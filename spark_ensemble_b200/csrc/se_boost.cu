// se_boost.cu — BoostingClassifier sample-weight update kernels (sm_90a).
//
// Reference: classification/BoostingClassifier.scala:168-187 (normalise), :198-230 (SAMME.R: error,
// weight update), :231-260 (SAMME), :269 (Σw').  The reference makes two (real) or three (discrete)
// passes over zipped RDDs per round; here SAMME.R is ONE pass (P[K][n] read once: 4K+8 B read, 4 B
// written per row) that also produces both scalars, and SAMME is the two passes its data dependence
// (β needs the error first) requires.  Weights are updated in place.
#include "se_kernels.h"
#include "se_loss.cuh"
#include "se_tma.cuh"

namespace se {

namespace {

constexpr float kSparkEps = 2.220446049250313e-16f;  // Spark ml.impl.Utils.EPSILON (2^-52)
constexpr int KU = 8;                                // classes loaded per batch (8 x 16 B in flight)

// Persistent grid: a multiple of the SM count, up to `ctas_per_sm` CTAs per SM, but never so many that a CTA
// gets fewer than ~8 work units (tiles): on large inputs later waves rebalance the tail, on small ones fewer,
// longer-lived CTAs amortise ramp-up and the per-CTA reduction epilogue.
inline int grid_for(int64_t work_items, int64_t per_cta, int ctas_per_sm, int sms) {
  int64_t units = (work_items + per_cta - 1) / per_cta;
  if (units < 1) units = 1;
  if (ctas_per_sm > 4) ctas_per_sm = 4;  // light grid-stride kernels (all CTAs resident)
  int64_t cap = (int64_t)ctas_per_sm * sms;
  if (cap > kMaxGridPartials) cap = (kMaxGridPartials / sms) * sms;
  int64_t want = (units / 8 / sms) * sms;  // >= 8 units per CTA, whole multiples of the SM count
  if (want < sms) want = sms;
  if (want > cap) want = cap;
  return (int)(units < want ? units : want);
}

// lg2 max(p, ε): the clamp is the exact constant lg2 2^-52 = -52, not an SFU approximation of it (NaN clamps too)
__device__ __forceinline__ float lg2_clamped(float p) { return (p > kSparkEps) ? lg2_approx(p) : -52.0f; }

// loss = Σ_k code_k log max(p_k, ε) with code_y = 1, code_{k≠y} = -1/(K-1)  (BoostingClassifier.scala:218-224)
//      = K/(K-1)·log p_y − (1/(K-1))·Σ_k log p_k,   so   −(K-1)/K·loss = ln 2·(Σ_k lg2 p_k / K − lg2 p_y)
// and w' = wₙ·2^x with x = Σ/K − lg2 p_y in [-52, 52] (:226).  Late in boosting most p_k clamp to ε, so Σ is ~K terms
// of -52: it is carried in fp64 (an fp32 sum loses ~1e-5 of the weight from K ~ 64), and x is split into an integer
// power of two (exact) and a fraction in [-0.5, 0.5] for the SFU.
struct RowState {
  float best, lg_y;
  double sum_lg;
  int am;
};

__device__ __forceinline__ void row_step(RowState& s, float p, int k, int yi) {
  if (p > s.best) {  // Vector.argmax: first maximum
    s.best = p;
    s.am = k;
  }
  const float lg = lg2_clamped(p);
  s.sum_lg += (double)lg;
  if (k == yi) s.lg_y = lg;
}

__device__ __forceinline__ float samme_r_weight(float wn, double sum_lg, float lg_y, double inv_k) {
  const double x = fma(sum_lg, inv_k, -(double)lg_y);
  const double xi = rint(x);
  return wn * ex2_approx((float)(x - xi)) * __int_as_float(((int)xi + 127) << 23);
}

__global__ void __launch_bounds__(kBlock) boost_real_kernel(const BoostArgs a) {
  const int K = a.K;
  const double inv_k = 1.0 / (double)K;
  double acc[2] = {0.0, 0.0};
  const int64_t n4 = a.n >> 2;
  for (int64_t g = (int64_t)blockIdx.x * kBlock + threadIdx.x; g < n4;
       g += (int64_t)gridDim.x * kBlock) {
    const float4 vy = ld_stream4(a.y + 4 * g);
    const float4 vw = ld_rw4(a.w + 4 * g);
    RowState st[4];
    int yi[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      st[e].best = -INFINITY; st[e].sum_lg = 0.0; st[e].lg_y = 0.f; st[e].am = 0;
      yi[e] = (int)f4at(vy, e);  // compared only (validity is checked once per label upload)
    }
    for (int k0 = 0; k0 < K; k0 += KU) {
      float4 vp[KU];
#pragma unroll
      for (int u = 0; u < KU; ++u)
        if (k0 + u < K) vp[u] = ld_stream4(a.proba + (int64_t)(k0 + u) * a.ld + 4 * g);
#pragma unroll
      for (int u = 0; u < KU; ++u)
        if (k0 + u < K) {
#pragma unroll
          for (int e = 0; e < 4; ++e) row_step(st[e], f4at(vp[u], e), k0 + u, yi[e]);
        }
    }
    float4 out;
    float err4 = 0.f, sum4 = 0.f;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float wn = f4at(vw, e) * a.inv_sum_w;  // :186
      err4 += (st[e].am != yi[e]) ? wn : 0.f;       // :202-209
      const float wo = samme_r_weight(wn, st[e].sum_lg, st[e].lg_y, inv_k);  // :218-226
      f4at(out, e) = wo;
      sum4 += wo;
    }
    st_stream4(a.w + 4 * g, out);
    acc[0] += (double)err4;
    acc[1] += (double)sum4;
  }
  if (blockIdx.x == 0 && threadIdx.x < (a.n & 3)) {
    const int64_t i = (n4 << 2) + threadIdx.x;
    RowState st{-INFINITY, 0.f, 0.0, 0};
    const int yi = (int)a.y[i];
    for (int k = 0; k < K; ++k) row_step(st, a.proba[(int64_t)k * a.ld + i], k, yi);
    const float wn = a.w[i] * a.inv_sum_w;
    const float wo = samme_r_weight(wn, st.sum_lg, st.lg_y, inv_k);
    a.w[i] = wo;
    acc[0] += (st.am != yi) ? (double)wn : 0.0;
    acc[1] += (double)wo;
  }
  block_reduce_publish<2>(acc, a.ws);
}

// SAMME.R through TMA tiles (K >= 5): the register-streaming kernel above keeps 8 x 16 B of P per thread in
// registers (99 registers, 2 CTAs/SM, ~64 KB of loads in flight per SM; long-scoreboard bound below the
// HBM roofline at large K).  Here a 2-warp CTA owns a 256-row x K tile of P that arrives as one 2-D tensor-map box
// (`cp.async.bulk.tensor.2d`, rows past n zero-filled), up to 8 CTAs per SM keep ~200 KB in flight, and a thread
// walks the classes of its four rows with 128-bit shared-memory reads: first-maximum argmax, Σ_k lg2 max(p, ε);
// log p_y is picked from the tile afterwards.  Same arithmetic as boost_real_kernel (BoostingClassifier.scala:198-230).
constexpr int kRT = 64;        // threads per CTA
constexpr int kRR = 4 * kRT;   // rows per tile
constexpr int kSammeTiledMinK = 5;  // SAMME.R: K <= 4 streams through registers (boost_real_kernel), wider K in tiles

__global__ void __launch_bounds__(kRT) boost_real_tiled_kernel(const BoostArgs a, const __grid_constant__ CUtensorMap mapP) {
  extern __shared__ __align__(128) unsigned char smem_dyn[];
  float* tileP = reinterpret_cast<float*>(smem_dyn + ((128u - (smem_u32(smem_dyn) & 127u)) & 127u));
  __shared__ __align__(8) uint64_t bar;
  const int K = a.K;
  const int tid = threadIdx.x;
  if (tid == 0) {
    mbar_init(&bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const double inv_k = 1.0 / (double)K;
  const int64_t ntiles = (a.n + kRR - 1) / kRR;
  double acc[2] = {0.0, 0.0};
  uint32_t it = 0;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
    if (tid == 0) {  // the other resident CTAs of the SM cover this tile's load latency
      mbar_expect_tx(&bar, (uint32_t)(K * kRR * sizeof(float)));
      tma_load_tile(tileP, &mapP, (int)(tile * kRR), &bar);
    }
    const int64_t row0 = tile * kRR + 4 * tid;
    const bool any_in = row0 < a.n, all_in = row0 + 3 < a.n;
    // slots are padded to 32 floats: 128-bit accesses at a 4-aligned row below n stay inside them
    const float4 vy = any_in ? ld_stream4(a.y + row0) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 vw = any_in ? ld_rw4(a.w + row0) : make_float4(0.f, 0.f, 0.f, 0.f);
    int yi[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) yi[e] = min(max((int)f4at(vy, e), 0), K - 1);  // clamp = memory safety; validity checked once per upload
    mbar_wait(&bar, it & 1);
    const float* sP = tileP + 4 * tid;
    float best[4];
    double sum_lg[4];
    int am[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) best[e] = -INFINITY, sum_lg[e] = 0.0, am[e] = 0;
#pragma unroll 2
    for (int k = 0; k < K; ++k) {
      const float4 p = *reinterpret_cast<const float4*>(sP + k * kRR);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pe = f4at(p, e);
        if (pe > best[e]) best[e] = pe, am[e] = k;  // Vector.argmax: first maximum
        sum_lg[e] += (double)lg2_clamped(pe);
      }
    }
    float4 out;
    float err4 = 0.f, sum4 = 0.f;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const bool in = row0 + e < a.n;
      const float lg_y = lg2_clamped(sP[yi[e] * kRR + e]);  // yi is clamped into [0, K)
      const float wn = f4at(vw, e) * a.inv_sum_w;          // :186
      const float wo = samme_r_weight(wn, sum_lg[e], lg_y, inv_k);  // :218-226
      f4at(out, e) = wo;
      err4 += (in && am[e] != yi[e]) ? wn : 0.f;                                   // :202-209
      sum4 += in ? wo : 0.f;
    }
    if (all_in) {
      st_stream4(a.w + row0, out);
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (row0 + e < a.n) a.w[row0 + e] = f4at(out, e);
    }
    acc[0] += (double)err4;
    acc[1] += (double)sum4;
    __syncthreads();  // everyone is done with the tile before it is refilled
  }
  block_reduce_publish<2, kRT>(acc, a.ws);
}

// SAMME: est_err = Σ wₙ·1[pred ≠ y]  (:232-242)
__global__ void __launch_bounds__(kBlock) boost_discrete_error_kernel(const BoostArgs a) {
  double acc[1] = {0.0};
  const int64_t n4 = a.n >> 2;
  constexpr int U = 4;  // 12 independent 16 B loads per thread in flight, contiguous tiles like the GBM kernels
  constexpr int64_t tile = (int64_t)kBlock * U;
  const int64_t ntiles = (n4 + tile - 1) / tile;
  for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int64_t base = t * tile + threadIdx.x;
    float4 vy[U], vp[U], vw[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t g = base + (int64_t)u * kBlock;
      if (g < n4) {
        vy[u] = ld_stream4(a.y + 4 * g);
        vp[u] = ld_stream4(a.pred + 4 * g);
        vw[u] = ld_stream4(a.w + 4 * g);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (base + (int64_t)u * kBlock < n4) {
        float e4 = 0.f;
#pragma unroll
        for (int e = 0; e < 4; ++e)
          e4 += (f4at(vy[u], e) != f4at(vp[u], e)) ? f4at(vw[u], e) * a.inv_sum_w : 0.f;
        acc[0] += (double)e4;
      }
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < (a.n & 3)) {
    const int64_t i = (n4 << 2) + threadIdx.x;
    if (a.y[i] != a.pred[i]) acc[0] += (double)(a.w[i] * a.inv_sum_w);
  }
  block_reduce_publish<1>(acc, a.ws);
}

// SAMME: w' = wₙ·(1/β)^err  (:254-258), Σw' (:269)
__global__ void __launch_bounds__(kBlock) boost_discrete_update_kernel(const BoostArgs a) {
  double acc[1] = {0.0};
  const int64_t n4 = a.n >> 2;
  for (int64_t g = (int64_t)blockIdx.x * kBlock + threadIdx.x; g < n4;
       g += (int64_t)gridDim.x * kBlock) {
    const float4 vy = ld_stream4(a.y + 4 * g), vp = ld_stream4(a.pred + 4 * g);
    const float4 vw = ld_rw4(a.w + 4 * g);
    float4 out;
    float s4 = 0.f;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float wn = f4at(vw, e) * a.inv_sum_w;
      // pow(1/β, 0) == 1 even for 1/β == Inf; wn·Inf for a mis-classified row is the reference's result too
      const float wo = (f4at(vy, e) != f4at(vp, e)) ? wn * a.inv_beta : wn;
      f4at(out, e) = wo;
      s4 += wo;
    }
    st_stream4(a.w + 4 * g, out);
    acc[0] += (double)s4;
  }
  if (blockIdx.x == 0 && threadIdx.x < (a.n & 3)) {
    const int64_t i = (n4 << 2) + threadIdx.x;
    const float wn = a.w[i] * a.inv_sum_w;
    const float wo = (a.y[i] != a.pred[i]) ? wn * a.inv_beta : wn;
    a.w[i] = wo;
    acc[0] += (double)wo;
  }
  block_reduce_publish<1>(acc, a.ws);
}

__global__ void __launch_bounds__(kBlock) sum_kernel(const float* x, int64_t n, const RedWs ws) {
  double acc[1] = {0.0};
  const int64_t n4 = n >> 2;
  for (int64_t g = (int64_t)blockIdx.x * kBlock + threadIdx.x; g < n4;
       g += (int64_t)gridDim.x * kBlock) {
    const float4 v = ld_stream4(x + 4 * g);
    acc[0] += (double)v.x + (double)v.y + (double)v.z + (double)v.w;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) acc[0] += (double)x[(n4 << 2) + threadIdx.x];
  block_reduce_publish<1>(acc, ws);
}

__global__ void __launch_bounds__(kBlock) dot_kernel(const float* a, const float* b, int64_t n, const RedWs ws) {
  double acc[1] = {0.0};
  const int64_t n4 = n >> 2;
  for (int64_t g = (int64_t)blockIdx.x * kBlock + threadIdx.x; g < n4; g += (int64_t)gridDim.x * kBlock) {
    const float4 va = ld_stream4(a + 4 * g);
    if (b) {
      const float4 vb = ld_stream4(b + 4 * g);
      acc[0] += (double)va.x * vb.x + (double)va.y * vb.y + (double)va.z * vb.z + (double)va.w * vb.w;
    } else {
      acc[0] += (double)va.x + (double)va.y + (double)va.z + (double)va.w;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const int64_t i = (n4 << 2) + threadIdx.x;
    acc[0] += b ? (double)a[i] * b[i] : (double)a[i];
  }
  block_reduce_publish<1>(acc, ws);
}

// ---- AdaBoost.R2 -----------------------------------------------------------------------------------
// loss(e) for e = |y - pred| / maxError in [0,1] (regression/BoostingRegressor.scala:97-106)
__device__ __forceinline__ float r2_loss(int loss_type, float e) {
  if (loss_type == 1) return e;
  if (loss_type == 2) return e * e;
  // 1 - exp(-e): series below 0.25 (no cancellation), SFU form above
  const float ser = e * fmaf(e, fmaf(e, fmaf(e, fmaf(e, fmaf(e, -1.0f / 720.0f, 1.0f / 120.0f), -1.0f / 24.0f),
                                              1.0f / 6.0f), -0.5f), 1.0f);
  return (e < 0.25f) ? ser : 1.0f - exp_neg_fast(-e);
}

__global__ void __launch_bounds__(kBlock) boostreg_max_kernel(const BoostRegArgs a) {
  float m = -INFINITY;
  const int64_t n4 = a.n >> 2;
  for (int64_t g = (int64_t)blockIdx.x * kBlock + threadIdx.x; g < n4; g += (int64_t)gridDim.x * kBlock) {
    const float4 vy = ld_stream4(a.y + 4 * g), vp = ld_stream4(a.pred + 4 * g);
#pragma unroll
    for (int e = 0; e < 4; ++e) m = fmaxf(m, fabsf(f4at(vy, e) - f4at(vp, e)));  // :169,231-234
  }
  if (blockIdx.x == 0 && threadIdx.x < (a.n & 3)) {
    const int64_t i = (n4 << 2) + threadIdx.x;
    m = fmaxf(m, fabsf(a.y[i] - a.pred[i]));
  }
  block_max_publish((double)m, a.ws.partials, a.ws.counter, a.ws.out);
}

template <bool UPDATE>
__global__ void __launch_bounds__(kBlock) boostreg_pass_kernel(const BoostRegArgs a) {
  double acc[1] = {0.0};
  const int64_t n4 = a.n >> 2;
  auto one = [&](float y, float p, float w, float& wo) -> float {
    const float l = r2_loss(a.loss_type, fabsf(y - p) * a.inv_max_err);  // :236-242
    const float wn = w * a.inv_sum_w;
    if (!UPDATE) return wn * l;                                            // :244-249
    wo = wn * ex2_approx((1.0f - l) * a.log2_beta);                        // wₙ·β^(1-loss) :256-260
    return wo;
  };
  for (int64_t g = (int64_t)blockIdx.x * kBlock + threadIdx.x; g < n4; g += (int64_t)gridDim.x * kBlock) {
    const float4 vy = ld_stream4(a.y + 4 * g), vp = ld_stream4(a.pred + 4 * g);
    const float4 vw = UPDATE ? ld_rw4(a.w + 4 * g) : ld_stream4(a.w + 4 * g);
    float4 out;
    float s4 = 0.f;
#pragma unroll
    for (int e = 0; e < 4; ++e) s4 += one(f4at(vy, e), f4at(vp, e), f4at(vw, e), f4at(out, e));
    if (UPDATE) st_stream4(a.w + 4 * g, out);
    acc[0] += (double)s4;
  }
  if (blockIdx.x == 0 && threadIdx.x < (a.n & 3)) {
    const int64_t i = (n4 << 2) + threadIdx.x;
    float wo = 0.f;
    acc[0] += (double)one(a.y[i], a.pred[i], a.w[i], wo);
    if (UPDATE) a.w[i] = wo;
  }
  block_reduce_publish<1>(acc, a.ws);
}

}  // namespace

cudaError_t launch_boostreg_max(const BoostRegArgs& a, int ctas_per_sm, int sms, cudaStream_t s) {
  boostreg_max_kernel<<<grid_for(a.n >> 2, kBlock, ctas_per_sm, sms), kBlock, 0, s>>>(a);
  return cudaGetLastError();
}
cudaError_t launch_boostreg_error(const BoostRegArgs& a, int ctas_per_sm, int sms, cudaStream_t s) {
  boostreg_pass_kernel<false><<<grid_for(a.n >> 2, kBlock, ctas_per_sm, sms), kBlock, 0, s>>>(a);
  return cudaGetLastError();
}
cudaError_t launch_boostreg_update(const BoostRegArgs& a, int ctas_per_sm, int sms, cudaStream_t s) {
  boostreg_pass_kernel<true><<<grid_for(a.n >> 2, kBlock, ctas_per_sm, sms), kBlock, 0, s>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_boost_real(const BoostArgs& a, int ctas_per_sm, int sms, cudaStream_t s) {
  const size_t tile_bytes = (size_t)a.K * kRR * sizeof(float);
  if (a.K >= kSammeTiledMinK && a.n > 0 && a.n < (int64_t)0x7fffff00 && tile_bytes <= 200 * 1024) {
    CUtensorMap mapP;
    cudaError_t e = make_tile_map(&mapP, a.proba, a.n, a.ld, a.K, kRR);
    if (e != cudaSuccess) return e;
    const size_t smem = tile_bytes + 128;
    int per_sm = (int)((228 * 1024) / (smem + 1536));  // + static shared memory and the 1 KB the system reserves
    if (per_sm > 8) per_sm = 8;
    const int64_t ntiles = (a.n + kRR - 1) / kRR;
    int64_t cap = (int64_t)per_sm * sms;
    if (cap > kMaxGridPartials) cap = kMaxGridPartials;
    const int grid = (int)(ntiles < cap ? ntiles : cap);
    e = cudaFuncSetAttribute(boost_real_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    boost_real_tiled_kernel<<<grid, kRT, smem, s>>>(a, mapP);
    return cudaGetLastError();
  }
  boost_real_kernel<<<grid_for(a.n >> 2, kBlock, ctas_per_sm, sms), kBlock, 0, s>>>(a);
  return cudaGetLastError();
}
cudaError_t launch_boost_discrete_error(const BoostArgs& a, int ctas_per_sm, int sms, cudaStream_t s) {
  boost_discrete_error_kernel<<<grid_for(a.n >> 2, kBlock, ctas_per_sm, sms), kBlock, 0, s>>>(a);
  return cudaGetLastError();
}
cudaError_t launch_boost_discrete_update(const BoostArgs& a, int ctas_per_sm, int sms, cudaStream_t s) {
  boost_discrete_update_kernel<<<grid_for(a.n >> 2, kBlock, ctas_per_sm, sms), kBlock, 0, s>>>(a);
  return cudaGetLastError();
}
cudaError_t launch_dot(const float* a, const float* b, int64_t n, const RedWs& ws, int ctas_per_sm, int sms,
                       cudaStream_t s) {
  dot_kernel<<<grid_for(n >> 2, kBlock, ctas_per_sm, sms), kBlock, 0, s>>>(a, b, n, ws);
  return cudaGetLastError();
}
cudaError_t launch_sum(const float* x, int64_t n, const RedWs& ws, int ctas_per_sm, int sms,
                       cudaStream_t s) {
  sum_kernel<<<grid_for(n >> 2, kBlock, ctas_per_sm, sms), kBlock, 0, s>>>(x, n, ws);
  return cudaGetLastError();
}

}  // namespace se
