// se_gbm_tiled.cu — LogLoss(K) GBM kernels for wide K: 2-D TMA tiles + four rows per thread.
//
// Reference arithmetic: boosting/GBMLoss.scala:196-263 (LogLoss), :50-74 (aggregator),
// classification/GBMClassifier.scala:337-375 (residuals), :437-449 (update).
//
// One CTA (2 warps) owns a tile of 256 rows x K classes of F (and h).  The tile is one box of a 2-D tensor map
// over the class-major [K][ld] array, so a whole stage arrives with ONE `cp.async.bulk.tensor.2d` per array
// (rows past n are zero-filled by the TMA unit), completion counted on an mbarrier.  A thread owns four
// consecutive rows and walks the classes with 128-bit shared-memory accesses:
//   A1  p = F + c_k h (written back into the F slot; F' stored to HBM when the mode updates F), running max / argmax
//   A2  e = 2^((p - m) log2 e) written back over p, srest = Σ_{k != argmax} e      (one MUFU per row and class)
//   B   row-wise outputs (residuals / newton weights) with 128-bit global stores, or — for the line-search
//       gradient Σ_i h_ik (softmax_ik - [y_i = k]) and newton's Σ_i hc_ik — a CLASS-wise sweep: warp w owns the
//       classes k ≡ w (mod 2), a lane sums eight rows of the tile per class and keeps one fp64 accumulator per
//       class in registers, so there are no per-tile shuffles and no per-row class registers.
// The one-hot term is folded in shared memory before pass B (e_y <- e_y - s, or -srest when y is the argmax, so that
// e_y / s = softmax_y - 1 keeps full relative precision on well-fitted rows).
// About 8 instructions per (row, class) instead of ~37 for the one-row-per-thread form which was
// issue-bound, far from the HBM roofline in eval mode.
#include "se_kernels.h"
#include "se_loss.cuh"
#include "se_tma.cuh"

namespace se {

namespace {

// W warps per CTA: 32 W threads, tiles of 128 W rows (<= 256: TMA box limit)

template <int MODE>
struct TiledTraits {
  static constexpr bool kReadH = (MODE == GBM_EVAL || MODE == GBM_UPDATE || MODE == GBM_UPDATE_RESID ||
                                  MODE == GBM_UPDATE_NEWTON);
  static constexpr bool kWriteF = (MODE == GBM_UPDATE || MODE == GBM_UPDATE_RESID || MODE == GBM_UPDATE_NEWTON);
  static constexpr bool kNewton = (MODE == GBM_RESID_NEWTON || MODE == GBM_UPDATE_NEWTON);
  static constexpr bool kWriteR = (MODE == GBM_RESID || MODE == GBM_UPDATE_RESID || kNewton);
  static constexpr bool kSumLoss = (MODE == GBM_EVAL || kWriteF || MODE == GBM_MEAN_LOSS);
  static constexpr bool kPerClassAcc = (MODE == GBM_EVAL || kNewton);
  static constexpr bool kKeepE = (MODE == GBM_EVAL || kWriteR);  // pass B needs the exponentials
  static constexpr bool kReduce = kSumLoss || kNewton;
};

// dynamic shared memory (128-byte aligned): [ {F,h} ][K][kTR] floats
template <int KMAX, int MODE, int W>
__global__ void __launch_bounds__(32 * W) gbm_logloss_tiled_kernel(const GbmArgs a,
                                                                const __grid_constant__ CUtensorMap mapF,
                                                                const __grid_constant__ CUtensorMap mapH) {
  using T = TiledTraits<MODE>;
  constexpr int kTT = 32 * W, kTR = 128 * W;
  extern __shared__ __align__(128) unsigned char smem_dyn[];
  // TMA tile destinations must be 128-byte aligned; the offset is applied to the shared array itself so that
  // the compiler keeps shared-memory addressing (LDS/STS) for everything derived from it
  float* stage = reinterpret_cast<float*>(smem_dyn + ((128u - (smem_u32(smem_dyn) & 127u)) & 127u));
  const int K = a.dim;
  constexpr int kArrays = T::kReadH ? 2 : 1;
  const int stage_floats = kArrays * K * kTR;
  __shared__ __align__(8) uint64_t bar;
  __shared__ float s_coef[kMaxDim];
  __shared__ __align__(16) float s_scale[T::kPerClassAcc ? kTR : 4];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int k = tid; k < K; k += kTT) s_coef[k] = a.coef[k];
  if (tid == 0) {
    mbar_init(&bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int64_t ntiles = (a.n + kTR - 1) / kTR;
  const int64_t ld = a.ld;
  const bool has_w = (a.w != nullptr);

  constexpr int NRED = T::kPerClassAcc ? KMAX + 1 : 1;
  constexpr int kAcc = T::kPerClassAcc ? KMAX / W : 1;
  double acc_loss = 0.0;
  double acc_c[kAcc];  // class k = warp + W*kk lives in acc_c[kk] of every lane of warp `warp`
#pragma unroll
  for (int kk = 0; kk < kAcc; ++kk) acc_c[kk] = 0.0;

  uint32_t it = 0;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
    // one elected thread loads the whole tile in <= 2 instructions; the other resident CTAs of the SM cover its latency
    if (tid == 0) {
      mbar_expect_tx(&bar, (uint32_t)(stage_floats * sizeof(float)));
      tma_load_tile(stage, &mapF, (int)(tile * kTR), &bar);
      if (T::kReadH) tma_load_tile(stage + K * kTR, &mapH, (int)(tile * kTR), &bar);
    }
    const int64_t row0 = tile * kTR + 4 * tid;
    const bool any_in = row0 < a.n;
    const bool all_in = row0 + 3 < a.n;
    // the slots are padded to 32 floats, so a 128-bit read at a 4-aligned row below n stays inside them
    const float4 y4 = any_in ? ld_stream4(a.y + row0) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 w4 = make_float4(1.f, 1.f, 1.f, 1.f), c4 = make_float4(1.f, 1.f, 1.f, 1.f);
    if (T::kNewton && has_w && any_in) w4 = ld_stream4(a.w + row0);
    if (T::kPerClassAcc && a.bag != nullptr && any_in) c4 = ld_stream4(a.bag + row0);  // bag multiplicities
    bool in[4];
    int yi[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      in[j] = row0 + j < a.n;
      yi[j] = in[j] ? min(max((int)f4at(y4, j), 0), K - 1) : 0;  // clamp = memory safety; validity is checked once per label upload
      if (!in[j]) f4at(c4, j) = 0.f;
    }
    mbar_wait(&bar, it & 1);
    float* sF = stage + 4 * tid;
    const float* sH = sF + K * kTR;

    // ---- A1: p = F + c_k h (GBMLoss.scala:56-59), running max and argmax (first maximum); p replaces F in shared memory
    float4 m4 = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    int am[4] = {0, 0, 0, 0};
#pragma unroll 2
    for (int k = 0; k < K; ++k) {
      float4 p = lds4(sF + k * kTR);
      if (T::kReadH) {
        const float4 hv = lds4(sH + k * kTR);
        const float c = s_coef[k];
        p.x = fmaf(c, hv.x, p.x), p.y = fmaf(c, hv.y, p.y), p.z = fmaf(c, hv.z, p.z), p.w = fmaf(c, hv.w, p.w);
        sts4(sF + k * kTR, p);
      }
      if (T::kWriteF) {
        float* g = a.F + k * ld + row0;
        if (all_in) {
          st_stream4(g, p);
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (in[j]) g[j] = f4at(p, j);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (f4at(p, j) > f4at(m4, j)) f4at(m4, j) = f4at(p, j), am[j] = k;
    }
    float py[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) py[j] = sF[yi[j] * kTR + j];

    // ---- A2: e = exp(p - m), srest = Σ_{k != argmax} e (the max term, exactly 1, is kept out of the sum so that a
    // well-fitted row keeps full relative precision in its loss and in 1 - softmax_argmax); e replaces p when pass B
    // needs it
    float4 r4 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 2
    for (int k = 0; k < K; ++k) {
      const float4 p = lds4(sF + k * kTR);
      float4 e;
      e.x = ex2_approx((p.x - m4.x) * kLog2e), e.y = ex2_approx((p.y - m4.y) * kLog2e);
      e.z = ex2_approx((p.z - m4.z) * kLog2e), e.w = ex2_approx((p.w - m4.w) * kLog2e);
      if (T::kKeepE) sts4(sF + k * kTR, e);
#pragma unroll
      for (int j = 0; j < 4; ++j) f4at(r4, j) += (k == am[j]) ? 0.f : f4at(e, j);
    }
    float inv_s[4];
    {
      float lsum = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float srest = f4at(r4, j);
        inv_s[j] = rcp_approx(1.0f + srest);
        // log Σ exp(p_k) - p_y = (m - p_y) + log1p(srest)                                 (GBMLoss.scala:206-221)
        const float l = (f4at(m4, j) - py[j]) + log1p_pos(srest);
        lsum += in[j] ? ((MODE == GBM_EVAL) ? f4at(c4, j) * l : l) : 0.f;
        // one-hot folded into the exponentials so that e_y / s = softmax_y - 1 (:223-238): -srest when y is the
        // argmax, e_y - s otherwise (|e_y - s| >= 1: no cancellation)
        if (T::kKeepE && !T::kNewton) {
          float& ey = sF[yi[j] * kTR + j];
          ey = (yi[j] == am[j]) ? -srest : ey - (1.0f + srest);
        }
      }
      if (T::kSumLoss) acc_loss += (double)lsum;
    }

    // ---- B: outputs
    if constexpr (MODE == GBM_EVAL) {
      // Σ_i c_i h_ik (softmax_ik - [y_i = k]) per class (:66-72): class-wise sweep over the whole tile
      sts4(s_scale + 4 * tid, make_float4(f4at(c4, 0) * inv_s[0], f4at(c4, 1) * inv_s[1], f4at(c4, 2) * inv_s[2],
                                          f4at(c4, 3) * inv_s[3]));
      __syncthreads();
      float4 sc[W];
#pragma unroll
      for (int q = 0; q < W; ++q) sc[q] = lds4(s_scale + 128 * q + 4 * lane);
      const float* tE = stage + 4 * lane;
      const float* tH = tE + K * kTR;
#pragma unroll
      for (int kk = 0; kk < kAcc; ++kk) {
        const int k = warp + W * kk;
        if (k < K) {
          float v = 0.f;
#pragma unroll
          for (int q = 0; q < W; ++q) {
            const float4 e = lds4(tE + k * kTR + 128 * q), hv = lds4(tH + k * kTR + 128 * q);
            v = fmaf(e.x * hv.x, sc[q].x, v), v = fmaf(e.y * hv.y, sc[q].y, v);
            v = fmaf(e.z * hv.z, sc[q].z, v), v = fmaf(e.w * hv.w, sc[q].w, v);
          }
          acc_c[kk] += (double)v;
        }
      }
    } else if constexpr (T::kNewton) {
      // R = -g/hc, WOUT = 1/2 hc w (x 1/S_k later), Σ_i c_i hc_ik       (:240-256, GBMClassifier.scala:342-364)
#pragma unroll 2
      for (int k = 0; k < K; ++k) {
        const float4 e = lds4(sF + k * kTR);
        float4 rr, ww, hh;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const bool top = (k == am[j]);
          const float sm = top ? inv_s[j] : f4at(e, j) * inv_s[j];
          const float om = f4at(r4, j) * inv_s[j];  // 1 - softmax of the argmax class
          const float gk = (k == yi[j]) ? (top ? -om : sm - 1.0f) : sm;
          const float hc = fmaxf(sm * (top ? om : 1.0f - sm), 1e-2f);
          f4at(rr, j) = -gk * rcp_approx(hc);
          f4at(ww, j) = 0.5f * hc * f4at(w4, j);
          f4at(hh, j) = f4at(c4, j) * hc;
        }
        sts4(sF + k * kTR, hh);
        float* gr = a.r + k * ld + row0;
        float* gw = a.wout + k * ld + row0;
        if (all_in) {
          st_stream4(gr, rr);
          st_stream4(gw, ww);
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (in[j]) gr[j] = f4at(rr, j), gw[j] = f4at(ww, j);
        }
      }
      __syncthreads();
      const float* tE = stage + 4 * lane;
#pragma unroll
      for (int kk = 0; kk < kAcc; ++kk) {
        const int k = warp + W * kk;
        if (k < K) {
          float v = 0.f;
#pragma unroll
          for (int q = 0; q < W; ++q) {
            const float4 e = lds4(tE + k * kTR + 128 * q);
            v += (e.x + e.y) + (e.z + e.w);
          }
          acc_c[kk] += (double)v;
        }
      }
    } else if constexpr (T::kWriteR) {
      // R = [y = k] - softmax_k                                                   (GBMClassifier.scala:371)
      const float4 ninv = make_float4(-inv_s[0], -inv_s[1], -inv_s[2], -inv_s[3]);
#pragma unroll 2
      for (int k = 0; k < K; ++k) {
        const float4 e = lds4(sF + k * kTR);
        const float4 rr = make_float4(e.x * ninv.x, e.y * ninv.y, e.z * ninv.z, e.w * ninv.w);
        float* gr = a.r + k * ld + row0;
        if (all_in) {
          st_stream4(gr, rr);
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (in[j]) gr[j] = f4at(rr, j);
        }
      }
    }
    fence_proxy_async_smem();
    __syncthreads();  // everyone is done with this stage before it is refilled
  }

  if (T::kReduce) {
    __shared__ double s_red[kTT / 32];
    __shared__ double s_tot[NRED];
    __shared__ bool is_last;
    {
      const double v = warp_sum(acc_loss);
      if (lane == 0) s_red[warp] = v;
    }
    if (T::kPerClassAcc) {
#pragma unroll
      for (int kk = 0; kk < kAcc; ++kk) {
        const double v = warp_sum(acc_c[kk]);  // 0 for k >= K
        if (lane == 0) a.ws.partials[(size_t)blockIdx.x * NRED + 1 + warp + W * kk] = v;
      }
    }
    __syncthreads();
    if (tid == 0) {
      double v = 0.0;
#pragma unroll
      for (int q = 0; q < W; ++q) v += s_red[q];
      a.ws.partials[(size_t)blockIdx.x * NRED] = v;
    }
    __threadfence();  // every writer publishes its partials before the ticket is taken
    __syncthreads();
    if (tid == 0) {
      __threadfence();
      const unsigned int ticket = atomicInc(a.ws.counter, gridDim.x - 1);
      is_last = (ticket == gridDim.x - 1);
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    // fixed-order cross-CTA reduction: warp w handles outputs w, w+W, ...; lanes stride over the CTAs
    for (int k = warp; k < NRED; k += kTT / 32) {
      double v = 0.0;
      for (unsigned int b = lane; b < gridDim.x; b += 32) v += __ldcg(&a.ws.partials[(size_t)b * NRED + k]);
      v = warp_sum(v);
      if (lane == 0) s_tot[k] = v;  // [0] = Σloss, [1 + k] per class (register-kernel convention)
    }
    __syncthreads();
    peer_exchange(s_tot, NRED, a.ws);
  }
}

template <int KMAX, int W>
cudaError_t launch_tiled_k(int mode, const GbmArgs& a, int sms, cudaStream_t st) {
  constexpr int kTT = 32 * W, kTR = 128 * W;
  const int K = a.dim;
  const bool read_h = (mode == GBM_EVAL || mode == GBM_UPDATE || mode == GBM_UPDATE_RESID || mode == GBM_UPDATE_NEWTON);
  if (a.n < 0 || a.n >= (int64_t)0x7fffff00) return cudaErrorInvalidValue;  // TMA coordinates are int32
  CUtensorMap mapF{}, mapH{};
  cudaError_t e = cudaSuccess;
  if (a.n > 0) {  // an empty shard launches one CTA with no tiles (it still publishes zero sums)
    e = make_tile_map(&mapF, a.F, a.n, a.ld, K, kTR);
    if (e != cudaSuccess) return e;
    e = make_tile_map(&mapH, read_h ? a.h : a.F, a.n, a.ld, K, kTR);
    if (e != cudaSuccess) return e;
  }
  const size_t stage_bytes = (size_t)(read_h ? 2 : 1) * K * kTR * sizeof(float);
  // one stage: with shared memory bounding occupancy, more resident CTAs beat double buffering at every K
  const size_t smem = stage_bytes + 128;
  int per_sm = (int)((228 * 1024) / (smem + 2560));  // + static shared memory and the 1 KB the system reserves per CTA
  if (per_sm < 1) return cudaErrorInvalidValue;
  if (per_sm > 16 / W) per_sm = 16 / W;  // at most 16 resident warps per SM
  int64_t need = (a.n + kTR - 1) / kTR;
  if (need < 1) need = 1;
  int64_t cap = (int64_t)per_sm * sms;
  if (cap > kMaxGridPartials) cap = kMaxGridPartials;
  const int grid = (int)(need < cap ? need : cap);
#define SE_CASE(M)                                                                                      \
  case M: {                                                                                             \
    auto kern = gbm_logloss_tiled_kernel<KMAX, M, W>;                                                     \
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);             \
    if (e != cudaSuccess) return e;                                                                     \
    kern<<<grid, kTT, smem, st>>>(a, mapF, mapH);                                                       \
    break;                                                                                              \
  }
  switch (mode) {
    SE_CASE(GBM_RESID)
    SE_CASE(GBM_RESID_NEWTON)
    SE_CASE(GBM_EVAL)
    SE_CASE(GBM_UPDATE)
    SE_CASE(GBM_UPDATE_RESID)
    SE_CASE(GBM_UPDATE_NEWTON)
    SE_CASE(GBM_MEAN_LOSS)
    default: return cudaErrorInvalidValue;
  }
#undef SE_CASE
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_gbm_logloss_tiled(int mode, const GbmArgs& a, int sms, cudaStream_t st) {
  const int K = a.dim;
  if (K < 1 || K > kMaxDim) return cudaErrorInvalidValue;
  // two warps per CTA (256-row tiles)
  if (K <= 8) return launch_tiled_k<8, 2>(mode, a, sms, st);
  if (K <= 16) return launch_tiled_k<16, 2>(mode, a, sms, st);
  if (K <= 32) return launch_tiled_k<32, 2>(mode, a, sms, st);
  // 33..64 classes: 128-row tiles (one warp) so that F and h of a tile still fit next to other CTAs' tiles; the warp
  // keeps all per-class fp64 sums (64 per lane) in registers
  return launch_tiled_k<64, 1>(mode, a, sms, st);
}

}  // namespace se
