// se_gbm.cu — GBM inner-loop kernels (sm_90a): pseudo-residuals, line-search evaluation,
// fused prediction update + next-round residual + loss, validation loss.
//
// Reference (fp64, Spark RDD closures): regression/GBMRegressor.scala:368-385 (residuals),
// :398-425 + boosting/GBMLoss.scala:50-74 (line search objective), :434-442 (F update),
// :444-456 (validation); classification/GBMClassifier.scala:337-375, :413-431, :437-449, :451-470.
//
// Design: every kernel is one streaming pass over column-major fp32 rows.  A CTA owns contiguous
// tiles of kBlock*U float4 groups; each thread issues all of its 128-bit loads for a tile before
// computing (U x 3 independent 16 B requests in flight per thread), evaluates the loss in fp32,
// accumulates sums in fp64, and the grid finishes with the deterministic last-CTA reduction from
// se_common.cuh.  HBM-bound: K1 (update+residual+loss) moves 20 B/row, K2 (eval) 12 B/row.
#include "se_kernels.h"
#include "se_loss.cuh"

namespace se {

namespace {

constexpr int U_SCALAR = 4;  // float4 groups per thread per tile (cheap losses: pure streaming)
constexpr int kLoglossTiledMinK = 5;  // LogLoss: K <= 4 classes per row in registers, wider K in TMA tiles

// Transcendental-heavy losses spend ~30 instructions per row: with U = 4 (76-80 registers, 3 CTAs/SM) the
// warps of an SM bunch up in the same load-then-compute phase (few eligible warps per cycle, low issue
// utilisation and DRAM throughput).  They use U = 2 and a 4-CTA/SM register budget (64 regs, no spills) instead: 32 warps per SM in
// different phases overlap one warp's math with another's loads.
template <int LOSS>
struct LossTune {
  static constexpr bool kHeavy = (LOSS == SE_LOSS_BERNOULLI || LOSS == SE_LOSS_EXPONENTIAL ||
                                  LOSS == SE_LOSS_LOGCOSH || LOSS == SE_LOSS_SCALED_LOGCOSH);
  static constexpr int kU = kHeavy ? 2 : U_SCALAR;
  static constexpr int kMinCtas = kHeavy ? 4 : 1;
};

template <int MODE>
struct ModeTraits {
  static constexpr bool kReadH = (MODE == GBM_EVAL || MODE == GBM_EVAL_LOSS || MODE == GBM_UPDATE ||
                                  MODE == GBM_UPDATE_RESID || MODE == GBM_UPDATE_NEWTON);
  static constexpr bool kWriteF = (MODE == GBM_UPDATE || MODE == GBM_UPDATE_RESID ||
                                   MODE == GBM_UPDATE_NEWTON);
  static constexpr bool kNewton = (MODE == GBM_RESID_NEWTON || MODE == GBM_UPDATE_NEWTON);
  static constexpr bool kWriteR = (MODE == GBM_RESID || MODE == GBM_UPDATE_RESID || kNewton);
  static constexpr bool kSumLoss = (MODE == GBM_EVAL || MODE == GBM_EVAL_LOSS || kWriteF || MODE == GBM_MEAN_LOSS);
  static constexpr bool kReduce = kSumLoss || kNewton;
};

__device__ __forceinline__ float device_step(const GbmArgs& a) {
  // squared loss closed form: alpha* = clip(Σh(y-F)/Σh², 0, 100) (Brent's interval, GBMRegressor.scala:412)
  const double s1 = a.dev_stats[1], s2 = a.dev_stats[2];
  double al = (s2 > 0.0) ? s1 / s2 : 1.0;
  al = fmin(fmax(al, 0.0), 100.0);
  return a.lr * (float)al;
}

// ------------------------------------------------------------------ scalar losses, dim == 1
// POL: accesses carry an explicit L2 eviction policy (se_common.cuh): always for the modes that write per-row
// results, for the read-only modes only on L2-sized shards (a.l2_hints)
template <int LOSS, int MODE, bool POL>
__global__ void __launch_bounds__(kBlock, LossTune<LOSS>::kMinCtas) gbm_scalar_kernel(const GbmArgs a) {
  using T = ModeTraits<MODE>;
  constexpr int U = LossTune<LOSS>::kU;
  float coef = a.coef[0];
  if (T::kWriteF && a.dev_stats != nullptr) coef = device_step(a);
  const float param = a.param;
  const bool has_w = (a.w != nullptr);
  // bag multiplicities (row sub-sampling, GBMRegressor.scala:357-359): the line search and newton's Σh run on
  // the bag (reference quirk 4), i.e. every per-row term of those sums is multiplied by the row's count
  constexpr bool kBagMode = (MODE == GBM_EVAL) || (MODE == GBM_EVAL_LOSS) || T::kNewton;
  const bool has_bag = kBagMode && (a.bag != nullptr);
  // [0] Σloss, [1] Σ h·g (eval) or Σ max(H,1e-2) (newton), [2] Σ h²·H (eval: curvature of the line-search objective)
  double acc[3] = {0.0, 0.0, 0.0};

  const int64_t n4 = a.n >> 2;
  constexpr int64_t tile = (int64_t)kBlock * U;
  const int64_t ntiles = (n4 + tile - 1) / tile;
  const uint64_t pol_keep = l2_policy(false), pol_stream = l2_policy(a.l2_hints != 0);

  auto row = [&](float y, float F, float h, float w, float c, float& Fo, float& ro, float& wo, float& l_acc,
                 float& x_acc, float& z_acc) {
    const float p = T::kReadH ? fmaf(coef, h, F) : F;
    const LGH o = eval_loss<LOSS>(y, p, param);
    if (T::kWriteF) Fo = p;
    if (T::kSumLoss) l_acc += (MODE == GBM_EVAL || MODE == GBM_EVAL_LOSS) ? c * o.l : o.l;
    if (MODE == GBM_EVAL) {
      x_acc = fmaf(c * h, o.g, x_acc);
      z_acc = fmaf(c * h * h, o.h, z_acc);
    }
    if (T::kNewton) {
      const float hc = fmaxf(o.h, 1e-2f);   // GBMRegressor.scala:371
      ro = -o.g * rcp_approx(hc);                      // :377
      wo = 0.5f * hc * w;                   // :379 (x 1/S applied when the weights leave the device: se_download)
      x_acc = fmaf(c, hc, x_acc);
    } else if (T::kWriteR) {
      ro = -o.g;                            // :383
    }
  };

  // tiles are interleaved across CTAs: at any moment the grid works inside one compact moving window of
  // each array (one contiguous region per CTA instead keeps thousands of distinct 2 MB pages live at once)
  for (int64_t t0 = blockIdx.x; t0 < ntiles; t0 += gridDim.x) {
    const int64_t t = a.reverse ? (ntiles - 1 - t0) : t0;
    const int64_t base = t * tile + threadIdx.x;
    float4 vy[U], vF[U], vh[U], vw[U], vb[U];
    bool ok[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t g = base + (int64_t)u * kBlock;
      ok[u] = g < n4;
      if (ok[u]) {
        vy[u] = a.y ? ld_s4<POL>(a.y + 4 * g, pol_stream) : make_float4(1.f, 1.f, 1.f, 1.f);  // y == nullptr: signed view, label 1
        vF[u] = T::kWriteF ? ld_r4<POL>(a.F + 4 * g, pol_stream) : ld_s4<POL>(a.F + 4 * g, pol_stream);
        if (T::kReadH) vh[u] = ld_s4<POL>(a.h + 4 * g, T::kWriteF ? pol_stream : pol_keep);  // an update is h's last reader
        if (T::kNewton && has_w) vw[u] = ld_stream4(a.w + 4 * g);
        if (has_bag) vb[u] = ld_stream4(a.bag + 4 * g);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (!ok[u]) continue;
      const int64_t g = base + (int64_t)u * kBlock;
      float4 oF, oR, oW;
      float l_acc = 0.f, x_acc = 0.f, z_acc = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float w = (T::kNewton && has_w) ? f4at(vw[u], e) : 1.0f;
        const float c = has_bag ? f4at(vb[u], e) : 1.0f;
        row(f4at(vy[u], e), f4at(vF[u], e), T::kReadH ? f4at(vh[u], e) : 0.f, w, c, f4at(oF, e),
            f4at(oR, e), f4at(oW, e), l_acc, x_acc, z_acc);
      }
      if (T::kWriteF) st_s4<POL>(a.F + 4 * g, oF, pol_stream);
      if (T::kWriteR) st_s4<POL>(a.r + 4 * g, oR, pol_keep);  // the next statistics pass starts where this one ends
      if (T::kNewton) st_stream4(a.wout + 4 * g, oW);
      if (T::kSumLoss) acc[0] += (double)l_acc;
      if (MODE == GBM_EVAL || T::kNewton) acc[1] += (double)x_acc;
      if (MODE == GBM_EVAL) acc[2] += (double)z_acc;
    }
  }
  // scalar tail (n % 4 rows)
  if (blockIdx.x == 0 && threadIdx.x < (a.n & 3)) {
    const int64_t i = (n4 << 2) + threadIdx.x;
    const float w = (T::kNewton && has_w) ? a.w[i] : 1.0f;
    const float c = has_bag ? a.bag[i] : 1.0f;
    float Fo = 0.f, ro = 0.f, wo = 0.f, l_acc = 0.f, x_acc = 0.f, z_acc = 0.f;
    row(a.y ? a.y[i] : 1.0f, a.F[i], T::kReadH ? a.h[i] : 0.f, w, c, Fo, ro, wo, l_acc, x_acc, z_acc);
    if (T::kWriteF) a.F[i] = Fo;
    if (T::kWriteR) a.r[i] = ro;
    if (T::kNewton) a.wout[i] = wo;
    if (T::kSumLoss) acc[0] += (double)l_acc;
    if (MODE == GBM_EVAL || T::kNewton) acc[1] += (double)x_acc;
    if (MODE == GBM_EVAL) acc[2] += (double)z_acc;
  }
  if (T::kReduce) block_reduce_publish<3>(acc, a.ws);
}

// squared loss: the three sufficient statistics of the line-search parabola, one pass (12 B/row)
// FROM_R: the residual slot already holds r = y - F for the current F (squared loss: r = -g, written by the
// previous fused update or by se_gbm_pseudo_residuals), so the statistics Σr², Σh·r, Σh² need r and h only:
// 8 B/row instead of 12.  Bit-identical: r was computed as the same fp32 difference y - F.
template <bool FROM_R, bool POL>
__global__ void __launch_bounds__(kBlock) gbm_sq_stats_kernel(const GbmArgs a) {
  constexpr int U = U_SCALAR;
  const bool has_bag = (a.bag != nullptr);
  const uint64_t pol_keep = l2_policy(false), pol_stream = l2_policy(a.l2_hints != 0);
  double acc[3] = {0.0, 0.0, 0.0};
  const int64_t n4 = a.n >> 2;
  constexpr int64_t tile = (int64_t)kBlock * U;
  const int64_t ntiles = (n4 + tile - 1) / tile;
  for (int64_t t0 = blockIdx.x; t0 < ntiles; t0 += gridDim.x) {
    const int64_t t = a.reverse ? (ntiles - 1 - t0) : t0;
    const int64_t base = t * tile + threadIdx.x;
    float4 vy[U], vF[U], vh[U], vb[U];
    bool ok[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t g = base + (int64_t)u * kBlock;
      ok[u] = g < n4;
      if (ok[u]) {
        if (FROM_R) {
          vy[u] = ld_s4<POL>(a.r + 4 * g, pol_stream);  // the update that follows rewrites r without reading it
        } else {
          vy[u] = ld_s4<POL>(a.y + 4 * g, pol_keep);
          vF[u] = ld_s4<POL>(a.F + 4 * g, pol_keep);
        }
        vh[u] = ld_s4<POL>(a.h + 4 * g, pol_keep);      // re-read by the update, from this pass's tail
        if (has_bag) vb[u] = ld_stream4(a.bag + 4 * g);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (!ok[u]) continue;
      float s0 = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float d = FROM_R ? f4at(vy[u], e) : f4at(vy[u], e) - f4at(vF[u], e), h = f4at(vh[u], e);
        const float c = has_bag ? f4at(vb[u], e) : 1.0f;
        s0 = fmaf(c * d, d, s0);
        s1 = fmaf(c * h, d, s1);
        s2 = fmaf(c * h, h, s2);
      }
      acc[0] += (double)s0;
      acc[1] += (double)s1;
      acc[2] += (double)s2;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < (a.n & 3)) {
    const int64_t i = (n4 << 2) + threadIdx.x;
    const float d = FROM_R ? a.r[i] : a.y[i] - a.F[i], h = a.h[i];
    const float c = has_bag ? a.bag[i] : 1.0f;
    acc[0] += (double)(c * d * d);
    acc[1] += (double)(c * h * d);
    acc[2] += (double)(c * h * h);
  }
  block_reduce_publish<3>(acc, a.ws);
}

// ------------------------------------------------------------------ LogLoss(K), dim == K
// boosting/GBMLoss.scala:196-263.  The reference's log Σ exp(p_k) has no max shift (overflows above
// ~709 in fp64); here the shifted form is used — identical wherever the reference is finite.
// Layout [K][ld]; a thread owns VEC consecutive rows and keeps all K classes in registers.
template <int KMAX, int MODE, int VEC>
__global__ void __launch_bounds__(kBlock) gbm_logloss_kernel(const GbmArgs a) {
  using T = ModeTraits<MODE>;
  const int K = a.dim;
  const int64_t ld = a.ld;
  const bool has_w = (a.w != nullptr);
  constexpr int NRED = KMAX + 1;
  double acc[NRED];
#pragma unroll
  for (int k = 0; k < NRED; ++k) acc[k] = 0.0;

  const int64_t ngroups = (a.n + VEC - 1) / VEC;
  for (int64_t g = (int64_t)blockIdx.x * kBlock + threadIdx.x; g < ngroups;
       g += (int64_t)gridDim.x * kBlock) {
    const int64_t i0 = g * VEC;
    const bool full = (i0 + VEC <= a.n);
    float p[KMAX][VEC], hh[KMAX][VEC], yv[VEC], wv[VEC], cv[VEC];
    constexpr bool kBagMode = (MODE == GBM_EVAL) || T::kNewton;
    const bool has_bag = kBagMode && (a.bag != nullptr);
#pragma unroll
    for (int e = 0; e < VEC; ++e) cv[e] = 1.0f;
    if (has_bag) {
#pragma unroll
      for (int e = 0; e < VEC; ++e) cv[e] = (i0 + e < a.n) ? a.bag[i0 + e] : 0.f;
    }
    // ---- loads
    if (VEC == 4 && full) {
      const float4 t = ld_stream4(a.y + i0);
#pragma unroll
      for (int e = 0; e < VEC; ++e) yv[e] = f4at(t, e);
      if (T::kNewton && has_w) {
        const float4 tw = ld_stream4(a.w + i0);
#pragma unroll
        for (int e = 0; e < VEC; ++e) wv[e] = f4at(tw, e);
      }
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
          const float4 tf = T::kWriteF ? ld_rw4(a.F + k * ld + i0) : ld_stream4(a.F + k * ld + i0);
#pragma unroll
          for (int e = 0; e < VEC; ++e) p[k][e] = f4at(tf, e);
          if (T::kReadH) {
            const float4 th = ld_stream4(a.h + k * ld + i0);
#pragma unroll
            for (int e = 0; e < VEC; ++e) hh[k][e] = f4at(th, e);
          }
        }
      }
    } else {
#pragma unroll
      for (int e = 0; e < VEC; ++e) {
        const bool in = (i0 + e < a.n);
        yv[e] = in ? a.y[i0 + e] : 0.f;
        if (T::kNewton && has_w) wv[e] = in ? a.w[i0 + e] : 0.f;
#pragma unroll
        for (int k = 0; k < KMAX; ++k) {
          if (k < K) {
            p[k][e] = in ? a.F[k * ld + i0 + e] : 0.f;
            if (T::kReadH) hh[k][e] = in ? a.h[k * ld + i0 + e] : 0.f;
          }
        }
      }
    }
    if (!(T::kNewton && has_w)) {
#pragma unroll
      for (int e = 0; e < VEC; ++e) wv[e] = 1.0f;
    }
    // ---- per-row math
    float outR[KMAX][VEC], outW[KMAX][VEC];
    // the VEC rows of a group are summed in fp32 and converted to fp64 once per group: the float->double
    // conversions share the SFU pipe with ex2/lg2/rcp (one conversion per row and class made the SFU pipe
    // the busiest)
    float g_loss = 0.f, g_cls[KMAX];
#pragma unroll
    for (int k = 0; k < KMAX; ++k) g_cls[k] = 0.f;
#pragma unroll
    for (int e = 0; e < VEC; ++e) {
      const bool in = (i0 + e < a.n);
      const float yf = yv[e];  // labels are compared as floats (exact small integers): no float->int conversion
      float m = -INFINITY;
      int am = 0;
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
          if (T::kReadH) p[k][e] = fmaf(a.coef[k], hh[k][e], p[k][e]);  // GBMLoss.scala:56-59
          if (p[k][e] > m) { m = p[k][e]; am = k; }
        }
      }
      // log Σ exp(p_k) = m + log1p(Σ_{k != argmax} exp(p_k - m)): the max term is exactly 1 and is kept
      // out of the sum so a well-fitted row (loss -> 0) keeps full relative precision; so does 1 - softmax of the
      // argmax class (= srest / (1 + srest)), which the label-class gradient and newton's hessian need
      float srest = 0.f, py = 0.f;
      float ex[KMAX];
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
          ex[k] = ex2_approx((p[k][e] - m) * kLog2e);
          if (k != am) srest += ex[k];
          if (yf == (float)k) py = p[k][e];
        }
      }
      const float inv_s = rcp_approx(1.0f + srest);
      const float om = srest * inv_s;  // 1 - softmax of the argmax class, without the cancellation of 1 - x
      if (T::kSumLoss && in) g_loss += ((MODE == GBM_EVAL) ? cv[e] : 1.0f) * ((m - py) + log1p_pos(srest));  // -Σ y_k (p_k - lse)  :206-221
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
          const bool top = (k == am);
          const float sm = top ? inv_s : ex[k] * inv_s;      // exp(p_k - lse)
          const float gk = (yf == (float)k) ? (top ? -om : sm - 1.0f) : sm;  // :223-238
          if (MODE == GBM_EVAL && in) g_cls[k] = fmaf(cv[e] * hh[k][e], gk, g_cls[k]);  // :66-72
          if (T::kNewton) {
            const float hc = fmaxf(sm * (top ? om : 1.0f - sm), 1e-2f);  // :240-256, GBMClassifier.scala:342
            outR[k][e] = -gk * rcp_approx(hc);                           // :362
            outW[k][e] = 0.5f * hc * wv[e];                   // :364 (× 1/S_k later)
            if (in) g_cls[k] = fmaf(cv[e], hc, g_cls[k]);
          } else if (T::kWriteR) {
            outR[k][e] = -gk;                                 // :371
          }
        }
      }
    }
    if (T::kSumLoss) acc[0] += (double)g_loss;
    if (MODE == GBM_EVAL || T::kNewton) {
#pragma unroll
      for (int k = 0; k < KMAX; ++k)
        if (k < K) acc[1 + k] += (double)g_cls[k];
    }
    // ---- stores
    if (VEC == 4 && full) {
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
          if (T::kWriteF) st_stream4(a.F + k * ld + i0, make_float4(p[k][0], p[k][1], p[k][2], p[k][3]));
          if (T::kWriteR)
            st_stream4(a.r + k * ld + i0, make_float4(outR[k][0], outR[k][1], outR[k][2], outR[k][3]));
          if (T::kNewton)
            st_stream4(a.wout + k * ld + i0, make_float4(outW[k][0], outW[k][1], outW[k][2], outW[k][3]));
        }
      }
    } else {
#pragma unroll
      for (int e = 0; e < VEC; ++e) {
        if (i0 + e < a.n) {
#pragma unroll
          for (int k = 0; k < KMAX; ++k) {
            if (k < K) {
              if (T::kWriteF) a.F[k * ld + i0 + e] = p[k][e];
              if (T::kWriteR) a.r[k * ld + i0 + e] = outR[k][e];
              if (T::kNewton) a.wout[k * ld + i0 + e] = outW[k][e];
            }
          }
        }
      }
    }
  }
  if (T::kReduce) block_reduce_publish<NRED>(acc, a.ws);
}

__global__ void __launch_bounds__(kBlock) pack_signed_kernel(const float* __restrict__ y, const float* __restrict__ F,
                                                            const float* __restrict__ h, float* __restrict__ u,
                                                            float* __restrict__ v, int64_t n) {
  const int64_t n4 = n >> 2;
  for (int64_t g = (int64_t)blockIdx.x * kBlock + threadIdx.x; g < n4; g += (int64_t)gridDim.x * kBlock) {
    const float4 vy = ld_stream4(y + 4 * g), vF = ld_stream4(F + 4 * g), vh = ld_stream4(h + 4 * g);
    float4 ou, ov;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float ye = 2.0f * f4at(vy, e) - 1.0f;  // GBMLoss.scala:272,297
      f4at(ou, e) = ye * f4at(vF, e);
      f4at(ov, e) = ye * f4at(vh, e);
    }
    st_stream4(u + 4 * g, ou);
    st_stream4(v + 4 * g, ov);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const int64_t i = (n4 << 2) + threadIdx.x;
    const float ye = 2.0f * y[i] - 1.0f;
    u[i] = ye * F[i];
    v[i] = ye * h[i];
  }
}

// F owed by the lazy squared-loss round: F = y - r, and r = y - F so that the pair is exactly what an eager update of
// this F leaves (reading F and uploading it again then changes nothing downstream)
__global__ void __launch_bounds__(kBlock) settle_f_kernel(const float* __restrict__ y, float* __restrict__ r,
                                                         float* __restrict__ F, int64_t n) {
  const int64_t n4 = n >> 2;
  for (int64_t g = (int64_t)blockIdx.x * kBlock + threadIdx.x; g < n4; g += (int64_t)gridDim.x * kBlock) {
    const float4 vy = ld_stream4(y + 4 * g), vr = ld_rw4(r + 4 * g);
    float4 oF, oR;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      f4at(oF, e) = f4at(vy, e) - f4at(vr, e);
      f4at(oR, e) = f4at(vy, e) - f4at(oF, e);
    }
    st_stream4(F + 4 * g, oF);
    st_stream4(r + 4 * g, oR);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const int64_t i = (n4 << 2) + threadIdx.x;
    const float f = y[i] - r[i];
    F[i] = f;
    r[i] = y[i] - f;
  }
}

// R pending after carried squared-loss rounds: apply their fp32 steps in place, in the order the rounds took them,
// with the fmaf each round's update applies (se_gbm_fused.cu) -- the r the last of them would have stored
__global__ void __launch_bounds__(kBlock) settle_r_kernel(float* __restrict__ r, const float* __restrict__ h,
                                                         const float* __restrict__ chain, int m, int64_t n) {
  __shared__ float s_chain[kSqDeferMax];
  for (int j = threadIdx.x; j < m; j += kBlock) s_chain[j] = chain[j];
  __syncthreads();
  const int64_t n4 = n >> 2;
  for (int64_t g = (int64_t)blockIdx.x * kBlock + threadIdx.x; g < n4; g += (int64_t)gridDim.x * kBlock) {
    float4 vr = ld_rw4(r + 4 * g);
    const float4 vh = ld_stream4(h + 4 * g);
    for (int j = 0; j < m; ++j) {
      const float c = s_chain[j];
#pragma unroll
      for (int e = 0; e < 4; ++e) f4at(vr, e) = fmaf(-c, f4at(vh, e), f4at(vr, e));
    }
    st_stream4(r + 4 * g, vr);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const int64_t i = (n4 << 2) + threadIdx.x;
    const float hi = h[i];
    float v = r[i];
    for (int j = 0; j < m; ++j) v = fmaf(-s_chain[j], hi, v);
    r[i] = v;
  }
}

__global__ void sq_alpha_kernel(const double* stats, double* out) {
  const double s1 = stats[1], s2 = stats[2];
  double al = (s2 > 0.0) ? s1 / s2 : 1.0;
  out[0] = fmin(fmax(al, 0.0), 100.0);
}

// Persistent grid: a multiple of the SM count, up to `ctas_per_sm` CTAs per SM, but never so many that a CTA
// gets fewer than ~8 work units (tiles): on large inputs later waves rebalance the tail, on small ones fewer,
// longer-lived CTAs amortise ramp-up and the per-CTA reduction epilogue.
inline int grid_for(int64_t work_items, int64_t per_cta, int ctas_per_sm, int sms) {
  int64_t units = (work_items + per_cta - 1) / per_cta;
  if (units < 1) units = 1;
  int64_t cap = (int64_t)ctas_per_sm * sms;
  if (cap > kMaxGridPartials) cap = (kMaxGridPartials / sms) * sms;
  int64_t want = (units / 8 / sms) * sms;  // >= 8 units per CTA, whole multiples of the SM count
  if (want < sms) want = sms;
  if (want > cap) want = cap;
  return (int)(units < want ? units : want);
}

template <int LOSS>
cudaError_t launch_scalar_loss(int mode, const GbmArgs& a, int ctas_per_sm, int sms, cudaStream_t st) {
  const int per_sm = LossTune<LOSS>::kHeavy ? (ctas_per_sm > 4 ? ctas_per_sm : 4) : ctas_per_sm;
  const int grid = grid_for(a.n >> 2, (int64_t)kBlock * LossTune<LOSS>::kU, per_sm, sms);
  switch (mode) {
#define SE_CASE_W(M) /* writes per-row results: explicit policy always */ \
  case M: gbm_scalar_kernel<LOSS, M, true><<<grid, kBlock, 0, st>>>(a); break;
#define SE_CASE_R(M) /* read-only pass: explicit policy only with the small-shard hints */ \
  case M:                                                                                  \
    if (a.l2_hints) gbm_scalar_kernel<LOSS, M, true><<<grid, kBlock, 0, st>>>(a);          \
    else gbm_scalar_kernel<LOSS, M, false><<<grid, kBlock, 0, st>>>(a);                    \
    break;
    SE_CASE_W(GBM_RESID)
    SE_CASE_W(GBM_RESID_NEWTON)
    SE_CASE_R(GBM_EVAL)
    SE_CASE_W(GBM_UPDATE)
    SE_CASE_W(GBM_UPDATE_RESID)
    SE_CASE_W(GBM_UPDATE_NEWTON)
    SE_CASE_R(GBM_MEAN_LOSS)
    SE_CASE_R(GBM_EVAL_LOSS)
#undef SE_CASE_W
#undef SE_CASE_R
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

template <int KMAX, int VEC>
cudaError_t launch_logloss_k(int mode, const GbmArgs& a, int grid, cudaStream_t st) {
  switch (mode) {
#define SE_CASE(M) \
  case M: gbm_logloss_kernel<KMAX, M, VEC><<<grid, kBlock, 0, st>>>(a); break;
    SE_CASE(GBM_RESID)
    SE_CASE(GBM_RESID_NEWTON)
    SE_CASE(GBM_EVAL)
    SE_CASE(GBM_UPDATE)
    SE_CASE(GBM_UPDATE_RESID)
    SE_CASE(GBM_UPDATE_NEWTON)
    SE_CASE(GBM_MEAN_LOSS)
#undef SE_CASE
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_gbm(int loss, int mode, const GbmArgs& a, int ctas_per_sm, int sms,
                       cudaStream_t st) {
  if (mode == GBM_SQ_STATS) {
    if (loss != SE_LOSS_SQUARED) return cudaErrorInvalidValue;
    const int grid = grid_for(a.n >> 2, (int64_t)kBlock * U_SCALAR, ctas_per_sm, sms);
    if (a.stats_from_r) {
      if (a.l2_hints) gbm_sq_stats_kernel<true, true><<<grid, kBlock, 0, st>>>(a);
      else gbm_sq_stats_kernel<true, false><<<grid, kBlock, 0, st>>>(a);
    } else {
      if (a.l2_hints) gbm_sq_stats_kernel<false, true><<<grid, kBlock, 0, st>>>(a);
      else gbm_sq_stats_kernel<false, false><<<grid, kBlock, 0, st>>>(a);
    }
    return cudaGetLastError();
  }
  if (loss != SE_LOSS_LOGLOSS) {
    switch (loss) {
      case SE_LOSS_SQUARED: return launch_scalar_loss<SE_LOSS_SQUARED>(mode, a, ctas_per_sm, sms, st);
      case SE_LOSS_ABSOLUTE: return launch_scalar_loss<SE_LOSS_ABSOLUTE>(mode, a, ctas_per_sm, sms, st);
      case SE_LOSS_HUBER: return launch_scalar_loss<SE_LOSS_HUBER>(mode, a, ctas_per_sm, sms, st);
      case SE_LOSS_QUANTILE: return launch_scalar_loss<SE_LOSS_QUANTILE>(mode, a, ctas_per_sm, sms, st);
      case SE_LOSS_LOGCOSH: return launch_scalar_loss<SE_LOSS_LOGCOSH>(mode, a, ctas_per_sm, sms, st);
      case SE_LOSS_SCALED_LOGCOSH: return launch_scalar_loss<SE_LOSS_SCALED_LOGCOSH>(mode, a, ctas_per_sm, sms, st);
      case SE_LOSS_BERNOULLI: return launch_scalar_loss<SE_LOSS_BERNOULLI>(mode, a, ctas_per_sm, sms, st);
      case SE_LOSS_EXPONENTIAL: return launch_scalar_loss<SE_LOSS_EXPONENTIAL>(mode, a, ctas_per_sm, sms, st);
      default: return cudaErrorInvalidValue;
    }
  }
  const int K = a.dim;
  if (K < 1 || K > kMaxDim) return cudaErrorInvalidValue;
  if (K >= kLoglossTiledMinK) return launch_gbm_logloss_tiled(mode, a, sms, st);
  if (ctas_per_sm > 4) ctas_per_sm = 4;  // register-resident K <= 4 kernels
  if (K <= 2) return launch_logloss_k<2, 4>(mode, a, grid_for((a.n + 3) / 4, kBlock, ctas_per_sm, sms), st);
  return launch_logloss_k<4, 4>(mode, a, grid_for((a.n + 3) / 4, kBlock, ctas_per_sm, sms), st);
}

cudaError_t launch_gbm_pack_signed(const float* y, const float* F, const float* h, float* u, float* v, int64_t n,
                                   int sms, cudaStream_t st) {
  pack_signed_kernel<<<grid_for(n >> 2, kBlock, 4, sms), kBlock, 0, st>>>(y, F, h, u, v, n);
  return cudaGetLastError();
}

cudaError_t launch_gbm_settle_f(const float* y, float* r, float* F, int64_t n, int sms, cudaStream_t st) {
  settle_f_kernel<<<grid_for(n >> 2, kBlock, 4, sms), kBlock, 0, st>>>(y, r, F, n);
  return cudaGetLastError();
}

cudaError_t launch_gbm_settle_r(float* r, const float* h, const float* chain, int m, int64_t n, int sms,
                                cudaStream_t st) {
  if (m < 1 || m > kSqDeferMax) return cudaErrorInvalidValue;
  settle_r_kernel<<<grid_for(n >> 2, kBlock, 4, sms), kBlock, 0, st>>>(r, h, chain, m, n);
  return cudaGetLastError();
}

cudaError_t launch_sq_alpha(const double* stats, double* out_alpha, cudaStream_t st) {
  sq_alpha_kernel<<<1, 1, 0, st>>>(stats, out_alpha);
  return cudaGetLastError();
}

}  // namespace se
