// se_gbm_generic.cu — LogLoss(K) for ANY number of classes (boosting/GBMLoss.scala:196-263 takes any numClasses; the
// register / TMA-tiled kernels of se_gbm.cu / se_gbm_tiled.cu specialise K <= 64).  General path, built for
// correctness and determinism rather than for the roofline: one WARP per CTA, one row per lane, three sweeps over the
// K classes of the lane's row (running max + F update, exp-sum + label term, outputs + per-class sums).  Accesses are
// coalesced (consecutive lanes = consecutive rows of one class row).  Per-class sums Σ_i c_i h_ik g_ik (line search,
// :66-72) / Σ_i c_i max(H_ik, 1e-2) (newton, GBMClassifier.scala:342-355) are folded warp-wide with shuffles and
// accumulated by lane 0 into the CTA's [K+1] fp64 accumulators in shared memory — a fixed order; the CTA partials go
// to global memory and the last CTA folds them in CTA order: results are deterministic for a launch configuration.
#include "se_kernels.h"
#include "se_loss.cuh"

namespace se {

namespace {

template <int MODE>
struct GenTraits {
  static constexpr bool kReadH = (MODE == GBM_EVAL || MODE == GBM_UPDATE || MODE == GBM_UPDATE_RESID || MODE == GBM_UPDATE_NEWTON);
  static constexpr bool kWriteF = (MODE == GBM_UPDATE || MODE == GBM_UPDATE_RESID || MODE == GBM_UPDATE_NEWTON);
  static constexpr bool kNewton = (MODE == GBM_RESID_NEWTON || MODE == GBM_UPDATE_NEWTON);
  static constexpr bool kWriteR = (MODE == GBM_RESID || MODE == GBM_UPDATE_RESID || kNewton);
  static constexpr bool kSumLoss = (MODE == GBM_EVAL || kWriteF || MODE == GBM_MEAN_LOSS);
  static constexpr bool kPerClass = (MODE == GBM_EVAL || kNewton);
  static constexpr bool kReduce = kSumLoss || kNewton;
};

template <int MODE>
__global__ void __launch_bounds__(32) gbm_logloss_generic_kernel(const GbmArgs a, const GenericArgs ga) {
  using T = GenTraits<MODE>;
  extern __shared__ double s_acc[];  // [K + 1]: [0] = Σloss, [1 + k] per class
  const int K = a.dim;
  const int64_t ld = a.ld;
  const int lane = threadIdx.x;
  for (int k = lane; k <= K; k += 32) s_acc[k] = 0.0;
  __syncwarp();
  const bool has_w = (a.w != nullptr);
  constexpr bool kBagMode = (MODE == GBM_EVAL) || T::kNewton;
  const bool has_bag = kBagMode && (a.bag != nullptr);
  double loss_acc = 0.0;
  const int64_t ngroups = (a.n + 31) / 32;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t i = g * 32 + lane;
    const bool in = i < a.n;
    const int64_t ii = in ? i : a.n - 1;  // out-of-range lanes shadow the last row (they never store or count)
    const float yf = a.y[ii];
    const int yi = min(max((int)yf, 0), K - 1);  // validity is checked once per label upload (se_api.cu)
    const float c = has_bag ? a.bag[ii] : 1.0f;
    const float w = (T::kNewton && has_w) ? a.w[ii] : 1.0f;
    // sweep 1: p_k = F_k + coef_k h_k (GBMLoss.scala:56-59), running max (first maximum), F update
    float m = -INFINITY, py = 0.f;
    int am = 0;
    for (int k = 0; k < K; ++k) {
      float p = a.F[(int64_t)k * ld + ii];
      if (T::kReadH) p = fmaf(__ldg(ga.coef + k), a.h[(int64_t)k * ld + ii], p);
      if (T::kWriteF && in) a.F[(int64_t)k * ld + ii] = p;
      if (p > m) m = p, am = k;
      if (k == yi) py = p;
    }
    auto pk = [&](int k) -> float {  // p_k again: from the updated F, or recomputed (same fma, same value)
      float p = a.F[(int64_t)k * ld + ii];
      if (T::kReadH && !(T::kWriteF && in)) p = fmaf(__ldg(ga.coef + k), a.h[(int64_t)k * ld + ii], p);
      return p;
    };
    // sweep 2: Σ_{k != argmax} exp(p_k - m) — shifted log-sum-exp (identical wherever the reference's unshifted form is
    // finite) with the max term, exactly 1, kept out of the sum: a well-fitted row keeps full relative precision in its
    // loss and in 1 - softmax_argmax
    float srest = 0.f;
    for (int k = 0; k < K; ++k)
      if (k != am) srest += ex2_approx((pk(k) - m) * kLog2e);
    const float inv_s = rcp_approx(1.0f + srest);
    const float om = srest * inv_s;  // 1 - softmax of the argmax class
    if (T::kSumLoss && in) {
      const float l = (m - py) + log1p_pos(srest);  // -Σ y_k (p_k - lse)  (:206-221)
      loss_acc += (double)(((MODE == GBM_EVAL) ? c : 1.0f) * l);
    }
    // sweep 3: gradients / outputs / per-class sums
    if (T::kWriteR || T::kPerClass) {
      for (int k = 0; k < K; ++k) {
        const bool top = (k == am);
        const float sm = top ? inv_s : ex2_approx((pk(k) - m) * kLog2e) * inv_s;   // exp(p_k - lse)
        const float gk = (k == yi) ? (top ? -om : sm - 1.0f) : sm;                // :223-238
        float term = 0.f;
        if (T::kNewton) {
          const float hc = fmaxf(sm * (top ? om : 1.0f - sm), 1e-2f);             // :240-256, GBMClassifier.scala:342
          if (in) {
            a.r[(int64_t)k * ld + ii] = -gk * rcp_approx(hc);        // :362
            a.wout[(int64_t)k * ld + ii] = 0.5f * hc * w;            // :364 (x 1/S_k when it leaves the device)
          }
          term = in ? c * hc : 0.f;
        } else {
          if (T::kWriteR && in) a.r[(int64_t)k * ld + ii] = -gk;     // :371
          if (MODE == GBM_EVAL) term = in ? c * a.h[(int64_t)k * ld + ii] * gk : 0.f;  // :66-72
        }
        if (T::kPerClass) {
          double t = (double)term;
#pragma unroll
          for (int off = 16; off > 0; off >>= 1) t += __shfl_down_sync(0xffffffffu, t, off);
          if (lane == 0) s_acc[1 + k] += t;
        }
      }
    }
  }
  if (!T::kReduce) return;
  loss_acc = warp_sum(loss_acc);
  if (lane == 0) s_acc[0] = loss_acc;
  __syncwarp();
  double* mine = ga.partials + (size_t)blockIdx.x * (K + 1);
  for (int k = lane; k <= K; k += 32) mine[k] = s_acc[k];
  __threadfence();
  __syncwarp();
  __shared__ bool is_last;
  if (lane == 0) {
    __threadfence();
    is_last = (atomicInc(a.ws.counter, gridDim.x - 1) == gridDim.x - 1);
  }
  __syncwarp();
  if (!is_last) return;
  __threadfence();
  for (int k = lane; k <= K; k += 32) {  // fixed order over the CTAs
    double v = 0.0;
    for (unsigned int b = 0; b < gridDim.x; ++b) v += __ldcg(&ga.partials[(size_t)b * (K + 1) + k]);
    ga.out[k] = v;
  }
}

}  // namespace

cudaError_t launch_gbm_logloss_generic(int mode, const GbmArgs& a, const GenericArgs& ga, int grid, cudaStream_t st) {
  const size_t smem = sizeof(double) * (size_t)(a.dim + 1);
  switch (mode) {
#define SE_CASE(M)                                                                                                   \
  case M: {                                                                                                          \
    auto kern = gbm_logloss_generic_kernel<M>;                                                                       \
    if (smem > 48 * 1024) {                                                                                          \
      cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);            \
      if (e != cudaSuccess) return e;                                                                                \
    }                                                                                                                \
    kern<<<grid, 32, smem, st>>>(a, ga);                                                                             \
    break;                                                                                                           \
  }
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

}  // namespace se
