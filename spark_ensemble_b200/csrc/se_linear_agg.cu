// se_linear_agg.cu — an ensemble of linear and logistic members scored in ONE pass over the resident features
// (se_linear_agg, DESIGN.md §3 "Linear ensembles in one pass").
//
// The member route runs se_logistic_predict once per member into SE_SLOT_P ([M][width][n] fp32) and se_agg_run over it:
// 4·M·width B per row written and read back.  Here a thread owns one row, forms every member's margins from the
// member's columns of X, turns them into the member's output with se_logistic_predict's own row steps and folds that
// output into the row's aggregate at once, then finishes the row with se_agg_run's epilogue.  X is read column by
// column, coalesced across the warp, through L1: a column that several members use comes from HBM once per tile.
// Coefficients and member records are uniform across the CTA and read through the read-only cache.
#include "se_kernels.h"
#include "se_row_steps.cuh"

namespace se {

namespace {

static_assert(kForestAggMaxClasses == SE_FOREST_AGG_MAX_CLASSES, "the classifier kinds' class limit is se_forest_agg's");

// The margins of member mb for row `row` (se_logistic_predict's lg_row_margins over the member's columns).
template <int MAXD>
__device__ __forceinline__ void member_margins(const LinearAggArgs& g, const LinearAggMember& mb, int64_t row,
                                               double (&m)[MAXD]) {
  const double* coef = g.coef + mb.coef0;
  const unsigned long long* coloff = g.coloff + mb.col0;
  const int p = mb.p;
  lg_row_margins<MAXD>(
      p, mb.D, [&](int k, int j) { return __ldg(coef + (size_t)k * p + j); },
      [&](int j) { return (double)__ldg(g.X + __ldg(coloff + j) + row); }, g.coef + mb.icpt0, m);
}

// Every kind but the median.  Per member, by kind:
//   sum kinds (GBM / Bagging regressor, Boosting mean)  its value v = (float) m_0 into agg_sum_kernel's fold (AggRowFold)
//   GBM classifier         w · v to class cls (the tree kernel's kFaTreeClass)
//   Bagging hard, SAMME    w to class label (kFaVote)
//   Bagging soft, SAMME.R  p_k, or lg2 max(p_k, ε), to every class k (kFaSoft, kFaReal)
// Classifier totals are fp64 in the row's own column of shared memory and added in model order; the row is finished by
// finalize_row / finalize_real_row / finalize_binary_row as se_forest_agg finishes it.
template <int MAXD>
__global__ void __launch_bounds__(kLinearAggTile) linear_agg_kernel(const __grid_constant__ LinearAggArgs g,
                                                                    const FinArgs fin) {
  constexpr int TILE = kLinearAggTile;
  extern __shared__ double s_tot[];  // [C][TILE]
  const int kind = g.kind, M = g.M, C = g.C;
  const bool sums = (kind == SE_AGG_GBM_REGRESSOR || kind == SE_AGG_BAGGING_REGRESSOR || kind == SE_AGG_BOOSTING_REG_MEAN);
  const bool real = (kind == SE_AGG_BOOSTING_REAL);
  double* tot = s_tot + threadIdx.x;  // this row's totals: own column, no synchronisation
  for (int64_t row = (int64_t)blockIdx.x * TILE + threadIdx.x; row < g.n; row += (int64_t)gridDim.x * TILE) {
    AggRowFold fold(M, row >= g.n4, g.init[0]);
    if (!sums)
      for (int c = 0; c < C; ++c) tot[c * TILE] = g.init[c];
    for (int i = 0; i < M; ++i) {
      const LinearAggMember& mb = g.members[i];
      double m[MAXD];
      member_margins<MAXD>(g, mb, row, m);
      if (sums) {
        fold.add(mb.wf, (float)m[0]);
      } else if (kind == SE_AGG_GBM_CLASSIFIER) {
        tot[mb.cls * TILE] += mb.w * (double)(float)m[0];
      } else {
        double mx;
        const int best = lg_row_argmax<MAXD>(mb.D, m, &mx);
        if (kind == SE_AGG_BAGGING_HARD || kind == SE_AGG_BOOSTING_DISCRETE) {
          tot[(int)lg_row_label(mb.D, m[0], best, mb.threshold) * TILE] += mb.w;
        } else {
          lg_row_probs<MAXD>(mb.D, m, mx, [&](int k, float v) {
            tot[k * TILE] += real ? (double)lg2_clamped(v) : (double)v;
          });
        }
      }
    }
    if (sums) {
      g.out[row] = fold.end(g.init[0], g.post_div);
    } else if (kind == SE_AGG_GBM_CLASSIFIER && g.dim == 1 && g.K == 2) {
      finalize_binary_row(fin, row, (float)tot[0]);
    } else if (real) {
      finalize_real_row(fin, row, [&](int c) { return tot[c * TILE]; });
    } else {
      finalize_row(fin, row, [&](int c) { return tot[c * TILE]; });
    }
  }
}

// The weighted median of at most 64 linear members: the row's M values (float) m_0 in its own column of shared memory
// ([M][TILE]), then se_forest_median's pick on them (wm_pick_row), so the result is se_agg_run's bit for bit.
template <int MP>
__global__ void __launch_bounds__(kLinearAggTile) linear_median_kernel(const __grid_constant__ LinearAggArgs g) {
  constexpr int TILE = kLinearAggTile;
  extern __shared__ float s_vals[];  // [M][TILE]
  __shared__ double s_a[kForestMedianMaxTrees];
  for (int m = threadIdx.x; m < kForestMedianMaxTrees; m += TILE) s_a[m] = (m < g.M) ? g.w[m] : 0.0;
  __syncthreads();
  float* vals = s_vals + threadIdx.x;
  for (int64_t row = (int64_t)blockIdx.x * TILE + threadIdx.x; row < g.n; row += (int64_t)gridDim.x * TILE) {
    for (int i = 0; i < g.M; ++i) {
      double m[1];
      member_margins<1>(g, g.members[i], row, m);
      vals[i * TILE] = (float)m[0];
    }
    bool exact;
    g.out[row] = wm_unkey(wm_pick_row<MP>(vals, TILE, g.M, g.mode, g.w, g.total, g.tau, s_a, true, exact));
  }
}

// Calls f(std::integral_constant<int, MP>()) for the power of two MP >= M the median kernel is instantiated for.
template <class F>
cudaError_t with_median_mp(int M, F f) {
  if (M <= 1) return f(std::integral_constant<int, 1>());
  if (M <= 2) return f(std::integral_constant<int, 2>());
  if (M <= 4) return f(std::integral_constant<int, 4>());
  if (M <= 8) return f(std::integral_constant<int, 8>());
  if (M <= 16) return f(std::integral_constant<int, 16>());
  if (M <= 32) return f(std::integral_constant<int, 32>());
  if (M <= 64) return f(std::integral_constant<int, 64>());
  return cudaErrorInvalidValue;
}

}  // namespace

cudaError_t launch_linear_agg(const LinearAggArgs& g, int max_d, int sms, cudaStream_t st) {
  if (g.M < 1 || g.n < 1 || g.C < 1 || g.C > kForestAggMaxClasses || max_d < 1 || max_d > kForestAggMaxClasses)
    return cudaErrorInvalidValue;
  const bool median = (g.kind == SE_AGG_BOOSTING_REG_MEDIAN);
  if (median && (g.M > kForestMedianMaxTrees || max_d != 1)) return cudaErrorInvalidValue;
  const size_t smem = median ? (size_t)g.M * kLinearAggTile * sizeof(float) : (size_t)g.C * kLinearAggTile * sizeof(double);
  int per_sm = (int)((220 * 1024) / (smem + 1024));
  if (per_sm < 1) per_sm = 1;
  if (per_sm > 16) per_sm = 16;
  const int grid = grid_rows(g.n, kLinearAggTile, per_sm, sms);
  if (median) {
    return with_median_mp(g.M, [&](auto mp) {
      auto kern = linear_median_kernel<decltype(mp)::value>;
      const cudaError_t e = allow_dynamic_smem(kern, smem);
      if (e != cudaSuccess) return e;
      kern<<<grid, kLinearAggTile, smem, st>>>(g);
      return cudaGetLastError();
    });
  }
  FinArgs f{};
  f.kind = g.kind; f.C = g.C; f.K = g.K; f.dim = g.dim; f.loss = g.loss; f.M = g.M;
  f.sum_a = g.sum_a;
  f.n = g.n; f.ld = g.ld_out; f.raw = g.raw; f.prob = g.prob; f.label = g.label;
  f.inv_km1 = 1.0 / (double)((g.K > 1 ? g.K : 2) - 1);
  return with_maxd(max_d, [&](auto md) {
    auto kern = linear_agg_kernel<decltype(md)::value>;
    const cudaError_t e = allow_dynamic_smem(kern, smem);
    if (e != cudaSuccess) return e;
    kern<<<grid, kLinearAggTile, smem, st>>>(g, f);
    return cudaGetLastError();
  });
}

}  // namespace se
