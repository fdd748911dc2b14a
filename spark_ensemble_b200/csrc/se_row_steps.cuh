// se_row_steps.cuh — the per-row steps that the aggregation kernels (se_agg.cu), the one-pass forest kernels and the
// linear scoring kernels (se_logistic.cu, se_linear_agg.cu) share, written once so that a one-pass kernel gives the
// bits of the member route it replaces: agg_sum_kernel's fold of a row's terms, the classifier epilogues, the weighted
// median's picks and se_logistic_predict's margins, probabilities and label.
#pragma once

#include <math.h>

#include <type_traits>

#include "se_common.cuh"
#include "se_loss.cuh"
#include "se_sortnet.h"
#include "../../include/se_abi.h"

namespace se {

namespace {

constexpr float kSparkEps = 2.220446049250313e-16f;
constexpr int MU = 8;  // models loaded per batch: 8 independent 16 B requests per thread

// lg2 max(p, ε): the clamp is the exact constant lg2 2^-52 = -52 (NaN clamps too), so the sums of pure-leaf outputs
// (exact 0s and 1s) are exact multiples of 52 and equal vote counts give equal totals
__device__ __forceinline__ float lg2_clamped(float p) { return (p > kSparkEps) ? lg2_approx(p) : -52.0f; }

// Per-row epilogue on the C per-class sums t_c (from shared memory or from the RAW slot): raw, prob, label.
struct FinArgs {
  int kind, C, K, dim, loss, M;
  double sum_a;  // Σ a_m (boosting discrete)
  int64_t n, ld;
  float* raw;
  float* prob;
  float* label;
  int* bad_label;  // raised when a vote is not a class index in [0, K)
  double inv_km1;  // 1 / (K - 1)
};

// raw value from the stage-1 sum.  Discrete: K·A_k − Σa subtracts nearly equal numbers and is formed in fp64 before
// the single rounding to the fp32 output.  (SAMME.R has its own epilogue, finalize_real_row.)
template <class T>
__device__ __forceinline__ float fin_raw(const FinArgs& f, T t, float mean_t) {
  switch (f.kind) {
    case SE_AGG_BOOSTING_DISCRETE:  // +a on the vote, −a/(K-1) elsewhere   :371-376
      return (float)(((double)t * (double)f.K - f.sum_a) * f.inv_km1);  // one reciprocal instead of an fp64 division per class
    default: return (float)t;
  }
}

// SAMME.R epilogue.  get(c) returns T_c = Σ_m lg2 max(p_mc, ε) in fp64 (exact for pure leaves).  With L = T ln 2:
// raw_c = (K-1)(L_c − mean L) (BoostingClassifier.scala:355-360) and prob = softmax(raw/(K-1)) = 2^(T_c − T_max) / Σ
// (:342-346), formed from the fp64 differences, not from the rounded raw (|raw| reaches (K-1)·36·M, where one fp32 ulp
// of raw is already 1e-5 of a probability).  First-maximum argmax of T, which orders the classes as raw does.
// Three sweeps over the classes, each reading get(c) again: the third overwrites what the stage-1 sums were read from.
template <class Get>
__device__ __forceinline__ void finalize_real_row(const FinArgs& f, int64_t i, Get get) {
  const int C = f.C;
  double s = 0.0, tmax = -INFINITY;
  int am = 0;
  for (int c = 0; c < C; ++c) {
    const double t = get(c);
    s += t;
    if (t > tmax) tmax = t, am = c;  // Vector.argmax: first maximum
  }
  const double mean = s / (double)C;
  const double rs = (double)(f.K - 1) * 0.6931471805599453;
  float ssum = 0.f;
  for (int c = 0; c < C; ++c) ssum += ex2_approx((float)(get(c) - tmax));
  const float inv = 1.0f / ssum;
  for (int c = 0; c < C; ++c) {
    const double t = get(c);
    f.prob[c * f.ld + i] = ex2_approx((float)(t - tmax)) * inv;
    f.raw[c * f.ld + i] = (float)(rs * (t - mean));
  }
  f.label[i] = (float)am;
}

// get(c) returns the stage-1 sum of class c for this row.  Two sweeps over the classes: (1) raw values with an
// online max / Σexp / first-argmax, (2) write raw and probability.
template <class Get>
__device__ __forceinline__ void finalize_row(const FinArgs& f, int64_t i, Get get) {
  const int C = f.C;
  const float mean_t = 0.f;
  const bool softmax = (f.kind == SE_AGG_BOOSTING_DISCRETE || f.kind == SE_AGG_GBM_CLASSIFIER);
  // boosting: softmax(raw/(K-1)) (BoostingClassifier.scala:342-346); GBM logloss: softmax(raw) (GBMLoss.scala:258-261)
  const float sc = (f.kind == SE_AGG_GBM_CLASSIFIER) ? kLog2e : kLog2e / (float)(f.K - 1);
  float best = -INFINITY, ssum = 0.f;
  int am = 0;
  for (int c = 0; c < C; ++c) {
    const float r = fin_raw(f, get(c), mean_t);
    if (r > best) am = c;  // Vector.argmax: first maximum
    const float mn = fmaxf(best, r);
    if (softmax) ssum = fmaf(ssum, ex2_approx((best - mn) * sc), ex2_approx((r - mn) * sc));
    best = mn;
  }
  f.label[i] = (float)am;
  const float inv = softmax ? rcp_approx(ssum) : 1.0f / (float)f.M;  // bagging: prob = raw·(1/M) (BaggingClassifier.scala:285-287)
  for (int c = 0; c < C; ++c) {
    const float r = fin_raw(f, get(c), mean_t);
    f.prob[c * f.ld + i] = softmax ? ex2_approx((r - best) * sc) * inv : r * inv;
    f.raw[c * f.ld + i] = r;
  }
}

// Binary GBM classifier with dim 1 (GBMClassifier.scala:583-584 + GBMLoss.scala:284-289,311-316): raw = (−F, F) from
// the one total F = res.
__device__ __forceinline__ void finalize_binary_row(const FinArgs& f, int64_t i, float res) {
  const float r0 = -res;
  // p1 = 1/(1+e^x), p0 = 1 - p1 with x = raw(0) (bernoulli) or -2 raw(0) (exponential); both
  // formed from t = e^-|x| so the small one keeps full relative precision
  const float x = (f.loss == SE_LOSS_EXPONENTIAL) ? -2.0f * r0 : r0;
  const float t = exp_neg_fast(-fabsf(x));
  const float inv = rcp_approx(1.0f + t);
  const float p1 = (x >= 0.f) ? t * inv : inv;
  const float p0 = (x >= 0.f) ? inv : t * inv;
  f.raw[i] = r0;
  f.raw[f.ld + i] = res;
  f.prob[i] = p0;
  f.prob[f.ld + i] = p1;
  f.label[i] = (res > r0) ? 1.0f : 0.0f;  // argmax, first maximum on ties
}

__device__ __forceinline__ uint32_t wm_key(float x) {
  const uint32_t u = __float_as_uint(x + 0.0f);  // -0 -> +0: equal values stay ties
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float wm_unkey(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// sort of the (key, model) words + the reference's sorted-order cumulative sums (ensemble/Utils.scala:31-38)
template <int MP>
__device__ __forceinline__ unsigned long long wm_exact_pick(unsigned long long (&w)[MP], int M, const double* s_a) {
  sortnet_oddeven<MP>(w, [](unsigned long long& x, unsigned long long& y) {
    const bool swap = x > y;
    const unsigned long long lo = swap ? y : x, hi = swap ? x : y;
    x = lo;
    y = hi;
  });
  double total = 0.0;
#pragma unroll
  for (int m = 0; m < MP; ++m)
    if (m < M) total += s_a[(unsigned)w[m]];
  const double half = 0.5 * total;
  double cum = 0.0;
  bool found = false;
  unsigned long long pick = 0ull;
#pragma unroll
  for (int m = 0; m < MP; ++m) {
    if (m < M) {
      cum += s_a[(unsigned)w[m]];
      const bool hit = !found && (cum >= half);
      pick = (hit || (!found && m == M - 1)) ? w[m] : pick;  // last element when nothing reaches half (NaN weights)
      found = found || hit;
    }
  }
  return pick;
}

// ---- weighted median, fast path (M <= 64, all weights finite and >= 0) -------------------------------------------
// The exact kernels above carry (key, model) words through the sort because the reference accumulates the weights in
// SORTED order (ensemble/Utils.scala:31-38) — 6 ALU-pipe instructions per compare-exchange, and the ALU pipe issues at
// half rate.  With weights >= 0 the answer is `the smallest value v whose group-end
// cumulative weight C(v) reaches h = total / 2` (cumulative sums are monotone in fp64 too).  C(v) and h are recursive
// fp64 sums of the same addends as Ĉ(v) = Σ_{x_j <= v} a_j and ĥ = T̂ / 2 taken in MODEL order, so
//     |(C(v) - h) - (Ĉ(v) - ĥ)| <= 3 (M - 1) 2^-53 T (1 + eps)
// and whenever both neighbours of the crossing clear the margin tau = 8 M 2^-53 T̂ the model-order decision IS the
// reference's decision.  So: sort the 32-bit keys alone (min/max, 2 instructions per compare-exchange, Batcher's
// 191-element network), bisect the sorted keys on Ĉ (5 x 32 predicated DADDs with the weights as constant-bank
// operands), and send the rows that do not clear the margin — none for generic weights, the exact ties for
// small-integer weights — to the exact kernel through a compacted list (mode 2: all weights equal, where both orders
// produce the same sums and no margin is needed).
struct WmWeights {
  double w[64];
};

template <int MP, int L>
__device__ __forceinline__ uint32_t wm_candidate(const uint32_t (&s)[MP], uint32_t t) {
  // level-L bisection probe: position step - 1 + t * 2 * step, t in [0, 2^L) — a select tree over static indices
  constexpr int step = MP >> (L + 1);
  uint32_t v = s[step - 1];
#pragma unroll
  for (int q = 1; q < (1 << L); ++q) v = (t == (uint32_t)q) ? s[step - 1 + q * 2 * step] : v;
  return v;
}

// The fast path's pick for a row of keys key[0..MP) in model order (padding keys ~0u carry weight 0): the smallest key
// whose model-order cumulative weight reaches half the total.  safe: the crossing clears the margin tau on both sides,
// so the reference's sorted-order sums pick the same key.  w is a __grid_constant__ parameter: the DFMAs of the
// bisection read the weights as constant-bank operands.
template <int MP>
__device__ __forceinline__ uint32_t wm_fast_pick(const uint32_t (&key)[MP], const double (&w)[64], double total,
                                                 double tau, bool& safe) {
  constexpr int LOG = (MP == 1) ? 0 : (MP == 2) ? 1 : (MP == 4) ? 2 : (MP == 8) ? 3 : (MP == 16) ? 4 : (MP == 32) ? 5 : 6;
  uint32_t s[MP];
#pragma unroll
  for (int m = 0; m < MP; ++m) s[m] = key[m];
  sortnet_oddeven<MP>(s, [](uint32_t& x, uint32_t& y) {
    const uint32_t lo = min(x, y), hi = max(x, y);
    x = lo;
    y = hi;
  });
  const double half = 0.5 * total;
  // invariant: P(lo) false, P(hi) true with P(k) := Ĉ(s[k]) >= ĥ; lo = t - 1, hi = t after LOG probes
  uint32_t t = 0, v_hi = s[MP - 1];
  double c_lo = 0.0, c_hi = total;
  auto probe = [&](uint32_t v) {
    double c = 0.0;
#pragma unroll
    for (int m = 0; m < MP; ++m) {
      // model order; padding (and m >= M) weights are 0.  fma(w, 1.0 or 0.0, c) is c + w rounded once, or c: one
      // select of the high word of the 0/1 factor instead of the two selects `if (...) c += w` compiles to
      const double b = __hiloint2double((key[m] <= v) ? 0x3ff00000 : 0, 0);
      c = fma(w[m], b, c);
    }
    const bool right = !(c >= half);
    c_lo = right ? c : c_lo;
    c_hi = right ? c_hi : c;
    v_hi = right ? v_hi : v;
    t = 2u * t + (right ? 1u : 0u);
  };
  if constexpr (LOG > 0) probe(wm_candidate<MP, 0>(s, t));
  if constexpr (LOG > 1) probe(wm_candidate<MP, 1>(s, t));
  if constexpr (LOG > 2) probe(wm_candidate<MP, 2>(s, t));
  if constexpr (LOG > 3) probe(wm_candidate<MP, 3>(s, t));
  if constexpr (LOG > 4) probe(wm_candidate<MP, 4>(s, t));
  if constexpr (LOG > 5) probe(wm_candidate<MP, 5>(s, t));
  safe = (c_hi - half > tau) && (half - c_lo > tau);
  return v_hi;
}

// ---- agg_sum_kernel's fold of one row's terms w_m·x_m (fp32 weights and values) ----------------------------------
// Each batch of MU terms is summed in fp32 in two chains (even and odd members, fmaf from 0); the batch sum joins an
// fp64 total when the row has more than two batches (wide), an fp32 carry otherwise.  The result is (total + init)
// / post_div (post_div 0: none), rounded once.  agg_sum_kernel's tail rows (the last n & 3) take another form: the
// total starts at init and every fp32 product is added in fp64 (agg_tail_add).
__device__ __forceinline__ void agg_fold_batch(bool wide, float s, double& d, float& carry) {
  if (wide) d += (double)s;
  else carry += s;
}
__device__ __forceinline__ float agg_fold_end(bool wide, double d, float carry, double init, float post_div) {
  if (!wide) d = (double)carry;
  d += init;
  if (post_div != 0.f) d /= (double)post_div;
  return (float)d;
}
__device__ __forceinline__ void agg_tail_add(double& d, float w, float x) { d += (double)(w * x); }

// The fold above for one row whose terms come one at a time, in model order.
struct AggRowFold {
  bool wide, tail;
  int u = 0;
  float s0 = 0.f, s1 = 0.f, carry = 0.f;
  double d = 0.0;
  __device__ __forceinline__ AggRowFold(int M, bool tail_row, double init) : wide(M > 2 * MU), tail(tail_row) {
    if (tail) d = init;
  }
  __device__ __forceinline__ void add(float w, float x) {
    if (tail) {
      agg_tail_add(d, w, x);
      return;
    }
    if (u & 1) s1 = fmaf(w, x, s1);
    else s0 = fmaf(w, x, s0);
    if (++u == MU) {
      agg_fold_batch(wide, s0 + s1, d, carry);
      s0 = s1 = 0.f;
      u = 0;
    }
  }
  __device__ __forceinline__ float end(double init, float post_div) {
    if (tail) {
      if (post_div != 0.f) d /= (double)post_div;
      return (float)d;
    }
    if (u) agg_fold_batch(wide, s0 + s1, d, carry);
    return agg_fold_end(wide, d, carry, init, post_div);
  }
};

// ---- the weighted median of one row's M values vals[m · stride] ---------------------------------------------------
// agg_wmedian_fast_kernel's pick (modes 1 and 2), and the exact (key, model) sort with sorted-order sums of
// agg_wmedian_list_kernel / agg_wmedian_reg_kernel for the rows inside the margin (mode 1) or for every row (mode 0):
// the key of the value se_agg_run(SE_AGG_BOOSTING_REG_MEDIAN) picks.  exact: the row took the exact sort.  w holds the
// weights (0 past M) and is a __grid_constant__ parameter of the caller; s_a holds them in shared memory.
template <int MP>
__device__ __forceinline__ uint32_t wm_pick_row(const float* vals, int stride, int M, int mode, const double (&w)[64],
                                                double total, double tau, const double* s_a, bool in, bool& exact) {
  uint32_t pick = 0;
  exact = (mode == 0);
  if constexpr (MP == 1) {  // one member: both routes return its value (one weight is always "all equal": no margin)
    pick = wm_key(vals[0]);
    exact = false;
  } else if (in && mode != 0) {
    uint32_t key[MP];
#pragma unroll
    for (int m = 0; m < MP; ++m) {
      key[m] = 0xFFFFFFFFu;  // padding sorts last and carries weight 0
      if (m < M) key[m] = wm_key(vals[m * stride]);
    }
    bool safe;
    pick = wm_fast_pick<MP>(key, w, total, tau, safe);
    exact = (mode == 1) && !safe;
  }
  if (in && exact) {
    unsigned long long wk[MP];
#pragma unroll
    for (int m = 0; m < MP; ++m) {
      wk[m] = ~0ull;
      if (m < M) wk[m] = ((unsigned long long)wm_key(vals[m * stride]) << 32) | (unsigned long long)(unsigned)m;
    }
    pick = (uint32_t)(wm_exact_pick<MP>(wk, M, s_a) >> 32);
  }
  return pick;
}

// ---- one row of a logistic or linear member, as se_logistic_predict scores it -------------------------------------
// The D margins m_k = Σ_j coef(k, j)·x(j) + intercept[k]: one fp64 fma per term in column order, the intercept added
// last.  MAXD >= D is the size of the caller's margin array: the loops over k unroll to it, so the margins stay in
// registers.
template <int MAXD, class Coef, class X>
__device__ __forceinline__ void lg_row_margins(int p, int D, Coef coef, X x, const double* intercept, double (&m)[MAXD]) {
#pragma unroll
  for (int k = 0; k < MAXD; ++k) m[k] = 0.0;
  for (int j = 0; j < p; ++j) {
    const double xj = x(j);
#pragma unroll
    for (int k = 0; k < MAXD; ++k)
      if (k < D) m[k] = fma(coef(k, j), xj, m[k]);
  }
#pragma unroll
  for (int k = 0; k < MAXD; ++k)
    if (k < D) m[k] += intercept[k];
}

// the first maximum of the margins (Vector.argmax) and its value *mx
template <int MAXD>
__device__ __forceinline__ int lg_row_argmax(int D, const double (&m)[MAXD], double* mx) {
  int best = 0;
  double b = m[0];
#pragma unroll
  for (int k = 1; k < MAXD; ++k)
    if (k < D && m[k] > b) b = m[k], best = k;
  *mx = b;
  return best;
}

__device__ __forceinline__ double lg_sigmoid(double m) { return 1.0 / (1.0 + exp(-m)); }

// the label: σ(m_0) > threshold for D = 1, else the first argmax `best`
__device__ __forceinline__ float lg_row_label(int D, double m0, int best, double threshold) {
  if (D == 1) return lg_sigmoid(m0) > threshold ? 1.f : 0.f;
  return (float)best;
}

// put(k, p_k) for the class probabilities: (1 − σ(m_0), σ(m_0)) for D = 1, else the softmax of the margins, where a
// maximum margin mx of +inf gives 1 to every +inf class and 0 to the others
template <int MAXD, class Put>
__device__ __forceinline__ void lg_row_probs(int D, const double (&m)[MAXD], double mx, Put put) {
  if (D == 1) {
    const double p1 = lg_sigmoid(m[0]);
    put(0, (float)(1.0 - p1));
    put(1, (float)p1);
    return;
  }
  if (mx == INFINITY) {
#pragma unroll
    for (int k = 0; k < MAXD; ++k)
      if (k < D) put(k, (m[k] == INFINITY) ? 1.f : 0.f);
    return;
  }
  double S = 0.0;
#pragma unroll
  for (int k = 0; k < MAXD; ++k)
    if (k < D) S += exp(m[k] - mx);
#pragma unroll
  for (int k = 0; k < MAXD; ++k)
    if (k < D) put(k, (float)(exp(m[k] - mx) / S));
}

}  // namespace

// Calls f(std::integral_constant<int, MAXD>()) for the margin-array size the linear scoring kernels are instantiated
// for: 1 (one margin), else the power of two from 4 to 64 that holds D margins.
template <class F>
cudaError_t with_maxd(int D, F f) {
  if (D <= 1) return f(std::integral_constant<int, 1>());
  if (D <= 4) return f(std::integral_constant<int, 4>());
  if (D <= 8) return f(std::integral_constant<int, 8>());
  if (D <= 16) return f(std::integral_constant<int, 16>());
  if (D <= 32) return f(std::integral_constant<int, 32>());
  if (D <= 64) return f(std::integral_constant<int, 64>());
  return cudaErrorInvalidValue;
}

}  // namespace se
