// se_brent.h — Brent's univariate minimiser, commons-math3 3.6.1 BrentOptimizer semantics (call site
// regression/GBMRegressor.scala:311,413-421), as ONE host/device template so that the host line search
// (se_gbm_linesearch_brent, se_brent_minimize) and the on-device line search of the squared-loss round
// (se_brent.cu, compiled with -fmad=false so that no multiply-add is contracted) execute the same IEEE operations
// in the same order and return the same iterates bit for bit.
// Golden-section fallback, parabolic interpolation when the fit lies inside the bracket and is shrinking, never
// evaluates closer than tol1 = rel*|x| + abs to a previous abscissa, stops when |x - mid| <= 2*tol1 - (hi-lo)/2;
// returns the best point evaluated.
#pragma once

#include <math.h>

#if defined(__CUDACC__) && !defined(SE_BRENT_HOST_ONLY)  // se_api.cu instantiates it with host callbacks only
#define SE_HD __host__ __device__
#else
#define SE_HD
#endif

namespace se {

constexpr int kBrentOk = 0;
constexpr int kBrentMaxEval = 1;  // MaxEval exceeded (commons-math throws TooManyEvaluationsException)

SE_HD inline bool within_one_ulp(double a, double b) {
  return a == b || (!isnan(a) && !isnan(b) && nextafter(a, b) == b);
}

// f: double -> double.  Returns kBrentOk or kBrentMaxEval; outputs are written in both cases.
template <class F>
SE_HD inline int brent_core(F f, double lo, double hi, double start, double rel, double abs_tol, int max_eval,
                            double* x_out, double* f_out, int* n_eval) {
  const double kGolden = 0x1.8722191a02d60p-2;  // 0.5 * (3 - sqrt(5))
  double left = lo < hi ? lo : hi, right = lo < hi ? hi : lo;
  double x = start, w = start, v = start;       // best, second best, previous second best
  double step = 0.0, prev_step = 0.0;           // "d" and "e" of the classic formulation
  int evals = 0;
  double fx = f(x);
  ++evals;
  double fw = fx, fv = fx;
  double bx = x, bf = fx;                       // best-of-all-evaluations bookkeeping
  double last_x = x, last_f = fx;
  bool have_two = false;
  double before_x = 0.0, before_f = 0.0;
  int status = kBrentOk;
  auto consider = [&](double cx, double cf) {
    if (!(bf <= cf)) { bx = cx; bf = cf; }
  };
  for (;;) {
    const double mid = 0.5 * (left + right);
    const double tol1 = rel * fabs(x) + abs_tol, tol2 = 2.0 * tol1;
    if (fabs(x - mid) <= tol2 - 0.5 * (right - left)) {
      if (have_two && before_f <= last_f) consider(before_x, before_f);
      else consider(last_x, last_f);
      break;
    }
    bool use_golden = true;
    double u;
    if (fabs(prev_step) > tol1) {
      double r = (x - w) * (fx - fv);
      double q = (x - v) * (fx - fw);
      double p = (x - v) * q - (x - w) * r;
      q = 2.0 * (q - r);
      if (q > 0.0) p = -p; else q = -q;
      r = prev_step;
      prev_step = step;
      if (p > q * (left - x) && p < q * (right - x) && fabs(p) < fabs(0.5 * q * r)) {
        step = p / q;
        u = x + step;
        if (u - left < tol2 || right - u < tol2) step = (x <= mid) ? tol1 : -tol1;
        use_golden = false;
      }
    }
    if (use_golden) {
      prev_step = (x < mid) ? right - x : left - x;
      step = kGolden * prev_step;
    }
    u = (fabs(step) < tol1) ? (step >= 0.0 ? x + tol1 : x - tol1) : x + step;
    if (evals >= max_eval) { status = kBrentMaxEval; break; }
    const double fu = f(u);
    ++evals;
    before_x = last_x; before_f = last_f; have_two = true;
    last_x = u; last_f = fu;
    if (before_f <= last_f) consider(before_x, before_f);
    else consider(last_x, last_f);
    if (fu <= fx) {
      if (u < x) right = x; else left = x;
      v = w; fv = fw;
      w = x; fw = fx;
      x = u; fx = fu;
    } else {
      if (u < x) left = u; else right = u;
      if (fu <= fw || within_one_ulp(w, x)) {
        v = w; fv = fw;
        w = u; fw = fu;
      } else if (fu <= fv || within_one_ulp(v, x) || within_one_ulp(v, w)) {
        v = u; fv = fu;
      }
    }
  }
  if (x_out) *x_out = bx;
  if (f_out) *f_out = bf;
  if (n_eval) *n_eval = evals;
  return status;
}

// squared-loss line-search objective from the sufficient statistics: Σ (y-F-αh)²/2 / Σw.  The division by 2Σw is a
// multiplication by its reciprocal, formed once: an fp64 division is a ~30-instruction dependent chain on the GPU and
// the objective is evaluated ~10-35 times per search by ONE thread while the whole grid waits for the step.  Host and device use this
// same struct, so their iterates stay bit-identical to each other.
struct BrentParabola {
  double s0, s1, s2, inv2ws;
  SE_HD BrentParabola(double a, double b, double c, double ws) : s0(a), s1(b), s2(c), inv2ws(1.0 / (2.0 * ws)) {}
  SE_HD double operator()(double x) const { return (s0 - 2.0 * x * s1 + x * x * s2) * inv2ws; }
};

}  // namespace se
