/*
 * se_oracle.c — CPU fp64 restatement of spark-ensemble's row-parallel boosting hot path.
 * TEST INFRASTRUCTURE ONLY (see se_oracle.h).  PARITY UNPINNED (no JVM here, no golden vectors
 * in the reference's tests); pinned against portable properties + an independent numpy restatement.
 *
 * Citations: paths relative to core/src/main/scala/org/apache/spark/ml/ of the reference repository.
 * Spark-internal helpers (softmax, log1pExp, EPSILON: org.apache.spark.ml.impl.Utils, Spark 3.3.1,
 * not vendored) are restated from their published definitions.
 */
#include "se_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define ORC_MAX_DIM 4096 /* stack arrays per row: LogLoss class counts used by the tests stay well below */

/* Spark ml.impl.Utils.EPSILON: smallest eps with 1 + eps/2 == 1  (= 2^-52). */
static const double SPARK_EPSILON = 2.220446049250313e-16;

int orc_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
void orc_set_num_threads(int t) {
#ifdef _OPENMP
  if (t > 0) omp_set_num_threads(t);
#else
  (void)t;
#endif
}

/* java.lang.Math.signum */
static inline double jsignum(double x) { return (x > 0.0) ? 1.0 : ((x < 0.0) ? -1.0 : x); }

/* Spark ml.impl.Utils.log1pExp */
static inline double log1p_exp(double x) { return (x > 0.0) ? x + log1p(exp(-x)) : log1p(exp(x)); }

/* ------------------------------------------------------------------ loss library */

double orc_encode_label(int loss, double label) {
  /* GBMLoss.scala:125 (regression: identity), :272-273 and :297-298 (2*label - 1) */
  if (loss == ORC_BERNOULLI || loss == ORC_EXPONENTIAL) return 2.0 * label - 1.0;
  return label;
}

int orc_has_hessian(int loss) {
  switch (loss) {
    case ORC_SQUARED: case ORC_LOGCOSH: case ORC_SCALED_LOGCOSH:
    case ORC_BERNOULLI: case ORC_EXPONENTIAL: case ORC_LOGLOSS: return 1;
    default: return 0;
  }
}

double orc_loss(int loss, double param, double y, double p) {
  switch (loss) {
    case ORC_SQUARED: /* :130-131 */
      return pow(y - p, 2.0) / 2.0;
    case ORC_ABSOLUTE: /* :140 */
      return fabs(y - p);
    case ORC_HUBER: /* :169-171 */
      if (fabs(y - p) <= param) return pow(y - p, 2.0) / 2.0;
      return param * (fabs(y - p) - param / 2.0);
    case ORC_QUANTILE: /* :181-183 */
      if (y > p) return param * (y - p);
      return (param - 1.0) * (y - p);
    case ORC_LOGCOSH: /* :146 */
      return log(cosh(y - p));
    case ORC_SCALED_LOGCOSH: /* :155-157 */
      if (y > p) return param * log(cosh(y - p));
      return (1.0 - param) * log(cosh(y - p));
    case ORC_BERNOULLI: /* :300-301 */
      return log1p_exp(-2.0 * y * p);
    case ORC_EXPONENTIAL: /* :275-276 */
      return exp(-y * p);
    default: return NAN;
  }
}

double orc_gradient(int loss, double param, double y, double p) {
  switch (loss) {
    case ORC_SQUARED: /* :133 */
      return -(y - p);
    case ORC_ABSOLUTE: /* :142 */
      return -jsignum(y - p);
    case ORC_HUBER: /* :173-175 */
      if (fabs(y - p) <= param) return -(y - p);
      return -param * jsignum(y - p);
    case ORC_QUANTILE: /* :185-186 */
      return (y > p) ? -param : (1.0 - param);
    case ORC_LOGCOSH: /* :148 */
      return -tanh(y - p);
    case ORC_SCALED_LOGCOSH: /* :159-161 */
      if (y > p) return param * -tanh(y - p);
      return (1.0 - param) * -tanh(y - p);
    case ORC_BERNOULLI: /* :303-304 */
      return -2.0 * y / (1.0 + exp(2.0 * y * p));
    case ORC_EXPONENTIAL: /* :278-279 */
      return -y * exp(-y * p);
    default: return NAN;
  }
}

double orc_hessian(int loss, double param, double y, double p) {
  switch (loss) {
    case ORC_SQUARED: /* :135 */
      return 1.0;
    case ORC_LOGCOSH: /* :150-151 */
      return 1.0 / pow(cosh(y - p), 2.0);
    case ORC_SCALED_LOGCOSH: /* :163-165 */
      if (y > p) return param * (1.0 / pow(cosh(y - p), 2.0));
      return (1.0 - param) * (1.0 / pow(cosh(y - p), 2.0));
    case ORC_BERNOULLI: /* :306-309 */
      return (4.0 * exp(2.0 * p * y) * pow(y, 2.0)) / pow(1.0 + exp(2.0 * p * y), 2.0);
    case ORC_EXPONENTIAL: /* :281-282 */
      return pow(y, 2.0) * exp(-y * p);
    default: return NAN;
  }
}

/* LogLoss(K) :206-221 — log Σ exp(p_k) WITHOUT max subtraction (reference quirk 7). */
static inline double logloss_lse(int K, const double* pred, int64_t stride) {
  double sum = 0.0;
  for (int k = 0; k < K; ++k) sum += exp(pred[k * stride]);
  return log(sum);
}

double orc_logloss_loss(int K, int label, const double* pred, int64_t stride) {
  const double lse = logloss_lse(K, pred, stride);
  double res = 0.0;
  for (int k = 0; k < K; ++k) {
    const double yk = (k == label) ? 1.0 : 0.0;
    res += -yk * (pred[k * stride] - lse);
  }
  return res;
}

void orc_logloss_gradient(int K, int label, const double* pred, int64_t stride, double* out) {
  /* :223-238 */
  const double lse = logloss_lse(K, pred, stride);
  for (int k = 0; k < K; ++k) {
    const double yk = (k == label) ? 1.0 : 0.0;
    out[k] = exp(pred[k * stride] - lse) - yk;
  }
}

void orc_logloss_hessian(int K, int label, const double* pred, int64_t stride, double* out) {
  /* :240-256 */
  (void)label;
  const double lse = logloss_lse(K, pred, stride);
  for (int k = 0; k < K; ++k) {
    const double s = exp(pred[k * stride] - lse);
    out[k] = s * (1.0 - s);
  }
}

/* ------------------------------------------------------------------ aggregator / line search */

void orc_linesearch_eval(int loss, double param, int dim, int64_t n, const double* y,
                         const double* w, const double* F, const double* h,
                         const double* alpha, double* out_loss, double* out_grad) {
  double loss_sum = 0.0, weight_sum = 0.0;
  double grad_sum[ORC_MAX_DIM];
  for (int j = 0; j < dim; ++j) grad_sum[j] = 0.0;

  if (loss != ORC_LOGLOSS) {
    /* dim == 1 (GBMScalarLoss :107-122) */
    double g0 = 0.0;
    const double a0 = alpha[0];
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : loss_sum, weight_sum, g0) schedule(static)
#endif
    for (int64_t i = 0; i < n; ++i) {
      const double label = orc_encode_label(loss, y[i]);
      const double p = F[i] + a0 * h[i];                 /* :56-59 */
      loss_sum += orc_loss(loss, param, label, p);       /* :60-64, dim == 1 */
      weight_sum += w ? w[i] : 1.0;                      /* :65 */
      g0 += h[i] * orc_gradient(loss, param, label, p);  /* :66-72 */
    }
    grad_sum[0] = g0;
  } else {
    const int K = dim;
#ifdef _OPENMP
#pragma omp parallel
#endif
    {
      double gl[ORC_MAX_DIM], arr[ORC_MAX_DIM], g[ORC_MAX_DIM];
      double ls = 0.0, ws = 0.0;
      for (int j = 0; j < K; ++j) gl[j] = 0.0;
#ifdef _OPENMP
#pragma omp for schedule(static) nowait
#endif
      for (int64_t i = 0; i < n; ++i) {
        for (int j = 0; j < K; ++j) arr[j] = F[j * n + i] + alpha[j] * h[j * n + i];
        const int label = (int)y[i];
        const double l = orc_logloss_loss(K, label, arr, 1);
        for (int j = 0; j < K; ++j) ls += l;             /* loss added dim times :60-64 */
        ws += w ? w[i] : 1.0;
        orc_logloss_gradient(K, label, arr, 1, g);
        for (int j = 0; j < K; ++j) gl[j] += h[j * n + i] * g[j];
      }
#ifdef _OPENMP
#pragma omp critical
#endif
      {
        loss_sum += ls;
        weight_sum += ws;
        for (int j = 0; j < K; ++j) grad_sum[j] += gl[j];
      }
    }
  }
  /* DifferentiableLossAggregator.loss / .gradient: divide by weightSum */
  *out_loss = loss_sum / weight_sum;
  if (out_grad)
    for (int j = 0; j < dim; ++j) out_grad[j] = grad_sum[j] / weight_sum;
}

/* ------------------------------------------------------------------ pseudo-residuals */

void orc_pseudo_residuals(int loss, double param, int dim, int64_t n, const double* y,
                          const double* w, const double* F, int newton, double* r,
                          double* wout, double* sum_hess) {
  if (loss != ORC_LOGLOSS) {
    if (newton) {
      /* GBMRegressor.scala:369-380 (and GBMClassifier.scala:338-368 with dim == 1) */
      double S = 0.0;
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : S) schedule(static)
#endif
      for (int64_t i = 0; i < n; ++i) {
        const double label = orc_encode_label(loss, y[i]);
        S += fmax(orc_hessian(loss, param, label, F[i]), 1e-2);
      }
      if (sum_hess) sum_hess[0] = S;
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
      for (int64_t i = 0; i < n; ++i) {
        const double label = orc_encode_label(loss, y[i]);
        const double hs = fmax(orc_hessian(loss, param, label, F[i]), 1e-2);
        const double ng = -orc_gradient(loss, param, label, F[i]);
        r[i] = ng / hs;
        wout[i] = 1.0 / 2.0 * hs / S * (w ? w[i] : 1.0);
      }
    } else {
      /* GBMRegressor.scala:381-384 ; GBMClassifier.scala:369-374 */
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
      for (int64_t i = 0; i < n; ++i) {
        const double label = orc_encode_label(loss, y[i]);
        r[i] = -orc_gradient(loss, param, label, F[i]);
        if (wout) wout[i] = w ? w[i] : 1.0;
      }
    }
    return;
  }
  const int K = dim;
  if (newton) {
    double S[ORC_MAX_DIM];
    for (int j = 0; j < K; ++j) S[j] = 0.0;
    double hs[ORC_MAX_DIM];
    for (int64_t i = 0; i < n; ++i) { /* GBMClassifier.scala:339-355 */
      orc_logloss_hessian(K, (int)y[i], F + i, n, hs);
      for (int j = 0; j < K; ++j) S[j] += fmax(hs[j], 1e-2);
    }
    if (sum_hess) memcpy(sum_hess, S, sizeof(double) * (size_t)K);
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
    for (int64_t i = 0; i < n; ++i) { /* :356-368 */
      double hh[ORC_MAX_DIM], g[ORC_MAX_DIM];
      orc_logloss_hessian(K, (int)y[i], F + i, n, hh);
      orc_logloss_gradient(K, (int)y[i], F + i, n, g);
      for (int j = 0; j < K; ++j) {
        const double hj = fmax(hh[j], 1e-2);
        r[j * n + i] = -g[j] / hj;
        wout[j * n + i] = 1.0 / 2.0 * hj / S[j] * (w ? w[i] : 1.0);
      }
    }
  } else {
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
    for (int64_t i = 0; i < n; ++i) { /* :369-374 */
      double g[ORC_MAX_DIM];
      orc_logloss_gradient(K, (int)y[i], F + i, n, g);
      for (int j = 0; j < K; ++j) {
        r[j * n + i] = -g[j];
        if (wout) wout[j * n + i] = w ? w[i] : 1.0;
      }
    }
  }
}

void orc_update(int dim, int64_t n, double* F, const double* h, const double* step) {
  for (int j = 0; j < dim; ++j) {
    const double s = step[j];
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
    for (int64_t i = 0; i < n; ++i) F[j * n + i] = F[j * n + i] + s * h[j * n + i];
  }
}

double orc_mean_loss(int loss, double param, int dim, int64_t n, const double* y,
                     const double* F) {
  double s = 0.0;
  if (loss != ORC_LOGLOSS) {
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : s) schedule(static)
#endif
    for (int64_t i = 0; i < n; ++i)
      s += orc_loss(loss, param, orc_encode_label(loss, y[i]), F[i]);
  } else {
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : s) schedule(static)
#endif
    for (int64_t i = 0; i < n; ++i) s += orc_logloss_loss(dim, (int)y[i], F + i, n);
  }
  return s / (double)n;
}

/* ------------------------------------------------------------------ Brent (commons-math3 3.6.1)
 * Restated from the published algorithm of org.apache.commons.math3.optim.univariate.BrentOptimizer
 * (doOptimize): golden-section constant 0.5*(3-sqrt 5); tol1 = rel*|x| + abs; stop when
 * |x - m| <= 2*tol1 - (b-a)/2; parabolic step accepted iff p in (q(a-x), q(b-x)) and |p| < |q*r/2|;
 * minimal step tol1; the returned point is the best of all evaluated points. */

static int ulp_equal(double a, double b) {
  /* commons-math3 Precision.equals(x, y): equal within 1 ulp */
  if (a == b) return 1;
  if (isnan(a) || isnan(b)) return 0;
  return nextafter(a, b) == b;
}

double orc_brent_minimize(orc_fn1 f, void* user, double lo, double hi, double start, double rel,
                          double abs_tol, int max_eval, int* n_eval, int* status) {
  const double golden = 0.5 * (3.0 - sqrt(5.0));
  double a = (lo < hi) ? lo : hi, b = (lo < hi) ? hi : lo;
  double x = start, v = start, wv = start, d = 0.0, e = 0.0;
  int evals = 0;
  if (status) *status = 0;
  double fx = f(x, user); ++evals;
  double fv = fx, fw = fx;
  double best_x = x, best_f = fx;
  double prev_x = 0.0, prev_f = 0.0, cur_x = x, cur_f = fx;
  int have_prev = 0;

  for (;;) {
    const double m = 0.5 * (a + b);
    const double tol1 = rel * fabs(x) + abs_tol;
    const double tol2 = 2.0 * tol1;
    if (fabs(x - m) <= tol2 - 0.5 * (b - a)) {
      /* best(best, best(previous, current)) */
      double cand_x = cur_x, cand_f = cur_f;
      if (have_prev && prev_f <= cur_f) { cand_x = prev_x; cand_f = prev_f; }
      if (!(best_f <= cand_f)) { best_x = cand_x; best_f = cand_f; }
      break;
    }
    double p = 0.0, q = 0.0, r = 0.0, u = 0.0;
    int golden_step = 1;
    if (fabs(e) > tol1) {
      r = (x - wv) * (fx - fv);
      q = (x - v) * (fx - fw);
      p = (x - v) * q - (x - wv) * r;
      q = 2.0 * (q - r);
      if (q > 0.0) p = -p; else q = -q;
      r = e;
      e = d;
      if (p > q * (a - x) && p < q * (b - x) && fabs(p) < fabs(0.5 * q * r)) {
        d = p / q;
        u = x + d;
        if (u - a < tol2 || b - u < tol2) d = (x <= m) ? tol1 : -tol1;
        golden_step = 0;
      }
    }
    if (golden_step) {
      e = (x < m) ? b - x : a - x;
      d = golden * e;
    }
    if (fabs(d) < tol1) u = (d >= 0.0) ? x + tol1 : x - tol1;
    else u = x + d;

    if (evals >= max_eval) { /* MaxEval(maxIter): TooManyEvaluationsException in the reference */
      if (status) *status = 1;
      break;
    }
    const double fu = f(u, user); ++evals;

    prev_x = cur_x; prev_f = cur_f; have_prev = 1;
    cur_x = u; cur_f = fu;
    {
      double cand_x = cur_x, cand_f = cur_f;
      if (prev_f <= cur_f) { cand_x = prev_x; cand_f = prev_f; }
      if (!(best_f <= cand_f)) { best_x = cand_x; best_f = cand_f; }
    }

    if (fu <= fx) {
      if (u < x) b = x; else a = x;
      v = wv; fv = fw;
      wv = x; fw = fx;
      x = u; fx = fu;
    } else {
      if (u < x) a = u; else b = u;
      if (fu <= fw || ulp_equal(wv, x)) {
        v = wv; fv = fw;
        wv = u; fw = fu;
      } else if (fu <= fv || ulp_equal(v, x) || ulp_equal(v, wv)) {
        v = u; fv = fu;
      }
    }
  }
  if (n_eval) *n_eval = evals;
  return best_x;
}

/* ------------------------------------------------------------------ BoostingClassifier */

double orc_sum(int64_t n, const double* w) {
  double s = 0.0;
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : s) schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) s += w[i];
  return s;
}

void orc_samme_r_update(int K, int64_t n, const double* y, const double* w, double sum_w,
                        const double* P, double* w_out, double* est_err, double* new_sum) {
  double err = 0.0, ns = 0.0;
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : err, ns) schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) {
    const double wn = w[i] / sum_w; /* BoostingClassifier.scala:184-187 */
    /* probability.argmax — first maximum (:205) */
    int am = 0;
    double best = P[i];
    for (int k = 1; k < K; ++k)
      if (P[(int64_t)k * n + i] > best) { best = P[(int64_t)k * n + i]; am = k; }
    err += wn * ((y[i] != (double)am) ? 1.0 : 0.0); /* :133,202-209 */
    double loss = 0.0;                              /* :218-224 */
    for (int k = 0; k < K; ++k) {
      const double code = (y[i] == (double)k) ? 1.0 : -1.0 / (K - 1.0);
      loss += code * log(fmax(P[(int64_t)k * n + i], SPARK_EPSILON));
    }
    const double wo = wn * exp(-((K - 1.0) / K) * loss); /* :226 */
    w_out[i] = wo;
    ns += wo; /* :269 */
  }
  *est_err = err;
  *new_sum = ns;
}

double orc_samme_error(int64_t n, const double* y, const double* w, double sum_w,
                       const double* pred) {
  double err = 0.0;
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : err) schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i)
    err += (w[i] / sum_w) * ((y[i] != pred[i]) ? 1.0 : 0.0);
  return err;
}

void orc_samme_update(int64_t n, const double* y, const double* w, double sum_w,
                      const double* pred, double beta, double* w_out, double* new_sum) {
  double ns = 0.0;
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : ns) schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) {
    const double e = (y[i] != pred[i]) ? 1.0 : 0.0;
    const double wo = (w[i] / sum_w) * pow(1.0 / beta, e); /* :254-258 */
    w_out[i] = wo;
    ns += wo;
  }
  *new_sum = ns;
}

/* ------------------------------------------------------------------ prediction aggregation */

void orc_agg_weighted_sum(int M, int64_t n, const double* P, const double* a, double init,
                          double* out) {
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) {
    double sum = init;
    for (int m = 0; m < M; ++m) sum += P[(int64_t)m * n + i] * a[m];
    out[i] = sum;
  }
}

void orc_agg_mean(int M, int64_t n, const double* P, double* out) {
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) {
    double sum = 0.0;
    for (int m = 0; m < M; ++m) sum += P[(int64_t)m * n + i];
    out[i] = sum / M;
  }
}

void orc_agg_gbm_classifier_raw(int M, int dim, int num_classes, int64_t n, const double* P,
                                const double* a, const double* init, double* raw) {
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) {
    double res[ORC_MAX_DIM];
    for (int j = 0; j < dim; ++j) res[j] = init[j];
    for (int m = 0; m < M; ++m)
      for (int j = 0; j < dim; ++j)
        res[j] += P[((int64_t)m * dim + j) * n + i] * a[m * dim + j];
    if (dim == 1 && num_classes == 2) { /* GBMClassifier.scala:583-584 */
      raw[i] = -res[0];
      raw[n + i] = res[0];
    } else {
      for (int j = 0; j < dim; ++j) raw[(int64_t)j * n + i] = res[j];
    }
  }
}

/* Spark ml.impl.Utils.softmax (in place): subtract max, exponentiate, normalise. */
static void spark_softmax(int K, double* v) {
  double mx = -INFINITY;
  for (int k = 0; k < K; ++k) if (v[k] > mx) mx = v[k];
  double sum = 0.0;
  for (int k = 0; k < K; ++k) { v[k] = exp(v[k] - mx); sum += v[k]; }
  for (int k = 0; k < K; ++k) v[k] /= sum;
}

void orc_gbm_raw2prob(int loss, int num_classes, int64_t n, const double* raw, double* prob) {
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) {
    if (loss == ORC_LOGLOSS) { /* GBMLoss.scala:258-261 */
      double v[ORC_MAX_DIM];
      for (int k = 0; k < num_classes; ++k) v[k] = raw[(int64_t)k * n + i];
      spark_softmax(num_classes, v);
      for (int k = 0; k < num_classes; ++k) prob[(int64_t)k * n + i] = v[k];
    } else if (loss == ORC_EXPONENTIAL) { /* :284-289 (raw(0) = -F) */
      const double p1 = 1.0 / (1.0 + exp(-2.0 * raw[i]));
      prob[n + i] = p1;
      prob[i] = 1.0 - p1;
    } else { /* BernoulliLoss :311-316 */
      const double p1 = 1.0 / (1.0 + exp(raw[i]));
      prob[n + i] = p1;
      prob[i] = 1.0 - p1;
    }
  }
}

void orc_agg_bagging_soft(int M, int K, int64_t n, const double* P, double* raw, double* prob) {
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i)
    for (int k = 0; k < K; ++k) {
      double s = 0.0;
      for (int m = 0; m < M; ++m) s += 1.0 * P[((int64_t)m * K + k) * n + i]; /* BLAS.axpy(1.0, ...) :279 */
      raw[(int64_t)k * n + i] = s;
      if (prob) prob[(int64_t)k * n + i] = s * (1.0 / (double)M); /* BLAS.scal(1/numModels) :285-287 */
    }
}

void orc_agg_bagging_hard(int M, int K, int64_t n, const double* votes, double* raw,
                          double* prob) {
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) {
    double cnt[ORC_MAX_DIM];
    for (int k = 0; k < K; ++k) cnt[k] = 0.0;
    for (int m = 0; m < M; ++m) cnt[(int)votes[(int64_t)m * n + i]] += 1.0; /* :271-275 */
    for (int k = 0; k < K; ++k) {
      raw[(int64_t)k * n + i] = cnt[k];
      if (prob) prob[(int64_t)k * n + i] = cnt[k] * (1.0 / (double)M);
    }
  }
}

void orc_agg_boosting_real(int M, int K, int64_t n, const double* P, double* raw, double* prob) {
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) {
    double res[ORC_MAX_DIM], lp[ORC_MAX_DIM];
    for (int k = 0; k < K; ++k) res[k] = 0.0;
    for (int m = 0; m < M; ++m) { /* BoostingClassifier.scala:348-364 */
      double sum_lp = 0.0;
      for (int k = 0; k < K; ++k) {
        lp[k] = log(fmax(P[((int64_t)m * K + k) * n + i], SPARK_EPSILON));
        sum_lp += lp[k];
      }
      for (int k = 0; k < K; ++k)
        res[k] += (double)(K - 1) * (lp[k] - (1.0 / K) * sum_lp); /* axpy(numClasses-1, decisions, res) */
    }
    for (int k = 0; k < K; ++k) raw[(int64_t)k * n + i] = res[k];
    if (prob) { /* :342-346 */
      for (int k = 0; k < K; ++k) res[k] *= 1.0 / (K - 1.0);
      spark_softmax(K, res);
      for (int k = 0; k < K; ++k) prob[(int64_t)k * n + i] = res[k];
    }
  }
}

void orc_agg_boosting_discrete(int M, int K, int64_t n, const double* votes, const double* a,
                               double* raw, double* prob) {
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) {
    double res[ORC_MAX_DIM];
    for (int k = 0; k < K; ++k) res[k] = 0.0;
    for (int m = 0; m < M; ++m) { /* :366-382 */
      const int pred = (int)votes[(int64_t)m * n + i];
      const double wt = a[m];
      for (int c = 0; c < K; ++c) {
        if (pred == c) res[c] += wt;
        else res[c] -= 1.0 / (K - 1) * wt;
      }
    }
    for (int k = 0; k < K; ++k) raw[(int64_t)k * n + i] = res[k];
    if (prob) {
      for (int k = 0; k < K; ++k) res[k] *= 1.0 / (K - 1.0);
      spark_softmax(K, res);
      for (int k = 0; k < K; ++k) prob[(int64_t)k * n + i] = res[k];
    }
  }
}

/* ------------------------------------------------------------------ BoostingRegressor (AdaBoost.R2) */

static inline double r2_loss(int loss_type, double e) {
  /* regression/BoostingRegressor.scala:97-106 */
  if (loss_type == 0) return 1.0 - exp(-e);
  if (loss_type == 1) return e;
  return pow(e, 2.0);
}

double orc_r2_max_error(int64_t n, const double* y, const double* pred) {
  double m = -INFINITY;
  for (int64_t i = 0; i < n; ++i) {
    const double e = fabs(y[i] - pred[i]); /* :169 */
    if (e > m) m = e;                      /* treeReduce(_ max _) :234 */
  }
  return m;
}

double orc_r2_estimator_error(int loss_type, int64_t n, const double* y, const double* pred,
                              const double* w, double sum_w, double max_error) {
  double acc = 0.0;
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : acc) schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) {
    const double e = fabs(y[i] - pred[i]);
    const double l = (max_error == 0.0) ? r2_loss(loss_type, e) : r2_loss(loss_type, e / max_error); /* :236-242 */
    acc += (w[i] / sum_w) * l;                                                                          /* :244-249 */
  }
  return acc;
}

void orc_r2_update(int loss_type, int64_t n, const double* y, const double* pred, const double* w,
                   double sum_w, double max_error, double beta, double* w_out, double* new_sum) {
  double ns = 0.0;
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : ns) schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) {
    const double e = fabs(y[i] - pred[i]);
    const double l = (max_error == 0.0) ? r2_loss(loss_type, e) : r2_loss(loss_type, e / max_error);
    const double wo = (w[i] / sum_w) * pow(beta, 1.0 - l); /* :256-260 */
    w_out[i] = wo;
    ns += wo;
  }
  *new_sum = ns;
}

void orc_agg_weighted_median(int M, int64_t n, const double* P, const double* a, double* out) {
  /* ensemble/Utils.scala:26-40: stable sort by value, cumulative weights, first index with cusum >= half */
  int* idx = (int*)malloc(sizeof(int) * (size_t)M);
  for (int64_t i = 0; i < n; ++i) {
    for (int m = 0; m < M; ++m) idx[m] = m;
    for (int m = 1; m < M; ++m) { /* stable insertion sort */
      const int v = idx[m];
      int j = m - 1;
      while (j >= 0 && P[(int64_t)idx[j] * n + i] > P[(int64_t)v * n + i]) { idx[j + 1] = idx[j]; --j; }
      idx[j + 1] = v;
    }
    double total = 0.0;
    for (int m = 0; m < M; ++m) total += a[idx[m]];
    double cum = 0.0;
    int pick = M - 1;
    for (int m = 0; m < M; ++m) {
      cum += a[idx[m]];
      if (cum >= 0.5 * total) { pick = m; break; }
    }
    out[i] = P[(int64_t)idx[pick] * n + i];
  }
  free(idx);
}

void orc_agg_weighted_mean(int M, int64_t n, const double* P, const double* a, double* out) {
  double sw = 0.0;
  for (int m = 0; m < M; ++m) sw += a[m];
  for (int64_t i = 0; i < n; ++i) {
    double dot = 0.0;
    for (int m = 0; m < M; ++m) dot += P[(int64_t)m * n + i] * a[m];
    out[i] = dot / sw; /* BLAS.dot(...) / sumWeights :340-342 */
  }
}

void orc_argmax(int C, int64_t n, const double* raw, double* pred) {
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) {
    int am = 0;
    double best = raw[i];
    for (int k = 1; k < C; ++k)
      if (raw[(int64_t)k * n + i] > best) { best = raw[(int64_t)k * n + i]; am = k; }
    pred[i] = (double)am;
  }
}
