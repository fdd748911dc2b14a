/*
 * se_oracle.h — CPU fp64 restatement of spark-ensemble's row-parallel boosting hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load it,
 * and there only as the checker or as the timed CPU baseline.
 *
 * PARITY UNPINNED: the reference is pure Scala on Spark 3.3.1; there is no JVM in this image
 * (java/javac/scala/sbt absent) and the reference's own tests hold no golden numbers for this
 * path (SURVEY.md §4, §8c).  The oracle is pinned only against the portable *properties* the
 * reference's tests assert (finite-difference gradient check, zero-sum raw predictions, ...),
 * against an independent numpy restatement (oracle/np_oracle.py) and against closed forms.
 *
 * All citations are relative to core/src/main/scala/org/apache/spark/ml/ of the reference repository.
 * Layout convention shared with the product: per-row arrays are [dim][n] ("class-major",
 * rows contiguous); model-output matrices are [M][n] or [M][K][n].
 */
#ifndef SE_ORACLE_H
#define SE_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Loss identifiers (boosting/GBMLoss.scala:129-318). */
enum {
  ORC_SQUARED = 0,        /* SquaredLoss        :129-137 */
  ORC_ABSOLUTE = 1,       /* AbsoluteLoss       :139-143 */
  ORC_HUBER = 2,          /* HuberLoss(delta)   :168-177 */
  ORC_QUANTILE = 3,       /* QuantileLoss(q)    :179-188 */
  ORC_LOGCOSH = 4,        /* LogCoshLoss        :145-152 */
  ORC_SCALED_LOGCOSH = 5, /* ScaledLogCoshLoss(alpha) :154-166 */
  ORC_BERNOULLI = 6,      /* BernoulliLoss      :293-318 */
  ORC_EXPONENTIAL = 7,    /* ExponentialLoss    :265-291 */
  ORC_LOGLOSS = 8         /* LogLoss(K)         :196-263 */
};

/* ---- per-row loss library (scalar losses take the *encoded* label) ---- */
double orc_encode_label(int loss, double label);           /* GBMLoss.scala:125,272-273,297-298 */
double orc_loss(int loss, double param, double label, double pred);
double orc_gradient(int loss, double param, double label, double pred);
double orc_hessian(int loss, double param, double label, double pred); /* NaN if loss has none */
int orc_has_hessian(int loss);
/* LogLoss(K): label is the class index, pred[K] strided by `stride` doubles. */
double orc_logloss_loss(int K, int label, const double* pred, int64_t stride);
void orc_logloss_gradient(int K, int label, const double* pred, int64_t stride, double* out);
void orc_logloss_hessian(int K, int label, const double* pred, int64_t stride, double* out);

/* ---- GBMLossAggregator.add + RDDLossFunction (GBMLoss.scala:50-74) ----
 * y[n] raw labels, w[n] or NULL (=1), F[dim][n], h[dim][n], alpha[dim].
 * out_loss = lossSum/weightSum (lossSum accumulated `dim` times per row — reference quirk),
 * out_grad[dim] = gradSum/weightSum. Instance weights enter weightSum only. */
void orc_linesearch_eval(int loss, double param, int dim, int64_t n, const double* y,
                         const double* w, const double* F, const double* h,
                         const double* alpha, double* out_loss, double* out_grad);

/* ---- pseudo-residuals (regression/GBMRegressor.scala:368-385, classification/GBMClassifier.scala:337-375)
 * newton != 0 requires a hessian. r[dim][n]; wout[dim][n] (may be NULL when newton == 0);
 * sum_hess[dim] (newton only). */
void orc_pseudo_residuals(int loss, double param, int dim, int64_t n, const double* y,
                          const double* w, const double* F, int newton, double* r,
                          double* wout, double* sum_hess);

/* F_j += step_j * h_j (GBMRegressor.scala:437-441, GBMClassifier.scala:437-448). */
void orc_update(int dim, int64_t n, double* F, const double* h, const double* step);

/* mean over rows of loss(encodeLabel(y), F) (GBMRegressor.scala:330-335,451-456; GBMClassifier.scala:315-320,465-470) */
double orc_mean_loss(int loss, double param, int dim, int64_t n, const double* y, const double* F);

/* ---- commons-math3 3.6.1 BrentOptimizer restated (call site GBMRegressor.scala:311,413-421) ----
 * Minimises f on [lo,hi] from `start` with rel/abs thresholds; returns the abscissa of the best
 * evaluated point. *status: 0 ok, 1 = MaxEval exceeded (the reference would throw). */
typedef double (*orc_fn1)(double x, void* user);
double orc_brent_minimize(orc_fn1 f, void* user, double lo, double hi, double start, double rel,
                          double abs_tol, int max_eval, int* n_eval, int* status);

/* ---- BoostingClassifier weight update (classification/BoostingClassifier.scala:168-269) ---- */
double orc_sum(int64_t n, const double* w);                                       /* :175,269 */
/* SAMME.R :198-230. P[K][n] class probabilities. w_out[n]. returns via pointers the
 * estimatorError (Σ w/sumW·1[argmax p != y]) and Σ w_out. */
void orc_samme_r_update(int K, int64_t n, const double* y, const double* w, double sum_w,
                        const double* P, double* w_out, double* est_err, double* new_sum);
/* SAMME :231-260. pred[n] predicted labels. beta/est_weight are outputs of the error pass. */
double orc_samme_error(int64_t n, const double* y, const double* w, double sum_w,
                       const double* pred);                                         /* :232-242 */
void orc_samme_update(int64_t n, const double* y, const double* w, double sum_w,
                      const double* pred, double beta, double* w_out, double* new_sum); /* :254-258 */

/* ---- ensemble Model prediction aggregation (the per-row bodies of predict/predictRaw) ---- */
/* GBMRegressionModel.predict regression/GBMRegressor.scala:531-539: out = init + Σ_m a_m·P[m] */
void orc_agg_weighted_sum(int M, int64_t n, const double* P, const double* a, double init,
                          double* out);
/* BaggingRegressionModel.predict regression/BaggingRegressor.scala:221-228: (Σ P[m]) / M */
void orc_agg_mean(int M, int64_t n, const double* P, double* out);
/* GBMClassificationModel.predictRaw classification/GBMClassifier.scala:567-589.
 * P[M][dim][n], a[M][dim], init[dim]; numClasses==2&&dim==1 -> raw[2][n] = (-res,res) else raw[dim][n]. */
void orc_agg_gbm_classifier_raw(int M, int dim, int num_classes, int64_t n, const double* P,
                                const double* a, const double* init, double* raw);
/* GBMClassificationLoss.raw2probabilityInPlace (GBMLoss.scala:258-261,284-289,311-316); raw[C][n] -> prob[C][n] */
void orc_gbm_raw2prob(int loss, int num_classes, int64_t n, const double* raw, double* prob);
/* BaggingClassificationModel.predictRaw/raw2probability classification/BaggingClassifier.scala:260-287.
 * soft: P[M][K][n] probabilities; hard: votes[M][n] predicted labels. raw[K][n]; prob = raw/M. */
void orc_agg_bagging_soft(int M, int K, int64_t n, const double* P, double* raw, double* prob);
void orc_agg_bagging_hard(int M, int K, int64_t n, const double* votes, double* raw, double* prob);
/* BoostingClassificationModel.predictRawReal/Discrete + raw2probability classification/BoostingClassifier.scala:342-382 */
void orc_agg_boosting_real(int M, int K, int64_t n, const double* P, double* raw, double* prob);
void orc_agg_boosting_discrete(int M, int K, int64_t n, const double* votes, const double* a,
                               double* raw, double* prob);
/* ---- BoostingRegressor (AdaBoost.R2) regression/BoostingRegressor.scala:97-106,169-171,225-263 ----
 * loss_type: 0 exponential (1 - exp(-e)), 1 linear (e), 2 squared (e^2). */
double orc_r2_max_error(int64_t n, const double* y, const double* pred);                  /* :231-234 */
/* losses_i = loss(err_i / maxError) (loss(err_i) when maxError == 0) ; returns Σ (w_i/sum_w)·loss_i :236-249 */
double orc_r2_estimator_error(int loss_type, int64_t n, const double* y, const double* pred,
                              const double* w, double sum_w, double max_error);
/* w'_i = (w_i/sum_w)·beta^(1 - loss_i) :256-260 ; *new_sum = Σ w' :263 */
void orc_r2_update(int loss_type, int64_t n, const double* y, const double* pred, const double* w,
                   double sum_w, double max_error, double beta, double* w_out, double* new_sum);
/* BoostingRegressionModel.predict :333-347 + ensemble/Utils.scala:26-40. P[M][n], a[M]. */
void orc_agg_weighted_median(int M, int64_t n, const double* P, const double* a, double* out);
void orc_agg_weighted_mean(int M, int64_t n, const double* P, const double* a, double* out);

/* Spark ClassificationModel.raw2prediction = argmax (first maximum). raw[C][n] -> pred[n] */
void orc_argmax(int C, int64_t n, const double* raw, double* pred);

/* ---- audit of a fitted tree over row chunks (oracle/tree_audit.py) ----
 * orc_ranks: out[i] = #{cand < x[i]} (the rank of x[i] among ncand sorted fp32 candidates), 255 for NaN.
 * orc_tree_walk: leaf[i] = the node where row i stops walking a tree over the ranks R[S][m] (left when rank <= bin).
 * orc_tree_hist: adds the rows [0, m) of a chunk to the fp64 statistics of every node of a node list (node 0 the
 * root; node v > 0 holds the rows of parent[v] < v whose rank in column col[v] is <= bin[v] when left[v], > bin[v]
 * otherwise; a row may reach several children of one node).  Only rows with c > 0 count (c NULL: all, as 1).  Per
 * row, K == 0 (regression, lab = label): (c, c·w, c·w·lab, c·w·lab²); K >= 2 (lab = class index): (c, c·w in class
 * lab), ns = 4 or K + 1 values.  totals[n_nodes][ns + 2] gets the node's sums, then Σ c·w·|lab| (regression) and its
 * row count; hist[h][S][256][ns] (h = hist_of[v] >= 0) the sums per column and rank. */
void orc_ranks(int64_t m, const float* x, int ncand, const float* cand, uint8_t* out);
void orc_tree_walk(int64_t m, const uint8_t* R, const int32_t* feature, const int32_t* bin, const int32_t* left,
                   const int32_t* right, int32_t* leaf);
void orc_tree_hist(int64_t m, int S, const uint8_t* R, int K, const double* lab, const double* w, const double* c,
                   int n_nodes, const int32_t* parent, const int32_t* col, const int32_t* bin, const int32_t* left,
                   const int32_t* hist_of, double* totals, double* hist);

/* number of OpenMP threads the library will use (1 when built without -fopenmp) */
int orc_num_threads(void);
void orc_set_num_threads(int t);

#ifdef __cplusplus
}
#endif
#endif
