// se_api_boost.cu — host side of Spark's Bernoulli sampler, the boosting weight updates (SAMME, SAMME.R, AdaBoost.R2)
// and the aggregation of member predictions.
#include "se_ctx.h"

using namespace se;
using namespace se_host;

// ---- Spark's Bernoulli row sampler, restated (host only) -----------------------------------------
// RDD.sample(withReplacement = false, fraction, seed) as the reference calls it (regression/GBMRegressor.scala:357-359,
// classification/GBMClassifier.scala:329-331) for data that sits in ONE partition:
//   PartitionwiseSampledRDD: partition p gets the seed  new java.util.Random(seed).nextLong()  (p-th call);
//   BernoulliSampler.setSeed -> XORShiftRandom(seed'): state = hashSeed(seed') (MurmurHash3 of the 8 big-endian bytes);
//   sample(): fraction <= 0.4 -> GapSampling (skip floor(log(max(u, 5e-11)) / log1p(-fraction)) rows between picks),
//             else keep the row iff nextDouble() <= fraction.
// java.util.Random is specified by the Java SE API documentation; MurmurHash3 and XORShift are pinned by published
// vectors / their definitions (tests/test_thirdparty_golden.py); the sampler logic itself is restated from the Spark
// 3.3.1 sources (org/apache/spark/util/random/RandomSampler.scala, rdd/PartitionwiseSampledRDD.scala) and is UNPINNED
// (no Spark in this image).  A Spark host uploads the multiplicities Spark itself drew (GBMRegressorNative.scala).
namespace {
struct JavaRandom {
  uint64_t seed;
  explicit JavaRandom(int64_t s) : seed(((uint64_t)s ^ 0x5DEECE66DULL) & ((1ULL << 48) - 1)) {}
  int32_t next(int bits) {
    seed = (seed * 0x5DEECE66DULL + 0xBULL) & ((1ULL << 48) - 1);
    return (int32_t)((int64_t)seed >> (48 - bits));
  }
  int64_t next_long() { const int64_t hi = next(32); const int64_t lo = next(32); return (int64_t)((uint64_t)hi << 32) + lo; }
};
uint32_t murmur3_bytes(const unsigned char* data, int len, uint32_t seed) {
  auto rotl = [](uint32_t x, int r) { return (x << r) | (x >> (32 - r)); };
  uint32_t h = seed;
  int i = 0;
  for (; len - i >= 4; i += 4) {
    uint32_t k = (uint32_t)data[i] | ((uint32_t)data[i + 1] << 8) | ((uint32_t)data[i + 2] << 16) | ((uint32_t)data[i + 3] << 24);
    k *= 0xcc9e2d51u; k = rotl(k, 15); k *= 0x1b873593u;
    h ^= k; h = rotl(h, 13); h = h * 5u + 0xe6546b64u;
  }
  uint32_t k = 0;
  const int rem = len - i;
  if (rem == 3) k ^= (uint32_t)data[i + 2] << 16;
  if (rem >= 2) k ^= (uint32_t)data[i + 1] << 8;
  if (rem >= 1) { k ^= (uint32_t)data[i]; k *= 0xcc9e2d51u; k = rotl(k, 15); k *= 0x1b873593u; h ^= k; }
  h ^= (uint32_t)len;
  h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
  return h;
}
struct XorShift {
  uint64_t s;
  explicit XorShift(int64_t init) {
    unsigned char b[8];
    for (int i = 0; i < 8; ++i) b[i] = (unsigned char)((uint64_t)init >> (56 - 8 * i));  // ByteBuffer.putLong: big endian
    const uint32_t low = murmur3_bytes(b, 8, 0x3c074a61u);  // MurmurHash3.arraySeed
    const uint32_t high = murmur3_bytes(b, 8, low);
    s = ((uint64_t)high << 32) | (uint64_t)low;
  }
  int32_t next(int bits) {
    s ^= s << 21; s ^= s >> 35; s ^= s << 4;
    return (int32_t)(s & ((1ULL << bits) - 1));
  }
  double next_double() { return (double)(((int64_t)next(26) << 27) + next(27)) * (1.0 / (double)(1LL << 53)); }
};
}  // namespace

int se_spark_bernoulli_sample(int64_t seed, double fraction, int64_t n, int partition, float* counts) {
  if (!counts || n < 0 || partition < 0) return fail(nullptr, SE_ERR_ARG, "bad argument");
  JavaRandom jr(seed);
  int64_t pseed = 0;
  for (int p = 0; p <= partition; ++p) pseed = jr.next_long();
  XorShift rng(pseed);
  if (fraction <= 0.0) { for (int64_t i = 0; i < n; ++i) counts[i] = 0.f; return SE_OK; }
  if (fraction >= 1.0) { for (int64_t i = 0; i < n; ++i) counts[i] = 1.f; return SE_OK; }
  if (fraction <= 0.4) {  // RandomSampler.defaultMaxGapSamplingFraction
    const double lnq = log1p(-fraction), eps = 5e-11;  // RandomSampler.rngEpsilon
    auto advance = [&]() { const double u = fmax(rng.next_double(), eps); return (int64_t)(log(u) / lnq); };
    int64_t drop = advance();  // the GapSampling constructor advances once
    for (int64_t i = 0; i < n; ++i) {
      if (drop > 0) { --drop; counts[i] = 0.f; }
      else { drop = advance(); counts[i] = 1.f; }
    }
  } else {
    for (int64_t i = 0; i < n; ++i) counts[i] = (rng.next_double() <= fraction) ? 1.f : 0.f;
  }
  return SE_OK;
}

// ---- Boosting ----------------------------------------------------------------------------------
int se_boost_configure(se_ctx* ctx, int64_t n, int num_classes, int real) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, n >= 0 && num_classes >= 2, SE_ERR_ARG, "need n >= 0 and numClasses >= 2");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  ctx->boost.on = true; ctx->boost.n = n; ctx->boost.K = num_classes; ctx->boost.real = real != 0;
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_Y, 1, n));
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_BW, 1, n));
  if (real) SE_TRY(slot_alloc2d(ctx, SE_SLOT_PROBA, num_classes, n));
  else SE_TRY(slot_alloc2d(ctx, SE_SLOT_PRED, 1, n));
  return SE_OK;
}

static BoostArgs boost_args(se_ctx* ctx, double sum_w) {
  ensure_labels_checked(ctx, 0, ctx->boost.K, ctx->boost.n);  // SAMME / SAMME.R compare (and index with) the label
  BoostArgs a;
  a.y = ctx->slot[SE_SLOT_Y].d;
  a.w = ctx->slot[SE_SLOT_BW].d;
  a.proba = ctx->slot[SE_SLOT_PROBA].d;
  a.pred = ctx->slot[SE_SLOT_PRED].d;
  a.n = ctx->boost.n;
  a.ld = ctx->slot[SE_SLOT_PROBA].ld;
  a.K = ctx->boost.K;
  a.inv_sum_w = (float)(1.0 / sum_w);
  a.ws = red_ws(ctx);
  return a;
}

int se_boost_real_update(se_ctx* ctx, double sum_w, double* est_err, double* new_sum) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, ctx->boost.on && ctx->boost.real, SE_ERR_STATE, "se_boost_configure(real=1) first");
  SE_TRY(begin(ctx));
  BoostArgs a = boost_args(ctx, sum_w);
  SE_LAUNCH_T(ctx, SE_KF_BOOST_REAL, launch_boost_real(a, ctx->ctas_per_sm, ctx->sms, ctx->stream));
  double s[2];
  SE_TRY(fetch_scalars(ctx, 0, 2, s));
  if (est_err) *est_err = s[0];
  if (new_sum) *new_sum = s[1];
  return SE_OK;
}

int se_boost_discrete_error(se_ctx* ctx, double sum_w, double* est_err) {
  if (!ctx || !est_err) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, ctx->boost.on && !ctx->boost.real, SE_ERR_STATE, "se_boost_configure(real=0) first");
  SE_TRY(begin(ctx));
  BoostArgs a = boost_args(ctx, sum_w);
  SE_LAUNCH_T(ctx, SE_KF_BOOST_ERR, launch_boost_discrete_error(a, ctx->ctas_per_sm, ctx->sms, ctx->stream));
  return fetch_scalars(ctx, 0, 1, est_err);
}

int se_boost_discrete_update(se_ctx* ctx, double sum_w, double beta, double* new_sum) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, ctx->boost.on && !ctx->boost.real, SE_ERR_STATE, "se_boost_configure(real=0) first");
  SE_TRY(begin(ctx));
  BoostArgs a = boost_args(ctx, sum_w);
  a.inv_beta = (float)(1.0 / beta);
  SE_LAUNCH_T(ctx, SE_KF_BOOST_UPD, launch_boost_discrete_update(a, ctx->ctas_per_sm, ctx->sms, ctx->stream));
  double s = 0.0;
  SE_TRY(fetch_scalars(ctx, 0, 1, &s));
  if (new_sum) *new_sum = s;
  return SE_OK;
}

// ---- BoostingRegressor (AdaBoost.R2) -----------------------------------------------------------
int se_boostreg_configure(se_ctx* ctx, int64_t n) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, n >= 0, SE_ERR_ARG, "negative row count");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  ctx->boostreg.on = true;
  ctx->boostreg.n = n;
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_Y, 1, n));
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_BW, 1, n));
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_PRED, 1, n));
  return SE_OK;
}

static BoostRegArgs boostreg_args(se_ctx* ctx, double sum_w, int loss_type, double max_error, bool exchange = true) {
  BoostRegArgs a;
  a.y = ctx->slot[SE_SLOT_Y].d;
  a.pred = ctx->slot[SE_SLOT_PRED].d;
  a.w = ctx->slot[SE_SLOT_BW].d;
  a.n = ctx->boostreg.n;
  a.loss_type = loss_type;
  a.inv_sum_w = (float)(1.0 / sum_w);
  a.inv_max_err = (max_error == 0.0) ? 1.0f : (float)(1.0 / max_error);
  a.ws = red_ws(ctx, 0, exchange);
  return a;
}

int se_boostreg_max_error(se_ctx* ctx, double* max_error) {
  if (!ctx || !max_error) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, ctx->boostreg.on, SE_ERR_STATE, "se_boostreg_configure first");
  SE_TRY(begin(ctx));
  BoostRegArgs a = boostreg_args(ctx, 1.0, 0, 0.0, /*exchange=*/false);  // max-reduction: NCCL max afterwards
  SE_LAUNCH_T(ctx, SE_KF_OTHER, launch_boostreg_max(a, ctx->ctas_per_sm, ctx->sms, ctx->stream));
  return fetch_scalars(ctx, 0, 1, max_error, kNcclMax);
}

int se_boostreg_error(se_ctx* ctx, double sum_w, int loss_type, double max_error, double* est_err) {
  if (!ctx || !est_err) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, ctx->boostreg.on, SE_ERR_STATE, "se_boostreg_configure first");
  SE_REQUIRE(ctx, loss_type >= SE_R2_EXPONENTIAL && loss_type <= SE_R2_SQUARED, SE_ERR_ARG, "bad loss type %d", loss_type);
  SE_TRY(begin(ctx));
  BoostRegArgs a = boostreg_args(ctx, sum_w, loss_type, max_error);
  SE_LAUNCH_T(ctx, SE_KF_BOOST_ERR, launch_boostreg_error(a, ctx->ctas_per_sm, ctx->sms, ctx->stream));
  return fetch_scalars(ctx, 0, 1, est_err);
}

int se_boostreg_update(se_ctx* ctx, double sum_w, int loss_type, double max_error, double beta, double* new_sum) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, ctx->boostreg.on, SE_ERR_STATE, "se_boostreg_configure first");
  SE_REQUIRE(ctx, loss_type >= SE_R2_EXPONENTIAL && loss_type <= SE_R2_SQUARED, SE_ERR_ARG, "bad loss type %d", loss_type);
  SE_TRY(begin(ctx));
  BoostRegArgs a = boostreg_args(ctx, sum_w, loss_type, max_error);
  a.log2_beta = (float)log2(beta);
  SE_LAUNCH_T(ctx, SE_KF_BOOST_UPD, launch_boostreg_update(a, ctx->ctas_per_sm, ctx->sms, ctx->stream));
  double s = 0.0;
  SE_TRY(fetch_scalars(ctx, 0, 1, &s));
  if (new_sum) *new_sum = s;
  return SE_OK;
}

// ---- Aggregation -------------------------------------------------------------------------------
// The weighted median's weights (se_agg_run, se_forest_median): 0 when one is negative or not finite (the exact sort
// for every row), 2 when all are equal (the fast path without a rounding margin), 1 otherwise (with one).
int se_host::wm_weight_mode(const double* w, int M) {
  bool ok = true, equal = true;
  for (int i = 0; i < M; ++i) {
    ok = ok && (w[i] >= 0.0) && (w[i] <= 1.7976931348623157e308);
    equal = equal && (w[i] == w[0]);
  }
  return !ok ? 0 : equal ? 2 : 1;
}

int se_agg_configure(se_ctx* ctx, int kind, int num_models, int num_classes, int dim, int loss, int64_t n) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, kind >= SE_AGG_GBM_REGRESSOR && kind <= SE_AGG_BOOSTING_REG_MEAN, SE_ERR_ARG, "bad kind %d", kind);
  SE_REQUIRE(ctx, num_models >= 0 && n >= 0, SE_ERR_ARG, "bad sizes");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  auto& g = ctx->agg;
  g.on = true; g.kind = kind; g.M = num_models; g.K = num_classes; g.dim = dim; g.loss = loss; g.n = n;
  switch (kind) {
    case SE_AGG_GBM_REGRESSOR:
    case SE_AGG_BAGGING_REGRESSOR:
    case SE_AGG_BOOSTING_REG_MEAN: g.width = 1; g.C = 1; break;
    case SE_AGG_BOOSTING_REG_MEDIAN:
      SE_REQUIRE(ctx, num_models >= 1 && num_models <= 8192, SE_ERR_ARG, "weighted median supports 1..8192 models (got %d)", num_models);
      g.width = 1; g.C = 1; break;
    case SE_AGG_GBM_CLASSIFIER:
      SE_REQUIRE(ctx, dim >= 1 && num_classes >= 2, SE_ERR_ARG, "bad dim/numClasses");
      g.width = dim; g.C = (dim == 1 && num_classes == 2) ? 2 : dim; break;
    case SE_AGG_BAGGING_SOFT:
    case SE_AGG_BOOSTING_REAL:
      SE_REQUIRE(ctx, num_classes >= 2, SE_ERR_ARG, "numClasses >= 2");
      g.width = num_classes; g.C = num_classes; break;
    default:
      SE_REQUIRE(ctx, num_classes >= 2, SE_ERR_ARG, "numClasses >= 2");
      g.width = 1; g.C = num_classes; break;
  }
  const int64_t prow = (int64_t)(num_models > 0 ? num_models : 1) * g.width;
  // P is allocated with rows >= 2 semantics (padded stride) so every model row is 128 B aligned
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_P, prow, n));
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_RAW, g.C, n));
  if (kind >= SE_AGG_GBM_CLASSIFIER && kind <= SE_AGG_BOOSTING_DISCRETE) {
    SE_TRY(slot_alloc2d(ctx, SE_SLOT_PROB, g.C, n));
    SE_TRY(slot_alloc2d(ctx, SE_SLOT_LABEL, 1, n));
  }
  return SE_OK;
}

int se_agg_run(se_ctx* ctx, const double* weights, const double* init) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, ctx->agg.on, SE_ERR_STATE, "se_agg_configure first");
  const auto& g = ctx->agg;
  SE_TRY(begin(ctx));
  AggArgs a;
  a.kind = g.kind; a.M = g.M; a.K = g.K; a.dim = g.dim; a.loss = g.loss; a.n = g.n;
  a.P = ctx->slot[SE_SLOT_P].d; a.ld = ctx->slot[SE_SLOT_P].ld;
  a.raw = ctx->slot[SE_SLOT_RAW].d;
  a.ld_out = ctx->slot[SE_SLOT_RAW].ld;
  a.prob = ctx->slot[SE_SLOT_PROB].d;
  a.label = ctx->slot[SE_SLOT_LABEL].d;
  a.bad_label = ctx->d_bad_label;
  // small operands: narrowed to fp32 and staged through pinned memory into d_small
  float* hs = reinterpret_cast<float*>(ctx->h_small.get());
  size_t used = 0;
  const bool uses_w = (g.kind == SE_AGG_GBM_REGRESSOR || g.kind == SE_AGG_GBM_CLASSIFIER || g.kind == SE_AGG_BOOSTING_DISCRETE ||
                       g.kind == SE_AGG_BOOSTING_REG_MEAN || g.kind == SE_AGG_BOOSTING_REG_MEDIAN);
  const int nw = g.M * ((g.kind == SE_AGG_GBM_CLASSIFIER) ? g.dim : 1);
  SE_REQUIRE(ctx, (size_t)(nw + kMaxDim) * sizeof(float) * 2 <= (size_t)kSmallBytes, SE_ERR_ARG, "too many models");
  // the previous run may still be reading d_small/h_small
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (uses_w) {
    SE_REQUIRE(ctx, weights || g.M == 0, SE_ERR_ARG, "weights required for this aggregation kind");
    double sw = 0.0;
    for (int i = 0; i < nw; ++i) { hs[i] = (float)weights[i]; sw += (double)hs[i]; }  // Σ of what the device sees
    a.weights = reinterpret_cast<const float*>(ctx->d_small.get());
    a.sum_weights = sw;
    used = (size_t)nw;
  }
  if ((g.kind == SE_AGG_GBM_REGRESSOR || g.kind == SE_AGG_GBM_CLASSIFIER) && init) {
    const size_t off = (used + 31) / 32 * 32;
    for (int j = 0; j < g.dim; ++j) hs[off + j] = (float)init[j];
    a.init = reinterpret_cast<const float*>(ctx->d_small.get()) + off;
    used = off + g.dim;
  }
  if (g.kind == SE_AGG_BOOSTING_REG_MEDIAN) {
    // cumulative weights are compared in fp64 like the reference: ship the weights as doubles too
    const size_t off = (used + 63) / 64 * 64;  // floats; keeps the doubles 8-byte aligned
    double* hd = reinterpret_cast<double*>(hs + off);
    for (int i = 0; i < g.M; ++i) hd[i] = weights[i];
    a.weights64 = reinterpret_cast<const double*>(reinterpret_cast<const float*>(ctx->d_small.get()) + off);
    used = off + 2 * (size_t)g.M;
    // fast path (launch_agg): every weight finite and >= 0; all equal -> no rounding margin needed
    ctx->last_wm_mode = 0;
    if (ctx->wm_fast && g.M >= 1 && g.M <= 64 && g.n > 0) {
      a.wm_mode = wm_weight_mode(weights, g.M);
      if (a.wm_mode) {
        a.weights64_host = weights;
        if (a.wm_mode == 1) {
          int64_t cap = ctx->wm_list_cap > 0 ? ctx->wm_list_cap : g.n / 4;
          if (cap < 1024 && ctx->wm_list_cap == 0) cap = 1024;
          if (cap > 2147483000LL) cap = 2147483000LL;
          if (ctx->d_wm.grow((size_t)cap + 1) != cudaSuccess) cudaGetLastError();
          if (ctx->d_wm) {
            a.wm_count = ctx->d_wm;
            a.wm_list = reinterpret_cast<int32_t*>(ctx->d_wm + 1);
            a.wm_cap = (unsigned int)cap;
          } else {
            a.wm_mode = 0;  // no room for the list: exact kernel
          }
        }
        ctx->last_wm_mode = a.wm_mode;
      }
    }
  }
  if (used) SE_CUDA(ctx, cudaMemcpyAsync(ctx->d_small, hs, used * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  SE_LAUNCH_T(ctx, SE_KF_AGG, launch_agg(a, 8, ctx->sms, ctx->stream));
  if (g.kind == SE_AGG_GBM_CLASSIFIER || g.kind == SE_AGG_BAGGING_SOFT || g.kind == SE_AGG_BOOSTING_REAL)
    ctx->launches++;  // separate finalize kernel (the vote kinds fuse their epilogue)
  return end(ctx);
}
