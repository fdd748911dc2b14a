// se_api_gbm.cu — host side of the GBM entry points: pseudo-residuals, updates, line searches (host Brent, the
// persistent device line search) and the one-launch squared-loss round.
#include "se_ctx.h"
#define SE_BRENT_HOST_ONLY
#include "se_brent.h"
#include "se_loss.cuh"

using namespace se;
using namespace se_host;

namespace {

int need_slot(se_ctx* ctx, int slot, int64_t rows, int64_t cols, const char* what) {
  const SlotBuf& s = ctx->slot[slot];
  if (!s.d || s.rows != rows || s.cols != cols)
    return fail(ctx, SE_ERR_STATE, "%s: slot %d must hold [%lld][%lld] (has [%lld][%lld])", what,
                slot, (long long)rows, (long long)cols, (long long)s.rows, (long long)s.cols);
  return SE_OK;
}

int ensure_counts(se_ctx* ctx) {
  if (ctx->gbm.counts_valid) return SE_OK;
  SE_CUDA(ctx, cudaSetDevice(ctx->device));  // callers may run before begin(): launches below need the right device
  double v[2] = {(double)ctx->gbm.n, (double)ctx->gbm.nv};
  SE_TRY(se_comm_allreduce_host(ctx, v, 2));
  ctx->gbm.n_global = v[0];
  ctx->gbm.nv_global = v[1];
  ctx->gbm.counts_valid = true;
  return SE_OK;
}

int ensure_wsum(se_ctx* ctx) {
  if (ctx->gbm.wsum_valid) return SE_OK;
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_TRY(ensure_counts(ctx));
  if (ctx->gbm.use_bag) {
    // weightSum over the bag: Σ c_i·w_i (GBMLoss.scala:65 adds instance.weight once per sampled copy)
    SE_TRY(need_slot(ctx, SE_SLOT_BAG, 1, ctx->gbm.n, "bag multiplicities"));
    SE_LAUNCH(ctx, launch_dot(ctx->slot[SE_SLOT_BAG].d, ctx->gbm.has_w ? ctx->slot[SE_SLOT_W].d.get() : nullptr,
                              ctx->gbm.n, red_ws(ctx), ctx->ctas_per_sm, ctx->sms, ctx->stream));
    double s = 0.0;
    SE_TRY(fetch_scalars(ctx, 0, 1, &s));
    ctx->gbm.wsum = s;
  } else if (!ctx->gbm.has_w) {
    ctx->gbm.wsum = ctx->gbm.n_global;
  } else {
    SE_TRY(need_slot(ctx, SE_SLOT_W, 1, ctx->gbm.n, "instance weights"));
    SE_LAUNCH(ctx, launch_sum(ctx->slot[SE_SLOT_W].d, ctx->gbm.n, red_ws(ctx), ctx->ctas_per_sm,
                              ctx->sms, ctx->stream));
    double s = 0.0;
    SE_TRY(fetch_scalars(ctx, 0, 1, &s));
    ctx->gbm.wsum = s;
  }
  ctx->gbm.wsum_valid = true;
  return SE_OK;
}

GbmArgs gbm_args(se_ctx* ctx, bool validation) {
  GbmArgs a;
  const auto& g = ctx->gbm;
  a.y = ctx->slot[validation ? SE_SLOT_VY : SE_SLOT_Y].d;
  a.F = ctx->slot[validation ? SE_SLOT_VF : SE_SLOT_F].d;
  a.h = ctx->slot[validation ? SE_SLOT_VH : SE_SLOT_H].d;
  a.w = (!validation && g.has_w) ? ctx->slot[SE_SLOT_W].d.get() : nullptr;
  a.bag = (!validation && g.use_bag) ? ctx->slot[SE_SLOT_BAG].d.get() : nullptr;
  a.r = validation ? nullptr : ctx->slot[SE_SLOT_R].d.get();
  a.wout = validation ? nullptr : ctx->slot[SE_SLOT_WOUT].d.get();
  a.n = validation ? g.nv : g.n;
  a.ld = ctx->slot[validation ? SE_SLOT_VF : SE_SLOT_F].ld;
  a.dim = g.dim;
  a.param = (float)g.param;
  a.reverse = (ctx->alternate && !validation) ? (int)(ctx->pass_parity++ & 1u) : 0;
  // shards whose four per-row arrays (y, F, h, r) are of the order of the L2: evict_first hints (se_common.cuh)
  a.l2_hints = ctx->l2_hints >= 0 ? ctx->l2_hints : ((validation ? ctx->gbm.nv : ctx->gbm.n) <= ctx->l2_hint_rows ? 1 : 0);
  a.ws = red_ws(ctx, 0, /*exchange=*/false);  // armed (sequence number taken) only at reducing launches
  return a;
}

// ---- Brent (se_brent.h): host wrapper over the shared host/device template
int brent_impl(se_fn1 f, void* user, double lo, double hi, double start, double rel, double abs_tol,
               int max_eval, double* x_out, double* f_out, int* n_eval) {
  const int rc = brent_core([&](double x) { return f(x, user); }, lo, hi, start, rel, abs_tol, max_eval, x_out, f_out,
                            n_eval);
  return rc == kBrentOk ? SE_OK : SE_ERR_OPT;
}

}  // namespace

// ---- GBM ---------------------------------------------------------------------------------------
int se_gbm_configure(se_ctx* ctx, int64_t n_train, int64_t n_valid, int dim, int loss, double param,
                     int has_weights) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, n_train >= 0 && n_valid >= 0, SE_ERR_ARG, "negative row count");
  SE_REQUIRE(ctx, loss >= SE_LOSS_SQUARED && loss <= SE_LOSS_LOGLOSS, SE_ERR_ARG, "unknown loss %d", loss);
  SE_REQUIRE(ctx, dim >= 1 && dim <= kMaxDimGeneric, SE_ERR_ARG, "dim %d outside [1,%d]", dim, kMaxDimGeneric);
  SE_REQUIRE(ctx, (loss == SE_LOSS_LOGLOSS) || dim == 1, SE_ERR_ARG, "scalar losses have dim 1 (got %d)", dim);
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_TRY(settle_f(ctx));  // F is kept across a reconfiguration that does not reallocate it
  auto& g = ctx->gbm;
  g.on = true; g.n = n_train; g.nv = n_valid; g.dim = dim; g.loss = loss; g.param = param;
  g.has_w = has_weights != 0;
  g.use_bag = false;
  g.r_current = false;
  g.sq_stats_current = false;
  g.sq_defer_ok = false;
  g.wsum_valid = false; g.counts_valid = false;
  ctx->y_state[0] = ctx->y_state[1] = 0;
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_Y, 1, n_train));
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_F, dim, n_train));
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_H, dim, n_train));
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_R, dim, n_train));
  if (g.has_w) SE_TRY(slot_alloc2d(ctx, SE_SLOT_W, 1, n_train));
  // validation slots exist even for an EMPTY local validation shard (trailing row shards may be empty,
  // ensemble.row_partition): the rank must still launch every validation reduction so that its peers' collectives complete
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_VY, 1, n_valid));
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_VF, dim, n_valid));
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_VH, dim, n_valid));
  return SE_OK;
}

int se_gbm_set_loss_param(se_ctx* ctx, double param) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, ctx->gbm.on, SE_ERR_STATE, "se_gbm_configure first");
  SE_TRY(settle_f(ctx));
  ctx->gbm.param = param;
  ctx->gbm.r_current = false;
  ctx->gbm.sq_stats_current = false;
  return SE_OK;
}

int se_gbm_set_bag(se_ctx* ctx, int on) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, ctx->gbm.on, SE_ERR_STATE, "se_gbm_configure first");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  if (on) SE_TRY(slot_alloc2d(ctx, SE_SLOT_BAG, 1, ctx->gbm.n));
  ctx->gbm.use_bag = on != 0;
  ctx->gbm.wsum_valid = false;
  ctx->gbm.sq_stats_current = false;
  return SE_OK;
}

namespace {
int ensure_big(se_ctx* ctx, int dim) {
  auto& b = ctx->big;
  b.grid = std::min(ctx->sms * 8, 1024);
  SE_CUDA(ctx, b.d_coef.grow((size_t)dim));
  SE_CUDA(ctx, b.h_coef.grow((size_t)dim));
  SE_CUDA(ctx, b.d_partials.grow((size_t)b.grid * (size_t)(dim + 1)));
  SE_CUDA(ctx, b.d_out.grow((size_t)(dim + 1)));
  SE_CUDA(ctx, b.h_out.grow((size_t)(dim + 1)));
  return SE_OK;
}
}  // namespace

// Labels as class indices: one validation pass per write of the label slot (see validate_labels_kernel).
int se_host::ensure_labels_checked(se_ctx* ctx, int which /*0 train, 1 validation*/, int K, int64_t n) {
  if (ctx->y_state[which] == 2 && ctx->y_state_k[which] == K) return SE_OK;
  const SlotBuf& y = ctx->slot[which ? SE_SLOT_VY : SE_SLOT_Y];
  if (!y.d || n <= 0) return SE_OK;
  SE_LAUNCH(ctx, launch_validate_labels(y.d, n, K, ctx->d_bad_label, ctx->sms, ctx->stream));
  ctx->y_state[which] = 1;
  ctx->y_state_k[which] = K;
  return SE_OK;
}

namespace {
// One GBM kernel launch for the configured loss.  `coef` (alpha or step, gbm.dim values, nullable) goes into the kernel
// arguments for dim <= kMaxDim and into a device buffer for the general LogLoss path beyond it.
int gbm_launch(se_ctx* ctx, int family, int mode, GbmArgs& a, const double* coef) {
  const int dim = ctx->gbm.dim;
  ctx->big.pending = false;
  if (ctx->gbm.loss == SE_LOSS_LOGLOSS) {
    const int which = (a.y == ctx->slot[SE_SLOT_VY].d && a.y != nullptr && a.y != ctx->slot[SE_SLOT_Y].d) ? 1 : 0;
    SE_TRY(ensure_labels_checked(ctx, which, dim, a.n));
  }
  if (dim <= kMaxDim) {
    if (coef)
      for (int j = 0; j < dim; ++j) a.coef[j] = (float)coef[j];
    SE_LAUNCH_T(ctx, family, launch_gbm(ctx->gbm.loss, mode, a, ctx->ctas_per_sm, ctx->sms, ctx->stream));
    return SE_OK;
  }
  SE_TRY(ensure_big(ctx, dim));
  auto& b = ctx->big;
  if (coef) {
    SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // h_coef may still feed the previous launch
    for (int j = 0; j < dim; ++j) b.h_coef[j] = (float)coef[j];
    SE_CUDA(ctx, cudaMemcpyAsync(b.d_coef, b.h_coef, sizeof(float) * (size_t)dim, cudaMemcpyHostToDevice, ctx->stream));
  }
  GenericArgs ga;
  ga.coef = b.d_coef;
  ga.partials = b.d_partials;
  ga.out = b.d_out;
  const int64_t groups = (a.n + 31) / 32;
  int grid = (int)(groups < (int64_t)b.grid ? (groups > 0 ? groups : 1) : b.grid);
  // the sums of this path are all-reduced by NCCL (fetch below): disarm the in-kernel exchange / host mirror
  ctx->last_reduce_global = false;
  ctx->mirror_valid = false;
  SE_LAUNCH_T(ctx, family, launch_gbm_logloss_generic(mode, a, ga, grid, ctx->stream));
  b.pending = true;
  return SE_OK;
}

// The sums of the last gbm_launch: [0] Σloss, [1 + j] per-dimension sums — global (summed across GPUs).
int gbm_fetch(se_ctx* ctx, int count, double* out) {
  if (!ctx->big.pending) return fetch_scalars(ctx, 0, count, out);
  auto& b = ctx->big;
  b.pending = false;
  if (ctx->comm && ctx->nranks > 1) {
    NcclApi& api = nccl();
    int rc = api.AllReduce(b.d_out, b.d_out, (size_t)(ctx->gbm.dim + 1), kNcclFloat64, kNcclSum, ctx->comm, ctx->stream);
    if (rc != 0) return fail(ctx, SE_ERR_NCCL, "ncclAllReduce: %s", api.GetErrorString(rc));
  }
  SE_CUDA(ctx, cudaMemcpyAsync(b.h_out, b.d_out, sizeof(double) * (size_t)count, cudaMemcpyDeviceToHost, ctx->stream));
  SE_TRY(end(ctx));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < count; ++i) out[i] = b.h_out[i];
  return check_labels(ctx);
}
}  // namespace

static int newton_finish(se_ctx* ctx, double* sum_hess) {
  // S_j (all-reduced) -> the base-learner weights are WOUT_j * 1/S_j  (GBMRegressor.scala:373,379;
  // GBMClassifier.scala:344-355,364).  The kernel left the unnormalised 1/2 hc w in SE_SLOT_WOUT; the per-dimension
  // factor 1/S_j is applied wherever WOUT is read as weights, and only there: where they LEAVE the device (se_download /
  // se_download_scaled on SE_SLOT_WOUT) and where a device fit reads them (se_linear_moments scales its matrix; a tree
  // fit needs no factor, its splits and leaves do not change when every weight is scaled) — no separate 8 B/row pass
  // over WOUT for it.
  const int dim = ctx->gbm.dim;
  std::vector<double> s((size_t)dim + 1);
  SE_TRY(gbm_fetch(ctx, 1 + dim, s.data()));
  ctx->wout_scale.assign((size_t)dim, 0.f);
  for (int j = 0; j < dim; ++j) {
    ctx->wout_scale[j] = (float)(1.0 / s[1 + j]);
    if (sum_hess) sum_hess[j] = s[1 + j];
  }
  ctx->wout_scaled = true;
  ctx->h_scal[0] = s[0];
  return SE_OK;
}

int se_gbm_pseudo_residuals(se_ctx* ctx, int newton, double* sum_hess) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, ctx->gbm.on, SE_ERR_STATE, "se_gbm_configure first");
  SE_REQUIRE(ctx, !newton || loss_has_hessian(ctx->gbm.loss), SE_ERR_ARG, "loss %d has no hessian (updates=newton)", ctx->gbm.loss);
  SE_TRY(begin(ctx));
  SE_TRY(settle_f(ctx));
  ctx->gbm.sq_stats_current = false;  // R is rewritten
  if (newton) SE_TRY(slot_alloc2d(ctx, SE_SLOT_WOUT, ctx->gbm.dim, ctx->gbm.n));
  GbmArgs a = gbm_args(ctx, false);
  if (newton) ctx->wout_scaled = false;  // a gradient-mode call leaves WOUT, and the 1/S of its download, as they were
  if (newton) a.ws = red_ws(ctx);  // Σ max(H,1e-2): reducing launch
  SE_TRY(gbm_launch(ctx, SE_KF_RESID, newton ? GBM_RESID_NEWTON : GBM_RESID, a, nullptr));
  if (newton) SE_TRY(newton_finish(ctx, sum_hess));
  ctx->gbm.r_current = true;  // squared loss: r = y - F for gradient and newton (h = 1) alike
  return end(ctx);
}

int se_gbm_linesearch_eval(se_ctx* ctx, const double* alpha, double* loss, double* grad) {
  if (!ctx || !alpha || !loss) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, ctx->gbm.on, SE_ERR_STATE, "se_gbm_configure first");
  SE_TRY(ensure_wsum(ctx));
  SE_TRY(begin(ctx));
  SE_TRY(settle_f(ctx));
  const int dim = ctx->gbm.dim;
  GbmArgs a = gbm_args(ctx, false);
  if (ctx->ls_packed) {  // inside se_gbm_linesearch_brent: bit-identical 8 B/row view
    a.y = nullptr;
    a.F = ctx->d_ls_u;
    a.h = ctx->d_ls_v;
  }
  a.ws = red_ws(ctx);
  // Brent consumes the objective value only: skip the gradient/curvature arithmetic when nobody asked for it
  const int eval_mode = (!grad && ctx->gbm.loss != SE_LOSS_LOGLOSS) ? GBM_EVAL_LOSS : GBM_EVAL;
  SE_TRY(gbm_launch(ctx, SE_KF_EVAL, eval_mode, a, alpha));
  std::vector<double> s((size_t)dim + 1);
  SE_TRY(gbm_fetch(ctx, 1 + dim, s.data()));
  // lossSum is accumulated `dim` times per row in the reference (GBMLoss.scala:60-64)
  *loss = (double)dim * s[0] / ctx->gbm.wsum;
  if (grad)
    for (int j = 0; j < dim; ++j) grad[j] = s[1 + j] / ctx->gbm.wsum;
  return SE_OK;
}

int se_gbm_linesearch_stats(se_ctx* ctx, double* stats4) {
  if (!ctx || !stats4) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, ctx->gbm.on && ctx->gbm.loss == SE_LOSS_SQUARED, SE_ERR_STATE, "squared loss only");
  SE_TRY(ensure_wsum(ctx));
  SE_TRY(begin(ctx));
  SE_TRY(settle_f(ctx));
  GbmArgs a = gbm_args(ctx, false);
  a.stats_from_r = ctx->gbm.r_current ? 1 : 0;
  a.ws = red_ws(ctx);
  SE_LAUNCH_T(ctx, SE_KF_SQ_STATS, launch_gbm(SE_LOSS_SQUARED, GBM_SQ_STATS, a, ctx->ctas_per_sm, ctx->sms, ctx->stream));
  SE_TRY(fetch_scalars(ctx, 0, 3, stats4));
  stats4[3] = ctx->gbm.wsum;
  return SE_OK;
}

int se_gbm_update(se_ctx* ctx, const double* step, int flags, double* loss_sum, double* sum_hess) {
  if (!ctx || !step) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, ctx->gbm.on, SE_ERR_STATE, "se_gbm_configure first");
  const bool newton = (flags & SE_UPD_NEWTON) != 0;
  SE_REQUIRE(ctx, !newton || loss_has_hessian(ctx->gbm.loss), SE_ERR_ARG, "loss %d has no hessian", ctx->gbm.loss);
  SE_TRY(begin(ctx));
  SE_TRY(settle_f(ctx));
  ctx->gbm.sq_stats_current = false;  // F or R is rewritten
  if (newton) SE_TRY(slot_alloc2d(ctx, SE_SLOT_WOUT, ctx->gbm.dim, ctx->gbm.n));
  GbmArgs a = gbm_args(ctx, false);
  const int mode = newton ? GBM_UPDATE_NEWTON : ((flags & SE_UPD_RESIDUAL) ? GBM_UPDATE_RESID : GBM_UPDATE);
  if (newton) ctx->wout_scaled = false;
  a.ws = red_ws(ctx);
  SE_TRY(gbm_launch(ctx, SE_KF_UPDATE, mode, a, step));
  ctx->gbm.r_current = (mode != GBM_UPDATE);  // the fused modes refresh R from the new F
  if (newton) {
    SE_TRY(newton_finish(ctx, sum_hess));
    if (loss_sum) *loss_sum = ctx->h_scal[0];
    return end(ctx);
  }
  if ((flags & SE_UPD_LOSS) && loss_sum) return gbm_fetch(ctx, 1, loss_sum);
  return end(ctx);
}

int se_gbm_mean_loss(se_ctx* ctx, int which, double* out) {
  if (!ctx || !out) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, ctx->gbm.on, SE_ERR_STATE, "se_gbm_configure first");
  SE_REQUIRE(ctx, which == 0 || which == 1, SE_ERR_ARG, "which must be 0 (train) or 1 (validation)");
  SE_TRY(ensure_counts(ctx));
  // the GLOBAL count decides: a rank whose local shard is empty still launches the reduction (n = 0) so that the
  // collective of its peers completes
  SE_REQUIRE(ctx, (which == 1 ? ctx->gbm.nv_global : ctx->gbm.n_global) > 0.0, SE_ERR_ARG,
             which == 1 ? "no validation rows on any rank" : "no training rows on any rank");
  SE_TRY(begin(ctx));
  if (which == 0) SE_TRY(settle_f(ctx));
  GbmArgs a = gbm_args(ctx, which == 1);
  a.ws = red_ws(ctx);
  SE_TRY(gbm_launch(ctx, SE_KF_MEAN_LOSS, GBM_MEAN_LOSS, a, nullptr));
  double s = 0.0;
  SE_TRY(gbm_fetch(ctx, 1, &s));
  *out = s / (which == 1 ? ctx->gbm.nv_global : ctx->gbm.n_global);
  return SE_OK;
}

int se_gbm_update_validation(se_ctx* ctx, const double* step, double* mean_loss) {
  if (!ctx || !step) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, ctx->gbm.on, SE_ERR_STATE, "se_gbm_configure first");
  SE_TRY(ensure_counts(ctx));
  SE_REQUIRE(ctx, ctx->gbm.nv_global > 0.0, SE_ERR_STATE, "no validation rows configured on any rank");
  SE_TRY(begin(ctx));
  GbmArgs a = gbm_args(ctx, true);
  a.ws = red_ws(ctx);
  SE_TRY(gbm_launch(ctx, SE_KF_UPDATE, GBM_UPDATE, a, step));
  double s = 0.0;
  SE_TRY(gbm_fetch(ctx, 1, &s));
  if (mean_loss) *mean_loss = s / ctx->gbm.nv_global;
  return SE_OK;
}

namespace {
struct EvalClosure {
  se_ctx* ctx;
  int rc;
};
double eval_cb(double x, void* user) {
  EvalClosure* c = static_cast<EvalClosure*>(user);
  double l = NAN;
  if (c->rc == SE_OK) c->rc = se_gbm_linesearch_eval(c->ctx, &x, &l, nullptr);
  return l;
}
using Parabola = BrentParabola;
double parabola_cb(double x, void* user) { return (*static_cast<const Parabola*>(user))(x); }
}  // namespace

namespace {

int ensure_ls_view(se_ctx* ctx) {
  // one allocation for both halves, v starting on a 256-byte boundary
  const size_t half = ((size_t)ctx->gbm.n + 32 + 63) / 64 * 64;
  SE_CUDA(ctx, ctx->d_ls_u.grow(2 * half));
  ctx->d_ls_v = ctx->d_ls_u + half;
  return SE_OK;
}

// One launch of the persistent line-search kernel (se_gbm_fused.cu): the whole Brent search (single == 0) or one
// evaluation of the objective at `start` with the tile direction of evaluation number `parity + 1` (single == 1).
int linesearch_persist(se_ctx* ctx, double lo, double hi, double start, double rel, double abs_tol, int max_eval,
                       int single, int parity, double* alpha, double* loss, int* n_eval) {
  SE_TRY(ensure_wsum(ctx));
  SE_TRY(begin(ctx));
  SE_TRY(settle_f(ctx));
  const int lossid = ctx->gbm.loss;
  const bool packed = gbm_linesearch_persist_packed(lossid);
  if (packed) SE_TRY(ensure_ls_view(ctx));
  LsArgs a;
  a.y = ctx->slot[SE_SLOT_Y].d;
  a.F = ctx->slot[SE_SLOT_F].d;
  a.h = ctx->slot[SE_SLOT_H].d;
  a.u = ctx->d_ls_u;
  a.v = ctx->d_ls_v;
  a.n = ctx->gbm.n;
  a.param = (float)ctx->gbm.param;
  a.wsum = ctx->gbm.wsum;
  a.lo = lo; a.hi = hi; a.start = start; a.rel = rel; a.abs_tol = abs_tol; a.max_eval = max_eval;
  a.single = single;
  a.timing = ctx->fused_timing;
  a.first_parity = parity;
  a.partials = ctx->d_partials;
  a.sync = ctx->d_fsync;
  a.epoch0 = ctx->fused_epoch;
  ctx->fused_epoch += (unsigned long long)(max_eval > 0 ? max_eval : 1) + 4;
  a.out = ctx->d_scal + kScalRound + 16;
  a.ws = red_ws(ctx, kScalRound + 16);  // takes ONE sequence number; the kernel uses seq, seq+1, ... per evaluation
  const unsigned long long seq0 = ctx->red_seq;
  LsLaunch cfg;
  // small shards (what strong scaling leaves per GPU) live entirely in shared memory + L2: fewer, fatter CTAs keep more
  // tiles resident and shorten the per-evaluation rendezvous; large shards want more CTAs in flight
  cfg.max_ctas_per_sm = (ctx->ls_ctas_per_sm == 4 && ctx->gbm.n <= 8000000) ? 3 : ctx->ls_ctas_per_sm;
  cfg.resident = ctx->ls_resident;
  int workers = 0;
  SE_LAUNCH_T(ctx, SE_KF_EVAL, launch_gbm_linesearch_persist(lossid, a, ctx->sms, cfg, ctx->stream, &workers));
  ctx->last_ls_workers = workers;
  double res[4] = {0, 0, 0, 0};
  const int rc = fetch_scalars(ctx, kScalRound + 16, 4, res);
  // every evaluation consumed one reduction sequence number on every rank (the first was taken by red_ws)
  const int passes = (int)res[3];
  if (ctx->p2p && ctx->nranks > 1 && passes > 1) ctx->red_seq = seq0 + (unsigned long long)(passes - 1);
  ctx->last_ls_passes = passes;
  if (ctx->fused_timing) {
    SE_CUDA(ctx, cudaMemcpyAsync(ctx->h_scal + kScalRound + 20, ctx->d_scal + kScalRound + 20, sizeof(double) * 2, cudaMemcpyDeviceToHost, ctx->stream));
    SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->last_fused_us[0] = ctx->h_scal[kScalRound + 20];  // worker passes
    ctx->last_fused_us[1] = ctx->h_scal[kScalRound + 21];  // fold + exchange + Brent step
    ctx->last_fused_us[2] = 0.0;
  }
  if (rc != SE_OK) return rc;
  if (alpha) *alpha = res[0];
  if (loss) *loss = res[1];
  if (n_eval) *n_eval = (int)fabs(res[2]);
  if (res[2] < 0.0) return fail(ctx, SE_ERR_OPT, "Brent exceeded MaxEval(%d)", max_eval);
  return SE_OK;
}

struct PersistEvalClosure {
  se_ctx* ctx;
  int rc;
  int k;  // evaluations so far
};
double persist_eval_cb(double x, void* user) {
  PersistEvalClosure* c = static_cast<PersistEvalClosure*>(user);
  double l = NAN;
  if (c->rc == SE_OK) c->rc = linesearch_persist(c->ctx, 0.0, 0.0, x, 1e-6, 1e-6, 1, /*single=*/1, /*parity=*/c->k, nullptr, &l, nullptr);
  c->k++;
  return l;
}

}  // namespace

int se_gbm_linesearch_brent(se_ctx* ctx, double lo, double hi, double start, double rel, double abs_tol,
                            int max_eval, double* alpha, double* loss, int* n_eval) {
  if (!ctx || !alpha) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, ctx->gbm.on && ctx->gbm.dim == 1, SE_ERR_STATE, "Brent line search needs dim == 1");
  SE_TRY(settle_f(ctx));  // the packed view below reads F
  if (ctx->gbm.loss == SE_LOSS_SQUARED) {
    double st[4];
    SE_TRY(se_gbm_linesearch_stats(ctx, st));
    Parabola p{st[0], st[1], st[2], st[3]};
    int rc = brent_impl(parabola_cb, &p, lo, hi, start, rel, abs_tol, max_eval, alpha, loss, n_eval);
    if (rc != SE_OK) return fail(ctx, rc, "Brent exceeded MaxEval(%d)", max_eval);
    return SE_OK;
  }
  // Default: ONE persistent launch runs all of Brent's evaluations on the device (no host round trip and no launch
  // per evaluation; tiles resident in shared memory / L2 between evaluations) — se_gbm_fused.cu.
  // (needs in-kernel cross-GPU sums: single GPU or the fused peer exchange, not the NCCL fallback)
  if (ctx->ls_mode != 0 && !ctx->gbm.use_bag && max_eval >= 1 && gbm_linesearch_persist_supported(ctx->gbm.loss) &&
      (ctx->nranks <= 1 || ctx->p2p)) {
    if (ctx->ls_mode == 1) return linesearch_persist(ctx, lo, hi, start, rel, abs_tol, max_eval, 0, 0, alpha, loss, n_eval);
    // mode 2: the HOST runs the same Brent template and asks the same kernel for one evaluation at a time; the
    // objective values, hence the iterates, must equal mode 1 bit for bit (tests/test_gpu_parity.py)
    PersistEvalClosure c{ctx, SE_OK, 0};
    int rc = brent_impl(persist_eval_cb, &c, lo, hi, start, rel, abs_tol, max_eval, alpha, loss, n_eval);
    if (c.rc != SE_OK) return c.rc;
    if (rc != SE_OK) return fail(ctx, rc, "Brent exceeded MaxEval(%d)", max_eval);
    return SE_OK;
  }
  // Round-1 path (one launch + one host poll per evaluation), kept for bags and as the A/B baseline.
  // Binary scalar losses depend on (2y-1)(F + αh) only: one 20 B/row pass builds u = (2y-1)F, v = (2y-1)h and
  // every one of Brent's 20-40 evaluations then reads 8 B/row instead of 12 — same values bit for bit
  // (multiplying by ±1 is exact and fma is sign-symmetric).
  const bool pack = (ctx->gbm.loss == SE_LOSS_BERNOULLI || ctx->gbm.loss == SE_LOSS_EXPONENTIAL) && max_eval >= 8 &&
                    !ctx->gbm.use_bag;
  if (pack) {
    SE_CUDA(ctx, cudaSetDevice(ctx->device));
    SE_TRY(ensure_ls_view(ctx));
    SE_LAUNCH_T(ctx, SE_KF_OTHER, launch_gbm_pack_signed(ctx->slot[SE_SLOT_Y].d, ctx->slot[SE_SLOT_F].d, ctx->slot[SE_SLOT_H].d,
                                                         ctx->d_ls_u, ctx->d_ls_v, ctx->gbm.n, ctx->sms, ctx->stream));
    ctx->ls_packed = true;
  }
  EvalClosure c{ctx, SE_OK};
  int rc = brent_impl(eval_cb, &c, lo, hi, start, rel, abs_tol, max_eval, alpha, loss, n_eval);
  ctx->ls_packed = false;
  if (c.rc != SE_OK) return c.rc;
  if (rc != SE_OK) return fail(ctx, rc, "Brent exceeded MaxEval(%d)", max_eval);
  return SE_OK;
}

namespace {
// Squared loss, one cooperative launch per round (se_gbm_fused.cu): statistics -> cross-GPU sum -> Brent -> update +
// residual + loss -> cross-GPU sum -> host mirror.  One launch and one host poll per round.
int round_squared_fused(se_ctx* ctx, double learning_rate, double tol, int max_iter, int flags, double* alpha,
                        double* loss_sum, int* n_eval) {
  SE_TRY(ensure_wsum(ctx));
  SE_TRY(begin(ctx));
  const int write_r = (flags & SE_UPD_RESIDUAL) ? 1 : 0;
  // residual mode reads r (or y and F on a round whose residual slot is not current) and leaves F owed; the eager
  // form updates F itself and needs it current
  if (!write_r) SE_TRY(settle_f(ctx));
  SqRoundArgs a;
  const auto& g = ctx->gbm;
  a.y = ctx->slot[SE_SLOT_Y].d;
  a.F = ctx->slot[SE_SLOT_F].d;
  a.h = ctx->slot[SE_SLOT_H].d;
  a.r = ctx->slot[SE_SLOT_R].d;
  a.bag = g.use_bag ? ctx->slot[SE_SLOT_BAG].d.get() : nullptr;
  a.n = g.n;
  a.stats_from_r = g.r_current ? 1 : 0;
  a.l2_hints = ctx->l2_hints >= 0 ? ctx->l2_hints : (g.n <= ctx->l2_hint_rows ? 1 : 0);
  a.lr = learning_rate;
  a.wsum = g.wsum;
  a.lo = 0.0; a.hi = 100.0; a.start = 1.0; a.rel = tol; a.abs_tol = tol; a.max_eval = max_iter;
  a.out = ctx->d_scal + kScalRound;
  // The train loss after the update follows from the (global) statistics in closed form — no second reduction, no
  // second cross-GPU exchange, and the host is served before the update phase ends.  With a bag the statistics run
  // over the bag while the loss runs over all rows: then the loss is reduced over the rows as in the two-launch path.
  const bool loss_reduce = g.use_bag || ctx->fused_loss_reduce;
  // Such a residual round's update pass also sums the statistics of what it writes, (r', h), one partial per CTA into
  // a parity of d_sq_carry: the next round over the same direction folds them and skips its statistics pass (12 B/row,
  // not 20).
  // The update then walks its tiles opposite to the previous one, so that it starts on what is still in the L2.
  const bool stats_out = write_r && !loss_reduce;
  const bool carried = stats_out && g.r_current && g.sq_stats_current;
  // Only a carried round reads a pending R (and applies its steps in registers); every other round reads it settled.
  if (!carried) SE_TRY(settle_r(ctx));
  a.carried = carried ? 1 : 0;
  a.forward = (carried && !g.sq_last_up) ? 1 : 0;
  // A carried round after another one whose R nobody read stores nothing (8 B/row, not 12) while fewer than
  // sq_defer_max steps are pending; the round that would exceed the cap stores r' with all of them applied.  The
  // first carried round over a direction stores: a caller that reads R after it pays no settle.
  a.r_chain = ctx->d_rchain;
  a.r_pending = carried ? g.r_pending : 0;
  a.r_defer = (carried && g.sq_defer_ok && g.r_pending < ctx->sq_defer_max) ? 1 : 0;
  // the carried partials: read from the parity the last such round stored, stored into the other one
  constexpr size_t kCarryParity = (size_t)(kMaxGridPartials / 2) * 3;
  const int carry_parity = g.sq_carry_parity ^ 1;
  a.carry_in = ctx->d_sq_carry + (size_t)g.sq_carry_parity * kCarryParity;
  a.carry_grid = g.sq_carry_grid;
  a.carry_out = stats_out ? ctx->d_sq_carry + (size_t)carry_parity * kCarryParity : nullptr;
  ctx->gbm.sq_stats_current = false;           // until the round has succeeded
  a.ws_a = red_ws(ctx, kScalRound);            // sequence number s (statistics)
  // on one GPU a carried round may start before the kernel before it ends: it loads r that early only when no
  // kernel since the last deferring round has written R (every write of R settles the pending steps first)
  a.r_early = (carried && (a.ws_a.nranks <= 1 || a.ws_a.mbox == nullptr) && a.r_pending > 0) ? 1 : 0;
  a.ws_a.host_out = nullptr;                   // the mirror ticket is written after Brent / the second reduction
  a.ws_a.host_flag = nullptr;
  if (ctx->mirror_valid) --ctx->mirror_ticket; // red_ws armed the mirror for ws_a: re-armed below
  constexpr int kMirrorRound = 32;             // mirror slots [32..38]: above what a reducing kernel writes before its ticket
  bool mirror = false;
  if (loss_reduce) {
    a.ws_b = red_ws(ctx, kScalRound + 8);      // sequence number s + 1 (loss), host mirror + ticket
    a.ws_b.partials = ctx->d_partials + (size_t)(kMaxGridPartials / 2) * 4;
    a.ws_b.counter = &ctx->d_fsync->counter_b;
    mirror = ctx->mirror_valid;
  } else {
    const bool global = ctx->last_reduce_global;  // keep what red_ws decided for the statistics
    mirror = ctx->use_mirror && ctx->h_mirror && (ctx->nranks <= 1 || ctx->p2p);
    if (mirror) {
      a.host_final = ctx->d_mirror;
      a.host_flag = reinterpret_cast<volatile unsigned long long*>(ctx->d_mirror + kMboxPayload);
      a.host_ticket = ++ctx->mirror_ticket;
      ctx->mirror_valid = true;
      ctx->mirror_off = kScalRound + 8;
    }
    ctx->last_reduce_global = global;
  }
  a.host_res = mirror ? ctx->d_mirror + kMirrorRound : nullptr;
  a.sync = ctx->d_fsync;
  a.epoch = ++ctx->fused_epoch;
  a.timing = ctx->fused_timing;
  int grid = 0, resident_slots = 0;
  auto launch = [&]() {
    return launch_gbm_round_sq_fused(a, write_r, loss_reduce ? 1 : 0, ctx->fused_resident, ctx->sms,
                                     ctx->fused_ctas_per_sm, ctx->stream, &grid, &resident_slots);
  };
  if (carried && (a.ws_a.nranks <= 1 || a.ws_a.mbox == nullptr)) {
    // a programmatic dependent launch: kernel timing takes the kernel's own stamps, not events around it
    SE_TRY(kernel_stamp_slot(ctx, SE_KF_UPDATE, &a.kstamp));
    const cudaError_t e = launch();
    ctx->launches++;
    if (e != cudaSuccess) {
      if (a.kstamp) --ctx->kpending;  // give back the slot claimed above: nothing will stamp it
      return fail(ctx, SE_ERR_CUDA, "%s:%d launch launch_gbm_round_sq_fused -> %s", __FILE__, __LINE__,
                  cudaGetErrorString(e));
    }
  } else {
    SE_LAUNCH_T(ctx, SE_KF_UPDATE, launch());
  }
  ctx->last_fused_grid = grid;
  ctx->last_round_carried = carried ? 1 : 0;
  ctx->gbm.r_pending = a.r_defer ? a.r_pending + 1 : 0;  // the kernel ran: its step joined the chain or R was stored
  ctx->gbm.sq_defer_ok = carried;
  ctx->last_round_deferred = a.r_defer;
  ctx->last_fused_resident_tiles = resident_slots / 4.0;  // float4 groups per thread, U_SQ = 4 to a tile
  const bool r_current_before = ctx->gbm.r_current;
  ctx->gbm.r_current = write_r != 0;
  const bool owed_before = ctx->gbm.f_owed;
  if (write_r) ctx->gbm.f_owed = true;  // F = y - r from here on (unless the step turns out to be 0, below)
  double ls = 0.0;
  SE_TRY(fetch_scalars(ctx, kScalRound + 8, 1, &ls));
  double res[7];
  if (mirror) {
    for (int i = 0; i < 7; ++i) res[i] = ctx->h_mirror[kMirrorRound + i];
  } else {
    SE_CUDA(ctx, cudaMemcpyAsync(ctx->h_scal + kScalRound, ctx->d_scal + kScalRound, sizeof(double) * 7, cudaMemcpyDeviceToHost, ctx->stream));
    SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < 7; ++i) res[i] = ctx->h_scal[kScalRound + i];
  }
  for (int i = 0; i < 3; ++i) ctx->last_round_stats[i] = res[i];
  if (ctx->fused_timing) {
    double t[4];
    SE_CUDA(ctx, cudaMemcpyAsync(ctx->h_scal + kScalRound + 10, ctx->d_scal + kScalRound + 10, sizeof(double) * 4, cudaMemcpyDeviceToHost, ctx->stream));
    SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < 4; ++i) t[i] = ctx->h_scal[kScalRound + 10 + i];
    ctx->last_fused_us[0] = t[1] - t[0]; ctx->last_fused_us[1] = t[2] - t[1]; ctx->last_fused_us[2] = t[3] - t[2];
  }
  if (alpha) *alpha = res[4];
  if (n_eval) *n_eval = (int)fabs(res[6]);
  if (loss_sum) *loss_sum = ls;
  if (res[6] < 0.0) {
    // the step was 0: F was not moved, so it is exactly as current as before the round, and a download returns it bit
    // for bit.  R too: a round that read r stored r - 0*h, one that read y and F (R not current) stored nothing.
    ctx->gbm.f_owed = owed_before;
    ctx->gbm.r_current = r_current_before;
    return fail(ctx, SE_ERR_OPT, "Brent exceeded MaxEval(%d)", max_iter);
  }
  if (stats_out) {
    ctx->gbm.sq_stats_current = true;
    ctx->gbm.sq_last_up = a.forward != 0;
    ctx->gbm.sq_carry_parity = carry_parity;
    ctx->gbm.sq_carry_grid = grid;
  }
  return SE_OK;
}
}  // namespace

int se_gbm_round(se_ctx* ctx, double learning_rate, int optimized, double tol, int max_iter, int flags,
                 double* alpha, double* loss_sum, int* n_eval) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, ctx->gbm.on && ctx->gbm.dim == 1, SE_ERR_STATE, "se_gbm_round needs dim == 1");
  ctx->last_round_fused = 0;
  ctx->last_round_carried = 0;
  ctx->last_round_deferred = 0;
  const bool sq_search = optimized && ctx->gbm.loss == SE_LOSS_SQUARED && !(flags & SE_UPD_NEWTON) && max_iter >= 1;
  if (sq_search) {
    // commons-math3 BrentOptimizer constructor checks (the host path performs them in brent_impl's caller)
    SE_REQUIRE(ctx, tol >= 2.0 * 2.220446049250313e-16 && tol > 0.0, SE_ERR_ARG, "tolerance %g too small for Brent", tol);
    // One cooperative launch per round: no host round trip between the line search and the update.
    // With a communicator it needs the fused peer exchange (an NCCL all-reduce cannot run inside the kernel).
    const bool can = (ctx->nranks <= 1 || ctx->p2p);
    const bool want = ctx->fused_round > 0 || (ctx->fused_round < 0 && ctx->gbm.n <= ctx->fused_round_max_rows);
    if (can && want) {
      ctx->last_round_fused = 1;
      return round_squared_fused(ctx, learning_rate, tol, max_iter, flags, alpha, loss_sum, n_eval);
    }
  }
  double a = 1.0, obj = 0.0;
  int ne = 0;
  if (optimized) SE_TRY(se_gbm_linesearch_brent(ctx, 0.0, 100.0, 1.0, tol, tol, max_iter, &a, &obj, &ne));
  const double step = learning_rate * a;
  SE_TRY(se_gbm_update(ctx, &step, flags, loss_sum, nullptr));
  if (alpha) *alpha = a;
  if (n_eval) *n_eval = ne;
  return SE_OK;
}

int se_gbm_linesearch_eval2(se_ctx* ctx, double alpha, double* loss, double* d1, double* d2) {
  if (!ctx || !loss || !d1 || !d2) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, ctx->gbm.on && ctx->gbm.dim == 1 && ctx->gbm.loss != SE_LOSS_LOGLOSS, SE_ERR_STATE, "needs a dim-1 scalar loss");
  SE_TRY(ensure_wsum(ctx));
  SE_TRY(begin(ctx));
  SE_TRY(settle_f(ctx));
  GbmArgs a = gbm_args(ctx, false);
  a.coef[0] = (float)alpha;
  a.ws = red_ws(ctx);
  SE_LAUNCH_T(ctx, SE_KF_EVAL, launch_gbm(ctx->gbm.loss, GBM_EVAL, a, ctx->ctas_per_sm, ctx->sms, ctx->stream));
  double s[3];
  SE_TRY(fetch_scalars(ctx, 0, 3, s));
  *loss = s[0] / ctx->gbm.wsum;
  *d1 = s[1] / ctx->gbm.wsum;
  *d2 = s[2] / ctx->gbm.wsum;
  return SE_OK;
}

int se_gbm_linesearch_newton(se_ctx* ctx, double lo, double hi, double start, double rel, double abs_tol,
                             int max_eval, double* alpha, double* loss, int* n_eval) {
  if (!ctx || !alpha) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, ctx->gbm.on && ctx->gbm.dim == 1, SE_ERR_STATE, "Newton line search needs dim == 1");
  SE_REQUIRE(ctx, loss_has_hessian(ctx->gbm.loss), SE_ERR_ARG, "loss %d has no hessian: use the Brent line search", ctx->gbm.loss);
  if (lo > hi) { const double t = lo; lo = hi; hi = t; }
  double a = lo, b = hi;
  double x = fmin(fmax(start, a), b);
  double f = NAN;
  int evals = 0;
  for (;;) {
    if (evals >= max_eval) return fail(ctx, SE_ERR_OPT, "Newton line search exceeded MaxEval(%d)", max_eval);
    double d1, d2;
    SE_TRY(se_gbm_linesearch_eval2(ctx, x, &f, &d1, &d2));
    ++evals;
    // the objective is convex along the line: the sign of the slope brackets the minimiser
    if (d1 > 0.0) b = x; else a = x;
    if ((x <= lo && d1 >= 0.0) || (x >= hi && d1 <= 0.0) || d1 == 0.0) break;  // boundary or stationary
    double xn = (d2 > 0.0) ? x - d1 / d2 : 0.5 * (a + b);
    // a Newton step that leaves the interval through an end that has not been evaluated yet: try that end
    // (a boundary minimum is then confirmed in one pass instead of ~20 bisections); otherwise bisect
    if (xn <= a) xn = (a == lo && x != lo) ? lo : 0.5 * (a + b);
    else if (xn >= b) xn = (b == hi && x != hi) ? hi : 0.5 * (a + b);
    if (fabs(xn - x) <= rel * fabs(x) + abs_tol) break;  // x is within tolerance of the minimiser
    x = xn;
  }
  *alpha = x;
  if (loss) *loss = f;
  if (n_eval) *n_eval = evals;
  return SE_OK;
}

int se_gbm_round_squared_async(se_ctx* ctx, double learning_rate) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, ctx->gbm.on && ctx->gbm.loss == SE_LOSS_SQUARED, SE_ERR_STATE, "squared loss only");
  SE_TRY(begin(ctx));
  SE_TRY(settle_f(ctx));
  ctx->gbm.sq_stats_current = false;  // R is rewritten
  GbmArgs a = gbm_args(ctx, false);
  a.stats_from_r = ctx->gbm.r_current ? 1 : 0;
  a.ws = red_ws(ctx, kScalRound);  // stats -> d_scal[kScalRound..+2]
  SE_LAUNCH_T(ctx, SE_KF_SQ_STATS, launch_gbm(SE_LOSS_SQUARED, GBM_SQ_STATS, a, ctx->ctas_per_sm, ctx->sms, ctx->stream));
  SE_TRY(allreduce_dev(ctx, kScalRound, 3));
  GbmArgs u = gbm_args(ctx, false);
  u.dev_stats = ctx->d_scal + kScalRound;
  u.lr = (float)learning_rate;
  u.ws = red_ws(ctx, kScalRound + 8);  // Σloss -> d_scal[kScalRound + 8]
  SE_LAUNCH_T(ctx, SE_KF_UPDATE, launch_gbm(SE_LOSS_SQUARED, GBM_UPDATE_RESID, u, ctx->ctas_per_sm, ctx->sms, ctx->stream));
  SE_TRY(allreduce_dev(ctx, kScalRound + 8, 1));
  ctx->gbm.r_current = true;
  return end(ctx);
}

int se_gbm_round_result(se_ctx* ctx, double* alpha, double* loss_sum) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_CUDA(ctx, cudaMemcpyAsync(ctx->h_scal + kScalRound, ctx->d_scal + kScalRound, sizeof(double) * 16,
                               cudaMemcpyDeviceToHost, ctx->stream));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const double s1 = ctx->h_scal[kScalRound + 1], s2 = ctx->h_scal[kScalRound + 2];
  double al = (s2 > 0.0) ? s1 / s2 : 1.0;
  al = fmin(fmax(al, 0.0), 100.0);
  if (alpha) *alpha = al;
  if (loss_sum) *loss_sum = ctx->h_scal[kScalRound + 8];
  return SE_OK;
}

int se_brent_minimize(se_fn1 f, void* user, double lo, double hi, double start, double rel, double abs_tol,
                      int max_eval, double* x_out, double* f_out, int* n_eval) {
  if (!f) return fail(nullptr, SE_ERR_ARG, "null objective");
  // commons-math3 BrentOptimizer constructor checks
  if (rel < 2.0 * 2.220446049250313e-16) return fail(nullptr, SE_ERR_ARG, "relative threshold %g too small", rel);
  if (abs_tol <= 0.0) return fail(nullptr, SE_ERR_ARG, "absolute threshold must be > 0");
  int rc = brent_impl(f, user, lo, hi, start, rel, abs_tol, max_eval, x_out, f_out, n_eval);
  if (rc != SE_OK) return fail(nullptr, rc, "Brent exceeded MaxEval(%d)", max_eval);
  return SE_OK;
}
