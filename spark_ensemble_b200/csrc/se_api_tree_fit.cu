// se_api_tree_fit.cu — host side of the device tree fits: regression, classification and forests of trees.
#include "se_ctx.h"

using namespace se;
using namespace se_host;

// ---- regression-tree fit over the rank matrix (se_tree_fit.cu) -----------------------------------
int se_tree_fit_bins(se_ctx* ctx, int n_cols, const int32_t* offsets, const float* thresholds) {
  if (!ctx || !offsets) return fail(ctx, SE_ERR_ARG, "null argument");
  const SlotBuf& X = ctx->slot[SE_SLOT_X];
  SE_REQUIRE(ctx, X.d && X.cols > 0, SE_ERR_STATE, "feature matrix slot not allocated");
  SE_REQUIRE(ctx, n_cols == X.rows, SE_ERR_ARG, "%d candidate lists for a feature matrix of %lld columns", n_cols, (long long)X.rows);
  SE_REQUIRE(ctx, X.rows <= 65535, SE_ERR_ARG, "the rank matrix holds at most 65535 columns");
  SE_REQUIRE(ctx, offsets[0] == 0, SE_ERR_ARG, "offsets[0] must be 0");
  for (int c = 0; c < n_cols; ++c) {
    const int32_t b = offsets[c], m = offsets[c + 1] - offsets[c];
    SE_REQUIRE(ctx, m >= 0 && m <= 255, SE_ERR_ARG, "column %d: %d candidates (0..255 supported)", c, m);
    SE_REQUIRE(ctx, m == 0 || thresholds, SE_ERR_ARG, "null thresholds");
    for (int i = 0; i < m; ++i) {
      SE_REQUIRE(ctx, isfinite(thresholds[b + i]), SE_ERR_ARG, "column %d: candidate %d is not finite", c, i);
      SE_REQUIRE(ctx, i == 0 || thresholds[b + i - 1] < thresholds[b + i], SE_ERR_ARG,
                 "column %d: candidates are not strictly increasing at %d", c, i);
    }
  }
  SE_TRY(begin(ctx));
  BinState& B = ctx->bins[0];
  SE_REQUIRE(ctx, bins_ensure(B, X), SE_ERR_CUDA, "no device memory for the rank matrix (%lld x %lld bytes)",
             (long long)X.rows, (long long)X.cols);
  for (int c = 0; c < n_cols; ++c) {
    B.edges[c].assign(thresholds ? thresholds + offsets[c] : nullptr, thresholds ? thresholds + offsets[c + 1] : nullptr);
    B.dirty[c] = 1;
    B.fit[c] = 1;
  }
  SE_TRY(bins_rerank(ctx, B, X));
  return end(ctx);
}

namespace {
// What the local part of a fit (tree_fit_prepare) hands to its level loop.
struct TreeFitPlan {
  const float *r = nullptr, *w = nullptr, *bag = nullptr;
  float* out = nullptr;
  int64_t n = 0, nw = 0, ld_out = 0;
  int nb = 0, sw = 0, top = 0;
  int n_trees = 0, total_cols = 0, max_cols = 0;  // the trees' subspaces: summed and largest size
  uint32_t hash = 0;  // 24 bits: the subspace, its columns' candidates and the validity rules
};

// The rank matrix holds the split candidates of a fit for the feature matrix as it is now.
int tree_fit_bins_ready(se_ctx* ctx) {
  const SlotBuf& X = ctx->slot[SE_SLOT_X];
  SE_REQUIRE(ctx, X.d && X.cols > 0, SE_ERR_STATE, "feature matrix slot not allocated");
  const BinState& B = ctx->bins[0];
  SE_REQUIRE(ctx, B.d8 && B.d == X.rows && B.n == X.cols, SE_ERR_STATE,
             "no split candidates for this feature matrix: call se_tree_fit_bins first");
  return SE_OK;
}

// One tree's subspace (cols null: columns 0 .. S - 1); tree >= 0 names the tree of a forest fit in the messages.
int tree_fit_check_subspace(se_ctx* ctx, const int32_t* cols, int S, int tree) {
  char who[32] = "";
  if (tree >= 0) snprintf(who, sizeof(who), "tree %d: ", tree);
  SE_REQUIRE(ctx, S >= 1, SE_ERR_ARG, "%sempty subspace", who);
  const SlotBuf& X = ctx->slot[SE_SLOT_X];
  const BinState& B = ctx->bins[0];
  for (int k = 0; k < S; ++k) {
    const int32_t c = cols ? cols[k] : k;
    SE_REQUIRE(ctx, c >= 0 && c < X.rows, SE_ERR_ARG, "%ssubspace entry %d: column %d outside X with %lld columns", who,
               k, c, (long long)X.rows);
    SE_REQUIRE(ctx, B.fit[c], SE_ERR_STATE,
               "%scolumn %d does not hold the fit's split candidates (never set, or a tree walk added a threshold to "
               "it): call se_tree_fit_bins again", who, c);
  }
  return SE_OK;
}

// FNV-1a over 32-bit words
inline uint32_t fnv_words(uint32_t h, const void* p, size_t words) {
  const uint32_t* q = static_cast<const uint32_t*>(p);
  for (size_t i = 0; i < words; ++i)
    for (int b = 0; b < 4; ++b) h = (h ^ ((q[i] >> (8 * b)) & 0xFFu)) * 16777619u;
  return h;
}

// The checks, the scratch and the uploads of a fit of n_trees trees, tree t over sub_cols[sub_off[t] .. sub_off[t + 1])
// (sub_cols null: columns 0 .. S - 1 of the one tree): everything that depends on this rank alone.  Under a
// communicator its failure is not returned to the caller straight away: tree_fit_agree tells every rank first.
// with_out: the fit writes every row's output into out_slot (the forest fit writes none).  first_tree: the index of
// tree 0 in a forest fit's messages (-1: a one-tree fit, whose messages name no tree).
int tree_fit_prepare(se_ctx* ctx, int K, int entropy, int out_proba, int label_slot, int label_row, int weight_slot,
                     int weight_row, int use_bag, int n_trees, int first_tree, const int32_t* sub_off,
                     const int32_t* sub_cols, int max_depth, int min_instances, double min_info_gain,
                     double min_weight_fraction, bool with_out, int out_slot, int out_row, TreeFitPlan& P) {
  SE_REQUIRE(ctx, max_depth >= 0 && max_depth <= 8, SE_ERR_ARG, "maxDepth %d outside [0, 8]", max_depth);
  SE_REQUIRE(ctx, min_instances >= 1, SE_ERR_ARG, "minInstancesPerNode %d < 1", min_instances);
  SE_REQUIRE(ctx, min_weight_fraction >= 0.0 && min_weight_fraction < 0.5, SE_ERR_ARG,
             "minWeightFractionPerNode %g outside [0, 0.5)", min_weight_fraction);
  SE_REQUIRE(ctx, !isnan(min_info_gain), SE_ERR_ARG, "minInfoGain is NaN");
  const SlotBuf& X = ctx->slot[SE_SLOT_X];
  SE_REQUIRE(ctx, X.d && X.cols > 0, SE_ERR_STATE, "feature matrix slot not allocated");
  const int64_t n = X.cols;
  auto row_of = [&](int slot, int row, const char* what, const float** p) -> int {
    SE_REQUIRE(ctx, slot >= 0 && slot < SE_NUM_SLOTS, SE_ERR_ARG, "bad %s slot %d", what, slot);
    const SlotBuf& s = ctx->slot[slot];
    SE_REQUIRE(ctx, s.d && s.cols == n && row >= 0 && row < s.rows, SE_ERR_STATE, "%s slot %d: no row %d of %lld values", what,
               slot, row, (long long)n);
    *p = s.d + (int64_t)row * s.ld;
    return SE_OK;
  };
  const float *r = nullptr, *w = nullptr, *bag = nullptr;
  SE_TRY(row_of(label_slot, label_row, "label", &r));
  if (weight_slot >= 0) SE_TRY(row_of(weight_slot, weight_row, "weight", &w));
  if (use_bag) SE_TRY(row_of(SE_SLOT_BAG, 0, "bag", &bag));
  SE_REQUIRE(ctx, sub_off[0] == 0 && sub_off[n_trees] - sub_off[0] >= 1, SE_ERR_ARG, "empty subspace");
  SE_TRY(tree_fit_bins_ready(ctx));
  BinState& B = ctx->bins[0];
  const int total = sub_off[n_trees];
  std::vector<int32_t> cols((size_t)total + (size_t)n_trees + 1);  // the columns, then the offsets: one upload
  int maxc = 0, maxS = 0;
  for (int t = 0; t < n_trees; ++t) {
    const int S = sub_off[t + 1] - sub_off[t];
    SE_TRY(tree_fit_check_subspace(ctx, sub_cols ? sub_cols + sub_off[t] : nullptr, S, first_tree >= 0 ? first_tree + t : -1));
    maxS = std::max(maxS, S);
    for (int k = sub_off[t]; k < sub_off[t + 1]; ++k) {
      const int32_t c = sub_cols ? sub_cols[k] : k;
      cols[k] = c;
      maxc = std::max(maxc, (int)B.edges[c].size());
    }
  }
  for (int t = 0; t <= n_trees; ++t) cols[(size_t)total + t] = sub_off[t];
  const int nb = std::min(256, maxc + 2);  // ranks 0..maxc, then NaN (rank 255) in the last bin
  SE_TRY(begin(ctx));
  SE_TRY(read_slot(ctx, label_slot));
  SE_TRY(read_slot(ctx, weight_slot));
  SE_TRY(bins_rerank(ctx, B, X));  // X was rewritten since the candidates were set
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // h_small is reused below
  // ---- scratch
  auto& T = ctx->tf;
  const int64_t nw = (n + 3) >> 2;
  SE_CUDA(ctx, T.d_nid.grow(2 * 4 * (size_t)nw * (size_t)n_trees));
  const int top = max_depth > 0 ? max_depth - 1 : 0;  // deepest level that is searched (or, at depth 0, only summed)
  const int sw = K > 0 ? K + (w ? 1 : 0) : 4;  // doubles per histogram bin
  const size_t hist_bytes = ((size_t)1 << top) * (size_t)total * (size_t)nb * (size_t)sw * sizeof(double);
  SE_CUDA(ctx, T.d_hist.grow(hist_bytes / sizeof(double)));
  SE_CUDA(ctx, T.d_nodes.grow(kTreeFitHeap * (size_t)n_trees));
  SE_CUDA(ctx, T.d_dec.grow(kTreeFitHeap * (size_t)n_trees));
  if (!T.smem_optin)
    SE_CUDA(ctx, cudaDeviceGetAttribute(&T.smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
  if (K > 0) {
    SE_CUDA(ctx, T.d_cw.grow(kTreeFitHeap * kTreeFitMaxClasses * (size_t)n_trees));
    SE_CUDA(ctx, T.d_prob.grow(kTreeFitHeap * kTreeFitMaxClasses * (size_t)n_trees));
    SE_CUDA(ctx, T.d_prn.grow(kTreeFitHeap * (size_t)n_trees));
  }
  const int ncols = (int)cols.size();
  SE_CUDA(ctx, T.d_cols.grow((size_t)ncols));
  SE_REQUIRE(ctx, sizeof(int32_t) * (size_t)ncols <= (size_t)kSmallBytes, SE_ERR_ARG, "subspace too large");
  memcpy(ctx->h_small, cols.data(), sizeof(int32_t) * (size_t)ncols);
  SE_CUDA(ctx, cudaMemcpyAsync(T.d_cols, ctx->h_small, sizeof(int32_t) * (size_t)ncols, cudaMemcpyHostToDevice, ctx->stream));
  if (K > 0 && label_slot == SE_SLOT_Y) SE_TRY(ensure_labels_checked(ctx, 0, K, n));  // class indices, checked per upload
  cols.resize((size_t)total);
  uint32_t h = 2166136261u;
  h = fnv_words(h, cols.data(), cols.size());
  for (int32_t c : cols) {
    const uint32_t m = (uint32_t)B.edges[c].size();
    h = fnv_words(h, &m, 1);
    h = fnv_words(h, B.edges[c].data(), m);
  }
  const int32_t rules[2] = {min_instances, entropy};
  const double frac[2] = {min_info_gain, min_weight_fraction};
  h = fnv_words(h, rules, 2);
  h = fnv_words(h, frac, sizeof(frac) / 4);
  // after the re-rank of X and the label check above: the output rows may be rows of X or Y themselves
  if (with_out) SE_TRY(out_rows(ctx, out_slot, out_row, out_proba ? K : 1, n, &P.out, &P.ld_out));
  P.r = r; P.w = w; P.bag = bag;
  P.n = n; P.nw = nw; P.nb = nb; P.sw = sw; P.top = top;
  P.n_trees = n_trees; P.total_cols = total; P.max_cols = maxS;
  P.hash = (h ^ (h >> 24)) & 0xFFFFFFu;
  return SE_OK;
}

// Under a communicator of two or more ranks, one max all-reduce of the fit's shape and of its negation, before the
// first histogram collective: every rank learns the minimum and maximum of each entry, and every rank fails when one
// rank failed its own checks (rc) or when any entry differs.  Without it a rank that stops alone would leave its peers
// blocked in the first histogram all-reduce.  The failing rank keeps its own error; its peers get SE_ERR_ARG.
int tree_fit_agree(se_ctx* ctx, int rc, const double* shape, int count) {
  static const char* const names[] = {"failed", "maxDepth", "the subspace size", "the bins per column",
                                      "the doubles per bin", "numClasses", "the weights", "the bag",
                                      "the subspace, its candidates or the validity rules (hash)"};
  constexpr int kMax = 16;
  const std::string local = ctx->err;
  double v[2 * kMax];
  for (int i = 0; i < count; ++i) {
    v[i] = i == 0 ? (rc != SE_OK ? 1.0 : 0.0) : shape[i];
    v[count + i] = -v[i];
  }
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  for (int i = 0; i < 2 * count; ++i) ctx->h_scal[kScalHost + i] = v[i];
  SE_CUDA(ctx, cudaMemcpyAsync(ctx->d_scal + kScalHost, ctx->h_scal + kScalHost, sizeof(double) * 2 * count,
                               cudaMemcpyHostToDevice, ctx->stream));
  NcclApi& api = nccl();
  const int nr = api.AllReduce(ctx->d_scal + kScalHost, ctx->d_scal + kScalHost, (size_t)(2 * count), kNcclFloat64,
                               kNcclMax, ctx->comm, ctx->stream);
  if (nr != 0) return fail(ctx, SE_ERR_NCCL, "ncclAllReduce: %s", api.GetErrorString(nr));
  SE_CUDA(ctx, cudaMemcpyAsync(ctx->h_scal + kScalHost, ctx->d_scal + kScalHost, sizeof(double) * 2 * count,
                               cudaMemcpyDeviceToHost, ctx->stream));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < 2 * count; ++i) v[i] = ctx->h_scal[kScalHost + i];
  if (rc != SE_OK) return fail(ctx, rc, "%s", local.c_str());
  SE_REQUIRE(ctx, v[0] == 0.0, SE_ERR_ARG, "ranks disagree on the fit: another rank failed its own checks");
  for (int i = 1; i < count; ++i)
    SE_REQUIRE(ctx, v[i] == -v[count + i], SE_ERR_ARG, "ranks disagree on the fit: %s is %.17g on one rank, %.17g on another",
               names[i], -v[count + i], v[i]);
  return SE_OK;
}

// Bytes of one tree's node records as tree_fit_run downloads them (K == 0: regression).
size_t tree_fit_record_bytes(int K) {
  return sizeof(TreeFitNode) * kTreeFitHeap +
         (K > 0 ? (sizeof(double) + sizeof(float)) * kTreeFitHeap * (size_t)K + sizeof(int4) * kTreeFitHeap : 0);
}

// The part of a fit that se_tree_fit, se_tree_fit_classifier and se_forest_fit share: argument checks, scratch, the
// level loop with its shared-memory / global-atomics choice, the classifier's pruning, the out kernel (with_out) and
// the download of the n_trees trees' node records into the pinned `records`: [T][kTreeFitHeap] TreeFitNode, then for
// K >= 2 the class weights ([T][kTreeFitHeap][K] double), the probabilities ([T][kTreeFitHeap][K] float) and the
// pruning tables ([T][kTreeFitHeap] int4).  K == 0: regression.  rc0 is the caller's own checks.
//
// The trees grow together: every kernel of the level loop covers all of them, so T trees cost one launch sequence.
// The shared-memory / global-atomics choice depends on the level's 2^L · nb · sw alone, so it is the same for all.
//
// Under a communicator the fit is collective (one tree only): each level's histogram is summed over the ranks (one
// fp64 NCCL all-reduce between the histogram and the split kernels), so every rank splits on the histogram of the
// union of the shards and writes its own rows' output.  The collective sequence is fixed by the shape tree_fit_agree
// checks.
int tree_fit_run(se_ctx* ctx, int rc0, int K, int entropy, int out_proba, int label_slot, int label_row,
                 int weight_slot, int weight_row, int use_bag, int n_trees, int first_tree, const int32_t* sub_off,
                 const int32_t* sub_cols, int max_depth, int min_instances, double min_info_gain,
                 double min_weight_fraction, bool with_out, int out_slot, int out_row, unsigned char* records) {
  TreeFitPlan P;
  int rc = rc0 != SE_OK ? rc0
                        : tree_fit_prepare(ctx, K, entropy, out_proba, label_slot, label_row, weight_slot, weight_row,
                                           use_bag, n_trees, first_tree, sub_off, sub_cols, max_depth, min_instances,
                                           min_info_gain, min_weight_fraction, with_out, out_slot, out_row, P);
  const bool collective = ctx->comm && ctx->nranks > 1;
  if (collective) {
    const double shape[] = {0.0, (double)max_depth, (double)(sub_off[1] - sub_off[0]), (double)P.nb, (double)P.sw,
                            (double)K, P.w ? 1.0 : 0.0, P.bag ? 1.0 : 0.0, (double)P.hash};
    rc = tree_fit_agree(ctx, rc, shape, (int)(sizeof(shape) / sizeof(shape[0])));
  }
  if (rc != SE_OK) return rc;
  // ---- the fit: a fixed sequence of launches, no host round trip
  auto& T = ctx->tf;
  BinState& B = ctx->bins[0];
  const int64_t n = P.n, nw = P.nw;
  const int nb = P.nb, sw = P.sw, top = P.top, nt = P.n_trees, total = P.total_cols, maxS = P.max_cols;
  const float *r = P.r, *w = P.w, *bag = P.bag;
  TreeFitArgs a;
  a.X8 = B.d8; a.ld8 = B.ld8; a.n = n;
  a.cols = T.d_cols; a.n_edges = B.d_nedges; a.edges = B.d_edges;
  a.S = maxS; a.nb = nb; a.max_depth = max_depth; a.search = max_depth > 0 ? 1 : 0;
  a.has_w = w ? 1 : 0; a.r = r; a.w = w; a.bag = bag;
  a.dec = T.d_dec; a.nodes = T.d_nodes; a.hist = T.d_hist;
  a.min_instances = min_instances; a.min_info_gain = min_info_gain; a.min_weight_fraction = min_weight_fraction;
  a.K = K; a.sw = sw; a.entropy = entropy; a.out_proba = out_proba;
  a.cw = T.d_cw; a.prob = T.d_prob; a.prn = T.d_prn;
  a.T = nt; a.sub_off = T.d_cols + total; a.nid_stride = 2 * 4 * nw;
  uint16_t* nid[2] = {T.d_nid, T.d_nid + 4 * nw};
  SE_LAUNCH_T(ctx, SE_KF_TREE, launch_tree_fit_init(T.d_nodes, T.d_dec, nt, ctx->stream));
  ctx->last_tree_fit_hist = 0;
  for (int L = 0; L <= top; ++L) {
    a.L = L;
    a.route = L >= 1;
    a.nid_in = L >= 2 ? nid[(L - 1) & 1] : nullptr;
    a.nid_out = L >= 1 ? nid[L & 1] : nullptr;
    const size_t per_col = ((size_t)1 << L) * (size_t)nb * (size_t)sw * sizeof(double);
    SE_CUDA(ctx, cudaMemsetAsync(T.d_hist, 0, per_col * (size_t)total, ctx->stream));
    int smem_mode = 1, per_sm = 4;
    size_t smem = 0;
    if (per_col <= (size_t)kTreeFitSmemBudget) {
      a.cb = (int)std::min<size_t>((size_t)maxS, kTreeFitSmemBudget / per_col);
    } else if (per_col <= (size_t)T.smem_optin) {
      a.cb = 1;
      per_sm = per_col <= (size_t)T.smem_optin / 2 ? 2 : 1;
    } else {  // one column's histogram of every node of the level does not fit: global fp64 atomics
      smem_mode = 0;
      a.cb = maxS;
      per_sm = 8;
    }
    if (smem_mode) smem = per_col * (size_t)a.cb;
    const int path = !smem_mode ? 4 : per_col > (size_t)kTreeFitSmemBudget ? (per_sm == 2 ? 2 : 3) : (a.cb > 1 ? 0 : 1);
    ctx->last_tree_fit_hist |= (int64_t)path << (3 * L);
    const int gx = smem_mode ? (maxS + a.cb - 1) / a.cb : 1;
    int64_t gy = ((int64_t)ctx->sms * per_sm + gx - 1) / gx;
    // T trees share the grid one tree would use, rounded down: rounding up would leave a few CTAs in a second wave,
    // each with a whole CTA's rows to do alone
    gy = std::max<int64_t>(gy / nt, 1);
    gy = std::min<int64_t>(gy, (nw + 255) / 256);
    gy = std::max<int64_t>(std::min<int64_t>(gy, 65535), 1);
    a.words_per_cta = (nw + gy - 1) / gy;
    SE_LAUNCH_T(ctx, SE_KF_TREE, launch_tree_fit_hist(a, smem_mode, (int)gy, smem, ctx->stream));
    if (collective) {  // the level's histogram over the union of the shards, bit-identical on every rank
      NcclApi& api = nccl();
      const int nr = api.AllReduce(T.d_hist, T.d_hist, per_col / sizeof(double) * (size_t)total, kNcclFloat64,
                                   kNcclSum, ctx->comm, ctx->stream);
      if (nr != 0) return fail(ctx, SE_ERR_NCCL, "ncclAllReduce: %s", api.GetErrorString(nr));
    }
    SE_LAUNCH_T(ctx, SE_KF_TREE, launch_tree_fit_split(a, ctx->stream));
  }
  a.route = max_depth >= 1;
  a.nid_in = max_depth >= 2 ? nid[(max_depth - 1) & 1] : nullptr;
  a.nid_out = nullptr;
  a.out = P.out;
  a.ld_out = P.ld_out;
  if (K > 0) SE_LAUNCH_T(ctx, SE_KF_TREE, launch_tree_fit_prune(a, ctx->stream));
  if (with_out) SE_LAUNCH_T(ctx, SE_KF_TREE, launch_tree_fit_out(a, ctx->sms, ctx->stream));
  char* hs = reinterpret_cast<char*>(records);
  size_t off = sizeof(TreeFitNode) * kTreeFitHeap * (size_t)nt;
  SE_CUDA(ctx, cudaMemcpyAsync(hs, T.d_nodes, off, cudaMemcpyDeviceToHost, ctx->stream));
  if (K > 0) {
    const size_t cwb = sizeof(double) * kTreeFitHeap * (size_t)K * nt, pb = sizeof(float) * kTreeFitHeap * (size_t)K * nt;
    SE_CUDA(ctx, cudaMemcpyAsync(hs + off, T.d_cw, cwb, cudaMemcpyDeviceToHost, ctx->stream));
    SE_CUDA(ctx, cudaMemcpyAsync(hs + off + cwb, T.d_prob, pb, cudaMemcpyDeviceToHost, ctx->stream));
    SE_CUDA(ctx, cudaMemcpyAsync(hs + off + cwb + pb, T.d_prn, sizeof(int4) * kTreeFitHeap * nt, cudaMemcpyDeviceToHost,
                                 ctx->stream));
  }
  SE_TRY(end(ctx));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (K > 0) SE_TRY(check_labels(ctx));  // a label outside [0, K) was clamped: the fit is invalid
  return SE_OK;
}

// One regression tree's records R in the array form of se_tree_predict: pruned bottom-up (two leaf children with
// equal fp64 predictions), numbered in BFS order.
int tree_fit_arrays(se_ctx* ctx, const TreeFitNode* R, int max_nodes, int32_t* feature, float* threshold,
                    int32_t* left, int32_t* right, float* value, double* gain, int* n_nodes) {
  std::vector<char> leaf(kTreeFitHeap, 1);
  std::vector<double> pred(kTreeFitHeap, 0.0);
  std::vector<float> val(kTreeFitHeap, 0.f);
  for (int h = 1; h < kTreeFitHeap; ++h) {
    leaf[h] = R[h].state != 2;
    pred[h] = R[h].pred;
    val[h] = R[h].value;
  }
  for (int h = kTreeFitHeap / 2 - 1; h >= 1; --h) {
    if (leaf[h] || !leaf[2 * h] || !leaf[2 * h + 1] || !(pred[2 * h] == pred[2 * h + 1])) continue;
    leaf[h] = 1;
    pred[h] = pred[2 * h];
    val[h] = val[2 * h];
  }
  std::vector<int> order;
  order.push_back(1);
  for (size_t q = 0; q < order.size(); ++q)
    if (!leaf[order[q]]) { order.push_back(2 * order[q]); order.push_back(2 * order[q] + 1); }
  SE_REQUIRE(ctx, (int)order.size() <= max_nodes, SE_ERR_ARG, "the fitted tree has %d nodes, max_nodes is %d",
             (int)order.size(), max_nodes);
  std::vector<int> id(kTreeFitHeap, 0);
  for (size_t q = 0; q < order.size(); ++q) id[order[q]] = (int)q;
  for (size_t q = 0; q < order.size(); ++q) {
    const int h = order[q];
    const bool lf = leaf[h];
    feature[q] = lf ? -1 : R[h].col;
    threshold[q] = lf ? 0.f : R[h].thr;
    left[q] = lf ? 0 : id[2 * h];
    right[q] = lf ? 0 : id[2 * h + 1];
    value[q] = val[h];
    if (gain) gain[q] = lf ? 0.0 : R[h].gain;
  }
  *n_nodes = (int)order.size();
  return SE_OK;
}

// One classification tree's records (pruned on the device by tree_prune_cls_kernel) in the array form of
// se_tree_predict_multi, numbered in BFS order.
int tree_fit_arrays_cls(se_ctx* ctx, const TreeFitNode* R, const double* CW, const float* PR, const int4* PN, int K,
                        int max_nodes, int32_t* feature, float* threshold, int32_t* left, int32_t* right, float* value,
                        float* proba, double* class_weights, double* gain, int* n_nodes) {
  std::vector<int> order;
  order.push_back(1);
  for (size_t q = 0; q < order.size(); ++q)
    if (!PN[order[q]].z) { order.push_back(2 * order[q]); order.push_back(2 * order[q] + 1); }
  SE_REQUIRE(ctx, (int)order.size() <= max_nodes, SE_ERR_ARG, "the fitted tree has %d nodes, max_nodes is %d",
             (int)order.size(), max_nodes);
  std::vector<int> id(kTreeFitHeap, 0);
  for (size_t q = 0; q < order.size(); ++q) id[order[q]] = (int)q;
  for (size_t q = 0; q < order.size(); ++q) {
    const int h = order[q];
    const bool lf = PN[h].z != 0;
    feature[q] = lf ? -1 : R[h].col;
    threshold[q] = lf ? 0.f : R[h].thr;
    left[q] = lf ? 0 : id[2 * h];
    right[q] = lf ? 0 : id[2 * h + 1];
    value[q] = (float)PN[h].y;  // a merged leaf keeps its children's label ...
    for (int k = 0; k < K; ++k) {  // ... and its own statistics
      proba[q * K + k] = PR[(size_t)h * K + k];
      if (class_weights) class_weights[q * K + k] = CW[(size_t)h * K + k];
    }
    if (gain) gain[q] = lf ? 0.0 : R[h].gain;
  }
  *n_nodes = (int)order.size();
  return SE_OK;
}
}  // namespace

int se_tree_fit(se_ctx* ctx, int label_slot, int label_row, int weight_slot, int weight_row, int use_bag,
                const int32_t* subspace, int n_subspace, int max_depth, int min_instances, double min_info_gain,
                double min_weight_fraction, int out_slot, int out_row, int max_nodes, int32_t* feature,
                float* threshold, int32_t* left, int32_t* right, float* value, double* gain, int* n_nodes) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  const int rc0 = (!feature || !threshold || !left || !right || !value || !n_nodes) ? fail(ctx, SE_ERR_ARG, "null argument")
                                                                                    : SE_OK;
  const int32_t sub_off[2] = {0, n_subspace};
  SE_TRY(tree_fit_run(ctx, rc0, 0, 0, 0, label_slot, label_row, weight_slot, weight_row, use_bag, 1, -1, sub_off,
                      subspace, max_depth, min_instances, min_info_gain, min_weight_fraction, true, out_slot, out_row,
                      ctx->h_small));
  return tree_fit_arrays(ctx, reinterpret_cast<const TreeFitNode*>(ctx->h_small.get()), max_nodes, feature, threshold, left,
                         right, value, gain, n_nodes);
}

// ---- classification-tree fit over the rank matrix (se_tree_fit.cu) -------------------------------
int se_tree_fit_classifier(se_ctx* ctx, int label_slot, int label_row, int weight_slot, int weight_row, int use_bag,
                           const int32_t* subspace, int n_subspace, int num_classes, int impurity, int max_depth,
                           int min_instances, double min_info_gain, double min_weight_fraction, int out_kind,
                           int out_slot, int out_row, int max_nodes, int32_t* feature, float* threshold, int32_t* left,
                           int32_t* right, float* value, float* proba, double* class_weights, double* gain,
                           int* n_nodes) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  auto checks = [&]() -> int {  // this rank's own: under a communicator tree_fit_run tells the other ranks
    SE_REQUIRE(ctx, feature && threshold && left && right && value && proba && n_nodes, SE_ERR_ARG, "null argument");
    SE_REQUIRE(ctx, num_classes >= 2 && num_classes <= kTreeFitMaxClasses, SE_ERR_ARG, "numClasses %d outside [2, %d]",
               num_classes, kTreeFitMaxClasses);
    SE_REQUIRE(ctx, impurity == SE_IMPURITY_GINI || impurity == SE_IMPURITY_ENTROPY, SE_ERR_ARG, "bad impurity %d", impurity);
    SE_REQUIRE(ctx, out_kind == SE_TREE_OUT_LABEL || out_kind == SE_TREE_OUT_PROBA, SE_ERR_ARG, "bad output kind %d", out_kind);
    return SE_OK;
  };
  const int K = num_classes;
  static_assert(sizeof(TreeFitNode) * kTreeFitHeap + (sizeof(double) + sizeof(float)) * kTreeFitHeap * kTreeFitMaxClasses +
                        sizeof(int4) * kTreeFitHeap <= (size_t)kSmallBytes,
                "one tree's node records fit the staging buffer");
  const int32_t sub_off[2] = {0, n_subspace};
  SE_TRY(tree_fit_run(ctx, checks(), K, impurity == SE_IMPURITY_ENTROPY, out_kind == SE_TREE_OUT_PROBA, label_slot,
                      label_row, weight_slot, weight_row, use_bag, 1, -1, sub_off, subspace, max_depth, min_instances,
                      min_info_gain, min_weight_fraction, true, out_slot, out_row, ctx->h_small));
  const char* hs = reinterpret_cast<const char*>(ctx->h_small.get());
  const TreeFitNode* R = reinterpret_cast<const TreeFitNode*>(hs);
  const double* CW = reinterpret_cast<const double*>(hs + sizeof(TreeFitNode) * kTreeFitHeap);
  const float* PR = reinterpret_cast<const float*>(CW + (size_t)kTreeFitHeap * K);
  const int4* PN = reinterpret_cast<const int4*>(PR + (size_t)kTreeFitHeap * K);
  return tree_fit_arrays_cls(ctx, R, CW, PR, PN, K, max_nodes, feature, threshold, left, right, value, proba,
                             class_weights, gain, n_nodes);
}

// ---- several trees over the same rows, labels, weights and bag, one subspace each (se_tree_fit.cu) ----------------
int se_forest_fit(se_ctx* ctx, int n_trees, const int32_t* sub_offsets, const int32_t* sub_cols, int label_slot,
                  int label_row, int weight_slot, int weight_row, int use_bag, int num_classes, int impurity,
                  int max_depth, int min_instances, double min_info_gain, double min_weight_fraction, int max_nodes,
                  int32_t* feature, float* threshold, int32_t* left, int32_t* right, float* value, float* proba,
                  double* class_weights, double* gain, int* n_nodes) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, !(ctx->comm && ctx->nranks > 1), SE_ERR_STATE,
             "se_forest_fit does not fit over row-sharded GPUs: call it without a communicator");
  SE_REQUIRE(ctx, n_trees >= 1 && sub_offsets && sub_cols, SE_ERR_ARG, "null argument or no tree");
  SE_REQUIRE(ctx, feature && threshold && left && right && value && n_nodes, SE_ERR_ARG, "null argument");
  const int K = num_classes;
  SE_REQUIRE(ctx, K == 0 || (K >= 2 && K <= kTreeFitMaxClasses), SE_ERR_ARG,
             "numClasses %d: 0 (regression) or [2, %d]", K, kTreeFitMaxClasses);
  if (K > 0) {
    SE_REQUIRE(ctx, proba, SE_ERR_ARG, "null argument");
    SE_REQUIRE(ctx, impurity == SE_IMPURITY_GINI || impurity == SE_IMPURITY_ENTROPY, SE_ERR_ARG, "bad impurity %d", impurity);
  }
  SE_REQUIRE(ctx, max_nodes >= 1, SE_ERR_ARG, "max_nodes %d < 1", max_nodes);
  SE_REQUIRE(ctx, sub_offsets[0] == 0, SE_ERR_ARG, "sub_offsets[0] must be 0");
  SE_TRY(tree_fit_bins_ready(ctx));
  const BinState& B = ctx->bins[0];
  int maxc = 0;
  for (int t = 0; t < n_trees; ++t) {
    const int S = sub_offsets[t + 1] - sub_offsets[t];
    SE_TRY(tree_fit_check_subspace(ctx, sub_cols + sub_offsets[t], S, t));
    for (int k = sub_offsets[t]; k < sub_offsets[t + 1]; ++k) maxc = std::max(maxc, (int)B.edges[sub_cols[k]].size());
  }
  // ---- batches: at most kBatch trees whose node ids (4 B/row) and deepest histograms take at most half of the free
  // device memory (plus the fit scratch this context already holds, which the batch reuses)
  constexpr int kBatch = 64;
  const int64_t n = ctx->slot[SE_SLOT_X].cols;
  const int64_t nw = (n + 3) >> 2;
  const int top = max_depth > 0 && max_depth <= 8 ? max_depth - 1 : 0;
  const int sw = K > 0 ? K + (weight_slot >= 0 ? 1 : 0) : 4;
  const int nb_all = std::min(256, maxc + 2);
  SE_TRY(begin(ctx));
  size_t free_b = 0, total_b = 0;
  SE_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
  auto& T = ctx->tf;
  const double budget = 0.5 * (double)free_b + (double)(sizeof(double) * T.d_hist.size()) +
                        (double)(sizeof(uint16_t) * T.d_nid.size());
  const size_t rec = tree_fit_record_bytes(K);
  ctx->last_forest_fit_batches = 0;
  std::vector<int32_t> off;
  for (int t0 = 0; t0 < n_trees;) {
    double bytes = 0.0;
    int t1 = t0;
    while (t1 < n_trees && t1 - t0 < kBatch) {
      const int S = sub_offsets[t1 + 1] - sub_offsets[t1];
      const double tree_b = 4.0 * 4.0 * (double)nw + (double)((size_t)1 << top) * S * nb_all * sw * sizeof(double);
      const int cols = sub_offsets[t1 + 1] - sub_offsets[t0] + (t1 + 1 - t0) + 1;  // one upload through h_small
      if (t1 > t0 && (bytes + tree_b > budget || (size_t)cols * sizeof(int32_t) > (size_t)kSmallBytes)) break;
      bytes += tree_b;
      ++t1;
    }
    const int nt = t1 - t0;
    off.assign(sub_offsets + t0, sub_offsets + t1 + 1);
    for (int32_t& o : off) o -= sub_offsets[t0];
    SE_CUDA(ctx, ctx->h_stage.grow((rec * nt + sizeof(float) - 1) / sizeof(float)));
    unsigned char* hs = reinterpret_cast<unsigned char*>(ctx->h_stage.get());
    SE_TRY(tree_fit_run(ctx, SE_OK, K, impurity == SE_IMPURITY_ENTROPY, 0, label_slot, label_row, weight_slot,
                        weight_row, use_bag, nt, t0, off.data(), sub_cols + sub_offsets[t0], max_depth, min_instances,
                        min_info_gain, min_weight_fraction, false, -1, 0, hs));
    ++ctx->last_forest_fit_batches;
    const TreeFitNode* R = reinterpret_cast<const TreeFitNode*>(hs);
    const double* CW = reinterpret_cast<const double*>(R + (size_t)kTreeFitHeap * nt);
    const float* PR = reinterpret_cast<const float*>(CW + (size_t)kTreeFitHeap * K * nt);
    const int4* PN = reinterpret_cast<const int4*>(PR + (size_t)kTreeFitHeap * K * nt);
    for (int i = 0; i < nt; ++i) {
      const size_t t = (size_t)(t0 + i), o = t * (size_t)max_nodes;
      int rc;
      if (K == 0) {
        rc = (tree_fit_arrays(ctx, R + (size_t)kTreeFitHeap * i, max_nodes, feature + o, threshold + o, left + o,
                               right + o, value + o, gain ? gain + o : nullptr, n_nodes + t));
      } else {
        rc = (tree_fit_arrays_cls(ctx, R + (size_t)kTreeFitHeap * i, CW + (size_t)kTreeFitHeap * K * i,
                                   PR + (size_t)kTreeFitHeap * K * i, PN + (size_t)kTreeFitHeap * i, K, max_nodes,
                                   feature + o, threshold + o, left + o, right + o, value + o, proba + o * K,
                                   class_weights ? class_weights + o * K : nullptr, gain ? gain + o : nullptr,
                                   n_nodes + t));
      }
      if (rc != SE_OK) {
        const std::string msg = ctx->err;
        return fail(ctx, rc, "tree %d: %s", (int)t, msg.c_str());
      }
    }
    t0 = t1;
  }
  // the batch's node ids and histograms were sized for up to 64 trees: give them back rather than hold them for the
  // life of the context (the next fit allocates what it needs)
  T.d_nid.reset();
  T.d_hist.reset();
  return SE_OK;
}
