// se_api_trees.cu — host side of the rank matrix and of tree, forest, weighted-median and linear scoring.
#include "se_ctx.h"

using namespace se;
using namespace se_host;

// ---- on-device base models ---------------------------------------------------------------------
namespace se_host {
// Makes the rank matrix of slot X cover every threshold of the given nodes (col[i] < 0: leaf): allocates it on first
// use, inserts new thresholds into the per-column edge lists and re-ranks the columns that changed.  Returns 1 when the
// matrix is ready, 0 when it cannot be used (disabled, no memory, NaN threshold, a column with more than 255 edges).
// Allocates the rank matrix of slot X on first use (or when the slot's shape changed).  False when there is no room.
bool bins_ensure(BinState& B, const SlotBuf& X) {
  const int d = (int)X.rows;
  if (B.d8 && B.d == d && B.n == X.cols) return true;
  B = BinState();
  const int64_t ld8 = ((X.cols + 127) / 128) * 128;
  bool ok = B.d8.grow((size_t)d * (size_t)ld8) == cudaSuccess && B.d_edges.grow(256 * (size_t)d) == cudaSuccess &&
            B.d_nedges.grow((size_t)d) == cudaSuccess && B.d_cols.grow((size_t)d) == cudaSuccess;
  if (!ok) {
    cudaGetLastError();
    B = BinState();
    return false;
  }
  B.ld8 = ld8; B.n = X.cols; B.d = d;
  B.edges.assign((size_t)d, std::vector<float>());
  B.dirty.assign((size_t)d, 0);
  B.fit.assign((size_t)d, 0);
  B.valid = true;
  return true;
}

// Re-ranks every dirty column (and every column with edges when the slot was rewritten)
int bins_rerank(se_ctx* ctx, BinState& B, const SlotBuf& X) {
  const int d = B.d;
  if (!B.valid) {  // the slot was rewritten: every column that has edges must be re-ranked
    for (int c = 0; c < d; ++c) B.dirty[c] = B.edges[c].empty() ? 0 : 1;
    B.valid = true;
  }
  std::vector<int32_t> cols;
  for (int c = 0; c < d; ++c)
    if (B.dirty[c]) cols.push_back(c);
  if (!cols.empty()) {
    std::vector<int32_t> ne((size_t)d);
    for (int c = 0; c < d; ++c) ne[c] = (int32_t)B.edges[c].size();
    for (int32_t c : cols)
      if (!B.edges[c].empty())
        SE_CUDA(ctx, cudaMemcpyAsync(B.d_edges + (size_t)c * 256, B.edges[c].data(), sizeof(float) * B.edges[c].size(), cudaMemcpyHostToDevice, ctx->stream));
    SE_CUDA(ctx, cudaMemcpyAsync(B.d_nedges, ne.data(), sizeof(int32_t) * (size_t)d, cudaMemcpyHostToDevice, ctx->stream));
    SE_CUDA(ctx, cudaMemcpyAsync(B.d_cols, cols.data(), sizeof(int32_t) * cols.size(), cudaMemcpyHostToDevice, ctx->stream));
    SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // the host vectors above go out of scope
    BinArgs b;
    b.X = X.d; b.X8 = B.d8; b.n = X.cols; b.ld = X.ld; b.ld8 = B.ld8;
    b.cols = B.d_cols; b.edges = B.d_edges; b.n_edges = B.d_nedges;
    SE_LAUNCH_T(ctx, SE_KF_OTHER, launch_bin_columns(b, (int)cols.size(), ctx->sms, ctx->stream));
    for (int32_t c : cols) B.dirty[c] = 0;
    ctx->last_tree_rebinned_cols = (int)cols.size();
  }
  return SE_OK;
}

int bins_prepare(se_ctx* ctx, int which, const SlotBuf& X, int n_nodes, const int32_t* col, const float* thr) {
  ctx->last_tree_rebinned_cols = 0;
  if (!ctx->tree_bins || X.rows > 65535 || X.cols == 0) return 0;
  BinState& B = ctx->bins[which];
  if (!bins_ensure(B, X)) {  // e.g. no room for another d x n bytes: keep walking the fp32 matrix
    ctx->tree_bins = 0;
    return 0;
  }
  for (int i = 0; i < n_nodes; ++i) {
    if (col[i] < 0) continue;
    if (!(thr[i] == thr[i])) return 0;  // NaN threshold: leave it to the fp32 walk
    std::vector<float>& E = B.edges[col[i]];
    auto it = std::lower_bound(E.begin(), E.end(), thr[i]);
    if (it != E.end() && *it == thr[i]) continue;
    if (E.size() >= 255) return 0;      // this column needs more ranks than a byte holds
    E.insert(it, thr[i]);
    B.dirty[col[i]] = 1;
    B.fit[col[i]] = 0;                  // no longer the fit's candidates: se_tree_fit refuses the column
  }
  SE_TRY(bins_rerank(ctx, B, X));
  return 1;
}
}  // namespace se_host

namespace {
// The device walks follow child links until they meet a leaf: anything but a tree rooted at node 0 could send them
// around a cycle forever.  Returns the first node reached twice (a cycle or a DAG) and sets *parent to the node that
// reached it, or -1 for a tree.  Every child index must already lie in [0, n).
int reached_twice(int n, const int32_t* feature, const int32_t* left, const int32_t* right, int* parent) {
  std::vector<char> seen((size_t)n, 0);
  std::vector<int32_t> stack(1, 0);
  seen[0] = 1;
  while (!stack.empty()) {
    const int32_t i = stack.back();
    stack.pop_back();
    if (feature[i] < 0) continue;  // leaf
    for (const int32_t c : {left[i], right[i]}) {
      if (seen[c]) {
        *parent = i;
        return c;
      }
      seen[c] = 1;
      stack.push_back(c);
    }
  }
  return -1;
}

// Walk the uint8 rank matrix instead of the fp32 features when every threshold of the tree fits the per-column edge
// lists (<= 255 per column; Spark's trees draw theirs from the <= maxBins - 1 candidates of findSplits, the same on
// every round).  Returns 1 with the tree staged in bins[which].d_nodes and its internal node count in n_internal, 0
// when the caller must take the fp32 walk.
int tree_nodes_binned(se_ctx* ctx, int which, const SlotBuf& X, int n_nodes, const int32_t* col, const float* thr,
                      const int32_t* left, const int32_t* right, int* n_internal) {
  if (n_nodes > 65535) return 0;
  {
    const int rc = bins_prepare(ctx, which, X, n_nodes, col, thr);
    if (rc <= 0) return rc;
  }
  BinState& B = ctx->bins[which];
  SE_CUDA(ctx, B.d_nodes.grow((size_t)n_nodes));
  std::vector<uint4> nodes((size_t)n_nodes);
  *n_internal = 0;
  for (int i = 0; i < n_nodes; ++i) {
    if (col[i] < 0) { nodes[i] = make_uint4(0u, 0u, 0x80000000u, 0u); continue; }
    ++*n_internal;
    const std::vector<float>& E = B.edges[col[i]];
    const uint32_t j = (uint32_t)(std::lower_bound(E.begin(), E.end(), thr[i]) - E.begin());  // x <= t_j  <=>  rank(x) <= j
    const uint64_t off = (uint64_t)col[i] * (uint64_t)B.ld8;
    nodes[i] = make_uint4((uint32_t)off, (uint32_t)(off >> 32), j, (uint32_t)left[i] | ((uint32_t)right[i] << 16));
  }
  SE_CUDA(ctx, cudaMemcpyAsync(B.d_nodes, nodes.data(), sizeof(uint4) * (size_t)n_nodes, cudaMemcpyHostToDevice, ctx->stream));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return 1;
}
}  // namespace

static int tree_predict_impl(se_ctx* ctx, int which, int n_nodes, const int32_t* feature, const float* threshold,
                             const int32_t* left, const int32_t* right, const float* value, int n_out,
                             const int32_t* subspace, int n_subspace, int out_slot, int out_row) {
  if (!ctx || !feature || !threshold || !left || !right || !value) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, n_out >= 1 && n_out <= 4096, SE_ERR_ARG, "bad leaf width %d", n_out);
  const size_t bytes = (size_t)n_nodes * (16 + 4 * (size_t)n_out);
  SE_REQUIRE(ctx, n_nodes >= 1 && bytes <= (size_t)kSmallBytes && (size_t)n_nodes * 20 <= 200 * 1024,
             SE_ERR_ARG, "tree of %d nodes x %d outputs not supported", n_nodes, n_out);
  const SlotBuf& X = ctx->slot[which ? SE_SLOT_VX : SE_SLOT_X];
  SE_REQUIRE(ctx, X.d, SE_ERR_STATE, "feature matrix slot not allocated");
  SE_TRY(begin(ctx));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  int32_t* hf = reinterpret_cast<int32_t*>(ctx->h_small.get());
  float* ht = reinterpret_cast<float*>(hf + n_nodes);
  int32_t* hl = reinterpret_cast<int32_t*>(ht + n_nodes);
  int32_t* hr = hl + n_nodes;
  float* hv = reinterpret_cast<float*>(hr + n_nodes);
  for (int i = 0; i < n_nodes; ++i) {
    int32_t f = feature[i];
    if (f >= 0) {
      if (subspace) {
        SE_REQUIRE(ctx, f < n_subspace, SE_ERR_ARG, "node %d: feature %d outside subspace of %d", i, f, n_subspace);
        f = subspace[f];
      }
      SE_REQUIRE(ctx, f >= 0 && f < X.rows, SE_ERR_ARG, "node %d: column %d outside X with %lld columns", i, f, (long long)X.rows);
      SE_REQUIRE(ctx, left[i] >= 0 && left[i] < n_nodes && right[i] >= 0 && right[i] < n_nodes, SE_ERR_ARG, "node %d: bad child", i);
    }
    hf[i] = f; ht[i] = threshold[i]; hl[i] = left[i]; hr[i] = right[i];
  }
  int parent = 0;
  const int twice = reached_twice(n_nodes, hf, hl, hr, &parent);
  SE_REQUIRE(ctx, twice < 0, SE_ERR_ARG, "node %d is reached twice (child of node %d): not a tree", twice, parent);
  memcpy(hv, value, sizeof(float) * (size_t)n_nodes * n_out);
  SE_CUDA(ctx, cudaMemcpyAsync(ctx->d_small, ctx->h_small, bytes, cudaMemcpyHostToDevice, ctx->stream));
  int n_internal = 0;
  const int binned = tree_nodes_binned(ctx, which, X, n_nodes, hf, ht, hl, hr, &n_internal);
  if (binned < 0) return binned;
  TreeArgs t;
  // after the rank matrix is prepared: a walk over X into a row of X leaves it invalid
  SE_TRY(out_rows(ctx, out_slot, out_row, n_out, X.cols, &t.out, &t.ld_out));
  t.X = X.d; t.n = X.cols; t.ld = X.ld; t.n_nodes = n_nodes;
  t.feature = reinterpret_cast<const int32_t*>(ctx->d_small.get());
  t.threshold = reinterpret_cast<const float*>(t.feature + n_nodes);
  t.left = reinterpret_cast<const int32_t*>(t.threshold + n_nodes);
  t.right = t.left + n_nodes;
  t.value = reinterpret_cast<const float*>(t.right + n_nodes);
  t.n_out = n_out;
  if (binned) {
    const BinState& B = ctx->bins[which];
    SE_LAUNCH_T(ctx, SE_KF_TREE, launch_tree_predict_binned(t, B.d8, B.d_nodes, n_internal, ctx->tree_mask, ctx->sms, ctx->stream));
  } else {
    SE_LAUNCH_T(ctx, SE_KF_TREE, launch_tree_predict(t, ctx->sms, ctx->stream));
  }
  ctx->last_tree_binned = binned;
  ctx->last_tree_mask = (binned && ctx->tree_mask && n_internal <= 64 && n_nodes <= 256) ? 1 : 0;
  return end(ctx);
}

int se_tree_predict(se_ctx* ctx, int which, int n_nodes, const int32_t* feature, const float* threshold,
                    const int32_t* left, const int32_t* right, const float* value,
                    const int32_t* subspace, int n_subspace, int out_slot, int out_row) {
  return tree_predict_impl(ctx, which, n_nodes, feature, threshold, left, right, value, 1, subspace, n_subspace,
                           out_slot, out_row);
}

int se_tree_predict_multi(se_ctx* ctx, int which, int n_nodes, const int32_t* feature, const float* threshold,
                          const int32_t* left, const int32_t* right, const float* values, int n_out,
                          const int32_t* subspace, int n_subspace, int out_slot) {
  return tree_predict_impl(ctx, which, n_nodes, feature, threshold, left, right, values, n_out, subspace, n_subspace,
                           out_slot, 0);
}

// ---- forests in one pass over the rank matrix (se_forest_predict, se_forest_agg) ----------------------------------
namespace {
// Every member must be a tree rooted at its first node, with tree-local child indices and GLOBAL column indices of X
// (d columns): anything else could send the device walk out of the tree or around a cycle.
int forest_check(se_ctx* ctx, int64_t d, int n_trees, const int32_t* offsets, const int32_t* feature, const int32_t* left,
                 const int32_t* right) {
  SE_REQUIRE(ctx, offsets[0] == 0, SE_ERR_ARG, "offsets[0] must be 0");
  const int64_t total = offsets[n_trees];
  SE_REQUIRE(ctx, total >= n_trees && total <= (1 << 26), SE_ERR_ARG, "bad node count %lld", (long long)total);
  for (int t = 0; t < n_trees; ++t) {
    const int32_t b = offsets[t], nn = offsets[t + 1] - offsets[t];
    SE_REQUIRE(ctx, nn >= 1 && nn <= 65535, SE_ERR_ARG, "tree %d: %d nodes (1..65535 supported)", t, nn);
    for (int i = 0; i < nn; ++i) {
      if (feature[b + i] < 0) continue;
      SE_REQUIRE(ctx, feature[b + i] < d, SE_ERR_ARG, "tree %d node %d: column %d outside X with %lld columns", t, i,
                 feature[b + i], (long long)d);
      SE_REQUIRE(ctx, left[b + i] >= 0 && left[b + i] < nn && right[b + i] >= 0 && right[b + i] < nn, SE_ERR_ARG,
                 "tree %d node %d: bad child", t, i);
    }
    int parent = 0;
    const int twice = reached_twice(nn, feature + b, left + b, right + b, &parent);
    SE_REQUIRE(ctx, twice < 0, SE_ERR_ARG, "tree %d: node %d is reached twice: not a tree", t, twice);
  }
  return SE_OK;
}

// Makes the rank matrix of X cover every threshold of the forest; SE_ERR_STATE when it cannot (a column with more than
// 255 distinct thresholds, a NaN threshold, tree_bins off).
int forest_bins(se_ctx* ctx, int which, const SlotBuf& X, int n_trees, const int32_t* offsets, const int32_t* feature,
                const float* threshold) {
  const int rc = bins_prepare(ctx, which, X, offsets[n_trees], feature, threshold);
  if (rc < 0) return rc;
  SE_REQUIRE(ctx, rc == 1, SE_ERR_STATE,
             "the forest kernel needs the uint8 rank matrix (tree_bins on, <= 255 distinct thresholds per column, no NaN "
             "threshold): evaluate the members with se_tree_predict + se_agg_run instead");
  return SE_OK;
}

// The prologue of the one-pass entry points: the X slot `which` names, checked against the forest, and its rank matrix
// made to cover every threshold of the forest.  *X and *B point into the context.
int forest_prepare(se_ctx* ctx, int which, int n_trees, const int32_t* offsets, const int32_t* feature,
                   const float* threshold, const int32_t* left, const int32_t* right, const SlotBuf** X,
                   const BinState** B) {
  const SlotBuf& x = ctx->slot[which ? SE_SLOT_VX : SE_SLOT_X];
  SE_REQUIRE(ctx, x.d, SE_ERR_STATE, "feature matrix slot not allocated");
  SE_TRY(forest_check(ctx, x.rows, n_trees, offsets, feature, left, right));
  SE_TRY(begin(ctx));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  SE_TRY(forest_bins(ctx, which, x, n_trees, offsets, feature, threshold));
  *X = &x;
  *B = &ctx->bins[which];
  return SE_OK;
}

// Trees [t0, t1) run as one launch; cols are the global columns they use (local column c = cols[c]).
struct ForestChunk {
  int t0 = 0, t1 = 0;
  size_t nodes = 0;
  std::vector<int32_t> cols;
};

size_t forest_pad(size_t v, size_t to) { return (v + to - 1) / to * to; }

// Blob layout of a chunk (ForestArgs): T trees, C columns, Nn nodes, with or without the per-tree class array.
void forest_layout(size_t T, size_t C, size_t Nn, bool cls, ForestArgs& a) {
  a.T = (int)T; a.C = (int)C;
  a.off_coloff = (int)(8 * T);
  a.off_nodes = a.off_coloff + (int)(8 * C);
  a.off_treeoff = a.off_nodes + (int)(8 * Nn);
  a.off_treecls = cls ? a.off_treeoff + (int)forest_pad(4 * (T + 1), 8) : 0;
  a.off_values = (cls ? a.off_treecls + (int)forest_pad(4 * T, 8) : a.off_treeoff + (int)forest_pad(4 * (T + 1), 8));
  a.blob_bytes = (int)forest_pad((size_t)a.off_values + 4 * Nn, 16);
  a.off_ranks = a.blob_bytes;
}

// Cuts the forest into chunks of consecutive trees whose blob, plus the ranks of their columns ([C][tile] bytes), plus
// `fixed` bytes the kernel keeps for itself fit one CTA's shared memory.  A chunk grows tree by tree under the
// four-CTAs-per-SM budget; a member that does not fit it alone gets two, then one CTA per SM.
int forest_plan(se_ctx* ctx, int64_t d, int n_trees, const int32_t* offsets, const int32_t* feature, bool cls, int tile,
                size_t fixed, std::vector<ForestChunk>& chunks, size_t first_budget = kForestSmemBudget) {
  chunks.clear();
  std::vector<int32_t> local((size_t)d, -1);  // global column -> local column of the current chunk
  std::vector<int32_t> used;
  int t0 = 0;
  while (t0 < n_trees) {
    size_t nodes = 0;
    int t1 = t0;
    for (const size_t budget : {first_budget, std::max(first_budget, (size_t)(100 * 1024)), (size_t)(216 * 1024)}) {
      for (int32_t c : used) local[c] = -1;
      used.clear();
      nodes = 0;
      for (t1 = t0; t1 < n_trees; ++t1) {
        const int32_t b = offsets[t1], nn = offsets[t1 + 1] - offsets[t1];
        std::vector<int32_t> added;
        for (int i = 0; i < nn; ++i) {
          const int32_t c = feature[b + i];
          if (c >= 0 && local[c] < 0) { local[c] = (int32_t)(used.size() + added.size()); added.push_back(c); }
        }
        ForestArgs a;
        forest_layout((size_t)(t1 - t0 + 1), used.size() + added.size(), nodes + (size_t)nn, cls, a);
        const size_t bytes = (size_t)a.blob_bytes + (size_t)a.C * tile + fixed;
        if (bytes > budget || a.C > 65535) {
          for (int32_t c : added) local[c] = -1;
          break;
        }
        used.insert(used.end(), added.begin(), added.end());
        nodes += (size_t)nn;
      }
      if (t1 > t0) break;
    }
    SE_REQUIRE(ctx, t1 > t0, SE_ERR_ARG, "tree %d alone (%d nodes) does not fit the forest kernel's shared memory", t0,
               offsets[t0 + 1] - offsets[t0]);
    ForestChunk ch;
    ch.t0 = t0; ch.t1 = t1; ch.nodes = nodes; ch.cols = used;
    chunks.push_back(std::move(ch));
    t0 = t1;
  }
  return SE_OK;
}

// Packs a chunk (weights NULL: all 1; tree_class NULL: no class array) into `blob` and sets the layout fields of `a`.
void forest_pack_chunk(const BinState& B, const ForestChunk& ch, const int32_t* offsets, const int32_t* feature,
                       const float* threshold, const int32_t* left, const int32_t* right, const float* value,
                       const double* weights, const int32_t* tree_class, ForestArgs& a, std::vector<unsigned char>& blob) {
  const size_t T = (size_t)(ch.t1 - ch.t0), C = ch.cols.size();
  forest_layout(T, C, ch.nodes, tree_class != nullptr, a);
  blob.assign((size_t)a.blob_bytes, 0);
  std::vector<int32_t> local((size_t)B.d, -1);
  for (size_t c = 0; c < C; ++c) local[ch.cols[c]] = (int32_t)c;
  double* bw = reinterpret_cast<double*>(blob.data());
  unsigned long long* bco = reinterpret_cast<unsigned long long*>(blob.data() + a.off_coloff);
  uint2* bn = reinterpret_cast<uint2*>(blob.data() + a.off_nodes);
  int32_t* bto = reinterpret_cast<int32_t*>(blob.data() + a.off_treeoff);
  int32_t* bcl = reinterpret_cast<int32_t*>(blob.data() + a.off_treecls);
  float* bv = reinterpret_cast<float*>(blob.data() + a.off_values);
  for (size_t c = 0; c < C; ++c) bco[c] = (unsigned long long)ch.cols[c] * (unsigned long long)B.ld8;
  size_t at = 0;
  for (int t = ch.t0; t < ch.t1; ++t) {
    const int32_t b = offsets[t], nn = offsets[t + 1] - offsets[t];
    bw[t - ch.t0] = weights ? weights[t] : 1.0;
    bto[t - ch.t0] = (int32_t)at;
    if (tree_class) bcl[t - ch.t0] = tree_class[t];
    for (int i = 0; i < nn; ++i) {
      const int32_t c = feature[b + i];
      bv[at + i] = value[b + i];
      if (c < 0) { bn[at + i] = make_uint2(0x80000000u, 0u); continue; }
      const std::vector<float>& E = B.edges[c];
      const uint32_t j = (uint32_t)(std::lower_bound(E.begin(), E.end(), threshold[b + i]) - E.begin());  // x <= t_j <=> rank <= j
      bn[at + i] = make_uint2((uint32_t)local[c] | (j << 16), (uint32_t)left[b + i] | ((uint32_t)right[b + i] << 16));
    }
    at += (size_t)nn;
  }
  bto[T] = (int32_t)at;
}

// Copies `bytes` of pageable host memory into ctx->d_forest.  Returns once the copy is done: the previous chunk's kernel
// may still be reading d_forest before it, and the next chunk reuses it after it.
int forest_upload(se_ctx* ctx, const unsigned char* host, size_t bytes) {
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  SE_CUDA(ctx, ctx->d_forest.grow(bytes));
  SE_CUDA(ctx, cudaMemcpyAsync(ctx->d_forest, host, bytes, cudaMemcpyHostToDevice, ctx->stream));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return SE_OK;
}

// Packs a chunk into ctx->d_forest and sets the layout fields of `a`.
int forest_upload_chunk(se_ctx* ctx, const BinState& B, const ForestChunk& ch, const int32_t* offsets,
                        const int32_t* feature, const float* threshold, const int32_t* left, const int32_t* right,
                        const float* value, const double* weights, const int32_t* tree_class, ForestArgs& a) {
  std::vector<unsigned char> blob;
  forest_pack_chunk(B, ch, offsets, feature, threshold, left, right, value, weights, tree_class, a, blob);
  SE_TRY(forest_upload(ctx, blob.data(), blob.size()));
  a.blob = ctx->d_forest;
  a.X8 = B.d8; a.ld8 = B.ld8;
  return SE_OK;
}
}  // namespace

// Σ_t weights[t] · tree_t(x) + init for every row in one pass over the rank matrix per chunk of trees
// (GBMRegressionModel.predict, regression/GBMRegressor.scala:531-539; BaggingRegressionModel.predict,
// regression/BaggingRegressor.scala:221-228 with weights 1 / M).
int se_forest_predict(se_ctx* ctx, int which, int n_trees, const int32_t* offsets, const int32_t* feature,
                      const float* threshold, const int32_t* left, const int32_t* right, const float* value,
                      const double* weights, double init, int out_slot, int out_row) {
  if (!ctx || !offsets || !feature || !threshold || !left || !right || !value) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, n_trees >= 1 && n_trees <= (1 << 20), SE_ERR_ARG, "bad tree count %d", n_trees);
  const SlotBuf* xs;
  const BinState* bs;
  SE_TRY(forest_prepare(ctx, which, n_trees, offsets, feature, threshold, left, right, &xs, &bs));
  const SlotBuf& X = *xs;
  const BinState& B = *bs;
  std::vector<ForestChunk> chunks;
  SE_TRY(forest_plan(ctx, X.rows, n_trees, offsets, feature, false, kForestTile, 0, chunks));
  ForestArgs a;
  SE_TRY(out_rows(ctx, out_slot, out_row, 1, X.cols, &a.out, nullptr));  // after forest_bins, as in tree_predict_impl
  a.n = X.cols;
  a.init = init;
  for (size_t k = 0; k < chunks.size(); ++k) {
    SE_TRY(forest_upload_chunk(ctx, B, chunks[k], offsets, feature, threshold, left, right, value, weights, nullptr, a));
    a.accumulate = k > 0 ? 1 : 0;
    SE_LAUNCH_T(ctx, SE_KF_TREE, launch_forest_predict(a, ctx->sms, ctx->stream));
  }
  ctx->last_forest_chunks = (int)chunks.size();
  ctx->last_tree_binned = 1;
  return end(ctx);
}

// A classifier ensemble of trees in one pass with the aggregation's epilogue (see se_abi.h).
int se_forest_agg(se_ctx* ctx, int which, int kind, int num_classes, int dim, int loss, int n_trees, const int32_t* offsets,
                  const int32_t* feature, const float* threshold, const int32_t* left, const int32_t* right,
                  const float* value, const float* probs, const int32_t* tree_class, const double* weights,
                  const double* init) {
  if (!ctx || !offsets || !feature || !threshold || !left || !right || !value) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, n_trees >= 1 && n_trees <= (1 << 20), SE_ERR_ARG, "bad tree count %d", n_trees);
  SE_REQUIRE(ctx, kind == SE_AGG_GBM_CLASSIFIER || kind == SE_AGG_BAGGING_SOFT || kind == SE_AGG_BAGGING_HARD ||
                      kind == SE_AGG_BOOSTING_REAL || kind == SE_AGG_BOOSTING_DISCRETE,
             SE_ERR_ARG, "se_forest_agg serves the classifier kinds (2..6), got %d", kind);
  SE_REQUIRE(ctx, num_classes >= 2 && num_classes <= SE_FOREST_AGG_MAX_CLASSES, SE_ERR_ARG,
             "se_forest_agg supports 2..%d classes, got %d", SE_FOREST_AGG_MAX_CLASSES, num_classes);
  const bool gbm = (kind == SE_AGG_GBM_CLASSIFIER);
  const bool vec = (kind == SE_AGG_BAGGING_SOFT || kind == SE_AGG_BOOSTING_REAL);
  if (gbm) {
    SE_REQUIRE(ctx, dim >= 1 && dim <= SE_FOREST_AGG_MAX_CLASSES && (dim > 1 || num_classes == 2), SE_ERR_ARG,
               "bad dim %d for %d classes", dim, num_classes);
    SE_REQUIRE(ctx, tree_class && weights, SE_ERR_ARG, "the GBM classifier needs tree_class and weights");
    for (int t = 0; t < n_trees; ++t)
      SE_REQUIRE(ctx, tree_class[t] >= 0 && tree_class[t] < dim, SE_ERR_ARG, "tree %d: class %d outside [0, %d)", t,
                 tree_class[t], dim);
  }
  SE_REQUIRE(ctx, !vec || probs, SE_ERR_ARG, "bagging soft / boosting real need the leaf probabilities");
  SE_REQUIRE(ctx, kind != SE_AGG_BOOSTING_DISCRETE || weights, SE_ERR_ARG, "boosting discrete needs the weights");
  const SlotBuf* xs;
  const BinState* bs;
  SE_TRY(forest_prepare(ctx, which, n_trees, offsets, feature, threshold, left, right, &xs, &bs));
  const SlotBuf& X = *xs;
  const BinState& B = *bs;
  const int C = gbm ? dim : num_classes;               // totals per row
  const int out_c = (gbm && dim == 1) ? 2 : C;         // classes of RAW / PROB
  const int64_t n = X.cols;
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_RAW, out_c, n));
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_PROB, out_c, n));
  SE_TRY(slot_alloc2d(ctx, SE_SLOT_LABEL, 1, n));
  std::vector<ForestChunk> chunks;
  SE_TRY(forest_plan(ctx, X.rows, n_trees, offsets, feature, gbm, kForestAggTile,
                     (size_t)C * kForestAggTile * sizeof(double), chunks));
  const int64_t total_nodes = offsets[n_trees];
  if (vec) {  // every node's K probabilities, read by the kernel through L1 at the leaf it reaches
    const size_t need = (size_t)total_nodes * (size_t)num_classes;
    SE_CUDA(ctx, ctx->d_forest_p.grow(need));
    SE_CUDA(ctx, cudaMemcpyAsync(ctx->d_forest_p, probs, sizeof(float) * need, cudaMemcpyHostToDevice, ctx->stream));
  }
  const int64_t ld_acc = ((n + 31) / 32) * 32;
  if (chunks.size() > 1) SE_CUDA(ctx, ctx->d_forest_acc.grow((size_t)C * (size_t)ld_acc));
  // the vote weights are narrowed to fp32 as se_agg_run does, and Σa is the sum of what the kernel adds
  std::vector<double> w((size_t)n_trees, 1.0);
  double sum_a = 0.0;
  for (int t = 0; t < n_trees; ++t) {
    if (kind == SE_AGG_BOOSTING_DISCRETE) w[t] = (double)(float)weights[t];
    else if (gbm) w[t] = weights[t];
    sum_a += w[t];
  }
  ForestAggArgs g;
  g.f.n = n;
  g.kind = kind; g.K = num_classes; g.C = C; g.dim = gbm ? dim : 1; g.loss = loss; g.M = n_trees;
  g.sum_a = sum_a;
  for (int c = 0; c < C; ++c) g.init[c] = (gbm && init) ? init[c] : 0.0;
  g.acc = ctx->d_forest_acc; g.ld_acc = ld_acc;
  const SlotBuf& R = ctx->slot[SE_SLOT_RAW];
  g.raw = R.d; g.prob = ctx->slot[SE_SLOT_PROB].d; g.label = ctx->slot[SE_SLOT_LABEL].d;
  g.ld_out = R.ld;
  g.bad_label = ctx->d_bad_label;
  for (size_t k = 0; k < chunks.size(); ++k) {
    SE_TRY(forest_upload_chunk(ctx, B, chunks[k], offsets, feature, threshold, left, right, value, w.data(),
                               gbm ? tree_class : nullptr, g.f));
    g.probs = vec ? ctx->d_forest_p + (size_t)offsets[chunks[k].t0] * (size_t)num_classes : nullptr;
    g.first = k == 0 ? 1 : 0;
    g.last = k + 1 == chunks.size() ? 1 : 0;
    SE_LAUNCH_T(ctx, SE_KF_TREE, launch_forest_agg(g, ctx->sms, ctx->stream));
  }
  ctx->last_forest_chunks = (int)chunks.size();
  ctx->last_tree_binned = 1;
  SE_TRY(end(ctx));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return check_labels(ctx);  // a leaf label that is not a class index in [0, K)
}

// The weighted median of at most 64 regression trees in one pass, the value se_tree_predict per member into SE_SLOT_P
// followed by se_agg_run(SE_AGG_BOOSTING_REG_MEDIAN) gives (see se_abi.h).
int se_forest_median(se_ctx* ctx, int which, int n_trees, const int32_t* offsets, const int32_t* feature,
                     const float* threshold, const int32_t* left, const int32_t* right, const float* value,
                     const double* weights, int out_slot, int out_row) {
  if (!ctx || !offsets || !feature || !threshold || !left || !right || !value || !weights)
    return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, n_trees >= 1 && n_trees <= SE_FOREST_MEDIAN_MAX_TREES, SE_ERR_ARG,
             "se_forest_median serves 1..%d trees, got %d: evaluate the members with se_tree_predict + se_agg_run",
             SE_FOREST_MEDIAN_MAX_TREES, n_trees);
  const SlotBuf* xs;
  const BinState* bs;
  SE_TRY(forest_prepare(ctx, which, n_trees, offsets, feature, threshold, left, right, &xs, &bs));
  const SlotBuf& X = *xs;
  const BinState& B = *bs;
  const size_t vals_bytes = (size_t)n_trees * kForestMedianTile * sizeof(float);
  // chunks as large as the CTAs its registers let an SM hold can use: every chunk beyond the first re-stages its trees
  // for each tile, and the median's registers (up to 252 at 64 trees) cap the CTAs per SM below four already
  int ctas = 0;
  SE_CUDA(ctx, forest_median_ctas_per_sm(n_trees, &ctas));
  if (ctas > 4) ctas = 4;
  const size_t budget = std::min((size_t)(216 * 1024), (size_t)(228 * 1024) / (size_t)ctas - 1024 - 512 - 16);
  std::vector<ForestChunk> chunks;
  SE_TRY(forest_plan(ctx, X.rows, n_trees, offsets, feature, false, kForestMedianTile, vals_bytes, chunks, budget));
  ForestMedianArgs g;
  SE_TRY(out_rows(ctx, out_slot, out_row, 1, X.cols, &g.out, nullptr));  // after forest_bins, as in tree_predict_impl
  // every chunk's packed trees in one buffer: the kernel walks them all for each tile
  g.n = X.cols;
  g.X8 = B.d8; g.ld8 = B.ld8;
  g.M = n_trees;
  g.n_chunks = (int)chunks.size();
  std::vector<unsigned char> all, blob;
  size_t stage = 0;  // the largest chunk's blob + ranks
  for (size_t k = 0; k < chunks.size(); ++k) {
    ForestArgs a;
    forest_pack_chunk(B, chunks[k], offsets, feature, threshold, left, right, value, nullptr, nullptr, a, blob);
    ForestMedianChunk& c = g.chunk[k];
    c.blob_off = (int)all.size(); c.blob_bytes = a.blob_bytes;
    c.T = a.T; c.C = a.C; c.t0 = chunks[k].t0;
    c.off_coloff = a.off_coloff; c.off_nodes = a.off_nodes; c.off_treeoff = a.off_treeoff; c.off_values = a.off_values;
    all.insert(all.end(), blob.begin(), blob.end());  // blob_bytes is a multiple of 16: every chunk stays aligned
    stage = std::max(stage, (size_t)a.blob_bytes + (size_t)a.C * kForestMedianTile);
  }
  g.vals_off = (int)forest_pad(stage, 16);
  SE_TRY(forest_upload(ctx, all.data(), all.size()));
  g.blob = ctx->d_forest;
  // the weights as se_agg_run takes them: the fast path when every weight is finite and >= 0 (without a margin when
  // they are all equal), the exact sort for every row otherwise
  g.mode = ctx->wm_fast ? wm_weight_mode(weights, n_trees) : 0;
  g.total = 0.0;
  for (int m = 0; m < kForestMedianMaxTrees; ++m) {
    g.w[m] = (m < n_trees) ? weights[m] : 0.0;
    g.total += g.w[m];  // model order, like the kernel's own sums
  }
  g.tau = (g.mode == 1) ? 8.0 * (double)n_trees * 1.1102230246251565e-16 * g.total : -1.0;
  if (g.mode == 1) {
    SE_CUDA(ctx, ctx->d_wm.grow(1));
    SE_CUDA(ctx, cudaMemsetAsync(ctx->d_wm, 0, sizeof(unsigned int), ctx->stream));
    g.deferred = ctx->d_wm;
  }
  SE_LAUNCH_T(ctx, SE_KF_TREE, launch_forest_median(g, (size_t)g.vals_off + vals_bytes, ctx->sms, ctx->stream));
  ctx->last_wm_mode = g.mode;
  ctx->last_forest_chunks = (int)chunks.size();
  ctx->last_tree_binned = 1;
  return end(ctx);
}

int se_linear_predict(se_ctx* ctx, int which, int n_coef, const float* coef, float intercept,
                      const int32_t* subspace, int out_slot, int out_row) {
  if (!ctx || (!coef && n_coef > 0)) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, n_coef >= 0 && (size_t)n_coef * 8 <= (size_t)kSmallBytes, SE_ERR_ARG, "bad coefficient count");
  const SlotBuf& X = ctx->slot[which ? SE_SLOT_VX : SE_SLOT_X];
  SE_REQUIRE(ctx, X.d, SE_ERR_STATE, "feature matrix slot not allocated");
  SE_TRY(begin(ctx));
  float* out = nullptr;
  SE_TRY(out_rows(ctx, out_slot, out_row, 1, X.cols, &out, nullptr));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  float* hc = reinterpret_cast<float*>(ctx->h_small.get());
  int32_t* hcol = reinterpret_cast<int32_t*>(hc + n_coef);
  for (int j = 0; j < n_coef; ++j) {
    hc[j] = coef[j];
    const int32_t col = subspace ? subspace[j] : j;
    SE_REQUIRE(ctx, col >= 0 && col < X.rows, SE_ERR_ARG, "column %d outside X", col);
    hcol[j] = col;
  }
  if (n_coef > 0)
    SE_CUDA(ctx, cudaMemcpyAsync(ctx->d_small, ctx->h_small, (size_t)n_coef * 8, cudaMemcpyHostToDevice, ctx->stream));
  const float* dc = reinterpret_cast<const float*>(ctx->d_small.get());
  const int32_t* dcol = reinterpret_cast<const int32_t*>(dc + n_coef);
  SE_LAUNCH_T(ctx, SE_KF_LINEAR, launch_linear_predict(X.d, X.cols, X.ld, n_coef, dc, dcol, intercept, out, ctx->sms,
                                                       ctx->stream));
  return end(ctx);
}

int se_linear_moments(se_ctx* ctx, int src_slot, int n_cols, const int32_t* cols, const double* shift,
                      double label_shift, int label_slot, int label_row, int weight_slot, int weight_row, int use_bag,
                      double* out) {
  if (!ctx || !out || (n_cols > 0 && !cols)) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, src_slot == SE_SLOT_X || src_slot == SE_SLOT_P, SE_ERR_ARG,
             "source slot %d: only SE_SLOT_X or SE_SLOT_P", src_slot);
  SE_REQUIRE(ctx, n_cols >= 0 && n_cols <= kLinearMomentsMaxCols, SE_ERR_ARG, "%d columns (0..%d supported)", n_cols,
             kLinearMomentsMaxCols);
  const SlotBuf& X = ctx->slot[src_slot];
  SE_REQUIRE(ctx, X.d && X.cols > 0, SE_ERR_STATE, "source slot %d not allocated", src_slot);
  const int64_t n = X.cols;
  for (int k = 0; k < n_cols; ++k)
    SE_REQUIRE(ctx, cols[k] >= 0 && cols[k] < X.rows, SE_ERR_ARG, "column list entry %d: column %d outside slot %d "
               "with %lld columns", k, cols[k], src_slot, (long long)X.rows);
  auto row_of = [&](int slot, int row, const char* what, const float** p) -> int {
    SE_REQUIRE(ctx, slot >= 0 && slot < SE_NUM_SLOTS, SE_ERR_ARG, "bad %s slot %d", what, slot);
    const SlotBuf& s = ctx->slot[slot];
    SE_REQUIRE(ctx, s.d && s.cols == n && row >= 0 && row < s.rows, SE_ERR_ARG, "%s slot %d: no row %d of %lld values",
               what, slot, row, (long long)n);
    *p = s.d + (int64_t)row * s.ld;
    return SE_OK;
  };
  LinearMomentsArgs a;
  SE_TRY(row_of(label_slot, label_row, "label", &a.y));
  if (weight_slot >= 0) SE_TRY(row_of(weight_slot, weight_row, "weight", &a.w));
  if (use_bag) SE_TRY(row_of(SE_SLOT_BAG, 0, "bag", &a.bag));
  SE_TRY(begin(ctx));
  SE_TRY(read_slot(ctx, src_slot));
  SE_TRY(read_slot(ctx, label_slot));
  SE_TRY(read_slot(ctx, weight_slot));
  const int m = n_cols + 2;
  size_t n_part = 0;
  int n_cnt = 0;
  linear_moments_scratch(n_cols, n, ctx->sms, &n_part, &n_cnt);
  auto& L = ctx->lm;
  SE_CUDA(ctx, L.d_part.grow(n_part));
  SE_CUDA(ctx, L.d_cnt.grow((size_t)n_cnt));
  SE_CUDA(ctx, L.d_out.grow((size_t)m * m));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // h_small is reused below
  int32_t* hcol = reinterpret_cast<int32_t*>(ctx->h_small.get());
  double* hs = reinterpret_cast<double*>(ctx->h_small.get() + 1024);  // 254 columns fit below it
  for (int k = 0; k < n_cols; ++k) {
    hcol[k] = cols[k];
    hs[k] = shift ? shift[k] : 0.0;
  }
  SE_CUDA(ctx, cudaMemcpyAsync(ctx->d_small, ctx->h_small, 1024 + sizeof(double) * (size_t)n_cols, cudaMemcpyHostToDevice,
                               ctx->stream));
  SE_CUDA(ctx, cudaMemsetAsync(L.d_cnt, 0, sizeof(unsigned int) * (size_t)n_cnt, ctx->stream));
  a.X = X.d; a.ld = X.ld; a.n = n; a.p = n_cols;
  a.cols = reinterpret_cast<const int32_t*>(ctx->d_small.get());
  a.shift = reinterpret_cast<const double*>(ctx->d_small.get() + 1024);
  a.y_shift = label_shift;
  a.partials = L.d_part; a.counters = L.d_cnt; a.out = L.d_out;
  SE_LAUNCH_T(ctx, SE_KF_LINEAR, launch_linear_moments(a, ctx->sms, ctx->stream));
  double* hout = reinterpret_cast<double*>(ctx->h_small.get());
  SE_CUDA(ctx, cudaMemcpyAsync(hout, L.d_out, sizeof(double) * (size_t)m * m, cudaMemcpyDeviceToHost, ctx->stream));
  SE_TRY(end(ctx));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  memcpy(out, hout, sizeof(double) * (size_t)m * m);
  if (weight_slot == SE_SLOT_WOUT && ctx->wout_scaled && (size_t)weight_row < ctx->wout_scale.size()) {
    // Newton weights: WOUT holds 1/2 hc w, the learner's weights are that x 1/S_row (newton_finish); the moments are
    // linear in the weights, so the factor se_download applies per value is applied to the matrix here
    const double s = (double)ctx->wout_scale[(size_t)weight_row];
    for (int i = 0; i < m * m; ++i) out[i] *= s;
  }
  return SE_OK;
}

namespace {
// The inputs se_logistic_stats and se_logistic_loss_grad share: the columns of src_slot, the label row and the weight
// row (none when weight_slot < 0), checked; the column list goes to d_small.
// (se_logistic_loss_grad_batch: cols is every member's list, one after another, max_cols their total's limit.)
int logistic_inputs(se_ctx* ctx, int src_slot, int n_cols, const int32_t* cols, int label_slot, int label_row,
                    int weight_slot, int weight_row, LogisticArgs* a, int max_cols = kLogisticMaxCols) {
  if (!ctx || (n_cols > 0 && !cols)) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, src_slot == SE_SLOT_X || src_slot == SE_SLOT_P, SE_ERR_ARG,
             "source slot %d: only SE_SLOT_X or SE_SLOT_P", src_slot);
  SE_REQUIRE(ctx, n_cols >= 0 && n_cols <= max_cols, SE_ERR_ARG, "%d columns (0..%d supported)", n_cols, max_cols);
  const SlotBuf& X = ctx->slot[src_slot];
  SE_REQUIRE(ctx, X.d && X.cols > 0, SE_ERR_STATE, "source slot %d not allocated", src_slot);
  const int64_t n = X.cols;
  for (int k = 0; k < n_cols; ++k)
    SE_REQUIRE(ctx, cols[k] >= 0 && cols[k] < X.rows, SE_ERR_ARG, "column list entry %d: column %d outside slot %d "
               "with %lld columns", k, cols[k], src_slot, (long long)X.rows);
  auto row_of = [&](int slot, int row, const char* what, const float** p) -> int {
    SE_REQUIRE(ctx, slot >= 0 && slot < SE_NUM_SLOTS, SE_ERR_ARG, "bad %s slot %d", what, slot);
    const SlotBuf& s = ctx->slot[slot];
    SE_REQUIRE(ctx, s.d && s.cols == n && row >= 0 && row < s.rows, SE_ERR_ARG, "%s slot %d: no row %d of %lld values",
               what, slot, row, (long long)n);
    *p = s.d + (int64_t)row * s.ld;
    return SE_OK;
  };
  SE_TRY(row_of(label_slot, label_row, "label", &a->y));
  if (weight_slot >= 0) SE_TRY(row_of(weight_slot, weight_row, "weight", &a->w));
  SE_TRY(begin(ctx));
  SE_TRY(read_slot(ctx, src_slot));
  SE_TRY(read_slot(ctx, label_slot));
  SE_TRY(read_slot(ctx, weight_slot));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // h_small is reused below
  memcpy(ctx->h_small.get(), cols, sizeof(int32_t) * (size_t)n_cols);
  a->X = X.d; a->ld = X.ld; a->n = n; a->p = n_cols;
  a->cols = reinterpret_cast<const int32_t*>(ctx->d_small.get());
  return SE_OK;
}

// Launches `launch` over scratch of the sizes `scratch` asks for, after uploading `doubles` values from h_small + 1024,
// and copies `len` results into out.
template <class Scratch, class Launch>
int logistic_run(se_ctx* ctx, LogisticArgs& a, size_t doubles, int len, Scratch scratch, Launch launch, double* out) {
  size_t n_part = 0;
  int n_cnt = 0;
  scratch(&n_part, &n_cnt);
  auto& L = ctx->lg;
  SE_CUDA(ctx, L.d_part.grow(n_part));
  SE_CUDA(ctx, L.d_cnt.grow((size_t)n_cnt));
  SE_CUDA(ctx, L.d_out.grow((size_t)len));
  SE_CUDA(ctx, cudaMemcpyAsync(ctx->d_small, ctx->h_small, 1024 + sizeof(double) * doubles, cudaMemcpyHostToDevice,
                               ctx->stream));
  SE_CUDA(ctx, cudaMemsetAsync(L.d_cnt, 0, sizeof(unsigned int) * (size_t)n_cnt, ctx->stream));
  a.partials = L.d_part; a.counters = L.d_cnt; a.out = L.d_out;
  SE_LAUNCH_T(ctx, SE_KF_LINEAR, launch());
  double* hout = reinterpret_cast<double*>(ctx->h_small.get());
  SE_CUDA(ctx, cudaMemcpyAsync(hout, L.d_out, sizeof(double) * (size_t)len, cudaMemcpyDeviceToHost, ctx->stream));
  SE_TRY(end(ctx));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  memcpy(out, hout, sizeof(double) * (size_t)len);
  return SE_OK;
}
}  // namespace

int se_logistic_stats(se_ctx* ctx, int src_slot, int n_cols, const int32_t* cols, const double* shift, int num_classes,
                      int label_slot, int label_row, int weight_slot, int weight_row, double* out) {
  if (!ctx || !out) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, num_classes >= 1 && num_classes <= kLogisticMaxClasses, SE_ERR_ARG, "%d classes (1..%d supported)",
             num_classes, kLogisticMaxClasses);
  LogisticArgs a;
  SE_TRY(logistic_inputs(ctx, src_slot, n_cols, cols, label_slot, label_row, weight_slot, weight_row, &a));
  double* hs = reinterpret_cast<double*>(ctx->h_small.get() + 1024);
  for (int k = 0; k < n_cols; ++k) hs[k] = shift ? shift[k] : 0.0;
  a.shift = reinterpret_cast<const double*>(ctx->d_small.get() + 1024);
  a.D = num_classes;
  const int64_t n = a.n;
  return logistic_run(
      ctx, a, (size_t)n_cols, 3 + 2 * n_cols + num_classes,
      [&](size_t* part, int* cnt) { logistic_stats_scratch(n_cols, num_classes, n, ctx->sms, part, cnt); },
      [&]() { return launch_logistic_stats(a, ctx->sms, ctx->stream); }, out);
}

int se_logistic_loss_grad(se_ctx* ctx, int src_slot, int n_cols, const int32_t* cols, const double* shift,
                          const double* scale, int n_sets, const double* coef, int label_slot, int label_row,
                          int weight_slot, int weight_row, double* out) {
  if (!ctx || !out || !coef) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, n_sets >= 1 && n_sets <= kLogisticMaxClasses, SE_ERR_ARG,
             "%d coefficient sets (1: binomial, 2..%d: multinomial)", n_sets, kLogisticMaxClasses);
  LogisticArgs a;
  SE_TRY(logistic_inputs(ctx, src_slot, n_cols, cols, label_slot, label_row, weight_slot, weight_row, &a));
  const int P1 = n_cols + 1;
  double* hs = reinterpret_cast<double*>(ctx->h_small.get() + 1024);
  for (int k = 0; k < n_cols; ++k) {
    hs[k] = shift ? shift[k] : 0.0;
    hs[n_cols + k] = scale ? scale[k] : 1.0;
  }
  memcpy(hs + 2 * n_cols, coef, sizeof(double) * (size_t)n_sets * P1);
  const double* ds = reinterpret_cast<const double*>(ctx->d_small.get() + 1024);
  a.shift = ds;
  a.scale = ds + n_cols;
  a.coef = ds + 2 * n_cols;
  a.D = n_sets;
  const int64_t n = a.n;
  return logistic_run(
      ctx, a, (size_t)2 * n_cols + (size_t)n_sets * P1, 1 + n_sets * P1,
      [&](size_t* part, int* cnt) { logistic_loss_grad_scratch(n_cols, n_sets, n, ctx->sms, part, cnt); },
      [&]() { return launch_logistic_loss_grad(a, ctx->sms, ctx->stream); }, out);
}

int se_logistic_loss_grad_batch(se_ctx* ctx, int src_slot, int n_members, const int32_t* n_cols, const int32_t* cols,
                                const double* shift, const double* scale, int n_sets, const double* coef,
                                int label_slot, int label_row, int weight_slot, int weight_row, double* out) {
  if (!ctx || !out || !coef || !n_cols) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, n_members >= 1 && n_members <= kLogisticMaxBatch, SE_ERR_ARG, "%d members (1..%d supported)",
             n_members, kLogisticMaxBatch);
  SE_REQUIRE(ctx, n_sets >= 1 && n_sets <= kLogisticMaxClasses, SE_ERR_ARG,
             "%d coefficient sets (1: binomial, 2..%d: multinomial)", n_sets, kLogisticMaxClasses);
  int64_t total = 0;
  for (int b = 0; b < n_members; ++b) {
    SE_REQUIRE(ctx, n_cols[b] >= 0 && n_cols[b] <= kLogisticMaxCols, SE_ERR_ARG,
               "member %d: %d columns (0..%d supported)", b, n_cols[b], kLogisticMaxCols);
    total += n_cols[b];
  }
  LogisticArgs a;  // every column of every member is checked against the slot here
  SE_TRY(logistic_inputs(ctx, src_slot, (int)total, cols, label_slot, label_row, weight_slot, weight_row, &a,
                         kLogisticMaxBatch * kLogisticMaxCols));
  const int D = n_sets;
  std::vector<LogisticArgs> mem((size_t)n_members, a);
  size_t n_part = 0, n_in_doubles = 0, n_out = 0;
  int n_cnt = 0;
  for (int b = 0; b < n_members; ++b) {
    size_t part = 0;
    int cnt = 0;
    logistic_loss_grad_scratch(n_cols[b], D, a.n, ctx->sms, &part, &cnt);
    LogisticArgs& m = mem[(size_t)b];
    m.p = n_cols[b];
    m.D = D;
    // offsets for now, pointers once the buffers exist
    m.partials = reinterpret_cast<double*>(n_part);
    m.counters = reinterpret_cast<unsigned int*>((size_t)n_cnt);
    m.out = reinterpret_cast<double*>(n_out);
    n_part += part;
    n_cnt += cnt;
    n_out += 1 + (size_t)D * (m.p + 1);
    n_in_doubles += 2 * (size_t)m.p + (size_t)D * (m.p + 1);
  }
  const int count = logistic_batch_items(mem.data(), n_members, ctx->sms, nullptr);
  const size_t items_bytes = ((sizeof(LogisticBatchItem) * (size_t)count + 15) / 16) * 16;
  const size_t cols_bytes = ((sizeof(int32_t) * (size_t)total + 15) / 16) * 16;
  const size_t in_bytes = items_bytes + cols_bytes + sizeof(double) * n_in_doubles;
  auto& L = ctx->lg;
  SE_CUDA(ctx, L.d_part.grow(n_part));
  SE_CUDA(ctx, L.d_cnt.grow((size_t)n_cnt));
  SE_CUDA(ctx, L.d_out.grow(n_out));
  SE_CUDA(ctx, L.d_in.grow(in_bytes));
  SE_CUDA(ctx, L.h_in.grow(std::max(in_bytes, sizeof(double) * n_out)));
  unsigned char* h = L.h_in.get();
  unsigned char* d = L.d_in.get();
  memcpy(h + items_bytes, cols, sizeof(int32_t) * (size_t)total);
  double* hd = reinterpret_cast<double*>(h + items_bytes + cols_bytes);
  const double* dd = reinterpret_cast<const double*>(d + items_bytes + cols_bytes);
  size_t col_off = 0, dbl_off = 0, coef_off = 0;
  for (int b = 0; b < n_members; ++b) {
    LogisticArgs& m = mem[(size_t)b];
    const int p = m.p, P1 = p + 1;
    for (int k = 0; k < p; ++k) {
      hd[dbl_off + k] = shift ? shift[col_off + k] : 0.0;
      hd[dbl_off + p + k] = scale ? scale[col_off + k] : 1.0;
    }
    memcpy(hd + dbl_off + 2 * p, coef + coef_off, sizeof(double) * (size_t)D * P1);
    m.cols = reinterpret_cast<const int32_t*>(d + items_bytes) + col_off;
    m.shift = dd + dbl_off;
    m.scale = dd + dbl_off + p;
    m.coef = dd + dbl_off + 2 * p;
    m.partials = L.d_part.get() + reinterpret_cast<size_t>(m.partials);
    m.counters = L.d_cnt.get() + reinterpret_cast<size_t>(m.counters);
    m.out = L.d_out.get() + reinterpret_cast<size_t>(m.out);
    col_off += (size_t)p;
    dbl_off += 2 * (size_t)p + (size_t)D * P1;
    coef_off += (size_t)D * P1;
  }
  LogisticBatchItem* items = reinterpret_cast<LogisticBatchItem*>(h);
  logistic_batch_items(mem.data(), n_members, ctx->sms, items);
  SE_CUDA(ctx, cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
  SE_CUDA(ctx, cudaMemsetAsync(L.d_cnt, 0, sizeof(unsigned int) * (size_t)n_cnt, ctx->stream));
  SE_LAUNCH_T(ctx, SE_KF_LINEAR, launch_logistic_loss_grad_batch(items, reinterpret_cast<const LogisticBatchItem*>(d),
                                                                 count, ctx->stream));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // the staged items are read by the copy above: reuse h_in after it
  double* hout = reinterpret_cast<double*>(L.h_in.get());
  SE_CUDA(ctx, cudaMemcpyAsync(hout, L.d_out, sizeof(double) * n_out, cudaMemcpyDeviceToHost, ctx->stream));
  SE_TRY(end(ctx));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  memcpy(out, hout, sizeof(double) * n_out);
  return SE_OK;
}

int se_logistic_predict(se_ctx* ctx, int n_coef, const int32_t* subspace, int n_sets, const double* coef,
                        const double* intercept, double threshold, int raw_slot, int raw_row, int prob_slot,
                        int prob_row, int label_slot, int label_row) {
  if (!ctx || !intercept || (n_coef > 0 && !coef)) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, n_coef >= 0 && n_coef <= kLogisticMaxCols, SE_ERR_ARG, "%d coefficients per set (0..%d supported)",
             n_coef, kLogisticMaxCols);
  SE_REQUIRE(ctx, n_sets >= 1 && n_sets <= kLogisticMaxClasses, SE_ERR_ARG,
             "%d coefficient sets (1: binomial, 2..%d: multinomial)", n_sets, kLogisticMaxClasses);
  const SlotBuf& X = ctx->slot[SE_SLOT_X];
  SE_REQUIRE(ctx, X.d && X.cols > 0, SE_ERR_STATE, "feature matrix slot not allocated");
  for (int j = 0; j < n_coef; ++j) {
    const int32_t col = subspace ? subspace[j] : j;
    SE_REQUIRE(ctx, col >= 0 && col < X.rows, SE_ERR_ARG, "column %d outside X", col);
  }
  SE_TRY(begin(ctx));
  LogisticPredictArgs a;
  const int width = n_sets == 1 ? 2 : n_sets;
  if (raw_slot >= 0) SE_TRY(out_rows(ctx, raw_slot, raw_row, width, X.cols, &a.raw, &a.ld_raw));
  if (prob_slot >= 0) SE_TRY(out_rows(ctx, prob_slot, prob_row, width, X.cols, &a.prob, &a.ld_prob));
  if (label_slot >= 0) SE_TRY(out_rows(ctx, label_slot, label_row, 1, X.cols, &a.label, nullptr));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // h_small is reused below
  int32_t* hcol = reinterpret_cast<int32_t*>(ctx->h_small.get());
  for (int j = 0; j < n_coef; ++j) hcol[j] = subspace ? subspace[j] : j;
  double* hd = reinterpret_cast<double*>(ctx->h_small.get() + 1024);
  memcpy(hd, coef, sizeof(double) * (size_t)n_sets * n_coef);
  memcpy(hd + (size_t)n_sets * n_coef, intercept, sizeof(double) * (size_t)n_sets);
  SE_CUDA(ctx, cudaMemcpyAsync(ctx->d_small, ctx->h_small, 1024 + sizeof(double) * (size_t)n_sets * (n_coef + 1),
                               cudaMemcpyHostToDevice, ctx->stream));
  const double* dd = reinterpret_cast<const double*>(ctx->d_small.get() + 1024);
  a.X = X.d; a.ld = X.ld; a.n = X.cols; a.p = n_coef; a.D = n_sets;
  a.cols = reinterpret_cast<const int32_t*>(ctx->d_small.get());
  a.coef = dd;
  a.intercept = dd + (size_t)n_sets * n_coef;
  a.threshold = threshold;
  SE_LAUNCH_T(ctx, SE_KF_LINEAR, launch_logistic_predict(a, ctx->sms, ctx->stream));
  return end(ctx);
}

// An ensemble of linear and logistic members in one pass over X with se_agg_run's results (see se_abi.h).
int se_linear_agg(se_ctx* ctx, int which, int kind, int num_classes, int dim, int loss, int n_members,
                  const int32_t* col_offsets, const int32_t* cols, const int32_t* n_sets, const double* coef,
                  const double* intercept, const double* threshold, const int32_t* member_class,
                  const double* weights, const double* init, int out_slot, int out_row) {
  if (!ctx || !col_offsets || !n_sets || !intercept) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, kind >= SE_AGG_GBM_REGRESSOR && kind <= SE_AGG_BOOSTING_REG_MEAN, SE_ERR_ARG, "bad kind %d", kind);
  SE_REQUIRE(ctx, n_members >= 1 && n_members <= (1 << 20), SE_ERR_ARG, "bad member count %d", n_members);
  const bool median = (kind == SE_AGG_BOOSTING_REG_MEDIAN);
  const bool reg = median || kind == SE_AGG_GBM_REGRESSOR || kind == SE_AGG_BAGGING_REGRESSOR ||
                   kind == SE_AGG_BOOSTING_REG_MEAN;
  const bool gbm = (kind == SE_AGG_GBM_CLASSIFIER);
  const bool vec = (kind == SE_AGG_BAGGING_SOFT || kind == SE_AGG_BOOSTING_REAL);
  const bool value = reg || gbm;  // the member's output is its value: one margin
  SE_REQUIRE(ctx, !median || n_members <= SE_FOREST_MEDIAN_MAX_TREES, SE_ERR_ARG,
             "the weighted median serves 1..%d members, got %d: evaluate the members with se_logistic_predict + "
             "se_agg_run", SE_FOREST_MEDIAN_MAX_TREES, n_members);
  if (!reg)
    SE_REQUIRE(ctx, num_classes >= 2 && num_classes <= SE_FOREST_AGG_MAX_CLASSES, SE_ERR_ARG,
               "se_linear_agg's classifier kinds support 2..%d classes, got %d", SE_FOREST_AGG_MAX_CLASSES, num_classes);
  if (gbm) {
    SE_REQUIRE(ctx, dim >= 1 && dim <= SE_FOREST_AGG_MAX_CLASSES && (dim > 1 || num_classes == 2), SE_ERR_ARG,
               "bad dim %d for %d classes", dim, num_classes);
    SE_REQUIRE(ctx, member_class, SE_ERR_ARG, "the GBM classifier needs member_class");
  }
  SE_REQUIRE(ctx, weights || !(kind == SE_AGG_GBM_REGRESSOR || gbm || kind == SE_AGG_BOOSTING_DISCRETE || median ||
                               kind == SE_AGG_BOOSTING_REG_MEAN),
             SE_ERR_ARG, "weights required for aggregation kind %d", kind);
  const SlotBuf& X = ctx->slot[which ? SE_SLOT_VX : SE_SLOT_X];
  SE_REQUIRE(ctx, X.d && X.cols > 0, SE_ERR_STATE, "feature matrix slot not allocated");
  SE_REQUIRE(ctx, col_offsets[0] == 0, SE_ERR_ARG, "col_offsets[0] must be 0");
  SE_REQUIRE(ctx, !reg || out_slot != (which ? SE_SLOT_VX : SE_SLOT_X), SE_ERR_ARG,
             "the output row cannot be a row of the feature matrix the members read");
  std::vector<LinearAggMember> mem((size_t)n_members);
  int max_d = 1;
  int64_t n_coef = 0, n_icpt = 0;
  for (int m = 0; m < n_members; ++m) {
    const int64_t p = (int64_t)col_offsets[m + 1] - col_offsets[m];
    const int D = n_sets[m];
    SE_REQUIRE(ctx, p >= 0 && p <= kLinearAggMaxCols, SE_ERR_ARG, "member %d: %lld columns (0..%d supported)", m,
               (long long)p, kLinearAggMaxCols);
    SE_REQUIRE(ctx, p == 0 || cols, SE_ERR_ARG, "null argument");
    SE_REQUIRE(ctx, value ? D == 1 : (D == 1 || D == num_classes), SE_ERR_ARG,
               "member %d: %d coefficient sets where %s", m, D, value ? "this kind takes the value of one" : "1 or K are");
    SE_REQUIRE(ctx, !vec || D > 1 || num_classes == 2, SE_ERR_ARG,
               "member %d: a binomial member gives 2 probabilities, not %d", m, num_classes);
    for (int64_t j = col_offsets[m]; j < col_offsets[m + 1]; ++j)
      SE_REQUIRE(ctx, cols[j] >= 0 && cols[j] < X.rows, SE_ERR_ARG, "member %d: column %d outside X with %lld columns",
                 m, cols[j], (long long)X.rows);
    if (gbm)
      SE_REQUIRE(ctx, member_class[m] >= 0 && member_class[m] < dim, SE_ERR_ARG, "member %d: class %d outside [0, %d)",
                 m, member_class[m], dim);
    LinearAggMember& mb = mem[(size_t)m];
    mb.col0 = col_offsets[m]; mb.p = (int)p; mb.D = D; mb.cls = gbm ? member_class[m] : 0;
    mb.coef0 = (int)n_coef;
    n_coef += (int64_t)D * p;
    mb.icpt0 = (int)n_icpt;  // moved past the coefficients below
    n_icpt += D;
    mb.threshold = threshold ? threshold[m] : 0.5;
    // the weights as se_agg_run takes them: fp32 for the sums and the SAMME votes, fp64 for the GBM classifier
    const bool sum_w = (kind == SE_AGG_GBM_REGRESSOR || kind == SE_AGG_BOOSTING_REG_MEAN);
    mb.wf = sum_w ? (float)weights[m] : 1.f;
    mb.w = kind == SE_AGG_BOOSTING_DISCRETE ? (double)(float)weights[m] : gbm ? weights[m] : 1.0;
    max_d = std::max(max_d, D);
  }
  SE_REQUIRE(ctx, n_coef == 0 || coef, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, n_coef + n_icpt <= (int64_t)1 << 28, SE_ERR_ARG, "%lld coefficients: too many",
             (long long)(n_coef + n_icpt));
  for (LinearAggMember& mb : mem) mb.icpt0 += (int)n_coef;
  const int64_t n = X.cols;
  SE_TRY(begin(ctx));
  LinearAggArgs g;
  g.kind = kind; g.K = num_classes; g.M = n_members; g.loss = loss;
  g.dim = gbm ? dim : 1;
  g.C = reg ? 1 : gbm ? dim : num_classes;
  const int out_c = (gbm && dim == 1) ? 2 : g.C;
  if (reg) {
    SE_TRY(out_rows(ctx, out_slot, out_row, 1, n, &g.out, nullptr));
  } else {
    SE_TRY(slot_alloc2d(ctx, SE_SLOT_RAW, out_c, n));
    SE_TRY(slot_alloc2d(ctx, SE_SLOT_PROB, out_c, n));
    SE_TRY(slot_alloc2d(ctx, SE_SLOT_LABEL, 1, n));
    const SlotBuf& R = ctx->slot[SE_SLOT_RAW];
    g.raw = R.d; g.prob = ctx->slot[SE_SLOT_PROB].d; g.label = ctx->slot[SE_SLOT_LABEL].d;
    g.ld_out = R.ld;
  }
  // se_agg_run's scalars: (float) init of the GBM regressor, the divisor of the mean kinds (M, or Σ of the fp32
  // weights), Σ of the SAMME vote weights
  double sum_f = 0.0;
  for (int m = 0; m < n_members; ++m) sum_f += (double)mem[(size_t)m].wf;
  if (kind == SE_AGG_GBM_REGRESSOR) g.init[0] = init ? (double)(float)init[0] : 0.0;
  if (kind == SE_AGG_BAGGING_REGRESSOR) g.post_div = (float)n_members;
  if (kind == SE_AGG_BOOSTING_REG_MEAN) g.post_div = (float)sum_f;
  if (gbm)
    for (int c = 0; c < dim; ++c) g.init[c] = init ? init[c] : 0.0;
  for (int m = 0; m < n_members; ++m) g.sum_a += mem[(size_t)m].w;
  g.n4 = reg ? (n & ~(int64_t)3) : n;
  if (median) {  // as se_forest_median
    g.mode = ctx->wm_fast ? wm_weight_mode(weights, n_members) : 0;
    for (int m = 0; m < kForestMedianMaxTrees; ++m) {
      g.w[m] = (m < n_members) ? weights[m] : 0.0;
      g.total += g.w[m];
    }
    g.tau = (g.mode == 1) ? 8.0 * (double)n_members * 1.1102230246251565e-16 * g.total : -1.0;
    ctx->last_wm_mode = g.mode;
  }
  // the members, the 64-bit offsets of their columns and their coefficients, in one blob
  const size_t total_cols = (size_t)col_offsets[n_members];
  const size_t mem_bytes = forest_pad(sizeof(LinearAggMember) * (size_t)n_members, 16);
  const size_t col_bytes = forest_pad(sizeof(unsigned long long) * total_cols, 16);
  std::vector<unsigned char> blob(mem_bytes + col_bytes + sizeof(double) * (size_t)(n_coef + n_icpt));
  memcpy(blob.data(), mem.data(), sizeof(LinearAggMember) * (size_t)n_members);
  unsigned long long* co = reinterpret_cast<unsigned long long*>(blob.data() + mem_bytes);
  for (size_t j = 0; j < total_cols; ++j) co[j] = (unsigned long long)cols[j] * (unsigned long long)X.ld;
  double* cf = reinterpret_cast<double*>(blob.data() + mem_bytes + col_bytes);
  if (n_coef) memcpy(cf, coef, sizeof(double) * (size_t)n_coef);
  memcpy(cf + n_coef, intercept, sizeof(double) * (size_t)n_icpt);
  SE_TRY(forest_upload(ctx, blob.data(), blob.size()));
  const unsigned char* d = ctx->d_forest;
  g.members = reinterpret_cast<const LinearAggMember*>(d);
  g.coloff = reinterpret_cast<const unsigned long long*>(d + mem_bytes);
  g.coef = reinterpret_cast<const double*>(d + mem_bytes + col_bytes);
  g.X = X.d; g.n = n;
  SE_LAUNCH_T(ctx, SE_KF_LINEAR, launch_linear_agg(g, max_d, ctx->sms, ctx->stream));
  return end(ctx);
}
