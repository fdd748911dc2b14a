// se_kernels.h — host-callable launchers of the sm_90a kernels (internal to libse_b200.so).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "se_common.cuh"

namespace se {

constexpr int kMaxDim = 64;  // LogLoss classes served by the specialised kernels: per-class sums reduced in one kernel (kMaxRed, mailbox width)
constexpr int kMaxDimGeneric = 16384;  // beyond kMaxDim: the general kernels of se_gbm_generic.cu (shared-memory accumulators)

// ---- GBM (se_gbm.cu) -------------------------------------------------------------------------
enum GbmMode {
  GBM_RESID = 0,         // R = -g(y,F)
  GBM_RESID_NEWTON = 1,  // R = -g/hc, WOUT = 1/2 hc w (unnormalised), Σhc
  GBM_EVAL = 2,          // p = F + a h : Σloss, Σ h g      (GBMLossAggregator.add)
  GBM_UPDATE = 3,        // F += s h : Σloss(F')
  GBM_UPDATE_RESID = 4,  // + R = -g(y,F')
  GBM_UPDATE_NEWTON = 5, // + R = -g/hc, WOUT = 1/2 hc w, Σhc
  GBM_MEAN_LOSS = 6,     // Σloss(y,F)
  GBM_SQ_STATS = 7,      // squared: Σ(y-F)², Σh(y-F), Σh²
  GBM_EVAL_LOSS = 8      // p = F + a h : Σloss only (Brent needs the objective value, not its gradient)
};

struct GbmArgs {
  const float* y = nullptr;
  const float* w = nullptr;  // nullable: unit weights
  const float* bag = nullptr;  // nullable: per-row bag multiplicities (RDD.sample counts) for line search / newton S
  float* F = nullptr;
  const float* h = nullptr;
  float* r = nullptr;
  float* wout = nullptr;
  int64_t n = 0;
  int64_t ld = 0;  // row stride of the [dim][n] arrays
  int dim = 1;
  float param = 0.f;
  float coef[kMaxDim] = {0};  // alpha (eval) or step (update), per dim
  // squared-loss device-resident step: step = lr * clip(stats[1]/stats[2], 0, 100) when non-null
  const double* dev_stats = nullptr;
  float lr = 1.f;
  // step = (float)(lr64 * *dev_alpha) when non-null: alpha comes from the on-device line search (se_brent.cu)
  const double* dev_alpha = nullptr;
  double lr64 = 1.0;
  int stats_from_r = 0;  // squared-loss statistics read the current residual slot r = y - F (8 B/row) instead of y, F (12 B/row)
  int l2_hints = 0; // L2-sized shard: evict_first for the arrays the next pass does not re-read (se_common.cuh)
  int reverse = 0; // walk the tiles from the end: consecutive passes alternate direction so the tail of one
                   // pass (still in the L2) is the head of the next
  RedWs ws{};
};

// reduction outputs (ws.out): scalar losses: [0]=Σloss [1]=Σ h·g or Σhc ; SQ_STATS: [0..2]
// logloss: [0]=Σloss, [1..K]=Σ h_j g_j  or Σhc_j
cudaError_t launch_gbm(int loss, int mode, const GbmArgs& a, int ctas_per_sm, int sms,
                       cudaStream_t stream);
// line-search view for the binary scalar losses: u = (2y-1)·F, v = (2y-1)·h (exact sign flips), so that every
// Brent evaluation reads two arrays instead of three (launch_gbm GBM_EVAL with y == nullptr, F = u, h = v)
cudaError_t launch_gbm_pack_signed(const float* y, const float* F, const float* h, float* u, float* v, int64_t n,
                                   int sms, cudaStream_t stream);
// squared loss, F owed after a residual-mode fused round: F = y - r, then r = y - F (the residual an update of that F
// would have left), 16 B/row
cudaError_t launch_gbm_settle_f(const float* y, float* r, float* F, int64_t n, int sms, cudaStream_t stream);
// LogLoss(K) for K > kMaxDim (se_gbm_generic.cu): coefficients, per-CTA partials [grid][K+1] and the K+1 sums live in
// device buffers sized for K; the cross-GPU sum of `out` is an NCCL all-reduce issued by the caller
struct GenericArgs {
  const float* coef = nullptr;  // device [K]
  double* partials = nullptr;   // device [grid][K+1]
  double* out = nullptr;        // device [K+1]
};
cudaError_t launch_gbm_logloss_generic(int mode, const GbmArgs& a, const GenericArgs& ga, int grid, cudaStream_t stream);
// LogLoss(K), wide K: 2-D TMA tiles of 256 rows x K classes, four rows per thread (se_gbm_tiled.cu)
cudaError_t launch_gbm_logloss_tiled(int mode, const GbmArgs& a, int sms, cudaStream_t stream);
// squared-loss line search on the device: Brent over the parabola of stats[0..2]; out[0] = alpha, out[1] = objective,
// out[2] = evaluations (negative: MaxEval exceeded); out_host (mapped pinned memory) is optional
cudaError_t launch_brent_parabola(const double* stats, double wsum, double lo, double hi, double start, double rel,
                                  double abs_tol, int max_eval, double* out_dev, double* out_host, cudaStream_t stream);
// squared-loss round result: out[0] = alpha*, computed on device from stats (for se_gbm_round_result)
cudaError_t launch_sq_alpha(const double* stats, double* out_alpha, cudaStream_t stream);

// ---- whole-round / whole-line-search cooperative kernels (se_gbm_fused.cu) ----------------------
// Device-side rendezvous of the cooperative kernels (owned by the context, zero-initialised).
struct FusedSync {
  unsigned long long flag;  // epoch published by the coordinating CTA / warp (monotonic across launches)
  double x;                 // published with the flag: the step (round kernel) or the next abscissa (line search)
  int cmd;                  // line search: 0 = evaluate x, 1 = stop
  int pad;
  unsigned int arrive;      // line search: worker arrival counter (reset by the coordinator)
  unsigned int counter_b;   // round kernel: ticket of the second (loss) reduction
};

// One squared-loss boosting round in one launch: statistics -> (cross-GPU sum) -> Brent -> update + residual + loss.
// write_r (residual mode): the update writes r' = r - c h only and leaves F for the host to rebuild as y - r'.
// A residual-mode round that reads r (no bag) carries its statistics pass's last tile in registers and, with
// `resident`, the groups before it in shared memory into the update pass; *resident_slots_out = groups per thread.
struct SqRoundArgs {
  const float* y = nullptr;
  float* F = nullptr;
  const float* h = nullptr;
  float* r = nullptr;
  const float* bag = nullptr;  // nullable: bag multiplicities for the line-search statistics
  int64_t n = 0;
  int stats_from_r = 0;
  int l2_hints = 0;
  int l2_mode = 0;         // 0: evict_normal / evict_first hints; 1: evict_last on r and h (experiment)
  int timing = 0;          // write %globaltimer stamps (us) to out[10..13]: start, statistics folded, step published, end
  int prefetch_tiles = 0;  // update-phase tiles (r/h, or y/F) each CTA prefetches into L2 while it waits for the step
  int resident_slots = 0;  // set by the launcher: float4 groups of r and h per thread carried in shared memory
  double lr = 1.0, wsum = 1.0;                                   // learning rate, Σw (objective scale)
  double lo = 0.0, hi = 100.0, start = 1.0, rel = 1e-6, abs_tol = 1e-6;
  int max_eval = 100;
  RedWs ws_a{};  // statistics: out = `out`, no host mirror
  RedWs ws_b{};  // loss (only when it is reduced over the rows: bags): out = out + 8, host mirror + ticket
  double* out = nullptr;       // [0..2] statistics, [4] alpha, [5] objective, [6] +-evaluations, [8] Σloss
  double* host_res = nullptr;  // mapped host copy of out[0..6] (nullable)
  // loss-from-statistics mode: the Brent thread also serves the host (final value + ticket) before the update phase ends
  double* host_final = nullptr;
  volatile unsigned long long* host_flag = nullptr;
  unsigned long long host_ticket = 0;
  FusedSync* sync = nullptr;
  unsigned long long epoch = 0;
};
cudaError_t launch_gbm_round_sq_fused(const SqRoundArgs& a, int write_r, int loss_reduce, int resident, int sms,
                                      int max_ctas_per_sm, cudaStream_t stream, int* grid_out, int* resident_slots_out,
                                      void* window_base = nullptr, size_t window_bytes = 0);

// Brent's whole line search for a dim-1 scalar loss in one launch (persistent workers + coordinator warp).
struct LsArgs {
  const float* y = nullptr;
  const float* F = nullptr;
  const float* h = nullptr;
  float* u = nullptr;  // binary losses: signed view written by the first evaluation, read by the others
  float* v = nullptr;
  int64_t n = 0;
  float param = 0.f;
  double wsum = 1.0;
  double lo = 0.0, hi = 100.0, start = 1.0, rel = 1e-6, abs_tol = 1e-6;
  int max_eval = 100;
  int timing = 0;        // diagnostics: out[4] = us spent in worker passes, out[5] = us in fold + cross-GPU exchange
  int single = 0;        // evaluate the objective at `start` once (host-driven search over the same kernel)
  int first_parity = 0;  // tile direction of evaluation e is (first_parity + e) & 1
  int resident_tiles = 0;
  int ring_stages = 0;   // > 0: streamed tiles go through a per-thread cp.async ring of this many stages in shared memory
  double* partials = nullptr;
  FusedSync* sync = nullptr;
  unsigned long long epoch0 = 0;
  RedWs ws{};            // peer exchange (seq = sequence of the FIRST evaluation) and host mirror
  double* out = nullptr; // [0] alpha, [1] objective, [2] +-evaluations (negative: MaxEval exceeded), [3] passes run
};
struct LsLaunch {
  int max_ctas_per_sm = 4;
  int resident = 1;             // keep each worker's first tiles in shared memory
  int ring = 0;                 // cp.async ring stages for the streamed tiles: 0 off (register prefetch), 2..4
  void* window_base = nullptr;  // L2 access-policy window (persisting) over the packed view
  size_t window_bytes = 0;
  float hit_ratio = 0.f;
};
bool gbm_linesearch_persist_supported(int loss);
bool gbm_linesearch_persist_packed(int loss);
cudaError_t launch_gbm_linesearch_persist(int loss, const LsArgs& a, int sms, const LsLaunch& cfg, cudaStream_t stream,
                                          int* workers_out);

// ---- Boosting (se_boost.cu) ------------------------------------------------------------------
struct BoostArgs {
  const float* y = nullptr;
  float* w = nullptr;         // updated in place
  const float* proba = nullptr;  // [K][n]
  const float* pred = nullptr;   // [n]
  int64_t n = 0, ld = 0;
  int K = 2;
  float inv_sum_w = 1.f;
  float inv_beta = 1.f;
  RedWs ws{};
};
cudaError_t launch_boost_real(const BoostArgs& a, int ctas_per_sm, int sms, cudaStream_t s);   // out: [0]=err [1]=Σw'
cudaError_t launch_boost_discrete_error(const BoostArgs& a, int ctas_per_sm, int sms, cudaStream_t s);  // out[0]
cudaError_t launch_boost_discrete_update(const BoostArgs& a, int ctas_per_sm, int sms, cudaStream_t s); // out[0]=Σw'
cudaError_t launch_sum(const float* x, int64_t n, const RedWs& ws, int ctas_per_sm, int sms,
                       cudaStream_t s);  // out[0]
// out[0] = Σ a_i·b_i (b nullable: Σ a_i)
cudaError_t launch_dot(const float* a, const float* b, int64_t n, const RedWs& ws, int ctas_per_sm, int sms,
                       cudaStream_t s);
// AdaBoost.R2 (regression/BoostingRegressor.scala:225-263). loss_type 0 exponential, 1 linear, 2 squared.
struct BoostRegArgs {
  const float* y = nullptr;
  const float* pred = nullptr;
  float* w = nullptr;  // updated in place by the update kernel
  int64_t n = 0;
  int loss_type = 0;
  float inv_sum_w = 1.f;
  float inv_max_err = 1.f;  // 1/maxError, or 1 when maxError == 0 (:236-242)
  float log2_beta = 0.f;
  RedWs ws{};
};
cudaError_t launch_boostreg_max(const BoostRegArgs& a, int ctas_per_sm, int sms, cudaStream_t s);     // out[0] = max|y-pred|
cudaError_t launch_boostreg_error(const BoostRegArgs& a, int ctas_per_sm, int sms, cudaStream_t s);   // out[0] = Σ wₙ·loss
cudaError_t launch_boostreg_update(const BoostRegArgs& a, int ctas_per_sm, int sms, cudaStream_t s);  // out[0] = Σ w'

// ---- Aggregation (se_agg.cu) -----------------------------------------------------------------
struct AggArgs {
  int kind = 0;
  const float* P = nullptr;  // [M][width][n] with row stride ld
  float* raw = nullptr;      // [C][n]
  float* prob = nullptr;     // [C][n] (classifiers)
  float* label = nullptr;    // [n]    (classifiers)
  const float* weights = nullptr;  // device [M] or [M][dim]
  const float* init = nullptr;     // device [dim]
  int M = 0, K = 0, dim = 1, loss = 0;
  int64_t n = 0, ld = 0, ld_out = 0;
  double sum_weights = 0.0;  // Σ a_m of the fp32-narrowed weights (boosting discrete epilogue, boosting-regressor mean)
  const double* weights64 = nullptr;  // device [M] fp64 (weighted median cumulative sums)
  int* bad_label = nullptr;           // raised (mapped host memory) when a vote is not a class index in [0, K)
  // weighted median fast path (M <= 64): 0 exact kernel only; 1 keys-only sort + model-order sums, rows within the
  // rounding margin of the half-weight deferred to the exact kernel through wm_list; 2 all weights equal (no margin)
  int wm_mode = 0;
  const double* weights64_host = nullptr;  // [M], the same values as weights64
  int32_t* wm_list = nullptr;              // [wm_cap] deferred rows
  unsigned int* wm_count = nullptr;        // number of deferred rows (may exceed wm_cap: the exact pass then covers all rows)
  unsigned int wm_cap = 0;
};
cudaError_t launch_agg(const AggArgs& a, int ctas_per_sm, int sms, cudaStream_t s);

// ---- base-model evaluators over column-major X (se_models.cu) --------------------------------
struct TreeArgs {
  const float* X = nullptr;  // [d][n], stride ld
  int64_t n = 0, ld = 0;
  int n_nodes = 0;
  const int32_t* feature = nullptr;  // device arrays [n_nodes]; feature already mapped through subspace
  const float* threshold = nullptr;
  const int32_t* left = nullptr;
  const int32_t* right = nullptr;
  const float* value = nullptr;      // [n_nodes][n_out]
  float* out = nullptr;              // n_out rows of stride ld_out
  int n_out = 1;                     // 1: regression value / label; K: class-probability vector of the leaf
  int64_t ld_out = 0;
};
cudaError_t launch_tree_predict(const TreeArgs& a, int sms, cudaStream_t s);
// uint8 rank matrix of X for the tree walk (se_models.cu): X8[col][i] = #{thresholds of col strictly below X[col][i]}
struct BinArgs {
  const float* X = nullptr;      // [d][ld]
  uint8_t* X8 = nullptr;         // [d][ld8]
  int64_t n = 0, ld = 0, ld8 = 0;
  const int32_t* cols = nullptr;     // device: the columns to (re)build, one per blockIdx.y
  const float* edges = nullptr;      // device [d][256]: sorted thresholds per column
  const int32_t* n_edges = nullptr;  // device [d]
};
cudaError_t launch_bin_columns(const BinArgs& a, int n_cols, int sms, cudaStream_t s);
// nodes: packed {x,y: byte offset of the column in X8 (64 bit); z: bin threshold | leaf << 31; w: left | right << 16}
// n_internal: number of internal nodes; mask_mode != 0 allows the all-nodes kernel for trees of <= 64 internal nodes
cudaError_t launch_tree_predict_binned(const TreeArgs& a, const uint8_t* X8, const uint4* nodes, int n_internal, int mask_mode,
                                       int sms, cudaStream_t s);
// A whole forest in ONE pass over the uint8 rank matrix: out = (accumulate ? out : init) + Σ_t w_t · tree_t(row)
// (GBMRegressionModel.predict, regression/GBMRegressor.scala:531-539; BaggingRegressionModel.predict,
// regression/BaggingRegressor.scala:221-228).  `blob` is the packed chunk of trees, copied verbatim into shared memory:
//   [0)            double   w[T]
//   [off_coloff)   uint64   byte offset of local column c in X8 (column * ld8), c < C
//   [off_nodes)    uint2    nodes: x = local column | rank threshold << 16 | leaf << 31, y = left | right << 16 (tree-local)
//   [off_treeoff)  int32    first node of tree t (T + 1 entries)
//   [off_treecls)  int32    class of tree t (T entries; se_forest_agg's GBM classifier only, else off_treecls == 0)
//   [off_values)   float    leaf value per node
//   [off_ranks)    uint8    (shared memory only) the tile's ranks, [C][tile rows]
struct ForestArgs {
  const uint8_t* X8 = nullptr;
  int64_t n = 0, ld8 = 0;
  const unsigned char* blob = nullptr;
  int blob_bytes = 0;  // multiple of 16
  int T = 0, C = 0;
  int off_coloff = 0, off_nodes = 0, off_treeoff = 0, off_treecls = 0, off_values = 0, off_ranks = 0;
  double init = 0.0;
  int accumulate = 0;
  float* out = nullptr;
};
constexpr int kForestTile = 256;              // rows per CTA tile (one row per thread)
constexpr int kForestSmemBudget = 54 * 1024;  // per CTA: four CTAs per SM (the walk is latency-bound: warps matter more than chunk size)
cudaError_t launch_forest_predict(const ForestArgs& a, int sms, cudaStream_t s);

// One level of a packed tree for the row whose ranks start at myr (rank of local column c at myr[c * TILE]).
template <int TILE>
__device__ __forceinline__ void forest_step(const uint2* __restrict__ nodes, const unsigned char* __restrict__ myr, int& nd,
                                            bool& live) {
  const uint2 w = nodes[nd];
  live = (w.x >> 31) == 0;
  if (live) {
    const uint32_t rank = myr[(w.x & 0xFFFFu) * TILE];
    nd = (int)((rank <= ((w.x >> 16) & 0xFFu)) ? (w.y & 0xFFFFu) : (w.y >> 16));
  }
}

// A classifier forest in ONE pass with the aggregation's epilogue (se_forest_agg, se_agg.cu): the chunk's trees are
// staged as for forest_predict_kernel, each row's C class totals are fp64 in shared memory ([C][kForestAggTile] after
// the ranks), carried between chunks in `acc` ([C][ld_acc] fp64) and finished by finalize_row / finalize_real_row.
constexpr int kForestAggTile = 128;        // rows per CTA tile: C x 128 fp64 totals (32 KB at the class limit)
constexpr int kForestAggMaxClasses = 32;   // SE_FOREST_AGG_MAX_CLASSES
struct ForestAggArgs {
  ForestArgs f;                  // the chunk (f.init, f.accumulate and f.out unused)
  int kind = 0, K = 0, C = 0, dim = 1, loss = 0, M = 0;
  double sum_a = 0.0;            // Σ of the tree weights (boosting discrete epilogue)
  double init[kForestAggMaxClasses] = {};  // GBM classifier: the totals of the first chunk start here
  const float* probs = nullptr;  // [chunk nodes][K] leaf class probabilities (bagging soft, boosting real), read through L1
  double* acc = nullptr;         // [C][ld_acc] totals between chunks
  int64_t ld_acc = 0;
  int first = 1, last = 1;       // the chunk starts from init / finishes the rows
  float* raw = nullptr;
  float* prob = nullptr;
  float* label = nullptr;
  int64_t ld_out = 0;
  int* bad_label = nullptr;
};
cudaError_t launch_forest_agg(const ForestAggArgs& a, int sms, cudaStream_t s);
// The weighted median of a forest of at most 64 regression trees in ONE pass (se_forest_median, se_agg.cu): a CTA walks
// every chunk of trees over its 128-row tile in turn, re-staging the chunk's packed trees and ranks as
// forest_predict_kernel stages them, and keeps each row's M leaf values in its own column of shared memory
// ([M][kForestMedianTile] fp32 at vals_off) until the last chunk; the median is then taken as agg_wmedian_fast_kernel
// takes it, and the rows inside its rounding margin (mode 1) or every row (mode 0) by wm_exact_pick on the same values.
constexpr int kForestMedianTile = 128;
constexpr int kForestMedianMaxTrees = 64;  // SE_FOREST_MEDIAN_MAX_TREES
struct ForestMedianChunk {
  int blob_off = 0, blob_bytes = 0;  // the chunk's packed trees at blob + blob_off (ForestArgs layout, multiple of 16)
  int T = 0, C = 0, t0 = 0;          // its trees are t0 .. t0 + T - 1 of the forest, over C local columns
  int off_coloff = 0, off_nodes = 0, off_treeoff = 0, off_values = 0;
};
struct ForestMedianArgs {
  const uint8_t* X8 = nullptr;
  int64_t n = 0, ld8 = 0;
  const unsigned char* blob = nullptr;
  int n_chunks = 0, M = 0;
  int vals_off = 0;               // shared-memory byte offset of the leaf values: past every chunk's blob and ranks
  int mode = 0;                   // 0: exact sort for every row; 1: fast path + margin; 2: all weights equal, no margin
  double total = 0.0, tau = -1.0; // Σ weights in model order, the margin 8·M·2⁻⁵³·total (mode 1)
  double w[kForestMedianMaxTrees] = {};
  ForestMedianChunk chunk[kForestMedianMaxTrees];
  unsigned int* deferred = nullptr;  // mode 1: counts the rows resolved by the exact sort (nullable)
  float* out = nullptr;
};
cudaError_t launch_forest_median(const ForestMedianArgs& a, size_t smem, int sms, cudaStream_t s);
// CTAs of the kernel for M trees one SM can hold by its registers alone (>= 1)
cudaError_t forest_median_ctas_per_sm(int M, int* ctas);
// ---- regression- and classification-tree fit over the uint8 rank matrix (se_tree_fit.cu) -----
// Nodes are heap-indexed (root 1, children 2h, 2h + 1), so depth <= 8 needs 511 records.
constexpr int kTreeFitHeap = 512;
constexpr int kTreeFitSmemBudget = 56 * 1024;  // shared-memory histograms per CTA: four CTAs per SM
constexpr int kTreeFitMaxClasses = 64;         // classification: two classes per lane of the split search's warp
struct TreeFitNode {                 // 64 B, downloaded once at the end of a fit
  double cnt, w, s, q;               // rawCount, W, S, Q of the node's in-bag rows (classification: s, q unused)
  double pred;                       // S / W (classification: the label)
  double gain;                       // of the chosen split (state 2)
  int32_t state;                     // 0 unused, 1 leaf, 2 split
  int32_t col, bin;                  // split: subspace-local column, left when rank <= bin
  float thr;                         // split: the fp32 candidate
  float value;                       // (float) pred
  int32_t pad;
};
struct TreeFitArgs {
  const uint8_t* X8 = nullptr;
  int64_t ld8 = 0, n = 0;
  const int32_t* cols = nullptr;     // device [S]: global column of subspace entry k
  const int32_t* n_edges = nullptr;  // device [d]: candidates per column
  const float* edges = nullptr;      // device [d][256]
  int S = 0, nb = 0, L = 0, cb = 1, max_depth = 0;
  int search = 1, route = 0, has_w = 0;
  const float* r = nullptr;          // labels
  const float* w = nullptr;          // weights (has_w)
  const float* bag = nullptr;        // multiplicities or nullptr
  const uint16_t* nid_in = nullptr;  // node of every row before this level's step (nullptr: the root)
  uint16_t* nid_out = nullptr;       // after it (written by the first column block)
  uint2* dec = nullptr;              // [kTreeFitHeap] x: global split column (~0: none), y: bin | open << 31
  TreeFitNode* nodes = nullptr;      // [kTreeFitHeap]
  double* hist = nullptr;            // [2^L][S][nb][sw]
  int64_t words_per_cta = 0;         // 4-row groups per CTA row range
  int min_instances = 1;
  double min_info_gain = 0.0, min_weight_fraction = 0.0;
  float* out = nullptr;              // final pass: leaf value per row (classification: label, or K rows of ld_out)
  // classification (K >= 2; K == 0 is the regression fit): labels in `r` are class indices
  int K = 0, sw = 4;                 // sw: doubles per histogram bin (regression 4; classification K, + 1 when has_w)
  int entropy = 0, out_proba = 0;
  int64_t ld_out = 0;
  double* cw = nullptr;              // [kTreeFitHeap][K] class weights of every node
  float* prob = nullptr;             // [kTreeFitHeap][K] fp32 of cw / W (all 0 when W == 0)
  int4* prn = nullptr;               // [kTreeFitHeap] after pruning: x the node whose statistics a row at h outputs,
                                     // y its label, z 1 when h is a leaf of the pruned tree
};
cudaError_t launch_tree_fit_init(TreeFitNode* nodes, uint2* dec, cudaStream_t s);
// smem_mode 1: shared-memory histograms of a.cb columns per CTA (smem bytes), folded into a.hist; 0: global atomics
cudaError_t launch_tree_fit_hist(const TreeFitArgs& a, int smem_mode, int grid_y, size_t smem, cudaStream_t s);
cudaError_t launch_tree_fit_split(const TreeFitArgs& a, cudaStream_t s);
cudaError_t launch_tree_fit_prune(const TreeFitArgs& a, cudaStream_t s);  // classification only
cudaError_t launch_tree_fit_out(const TreeFitArgs& a, int sms, cudaStream_t s);

cudaError_t launch_linear_predict(const float* X, int64_t n, int64_t ld, int n_coef,
                                  const float* coef, const int32_t* cols, float intercept,
                                  float* out, int sms, cudaStream_t s);

// ---- exact quantile by radix select (se_util.cu) ---------------------------------------------
// One pass: histogram (256 bins, fp64 counts in `hist`) of byte `shift/8` of the order-preserving key of each
// value whose higher bytes equal `prefix` (mask = bits above the byte).  value = a[i], or |a[i] - b[i]| when b.
cudaError_t launch_radix_hist(const float* a, const float* b, int64_t n, uint32_t prefix, uint32_t mask,
                              int shift, double* hist, int sms, cudaStream_t s);

// ---- ingest (se_util.cu): row-major host chunk [rows][d] -> column-major X[d][ld] rows [row0, row0+rows)
cudaError_t launch_transpose_rows(const float* src, int64_t rows, int d, float* X, int64_t ld, int64_t row0,
                                  cudaStream_t s);

// ---- utilities (se_util.cu) ------------------------------------------------------------------
// raises *bad (mapped host memory) when a label is not an integer class index in [0, K)
cudaError_t launch_validate_labels(const float* y, int64_t n, int K, int* bad, int sms, cudaStream_t s);
cudaError_t launch_fill(float* p, float v, int64_t n, int sms, cudaStream_t s);
cudaError_t launch_fill_synthetic(float* p, int kind, uint64_t seed, double a, double b, int64_t n,
                                  int64_t index_offset, int sms, cudaStream_t s);
cudaError_t launch_f64_to_f32(const double* src, float* dst, int64_t n, int sms, cudaStream_t s);
cudaError_t launch_scale_copy(const float* src, float* dst, float scale, int64_t n, int sms,
                              cudaStream_t s);

}  // namespace se
