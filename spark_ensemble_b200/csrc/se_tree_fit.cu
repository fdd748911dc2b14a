// se_tree_fit.cu — regression-tree learner over the uint8 rank matrix (DESIGN.md §3 "Device tree fit").
//
// Spark's DecisionTreeRegressor (RandomForest.run for one tree: variance impurity, continuous features, level-wise best
// split over binned candidates, prune = true) as a fixed sequence of launches.  The rank matrix of SE_SLOT_X holds, per
// column, the fit's split candidates t_0 < ... < t_{m-1} (se_tree_fit_bins); rank(x) = #{t_j < x}, so `x <= t_j` is
// `rank <= j` and a row's bin in the histogram of a column IS its rank (NaN ranks 255 and goes right of every candidate).
//
// Nodes carry heap indices (root 1, children 2h and 2h + 1; depth <= 8 keeps them below 512).  Per level L:
//   tree_hist_kernel   every row moves one level down with one rank gather of its node's split column (rows whose node
//                      is a leaf stay), then adds (rawCount, W, S, Q) = (c, c·w, c·w·r, c·w·r²) of in-bag rows at open
//                      nodes to hist[node][column][bin] — per CTA in shared memory over a block of columns, folded into
//                      fp64 global totals, or straight into the global totals when one column's histogram for every
//                      node of the level does not fit in shared memory;
//   tree_split_kernel  one CTA per node of the level: prefix sums over the bins of every column, Spark's validity rules
//                      and gain, best split by (gain, first column, first candidate); writes the routing decision and the
//                      child records the next level reads.
// tree_out_kernel routes every row to its leaf and writes the leaf value.  Nothing returns to the host in between.
//
// Classification (DecisionTreeClassifier, gini or entropy; a.K >= 2 classes) reuses the routing, the level loop and the
// histogram kernel; a bin then holds the class weights Σ c·w per class (plus rawCount Σ c when weighted), the split
// search runs a warp per (node, column) with the classes over the lanes (tree_split_cls_kernel), and
// tree_prune_cls_kernel applies Spark's pruning before tree_out_kernel writes the label or the K probabilities.
//
// One launch sequence can grow T independent trees over the same rows, labels, weights and bag, each over its own
// column subspace (se_forest_fit, bagging's members): the tree is a grid dimension of every kernel (TreeView).  The
// batch shares one bin count nb, the largest of its columns', so a tree's histogram only gains empty bins between its
// candidates and the NaN bin: its sums, and so its splits, are those of its own fit.
#include "se_kernels.h"

namespace se {

namespace {

constexpr int kTfBlock = 256;
constexpr unsigned kDecNone = 0xFFFFFFFFu;  // dec.x: node does not split
constexpr unsigned kDecOpen = 0x80000000u;  // dec.y: node is searched at its level

struct Stat4 {
  double c, w, s, q;
};

__device__ __forceinline__ double impurity(const Stat4& a) { return a.w == 0.0 ? 0.0 : (a.q - a.s * a.s / a.w) / a.w; }

__device__ __forceinline__ Stat4 load4(const double* p) { return Stat4{p[0], p[1], p[2], p[3]}; }

// Tree t of a fit (TreeFitArgs: T trees): its columns, records, level-L histogram and node ids.
struct TreeView {
  const int32_t* cols;
  int S;
  uint2* dec;
  TreeFitNode* nodes;
  double* hist;
  double* cw;
  float* prob;
  int4* prn;
  const uint16_t* nid_in;
  uint16_t* nid_out;
};

__device__ __forceinline__ TreeView tree_view(const TreeFitArgs& a, int t) {
  const int off = __ldg(a.sub_off + t);
  TreeView v;
  v.cols = a.cols + off;
  v.S = __ldg(a.sub_off + t + 1) - off;
  v.dec = a.dec + (int64_t)t * kTreeFitHeap;
  v.nodes = a.nodes + (int64_t)t * kTreeFitHeap;
  v.hist = a.hist + ((int64_t)a.nb * a.sw << a.L) * off;
  v.cw = a.cw + (int64_t)t * kTreeFitHeap * a.K;
  v.prob = a.prob + (int64_t)t * kTreeFitHeap * a.K;
  v.prn = a.prn + (int64_t)t * kTreeFitHeap;
  v.nid_in = a.nid_in ? a.nid_in + (int64_t)t * a.nid_stride : nullptr;
  v.nid_out = a.nid_out ? a.nid_out + (int64_t)t * a.nid_stride : nullptr;
  return v;
}

// One tile = 4 consecutive rows per thread: node indices in, one routing step, node indices out.
__device__ __forceinline__ void route4(const TreeFitArgs& a, const TreeView& tv, int64_t i0, unsigned (&h)[4]) {
  if (tv.nid_in) {
    const uint2 v = *reinterpret_cast<const uint2*>(tv.nid_in + i0);
    h[0] = v.x & 0xFFFFu; h[1] = v.x >> 16; h[2] = v.y & 0xFFFFu; h[3] = v.y >> 16;
  } else {
    h[0] = h[1] = h[2] = h[3] = 1u;
  }
  if (!a.route) return;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const uint2 d = __ldg(tv.dec + h[e]);
    if (d.x != kDecNone && i0 + e < a.n) {
      const unsigned rk = __ldg(a.X8 + (int64_t)d.x * a.ld8 + i0 + e);
      h[e] = 2u * h[e] + (rk > (d.y & 0xFFFFu) ? 1u : 0u);
    }
  }
}

// CLS: a classification fit adds c·w to the bin entry of the row's class (labels are class indices, clamped into
// [0, K) for memory safety) and c to entry K when weighted: a bin holds sw = K (+ 1) doubles instead of 4.
// blockIdx.z is the tree.  The column blocks are sized by the largest subspace: a CTA whose block starts past its own
// tree's columns has nothing to do (block 0 always has a column, so the node ids are still written).
template <bool SMEM, bool HAS_W, bool CLS>
__global__ void __launch_bounds__(kTfBlock) tree_hist_kernel(const TreeFitArgs a) {
  extern __shared__ double s_hist[];  // [2^L][cb][nb][sw]
  const int SW = CLS ? a.sw : 4;
  const TreeView tv = tree_view(a, blockIdx.z);
  const int k0 = blockIdx.x * a.cb;
  if (k0 >= tv.S) return;
  const int ncb = min(a.cb, tv.S - k0);
  const int nodes = 1 << a.L;
  const int64_t sz = (int64_t)nodes * a.cb * a.nb * SW;
  if (SMEM) {
    for (int64_t t = threadIdx.x; t < sz; t += kTfBlock) s_hist[t] = 0.0;
    __syncthreads();
  }
  const int64_t nw = (a.n + 3) >> 2;
  const int64_t w0 = (int64_t)blockIdx.y * a.words_per_cta;
  const int64_t w1 = min(nw, w0 + a.words_per_cta);
  const unsigned hbase = 1u << a.L;
  for (int64_t g = w0 + threadIdx.x; g < w1; g += kTfBlock) {
    const int64_t i0 = 4 * g;
    unsigned h[4];
    route4(a, tv, i0, h);
    if (tv.nid_out && blockIdx.x == 0)
      *reinterpret_cast<uint2*>(tv.nid_out + i0) = make_uint2(h[0] | (h[1] << 16), h[2] | (h[3] << 16));
    const float4 r4 = *reinterpret_cast<const float4*>(a.r + i0);
    const float4 w4 = HAS_W ? *reinterpret_cast<const float4*>(a.w + i0) : make_float4(1.f, 1.f, 1.f, 1.f);
    const float4 c4 = a.bag ? *reinterpret_cast<const float4*>(a.bag + i0) : make_float4(1.f, 1.f, 1.f, 1.f);
    const float rr[4] = {r4.x, r4.y, r4.z, r4.w}, ww[4] = {w4.x, w4.y, w4.z, w4.w}, cc[4] = {c4.x, c4.y, c4.z, c4.w};
    int node[4], cls[4] = {0, 0, 0, 0};  // initialised: otherwise ptxas keeps cls in local memory
    double vc[4], vw[4], vs[4], vq[4];
    bool any = false;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      node[e] = -1;
      if (i0 + e < a.n && cc[e] > 0.f && h[e] >= hbase && (__ldg(tv.dec + h[e]).y & kDecOpen)) {
        node[e] = (int)(h[e] - hbase);
        vc[e] = (double)cc[e];
        vw[e] = (double)cc[e] * (double)ww[e];
        if constexpr (CLS) {
          cls[e] = min(max((int)rr[e], 0), a.K - 1);
        } else {
          vs[e] = vw[e] * (double)rr[e];
          vq[e] = vs[e] * (double)rr[e];
        }
        any = true;
      }
    }
    if (!any) continue;
    for (int kk = 0; kk < ncb; ++kk) {
      const int k = k0 + kk;
      const unsigned word = *reinterpret_cast<const unsigned*>(a.X8 + (int64_t)__ldg(tv.cols + k) * a.ld8 + i0);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (node[e] < 0) continue;
        unsigned b = (word >> (8 * e)) & 0xFFu;
        if (b == 255u) b = (unsigned)a.nb - 1u;
        double* p = SMEM ? s_hist + (((int64_t)node[e] * a.cb + kk) * a.nb + b) * SW
                         : tv.hist + (((int64_t)node[e] * tv.S + k) * a.nb + b) * SW;
        if constexpr (CLS) {
          atomicAdd(p + cls[e], vw[e]);
          if (HAS_W) atomicAdd(p + a.K, vc[e]);
        } else {
          atomicAdd(p + 0, vc[e]);
          if (HAS_W) atomicAdd(p + 1, vw[e]);
          atomicAdd(p + 2, vs[e]);
          atomicAdd(p + 3, vq[e]);
        }
      }
    }
  }
  if (SMEM) {
    __syncthreads();
    if constexpr (CLS) {  // entry by entry: most class entries of a bin are empty
      for (int64_t t = threadIdx.x; t < sz; t += kTfBlock) {
        const double s = s_hist[t];
        if (s == 0.0) continue;
        const int64_t cell = t / SW;
        const int b = (int)(cell % a.nb);
        const int kk = (int)((cell / a.nb) % a.cb);
        const int p = (int)(cell / ((int64_t)a.nb * a.cb));
        if (kk >= ncb) continue;
        atomicAdd(tv.hist + (((int64_t)p * tv.S + k0 + kk) * a.nb + b) * SW + (int)(t - cell * SW), s);
      }
    } else {
      const int64_t cells = (int64_t)nodes * a.cb * a.nb;
      for (int64_t t = threadIdx.x; t < cells; t += kTfBlock) {
        const double* s = s_hist + 4 * t;
        if (s[0] == 0.0) continue;  // no in-bag row fell into this bin
        const int b = (int)(t % a.nb);
        const int kk = (int)((t / a.nb) % a.cb);
        const int p = (int)(t / ((int64_t)a.nb * a.cb));
        if (kk >= ncb) continue;
        double* g = tv.hist + (((int64_t)p * tv.S + k0 + kk) * a.nb + b) * 4;
        atomicAdd(g + 0, s[0]);
        if (HAS_W) atomicAdd(g + 1, s[1]);
        atomicAdd(g + 2, s[2]);
        atomicAdd(g + 3, s[3]);
      }
    }
  }
}

__device__ __forceinline__ Stat4 bin_stat(const double* hk, int b, bool has_w) {
  Stat4 v = load4(hk + 4 * b);
  if (!has_w) v.w = v.c;  // unweighted: W is the (integer, exact) count
  return v;
}

// Best split of one column: max gain over its candidates, first candidate on ties; gain -inf when none is valid.
__device__ void best_of_column(const TreeFitArgs& a, const double* hk, int ncand, double minW, Stat4& tot, double& best_g,
                               int& best_j) {
  tot = Stat4{0, 0, 0, 0};
  for (int b = 0; b < a.nb; ++b) {
    const Stat4 v = bin_stat(hk, b, a.has_w);
    tot.c += v.c; tot.w += v.w; tot.s += v.s; tot.q += v.q;
  }
  best_g = -INFINITY;
  best_j = -1;
  const double imp = impurity(tot);
  Stat4 l{0, 0, 0, 0};
  for (int j = 0; j < ncand; ++j) {
    const Stat4 v = bin_stat(hk, j, a.has_w);
    l.c += v.c; l.w += v.w; l.s += v.s; l.q += v.q;
    // no in-bag row ranks j: candidate j repeats candidate j - 1's partition, which is taken first.  Skipped rather
    // than left to the strict > below: the compiled gain of equal sums is not guaranteed the same bits in every
    // iteration of this loop, and a later equal candidate must not win by a rounding
    if (j > 0 && v.c == 0.0) continue;
    const Stat4 rt{tot.c - l.c, tot.w - l.w, tot.s - l.s, tot.q - l.q};
    if (l.c < (double)a.min_instances || rt.c < (double)a.min_instances) continue;
    if (l.w < minW || rt.w < minW) continue;
    const double g = imp - (l.w / tot.w) * impurity(l) - (rt.w / tot.w) * impurity(rt);
    if (g < a.min_info_gain) continue;
    if (g > best_g) { best_g = g; best_j = j; }
  }
}

__device__ __forceinline__ void set_node(TreeFitNode& nd, const Stat4& s) {
  nd.cnt = s.c; nd.w = s.w; nd.s = s.s; nd.q = s.q;
  nd.pred = s.s / s.w;
  nd.value = (float)nd.pred;
}

// grid (2^L, T): node p of the level of tree blockIdx.y
__global__ void __launch_bounds__(kTfBlock) tree_split_kernel(const TreeFitArgs a) {
  const int p = blockIdx.x;
  const unsigned h = (1u << a.L) + (unsigned)p;
  const TreeView tv = tree_view(a, blockIdx.y);
  if (!(tv.dec[h].y & kDecOpen)) return;
  TreeFitNode* nodes = tv.nodes;
  const double* hp = tv.hist + (int64_t)p * tv.S * a.nb * 4;
  __shared__ double s_g[kTfBlock / 32];
  __shared__ int s_k[kTfBlock / 32], s_j[kTfBlock / 32];
  if (a.L == 0 && threadIdx.x == 0) {  // the root's statistics: totals of the first column
    Stat4 t{0, 0, 0, 0};
    for (int b = 0; b < a.nb; ++b) {
      const Stat4 v = bin_stat(hp, b, a.has_w);
      t.c += v.c; t.w += v.w; t.s += v.s; t.q += v.q;
    }
    set_node(nodes[1], t);
    nodes[1].state = 1;
  }
  __syncthreads();
  const double minW = a.min_weight_fraction * nodes[1].w;
  double bg = -INFINITY;
  int bk = 0x7FFFFFFF, bj = -1;
  if (a.search) {
    for (int k = threadIdx.x; k < tv.S; k += kTfBlock) {
      const int ncand = __ldg(a.n_edges + __ldg(tv.cols + k));
      if (ncand <= 0) continue;
      Stat4 tot;
      double g;
      int j;
      best_of_column(a, hp + (int64_t)k * a.nb * 4, ncand, minW, tot, g, j);
      if (j >= 0 && g > bg) { bg = g; bk = k; bj = j; }  // k ascends per thread: strict > keeps the first column
    }
  }
  // block arg-max by (gain desc, column asc)
  for (int off = 16; off > 0; off >>= 1) {
    const double og = __shfl_down_sync(0xFFFFFFFFu, bg, off);
    const int ok = __shfl_down_sync(0xFFFFFFFFu, bk, off);
    const int oj = __shfl_down_sync(0xFFFFFFFFu, bj, off);
    if (oj >= 0 && (bj < 0 || og > bg || (og == bg && ok < bk))) { bg = og; bk = ok; bj = oj; }
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { s_g[wid] = bg; s_k[wid] = bk; s_j[wid] = bj; }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 1; w < kTfBlock / 32; ++w)
    if (s_j[w] >= 0 && (bj < 0 || s_g[w] > bg || (s_g[w] == bg && s_k[w] < bk))) { bg = s_g[w]; bk = s_k[w]; bj = s_j[w]; }
  TreeFitNode& nd = nodes[h];
  if (bj < 0 || !(bg > 0.0)) {  // no valid split, or no positive gain: leaf
    nd.state = 1;
    tv.dec[h] = make_uint2(kDecNone, 0u);
    return;
  }
  const int gcol = __ldg(tv.cols + bk);
  const double* hk = hp + (int64_t)bk * a.nb * 4;
  Stat4 tot{0, 0, 0, 0}, l{0, 0, 0, 0};
  for (int b = 0; b < a.nb; ++b) {
    const Stat4 v = bin_stat(hk, b, a.has_w);
    tot.c += v.c; tot.w += v.w; tot.s += v.s; tot.q += v.q;
    if (b <= bj) { l.c += v.c; l.w += v.w; l.s += v.s; l.q += v.q; }
  }
  const Stat4 rt{tot.c - l.c, tot.w - l.w, tot.s - l.s, tot.q - l.q};
  nd.state = 2;
  nd.gain = bg;
  nd.col = bk;
  nd.bin = bj;
  nd.thr = __ldg(a.edges + (int64_t)gcol * 256 + bj);
  tv.dec[h] = make_uint2((unsigned)gcol, (unsigned)bj);
  const bool last = a.L + 1 >= a.max_depth;
  const Stat4 ch[2] = {l, rt};
  for (int s = 0; s < 2; ++s) {
    TreeFitNode& c = nodes[2 * h + s];
    set_node(c, ch[s]);
    const bool leaf = last || fabs(impurity(ch[s])) < 0x1p-52;
    c.state = 1;
    tv.dec[2 * h + s] = make_uint2(kDecNone, leaf ? 0u : kDecOpen);
  }
}

// ---- classification: a warp per (node, column), lane l holds classes l and l + 32 -------------------------------
constexpr unsigned kFull = 0xFFFFFFFFu;

// Butterfly sum: a + b == b + a, so every lane ends with the same bits.
__device__ __forceinline__ double warp_sum(double v) {
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(kFull, v, off);
  return v;
}

// Spark's Gini / Entropy calculators over the class weights (n0, n1) of every lane, W = Σ_k n_k (0 when W == 0).
// Classes with zero weight add nothing; the classes' terms are summed by the butterfly, not in class order.
template <bool ENTROPY>
__device__ __forceinline__ double warp_impurity(double n0, double n1, double W) {
  if (W == 0.0) return 0.0;
  double t = 0.0;
  if (n0 != 0.0) { const double p = n0 / W; t += ENTROPY ? p * (log(p) / log(2.0)) : p * p; }
  if (n1 != 0.0) { const double p = n1 / W; t += ENTROPY ? p * (log(p) / log(2.0)) : p * p; }
  t = warp_sum(t);
  return ENTROPY ? -t : 1.0 - t;
}

// Spark's indexOfLargestArrayElement: the first class of the largest weight.
__device__ __forceinline__ int warp_argmax(double n0, double n1, int K) {
  const int lane = threadIdx.x & 31;
  double v = lane < K ? n0 : -1.0;
  int i = lane;
  if (lane + 32 < K && n1 > v) { v = n1; i = lane + 32; }
  for (int off = 16; off > 0; off >>= 1) {
    const double ov = __shfl_xor_sync(kFull, v, off);
    const int oi = __shfl_xor_sync(kFull, i, off);
    if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
  }
  return i;
}

// Class weights of bins [0, nbins) of one column's histogram: (lane's two classes, rawCount)
__device__ __forceinline__ void cls_sums(const TreeFitArgs& a, const double* hk, int nbins, double& n0, double& n1,
                                         double& c) {
  const int lane = threadIdx.x & 31;
  n0 = n1 = c = 0.0;
  for (int b = 0; b < nbins; ++b) {
    const double* e = hk + (int64_t)b * a.sw;
    if (lane < a.K) n0 += e[lane];
    if (lane + 32 < a.K) n1 += e[lane + 32];
    if (a.has_w) c += e[a.K];
  }
}

// Writes node h's records from its class weights (the whole warp): rawCount c, W, label, probabilities; returns the
// impurity.  An unweighted fit's rawCount is W.
template <bool ENTROPY>
__device__ double cls_set_node(const TreeFitArgs& a, const TreeView& tv, int h, double n0, double n1, double c) {
  const int lane = threadIdx.x & 31;
  const double W = warp_sum(n0 + n1);
  const double imp = warp_impurity<ENTROPY>(n0, n1, W);
  const int label = warp_argmax(n0, n1, a.K);
  double* cw = tv.cw + (int64_t)h * a.K;
  float* pr = tv.prob + (int64_t)h * a.K;
  if (lane < a.K) { cw[lane] = n0; pr[lane] = W == 0.0 ? 0.f : (float)(n0 / W); }
  if (lane + 32 < a.K) { cw[lane + 32] = n1; pr[lane + 32] = W == 0.0 ? 0.f : (float)(n1 / W); }
  if (lane == 0) {
    TreeFitNode& nd = tv.nodes[h];
    nd.cnt = a.has_w ? c : W;
    nd.w = W;
    nd.pred = (double)label;
    nd.value = (float)label;
  }
  return imp;
}

// grid (2^L, T): node p of the level of tree blockIdx.y
template <bool ENTROPY>
__global__ void __launch_bounds__(kTfBlock) tree_split_cls_kernel(const TreeFitArgs a) {
  const int p = blockIdx.x;
  const unsigned h = (1u << a.L) + (unsigned)p;
  const TreeView tv = tree_view(a, blockIdx.y);
  if (!(tv.dec[h].y & kDecOpen)) return;
  TreeFitNode* nodes = tv.nodes;
  const int64_t col_stride = (int64_t)a.nb * a.sw;
  const double* hp = tv.hist + (int64_t)p * tv.S * col_stride;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __shared__ double s_g[kTfBlock / 32];
  __shared__ int s_k[kTfBlock / 32], s_j[kTfBlock / 32];
  if (a.L == 0 && wid == 0) {  // the root's statistics: totals of the first column
    double n0, n1, c;
    cls_sums(a, hp, a.nb, n0, n1, c);
    cls_set_node<ENTROPY>(a, tv, 1, n0, n1, c);
    if (lane == 0) nodes[1].state = 1;
  }
  __syncthreads();
  const double minW = a.min_weight_fraction * nodes[1].w;
  double bg = -INFINITY;
  int bk = 0x7FFFFFFF, bj = -1;
  if (a.search) {
    for (int k = wid; k < tv.S; k += kTfBlock / 32) {  // k ascends per warp: strict > keeps the first column
      const int ncand = __ldg(a.n_edges + __ldg(tv.cols + k));
      if (ncand <= 0) continue;
      const double* hk = hp + (int64_t)k * col_stride;
      double t0, t1, tc;
      cls_sums(a, hk, a.nb, t0, t1, tc);
      const double W = warp_sum(t0 + t1);
      const double imp = warp_impurity<ENTROPY>(t0, t1, W);
      const double tcount = a.has_w ? tc : W;
      double l0 = 0.0, l1 = 0.0, lc = 0.0, prev = -1.0;
      for (int j = 0; j < ncand; ++j) {
        const double* e = hk + (int64_t)j * a.sw;
        if (lane < a.K) l0 += e[lane];
        if (lane + 32 < a.K) l1 += e[lane + 32];
        if (a.has_w) lc += e[a.K];
        const double r0 = t0 - l0, r1 = t1 - l1;
        const double lw = warp_sum(l0 + l1), rw = warp_sum(r0 + r1);
        const double lcount = a.has_w ? lc : lw, rcount = a.has_w ? tcount - lc : rw;
        // the left rawCount (integer sums, exact) did not grow: no in-bag row ranks j, candidate j repeats candidate
        // j - 1's partition, which is taken first (as in tree_split_kernel).  The same on every lane: warp-uniform
        const bool repeat = j > 0 && lcount == prev;
        prev = lcount;
        if (repeat) continue;
        if (lcount < (double)a.min_instances || rcount < (double)a.min_instances) continue;
        if (lw < minW || rw < minW) continue;
        const double tw = lw + rw;
        const double g = imp - (lw / tw) * warp_impurity<ENTROPY>(l0, l1, lw) - (rw / tw) * warp_impurity<ENTROPY>(r0, r1, rw);
        if (g < a.min_info_gain) continue;
        if (g > bg) { bg = g; bk = k; bj = j; }
      }
    }
  }
  if (lane == 0) { s_g[wid] = bg; s_k[wid] = bk; s_j[wid] = bj; }
  __syncthreads();
  if (wid != 0) return;
  // block arg-max by (gain desc, column asc); every lane of warp 0 reads the same values
  bg = s_g[0]; bk = s_k[0]; bj = s_j[0];
  for (int w = 1; w < kTfBlock / 32; ++w)
    if (s_j[w] >= 0 && (bj < 0 || s_g[w] > bg || (s_g[w] == bg && s_k[w] < bk))) { bg = s_g[w]; bk = s_k[w]; bj = s_j[w]; }
  TreeFitNode& nd = nodes[h];
  if (bj < 0 || !(bg > 0.0)) {  // no valid split, or no positive gain: leaf
    if (lane == 0) {
      nd.state = 1;
      tv.dec[h] = make_uint2(kDecNone, 0u);
    }
    return;
  }
  const int gcol = __ldg(tv.cols + bk);
  const double* hk = hp + (int64_t)bk * col_stride;
  double t0, t1, tc, l0, l1, lc;
  cls_sums(a, hk, a.nb, t0, t1, tc);
  cls_sums(a, hk, bj + 1, l0, l1, lc);
  if (lane == 0) {
    nd.state = 2;
    nd.gain = bg;
    nd.col = bk;
    nd.bin = bj;
    nd.thr = __ldg(a.edges + (int64_t)gcol * 256 + bj);
    tv.dec[h] = make_uint2((unsigned)gcol, (unsigned)bj);
  }
  const bool last = a.L + 1 >= a.max_depth;
  for (int s = 0; s < 2; ++s) {
    const unsigned c = 2 * h + s;
    const double imp = s == 0 ? cls_set_node<ENTROPY>(a, tv, c, l0, l1, lc)
                              : cls_set_node<ENTROPY>(a, tv, c, t0 - l0, t1 - l1, tc - lc);
    const bool leaf = last || fabs(imp) < 0x1p-52;
    if (lane == 0) {
      nodes[c].state = 1;
      tv.dec[c] = make_uint2(kDecNone, leaf ? 0u : kDecOpen);
    }
  }
}

// Spark's LearningNode.toNode(prune = true), bottom-up: an internal node whose two children are leaves with the same
// label becomes a leaf that keeps the children's label and the node's OWN statistics (so its probabilities are the
// parent's).  Then, top-down, every heap index gets the node whose statistics its rows output.  One thread per tree
// (CTA blockIdx.x): 511 nodes.
__global__ void tree_prune_cls_kernel(const TreeFitArgs a) {
  if (threadIdx.x != 0) return;
  const TreeView tv = tree_view(a, blockIdx.x);
  __shared__ unsigned char leaf[kTreeFitHeap];
  __shared__ int label[kTreeFitHeap], rep[kTreeFitHeap];
  for (int h = 1; h < kTreeFitHeap; ++h) {
    leaf[h] = tv.nodes[h].state != 2;
    label[h] = (int)tv.nodes[h].pred;
  }
  for (int h = kTreeFitHeap / 2 - 1; h >= 1; --h)
    if (!leaf[h] && leaf[2 * h] && leaf[2 * h + 1] && label[2 * h] == label[2 * h + 1]) {
      leaf[h] = 1;
      label[h] = label[2 * h];
    }
  rep[1] = 1;
  tv.prn[0] = make_int4(0, 0, 0, 0);
  for (int h = 1; h < kTreeFitHeap; ++h) {
    if (h > 1) rep[h] = leaf[h >> 1] ? rep[h >> 1] : h;  // below a leaf of the pruned tree: that leaf
    tv.prn[h] = make_int4(rep[h], label[rep[h]], leaf[h], 0);
  }
}

// one CTA per tree
__global__ void tree_fit_init_kernel(TreeFitNode* nodes, uint2* dec) {
  nodes += (int64_t)blockIdx.x * kTreeFitHeap;
  dec += (int64_t)blockIdx.x * kTreeFitHeap;
  for (int h = threadIdx.x; h < kTreeFitHeap; h += blockDim.x) {
    TreeFitNode z = {};
    nodes[h] = z;
    dec[h] = make_uint2(kDecNone, h == 1 ? kDecOpen : 0u);
  }
}

// CLS: the output of the pruned tree (tree_prune_cls_kernel): the label, or the K probabilities into rows of ld_out
template <bool CLS>
__global__ void __launch_bounds__(kTfBlock) tree_out_kernel(const TreeFitArgs a) {
  const int64_t nw = (a.n + 3) >> 2;
  const TreeView tv = tree_view(a, 0);
  for (int64_t g = (int64_t)blockIdx.x * kTfBlock + threadIdx.x; g < nw; g += (int64_t)gridDim.x * kTfBlock) {
    const int64_t i0 = 4 * g;
    unsigned h[4];
    route4(a, tv, i0, h);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (i0 + e >= a.n) continue;
      if constexpr (CLS) {
        const int4 p = __ldg(a.prn + h[e]);
        if (!a.out_proba) {
          a.out[i0 + e] = (float)p.y;
        } else {
          const float* pr = a.prob + (int64_t)p.x * a.K;
          for (int k = 0; k < a.K; ++k) a.out[(int64_t)k * a.ld_out + i0 + e] = __ldg(pr + k);
        }
      } else {
        a.out[i0 + e] = a.nodes[h[e]].value;
      }
    }
  }
}

}  // namespace

cudaError_t launch_tree_fit_init(TreeFitNode* nodes, uint2* dec, int T, cudaStream_t st) {
  tree_fit_init_kernel<<<T, 512, 0, st>>>(nodes, dec);
  return cudaGetLastError();
}

cudaError_t launch_tree_fit_hist(const TreeFitArgs& a, int smem_mode, int grid_y, size_t smem, cudaStream_t st) {
  const int gx = smem_mode ? (a.S + a.cb - 1) / a.cb : 1;
  const dim3 grid((unsigned)gx, (unsigned)grid_y, (unsigned)a.T);
  const bool cls = a.K > 0;
  if (smem_mode) {
    auto k = cls ? (a.has_w ? tree_hist_kernel<true, true, true> : tree_hist_kernel<true, false, true>)
                 : (a.has_w ? tree_hist_kernel<true, true, false> : tree_hist_kernel<true, false, false>);
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    k<<<grid, kTfBlock, smem, st>>>(a);
  } else {
    auto k = cls ? (a.has_w ? tree_hist_kernel<false, true, true> : tree_hist_kernel<false, false, true>)
                 : (a.has_w ? tree_hist_kernel<false, true, false> : tree_hist_kernel<false, false, false>);
    k<<<grid, kTfBlock, 0, st>>>(a);
  }
  return cudaGetLastError();
}

cudaError_t launch_tree_fit_split(const TreeFitArgs& a, cudaStream_t st) {
  const dim3 grid(1u << a.L, (unsigned)a.T);
  if (a.K == 0)
    tree_split_kernel<<<grid, kTfBlock, 0, st>>>(a);
  else if (a.entropy)
    tree_split_cls_kernel<true><<<grid, kTfBlock, 0, st>>>(a);
  else
    tree_split_cls_kernel<false><<<grid, kTfBlock, 0, st>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_tree_fit_prune(const TreeFitArgs& a, cudaStream_t st) {
  tree_prune_cls_kernel<<<a.T, 32, 0, st>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_tree_fit_out(const TreeFitArgs& a, int sms, cudaStream_t st) {
  const int64_t nw = (a.n + 3) >> 2;
  int64_t gx = (nw + kTfBlock - 1) / kTfBlock;
  if (gx > (int64_t)sms * 8) gx = (int64_t)sms * 8;
  if (gx < 1) gx = 1;
  if (a.K > 0)
    tree_out_kernel<true><<<(unsigned)gx, kTfBlock, 0, st>>>(a);
  else
    tree_out_kernel<false><<<(unsigned)gx, kTfBlock, 0, st>>>(a);
  return cudaGetLastError();
}

}  // namespace se
