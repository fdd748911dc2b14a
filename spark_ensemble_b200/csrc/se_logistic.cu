// se_logistic.cu — logistic regression over resident columns (DESIGN.md §3 "Device logistic fit"): the one-off
// statistics pass, the loss and gradient of one optimiser evaluation, and the scoring of a fitted model.
//
// For columns S (p of them) of a [cols][n] slot, z_j = (x_{S[j]} − shift_j)·scale_j and z_p = 1, the margins
// m_k = Σ_j coef[k][j]·z_j of D coefficient sets, and the loss ℓ (binomial: log1pExp(m) − [y=1]·m; multinomial:
// logsumexp(m) − m_y).  Every term is formed and summed in fp64, the CTA partials are folded in a fixed order by the
// last CTA (lm_fold_last), and no kernel indexes memory by a label value: labels are compared with class indices.
// Two loss-gradient kernels:
//   * D = 1 and p + 1 <= 40: every thread keeps z, the margin and the p + 1 gradient sums of its rows in registers
//     (a binomial stacker over up to a few dozen member outputs: bandwidth-bound, one read of the columns, labels and
//     weights), in two widths so that a few columns do not pay the registers of 40;
//   * otherwise a CTA stages 32 rows of z in shared memory in fp64, forms their D margins, turns them into residuals
//     c·(π_k − [y=k]) and accumulates a (4·nk)×(4·nj) tile of the gradient, 4×4 entries per thread, with FFMA64.
#include <algorithm>

#include "se_common.cuh"
#include "se_kernels.h"
#include "se_row_steps.cuh"

namespace se {
namespace {

constexpr int kLsRows = 32;     // rows per step of the statistics pass
constexpr int kLgNarrow = 16;   // D = 1: the register kernel's widths (p + 1 <= 16, p + 1 <= 40)
constexpr int kLgWide = 40;
constexpr int kLgRows = 32;     // rows staged per step of the tiled kernel
constexpr int kLgTileEntries = 16 * kBlock;  // 4×4 gradient entries per thread
constexpr int kLgPart = kLgTileEntries + 1;  // + the loss

// butterfly reductions: every lane gets the same total, in the same order
__device__ __forceinline__ double warp_allsum(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}
__device__ __forceinline__ double warp_allmax(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, off));
  return v;
}

__device__ __forceinline__ double lg_weight(const float* w, int64_t i) { return w ? (double)ld_stream1(w + i) : 1.0; }

// binomial terms of one row: adds c·ℓ to *loss and returns c·(σ(m) − [y=1])
__device__ __forceinline__ double lg_binomial(double m, float y, double c, double* loss) {
  const double yy = (y == 1.f) ? 1.0 : 0.0;
  const double e = exp(-fabs(m));
  *loss = fma(c, fmax(m, 0.0) + log1p(e) - yy * m, *loss);
  const double pi = (m >= 0.0) ? 1.0 / (1.0 + e) : e / (1.0 + e);
  return c * (pi - yy);
}

// rows [r0, r1) of CTA blockIdx.x: `rows` per step, about `target` CTAs
void lg_row_grid(int64_t n, int rows, int64_t target, int* grid, int64_t* rows_per_cta) {
  const int64_t steps = (n + rows - 1) / rows;
  int64_t g = target < steps ? target : steps;
  if (g < 1) g = 1;
  const int64_t per = (steps + g - 1) / g;
  *rows_per_cta = per * rows;
  *grid = (int)((steps + per - 1) / per);
}

// ---- statistics ------------------------------------------------------------------------------------------------------
// Thread j < p owns column j's two sums, thread k < K class k's weight, the last thread Σc, Σc² and the invalid rows.
__global__ void __launch_bounds__(kBlock) logistic_stats_kernel(LogisticArgs a, int64_t rows_per_cta) {
  __shared__ float xs[kLogisticMaxCols][kLsRows + 1];
  __shared__ int32_t s_col[kLogisticMaxCols];
  __shared__ double cs[kLsRows];
  __shared__ float ys[kLsRows];
  __shared__ int bad[kLsRows];
  const int p = a.p, K = a.D, t = threadIdx.x;
  for (int j = t; j < p; j += kBlock) s_col[j] = a.cols[j];
  const double shift = t < p ? a.shift[t] : 0.0;
  double s1 = 0.0, s2 = 0.0, hk = 0.0, sc = 0.0, sc2 = 0.0, nbad = 0.0;
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_cta;
  const int64_t r1 = min(a.n, r0 + rows_per_cta);
  for (int64_t base = r0; base < r1; base += kLsRows) {
    if (t < kLsRows) {
      const int64_t i = base + t;
      double c = 0.0;
      float yv = -1.f;
      bool b = false;
      if (i < r1) {
        const float wv = a.w ? ld_stream1(a.w + i) : 1.f;
        const float y = ld_stream1(a.y + i);
        bool bl = false;
        const int k = checked_label(y, K, bl);
        b = bl || !(isfinite(wv) && wv >= 0.f);
        yv = bl ? -1.f : (float)k;
        c = (double)wv;
      }
      cs[t] = c;
      ys[t] = yv;
      bad[t] = b ? 1 : 0;
    }
    __syncthreads();
    for (int j = t / kLsRows; j < p; j += kBlock / kLsRows) {
      const int r = t % kLsRows;
      const int64_t i = base + r;
      float v = 0.f;
      if (i < r1) {
        v = ld_stream1(a.X + (int64_t)s_col[j] * a.ld + i);
        if (!isfinite(v)) atomicOr(&bad[r], 1);
      }
      xs[j][r] = v;
    }
    __syncthreads();
    if (t < p) {
#pragma unroll 8
      for (int r = 0; r < kLsRows; ++r) {
        const double d = (double)xs[t][r] - shift;
        const double cd = cs[r] * d;
        s1 += cd;
        s2 = fma(cd, d, s2);
      }
    }
    if (t < K) {
      const float k = (float)t;
      for (int r = 0; r < kLsRows; ++r) hk += (ys[r] == k) ? cs[r] : 0.0;
    }
    if (t == kBlock - 1) {
      for (int r = 0; r < kLsRows; ++r) {
        sc += cs[r];
        sc2 = fma(cs[r], cs[r], sc2);
        nbad += (double)bad[r];
      }
    }
    __syncthreads();
  }
  const int len = 3 + 2 * p + K;
  double* part = a.partials + (size_t)blockIdx.x * len;
  if (t < p) {
    part[2 + t] = s1;
    part[2 + p + t] = s2;
  }
  if (t < K) part[2 + 2 * p + t] = hk;
  if (t == kBlock - 1) {
    part[0] = sc;
    part[1] = sc2;
    part[2 + 2 * p + K] = nbad;
  }
  lm_fold_last(a.partials, len, gridDim.x, a.counters, [&](int e, double s) { a.out[e] = s; });
}

// ---- loss and gradient: registers (D = 1, p + 1 <= kLgSmall) ----------------------------------------------------------
// CTA `cta` of `ctas` over the rows of member a.  kSkipZero: rows of weight 0 are skipped before any of their values is
// read (a batch's out-of-bag rows), so that a non-finite feature there contributes nothing.
template <int kLgSmall, bool kSkipZero>
__device__ __forceinline__ void lg_small_body(const LogisticArgs& a, int cta, int ctas) {
  __shared__ int32_t s_col[kLgSmall];
  __shared__ double s_shift[kLgSmall], s_scale[kLgSmall], s_coef[kLgSmall];
  const int p = a.p;
  if (threadIdx.x < kLgSmall) {
    const int j = threadIdx.x;
    s_col[j] = j < p ? a.cols[j] : 0;
    s_shift[j] = j < p ? a.shift[j] : 0.0;
    s_scale[j] = j < p ? a.scale[j] : 0.0;
    s_coef[j] = j <= p ? a.coef[j] : 0.0;
  }
  __syncthreads();
  double acc[kLgSmall];
#pragma unroll
  for (int j = 0; j < kLgSmall; ++j) acc[j] = 0.0;
  double loss = 0.0;
  for (int64_t i = (int64_t)cta * kBlock + threadIdx.x; i < a.n; i += (int64_t)ctas * kBlock) {
    const double c = lg_weight(a.w, i);
    if (kSkipZero && c == 0.0) continue;
    double z[kLgSmall];
    double m = 0.0;
#pragma unroll
    for (int j = 0; j < kLgSmall; ++j) {
      double v = 0.0;
      if (j < p) v = ((double)ld_stream1(a.X + (int64_t)s_col[j] * a.ld + i) - s_shift[j]) * s_scale[j];
      else if (j == p) v = 1.0;
      z[j] = v;
      m = fma(s_coef[j], v, m);
    }
    const double r = lg_binomial(m, ld_stream1(a.y + i), c, &loss);
#pragma unroll
    for (int j = 0; j < kLgSmall; ++j) acc[j] = fma(r, z[j], acc[j]);
  }
  constexpr int kLen = kLgSmall + 1;
  __shared__ double sm[kLen][kBlock / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int e = 0; e < kLen; ++e) {
    const double v = warp_sum(e == 0 ? loss : acc[e - 1]);
    if (lane == 0) sm[e][warp] = v;
  }
  __syncthreads();
  if (threadIdx.x < kLen) {
    double v = 0.0;
    for (int w = 0; w < kBlock / 32; ++w) v += sm[threadIdx.x][w];
    a.partials[(size_t)cta * kLen + threadIdx.x] = v;
  }
  lm_fold_last(a.partials, kLen, ctas, a.counters, [&](int e, double s) {
    if (e <= p + 1) a.out[e] = s;
  });
}
template <int kLgSmall>
__global__ void __launch_bounds__(kBlock) logistic_small_kernel(LogisticArgs a) {
  lg_small_body<kLgSmall, false>(a, blockIdx.x, gridDim.x);
}

// ---- loss and gradient: shared-memory row blocks and a register-tiled gradient ----------------------------------------
// Thread t owns gradient entries (k, j) = (tk + nk·u, j0 + tj + nj·v), u, v < 4, with tk = t / nj, tj = t % nj and
// j0 = blockIdx.y·4·nj.  Margins: L lanes per (row, class) pair split the p + 1 products and add them butterfly-wise.
// CTA `cta` of `ctas` over j-tile `tile` of member a, whose partials start at a.partials + tile·ctas·kLgPart and whose
// ticket is a.counters[tile].  kSkipZero: a row of weight 0 is staged as z = 0 (the intercept's 1 aside), so that its
// terms are exact zeros whatever its features.
template <bool kSkipZero>
__device__ __forceinline__ void lg_tile_body(const LogisticArgs& a, int cta, int ctas, int tile, int64_t rows_per_cta,
                                             int nk, int L, int zs) {
  extern __shared__ double lg_smem[];
  double* Z = lg_smem;                           // [kLgRows][zs]
  double* Rs = Z + kLgRows * zs;                 // [kLgRows][64]: margins, then residuals
  double* cs = Rs + kLgRows * kLogisticMaxClasses;
  float* ys = reinterpret_cast<float*>(cs + kLgRows);
  int32_t* s_col = reinterpret_cast<int32_t*>(ys + kLgRows);
  const int p = a.p, P1 = p + 1, D = a.D, t = threadIdx.x;
  const int lane = t & 31, warp = t >> 5;
  for (int j = t; j < p; j += kBlock) s_col[j] = a.cols[j];
  const int nj = kBlock / nk, tk = t / nj, tj = t % nj;
  const int j0 = tile * 4 * nj;
  int nu = 0;
#pragma unroll
  for (int u = 0; u < 4; ++u) nu += (tk + nk * u < D) ? 1 : 0;
  double acc[4][4];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) acc[u][v] = 0.0;
  double loss = 0.0;
  __syncthreads();
  const int64_t r0 = (int64_t)cta * rows_per_cta;
  const int64_t r1 = min(a.n, r0 + rows_per_cta);
  for (int64_t base = r0; base < r1; base += kLgRows) {
    if (t < kLgRows) {
      const int64_t i = base + t;
      const bool ok = i < r1;
      cs[t] = ok ? lg_weight(a.w, i) : 0.0;
      ys[t] = ok ? ld_stream1(a.y + i) : -1.f;
    }
    for (int j = t / kLgRows; j <= p; j += kBlock / kLgRows) {
      const int r = t % kLgRows;
      const int64_t i = base + r;
      double v = 0.0;
      const bool live = !kSkipZero || j == p || (i < r1 && (!a.w || __ldg(a.w + i) != 0.f));
      if (i < r1 && live)
        v = (j < p) ? ((double)ld_stream1(a.X + (int64_t)s_col[j] * a.ld + i) - a.shift[j]) * a.scale[j] : 1.0;
      Z[r * zs + j] = v;
    }
    __syncthreads();
    // margins: pair pr = (row pr % 32, class pr / 32)
    const int npair = kLgRows * D;
    for (int b0 = 0; b0 < npair; b0 += kBlock / L) {
      const int pr = b0 + t / L, l = t % L;
      const int r = pr % kLgRows, k = pr / kLgRows;
      double s = 0.0;
      if (pr < npair) {
        const double* th = a.coef + (size_t)k * P1;
        const double* zr = Z + r * zs;
        for (int j = l; j < P1; j += L) s = fma(__ldg(th + j), zr[j], s);
      }
      for (int o = L / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (pr < npair && l == 0) Rs[r * kLogisticMaxClasses + k] = s;
    }
    __syncthreads();
    // residuals c·(π_k − [y=k]) in place of the margins, and the loss
    if (D == 1) {
      if (t < kLgRows) Rs[t * kLogisticMaxClasses] = lg_binomial(Rs[t * kLogisticMaxClasses], ys[t], cs[t], &loss);
    } else {
      for (int r = warp; r < kLgRows; r += kBlock / 32) {
        double* mr = Rs + r * kLogisticMaxClasses;
        const bool h0 = lane < D, h1 = lane + 32 < D;
        const double m0 = h0 ? mr[lane] : -INFINITY, m1 = h1 ? mr[lane + 32] : -INFINITY;
        const double mx = warp_allmax(fmax(m0, m1));
        const double e0 = h0 ? exp(m0 - mx) : 0.0, e1 = h1 ? exp(m1 - mx) : 0.0;
        const double S = warp_allsum(e0 + e1);
        const float y = ys[r];
        const bool y0 = h0 && y == (float)lane, y1 = h1 && y == (float)(lane + 32);
        const double my = warp_allsum((y0 ? m0 : 0.0) + (y1 ? m1 : 0.0));
        const double c = cs[r];
        if (lane == 0) loss = fma(c, mx + log(S) - my, loss);
        if (h0) mr[lane] = c * (e0 / S - (y0 ? 1.0 : 0.0));
        if (h1) mr[lane + 32] = c * (e1 / S - (y1 ? 1.0 : 0.0));
      }
    }
    __syncthreads();
#pragma unroll 4
    for (int r = 0; r < kLgRows; ++r) {
      double x[4], y[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) x[u] = Rs[r * kLogisticMaxClasses + tk + nk * u];
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        const int j = j0 + tj + nj * v;
        y[v] = j < P1 ? Z[r * zs + j] : 0.0;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (u < nu) {
#pragma unroll
          for (int v = 0; v < 4; ++v) acc[u][v] = fma(x[u], y[v], acc[u][v]);
        }
    }
    __syncthreads();
  }
  double* part = a.partials + (size_t)tile * ctas * kLgPart + (size_t)cta * kLgPart;
  const int TJ = 4 * nj;
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) part[(tk + nk * u) * TJ + tj + nj * v] = acc[u][v];
  __shared__ double sl[kBlock / 32];
  const double lw = warp_sum(loss);
  if (lane == 0) sl[warp] = lw;
  __syncthreads();
  if (t == 0) {
    double s = 0.0;
    for (int w = 0; w < kBlock / 32; ++w) s += sl[w];
    part[kLgTileEntries] = s;
  }
  lm_fold_last(a.partials + (size_t)tile * ctas * kLgPart, kLgPart, ctas, a.counters + tile,
               [&](int e, double s) {
                 if (e == kLgTileEntries) {
                   if (tile == 0) a.out[0] = s;
                   return;
                 }
                 const int k = e / TJ, j = j0 + e % TJ;
                 if (k < D && j < P1) a.out[1 + (size_t)k * P1 + j] = s;
               });
}
__global__ void __launch_bounds__(kBlock) logistic_tile_kernel(LogisticArgs a, int64_t rows_per_cta, int nk, int L,
                                                               int zs) {
  lg_tile_body<false>(a, blockIdx.x, gridDim.x, blockIdx.y, rows_per_cta, nk, L, zs);
}

// the tiled kernel's shape: nk thread rows (4·nk >= D), L lanes per margin, j-tiles, shared memory
struct LgShape {
  int nk, L, zs, tiles;
  size_t smem;
};
LgShape lg_shape(int p, int D) {
  LgShape s;
  s.nk = 1;
  while (4 * s.nk < D) s.nk *= 2;
  s.L = 1;
  while (s.L < 32 && kLgRows * D * s.L * 2 <= kBlock) s.L *= 2;
  s.zs = (p + 1) | 1;  // odd stride: rows land in different banks
  const int TJ = 4 * (kBlock / s.nk);
  s.tiles = (p + 1 + TJ - 1) / TJ;
  s.smem = sizeof(double) * ((size_t)kLgRows * s.zs + (size_t)kLgRows * kLogisticMaxClasses + kLgRows) +
           sizeof(float) * kLgRows + sizeof(int32_t) * kLogisticMaxCols;
  return s;
}
// the register kernel's width for (p, D), 0 for the tiled kernel
int lg_small(int p, int D) {
  if (D != 1 || p + 1 > kLgWide) return 0;
  return p + 1 <= kLgNarrow ? kLgNarrow : kLgWide;
}

// ---- loss and gradient of a batch of members (se_logistic_loss_grad_batch) ------------------------------------------
// blockIdx.x is the work item, blockIdx.y the CTA of its rows: the members' CTAs over the same rows are adjacent in
// launch order, so they run together and the L2 serves the members' repeated reads of the columns they share.  An item
// runs its member's own kernel body, grid and partials, so a member's bits do not depend on the rest of the batch; CTAs
// beyond an item's own grid return at once.
template <int kLgSmall>
__global__ void __launch_bounds__(kBlock) logistic_small_batch_kernel(const LogisticBatchItem* items) {
  const LogisticBatchItem& it = items[blockIdx.x];
  if ((int)blockIdx.y >= it.ctas) return;
  lg_small_body<kLgSmall, true>(it.a, blockIdx.y, it.ctas);
}
__global__ void __launch_bounds__(kBlock) logistic_tile_batch_kernel(const LogisticBatchItem* items) {
  const LogisticBatchItem& it = items[blockIdx.x];
  if ((int)blockIdx.y >= it.ctas) return;
  lg_tile_body<true>(it.a, blockIdx.y, it.ctas, it.tile, it.rows_per_cta, it.nk, it.L, it.zs);
}

// ---- scoring --------------------------------------------------------------------------------------------------------
// The per-row steps are se_row_steps.cuh's (lg_row_*), which se_linear_agg's kernels share.  The binomial case (D = 1)
// keeps its coefficients in shared memory; the multinomial case reads them through the read-only cache.  MAXD >= D
// keeps the margins in registers.
template <int MAXD>
__global__ void __launch_bounds__(kBlock) logistic_predict_kernel(LogisticPredictArgs a) {
  __shared__ int32_t s_col[kLogisticMaxCols];
  __shared__ double s_coef[kLogisticMaxCols];
  const int p = a.p, D = a.D;
  for (int j = threadIdx.x; j < p; j += kBlock) {
    s_col[j] = a.cols[j];
    s_coef[j] = D == 1 ? a.coef[j] : 0.0;
  }
  __syncthreads();
  for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * kBlock) {
    const auto x = [&](int j) { return (double)ld_stream1(a.X + (int64_t)s_col[j] * a.ld + i); };
    double m[MAXD];
    if (D == 1) lg_row_margins<MAXD>(p, 1, [&](int, int j) { return s_coef[j]; }, x, a.intercept, m);
    else lg_row_margins<MAXD>(p, D, [&](int k, int j) { return __ldg(a.coef + (size_t)k * p + j); }, x, a.intercept, m);
    double mx;
    const int best = lg_row_argmax<MAXD>(D, m, &mx);
    if (a.raw) {
      if (D == 1) {
        a.raw[i] = (float)(-m[0]);
        a.raw[a.ld_raw + i] = (float)m[0];
      } else {
#pragma unroll
        for (int k = 0; k < MAXD; ++k)
          if (k < D) a.raw[(int64_t)k * a.ld_raw + i] = (float)m[k];
      }
    }
    if (a.prob) lg_row_probs<MAXD>(D, m, mx, [&](int k, float v) { a.prob[(int64_t)k * a.ld_prob + i] = v; });
    if (a.label) a.label[i] = lg_row_label(D, m[0], best, a.threshold);
  }
}

}  // namespace

void logistic_stats_scratch(int p, int K, int64_t n, int sms, size_t* partials, int* counters) {
  int g;
  int64_t per;
  lg_row_grid(n, kLsRows, 4 * (int64_t)sms, &g, &per);
  *partials = (size_t)g * (size_t)(3 + 2 * p + K);
  *counters = 1;
}

cudaError_t launch_logistic_stats(const LogisticArgs& a, int sms, cudaStream_t st) {
  if (a.p < 0 || a.p > kLogisticMaxCols || a.D < 1 || a.D > kLogisticMaxClasses || a.n < 1) return cudaErrorInvalidValue;
  int g;
  int64_t per;
  lg_row_grid(a.n, kLsRows, 4 * (int64_t)sms, &g, &per);
  logistic_stats_kernel<<<g, kBlock, 0, st>>>(a, per);
  return cudaGetLastError();
}

void logistic_loss_grad_scratch(int p, int D, int64_t n, int sms, size_t* partials, int* counters) {
  if (const int w = lg_small(p, D)) {
    *partials = (size_t)grid_rows(n, kBlock, 4, sms) * (w + 1);
    *counters = 1;
    return;
  }
  const LgShape s = lg_shape(p, D);
  int g;
  int64_t per;
  lg_row_grid(n, kLgRows, (2 * (int64_t)sms + s.tiles - 1) / s.tiles, &g, &per);
  *partials = (size_t)s.tiles * (size_t)g * kLgPart;
  *counters = s.tiles;
}

cudaError_t launch_logistic_loss_grad(const LogisticArgs& a, int sms, cudaStream_t st) {
  if (a.p < 0 || a.p > kLogisticMaxCols || a.D < 1 || a.D > kLogisticMaxClasses || a.n < 1) return cudaErrorInvalidValue;
  if (const int w = lg_small(a.p, a.D)) {
    if (w == kLgNarrow) logistic_small_kernel<kLgNarrow><<<grid_rows(a.n, kBlock, 4, sms), kBlock, 0, st>>>(a);
    else logistic_small_kernel<kLgWide><<<grid_rows(a.n, kBlock, 4, sms), kBlock, 0, st>>>(a);
    return cudaGetLastError();
  }
  const LgShape s = lg_shape(a.p, a.D);
  int g;
  int64_t per;
  lg_row_grid(a.n, kLgRows, (2 * (int64_t)sms + s.tiles - 1) / s.tiles, &g, &per);
  cudaError_t e = allow_dynamic_smem(logistic_tile_kernel, s.smem);
  if (e != cudaSuccess) return e;
  logistic_tile_kernel<<<dim3((unsigned)g, (unsigned)s.tiles), kBlock, s.smem, st>>>(a, per, s.nk, s.L, s.zs);
  return cudaGetLastError();
}

int logistic_batch_items(const LogisticArgs* members, int B, int sms, LogisticBatchItem* items) {
  int count = 0;
  for (int kind = 0; kind < 3; ++kind)  // grouped by kernel: narrow registers, wide registers, tiled
    for (int b = 0; b < B; ++b) {
      const LogisticArgs& a = members[b];
      const int w = lg_small(a.p, a.D);
      if (kind != (w == kLgNarrow ? 0 : w == kLgWide ? 1 : 2)) continue;
      if (kind < 2) {
        if (items) {
          LogisticBatchItem& it = items[count];
          it = LogisticBatchItem{};
          it.a = a;
          it.kind = kind;
          it.ctas = grid_rows(a.n, kBlock, 4, sms);
        }
        ++count;
        continue;
      }
      const LgShape s = lg_shape(a.p, a.D);
      int g;
      int64_t per;
      lg_row_grid(a.n, kLgRows, (2 * (int64_t)sms + s.tiles - 1) / s.tiles, &g, &per);
      for (int t = 0; t < s.tiles; ++t, ++count) {
        if (!items) continue;
        LogisticBatchItem& it = items[count];
        it = LogisticBatchItem{};
        it.a = a;
        it.kind = kind;
        it.ctas = g;
        it.rows_per_cta = per;
        it.tile = t;
        it.nk = s.nk; it.L = s.L; it.zs = s.zs;
        it.smem = s.smem;
      }
    }
  return count;
}

cudaError_t launch_logistic_loss_grad_batch(const LogisticBatchItem* items, const LogisticBatchItem* d_items,
                                            int count, cudaStream_t st) {
  for (int i0 = 0; i0 < count;) {
    const int kind = items[i0].kind;
    int i1 = i0, ctas = 1;
    size_t smem = 0;
    for (; i1 < count && items[i1].kind == kind; ++i1) {
      const LogisticArgs& a = items[i1].a;
      if (a.p < 0 || a.p > kLogisticMaxCols || a.D < 1 || a.D > kLogisticMaxClasses || a.n < 1) return cudaErrorInvalidValue;
      ctas = max(ctas, items[i1].ctas);
      smem = std::max(smem, items[i1].smem);
    }
    const dim3 grid((unsigned)(i1 - i0), (unsigned)ctas);
    if (kind == 0) {
      logistic_small_batch_kernel<kLgNarrow><<<grid, kBlock, 0, st>>>(d_items + i0);
    } else if (kind == 1) {
      logistic_small_batch_kernel<kLgWide><<<grid, kBlock, 0, st>>>(d_items + i0);
    } else {
      const cudaError_t e = allow_dynamic_smem(logistic_tile_batch_kernel, smem);
      if (e != cudaSuccess) return e;
      logistic_tile_batch_kernel<<<grid, kBlock, smem, st>>>(d_items + i0);
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    i0 = i1;
  }
  return cudaSuccess;
}

cudaError_t launch_logistic_predict(const LogisticPredictArgs& a, int sms, cudaStream_t st) {
  if (a.p < 0 || a.D < 1 || a.D > kLogisticMaxClasses || a.n < 1) return cudaErrorInvalidValue;
  return with_maxd(a.D, [&](auto md) {
    logistic_predict_kernel<decltype(md)::value><<<grid_rows(a.n, kBlock, 4, sms), kBlock, 0, st>>>(a);
    return cudaGetLastError();
  });
}

}  // namespace se
