// se_linear_fit.cu — the weighted moment matrix of resident columns (se_linear_moments, DESIGN.md §3 "Device linear fit").
//
// For columns S (p of them) of a [cols][n] slot, z = (x_S − s, 1, y − s_y) and the fp64 (p+2)×(p+2) matrix
// Σ_rows c·w·z zᵀ.  Every term is formed and summed in fp64: c·w is exact (two fp32 factors), z is one fp64 rounding, and
// the CTA partials are folded in a fixed order by the last CTA of each output tile, so a launch configuration gives the
// same bits every time.  Two kernels:
//   * m = p + 2 <= 8: every thread keeps the 36 entries of an 8×8 upper triangle in registers over its rows (the
//     stacking case: bandwidth-bound, one read of the p columns, the label, the weights and the bag);
//   * m > 8: 64×64 output tiles of the upper triangle, one tile per blockIdx.y; a CTA stages 32 rows of the tile's
//     64 + 64 z values in shared memory in fp64 (c·w folded into the row side) and each thread accumulates a 4×4
//     sub-block with FFMA64 (fp64-compute-bound from p of a few dozen on).
#include "se_common.cuh"
#include "se_kernels.h"

namespace se {
namespace {

constexpr int kLmSmall = 8;                              // m <= 8: the register kernel
constexpr int kLmSmallTri = kLmSmall * (kLmSmall + 1) / 2;
constexpr int kLmTile = 64;                              // output tile edge of the tiled kernel
constexpr int kLmRows = 32;                              // rows staged per step
constexpr int kLmTileEntries = kLmTile * kLmTile;

__device__ __forceinline__ double lm_weight(const LinearMomentsArgs& a, int64_t i) {
  double c = 1.0;
  if (a.w) c = (double)a.w[i];
  if (a.bag) c *= (double)a.bag[i];  // the product of two fp32 values is exact in fp64
  return c;
}

__global__ void __launch_bounds__(kBlock) linear_moments_small_kernel(LinearMomentsArgs a) {
  __shared__ int32_t s_col[kLmSmall];
  __shared__ double s_shift[kLmSmall];
  if (threadIdx.x < kLmSmall) {
    s_col[threadIdx.x] = threadIdx.x < a.p ? a.cols[threadIdx.x] : 0;
    s_shift[threadIdx.x] = threadIdx.x < a.p ? a.shift[threadIdx.x] : 0.0;
  }
  __syncthreads();
  double acc[kLmSmallTri];
#pragma unroll
  for (int k = 0; k < kLmSmallTri; ++k) acc[k] = 0.0;
  const int p = a.p;
  for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * kBlock) {
    double z[kLmSmall];
#pragma unroll
    for (int k = 0; k < kLmSmall; ++k) {
      double v = 0.0;
      if (k < p) v = (double)ld_stream1(a.X + (int64_t)s_col[k] * a.ld + i) - s_shift[k];
      else if (k == p) v = 1.0;
      else if (k == p + 1) v = (double)ld_stream1(a.y + i) - a.y_shift;
      z[k] = v;
    }
    const double c = lm_weight(a, i);
    int e = 0;
#pragma unroll
    for (int r = 0; r < kLmSmall; ++r) {
      const double cz = c * z[r];
#pragma unroll
      for (int q = r; q < kLmSmall; ++q, ++e) acc[e] = fma(cz, z[q], acc[e]);
    }
  }
  // block totals -> partials[blockIdx.x]
  __shared__ double sm[kLmSmallTri][kBlock / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < kLmSmallTri; ++k) {
    const double v = warp_sum(acc[k]);
    if (lane == 0) sm[k][warp] = v;
  }
  __syncthreads();
  if (threadIdx.x < kLmSmallTri) {
    double v = 0.0;
    for (int w = 0; w < kBlock / 32; ++w) v += sm[threadIdx.x][w];
    a.partials[(size_t)blockIdx.x * kLmSmallTri + threadIdx.x] = v;
  }
  const int m = p + 2;
  lm_fold_last(a.partials, kLmSmallTri, gridDim.x, a.counters, [&](int e, double s) {
    int r = 0, q = e;  // entry e of the packed upper triangle -> (r, q), q >= r
    while (q >= kLmSmall - r) { q -= kLmSmall - r; ++r; }
    q += r;
    if (r < m && q < m) {
      a.out[(size_t)r * m + q] = s;
      a.out[(size_t)q * m + r] = s;
    }
  });
}

// z entry k of tile side: code >= 0 a column of X, -1 the intercept's 1, -2 the shifted label, -3 padding (0)
__device__ __forceinline__ double lm_z(const LinearMomentsArgs& a, int code, double shift, int64_t i) {
  if (code >= 0) return (double)ld_stream1(a.X + (int64_t)code * a.ld + i) - shift;
  if (code == -1) return 1.0;
  if (code == -2) return (double)ld_stream1(a.y + i) - a.y_shift;
  return 0.0;
}

__global__ void __launch_bounds__(kBlock) linear_moments_tile_kernel(LinearMomentsArgs a, int64_t rows_per_cta) {
  const int m = a.p + 2;
  const int nt = (m + kLmTile - 1) / kLmTile;
  int ti = 0, tj = blockIdx.y;  // upper-triangle tile blockIdx.y -> (ti, tj), tj >= ti
  while (tj >= nt - ti) { tj -= nt - ti; ++ti; }
  tj += ti;
  __shared__ double zi[kLmRows][kLmTile + 1];  // c·w·z of the tile's row side (padded: conflict-free stores)
  __shared__ double zj[kLmRows][kLmTile + 1];
  __shared__ int32_t ci[kLmTile], cj[kLmTile];
  __shared__ double si[kLmTile], sj[kLmTile];
  if (threadIdx.x < 2 * kLmTile) {
    const bool side_j = threadIdx.x >= kLmTile;
    const int t = threadIdx.x & (kLmTile - 1);
    const int k = (side_j ? tj : ti) * kLmTile + t;
    const int code = k < a.p ? a.cols[k] : (k == a.p ? -1 : (k == a.p + 1 ? -2 : -3));
    const double s = k < a.p ? a.shift[k] : 0.0;
    if (side_j) { cj[t] = code; sj[t] = s; } else { ci[t] = code; si[t] = s; }
  }
  __syncthreads();
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;  // entry (ty + 16u, tx + 16v) of the tile
  const int lr = threadIdx.x & (kLmRows - 1), lk = threadIdx.x >> 5;  // loader: row lr, columns lk + 8q
  double acc[4][4];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) acc[u][v] = 0.0;
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_cta;
  const int64_t r1 = min(a.n, r0 + rows_per_cta);
  for (int64_t base = r0; base < r1; base += kLmRows) {
    const int64_t i = base + lr;
    const bool ok = i < r1;
    const double c = ok ? lm_weight(a, i) : 0.0;
#pragma unroll
    for (int q = 0; q < kLmTile / (kBlock / kLmRows); ++q) {
      const int k = lk + (kBlock / kLmRows) * q;
      zi[lr][k] = ok ? c * lm_z(a, ci[k], si[k], i) : 0.0;
      zj[lr][k] = ok ? lm_z(a, cj[k], sj[k], i) : 0.0;
    }
    __syncthreads();
#pragma unroll 4
    for (int r = 0; r < kLmRows; ++r) {
      double x[4], y[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) x[u] = zi[r][ty + 16 * u];
#pragma unroll
      for (int v = 0; v < 4; ++v) y[v] = zj[r][tx + 16 * v];
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) acc[u][v] = fma(x[u], y[v], acc[u][v]);
    }
    __syncthreads();
  }
  double* part = a.partials + (size_t)blockIdx.y * gridDim.x * kLmTileEntries;
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v)
      part[(size_t)blockIdx.x * kLmTileEntries + (ty + 16 * u) * kLmTile + tx + 16 * v] = acc[u][v];
  lm_fold_last(part, kLmTileEntries, gridDim.x, a.counters + blockIdx.y, [&](int e, double s) {
    const int r = ti * kLmTile + e / kLmTile, q = tj * kLmTile + e % kLmTile;
    if (r < m && q < m && q >= r) {
      a.out[(size_t)r * m + q] = s;
      a.out[(size_t)q * m + r] = s;
    }
  });
}

// grid.x of the tiled kernel and its rows per CTA
void lm_tile_grid(int p, int64_t n, int sms, int* grid, int64_t* rows_per_cta) {
  const int nt = (p + 2 + kLmTile - 1) / kLmTile;
  const int tiles = nt * (nt + 1) / 2;
  const int64_t steps = (n + kLmRows - 1) / kLmRows;
  int64_t g = ((int64_t)4 * sms + tiles - 1) / tiles;
  if (g > steps) g = steps;
  if (g < 1) g = 1;
  const int64_t per = (steps + g - 1) / g;
  *rows_per_cta = per * kLmRows;
  *grid = (int)((steps + per - 1) / per);
}

}  // namespace

void linear_moments_scratch(int p, int64_t n, int sms, size_t* partials, int* counters) {
  if (p + 2 <= kLmSmall) {
    *partials = (size_t)grid_rows(n, kBlock, 4, sms) * kLmSmallTri;
    *counters = 1;
    return;
  }
  int g;
  int64_t per;
  lm_tile_grid(p, n, sms, &g, &per);
  const int nt = (p + 2 + kLmTile - 1) / kLmTile;
  *counters = nt * (nt + 1) / 2;
  *partials = (size_t)*counters * (size_t)g * kLmTileEntries;
}

cudaError_t launch_linear_moments(const LinearMomentsArgs& a, int sms, cudaStream_t st) {
  if (a.p < 0 || a.p > kLinearMomentsMaxCols || a.n < 1) return cudaErrorInvalidValue;
  if (a.p + 2 <= kLmSmall) {
    linear_moments_small_kernel<<<grid_rows(a.n, kBlock, 4, sms), kBlock, 0, st>>>(a);
    return cudaGetLastError();
  }
  int g;
  int64_t per;
  lm_tile_grid(a.p, a.n, sms, &g, &per);
  const int nt = (a.p + 2 + kLmTile - 1) / kLmTile;
  linear_moments_tile_kernel<<<dim3((unsigned)g, (unsigned)(nt * (nt + 1) / 2)), kBlock, 0, st>>>(a, per);
  return cudaGetLastError();
}

}  // namespace se
