// se_agg.cu — ensemble Model.predict / predictRaw aggregation kernels (sm_90a).
//
// Reference per-row bodies (one JVM call per row through a UDF, SURVEY.md §3.4):
//   regression/GBMRegressor.scala:531-539        init + Σ_m a_m·P[m]
//   regression/BaggingRegressor.scala:221-228    (Σ_m P[m]) / M
//   classification/GBMClassifier.scala:564-589   res_j = init_j + Σ_m a_mj·P[m][j]; binary dim 1 -> (-res,res)
//   classification/BaggingClassifier.scala:260-287   soft: Σ_m p_m ; hard: Σ_m onehot(ŷ_m) ; prob = raw/M
//   classification/BoostingClassifier.scala:342-382  real: Σ_m (K-1)(ℓ_mk − mean_k ℓ_mk) ; discrete: ±a_m votes;
//                                                    prob = softmax(raw/(K-1))
//
// All of them are one streaming pass over the stacked base-model outputs P (the only large operand:
// 4·M·width B/row) followed by a tiny per-row epilogue.  Stage 1 (sum / vote histogram) is the
// HBM-bound kernel; stage 2 (finalize) touches only C values per row.
#include "se_kernels.h"
#include "se_loss.cuh"
#include "se_tma.cuh"
#include "se_sortnet.h"
#include "se_row_steps.cuh"
#include <type_traits>
#include "../../include/se_abi.h"

namespace se {

namespace {

// out[c][i] = init_c + Σ_m a[m][c] · f(P[m][c][i]),  f = identity
// P row (m,c) lives at P + (cols ? cols[m] : m*width + c) * ld.
// LOGP (SAMME.R): f = lg2 max(·,ε), every term added in fp64 (a batch of fp32 sums of terms of ~-52 would lose 1e-5 of
// the probabilities), and the fp64 total is stored as an fp32 pair: out = hi, out_lo = total - hi.
template <bool LOGP>
__global__ void __launch_bounds__(kBlock) agg_sum_kernel(const float* __restrict__ P, int64_t n,
                                                        int64_t ld, int M, int width,
                                                        const float* __restrict__ a,
                                                        const float* __restrict__ init,
                                                        const int32_t* __restrict__ cols,
                                                        float post_div, float* __restrict__ out,
                                                        int64_t ld_out, float* __restrict__ out_lo = nullptr) {
  const int64_t n4 = n >> 2;
  for (int64_t g = (int64_t)blockIdx.x * kBlock + threadIdx.x; g < n4;
       g += (int64_t)gridDim.x * kBlock) {
    for (int c = 0; c < width; ++c) {
      // every batch of MU models is summed in fp32 (two short chains) and folded into fp64 accumulators: the
      // rounding error stays at the magnitude of one batch instead of growing with M (M = 512 in config 5)
      // (up to two batches there is nothing to gain: plain fp32 carry)
      const bool wide = M > 2 * MU;
      double d0 = 0.0, d1 = 0.0, d2 = 0.0, d3 = 0.0;
      float4 carry = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int m0 = 0; m0 < M; m0 += MU) {
        float4 v[MU];
        float wv[MU];
#pragma unroll
        for (int u = 0; u < MU; ++u) {
          const int m = m0 + u;
          if (m < M) {
            const int64_t rowi = cols ? (int64_t)cols[m] : (int64_t)m * width + c;
            v[u] = ld_stream4(P + rowi * ld + 4 * g);
            wv[u] = a ? a[(int64_t)m * width + c] : 1.0f;
          }
        }
        if constexpr (LOGP) {
#pragma unroll
          for (int u = 0; u < MU; ++u) {
            if (m0 + u < M) {
              d0 += (double)lg2_clamped(v[u].x); d1 += (double)lg2_clamped(v[u].y);
              d2 += (double)lg2_clamped(v[u].z); d3 += (double)lg2_clamped(v[u].w);
            }
          }
          continue;
        }
        float4 s0 = make_float4(0.f, 0.f, 0.f, 0.f), s1 = s0;
#pragma unroll
        for (int u = 0; u < MU; ++u) {
          if (m0 + u < M) {
            const float4 x = v[u];
            float4& s = (u & 1) ? s1 : s0;  // two accumulator sets: shorter dependency chains
            s.x = fmaf(wv[u], x.x, s.x); s.y = fmaf(wv[u], x.y, s.y);
            s.z = fmaf(wv[u], x.z, s.z); s.w = fmaf(wv[u], x.w, s.w);
          }
        }
        agg_fold_batch(wide, s0.x + s1.x, d0, carry.x); agg_fold_batch(wide, s0.y + s1.y, d1, carry.y);
        agg_fold_batch(wide, s0.z + s1.z, d2, carry.z); agg_fold_batch(wide, s0.w + s1.w, d3, carry.w);
      }
      if constexpr (LOGP) {
        const float4 hi = make_float4((float)d0, (float)d1, (float)d2, (float)d3);
        st_stream4(out + c * ld_out + 4 * g, hi);
        st_stream4(out_lo + c * ld_out + 4 * g, make_float4((float)(d0 - (double)hi.x), (float)(d1 - (double)hi.y),
                                                            (float)(d2 - (double)hi.z), (float)(d3 - (double)hi.w)));
        continue;
      }
      const double b = init ? (double)init[c] : 0.0;
      const float4 r = make_float4(agg_fold_end(wide, d0, carry.x, b, post_div), agg_fold_end(wide, d1, carry.y, b, post_div),
                                   agg_fold_end(wide, d2, carry.z, b, post_div), agg_fold_end(wide, d3, carry.w, b, post_div));
      st_stream4(out + c * ld_out + 4 * g, r);
    }
  }
  // tail rows
  const int tail = (int)(n & 3);
  if (blockIdx.x == 0 && threadIdx.x < tail) {
    const int64_t i = (n4 << 2) + threadIdx.x;
    for (int c = 0; c < width; ++c) {
      double sd = init ? (double)init[c] : 0.0;
      for (int m = 0; m < M; ++m) {
        const int64_t rowi = cols ? (int64_t)cols[m] : (int64_t)m * width + c;
        const float x = P[rowi * ld + i];
        if (LOGP) sd += (double)lg2_clamped(x);
        else agg_tail_add(sd, a ? a[(int64_t)m * width + c] : 1.0f, x);
      }
      if (LOGP) {
        out[c * ld_out + i] = (float)sd;
        out_lo[c * ld_out + i] = (float)(sd - (double)(float)sd);
        continue;
      }
      if (post_div != 0.f) sd /= (double)post_div;
      out[c * ld_out + i] = (float)sd;
    }
  }
}

// Vote histogram: A_c = Σ_{m: vote_m == c} a_m (a_m = 1 when a == nullptr).  One row per thread, per-thread
// histogram in shared memory laid out [K][kBlock] (conflict-free); the epilogue (raw, probability, argmax)
// runs straight out of shared memory — no intermediate [K][n] round trip through HBM.
// ncu / SASS on the first form of this kernel (weighted votes, M = 64, K = 26): 3860 instructions per row — per vote a
// 64-bit multiply for the address, a bounds predicate, a branch around the update and a global load + conversion of the
// model weight; per class an fp64 DIVISION in the epilogue.  This form walks the vote column with a pointer increment,
// stages the weights in shared memory in the histogram's type, updates branch-free (an invalid vote lands in a spare
// bin K and raises the error flag) and multiplies by 1/(K-1).
template <typename HT>  // float: unweighted counts (exact); double: weighted votes (error independent of M)
__global__ void __launch_bounds__(kBlock) agg_votes_kernel(const float* __restrict__ votes, int64_t ld, int M,
                                                          const float* __restrict__ a, const FinArgs f) {
  extern __shared__ __align__(8) unsigned char hist_raw[];
  HT* hist = reinterpret_cast<HT*>(hist_raw);  // [K + 1][kBlock]: bin K swallows invalid votes
  const int K = f.K;
  HT* s_a = hist + (size_t)(K + 1) * kBlock;    // [M] model weights (1 for plain votes)
  for (int m = threadIdx.x; m < M; m += kBlock) s_a[m] = a ? (HT)a[m] : (HT)1;
  __syncthreads();
  bool bad_vote = false;
  for (int64_t i0 = (int64_t)blockIdx.x * kBlock; i0 < f.n; i0 += (int64_t)gridDim.x * kBlock) {
    const int64_t i = i0 + threadIdx.x;
    HT* col = hist + threadIdx.x;
    for (int c = 0; c <= K; ++c) col[c * kBlock] = (HT)0;
    if (i < f.n) {
      const float* p = votes + i;
      int m0 = 0;
      for (; m0 + MU <= M; m0 += MU) {  // full batches: MU independent loads in flight, no per-vote predicates
        float v[MU];
#pragma unroll
        for (int u = 0; u < MU; ++u) v[u] = ld_stream1(p + (int64_t)u * ld);
        p += (int64_t)MU * ld;
#pragma unroll
        for (int u = 0; u < MU; ++u) {
          const int c = __float2int_rz(v[u]);
          const bool ok = ((unsigned)c < (unsigned)K) && ((float)c == v[u]);  // a vote is a predicted class index
          bad_vote = bad_vote || !ok;
          col[(ok ? c : K) * kBlock] += s_a[m0 + u];
        }
      }
      for (; m0 < M; ++m0, p += ld) {
        const float x = ld_stream1(p);
        const int c = __float2int_rz(x);
        const bool ok = ((unsigned)c < (unsigned)K) && ((float)c == x);
        bad_vote = bad_vote || !ok;
        col[(ok ? c : K) * kBlock] += s_a[m0];
      }
      // epilogue out of the thread's own histogram column, which doubles as fp32 scratch (ncu on the generic
      // two-sweep finalize_row: ~55 instructions per class; this form: 8 for plain votes, ~25 with the soft-max)
      float best = -INFINITY;
      int am = 0;
      if (f.kind == SE_AGG_BAGGING_HARD) {
        const float inv = 1.0f / (float)f.M;  // prob = raw·(1/M)  (BaggingClassifier.scala:285-287)
        for (int c = 0; c < K; ++c) {
          const float r = (float)col[c * kBlock];
          if (r > best) best = r, am = c;  // Vector.argmax: first maximum
          f.raw[c * f.ld + i] = r;
          f.prob[c * f.ld + i] = r * inv;
        }
      } else {
        const float sc = kLog2e / (float)(f.K - 1);  // prob = softmax(raw/(K-1))  (BoostingClassifier.scala:342-346)
        for (int c = 0; c < K; ++c) {
          const float r = fin_raw(f, col[c * kBlock], 0.f);
          if (r > best) best = r, am = c;
          f.raw[c * f.ld + i] = r;
          *reinterpret_cast<float*>(col + c * kBlock) = r;
        }
        float ssum = 0.f;
        for (int c = 0; c < K; ++c) {
          float* sp = reinterpret_cast<float*>(col + c * kBlock);
          const float e = ex2_approx((*sp - best) * sc);
          ssum += e;
          *sp = e;
        }
        const float inv = rcp_approx(ssum);
        for (int c = 0; c < K; ++c) f.prob[c * f.ld + i] = *reinterpret_cast<const float*>(col + c * kBlock) * inv;
      }
      f.label[i] = (float)am;
    }
  }
  if (bad_vote && f.bad_label != nullptr) *reinterpret_cast<volatile int*>(f.bad_label) = 1;
}

// Vote histogram for class counts whose shared-memory histogram does not fit (K + 1 bins x kBlock threads: K >= 99
// weighted, K >= 199 plain).  Each row's histogram lives in its own RAW and PROB columns: RAW holds the fp32 sum of
// the row's vote weights per class and PROB the rounding error of that sum (a two-sum per vote), so the weighted total
// is good to ~2^-48 like the fp64 histogram; plain counts are exact integers in RAW.  The votes of a warp scatter over
// K classes, so this is the slow path, kept for correctness at any K.
__global__ void __launch_bounds__(kBlock) agg_votes_global_kernel(const float* __restrict__ votes, int64_t ld, int M,
                                                                 const float* __restrict__ a, const FinArgs f) {
  const int K = f.K;
  bool bad_vote = false;
  for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < f.n; i += (int64_t)gridDim.x * kBlock) {
    float* hi = f.raw + i;
    float* lo = f.prob + i;
    for (int c = 0; c < K; ++c) hi[c * f.ld] = 0.f, lo[c * f.ld] = 0.f;
    for (int m = 0; m < M; ++m) {
      const float x = ld_stream1(votes + (int64_t)m * ld + i);
      const int c = __float2int_rz(x);
      const bool ok = ((unsigned)c < (unsigned)K) && ((float)c == x);  // a vote is a predicted class index
      bad_vote = bad_vote || !ok;
      if (!ok) continue;
      const float w = a ? __ldg(a + m) : 1.0f;
      const float s = hi[c * f.ld], t = s + w, bp = t - s;
      hi[c * f.ld] = t;
      lo[c * f.ld] += (s - (t - bp)) + (w - bp);
    }
    float best = -INFINITY;
    int am = 0;
    if (f.kind == SE_AGG_BAGGING_HARD) {
      const float inv = 1.0f / (float)f.M;  // prob = raw·(1/M)  (BaggingClassifier.scala:285-287)
      for (int c = 0; c < K; ++c) {
        const float r = hi[c * f.ld];
        if (r > best) best = r, am = c;  // Vector.argmax: first maximum
        lo[c * f.ld] = r * inv;
      }
    } else {
      const float sc = kLog2e / (float)(f.K - 1);  // prob = softmax(raw/(K-1))  (BoostingClassifier.scala:342-346)
      for (int c = 0; c < K; ++c) {
        const float r = fin_raw(f, (double)hi[c * f.ld] + (double)lo[c * f.ld], 0.f);
        if (r > best) best = r, am = c;
        hi[c * f.ld] = r;
      }
      double ssum = 0.0;  // up to thousands of terms of similar size: an fp32 sum drifts by 1e-5
      for (int c = 0; c < K; ++c) {
        const float e = ex2_approx((hi[c * f.ld] - best) * sc);
        ssum += (double)e;
        lo[c * f.ld] = e;
      }
      const float inv = (float)(1.0 / ssum);
      for (int c = 0; c < K; ++c) lo[c * f.ld] *= inv;
    }
    f.label[i] = (float)am;
  }
  if (bad_vote && f.bad_label != nullptr) *reinterpret_cast<volatile int*>(f.bad_label) = 1;
}

// Unweighted (hard) votes, the packed form: ncu on the histogram kernel above (M = 64, K = 26, 10 M rows): 2660
// instructions per row — 41 per vote — at 60 % issue utilisation and about half of the DRAM peak: issue-bound, not
// memory-bound.  Here a thread owns FOUR consecutive rows (one 128-bit load per model), counts are 8-bit fields packed
// four to a 32-bit word (class c -> word c >> 2, byte c & 3: M <= 255 never overflows a field), the words live in the
// thread's own shared-memory column (conflict-free, 4x less shared memory than one float per class), and the four
// rows give four independent read-modify-write chains.  Exact: integer counts.
constexpr int kVR = 4;  // rows per thread
__global__ void __launch_bounds__(kBlock) agg_hard_votes_packed_kernel(const float* __restrict__ votes, int64_t ld, int M,
                                                                      const FinArgs f) {
  extern __shared__ __align__(8) unsigned char hist_raw[];
  uint32_t* hist = reinterpret_cast<uint32_t*>(hist_raw);  // [W][kVR][kBlock]
  const int K = f.K;
  const int W = (K + 3) >> 2;
  bool bad_vote = false;
  const int64_t ngroups = (f.n + kVR - 1) / kVR;
  const float inv = 1.0f / (float)f.M;  // prob = raw·(1/M)  (BaggingClassifier.scala:285-287)
  for (int64_t g0 = (int64_t)blockIdx.x * kBlock; g0 < ngroups; g0 += (int64_t)gridDim.x * kBlock) {
    const int64_t g = g0 + threadIdx.x;
    for (int w = 0; w < W * kVR; ++w) hist[w * kBlock + threadIdx.x] = 0u;
    if (g >= ngroups) continue;
    const int64_t i0 = g * kVR;
    const bool full = (i0 + kVR <= f.n);  // rows are padded to 32 floats: the 128-bit load itself is always in bounds
    for (int m0 = 0; m0 < M; m0 += MU) {
      float4 v[MU];
#pragma unroll
      for (int u = 0; u < MU; ++u)
        if (m0 + u < M) v[u] = ld_stream4(votes + (int64_t)(m0 + u) * ld + i0);
#pragma unroll
      for (int u = 0; u < MU; ++u) {
        if (m0 + u >= M) break;
#pragma unroll
        for (int e = 0; e < kVR; ++e) {
          const float x = f4at(v[u], e);
          const int c = __float2int_rz(x);
          const bool ok = ((unsigned)c < (unsigned)K) && ((float)c == x);
          bad_vote = bad_vote || (!ok && (full || i0 + e < f.n));
          if (ok) hist[((c >> 2) * kVR + e) * kBlock + threadIdx.x] += 1u << ((c & 3) << 3);
        }
      }
    }
    // epilogue: one 128-bit store per class and output array for the thread's four rows
    int best[kVR] = {-1, -1, -1, -1}, am[kVR] = {0, 0, 0, 0};
    for (int c = 0; c < K; ++c) {
      float4 r;
#pragma unroll
      for (int e = 0; e < kVR; ++e) {
        const int cnt = (int)((hist[((c >> 2) * kVR + e) * kBlock + threadIdx.x] >> ((c & 3) << 3)) & 0xFFu);
        if (cnt > best[e]) best[e] = cnt, am[e] = c;  // Vector.argmax: first maximum
        f4at(r, e) = (float)cnt;
      }
      if (full) {
        st_stream4(f.raw + c * f.ld + i0, r);
        st_stream4(f.prob + c * f.ld + i0, make_float4(r.x * inv, r.y * inv, r.z * inv, r.w * inv));
      } else {
#pragma unroll
        for (int e = 0; e < kVR; ++e)
          if (i0 + e < f.n) {
            f.raw[c * f.ld + i0 + e] = f4at(r, e);
            f.prob[c * f.ld + i0 + e] = f4at(r, e) * inv;
          }
      }
    }
    if (full) {
      st_stream4(f.label + i0, make_float4((float)am[0], (float)am[1], (float)am[2], (float)am[3]));
    } else {
#pragma unroll
      for (int e = 0; e < kVR; ++e)
        if (i0 + e < f.n) f.label[i0 + e] = (float)am[e];
    }
  }
  if (bad_vote && f.bad_label != nullptr) *reinterpret_cast<volatile int*>(f.bad_label) = 1;
}

// (A four-rows-per-thread fp64 form of the WEIGHTED vote histogram was tried too: [K][4][128] doubles leave two
// 128-thread CTAs per SM and it was slower than agg_votes_kernel<double> — the
// fp64 read-modify-write chains need the resident warps more than they need wider loads.  Not kept.)

// ------------------------------------------------------------------ class-wide sums through TMA tiles
// For the classifiers every row needs all C class sums before its epilogue (argmax, soft-max).  The streaming path
// (agg_sum_kernel + agg_finalize_kernel) round-trips a [C][n] intermediate through HBM and, per ncu, is
// instruction-bound: 15.8 instructions per element in stage 1 and 55 per (row, class) in the epilogue.  Here a one-warp
// CTA owns 128 rows; the stacked model outputs arrive as 2-D tensor-map TMA boxes of G models x C classes x 128 rows;
// a thread owns four rows and keeps the C x 4 sums of the current batch of <= 8 models in REGISTERS (one 128-bit
// shared-memory read and 4 FMAs — plus 4 lg2 for SAMME.R — per class and model); each batch is folded into the
// tile's running totals [C][128] in shared memory (own columns only), and the epilogue runs out of shared memory
// with 128-bit stores: P is read once, nothing is re-read.  Latency is covered by the other resident CTAs (up to 8
// per SM), not by per-CTA double buffering.
constexpr int kClassTileRows = 128;  // one warp per CTA, four rows per thread

struct ClassTileArgs {
  int M, C;          // models, classes
  int G;             // models per TMA box
  int logp;          // f = log max(p, eps) (boosting real)
  const float* a;    // weights [M][C] (GBM classifier) or null
  const float* init; // [C] or null
};

// epilogue of four rows whose C stage-1 sums sit in T[c * kAR + j] (this thread's own columns)
template <int kAR>
__device__ __forceinline__ void finalize_tile4(const FinArgs& f, float* T, int64_t row0) {
  const int C = f.C;
  const bool all_in = row0 + 3 < f.n;
  auto store4 = [&](float* base, const float4& v) {
    if (all_in) {
      st_stream4(base + row0, v);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (row0 + j < f.n) base[row0 + j] = f4at(v, j);
    }
  };
  const float4 mean = make_float4(0.f, 0.f, 0.f, 0.f);
  const bool softmax = (f.kind == SE_AGG_GBM_CLASSIFIER);
  const float sc = kLog2e;
  // pass 1: raw (kept in the tile, written to HBM), max and first argmax
  float4 best = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  float4 am = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int c = 0; c < C; ++c) {
    const float4 t = *reinterpret_cast<const float4*>(T + c * kAR);
    float4 r;
    r.x = fin_raw(f, t.x, mean.x), r.y = fin_raw(f, t.y, mean.y), r.z = fin_raw(f, t.z, mean.z), r.w = fin_raw(f, t.w, mean.w);
    const float cf = (float)c;  // Vector.argmax: first maximum
    if (r.x > best.x) best.x = r.x, am.x = cf;
    if (r.y > best.y) best.y = r.y, am.y = cf;
    if (r.z > best.z) best.z = r.z, am.z = cf;
    if (r.w > best.w) best.w = r.w, am.w = cf;
    *reinterpret_cast<float4*>(T + c * kAR) = r;
    store4(f.raw + c * f.ld, r);
  }
  store4(f.label, am);
  if (softmax) {
    float4 ssum = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int c = 0; c < C; ++c) {
      const float4 r = *reinterpret_cast<const float4*>(T + c * kAR);
      float4 e;
      e.x = ex2_approx((r.x - best.x) * sc), e.y = ex2_approx((r.y - best.y) * sc);
      e.z = ex2_approx((r.z - best.z) * sc), e.w = ex2_approx((r.w - best.w) * sc);
      ssum.x += e.x, ssum.y += e.y, ssum.z += e.z, ssum.w += e.w;
      *reinterpret_cast<float4*>(T + c * kAR) = e;
    }
    const float4 inv = make_float4(rcp_approx(ssum.x), rcp_approx(ssum.y), rcp_approx(ssum.z), rcp_approx(ssum.w));
    for (int c = 0; c < C; ++c) {
      const float4 e = *reinterpret_cast<const float4*>(T + c * kAR);
      store4(f.prob + c * f.ld, make_float4(e.x * inv.x, e.y * inv.y, e.z * inv.z, e.w * inv.w));
    }
  } else {
    const float inv = 1.0f / (float)f.M;  // bagging: prob = raw·(1/M) (BaggingClassifier.scala:285-287)
    for (int c = 0; c < C; ++c) {
      const float4 r = *reinterpret_cast<const float4*>(T + c * kAR);
      store4(f.prob + c * f.ld, make_float4(r.x * inv, r.y * inv, r.z * inv, r.w * inv));
    }
  }
}

// dynamic shared memory (128-byte aligned): [G*C][kAR] floats (one box), then the running totals [C][kAR] (fp32, or
// fp64 for LOGP)
// LOGP (SAMME.R): every model's lg2 max(p, eps) is added straight into fp64 totals in shared memory: late in boosting
// most terms are -52 (exact for pure leaves), and fp32 batch sums of them lose 1e-5 of the probabilities from M ~ 8.
template <int CMAX, bool LOGP>
__global__ void __launch_bounds__(32) agg_class_tile_kernel(const ClassTileArgs ta, const FinArgs f,
                                                         const __grid_constant__ CUtensorMap mapP) {
  constexpr int kAR = kClassTileRows;
  extern __shared__ __align__(128) unsigned char smem_dyn[];
  float* stage = reinterpret_cast<float*>(smem_dyn + ((128u - (smem_u32(smem_dyn) & 127u)) & 127u));
  __shared__ __align__(8) uint64_t full;
  const int C = ta.C, M = ta.M;
  const int box_rows = ta.G * C;
  const int stage_floats = box_rows * kAR;
  const int tid = threadIdx.x;
  float* total = stage + stage_floats + 4 * tid;  // this thread's four columns
  double* total_lg = reinterpret_cast<double*>(stage + stage_floats) + 4 * tid;  // LOGP
  if (tid == 0) {
    mbar_init(&full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int64_t ntiles = (f.n + kAR - 1) / kAR;
  const int64_t my_tiles = (ntiles > blockIdx.x) ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  const int steps = (M + ta.G - 1) / ta.G;            // boxes per tile
  const int64_t nbox = my_tiles * steps;              // boxes this CTA consumes, in order
  auto issue = [&](int64_t q) {                       // one elected thread
    const int64_t tile = blockIdx.x + (q / steps) * gridDim.x;
    const int step = (int)(q % steps);
    mbar_expect_tx(&full, (uint32_t)(stage_floats * sizeof(float)));
    tma_load_tile_at(stage, &mapP, (int)(tile * kAR), step * box_rows, &full);
  };
  if (tid == 0 && nbox > 0) issue(0);

  uint32_t phase = 0;
  int64_t q = 0;
  for (int64_t ti = 0; ti < my_tiles; ++ti) {
    const int64_t row0 = (blockIdx.x + ti * gridDim.x) * kAR + 4 * tid;
    float4 acc[CMAX];
#pragma unroll
    for (int c = 0; c < CMAX; ++c) acc[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    int in_batch = 0;
    bool first_fold = true;
    if constexpr (LOGP) {
      for (int c = 0; c < C; ++c) {
        double2* t = reinterpret_cast<double2*>(total_lg + c * kAR);
        t[0] = make_double2(0.0, 0.0), t[1] = make_double2(0.0, 0.0);
      }
    }
    for (int step = 0; step < steps; ++step, ++q) {
      mbar_wait(&full, phase);
      const float* box = stage + 4 * tid;
      const int m0 = step * ta.G;
      const int gcount = min(ta.G, M - m0);
      for (int g = 0; g < gcount; ++g) {
        const float* bg = box + g * C * kAR;
        if constexpr (LOGP) {
          for (int c = 0; c < C; ++c) {
            const float4 x = *reinterpret_cast<const float4*>(bg + c * kAR);
            double2* t = reinterpret_cast<double2*>(total_lg + c * kAR);
            double2 t0 = t[0], t1 = t[1];
            t0.x += (double)lg2_clamped(x.x), t0.y += (double)lg2_clamped(x.y);
            t1.x += (double)lg2_clamped(x.z), t1.y += (double)lg2_clamped(x.w);
            t[0] = t0, t[1] = t1;
          }
          continue;
        }
        const float* wg = ta.a ? ta.a + (int64_t)(m0 + g) * C : nullptr;
#pragma unroll
        for (int c = 0; c < CMAX; ++c) {
          if (c < C) {
            const float4 x = *reinterpret_cast<const float4*>(bg + c * kAR);
            const float wv = wg ? __ldg(wg + c) : 1.0f;
            acc[c].x = fmaf(wv, x.x, acc[c].x), acc[c].y = fmaf(wv, x.y, acc[c].y);
            acc[c].z = fmaf(wv, x.z, acc[c].z), acc[c].w = fmaf(wv, x.w, acc[c].w);
          }
        }
      }
      __syncthreads();  // every thread is done with the box: the stage can be refilled
      if (tid == 0 && q + 1 < nbox) issue(q + 1);
      phase ^= 1;
      in_batch += gcount;
      if (!LOGP && (in_batch >= 8 || step == steps - 1)) {
        // fold the batch into the running totals: the rounding error stays at the magnitude of one batch
#pragma unroll
        for (int c = 0; c < CMAX; ++c) {
          if (c < C) {
            float4 t;
            if (first_fold) {
              const float b = ta.init ? __ldg(ta.init + c) : 0.f;
              t = make_float4(b, b, b, b);
            } else {
              t = *reinterpret_cast<const float4*>(total + c * kAR);
            }
            t.x += acc[c].x, t.y += acc[c].y, t.z += acc[c].z, t.w += acc[c].w;
            *reinterpret_cast<float4*>(total + c * kAR) = t;
            acc[c] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
        first_fold = false;
        in_batch = 0;
      }
    }
    if (row0 < f.n) {
      if constexpr (LOGP) {
        for (int j = 0; j < 4; ++j)
          if (row0 + j < f.n) finalize_real_row(f, row0 + j, [&](int c) { return total_lg[c * kAR + j]; });
      } else {
        finalize_tile4<kAR>(f, total, row0);
      }
    }
  }
}

// Stage 2 for the sum-based kinds: per-row epilogue on tmp[C][n] (in RAW) -> raw, prob, label.
__global__ void __launch_bounds__(kBlock) agg_finalize_kernel(const FinArgs f) {
  for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < f.n;
       i += (int64_t)gridDim.x * kBlock) {
    if (f.kind == SE_AGG_GBM_CLASSIFIER && f.dim == 1 && f.K == 2) {
      finalize_binary_row(f, i, f.raw[i]);
      continue;
    }
    if (f.kind == SE_AGG_BOOSTING_REAL)
      finalize_real_row(f, i, [&](int c) { return (double)f.raw[c * f.ld + i] + (double)f.prob[c * f.ld + i]; });
    else
      finalize_row(f, i, [&](int c) { return f.raw[c * f.ld + i]; });
  }
}

// Weighted median over M model outputs per row (ensemble/Utils.scala:26-40 via
// regression/BoostingRegressor.scala:333-337): stable sort of (value, weight) by value, cumulative weights in sorted
// order, first element whose cumulative weight reaches half of the total.
// One thread per row.  The row's M values become 64-bit words (order-preserving key << 32 | model index: all words
// distinct, ties keep model order = stable sort) in the thread's own column of shared memory [Mp][T] (conflict-free),
// padded to a power of two Mp with +inf words, and are sorted by a bitonic network — uniform control flow for the
// whole warp, O(M log² M) compare-exchanges instead of the O(M²) threshold scan it replaces (far from the HBM
// roofline because per-lane pruning diverges).  Total and running sums are then accumulated in fp64 in
// sorted order, exactly like the reference.
template <int T>
__global__ void __launch_bounds__(T) agg_wmedian_kernel(const float* __restrict__ P, int64_t n, int64_t ld, int M,
                                                       int Mp, const double* __restrict__ a,
                                                       float* __restrict__ out) {
  extern __shared__ __align__(128) unsigned char wm_raw[];
  double* s_a = reinterpret_cast<double*>(wm_raw);                        // [M]
  unsigned long long* col = reinterpret_cast<unsigned long long*>(s_a + M) + threadIdx.x;  // [Mp][T], own column
  for (int m = threadIdx.x; m < M; m += T) s_a[m] = a[m];
  __syncthreads();
  for (int64_t r0 = (int64_t)blockIdx.x * T; r0 < n; r0 += (int64_t)gridDim.x * T) {
    const int64_t row = r0 + threadIdx.x;
    const bool in = row < n;
    for (int m = 0; m < Mp; ++m) {
      unsigned long long w = ~0ull;  // padding sorts last
      if (m < M) {
        const float v = in ? ld_stream1(P + (int64_t)m * ld + row) : 0.f;
        w = ((unsigned long long)wm_key(v) << 32) | (unsigned long long)(unsigned)m;
      }
      col[(size_t)m * T] = w;
    }
    // bitonic sort, ascending (own column only: no synchronisation)
    for (int k = 2; k <= Mp; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int e = 0; e < Mp; ++e) {
          const int l = e ^ j;
          if (l > e) {
            const unsigned long long x = col[(size_t)e * T], y = col[(size_t)l * T];
            const bool up = ((e & k) == 0);
            if ((x > y) == up) {
              col[(size_t)e * T] = y;
              col[(size_t)l * T] = x;
            }
          }
        }
      }
    }
    double total = 0.0;
    for (int m = 0; m < M; ++m) total += s_a[(unsigned)col[(size_t)m * T]];
    const double half = 0.5 * total;
    double cum = 0.0;
    unsigned long long pick = col[(size_t)(M - 1) * T];
    for (int m = 0; m < M; ++m) {
      const unsigned long long w = col[(size_t)m * T];
      cum += s_a[(unsigned)w];
      if (cum >= half) {
        pick = w;
        break;
      }
    }
    if (in) out[row] = wm_unkey((uint32_t)(pick >> 32));
  }
}

// Any number of models (M <= 8192): ONE WARP per row.  The row's words live in the warp's slice of shared memory and
// are sorted by a warp-cooperative bitonic network (lane e handles the pairs (e, e^j), e^j > e, 32 at a time); lane 0
// then accumulates the weights in sorted order, sequentially in fp64 — the reference's order (ensemble/Utils.scala:
// 26-40), so the selected element is identical.  The reference has no bound on M (JVM arrays); this is the general
// path behind the register (M <= 64) and thread-per-row (M <= 256) kernels.
constexpr int kWmWarps = 2;
__global__ void __launch_bounds__(32 * kWmWarps) agg_wmedian_warp_kernel(const float* __restrict__ P, int64_t n, int64_t ld,
                                                                         int M, int Mp, const double* __restrict__ a,
                                                                         float* __restrict__ out) {
  extern __shared__ __align__(128) unsigned char wm_raw[];
  double* s_a = reinterpret_cast<double*>(wm_raw);  // [M]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long* words = reinterpret_cast<unsigned long long*>(s_a + M) + (size_t)warp * Mp;  // [Mp], this warp's
  for (int m = threadIdx.x; m < M; m += 32 * kWmWarps) s_a[m] = a[m];
  __syncthreads();
  for (int64_t row = (int64_t)blockIdx.x * kWmWarps + warp; row < n; row += (int64_t)gridDim.x * kWmWarps) {
    for (int m = lane; m < Mp; m += 32) {
      unsigned long long w = ~0ull;  // padding sorts last
      if (m < M) w = ((unsigned long long)wm_key(ld_stream1(P + (int64_t)m * ld + row)) << 32) | (unsigned long long)(unsigned)m;
      words[m] = w;
    }
    __syncwarp();
    for (int k = 2; k <= Mp; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int e = lane; e < Mp; e += 32) {
          const int l = e ^ j;
          if (l > e) {
            const unsigned long long x = words[e], y = words[l];
            const bool up = ((e & k) == 0);
            if ((x > y) == up) {
              words[e] = y;
              words[l] = x;
            }
          }
        }
        __syncwarp();
      }
    }
    if (lane == 0) {
      double total = 0.0;
      for (int m = 0; m < M; ++m) total += s_a[(unsigned)words[m]];
      const double half = 0.5 * total;
      double cum = 0.0;
      unsigned long long pick = words[M - 1];
      for (int m = 0; m < M; ++m) {
        const unsigned long long w = words[m];
        cum += s_a[(unsigned)w];
        if (cum >= half) {
          pick = w;
          break;
        }
      }
      out[row] = wm_unkey((uint32_t)(pick >> 32));
    }
    __syncwarp();
  }
}

// Same algorithm with the row's words in REGISTERS (Mp <= 64): the network is fully unrolled, so every
// compare-exchange is ~6 ALU instructions and no memory traffic — the shared-memory form above moves 32 B per
// compare-exchange and thread and is bound by shared-memory bandwidth.
template <int MP>
__global__ void __launch_bounds__(128) agg_wmedian_reg_kernel(const __grid_constant__ CUtensorMap mapP, int64_t n,
                                                              int M, const double* __restrict__ a,
                                                              float* __restrict__ out) {
  // the sort is ALU work with no loads in flight, so the next tile of [M][128] values is prefetched into the other
  // shared-memory stage by one 2-D TMA box while the current tile is sorted (ncu on the direct-load form: 20 % issue
  // utilisation, long-scoreboard bound)
  extern __shared__ __align__(128) unsigned char wm_raw[];
  float* stage0 = reinterpret_cast<float*>(wm_raw + ((128u - (smem_u32(wm_raw) & 127u)) & 127u));
  const int stage_floats = M * 128;
  double* s_a = reinterpret_cast<double*>(stage0 + 2 * stage_floats);  // [M]
  __shared__ __align__(8) uint64_t full[2];
  if (threadIdx.x == 0) {
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int m = threadIdx.x; m < M; m += 128) s_a[m] = a[m];
  __syncthreads();
  const int64_t ntiles = (n + 127) / 128;
  auto issue = [&](int64_t tile, int st) {
    mbar_expect_tx(&full[st], (uint32_t)(stage_floats * sizeof(float)));
    tma_load_tile(stage0 + (size_t)st * stage_floats, &mapP, (int)(tile * 128), &full[st]);
  };
  if (threadIdx.x == 0 && blockIdx.x < ntiles) issue(blockIdx.x, 0);
  uint32_t it = 0;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
    const int st = it & 1;
    if (threadIdx.x == 0 && tile + gridDim.x < ntiles) issue(tile + gridDim.x, st ^ 1);  // freed by the barrier below
    const int64_t row = tile * 128 + threadIdx.x;
    const bool in = row < n;
    mbar_wait(&full[st], (it >> 1) & 1);
    const float* src = stage0 + (size_t)st * stage_floats + threadIdx.x;
    unsigned long long w[MP];
#pragma unroll
    for (int m = 0; m < MP; ++m) {
      w[m] = ~0ull;  // padding sorts last
      if (m < M) w[m] = ((unsigned long long)wm_key(src[m * 128]) << 32) | (unsigned long long)(unsigned)m;
    }
    __syncthreads();  // the tile is in registers: its stage may be refilled
    const unsigned long long pick = wm_exact_pick<MP>(w, M, s_a);
    if (in) out[row] = wm_unkey((uint32_t)(pick >> 32));
  }
}

template <int MP>
__global__ void __launch_bounds__(128) agg_wmedian_fast_kernel(const __grid_constant__ CUtensorMap mapP, int64_t n, int M,
                                                               const __grid_constant__ WmWeights wts, double total,
                                                               double tau, int32_t* __restrict__ list,
                                                               unsigned int* __restrict__ count, unsigned int cap,
                                                               float* __restrict__ out) {
  extern __shared__ __align__(128) unsigned char wm_raw[];
  float* stage0 = reinterpret_cast<float*>(wm_raw + ((128u - (smem_u32(wm_raw) & 127u)) & 127u));
  const int stage_floats = M * 128;
  __shared__ __align__(8) uint64_t full[2];
  if (threadIdx.x == 0) {
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int64_t ntiles = (n + 127) / 128;
  auto issue = [&](int64_t tile, int st) {
    mbar_expect_tx(&full[st], (uint32_t)(stage_floats * sizeof(float)));
    tma_load_tile(stage0 + (size_t)st * stage_floats, &mapP, (int)(tile * 128), &full[st]);
  };
  if (threadIdx.x == 0 && blockIdx.x < ntiles) issue(blockIdx.x, 0);
  uint32_t it = 0;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
    const int st = it & 1;
    if (threadIdx.x == 0 && tile + gridDim.x < ntiles) issue(tile + gridDim.x, st ^ 1);  // freed by the barrier below
    const int64_t row = tile * 128 + threadIdx.x;
    const bool in = row < n;
    mbar_wait(&full[st], (it >> 1) & 1);
    const float* src = stage0 + (size_t)st * stage_floats + threadIdx.x;
    uint32_t key[MP];
#pragma unroll
    for (int m = 0; m < MP; ++m) {
      key[m] = 0xFFFFFFFFu;  // padding sorts last and carries weight 0
      if (m < M) key[m] = wm_key(src[m * 128]);
    }
    __syncthreads();  // the tile is in registers: its stage may be refilled
    bool safe;
    const uint32_t pick = wm_fast_pick<MP>(key, wts.w, total, tau, safe);
    if (in) out[row] = wm_unkey(pick);
    // rows whose decision could depend on the order of summation go to the exact kernel (warp-aggregated append)
    const bool defer = in && list != nullptr && !safe;
    const unsigned mask = __ballot_sync(0xffffffffu, defer);
    if (mask) {
      const int lane = threadIdx.x & 31, leader = __ffs(mask) - 1;
      unsigned base = 0;
      if (lane == leader) base = atomicAdd(count, (unsigned)__popc(mask));
      base = __shfl_sync(0xffffffffu, base, leader);
      const unsigned idx = base + (unsigned)__popc(mask & ((1u << lane) - 1u));
      if (defer && idx < cap) list[idx] = (int32_t)row;
    }
  }
}

// exact pass over the deferred rows (or over ALL rows when the list overflowed): gathers, (key, model) words, the
// reference's sorted-order sums
template <int MP>
__global__ void __launch_bounds__(128) agg_wmedian_list_kernel(const float* __restrict__ P, int64_t n, int64_t ld, int M,
                                                               const double* __restrict__ a,
                                                               const int32_t* __restrict__ list,
                                                               const unsigned int* __restrict__ count, unsigned int cap,
                                                               float* __restrict__ out) {
  __shared__ double s_a[64];
  for (int m = threadIdx.x; m < 64; m += 128) s_a[m] = (m < M) ? a[m] : 0.0;
  __syncthreads();
  const unsigned int c = *count;
  if (c == 0) return;
  const bool all = c > cap;
  const int64_t items = all ? n : (int64_t)c;
  for (int64_t i = (int64_t)blockIdx.x * 128 + threadIdx.x; i < items; i += (int64_t)gridDim.x * 128) {
    const int64_t row = all ? i : (int64_t)list[i];
    unsigned long long w[MP];
#pragma unroll
    for (int m = 0; m < MP; ++m) {
      w[m] = ~0ull;
      if (m < M) w[m] = ((unsigned long long)wm_key(__ldg(P + (int64_t)m * ld + row)) << 32) | (unsigned long long)(unsigned)m;
    }
    out[row] = wm_unkey((uint32_t)(wm_exact_pick<MP>(w, M, s_a) >> 32));
  }
}

// class-wide sum kinds through the tile kernel (2 <= C <= 32 classes, the tile fits in shared memory)
cudaError_t try_launch_agg_class_tile(const AggArgs& a, const FinArgs& f0, int sms, cudaStream_t st, bool* launched) {
  *launched = false;
  if (a.M < 1 || a.n < 1 || a.n >= (int64_t)0x7fffff00) return cudaSuccess;
  // one warp per CTA (128-row tiles), one stage: shared memory bounds occupancy and what counts is the number of
  // boxes in flight per SM (more warps or stages per CTA leave fewer CTAs resident)
  constexpr int kAR = kClassTileRows;
  ClassTileArgs ta{};
  FinArgs f = f0;
  ta.M = a.M;
  switch (a.kind) {
    case SE_AGG_GBM_CLASSIFIER:
      if (a.dim < 2) return cudaSuccess;  // binary dim-1 form: two outputs from one sum (streaming path)
      ta.C = a.dim; ta.a = a.weights; ta.init = a.init; break;
    case SE_AGG_BAGGING_SOFT: ta.C = a.K; break;
    case SE_AGG_BOOSTING_REAL: ta.C = a.K; ta.logp = 1; break;
    default: return cudaSuccess;
  }
  const int C = ta.C;
  if (C < 2 || C > 32) return cudaSuccess;
  f.C = C;
  ta.G = 32 / C;
  if (ta.G > a.M) ta.G = a.M;
  if (ta.G > 8) ta.G = 8;
  const int box_rows = ta.G * C;
  const size_t stage_bytes = (size_t)box_rows * kAR * sizeof(float);
  const size_t total_bytes = (size_t)C * kAR * (ta.logp ? sizeof(double) : sizeof(float));
  const size_t smem = total_bytes + stage_bytes + 128;
  CUtensorMap mapP;
  cudaError_t e = make_tile_map_rows(&mapP, a.P, a.n, a.ld, (int64_t)a.M * C, kAR, box_rows);
  if (e != cudaSuccess) return e;
  int per_sm = (int)((228 * 1024) / (smem + 1280));
  if (per_sm > 16) per_sm = 16;
  if (per_sm < 1) return cudaSuccess;
  const int grid = grid_rows(a.n, kAR, per_sm, sms);
  auto launch = [&](auto kern) {
    const cudaError_t e = allow_dynamic_smem(kern, smem);
    if (e != cudaSuccess) return e;
    kern<<<grid, 32, smem, st>>>(ta, f, mapP);
    *launched = true;
    return cudaGetLastError();
  };
  if (ta.logp) return launch(agg_class_tile_kernel<32, true>);  // no register batch: CMAX is unused
  if (C <= 4) return launch(agg_class_tile_kernel<4, false>);
  if (C <= 8) return launch(agg_class_tile_kernel<8, false>);
  if (C <= 16) return launch(agg_class_tile_kernel<16, false>);
  return launch(agg_class_tile_kernel<32, false>);
}

// Calls f(std::integral_constant<int, MP>()) for the power of two MP >= M that the kernels for M <= 64 models are
// instantiated for.
template <class F>
cudaError_t with_mp(int M, F f) {
  int Mp = 1;
  while (Mp < M) Mp <<= 1;
  switch (Mp) {
    case 1: return f(std::integral_constant<int, 1>());
    case 2: return f(std::integral_constant<int, 2>());
    case 4: return f(std::integral_constant<int, 4>());
    case 8: return f(std::integral_constant<int, 8>());
    case 16: return f(std::integral_constant<int, 16>());
    case 32: return f(std::integral_constant<int, 32>());
    case 64: return f(std::integral_constant<int, 64>());
    default: return cudaErrorInvalidValue;
  }
}

// ---- a classifier forest in one pass (se_forest_agg) -------------------------------------------------------------
// What tree t adds to its row's class totals, for its leaf node `leaf` (chunk-local node index):
//   kFaTreeClass  GBM classifier: w_t · value(leaf) to class cls_t                (GBMClassifier.scala:567-589)
//   kFaVote       bagging hard / boosting discrete: w_t (1 for hard) to class value(leaf) (BaggingClassifier.scala:
//                 260-283, BoostingClassifier.scala:366-382); a value that is not a class index raises bad_label
//   kFaSoft       bagging soft: p_leaf,k to every class k                         (BaggingClassifier.scala:260-287)
//   kFaReal       boosting real: lg2_clamped(p_leaf,k) to every class k           (BoostingClassifier.scala:348-364)
// Every term is added in fp64 in model order, so SAMME.R totals equal the member route's sums term for term.
enum { kFaTreeClass = 0, kFaVote = 1, kFaSoft = 2, kFaReal = 3 };
static_assert(kForestAggMaxClasses == SE_FOREST_AGG_MAX_CLASSES, "the kernel's class limit is the ABI's");

template <int MODE>
__global__ void __launch_bounds__(kForestAggTile) forest_agg_kernel(const ForestAggArgs g, const FinArgs fin) {
  constexpr int TILE = kForestAggTile;
  extern __shared__ __align__(16) unsigned char fsm[];
  const ForestArgs& a = g.f;
  for (int i = threadIdx.x; i < a.blob_bytes / 16; i += TILE)
    reinterpret_cast<uint4*>(fsm)[i] = __ldg(reinterpret_cast<const uint4*>(a.blob) + i);
  const double* s_w = reinterpret_cast<const double*>(fsm);
  const unsigned long long* s_coloff = reinterpret_cast<const unsigned long long*>(fsm + a.off_coloff);
  const uint2* s_nodes = reinterpret_cast<const uint2*>(fsm + a.off_nodes);
  const int* s_toff = reinterpret_cast<const int*>(fsm + a.off_treeoff);
  const int* s_cls = reinterpret_cast<const int*>(fsm + a.off_treecls);
  const float* s_val = reinterpret_cast<const float*>(fsm + a.off_values);
  unsigned char* s_rank = fsm + a.off_ranks;
  double* s_tot = reinterpret_cast<double*>(s_rank + (size_t)a.C * TILE);  // [C][TILE]: off_ranks and C * TILE are 8-aligned
  const int C = g.C, K = g.K;
  bool bad_vote = false;
  const int64_t ntiles = (a.n + TILE - 1) / TILE;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    __syncthreads();  // the packed trees are staged (first tile) / the previous tile's walks are over
    const int64_t row0 = tile * TILE;
    // forest_stage_ranks written out: through the helper, nvcc 12.9 allocates the kFaSoft instantiation 32 instead of
    // 40 registers and it runs 21 % slower (2 M rows, K = 26, H100)
    for (int i = threadIdx.x; i < a.C * (TILE / 4); i += TILE) {
      const int c = i / (TILE / 4), q = i % (TILE / 4);
      const int64_t r = row0 + 4 * q;  // columns are padded to 128 rows: a word at r < ld8 stays inside its column
      uint32_t v = 0;
      if (r < a.ld8) v = __ldg(reinterpret_cast<const uint32_t*>(a.X8 + s_coloff[c] + r));
      *reinterpret_cast<uint32_t*>(s_rank + c * TILE + 4 * q) = v;
    }
    __syncthreads();
    const int64_t row = row0 + threadIdx.x;
    if (row >= a.n) continue;
    double* tot = s_tot + threadIdx.x;  // this row's totals: own column, no synchronisation
    for (int c = 0; c < C; ++c) tot[c * TILE] = g.first ? g.init[c] : g.acc[c * g.ld_acc + row];
    const unsigned char* myr = s_rank + threadIdx.x;
    auto add = [&](int t, int leaf) {
      const int node = s_toff[t] + leaf;
      if constexpr (MODE == kFaTreeClass) {
        tot[s_cls[t] * TILE] += s_w[t] * (double)s_val[node];
      } else if constexpr (MODE == kFaVote) {
        const float v = s_val[node];
        const int c = __float2int_rz(v);
        const bool ok = ((unsigned)c < (unsigned)K) && ((float)c == v);  // a vote is a predicted class index
        bad_vote = bad_vote || !ok;
        if (ok) tot[c * TILE] += s_w[t];
      } else {
        const float* p = g.probs + (size_t)node * K;
        for (int k = 0; k < K; ++k) {
          const float pk = __ldg(p + k);
          tot[k * TILE] += (MODE == kFaReal) ? (double)lg2_clamped(pk) : (double)pk;
        }
      }
    };
    forest_walk<TILE>(s_nodes, s_toff, a.T, myr, add);
    if (!g.last) {
      for (int c = 0; c < C; ++c) g.acc[c * g.ld_acc + row] = tot[c * TILE];
    } else if (MODE == kFaTreeClass && g.dim == 1 && g.K == 2) {
      finalize_binary_row(fin, row, (float)tot[0]);
    } else if (MODE == kFaReal) {
      finalize_real_row(fin, row, [&](int c) { return tot[c * TILE]; });
    } else {
      finalize_row(fin, row, [&](int c) { return tot[c * TILE]; });
    }
  }
  if (bad_vote && g.bad_label != nullptr) *reinterpret_cast<volatile int*>(g.bad_label) = 1;
}

// ---- the weighted median of a regression forest in one pass (se_forest_median) -----------------------------------
// The member route writes every tree's outputs to SE_SLOT_P ([M][n], 4·M B per row) and reads them back in
// agg_wmedian_fast_kernel / agg_wmedian_list_kernel.  Here the row's M leaf values go to its own column of shared
// memory instead, chunk after chunk, and the same decisions are taken on them: the keys-only sort and model-order
// bisection, and the exact (key, model) sort with sorted-order sums for the rows inside the margin (mode 1) or for all
// rows (mode 0: a weight that is negative or not finite, or the fast path switched off).  So every row picks the
// member route's value, bit for bit.
static_assert(kForestMedianMaxTrees == SE_FOREST_MEDIAN_MAX_TREES, "the kernel's tree limit is the ABI's");

// (min blocks 1: with the default bounds ptxas spilled a few bytes at MP = 1; shared memory holds the CTAs per SM to
// four at most anyway)
template <int MP>
__global__ void __launch_bounds__(kForestMedianTile, 1) forest_median_kernel(const __grid_constant__ ForestMedianArgs g) {
  constexpr int TILE = kForestMedianTile;
  extern __shared__ __align__(16) unsigned char fsm[];
  __shared__ double s_a[kForestMedianMaxTrees];
  for (int m = threadIdx.x; m < kForestMedianMaxTrees; m += TILE) s_a[m] = (m < g.M) ? g.w[m] : 0.0;
  const int M = g.M;
  float* vals = reinterpret_cast<float*>(fsm + g.vals_off) + threadIdx.x;  // this row's leaf values: own column
  const unsigned char* myr = fsm + threadIdx.x;  // + the chunk's blob_bytes: this row's ranks
  const int64_t ntiles = (g.n + TILE - 1) / TILE;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * TILE, row = row0 + threadIdx.x;
    const bool in = row < g.n;
    for (int k = 0; k < g.n_chunks; ++k) {
      const ForestMedianChunk ch = g.chunk[k];  // a copy: a reference into the parameters spilled at MP = 16
      const unsigned char* blob = g.blob + ch.blob_off;
      __syncthreads();  // the previous chunk's (or tile's) walks are over
      if (g.n_chunks > 1 || tile == blockIdx.x)  // one chunk stays staged for every tile of the CTA
        for (int i = threadIdx.x; i < ch.blob_bytes / 16; i += TILE)
          reinterpret_cast<uint4*>(fsm)[i] = __ldg(reinterpret_cast<const uint4*>(blob) + i);
      const unsigned long long* coloff = reinterpret_cast<const unsigned long long*>(blob + ch.off_coloff);
      unsigned char* s_rank = fsm + ch.blob_bytes;
      // the offsets are read from the global blob: no barrier orders the blob's staging above before this read
      forest_stage_ranks<TILE>(s_rank, g.X8, g.ld8, ch.C, row0, [&](int c) { return __ldg(coloff + c); });
      __syncthreads();
      if (!in) continue;
      const uint2* s_nodes = reinterpret_cast<const uint2*>(fsm + ch.off_nodes);
      const int* s_toff = reinterpret_cast<const int*>(fsm + ch.off_treeoff);
      const float* s_val = reinterpret_cast<const float*>(fsm + ch.off_values);
      float* v = vals + (size_t)ch.t0 * TILE;
      forest_walk<TILE>(s_nodes, s_toff, ch.T, myr + ch.blob_bytes,
                        [&](int t, int leaf) { v[t * TILE] = s_val[s_toff[t] + leaf]; });
    }
    bool exact;
    const uint32_t pick = wm_pick_row<MP>(vals, TILE, M, g.mode, g.w, g.total, g.tau, s_a, in, exact);
    if (in) g.out[row] = wm_unkey(pick);
    if (g.mode == 1 && g.deferred != nullptr) {  // rows inside the margin, for se_ctx_get_option("last_wm_deferred")
      const unsigned mask = __ballot_sync(0xffffffffu, in && exact);
      if (mask && (threadIdx.x & 31) == __ffs(mask) - 1) atomicAdd(g.deferred, (unsigned)__popc(mask));
    }
  }
}

}  // namespace

cudaError_t launch_agg(const AggArgs& a, int ctas_per_sm, int sms, cudaStream_t st) {
  const int grid4 = grid_rows(a.n >> 2, kBlock, ctas_per_sm, sms);
  const int grid1 = grid_rows(a.n, kBlock, ctas_per_sm, sms);
  FinArgs f{};
  f.kind = a.kind; f.K = a.K; f.dim = a.dim; f.loss = a.loss; f.M = a.M;
  f.n = a.n; f.ld = a.ld_out; f.raw = a.raw; f.prob = a.prob; f.label = a.label;
  f.bad_label = a.bad_label;
  f.inv_km1 = 1.0 / (double)((a.K > 1 ? a.K : 2) - 1);
  f.sum_a = 0.0;
  {
    bool launched = false;
    const cudaError_t e = try_launch_agg_class_tile(a, f, sms, st, &launched);
    if (e != cudaSuccess || launched) return e;
  }
  switch (a.kind) {
    case SE_AGG_GBM_REGRESSOR:
      agg_sum_kernel<false><<<grid4, kBlock, 0, st>>>(a.P, a.n, a.ld, a.M, 1, a.weights, a.init,
                                                       nullptr, 0.f, a.raw, a.ld_out);
      return cudaGetLastError();
    case SE_AGG_BAGGING_REGRESSOR:
      agg_sum_kernel<false><<<grid4, kBlock, 0, st>>>(a.P, a.n, a.ld, a.M, 1, nullptr, nullptr,
                                                       nullptr, (float)a.M, a.raw, a.ld_out);
      return cudaGetLastError();
    case SE_AGG_BOOSTING_REG_MEAN:  // dot(predictions, weights) / Σ weights  (BoostingRegressor.scala:339-342)
      agg_sum_kernel<false><<<grid4, kBlock, 0, st>>>(a.P, a.n, a.ld, a.M, 1, a.weights, nullptr,
                                                       nullptr, (float)a.sum_weights, a.raw, a.ld_out);
      return cudaGetLastError();
    case SE_AGG_BOOSTING_REG_MEDIAN: {
      if (a.M < 1) return cudaErrorInvalidValue;
      int Mp = 1;
      while (Mp < a.M) Mp <<= 1;
      if (Mp <= 64 && a.n > 0 && a.n < (int64_t)0x7fffff00) {  // registers, tiles prefetched by TMA
        CUtensorMap mapP;
        cudaError_t e = make_tile_map(&mapP, a.P, a.n, a.ld, a.M, 128);
        if (e != cudaSuccess) return e;
        const size_t smem = 2 * (size_t)a.M * 128 * sizeof(float) + (size_t)a.M * sizeof(double) + 128;
        const int grid = grid_rows(a.n, 128, 8, sms);
        if (a.wm_mode != 0 && a.weights64_host != nullptr && (a.wm_mode == 2 || (a.wm_list != nullptr && a.wm_count != nullptr))) {
          // fast path: keys-only sort + model-order sums; rows inside the rounding margin go to the exact list kernel
          WmWeights wts;
          double total = 0.0;
          for (int m = 0; m < 64; ++m) {
            wts.w[m] = (m < a.M) ? a.weights64_host[m] : 0.0;
            total += wts.w[m];  // model order, like the kernel's own sums
          }
          const bool margin = (a.wm_mode == 1);
          const double tau = margin ? 8.0 * (double)a.M * 1.1102230246251565e-16 * total : -1.0;  // mode 2: every row is safe
          const size_t fsmem = 2 * (size_t)a.M * 128 * sizeof(float) + 128;
          if (margin) {
            e = cudaMemsetAsync(a.wm_count, 0, sizeof(unsigned int), st);
            if (e != cudaSuccess) return e;
          }
          return with_mp(a.M, [&](auto mp) {
            constexpr int MP = decltype(mp)::value;
            const cudaError_t e = allow_dynamic_smem(agg_wmedian_fast_kernel<MP>, fsmem);
            if (e != cudaSuccess) return e;
            agg_wmedian_fast_kernel<MP><<<grid, 128, fsmem, st>>>(mapP, a.n, a.M, wts, total, tau,
                                                                   margin ? a.wm_list : nullptr, a.wm_count, a.wm_cap,
                                                                   a.raw);
            if (margin)
              agg_wmedian_list_kernel<MP><<<sms * 4, 128, 0, st>>>(a.P, a.n, a.ld, a.M, a.weights64, a.wm_list,
                                                                    a.wm_count, a.wm_cap, a.raw);
            return cudaGetLastError();
          });
        }
        return with_mp(a.M, [&](auto mp) {
          constexpr int MP = decltype(mp)::value;
          const cudaError_t e = allow_dynamic_smem(agg_wmedian_reg_kernel<MP>, smem);
          if (e != cudaSuccess) return e;
          agg_wmedian_reg_kernel<MP><<<grid, 128, smem, st>>>(mapP, a.n, a.M, a.weights64, a.raw);
          return cudaGetLastError();
        });
      }
      const int T = 64;
      const size_t smem = (size_t)a.M * sizeof(double) + (size_t)Mp * T * sizeof(unsigned long long);
      if (smem > 200 * 1024) {  // M > 256: one warp per row
        const size_t wsmem = (size_t)a.M * sizeof(double) + (size_t)kWmWarps * Mp * sizeof(unsigned long long);
        if (wsmem > 200 * 1024) return cudaErrorInvalidValue;  // M > 8192
        cudaError_t e = allow_dynamic_smem(agg_wmedian_warp_kernel, wsmem);
        if (e != cudaSuccess) return e;
        int per_sm_w = (int)((220 * 1024) / (wsmem + 1024));
        if (per_sm_w < 1) per_sm_w = 1;
        if (per_sm_w > 16) per_sm_w = 16;
        const int gridw = grid_rows(a.n, kWmWarps, per_sm_w, sms);
        agg_wmedian_warp_kernel<<<gridw, 32 * kWmWarps, wsmem, st>>>(a.P, a.n, a.ld, a.M, Mp, a.weights64, a.raw);
        return cudaGetLastError();
      }
      auto kern = agg_wmedian_kernel<64>;
      const cudaError_t e = allow_dynamic_smem(kern, smem);
      if (e != cudaSuccess) return e;
      int per_sm = (int)((220 * 1024) / (smem + 1024));
      if (per_sm < 1) per_sm = 1;
      const int grid = grid_rows(a.n, T, per_sm, sms);
      kern<<<grid, T, smem, st>>>(a.P, a.n, a.ld, a.M, Mp, a.weights64, a.raw);
      return cudaGetLastError();
    }
    case SE_AGG_GBM_CLASSIFIER:
      agg_sum_kernel<false><<<grid4, kBlock, 0, st>>>(a.P, a.n, a.ld, a.M, a.dim, a.weights, a.init,
                                                       nullptr, 0.f, a.raw, a.ld_out);
      f.C = (a.dim == 1 && a.K == 2) ? 2 : a.dim;
      break;
    case SE_AGG_BAGGING_SOFT:
      agg_sum_kernel<false><<<grid4, kBlock, 0, st>>>(a.P, a.n, a.ld, a.M, a.K, nullptr, nullptr,
                                                       nullptr, 0.f, a.raw, a.ld_out);
      f.C = a.K;
      break;
    case SE_AGG_BOOSTING_REAL:  // fp64 totals as (hi, lo) pairs in RAW and PROB, read back by finalize_real_row
      agg_sum_kernel<true><<<grid4, kBlock, 0, st>>>(a.P, a.n, a.ld, a.M, a.K, nullptr, nullptr,
                                                      nullptr, 0.f, a.raw, a.ld_out, a.prob);
      f.C = a.K;
      break;
    case SE_AGG_BAGGING_HARD:
    case SE_AGG_BOOSTING_DISCRETE: {
      const bool weighted = (a.kind == SE_AGG_BOOSTING_DISCRETE);
      if (!weighted && a.M <= 255 && (size_t)((a.K + 3) / 4) * kVR * kBlock * 4 <= 160 * 1024) {
        const size_t psmem = (size_t)((a.K + 3) / 4) * kVR * kBlock * sizeof(uint32_t);
        const cudaError_t e = allow_dynamic_smem(agg_hard_votes_packed_kernel, psmem);
        if (e != cudaSuccess) return e;
        f.C = a.K;
        const int gridp = grid_rows((a.n + kVR - 1) / kVR, kBlock, ctas_per_sm, sms);
        agg_hard_votes_packed_kernel<<<gridp, kBlock, psmem, st>>>(a.P, a.ld, a.M, f);
        return cudaGetLastError();
      }
      const size_t hsz = weighted ? sizeof(double) : sizeof(float);
      const size_t smem = (size_t)(a.K + 1) * kBlock * hsz + (size_t)a.M * hsz;
      f.C = a.K;
      f.sum_a = a.sum_weights;
      if (smem > 200 * 1024) {  // the histogram does not fit in shared memory: keep it in the output columns
        agg_votes_global_kernel<<<grid1, kBlock, 0, st>>>(a.P, a.ld, a.M, weighted ? a.weights : nullptr, f);
        return cudaGetLastError();
      }
      auto kern = weighted ? agg_votes_kernel<double> : agg_votes_kernel<float>;
      const cudaError_t e = allow_dynamic_smem(kern, smem);
      if (e != cudaSuccess) return e;
      kern<<<grid1, kBlock, smem, st>>>(a.P, a.ld, a.M, weighted ? a.weights : nullptr, f);
      return cudaGetLastError();  // epilogue fused: no separate finalize launch
    }
    default: return cudaErrorInvalidValue;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  if (a.kind == SE_AGG_BOOSTING_DISCRETE) {
    // Σ a_m is needed by the epilogue (host-side sum of the tiny weight vector)
    f.sum_a = a.sum_weights;
  }
  agg_finalize_kernel<<<grid1, kBlock, 0, st>>>(f);
  return cudaGetLastError();
}

cudaError_t launch_forest_agg(const ForestAggArgs& g, int sms, cudaStream_t st) {
  const ForestArgs& a = g.f;
  const size_t smem = (size_t)a.off_ranks + (size_t)a.C * kForestAggTile + (size_t)g.C * kForestAggTile * sizeof(double);
  if (a.T < 1 || a.C < 0 || g.C < 1 || g.C > kForestAggMaxClasses || smem > 220 * 1024 || (a.blob_bytes & 15) != 0)
    return cudaErrorInvalidValue;
  FinArgs f{};
  f.kind = g.kind; f.C = g.C; f.K = g.K; f.dim = g.dim; f.loss = g.loss; f.M = g.M;
  f.sum_a = g.sum_a;
  f.n = a.n; f.ld = g.ld_out; f.raw = g.raw; f.prob = g.prob; f.label = g.label;
  f.bad_label = g.bad_label;
  f.inv_km1 = 1.0 / (double)((g.K > 1 ? g.K : 2) - 1);
  int per_sm = (int)((220 * 1024) / (smem + 1024));
  if (per_sm < 1) per_sm = 1;
  if (per_sm > 16) per_sm = 16;
  const int grid = grid_rows(a.n, kForestAggTile, per_sm, sms);
  auto launch = [&](auto kern) {
    const cudaError_t e = allow_dynamic_smem(kern, smem);
    if (e != cudaSuccess) return e;
    kern<<<grid, kForestAggTile, smem, st>>>(g, f);
    return cudaGetLastError();
  };
  switch (g.kind) {
    case SE_AGG_GBM_CLASSIFIER: return launch(forest_agg_kernel<kFaTreeClass>);
    case SE_AGG_BAGGING_HARD:
    case SE_AGG_BOOSTING_DISCRETE: return launch(forest_agg_kernel<kFaVote>);
    case SE_AGG_BAGGING_SOFT: return launch(forest_agg_kernel<kFaSoft>);
    case SE_AGG_BOOSTING_REAL: return launch(forest_agg_kernel<kFaReal>);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t forest_median_ctas_per_sm(int M, int* ctas) {
  cudaFuncAttributes fa{};
  const cudaError_t e =
      with_mp(M, [&](auto mp) { return cudaFuncGetAttributes(&fa, forest_median_kernel<decltype(mp)::value>); });
  if (e != cudaSuccess) return e;
  const int regs = (fa.numRegs + 7) / 8 * 8;  // allocated per thread in units of 8
  *ctas = regs > 0 ? 65536 / (regs * kForestMedianTile) : 16;
  if (*ctas < 1) *ctas = 1;
  return cudaSuccess;
}

cudaError_t launch_forest_median(const ForestMedianArgs& g, size_t smem, int sms, cudaStream_t st) {
  if (g.M < 1 || g.M > kForestMedianMaxTrees || g.n_chunks < 1 || g.n_chunks > g.M || smem > 220 * 1024)
    return cudaErrorInvalidValue;
  int per_sm = (int)((228 * 1024) / (smem + sizeof(double) * kForestMedianMaxTrees + 1024));
  if (per_sm < 1) per_sm = 1;
  if (per_sm > 16) per_sm = 16;
  const int grid = grid_rows(g.n, kForestMedianTile, per_sm, sms);
  return with_mp(g.M, [&](auto mp) {
    auto kern = forest_median_kernel<decltype(mp)::value>;
    const cudaError_t e = allow_dynamic_smem(kern, smem);
    if (e != cudaSuccess) return e;
    kern<<<grid, kForestMedianTile, smem, st>>>(g);
    return cudaGetLastError();
  });
}

}  // namespace se
