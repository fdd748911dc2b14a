// se_gbm_fused.cu — whole-round and whole-line-search kernels (sm_90a): the per-round fixed costs (kernel
// launches, host round trips between the line search and the update, one cross-GPU exchange per launch) are what
// bounds small row shards — exactly the shards STRONG scaling produces (100 M rows / 8 GPUs = 12.5 M rows per GPU,
// tens of microseconds per round at the HBM roofline).  Two cooperative (co-resident, persistent) kernels remove them:
//
//  * gbm_round_sq_fused_kernel — a complete squared-loss boosting round (regression/GBMRegressor.scala:398-442 +
//    :368-385 of the reference) in ONE launch: statistics pass (8 B/row) -> last CTA folds the partials, sums them
//    across GPUs over peer memory and runs Brent (se_brent.h, the same template as the host line search) -> the step
//    is published through an acquire/release flag while every other CTA already has the first update tile's loads in
//    flight -> next pseudo-residuals r' = r - c h + loss (12 B/row), walking the tiles in the opposite direction
//    so that the statistics pass's tail of r and h is still on chip (residual rounds without a bag keep each CTA's
//    last tile in registers and the groups before it in shared memory; otherwise the tail is in the L2) -> loss
//    reduction + second exchange + host mirror.  1 launch, 0 host round trips inside the round.
//    The round (residual mode) does not read or write F: nothing reads it between rounds, and for the squared loss
//    F = y - r.  The host marks F as owed and rebuilds it from y and r when F is next accessed (se_api.cu settle_f).
//    A round whose residual slot is not current (Y, F or R were just written) reads (y, F, h) instead of (r, h):
//    r' = (y - F) - c h, 16 B/row.  Without residual mode the update is F' = F + c h (F, y, h read; F written).
//
//  * gbm_linesearch_persist_kernel — Brent's <= MaxEval evaluations of the line-search objective
//    (boosting/GBMLoss.scala:50-74 through RDDLossFunction; GBMRegressor.scala:408-421) for the non-squared scalar
//    losses in ONE launch: worker CTAs own a fixed set of tiles, keep the first of them in SHARED MEMORY for the whole
//    search (132 SMs x ~190 KB = 25 MB on an H100 that never touch HBM again) and stream the rest (the caller marks the packed
//    view as L2-persisting); a coordinator warp folds the per-CTA partials in a fixed order, performs the cross-GPU
//    sum, advances Brent and publishes the next abscissa.  The first evaluation of the binary losses also BUILDS the
//    signed view u = (2y-1)F, v = (2y-1)h (exact sign flips: later evaluations read 8 B/row and are bit-identical to
//    evaluating on (y, F, h)).
//
// This translation unit is compiled with -fmad=false so that Brent executes the same IEEE operations as the host
// build of the template (bit-identical iterates); the per-row arithmetic below uses explicit fmaf().
#include "se_brent.h"
#include "se_kernels.h"
#include "se_loss.cuh"

namespace se {

namespace {

__device__ __forceinline__ unsigned long long ld_acquire_gpu_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_gpu_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu_add_u32(unsigned int* p, unsigned int v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// bulk L2 prefetch of a contiguous global range (bytes: multiple of 16, address 16 B aligned)
__device__ __forceinline__ double global_timer_us() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return (double)t * 1e-3;
}
__device__ __forceinline__ void prefetch_l2_bulk(const void* p, unsigned int bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}

// =================================================================================== squared-loss round, one launch
constexpr int U_SQ = 4;  // float4 groups per thread per tile (as the two-launch kernels)
// Residual-mode rounds that read r (no bag) carry phase A's tail into phase B on chip: the CTA's last tile stays in
// registers and the groups before it in shared memory, one slot per float4 group of r and of h (8 KB per CTA), so
// that a slot, not a whole 32 KB tile, is the unit the SM's shared memory is split into.
constexpr int kSqSlotBytes = 2 * kBlock * 16;

// The line search of the fused round, executed by ONE thread of the last CTA once the statistics are folded (and
// summed across GPUs) while every other CTA waits for the step with its first update tile's loads in flight.
template <bool LOSS_REDUCE>
__device__ __forceinline__ void fused_round_brent(const SqRoundArgs& a) {
  if (a.timing) a.out[11] = global_timer_us();  // statistics folded (and summed across GPUs)
  const double s0 = a.out[0], s1 = a.out[1], s2 = a.out[2];
  const BrentParabola f{s0, s1, s2, a.wsum};
  double x = 1.0, fx = 0.0;
  int evals = 0;
  const int rc = brent_core(f, a.lo, a.hi, a.start, a.rel, a.abs_tol, a.max_eval, &x, &fx, &evals);
  const double ne = (rc == kBrentOk) ? (double)evals : -(double)evals;  // negative: MaxEval exceeded
  a.out[4] = x, a.out[5] = fx, a.out[6] = ne;
  // MaxEval exceeded: the host reports SE_ERR_OPT and F must stay what it was (r - 0*h == r, F + 0*h == F; the host
  // does not mark F as owed)
  const double step = (rc == kBrentOk) ? a.lr * x : 0.0;
  a.sync->x = step;
  st_release_gpu_u64(&a.sync->flag, a.epoch);  // the grid starts the update NOW; the host is served next
  if (a.timing) a.out[12] = global_timer_us();  // step published
  if (a.host_res) {  // mapped host memory, above what a reducing kernel writes before its ticket
    a.host_res[0] = s0, a.host_res[1] = s1, a.host_res[2] = s2;
    a.host_res[4] = x, a.host_res[5] = fx, a.host_res[6] = ne;
  }
  if constexpr (!LOSS_REDUCE) {
    // Train loss after the update WITHOUT a second pass-wide reduction (and, across GPUs, without a second
    // exchange): Σ (y - F - c h)²/2 = (s0 - 2 c s1 + c² s2)/2 exactly, from the GLOBAL statistics every GPU already
    // holds; c is the fp32 step the update applies.  (Differs from summing the fp32 rows by their rounding only,
    // ~1e-7 relative.)  The host gets alpha, the loss and its ticket here — while the update phase is still
    // running — so the next round's launch overlaps this round's tail.
    const double c = (double)(float)step;
    const double loss = 0.5 * (s0 - 2.0 * c * s1 + c * c * s2);
    a.out[8] = loss;
    if (a.host_final) {
      a.host_final[0] = loss;
      __threadfence_system();
      *a.host_flag = a.host_ticket;
    }
  } else if (a.host_res) {
    __threadfence_system();
  }
}

// FROM_R (the path a fit and the benchmark take: residual mode, the residual slot current, no bag) is a compile-time
// specialisation: it carries phase A's tail into phase B on chip (kSqSlotBytes) and has no y / F / bag arrays live.
template <bool WRITE_R, bool LOSS_REDUCE, bool FROM_R>
__global__ void __launch_bounds__(kBlock, 3) gbm_round_sq_fused_kernel(const SqRoundArgs a) {
  static_assert(WRITE_R || !FROM_R, "FROM_R is a residual-mode round");
  constexpr int U = U_SQ;
  extern __shared__ float4 s_res[];  // FROM_R: [slot][r, h][kBlock]
  __shared__ float s_coef;
  __shared__ float4 s_brent_regs[2 * U];  // FROM_R: the Brent thread's carried groups while it runs Brent
  const int64_t n4 = a.n >> 2;
  constexpr int64_t tile = (int64_t)kBlock * U;
  const int64_t ntiles = (n4 + tile - 1) / tile;
  const int64_t G = gridDim.x;
  const int64_t cnt = (ntiles > (int64_t)blockIdx.x) ? (ntiles - 1 - blockIdx.x) / G + 1 : 0;  // tiles b, b+G, ...
  const bool has_bag = !FROM_R && (a.bag != nullptr);
  const bool stats_from_r = FROM_R || a.stats_from_r;
  // FROM_R: group u of tile i has the flat index i*U + u.  The last tile (cnt-1) stays in registers, the S groups
  // before it in shared memory: every group from p_res on is carried to phase B.
  const int64_t S = FROM_R ? min((int64_t)a.resident_slots, (cnt > 0 ? cnt - 1 : 0) * U) : 0;
  const int64_t p_res = (cnt - 1) * U - S;
  // l2_mode 1: r and h are the arrays worth keeping between phases / rounds (r: written by the update, read by the
  // next statistics pass; h: read by both phases) -> evict_last; y and F stream through -> evict_first
  const uint64_t pol_stream = l2_policy(a.l2_hints != 0);
  const uint64_t pol_keep = (a.l2_mode == 1) ? l2_policy_evict_last() : l2_policy(false);
  const uint64_t pol_r_in = (a.l2_mode == 1) ? pol_keep : pol_stream;
  const uint64_t pol_h_b = (a.l2_mode == 1) ? pol_keep : pol_stream;
  // carried groups are served from chip in phase B: their L2 lines go first, so that the L2 keeps the groups before
  // them, which phase B reads next
  const uint64_t pol_carried = l2_policy(true);

  if (a.timing && blockIdx.x == 0 && threadIdx.x == 0) a.out[10] = global_timer_us();
  // ---- phase A: Σ(y-F)², Σh(y-F), Σh² (from the current residual slot when it is valid: 8 B/row)
  double acc[3] = {0.0, 0.0, 0.0};
  auto stats_tile = [&](int64_t i, float4 (&vy)[U], float4 (&vF)[U], float4 (&vh)[U], bool (&ok)[U]) {
    const int64_t base = (blockIdx.x + i * G) * tile + threadIdx.x;
    float4 vb[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t g = base + (int64_t)u * kBlock;
      ok[u] = g < n4;
      if (ok[u]) {
        if constexpr (FROM_R) {
          const bool carried = i * U + u >= p_res;
          vy[u] = ld_rw4_p(a.r + 4 * g, carried ? pol_carried : pol_r_in);
          vh[u] = ld_stream4_p(a.h + 4 * g, carried ? pol_carried : pol_keep);
        } else {
          if (stats_from_r) {
            vy[u] = ld_rw4_p(a.r + 4 * g, pol_r_in);  // read again and rewritten by phase B
          } else {
            vy[u] = ld_stream4_p(a.y + 4 * g, pol_keep);
            vF[u] = ld_rw4_p(a.F + 4 * g, pol_keep);
          }
          vh[u] = ld_stream4_p(a.h + 4 * g, pol_keep);   // re-read by phase B, starting from this pass's tail
          if (has_bag) vb[u] = ld_stream4(a.bag + 4 * g);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (!ok[u]) continue;
      float s0 = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float d = stats_from_r ? f4at(vy[u], e) : f4at(vy[u], e) - f4at(vF[u], e), h = f4at(vh[u], e);
        const float c = has_bag ? f4at(vb[u], e) : 1.0f;
        s0 = fmaf(c * d, d, s0);
        s1 = fmaf(c * h, d, s1);
        s2 = fmaf(c * h, h, s2);
      }
      acc[0] += (double)s0;
      acc[1] += (double)s1;
      acc[2] += (double)s2;
    }
    if constexpr (FROM_R) {
      if (i < cnt - 1) {  // each thread writes, and in phase B reads back, only its own slots: no barrier
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int64_t s = i * U + u - p_res;
          if (s >= 0 && ok[u]) {
            s_res[(2 * s) * kBlock + threadIdx.x] = vy[u];
            s_res[(2 * s + 1) * kBlock + threadIdx.x] = vh[u];
          }
        }
      }
    }
  };
  // phase B's tile registers.  FROM_R: phase A loads into them, so that its last tile is where phase B starts; the
  // other rounds keep phase A's tiles local, so that nothing is live across the wait but what phase B loads.
  float4 vy[U], vF[U], vh[U];  // from_r: vy holds r and vF is unused
  bool ok[U];
  for (int64_t i = 0; i < cnt; ++i) {
    if constexpr (FROM_R) {
      stats_tile(i, vy, vF, vh, ok);
    } else {
      float4 ty[U], tF[U], th[U];
      bool tok[U];
      stats_tile(i, ty, tF, th, tok);
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < (a.n & 3)) {
    const int64_t i = (n4 << 2) + threadIdx.x;
    const float d = stats_from_r ? a.r[i] : a.y[i] - a.F[i], h = a.h[i];
    const float c = has_bag ? a.bag[i] : 1.0f;
    acc[0] += (double)(c * d * d);
    acc[1] += (double)(c * h * d);
    acc[2] += (double)(c * h * h);
  }
  const bool last = block_reduce_publish<3>(acc, a.ws_a);  // the last CTA also sums across GPUs (peer_exchange)
  if (last) {
    __syncthreads();  // a.out[0..2] were written by other threads of this CTA
    if (threadIdx.x == 0) {
      // FROM_R: Brent needs more registers than are left beside the carried tile; its thread parks that tile in
      // shared memory meanwhile instead of spilling to local memory
      if constexpr (FROM_R) {
#pragma unroll
        for (int u = 0; u < U; ++u) s_brent_regs[u] = vy[u], s_brent_regs[U + u] = vh[u];
      }
      fused_round_brent<LOSS_REDUCE>(a);
      if constexpr (FROM_R) {
#pragma unroll
        for (int u = 0; u < U; ++u) vy[u] = s_brent_regs[u], vh[u] = s_brent_regs[U + u];
      }
    }
  }

  // ---- phase B, tiles in the opposite direction.  WRITE_R (residual mode): r' = r - step*h, Σ r'²/2; F is not
  // touched (the host rebuilds it as y - r' when it is next accessed), or r' = (y - F) - step*h on a round whose
  // residual slot is not current.  Otherwise: F' = F + step*h, Σ (y-F')²/2.  The order of the tiles, and so of the
  // loss sum, is the same whether a tile comes from registers, shared memory or global memory.
  const bool from_r = WRITE_R && stats_from_r;
  auto load_tile = [&](int64_t i) {
    const int64_t base = (blockIdx.x + i * G) * tile + threadIdx.x;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t g = base + (int64_t)u * kBlock;
      ok[u] = g < n4;
      if (ok[u]) {
        const int64_t s = i * U + u - p_res;
        if (FROM_R && s >= 0) {
          vy[u] = s_res[(2 * s) * kBlock + threadIdx.x];
          vh[u] = s_res[(2 * s + 1) * kBlock + threadIdx.x];
          continue;
        }
        if (from_r) {
          vy[u] = ld_rw4_p(a.r + 4 * g, pol_stream);
        } else {
          vy[u] = ld_stream4_p(a.y + 4 * g, pol_stream);
          vF[u] = ld_rw4_p(a.F + 4 * g, pol_stream);
        }
        vh[u] = ld_stream4_p(a.h + 4 * g, pol_h_b);  // the update is h's last reader
      }
    }
  };
  int64_t i = cnt - 1;
  // in flight while the last CTA reduces, exchanges and runs Brent (FROM_R: still in registers from phase A)
  if (!FROM_R && i >= 0) load_tile(i);
  if (threadIdx.x == 0) {
    // The wait (partials fold + cross-GPU exchange + ~30 dependent fp64 Brent iterations) is turned into
    // useful HBM time: every CTA pulls the ranges its next update tiles read (r and h, or y and F) into the L2 with
    // bulk prefetches (one instruction per 16 KB), bounded so that the whole grid stays within a.prefetch_tiles tiles
    // per CTA.
    const float* pf0 = from_r ? a.r : a.y;
    const float* pf1 = from_r ? a.h : a.F;
    int64_t pf = i - 1;
    if constexpr (FROM_R) {
      // nothing of the carried tail is loaded: the loads issued before the wait are those of the first tile phase B
      // reads from global memory (its groups below p_res)
      pf = p_res > 0 ? (p_res - 1) / U : -1;
      if (pf >= 0) {
        const int64_t g0 = (blockIdx.x + pf * G) * tile;
        int64_t groups = (p_res - pf * U) * kBlock;
        if (groups > n4 - g0) groups = n4 - g0;
        if (groups > 0) {
          prefetch_l2_bulk(pf0 + 4 * g0, (unsigned int)(groups * 16));
          prefetch_l2_bulk(pf1 + 4 * g0, (unsigned int)(groups * 16));
        }
        --pf;
      }
    }
    int budget = a.prefetch_tiles;
    while (ld_acquire_gpu_u64(&a.sync->flag) != a.epoch) {
      if (budget > 0 && pf >= 0) {
        const int64_t g0 = (blockIdx.x + pf * G) * tile;           // first float4 group of the tile
        int64_t groups = n4 - g0;
        if (groups > tile) groups = tile;
        if (groups > 0) {
          prefetch_l2_bulk(pf0 + 4 * g0, (unsigned int)(groups * 16));
          prefetch_l2_bulk(pf1 + 4 * g0, (unsigned int)(groups * 16));
        }
        --pf;
        --budget;
      }
    }
    s_coef = (float)a.sync->x;  // same rounding as the host path: (float)(lr * alpha)
  }
  __syncthreads();
  const float coef = s_coef;
  double accb[1] = {0.0};
  while (i >= 0) {
    const int64_t base = (blockIdx.x + i * G) * tile + threadIdx.x;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (!ok[u]) continue;
      const int64_t g = base + (int64_t)u * kBlock;
      float4 o;
      float l_acc = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float d;
        if constexpr (WRITE_R) {
          // -g(y, F + step*h) = (y - F) - step*h (GBMRegressor.scala:383, 434-441)
          const float r = from_r ? f4at(vy[u], e) : f4at(vy[u], e) - f4at(vF[u], e);
          d = fmaf(-coef, f4at(vh[u], e), r);
          f4at(o, e) = d;
        } else {
          const float p = fmaf(coef, f4at(vh[u], e), f4at(vF[u], e));  // GBMRegressor.scala:434-441
          d = f4at(vy[u], e) - p;
          f4at(o, e) = p;
        }
        if (LOSS_REDUCE) l_acc = fmaf(0.5f * d, d, l_acc);           // GBMLoss.scala:129-137
      }
      if (WRITE_R) st_stream4_p(a.r + 4 * g, o, pol_keep);  // the next statistics pass starts where this one ends
      else st_stream4_p(a.F + 4 * g, o, pol_stream);
      if (LOSS_REDUCE) accb[0] += (double)l_acc;
    }
    --i;
    if (i >= 0) load_tile(i);
  }
  if (blockIdx.x == 0 && threadIdx.x < (a.n & 3)) {
    const int64_t j = (n4 << 2) + threadIdx.x;
    float d;
    if constexpr (WRITE_R) {
      d = fmaf(-coef, a.h[j], from_r ? a.r[j] : a.y[j] - a.F[j]);
      a.r[j] = d;
    } else {
      const float p = fmaf(coef, a.h[j], a.F[j]);
      d = a.y[j] - p;
      a.F[j] = p;
    }
    accb[0] += (double)(0.5f * d * d);
  }
  if constexpr (LOSS_REDUCE) {
    const bool last_b = block_reduce_publish<1>(accb, a.ws_b);  // Σloss -> a.ws_b.out (+ cross-GPU sum, host mirror + ticket)
    if (a.timing && last_b && threadIdx.x == 0) a.out[13] = global_timer_us();
  } else if (a.timing) {
    // no reduction (the loss came from the statistics): the latest stamp of any CTA marks the end of the update
    __syncthreads();
    if (threadIdx.x == 0) atomicMax(reinterpret_cast<unsigned long long*>(&a.out[13]), (unsigned long long)__double_as_longlong(global_timer_us()));
  }
}

// =================================================================================== persistent line search
// 16-byte asynchronous global -> shared copies (LDGSTS).  Every thread copies, waits for and reads back ONLY its own
// 16-byte slots, so the ring needs no block barrier: cp.async.wait_group orders the executing thread's own copies.
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_pending(int pending) {  // at most `pending` newest groups still in flight
  switch (pending) {
    case 0: asm volatile("cp.async.wait_group 0;" ::: "memory"); break;
    case 1: asm volatile("cp.async.wait_group 1;" ::: "memory"); break;
    case 2: asm volatile("cp.async.wait_group 2;" ::: "memory"); break;
    default: asm volatile("cp.async.wait_group 3;" ::: "memory"); break;
  }
}

// Tiles hold U float4 groups per thread of NARR arrays: (u, v) for the binary losses, (y, F, h) otherwise.
template <int LOSS>
struct LsTraits {
  static constexpr bool kPacked = (LOSS == SE_LOSS_BERNOULLI || LOSS == SE_LOSS_EXPONENTIAL);
  static constexpr int kNarr = kPacked ? 2 : 3;
  static constexpr int kU = 2;
  static constexpr int kTileBytes = kNarr * kU * kBlock * 16;
};

// Binary losses as functions of their argument z, with the label encoding and constant factors folded into the
// packed view (multiplications by +-1 / +-2 are exact, so z equals the argument the plain evaluators form bit for bit):
//   bernoulli   (GBMLoss.scala:297-301): loss = log1pExp(-2 y~ p),  z = 2 y~ p  -> scale 2 y~
//   exponential (:272-276):               loss = exp(-y~ p),         z = y~ p    -> scale y~
template <int LOSS>
__device__ __forceinline__ float signed_scale(float y) {
  const float ye = 2.0f * y - 1.0f;
  return (LOSS == SE_LOSS_BERNOULLI) ? 2.0f * ye : ye;
}
template <int LOSS>
__device__ __forceinline__ float binary_loss_of_z(float z) {
  if constexpr (LOSS == SE_LOSS_BERNOULLI) {
    const float t = exp_neg_fast(-fabsf(z));
    return fmaxf(-z, 0.f) + log1p_unit(t);
  } else {
    return exp_fast(-z);
  }
}

template <int LOSS>
__global__ void __launch_bounds__(kBlock, 4) gbm_linesearch_persist_kernel(const LsArgs a) {
  using T = LsTraits<LOSS>;
  constexpr int U = T::kU, NARR = T::kNarr;
  constexpr bool PACKED = T::kPacked;
  extern __shared__ float4 s_dyn[];  // [ring stage][NARR][U][kBlock] then [resident][NARR][U][kBlock]
  __shared__ double s_red[kBlock / 32];
  __shared__ double s_x;
  __shared__ int s_cmd;
  const int W = (int)gridDim.x - 1;  // worker CTAs; the last CTA coordinates
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if ((int)blockIdx.x == W) {
    // ------------------------------------------------------------------ coordinator: warp 0, all lanes in lockstep
    if (warp != 0) return;
    int e = 0;
    bool failed = false;
    double t_pub = a.timing ? global_timer_us() : 0.0, t_pass = 0.0, t_fold = 0.0;  // diagnostics (lane 0)
    auto f = [&](double x) -> double {
      ++e;
      if (e > 1) {  // the first abscissa (start / the single point) is known to every worker at launch
        if (lane == 0) {
          a.sync->x = x;
          a.sync->cmd = 0;
          st_release_gpu_u64(&a.sync->flag, a.epoch0 + (unsigned long long)e);
        }
        __syncwarp();
      }
      if (a.timing && e > 1) t_pub = global_timer_us();
      const unsigned int want = (unsigned int)W * (unsigned int)e;
      while (ld_acquire_gpu_u32(&a.sync->arrive) != want) {}
      const double t_arr = a.timing ? global_timer_us() : 0.0;
      if (a.timing) t_pass += t_arr - t_pub;
      double s = 0.0;
      for (int b = lane; b < W; b += 32) s += __ldcg(&a.partials[b]);  // fixed order: deterministic sums
      s = warp_sum(s);
      s = __shfl_sync(0xffffffffu, s, 0);
      if (a.ws.nranks > 1 && a.ws.mbox != nullptr) {
        RedWs ws = a.ws;
        ws.seq = a.ws.seq + (unsigned long long)(e - 1);
        double tot = s, g = 0.0;
        const bool ok = peer_allreduce_warp(&tot, 1, ws, [&](int, double v) { g = v; });
        s = __shfl_sync(0xffffffffu, g, 0);
        if (!ok) failed = true;
      }
      if (a.timing) { const double t1 = global_timer_us(); t_fold += t1 - t_arr; t_pub = t1; }
      return s / a.wsum;  // dim == 1: lossSum / weightSum (GBMLoss.scala:60-65)
    };
    double x = a.start, fx = 0.0;
    int evals = 0, rc = kBrentOk;
    if (a.single) {
      fx = f(a.start);
      evals = 1;
    } else {
      // a dead peer turns every further sum into NaN: stop the search instead of waiting MaxEval timeouts
      auto guarded = [&](double xx) -> double { return failed ? __longlong_as_double(0x7ff8000000000000ll) : f(xx); };
      rc = brent_core(guarded, a.lo, a.hi, a.start, a.rel, a.abs_tol, failed ? 1 : a.max_eval, &x, &fx, &evals);
    }
    if (lane == 0) {
      a.sync->cmd = 1;  // stop
      a.sync->arrive = 0;
      st_release_gpu_u64(&a.sync->flag, a.epoch0 + (unsigned long long)(e + 1));
      const double ne = (rc == kBrentOk) ? (double)evals : -(double)evals;
      a.out[0] = x, a.out[1] = fx, a.out[2] = ne, a.out[3] = (double)e;
      if (a.timing) a.out[4] = t_pass, a.out[5] = t_fold;  // us in worker passes (publish -> all arrived) / in fold + exchange
      if (a.ws.host_out) {
        a.ws.host_out[0] = x, a.ws.host_out[1] = fx, a.ws.host_out[2] = ne, a.ws.host_out[3] = (double)e;
        __threadfence_system();
        *a.ws.host_flag = a.ws.host_ticket;
      }
    }
    return;
  }

  // -------------------------------------------------------------------- workers
  const int64_t n4 = a.n >> 2;
  constexpr int64_t tile = (int64_t)kBlock * U;
  const int64_t ntiles = (n4 + tile - 1) / tile;
  const int64_t cnt = (ntiles > (int64_t)blockIdx.x) ? (ntiles - 1 - blockIdx.x) / W + 1 : 0;  // tiles b, b+W, ...
  const int64_t R = cnt < a.resident_tiles ? cnt : a.resident_tiles;                           // kept in shared memory
  const float param = a.param;
  const uint64_t pol_keep = l2_policy(false);
  const int S = a.ring_stages;
  float4* const s_ring = s_dyn;
  float4* const s_tiles = s_dyn + (size_t)S * NARR * U * kBlock;

  auto row_loss = [&](float c0, float c1, float c2, float coef) -> float {
    // PACKED: (u, v) hold the loss ARGUMENT directly (signed_scale folded in, exact): z = u + coef*v
    if constexpr (PACKED) return binary_loss_of_z<LOSS>(fmaf(coef, c1, c0));
    else return eval_loss<LOSS>(c0, fmaf(coef, c2, c1), param).l;
  };

  for (int e = 1;; ++e) {
    float4 reg[NARR][U];
    bool ok[U];
    const int dir = (a.first_parity + e) & 1;
    const bool first = (e == 1);
    // issue the loads of the first streamed tile, then wait for the abscissa
    auto stream_index = [&](int64_t k) { return dir ? (cnt - 1 - k) : (R + k); };  // k-th streamed tile of this pass
    const int64_t nstream = cnt - R;
    auto load_tile = [&](int64_t i, bool from_source) {
      const int64_t base = (blockIdx.x + i * (int64_t)W) * tile + tid;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t g = base + (int64_t)u * kBlock;
        ok[u] = g < n4;
        if (!ok[u]) continue;
        if (PACKED && !from_source) {
          reg[0][u] = ld_rw4(a.u + 4 * g);  // written by this very thread in the first evaluation
          reg[1][u] = ld_rw4(a.v + 4 * g);
        } else {
          const float4 y4 = ld_stream4_p(a.y + 4 * g, pol_keep), F4 = ld_stream4_p(a.F + 4 * g, pol_keep),
                       h4 = ld_stream4_p(a.h + 4 * g, pol_keep);
          if constexpr (PACKED) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float ye = signed_scale<LOSS>(f4at(y4, q));
              f4at(reg[0][u], q) = ye * f4at(F4, q);
              f4at(reg[1][u], q) = ye * f4at(h4, q);
            }
          } else {
            reg[0][u] = y4; reg[1][u] = F4; reg[NARR - 1][u] = h4;
          }
        }
      }
    };
    // ring: the streamed tiles of this pass travel global -> shared by cp.async, S stages ahead of the arithmetic.
    // The first S of them are requested BEFORE the wait for the abscissa (they do not depend on it), so the
    // coordinator's fold + exchange hides their latency.  The first evaluation of a packed loss converts (y, F, h)
    // on the way and keeps the register path.
    const bool ring = S > 0 && !(PACKED && first);
    auto ring_issue = [&](int stage, int64_t i) {
      const int64_t base = (blockIdx.x + i * (int64_t)W) * tile + tid;
      float4* st = s_ring + (size_t)stage * NARR * U * kBlock;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t g = base + (int64_t)u * kBlock;
        if (g >= n4) continue;
        if constexpr (PACKED) {
          cp_async16(&st[(0 * U + u) * kBlock + tid], a.u + 4 * g);
          cp_async16(&st[(1 * U + u) * kBlock + tid], a.v + 4 * g);
        } else {
          cp_async16(&st[(0 * U + u) * kBlock + tid], a.y + 4 * g);
          cp_async16(&st[(1 * U + u) * kBlock + tid], a.F + 4 * g);
          cp_async16(&st[(2 * U + u) * kBlock + tid], a.h + 4 * g);
        }
      }
    };
    if (ring) {
      for (int s = 0; s < S; ++s) {  // exactly S groups (empty ones past the end keep the wait_group count uniform)
        if (s < nstream) ring_issue(s, stream_index(s));
        cp_async_commit();
      }
    } else if (nstream > 0) {
      load_tile(stream_index(0), first || !PACKED);
    }
    double x;
    if (first) {
      x = a.start;
    } else {
      if (tid == 0) {
        while (ld_acquire_gpu_u64(&a.sync->flag) != a.epoch0 + (unsigned long long)e) {}
        s_cmd = a.sync->cmd;
        s_x = a.sync->x;
      }
      __syncthreads();
      if (s_cmd) return;
      x = s_x;
    }
    const float coef = (float)x;  // same narrowing as se_gbm_linesearch_eval
    double acc = 0.0;
    if (ring) {
      int stage = 0;
      for (int64_t k = 0; k < nstream; ++k) {
        cp_async_wait_pending(S - 1);  // group k (the oldest of the S outstanding) has landed
        const int64_t base = (blockIdx.x + stream_index(k) * (int64_t)W) * tile + tid;
        const float4* st = s_ring + (size_t)stage * NARR * U * kBlock;
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (base + (int64_t)u * kBlock >= n4) continue;
          float4 c[NARR];
#pragma unroll
          for (int q = 0; q < NARR; ++q) c[q] = st[(q * U + u) * kBlock + tid];
          float l = 0.f;
#pragma unroll
          for (int q = 0; q < 4; ++q) l += row_loss(f4at(c[0], q), f4at(c[1], q), f4at(c[NARR - 1], q), coef);
          acc += (double)l;
        }
        // refill this stage only after its values were consumed (the thread's own reads precede its own new copy)
        if (k + S < nstream) ring_issue(stage, stream_index(k + S));
        cp_async_commit();
        stage = (stage + 1 == S) ? 0 : stage + 1;
      }
      cp_async_wait_pending(0);
    }
    // streamed tiles, register path (the first one is already in registers)
    for (int64_t k = 0; !ring && k < nstream; ++k) {
      const int64_t i = stream_index(k);
      const int64_t base = (blockIdx.x + i * (int64_t)W) * tile + tid;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (!ok[u]) continue;
        const int64_t g = base + (int64_t)u * kBlock;
        if (PACKED && first) {
          st_stream4_p(a.u + 4 * g, reg[0][u], pol_keep);
          st_stream4_p(a.v + 4 * g, reg[1][u], pol_keep);
        }
        float l = 0.f;
#pragma unroll
        for (int q = 0; q < 4; ++q)
          l += row_loss(f4at(reg[0][u], q), f4at(reg[1][u], q), f4at(reg[NARR - 1][u], q), coef);
        acc += (double)l;
      }
      if (k + 1 < nstream) load_tile(stream_index(k + 1), first || !PACKED);
    }
    // resident tiles: filled in the first evaluation, served from shared memory afterwards
    for (int64_t i = 0; i < R; ++i) {
      float4* st = s_tiles + (size_t)i * NARR * U * kBlock;
      if (first) {
        load_tile(i, true);
#pragma unroll
        for (int u = 0; u < U; ++u) {
#pragma unroll
          for (int c = 0; c < NARR; ++c)
            if (ok[u]) st[(c * U + u) * kBlock + tid] = reg[c][u];
        }
      } else {
        const int64_t base = (blockIdx.x + i * (int64_t)W) * tile + tid;
#pragma unroll
        for (int u = 0; u < U; ++u) {
          ok[u] = base + (int64_t)u * kBlock < n4;
#pragma unroll
          for (int c = 0; c < NARR; ++c)
            if (ok[u]) reg[c][u] = st[(c * U + u) * kBlock + tid];
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (!ok[u]) continue;
        float l = 0.f;
#pragma unroll
        for (int q = 0; q < 4; ++q)
          l += row_loss(f4at(reg[0][u], q), f4at(reg[1][u], q), f4at(reg[NARR - 1][u], q), coef);
        acc += (double)l;
      }
    }
    if (blockIdx.x == 0 && tid < (a.n & 3)) {  // scalar tail (n % 4 rows), always from the source arrays
      const int64_t j = (n4 << 2) + tid;
      if constexpr (PACKED) {
        const float ye = signed_scale<LOSS>(a.y[j]);
        acc += (double)row_loss(ye * a.F[j], ye * a.h[j], 0.f, coef);
      } else {
        acc += (double)row_loss(a.y[j], a.F[j], a.h[j], coef);
      }
    }
    acc = warp_sum(acc);
    if (lane == 0) s_red[warp] = acc;
    __syncthreads();
    if (warp == 0) {
      double v = (lane < kBlock / 32) ? s_red[lane] : 0.0;
      v = warp_sum(v);
      if (lane == 0) {
        a.partials[blockIdx.x] = v;
        __threadfence();
        red_release_gpu_add_u32(&a.sync->arrive, 1u);
      }
    }
    __syncthreads();  // s_red / s_x / s_cmd are reused by the next evaluation
  }
}

template <int LOSS>
cudaError_t launch_ls(const LsArgs& a0, int sms, const LsLaunch& cfg, cudaStream_t st, int* workers_out) {
  using T = LsTraits<LOSS>;
  auto kern = gbm_linesearch_persist_kernel<LOSS>;
  // function attributes are per DEVICE: a process that drives several GPUs (sharded.ShardedContext, a JVM executor with
  // `devices`) must opt in to the large dynamic shared memory on each of them
  constexpr int kMaxDev = 64;
  static int max_smem_dev[kMaxDev];
  static int blocks_full_dev[kMaxDev];
  static size_t smem_cap_dev[kMaxDev];
  static bool ready_dev[kMaxDev] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDev) return cudaErrorInvalidDevice;
  int& max_smem = max_smem_dev[dev];
  int& blocks_full = blocks_full_dev[dev];
  size_t& smem_cap = smem_cap_dev[dev];
  if (!ready_dev[dev]) {
    int optin = 0;
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, kern);
    if (e != cudaSuccess) return e;
    // static + dynamic shared memory together must stay within the opt-in limit
    const int dyn_max = optin - (int)fa.sharedSizeBytes;
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_max);
    if (e != cudaSuccess) return e;
    max_smem = dyn_max;
    // co-resident CTAs per SM are bounded by registers / threads (4 by __launch_bounds__): share the SM's shared
    // memory between them
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_full, kern, kBlock, 0);
    if (e != cudaSuccess) return e;
    if (blocks_full < 1) return cudaErrorLaunchOutOfResources;
    int per_sm = 0;
    cudaDeviceGetAttribute(&per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
    smem_cap = (size_t)per_sm;
    ready_dev[dev] = true;
  }
  LsArgs a = a0;
  int per_sm_ctas = blocks_full > cfg.max_ctas_per_sm ? cfg.max_ctas_per_sm : blocks_full;
  if (per_sm_ctas < 1) per_sm_ctas = 1;
  const int64_t ntiles = ((a.n >> 2) + (int64_t)kBlock * T::kU - 1) / ((int64_t)kBlock * T::kU);
  int64_t workers = (int64_t)per_sm_ctas * sms - 1;
  if (workers > ntiles) workers = ntiles;
  if (workers < 1) workers = 1;
  if (workers > kMaxGridPartials) workers = kMaxGridPartials;
  // shared-memory budget per CTA: the SM's capacity split between the co-resident CTAs (1 KB reserved per CTA)
  int64_t budget = (int64_t)smem_cap / per_sm_ctas - 1024 - 256;
  if (budget > max_smem) budget = max_smem;
  const int64_t per_cta = (ntiles + workers - 1) / workers;
  // ring stages for the tiles that do not stay resident: none when every tile of a worker fits in shared memory,
  // else cfg.ring as far as the budget allows; what is left of the budget holds resident tiles.  Off by default:
  // the ring costs resident tiles on small shards.
  const int64_t tb = T::kTileBytes;
  int ring = 0;
  if (per_cta > (cfg.resident ? budget / tb : 0)) {
    ring = cfg.ring < 0 ? 0 : (cfg.ring > 4 ? 4 : cfg.ring);
    if (ring == 1) ring = 2;
    if ((int64_t)ring * tb > budget) ring = (int)(budget / tb);
    if (ring < 2) ring = 0;
  }
  int64_t resident = cfg.resident ? (budget - (int64_t)ring * tb) / tb : 0;
  if (resident > per_cta) resident = per_cta;
  if (resident < 0) resident = 0;
  a.resident_tiles = (int)resident;
  a.ring_stages = ring;
  const size_t dyn = (size_t)(resident + ring) * T::kTileBytes;
  // the occupancy with this much dynamic shared memory must still cover the grid (cooperative launch would fail)
  int blocks = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, kern, kBlock, dyn);
  if (e != cudaSuccess) return e;
  if ((int64_t)blocks * sms < workers + 1) return cudaErrorCooperativeLaunchTooLarge;
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3((unsigned)(workers + 1));
  lc.blockDim = dim3(kBlock);
  lc.dynamicSmemBytes = dyn;
  lc.stream = st;
  cudaLaunchAttribute attrs[2];
  int na = 0;
  attrs[na].id = cudaLaunchAttributeCooperative;
  attrs[na].val.cooperative = 1;
  ++na;
  if (cfg.window_bytes > 0 && cfg.window_base != nullptr) {
    attrs[na].id = cudaLaunchAttributeAccessPolicyWindow;
    attrs[na].val.accessPolicyWindow.base_ptr = cfg.window_base;
    attrs[na].val.accessPolicyWindow.num_bytes = cfg.window_bytes;
    attrs[na].val.accessPolicyWindow.hitRatio = cfg.hit_ratio;
    attrs[na].val.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    attrs[na].val.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    ++na;
  }
  lc.attrs = attrs;
  lc.numAttrs = na;
  if (workers_out) *workers_out = (int)workers;
  return cudaLaunchKernelEx(&lc, kern, a);
}

}  // namespace

cudaError_t launch_gbm_round_sq_fused(const SqRoundArgs& a0, int write_r, int loss_reduce, int resident, int sms,
                                      int max_ctas_per_sm, cudaStream_t st, int* grid_out, int* resident_slots_out,
                                      void* window_base, size_t window_bytes) {
  constexpr int kKerns = 6;
  void (*kerns[kKerns])(const SqRoundArgs) = {
      gbm_round_sq_fused_kernel<false, false, false>, gbm_round_sq_fused_kernel<false, true, false>,
      gbm_round_sq_fused_kernel<true, false, false>,  gbm_round_sq_fused_kernel<true, true, false>,
      gbm_round_sq_fused_kernel<true, false, true>,   gbm_round_sq_fused_kernel<true, true, true>};
  const bool from_r = write_r && a0.stats_from_r && a0.bag == nullptr;
  const int which = from_r ? 4 + (loss_reduce ? 1 : 0) : (write_r ? 2 : 0) + (loss_reduce ? 1 : 0);
  // function attributes and occupancy are per DEVICE (a process may drive several GPUs, as in launch_ls)
  constexpr int kMaxDev = 64;
  struct KernInfo {
    int blocks, max_dyn, static_smem;
    // occupancy at the dynamic size of the last launch: consecutive rounds repeat it, and on small shards the host
    // must issue the next launch within the current round's update phase
    size_t dyn_checked;
    int blocks_dyn;
    bool ready;
  };
  static KernInfo info_dev[kMaxDev][kKerns] = {};
  static int smem_per_sm_dev[kMaxDev];
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDev) return cudaErrorInvalidDevice;
  KernInfo& info = info_dev[dev][which];
  if (!info.ready) {
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, kerns[which]);
    if (e != cudaSuccess) return e;
    info.static_smem = (int)fa.sharedSizeBytes;
    info.max_dyn = 0;
    if (which >= 4) {  // the carry-over sizes its dynamic shared memory past the default 48 KB
      int optin = 0;
      cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
      info.max_dyn = optin - info.static_smem;
      e = cudaFuncSetAttribute(kerns[which], cudaFuncAttributeMaxDynamicSharedMemorySize, info.max_dyn);
      if (e != cudaSuccess) return e;
    }
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&info.blocks, kerns[which], kBlock, 0);
    if (e != cudaSuccess) return e;
    cudaDeviceGetAttribute(&smem_per_sm_dev[dev], cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
    info.ready = true;
  }
  int per_sm = info.blocks;
  if (per_sm > max_ctas_per_sm) per_sm = max_ctas_per_sm;
  if (per_sm < 1) return cudaErrorLaunchOutOfResources;
  const int64_t ntiles = ((a0.n >> 2) + (int64_t)kBlock * U_SQ - 1) / ((int64_t)kBlock * U_SQ);
  int64_t grid = (int64_t)per_sm * sms;
  if (grid > ntiles) grid = ntiles;
  if (grid < 1) grid = 1;
  if (grid > kMaxGridPartials / 2) grid = kMaxGridPartials / 2;
  // carried slots per CTA: the SM's shared memory split between its co-resident CTAs (1 KB per CTA is reserved by
  // the system), and no more than the busiest CTA has groups before its last tile
  int64_t slots = 0;
  if (from_r && resident) {
    int64_t budget = (int64_t)smem_per_sm_dev[dev] / per_sm - 1024 - info.static_smem;
    if (budget > info.max_dyn) budget = info.max_dyn;
    slots = budget / kSqSlotBytes;
    const int64_t per_cta = (ntiles + grid - 1) / grid;
    if (slots > (per_cta - 1) * U_SQ) slots = (per_cta - 1) * U_SQ;
    if (slots < 0) slots = 0;
  }
  const size_t dyn = (size_t)slots * kSqSlotBytes;
  if (dyn > 0) {  // the whole grid must still be co-resident with this much shared memory per CTA
    if (dyn != info.dyn_checked) {
      cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&info.blocks_dyn, kerns[which], kBlock, dyn);
      if (e != cudaSuccess) return e;
      info.dyn_checked = dyn;
    }
    if ((int64_t)info.blocks_dyn * sms < grid) return cudaErrorCooperativeLaunchTooLarge;
  }
  SqRoundArgs a = a0;
  a.resident_slots = (int)slots;
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3((unsigned)grid);
  lc.blockDim = dim3(kBlock);
  lc.dynamicSmemBytes = dyn;
  lc.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;  // co-residency of all CTAs is what makes the in-kernel flag wait deadlock-free
  int na = 1;
  if (window_base != nullptr && window_bytes > 0) {
    attr[na].id = cudaLaunchAttributeAccessPolicyWindow;
    attr[na].val.accessPolicyWindow.base_ptr = window_base;
    attr[na].val.accessPolicyWindow.num_bytes = window_bytes;
    attr[na].val.accessPolicyWindow.hitRatio = 1.0f;
    attr[na].val.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    attr[na].val.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    ++na;
  }
  lc.attrs = attr;
  lc.numAttrs = na;
  if (grid_out) *grid_out = (int)grid;
  if (resident_slots_out) *resident_slots_out = (int)slots;
  return cudaLaunchKernelEx(&lc, kerns[which], a);
}

bool gbm_linesearch_persist_supported(int loss) {
  switch (loss) {
    case SE_LOSS_ABSOLUTE: case SE_LOSS_HUBER: case SE_LOSS_QUANTILE: case SE_LOSS_LOGCOSH:
    case SE_LOSS_SCALED_LOGCOSH: case SE_LOSS_BERNOULLI: case SE_LOSS_EXPONENTIAL: return true;
    default: return false;
  }
}

bool gbm_linesearch_persist_packed(int loss) { return loss == SE_LOSS_BERNOULLI || loss == SE_LOSS_EXPONENTIAL; }

cudaError_t launch_gbm_linesearch_persist(int loss, const LsArgs& a, int sms, const LsLaunch& cfg, cudaStream_t st,
                                          int* workers_out) {
  switch (loss) {
    case SE_LOSS_ABSOLUTE: return launch_ls<SE_LOSS_ABSOLUTE>(a, sms, cfg, st, workers_out);
    case SE_LOSS_HUBER: return launch_ls<SE_LOSS_HUBER>(a, sms, cfg, st, workers_out);
    case SE_LOSS_QUANTILE: return launch_ls<SE_LOSS_QUANTILE>(a, sms, cfg, st, workers_out);
    case SE_LOSS_LOGCOSH: return launch_ls<SE_LOSS_LOGCOSH>(a, sms, cfg, st, workers_out);
    case SE_LOSS_SCALED_LOGCOSH: return launch_ls<SE_LOSS_SCALED_LOGCOSH>(a, sms, cfg, st, workers_out);
    case SE_LOSS_BERNOULLI: return launch_ls<SE_LOSS_BERNOULLI>(a, sms, cfg, st, workers_out);
    case SE_LOSS_EXPONENTIAL: return launch_ls<SE_LOSS_EXPONENTIAL>(a, sms, cfg, st, workers_out);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace se
