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
//    F = y - r.  The host marks F as owed and rebuilds it from y and r when F is next accessed (se_api_ctx.cu settle_f).
//    A round whose residual slot is not current (Y, F or R were just written) reads (y, F, h) instead of (r, h):
//    r' = (y - F) - c h, 16 B/row.  Without residual mode the update is F' = F + c h (F, y, h read; F written).
//    A residual round without a bag also sums the statistics of (r', h) in its update pass, one partial per CTA;
//    while R and H stay as it left them, the next round folds those partials and skips the statistics pass
//    (12 B/row).  On one GPU every CTA of that carried round folds them and runs Brent itself: no CTA waits for
//    another, and the round is launched as a programmatic dependent that starts while the round before it drains.
//    Such a carried round may also leave R pending (se_api_ctx.cu settle_r): it stores nothing (8 B/row), and the
//    Brent thread appends its fp32 step to a chain on the device.  The next carried round reads the older r0 and
//    applies the chain in registers, t = fmaf(-c_j, h, t), before its own step -- the fmaf a storing round applies,
//    so every r it sums its statistics over, and the r it stores when the chain reaches the context's cap, is the one
//    the storing rounds would have left, bit for bit.
//
//  * gbm_linesearch_persist_kernel — Brent's <= MaxEval evaluations of the line-search objective
//    (boosting/GBMLoss.scala:50-74 through RDDLossFunction; GBMRegressor.scala:408-421) for the non-squared scalar
//    losses in ONE launch: worker CTAs own a fixed set of tiles, keep the first of them in SHARED MEMORY for the whole
//    search (132 SMs x ~190 KB = 25 MB on an H100 that never touch HBM again) and stream the rest; a coordinator
//    warp folds the per-CTA partials in a fixed order, performs the cross-GPU sum, advances Brent and publishes the
//    next abscissa.  The first evaluation of the binary losses also BUILDS the
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

__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ double global_timer_us() { return (double)global_timer_ns() * 1e-3; }
// bulk L2 prefetch of a contiguous global range (bytes: multiple of 16, address 16 B aligned)
__device__ __forceinline__ void prefetch_l2_bulk(const void* p, unsigned int bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}

// =================================================================================== squared-loss round, one launch
constexpr int U_SQ = 4;  // float4 groups per thread per tile (as the two-launch kernels)
// Residual-mode rounds that read r (no bag) carry phase A's tail into phase B on chip: the CTA's last tile stays in
// registers and the groups before it in shared memory, one slot per float4 group of r and of h (8 KB per CTA), so
// that a slot, not a whole 32 KB tile, is the unit the SM's shared memory is split into.
constexpr int kSqSlotBytes = 2 * kBlock * 16;

// The line search of the fused round, executed by ONE thread once the statistics s0, s1, s2 are folded (and summed
// across GPUs): by the last CTA while every other CTA waits for the step with its first update tile's loads in flight,
// or, in a carried round on one GPU, by every CTA for itself.  Returns the step.  `serve`: this thread also writes the
// round's results (out[4..8], the host mirror and its ticket) and appends a deferring round's step to the chain;
// `release`: it hands the step to the grid through a.sync.
template <bool LOSS_REDUCE>
__device__ __forceinline__ double fused_round_brent(const SqRoundArgs& a, double s0, double s1, double s2, bool serve,
                                                    bool release) {
  if (a.timing && serve) a.out[11] = global_timer_us();  // statistics folded (and summed across GPUs)
  const BrentParabola f{s0, s1, s2, a.wsum};
  double x = 1.0, fx = 0.0;
  int evals = 0;
  const int rc = brent_core(f, a.lo, a.hi, a.start, a.rel, a.abs_tol, a.max_eval, &x, &fx, &evals);
  // MaxEval exceeded: the host reports SE_ERR_OPT and F must stay what it was (r - 0*h == r, F + 0*h == F; the host
  // does not mark F as owed)
  const double step = (rc == kBrentOk) ? a.lr * x : 0.0;
  if (!serve) return step;
  const double ne = (rc == kBrentOk) ? (double)evals : -(double)evals;  // negative: MaxEval exceeded
  a.out[4] = x, a.out[5] = fx, a.out[6] = ne;
  // a deferring round's step, as phase B rounds it, joins the pending chain (a 0 step too: fmaf(-0, h, r) is what
  // the stored round applies)
  if (a.r_defer) a.r_chain[a.r_pending] = (float)step;
  if (release) {
    a.sync->x = step;
    st_release_gpu_u64(&a.sync->flag, a.epoch);  // the grid starts the update NOW; the host is served next
  }
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
  return step;
}

__device__ __forceinline__ void cp_async16(float4* smem, const float* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem)), "l"(gmem)
               : "memory");
}

// FROM_R (a fit's round after a new direction: residual mode, the residual slot current, no bag) is a compile-time
// specialisation: it carries phase A's tail into phase B on chip (kSqSlotBytes) and has no y / F / bag arrays live.
// CARRIED (the rounds after it over the same direction) has no phase A at all: the previous round's update pass left
// each CTA's partial statistics of (r, h) in a.carry_in.  They are folded and Brent runs while every CTA has its first
// update tile in registers and, with resident slots, the groups after it in flight to shared memory.  Across GPUs
// CTA 0 folds, sums across GPUs, runs Brent and publishes the step to the others (a cooperative launch).  On one GPU
// every CTA folds the same partials in the same order and runs Brent itself, so no CTA waits for another: the launch
// is an ordinary one, a programmatic dependent of the kernel before it (griddepcontrol), and CTA 0 alone serves the
// host and the chain.
// Residual rounds whose loss comes from the statistics (STATS_OUT) store the next round's partial statistics in
// phase B.
template <bool WRITE_R, bool LOSS_REDUCE, bool FROM_R, bool CARRIED>
__global__ void __launch_bounds__(kBlock, 3) gbm_round_sq_fused_kernel(const SqRoundArgs a) {
  static_assert(WRITE_R || !FROM_R, "FROM_R is a residual-mode round");
  static_assert(!CARRIED || (WRITE_R && !LOSS_REDUCE && !FROM_R), "CARRIED is a residual round without a bag");
  constexpr bool STATS_OUT = WRITE_R && !LOSS_REDUCE;
  constexpr int U = U_SQ;
  extern __shared__ float4 s_res[];  // FROM_R, CARRIED: [slot][r, h][kBlock]
  __shared__ float s_coef;
  __shared__ bool s_store_r;
  __shared__ double s_stats[3];  // CARRIED: the folded statistics
  __shared__ float s_chain[kSqDeferMax];  // CARRIED: the steps pending on the residual slot
  __shared__ float4 s_brent_regs[2 * U];  // FROM_R, CARRIED: the Brent thread's tile registers while it runs Brent
  const int64_t n4 = a.n >> 2;
  constexpr int64_t tile = (int64_t)kBlock * U;
  const int64_t ntiles = (n4 + tile - 1) / tile;
  const int64_t G = gridDim.x;
  const int64_t cnt = (ntiles > (int64_t)blockIdx.x) ? (ntiles - 1 - blockIdx.x) / G + 1 : 0;  // tiles b, b+G, ...
  const bool has_bag = !FROM_R && !CARRIED && (a.bag != nullptr);
  const bool stats_from_r = FROM_R || CARRIED || a.stats_from_r;
  // Phase B's k-th tile is i = cnt-1-k (downwards, from where phase A ended), or i = k on a carried round that walks
  // upwards.  FROM_R: group u of tile i has the flat index i*U + u.  The last tile (cnt-1) stays in registers, the S
  // groups before it in shared memory: every group from p_res on is carried to phase B.  CARRIED: the first tile is
  // in registers and the S groups after it, in phase B's order, in shared memory.
  const bool up = CARRIED && a.forward;
  const int64_t S = (FROM_R || CARRIED) ? min((int64_t)a.resident_slots, (cnt > 0 ? cnt - 1 : 0) * U) : 0;
  const int64_t p_res = (cnt - 1) * U - S;
  auto slot_of = [&](int64_t k, int64_t i, int u) -> int64_t {  // shared-memory slot of a phase-B group, or -1
    if constexpr (FROM_R) return i * U + u - p_res;
    if constexpr (CARRIED) return (k >= 1 && (k - 1) * U + u < S) ? (k - 1) * U + u : -1;
    return -1;
  };
  const uint64_t pol_stream = l2_policy(a.l2_hints != 0);
  const uint64_t pol_keep = l2_policy(false);
  // carried groups are served from chip in phase B: their L2 lines go first, so that the L2 keeps the groups before
  // them, which phase B reads next
  const uint64_t pol_carried = l2_policy(true);

  if (a.timing && blockIdx.x == 0 && threadIdx.x == 0) a.out[10] = global_timer_us();
  if (a.kstamp && blockIdx.x == 0 && threadIdx.x == 0) a.kstamp[0] = global_timer_ns();
  // phase B's tile registers.  FROM_R: phase A loads into them, so that its last tile is where phase B starts; the
  // other rounds keep phase A's tiles local, so that nothing is live across the wait but what phase B loads.
  float4 vy[U], vF[U], vh[U];  // from_r: vy holds r and vF is unused
  bool ok[U];
  // the Brent thread parks the tile registers in shared memory meanwhile: Brent needs more registers than are left
  // beside them, and local memory would be the alternative
  auto run_brent = [&](const double* s, bool serve, bool release) {
    if constexpr (FROM_R || CARRIED) {
#pragma unroll
      for (int u = 0; u < U; ++u) s_brent_regs[u] = vy[u], s_brent_regs[U + u] = vh[u];
    }
    s_coef = (float)fused_round_brent<LOSS_REDUCE>(a, s[0], s[1], s[2], serve, release);
    if constexpr (FROM_R || CARRIED) {
#pragma unroll
      for (int u = 0; u < U; ++u) vy[u] = s_brent_regs[u], vh[u] = s_brent_regs[U + u];
    }
  };
  const bool from_r = WRITE_R && stats_from_r;
  auto load_tile = [&](int64_t k) {
    const int64_t i = up ? k : cnt - 1 - k;
    const int64_t base = (blockIdx.x + i * G) * tile + threadIdx.x;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t g = base + (int64_t)u * kBlock;
      ok[u] = g < n4;
      if (ok[u]) {
        const int64_t s = slot_of(k, i, u);
        if ((FROM_R || CARRIED) && s >= 0) {
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
        vh[u] = ld_stream4_p(a.h + 4 * g, pol_stream);  // the update is h's last reader
      }
    }
  };

  // CARRIED: the pending steps, read before the Brent thread appends this round's (the barrier before phase B
  // publishes them).  The count and the store flag are read from the kernel parameters where they are used: kept in
  // registers they would spill.
  const bool solo = CARRIED && (a.ws_a.nranks <= 1 || a.ws_a.mbox == nullptr);
  if constexpr (CARRIED) {
    // the first tile into registers, the S groups after it into shared memory (each thread copies, and in phase B
    // reads back, only its own slots: no barrier)
    auto prologue = [&]() {
      if (cnt > 0) load_tile(0);
      for (int64_t s = 0; s < S; ++s) {
        const int64_t k = 1 + s / U, i = up ? k : cnt - 1 - k;
        const int64_t g = (blockIdx.x + i * G) * tile + threadIdx.x + (s % U) * (int64_t)kBlock;
        if (g < n4) {
          cp_async16(&s_res[(2 * s) * kBlock + threadIdx.x], a.r + 4 * g);
          cp_async16(&s_res[(2 * s + 1) * kBlock + threadIdx.x], a.h + 4 * g);
        }
      }
    };
    // On one GPU this kernel may start while the one before it still runs (programmatic dependent launch): until
    // griddepcontrol.wait returns, it reads nothing but h, which nothing between two carried rounds writes, and r
    // when the host says R has not been written since the last deferring round.  Everything the kernel before it
    // writes (r', the chain, the partials, the results) is read after the wait.  A CTA lets the next kernel start only
    // once its own wait has returned, so that kernel cannot begin before this one's predecessor has completed.
    if (a.r_early) prologue();
    if (solo) {
      asm volatile("griddepcontrol.wait;" ::: "memory");
      asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    }
    if (!a.r_early) prologue();
    for (int j = threadIdx.x; j < a.r_pending; j += kBlock) s_chain[j] = a.r_chain[j];
    if (solo) {
      // the statistics, bit for bit as CTA 0 would fold them, and the step, in every CTA
      fold_partials<3>(a.carry_in, (unsigned)a.carry_grid, s_stats);
      if (blockIdx.x == 0 && threadIdx.x < 3) a.out[threadIdx.x] = s_stats[threadIdx.x];
      if (threadIdx.x == 0) run_brent(s_stats, blockIdx.x == 0, false);
    } else if (blockIdx.x == 0) {
      fold_partials<3>(a.carry_in, (unsigned)a.carry_grid, s_stats);
      peer_exchange(s_stats, 3, a.ws_a);  // this GPU's statistics -> a.out[0..2], summed across GPUs
      __syncthreads();
      if (threadIdx.x == 0) run_brent(a.out, true, true);
    }
  } else {
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
          vy[u] = ld_rw4_p(a.r + 4 * g, carried ? pol_carried : pol_stream);
          vh[u] = ld_stream4_p(a.h + 4 * g, carried ? pol_carried : pol_keep);
        } else {
          if (stats_from_r) {
            vy[u] = ld_rw4_p(a.r + 4 * g, pol_stream);  // read again and rewritten by phase B
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
    if (threadIdx.x == 0) run_brent(a.out, true, true);
  }
  // in flight while the last CTA reduces, exchanges and runs Brent (FROM_R: still in registers from phase A)
  if (!FROM_R && cnt > 0) load_tile(0);
  }  // phase A

  // ---- phase B, tiles in the opposite direction.  WRITE_R (residual mode): r' = r - step*h, Σ r'²/2; F is not
  // touched (the host rebuilds it as y - r' when it is next accessed), or r' = (y - F) - step*h on a round whose
  // residual slot is not current.  Otherwise: F' = F + step*h, Σ (y-F')²/2.  The order of the tiles, and so of the
  // loss sum, is the same whether a tile comes from registers, shared memory or global memory.
  if (threadIdx.x == 0) {
    if constexpr (FROM_R) {
      // nothing of the carried tail is loaded: while the grid waits for the step, the first tile phase B reads from
      // global memory (its groups below p_res) is pulled into the L2 with bulk prefetches of r and h
      const int64_t pf = p_res > 0 ? (p_res - 1) / U : -1;
      if (pf >= 0) {
        const int64_t g0 = (blockIdx.x + pf * G) * tile;
        int64_t groups = (p_res - pf * U) * kBlock;
        if (groups > n4 - g0) groups = n4 - g0;
        if (groups > 0) {
          prefetch_l2_bulk(a.r + 4 * g0, (unsigned int)(groups * 16));
          prefetch_l2_bulk(a.h + 4 * g0, (unsigned int)(groups * 16));
        }
      }
    }
    if (!solo) {  // on one GPU a carried round's thread 0 computed the step itself
      while (ld_acquire_gpu_u64(&a.sync->flag) != a.epoch) {}
      s_coef = (float)a.sync->x;  // same rounding as the host path: (float)(lr * alpha)
    }
    // MaxEval exceeded on a round that read y and F: its residual slot was not current, and the failed round must
    // leave it as it was rather than store y - F (the Brent thread wrote the count before it released the step)
    s_store_r = !(WRITE_R && !from_r && a.out[6] < 0.0);
  }
  if constexpr (CARRIED) asm volatile("cp.async.wait_all;" ::: "memory");  // this thread's slots have landed
  __syncthreads();
  const float coef = s_coef;
  const bool store_r = s_store_r;
  double accb[1] = {0.0};
  double accn[3] = {0.0, 0.0, 0.0};  // STATS_OUT: Σr'², Σhr', Σh² over what this pass writes, as phase A sums them
  for (int64_t k = 0; k < cnt; ++k) {
    const int64_t i = up ? k : cnt - 1 - k;
    const int64_t base = (blockIdx.x + i * G) * tile + threadIdx.x;
    if constexpr (CARRIED) {
      // the pending steps, in the order the rounds took them: the r each of them would have stored and the next read
      for (int j = 0; j < a.r_pending; ++j) {
        const float c = s_chain[j];
#pragma unroll
        for (int u = 0; u < U; ++u) {
#pragma unroll
          for (int e = 0; e < 4; ++e) f4at(vy[u], e) = fmaf(-c, f4at(vh[u], e), f4at(vy[u], e));
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t g = base + (int64_t)u * kBlock;
      // CARRIED: the bound is tested again rather than kept from the load, which leaves the chain's registers free
      if (CARRIED ? g >= n4 : !ok[u]) continue;
      float4 o;
      float l_acc = 0.f, s0 = 0.f, s1 = 0.f, s2 = 0.f;
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
        if (STATS_OUT) {
          const float h = f4at(vh[u], e);
          s0 = fmaf(d, d, s0);
          s1 = fmaf(h, d, s1);
          s2 = fmaf(h, h, s2);
        }
      }
      // the next statistics pass starts where this one ends; a deferring round stores nothing
      if (WRITE_R) {
        if ((!CARRIED || !a.r_defer) && store_r) st_stream4_p(a.r + 4 * g, o, pol_keep);
      } else {
        st_stream4_p(a.F + 4 * g, o, pol_stream);
      }
      if (LOSS_REDUCE) accb[0] += (double)l_acc;
      if (STATS_OUT) accn[0] += (double)s0, accn[1] += (double)s1, accn[2] += (double)s2;
    }
    if (k + 1 < cnt) load_tile(k + 1);
  }
  if (blockIdx.x == 0 && threadIdx.x < (a.n & 3)) {
    const int64_t j = (n4 << 2) + threadIdx.x;
    float d;
    if constexpr (WRITE_R) {
      const float h = a.h[j];
      float r = from_r ? a.r[j] : a.y[j] - a.F[j];
      if constexpr (CARRIED)
        for (int q = 0; q < a.r_pending; ++q) r = fmaf(-s_chain[q], h, r);
      d = fmaf(-coef, h, r);
      if ((!CARRIED || !a.r_defer) && store_r) a.r[j] = d;
    } else {
      const float p = fmaf(coef, a.h[j], a.F[j]);
      d = a.y[j] - p;
      a.F[j] = p;
    }
    accb[0] += (double)(0.5f * d * d);
    if (STATS_OUT) {
      const float h = a.h[j];
      accn[0] += (double)(d * d), accn[1] += (double)(h * d), accn[2] += (double)(h * h);
    }
  }
  if constexpr (LOSS_REDUCE) {
    const bool last_b = block_reduce_publish<1>(accb, a.ws_b);  // Σloss -> a.ws_b.out (+ cross-GPU sum, host mirror + ticket)
    if (a.timing && last_b && threadIdx.x == 0) a.out[13] = global_timer_us();
  } else {
    // the next round's statistics, this GPU's, as one partial per CTA.  A carried round stores them into the other of
    // the context's two buffers than the one it folded, which its slower CTAs may still be reading.
    if constexpr (STATS_OUT) block_reduce_store<3>(accn, a.carry_out);
    if (a.timing) {
      // the loss came from the statistics: the latest stamp of any CTA marks the end of the update
      __syncthreads();
      if (threadIdx.x == 0) atomicMax(reinterpret_cast<unsigned long long*>(&a.out[13]), (unsigned long long)__double_as_longlong(global_timer_us()));
    }
    if (a.kstamp) {
      __syncthreads();
      if (threadIdx.x == 0) atomicMax(a.kstamp + 1, global_timer_ns());
    }
  }
}

// =================================================================================== persistent line search
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
  extern __shared__ float4 s_tiles[];  // [resident][NARR][U][kBlock]
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
    if (nstream > 0) load_tile(stream_index(0), first || !PACKED);
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
    // streamed tiles (the first one is already in registers)
    for (int64_t k = 0; k < nstream; ++k) {
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
  int64_t resident = cfg.resident ? budget / T::kTileBytes : 0;
  if (resident > per_cta) resident = per_cta;
  if (resident < 0) resident = 0;
  a.resident_tiles = (int)resident;
  const size_t dyn = (size_t)resident * T::kTileBytes;
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
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeCooperative;
  attr.val.cooperative = 1;
  lc.attrs = &attr;
  lc.numAttrs = 1;
  if (workers_out) *workers_out = (int)workers;
  return cudaLaunchKernelEx(&lc, kern, a);
}

}  // namespace

cudaError_t launch_gbm_round_sq_fused(const SqRoundArgs& a0, int write_r, int loss_reduce, int resident, int sms,
                                      int max_ctas_per_sm, cudaStream_t st, int* grid_out, int* resident_slots_out) {
  constexpr int kKerns = 7;
  void (*kerns[kKerns])(const SqRoundArgs) = {
      gbm_round_sq_fused_kernel<false, false, false, false>, gbm_round_sq_fused_kernel<false, true, false, false>,
      gbm_round_sq_fused_kernel<true, false, false, false>,  gbm_round_sq_fused_kernel<true, true, false, false>,
      gbm_round_sq_fused_kernel<true, false, true, false>,   gbm_round_sq_fused_kernel<true, true, true, false>,
      gbm_round_sq_fused_kernel<true, false, false, true>};
  const bool carried = a0.carried != 0;
  if (carried && !(write_r && !loss_reduce && a0.bag == nullptr)) return cudaErrorInvalidValue;
  // only a carried round reads pending steps or defers its own, and the chain holds at most kSqDeferMax of them
  if ((a0.r_pending || a0.r_defer) && !(carried && a0.r_chain)) return cudaErrorInvalidValue;
  if (a0.r_pending < 0 || a0.r_pending + (a0.r_defer ? 1 : 0) > kSqDeferMax) return cudaErrorInvalidValue;
  // a carried round folds the partials of a grid that fit the buffer; a residual round without a bag stores its own
  if (carried && !(a0.carry_in && a0.carry_grid >= 1 && a0.carry_grid <= kMaxGridPartials / 2))
    return cudaErrorInvalidValue;
  if (write_r && !loss_reduce && !a0.carry_out) return cudaErrorInvalidValue;
  // the same test as the kernel's (and peer_exchange's): one GPU, or no peer communicator attached
  const bool solo = a0.ws_a.nranks <= 1 || a0.ws_a.mbox == nullptr;
  // r is read before the kernel before this one is waited for only when that kernel cannot have written it
  if (a0.r_early && !(carried && solo && a0.r_pending > 0)) return cudaErrorInvalidValue;
  if (a0.kstamp && !(carried && solo)) return cudaErrorInvalidValue;
  const bool from_r = !carried && write_r && a0.stats_from_r && a0.bag == nullptr;
  const int which = carried ? 6 : from_r ? 4 + (loss_reduce ? 1 : 0) : (write_r ? 2 : 0) + (loss_reduce ? 1 : 0);
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
    if (which >= 4) {  // the shared-memory carry sizes its dynamic shared memory past the default 48 KB
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
  // the system), and no more than the busiest CTA has groups besides the tile it keeps in registers
  int64_t slots = 0;
  if ((from_r || carried) && resident) {
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
  cudaLaunchAttribute attr;
  if (carried && solo) {
    // no CTA waits for another: the round may start while the kernel before it drains (griddepcontrol in the kernel)
    attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr.val.programmaticStreamSerializationAllowed = 1;
  } else {
    attr.id = cudaLaunchAttributeCooperative;
    attr.val.cooperative = 1;  // co-residency of all CTAs is what makes the in-kernel flag wait deadlock-free
  }
  lc.attrs = &attr;
  lc.numAttrs = 1;
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
