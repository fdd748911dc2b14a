// se_common.cuh — shared device helpers for the sm_90a streaming kernels.
//
// Every kernel on this path is elementwise + reduction and HBM-bound (no tensor cores): the
// helpers here are the 128-bit streaming loads/stores (read-once data bypasses L1 allocation),
// the per-thread -> warp-shuffle -> shared-memory fp64 block reduction, and the deterministic
// cross-block "last block reduces" epilogue that leaves the global sums in a device scalar block
// (consumed in-stream by NCCL or by the next kernel, no host round-trip required).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace se {

constexpr int kBlock = 256;          // threads per CTA for the streaming kernels
constexpr int kMaxGridPartials = 4096;  // upper bound on gridDim.x of reducing kernels
constexpr int kMaxRed = 72;          // max number of fp64 sums one kernel reduces (dim <= 64 -> dim+1)

// ---- 128-bit streaming global accesses ------------------------------------------------------
__device__ __forceinline__ float4 ld_stream4(const float* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}
__device__ __forceinline__ float ld_stream1(const float* p) {
  float v;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
// read-write arrays (F is read then overwritten by the same thread): plain coherent load, no L1 allocation
__device__ __forceinline__ float4 ld_rw4(const float* p) {
  float4 v;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}
__device__ __forceinline__ float ld_rw1(const float* p) {
  float v;
  asm volatile("ld.global.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_stream4(float* p, const float4& v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w)
               : "memory");
}
__device__ __forceinline__ void st_stream1(float* p, float v) {
  asm volatile("st.global.L1::no_allocate.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// ---- the same accesses with an explicit L2 eviction policy (createpolicy + .L2::cache_hint) -----------------
//  * kernels that WRITE per-row results (K1: read y,F,h, write F,r) may carry an explicit evict_normal policy on
//    every access while read-only passes use the plain instructions — so POL is a template flag set per mode;
//  * on shards whose four arrays are of the order of the L2, marking what the next pass does not re-read as
//    evict_first keeps r and h resident between the statistics pass and the update; on shards much larger than the
//    L2 the hints buy nothing, so they are enabled by size (se_api_gbm.cu gbm_args, l2_hint_rows from the device's L2).
__device__ __forceinline__ uint64_t l2_policy(bool evict_first) {
  uint64_t p;
  if (evict_first) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  else asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ float4 ld_stream4_p(const float* p, uint64_t pol) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ float4 ld_rw4_p(const float* p, uint64_t pol) {
  float4 v;
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void st_stream4_p(float* p, const float4& v, uint64_t pol) {
  asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "f"(v.x),
               "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol)
               : "memory");
}

template <bool POL>
__device__ __forceinline__ float4 ld_s4(const float* p, uint64_t pol) {
  if constexpr (POL) return ld_stream4_p(p, pol);
  else return ld_stream4(p);
}
template <bool POL>
__device__ __forceinline__ float4 ld_r4(const float* p, uint64_t pol) {
  if constexpr (POL) return ld_rw4_p(p, pol);
  else return ld_rw4(p);
}
template <bool POL>
__device__ __forceinline__ void st_s4(float* p, const float4& v, uint64_t pol) {
  if constexpr (POL) st_stream4_p(p, v, pol);
  else st_stream4(p, v);
}

__device__ __forceinline__ float& f4at(float4& v, int i) { return (&v.x)[i]; }
__device__ __forceinline__ const float& f4at(const float4& v, int i) { return (&v.x)[i]; }

// ---- fp64 reductions ------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = fmax(v, __shfl_down_sync(0xffffffffu, v, off));
  return v;
}
// max-reduction twin of block_reduce_publish (one value): AdaBoost.R2's maxError
__device__ __forceinline__ void block_max_publish(double v, double* partials, unsigned int* counter,
                                                  double* out) {
  __shared__ double smx[kBlock / 32];
  __shared__ bool last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_max(v);
  if (lane == 0) smx[warp] = v;
  __syncthreads();
  if (warp == 0) {
    double m = (lane < kBlock / 32) ? smx[lane] : -INFINITY;
    m = warp_max(m);
    if (lane == 0) partials[blockIdx.x] = m;
  }
  if (threadIdx.x == 0) {
    __threadfence();
    last = (atomicInc(counter, gridDim.x - 1) == gridDim.x - 1);
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  double m = -INFINITY;
  for (unsigned int b = threadIdx.x; b < gridDim.x; b += kBlock) m = fmax(m, __ldcg(&partials[b]));
  m = warp_max(m);
  if (lane == 0) smx[warp] = m;
  __syncthreads();
  if (warp == 0) {
    double t = (lane < kBlock / 32) ? smx[lane] : -INFINITY;
    t = warp_max(t);
    if (lane == 0) out[0] = t;
  }
}

// Reduction workspace owned by the context: partials[kMaxGridPartials][nred], a self-resetting
// ticket counter, and the output scalar block.  With a peer-memory communicator attached (nranks > 1,
// mbox != nullptr) the kernel that reduces ALSO performs the cross-GPU sum itself (see peer_exchange).
constexpr int kMboxPayload = 72;   // totals per mailbox row (>= kMaxRed); also the width of the host mirror
constexpr int kMboxStride = 160;   // 64-bit words per row: two flagged packets per total (144) + padding (1280 B)
struct RedWs {
  double* partials;
  unsigned int* counter;
  double* out;  // [nred] sums: per-GPU, or global when the peer exchange is active
  // ---- fused NVLink all-reduce (one process per GPU, mailboxes mapped with CUDA IPC)
  double* const* mbox = nullptr;   // device table [nranks]: base of every rank's mailbox [nranks][2][kMboxStride]
  int nranks = 1, rank = 0;
  unsigned long long seq = 0;      // reduction sequence number (same on every rank), >= 1
  int* err = nullptr;              // set to 1 if a peer never showed up (bounded spin) or poisoned the reduction
  long long timeout_clocks = 0;    // spin bound of the peer exchange in SM clocks (0 = wait forever)
  // ---- label validation (Classifier.validateLabel / GBMLoss.scala:200-204 `res(label.toInt) = 1.0` throws on the JVM):
  // kernels that use a label as a class index set this flag (mapped host memory) instead of indexing out of bounds
  int* bad_label = nullptr;
  // ---- host mirror: the final sums are also stored into mapped pinned host memory, followed by a ticket, so
  // the host can pick them up by polling one cache line instead of a D2H copy + stream synchronisation
  double* host_out = nullptr;
  volatile unsigned long long* host_flag = nullptr;
  unsigned long long host_ticket = 0;
};

__device__ __forceinline__ void st_release_sys_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_sys_f64(double* p, double v) {
  asm volatile("st.relaxed.sys.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
__device__ __forceinline__ double ld_relaxed_sys_f64(const double* p) {
  double v;
  asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}

// Cross-GPU sum of `nred` per-GPU totals, executed by ONE WARP (all 32 lanes converged) — the collective is part
// of the reducing kernel, not a separate NCCL launch.  Mailbox rows are written in 8-BYTE PACKETS that carry their own
// validity flag (the low-latency protocol NCCL calls LL): every fp64 total travels as two 64-bit words
// {low 32 bits, flag} and {high 32 bits, flag}, flag = the reduction's sequence number (31 bits).  An aligned 8-byte
// store is single-copy atomic, so a receiver that sees the flag has the data — NO release/acquire fence pair, no
// separate "ready" word, one NVLink hop:
//   1. lane p < nranks stores this GPU's packets into rank p's mailbox row [my rank][seq parity] (plain relaxed
//      system-scope P2P stores over NVLink);
//   2. lane k < nred then polls its OWN mailbox, rank by rank, until both packets of total k carry this sequence
//      (bounded by ws.timeout_clocks; 0 = unbounded), and adds the values in rank order: bit-identical sums on every GPU;
//      emit(k, sum_k) is called by lane k % 32.
// Rows are double-buffered by sequence parity: a peer can be at most one reduction ahead.
// Failure protocol: a rank that gives up (timeout) or meets a poisoned packet overwrites ITS packets in every peer's
// mailbox with the poison flag (seq | 0x80000000), so that a late peer fails the SAME reduction instead of completing it
// with a sum its partners never saw; every rank then reports NaN sums + the sticky error flag (-> SE_ERR_NCCL).
constexpr unsigned int kPoisonFlag = 0x80000000u;
__device__ __forceinline__ void st_relaxed_sys_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
template <class Emit>
__device__ __forceinline__ bool peer_allreduce_warp(const double* tot, int nred, const RedWs& ws, Emit emit) {
  const int lane = threadIdx.x & 31;
  const int par = (int)(ws.seq & 1ull);
  const unsigned int flag = (unsigned int)(ws.seq & 0x7fffffffull);
  for (int p = lane; p < ws.nranks; p += 32) {
    unsigned long long* row = reinterpret_cast<unsigned long long*>(ws.mbox[p]) + (size_t)(ws.rank * 2 + par) * kMboxStride;
    for (int k = 0; k < nred; ++k) {
      const unsigned long long bits = (unsigned long long)__double_as_longlong(tot[k]);
      st_relaxed_sys_u64(row + 2 * k, ((bits & 0xffffffffull) << 32) | flag);
      st_relaxed_sys_u64(row + 2 * k + 1, ((bits >> 32) << 32) | flag);
    }
  }
  bool ok = true;
  const unsigned long long* mine = reinterpret_cast<const unsigned long long*>(ws.mbox[ws.rank]);
  const int rounds = (nred + 31) / 32;
  double sums[3] = {0.0, 0.0, 0.0};  // nred <= kMboxPayload = 72 -> at most 3 totals per lane
  for (int q = 0; q < rounds; ++q) {
    const int k = lane + 32 * q;
    if (k >= nred) break;
    double sum = 0.0;
    const long long t0 = clock64();
    for (int p = 0; p < ws.nranks && ok; ++p) {
      const unsigned long long* row = mine + (size_t)(p * 2 + par) * kMboxStride;
      unsigned long long lo, hi;
      for (;;) {
        lo = ld_relaxed_sys_u64(row + 2 * k);
        hi = ld_relaxed_sys_u64(row + 2 * k + 1);
        const unsigned int fl = (unsigned int)lo, fh = (unsigned int)hi;
        if (fl == flag && fh == flag) break;
        if (fl == (flag | kPoisonFlag) || fh == (flag | kPoisonFlag)) { ok = false; break; }   // the peer gave up on this one
        if (ws.timeout_clocks > 0 && clock64() - t0 > ws.timeout_clocks) { ok = false; break; }  // it never launched
      }
      sum += __longlong_as_double((long long)((hi & 0xffffffff00000000ull) | (lo >> 32)));
    }
    sums[q] = sum;
  }
  ok = __all_sync(0xffffffffu, ok);
  if (!ok) {
    for (int p = lane; p < ws.nranks; p += 32) {
      unsigned long long* row = reinterpret_cast<unsigned long long*>(ws.mbox[p]) + (size_t)(ws.rank * 2 + par) * kMboxStride;
      for (int k = 0; k < 2 * nred; ++k) st_relaxed_sys_u64(row + k, (unsigned long long)(flag | kPoisonFlag));
    }
    if (lane == 0 && ws.err) *ws.err = 1;
  }
  for (int q = 0; q < rounds; ++q) {
    const int k = lane + 32 * q;
    if (k < nred) emit(k, ok ? sums[q] : __longlong_as_double(0x7ff8000000000000ll));
  }
  return ok;
}

// The epilogue of every reducing kernel, executed by the LAST CTA: per-GPU totals -> ws.out (summed across GPUs by
// warp 0 when a peer communicator is attached), mirrored to mapped host memory + ticket when requested.
__device__ __forceinline__ void peer_exchange(const double* tot, int nred, const RedWs& ws) {
  if (ws.nranks <= 1 || ws.mbox == nullptr) {
    for (int k = threadIdx.x; k < nred; k += blockDim.x) {
      ws.out[k] = tot[k];
      if (ws.host_out) ws.host_out[k] = tot[k];
    }
    if (ws.host_out) {
      __threadfence_system();  // every writer orders its mirror stores before the barrier ...
      __syncthreads();         // (all threads of the last CTA reach this point together)
      if (threadIdx.x == 0) *ws.host_flag = ws.host_ticket;  // ... so the ticket is the last thing the host sees
    }
    return;
  }
  if ((threadIdx.x >> 5) != 0) return;
  const int lane = threadIdx.x & 31;
  peer_allreduce_warp(tot, nred, ws, [&](int k, double res) {
    ws.out[k] = res;
    if (ws.host_out) ws.host_out[k] = res;
  });
  if (ws.host_out) {
    __threadfence_system();
    __syncwarp();
    if (lane == 0) *ws.host_flag = ws.host_ticket;
  }
}

// The two halves of block_reduce_publish.  block_reduce_store: block-reduce NRED per-thread fp64 accumulators and
// store the CTA's partial at partials[blockIdx.x * NRED + k] (written by lane 0 of warp 0; every thread calls it).
template <int NRED, int BLOCK = kBlock>
__device__ __forceinline__ void block_reduce_store(double (&acc)[NRED], double* partials) {
  __shared__ double sm[NRED][BLOCK / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NRED; ++k) {
    const double v = warp_sum(acc[k]);
    if (lane == 0) sm[k][warp] = v;
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < NRED; ++k) {
      double v = (lane < BLOCK / 32) ? sm[k][lane] : 0.0;
      v = warp_sum(v);
      if (lane == 0) partials[(size_t)blockIdx.x * NRED + k] = v;
    }
  }
}

// fold_partials: the `grid` partials of NRED entries in a fixed order -- thread t takes blocks t, t+BLOCK, ..., then
// the warps and the CTA sum what they hold -- into tot (shared memory, complete in every thread on return).  The same
// partials give the same bits whichever CTA, or however many CTAs, fold them.
template <int NRED, int BLOCK = kBlock>
__device__ __forceinline__ void fold_partials(const double* partials, unsigned int grid, double* tot) {
  __shared__ double sm[NRED][BLOCK / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NRED; ++k) {
    double v = 0.0;
    for (unsigned int b = threadIdx.x; b < grid; b += BLOCK) v += __ldcg(&partials[(size_t)b * NRED + k]);
    v = warp_sum(v);
    if (lane == 0) sm[k][warp] = v;
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < NRED; ++k) {
      double v = (lane < BLOCK / 32) ? sm[k][lane] : 0.0;
      v = warp_sum(v);
      if (lane == 0) tot[k] = v;
    }
  }
  __syncthreads();
}

// Block-reduce NRED per-thread fp64 accumulators, publish the block partial, and let the last CTA
// to arrive reduce all partials in a fixed order (deterministic for a fixed launch configuration).
// Returns true in every thread of the CTA that performed the final reduction (its ws.out writes are then complete
// after a __syncthreads()).
template <int NRED, int BLOCK = kBlock>
__device__ __forceinline__ bool block_reduce_publish(double (&acc)[NRED], const RedWs& ws) {
  __shared__ double tot[NRED];
  __shared__ bool is_last;
  block_reduce_store<NRED, BLOCK>(acc, ws.partials);
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned int ticket = atomicInc(ws.counter, gridDim.x - 1);  // wraps to 0: self-resetting
    is_last = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return false;
  __threadfence();
  fold_partials<NRED, BLOCK>(ws.partials, gridDim.x, tot);
  peer_exchange(tot, NRED, ws);  // per-GPU totals -> ws.out (summed across GPUs when a peer communicator is attached)
  return true;
}

// The last CTA to finish (ticket on *counter) folds the `grid` partials of `len` entries that start at part, in CTA
// order, and hands every total to emit(entry, total).  The fixed order makes identical launches give identical bits.
template <class Emit>
__device__ __forceinline__ void lm_fold_last(const double* part, int len, int grid, unsigned int* counter, Emit emit) {
  __shared__ bool last;
  __threadfence();  // every thread's partials, before the ticket
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    last = (atomicInc(counter, (unsigned int)grid - 1) == (unsigned int)grid - 1);
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int e = threadIdx.x; e < len; e += blockDim.x) {
    double s = 0.0;
    for (int g = 0; g < grid; ++g) s += __ldcg(&part[(size_t)g * len + e]);
    emit(e, s);
  }
}

// Class index of a label, validated: integer-valued and inside [0, K).  Anything else (negative, >= K, fractional,
// NaN) raises `bad` and maps to class 0, so no kernel ever forms an out-of-range shared/global address from a label.
__device__ __forceinline__ int checked_label(float y, int K, bool& bad) {
  const int yi = (int)y;
  const bool ok = (y >= 0.f) && (yi < K) && ((float)yi == y);
  bad = bad || !ok;
  return ok ? yi : 0;
}
__device__ __forceinline__ void report_bad_label(bool bad, const RedWs& ws) {
  if (bad && ws.bad_label != nullptr) *reinterpret_cast<volatile int*>(ws.bad_label) = 1;
}

// ---- counter-based synthetic generator (bench / tests): identical integer stream on host -----
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__host__ __device__ __forceinline__ float u01_from_bits(uint64_t bits) {
  return (float)(uint32_t)(bits >> 40) * (1.0f / 16777216.0f);  // 24 random bits -> [0,1)
}

}  // namespace se
