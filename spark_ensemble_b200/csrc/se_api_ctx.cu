// se_api_ctx.cu — host side of libse_b200.so (the extern "C" ABI declared in include/se_abi.h): the NCCL loader,
// errors, context create/destroy, timing, options, host allocations and the communicator, plus the helpers every
// se_api_*.cu file shares (se_ctx.h).
//
// A context owns the per-GPU state (stream, device slots, reduction workspace, scalar block, NCCL communicator) and
// each ABI call turns into kernel launches on the context stream.  No CPU fallback exists: every compute entry point
// needs a working CUDA device.
#include <dlfcn.h>
#include <sched.h>
#include <stdarg.h>
#include <unistd.h>

#include <memory>
#include <mutex>

#include "se_ctx.h"

using namespace se;
using namespace se_host;

// ------------------------------------------------------------------------------------------------
// NCCL is bound at run time (dlopen) so the library loads on boxes/processes without it and never
// clashes with a copy another component (e.g. a host framework) already loaded.
// ------------------------------------------------------------------------------------------------
namespace se_host {

void nccl_load(NcclApi& api);

NcclApi& nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] { nccl_load(api); });
  return api;
}

void nccl_load(NcclApi& api) {
  const char* names[] = {getenv("SE_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
  for (const char* nm : names) {
    if (!nm || !*nm) continue;
    api.handle = dlopen(nm, RTLD_NOW | RTLD_LOCAL);
    if (api.handle) break;
  }
  if (!api.handle) {
    const char* de = dlerror();
    api.why = std::string("dlopen(libnccl.so.2) failed: ") + (de ? de : "?");
    return;
  }
#define SE_SYM(field, name)                                                     \
  api.field = reinterpret_cast<decltype(api.field)>(dlsym(api.handle, name));   \
  if (!api.field) { api.why = std::string("missing symbol ") + name; return; }
  SE_SYM(GetUniqueId, "ncclGetUniqueId")
  SE_SYM(CommInitRank, "ncclCommInitRank")
  SE_SYM(CommDestroy, "ncclCommDestroy")
  SE_SYM(AllReduce, "ncclAllReduce")
  SE_SYM(AllGather, "ncclAllGather")
  SE_SYM(GetErrorString, "ncclGetErrorString")
  SE_SYM(GetVersion, "ncclGetVersion")
#undef SE_SYM
  api.ok = true;
}
thread_local std::string g_last_error;

int fail(se_ctx* ctx, int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  if (ctx) ctx->err = buf;
  return code;
}

int drain_kernel_events(se_ctx* ctx) {
  if (ctx->kpending == 0) return SE_OK;
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  unsigned long long st[2 * se_ctx::kRing];
  if (ctx->d_kstamp)
    SE_CUDA(ctx, cudaMemcpy(st, ctx->d_kstamp, sizeof(unsigned long long) * 2 * ctx->kpending, cudaMemcpyDeviceToHost));
  for (int i = 0; i < ctx->kpending; ++i) {
    float ms = 0.f;
    if (ctx->kstamped[i]) ms = (float)(1e-6 * (double)(st[2 * i + 1] - st[2 * i]));
    else SE_CUDA(ctx, cudaEventElapsedTime(&ms, ctx->kev[i][0], ctx->kev[i][1]));
    ctx->kms[ctx->kfam[i]] += (double)ms;
    ctx->kcount[ctx->kfam[i]] += 1;
  }
  ctx->kpending = 0;
  return SE_OK;
}

int kernel_stamp_slot(se_ctx* ctx, int family, unsigned long long** stamps) {
  *stamps = nullptr;
  if (!ctx->ktiming) return SE_OK;
  if (ctx->kpending == se_ctx::kRing) SE_TRY(drain_kernel_events(ctx));
  if (!ctx->d_kstamp) {
    // zeroed once: a slot's exit stamp is an atomicMax, and what an earlier launch left there is older
    SE_CUDA(ctx, ctx->d_kstamp.grow(2 * se_ctx::kRing));
    SE_CUDA(ctx, cudaMemsetAsync(ctx->d_kstamp, 0, sizeof(unsigned long long) * 2 * se_ctx::kRing, ctx->stream));
  }
  const int slot = ctx->kpending++;
  ctx->kfam[slot] = family;
  ctx->kstamped[slot] = true;
  *stamps = ctx->d_kstamp + 2 * slot;
  return SE_OK;
}

// A non-sticky error left behind by an unrelated earlier runtime call (e.g. a query that reported "not ready")
// must not be mistaken for a failure of the next kernel launch, which is checked with cudaGetLastError().
void clear_stale_error(const char* where) {
  const cudaError_t stale = cudaGetLastError();
  if (stale != cudaSuccess && getenv("SE_DEBUG"))
    fprintf(stderr, "[se_b200] cleared stale CUDA error at %s: %s\n", where, cudaGetErrorString(stale));
}

int begin(se_ctx* ctx) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  clear_stale_error("begin");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  if (ctx->timing) SE_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
  return SE_OK;
}

int end(se_ctx* ctx) {
  if (ctx->timing) SE_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
  if (getenv("SE_DEBUG")) clear_stale_error("end");
  return SE_OK;
}

RedWs red_ws(se_ctx* ctx, int out_offset, bool exchange) {
  RedWs ws;
  ws.partials = ctx->d_partials;
  ws.counter = ctx->d_counter;
  ws.out = ctx->d_scal + out_offset;
  ws.bad_label = ctx->d_bad_label;
  ctx->last_reduce_global = false;
  ctx->mirror_valid = false;
  // results can be mirrored to the host by the kernel itself when they are final on this GPU: single GPU, or
  // the fused peer exchange (with the NCCL fallback the all-reduce still has to run after the kernel)
  if (exchange && ctx->use_mirror && ctx->h_mirror && (ctx->nranks <= 1 || ctx->p2p)) {
    ws.host_out = ctx->d_mirror;
    ws.host_flag = reinterpret_cast<volatile unsigned long long*>(ctx->d_mirror + kMboxPayload);
    ws.host_ticket = ++ctx->mirror_ticket;
    ctx->mirror_valid = true;
    ctx->mirror_off = out_offset;
  }
  if (exchange && ctx->p2p && ctx->nranks > 1) {
    ws.mbox = ctx->d_mbox_table;
    ws.nranks = ctx->nranks;
    ws.rank = ctx->rank;
    ws.seq = ++ctx->red_seq;
    ws.err = ctx->d_p2p_err;
    ws.timeout_clocks = (long long)(ctx->peer_timeout_ms * (double)ctx->clock_khz);
    ctx->last_reduce_global = true;
  }
  return ws;
}

// all-reduce d_scal[off..off+count) in-stream (no-op without communicator)
int allreduce_dev(se_ctx* ctx, int off, int count, int op) {
  if (!ctx->comm || ctx->nranks <= 1) return SE_OK;
  if (ctx->last_reduce_global && op == kNcclSum) {  // already summed across GPUs inside the kernel
    ctx->last_reduce_global = false;
    return SE_OK;
  }
  NcclApi& api = nccl();
  int rc = api.AllReduce(ctx->d_scal + off, ctx->d_scal + off, (size_t)count, kNcclFloat64, op,
                         ctx->comm, ctx->stream);
  if (rc != 0) return fail(ctx, SE_ERR_NCCL, "ncclAllReduce: %s", api.GetErrorString(rc));
  return SE_OK;
}

// Labels are class indices for LogLoss / SAMME(.R) / vote aggregation.  The reference throws on the JVM for a label
// outside [0, numClasses) or a fractional one (GBMLoss.scala:200-204 `res(label.toInt) = 1.0`, Classifier.validateLabel);
// here the kernels raise a flag instead of indexing out of bounds and the call that observes it fails with SE_ERR_ARG.
int check_labels(se_ctx* ctx) {
  if (!(ctx->h_bad_label && *reinterpret_cast<volatile int*>(ctx->h_bad_label.get()))) {
    for (int& st : ctx->y_state)
      if (st == 1) st = 2;  // a validation pass completed before this point (same stream) and raised nothing
    return SE_OK;
  }
  if (ctx->h_bad_label) {
    ctx->y_state[0] = ctx->y_state[1] = 0;  // unknown again: the next call re-validates (and fails again if unchanged)
    *reinterpret_cast<volatile int*>(ctx->h_bad_label.get()) = 0;
    return fail(ctx, SE_ERR_ARG, "a label (or vote) is not an integer class index in [0, numClasses): results of this call are invalid");
  }
  return SE_OK;
}

int check_p2p(se_ctx* ctx) {
  if (ctx->p2p && ctx->h_p2p_err && *reinterpret_cast<volatile int*>(ctx->h_p2p_err.get()))
    return fail(ctx, SE_ERR_NCCL, "peer-memory all-reduce failed: a rank did not launch the matching reduction within "
                "%.0f ms (or gave up on it); se_comm_clear_error() re-arms the communicator", ctx->peer_timeout_ms);
  return SE_OK;
}

// Wait until the kernel's last CTA has written the current mirror ticket into mapped host memory.  Spins on the
// cache line with PAUSE for the first ~100 us (the common case: the kernel is already running), then yields the core
// between polls so that a long kernel / a slow peer does not burn the driver thread.
int wait_mirror(se_ctx* ctx) {
  volatile unsigned long long* flag = reinterpret_cast<volatile unsigned long long*>(ctx->h_mirror + kMboxPayload);
  for (unsigned long spin = 0;; ++spin) {
    if (*flag == ctx->mirror_ticket) return SE_OK;
    if (spin < 20000) {
#if defined(__x86_64__) || defined(__i386__)
      __builtin_ia32_pause();
#endif
      continue;
    }
    if ((spin & 0x3F) == 0) {
      const cudaError_t q = cudaStreamQuery(ctx->stream);
      if (q != cudaErrorNotReady) {  // finished or failed
        if (*flag == ctx->mirror_ticket) return SE_OK;
        if (q != cudaSuccess) return fail(ctx, SE_ERR_CUDA, "kernel failed before publishing its results: %s", cudaGetErrorString(q));
        SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (*flag == ctx->mirror_ticket) return SE_OK;
        return fail(ctx, SE_ERR_CUDA, "reduction results never reached the host mirror");
      }
    }
    sched_yield();
  }
}

// (all-reduce and) bring d_scal[off..off+count) to the host; synchronises the stream
int fetch_scalars(se_ctx* ctx, int off, int count, double* out, int op) {
  if (ctx->mirror_valid && ctx->mirror_off == off && op == kNcclSum && count <= kMboxPayload) {
    // poll the ticket the last CTA writes after the sums: no D2H copy, no stream synchronisation
    ctx->mirror_valid = false;
    ctx->last_reduce_global = false;
    SE_TRY(end(ctx));
    SE_TRY(wait_mirror(ctx));
    for (int i = 0; i < count; ++i) out[i] = ctx->h_mirror[i];
    SE_TRY(check_labels(ctx));
    return check_p2p(ctx);
  }
  SE_TRY(allreduce_dev(ctx, off, count, op));
  SE_CUDA(ctx, cudaMemcpyAsync(ctx->h_scal + off, ctx->d_scal + off, sizeof(double) * count,
                               cudaMemcpyDeviceToHost, ctx->stream));
  SE_TRY(end(ctx));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < count; ++i) out[i] = ctx->h_scal[off + i];
  SE_TRY(check_labels(ctx));
  return check_p2p(ctx);
}

// Carried fused squared rounds may leave R pending (gbm.r_pending): apply the steps before anything else touches R or
// writes H.  The stored values are the ones the carried statistics were summed over, so they stay current.
int settle_r(se_ctx* ctx) {
  if (ctx->gbm.r_pending == 0) return SE_OK;
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_LAUNCH_T(ctx, SE_KF_OTHER, launch_gbm_settle_r(ctx->slot[SE_SLOT_R].d, ctx->slot[SE_SLOT_H].d, ctx->d_rchain,
                                                    ctx->gbm.r_pending, ctx->gbm.n, ctx->sms, ctx->stream));
  ctx->gbm.r_pending = 0;
  return SE_OK;
}

// The residual-mode fused squared round leaves F owed (gbm.f_owed): rebuild it as y - r before anything reads train F
// or writes Y, F or R.  R is re-derived from the rebuilt F (y - F), as an eager update would have left it.  A pending
// R is settled first: F = y - r.
int settle_f(se_ctx* ctx) {
  SE_TRY(settle_r(ctx));
  if (!ctx->gbm.f_owed) return SE_OK;
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_LAUNCH_T(ctx, SE_KF_OTHER, launch_gbm_settle_f(ctx->slot[SE_SLOT_Y].d, ctx->slot[SE_SLOT_R].d, ctx->slot[SE_SLOT_F].d,
                                                    ctx->gbm.n, ctx->sms, ctx->stream));
  ctx->gbm.f_owed = false;
  ctx->gbm.sq_stats_current = false;  // y - (y - r) need not equal r bit for bit
  return SE_OK;
}

// Every entry point that writes a caller-chosen slot calls this once its own checks have passed, before the write is
// enqueued: it drops what the context derived from the slot's old contents.  The owed F is rebuilt from Y and R first.
// A call that derives something from the slot it writes (a walk over X into a row of X re-ranks X) calls it after that.
int write_slot(se_ctx* ctx, int slot) {
  switch (slot) {
    case SE_SLOT_Y: case SE_SLOT_F: case SE_SLOT_R:
      SE_TRY(settle_f(ctx));
      ctx->gbm.r_current = false;
      ctx->gbm.sq_stats_current = false;
      if (slot == SE_SLOT_Y) ctx->y_state[0] = 0;  // labels checked as class indices
      break;
    case SE_SLOT_H:
      SE_TRY(settle_r(ctx));  // the pending steps go along the old h
      ctx->gbm.sq_stats_current = false;  // the squared round's carried statistics
      break;
    case SE_SLOT_VY: ctx->y_state[1] = 0; break;
    case SE_SLOT_W: case SE_SLOT_BAG: ctx->gbm.wsum_valid = false; break;
    case SE_SLOT_WOUT: ctx->wout_scaled = false; break;  // se_download's 1/S factor
    case SE_SLOT_X: ctx->bins[0].valid = false; break;   // rank matrix
    case SE_SLOT_VX: ctx->bins[1].valid = false; break;
  }
  return SE_OK;
}

// Every entry point that reads a caller-chosen slot calls this first.  A caller that reads R between rounds over one
// direction would pay a settle for every deferred round: the next carried round stores r' instead.
int read_slot(se_ctx* ctx, int slot) {
  if (slot == SE_SLOT_F) return settle_f(ctx);
  if (slot == SE_SLOT_R) {
    ctx->gbm.sq_defer_ok = false;
    return settle_r(ctx);
  }
  return SE_OK;
}
int slot_alloc2d(se_ctx* ctx, int slot, int64_t rows, int64_t cols) {
  SE_REQUIRE(ctx, slot >= 0 && slot < SE_NUM_SLOTS, SE_ERR_ARG, "bad slot %d", slot);
  SE_REQUIRE(ctx, rows >= 1 && cols >= 0, SE_ERR_ARG, "bad slot shape %lld x %lld", (long long)rows,
             (long long)cols);
  SE_TRY(write_slot(ctx, slot));
  SlotBuf& s = ctx->slot[slot];
  const int64_t ld = (rows > 1) ? ((cols + 31) / 32) * 32 : cols;
  s.rows = s.cols = s.ld = 0;  // an empty slot if the allocation fails
  SE_CUDA(ctx, s.d.grow((size_t)(rows * ld + 32)));
  s.rows = rows; s.cols = cols; s.ld = ld;
  return SE_OK;
}

// Rows [row, row + count) of a caller's output slot, n values each: records the write (write_slot) and hands out the
// first row and the row stride (ld may be NULL).
int out_rows(se_ctx* ctx, int slot, int row, int count, int64_t n, float** out, int64_t* ld) {
  SE_REQUIRE(ctx, slot >= 0 && slot < SE_NUM_SLOTS, SE_ERR_ARG, "bad output slot %d", slot);
  const SlotBuf& s = ctx->slot[slot];
  SE_REQUIRE(ctx, s.d && s.cols == n && row >= 0 && (int64_t)row + count <= s.rows, SE_ERR_STATE,
             "output slot %d: no rows %d..%d of %lld values", slot, row, row + count - 1, (long long)n);
  SE_TRY(write_slot(ctx, slot));
  *out = s.d + (int64_t)row * s.ld;
  if (ld) *ld = s.ld;
  return SE_OK;
}

}  // namespace se_host

int se_abi_version(void) { return SE_ABI_VERSION; }

const char* se_last_error(const se_ctx* ctx) {
  if (ctx && !ctx->err.empty()) return ctx->err.c_str();
  return g_last_error.c_str();
}

int se_device_count(int* out) {
  if (!out) return fail(nullptr, SE_ERR_ARG, "null out");
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) {
    *out = 0;
    return fail(nullptr, SE_ERR_CUDA, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
  }
  *out = n;
  return SE_OK;
}

int se_ctx_create(int device, se_ctx** out) {
  if (!out) return fail(nullptr, SE_ERR_ARG, "null out");
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0)
    return fail(nullptr, SE_ERR_CUDA, "no CUDA device available (%s): the hot path has no CPU fallback",
                e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
  if (device < 0 || device >= n) return fail(nullptr, SE_ERR_ARG, "device %d out of range [0,%d)", device, n);
  std::unique_ptr<se_ctx> owner(new se_ctx());  // a failed step frees what the steps before it created
  se_ctx* ctx = owner.get();
  ctx->device = device;
  SE_CUDA(nullptr, cudaSetDevice(device));
  cudaDeviceProp prop;
  SE_CUDA(nullptr, cudaGetDeviceProperties(&prop, device));
  ctx->sms = prop.multiProcessorCount;
  ctx->l2_hint_rows = 2 * (int64_t)prop.l2CacheSize / 16;
  if (const char* s = getenv("SE_ALTERNATE_PASSES")) ctx->alternate = atoi(s) != 0;
  if (const char* s = getenv("SE_L2_HINTS")) ctx->l2_hints = atoi(s) != 0 ? 1 : 0;
  if (const char* s = getenv("SE_CTAS_PER_SM")) {
    const int v = atoi(s);
    if (v >= 1 && v <= 16) ctx->ctas_per_sm = v;
  }
  SE_CUDA(nullptr, ctx->stream.create(cudaStreamNonBlocking));
  SE_CUDA(nullptr, ctx->ev0.create());
  SE_CUDA(nullptr, ctx->ev1.create());
  SE_CUDA(nullptr, ctx->d_scal.grow(kScal));
  SE_CUDA(nullptr, cudaMemset(ctx->d_scal, 0, sizeof(double) * kScal));
  SE_CUDA(nullptr, ctx->h_scal.grow(kScal));
  SE_CUDA(nullptr, ctx->d_partials.grow((size_t)kMaxGridPartials * kMaxRed));
  SE_CUDA(nullptr, ctx->d_counter.grow(1));
  SE_CUDA(nullptr, cudaMemset(ctx->d_counter, 0, sizeof(unsigned int)));
  SE_CUDA(nullptr, ctx->h_bad_label.grow(1));
  *ctx->h_bad_label = 0;
  SE_CUDA(nullptr, cudaHostGetDevicePointer(&ctx->d_bad_label, ctx->h_bad_label, 0));
  SE_CUDA(nullptr, ctx->d_fsync.grow(1));
  SE_CUDA(nullptr, cudaMemset(ctx->d_fsync, 0, sizeof(FusedSync)));
  SE_CUDA(nullptr, ctx->d_rchain.grow(kSqDeferMax));
  SE_CUDA(nullptr, ctx->d_sq_carry.grow((size_t)2 * (kMaxGridPartials / 2) * 3));
  ctx->clock_khz = prop.clockRate > 0 ? prop.clockRate : 1965000;
  if (const char* s = getenv("SE_FUSED_ROUND")) ctx->fused_round = atoi(s) != 0 ? 1 : 0;
  if (const char* s = getenv("SE_FUSED_RESIDENT")) ctx->fused_resident = atoi(s) != 0;
  if (const char* s = getenv("SE_LS_MODE")) { const int v = atoi(s); if (v >= 0 && v <= 2) ctx->ls_mode = v; }
  if (const char* s = getenv("SE_LS_RESIDENT")) ctx->ls_resident = atoi(s) != 0;
  if (const char* s = getenv("SE_PEER_TIMEOUT_MS")) { const double v = atof(s); if (v >= 0.0) ctx->peer_timeout_ms = v; }
  SE_CUDA(nullptr, ctx->h_mirror.grow(kMboxPayload + 8));
  memset(ctx->h_mirror, 0, sizeof(double) * (kMboxPayload + 8));
  SE_CUDA(nullptr, cudaHostGetDevicePointer(&ctx->d_mirror, ctx->h_mirror, 0));
  if (const char* s = getenv("SE_HOST_MIRROR")) ctx->use_mirror = atoi(s) != 0;
  SE_CUDA(nullptr, ctx->d_small.grow(kSmallBytes));
  SE_CUDA(nullptr, ctx->h_small.grow(kSmallBytes));
  SE_CUDA(nullptr, cudaDeviceSynchronize());
  *out = owner.release();
  return SE_OK;
}

static void release_p2p(se_ctx* ctx);

int se_ctx_destroy(se_ctx* ctx) {
  if (!ctx) return SE_OK;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  if (ctx->comm && nccl().ok) {
    release_p2p(ctx);
    nccl().CommDestroy(ctx->comm);
  }
  delete ctx;
  return SE_OK;
}

int se_ctx_sync(se_ctx* ctx) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return check_labels(ctx);
}

int se_ctx_device(const se_ctx* ctx, int* device) {
  if (!ctx || !device) return fail(nullptr, SE_ERR_ARG, "null argument");
  *device = ctx->device;
  return SE_OK;
}

int se_ctx_launch_count(const se_ctx* ctx, int64_t* out) {
  if (!ctx || !out) return fail(nullptr, SE_ERR_ARG, "null argument");
  *out = ctx->launches;
  return SE_OK;
}

int se_ctx_set_timing(se_ctx* ctx, int on) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  ctx->timing = on != 0;
  return SE_OK;
}

int se_ctx_last_ms(se_ctx* ctx, double* out) {
  if (!ctx || !out) return fail(nullptr, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, ctx->timing, SE_ERR_STATE, "timing is off (se_ctx_set_timing)");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
  float ms = 0.f;
  SE_CUDA(ctx, cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
  *out = (double)ms;
  return SE_OK;
}

int se_ctx_timer_start(se_ctx* ctx) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  if (!ctx->tm0) {
    SE_CUDA(ctx, ctx->tm0.create());
    SE_CUDA(ctx, ctx->tm1.create());
  }
  SE_CUDA(ctx, cudaEventRecord(ctx->tm0, ctx->stream));
  return SE_OK;
}

int se_ctx_timer_stop(se_ctx* ctx, double* ms) {
  if (!ctx || !ms) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, ctx->tm0, SE_ERR_STATE, "se_ctx_timer_start first");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_CUDA(ctx, cudaEventRecord(ctx->tm1, ctx->stream));
  SE_CUDA(ctx, cudaEventSynchronize(ctx->tm1));
  float f = 0.f;
  SE_CUDA(ctx, cudaEventElapsedTime(&f, ctx->tm0, ctx->tm1));
  *ms = (double)f;
  return SE_OK;
}

int se_ctx_kernel_timing(se_ctx* ctx, int on) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  if (!on) SE_TRY(drain_kernel_events(ctx));
  ctx->ktiming = on != 0;
  return SE_OK;
}

int se_ctx_kernel_time(se_ctx* ctx, int family, double* total_ms, int64_t* launches) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, family >= 0 && family < SE_KF_COUNT, SE_ERR_ARG, "bad kernel family %d", family);
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_TRY(drain_kernel_events(ctx));
  if (total_ms) *total_ms = ctx->kms[family];
  if (launches) *launches = ctx->kcount[family];
  return SE_OK;
}

int se_ctx_kernel_time_reset(se_ctx* ctx) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_TRY(drain_kernel_events(ctx));
  for (int i = 0; i < SE_KF_COUNT; ++i) { ctx->kms[i] = 0.0; ctx->kcount[i] = 0; }
  return SE_OK;
}

namespace {
// One entry per option of se_ctx_set_option / se_ctx_get_option.  `set` is null for a read-only diagnostic; `ok`, when
// set, refuses a value with the message `range`.
struct Option {
  const char* name;
  int (*get)(const se_ctx* c, double* v);
  void (*set)(se_ctx* c, double v);
  bool (*ok)(double v);
  const char* range;
};
#define SE_GET(expr) [](const se_ctx* c, double* v) { *v = (double)(expr); return (int)SE_OK; }
#define SE_SET(stmt) [](se_ctx* c, double v) { const int iv = (int)v; (void)iv; stmt; }
#define SE_IN(cond) [](double v) { const int iv = (int)v; (void)iv; return (bool)(cond); }

// rows the last weighted median sent to the exact kernel (synchronises the stream)
int last_wm_deferred(const se_ctx* c, double* v) {
  unsigned int n = 0;
  if (c->d_wm && c->last_wm_mode == 1) {
    cudaSetDevice(c->device);
    if (cudaStreamSynchronize(c->stream) != cudaSuccess || cudaMemcpy(&n, c->d_wm, sizeof(n), cudaMemcpyDeviceToHost) != cudaSuccess) {
      cudaGetLastError();
      return SE_ERR_CUDA;
    }
  }
  *v = (double)n;
  return SE_OK;
}

const Option kOptions[] = {
  {"fused_round", SE_GET(c->fused_round), SE_SET(c->fused_round = v < 0 ? -1 : (iv != 0))},
  {"fused_round_max_rows", SE_GET(c->fused_round_max_rows), SE_SET(c->fused_round_max_rows = (int64_t)v)},
  {"fused_timing", SE_GET(c->fused_timing), SE_SET(c->fused_timing = iv != 0)},
  {"fused_loss_reduce", SE_GET(c->fused_loss_reduce), SE_SET(c->fused_loss_reduce = iv != 0)},
  {"tree_bins", SE_GET(c->tree_bins), SE_SET(c->tree_bins = iv != 0)},
  {"tree_mask", SE_GET(c->tree_mask), SE_SET(c->tree_mask = iv != 0)},
  {"wm_fast", SE_GET(c->wm_fast), SE_SET(c->wm_fast = iv != 0)},
  {"wm_list_cap", SE_GET(c->wm_list_cap), SE_SET(c->wm_list_cap = (int64_t)v), SE_IN(v >= 0 && v < 2147483000.0),
   "wm_list_cap in [0, 2^31)"},
  {"fused_ctas_per_sm", SE_GET(c->fused_ctas_per_sm), SE_SET(c->fused_ctas_per_sm = iv), SE_IN(iv >= 1 && iv <= 8),
   "fused_ctas_per_sm in [1,8]"},
  {"fused_resident", SE_GET(c->fused_resident), SE_SET(c->fused_resident = iv != 0)},
  {"sq_defer_max", SE_GET(c->sq_defer_max), SE_SET(c->sq_defer_max = iv), SE_IN(iv >= 0 && iv <= kSqDeferMax),
   "sq_defer_max in [0,64]"},
  {"ls_mode", SE_GET(c->ls_mode), SE_SET(c->ls_mode = iv), SE_IN(iv >= 0 && iv <= 2), "ls_mode in {0,1,2}"},
  {"ls_resident", SE_GET(c->ls_resident), SE_SET(c->ls_resident = iv != 0)},
  {"ls_ctas_per_sm", SE_GET(c->ls_ctas_per_sm), SE_SET(c->ls_ctas_per_sm = iv), SE_IN(iv >= 1 && iv <= 8),
   "ls_ctas_per_sm in [1,8]"},
  {"peer_timeout_ms", SE_GET(c->peer_timeout_ms), SE_SET(c->peer_timeout_ms = v), SE_IN(v >= 0.0), "peer_timeout_ms >= 0"},
  {"alternate_passes", SE_GET(c->alternate), SE_SET(c->alternate = iv != 0)},
  {"l2_hints", SE_GET(c->l2_hints), SE_SET(c->l2_hints = v < 0 ? -1 : (iv != 0))},
  {"ctas_per_sm", SE_GET(c->ctas_per_sm), SE_SET(c->ctas_per_sm = iv), SE_IN(iv >= 1 && iv <= 16), "ctas_per_sm in [1,16]"},
  {"host_mirror", SE_GET(c->use_mirror), SE_SET(c->use_mirror = iv != 0)},
  // read-only diagnostics
  {"last_forest_chunks", SE_GET(c->last_forest_chunks)},
  {"last_wm_mode", SE_GET(c->last_wm_mode)},
  {"last_wm_deferred", last_wm_deferred},
  {"last_tree_mask", SE_GET(c->last_tree_mask)},
  {"last_tree_binned", SE_GET(c->last_tree_binned)},
  {"last_tree_rebinned_cols", SE_GET(c->last_tree_rebinned_cols)},
  {"last_tree_fit_hist", SE_GET(c->last_tree_fit_hist)},
  {"last_forest_fit_batches", SE_GET(c->last_forest_fit_batches)},
  {"last_fused_stats_us", SE_GET(c->last_fused_us[0])},
  {"last_fused_brent_us", SE_GET(c->last_fused_us[1])},
  {"last_fused_update_us", SE_GET(c->last_fused_us[2])},
  {"last_round_fused", SE_GET(c->last_round_fused)},
  {"last_round_stats_carried", SE_GET(c->last_round_carried)},
  {"last_round_deferred", SE_GET(c->last_round_deferred)},
  {"r_pending", SE_GET(c->gbm.r_pending)},
  {"last_ls_workers", SE_GET(c->last_ls_workers)},
  {"last_ls_passes", SE_GET(c->last_ls_passes)},
  {"last_ls_hit_ratio", SE_GET(0.0)},  // kept for compatibility: no L2 window is ever requested
  {"last_fused_grid", SE_GET(c->last_fused_grid)},
  {"last_fused_resident_tiles", SE_GET(c->last_fused_resident_tiles)},
  {"last_round_stat0", SE_GET(c->last_round_stats[0])},
  {"last_round_stat1", SE_GET(c->last_round_stats[1])},
  {"last_round_stat2", SE_GET(c->last_round_stats[2])},
};
#undef SE_GET
#undef SE_SET
#undef SE_IN

const Option* find_option(const char* key) {
  if (!key) return nullptr;
  for (const Option& o : kOptions)
    if (strcmp(o.name, key) == 0) return &o;
  return nullptr;
}
}  // namespace

int se_ctx_set_option(se_ctx* ctx, const char* key, double value) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  const Option* o = find_option(key);
  if (!o || !o->set) return fail(ctx, SE_ERR_ARG, "unknown or read-only option '%s'", key ? key : "(null)");
  SE_REQUIRE(ctx, !o->ok || o->ok(value), SE_ERR_ARG, "%s", o->range);
  o->set(ctx, value);
  return SE_OK;
}

int se_ctx_get_option(const se_ctx* ctx, const char* key, double* value) {
  if (!ctx || !value) return fail(nullptr, SE_ERR_ARG, "null argument");
  const Option* o = find_option(key);
  if (!o) return fail(const_cast<se_ctx*>(ctx), SE_ERR_ARG, "unknown option '%s'", key ? key : "(null)");
  return o->get(ctx, value);
}

int se_host_alloc(int64_t bytes, void** out) {
  if (!out || bytes < 0) return fail(nullptr, SE_ERR_ARG, "bad argument");
  *out = nullptr;
  cudaError_t e = PinnedMem::alloc(out, (size_t)(bytes > 0 ? bytes : 1));
  if (e != cudaSuccess) return fail(nullptr, SE_ERR_CUDA, "cudaMallocHost(%lld): %s", (long long)bytes, cudaGetErrorString(e));
  return SE_OK;
}

int se_host_free(void* ptr) {
  if (!ptr) return SE_OK;
  cudaError_t e = PinnedMem::release(ptr);
  if (e != cudaSuccess) return fail(nullptr, SE_ERR_CUDA, "cudaFreeHost: %s", cudaGetErrorString(e));
  return SE_OK;
}

// ---- communicator ------------------------------------------------------------------------------
int se_comm_unique_id(void* out, int bytes) {
  if (!out || bytes < SE_COMM_ID_BYTES) return fail(nullptr, SE_ERR_ARG, "id buffer must hold %d bytes", SE_COMM_ID_BYTES);
  NcclApi& api = nccl();
  if (!api.ok) return fail(nullptr, SE_ERR_NCCL, "NCCL unavailable: %s", api.why.c_str());
  nccl_uid_t id;
  int rc = api.GetUniqueId(&id);
  if (rc != 0) return fail(nullptr, SE_ERR_NCCL, "ncclGetUniqueId: %s", api.GetErrorString(rc));
  memcpy(out, &id, sizeof(id));
  return SE_OK;
}

int se_comm_init(se_ctx* ctx, int nranks, int rank, const void* id, int bytes) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, nranks >= 1 && rank >= 0 && rank < nranks, SE_ERR_ARG, "bad rank %d of %d", rank, nranks);
  SE_REQUIRE(ctx, !ctx->comm, SE_ERR_STATE, "communicator already attached");
  ctx->nranks = nranks;
  ctx->rank = rank;
  ctx->gbm.counts_valid = ctx->gbm.wsum_valid = false;
  if (nranks == 1) return SE_OK;
  SE_REQUIRE(ctx, id && bytes >= SE_COMM_ID_BYTES, SE_ERR_ARG, "unique id of %d bytes required", SE_COMM_ID_BYTES);
  NcclApi& api = nccl();
  if (!api.ok) return fail(ctx, SE_ERR_NCCL, "NCCL unavailable: %s", api.why.c_str());
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  nccl_uid_t uid;
  memcpy(&uid, id, sizeof(uid));
  int rc = api.CommInitRank(&ctx->comm, nranks, uid, rank);
  if (rc != 0) {
    ctx->comm = nullptr;
    return fail(ctx, SE_ERR_NCCL, "ncclCommInitRank: %s", api.GetErrorString(rc));
  }
  // ---- peer-memory mailboxes for the fused all-reduce (falls back to NCCL if any rank cannot map them)
  const char* env = getenv("SE_P2P_ALLREDUCE");
  int want = (env && atoi(env) == 0) ? 0 : 1;
  const size_t mbox_bytes = sizeof(double) * (size_t)nranks * 2 * kMboxStride;
  int ok = want;
  cudaIpcMemHandle_t mine;
  memset(&mine, 0, sizeof(mine));
  if (ok) {
    ok = ctx->mbox_local.grow(mbox_bytes / sizeof(double)) == cudaSuccess && cudaMemset(ctx->mbox_local, 0, mbox_bytes) == cudaSuccess &&
         ctx->h_p2p_err.grow(1) == cudaSuccess &&
         cudaHostGetDevicePointer(&ctx->d_p2p_err, ctx->h_p2p_err, 0) == cudaSuccess &&
         ctx->d_mbox_table.grow(nranks) == cudaSuccess &&
         cudaIpcGetMemHandle(&mine, ctx->mbox_local) == cudaSuccess;
    cudaGetLastError();
  }
  // exchange the handles (and everyone's readiness) through NCCL.  Ranks that live in the SAME process (one JVM /
  // one Python process driving several GPUs: sharded.ShardedContext) cannot open each other's IPC handles — they
  // exchange the raw device pointer instead and enable peer access between the two devices.
  struct PeerBlob { cudaIpcMemHandle_t handle; unsigned char ok; unsigned char pad[3]; int32_t pid; int32_t device; int32_t pad2; uint64_t ptr; };
  const size_t hb = sizeof(PeerBlob);
  std::vector<unsigned char> send(hb, 0), recv(hb * nranks, 0);
  {
    PeerBlob b;
    memset(&b, 0, sizeof(b));
    b.handle = mine; b.ok = (unsigned char)ok; b.pid = (int32_t)getpid(); b.device = ctx->device;
    b.ptr = (uint64_t)(uintptr_t)ctx->mbox_local.get();
    memcpy(send.data(), &b, sizeof(b));
  }
  DevBuf<unsigned char> d_send, d_recv;
  SE_CUDA(ctx, d_send.grow(hb));
  SE_CUDA(ctx, d_recv.grow(hb * nranks));
  SE_CUDA(ctx, cudaMemcpyAsync(d_send, send.data(), hb, cudaMemcpyHostToDevice, ctx->stream));
  rc = api.AllGather(d_send, d_recv, hb, kNcclChar, ctx->comm, ctx->stream);
  if (rc != 0) return fail(ctx, SE_ERR_NCCL, "ncclAllGather: %s", api.GetErrorString(rc));
  SE_CUDA(ctx, cudaMemcpyAsync(recv.data(), d_recv, hb * nranks, cudaMemcpyDeviceToHost, ctx->stream));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  int all_ok = 1;
  for (int p = 0; p < nranks; ++p) all_ok &= reinterpret_cast<const PeerBlob*>(recv.data() + p * hb)->ok;
  ctx->mbox_peers.assign(nranks, nullptr);
  ctx->mbox_ipc.assign(nranks, 0);
  if (all_ok) {
    for (int p = 0; p < nranks && all_ok; ++p) {
      if (p == rank) { ctx->mbox_peers[p] = ctx->mbox_local; continue; }
      PeerBlob b;
      memcpy(&b, recv.data() + p * hb, sizeof(b));
      void* ptr = nullptr;
      if (b.pid == (int32_t)getpid()) {
        int can = 0;
        if (b.device == ctx->device) can = 1;
        else if (cudaDeviceCanAccessPeer(&can, ctx->device, b.device) == cudaSuccess && can) {
          const cudaError_t pe = cudaDeviceEnablePeerAccess(b.device, 0);
          if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) can = 0;
        }
        cudaGetLastError();
        if (can) ptr = (void*)(uintptr_t)b.ptr; else all_ok = 0;
      } else {
        if (cudaIpcOpenMemHandle(&ptr, b.handle, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { all_ok = 0; cudaGetLastError(); }
        else ctx->mbox_ipc[p] = 1;
      }
      ctx->mbox_peers[p] = ptr;
    }
  }
  // second round: did every rank manage to open every peer?
  send[0] = (unsigned char)all_ok;
  SE_CUDA(ctx, cudaMemcpyAsync(d_send, send.data(), hb, cudaMemcpyHostToDevice, ctx->stream));
  rc = api.AllGather(d_send, d_recv, hb, kNcclChar, ctx->comm, ctx->stream);
  if (rc != 0) return fail(ctx, SE_ERR_NCCL, "ncclAllGather: %s", api.GetErrorString(rc));
  SE_CUDA(ctx, cudaMemcpyAsync(recv.data(), d_recv, hb * nranks, cudaMemcpyDeviceToHost, ctx->stream));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int p = 0; p < nranks; ++p) all_ok &= recv[p * hb];
  if (all_ok) {
    *ctx->h_p2p_err = 0;
    SE_CUDA(ctx, cudaMemcpy(ctx->d_mbox_table, ctx->mbox_peers.data(), sizeof(double*) * nranks, cudaMemcpyHostToDevice));
    ctx->p2p = true;
    ctx->red_seq = 0;
  } else {
    ctx->p2p = false;  // NCCL all-reduce of the scalar block after each reducing kernel
  }
  return SE_OK;
}

int se_comm_p2p_active(const se_ctx* ctx, int* active) {
  if (!ctx || !active) return fail(nullptr, SE_ERR_ARG, "null argument");
  *active = ctx->p2p ? 1 : 0;
  return SE_OK;
}

int se_comm_clear_error(se_ctx* ctx) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (ctx->h_p2p_err) *reinterpret_cast<volatile int*>(ctx->h_p2p_err.get()) = 0;
  ctx->err.clear();
  return SE_OK;
}

static void release_p2p(se_ctx* ctx) {
  for (int p = 0; p < (int)ctx->mbox_peers.size(); ++p)
    if (p != ctx->rank && ctx->mbox_peers[p] && ctx->mbox_ipc[p]) cudaIpcCloseMemHandle(ctx->mbox_peers[p]);
  ctx->mbox_peers.clear();
  ctx->mbox_ipc.clear();
  ctx->mbox_local.reset();
  ctx->d_mbox_table.reset();
  ctx->h_p2p_err.reset();
  ctx->d_p2p_err = nullptr;
  ctx->p2p = false;
}

int se_comm_destroy(se_ctx* ctx) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  if (ctx->comm) {
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    release_p2p(ctx);
    nccl().CommDestroy(ctx->comm);
    ctx->comm = nullptr;
  }
  ctx->nranks = 1;
  ctx->rank = 0;
  ctx->gbm.counts_valid = ctx->gbm.wsum_valid = false;
  return SE_OK;
}

int se_comm_info(const se_ctx* ctx, int* nranks, int* rank) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  if (nranks) *nranks = ctx->nranks;
  if (rank) *rank = ctx->rank;
  return SE_OK;
}

int se_comm_allreduce_host(se_ctx* ctx, double* values, int count) {
  if (!ctx || !values) return fail(nullptr, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, count >= 0 && count <= kScalHist - kScalHost, SE_ERR_ARG, "count %d too large", count);
  if (!ctx->comm || ctx->nranks <= 1 || count == 0) return SE_OK;
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  for (int i = 0; i < count; ++i) ctx->h_scal[kScalHost + i] = values[i];
  SE_CUDA(ctx, cudaMemcpyAsync(ctx->d_scal + kScalHost, ctx->h_scal + kScalHost, sizeof(double) * count,
                               cudaMemcpyHostToDevice, ctx->stream));
  ctx->last_reduce_global = false;
  SE_TRY(allreduce_dev(ctx, kScalHost, count));
  SE_CUDA(ctx, cudaMemcpyAsync(ctx->h_scal + kScalHost, ctx->d_scal + kScalHost, sizeof(double) * count,
                               cudaMemcpyDeviceToHost, ctx->stream));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < count; ++i) values[i] = ctx->h_scal[kScalHost + i];
  return SE_OK;
}
