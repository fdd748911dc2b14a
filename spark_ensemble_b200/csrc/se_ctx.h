// se_ctx.h — private to the host side of libse_b200.so (se_api_*.cu): the per-GPU context, the handles that own its
// CUDA resources, and the helpers the entry points share.
#pragma once

#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <utility>
#include <vector>

#include "../../include/se_abi.h"
#include "se_kernels.h"

namespace se_host {

typedef struct { char internal[128]; } nccl_uid_t;
typedef void* nccl_comm_t;
struct NcclApi {
  void* handle = nullptr;
  int (*GetUniqueId)(nccl_uid_t*) = nullptr;
  int (*CommInitRank)(nccl_comm_t*, int, nccl_uid_t, int) = nullptr;
  int (*CommDestroy)(nccl_comm_t) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, nccl_comm_t, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  int (*GetVersion)(int*) = nullptr;
  bool ok = false;
  std::string why;
};
constexpr int kNcclFloat64 = 8;  // ncclDouble
constexpr int kNcclSum = 0;
constexpr int kNcclMax = 2;
constexpr int kNcclChar = 0;

extern thread_local std::string g_last_error;

constexpr int kScal = 1024;         // doubles in the device/host scalar blocks ([0, 160): generic reductions)
constexpr int kScalHist = 704;      // 256-bin radix-select histogram
constexpr int kScalRound = 160;     // offset of the squared-round results (statistics, alpha, loss)
constexpr int kScalHost = 192;      // offset used by se_comm_allreduce_host (up to kScalHist - kScalHost values)
constexpr int kSmallBytes = 1 << 20;  // small device scratch: weights, init, tree arrays, factors

// ---- owning handles of CUDA resources: each frees what it holds when it is destroyed or reassigned
struct DeviceMem {
  static cudaError_t alloc(void** p, size_t bytes) { return cudaMalloc(p, bytes); }
  static cudaError_t release(void* p) { return cudaFree(p); }
};
struct PinnedMem {
  static cudaError_t alloc(void** p, size_t bytes) { return cudaMallocHost(p, bytes); }
  static cudaError_t release(void* p) { return cudaFreeHost(p); }
};
struct MappedMem {  // pinned and mapped: cudaHostGetDevicePointer gives the device alias
  static cudaError_t alloc(void** p, size_t bytes) { return cudaHostAlloc(p, bytes, cudaHostAllocMapped); }
  static cudaError_t release(void* p) { return cudaFreeHost(p); }
};

// A buffer of `size()` elements of T.  It converts to T* so that it can be handed to launchers and copies as is.
template <class T, class Mem>
class Buffer {
 public:
  Buffer() = default;
  Buffer(Buffer&& o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
  Buffer& operator=(Buffer&& o) noexcept {
    std::swap(p_, o.p_);
    std::swap(n_, o.n_);
    return *this;
  }
  ~Buffer() { reset(); }
  operator T*() const { return p_; }
  T* operator->() const { return p_; }
  T* get() const { return p_; }
  size_t size() const { return n_; }
  cudaError_t reset() {
    const cudaError_t e = p_ ? Mem::release(p_) : cudaSuccess;
    p_ = nullptr;
    n_ = 0;
    return e;
  }
  // At least n elements.  A smaller buffer is freed before the new one is allocated, so the peak stays one buffer;
  // the old contents are not kept.  On failure the buffer is left empty.
  cudaError_t grow(size_t n) {
    if (p_ && n_ >= n) return cudaSuccess;
    cudaError_t e = reset();
    if (e == cudaSuccess) e = Mem::alloc(reinterpret_cast<void**>(&p_), sizeof(T) * n);
    if (e != cudaSuccess) {
      p_ = nullptr;
      return e;
    }
    n_ = n;
    return cudaSuccess;
  }

 private:
  T* p_ = nullptr;
  size_t n_ = 0;
};
template <class T> using DevBuf = Buffer<T, DeviceMem>;
template <class T> using PinnedBuf = Buffer<T, PinnedMem>;
template <class T> using MappedBuf = Buffer<T, MappedMem>;

class Stream {
 public:
  Stream() = default;
  Stream(Stream&& o) noexcept : s_(std::exchange(o.s_, nullptr)) {}
  Stream& operator=(Stream&& o) noexcept { std::swap(s_, o.s_); return *this; }
  ~Stream() { if (s_) cudaStreamDestroy(s_); }
  cudaError_t create(unsigned flags) { return cudaStreamCreateWithFlags(&s_, flags); }
  operator cudaStream_t() const { return s_; }

 private:
  cudaStream_t s_ = nullptr;
};

class Event {
 public:
  Event() = default;
  Event(Event&& o) noexcept : e_(std::exchange(o.e_, nullptr)) {}
  Event& operator=(Event&& o) noexcept { std::swap(e_, o.e_); return *this; }
  ~Event() { if (e_) cudaEventDestroy(e_); }
  cudaError_t create(unsigned flags = cudaEventDefault) { return cudaEventCreateWithFlags(&e_, flags); }
  operator cudaEvent_t() const { return e_; }

 private:
  cudaEvent_t e_ = nullptr;
};

struct SlotBuf {
  DevBuf<float> d;
  int64_t rows = 0, cols = 0, ld = 0;  // ld: row stride in floats, cols itself when rows == 1
};

// uint8 rank matrix of a feature-matrix slot for the tree walk (se_models.cu): per column the sorted thresholds seen
// so far (<= 255), X8[col][i] = #{thresholds of col strictly below X[col][i]}
struct BinState {
  DevBuf<uint8_t> d8;
  int64_t ld8 = 0, n = 0;
  int d = 0;
  bool valid = false;                      // X8 reflects the current contents of the slot for every column with edges
  std::vector<std::vector<float>> edges;   // per column
  std::vector<char> dirty;
  std::vector<char> fit;                   // per column: the edges are exactly the candidates se_tree_fit_bins set
  DevBuf<float> d_edges;                   // [d][256]
  DevBuf<int32_t> d_nedges;                // [d]
  DevBuf<int32_t> d_cols;                  // [d]
  DevBuf<uint4> d_nodes;
};

}  // namespace se_host

struct se_ctx {
  int device = 0;
  se_host::Stream stream;  // declared first: destroyed after every buffer below
  se_host::Event ev0, ev1;
  bool timing = false;
  double last_ms = 0.0;
  int sms = 132;
  int ctas_per_sm = 8;  // upper bound; launchers scale the grid down for small shards (se_gbm.cu grid_for)
  int64_t launches = 0;
  se_host::SlotBuf slot[SE_NUM_SLOTS];
  se_host::DevBuf<double> d_scal;
  se_host::PinnedBuf<double> h_scal;
  se_host::DevBuf<double> d_partials;
  se_host::DevBuf<unsigned int> d_counter;
  se_host::DevBuf<unsigned char> d_small;
  se_host::PinnedBuf<unsigned char> h_small;  // staging for d_small
  se_host::PinnedBuf<float> h_stage;          // staging for f64 uploads / scaled downloads
  struct {
    bool on = false;
    int64_t n = 0, nv = 0;
    int dim = 1, loss = 0;
    double param = 0.0;
    bool has_w = false;
    bool use_bag = false;
    bool r_current = false;  // SE_SLOT_R holds -g(y, F) of the CURRENT F (squared loss: y - F)
    bool f_owed = false;     // SE_SLOT_F is stale: its value is y - r (residual-mode fused squared round); settle_f
                             // rebuilds it.  Implies r_current.
    // d_sq_carry's parity sq_carry_parity holds this GPU's Σr², Σhr, Σh² over the current R and H as the
    // sq_carry_grid partials of the CTAs of the last residual fused round's update pass, which summed them over what it
    // wrote.  Dropped by every write of Y, F, R or H.
    bool sq_stats_current = false;
    int sq_carry_parity = 0;
    int sq_carry_grid = 0;
    bool sq_last_up = false;  // the last fused round's update pass walked its tiles upwards (ended on the highest)
    // SE_SLOT_R is pending: it holds an older r0, and the residual is r0 after the r_pending fp32 steps in d_rchain
    // along H (carried rounds that stored nothing).  settle_r applies them; nothing else may touch R, or write H,
    // while r_pending > 0.
    int r_pending = 0;
    bool sq_defer_ok = false;  // the last round was carried and R has not been read since: the next may defer
    double wsum = 0.0;
    bool wsum_valid = false;
    double n_global = 0.0, nv_global = 0.0;
    bool counts_valid = false;
  } gbm;
  struct {
    bool on = false;
    int64_t n = 0;
    int K = 2;
    bool real = false;
  } boost;
  struct {
    bool on = false;
    int kind = 0, M = 0, K = 0, dim = 1, loss = 0, width = 1, C = 1;
    int64_t n = 0;
  } agg;
  struct {
    bool on = false;
    int64_t n = 0;
  } boostreg;
  se_host::nccl_comm_t comm = nullptr;
  int nranks = 1, rank = 0;
  // fused NVLink all-reduce: mailboxes of all ranks mapped into this process with CUDA IPC
  bool p2p = false;
  se_host::DevBuf<double> mbox_local;
  std::vector<void*> mbox_peers;      // opened IPC mappings (index = rank; own entry = mbox_local)
  std::vector<char> mbox_ipc;         // 1: mbox_peers[p] came from cudaIpcOpenMemHandle (close it); 0: same-process peer pointer
  se_host::DevBuf<double*> d_mbox_table;  // device copy of the pointer table
  int* d_p2p_err = nullptr;           // device alias of h_p2p_err (mapped pinned host memory: no copy to poll it)
  se_host::MappedBuf<int> h_p2p_err;
  se_host::MappedBuf<int> h_bad_label;  // raised by kernels that met a label / vote outside [0, K)
  int* d_bad_label = nullptr;         // device alias of h_bad_label
  // labels used as class indices are validated once per write: 0 unknown, 1 validation launched (result not yet
  // observed), 2 known good — per label slot (SE_SLOT_Y, SE_SLOT_VY) together with the K they were checked for
  int y_state[2] = {0, 0};
  int y_state_k[2] = {0, 0};
  unsigned long long red_seq = 0;
  bool last_reduce_global = false;    // the kernel just launched already produced cross-GPU sums
  // host mirror of the scalar block (mapped pinned memory written by the reducing kernel's last CTA)
  se_host::MappedBuf<double> h_mirror;  // [kMboxPayload] + ticket word
  double* d_mirror = nullptr;         // device alias
  unsigned long long mirror_ticket = 0;
  bool mirror_valid = false;
  int mirror_off = 0;
  bool use_mirror = true;
  se_host::DevBuf<float> d_ls_u;      // line-search view (signed): u = (2y-1)F, v = (2y-1)h; holds both
  float* d_ls_v = nullptr;            // alias into d_ls_u
  bool ls_packed = false;             // evaluations currently read (u, v) instead of (y, F, h)
  unsigned pass_parity = 0;           // alternates the tile direction of consecutive GBM passes (L2 reuse)
  bool alternate = true;
  int l2_hints = -1;                  // evict_first hints on the GBM streams: -1 by shard size, 0 off, 1 on (SE_L2_HINTS)
  int64_t l2_hint_rows = 0;           // shard size up to which l2_hints = -1 turns them on: 16 B/row of y, F, h, r up to ~2x the L2
  // ---- cooperative whole-round / whole-line-search kernels (se_gbm_fused.cu)
  se_host::DevBuf<se::FusedSync> d_fsync;
  unsigned long long fused_epoch = 0;
  int fused_round = -1;               // squared-loss round in one launch: -1 by shard size, 0 off, 1 on
  int64_t fused_round_max_rows = (int64_t)1 << 40;  // no size limit by default
  int fused_ctas_per_sm = 3;
  int fused_loss_reduce = 0;          // 1: reduce the train loss over the rows even when the closed form applies
  int fused_timing = 0;               // diagnostic: in-kernel %globaltimer stamps of the fused round
  int fused_resident = 1;             // residual rounds reading r carry the statistics pass's tail in shared memory
  // carried rounds leave at most this many steps pending on R before one stores it (0: every round stores r')
  int sq_defer_max = 16;
  se_host::DevBuf<float> d_rchain;    // the pending steps [kSqDeferMax]
  // the squared round's carried statistics: two parities of [kMaxGridPartials / 2][3] CTA partials.  A round stores
  // into the parity its predecessor did not, so its first CTAs to finish never overwrite what its last ones fold.  Not
  // the shared reduction workspace: the partials must outlive the calls between two rounds, a read of R among them.
  se_host::DevBuf<double> d_sq_carry;
  double last_fused_resident_tiles = 0.0;  // tiles per CTA the last fused round carried in shared memory
  double last_fused_us[3] = {0, 0, 0};  // statistics phase, fold+exchange+Brent, update phase
  int ls_mode = 1;                    // non-squared line search: 0 one launch per evaluation (round-1 kernels), 1 one
                                      // persistent launch (device Brent), 2 host Brent over single-evaluation launches of
                                      // the persistent kernel (bit-identity check of mode 1)
  int ls_resident = 1;                // workers keep their first tiles in shared memory
  int ls_ctas_per_sm = 4;
  int clock_khz = 1965000;
  double peer_timeout_ms = 120000.0;  // spin bound of the fused peer exchange (0 = wait forever)
  // diagnostics of the last call (se_ctx_get_option)
  int last_round_fused = 0, last_round_carried = 0, last_round_deferred = 0, last_ls_workers = 0, last_ls_resident = 0, last_ls_passes = 0, last_fused_grid = 0;
  double last_round_stats[3] = {0.0, 0.0, 0.0};
  // newton updates: SE_SLOT_WOUT holds 1/2 hc w; the 1/S_j of each dimension is applied on download
  std::vector<float> wout_scale;
  bool wout_scaled = false;
  // LogLoss with more than kMaxDim classes (se_gbm_generic.cu): buffers sized for the configured dim
  struct {
    int grid = 0;
    se_host::DevBuf<float> d_coef;
    se_host::PinnedBuf<float> h_coef;
    se_host::DevBuf<double> d_partials;  // [grid][dim + 1]
    se_host::DevBuf<double> d_out;       // [dim + 1]
    se_host::PinnedBuf<double> h_out;
    bool pending = false;         // the last GBM launch left its sums in d_out
  } big;
  // binned (uint8) copies of X / VX for the tree walk
  se_host::BinState bins[2];
  int tree_bins = 1;                  // 0: always walk the fp32 matrix
  se_host::DevBuf<unsigned char> d_forest;  // packed chunk of trees for se_forest_predict / se_forest_agg
  se_host::DevBuf<float> d_forest_p;        // se_forest_agg: leaf class probabilities of every node [nodes][K]
  se_host::DevBuf<double> d_forest_acc;     // se_forest_agg: fp64 class totals carried between chunks [C][n]
  int last_forest_chunks = 0;
  int wm_fast = 1;                    // weighted median (M <= 64, weights >= 0): keys-only sort + margin check, exact kernel for the rest
  int64_t wm_list_cap = 0;            // deferred-row list capacity (0: n / 4)
  se_host::DevBuf<unsigned int> d_wm;  // [0] deferred count, [1..] row list
  int last_wm_mode = 0;
  int tree_mask = 1;                  // shallow trees (<= 64 internal nodes): all-nodes comparison kernel over the rank matrix
  int last_tree_mask = 0;
  int last_tree_binned = 0, last_tree_rebinned_cols = 0;
  // the last tree fit's histogram path per level L, in octal digit L: 0 several columns per CTA in shared memory, 1 one
  // column per CTA, 2 one column with opt-in shared memory at 2 CTAs/SM, 3 the same at 1 CTA/SM, 4 global fp64 atomics
  int64_t last_tree_fit_hist = 0;
  int last_forest_fit_batches = 0;    // launch sequences of the last se_forest_fit
  // tree fits (se_tree_fit, se_forest_fit): scratch kept across the rounds of a fit, sized for the most trees at once
  struct {
    se_host::DevBuf<uint16_t> d_nid;  // per tree two [4 nw] node-index buffers (levels alternate)
    se_host::DevBuf<double> d_hist;
    se_host::DevBuf<se::TreeFitNode> d_nodes;  // [trees][kTreeFitHeap]
    se_host::DevBuf<uint2> d_dec;     // [trees][kTreeFitHeap]
    se_host::DevBuf<int32_t> d_cols;  // the trees' subspace columns, then their T + 1 offsets
    int smem_optin = 0;
    se_host::DevBuf<double> d_cw;     // classification: [trees][kTreeFitHeap][kTreeFitMaxClasses]
    se_host::DevBuf<float> d_prob;    // [trees][kTreeFitHeap][kTreeFitMaxClasses]
    se_host::DevBuf<int4> d_prn;      // [trees][kTreeFitHeap]
  } tf;
  struct {  // se_linear_moments: CTA partials, tile tickets and the matrix, kept across calls
    se_host::DevBuf<double> d_part;
    se_host::DevBuf<unsigned int> d_cnt;
    se_host::DevBuf<double> d_out;
  } lm;
  struct {  // se_logistic_stats / se_logistic_loss_grad: the same, kept across the evaluations of a fit
    se_host::DevBuf<double> d_part;
    se_host::DevBuf<unsigned int> d_cnt;
    se_host::DevBuf<double> d_out;
    // se_logistic_loss_grad_batch: the work items and the members' columns and coefficients, staged and on the device
    se_host::PinnedBuf<unsigned char> h_in;
    se_host::DevBuf<unsigned char> d_in;
  } lg;
  std::string err;
  // stopwatch + per-kernel-family timing
  se_host::Event tm0, tm1;
  bool ktiming = false;
  static constexpr int kRing = 128;
  se_host::Event kev[kRing][2];
  int kfam[kRing] = {};
  // a launch timed by its own %globaltimer stamps instead of events: d_kstamp[2 * slot] is CTA 0's entry and
  // [2 * slot + 1] the latest exit of any CTA, in ns (kernel_stamp_slot)
  bool kstamped[kRing] = {};
  se_host::DevBuf<unsigned long long> d_kstamp;
  int kpending = 0;
  double kms[SE_KF_COUNT] = {};
  int64_t kcount[SE_KF_COUNT] = {};
};

namespace se_host {

int fail(se_ctx* ctx, int code, const char* fmt, ...);

#define SE_CUDA(ctx, call)                                                                    \
  do {                                                                                        \
    cudaError_t e__ = (call);                                                                 \
    if (e__ != cudaSuccess)                                                                   \
      return fail(ctx, SE_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call,              \
                  cudaGetErrorString(e__));                                                   \
  } while (0)

#define SE_LAUNCH(ctx, call)                                                                  \
  do {                                                                                        \
    cudaError_t e__ = (call);                                                                 \
    (ctx)->launches++;                                                                        \
    if (e__ != cudaSuccess)                                                                   \
      return fail(ctx, SE_ERR_CUDA, "%s:%d launch %s -> %s", __FILE__, __LINE__, #call,       \
                  cudaGetErrorString(e__));                                                   \
  } while (0)

int drain_kernel_events(se_ctx* ctx);
// With kernel timing on: a slot of the timing ring for a launch that stamps its own start and end (*stamps, nullptr
// with kernel timing off).  CUDA events recorded around a programmatic dependent launch would order it after the
// kernel before it in full, so such a launch is timed from inside instead.
int kernel_stamp_slot(se_ctx* ctx, int family, unsigned long long** stamps);

// launch bracketed by CUDA events on the context stream when kernel timing is on
#define SE_LAUNCH_T(ctx, family, call)                                                        \
  do {                                                                                        \
    int slot__ = -1;                                                                          \
    if ((ctx)->ktiming) {                                                                     \
      if ((ctx)->kpending == se_ctx::kRing) {                                                 \
        int rc__ = drain_kernel_events(ctx);                                                  \
        if (rc__ != SE_OK) return rc__;                                                       \
      }                                                                                       \
      slot__ = (ctx)->kpending;                                                               \
      if (!(ctx)->kev[slot__][0]) {                                                           \
        SE_CUDA(ctx, (ctx)->kev[slot__][0].create());                                         \
        SE_CUDA(ctx, (ctx)->kev[slot__][1].create());                                         \
      }                                                                                       \
      SE_CUDA(ctx, cudaEventRecord((ctx)->kev[slot__][0], (ctx)->stream));                    \
    }                                                                                         \
    SE_LAUNCH(ctx, call);                                                                     \
    if (slot__ >= 0) {                                                                        \
      SE_CUDA(ctx, cudaEventRecord((ctx)->kev[slot__][1], (ctx)->stream));                    \
      (ctx)->kfam[slot__] = (family);                                                         \
      (ctx)->kstamped[slot__] = false;                                                        \
      (ctx)->kpending = slot__ + 1;                                                           \
    }                                                                                         \
  } while (0)

#define SE_TRY(expr)                \
  do {                              \
    int rc__ = (expr);              \
    if (rc__ != SE_OK) return rc__; \
  } while (0)

#define SE_REQUIRE(ctx, cond, code, ...) \
  do {                                   \
    if (!(cond)) return fail(ctx, code, __VA_ARGS__); \
  } while (0)

// ---- shared by the entry points (se_api_ctx.cu unless noted)
NcclApi& nccl();
int begin(se_ctx* ctx);
int end(se_ctx* ctx);
// exchange = true: the launched kernel ends in block_reduce_publish/peer_exchange (sum); it then performs
// the cross-GPU reduction itself over peer memory and the NCCL all-reduce is skipped.
se::RedWs red_ws(se_ctx* ctx, int out_offset = 0, bool exchange = true);
int allreduce_dev(se_ctx* ctx, int off, int count, int op = kNcclSum);
int check_labels(se_ctx* ctx);
int fetch_scalars(se_ctx* ctx, int off, int count, double* out, int op = kNcclSum);
int settle_r(se_ctx* ctx);
int settle_f(se_ctx* ctx);
int write_slot(se_ctx* ctx, int slot);
int read_slot(se_ctx* ctx, int slot);
int slot_alloc2d(se_ctx* ctx, int slot, int64_t rows, int64_t cols);
int out_rows(se_ctx* ctx, int slot, int row, int count, int64_t n, float** out, int64_t* ld);
int ensure_labels_checked(se_ctx* ctx, int which, int K, int64_t n);  // se_api_gbm.cu
int wm_weight_mode(const double* w, int M);                           // se_api_boost.cu
// the rank matrix (se_api_trees.cu)
bool bins_ensure(BinState& B, const SlotBuf& X);
int bins_rerank(se_ctx* ctx, BinState& B, const SlotBuf& X);
int bins_prepare(se_ctx* ctx, int which, const SlotBuf& X, int n_nodes, const int32_t* col, const float* thr);

}  // namespace se_host
