// se_api_slots.cu — host side of the slot entry points: allocation, uploads and downloads, fill, sum, quantile.
#include "se_ctx.h"

using namespace se;
using namespace se_host;

namespace {

// logical flat [rows][cols] range -> per-row physical segments
template <class Fn>
int for_segments(se_ctx* ctx, const SlotBuf& s, int64_t count, int64_t offset, Fn fn) {
  SE_REQUIRE(ctx, s.d, SE_ERR_STATE, "slot not allocated");
  SE_REQUIRE(ctx, offset >= 0 && count >= 0 && offset + count <= s.rows * s.cols, SE_ERR_ARG,
             "range [%lld,+%lld) outside slot of %lld elements", (long long)offset,
             (long long)count, (long long)(s.rows * s.cols));
  int64_t done = 0;
  while (done < count) {
    const int64_t pos = offset + done;
    const int64_t r = (s.cols > 0) ? pos / s.cols : 0, c = (s.cols > 0) ? pos % s.cols : 0;
    int64_t len = s.cols - c;
    if (len > count - done) len = count - done;
    SE_TRY(fn(s.d + r * s.ld + c, done, len));
    done += len;
  }
  return SE_OK;
}

}  // namespace

// ---- slots -------------------------------------------------------------------------------------
int se_slot_alloc(se_ctx* ctx, int slot, int64_t count) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  return slot_alloc2d(ctx, slot, 1, count);
}

int se_slot_alloc2d(se_ctx* ctx, int slot, int64_t rows, int64_t cols) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  return slot_alloc2d(ctx, slot, rows, cols);
}

int se_slot_free(se_ctx* ctx, int slot) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, slot >= 0 && slot < SE_NUM_SLOTS, SE_ERR_ARG, "bad slot %d", slot);
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_TRY(write_slot(ctx, slot));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  SE_CUDA(ctx, ctx->slot[slot].d.reset());
  ctx->slot[slot] = SlotBuf();
  if (slot == SE_SLOT_X) ctx->bins[0] = BinState();
  if (slot == SE_SLOT_VX) ctx->bins[1] = BinState();
  return SE_OK;
}

int se_slot_info(const se_ctx* ctx, int slot, void** device_ptr, int64_t* count) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  if (slot < 0 || slot >= SE_NUM_SLOTS) return fail(nullptr, SE_ERR_ARG, "bad slot %d", slot);
  if (device_ptr) {
    // the caller may read or write through the raw pointer
    se_ctx* mctx = const_cast<se_ctx*>(ctx);
    const int64_t launches = ctx->launches;
    SE_TRY(write_slot(mctx, slot));
    // F was just rebuilt or R settled: the caller's own stream may touch the slot next
    if (ctx->launches != launches) SE_CUDA(mctx, cudaStreamSynchronize(ctx->stream));
    *device_ptr = ctx->slot[slot].d;
  }
  if (count) *count = ctx->slot[slot].rows * ctx->slot[slot].cols;
  return SE_OK;
}

int se_slot_layout(const se_ctx* ctx, int slot, int64_t* rows, int64_t* cols, int64_t* ld) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  if (slot < 0 || slot >= SE_NUM_SLOTS) return fail(nullptr, SE_ERR_ARG, "bad slot %d", slot);
  if (rows) *rows = ctx->slot[slot].rows;
  if (cols) *cols = ctx->slot[slot].cols;
  if (ld) *ld = ctx->slot[slot].ld;
  return SE_OK;
}

int se_upload(se_ctx* ctx, int slot, const float* host, int64_t count, int64_t offset) {
  if (!ctx || !host) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, slot >= 0 && slot < SE_NUM_SLOTS, SE_ERR_ARG, "bad slot %d", slot);
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_TRY(write_slot(ctx, slot));
  SE_TRY(for_segments(ctx, ctx->slot[slot], count, offset, [&](float* d, int64_t done, int64_t len) {
    SE_CUDA(ctx, cudaMemcpyAsync(d, host + done, sizeof(float) * len, cudaMemcpyHostToDevice, ctx->stream));
    return SE_OK;
  }));
  // host buffers are borrowed for the duration of the call only
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return SE_OK;
}

int se_upload_f64(se_ctx* ctx, int slot, const double* host, int64_t count, int64_t offset) {
  if (!ctx || !host) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, slot >= 0 && slot < SE_NUM_SLOTS, SE_ERR_ARG, "bad slot %d", slot);
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_TRY(write_slot(ctx, slot));
  // narrow on the host (halves PCIe bytes) through pinned staging, in chunks
  const int64_t chunk = 1 << 22;
  SE_CUDA(ctx, ctx->h_stage.grow((size_t)chunk));
  SE_TRY(for_segments(ctx, ctx->slot[slot], count, offset, [&](float* d, int64_t done, int64_t len) {
    for (int64_t c0 = 0; c0 < len; c0 += chunk) {
      const int64_t m = (len - c0 < chunk) ? len - c0 : chunk;
      for (int64_t i = 0; i < m; ++i) ctx->h_stage[i] = (float)host[done + c0 + i];
      SE_CUDA(ctx, cudaMemcpyAsync(d + c0, ctx->h_stage, sizeof(float) * m, cudaMemcpyHostToDevice, ctx->stream));
      SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return SE_OK;
  }));
  return SE_OK;
}

int se_upload_rowmajor(se_ctx* ctx, int slot, const float* host, int64_t n_rows, int d, int64_t row_offset) {
  if (!ctx || (!host && n_rows > 0)) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, slot >= 0 && slot < SE_NUM_SLOTS, SE_ERR_ARG, "bad slot %d", slot);
  const SlotBuf& X = ctx->slot[slot];
  SE_REQUIRE(ctx, X.d && X.rows == d, SE_ERR_STATE, "slot %d must be allocated as [%d][n] (has [%lld][%lld])", slot, d,
             (long long)X.rows, (long long)X.cols);
  SE_REQUIRE(ctx, n_rows >= 0 && row_offset >= 0 && row_offset + n_rows <= X.cols, SE_ERR_ARG,
             "rows [%lld,+%lld) outside the slot's %lld rows", (long long)row_offset, (long long)n_rows, (long long)X.cols);
  if (n_rows == 0) return SE_OK;
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_TRY(write_slot(ctx, slot));
  // ~32 MB chunks, whole rows, multiple of 32 rows
  int64_t chunk_rows = (int64_t)(32u << 20) / ((int64_t)d * (int64_t)sizeof(float));
  chunk_rows = (chunk_rows / 32) * 32;
  if (chunk_rows < 32) chunk_rows = 32;
  if (chunk_rows > n_rows) chunk_rows = n_rows;
  const size_t chunk_floats = (size_t)chunk_rows * d;
  cudaPointerAttributes attr;
  const bool pinned_src = (cudaPointerGetAttributes(&attr, host) == cudaSuccess && attr.type == cudaMemoryTypeHost);
  cudaGetLastError();
  Stream copy_stream;
  DevBuf<float> dstage[2];
  PinnedBuf<float> hstage[2];
  Event copied[2], consumed[2];
  struct Drain {  // declared last: on every return both streams are done with the staging buffers before they are freed
    const Stream& copy;
    cudaStream_t stream;
    ~Drain() {
      if (copy) cudaStreamSynchronize(copy);
      cudaStreamSynchronize(stream);
    }
  } drain{copy_stream, ctx->stream};
  SE_CUDA(ctx, copy_stream.create(cudaStreamNonBlocking));
  for (int i = 0; i < 2; ++i) {
    SE_CUDA(ctx, dstage[i].grow(chunk_floats));
    if (!pinned_src) SE_CUDA(ctx, hstage[i].grow(chunk_floats));
    SE_CUDA(ctx, copied[i].create(cudaEventDisableTiming));
    SE_CUDA(ctx, consumed[i].create(cudaEventDisableTiming));
  }
  int64_t done = 0;
  for (int c = 0; done < n_rows; ++c) {
    const int b = c & 1;
    const int64_t rows = (n_rows - done < chunk_rows) ? n_rows - done : chunk_rows;
    const size_t bytes = (size_t)rows * d * sizeof(float);
    if (c >= 2) SE_CUDA(ctx, cudaEventSynchronize(consumed[b]));  // staging buffers of chunk c-2 are free again
    const float* src = host + done * d;
    if (!pinned_src) {
      memcpy(hstage[b], src, bytes);  // overlaps the DMA of chunk c-1 and the transpose of chunk c-2
      src = hstage[b];
    }
    SE_CUDA(ctx, cudaMemcpyAsync(dstage[b], src, bytes, cudaMemcpyHostToDevice, copy_stream));
    SE_CUDA(ctx, cudaEventRecord(copied[b], copy_stream));
    SE_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, copied[b], 0));
    const cudaError_t le = launch_transpose_rows(dstage[b], rows, d, X.d, X.ld, row_offset + done, ctx->stream);
    ctx->launches++;
    SE_CUDA(ctx, le);
    SE_CUDA(ctx, cudaEventRecord(consumed[b], ctx->stream));
    done += rows;
  }
  return SE_OK;
}

int se_download(se_ctx* ctx, int slot, float* host, int64_t count, int64_t offset) {
  if (!ctx || !host) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, slot >= 0 && slot < SE_NUM_SLOTS, SE_ERR_ARG, "bad slot %d", slot);
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_TRY(read_slot(ctx, slot));
  SE_TRY(for_segments(ctx, ctx->slot[slot], count, offset, [&](float* d, int64_t done, int64_t len) {
    SE_CUDA(ctx, cudaMemcpyAsync(host + done, d, sizeof(float) * len, cudaMemcpyDeviceToHost, ctx->stream));
    return SE_OK;
  }));
  SE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (slot == SE_SLOT_WOUT && ctx->wout_scaled) {
    // newton base-learner weights: 1/2 hc w on the device, x 1/S_dim here (GBMRegressor.scala:379)
    const int64_t cols = ctx->slot[slot].cols;
    for (int64_t i = 0; i < count; ++i) {
      const size_t j = (size_t)(cols > 0 ? (offset + i) / cols : 0);
      if (j < ctx->wout_scale.size()) host[i] *= ctx->wout_scale[j];
    }
  }
  return check_labels(ctx);  // e.g. the probabilities of an aggregation that met a vote outside [0, K)
}

int se_download_scaled(se_ctx* ctx, int slot, double scale, float* host, int64_t count, int64_t offset) {
  if (!ctx || !host) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_TRY(se_download(ctx, slot, host, count, offset));
  const float s = (float)scale;
  for (int64_t i = 0; i < count; ++i) host[i] *= s;
  return SE_OK;
}

int se_fill(se_ctx* ctx, int slot, float value, int64_t count, int64_t offset) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, slot >= 0 && slot < SE_NUM_SLOTS, SE_ERR_ARG, "bad slot %d", slot);
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_TRY(write_slot(ctx, slot));
  return for_segments(ctx, ctx->slot[slot], count, offset, [&](float* d, int64_t, int64_t len) {
    SE_LAUNCH(ctx, launch_fill(d, value, len, ctx->sms, ctx->stream));
    return SE_OK;
  });
}

int se_copy_slot(se_ctx* ctx, int dst_slot, int src_slot) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, dst_slot >= 0 && dst_slot < SE_NUM_SLOTS && src_slot >= 0 && src_slot < SE_NUM_SLOTS,
             SE_ERR_ARG, "bad slot");
  const SlotBuf &d = ctx->slot[dst_slot], &s = ctx->slot[src_slot];
  SE_REQUIRE(ctx, d.d && s.d && d.rows == s.rows && d.cols == s.cols, SE_ERR_STATE, "slot shapes differ");
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_TRY(read_slot(ctx, src_slot));
  SE_TRY(write_slot(ctx, dst_slot));
  SE_CUDA(ctx, cudaMemcpyAsync(d.d, s.d, sizeof(float) * (size_t)(s.rows * s.ld), cudaMemcpyDeviceToDevice, ctx->stream));
  return SE_OK;
}

int se_copy_rows(se_ctx* ctx, int dst_slot, int dst_row, int src_slot, int src_row, int count) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, dst_slot >= 0 && dst_slot < SE_NUM_SLOTS && src_slot >= 0 && src_slot < SE_NUM_SLOTS,
             SE_ERR_ARG, "bad slot");
  const SlotBuf &d = ctx->slot[dst_slot], &s = ctx->slot[src_slot];
  SE_REQUIRE(ctx, d.d && s.d && d.cols == s.cols, SE_ERR_STATE, "slots %d and %d do not hold rows of the same length",
             dst_slot, src_slot);
  SE_REQUIRE(ctx, count >= 0 && src_row >= 0 && dst_row >= 0 && (int64_t)src_row + count <= s.rows &&
             (int64_t)dst_row + count <= d.rows, SE_ERR_ARG, "rows %d..%d of slot %d into rows %d.. of slot %d: out of range",
             src_row, src_row + count - 1, src_slot, dst_row, dst_slot);
  SE_REQUIRE(ctx, dst_slot != src_slot || count == 0 || src_row + count <= dst_row || dst_row + count <= src_row,
             SE_ERR_ARG, "overlapping rows");
  if (count == 0 || s.cols == 0) return SE_OK;
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_TRY(read_slot(ctx, src_slot));
  SE_TRY(write_slot(ctx, dst_slot));
  SE_CUDA(ctx, cudaMemcpy2DAsync(d.d + (int64_t)dst_row * d.ld, sizeof(float) * (size_t)d.ld, s.d + (int64_t)src_row * s.ld,
                                 sizeof(float) * (size_t)s.ld, sizeof(float) * (size_t)s.cols, (size_t)count,
                                 cudaMemcpyDeviceToDevice, ctx->stream));
  return SE_OK;
}

int se_fill_synthetic(se_ctx* ctx, int slot, int kind, uint64_t seed, double a, double b, int64_t count,
                      int64_t offset) {
  if (!ctx) return fail(nullptr, SE_ERR_ARG, "null context");
  SE_REQUIRE(ctx, slot >= 0 && slot < SE_NUM_SLOTS, SE_ERR_ARG, "bad slot %d", slot);
  SE_REQUIRE(ctx, kind >= 0 && kind <= 3, SE_ERR_ARG, "bad synthetic kind %d", kind);
  SE_CUDA(ctx, cudaSetDevice(ctx->device));
  SE_TRY(write_slot(ctx, slot));
  return for_segments(ctx, ctx->slot[slot], count, offset, [&](float* d, int64_t done, int64_t len) {
    SE_LAUNCH(ctx, launch_fill_synthetic(d, kind, seed, a, b, len, offset + done, ctx->sms, ctx->stream));
    return SE_OK;
  });
}

int se_slot_sum(se_ctx* ctx, int slot, int64_t count, double* out) {
  if (!ctx || !out) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, slot >= 0 && slot < SE_NUM_SLOTS, SE_ERR_ARG, "bad slot %d", slot);
  const SlotBuf& s = ctx->slot[slot];
  SE_REQUIRE(ctx, s.d && s.rows == 1 && count <= s.cols, SE_ERR_STATE, "slot %d is not a [n] vector of >= %lld", slot, (long long)count);
  SE_TRY(begin(ctx));
  SE_TRY(read_slot(ctx, slot));
  SE_LAUNCH(ctx, launch_sum(s.d, count, red_ws(ctx), ctx->ctas_per_sm, ctx->sms, ctx->stream));
  return fetch_scalars(ctx, 0, 1, out);
}

int se_quantile(se_ctx* ctx, int which, int slot, int64_t count, double q, double* out) {
  if (!ctx || !out) return fail(ctx, SE_ERR_ARG, "null argument");
  SE_REQUIRE(ctx, q >= 0.0 && q <= 1.0, SE_ERR_ARG, "quantile %g outside [0,1]", q);
  const float *a = nullptr, *b = nullptr;
  int64_t n = count;
  if (which == 1) {
    SE_REQUIRE(ctx, ctx->gbm.on && ctx->gbm.dim == 1, SE_ERR_STATE, "|y - F| quantile needs a dim-1 GBM problem");
    a = ctx->slot[SE_SLOT_Y].d;
    b = ctx->slot[SE_SLOT_F].d;
    n = ctx->gbm.n;
  } else {
    SE_REQUIRE(ctx, slot >= 0 && slot < SE_NUM_SLOTS, SE_ERR_ARG, "bad slot %d", slot);
    const SlotBuf& s = ctx->slot[slot];
    SE_REQUIRE(ctx, s.d && s.rows == 1 && count <= s.cols, SE_ERR_STATE, "slot %d is not a [n] vector of >= %lld", slot, (long long)count);
    a = s.d;
  }
  SE_TRY(begin(ctx));
  SE_TRY(read_slot(ctx, which == 1 ? SE_SLOT_F : slot));
  double total = (double)n;
  SE_TRY(se_comm_allreduce_host(ctx, &total, 1));
  SE_REQUIRE(ctx, total >= 1.0, SE_ERR_ARG, "quantile of an empty column");
  // 1-based target rank: ceil(q·N), at least 1
  double rank = ceil(q * total);
  if (rank < 1.0) rank = 1.0;
  uint32_t prefix = 0, mask = 0;
  double hist[256];
  for (int shift = 24; shift >= 0; shift -= 8) {
    SE_CUDA(ctx, cudaMemsetAsync(ctx->d_scal + kScalHist, 0, sizeof(double) * 256, ctx->stream));
    ctx->last_reduce_global = false;  // histogram bins: summed by NCCL
    SE_LAUNCH_T(ctx, SE_KF_OTHER, launch_radix_hist(a, b, n, prefix, mask, shift, ctx->d_scal + kScalHist, ctx->sms, ctx->stream));
    SE_TRY(fetch_scalars(ctx, kScalHist, 256, hist));
    double cum = 0.0;
    int bin = 255;
    for (int i = 0; i < 256; ++i) {
      if (cum + hist[i] >= rank) { bin = i; break; }
      cum += hist[i];
    }
    rank -= cum;
    prefix |= (uint32_t)bin << shift;
    mask |= 0xFFu << shift;
  }
  // invert the order-preserving key
  const uint32_t bits = (prefix & 0x80000000u) ? (prefix & 0x7FFFFFFFu) : ~prefix;
  float v;
  memcpy(&v, &bits, sizeof(v));
  *out = (double)v;
  return SE_OK;
}
