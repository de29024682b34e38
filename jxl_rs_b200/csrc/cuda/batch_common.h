// Pieces shared by the VarDCT batch (batch.cc) and the Modular batch (modular_batch.cc): error plumbing, pooled
// device buffers, the pinned staging arena and the per-device context.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "../../../include/jxg.h"

namespace jxgpu {
int sm_count();  // kernels.cu

namespace detail {

extern thread_local std::string g_error;
inline int set_error(int code, const std::string& what) {
  g_error = what;
  return code;
}
#define CUDA_TRY(expr)                                                                        \
  do {                                                                                        \
    cudaError_t e__ = (expr);                                                                 \
    if (e__ != cudaSuccess) return set_error(JXG_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e__)); \
  } while (0)

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes) {
    if (bytes <= cap) return 0;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    if (cudaMalloc(&p, want) != cudaSuccess) return set_error(JXG_ERR_CUDA, "cudaMalloc of " + std::to_string(want) + " bytes failed");
    cap = want;
    return 0;
  }
  ~DevBuf() {
    if (p) cudaFree(p);
  }
};

// Growable pinned host arena: the batch blob is assembled directly in pinned
// memory so that the upload is one cudaMemcpyAsync.
struct PinnedArena {
  uint8_t* p = nullptr;
  size_t size = 0, cap = 0;
  int fill = -1;  // the context's pool fill byte for this batch (jxg_context_set_pool_fill), -1: off
  ~PinnedArena() {
    if (p) cudaFreeHost(p);
  }
  bool reserve(size_t want) {
    if (want <= cap) return true;
    size_t ncap = std::max(want, cap * 2);
    ncap = std::max<size_t>(ncap, 1 << 20);
    uint8_t* np = nullptr;
    if (cudaHostAlloc(reinterpret_cast<void**>(&np), ncap, cudaHostAllocDefault) != cudaSuccess) return false;
    if (p) {
      memcpy(np, p, size);
      cudaFreeHost(p);
    }
    if (fill >= 0) memset(np + size, fill, ncap - size);
    p = np;
    cap = ncap;
    return true;
  }
  // Deferred mode (jxg_batch_set_deferred_copy): large copies are only recorded here and executed by
  // flush() on several host threads right before the upload; sources must stay valid until then.
  struct Pending {
    size_t off;
    const void* src;
    size_t bytes;
  };
  std::vector<Pending> pending;
  int deferred_threads = 0;
  // returns offset; pads with zeros up to `align`, appends `bytes` (+ `tail_zero` zero bytes)
  int64_t append(const void* src, size_t bytes, size_t align = 16, size_t tail_zero = 0) {
    size_t off = (size + align - 1) / align * align;
    size_t end = off + bytes + tail_zero;
    if (!reserve(end)) return -1;
    memset(p + size, 0, off - size);
    if (bytes) {
      if (deferred_threads > 0 && bytes >= 4096) pending.push_back(Pending{off, src, bytes});
      else memcpy(p + off, src, bytes);
    }
    if (tail_zero) memset(p + off + bytes, 0, tail_zero);
    size = end;
    return int64_t(off);
  }
  void flush() {
    if (pending.empty()) return;
    const int nt = std::max(1, std::min<int>(deferred_threads, int(pending.size())));
    std::atomic<size_t> next{0};
    auto work = [&] {
      for (;;) {
        const size_t i = next.fetch_add(8);
        if (i >= pending.size()) return;
        for (size_t j = i; j < std::min(i + 8, pending.size()); j++) memcpy(p + pending[j].off, pending[j].src, pending[j].bytes);
      }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < nt; t++) th.emplace_back(work);
    work();
    for (auto& t : th) t.join();
    pending.clear();
  }
};

// One D2H stream per DEVICE, shared by all its contexts: output copies leave in launch order. With a copy stream per
// context the copies of all batches in flight share the host link evenly, so they all end together, all contexts come
// free together and the next batches start together: a convoy that leaves the SMs idle for the length of the D2H tail.
// First in, first out retires the oldest batch early and keeps the launches staggered. Created on first use; nullptr
// when that fails.
cudaStream_t device_d2h_stream(int device);

struct Context {
  int device = 0;
  cudaStream_t stream = nullptr;
  // Output copies of a batch leave on the device's D2H stream (device_d2h_stream) in up to kMaxRanges frame ranges: the
  // copy of a finished range overlaps the filtering of the later ones.
  cudaStream_t d2h = nullptr;
  static constexpr int kMaxRanges = 8;
  cudaEvent_t range_done[kMaxRanges] = {nullptr}, copy_done = nullptr;
  DevBuf dequant_default, dequant_default_off, natural_orders, natural_order_off;
  // Pools reused by successive batches (one live batch per context): device
  // intermediates and the pinned staging arena survive jxg_batch_end so that a
  // steady-state decode loop does no cudaMalloc / cudaHostAlloc.
  PinnedArena blob;
  DevBuf d_blob, d_coeffs, d_planes_a, d_status, d_out, d_desc, d_nblk, d_cls_n, d_cls_list, d_orient, d_lzwin,
      d_modular_lzwin, d_modular_wp;
  int pool_fill = -1;  // test hook (jxg_context_set_pool_fill): byte written over the pools before each run, -1: off
  int sm_budget = 0;   // test hook (jxg_context_set_sm_budget): SMs every schedule of the context assumes, 0: the device's
  bool batch_live = false;
  // pinned status readback buffer, owned by the context: cudaHostAlloc / cudaFreeHost synchronise the whole
  // device, so they must not happen per batch when batches of several contexts are in flight
  int32_t* status_host = nullptr;
  size_t status_cap = 0;
};

// SMs the launch schedules of the context's batches are sized for: the device's count, or the test hook's budget.
inline uint32_t schedule_sms(const Context* cx) {
  return cx->sm_budget > 0 ? uint32_t(cx->sm_budget) : uint32_t(sm_count());
}

// What a batch of either engine holds besides its frames. ev0: before the upload; ev1: behind everything of the last run.
struct BatchCore {
  Context* ctx = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  bool uploaded = false;
  cudaStream_t last_stream = nullptr;  // stream of the last run / rerun (the context's or the caller's)
  int32_t* status_host = nullptr;      // pinned (context-owned): a D2H copy into pageable memory would block the run
  size_t status_n = 0;
  uint64_t launches = 0, h2d = 0, d2h = 0;
};

// One live batch per context. Creates ev0, ev1 and, if `extra` is given, the engine's own timing event; on failure the
// context stays free.
inline int batch_begin(BatchCore& b, Context* cx, cudaEvent_t* extra = nullptr) {
  if (cx->batch_live) return set_error(JXG_ERR_ARGUMENT, "one live batch per context: end the previous batch first");
  CUDA_TRY(cudaSetDevice(cx->device));
  b.ctx = cx;
  cx->blob.size = 0;
  cx->blob.pending.clear();
  cx->blob.deferred_threads = 0;
  cx->blob.fill = cx->pool_fill;
  if (cx->pool_fill >= 0 && cx->blob.p) memset(cx->blob.p, cx->pool_fill, cx->blob.cap);
  cudaError_t e = cudaEventCreate(&b.ev0);
  if (e == cudaSuccess) e = cudaEventCreate(&b.ev1);
  if (e == cudaSuccess && extra) e = cudaEventCreate(extra);
  if (e != cudaSuccess) {
    for (cudaEvent_t ev : {b.ev0, b.ev1, extra ? *extra : nullptr})
      if (ev) cudaEventDestroy(ev);
    return set_error(JXG_ERR_CUDA, std::string("cudaEventCreate: ") + cudaGetErrorString(e));
  }
  cx->batch_live = true;  // only once nothing can fail any more
  return 0;
}

// The stream of a run or rerun, `cuda_stream` of the entry point: the caller's, or else the context's; kept as last_stream.
inline cudaStream_t batch_stream(BatchCore& b, void* cuda_stream) {
  b.last_stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : b.ctx->stream;
  return b.last_stream;
}

// Waits for the last run (the context's pools are then free for the next batch); the engine destroys its own events.
inline void batch_end(BatchCore& b) {
  cudaSetDevice(b.ctx->device);
  if (b.uploaded) cudaEventSynchronize(b.ev1);
  cudaEventDestroy(b.ev0);
  cudaEventDestroy(b.ev1);
  b.ctx->batch_live = false;
}

// The batch's status words: the first n of the context's pinned status buffer (grown if needed), zeroed.
inline int batch_status(BatchCore& b, size_t n) {
  Context* cx = b.ctx;
  if (n > cx->status_cap) {
    if (cx->status_host) cudaFreeHost(cx->status_host);
    cx->status_host = nullptr;
    cx->status_cap = 0;
    const size_t cap = std::max<size_t>(n * 2, 1 << 16);
    CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(&cx->status_host), cap * 4, cudaHostAllocDefault));
    cx->status_cap = cap;
  }
  b.status_host = cx->status_host;
  b.status_n = n;
  memset(b.status_host, 0, n * 4);
  return 0;
}

// The first non-zero status word of a stream as the batch's error: "<what><frame> group <group>" of that stream. The
// words after the streams' (status_n may count more) are not statuses.
template <typename Stream>
int batch_first_failure(const BatchCore& b, const std::vector<Stream>& streams, const char* what, uint32_t* frame, uint32_t* group) {
  for (size_t i = 0; i < std::min(b.status_n, streams.size()); i++)
    if (b.status_host[i] != 0) {
      if (frame) *frame = streams[i].frame;
      if (group) *group = streams[i].group;
      return set_error(b.status_host[i], what + std::to_string(streams[i].frame) + " group " + std::to_string(streams[i].group));
    }
  return 0;
}

// Appends a batch table to the pinned blob, so that it travels with the one H2D copy; `off`: its offset in the blob.
template <typename T>
bool batch_table(PinnedArena& blob, const std::vector<T>& v, uint64_t& off) {
  const int64_t o = blob.append(v.empty() ? nullptr : v.data(), v.size() * sizeof(T), 16, 16);
  off = uint64_t(o);
  return o >= 0;
}

// Test hook (jxg_context_set_pool_fill): writes the fill byte over the whole capacity of every pool of the context, on
// the stream of the upload, so that a kernel reading a word its batch did not write sees the pattern, not what an
// earlier batch left there. A run fills d_blob as well (the upload then overwrites its own part); a rerun keeps it.
inline int fill_pools(Context* cx, cudaStream_t s, bool with_blob) {
  if (cx->pool_fill < 0) return 0;
  for (DevBuf* d : {&cx->d_blob, &cx->d_coeffs, &cx->d_planes_a, &cx->d_status, &cx->d_out, &cx->d_desc, &cx->d_nblk,
                    &cx->d_cls_n, &cx->d_cls_list, &cx->d_orient, &cx->d_lzwin, &cx->d_modular_lzwin, &cx->d_modular_wp})
    if (d->p && (with_blob || d != &cx->d_blob)) CUDA_TRY(cudaMemsetAsync(d->p, cx->pool_fill, d->cap, s));
  return 0;
}

// Read taps copy device buffers of the last run, which may have run on a caller's stream: they wait for its ev1.
inline int batch_wait_last_run(const BatchCore& b) {
  CUDA_TRY(cudaSetDevice(b.ctx->device));
  CUDA_TRY(cudaEventSynchronize(b.ev1));
  return 0;
}

template <typename T>
int upload(DevBuf& b, const std::vector<T>& v, cudaStream_t s) {
  if (int r = b.ensure(std::max<size_t>(v.size() * sizeof(T), 16))) return r;
  if (!v.empty()) CUDA_TRY(cudaMemcpyAsync(b.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, s));
  return 0;
}

}  // namespace detail
}  // namespace jxgpu
