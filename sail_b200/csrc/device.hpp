// device.hpp -- context, HBM buffers, device-resident columns/batches and Arrow C (Device) Data
// Interface import/export.  Data layout in HBM is Arrow's own (values buffers, LSB bitmaps,
// 16-byte string views) so an imported device batch is used in place; the only normalisation is
// that string views longer than 12 bytes carry an absolute device pointer in their last 8 bytes
// ("resolved views") so kernels can dereference them without a buffer table.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <functional>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "common.hpp"

namespace sg {

#define SG_CUDA(call)                                                                                  \
  do {                                                                                                 \
    cudaError_t _e = (call);                                                                           \
    if (_e != cudaSuccess)                                                                             \
      ::sg::fail(SAILGPU_ERR_CUDA, std::string("CUDA error: ") + cudaGetErrorString(_e) + " at " #call); \
  } while (0)

struct PackPool;

struct Ctx {
  int device = 0;
  int sm_count = 132;
  size_t max_smem = 227 * 1024;
  cudaStream_t stream = nullptr;        // compute stream
  // compiled pipelines shared by every operator instance created from the same spec over the same schema (engine.cu): an
  // executor creates one operator per partition and per query run, the tile program / specialised kernel is built once
  std::map<std::string, std::shared_ptr<void>> shared_objects;
  PackPool* pack_pool = nullptr;        // host-batch ingest: packer threads, pinned staging, copy streams (h2d.cu)
  std::string last_error;
  // One compute stream, one allocation cache and one D2H bounce buffer per context: calls that touch the device are
  // serialised per context (capi.cu takes this lock), different contexts run concurrently.
  std::recursive_mutex mu;
  void* nccl_comm = nullptr;
  int rank = 0, world = 1;
  std::atomic<bool> dead{false};     // context destroyed; buffers that outlive it fall back to cudaFree
  // metrics shared by all ops of the context
  std::atomic<uint64_t> h2d_bytes{0}, d2h_bytes{0};
  // all-to-all exchanges of this context: bytes put on / taken off NVLink and device time of the grouped send/recv
  std::atomic<uint64_t> exch_sent_bytes{0}, exch_recv_bytes{0}, exch_ns{0}, exch_calls{0};
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> exch_events;      // grouped send/recv of finished exchanges, not yet read (resolve_exchange_timing)
  // small device->host exports (operator results of a few rows) bounce through one pinned block so that all their
  // copies are asynchronous and the export costs one synchronisation instead of one per buffer
  struct D2HItem { void* host; size_t off, bytes; };
  void* d2h_stage = nullptr;
  size_t d2h_used = 0;
  std::vector<D2HItem> d2h_pending;
  static constexpr size_t D2H_STAGE_BYTES = 1 << 20, D2H_SMALL = 64 << 10;
  // Size-class cache in front of the stream-ordered pool.  Everything (allocation, copies, kernels) runs on `stream`,
  // so a block released by the host can be handed to the next request of its size class at once: its new first use is
  // ordered after the old last use.  Operators re-allocate the same sizes batch after batch; going to the driver's
  // pool each time costs microseconds per call and, when differently sized operators alternate, fresh mappings of
  // gigabytes (a join became several times slower after an aggregation had reshaped the pool).
  std::mutex cache_mu;
  std::unordered_map<size_t, std::vector<void*>> cache;
  size_t cached_bytes = 0;
  static constexpr size_t CACHE_LIMIT = 64ull << 30;
  static size_t size_class(size_t padded) { return padded <= (1u << 20) ? (padded + 511) & ~(size_t)511 : (padded + (1u << 20) - 1) & ~(size_t)((1u << 20) - 1); }
  // times the host waited for `stream` to drain (stream_sync); capi.cu charges each call's share to the operator it served
  std::atomic<uint64_t> host_syncs{0};
  // pinned 128-byte slots for the asynchronous read-backs of operators (pinned_slot_acquire / release): one block per context,
  // because pinning memory per operator would cost more than the round trips it saves
  static constexpr size_t PINNED_SLOT = 128, PINNED_SLOTS = 512;
  void* pinned_block = nullptr;
  std::vector<uint32_t> pinned_free;
  uint32_t pinned_next = 0;
  // the ZSTD work of the last sailgpu_parquet_decode call (parquet.cu; sailgpu_parquet_stats): pages, bytes they decompressed
  // to, bytes read back, and the device time of the decompression launch and of the read-back (CUDA events)
  struct ParquetZstd { uint64_t pages = 0, out_bytes = 0, image_bytes = 0; float decompress_ms = 0, readback_ms = 0; };
  ParquetZstd parquet_zstd;
};

// Waits until everything queued on the context's stream has run.  Every such wait leaves the device without work until the
// host queues more, so the library counts them (gpu.host_syncs).
inline void stream_sync(Ctx* ctx) {
  ctx->host_syncs++;
  SG_CUDA(cudaStreamSynchronize(ctx->stream));
}

// A pinned, device-mapped host slot of Ctx::PINNED_SLOT bytes (kernels may write it through cudaHostGetDevicePointer); null
// when pinning fails.
inline void* pinned_slot_acquire(Ctx* ctx) {
  if (!ctx->pinned_block) {
    if (cudaHostAlloc(&ctx->pinned_block, Ctx::PINNED_SLOT * Ctx::PINNED_SLOTS, cudaHostAllocMapped) != cudaSuccess) { cudaGetLastError(); ctx->pinned_block = nullptr; return nullptr; }
  }
  uint32_t i;
  if (!ctx->pinned_free.empty()) { i = ctx->pinned_free.back(); ctx->pinned_free.pop_back(); }
  else if (ctx->pinned_next < Ctx::PINNED_SLOTS) i = ctx->pinned_next++;
  else return nullptr;
  return static_cast<uint8_t*>(ctx->pinned_block) + (size_t)i * Ctx::PINNED_SLOT;
}
inline void pinned_slot_release(Ctx* ctx, void* p) {
  if (!p || !ctx->pinned_block) return;
  ctx->pinned_free.push_back((uint32_t)((static_cast<uint8_t*>(p) - static_cast<uint8_t*>(ctx->pinned_block)) / Ctx::PINNED_SLOT));
}

// set by an atexit hook: CUDA may already be torn down when late destructors run at process exit
extern std::atomic<bool> g_exiting;

// A reference-counted HBM allocation (stream-ordered pool) or a borrowed foreign pointer.
struct DevBuf {
  void* ptr = nullptr;
  size_t bytes = 0;
  size_t cls = 0;                     // size class of an owned allocation (0: borrowed / view)
  Ctx* ctx = nullptr;
  std::function<void()> on_release;   // borrowed buffers: drop the producer's reference
  ~DevBuf() {
    if (g_exiting.load()) return;
    if (on_release) { on_release(); return; }
    if (!ptr || !ctx) return;
    if (ctx->dead.load()) { cudaFree(ptr); return; }
    if (cls) {
      std::lock_guard<std::mutex> g(ctx->cache_mu);
      if (ctx->cached_bytes + cls <= Ctx::CACHE_LIMIT) { ctx->cache[cls].push_back(ptr); ctx->cached_bytes += cls; return; }
    }
    cudaFreeAsync(ptr, ctx->stream);
  }
};
using BufPtr = std::shared_ptr<DevBuf>;

inline BufPtr dev_alloc(Ctx* ctx, size_t bytes) {
  auto b = std::make_shared<DevBuf>();
  b->ctx = ctx;
  b->bytes = bytes;
  const size_t padded = ((bytes + 255) & ~(size_t)255) + 256;   // room for 16-byte over-reads of tails
  const size_t cls = Ctx::size_class(padded);
  {
    std::lock_guard<std::mutex> g(ctx->cache_mu);
    auto it = ctx->cache.find(cls);
    if (it != ctx->cache.end() && !it->second.empty()) {
      b->ptr = it->second.back(); it->second.pop_back(); ctx->cached_bytes -= cls; b->cls = cls;
      return b;
    }
  }
  cudaError_t e = cudaMallocAsync(&b->ptr, cls, ctx->stream);
  if (e == cudaErrorMemoryAllocation) {       // out of HBM with blocks parked in the cache: give them back and retry
    cudaGetLastError();
    {
      std::lock_guard<std::mutex> g(ctx->cache_mu);
      for (auto& kv : ctx->cache) for (void* p : kv.second) cudaFreeAsync(p, ctx->stream);
      ctx->cache.clear(); ctx->cached_bytes = 0;
    }
    cudaStreamSynchronize(ctx->stream);
    e = cudaMallocAsync(&b->ptr, cls, ctx->stream);
  }
  if (e != cudaSuccess) { b->ptr = nullptr; ::sg::fail(SAILGPU_ERR_CUDA, std::string("CUDA error: ") + cudaGetErrorString(e) + " at cudaMallocAsync"); }
  b->cls = cls;
  return b;
}
inline BufPtr dev_alloc_zero(Ctx* ctx, size_t bytes) {
  BufPtr b = dev_alloc(ctx, bytes);
  SG_CUDA(cudaMemsetAsync(b->ptr, 0, ((bytes + 255) & ~(size_t)255) + 256, ctx->stream));
  return b;
}

struct DevColumn {
  DataType type;
  int64_t length = 0;
  BufPtr data;                 // values / views (Utf8 columns are converted to resolved views)
  BufPtr validity;             // Arrow bitmap (bit i at offset 0) or null when no nulls
  int64_t null_count = 0;
  std::vector<BufPtr> heaps;   // keep-alive for string bytes the views point into
  bool arrow_is_utf8 = false;  // the Arrow-facing type is Utf8 (export converts views back)
};

struct DevBatch {
  std::vector<DevColumn> cols;
  int64_t rows = 0;
};
using BatchPtr = std::shared_ptr<DevBatch>;

// ---- Arrow import / export (device.cu) -------------------------------------------------------------
Schema schema_from_arrow(const ArrowSchema* s);
void schema_to_arrow(const Schema& s, ArrowSchema* out);

// Host ArrowArray (struct) -> HBM.  Copies are issued on ctx->stream (one stream: allocation, copies and kernels stay ordered).
BatchPtr import_host_batch(Ctx* ctx, const Schema& schema, ArrowArray* arr);
// Device ArrowDeviceArray -> batch without copying values (string views are copied + resolved).
BatchPtr import_device_batch(Ctx* ctx, const Schema& schema, ArrowDeviceArray* arr);
// HBM -> host ArrowArray (malloc'ed buffers released by the consumer).
void export_host_batch(Ctx* ctx, const Schema& schema, const BatchPtr& b, ArrowArray* out);
// HBM -> ArrowDeviceArray sharing the buffers.
void export_device_batch(Ctx* ctx, const Schema& schema, const BatchPtr& b, ArrowDeviceArray* out, bool handle_only = false);

BatchPtr concat_batches(Ctx* ctx, const Schema& schema, const std::vector<BatchPtr>& parts);
BatchPtr empty_batch(Ctx* ctx, const Schema& schema);

}  // namespace sg
