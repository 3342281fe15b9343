// capi.cu -- the extern "C" surface declared in include/sailgpu.h.
#include <cstdio>

#include "h2d.hpp"
#include "runner.hpp"

using namespace sg;

struct sailgpu_ctx {
  Ctx ctx;
};
struct sailgpu_op {
  std::unique_ptr<Op> op;
  sailgpu_ctx* owner = nullptr;
  std::string last_error;
  std::vector<bool> input_finished;
};

namespace sg { std::atomic<bool> g_exiting{false}; }

namespace {
thread_local std::string g_ctx_error;
void mark_exiting() { sg::g_exiting.store(true); }

template <typename F>
int32_t guard(std::string* err, F&& f) {
  try {
    f();
    return SAILGPU_OK;
  } catch (const Error& e) {
    if (err) *err = e.what();
    return e.code;
  } catch (const std::exception& e) {
    if (err) *err = std::string("internal error: ") + e.what();
    return SAILGPU_ERR_CUDA;
  }
}
void set_device(const Ctx& c) { SG_CUDA(cudaSetDevice(c.device)); }
// charges the stream drains of one call on an operator handle to that operator (a chain's handle gets those of its stages)
struct SyncCharge {
  sailgpu_op* h; uint64_t s0;
  explicit SyncCharge(sailgpu_op* op) : h(op), s0(op->owner->ctx.host_syncs.load()) {}
  ~SyncCharge() { if (h->op) h->op->m.host_syncs += h->owner->ctx.host_syncs.load() - s0; }
};
using CtxLock = std::lock_guard<std::recursive_mutex>;
}  // namespace

namespace sg { void set_ctx_error(const std::string& m) { g_ctx_error = m; } }   // ops_more.cu: comm_init / exchange report through sailgpu_ctx_last_error
namespace sg { void resolve_exchange_timing(Ctx* ctx);
void pipeline_static_check(const Json& spec, const std::vector<Schema>& inputs);
size_t pipeline_precompile(const Json& spec, const std::vector<Schema>& inputs, uint64_t validity_mask, bool cold, bool compile, std::string* source); }

namespace sg {
struct ParquetColumnDesc { const uint8_t* chunk; uint64_t chunk_len; int32_t physical_type, type_length, max_def_level, codec; int64_t num_values; };
void decode_parquet_row_group(Ctx* ctx, const Schema& schema, const std::vector<ParquetColumnDesc>& cols, int64_t n_rows, DevBatch* b);
std::string parquet_plan_summary(const Field& f, const ParquetColumnDesc& c, int64_t n_rows);
}

extern "C" {

// release callback for a borrowed (non-owning) copy of an Arrow array struct: marks it released, frees nothing
SAILGPU_API void sailgpu_borrowed_release(struct ArrowArray* a) { if (a) a->release = nullptr; }

SAILGPU_API uint32_t sailgpu_version(void) { return (0u << 16) | 1u; }

SAILGPU_API int32_t sailgpu_ctx_create(int32_t device, sailgpu_ctx** out) {
  return guard(&g_ctx_error, [&] {
    SG_CHECK(out != nullptr, SAILGPU_ERR_INVALID, "out is null");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
      fail(SAILGPU_ERR_NO_DEVICE, std::string("no usable CUDA device (") + cudaGetErrorString(e) + "); libsailgpu has no CPU fallback");
    SG_CHECK(device >= 0 && device < n, SAILGPU_ERR_INVALID, "device ordinal out of range");
    static const int hooked = std::atexit(mark_exiting);
    (void)hooked;
    auto c = std::make_unique<sailgpu_ctx>();
    c->ctx.device = device;
    SG_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    SG_CUDA(cudaGetDeviceProperties(&prop, device));
    SG_CHECK(prop.major == 9 && prop.minor == 0, SAILGPU_ERR_NO_DEVICE, std::string("device '") + prop.name + "' is not sm_90 (Hopper); this library only carries sm_90a code");
    c->ctx.sm_count = prop.multiProcessorCount;
    c->ctx.max_smem = prop.sharedMemPerBlockOptin;
    SG_CUDA(cudaStreamCreateWithFlags(&c->ctx.stream, cudaStreamNonBlocking));
    cudaMemPool_t pool;
    SG_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
    uint64_t threshold = UINT64_MAX;   // keep freed HBM in the pool: operators re-allocate the same sizes every batch
    SG_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &threshold));
    *out = c.release();
  });
}

SAILGPU_API void sailgpu_ctx_destroy(sailgpu_ctx* c) {
  if (!c) return;
  if (sg::g_exiting.load()) return;
  CtxLock lk(c->ctx.mu);
  cudaSetDevice(c->ctx.device);
  // Batches handed out through pull_device may outlive the context: the (tiny) Ctx block is intentionally never freed,
  // it is only marked dead so that late buffer releases use cudaFree instead of the destroyed stream.
  c->ctx.shared_objects.clear();      // compiled pipelines and their literal buffers
  c->ctx.dead.store(true);
  if (c->ctx.stream) { cudaStreamSynchronize(c->ctx.stream); cudaStreamDestroy(c->ctx.stream); c->ctx.stream = nullptr; }
  if (c->ctx.pinned_block) { cudaFreeHost(c->ctx.pinned_block); c->ctx.pinned_block = nullptr; }
  destroy_pack_pool(&c->ctx);
}

SAILGPU_API const char* sailgpu_ctx_last_error(const sailgpu_ctx*) { return g_ctx_error.c_str(); }

SAILGPU_API void* sailgpu_ctx_stream(sailgpu_ctx* c) { return c ? (void*)c->ctx.stream : nullptr; }
SAILGPU_API int32_t sailgpu_ctx_synchronize(sailgpu_ctx* c) {
  return guard(&g_ctx_error, [&] {
    SG_CHECK(c != nullptr, SAILGPU_ERR_INVALID, "null context");
    CtxLock lk(c->ctx.mu);
    set_device(c->ctx);
    SG_CUDA(cudaStreamSynchronize(c->ctx.stream));
  });
}

SAILGPU_API int32_t sailgpu_op_create(sailgpu_ctx* c, const char* spec_json, size_t spec_len, const struct ArrowSchema* const* input_schemas,
                          int32_t n_inputs, int32_t partition, sailgpu_op** out, struct ArrowSchema* out_schema) {
  return guard(&g_ctx_error, [&] {
    SG_CHECK(c && spec_json && out && out_schema, SAILGPU_ERR_INVALID, "null argument");
    CtxLock lk(c->ctx.mu);
    set_device(c->ctx);
    Json spec = JsonParser(spec_json, spec_len).parse();
    std::vector<Schema> ins;
    for (int i = 0; i < n_inputs; ++i) ins.push_back(schema_from_arrow(input_schemas[i]));
    auto h = std::make_unique<sailgpu_op>();
    h->owner = c;
    const uint64_t s0 = c->ctx.host_syncs.load();
    h->op = make_op(&c->ctx, spec, ins, partition);
    h->op->m.host_syncs += c->ctx.host_syncs.load() - s0;
    h->input_finished.assign((size_t)n_inputs, false);
    schema_to_arrow(h->op->out_schema, out_schema);
    *out = h.release();
  });
}

// Plan-time check used by the rewrite pass: parses the spec, runs type inference and reports the output schema or
// why the operator cannot run on the GPU.  Touches no device: works on a machine without a GPU.
SAILGPU_API int32_t sailgpu_spec_validate(const char* spec_json, size_t spec_len, const struct ArrowSchema* const* input_schemas,
                                          int32_t n_inputs, struct ArrowSchema* out_schema, char* err_buf, size_t err_cap) {
  std::string err;
  const int32_t rc = guard(&err, [&] {
    SG_CHECK(spec_json && out_schema, SAILGPU_ERR_INVALID, "null argument");
    Json spec = JsonParser(spec_json, spec_len).parse();
    std::vector<Schema> ins;
    for (int i = 0; i < n_inputs; ++i) ins.push_back(schema_from_arrow(input_schemas[i]));
    std::unique_ptr<Op> op = make_op(nullptr, spec, ins, 0);
    pipeline_static_check(spec, ins);
    schema_to_arrow(op->out_schema, out_schema);
  });
  if (rc != 0 && err_buf && err_cap) { const size_t k = std::min(err.size(), err_cap - 1); memcpy(err_buf, err.data(), k); err_buf[k] = 0; }
  return rc;
}

SAILGPU_API int64_t sailgpu_jit_precompile(const char* spec_json, size_t spec_len, const struct ArrowSchema* const* input_schemas, int32_t n_inputs,
                                           uint64_t validity_mask, int32_t flags, char* buf, size_t cap) {
  std::string err, source;
  size_t cubin = 0;
  const int32_t rc = guard(&err, [&] {
    SG_CHECK(spec_json && n_inputs >= 1, SAILGPU_ERR_INVALID, "null argument");
    Json spec = JsonParser(spec_json, spec_len).parse();
    std::vector<Schema> ins;
    for (int i = 0; i < n_inputs; ++i) ins.push_back(schema_from_arrow(input_schemas[i]));
    cubin = pipeline_precompile(spec, ins, validity_mask, (flags & SAILGPU_JIT_COLD_VARIANT) != 0, (flags & SAILGPU_JIT_COMPILE) != 0, &source);
  });
  const std::string& text = rc != 0 ? err : source;
  if (buf && cap) { const size_t k = std::min(text.size(), cap - 1); memcpy(buf, text.data(), k); buf[k] = 0; }
  if (rc != 0) return -(int64_t)(rc < 0 ? -rc : rc);
  return (flags & SAILGPU_JIT_COMPILE) ? (int64_t)cubin : (int64_t)source.size();
}

// host-only: what the page / run-header walk found in one column chunk, as JSON (no device is touched)
SAILGPU_API int32_t sailgpu_parquet_inspect(const struct ArrowSchema* schema_c, const sailgpu_parquet_column* cols, int32_t n_cols, int64_t n_rows, int32_t column,
                                            char* buf, size_t cap) {
  std::string err, out;
  const int32_t rc = guard(&err, [&] {
    SG_CHECK(schema_c && cols && column >= 0 && column < n_cols, SAILGPU_ERR_INVALID, "bad argument");
    Schema schema = schema_from_arrow(schema_c);
    SG_CHECK((int)schema.size() == n_cols, SAILGPU_ERR_INVALID, "parquet: column count mismatch");
    ParquetColumnDesc d{cols[column].chunk, cols[column].chunk_len, cols[column].physical_type, cols[column].type_length, cols[column].max_def_level, cols[column].codec, cols[column].num_values};
    out = parquet_plan_summary(schema[(size_t)column], d, n_rows);
  });
  const std::string& text = rc != 0 ? err : out;
  if (buf && cap) { const size_t k = std::min(text.size(), cap - 1); memcpy(buf, text.data(), k); buf[k] = 0; }
  return rc;
}
SAILGPU_API int32_t sailgpu_parquet_decode(sailgpu_ctx* c, const struct ArrowSchema* schema_c, const sailgpu_parquet_column* cols, int32_t n_cols, int64_t n_rows,
                                           struct ArrowDeviceArray* out) {
  return guard(&g_ctx_error, [&] {
    SG_CHECK(c && schema_c && cols && out && n_rows >= 0, SAILGPU_ERR_INVALID, "null argument");
    CtxLock lk(c->ctx.mu);
    set_device(c->ctx);
    Schema schema = schema_from_arrow(schema_c);
    SG_CHECK((int)schema.size() == n_cols, SAILGPU_ERR_INVALID, "parquet: " + std::to_string(n_cols) + " column chunks for a schema of " + std::to_string(schema.size()) + " fields");
    auto b = std::make_shared<DevBatch>();
    b->rows = n_rows;
    std::vector<ParquetColumnDesc> descs;
    for (int i = 0; i < n_cols; ++i)
      descs.push_back(ParquetColumnDesc{cols[i].chunk, cols[i].chunk_len, cols[i].physical_type, cols[i].type_length, cols[i].max_def_level, cols[i].codec, cols[i].num_values});
    decode_parquet_row_group(&c->ctx, schema, descs, n_rows, b.get());
    export_device_batch(&c->ctx, schema, b, out);
  });
}
SAILGPU_API int32_t sailgpu_parquet_stats(sailgpu_ctx* c, char* buf, size_t cap) {
  return guard(&g_ctx_error, [&] {
    SG_CHECK(c && buf && cap, SAILGPU_ERR_INVALID, "null argument");
    CtxLock lk(c->ctx.mu);
    const Ctx::ParquetZstd& s = c->ctx.parquet_zstd;
    snprintf(buf, cap, "{\"zstd_pages\":%llu,\"zstd_out_bytes\":%llu,\"image_bytes\":%llu,\"decompress_ms\":%.4f,\"readback_ms\":%.4f}", (unsigned long long)s.pages,
             (unsigned long long)s.out_bytes, (unsigned long long)s.image_bytes, (double)s.decompress_ms, (double)s.readback_ms);
  });
}

SAILGPU_API int32_t sailgpu_op_push(sailgpu_op* h, int32_t input_idx, struct ArrowArray* batch) {
  if (!h) return SAILGPU_ERR_INVALID;
  return guard(&h->last_error, [&] {
    CtxLock lk(h->owner->ctx.mu);
    SyncCharge charge(h);
    set_device(h->owner->ctx);
    SG_CHECK(input_idx >= 0 && input_idx < (int)h->op->in_schemas.size(), SAILGPU_ERR_INVALID, "input index out of range");
    SG_CHECK(!h->input_finished[(size_t)input_idx], SAILGPU_ERR_STATE, "push after finish_input");
    BatchPtr b = import_host_batch(&h->owner->ctx, h->op->in_schemas[(size_t)input_idx], batch);
    h->op->push(input_idx, b);
  });
}

SAILGPU_API int32_t sailgpu_op_push_device(sailgpu_op* h, int32_t input_idx, struct ArrowDeviceArray* batch) {
  if (!h) return SAILGPU_ERR_INVALID;
  return guard(&h->last_error, [&] {
    CtxLock lk(h->owner->ctx.mu);
    SyncCharge charge(h);
    set_device(h->owner->ctx);
    SG_CHECK(input_idx >= 0 && input_idx < (int)h->op->in_schemas.size(), SAILGPU_ERR_INVALID, "input index out of range");
    SG_CHECK(!h->input_finished[(size_t)input_idx], SAILGPU_ERR_STATE, "push after finish_input");
    SG_CHECK(batch && batch->array.release, SAILGPU_ERR_INVALID, "batch is null or released");
    BatchPtr b = take_internal_batch(batch, &h->owner->ctx);
    if (!b) { SG_CHECK(batch->array.n_children == (int64_t)h->op->in_schemas[(size_t)input_idx].size(), SAILGPU_ERR_INVALID, "device batch has no column arrays (a handle of another library instance?)"); }
    if (!b) { Trace t(&h->owner->ctx, "import_device_batch"); b = import_device_batch(&h->owner->ctx, h->op->in_schemas[(size_t)input_idx], batch); }
    Trace t2(&h->owner->ctx, "op.push");
    h->op->push(input_idx, b);
  });
}

SAILGPU_API int32_t sailgpu_op_finish_input(sailgpu_op* h, int32_t input_idx) {
  if (!h) return SAILGPU_ERR_INVALID;
  return guard(&h->last_error, [&] {
    CtxLock lk(h->owner->ctx.mu);
    SyncCharge charge(h);
    set_device(h->owner->ctx);
    SG_CHECK(input_idx >= 0 && input_idx < (int)h->op->in_schemas.size(), SAILGPU_ERR_INVALID, "input index out of range");
    if (h->input_finished[(size_t)input_idx]) return;
    h->input_finished[(size_t)input_idx] = true;
    Trace t(&h->owner->ctx, "op.finish");
    h->op->finish(input_idx);
  });
}

static int32_t pull_common(sailgpu_op* h, int part, struct ArrowArray* host_out, struct ArrowDeviceArray* dev_out, int32_t* has_more, bool handle_only = false) {
  if (!h) return SAILGPU_ERR_INVALID;
  return guard(&h->last_error, [&] {
    CtxLock lk(h->owner->ctx.mu);
    SyncCharge charge(h);
    set_device(h->owner->ctx);
    SG_CHECK(has_more && (host_out || dev_out), SAILGPU_ERR_INVALID, "null argument");
    BatchPtr b;
    bool more;
    { Trace t(&h->owner->ctx, "op.pull"); more = part >= 0 ? h->op->pull_partition(part, &b) : h->op->pull(&b); }
    Trace t2(&h->owner->ctx, "export");
    *has_more = more ? 1 : 0;
    if (!b) b = empty_batch(&h->owner->ctx, h->op->out_schema);
    if (host_out) export_host_batch(&h->owner->ctx, h->op->out_schema, b, host_out);
    else export_device_batch(&h->owner->ctx, h->op->out_schema, b, dev_out, handle_only);
  });
}

SAILGPU_API int32_t sailgpu_op_pull(sailgpu_op* h, struct ArrowArray* out, int32_t* has_more) { return pull_common(h, -1, out, nullptr, has_more); }
SAILGPU_API int32_t sailgpu_op_pull_device(sailgpu_op* h, struct ArrowDeviceArray* out, int32_t* has_more) { return pull_common(h, -1, nullptr, out, has_more); }
SAILGPU_API int32_t sailgpu_op_pull_device_handle(sailgpu_op* h, struct ArrowDeviceArray* out, int32_t* has_more) { return pull_common(h, -1, nullptr, out, has_more, true); }
SAILGPU_API int32_t sailgpu_op_pull_partition(sailgpu_op* h, int32_t part, struct ArrowDeviceArray* out, int32_t* has_more) {
  if (part < 0) return SAILGPU_ERR_INVALID;
  return pull_common(h, part, nullptr, out, has_more);
}

// Result sink: the next output batch as one self-contained Arrow IPC stream (ipc.cpp), the bytes Sail's Spark Connect executor
// sends for a result batch (crates/sail-spark-connect/src/executor.rs:320-330).  pull to the host + framing.
SAILGPU_API int32_t sailgpu_op_pull_ipc(sailgpu_op* h, uint8_t** data, size_t* len, int64_t* rows, int32_t* has_more) {
  if (!h || !data || !len || !has_more) return SAILGPU_ERR_INVALID;
  struct ArrowArray batch;
  memset(&batch, 0, sizeof(batch));
  int32_t rc = pull_common(h, -1, &batch, nullptr, has_more);
  if (rc != SAILGPU_OK) return rc;
  struct ArrowSchema schema;
  memset(&schema, 0, sizeof(schema));
  rc = guard(&h->last_error, [&] { schema_to_arrow(h->op->out_schema, &schema); });
  if (rc == SAILGPU_OK) {
    rc = sailgpu_ipc_stream(&schema, &batch, data, len);
    if (rc != SAILGPU_OK) h->last_error = sailgpu_ipc_last_error();
    else if (rows) *rows = batch.length;
  }
  if (schema.release) schema.release(&schema);
  if (batch.release) batch.release(&batch);
  return rc;
}

SAILGPU_API int64_t sailgpu_op_metrics(sailgpu_op* h, char* json_buf, size_t cap) {
  if (!h) return -1;
  CtxLock lk(h->owner->ctx.mu);
  cudaSetDevice(h->owner->ctx.device);
  const Metrics& m = h->op->m;
  char tmp[2048];
  sg::resolve_exchange_timing(&h->owner->ctx);
  int n = snprintf(tmp, sizeof(tmp),
                   "{\"output_rows\":%llu,\"output_batches\":%llu,\"input_rows\":%llu,\"input_batches\":%llu,"
                   "\"elapsed_compute\":%llu,\"build_input_rows\":%llu,\"build_input_batches\":%llu,\"build_time\":%llu,"
                   "\"join_time\":%llu,\"gpu.kernel_launches\":%llu,\"gpu.h2d_bytes\":%llu,\"gpu.d2h_bytes\":%llu,"
                   "\"gpu.pipeline_launches\":%llu,\"gpu.jit_launches\":%llu,\"gpu.pipeline_kernel_ns\":%llu,"
                   "\"gpu.exchange_sent_bytes\":%llu,\"gpu.exchange_recv_bytes\":%llu,\"gpu.exchange_ns\":%llu,\"gpu.exchange_calls\":%llu,"
                   "\"gpu.host_syncs\":%llu}",
                   (unsigned long long)m.output_rows, (unsigned long long)m.output_batches, (unsigned long long)m.input_rows,
                   (unsigned long long)m.input_batches, (unsigned long long)m.elapsed_compute_ns, (unsigned long long)m.build_input_rows,
                   (unsigned long long)m.build_input_batches, (unsigned long long)m.build_time_ns, (unsigned long long)m.join_time_ns,
                   (unsigned long long)m.kernel_launches, (unsigned long long)h->owner->ctx.h2d_bytes.load(),
                   (unsigned long long)h->owner->ctx.d2h_bytes.load(), (unsigned long long)h->op->m.pipeline_launches, (unsigned long long)h->op->m.jit_launches,
                   (unsigned long long)h->op->pipeline_kernel_ns(), (unsigned long long)h->owner->ctx.exch_sent_bytes.load(),
                   (unsigned long long)h->owner->ctx.exch_recv_bytes.load(), (unsigned long long)h->owner->ctx.exch_ns.load(),
                   (unsigned long long)h->owner->ctx.exch_calls.load(), (unsigned long long)m.host_syncs);
  std::string js(tmp, (size_t)std::max(0, std::min(n, (int)sizeof(tmp) - 1)));
  if (m.agg_spills) {      // an aggregate that went into partitioned mode
    js.pop_back();
    js += ",\"gpu.agg_spills\":" + std::to_string(m.agg_spills) + ",\"gpu.agg_partitions\":" + std::to_string(m.agg_partitions) + ",\"gpu.agg_partition_groups\":[";
    for (size_t i = 0; i < m.agg_partition_groups.size(); ++i) js += (i ? "," : "") + std::to_string(m.agg_partition_groups[i]);
    js += "]}";
  }
  if (json_buf && cap) { size_t k = std::min<size_t>(js.size(), cap - 1); memcpy(json_buf, js.data(), k); json_buf[k] = 0; }
  return (int64_t)js.size() + 1;
}

SAILGPU_API const char* sailgpu_last_error(const sailgpu_op* h) { return h ? h->last_error.c_str() : "null handle"; }

SAILGPU_API void sailgpu_op_destroy(sailgpu_op* h) {
  if (!h) return;
  if (sg::g_exiting.load()) return;
  CtxLock lk(h->owner->ctx.mu);
  cudaSetDevice(h->owner->ctx.device);
  cudaStreamSynchronize(h->owner->ctx.stream);
  delete h;
}

SAILGPU_API int32_t sailgpu_host_alloc(sailgpu_ctx* c, size_t bytes, void** out) {
  return guard(&g_ctx_error, [&] {
    SG_CHECK(c && out, SAILGPU_ERR_INVALID, "null argument");
    CtxLock lk(c->ctx.mu);
    set_device(c->ctx);
    SG_CUDA(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
  });
}
SAILGPU_API void sailgpu_host_free(sailgpu_ctx* c, void* p) {
  if (!c || !p) return;
  CtxLock lk(c->ctx.mu);
  cudaSetDevice(c->ctx.device);
  cudaFreeHost(p);
}

}  // extern "C"
