// device.cu -- Arrow C Data / C Device Data Interface <-> HBM batches.
//
// This is the boundary the Rust shim crosses per RecordBatch (arrow::ffi::to_ffi / from_ffi);
// ownership rules follow SURVEY.md section 8b "Ownership": inputs are producer-owned until their
// release callback runs; outputs are library-owned until the consumer calls release.
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "device.hpp"
#include "h2d.hpp"
#include "kernels.hpp"
#include "relational.hpp"

namespace sg {

// ---------------------------------------------------------------------------------------------
// schema
// ---------------------------------------------------------------------------------------------
Schema schema_from_arrow(const ArrowSchema* s) {
  SG_CHECK(s && s->format && std::string(s->format) == "+s", SAILGPU_ERR_INVALID, "input schema must be a struct (+s)");
  Schema out;
  for (int64_t i = 0; i < s->n_children; ++i) {
    const ArrowSchema* c = s->children[i];
    Field f;
    f.name = c->name ? c->name : "";
    f.type = type_from_arrow_format(c->format);
    f.nullable = (c->flags & ARROW_FLAG_NULLABLE) != 0;
    out.push_back(f);
  }
  return out;
}

namespace {
struct SchemaPriv {
  std::string format, name;
  std::vector<ArrowSchema> children;
  std::vector<ArrowSchema*> child_ptrs;
};
void release_schema(ArrowSchema* s) {
  if (!s || !s->release) return;
  for (int64_t i = 0; i < s->n_children; ++i)
    if (s->children[i]->release) s->children[i]->release(s->children[i]);
  delete static_cast<SchemaPriv*>(s->private_data);
  s->release = nullptr;
}
void fill_schema(ArrowSchema* out, const std::string& fmt, const std::string& name, bool nullable, SchemaPriv* p) {
  p->format = fmt; p->name = name;
  out->format = p->format.c_str(); out->name = p->name.c_str(); out->metadata = nullptr;
  out->flags = nullable ? ARROW_FLAG_NULLABLE : 0;
  out->n_children = 0; out->children = nullptr; out->dictionary = nullptr;
  out->release = release_schema; out->private_data = p;
}
}  // namespace

void schema_to_arrow(const Schema& s, ArrowSchema* out) {
  auto* p = new SchemaPriv();
  fill_schema(out, "+s", "", false, p);
  p->children.resize(s.size());
  p->child_ptrs.resize(s.size());
  for (size_t i = 0; i < s.size(); ++i) {
    fill_schema(&p->children[i], s[i].type.arrow_format(), s[i].name, s[i].nullable, new SchemaPriv());
    p->child_ptrs[i] = &p->children[i];
  }
  out->n_children = (int64_t)s.size();
  out->children = p->child_ptrs.data();
}

// ---------------------------------------------------------------------------------------------
// import
// ---------------------------------------------------------------------------------------------
namespace {

// What an import needs besides the column itself: the staged host->device copies (host batches only) and the device
// work that may only run once the copied bytes are in place (conversions of Utf8 / long views / unaligned bitmaps).
struct ImportJob {
  Ctx* ctx;
  bool on_device;
  cudaStream_t stream;
  HostStager stager;
  std::vector<std::function<void()>> post;
  ImportJob(Ctx* c, bool dev, cudaStream_t s) : ctx(c), on_device(dev), stream(s), stager(c) {}
  // `n` elements of `width` bytes from a host (staged, possibly packed on the wire) or device (plain copy) pointer into a fresh HBM buffer
  BufPtr upload(const void* src, int64_t n, int width, HostCol kind = HostCol::Raw) {
    const size_t bytes = (size_t)n * (size_t)width;
    BufPtr b = dev_alloc(ctx, bytes);
    if (!bytes) return b;
    if (on_device) SG_CUDA(cudaMemcpyAsync(b->ptr, src, bytes, cudaMemcpyDeviceToDevice, stream));
    else if (kind == HostCol::Raw) stager.add_raw(b->ptr, src, bytes);
    else stager.add(kind, b->ptr, src, n, width);
    return b;
  }
  // run `f` now (device import: the data is there) or after the staged copies (host import)
  void after(std::function<void()> f) { if (on_device) f(); else post.push_back(std::move(f)); }
};

struct ReleaseToken {     // drops the producer's ArrowArray when the last borrowed buffer dies
  ArrowArray arr;
  ~ReleaseToken() { if (arr.release) arr.release(&arr); }
};

// bitmap slice [offset, offset+len) -> bitmap at bit 0
BufPtr import_bitmap(ImportJob& J, const uint8_t* src, int64_t offset, int64_t len) {
  Ctx* ctx = J.ctx;
  const int64_t first_byte = offset >> 3;
  const int64_t nbytes = ((offset + len + 7) >> 3) - first_byte;
  if ((offset & 7) == 0) {
    if (J.on_device) {
      auto b = std::make_shared<DevBuf>();   // borrowed: lifetime tied to the batch token held elsewhere
      b->ptr = const_cast<uint8_t*>(src) + first_byte; b->bytes = (size_t)nbytes; b->on_release = [] {};
      return b;
    }
    return J.upload(src + first_byte, nbytes, 1);
  }
  BufPtr raw = J.on_device ? nullptr : J.upload(src + first_byte, nbytes, 1);
  const uint8_t* dsrc = J.on_device ? src + first_byte : static_cast<const uint8_t*>(raw->ptr);
  BufPtr bytes = dev_alloc(ctx, (size_t)len);
  BufPtr bits = dev_alloc_zero(ctx, (size_t)((len + 31) / 32 * 4));
  cudaStream_t stream = J.stream;
  J.after([=] {
    (void)raw;
    SG_CUDA(launch_unpack_bits(dsrc, static_cast<uint8_t*>(bytes->ptr), len, offset & 7, stream));
    SG_CUDA(launch_pack_bytes(static_cast<const uint8_t*>(bytes->ptr), static_cast<uint32_t*>(bits->ptr), len, nullptr, stream));
  });
  return bits;
}

DevColumn import_column(ImportJob& J, const Field& f, const ArrowArray* a, const std::shared_ptr<ReleaseToken>& token) {
  Ctx* ctx = J.ctx;
  const bool on_device = J.on_device;
  cudaStream_t stream = J.stream;
  DevColumn c;
  c.type = f.type;
  c.length = a->length;
  c.null_count = a->null_count;
  auto borrow = [&](const void* p, size_t bytes) {
    auto b = std::make_shared<DevBuf>();
    b->ptr = const_cast<void*>(p); b->bytes = bytes;
    b->on_release = [token] {};
    return b;
  };
  const uint8_t* vbits = a->n_buffers > 0 ? static_cast<const uint8_t*>(a->buffers[0]) : nullptr;
  if (vbits && a->null_count != 0 && a->length > 0) {
    c.validity = import_bitmap(J, vbits, a->offset, a->length);
    if (on_device && c.validity->on_release) c.validity->on_release = [token] {};
    if (c.null_count < 0) c.null_count = -1;   // unknown: treated as "may contain nulls"
  } else {
    c.null_count = 0;
  }
  const int w = f.type.arrow_width();
  switch (f.type.id) {
    case TypeId::Bool: {
      const uint8_t* bits = static_cast<const uint8_t*>(a->buffers[1]);
      c.data = a->length ? import_bitmap(J, bits, a->offset, a->length) : dev_alloc(ctx, 0);
      if (on_device && c.data->on_release) c.data->on_release = [token] {};
      break;
    }
    case TypeId::Utf8: {
      const int32_t* offs = static_cast<const int32_t*>(a->buffers[1]) + a->offset;
      const uint8_t* bytes = static_cast<const uint8_t*>(a->buffers[2]);
      BufPtr doffs, dbytes;
      if (on_device) {
        doffs = borrow(offs, (size_t)(a->length + 1) * 4);
        int32_t last = 0;
        if (a->length) SG_CUDA(cudaMemcpyAsync(&last, offs + a->length, 4, cudaMemcpyDeviceToHost, stream));
        stream_sync(ctx);
        dbytes = borrow(bytes, (size_t)last);
      } else {
        doffs = J.upload(offs, a->length + 1, 4);
        const int32_t last = a->length ? offs[a->length] : 0;
        dbytes = J.upload(bytes, last, 1);   // absolute offsets: copy from byte 0
      }
      c.data = dev_alloc(ctx, (size_t)a->length * 16);
      {
        BufPtr views = c.data;
        const int64_t n = a->length;
        J.after([=] { SG_CUDA(launch_utf8_to_views(static_cast<const int32_t*>(doffs->ptr), static_cast<const uint8_t*>(dbytes->ptr), views->ptr, n, stream)); });
      }
      c.heaps = {dbytes, doffs};
      c.arrow_is_utf8 = true;
      break;
    }
    case TypeId::Utf8View: {
      const uint8_t* views = static_cast<const uint8_t*>(a->buffers[1]) + a->offset * 16;
      const int64_t n_data = a->n_buffers - 3;   // validity, views, data..., sizes
      // views without data buffers are all inline (<= 12 bytes): a device batch can be used in place, a host batch travels packed
      if (on_device && n_data <= 0) c.data = borrow(views, (size_t)a->length * 16);
      else c.data = J.upload(views, a->length, 16, n_data <= 0 ? HostCol::View16 : HostCol::Raw);
      if (n_data > 0) {
        std::vector<int64_t> sizes((size_t)n_data);
        const int64_t* size_buf = static_cast<const int64_t*>(a->buffers[a->n_buffers - 1]);
        if (on_device) { SG_CUDA(cudaMemcpyAsync(sizes.data(), size_buf, (size_t)n_data * 8, cudaMemcpyDeviceToHost, stream)); stream_sync(ctx); }
        else std::memcpy(sizes.data(), size_buf, (size_t)n_data * 8);
        auto bases = std::make_shared<std::vector<uint64_t>>((size_t)n_data);
        for (int64_t k = 0; k < n_data; ++k) {
          BufPtr h = on_device ? borrow(a->buffers[2 + k], (size_t)sizes[k]) : J.upload(a->buffers[2 + k], sizes[k], 1);
          (*bases)[(size_t)k] = reinterpret_cast<uint64_t>(h->ptr);
          c.heaps.push_back(h);
        }
        BufPtr dbases = dev_alloc(ctx, (size_t)n_data * 8);
        BufPtr vdata = c.data;
        const int64_t n = a->length;
        J.after([=] {
          SG_CUDA(cudaMemcpyAsync(dbases->ptr, bases->data(), (size_t)n_data * 8, cudaMemcpyHostToDevice, stream));
          SG_CUDA(launch_resolve_views(vdata->ptr, n, static_cast<const uint64_t*>(dbases->ptr), stream));
          stream_sync(ctx);   // `bases` is host memory owned by this closure
        });
        c.heaps.push_back(dbases);
      }
      break;
    }
    default: {
      SG_CHECK(w > 0, SAILGPU_ERR_UNSUPPORTED, "unsupported column type " + f.type.str());
      const uint8_t* p = static_cast<const uint8_t*>(a->buffers[1]) + a->offset * w;
      if (on_device) c.data = borrow(p, (size_t)a->length * w);
      else {
        const TypeId id = f.type.storage().id;
        const HostCol kind = id == TypeId::Decimal128 ? HostCol::Dec128
                           : (id == TypeId::Int64 || id == TypeId::UInt64) ? HostCol::Int64
                           : (id == TypeId::Int32 || id == TypeId::UInt32 || id == TypeId::Date32) ? HostCol::Int32 : HostCol::Raw;
        c.data = J.upload(p, a->length, w, kind);
      }
    }
  }
  return c;
}

BatchPtr import_batch(Ctx* ctx, const Schema& schema, ArrowArray* arr, bool on_device, cudaStream_t stream) {
  SG_CHECK(arr && arr->release, SAILGPU_ERR_INVALID, "batch is null or already released");
  SG_CHECK(arr->n_children == (int64_t)schema.size(), SAILGPU_ERR_INVALID,
           "batch has " + std::to_string(arr->n_children) + " columns, schema has " + std::to_string(schema.size()));
  SG_CHECK(arr->offset == 0, SAILGPU_ERR_UNSUPPORTED, "struct-level offset is not supported");
  auto token = std::make_shared<ReleaseToken>();
  token->arr = *arr;          // move: we now own the producer's reference
  arr->release = nullptr;
  auto b = std::make_shared<DevBatch>();
  b->rows = token->arr.length;
  ImportJob J(ctx, on_device, stream);
  for (size_t i = 0; i < schema.size(); ++i) {
    const ArrowArray* ch = token->arr.children[i];
    SG_CHECK(ch->length == b->rows, SAILGPU_ERR_INVALID, "column length mismatch");
    b->cols.push_back(import_column(J, schema[i], ch, token));
  }
  if (!on_device) {
    // the packer threads read every host buffer into pinned staging memory before flush() returns; the copies themselves
    // may still be in flight (the compute stream waits for them through an event), so the next batch can be packed meanwhile
    J.stager.flush();
    for (auto& f : J.post) f();
    token.reset();
  }
  return b;
}

}  // namespace

BatchPtr import_host_batch(Ctx* ctx, const Schema& schema, ArrowArray* arr) {
  // copies + import kernels run on the compute stream: one ordering domain, no cross-stream events
  return import_batch(ctx, schema, arr, false, ctx->stream);
}

BatchPtr import_device_batch(Ctx* ctx, const Schema& schema, ArrowDeviceArray* arr) {
  SG_CHECK(arr->device_type == ARROW_DEVICE_CUDA, SAILGPU_ERR_INVALID, "device batch must be ARROW_DEVICE_CUDA");
  if (arr->sync_event) SG_CUDA(cudaStreamWaitEvent(ctx->stream, *static_cast<cudaEvent_t*>(arr->sync_event), 0));
  return import_batch(ctx, schema, &arr->array, true, ctx->stream);
}

// ---------------------------------------------------------------------------------------------
// export
// ---------------------------------------------------------------------------------------------
namespace {

struct ArrayPriv {
  std::vector<void*> host_allocs;            // free() on release
  std::vector<const void*> buffers;
  std::vector<ArrowArray> children;
  std::vector<ArrowArray*> child_ptrs;
  std::vector<BufPtr> keep;                  // device export keeps HBM alive
  BatchPtr batch;                            // internal fast path for chained operators
  Ctx* ctx = nullptr;                        // exporting context (a handle taken by another context waits for its stream)
  bool opaque = false;                       // handle export: no Arrow children were materialised
};
void release_array(ArrowArray* a) {
  if (!a || !a->release) return;
  for (int64_t i = 0; i < a->n_children; ++i)
    if (a->children[i]->release) a->children[i]->release(a->children[i]);
  auto* p = static_cast<ArrayPriv*>(a->private_data);
  for (void* h : p->host_allocs) free(h);
  delete p;
  a->release = nullptr;
}
void init_array(ArrowArray* a, int64_t length, int64_t null_count, ArrayPriv* p) {
  a->length = length; a->null_count = null_count; a->offset = 0;
  a->n_buffers = (int64_t)p->buffers.size(); a->buffers = p->buffers.data();
  a->n_children = 0; a->children = nullptr; a->dictionary = nullptr;
  a->release = release_array; a->private_data = p;
}

// strings: produce Arrow-conformant buffers on the device from resolved views
struct StringExport { BufPtr views_or_offsets, heap; int64_t heap_bytes = 0; };
// `inline_known`: the caller has established that every view of the column is inline (<= 12 bytes)
StringExport export_strings(Ctx* ctx, const DevColumn& c, bool as_utf8, bool inline_known) {
  StringExport out;
  const int64_t n = c.length;
  if (n == 0) {
    out.views_or_offsets = dev_alloc_zero(ctx, as_utf8 ? 4 : 0);
    out.heap = dev_alloc(ctx, 0);
    return out;
  }
  if (inline_known) {
    out.views_or_offsets = c.data;
    out.heap = dev_alloc(ctx, 0);
    return out;
  }
  if (!as_utf8) {
    // all strings inline (<= 12 bytes, e.g. flags and codes): the resolved views already are Arrow views -> zero copy
    BufPtr mx = dev_alloc_zero(ctx, 8);
    unsigned int max_len = 0;
    SG_CUDA(launch_max_view_len(c.data->ptr, n, static_cast<unsigned int*>(mx->ptr), ctx->stream));
    SG_CUDA(cudaMemcpyAsync(&max_len, mx->ptr, 4, cudaMemcpyDeviceToHost, ctx->stream));
    stream_sync(ctx);
    if (max_len <= 12) {
      out.views_or_offsets = c.data;
      out.heap = dev_alloc(ctx, 0);
      return out;
    }
  }
  BufPtr lens = dev_alloc(ctx, (size_t)n * 4);
  BufPtr offs = dev_alloc(ctx, (size_t)n * 8);
  BufPtr scratch = dev_alloc(ctx, 1026 * 8);
  SG_CUDA(launch_view_lengths(c.data->ptr, n, static_cast<uint32_t*>(lens->ptr), as_utf8 ? 1 : 0, ctx->stream));
  SG_CUDA(launch_exclusive_scan_u32(static_cast<uint32_t*>(lens->ptr), n, static_cast<uint64_t*>(offs->ptr), static_cast<uint64_t*>(scratch->ptr), ctx->stream));
  const int64_t nblocks = std::min<int64_t>(1024, (n + 4095) / 4096);
  uint64_t total = 0;
  SG_CUDA(cudaMemcpyAsync(&total, static_cast<uint64_t*>(scratch->ptr) + nblocks, 8, cudaMemcpyDeviceToHost, ctx->stream));
  stream_sync(ctx);
  out.heap_bytes = (int64_t)total;
  out.heap = dev_alloc(ctx, (size_t)total);
  if (as_utf8) {
    SG_CHECK(total < (1ull << 31), SAILGPU_ERR_UNSUPPORTED, "Utf8 output exceeds 2 GiB of string data; use Utf8View");
    out.views_or_offsets = dev_alloc(ctx, (size_t)(n + 1) * 4);
    SG_CUDA(launch_views_to_utf8(c.data->ptr, n, static_cast<uint64_t*>(offs->ptr), static_cast<int32_t*>(out.views_or_offsets->ptr),
                                 static_cast<uint8_t*>(out.heap->ptr), ctx->stream));
  } else {
    SG_CHECK(total < (1ull << 31), SAILGPU_ERR_UNSUPPORTED, "string heap of one output batch exceeds 2 GiB");
    out.views_or_offsets = dev_alloc(ctx, (size_t)n * 16);
    SG_CUDA(cudaMemcpyAsync(out.views_or_offsets->ptr, c.data->ptr, (size_t)n * 16, cudaMemcpyDeviceToDevice, ctx->stream));
    SG_CUDA(launch_views_to_arrow(out.views_or_offsets->ptr, n, static_cast<uint64_t*>(offs->ptr), static_cast<uint8_t*>(out.heap->ptr), ctx->stream));
  }
  return out;
}

void* to_host(Ctx* ctx, const void* dptr, size_t bytes, ArrayPriv* p) {
  void* h = malloc(bytes ? bytes : 1);
  SG_CHECK(h != nullptr, SAILGPU_ERR_CUDA, "host allocation failed");
  p->host_allocs.push_back(h);
  ctx->d2h_bytes += bytes;
  if (!bytes) return h;
  if (bytes <= Ctx::D2H_SMALL) {
    if (!ctx->d2h_stage && cudaHostAlloc(&ctx->d2h_stage, Ctx::D2H_STAGE_BYTES, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); ctx->d2h_stage = nullptr; }
    const size_t off = (ctx->d2h_used + 15) & ~(size_t)15;
    if (ctx->d2h_stage && off + bytes <= Ctx::D2H_STAGE_BYTES) {
      SG_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(ctx->d2h_stage) + off, dptr, bytes, cudaMemcpyDeviceToHost, ctx->stream));
      ctx->d2h_pending.push_back({h, off, bytes});
      ctx->d2h_used = off + bytes;
      return h;
    }
  }
  SG_CUDA(cudaMemcpyAsync(h, dptr, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  return h;
}

// after the stream has been synchronised: move the bounced pieces to their host buffers
void finish_small_d2h(Ctx* ctx) {
  for (auto& it : ctx->d2h_pending) memcpy(it.host, static_cast<const uint8_t*>(ctx->d2h_stage) + it.off, it.bytes);
  ctx->d2h_pending.clear();
  ctx->d2h_used = 0;
}

void export_column(Ctx* ctx, const Field& f, const DevColumn& c, ArrowArray* out, bool to_device, bool inline_known = false) {
  auto* p = new ArrayPriv();
  const int64_t n = c.length;
  auto emit = [&](const BufPtr& b, size_t bytes) -> const void* {
    if (!b) return nullptr;
    if (to_device) { p->keep.push_back(b); return b->ptr; }
    return to_host(ctx, b->ptr, bytes, p);
  };
  int64_t null_count = c.validity ? c.null_count : 0;
  p->buffers.push_back(c.validity ? emit(c.validity, (size_t)((n + 7) / 8)) : nullptr);
  if (f.type.is_string()) {
    const bool as_utf8 = f.type.id == TypeId::Utf8;
    StringExport s = export_strings(ctx, c, as_utf8, inline_known);
    if (as_utf8) {
      p->buffers.push_back(emit(s.views_or_offsets, (size_t)(n + 1) * 4));
      p->buffers.push_back(emit(s.heap, (size_t)s.heap_bytes));
    } else {
      p->buffers.push_back(emit(s.views_or_offsets, (size_t)n * 16));
      const bool has_heap = s.heap_bytes > 0;          // all-inline columns carry no variadic data buffer
      if (has_heap) p->buffers.push_back(emit(s.heap, (size_t)s.heap_bytes));
      // variadic buffer sizes (host array in both modes: tiny)
      int64_t* sizes = static_cast<int64_t*>(malloc(8));
      sizes[0] = s.heap_bytes;
      p->host_allocs.push_back(sizes);
      if (to_device) {
        BufPtr dsz = dev_alloc(ctx, 8);
        SG_CUDA(cudaMemcpyAsync(dsz->ptr, sizes, 8, cudaMemcpyHostToDevice, ctx->stream));
        p->keep.push_back(dsz);
        p->buffers.push_back(dsz->ptr);
      } else {
        p->buffers.push_back(sizes);
      }
    }
  } else if (f.type.id == TypeId::Bool) {
    p->buffers.push_back(emit(c.data, (size_t)((n + 7) / 8)));
  } else {
    p->buffers.push_back(emit(c.data, (size_t)n * f.type.arrow_width()));
  }
  init_array(out, n, null_count, p);
}

}  // namespace

// One synchronisation per batch: every Utf8View column is first exported as if all its strings were inline (its views are
// then the Arrow views), with the longest length of each such column read back together with the data.  Only a column that
// really holds longer strings is exported a second time, through the heap.
void export_host_batch(Ctx* ctx, const Schema& schema, const BatchPtr& b, ArrowArray* out) {
  ctx->d2h_pending.clear(); ctx->d2h_used = 0;      // leftovers of an export that failed half way
  auto* p = new ArrayPriv();
  p->buffers.push_back(nullptr);
  p->children.resize(schema.size());
  p->child_ptrs.resize(schema.size());
  std::vector<size_t> view_cols;
  for (size_t i = 0; i < schema.size(); ++i)
    if (schema[i].type.id == TypeId::Utf8View && b->cols[i].length > 0) view_cols.push_back(i);
  const unsigned int* max_len = nullptr;
  if (!view_cols.empty()) {
    BufPtr mx = dev_alloc_zero(ctx, view_cols.size() * 4);
    for (size_t k = 0; k < view_cols.size(); ++k)
      SG_CUDA(launch_max_view_len(b->cols[view_cols[k]].data->ptr, b->cols[view_cols[k]].length, static_cast<unsigned int*>(mx->ptr) + k, ctx->stream));
    max_len = static_cast<const unsigned int*>(to_host(ctx, mx->ptr, view_cols.size() * 4, p));
  }
  auto is_view = [&](size_t i) { return std::find(view_cols.begin(), view_cols.end(), i) != view_cols.end(); };
  for (size_t i = 0; i < schema.size(); ++i) {
    p->children[i].release = nullptr;
    export_column(ctx, schema[i], b->cols[i], &p->children[i], false, is_view(i));
    p->child_ptrs[i] = &p->children[i];
  }
  stream_sync(ctx);
  finish_small_d2h(ctx);
  bool again = false;
  for (size_t k = 0; k < view_cols.size(); ++k) {
    if (max_len[k] <= 12) continue;
    const size_t i = view_cols[k];
    p->children[i].release(&p->children[i]);
    export_column(ctx, schema[i], b->cols[i], &p->children[i], false, false);
    again = true;
  }
  if (again) {
    stream_sync(ctx);
    finish_small_d2h(ctx);
  }
  init_array(out, b->rows, 0, p);
  out->n_children = (int64_t)schema.size();
  out->children = p->child_ptrs.data();
}

void export_device_batch(Ctx* ctx, const Schema& schema, const BatchPtr& b, ArrowDeviceArray* out, bool handle_only) {
  auto* p = new ArrayPriv();
  p->buffers.push_back(nullptr);
  p->batch = b;
  p->ctx = ctx;
  if (handle_only) {
    // a HANDLE: the batch stays in the library's internal form (resolved string views, no compacted heaps, no Arrow child
    // structs) and nothing is waited for -- only sailgpu_op_push_device of this library can consume it (take_internal_batch)
    p->opaque = true;
    init_array(&out->array, b->rows, 0, p);
    out->array.n_children = 0;
    out->array.children = nullptr;
  } else {
    p->children.resize(schema.size());
    p->child_ptrs.resize(schema.size());
    for (size_t i = 0; i < schema.size(); ++i) {
      p->children[i].release = nullptr;
      export_column(ctx, schema[i], b->cols[i], &p->children[i], true);
      p->child_ptrs[i] = &p->children[i];
    }
    stream_sync(ctx);   // consumer may use any stream: hand over completed data
    init_array(&out->array, b->rows, 0, p);
    out->array.n_children = (int64_t)schema.size();
    out->array.children = p->child_ptrs.data();
  }
  out->device_id = ctx->device;
  out->device_type = ARROW_DEVICE_CUDA;
  out->sync_event = nullptr;
  out->reserved[0] = out->reserved[1] = out->reserved[2] = 0;
}

// internal fast path: a device array we exported ourselves carries the batch
BatchPtr take_internal_batch(ArrowDeviceArray* arr, Ctx* consumer) {
  if (arr->array.release != release_array) return nullptr;
  auto* p = static_cast<ArrayPriv*>(arr->array.private_data);
  BatchPtr b = p->batch;
  if (b) {
    // a handle was not waited for at export: work queued on another context's stream must be complete before this one reads it
    if (p->opaque && p->ctx && p->ctx != consumer) cudaStreamSynchronize(p->ctx->stream);
    arr->array.release(&arr->array);
  }
  return b;
}

// ---------------------------------------------------------------------------------------------
// concat / empty
// ---------------------------------------------------------------------------------------------
BatchPtr empty_batch(Ctx* ctx, const Schema& schema) {
  auto b = std::make_shared<DevBatch>();
  for (auto& f : schema) {
    DevColumn c; c.type = f.type; c.length = 0; c.data = dev_alloc(ctx, 0);
    c.arrow_is_utf8 = f.type.id == TypeId::Utf8;
    b->cols.push_back(c);
  }
  return b;
}

BatchPtr concat_batches(Ctx* ctx, const Schema& schema, const std::vector<BatchPtr>& parts) {
  if (parts.empty()) return empty_batch(ctx, schema);
  if (parts.size() == 1) return parts[0];
  auto out = std::make_shared<DevBatch>();
  int64_t total = 0;
  for (auto& p : parts) total += p->rows;
  out->rows = total;
  for (size_t ci = 0; ci < schema.size(); ++ci) {
    const DataType& t = schema[ci].type;
    DevColumn c; c.type = t; c.length = total; c.arrow_is_utf8 = t.id == TypeId::Utf8;
    bool any_valid = false;
    for (auto& p : parts) any_valid |= (bool)p->cols[ci].validity;
    const bool bits = t.id == TypeId::Bool;
    const int w = t.is_string() ? 16 : t.arrow_width();
    if (!bits) {
      c.data = dev_alloc(ctx, (size_t)total * w);
      int64_t off = 0;
      for (auto& p : parts) {
        const DevColumn& s = p->cols[ci];
        if (s.length) SG_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(c.data->ptr) + off * w, s.data->ptr, (size_t)s.length * w, cudaMemcpyDeviceToDevice, ctx->stream));
        off += s.length;
        for (auto& h : s.heaps) c.heaps.push_back(h);
      }
    }
    if (bits || any_valid) {
      // go through bytes: unpack every part at its row offset, pack once
      BufPtr bytes = dev_alloc(ctx, (size_t)total);
      auto gather_bits = [&](bool validity) {
        int64_t off = 0;
        for (auto& p : parts) {
          const DevColumn& s = p->cols[ci];
          const BufPtr& src = validity ? s.validity : s.data;
          if (s.length) {
            if (src) SG_CUDA(launch_unpack_bits(static_cast<const uint8_t*>(src->ptr), static_cast<uint8_t*>(bytes->ptr) + off, s.length, 0, ctx->stream));
            else SG_CUDA(cudaMemsetAsync(static_cast<uint8_t*>(bytes->ptr) + off, 1, (size_t)s.length, ctx->stream));
          }
          off += s.length;
        }
        BufPtr packed = dev_alloc_zero(ctx, (size_t)((total + 31) / 32 * 4));
        SG_CUDA(launch_pack_bytes(static_cast<const uint8_t*>(bytes->ptr), static_cast<uint32_t*>(packed->ptr), total, nullptr, ctx->stream));
        return packed;
      };
      if (bits) c.data = gather_bits(false);
      if (any_valid) { c.validity = gather_bits(true); c.null_count = -1; }
    }
    out->cols.push_back(c);
  }
  return out;
}

}  // namespace sg
