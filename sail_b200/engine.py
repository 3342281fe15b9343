"""Host-side mirror of the reference's operator interface over the libsailgpu C ABI.

In Sail the callers are Rust: `ExecutionPlan::execute(partition, ctx) -> SendableRecordBatchStream`
(shape: crates/sail-execution/src/plan/shuffle_write.rs:146-206) and the stream's `poll_next`.
The Rust toolchain is absent from this image, so this module plays that role for tests and the
bench: `GpuExec` <-> a DataFusion `ExecutionPlan` node, `push/finish/pull` <-> what the shim's
`poll_next` does with each child batch (INTEGRATION.md has the Rust side).  Everything below goes
through `include/sailgpu.h` entry points with Arrow C Data Interface structs -- no torch types.

There is no CPU fallback: importing works anywhere (so symbol/ABI tests run on CPU), but creating a
`Context` without an H100 raises `GpuUnavailable`.
"""
from __future__ import annotations

import ctypes
import json
import os
import sys

import pyarrow as pa

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_build", "libsailgpu.so")


class ArrowSchemaC(ctypes.Structure):
    _fields_ = [("format", ctypes.c_char_p), ("name", ctypes.c_char_p), ("metadata", ctypes.c_char_p),
                ("flags", ctypes.c_int64), ("n_children", ctypes.c_int64), ("children", ctypes.c_void_p),
                ("dictionary", ctypes.c_void_p), ("release", ctypes.c_void_p), ("private_data", ctypes.c_void_p)]


class ArrowArrayC(ctypes.Structure):
    _fields_ = [("length", ctypes.c_int64), ("null_count", ctypes.c_int64), ("offset", ctypes.c_int64),
                ("n_buffers", ctypes.c_int64), ("n_children", ctypes.c_int64), ("buffers", ctypes.c_void_p),
                ("children", ctypes.c_void_p), ("dictionary", ctypes.c_void_p), ("release", ctypes.c_void_p),
                ("private_data", ctypes.c_void_p)]


class ArrowDeviceArrayC(ctypes.Structure):
    _fields_ = [("array", ArrowArrayC), ("device_id", ctypes.c_int64), ("device_type", ctypes.c_int32),
                ("sync_event", ctypes.c_void_p), ("reserved", ctypes.c_int64 * 3)]


class SailGpuError(RuntimeError):
    def __init__(self, code, message):
        super().__init__(f"[sailgpu {code}] {message}")
        self.code = code


class GpuUnavailable(SailGpuError):
    pass


ERR_NO_DEVICE = 5
_lib = None


def lib():
    """Loads libsailgpu.so (built in-tree by sail_b200/build.py).  Fails loudly when it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SailGpuError(-1, f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
        L = ctypes.CDLL(LIB_PATH)
        vp, i32, i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
        L.sailgpu_version.restype = ctypes.c_uint32
        L.sailgpu_ctx_create.argtypes = [i32, ctypes.POINTER(vp)]
        L.sailgpu_ctx_destroy.argtypes = [vp]
        L.sailgpu_ctx_destroy.restype = None
        L.sailgpu_ctx_last_error.argtypes = [vp]
        L.sailgpu_ctx_last_error.restype = ctypes.c_char_p
        L.sailgpu_ctx_stream.argtypes = [vp]
        L.sailgpu_ctx_stream.restype = vp
        L.sailgpu_ctx_synchronize.argtypes = [vp]
        L.sailgpu_op_create.argtypes = [vp, ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(vp), i32, i32,
                                        ctypes.POINTER(vp), vp]
        L.sailgpu_spec_validate.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(vp), i32, vp, ctypes.c_char_p, ctypes.c_size_t]
        L.sailgpu_jit_precompile.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(vp), i32, ctypes.c_uint64, i32, ctypes.c_char_p, ctypes.c_size_t]
        L.sailgpu_jit_precompile.restype = i64
        L.sailgpu_parquet_decode.argtypes = [vp, vp, vp, i32, i64, vp]
        L.sailgpu_parquet_inspect.argtypes = [vp, vp, i32, i64, i32, ctypes.c_char_p, ctypes.c_size_t]
        L.sailgpu_parquet_stats.argtypes = [vp, ctypes.c_char_p, ctypes.c_size_t]
        L.sailgpu_op_push.argtypes = [vp, i32, vp]
        L.sailgpu_op_push_device.argtypes = [vp, i32, vp]
        L.sailgpu_op_finish_input.argtypes = [vp, i32]
        L.sailgpu_op_pull.argtypes = [vp, vp, ctypes.POINTER(i32)]
        L.sailgpu_op_pull_device.argtypes = [vp, vp, ctypes.POINTER(i32)]
        L.sailgpu_op_pull_device_handle.argtypes = [vp, vp, ctypes.POINTER(i32)]
        L.sailgpu_op_pull_partition.argtypes = [vp, i32, vp, ctypes.POINTER(i32)]
        L.sailgpu_op_metrics.argtypes = [vp, ctypes.c_char_p, ctypes.c_size_t]
        L.sailgpu_op_metrics.restype = i64
        L.sailgpu_last_error.argtypes = [vp]
        L.sailgpu_last_error.restype = ctypes.c_char_p
        L.sailgpu_op_destroy.argtypes = [vp]
        L.sailgpu_op_destroy.restype = None
        L.sailgpu_host_alloc.argtypes = [vp, ctypes.c_size_t, ctypes.POINTER(vp)]
        L.sailgpu_host_free.argtypes = [vp, vp]
        L.sailgpu_host_free.restype = None
        L.sailgpu_comm_unique_id.argtypes = [ctypes.c_char_p]
        L.sailgpu_ctx_comm_init.argtypes = [vp, ctypes.c_char_p, i32, i32]
        L.sailgpu_exchange.argtypes = [vp, vp, vp, i32, vp]
        L.sailgpu_ipc_stream.argtypes = [vp, vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_size_t)]
        L.sailgpu_op_pull_ipc.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(i64), ctypes.POINTER(i32)]
        L.sailgpu_ipc_last_error.restype = ctypes.c_char_p
        L.sailgpu_ipc_free.argtypes = [vp]
        L.sailgpu_ipc_free.restype = None
        _lib = L
    return _lib


class Context:
    def __init__(self, device: int = 0):
        self._h = ctypes.c_void_p()
        rc = lib().sailgpu_ctx_create(device, ctypes.byref(self._h))
        if rc != 0:
            msg = lib().sailgpu_ctx_last_error(None).decode()
            raise (GpuUnavailable if rc == ERR_NO_DEVICE else SailGpuError)(rc, msg)
        self.device = device

    def close(self):
        if self._h:
            lib().sailgpu_ctx_destroy(self._h)
            self._h = ctypes.c_void_p()

    def stream(self) -> int:
        """cudaStream_t of this context as an integer (wrap with torch.cuda.ExternalStream to record events)"""
        return int(lib().sailgpu_ctx_stream(self._h) or 0)

    def synchronize(self):
        rc = lib().sailgpu_ctx_synchronize(self._h)
        if rc != 0:
            raise SailGpuError(rc, lib().sailgpu_ctx_last_error(None).decode())

    def comm_init(self, unique_id: bytes, rank: int, world: int):
        rc = lib().sailgpu_ctx_comm_init(self._h, unique_id, rank, world)
        if rc != 0:
            raise SailGpuError(rc, lib().sailgpu_ctx_last_error(None).decode())

    def __del__(self):
        try:
            if not sys.is_finalizing():
                self.close()
        except Exception:
            pass


def comm_unique_id() -> bytes:
    buf = ctypes.create_string_buffer(128)
    rc = lib().sailgpu_comm_unique_id(buf)
    if rc != 0:
        raise SailGpuError(rc, "sailgpu_comm_unique_id failed")
    return buf.raw


_default_ctx = None


def default_context() -> Context:
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context(int(os.environ.get("LOCAL_RANK", "0")))
    return _default_ctx


class DeviceBatch:
    """An Arrow C Device array (ARROW_DEVICE_CUDA) resident in HBM.  Owns the C struct until it is
    pushed into an operator (push takes ownership) or dropped."""

    def __init__(self, schema: pa.Schema):
        self.schema = schema
        self.c = ArrowDeviceArrayC()
        self._live = False

    @property
    def num_rows(self) -> int:
        return self.c.array.length

    def borrow(self) -> "DeviceBatch":
        """A second handle on the same HBM buffers whose release is a no-op: lets a resident batch be
        pushed into many operators (each push consumes only the borrowed handle)."""
        b = DeviceBatch(self.schema)
        ctypes.memmove(ctypes.addressof(b.c), ctypes.addressof(self.c), ctypes.sizeof(ArrowDeviceArrayC))
        b.c.array.release = ctypes.cast(lib().sailgpu_borrowed_release, ctypes.c_void_p).value   # C callback: safe at interpreter exit
        b.c.array.private_data = None
        b._live = True
        b._owner = self          # keep the buffers alive
        return b

    def release(self):
        if getattr(self, "_owner", None) is not None:
            self._live = False
            return
        if self._live and self.c.array.release:
            fn = ctypes.CFUNCTYPE(None, ctypes.c_void_p)(self.c.array.release)
            fn(ctypes.addressof(self.c.array))
        self._live = False

    def __del__(self):
        try:
            if not sys.is_finalizing():
                self.release()
        except Exception:
            pass


@ctypes.CFUNCTYPE(None, ctypes.c_void_p)
def _NOOP_RELEASE(ptr):
    a = ArrowArrayC.from_address(ptr)
    a.release = None


def _export_schema(schema: pa.Schema) -> ArrowSchemaC:
    c = ArrowSchemaC()
    schema._export_to_c(ctypes.addressof(c))
    return c


def _release_schema(c: ArrowSchemaC):
    if c.release:
        ctypes.CFUNCTYPE(None, ctypes.c_void_p)(c.release)(ctypes.addressof(c))


class GpuExec:
    """One GPU operator instance (the analogue of a DataFusion ExecutionPlan node + its stream).

    spec: operator spec dict (see include/sailgpu.h); inputs: list of pyarrow.Schema.
    """

    def __init__(self, spec: dict, inputs: list, ctx: Context | None = None, partition: int = 0):
        self.ctx = ctx or default_context()
        self.spec = spec
        self.inputs = list(inputs)
        text = json.dumps(spec).encode()
        cs = [_export_schema(s) for s in inputs]
        arr = (ctypes.c_void_p * len(cs))(*[ctypes.addressof(c) for c in cs])
        out_schema = ArrowSchemaC()
        self._h = ctypes.c_void_p()
        rc = lib().sailgpu_op_create(self.ctx._h, text, len(text), arr, len(cs), partition, ctypes.byref(self._h),
                                     ctypes.addressof(out_schema))
        for c in cs:
            _release_schema(c)
        if rc != 0:
            raise SailGpuError(rc, lib().sailgpu_ctx_last_error(None).decode())
        self.schema = pa.Schema._import_from_c(ctypes.addressof(out_schema))

    def name(self) -> str:
        return {"filter": "GpuFilterExec", "projection": "GpuProjectionExec", "aggregate": "GpuAggregateExec",
                "hash_join": "GpuHashJoinExec", "sort": "GpuSortExec", "sort_preserving_merge": "GpuSortPreservingMergeExec", "repartition": "GpuRepartitionExec",
                "pipeline": "GpuPipelineExec", "chain": "GpuChainExec"}.get(self.spec.get("op"), "GpuExec")

    def _check(self, rc):
        if rc != 0:
            raise SailGpuError(rc, lib().sailgpu_last_error(self._h).decode())

    def push(self, batch, input_idx: int = 0):
        """batch: pyarrow RecordBatch/Table (host) or DeviceBatch (HBM)."""
        if isinstance(batch, DeviceBatch):
            if not batch._live:
                raise SailGpuError(6, "device batch was already consumed")
            self._check(lib().sailgpu_op_push_device(self._h, input_idx, ctypes.addressof(batch.c)))
            batch._live = False
            return
        if isinstance(batch, pa.Table):
            batch = batch.combine_chunks()
            batches = batch.to_batches()
            if not batches:
                batches = [pa.RecordBatch.from_arrays([pa.array([], type=f.type) for f in batch.schema], schema=batch.schema)]
            for b in batches:
                self.push(b, input_idx)
            return
        c = ArrowArrayC()
        batch._export_to_c(ctypes.addressof(c))
        self._check(lib().sailgpu_op_push(self._h, input_idx, ctypes.addressof(c)))

    def finish(self, input_idx: int = 0):
        self._check(lib().sailgpu_op_finish_input(self._h, input_idx))

    def pull(self):
        """-> (RecordBatch, has_more)"""
        c = ArrowArrayC()
        more = ctypes.c_int32(0)
        self._check(lib().sailgpu_op_pull(self._h, ctypes.addressof(c), ctypes.byref(more)))
        sc = _export_schema(self.schema)
        batch = pa.RecordBatch._import_from_c(ctypes.addressof(c), ctypes.addressof(sc))
        return batch, bool(more.value)

    def pull_ipc(self):
        """-> (bytes of one Arrow IPC stream holding the next batch, rows, has_more): the result sink (sailgpu_op_pull_ipc)"""
        data, n = ctypes.c_void_p(), ctypes.c_size_t(0)
        rows, more = ctypes.c_int64(0), ctypes.c_int32(0)
        self._check(lib().sailgpu_op_pull_ipc(self._h, ctypes.byref(data), ctypes.byref(n), ctypes.byref(rows), ctypes.byref(more)))
        try:
            return ctypes.string_at(data.value, n.value), rows.value, bool(more.value)
        finally:
            lib().sailgpu_ipc_free(data)

    def pull_device(self, partition: int | None = None, handle: bool = False):
        """-> (DeviceBatch, has_more).  handle=True: sailgpu_op_pull_device_handle -- no Arrow column arrays are materialised; the
        batch can only be pushed (once, not borrowed) into another operator of this library"""
        d = DeviceBatch(self.schema)
        more = ctypes.c_int32(0)
        if partition is None:
            fn = lib().sailgpu_op_pull_device_handle if handle else lib().sailgpu_op_pull_device
            self._check(fn(self._h, ctypes.addressof(d.c), ctypes.byref(more)))
        else:
            self._check(lib().sailgpu_op_pull_partition(self._h, partition, ctypes.addressof(d.c), ctypes.byref(more)))
        d._live = True
        return d, bool(more.value)

    def metrics(self) -> dict:
        buf = ctypes.create_string_buffer(2048)
        need = lib().sailgpu_op_metrics(self._h, buf, 2048)
        if need > 2048:      # a partitioned aggregate lists the groups of every partition
            buf = ctypes.create_string_buffer(need)
            lib().sailgpu_op_metrics(self._h, buf, need)
        return json.loads(buf.value.decode())

    def collect(self) -> pa.Table:
        out = []
        while True:
            b, more = self.pull()
            if b.num_rows or not more:
                out.append(b)
            if not more:
                break
        return pa.Table.from_batches(out, schema=self.schema)

    def collect_device(self, handle: bool = False) -> list:
        out = []
        while True:
            d, more = self.pull_device(handle=handle)
            if d.num_rows or not more:
                out.append(d)
            if not more:
                break
        return out

    def close(self):
        if self._h:
            lib().sailgpu_op_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            if not sys.is_finalizing():
                self.close()
        except Exception:
            pass


def ipc_stream(batch: pa.RecordBatch | None, schema: pa.Schema | None = None) -> bytes:
    """A host batch framed as one self-contained Arrow IPC stream (sailgpu_ipc_stream; batch None: schema + end-of-stream only).
    Needs no GPU and no context."""
    sc = _export_schema(batch.schema if batch is not None else schema)
    c = ArrowArrayC()
    if batch is not None:
        batch._export_to_c(ctypes.addressof(c))
    data, n = ctypes.c_void_p(), ctypes.c_size_t(0)
    try:
        rc = lib().sailgpu_ipc_stream(ctypes.addressof(sc), ctypes.addressof(c) if batch is not None else None, ctypes.byref(data), ctypes.byref(n))
        if rc != 0:
            raise SailGpuError(rc, lib().sailgpu_ipc_last_error().decode())
        return ctypes.string_at(data.value, n.value)
    finally:
        lib().sailgpu_ipc_free(data)
        _release_schema(sc)
        if batch is not None and c.release:
            ctypes.CFUNCTYPE(None, ctypes.c_void_p)(c.release)(ctypes.addressof(c))


def validate(spec: dict, inputs: list) -> pa.Schema:
    """Plan-time check (no GPU needed): output schema of `spec` over the input schemas, or SailGpuError."""
    text = json.dumps(spec).encode()
    cs = [_export_schema(s) for s in inputs]
    arr = (ctypes.c_void_p * len(cs))(*[ctypes.addressof(c) for c in cs])
    out = ArrowSchemaC()
    err = ctypes.create_string_buffer(1024)
    rc = lib().sailgpu_spec_validate(text, len(text), arr, len(cs), ctypes.addressof(out), err, 1024)
    for c in cs:
        _release_schema(c)
    if rc != 0:
        raise SailGpuError(rc, err.value.decode())
    return pa.Schema._import_from_c(ctypes.addressof(out))


JIT_COLD_VARIANT, JIT_COMPILE = 1, 2


def jit_precompile(spec: dict, inputs: list, validity_mask: int = 0, flags: int = 0) -> tuple[int, str]:
    """Plan-time kernel specialisation (no GPU needed): returns (cubin bytes or source length, generated CUDA source)
    of the specialised kernel for `spec`; with JIT_COMPILE the cubin lands in the kernel cache."""
    text = json.dumps(spec).encode()
    cs = [_export_schema(s) for s in inputs]
    arr = (ctypes.c_void_p * len(cs))(*[ctypes.addressof(c) for c in cs])
    cap = 1 << 20
    buf = ctypes.create_string_buffer(cap)
    n = lib().sailgpu_jit_precompile(text, len(text), arr, len(cs), validity_mask, flags, buf, cap)
    for c in cs:
        _release_schema(c)
    if n < 0:
        raise SailGpuError(int(-n), buf.value.decode())
    return int(n), buf.value.decode()


def run_op(spec: dict, *tables, ctx: Context | None = None) -> pa.Table:
    """Execute one operator over whole tables through the C ABI (host buffers in, host buffers out)."""
    op = GpuExec(spec, [t.schema for t in tables], ctx)
    try:
        for i, t in enumerate(tables):
            op.push(t, i)
            op.finish(i)
        return op.collect()
    finally:
        op.close()


def exchange(send: list, schema: pa.Schema, ctx: Context | None = None) -> DeviceBatch:
    """All-to-all over NCCL/NVLink: send[p] (DeviceBatch) goes to rank p; returns what this rank received.
    Replaces the body of shuffle_write/shuffle_read for Partitioning::Hash
    (crates/sail-execution/src/plan/shuffle_write.rs:209-267, shuffle_read.rs:107-117)."""
    ctx = ctx or default_context()
    n = len(send)
    arr = (ArrowDeviceArrayC * n)()
    for i, d in enumerate(send):
        if d is None:
            continue                      # zeroed struct (release == NULL): nothing for rank i
        if not d._live:
            raise SailGpuError(6, "device batch was already consumed")
        ctypes.memmove(ctypes.addressof(arr[i]), ctypes.addressof(d.c), ctypes.sizeof(ArrowDeviceArrayC))
        d._live = False
    out = DeviceBatch(schema)
    sc = _export_schema(schema)
    rc = lib().sailgpu_exchange(ctx._h, ctypes.addressof(sc), ctypes.addressof(arr), n, ctypes.addressof(out.c))
    _release_schema(sc)
    if rc != 0:
        raise SailGpuError(rc, "sailgpu_exchange failed")
    out._live = True
    return out


_FOREIGN_KEEP = {}     # id -> objects a foreign device batch borrows from (dropped by its release callback)


@ctypes.CFUNCTYPE(None, ctypes.c_void_p)
def _foreign_release(ptr):
    a = ArrowArrayC.from_address(ptr)
    _FOREIGN_KEEP.pop(int(a.private_data or 0), None)
    a.release = None


def device_batch_from_buffers(schema: pa.Schema, n_rows: int, tensors: list, ctx: Context | None = None) -> DeviceBatch:
    """Wraps caller-owned device memory (objects with .data_ptr(), e.g. torch tensors; one values buffer per column, no
    nulls, strings as inline Utf8View) as an ARROW_DEVICE_CUDA batch -- what a GPU-side producer (a Parquet decoder, the
    data generator) hands to sailgpu_op_push_device without a copy."""
    ctx = ctx or default_context()
    n = len(tensors)
    assert n == len(schema)
    children = (ArrowArrayC * n)()
    child_ptrs = (ctypes.c_void_p * n)()
    bufs = []
    for i, t in enumerate(tensors):
        is_view = schema.field(i).type == pa.string_view()
        nb = 3 if is_view else 2           # views: validity, views, variadic sizes (no data buffers: every view is inline)
        b = (ctypes.c_void_p * nb)()
        b[1] = t.data_ptr()
        bufs.append(b)
        c = children[i]
        c.length, c.null_count, c.offset, c.n_buffers, c.n_children = n_rows, 0, 0, nb, 0
        c.buffers = ctypes.cast(b, ctypes.c_void_p)
        c.release = ctypes.cast(_NOOP_RELEASE, ctypes.c_void_p).value
        child_ptrs[i] = ctypes.addressof(c)
    d = DeviceBatch(schema)
    top = (ctypes.c_void_p * 1)()
    a = d.c.array
    a.length, a.null_count, a.offset, a.n_buffers, a.n_children = n_rows, 0, 0, 1, n
    a.buffers = ctypes.cast(top, ctypes.c_void_p)
    a.children = ctypes.cast(child_ptrs, ctypes.c_void_p)
    key = id(d)
    a.private_data = key
    a.release = ctypes.cast(_foreign_release, ctypes.c_void_p).value
    _FOREIGN_KEEP[key] = (children, child_ptrs, bufs, top, list(tensors))
    d.c.device_id = ctx.device
    d.c.device_type = 2      # ARROW_DEVICE_CUDA
    d._live = True
    return d


class ParquetColumnC(ctypes.Structure):
    _fields_ = [("chunk", ctypes.c_void_p), ("chunk_len", ctypes.c_uint64), ("physical_type", ctypes.c_int32), ("type_length", ctypes.c_int32),
                ("max_def_level", ctypes.c_int32), ("codec", ctypes.c_int32), ("num_values", ctypes.c_int64)]


_PQ_PHYSICAL = {"BOOLEAN": 0, "INT32": 1, "INT64": 2, "INT96": 3, "FLOAT": 4, "DOUBLE": 5, "BYTE_ARRAY": 6, "FIXED_LEN_BYTE_ARRAY": 7}
_PQ_CODEC = {"UNCOMPRESSED": 0, "SNAPPY": 1, "GZIP": 2, "LZO": 3, "BROTLI": 4, "LZ4": 5, "ZSTD": 6, "LZ4_RAW": 7}


def _parquet_descriptors(file_bytes, row_group: int, columns: list | None, binary_as_string: bool = False):
    import pyarrow.parquet as pq
    buf = pa.py_buffer(file_bytes)
    f = pq.ParquetFile(pa.BufferReader(buf))
    rg = f.metadata.row_group(row_group)
    names = [f.schema.column(i).name for i in range(rg.num_columns)]
    columns = list(columns or names)
    fields, cols = [], (ParquetColumnC * len(columns))()
    for k, name in enumerate(columns):
        i = names.index(name)
        cm, cs = rg.column(i), f.schema.column(i)
        t = f.schema_arrow.field(name).type
        if pa.types.is_string(t) or pa.types.is_large_string(t):
            t = pa.string_view()
        elif binary_as_string and (pa.types.is_binary(t) or pa.types.is_large_binary(t)):
            t = pa.string_view()         # DataFusion's `binary_as_string`: unannotated BYTE_ARRAY columns read as strings
        fields.append(pa.field(name, t, nullable=cs.max_definition_level > 0))
        start = cm.data_page_offset
        if cm.has_dictionary_page and cm.dictionary_page_offset is not None:
            start = min(start, cm.dictionary_page_offset)
        c = cols[k]
        c.chunk = buf.address + start
        c.chunk_len = cm.total_compressed_size
        c.physical_type = _PQ_PHYSICAL[cm.physical_type]
        c.type_length = cs.length if cm.physical_type == "FIXED_LEN_BYTE_ARRAY" else 0
        c.max_def_level = cs.max_definition_level
        c.codec = _PQ_CODEC.get(cm.compression, 99)
        c.num_values = cm.num_values
    return buf, pa.schema(fields), cols, rg.num_rows


def parquet_decode(file_bytes, row_group: int = 0, columns: list | None = None, ctx: Context | None = None,
                   binary_as_string: bool = False) -> DeviceBatch:
    """One row group of a Parquet file (bytes in host memory) decoded on the device: the footer is read here with pyarrow (the
    Rust side uses the `parquet` crate), the column chunks go to sailgpu_parquet_decode as stored.  binary_as_string: BYTE_ARRAY
    columns without a UTF8 annotation decode to Utf8View (their bytes unchanged, not validated as UTF-8); without it such a
    column is refused (SAILGPU_ERR_UNSUPPORTED), as the library has no binary type."""
    ctx = ctx or default_context()
    buf, schema, cols, n_rows = _parquet_descriptors(file_bytes, row_group, columns, binary_as_string)
    cschema = _export_schema(schema)
    d = DeviceBatch(schema)
    rc = lib().sailgpu_parquet_decode(ctx._h, ctypes.addressof(cschema), ctypes.addressof(cols), len(cols), n_rows, ctypes.addressof(d.c))
    _release_schema(cschema)
    del buf
    if rc != 0:
        raise SailGpuError(rc, lib().sailgpu_ctx_last_error(None).decode())
    d._live = True
    return d


def parquet_inspect(file_bytes, column: int, row_group: int = 0, columns: list | None = None, binary_as_string: bool = False) -> dict:
    """Host-only: what the page / run-header walk of sailgpu_parquet_decode finds in one column chunk (no GPU needed)."""
    buf, schema, cols, n_rows = _parquet_descriptors(file_bytes, row_group, columns, binary_as_string)
    cschema = _export_schema(schema)
    out = ctypes.create_string_buffer(1024)
    rc = lib().sailgpu_parquet_inspect(ctypes.addressof(cschema), ctypes.addressof(cols), len(cols), n_rows, column, out, 1024)
    _release_schema(cschema)
    del buf
    if rc != 0:
        raise SailGpuError(rc, out.value.decode())
    return json.loads(out.value.decode())


def parquet_stats(ctx: Context | None = None) -> dict:
    """What the last parquet_decode on `ctx` spent on ZSTD pages: page count, decompressed bytes, image bytes read back, and the
    device milliseconds of the decompression launch and of the read-back."""
    ctx = ctx or default_context()
    out = ctypes.create_string_buffer(512)
    rc = lib().sailgpu_parquet_stats(ctx._h, out, 512)
    if rc != 0:
        raise SailGpuError(rc, lib().sailgpu_ctx_last_error(None).decode())
    return json.loads(out.value.decode())


def to_device(table: pa.Table, ctx: Context | None = None) -> DeviceBatch:
    """Upload a table once; the returned DeviceBatch is HBM-resident Arrow (used by the bench's
    'inputs already resident in HBM' leg)."""
    spec = {"op": "projection", "exprs": [{"expr": {"col": i}, "name": n} for i, n in enumerate(table.schema.names)]}
    op = GpuExec(spec, [table.schema], ctx)
    try:
        op.push(table)
        op.finish()
        parts = op.collect_device()
        assert len(parts) == 1, "to_device expects a single-chunk table"
        d = parts[0]
        d.schema = table.schema
        return d
    finally:
        op.close()
