"""datagen/tpch_gpu.py -- TPC-H orders / lineitem generated on the GPU (datagen/tpch_dbgen_gpu.cu) as HBM-resident
Arrow batches.  Bench / test infrastructure; bit-identical to datagen/tpch.py (tests/test_gpu_datagen.py)."""
from __future__ import annotations

import ctypes
import os
import subprocess

import pyarrow as pa

from . import tpch

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libtpch_dbgen_gpu.so")
_lib = None

ORDERS_TYPES = {"o_orderkey": pa.int64(), "o_custkey": pa.int64(), "o_orderdate": pa.date32(), "o_shippriority": pa.int32(),
                "o_totalprice": pa.decimal128(15, 2), "o_orderstatus": pa.string_view()}
LINEITEM_TYPES = {"l_orderkey": pa.int64(), "l_partkey": pa.int64(), "l_suppkey": pa.int64(), "l_linenumber": pa.int32(),
                  "l_quantity": pa.decimal128(15, 2), "l_extendedprice": pa.decimal128(15, 2), "l_discount": pa.decimal128(15, 2),
                  "l_tax": pa.decimal128(15, 2), "l_returnflag": pa.string_view(), "l_linestatus": pa.string_view(),
                  "l_shipdate": pa.date32(), "l_commitdate": pa.date32(), "l_receiptdate": pa.date32()}
_FIELDS = list(ORDERS_TYPES) + list(LINEITEM_TYPES)


class _Out(ctypes.Structure):
    _fields_ = [(f, ctypes.c_void_p) for f in _FIELDS]


_ARCH = "arch=compute_90a,code=sm_90a"


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "tpch_dbgen_gpu.cu")
    stamp = _SO + ".arch"
    if not os.path.exists(stamp) or open(stamp).read() != _ARCH:
        force = True        # a library built for another architecture
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.check_call([nvcc, "-gencode", _ARCH, "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-o", _SO, src, "-lcudart"])
        with open(stamp, "w") as f:
            f.write(_ARCH)
    return _SO


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build())
        _lib.tpch_gpu_count_lines.argtypes = [ctypes.c_longlong, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_void_p]
        _lib.tpch_gpu_generate.argtypes = [ctypes.c_longlong] * 5 + [ctypes.c_void_p, ctypes.POINTER(_Out), ctypes.c_void_p]
    return _lib


def _width(t: pa.DataType) -> int:
    return 16 if (pa.types.is_decimal(t) or t == pa.string_view()) else t.bit_width // 8


class Generated:
    """Columns of one generated table as raw device buffers (torch uint8 tensors in Arrow layout)."""

    def __init__(self, schema: pa.Schema, rows: int, buffers: list):
        self.schema, self.rows, self.buffers = schema, rows, buffers

    def device_batch(self, ctx=None):
        from sail_b200 import engine
        return engine.device_batch_from_buffers(self.schema, self.rows, self.buffers, ctx)

    def host_table(self) -> pa.Table:
        """D2H copy (torch, pageable host memory) wrapped as a pyarrow table: no library of the product involved"""
        arrays = []
        for f, t in zip(self.schema, self.buffers):
            w = _width(f.type)
            host = t[: self.rows * w].cpu().numpy()
            bufs = [None, pa.py_buffer(host)]
            if f.type == pa.string_view():
                arrays.append(pa.Array.from_buffers(f.type, self.rows, bufs))
            else:
                arrays.append(pa.Array.from_buffers(f.type, self.rows, bufs, null_count=0))
        return pa.table(arrays, schema=self.schema)


def generate_buffers(sf: float, first: int, n: int, orders_cols=(), lineitem_cols=(), device: int = 0):
    """Order rows [first, first+n) of an SF `sf` database and their lineitems, generated in HBM.
    Returns (orders Generated | None, lineitem Generated | None)."""
    import torch
    dev = torch.device("cuda", device)
    c = tpch.counts(sf)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev)
        lines = torch.empty(n, dtype=torch.int32, device=dev)
        rc = lib().tpch_gpu_count_lines(first, n, lines.data_ptr(), stream.cuda_stream)
        assert rc == 0, f"count_lines kernel failed: {rc}"
        incl = torch.cumsum(lines, 0, dtype=torch.int64)
        n_lines = int(incl[-1].item()) if n else 0
        offs = incl - lines
        out = _Out()
        bufs_o, bufs_l = {}, {}
        for name in orders_cols:
            bufs_o[name] = torch.empty(n * _width(ORDERS_TYPES[name]) + 256, dtype=torch.uint8, device=dev)
            setattr(out, name, bufs_o[name].data_ptr())
        for name in lineitem_cols:
            bufs_l[name] = torch.empty(n_lines * _width(LINEITEM_TYPES[name]) + 256, dtype=torch.uint8, device=dev)
            setattr(out, name, bufs_l[name].data_ptr())
        rc = lib().tpch_gpu_generate(c["part"], c["supplier"], c["customer"], first, n, offs.data_ptr(), ctypes.byref(out), stream.cuda_stream)
        assert rc == 0, f"generate kernel failed: {rc}"
        stream.synchronize()
    del lines, incl, offs
    o = Generated(pa.schema([(k, ORDERS_TYPES[k]) for k in orders_cols]), n, [bufs_o[k] for k in orders_cols]) if orders_cols else None
    l = Generated(pa.schema([(k, LINEITEM_TYPES[k]) for k in lineitem_cols]), n_lines, [bufs_l[k] for k in lineitem_cols]) if lineitem_cols else None
    return o, l


def generate(sf: float, first: int, n: int, orders_cols=(), lineitem_cols=(), ctx=None):
    """Same, as HBM-resident Arrow batches (engine.DeviceBatch) of `ctx`."""
    from sail_b200 import engine
    ctx = ctx or engine.default_context()
    o, l = generate_buffers(sf, first, n, orders_cols, lineitem_cols, ctx.device)
    return (o.device_batch(ctx) if o else None), (l.device_batch(ctx) if l else None)
