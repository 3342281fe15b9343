"""Plan-time kernel specialisation for the pipelines bench.py and the evidence scripts run: generates and NVRTC-compiles
their specialised kernels into sail_b200/_build/jit_cache (no GPU needed), so that the first batch on the GPU finds
the cubin instead of paying a compilation.  What a rewrite pass does through sailgpu_jit_precompile while planning."""
from __future__ import annotations

import pyarrow as pa

from . import engine

D152 = pa.decimal128(15, 2)


def pipelines():
    import bench
    fused, final, sort = bench.q1_specs()
    q1_schema = pa.schema([("l_quantity", D152), ("l_extendedprice", D152), ("l_discount", D152), ("l_tax", D152),
                           ("l_returnflag", pa.string_view()), ("l_linestatus", pa.string_view()), ("l_shipdate", pa.date32())])
    out = [("q1 fused partial", fused, q1_schema, 0, 0)]
    xs = pa.schema([("l_orderkey", pa.int64()), ("l_quantity", D152)])
    partial = {"op": "aggregate", "mode": "partial", "group_by": [{"expr": {"col": 0}, "name": "l_orderkey"}],
               "aggs": [{"fn": "sum", "name": "sum_qty", "input_type": "Decimal128(15,2)", "args": [{"col": 1}]}, {"fn": "count", "name": "cnt", "input_type": None, "args": []}]}
    out.append(("group by l_orderkey (dictionary)", partial, xs, 0, 0))
    out.append(("group by l_orderkey (global table)", partial, xs, 0, engine.JIT_COLD_VARIANT))
    return out


def warm(verbose: bool = False) -> int:
    n = 0
    for name, spec, schema, mask, flags in pipelines():
        try:
            size, _ = engine.jit_precompile(spec, [schema], mask, flags | engine.JIT_COMPILE)
            n += 1
            if verbose:
                print(f"[jit_warm] {name}: {size} B")
        except engine.SailGpuError as e:      # a pipeline the specialiser does not cover stays interpreted
            if verbose:
                print(f"[jit_warm] {name}: {e}")
    return n


if __name__ == "__main__":
    warm(True)
