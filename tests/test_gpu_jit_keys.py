"""GPU parity of the SPECIALISED aggregate kernel across group-key shapes.  The key travels in registers as G::Key (jit.cu,
jit_rt.cuh), padded to the dictionary's four words: Q1's two Utf8View keys (four words, register tier), a nullable key
(a null-mask word in front), a single 8-byte key (one-word global table), a float sum (dictionary tier) and three Decimal128
keys (six words: wider than the dictionary, global table only).  Specialisation is forced from the first row; batch sizes
include a partial last tile and more tiles than CTAs."""
import decimal

import numpy as np
import pyarrow as pa
import pytest

from tests.util import assert_same, oracle_op

pytestmark = pytest.mark.gpu

D152 = pa.decimal128(15, 2)


@pytest.fixture(autouse=True)
def specialised(monkeypatch):
    monkeypatch.setenv("SAILGPU_JIT_MIN_ROWS", "0")
    monkeypatch.setenv("SAILGPU_JIT_STRICT", "1")


def run(spec, t):
    from sail_b200 import engine
    op = engine.GpuExec(spec, [t.schema])
    op.push(t)
    op.finish()
    got = op.collect()
    m = op.metrics()
    op.close()
    assert m.get("gpu.jit_launches", 0) >= 1
    return got


def dec(rng, n, lo=-10**9, hi=10**9):
    return pa.array([decimal.Decimal(int(x)) / 100 for x in rng.integers(lo, hi, n)], type=D152)


def table(shape, n):
    rng = np.random.default_rng(n)
    if shape == "nullable":
        k = pa.array(rng.integers(0, 5, n).astype(np.int32), mask=rng.random(n) < 0.1)
        return pa.table({"k": k, "k2": pa.array(rng.integers(0, 2, n).astype(np.int64)), "v": dec(rng, n)}), ["k", "k2"]
    if shape == "int64":
        return pa.table({"k": pa.array(rng.integers(0, 3, n).astype(np.int64)), "v": dec(rng, n)}), ["k"]
    if shape == "float":
        return pa.table({"k": pa.array(rng.integers(0, 6, n).astype(np.int32)), "v": pa.array(rng.standard_normal(n))}), ["k"]
    if shape == "wide":
        return pa.table({"a": dec(rng, n, 0, 3), "b": dec(rng, n, 0, 2), "c": dec(rng, n, 0, 2), "v": dec(rng, n)}), ["a", "b", "c"]
    raise ValueError(shape)


@pytest.mark.parametrize("n", [513, 200_003])
@pytest.mark.parametrize("shape", ["nullable", "int64", "float", "wide"])
def test_specialised_aggregate_key_shapes(shape, n):
    t, keys = table(shape, n)
    spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": t.schema.get_field_index(k)}, "name": k} for k in keys],
            "aggs": [{"fn": "sum", "args": [{"col": t.num_columns - 1}], "name": "s"}, {"fn": "count", "args": [], "name": "c"}]}
    assert_same(run(spec, t), oracle_op(spec, t), float_cols=(len(keys),) if shape == "float" else ())


@pytest.mark.parametrize("sf", [0.01, 0.05])
def test_specialised_q1_partial(sf):
    """Q1's fused Filter -> Projection -> Aggregate(Partial) over two Utf8View keys, then the final aggregate and the sort,
    against the oracle's Q1 plan"""
    import bench
    from datagen import tpch
    from sail_b200 import engine, plans
    lineitem = tpch.lineitem(sf)
    fused, final, sort = bench.q1_specs()
    got = engine.run_op(sort, engine.run_op(final, run(fused, lineitem.select(bench.Q1_COLS))))
    assert_same(got, plans.execute(plans.q1(), {"lineitem": lineitem}, oracle_op))
