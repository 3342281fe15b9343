"""GPU parity of the SPECIALISED pipeline kernel (jit.cu / jit_rt.cuh): the pipeline parity cases of test_gpu_pipeline,
run again with specialisation forced from the first row (SAILGPU_JIT_MIN_ROWS=0; a kernel that fails to build is an
error, SAILGPU_JIT_STRICT=1) at the planner's stage count and at four stages.  The batch sizes of those cases include
ones with a partial last tile and ones with fewer tiles than CTAs; the bounded-table cases below give every CTA many
tiles, so hand-backs are decided in the middle of a CTA's tile loop."""
import decimal

import numpy as np
import pyarrow as pa
import pytest

from tests.test_gpu_pipeline import (  # noqa: F401  (collected here, under the fixture below)
    test_aggregate_bounded_table_grows_by_itself,
    test_aggregate_bounded_table_hands_tiles_back,
    test_aggregate_many_groups_multi_batch_growth,
    test_aggregate_single,
    test_filter,
    test_filter_two_pass,
    test_fused_pipeline_matches_operator_chain,
    test_projection,
    test_tpch_pipeline_queries,
)
from tests.util import assert_same, oracle_op

pytestmark = pytest.mark.gpu

# SAILGPU_JIT_STAGES; "" keeps the planner's choice
STAGES = ["", "4"]


@pytest.fixture(autouse=True, params=STAGES, ids=lambda s: f"stages{s or 'D'}")
def specialised(request, monkeypatch):
    monkeypatch.setenv("SAILGPU_JIT_MIN_ROWS", "0")
    monkeypatch.setenv("SAILGPU_JIT_STRICT", "1")
    if request.param:
        monkeypatch.setenv("SAILGPU_JIT_STAGES", request.param)
    else:
        monkeypatch.delenv("SAILGPU_JIT_STAGES", raising=False)
    return request.param


@pytest.mark.parametrize("n", [1, 255, 511, 513, 5 * 256 + 7, 200_003])
def test_specialised_kernel_runs_and_matches(n):
    """the operator really launches the specialised kernel (metrics), over partial last tiles and short batches"""
    from sail_b200 import engine
    rng = np.random.default_rng(n)
    k = rng.integers(0, 3, n).astype(np.int32)
    v = [decimal.Decimal(int(x)) / 100 for x in rng.integers(-10**9, 10**9, n)]
    t = pa.table({"k": pa.array(k), "v": pa.array(v, type=pa.decimal128(15, 2)), "i": pa.array(rng.integers(-50, 50, n).astype(np.int64))})
    spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": 0}, "name": "k"}],
            "aggs": [{"fn": "sum", "args": [{"col": 1}], "name": "sv"}, {"fn": "count", "args": [], "name": "c"},
                     {"fn": "sum", "args": [{"col": 2}], "name": "si"}]}
    op = engine.GpuExec(spec, [t.schema])
    op.push(t)
    op.finish()
    got = op.collect()
    m = op.metrics()
    op.close()
    assert m.get("gpu.jit_launches", 0) >= 1
    assert_same(got, oracle_op(spec, t))


@pytest.mark.parametrize("first_limit", ["0", "3000", "200000"])
def test_specialised_hand_back_with_many_tiles_per_cta(first_limit, monkeypatch):
    """1 M rows (about 15 tiles per CTA) and a forced group limit: CTAs stop after some of their tiles, hand the rest back
    and the re-launches over the deferred list finish the batch; sums and counts are checked against numpy"""
    from sail_b200 import engine
    monkeypatch.setenv("SAILGPU_AGG_FIRST_LIMIT", first_limit)
    n = 1_000_003
    rng = np.random.default_rng(17)
    k = rng.integers(0, 400_000, n).astype(np.int64)
    v = rng.integers(-1000, 1000, n).astype(np.int64)
    t = pa.table({"k": pa.array(k), "v": pa.array(v)})
    spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": 0}, "name": "k"}],
            "aggs": [{"fn": "sum", "args": [{"col": 1}], "name": "s"}, {"fn": "count", "args": [], "name": "c"}]}
    op = engine.GpuExec(spec, [t.schema])
    op.push(t)
    op.finish()
    got = op.collect()
    m = op.metrics()
    op.close()
    assert m.get("gpu.jit_launches", 0) >= 1
    uk, inv, cnt = np.unique(k, return_inverse=True, return_counts=True)
    sums = np.bincount(inv, weights=v.astype(np.float64)).astype(np.int64)
    order = np.argsort(got.column("k").to_numpy())
    assert got.num_rows == len(uk)
    assert np.array_equal(got.column("k").to_numpy()[order], uk)
    assert np.array_equal(got.column("s").to_numpy()[order], sums)
    assert np.array_equal(got.column("c").to_numpy()[order], cnt)
