"""The aggregate's launches are pipelined one deep (engine.cu, PipelineOp): batch k is queued before the host looks at what
batch k-1 handed back.  These cases cover the paths that depend on that order -- hand-backs discovered a batch late, a
validity signature that widens while a launch is in flight, a device error in the middle of a stream -- plus the tail of a
Q1 step that no longer waits for the device: the small sort and the host export of string views.  Each runs on the
interpreted and on the specialised kernel."""
import decimal

import numpy as np
import pyarrow as pa
import pytest

from sail_b200 import plans
from tests.util import assert_same, oracle_op

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=["interpreted", "specialised"])
def kernel(request, monkeypatch):
    if request.param == "interpreted":
        monkeypatch.setenv("SAILGPU_JIT", "0")
    else:
        monkeypatch.setenv("SAILGPU_JIT", "1")
        monkeypatch.setenv("SAILGPU_JIT_MIN_ROWS", "0")
        monkeypatch.setenv("SAILGPU_JIT_STRICT", "1")
    return request.param


def run_batches(spec, batches):
    """pushes every batch into one operator; returns (result, metrics)"""
    from sail_b200 import engine
    op = engine.GpuExec(spec, [batches[0].schema])
    try:
        for t in batches:
            op.push(t)
        op.finish()
        got = op.collect()
        m = op.metrics()
    finally:
        op.close()
    return got, m


def test_q1_chain_five_batches():
    """the whole Q1 plan as one chain over five resident batches, against the oracle; the step waits for the device at most
    five times (the two aggregates' group counts, the final aggregate's null counts, the export)"""
    import bench
    from datagen import tpch
    from oracle import render
    from sail_b200 import engine
    table = tpch.lineitem(0.05)
    want = plans.execute(plans.q1(), {"lineitem": table}, oracle_op)
    q1 = table.select(bench.Q1_COLS)
    n = q1.num_rows
    cuts = [0, n // 5, 2 * n // 5, 3 * n // 5, 4 * n // 5, n]
    ctx = engine.default_context()
    devs = [engine.to_device(q1.slice(a, b - a).combine_chunks(), ctx) for a, b in zip(cuts, cuts[1:])]
    fused, final, sort = bench.q1_specs()
    for _ in range(2):      # the second execution re-creates the same plan: nothing is compiled again
        op = engine.GpuExec({"op": "chain", "ops": [fused, final, sort]}, [q1.schema], ctx)
        for d in devs:
            op.push(d.borrow())
        op.finish()
        got = op.collect()
        m = op.metrics()
        op.close()
        assert got.schema.names == want.schema.names
        assert render.rows(got) == render.rows(want)
        assert m["input_batches"] == 5
        assert m["gpu.host_syncs"] <= 5, m


@pytest.mark.parametrize("first_limit", [None, "0", "1000"])
def test_hand_back_found_after_next_launch(first_limit, monkeypatch):
    """a first table of 512 Ki slots (half of it may fill, and one launch's rows fit in the other half) and key domains
    that keep widening, with or without a forced early hand-back: batch k's deferred tiles are only looked at after batch
    k+1 was launched on the too-small table, so both are resolved together (grow, rehash, re-launch, many-groups variant)"""
    if first_limit is not None:
        monkeypatch.setenv("SAILGPU_AGG_FIRST_LIMIT", first_limit)
    monkeypatch.setenv("SAILGPU_AGG_MIN_CAPACITY", str(1 << 19))
    rng = np.random.default_rng(7)
    batches, ks, vs = [], [], []
    for b in range(5):
        n = 200_000 + 1234 * b
        k = rng.integers(0, 150_000 * (b + 1), n).astype(np.int64)
        v = rng.integers(-1000, 1000, n).astype(np.int64)
        ks.append(k)
        vs.append(v)
        batches.append(pa.table({"k": pa.array(k), "v": pa.array(v)}))
    spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": 0}, "name": "k"}],
            "aggs": [{"fn": "sum", "args": [{"col": 1}], "name": "s"}, {"fn": "count", "args": [], "name": "c"}]}
    got, _ = run_batches(spec, batches)
    k, v = np.concatenate(ks), np.concatenate(vs)
    uk, inv, cnt = np.unique(k, return_inverse=True, return_counts=True)
    sums = np.bincount(inv, weights=v.astype(np.float64)).astype(np.int64)
    assert got.num_rows == len(uk)
    order = np.argsort(got.column("k").to_numpy())
    assert np.array_equal(got.column("k").to_numpy()[order], uk)
    assert np.array_equal(got.column("s").to_numpy()[order], sums)
    assert np.array_equal(got.column("c").to_numpy()[order], cnt)


@pytest.mark.parametrize("first_limit", [None, "50"])
def test_validity_widens_while_a_launch_is_in_flight(first_limit, monkeypatch):
    """batches 1 and 2 carry no validity buffers, batch 3 does: the table is migrated to the wider layout while batch 2's
    launch is still unresolved"""
    if first_limit:
        monkeypatch.setenv("SAILGPU_AGG_FIRST_LIMIT", first_limit)
    rng = np.random.default_rng(11)
    batches = []
    for b in range(4):
        n = 40_000 + 17 * b
        mask = (rng.random(n) < 0.2) if b == 2 else None
        d = [decimal.Decimal(int(x)) / 100 for x in rng.integers(-10**7, 10**7, n)]
        batches.append(pa.table({"k": pa.array(rng.integers(0, 3000, n).astype(np.int32)),
                                 "v": pa.array(rng.integers(-100, 100, n).astype(np.int64), mask=mask),
                                 "d": pa.array(d, type=pa.decimal128(15, 2))}))
    schema = pa.schema([pa.field("k", pa.int32()), pa.field("v", pa.int64(), nullable=True), pa.field("d", pa.decimal128(15, 2))])
    batches = [t.cast(schema) for t in batches]
    spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": 0}, "name": "k"}],
            "aggs": [{"fn": "sum", "args": [{"col": 1}], "name": "sv"}, {"fn": "count", "args": [{"col": 1}], "name": "cv"},
                     {"fn": "avg", "args": [{"col": 1}], "name": "av"}, {"fn": "sum", "args": [{"col": 2}], "name": "sd"}]}
    got, _ = run_batches(spec, batches)
    assert_same(got, oracle_op(spec, pa.concat_tables(batches)), float_cols={3})


@pytest.mark.parametrize("grouped", [True, False])
def test_device_error_in_second_batch_raises_and_closes(grouped):
    """a division by zero in batch 2 of 4 surfaces as SailGpuError by finish / collect, and the operator still closes"""
    from sail_b200 import engine
    batches = []
    for b in range(4):
        n = 50_000
        div = np.full(n, 3, dtype=np.int64)
        if b == 1:
            div[n // 2] = 0
        batches.append(pa.table({"k": pa.array(np.arange(n, dtype=np.int64) % 97), "a": pa.array(np.arange(n, dtype=np.int64)), "b": pa.array(div)}))
    spec = {"op": "pipeline", "stages": [
        {"op": "projection", "exprs": [{"expr": {"col": 0}, "name": "k"}, {"expr": plans.binop("/", {"col": 1}, {"col": 2}), "name": "q"}]},
        {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": 0}, "name": "k"}] if grouped else [],
         "aggs": [{"fn": "sum", "args": [{"col": 1}], "name": "s"}]}]}
    op = engine.GpuExec(spec, [batches[0].schema])
    with pytest.raises(engine.SailGpuError) as e:
        for t in batches:
            op.push(t)
        op.finish()
        op.collect()
    assert "ivide by zero" in str(e.value)
    op.close()
    # the context stays usable
    ok, _ = run_batches(spec, batches[:1])
    assert ok.num_rows == (97 if grouped else 1)


@pytest.mark.parametrize("n", [1, 7, 300, 1024])
def test_small_sort_long_strings_and_nulls(n):
    """the small-input sort ranks rows straight from the key columns: strings longer than 12 bytes (and longer than the
    256-byte bound of the encoded sort), shared prefixes, nulls first and last, a descending second key"""
    rng = np.random.default_rng(n)
    words = ["", "a", "ab", "ab\x00", "abc", "inline-12chr", "inline-12chrX", "a much longer string value that lives in a heap",
             "a much longer string value that lives in a heap, too", "z" * 300, "z" * 300 + "a"]
    s = [words[i] for i in rng.integers(0, len(words), n)]
    t = pa.table({"s": pa.array(s, type=pa.string_view(), mask=rng.random(n) < 0.2),
                  "i": pa.array(rng.integers(-5, 5, n).astype(np.int64), mask=rng.random(n) < 0.1),
                  "p": pa.array(np.arange(n, dtype=np.int64))})
    for nulls_first in (True, False):
        spec = {"op": "sort", "keys": [{"expr": {"col": 0}, "asc": True, "nulls_first": nulls_first},
                                       {"expr": {"col": 1}, "asc": False, "nulls_first": not nulls_first}]}
        got, _ = run_batches(spec, [t])
        assert_same(got, oracle_op(spec, t), ordered=True)


@pytest.mark.parametrize("long_strings", [False, True])
def test_host_export_of_string_views(long_strings):
    """Utf8View columns come back to the host intact, inline-only or not (the export first assumes every column is inline
    and exports a column with longer strings a second time)"""
    rng = np.random.default_rng(3)
    n = 5000
    short = ["", "x", "flag", "twelve bytes"]
    longer = short + ["thirteen bytes", "a string that does not fit into the view"]
    a = [short[i] for i in rng.integers(0, len(short), n)]
    b = [(longer if long_strings else short)[i] for i in rng.integers(0, len(longer if long_strings else short), n)]
    t = pa.table({"a": pa.array(a, type=pa.string_view(), mask=rng.random(n) < 0.1), "b": pa.array(b, type=pa.string_view()),
                  "c": pa.array(np.arange(n, dtype=np.int64))})
    spec = {"op": "projection", "exprs": [{"expr": {"col": i}, "name": nm} for i, nm in enumerate(t.schema.names)]}
    got, _ = run_batches(spec, [t])
    assert got.schema == t.schema
    assert got.column("a").to_pylist() == t.column("a").to_pylist()
    assert got.column("b").to_pylist() == t.column("b").to_pylist()
    assert got.column("c").to_pylist() == t.column("c").to_pylist()
