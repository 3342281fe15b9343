"""Partitioned mode of the hash aggregate (engine.cu, PipelineOp): a group table that would need more slots than its ceiling
empties itself as partial-aggregate state rows and starts over.  A partial aggregate emits those rows at once; the other modes
scatter them into key-hash partitions and merge every partition with a final aggregate of its own.  SAILGPU_AGG_MAX_CAPACITY
lowers the ceiling (2^28 slots) so that these tests reach partitioned mode with 10^4 - 10^6 groups; results are compared with
the numpy oracle as sets of rows, Float64 within 1e-6 relative."""
import decimal

import numpy as np
import pyarrow as pa
import pytest

from sail_b200 import plans
from tests.util import assert_same, oracle_op

pytestmark = pytest.mark.gpu


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


@pytest.fixture
def ceiling(monkeypatch):
    def set_(slots):
        monkeypatch.setenv("SAILGPU_AGG_MAX_CAPACITY", str(slots))
    return set_


# ---- data -------------------------------------------------------------------------------------------
LONG = "a group key much longer than twelve bytes #"


def key_column(kind, ids, rng):
    """the group key(s) for group numbers `ids`: {name: array}"""
    if kind == "int64":
        return {"k": pa.array(ids * 7919 - 10**12)}
    if kind == "int32":
        return {"k": pa.array((ids - 50_000).astype(np.int32))}
    if kind == "int16":          # 65536 values at most: ids are folded, the sums still differ per group
        return {"k": pa.array((ids % 60_000 - 30_000).astype(np.int16))}
    if kind == "date32":
        return {"k": pa.array((ids + 1000).astype(np.int32), type=pa.int32()).cast(pa.date32())}
    if kind == "decimal":
        return {"k": pa.array([decimal.Decimal(int(i) * 10**15 + 7) / 100 for i in ids], type=pa.decimal128(25, 2))}
    if kind == "utf8view_inline":
        return {"k": pa.array([f"k{i}" for i in ids], type=pa.string_view())}
    if kind == "utf8view_long":
        return {"k": pa.array([LONG + str(i) for i in ids], type=pa.string_view())}
    if kind == "multi":
        return {"k": pa.array((ids % 1000).astype(np.int32)), "k2": pa.array([f"s{i // 1000}" for i in ids], type=pa.string_view())}
    if kind == "nullable":
        return {"k": pa.array(ids.astype(np.int64), mask=(ids % 97) == 0)}     # the null group collects every 97th group
    raise AssertionError(kind)


def make_batches(kind, sizes, seed=1):
    """batches of the given row counts; batch i draws its groups mostly from a fresh range, so distinct groups keep growing"""
    rng = np.random.default_rng(seed)
    out, base = [], 0
    for n in sizes:
        ids = base + rng.integers(0, int(n * 1.1), n)          # ~0.6 n distinct groups per batch, repeats inside the batch
        ids[: n // 20] = rng.integers(0, max(1, base), n // 20) if base else ids[: n // 20]     # and some groups seen before
        base += int(n * 1.1)
        cols = key_column(kind, ids, rng)
        v = rng.integers(-10**6, 10**6, n).astype(np.int64)
        cols["v"] = pa.array(v, mask=rng.random(n) < 0.05)
        cols["d"] = pa.array([decimal.Decimal(int(x)) / 100 for x in rng.integers(-10**9, 10**9, n)], type=pa.decimal128(15, 2))
        cols["f"] = pa.array(rng.standard_normal(n) * 100)
        out.append(pa.table(cols))
    schema = out[0].schema
    return [t.cast(schema) for t in out]


def agg_spec(mode, keys, schema):
    idx = {n: i for i, n in enumerate(schema.names)}
    aggs = [("sum", "v", "sv", "Int64"), ("count", None, "c", None), ("count", "v", "cv", "Int64"), ("min", "v", "mnv", "Int64"),
            ("max", "d", "mxd", "Decimal128(15,2)"), ("avg", "v", "av", "Int64"), ("sum", "d", "sd", "Decimal128(15,2)"),
            ("avg", "d", "ad", "Decimal128(15,2)"), ("sum", "f", "sf", "Float64"), ("min", "f", "mnf", "Float64"), ("avg", "f", "af", "Float64")]
    gb = [{"expr": {"col": idx[k]}, "name": k} for k in keys]
    if mode in ("final", "final_partitioned"):
        return {"op": "aggregate", "mode": mode, "group_by": [{"expr": {"col": i}, "name": k} for i, k in enumerate(keys)],
                "aggs": [{"fn": f, "name": nm, "input_type": t} for f, _, nm, t in aggs]}
    return {"op": "aggregate", "mode": mode, "group_by": gb,
            "aggs": [{"fn": f, "name": nm, "input_type": t, "args": [] if a is None else [{"col": idx[a]}]} for f, a, nm, t in aggs]}


FLOATS_OUT = {"af", "sf", "mnf"}


def float_cols(t):
    return {i for i, n in enumerate(t.schema.names) if n in FLOATS_OUT}


def keys_of(batches):
    return [n for n in batches[0].schema.names if n in ("k", "k2")]


def check_single(batches, got):
    keys = keys_of(batches)
    want = oracle_op(agg_spec("single", keys, batches[0].schema), pa.concat_tables(batches))
    assert_same(got, want, float_cols=float_cols(want))


# overflow in the first batch, in the middle of the stream, in the last one: a batch of 50 K rows into a table of 2^17 slots
# (half of which may fill, less what one launch's tiles can add) hands tiles back; batches of 20 K rows do not, until the
# table holds enough groups.  Every batch is queued before the hand-back of the one before it is looked at.
LAYOUTS = {"first": [50_000, 20_000, 20_000], "mid": [20_000, 20_000, 50_000, 20_000], "last": [20_000, 20_000, 50_000]}
KINDS = ["int64", "int32", "int16", "date32", "decimal", "utf8view_inline", "utf8view_long", "multi", "nullable"]


@pytest.mark.parametrize("kind", KINDS)
def test_single_mode_key_types(kind, ceiling):
    ceiling(1 << 17)
    batches = make_batches(kind, LAYOUTS["mid"])
    got, m = run_batches(agg_spec("single", keys_of(batches), batches[0].schema), batches)
    check_single(batches, got)
    assert m["gpu.agg_spills"] >= 1 and m["gpu.agg_partitions"] >= 2, m
    assert sum(m["gpu.agg_partition_groups"]) == got.num_rows == m["output_rows"]
    assert len(m["gpu.agg_partition_groups"]) == m["gpu.agg_partitions"] and m["output_batches"] <= m["gpu.agg_partitions"]


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("jit", ["interpreted", "specialised"])
def test_overflow_position(layout, jit, ceiling, monkeypatch):
    if jit == "interpreted":
        monkeypatch.setenv("SAILGPU_JIT", "0")
    else:
        monkeypatch.setenv("SAILGPU_JIT", "1")
        monkeypatch.setenv("SAILGPU_JIT_MIN_ROWS", "0")
    ceiling(1 << 17)
    batches = make_batches("int64", LAYOUTS[layout], seed=3)
    got, m = run_batches(agg_spec("single", ["k"], batches[0].schema), batches)
    check_single(batches, got)
    assert m["gpu.agg_spills"] >= 1, m


@pytest.mark.parametrize("kind", ["int64", "utf8view_long", "multi", "nullable", "decimal"])
def test_partial_emits_early_and_final_merges_repeats(kind, ceiling):
    """partial -> final_partitioned, both in partitioned mode: the partial aggregate emits a group once per time its table was
    emptied, the final merges the repeats"""
    ceiling(1 << 17)
    batches = make_batches(kind, LAYOUTS["mid"], seed=5)
    keys = keys_of(batches)
    partial, pm = run_batches(agg_spec("partial", keys, batches[0].schema), batches)
    assert pm["gpu.agg_spills"] >= 1 and pm["output_batches"] >= 2, pm
    distinct = oracle_op(agg_spec("single", keys, batches[0].schema), pa.concat_tables(batches)).num_rows
    assert partial.num_rows > distinct          # some group was emitted more than once
    want_partial = oracle_op(agg_spec("partial", keys, batches[0].schema), pa.concat_tables(batches))
    assert partial.schema.names == want_partial.schema.names
    final_spec = agg_spec("final_partitioned", keys, batches[0].schema)
    parts = [partial.slice(i, 30_000) for i in range(0, partial.num_rows, 30_000)]
    got, fm = run_batches(final_spec, parts)
    check_single(batches, got)
    assert fm["gpu.agg_spills"] >= 1, fm


@pytest.mark.parametrize("mode", ["final", "final_partitioned"])
@pytest.mark.parametrize("kind", ["int64", "utf8view_inline", "nullable"])
def test_final_modes(mode, kind, ceiling):
    """state rows from the oracle's partial aggregate of each batch, merged on the GPU by a final aggregate past its ceiling"""
    ceiling(1 << 17)
    batches = make_batches(kind, [30_000] * 5, seed=9)
    keys = keys_of(batches)
    pspec = agg_spec("partial", keys, batches[0].schema)
    states = [oracle_op(pspec, t) for t in batches]
    got, m = run_batches(agg_spec(mode, keys, batches[0].schema), states)
    check_single(batches, got)
    assert m["gpu.agg_spills"] >= 1 and m["gpu.agg_partitions"] >= 2, m


def test_jit_above_specialiser_threshold(ceiling, monkeypatch):
    """two batches of 5 Mi rows (above SAILGPU_JIT_MIN_ROWS' default of 4 Mi) through the specialised kernel, 2^24 slots at most"""
    monkeypatch.setenv("SAILGPU_JIT", "1")
    monkeypatch.delenv("SAILGPU_JIT_MIN_ROWS", raising=False)
    ceiling(1 << 24)
    n = 5 << 20
    batches, vals = [], []
    for b in range(2):
        i = np.arange(b * n, (b + 1) * n, dtype=np.int64)
        k = (i * 2654435761) % (1 << 40)               # distinct keys, in no order
        v = (i % 1000) - 500
        vals.append(v)
        batches.append(pa.table({"k": pa.array(k), "v": pa.array(v)}))
    spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": 0}, "name": "k"}],
            "aggs": [{"fn": "sum", "args": [{"col": 1}], "name": "s"}, {"fn": "count", "args": [], "name": "c"}]}
    got, m = run_batches(spec, batches)
    assert m["gpu.agg_spills"] >= 1 and m["gpu.jit_launches"] >= 2, m
    assert got.num_rows == 2 * n
    k = np.concatenate([t.column("k").to_numpy() for t in batches])
    v = np.concatenate(vals)
    order, gorder = np.argsort(k), np.argsort(got.column("k").to_numpy())
    assert np.array_equal(got.column("k").to_numpy()[gorder], k[order])
    assert np.array_equal(got.column("s").to_numpy()[gorder], v[order])
    assert (got.column("c").to_numpy() == 1).all()


# ---- whole queries ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tpch_small():
    from datagen import tpch
    return tpch.tables(0.01)


@pytest.mark.parametrize("q", ["q18", "q10"])
def test_tpch(q, tpch_small, ceiling):
    """every aggregate of the plan under a ceiling of 2^17 slots: GROUP BY l_orderkey (15 K groups over 60 K rows) of Q18 goes
    into partitioned mode; Q10's seven-column key takes the sort-based path, whose aggregate runs on a dense group number"""
    from oracle import render
    from sail_b200 import engine
    ceiling(1 << 17)
    plan = plans.q18() if q == "q18" else plans.q10()
    want = plans.execute(plan, tpch_small, oracle_op)
    got = plans.execute(plan, tpch_small, engine.run_op)
    assert got.schema.names == want.schema.names
    assert sorted(render.rows(got)) == sorted(render.rows(want))


@pytest.mark.parametrize("name", ["c15", "c16", "c31", "c32"])
def test_clickbench(name, ceiling):
    """ClickBench [15], [16], [31], [32] over 100 K rows with a ceiling of 2^18 slots; [32] has one group per row"""
    from datagen import hits as gen
    from tests import clickbench_sql as sql
    from tests.test_clickbench import check
    from tests.util import gpu_op
    ceiling(1 << 18)
    hits = gen.hits(100_000, seed=7)
    check(name, sql.frame(hits), {"hits": hits}, gpu_op)


# ---- the real ceiling ---------------------------------------------------------------------------------
def test_160m_groups_without_the_knob(monkeypatch):
    """about 160 M distinct Int64 keys through one single-mode aggregate at the real ceiling of 2^28 slots: group count, every
    count 1, sum of sums equal to the input's sum"""
    from sail_b200 import engine
    monkeypatch.delenv("SAILGPU_AGG_MAX_CAPACITY", raising=False)
    n_batches, per = 8, 20_000_000
    spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": 0}, "name": "k"}],
            "aggs": [{"fn": "sum", "args": [{"col": 1}], "name": "s"}, {"fn": "count", "args": [], "name": "c"}]}
    schema = pa.schema([("k", pa.int64()), ("v", pa.int64())])
    op = engine.GpuExec(spec, [schema])
    total = 0
    try:
        for b in range(n_batches):
            i = np.arange(b * per, (b + 1) * per, dtype=np.int64)
            k = i * np.int64(-7046029254386353131)          # odd multiplier: a bijection of Int64, keys in no order
            v = (i % 2001) - 1000
            total += int(v.sum())
            op.push(pa.table({"k": pa.array(k), "v": pa.array(v)}, schema=schema))
        op.finish()
        groups, ones, sum_s = 0, True, 0
        while True:
            d, more = op.pull()
            if d.num_rows:
                groups += d.num_rows
                ones &= bool((d.column(2).to_numpy() == 1).all())
                sum_s += int(d.column(1).to_numpy().sum())
            if not more:
                break
        m = op.metrics()
    finally:
        op.close()
    assert groups == n_batches * per
    assert ones
    assert sum_s == total
    assert m["gpu.agg_spills"] >= 1 and m["gpu.agg_partitions"] >= 2, m
    assert sum(m["gpu.agg_partition_groups"]) == groups
