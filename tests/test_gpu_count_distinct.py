"""DISTINCT aggregates on the GPU: count / sum / avg(DISTINCT x) behind the per-pair gate of single-mode aggregates, against the
reference of tests/distinct_ref.py -- every argument type with and without nulls, keyless and with 1-3 keys, next to plain
aggregates, behind a filter, across batches, through pair-set growth and partitioned mode, and ClickBench [09] in the
reference's plan shape, resident and from Parquet."""
import decimal
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from sail_b200 import clickbench as cb, engine, plans
from tests import distinct_ref as ref
from tests.util import assert_same, assert_topk

pytestmark = pytest.mark.gpu

LONG = "a DISTINCT argument longer than twelve bytes #"


def run(spec, batches):
    op = engine.GpuExec(spec, [batches[0].schema])
    try:
        for t in batches:
            op.push(t)
        op.finish()
        return op.collect(), op.metrics()
    finally:
        op.close()


def check(spec, table, batches=None, float_cols=()):
    """float_cols: names of the Float64 results (compared within 1e-6 relative)"""
    got, m = run(spec, batches or [table])
    assert_same(got, ref.ref_op(spec, table), float_cols=[got.schema.names.index(c) for c in float_cols if c in got.schema.names])
    return got, m


def agg(aggs, keys, pre=None):
    spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": k}, "name": f"k{k}"} for k in keys], "aggs": aggs}
    return spec if pre is None else {"op": "pipeline", "stages": [pre, spec]}


def d(fn, arg, name, distinct=True, input_type=None):
    out = {"fn": fn, "name": name, "args": [{"col": arg}]}
    if distinct:
        out["distinct"] = True
    if input_type:
        out["input_type"] = input_type
    return out


def values(kind, v):
    """argument values for integer codes v (few distinct values, so that pairs repeat)"""
    if kind in ("int16", "int32", "int64"):
        return pa.array(v - 500, type=getattr(pa, kind)())
    if kind == "uint64":
        return pa.array(v.astype(np.uint64) + np.uint64(2**53), type=pa.uint64())
    if kind == "dec15":
        return pa.array([decimal.Decimal(int(x) * 1234567 - 10**9) / 100 for x in v], type=pa.decimal128(15, 2))
    if kind == "dec38":
        return pa.array([decimal.Decimal((int(x) - 300) * 10**25 + 7) for x in v], type=pa.decimal128(38, 0))
    if kind == "date32":
        return pa.array(v.astype(np.int32) + 15000, type=pa.int32()).cast(pa.date32())
    if kind == "timestamp":
        return pa.array(v.astype(np.int64) * 1_000_003 + 1_600_000_000_000_000, type=pa.int64()).cast(pa.timestamp("us", tz="UTC"))
    if kind in ("utf8", "utf8view"):
        return pa.array([f"v{x}" if x % 3 else LONG + str(x) for x in v], type=pa.string() if kind == "utf8" else pa.string_view())
    raise AssertionError(kind)


NUMERIC = ["int16", "int32", "int64", "uint64", "dec15", "dec38"]
KINDS = NUMERIC + ["date32", "timestamp", "utf8", "utf8view"]


def table(kind, n_keys, nulls, n=24_000, seed=3, card=700):
    rng = np.random.default_rng(seed)
    cols, names = [], []
    for i in range(n_keys):
        k = rng.integers(0, [7, 3, 5][i], n)
        cols.append(pa.array(k.astype(np.int32), mask=(rng.random(n) < 0.05) if nulls else None) if i != 1 else pa.array([f"key{x}" for x in k], type=pa.string_view()))
        names.append(f"k{i}")
    x = values(kind, rng.integers(0, card, n))
    if nulls:
        x = pa.array(x.to_pylist(), type=x.type, mask=rng.random(n) < 0.2)
    return pa.table(cols + [x], names=names + ["x"])


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n_keys", [0, 1, 3])
@pytest.mark.parametrize("nulls", [False, True])
def test_argument_types(kind, n_keys, nulls):
    t = table(kind, n_keys, nulls)
    x = n_keys
    aggs = [d("count", x, "n")]
    if kind in NUMERIC:
        aggs += [d("sum", x, "s"), d("avg", x, "a")]
    # two batches, the second a slice of a larger array (offset views / bitmaps)
    big = pa.concat_tables([t, t])
    batches = [t.slice(0, 10_000), big.slice(10_000, t.num_rows - 10_000)]
    if kind == "timestamp":          # the oracle has no Timestamp type: the reference counts the instants as Int64
        t = t.set_column(n_keys, "x", t.column("x").cast(pa.int64()))
    got, m = check(agg(aggs, range(n_keys)), t, batches, float_cols=("a",))
    assert m.get("gpu.jit_launches", 0) == 0


@pytest.mark.parametrize("n_keys", [1, 2])
def test_distinct_and_plain_aggregates_over_one_column_differ(n_keys):
    t = table("int64", n_keys, True, card=50)
    spec = agg([d("count", n_keys, "cd"), d("count", n_keys, "c", distinct=False), d("sum", n_keys, "sd"), d("sum", n_keys, "s", distinct=False),
                d("avg", n_keys, "ad"), d("avg", n_keys, "a", distinct=False)], range(n_keys))
    got, _ = check(spec, t, float_cols=("ad", "a"))
    assert got.column("cd").to_pylist() != got.column("c").to_pylist() and got.column("sd").to_pylist() != got.column("s").to_pylist()


def test_two_distinct_arguments_and_a_shared_gate():
    rng = np.random.default_rng(8)
    n = 50_000
    t = pa.table({"k": pa.array(rng.integers(0, 40, n).astype(np.int32)), "u": pa.array(rng.integers(0, 900, n)),
                  "s": pa.array([f"s{i}" for i in rng.integers(0, 300, n)], type=pa.string_view())})
    spec = agg([d("count", 1, "cu"), d("sum", 1, "su"), d("avg", 1, "au"), d("count", 2, "cs"), {"fn": "count", "name": "c", "args": []}], [0])
    check(spec, t, float_cols=("au",))


@pytest.mark.parametrize("fn", ["min", "max"])
def test_min_max_with_the_flag_equal_their_results_without(fn):
    t = table("int64", 1, True)
    with_flag, _ = run(agg([d(fn, 1, "m")], [0]), [t])
    without, _ = run(agg([d(fn, 1, "m", distinct=False)], [0]), [t])
    assert_same(with_flag, without)


def test_filtered_rows_neither_count_nor_claim_pairs():
    # every pair appears first on a row the filter drops and later on a kept row: the kept row must still count
    k = np.repeat(np.arange(100, dtype=np.int32), 40)
    x = np.tile(np.repeat(np.arange(20, dtype=np.int64), 2), 100)
    keep = np.tile(np.array([0, 1], dtype=np.int32), 2000)
    t = pa.table({"k": k, "x": x, "f": keep})
    flt = {"op": "filter", "predicate": {"op": "=", "l": {"col": 2}, "r": {"lit": 1, "type": "Int32"}}}
    spec = agg([d("count", 1, "n"), d("sum", 1, "s")], [0], pre=flt)
    got, _ = run(spec, [t])
    want = ref.ref_op(agg([d("count", 1, "n"), d("sum", 1, "s")], [0]), ref.oracle_op(flt, t))
    assert_same(got, want)
    assert set(got.column("n").to_pylist()) == {20}


def test_many_batches_whose_pairs_repeat_and_long_strings_in_later_batches():
    rng = np.random.default_rng(4)
    batches = []
    for b in range(12):
        n = 9_000
        xs = [LONG + str(i) if i % 2 else f"s{i}" for i in rng.integers(0, 2_000, n)]
        # a fresh heap per batch: equal long strings of later batches point into other buffers
        batches.append(pa.table({"k": pa.array(rng.integers(0, 30, n).astype(np.int64)), "x": pa.array(xs, type=pa.string_view())}))
    spec = agg([d("count", 1, "n"), {"fn": "count", "name": "c", "args": []}], [0])
    whole = pa.concat_tables(batches)
    got, _ = run(spec, batches)
    assert_same(got, ref.ref_op(spec, whole))


def test_three_million_pairs_grow_the_pair_set_through_hand_backs():
    n = 6_000_000
    rng = np.random.default_rng(5)
    x = rng.permutation(3_000_000).repeat(2)
    t = pa.table({"k": pa.array((x % 1000).astype(np.int32)), "x": pa.array(x.astype(np.int64))})
    spec = agg([d("count", 1, "n"), d("sum", 1, "s"), {"fn": "count", "name": "c", "args": []}], [0])
    got, m = run(spec, [t.slice(i, 1_000_000) for i in range(0, n, 1_000_000)])
    want = ref.ref_op(spec, t)
    assert_same(got, want)
    assert sum(got.column("n").to_pylist()) == 3_000_000


def test_one_group_with_one_value_over_ten_million_rows():
    n = 10_000_000
    t = pa.table({"k": pa.array(np.zeros(n, np.int32)), "x": pa.array(np.full(n, 42, np.int64))})
    got, _ = run(agg([d("count", 1, "n"), d("sum", 1, "s"), {"fn": "count", "name": "c", "args": []}], [0]), [t])
    assert got.to_pylist() == [{"k0": 0, "n": 1, "s": 42, "c": n}]


def test_one_group_where_every_value_is_distinct():
    n = 2_000_000
    x = np.random.default_rng(6).permutation(n).astype(np.int64)
    t = pa.table({"x": x})
    got, _ = run(agg([d("count", 0, "n"), d("sum", 0, "s"), d("avg", 0, "a")], []), [t.slice(0, 700_000), t.slice(700_000)])
    assert got.to_pylist() == [{"n": n, "s": int(x.sum()), "a": float(x.sum()) / n}]


def test_partitioned_mode_with_pairs_under_the_ceiling(monkeypatch):
    # unique keys overflow a 2^14-slot group table; x is null on all but every 50th row, so the pairs stay far under the ceiling
    monkeypatch.setenv("SAILGPU_AGG_MAX_CAPACITY", str(1 << 14))
    rng = np.random.default_rng(9)
    n = 60_000
    x = rng.integers(0, 5, n)
    t = pa.table({"k": pa.array(np.arange(n, dtype=np.int64) // 2), "x": pa.array(x, mask=(np.arange(n) % 50) != 0)})
    spec = agg([d("count", 1, "n"), d("sum", 1, "s"), d("avg", 1, "a"), {"fn": "count", "name": "c", "args": []}], [0])
    got, m = run(spec, [t.slice(i, 1_000) for i in range(0, n, 1_000)])
    assert m.get("gpu.agg_spills", 0) > 0 or m.get("gpu.agg_partitions", 0) > 1, m
    assert_same(got, ref.ref_op(spec, t), float_cols=(3,))


def test_more_pairs_than_the_ceiling_is_refused_cleanly(monkeypatch):
    monkeypatch.setenv("SAILGPU_AGG_MAX_CAPACITY", str(1 << 14))
    n = 60_000
    t = pa.table({"k": pa.array(np.zeros(n, np.int32)), "x": pa.array(np.arange(n, dtype=np.int64))})
    with pytest.raises(engine.SailGpuError) as e:
        run(agg([d("count", 1, "n")], [0]), [t.slice(i, 1_000) for i in range(0, n, 1_000)])
    assert e.value.code == 2 and "pair slots" in str(e.value)


def test_the_specialiser_leaves_the_gated_pipeline_interpreted(monkeypatch):
    monkeypatch.setenv("SAILGPU_JIT_MIN_ROWS", "0")
    t = table("int64", 2, True, n=200_000)
    spec = agg([d("count", 2, "n"), d("sum", 2, "s"), {"fn": "count", "name": "c", "args": []}], [0, 1])
    got, m = check(spec, t)
    assert m.get("gpu.jit_launches", 0) == 0


# ---- ClickBench [09] ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hits_table():
    from datagen import hits as gen
    return gen.hits(100_000, seed=7)


@pytest.fixture(scope="module")
def frame(hits_table):
    from tests import clickbench_sql as sql
    return sql.frame(hits_table)


def check9(got, frame, hits_table, gpu):
    from tests import clickbench_sql as sql
    from tests.test_clickbench import as_table
    q = cb.DISTINCT_QUERIES["c9_single"]
    assert got.num_rows == 10
    assert_topk(got, as_table(sql.q9(frame), got.schema), list(q.order), 10, float_cols=q.floats)
    # and the whole result equals the two-level rewrite's on the GPU
    assert_same(plans.execute(cb.without_limit(q.plan()), {"hits": hits_table}, gpu), plans.execute(cb.without_limit(cb.c9()), {"hits": hits_table}, gpu), float_cols=q.floats)


def test_clickbench_9_single_resident(hits_table, frame):
    from tests.util import gpu_op
    got = plans.execute(cb.top_sort(cb.DISTINCT_QUERIES["c9_single"].plan()), {"hits": hits_table}, gpu_op)
    check9(got, frame, hits_table, gpu_op)


def test_clickbench_9_single_from_parquet(hits_table, frame):
    from datagen import hits as gen
    from tests.test_gpu_parquet_clickbench import run_gpu
    from tests.util import gpu_op
    cols = ["RegionID", "UserID", "AdvEngineID", "ResolutionWidth"]
    buf = io.BytesIO()
    pq.write_table(gen.stored(hits_table.select(cols)), buf, compression="zstd", compression_level=3, row_group_size=30_000)
    raw = buf.getvalue()
    n_groups = pq.ParquetFile(io.BytesIO(raw)).metadata.num_row_groups
    assert n_groups > 1
    parts = [engine.parquet_decode(raw, row_group=g, binary_as_string=True) for g in range(n_groups)]
    got = run_gpu(cb.over_view(cb.top_sort(cb.DISTINCT_QUERIES["c9_single"].plan())), {"hits": (parts, parts[0].schema.names)})
    check9(got, frame, hits_table, gpu_op)
