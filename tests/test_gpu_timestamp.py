"""The Timestamp type on the GPU, against the numpy reference of tests/timestamp_ref.py: date_part / date_trunc / casts in the
interpreted and the specialised kernel over every unit and the supported zones, the operators that carry timestamps without
reading wall-clock time, host and device round trips, Parquet TIMESTAMP columns, and ClickBench [18] / [42] against their SQL
restated in pandas."""
import io

import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from sail_b200 import clickbench as cb, engine, plans
from tests import timestamp_ref as ref
from tests.test_timestamp_plan import UNITS, ZONES, col, exprs_over, fn, ts_table
from tests.util import assert_same, assert_topk

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["interpreted", "specialised"])
def kernel(request, monkeypatch):
    if request.param == "interpreted":
        monkeypatch.setenv("SAILGPU_JIT", "0")
    else:
        monkeypatch.delenv("SAILGPU_JIT", raising=False)
        monkeypatch.setenv("SAILGPU_JIT_MIN_ROWS", "0")
        monkeypatch.setenv("SAILGPU_JIT_STRICT", "1")
    return request.param


def assert_columns_equal(got: pa.Table, want: pa.Table):
    """row for row, column by column (Arrow equality: values, validity and type)"""
    assert got.schema.names == want.schema.names
    for name in want.schema.names:
        g, w = got.column(name).combine_chunks(), want.column(name).combine_chunks()
        assert g.type == w.type, (name, g.type, w.type)
        assert g.equals(w), name


def as_storage(t: pa.Table) -> pa.Table:
    """timestamp columns as their int64 values: rendering zone-aware timestamps row by row costs a tz-aware datetime per cell"""
    return pa.table([c.cast(pa.int64()) if pa.types.is_timestamp(c.type) else c for c in t.columns], names=t.schema.names)


def assert_same_rows(got: pa.Table, want: pa.Table):
    """tests.util.assert_same (rows as multisets) with the types checked first and timestamps compared by value"""
    assert [(f.name, f.type) for f in got.schema] == [(f.name, f.type) for f in want.schema], (got.schema, want.schema)
    assert_same(as_storage(got), as_storage(want))


def run(spec, *tables):
    op = engine.GpuExec(spec, [t.schema for t in tables])
    try:
        for i, t in enumerate(tables):
            op.push(t, i)
            op.finish(i)
        return op.collect(), op.metrics()
    finally:
        op.close()


# ---- functions ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 1000, 300_007])           # a partial last tile; more tiles than CTAs
@pytest.mark.parametrize("unit", UNITS)
@pytest.mark.parametrize("tz", ZONES)
def test_functions_match_the_reference(kernel, unit, tz, n):
    t = ts_table(n, unit, tz, seed=n)
    spec = {"op": "projection", "exprs": [{"expr": e, "name": nm} for e, nm in exprs_over(unit, tz)]}
    got, m = run(spec, t)
    assert_columns_equal(got, ref.ref_op(spec, t))
    if kernel == "specialised":
        assert m["gpu.jit_launches"] >= 1


def test_filter_on_a_timestamp_range(kernel):
    t = ts_table(100_000, "us", "UTC", seed=4)
    lo, hi = {"lit": 0, "type": "Timestamp(us, UTC)"}, {"lit": 1_500_000_000_000_000, "type": "Timestamp(us, UTC)"}
    spec = {"op": "filter", "predicate": {"op": "and", "l": {"op": ">=", "l": col(0), "r": lo}, "r": {"op": "<", "l": col(0), "r": hi}}}
    got, _ = run(spec, t)
    assert got.num_rows > 0
    assert_columns_equal(got, ref.ref_op(spec, t))


# ---- operators --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("asc", [True, False])
@pytest.mark.parametrize("fetch", [None, 25])
def test_sort_and_topk_with_nulls(asc, fetch):
    t = ts_table(30_000, "ns", "+05:30", seed=6)
    spec = {"op": "sort", "keys": [{"expr": col(0), "asc": asc, "nulls_first": asc}, {"expr": col(1), "asc": True, "nulls_first": True}], "fetch": fetch}
    got, _ = run(spec, t)
    assert_columns_equal(got, ref.ref_op(spec, t))


@pytest.mark.parametrize("mode", ["single", "two_phase"])
def test_aggregate_grouped_by_date_trunc_with_min_max_count(kernel, mode):
    t = ts_table(120_000, "us", "-08:00", seed=8)
    days = pa.array(np.random.default_rng(8).integers(15_000, 18_650, 120_000) * 86_400_000_000 + 12_345_678)    # ten years: ~3.6 k groups
    t = t.set_column(0, "t", pa.array(days.to_numpy(), type=pa.int64(), mask=t.column("t").is_null().to_numpy(zero_copy_only=False)).cast(pa.timestamp("us", tz="-08:00")))
    gb = [{"expr": fn("date_trunc", "day", col(0)), "name": "d"}]
    ty = "Timestamp(us, -08:00)"
    aggs = [{"fn": "min", "args": [col(0)], "name": "mn", "input_type": ty}, {"fn": "max", "args": [col(0)], "name": "mx", "input_type": ty},
            {"fn": "count", "args": [col(0)], "name": "c", "input_type": ty}]
    if mode == "single":
        spec = {"op": "aggregate", "mode": "single", "group_by": gb, "aggs": aggs}
        assert_same_rows(run(spec, t)[0], ref.ref_op(spec, t))
        return
    partial = {"op": "aggregate", "mode": "partial", "group_by": gb, "aggs": aggs}
    final = {"op": "aggregate", "mode": "final_partitioned", "group_by": [{"expr": col(0), "name": "d"}],
             "aggs": [{k: v for k, v in a.items() if k != "args"} for a in aggs]}
    halves = [run(partial, t.slice(0, 60_000))[0], run(partial, t.slice(60_000))[0]]
    want = ref.ref_op(final, pa.concat_tables([ref.ref_op(partial, t.slice(0, 60_000)), ref.ref_op(partial, t.slice(60_000))]))
    assert_same_rows(run(final, pa.concat_tables(halves))[0], want)


def test_hash_join_on_a_timestamp_key():
    rng = np.random.default_rng(12)
    keys = rng.choice(np.arange(0, 10_000, dtype=np.int64) * 60_000_000, 5000, replace=False)
    build = pa.table({"k": pa.array(keys).cast(pa.timestamp("us", tz="UTC")), "b": pa.array(np.arange(5000))})
    probe = pa.table({"k": pa.array(rng.choice(keys, 40_000)).cast(pa.timestamp("us", tz="UTC")), "p": pa.array(np.arange(40_000))})
    spec = {"op": "hash_join", "join_type": "inner", "mode": "collect_left", "on": [[0, 0]], "filter": None, "projection": None}
    got, _ = run(spec, build, probe)
    assert got.num_rows == 40_000
    assert_same_rows(got, ref.ref_op(spec, build, probe))


def test_hash_repartition_keeps_every_row_and_the_type():
    t = ts_table(50_000, "ms", "UTC", seed=13)
    spec = {"op": "repartition", "exprs": [col(0)], "n": 4}
    op = engine.GpuExec(spec, [t.schema])
    op.push(t)
    op.finish()
    parts = []
    for p in range(4):
        d, _ = op.pull_device(partition=p)
        from tests.test_gpu_parquet_clickbench import host
        parts.append(host([d], op.schema))
    op.close()
    want = ref.ref_op(spec, t)
    for g, w in zip(parts, want):
        assert g.schema.field("t").type == pa.timestamp("ms", tz="UTC")
        assert_same_rows(g, w)


# ---- round trips -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("unit", UNITS)
@pytest.mark.parametrize("tz", ZONES)
def test_push_pull_and_device_round_trips_keep_the_type(unit, tz):
    from tests.test_gpu_parquet_clickbench import host
    t = ts_table(10_001, unit, tz, seed=21)
    spec = {"op": "projection", "exprs": [{"expr": col(0), "name": "t"}]}
    got, _ = run(spec, t)
    assert got.column("t").combine_chunks().equals(t.column("t").combine_chunks())
    op = engine.GpuExec(spec, [t.schema])
    op.push(t)
    op.finish()
    dev = op.collect_device()
    op.close()
    back = host(dev, op.schema)
    assert back.schema.field("t").type == pa.timestamp(unit, tz=tz)
    assert back.column("t").combine_chunks().equals(t.column("t").combine_chunks())


# ---- Parquet -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("unit", ["ms", "us", "ns"])
@pytest.mark.parametrize("tz", [None, "UTC"])
@pytest.mark.parametrize("codec,level", [("none", None), ("zstd", 1), ("zstd", 19)])
def test_parquet_timestamps_decode_like_pyarrow(unit, tz, codec, level):
    from tests.test_gpu_parquet_clickbench import host
    from tests.test_timestamp_plan import ts_parquet
    _, raw = ts_parquet(unit, tz, codec, level, n=70_001)
    want = pq.read_table(io.BytesIO(raw)).column("t").combine_chunks()
    got = host([engine.parquet_decode(raw)]).column("t").combine_chunks()
    assert got.type == want.type and got.equals(want)


# ---- ClickBench [18] and [42] --------------------------------------------------------------------------------------------------
N_HITS = 1_000_000       # below ~1 M rows [42] has fewer than 1,010 minute groups and its OFFSET leaves nothing to compare


def sql18(h):
    """SELECT UserID, extract(minute FROM CAST(EventTime AS TIMESTAMP)) AS m, SearchPhrase, COUNT(*) .. GROUP BY UserID, m, SearchPhrase
    ORDER BY COUNT(*) DESC"""
    df = pd.DataFrame({"UserID": h.UserID, "m": ((h.EventTime // 60) % 60).astype(np.int32), "SearchPhrase": h.SearchPhrase})
    out = df.groupby(["UserID", "m", "SearchPhrase"], sort=False).size().reset_index(name="count(*)")
    return out.sort_values("count(*)", ascending=False, kind="stable").reset_index(drop=True)


def sql42(h):
    """SELECT DATE_TRUNC('minute', CAST(EventTime AS TIMESTAMP)) AS M, COUNT(*) AS PageViews .. WHERE CounterID = 62 AND EventDate
    BETWEEN '2013-07-14' AND '2013-07-15' AND IsRefresh = 0 AND DontCountHits = 0 GROUP BY M ORDER BY M"""
    import datetime
    f = h[(h.CounterID == 62) & (h.EventDate >= datetime.date(2013, 7, 14)) & (h.EventDate <= datetime.date(2013, 7, 15)) & (h.IsRefresh == 0) & (h.DontCountHits == 0)]
    m = pd.to_datetime(f.EventTime // 60 * 60, unit="s", utc=True).astype("datetime64[us, UTC]")
    out = pd.DataFrame({"M": m}).groupby("M", sort=True).size().reset_index(name="PageViews")
    return out.reset_index(drop=True)


@pytest.fixture(scope="module")
def hits_table():
    from datagen import hits as gen
    return gen.hits(N_HITS, seed=7)


def check_timestamp_query(name, got, frame):
    from tests.test_clickbench import as_table
    q = cb.TIMESTAMP_QUERIES[name]
    full = as_table({"c18": sql18, "c42": sql42}[name](frame), got.schema)
    fetch = cb.top_sort(q.plan()).spec["fetch"]
    assert_topk(got, full, list(q.order), fetch)
    assert got.slice(q.skip).num_rows > 0, "the OFFSET leaves rows to compare"


@pytest.fixture(scope="module")
def frame(hits_table):
    from tests import clickbench_sql as sql
    return sql.frame(hits_table)


@pytest.mark.parametrize("name", list(cb.TIMESTAMP_QUERIES))
def test_clickbench_timestamp_query_resident(name, hits_table, frame):
    q = cb.TIMESTAMP_QUERIES[name]
    node = cb.top_sort(q.plan())
    got = plans.execute(node, {"hits": hits_table}, lambda spec, *ts: run(spec, *ts)[0])
    check_timestamp_query(name, got, frame)


@pytest.mark.parametrize("name", list(cb.TIMESTAMP_QUERIES))
def test_clickbench_timestamp_query_from_parquet(name, hits_table, frame):
    from datagen import hits as gen
    from tests.test_gpu_parquet_clickbench import run_gpu
    buf = io.BytesIO()
    pq.write_table(gen.stored(hits_table), buf, compression="zstd", compression_level=3, row_group_size=300_000)
    raw = buf.getvalue()
    n_groups = pq.ParquetFile(io.BytesIO(raw)).metadata.num_row_groups
    parts = [engine.parquet_decode(raw, row_group=g, binary_as_string=True) for g in range(n_groups)]
    got = run_gpu(cb.over_view(cb.top_sort(cb.TIMESTAMP_QUERIES[name].plan())), {"hits": (parts, parts[0].schema.names)})
    check_timestamp_query(name, got, frame)
