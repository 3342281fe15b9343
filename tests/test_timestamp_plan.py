"""CPU tests of the Timestamp type: Arrow formats and spec strings, plan-time typing of the new expressions against the numpy
reference (tests/timestamp_ref.py), the refusals, the reference's wall-clock arithmetic against Python's `datetime` and
`pyarrow.compute`, the ClickBench plans [18] and [42], the specialised kernels' resources, and the Parquet walk over TIMESTAMP
columns."""
import datetime as dt
import io
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from sail_b200 import clickbench as cb, engine, plans
from tests import timestamp_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ZONES = [None, "UTC", "+05:30", "-08:00"]
UNITS = ["s", "ms", "us", "ns"]

# hand-picked instants (UTC): before 1970, leap days, century years, the last microsecond of a year, ISO week boundaries
INSTANTS = [dt.datetime(1969, 12, 31, 23, 59, 59, 999999), dt.datetime(1960, 2, 29, 12, 0, 1, 5), dt.datetime(1900, 3, 1, 0, 0),
            dt.datetime(1899, 12, 31, 23, 59, 59), dt.datetime(2000, 2, 29, 23, 30, 0, 250000), dt.datetime(2100, 2, 28, 18, 31, 7),
            dt.datetime(2012, 12, 31, 23, 59, 59, 999999), dt.datetime(2013, 7, 14, 0, 0), dt.datetime(2013, 7, 15, 23, 59, 59, 1),
            dt.datetime(2021, 1, 3, 23, 59, 59), dt.datetime(2021, 1, 4, 0, 0), dt.datetime(1970, 1, 1), dt.datetime(1970, 1, 5, 3, 4, 5)]


def micros(d: dt.datetime) -> int:
    return (d - dt.datetime(1970, 1, 1)) // dt.timedelta(microseconds=1)


def zone(tz):
    if tz in (None, "UTC"):
        return dt.timezone.utc
    return dt.timezone(dt.timedelta(seconds=ref.zone_seconds(tz)))


def col(i):
    return {"col": i}


def fn(name, part, arg):
    return {"fn": name, "part": part, "args": [arg]}


def ts_table(n, unit, tz, seed=1, nulls=True):
    rng = np.random.default_rng(seed)
    ups = ref.UNITS[unit]
    v = rng.integers(-2_000_000_000, 4_200_000_000, n).astype(np.int64) * ups + rng.integers(0, ups, n)
    mask = rng.random(n) < 0.1 if nulls else None
    return pa.table({"t": pa.array(v, type=pa.int64(), mask=mask).cast(pa.timestamp(unit, tz=tz)), "i": pa.array(rng.integers(0, 100, n))})


# ---- types --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("unit", UNITS)
@pytest.mark.parametrize("tz", [None, "UTC", "+05:30", "Europe/Paris"])
def test_formats_round_trip(unit, tz):
    t = pa.timestamp(unit, tz=tz)
    spec = {"op": "projection", "exprs": [{"expr": col(0), "name": "t"},
                                          {"expr": {"cast": {"cast": col(0), "to": "Int64"}, "to": ref.ts_type(unit, tz or "")}, "name": "r"}]}
    out = engine.validate(spec, [pa.schema([("t", t)])])
    assert out.field("t").type == t and out.field("r").type == t


def exprs_over(unit, tz):
    t = ref.ts_type(unit, tz or "")
    finer = ref.UNIT_ORDER[min(3, ref.UNIT_ORDER.index(unit) + 1)]
    out = [(fn("date_part", p, col(0)), f"p_{p}") for p in ref.PARTS]
    out += [(fn("date_trunc", p, col(0)), f"t_{p}") for p in ref.TRUNC_PARTS]
    out += [({"cast": col(0), "to": "Date32"}, "d"), ({"cast": col(0), "to": "Int64"}, "i64"),
            ({"cast": col(0), "to": ref.ts_type(finer, tz or "")}, "finer"),
            ({"op": ">=", "l": col(0), "r": {"lit": 0, "type": t}}, "ge"),
            ({"in": col(0), "set": [{"lit": 0, "type": t}, {"lit": 86400 * ref.UNITS[unit], "type": t}]}, "inl")]
    return out


@pytest.mark.parametrize("unit", UNITS)
@pytest.mark.parametrize("tz", ZONES)
def test_validate_gives_the_reference_types(unit, tz):
    t = ts_table(50, unit, tz)
    spec = {"op": "projection", "exprs": [{"expr": e, "name": n} for e, n in exprs_over(unit, tz)]}
    got, want = engine.validate(spec, [t.schema]), ref.ref_op(spec, t).schema
    assert [(f.name, f.type) for f in got] == [(f.name, f.type) for f in want]


def refused(spec, schema):
    with pytest.raises(engine.SailGpuError) as e:
        engine.validate(spec, [schema])
    return e.value.code


@pytest.mark.parametrize("expr", [
    fn("date_part", "minute", {"cast": col(1), "to": "Timestamp(us, Europe/Paris)"}),
    fn("date_trunc", "minute", {"cast": col(1), "to": "Timestamp(us, America/New_York)"}),
    {"cast": {"cast": col(1), "to": "Timestamp(us, Asia/Tokyo)"}, "to": "Date32"},
    fn("date_part", "fortnight", col(0)), fn("date_trunc", "millennium", col(0)), fn("date_part", "week", col(0)),
    {"op": "+", "l": col(0), "r": col(0)}, {"op": "-", "l": col(0), "r": {"lit": 1, "type": "Int64"}}, {"neg": col(0)},
    {"op": "<", "l": col(0), "r": col(2)}, {"op": "=", "l": col(0), "r": col(1)},
    {"cast": col(2), "to": "Timestamp(us, UTC)"}, {"cast": col(3), "to": "Timestamp(us, UTC)"}, {"cast": col(0), "to": "Timestamp(s, UTC)"},
    {"cast": col(0), "to": "Float64"}, {"cast": col(0), "to": "Timestamp(us)"},
    # CASE brings its branches to the first one's type with implied casts: they follow the same rules as written ones
    {"case": [[col(4), col(5)]], "else": col(0)}, {"case": [[col(4), col(7)]], "else": col(0)}, {"case": [[col(4), col(6)]], "else": col(0)},
    {"case": [[col(4), col(0)]], "else": col(3)}, {"case": [[col(4), col(0)]], "else": col(5)}, {"case": [[col(4), col(0)]], "else": col(2)},
], ids=lambda e: json.dumps(e)[:60])
def test_unsupported_expressions_are_refused_at_plan_time(expr):
    assert refused({"op": "projection", "exprs": [{"expr": expr, "name": "x"}]}, MIXED) == 2      # SAILGPU_ERR_UNSUPPORTED


MIXED = pa.schema([("t", pa.timestamp("us", tz="UTC")), ("i", pa.int64()), ("n", pa.timestamp("ns", tz="UTC")), ("d", pa.date32()),
                   ("b", pa.bool_()), ("s", pa.string_view()), ("f", pa.float64()), ("ts", pa.timestamp("s", tz="UTC"))])


def test_case_over_timestamps_of_one_type_is_accepted():
    spec = {"op": "projection", "exprs": [{"expr": {"case": [[col(4), col(0)]], "else": {"lit": 0, "type": "Timestamp(us, UTC)"}}, "name": "x"},
                                          {"expr": {"case": [[col(4), {"cast": col(7), "to": "Timestamp(us, UTC)"}]], "else": col(0)}, "name": "y"}]}
    out = engine.validate(spec, [MIXED])
    assert out.field("x").type == pa.timestamp("us", tz="UTC") and out.field("y").type == pa.timestamp("us", tz="UTC")
    cols = [pa.array([0, 1], type=pa.int64()).cast(f.type) if pa.types.is_timestamp(f.type) else pa.array([1, 2], type=pa.int64())
            for f in (MIXED.field(i) for i in range(3))]
    cols += [pa.array([1, 2], type=pa.date32()), pa.array([True, False]), pa.array(["a", "b"], type=pa.string_view()),
             pa.array([1.0, 2.0]), pa.array([3, 4], type=pa.int64()).cast(MIXED.field("ts").type)]
    t = pa.Table.from_arrays(cols, schema=MIXED)
    got = ref.ref_op(spec, t)
    assert [(f.name, f.type) for f in got.schema] == [(f.name, f.type) for f in out]


@pytest.mark.parametrize("fn_", ["sum", "avg"])
def test_sum_and_avg_of_timestamps_are_refused(fn_):
    s = pa.schema([("t", pa.timestamp("us", tz="UTC"))])
    spec = {"op": "aggregate", "mode": "single", "group_by": [], "aggs": [{"fn": fn_, "args": [col(0)], "name": "x", "input_type": "Timestamp(us, UTC)"}]}
    assert refused(spec, s) == 2


def test_zones_pass_through_operators_that_do_not_read_wall_clock_time():
    s = pa.schema([("t", pa.timestamp("us", tz="Europe/Paris")), ("i", pa.int64())])
    specs = [{"op": "filter", "predicate": {"op": ">", "l": col(0), "r": {"lit": 5, "type": "Timestamp(us, Europe/Paris)"}}},
             {"op": "sort", "keys": [{"expr": col(0), "asc": True, "nulls_first": True}], "fetch": 3},
             {"op": "aggregate", "mode": "single", "group_by": [{"expr": col(0), "name": "t"}],
              "aggs": [{"fn": "min", "args": [col(0)], "name": "mn", "input_type": "Timestamp(us, Europe/Paris)"}]}]
    for spec in specs:
        out = engine.validate(spec, [s])
        assert out.field("t").type == pa.timestamp("us", tz="Europe/Paris")


# ---- the reference's wall-clock arithmetic ---------------------------------------------------------------------------------------
def python_parts(local: dt.datetime):
    return {"year": local.year, "quarter": (local.month - 1) // 3 + 1, "month": local.month, "day": local.day, "hour": local.hour,
            "minute": local.minute, "second": local.second * 1_000_000 + local.microsecond}


def python_trunc(local: dt.datetime, part):
    if part == "week":
        d = local.replace(hour=0, minute=0, second=0, microsecond=0)
        return d - dt.timedelta(days=d.weekday())
    keep = ["year", "month", "day", "hour", "minute", "second"]
    if part == "quarter":
        return local.replace(month=(local.month - 1) // 3 * 3 + 1, day=1, hour=0, minute=0, second=0, microsecond=0)
    cut = keep[keep.index(part) + 1:]
    repl = {k: (1 if k in ("month", "day") else 0) for k in cut}
    repl["microsecond"] = 0
    return local.replace(**repl)


@pytest.mark.parametrize("tz", ZONES)
def test_reference_agrees_with_python_datetime(tz):
    v = np.array([micros(d) for d in INSTANTS], dtype=np.int64)
    z = zone(tz)
    for i, d in enumerate(INSTANTS):
        local = d.replace(tzinfo=dt.timezone.utc).astimezone(z)
        want = python_parts(local)
        for p in ref.PARTS:
            assert int(ref.date_part(v[i:i + 1], p, "us", tz or "")[1][0]) == want[p], (d, tz, p)
        for p in ref.TRUNC_PARTS:
            w = python_trunc(local, p)
            assert int(ref.date_trunc(v[i:i + 1], p, "us", tz or "")[0]) == micros(w.astimezone(dt.timezone.utc).replace(tzinfo=None)), (d, tz, p)
        assert int(ref.cast_to_date(v[i:i + 1], "us", tz or "")[0]) == (local.date() - dt.date(1970, 1, 1)).days


@pytest.mark.parametrize("unit", UNITS)
@pytest.mark.parametrize("tz", ZONES)
def test_reference_agrees_with_pyarrow_compute(unit, tz):
    arr = ts_table(2000, unit, tz, seed=3, nulls=False).column("t").combine_chunks()
    v = arr.cast(pa.int64()).to_numpy()
    local = arr if tz is None else pc.local_timestamp(arr)
    for p, f in [("year", pc.year), ("quarter", pc.quarter), ("month", pc.month), ("day", pc.day), ("hour", pc.hour), ("minute", pc.minute)]:
        assert np.array_equal(ref.date_part(v, p, unit, tz or "")[1], f(local).to_numpy().astype(np.int32)), p
    for p in ref.TRUNC_PARTS:
        if ref.UNITS[unit] == 1 and p == "second":
            continue
        want = pc.floor_temporal(local, unit=p, week_starts_monday=True).cast(pa.int64()).to_numpy() - ref.zone_seconds(tz or "") * ref.UNITS[unit]
        assert np.array_equal(ref.date_trunc(v, p, unit, tz or ""), want), p


# ---- ClickBench [18] and [42] ----------------------------------------------------------------------------------------------------
def hits(n=30000):
    from datagen import hits as gen
    return gen.hits(n, seed=7)


@pytest.mark.parametrize("name", list(cb.TIMESTAMP_QUERIES))
def test_clickbench_timestamp_plans_validate_node_by_node(name):
    t = hits()
    plan = cb.TIMESTAMP_QUERIES[name].plan()

    def walk(node):
        if node.spec["op"] == "scan":
            return t.select(node.spec["columns"])
        ins = [walk(c) for c in node.inputs]
        want = ref.ref_op(node.spec, *ins)
        got = engine.validate(node.spec, [i.schema for i in ins])
        assert [(f.name, f.type) for f in got] == [(f.name, f.type) for f in want.schema], node.spec["op"]
        return want
    walk(plan)


def test_clickbench_timestamp_plans_keep_the_snapshot_limits():
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "clickbench_plan_ops.json")))["queries"]
    for name, q in cb.TIMESTAMP_QUERIES.items():
        top = cb.top_sort(q.plan())
        assert top.spec["fetch"] == golden[name]["topk"] and q.skip == golden[name]["skip"], name
    assert set(cb.QUERIES).isdisjoint(cb.TIMESTAMP_QUERIES) and {q.sql for q in cb.TIMESTAMP_QUERIES.values()} == {18, 42}


# ---- specialised kernels -------------------------------------------------------------------------------------------------------
SCRIPT = r"""
import json, os, sys
sys.path.insert(0, sys.argv[1])
import pyarrow as pa
from sail_b200 import engine, plans, clickbench as cb
for name, spec, schema in json.loads(sys.argv[2]):
    schema = pa.schema([(n, pa.timestamp("us", tz="UTC") if t == "ts" else pa.int64()) for n, t in schema])
    before = set(os.listdir(os.environ["SAILGPU_JIT_CACHE"]))
    engine.jit_precompile(spec, [schema], 0, engine.JIT_COMPILE)
    new = sorted(set(os.listdir(os.environ["SAILGPU_JIT_CACHE"])) - before)
    print(name + "\t" + (new[-1] if new else ""))
"""


def kernels_to_compile():
    proj = {"op": "projection", "exprs": [{"expr": fn("date_trunc", "minute", col(0)), "name": "m"},
                                          {"expr": fn("date_part", "minute", col(0)), "name": "pm"},
                                          {"expr": fn("date_part", "hour", col(0)), "name": "ph"}]}
    partial = cb.c42().inputs[0].inputs[0]          # sort <- final <- partial
    assert partial.spec["mode"] == "partial"
    return [("projection", proj, [("t", "ts")]), ("c42_partial", partial.spec, [("EventTime", "i64")])]


@pytest.mark.skipif(not os.path.exists("/usr/local/cuda/bin/cuobjdump") and shutil.which("cuobjdump") is None, reason="cuobjdump not installed")
def test_specialised_timestamp_kernels_use_no_local_memory():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    with tempfile.TemporaryDirectory(prefix="sailgpu_jit_") as cache:
        env = dict(os.environ, SAILGPU_JIT_CACHE=cache)
        out = subprocess.run([sys.executable, "-c", SCRIPT, ROOT, json.dumps(kernels_to_compile())], env=env, capture_output=True, text=True, check=True).stdout
        kernels = [line.split("\t") for line in out.strip().splitlines()]
        assert len(kernels) == 2
        for name, f in kernels:
            assert f, f"{name}: no kernel compiled"
            path = os.path.join(cache, f)
            res = subprocess.run([cuobjdump, "--dump-resource-usage", path], capture_output=True, text=True, check=True).stdout
            m = re.search(r"REG:(\d+) STACK:(\d+)", res)
            assert m and int(m.group(2)) == 0, f"{name}: {res}"
            sass = subprocess.run([cuobjdump, "-sass", path], capture_output=True, text=True, check=True).stdout
            assert not re.search(r"\b(STL|LDL)\b", sass), f"{name}: local loads or stores in the SASS"


# ---- Parquet ---------------------------------------------------------------------------------------------------------------------
def ts_parquet(unit, tz, codec, level=None, n=5000):
    t = ts_table(n, unit, tz, seed=9)
    buf = io.BytesIO()
    pq.write_table(t.select(["t"]), buf, compression=codec, compression_level=level, coerce_timestamps=None if unit != "s" else "ms",
                   allow_truncated_timestamps=False, store_schema=True)
    return t, buf.getvalue()


@pytest.mark.parametrize("unit", ["ms", "us", "ns"])
@pytest.mark.parametrize("codec,level", [("none", None), ("zstd", 1), ("zstd", 19)])
def test_parquet_walk_accepts_timestamp_int64_chunks(unit, codec, level):
    t, raw = ts_parquet(unit, "UTC", codec, level)
    f = pq.ParquetFile(io.BytesIO(raw))
    assert f.metadata.row_group(0).column(0).physical_type == "INT64"
    assert f.schema_arrow.field("t").type == pa.timestamp(unit, tz="UTC")
    info = engine.parquet_inspect(raw, 0)
    assert info["dense"] == t.num_rows - t.column("t").null_count and info["level_values"] == t.num_rows


def test_int96_timestamps_stay_refused():
    t = ts_table(100, "ns", None, seed=2)
    buf = io.BytesIO()
    pq.write_table(t.select(["t"]), buf, use_deprecated_int96_timestamps=True)
    with pytest.raises(engine.SailGpuError) as e:
        engine.parquet_inspect(buf.getvalue(), 0)
    assert e.value.code == 2
