"""GPU parity: FilterExec / ProjectionExec / AggregateExec (and their fused pipeline) through the
C ABI vs the oracle, bit-exact for integer/decimal/date/string columns."""
import decimal

import numpy as np
import pyarrow as pa
import pytest

from sail_b200 import plans
from tests.util import assert_same, gpu_op, oracle_op

pytestmark = pytest.mark.gpu


def make_table(n, seed=0, nulls=False):
    rng = np.random.default_rng(seed)
    a = rng.integers(-1000, 1000, n).astype(np.int64)
    b = rng.integers(0, 50, n).astype(np.int32)
    d = [decimal.Decimal(int(x)) / 100 for x in rng.integers(-10**9, 10**9, n)]
    f = rng.normal(size=n)
    s = [["alpha", "beta", "gamma", "a considerably longer string value", ""][i] for i in rng.integers(0, 5, n)]
    dt = rng.integers(8000, 11000, n).astype(np.int32)
    mask = (rng.random(n) < 0.2) if nulls else None
    cols = {
        "a": pa.array(a, mask=mask),
        "b": pa.array(b, mask=None if not nulls else rng.random(n) < 0.1),
        "d": pa.array(d, type=pa.decimal128(15, 2), mask=None if not nulls else rng.random(n) < 0.15),
        "f": pa.array(f),
        "s": pa.array(s, type=pa.string_view(), mask=None if not nulls else rng.random(n) < 0.1),
        "dt": pa.array(dt, type=pa.int32()).cast(pa.date32()),
    }
    return pa.table(cols)


C = plans.col


def resolve(e, t):
    return plans.resolve(e, t.schema.names)


@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 1000, 5000, 70001])
@pytest.mark.parametrize("nulls", [False, True])
def test_projection(n, nulls):
    t = make_table(n, seed=n, nulls=nulls)
    exprs = [
        (plans.binop("+", C("a"), plans.lit(7, "Int64")), "a7"),
        (plans.binop("*", C("d"), plans.binop("-", plans.dec(1, 10, 0), C("d"))), "dd"),
        (plans.binop("<=", C("dt"), plans.date("1995-06-17")), "early"),
        (plans.binop("=", C("s"), plans.string("beta")), "is_beta"),
        (plans.binop("=", C("s"), plans.string("a considerably longer string value")), "is_long"),
        (plans.binop("*", C("f"), plans.lit(2.5, "Float64")), "f2"),
        (C("s"), "s"),
        (C("d"), "d"),
        (plans.binop("and", plans.binop(">", C("a"), plans.lit(0, "Int64")), plans.binop("<", C("b"), plans.lit(25, "Int32"))), "both"),
        ({"cast": C("b"), "to": "Int64"}, "b64"),
        ({"case": [[plans.binop(">", C("a"), plans.lit(0, "Int64")), C("d")]], "else": plans.dec(0, 15, 2)}, "casewhen"),
    ]
    spec = {"op": "projection", "exprs": [{"expr": resolve(e, t), "name": nm} for e, nm in exprs]}
    assert_same(gpu_op(spec, t), oracle_op(spec, t), ordered=True, float_cols={5})


@pytest.mark.parametrize("n", [0, 1, 300, 4097, 100003])
@pytest.mark.parametrize("nulls", [False, True])
def test_filter(n, nulls):
    t = make_table(n, seed=n + 1, nulls=nulls)
    pred = plans.and_(plans.binop(">=", C("a"), plans.lit(-500, "Int64")),
                      plans.or_(plans.binop("<", C("d"), plans.dec(12345, 15, 2)), plans.binop("=", C("s"), plans.string("gamma"))))
    spec = {"op": "filter", "predicate": resolve(pred, t), "projection": [0, 2, 4, 5]}
    assert_same(gpu_op(spec, t), oracle_op(spec, t), ordered=True)
    spec = {"op": "filter", "predicate": resolve(plans.binop(">", C("a"), plans.lit(10**6, "Int64")), t), "projection": None}
    assert_same(gpu_op(spec, t), oracle_op(spec, t), ordered=True)


@pytest.mark.parametrize("n", [1, 300, 1024, 4097, 100003, 300007])
@pytest.mark.parametrize("nulls", [False, True])
def test_filter_two_pass(n, nulls, monkeypatch):
    """Large batches filter in two passes (mask pass, scan of the per-tile popcounts, store pass at known offsets);
    the threshold is lowered so that the small and ragged sizes take that path too."""
    monkeypatch.setenv("SAILGPU_TWO_PASS_MIN", "1")
    t = make_table(n, seed=n + 5, nulls=nulls)
    pred = plans.and_(plans.binop(">=", C("a"), plans.lit(-500, "Int64")),
                      plans.or_(plans.binop("<", C("d"), plans.dec(12345, 15, 2)), plans.binop("=", C("s"), plans.string("gamma"))))
    spec = {"op": "filter", "predicate": resolve(pred, t), "projection": [0, 2, 4, 5]}
    assert_same(gpu_op(spec, t), oracle_op(spec, t), ordered=True)
    # nothing / everything passes, no projection list
    spec = {"op": "filter", "predicate": resolve(plans.binop(">", C("a"), plans.lit(10**6, "Int64")), t), "projection": None}
    assert_same(gpu_op(spec, t), oracle_op(spec, t), ordered=True)
    spec = {"op": "filter", "predicate": resolve(plans.binop("<", C("b"), plans.lit(10**6, "Int32")), t), "projection": None}
    assert_same(gpu_op(spec, t), oracle_op(spec, t), ordered=True)
    # filter + computed projection fused in one pipeline
    spec = {"op": "pipeline", "stages": [
        {"op": "filter", "predicate": resolve(plans.binop("<", C("b"), plans.lit(20, "Int32")), t), "projection": None},
        {"op": "projection", "exprs": [{"expr": resolve(plans.binop("+", C("a"), plans.lit(1, "Int64")), t), "name": "a1"},
                                       {"expr": resolve(C("s"), t), "name": "s"}]}]}
    want = oracle_op(spec["stages"][1], oracle_op(spec["stages"][0], t))
    assert_same(gpu_op(spec, t), want, ordered=True)


def test_filter_large_batch_order_and_content_vs_numpy():
    """8 M rows through the default (two-pass) FilterExec path: exactly the rows numpy selects, in input order"""
    n = 8_000_003
    rng = np.random.default_rng(123)
    a = rng.integers(0, 1000, n).astype(np.int64)
    b = rng.integers(0, 100, n).astype(np.int32)
    t = pa.table({"a": pa.array(a), "b": pa.array(b), "i": pa.array(np.arange(n, dtype=np.int64))})
    for lo, hi in ((0, 1000), (10, 20), (999, 1000), (1000, 1001)):          # everything / 1 % / 0.1 % / nothing
        pred = plans.and_(plans.binop(">=", {"col": 0}, plans.lit(lo, "Int64")), plans.binop("<", {"col": 0}, plans.lit(hi, "Int64")))
        got = gpu_op({"op": "filter", "predicate": pred, "projection": [2, 1]}, t)
        keep = (a >= lo) & (a < hi)
        assert got.num_rows == int(keep.sum())
        assert np.array_equal(got.column(0).to_numpy(), np.nonzero(keep)[0])
        assert np.array_equal(got.column(1).to_numpy(), b[keep])


def test_filter_two_pass_matches_single_pass(monkeypatch):
    t = make_table(400001, seed=77, nulls=True)
    spec = {"op": "filter", "predicate": resolve(plans.binop("<", C("b"), plans.lit(3, "Int32")), t), "projection": [0, 1, 2, 4]}
    monkeypatch.setenv("SAILGPU_TWO_PASS_MIN", "off")
    one = gpu_op(spec, t)
    monkeypatch.setenv("SAILGPU_TWO_PASS_MIN", "1")
    two = gpu_op(spec, t)
    assert_same(two, one, ordered=True)
    assert_same(two, oracle_op(spec, t), ordered=True)


@pytest.mark.parametrize("n", [0, 1, 999, 50000])
@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("keys", [[], ["b"], ["s"], ["b", "s", "dt"], ["s", "d", "b"]])      # the last one: 5 key words (no CTA dictionary)
def test_aggregate_single(n, nulls, keys):
    t = make_table(n, seed=n + 2, nulls=nulls)
    aggs = [("sum", "d"), ("avg", "d"), ("count", None), ("count", "a"), ("min", "a"), ("max", "d"), ("sum", "a"), ("avg", "f"), ("sum", "f"), ("min", "dt")]
    spec = {"op": "aggregate", "mode": "single",
            "group_by": [{"expr": resolve(C(k), t), "name": k} for k in keys],
            "aggs": [{"fn": fn, "args": [] if c is None else [resolve(C(c), t)], "name": f"{fn}_{c}"} for fn, c in aggs]}
    nk = len(keys)
    assert_same(gpu_op(spec, t), oracle_op(spec, t), float_cols={nk + 7, nk + 8})


@pytest.mark.parametrize("nulls", [False, True])
def test_aggregate_wide_keys_integer_sums(nulls):
    """sums/counts that qualify for the register fast path, but grouped by more key words than the CTA dictionary holds
    (TPC-H Q7's shape: two strings + a year): must take the general path"""
    t = make_table(30011, seed=77, nulls=nulls)
    names = t.schema.names
    spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": names.index(c)}, "name": c} for c in ("s", "d", "b")],
            "aggs": [{"fn": "sum", "args": [{"col": names.index("a")}], "name": "sa"}, {"fn": "count", "args": [], "name": "c"}]}
    assert_same(gpu_op(spec, t), oracle_op(spec, t))


def test_two_phase_aggregate():
    t = make_table(20000, seed=5, nulls=True)
    aggs = [("sum", "d", "Decimal128(15,2)"), ("avg", "d", "Decimal128(15,2)"), ("count", None, None), ("min", "a", "Int64"), ("avg", "a", "Int64")]
    def mk(mode, names):
        merging = mode != "partial"
        return {"op": "aggregate", "mode": mode,
                "group_by": [{"expr": {"col": names.index("b")}, "name": "b"}],
                "aggs": [{"fn": fn, "args": [] if (c is None or merging) else [{"col": names.index(c)}], "name": f"{fn}_{c}", "input_type": it}
                         for fn, c, it in aggs]}
    part = mk("partial", t.schema.names)
    halves = [t.slice(0, 9000), t.slice(9000)]
    partial_tables = [gpu_op(part, h) for h in halves]
    want_partial = [oracle_op(part, h) for h in halves]
    for g, w in zip(partial_tables, want_partial):
        assert_same(g, w, float_cols={6})
    merged = pa.concat_tables(partial_tables)
    fin = mk("final_partitioned", merged.schema.names)
    fin["group_by"] = [{"expr": {"col": 0}, "name": "b"}]
    assert_same(gpu_op(fin, merged), oracle_op(fin, merged), float_cols={5})


def strip_sort(node):
    return node.inputs[0] if node.spec["op"] == "sort" else node


@pytest.mark.parametrize("sf", [0.001, 0.01])
@pytest.mark.parametrize("q", ["q1", "q6"])
def test_tpch_pipeline_queries(q, sf):
    from datagen import tpch
    tables = {"lineitem": tpch.lineitem(sf)}
    plan = strip_sort(plans.TPCH[q]())
    got = plans.execute(plan, tables, gpu_op)
    want = plans.execute(plan, tables, oracle_op)
    assert_same(got, want)


def fuse(node):
    """collapse a Filter/Projection/.../Aggregate(partial) chain into one pipeline spec"""
    stages = []
    n = node
    while n.spec["op"] in ("filter", "projection", "aggregate"):
        stages.append(n.spec)
        n = n.inputs[0]
    return plans.Node({"op": "pipeline", "stages": stages[::-1]}, [n], node.names)


@pytest.mark.parametrize("q", ["q1", "q6"])
def test_fused_pipeline_matches_operator_chain(q):
    from datagen import tpch
    tables = {"lineitem": tpch.lineitem(0.01)}
    final = strip_sort(plans.TPCH[q]())
    partial = final.inputs[0]
    fused_partial = fuse(partial)
    assert fused_partial.spec["op"] == "pipeline" and len(fused_partial.spec["stages"]) == 3
    fused = plans.Node(final.spec, [fused_partial], final.names)
    got = plans.execute(fused, tables, gpu_op)
    want = plans.execute(final, tables, oracle_op)
    assert_same(got, want)


def test_divide_by_zero_is_an_error():
    from sail_b200 import engine
    t = pa.table({"a": pa.array([1, 2, 3], type=pa.int64()), "b": pa.array([1, 0, 2], type=pa.int64())})
    spec = {"op": "projection", "exprs": [{"expr": plans.binop("/", {"col": 0}, {"col": 1}), "name": "q"}]}
    with pytest.raises(engine.SailGpuError) as e:
        gpu_op(spec, t)
    assert "ivide by zero" in str(e.value)


def test_aggregate_many_groups_multi_batch_growth():
    """streams 16 batches into one AggregateExec: the global table grows (rehash) several times, most rows take the
    cold (global-table) path, keys include long strings"""
    from sail_b200 import engine
    rng = np.random.default_rng(42)
    n_batches, n = 16, 40000
    words = [f"key-{i:06d}-{'x' * (i % 17)}" for i in range(3000)]
    batches = []
    for b in range(n_batches):
        k = rng.integers(0, 20000 * (b + 1), n).astype(np.int64)          # key domain keeps widening -> growth
        s = [words[i] for i in rng.integers(0, len(words), n)]
        v = [decimal.Decimal(int(x)) / 100 for x in rng.integers(-10**7, 10**7, n)]
        batches.append(pa.table({"k": pa.array(k), "s": pa.array(s, type=pa.string_view()), "v": pa.array(v, type=pa.decimal128(15, 2))}))
    whole = pa.concat_tables(batches)
    for keys in (["k"], ["s"], ["k", "s"]):
        spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": whole.schema.names.index(c)}, "name": c} for c in keys],
                "aggs": [{"fn": "sum", "args": [{"col": 2}], "name": "sv"}, {"fn": "count", "args": [], "name": "c"},
                         {"fn": "max", "args": [{"col": 2}], "name": "mx"}, {"fn": "avg", "args": [{"col": 2}], "name": "av"}]}
        op = engine.GpuExec(spec, [whole.schema])
        for t in batches:
            op.push(t)
        op.finish()
        got = op.collect()
        op.close()
        assert_same(got, oracle_op(spec, whole))


@pytest.mark.parametrize("late_nulls", [False, True])
@pytest.mark.parametrize("ktype", ["int64", "date32", "decimal"])
@pytest.mark.parametrize("kernel", ["interpreted", "specialised"])
def test_aggregate_single_word_key(ktype, late_nulls, kernel, monkeypatch):
    """One never-null 8-byte key word, in the interpreted and in the specialised kernel (whose global table is compiled for a
    one-word key).  Covers INT64_MIN and 0 as real keys, growth with re-hashing over many batches, min/max identities, and a
    late batch with NULL keys, which moves the table to a layout with a null-mask word in the middle of the stream."""
    from sail_b200 import engine
    if kernel == "interpreted":
        monkeypatch.setenv("SAILGPU_JIT", "0")
    else:
        monkeypatch.setenv("SAILGPU_JIT_MIN_ROWS", "0")
        monkeypatch.setenv("SAILGPU_JIT_STRICT", "1")
    rng = np.random.default_rng(11)
    n_batches, n = 12, 50000
    batches = []
    for b in range(n_batches):
        k = rng.integers(-30000 * (b + 1), 30000 * (b + 1), n).astype(np.int64)
        if ktype == "int64":
            k[::997] = np.iinfo(np.int64).min
            k[1::1999] = 0
            karr = pa.array(k, mask=(rng.random(n) < 0.05) if (late_nulls and b >= 8) else None)
        elif ktype == "date32":
            karr = pa.array((k % 20000).astype(np.int32), type=pa.int32()).cast(pa.date32())
            if late_nulls and b >= 8:
                karr = pa.array(karr.to_pylist()[: n // 2] + [None] * (n - n // 2), type=pa.date32())
        else:
            vals = [decimal.Decimal(int(x)) / 100 for x in k]
            if late_nulls and b >= 8:
                vals[::13] = [None] * len(vals[::13])
            karr = pa.array(vals, type=pa.decimal128(15, 2))
        v = pa.array([decimal.Decimal(int(x)) / 100 for x in rng.integers(-10**7, 10**7, n)], type=pa.decimal128(15, 2))
        i = pa.array(rng.integers(-1000, 1000, n).astype(np.int64))
        batches.append(pa.table({"k": karr, "v": v, "i": i}))
    whole = pa.concat_tables(batches)
    spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": 0}, "name": "k"}],
            "aggs": [{"fn": "sum", "args": [{"col": 1}], "name": "sv"}, {"fn": "count", "args": [], "name": "c"}, {"fn": "min", "args": [{"col": 1}], "name": "mn"},
                     {"fn": "max", "args": [{"col": 2}], "name": "mx"}, {"fn": "avg", "args": [{"col": 1}], "name": "av"}, {"fn": "sum", "args": [{"col": 2}], "name": "si"}]}
    op = engine.GpuExec(spec, [whole.schema])
    for t in batches:
        op.push(t)
    op.finish()
    got = op.collect()
    m = op.metrics()
    op.close()
    assert_same(got, oracle_op(spec, whole))
    assert (m.get("gpu.jit_launches", 0) > 0) == (kernel == "specialised"), m


@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("keys", [["b"], ["a"], ["a", "s"]])
@pytest.mark.parametrize("first_limit", ["0", "40", "700"])
def test_aggregate_bounded_table_hands_tiles_back(keys, nulls, first_limit, monkeypatch):
    """The group table is bounded: CTAs that find it above the launch's group limit hand their remaining tiles back and
    the operator grows the table, rehashes and re-launches over the deferred list (switching to the many-groups variant
    of the pipeline).  SAILGPU_AGG_FIRST_LIMIT forces that on the first pass (0: everything is handed back)."""
    monkeypatch.setenv("SAILGPU_AGG_FIRST_LIMIT", first_limit)
    t = make_table(60001, seed=31, nulls=nulls)
    names = t.schema.names
    spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": names.index(c)}, "name": c} for c in keys],
            "aggs": [{"fn": "sum", "args": [{"col": names.index("d")}], "name": "sd"}, {"fn": "count", "args": [], "name": "c"},
                     {"fn": "min", "args": [{"col": names.index("dt")}], "name": "mn"}, {"fn": "avg", "args": [{"col": names.index("d")}], "name": "av"},
                     {"fn": "sum", "args": [{"col": names.index("f")}], "name": "sf"}]}
    assert_same(gpu_op(spec, t), oracle_op(spec, t), float_cols={len(keys) + 4})


def test_aggregate_bounded_table_grows_by_itself():
    """no forcing: 3 M distinct keys overflow the initial 4 M-slot table's group limit, so the natural hand-back /
    grow / re-launch path runs; sums and counts are checked against numpy"""
    from sail_b200 import engine
    n, domain = 4_000_000, 3_000_000
    rng = np.random.default_rng(5)
    k = rng.integers(0, domain, n).astype(np.int64)
    v = rng.integers(-1000, 1000, n).astype(np.int64)
    t = pa.table({"k": pa.array(k), "v": pa.array(v)})
    spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": 0}, "name": "k"}],
            "aggs": [{"fn": "sum", "args": [{"col": 1}], "name": "s"}, {"fn": "count", "args": [], "name": "c"}]}
    got = engine.run_op(spec, t)
    gk = got.column("k").to_numpy()
    order = np.argsort(gk)
    uk, inv, cnt = np.unique(k, return_inverse=True, return_counts=True)
    sums = np.bincount(inv, weights=v.astype(np.float64)).astype(np.int64)
    assert got.num_rows == len(uk)
    assert np.array_equal(gk[order], uk)
    assert np.array_equal(got.column("s").to_numpy()[order], sums)
    assert np.array_equal(got.column("c").to_numpy()[order], cnt)


def test_filter_streams_many_batches_in_order():
    from sail_b200 import engine
    t = make_table(30000, seed=9, nulls=True)
    spec = {"op": "filter", "predicate": resolve(plans.binop("<", C("b"), plans.lit(20, "Int32")), t), "projection": [0, 1, 4]}
    op = engine.GpuExec(spec, [t.schema])
    for o in range(0, t.num_rows, 777):          # ragged batch sizes
        op.push(t.slice(o, 777))
    op.finish()
    assert_same(op.collect(), oracle_op(spec, t), ordered=True)
    op.close()


@pytest.mark.parametrize("order", ["nulls_first", "nulls_last", "alternating"])
@pytest.mark.parametrize("keys", [["b"], ["s"], []])
def test_aggregate_batches_differ_in_validity_buffers(order, keys):
    """Arrow producers drop the validity buffer of a batch without nulls, so the batches of one stream differ in which
    columns carry one.  The table layout (null-mask word, seen bits, per-argument counters) must survive that in any order:
    groups that only appear in null-free batches, all-NULL groups, and nullable group keys."""
    from sail_b200 import engine
    rng = np.random.default_rng(5)

    def part(n, with_nulls, lo):
        b = rng.integers(lo, lo + 6, n).astype(np.int32)
        s = [f"g{int(x) % 5}" for x in rng.integers(lo, lo + 9, n)]
        v = [decimal.Decimal(int(x)) / 100 for x in rng.integers(-10**6, 10**6, n)]
        f = rng.normal(size=n)
        if with_nulls:
            mb, ms, mv = rng.random(n) < 0.2, rng.random(n) < 0.2, rng.random(n) < 0.5
            mv |= b == lo                      # one whole group whose argument is always NULL
            return pa.table({"b": pa.array(b, mask=mb), "s": pa.array(s, type=pa.string_view(), mask=ms),
                             "v": pa.array(v, type=pa.decimal128(15, 2), mask=mv), "f": pa.array(f, mask=mv)})
        return pa.table({"b": pa.array(b), "s": pa.array(s, type=pa.string_view()), "v": pa.array(v, type=pa.decimal128(15, 2)), "f": pa.array(f)})

    clean = [part(5000, False, 0), part(3000, False, 4)]        # group ids 0..9, some only here
    dirty = [part(4000, True, 2), part(2500, True, 8)]          # group ids 2..13, some only here
    batches = {"nulls_first": dirty + clean, "nulls_last": clean + dirty, "alternating": [clean[0], dirty[0], clean[1], dirty[1]]}[order]
    whole = pa.concat_tables(batches)
    spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": whole.schema.names.index(c)}, "name": c} for c in keys],
            "aggs": [{"fn": "sum", "args": [{"col": 2}], "name": "sv"}, {"fn": "count", "args": [], "name": "c"}, {"fn": "count", "args": [{"col": 2}], "name": "cv"},
                     {"fn": "min", "args": [{"col": 2}], "name": "mn"}, {"fn": "avg", "args": [{"col": 2}], "name": "av"}, {"fn": "max", "args": [{"col": 3}], "name": "mf"},
                     {"fn": "avg", "args": [{"col": 3}], "name": "af"}]}
    op = engine.GpuExec(spec, [whole.schema])
    for t in batches:
        op.push(t)
    op.finish()
    got = op.collect()
    op.close()
    n_key = len(keys)
    assert_same(got, oracle_op(spec, whole), float_cols=(n_key + 5, n_key + 6))


@pytest.mark.parametrize("shared_context", [True, False])
def test_concurrent_handles_from_two_threads(shared_context):
    """include/sailgpu.h threading contract: handles may be driven from any threads at once; handles of one context are
    serialised inside the library, handles of different contexts overlap.  DataFusion polls partitions from a thread pool."""
    import threading
    from sail_b200 import engine
    t = make_table(60000, seed=21, nulls=True)
    specs = [
        {"op": "aggregate", "mode": "single", "group_by": [{"expr": resolve(C("b"), t), "name": "b"}],
         "aggs": [{"fn": "sum", "args": [resolve(C("d"), t)], "name": "sd"}, {"fn": "count", "args": [], "name": "c"}]},
        {"op": "filter", "predicate": resolve(plans.binop("<", C("b"), plans.lit(25, "Int32")), t), "projection": [0, 2, 4]},
    ]
    want = [oracle_op(s, t) for s in specs]
    ctxs = [engine.default_context(), engine.default_context() if shared_context else engine.Context(0)]
    errors, got = [], [[None] * 6, [None] * 6]

    def work(k):
        try:
            for it in range(6):
                op = engine.GpuExec(specs[k], [t.schema], ctxs[k])
                for o in range(0, t.num_rows, 7001):
                    op.push(t.slice(o, 7001))
                op.finish()
                got[k][it] = op.collect()
                op.close()
        except Exception as e:      # surfaced below: an exception in a thread would otherwise be lost
            errors.append(e)

    threads = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    if not shared_context:
        ctxs[1].close()
    assert not errors, errors
    for k in range(2):
        for it in range(6):
            assert_same(got[k][it], want[k], ordered=(k == 1))
