"""DISTINCT aggregates on the CPU: plan-time types, nullability and refusals from the library, the reference of
tests/distinct_ref.py against ClickBench [09]'s SQL restated in pandas and against the two-level rewrite c9, the plan shape of
c9_single, and the specialiser declining a gated pipeline."""
import pyarrow as pa
import pytest

from sail_b200 import clickbench as cb, engine, plans
from tests import distinct_ref as ref
from tests.test_clickbench import as_table
from tests.util import assert_same, assert_topk

UNSUPPORTED, INVALID = 2, 1


def agg(aggs, keys=(0,), mode="single"):
    return {"op": "aggregate", "mode": mode, "group_by": [{"expr": {"col": k}, "name": f"k{k}"} for k in keys], "aggs": aggs}


def a(fn, arg=1, distinct=True, name="r", **kw):
    out = {"fn": fn, "name": name, "args": [] if arg is None else [{"col": arg}], **kw}
    if distinct is not None:
        out["distinct"] = distinct
    return out


def schema(x_type, k_type=pa.int32(), nullable=True):
    return [pa.schema([pa.field("k", k_type), pa.field("x", x_type, nullable=nullable)])]


ARG_TYPES = [pa.int16(), pa.int32(), pa.int64(), pa.uint64(), pa.decimal128(15, 2), pa.decimal128(38, 0), pa.date32(),
             pa.timestamp("us", tz="UTC"), pa.string(), pa.string_view()]


@pytest.mark.parametrize("t", ARG_TYPES, ids=str)
@pytest.mark.parametrize("nullable", [False, True])
def test_count_distinct_is_int64_not_null(t, nullable):
    out = engine.validate(agg([a("count")]), schema(t, nullable=nullable))
    assert out.field("r").type == pa.int64() and not out.field("r").nullable


@pytest.mark.parametrize("fn", ["sum", "avg"])
@pytest.mark.parametrize("t", [pa.int16(), pa.int32(), pa.int64(), pa.uint64(), pa.decimal128(15, 2), pa.decimal128(38, 0)], ids=str)
def test_sum_and_avg_distinct_have_the_plain_type_and_are_nullable(fn, t):
    got = engine.validate(agg([a(fn)]), schema(t, nullable=False)).field("r")
    plain = engine.validate(agg([a(fn, distinct=None)]), schema(t, nullable=False)).field("r")
    assert got.type == plain.type and got.nullable


@pytest.mark.parametrize("fn", ["min", "max"])
@pytest.mark.parametrize("t", [pa.int32(), pa.int64(), pa.decimal128(38, 0), pa.float64(), pa.date32()], ids=str)
def test_min_max_distinct_is_a_no_op(fn, t):
    got = engine.validate(agg([a(fn)]), schema(t))
    assert got == engine.validate(agg([a(fn, distinct=None)]), schema(t))


@pytest.mark.parametrize("fn", ["count", "sum", "avg", "min"])
def test_distinct_false_gives_the_schema_of_no_key(fn):
    s = schema(pa.int64())
    assert engine.validate(agg([a(fn, distinct=False)]), s) == engine.validate(agg([a(fn, distinct=None)]), s)


def refused(spec, s):
    with pytest.raises(engine.SailGpuError) as e:
        engine.validate(spec, s)
    return e.value


@pytest.mark.parametrize("mode", ["partial", "final", "final_partitioned"])
def test_distinct_outside_single_mode_is_unsupported(mode):
    s = schema(pa.int64()) if mode == "partial" else [pa.schema([("k", pa.int32()), ("s", pa.int64())])]
    e = refused(agg([a("count", input_type="Int64")], mode=mode), s)
    assert e.code == UNSUPPORTED and "List" in str(e)


def test_two_arguments_are_unsupported():
    spec = agg([{"fn": "count", "name": "r", "args": [{"col": 1}, {"col": 0}], "distinct": True}])
    assert refused(spec, schema(pa.int64())).code == UNSUPPORTED


@pytest.mark.parametrize("fn", ["count", "sum", "avg"])
@pytest.mark.parametrize("t", [pa.float32(), pa.float64(), pa.bool_()], ids=str)
def test_float_and_boolean_arguments_are_unsupported(fn, t):
    if fn != "count" and t == pa.bool_():
        pytest.skip("sum / avg over Boolean are refused without DISTINCT as well")
    assert refused(agg([a(fn)]), schema(t)).code == UNSUPPORTED


def test_distinct_without_an_argument_is_invalid():
    assert refused(agg([a("count", arg=None)]), schema(pa.int64())).code == INVALID


def test_a_pair_key_wider_than_the_table_packs_is_unsupported():
    # seven columns: six group keys are what the hash table packs, the argument makes seven
    s = [pa.schema([(f"c{i}", pa.int32()) for i in range(7)])]
    assert refused(agg([a("count", arg=6)], keys=range(6)), s).code == UNSUPPORTED
    # 64 bytes: four strings (8 words) leave no room for the null-mask word and the argument -- the plain aggregate takes them
    s = [pa.schema([(f"c{i}", pa.string_view()) for i in range(4)] + [("x", pa.int64())])]
    assert refused(agg([a("count", arg=4)], keys=range(4)), s).code == UNSUPPORTED
    engine.validate(agg([a("count", arg=4, distinct=None)], keys=range(4)), s)
    # group keys wide enough for the sort-based aggregate: refused as well, not handed to it
    s = [pa.schema([(f"c{i}", pa.string_view()) for i in range(5)] + [("x", pa.int64())])]
    assert refused(agg([a("count", arg=5)], keys=range(5)), s).code == UNSUPPORTED


def test_more_than_four_distinct_arguments_are_unsupported():
    s = [pa.schema([("k", pa.int32())] + [(f"x{i}", pa.int64()) for i in range(5)])]
    assert refused(agg([a("count", arg=1 + i, name=f"r{i}") for i in range(5)]), s).code == UNSUPPORTED
    # count and sum over one argument share a gate: four arguments are fine
    engine.validate(agg([a(fn, arg=1 + i, name=f"{fn}{i}") for i in range(4) for fn in ("count", "sum")]), s)


def test_distinct_must_be_a_boolean():
    assert refused(agg([a("count", distinct="yes")]), schema(pa.int64())).code == INVALID


def test_plans_aggregate_marks_distinct_and_leaves_other_specs_as_they_were():
    t = plans.scan("t", ["k", "x"])
    old = plans.aggregate(t, "single", ["k"], [("count", plans.col("x"), "n", "Int64"), ("sum", plans.col("x"), "s", "Int64")])
    assert all("distinct" not in s for s in old.spec["aggs"])
    new = plans.aggregate(t, "single", ["k"], [("count", plans.col("x"), "n", "Int64", True), ("sum", plans.col("x"), "s", "Int64", False)])
    assert new.spec["aggs"][0]["distinct"] is True and "distinct" not in new.spec["aggs"][1]
    assert {**new.spec["aggs"][0], "distinct": None} == {**old.spec["aggs"][0], "distinct": None}


# ---- ClickBench [09] ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hits():
    from datagen import hits as gen
    return gen.hits(30000, seed=7)


@pytest.fixture(scope="module")
def frame(hits):
    from tests import clickbench_sql as sql
    return sql.frame(hits)


def test_c9_single_has_the_reference_shape():
    q = cb.DISTINCT_QUERIES["c9_single"]
    assert q.sql == 9 and set(cb.QUERIES).isdisjoint(cb.DISTINCT_QUERIES) and "c9" in cb.QUERIES and len(cb.QUERIES) == 37
    node = q.plan()
    ops = []

    def walk(n):
        ops.append(n.spec["op"])
        for c in n.inputs:
            walk(c)
    walk(node)
    assert ops == ["sort", "projection", "aggregate", "scan"]
    assert node.spec["fetch"] == 10
    a = node.inputs[0].inputs[0].spec
    assert a["mode"] == "single" and [g["name"] for g in a["group_by"]] == ["RegionID"]
    assert [(x["fn"], bool(x.get("distinct"))) for x in a["aggs"]] == [("sum", False), ("count", False), ("avg", False), ("count", True)]
    assert "alias1" not in str(node.spec) + str(a)
    assert node.names == cb.c9().names


def test_every_c9_single_node_validates_with_the_reference_schema(hits):
    seen = []

    def walk(node):
        if node.spec["op"] == "scan":
            return hits.select(node.spec["columns"]).slice(0, 3000)
        ins = [walk(c) for c in node.inputs]
        want = ref.ref_op(node.spec, *ins)
        got = engine.validate(node.spec, [t.schema for t in ins])
        assert got.names == want.schema.names and [str(f.type) for f in got] == [str(f.type) for f in want.schema], (node.spec["op"], got, want.schema)
        seen.append(node.spec["op"])
        return want
    walk(cb.c9_single())
    assert seen == ["aggregate", "projection", "sort"]


def test_reference_c9_single_equals_the_sql_and_the_two_level_plan(hits, frame):
    from tests import clickbench_sql as sql
    q = cb.DISTINCT_QUERIES["c9_single"]
    node = q.plan()
    got = plans.execute(node, {"hits": hits}, ref.ref_op)
    assert got.num_rows == 10
    assert_topk(got, as_table(sql.q9(frame), got.schema), list(q.order), node.spec["fetch"], float_cols=q.floats)
    full = plans.execute(cb.without_limit(node), {"hits": hits}, ref.ref_op)
    two_level = plans.execute(cb.without_limit(cb.c9()), {"hits": hits}, ref.oracle_op)
    assert_same(full, two_level, float_cols=q.floats)


def test_reference_counts_distinct_pairs_per_group():
    t = pa.table({"k": pa.array([1, 1, 1, 2, 2, None, None, 3], pa.int32()), "x": pa.array([5, 5, 6, None, None, 7, 7, 8], pa.int64())})
    got = ref.ref_op(agg([a("count", name="n"), a("sum", name="s"), a("count", name="c", distinct=None), a("max", name="m")]), t)
    rows = sorted(zip(*[got.column(i).to_pylist() for i in range(got.num_columns)]), key=str)
    assert rows == sorted([(1, 2, 11, 3, 6), (2, 0, None, 0, None), (None, 1, 7, 2, 7), (3, 1, 8, 1, 8)], key=str)


def test_the_specialiser_declines_a_gated_pipeline():
    spec = agg([a("count", name="n"), a("count", name="c", distinct=None)])
    with pytest.raises(engine.SailGpuError) as e:
        engine.jit_precompile(spec, schema(pa.int64()), 0, 0)
    assert e.value.code == UNSUPPORTED and "DISTINCT" in str(e.value)
    n, src = engine.jit_precompile(agg([a("count", name="c", distinct=None)]), schema(pa.int64()), 0, 0)
    assert n == len(src) > 1000
