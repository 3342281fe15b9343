"""character_length on the CPU: plan-time types and refusals from the library, the reference of tests/char_length_ref.py against
pyarrow and against ClickBench [27]'s SQL restated in pandas, and the specialised kernel's source for every pipeline of [27]."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from sail_b200 import clickbench as cb, engine, plans
from tests import char_length_ref as ref
from tests.test_clickbench import as_table
from tests.util import assert_topk

STRINGS = ["", "a", "héllo", "日本語", "🦀🦀", "x" * 12, "é" * 6, "abcdefghijk€", "€" * 40, None]


def length_of(i):
    return {"op": "projection", "exprs": [{"expr": plans.char_length({"col": i}), "name": "n"}]}


@pytest.mark.parametrize("t", [pa.string(), pa.string_view()])
def test_validate_gives_int32_for_utf8_and_utf8view(t):
    out = engine.validate(length_of(0), [pa.schema([("s", t)])])
    assert out.names == ["n"] and out.field("n").type == pa.int32()


@pytest.mark.parametrize("nullable", [False, True])
def test_result_is_nullable_exactly_when_the_input_is(nullable):
    out = engine.validate(length_of(0), [pa.schema([pa.field("s", pa.string_view(), nullable=nullable)])])
    assert out.field("n").nullable == nullable


def test_a_non_string_argument_is_refused_as_invalid():
    with pytest.raises(engine.SailGpuError) as e:
        engine.validate(length_of(0), [pa.schema([("x", pa.int64())])])
    assert e.value.code == 1


def test_only_the_physical_plan_name_is_accepted():
    for name in ("length", "char_length", "octet_length"):
        with pytest.raises(engine.SailGpuError) as e:
            engine.validate({"op": "projection", "exprs": [{"expr": {"fn": name, "args": [{"col": 0}]}, "name": "n"}]}, [pa.schema([("s", pa.string())])])
        assert e.value.code == 2, name


@pytest.mark.parametrize("t", [pa.string(), pa.string_view()])
def test_reference_counts_equal_pyarrow_utf8_length(t):
    rng = np.random.default_rng(5)
    vals = STRINGS + ["".join(rng.choice(["a", "ж", "€", "𝄞"], int(k))) for k in rng.integers(0, 300, 200)]
    tbl = pa.table({"s": pa.array(vals, type=t)})
    got = ref.ref_op(length_of(0), tbl).column("n")
    assert got.type == pa.int32()
    assert got.equals(pc.utf8_length(tbl.column("s").cast(pa.string())))


# ---- ClickBench [27] -------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hits():
    from datagen import hits as gen
    return gen.hits(30000, seed=7)


@pytest.fixture(scope="module")
def frame(hits):
    from tests import clickbench_sql as sql
    return sql.frame(hits)


def test_c27_is_planned_outside_queries_with_the_snapshot_limit():
    import json
    import os
    golden = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "clickbench_plan_ops.json")))["queries"]["c27"]
    q = cb.LENGTH_QUERIES["c27"]
    assert q.sql == 27 and 27 in cb.NOT_PLANNED and set(cb.QUERIES).isdisjoint(cb.LENGTH_QUERIES)
    assert cb.top_sort(q.plan()).spec["fetch"] == golden["topk"] and q.skip == golden["skip"]
    assert q.plan().names == ["CounterID", "l", "c"]


def test_every_c27_node_is_accepted_with_the_reference_schema(hits):
    seen = []

    def walk(node):
        if node.spec["op"] == "scan":
            return hits.select(node.spec["columns"]).slice(0, 2000)
        ins = [walk(c) for c in node.inputs]
        want = ref.ref_op(node.spec, *ins)
        got = engine.validate(node.spec, [t.schema for t in ins])
        assert got.names == want.schema.names and [str(f.type) for f in got] == [str(f.type) for f in want.schema], (node.spec["op"], got, want.schema)
        seen.append(node.spec["op"])
        return want
    walk(cb.c27())
    assert seen == ["filter", "aggregate", "aggregate", "filter", "sort"]


def test_reference_c27_equals_the_sql_restated_in_pandas(hits, frame):
    q = cb.LENGTH_QUERIES["c27"]
    min_count = ref.q27_min_count(frame)
    node = cb.top_sort(q.plan(min_count=min_count))
    got = plans.execute(node, {"hits": hits}, ref.ref_op)
    assert got.num_rows >= 10
    assert_topk(got, as_table(ref.q27(frame, min_count), got.schema), list(q.order), node.spec["fetch"], float_cols=q.floats)


def test_specialised_kernel_source_is_generated_for_every_c27_pipeline(hits):
    """as tests/test_jit_codegen.py does for QUERIES, with the inputs computed by the reference of this file"""
    out = []

    def walk(node):
        if node.spec["op"] == "scan":
            return hits.select(node.spec["columns"]).slice(0, 2000)
        ins = [walk(c) for c in node.inputs]
        if node.spec["op"] in ("filter", "aggregate"):
            for flags in (0, engine.JIT_COLD_VARIANT) if node.spec["op"] == "aggregate" else (0,):
                n, src = engine.jit_precompile(node.spec, [ins[0].schema], 0, flags)
                assert n == len(src) > 1000 and "struct G" in src
                out.append((node.spec["op"], src))
        return ref.ref_op(node.spec, *ins)
    walk(cb.c27())
    assert [op for op, _ in out] == ["filter", "aggregate", "aggregate", "aggregate", "aggregate", "filter"]
    assert sum("view_char_length(" in src for _, src in out) == 2        # both variants of the partial aggregate
