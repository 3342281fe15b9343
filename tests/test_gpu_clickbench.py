"""ClickBench (BASELINE.json configs[4]) on the GPU: the 37 plans of sail_b200/clickbench.py through the C ABI on a synthetic hits
table, each result checked against the query's SQL restated in pandas (tests/clickbench_sql.py) -- up to ties for ORDER BY ..
LIMIT, Float64 AVG within 1e-6 relative, everything else bit-exact.  The same check runs the oracle on the CPU
(tests/test_clickbench.py)."""
import numpy as np
import pyarrow as pa
import pytest

from sail_b200 import clickbench as cb
from tests import clickbench_sql as sql
from tests.test_clickbench import check
from tests.util import assert_same, gpu_op, oracle_op

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def hits():
    from datagen import hits as gen
    return gen.hits(100_000, seed=7)


@pytest.fixture(scope="module")
def frame(hits):
    return sql.frame(hits)


@pytest.mark.parametrize("name", list(cb.QUERIES))
def test_clickbench_query_equals_its_sql(name, hits, frame):
    check(name, frame, {"hits": hits}, gpu_op)


@pytest.mark.parametrize("mode", ["single", "two_phase"])
@pytest.mark.parametrize("nulls", [False, True])
def test_two_byte_group_keys_keep_both_bytes(mode, nulls):
    """Int16 / UInt16 group keys beyond one byte and below zero (ClickBench [39] TraficSourceID = -1, [41] WindowClientWidth up to
    2560): the aggregate's output kernel once wrote only the low byte of a 2-byte key column."""
    rng = np.random.default_rng(5)
    n = 40000
    k = rng.integers(-700, 700, n).astype(np.int16)
    u = rng.choice(np.array([0, 255, 256, 1280, 2560, 40000, 65535], dtype=np.uint16), n)
    mask = (rng.random(n) < 0.1) if nulls else None
    t = pa.table({"k": pa.array(k, mask=mask), "u": pa.array(u), "v": pa.array(rng.integers(-1000, 1000, n).astype(np.int64))})
    gb = [{"expr": {"col": 0}, "name": "k"}, {"expr": {"col": 1}, "name": "u"}]
    aggs = [{"fn": "sum", "args": [{"col": 2}], "name": "s", "input_type": "Int64"}, {"fn": "count", "args": [], "name": "c", "input_type": None},
            {"fn": "min", "args": [{"col": 0}], "name": "mk", "input_type": "Int16"}, {"fn": "max", "args": [{"col": 1}], "name": "mu", "input_type": "UInt16"}]
    if mode == "single":
        spec = {"op": "aggregate", "mode": "single", "group_by": gb, "aggs": aggs}
        assert_same(gpu_op(spec, t), oracle_op(spec, t))
        return
    partial = {"op": "aggregate", "mode": "partial", "group_by": gb, "aggs": aggs}
    final = {"op": "aggregate", "mode": "final_partitioned", "group_by": gb, "aggs": [{k2: v for k2, v in a.items() if k2 != "args"} for a in aggs]}
    halves = [gpu_op(partial, t.slice(0, n // 2)), gpu_op(partial, t.slice(n // 2))]
    want = oracle_op(final, pa.concat_tables([oracle_op(partial, t.slice(0, n // 2)), oracle_op(partial, t.slice(n // 2))]))
    assert_same(gpu_op(final, pa.concat_tables(halves)), want)
