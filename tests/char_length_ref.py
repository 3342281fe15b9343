"""TEST INFRASTRUCTURE.  character_length for the numpy oracle (oracle/ops.py), restated independently of the library.

`run_op` runs a spec through the oracle after evaluating every `{"fn": "character_length", "args": [E]}` node here -- the code
points of each value of E as Int32, null where E is null -- and handing the result to the oracle as an extra column.  Outputs
that pass input columns through (filter, sort, repartition) drop the extra columns again.  `q27` is ClickBench [27] restated in
pandas from its SQL text, next to the other queries of tests/clickbench_sql.py.
"""
import numpy as np
import pandas as pd

from oracle import ops


def char_lengths(c: ops.Col) -> ops.Col:
    assert ops.is_string(c.type), c.type
    return ops.Col("Int32", np.array([len(v.decode()) for v in c.data], dtype=np.int32), c.valid)


def lower(b: ops.Batch, e):
    """`e` with its character_length nodes replaced by columns appended to `b`"""
    if isinstance(e, list):
        return [lower(b, x) for x in e]
    if not isinstance(e, dict):
        return e
    if e.get("fn") == "character_length":
        assert len(e["args"]) == 1
        b.cols.append(char_lengths(ops.eval_expr(b, lower(b, e["args"][0]))))
        b.names.append(f"__len{len(b.cols)}")
        return {"col": len(b.cols) - 1}
    return {k: lower(b, v) for k, v in e.items()}


def run_op(spec: dict, *inputs: ops.Batch):
    """oracle.ops.run_op for specs whose expressions may call character_length"""
    kind = spec["op"]
    if kind not in ("filter", "projection", "aggregate", "sort", "repartition"):
        return ops.run_op(spec, *inputs)
    b = ops.Batch(list(inputs[0].names), list(inputs[0].cols))
    keep = list(range(len(b.cols)))
    s = dict(spec)
    if kind == "filter":
        s["predicate"] = lower(b, spec["predicate"])
        s["projection"] = spec.get("projection") if spec.get("projection") is not None else keep
        return ops.op_filter(b, s)
    if kind == "projection":
        s["exprs"] = lower(b, spec["exprs"])
        return ops.op_projection(b, s)
    if kind == "aggregate":
        s["group_by"], s["aggs"] = lower(b, spec["group_by"]), lower(b, spec["aggs"])
        return ops.op_aggregate(b, s)
    if kind == "sort":
        s["keys"] = lower(b, spec["keys"])
        return ops.op_sort(b, s).select(keep)
    s["exprs"] = lower(b, spec.get("exprs", []))
    return [p.select(keep) for p in ops.op_repartition(b, s)]


def ref_op(spec, *tables):
    """tests.util.oracle_op with character_length"""
    out = run_op(spec, *[ops.batch_from_arrow(t) for t in tables])
    if isinstance(out, list):
        return [ops.batch_to_arrow(x) for x in out]
    return ops.batch_to_arrow(out)


def q27(h: pd.DataFrame, min_count: int) -> pd.DataFrame:
    """SELECT CounterID, AVG(length(URL)) AS l, COUNT(*) AS c FROM hits WHERE URL <> '' GROUP BY CounterID
    HAVING COUNT(*) > min_count ORDER BY l DESC -- without the LIMIT 25; `str.len` counts code points"""
    f = h[h.URL != ""]
    g = f.assign(n=f.URL.str.len()).groupby("CounterID", sort=False)
    out = pd.DataFrame({"l": g.n.mean().astype(np.float64), "c": g.size()}).reset_index()
    out = out[out.c > min_count]
    return out.sort_values("l", ascending=False, kind="stable").reset_index(drop=True)


def q27_min_count(h: pd.DataFrame, rank: int = 10) -> int:
    """a HAVING threshold that `rank` CounterID groups pass on a synthetic table: at the SQL's 100000 a small table returns nothing"""
    sizes = h[h.URL != ""].groupby("CounterID").size().sort_values(ascending=False)
    return int(sizes.iloc[min(rank, len(sizes)) - 1]) - 1
