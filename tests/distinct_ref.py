"""TEST INFRASTRUCTURE.  DISTINCT aggregates for the numpy oracle (oracle/ops.py), which ignores an aggregate's "distinct" key.

`ref_op` evaluates an aggregate spec whose entries may carry `"distinct": true`: the group keys and the DISTINCT arguments are
evaluated by the oracle (a projection), pyarrow's hash aggregation gives each group's count of distinct non-null values and their
list, and sum / avg DISTINCT are the oracle's plain sum / avg over those lists (so their types and decimal rounding are the
oracle's).  The plain aggregates of the spec, min / max with the flag among them (a no-op, as in DataFusion), go to the oracle
as they are.  Every other spec goes to the oracle unchanged.
"""
import pyarrow as pa
import pyarrow.compute as pc

from oracle import ops


def oracle_op(spec, *tables):
    out = ops.run_op(spec, *[ops.batch_from_arrow(t) for t in tables])
    if isinstance(out, list):
        return [ops.batch_to_arrow(x) for x in out]
    return ops.batch_to_arrow(out)


def _gated(a):
    return bool(a.get("distinct")) and a["fn"] in ("count", "sum", "avg")


def _plain(a):
    return {k: v for k, v in a.items() if k != "distinct"}


def _for_pyarrow(c):
    return c.cast(pa.string()) if pa.types.is_string_view(c.type) else c


def ref_op(spec, *tables):
    if spec["op"] != "aggregate" or not any(_gated(a) for a in spec["aggs"]):
        return oracle_op({**spec, "aggs": [_plain(a) for a in spec["aggs"]]} if spec["op"] == "aggregate" else spec, *tables)
    assert spec.get("mode", "single") == "single"
    t = tables[0]
    n_keys = len(spec["group_by"])
    gated = [a for a in spec["aggs"] if _gated(a)]
    plain = oracle_op({**spec, "aggs": [_plain(a) for a in spec["aggs"] if not _gated(a)]}, t)
    keys_of = lambda tbl: list(zip(*[tbl.column(i).to_pylist() for i in range(n_keys)])) if n_keys else [()] * tbl.num_rows
    n_rows = plain.num_rows if n_keys else 1            # (a keyless aggregate without plain aggregates has no column to count)
    row_of = {k: i for i, k in enumerate(keys_of(plain))} if n_keys else {(): 0}
    # keys and every distinct argument, evaluated by the oracle; one more constant key so that a keyless aggregate groups too
    args = []
    for a in gated:
        if a["args"][0] not in args:
            args.append(a["args"][0])
    exprs = [{"expr": g["expr"], "name": f"k{i}"} for i, g in enumerate(spec["group_by"])] + [{"expr": x, "name": f"d{j}"} for j, x in enumerate(args)]
    proj = oracle_op({"op": "projection", "exprs": exprs}, t)
    base = [_for_pyarrow(proj.column(i)) for i in range(n_keys)] + [pa.array([0] * proj.num_rows, pa.int8())]
    key_names = [f"k{i}" for i in range(n_keys)] + ["__one"]
    results = {}
    for j, x in enumerate(args):
        d = proj.column(n_keys + j)
        tbl = pa.table(base + [_for_pyarrow(d)], names=key_names + ["d"])
        g = tbl.group_by(key_names, use_threads=False).aggregate([("d", "count_distinct", pc.CountOptions("only_valid")), ("d", "distinct", pc.CountOptions("only_valid"))])
        g = g.select(key_names + ["d_count_distinct", "d_distinct"])          # (pyarrow puts the aggregates first)
        counts = {k[:-1]: n for k, n in zip(zip(*[g.column(c).to_pylist() for c in key_names]), g.column("d_count_distinct").to_pylist())}
        lists = g.column("d_distinct")
        parents = pc.list_parent_indices(lists)
        flat = pc.list_flatten(lists)
        # the distinct values of every group, one row each, in the argument's own type: the input of the plain sum / avg
        dedup = pa.table([pc.take(g.column(i), parents) for i in range(n_keys)] + [flat.cast(d.type)], names=key_names[:-1] + ["d"])
        results[json_key(x)] = (counts, dedup)
    cols, fields = [], []
    for i in range(n_keys):
        cols.append(plain.column(i)); fields.append(plain.schema.field(i))
    for a in spec["aggs"]:
        if not _gated(a):
            cols.append(plain.column(a["name"])); fields.append(plain.schema.field(a["name"]))
            continue
        counts, dedup = results[json_key(a["args"][0])]
        if a["fn"] == "count":
            v = [0] * n_rows
            for k, n in counts.items():
                v[row_of[k]] = n
            cols.append(pa.array(v, pa.int64())); fields.append(pa.field(a["name"], pa.int64(), nullable=False))
            continue
        agg = oracle_op({"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": i}, "name": f"k{i}"} for i in range(n_keys)],
                         "aggs": [{"fn": a["fn"], "name": a["name"], "input_type": a.get("input_type"), "args": [{"col": n_keys}]}]}, dedup)
        v = [None] * n_rows
        for k, val in zip(keys_of(agg), agg.column(a["name"]).to_pylist()):
            v[row_of[k]] = val
        typ = agg.schema.field(a["name"]).type
        cols.append(pa.array(v, typ)); fields.append(pa.field(a["name"], typ))
    return pa.table(cols, schema=pa.schema(fields))


def json_key(x):
    import json
    return json.dumps(x, sort_keys=True)
