"""TEST INFRASTRUCTURE.  Timestamps for the numpy oracle (oracle/ops.py), restated independently of the library.

A Timestamp column is an oracle `Col` whose type is the spec string (`Timestamp(us, UTC)`) over int64 values.  `run_op` runs a spec
through the oracle after lowering what only timestamps have: every timestamp literal, cast, `date_part` and `date_trunc` is
evaluated here with numpy floor arithmetic (wall-clock time in the column's zone, the oracle's `civil_from_days` for the calendar)
and handed to the oracle as an extra column; aggregates and joins see timestamps as their Int64 values and get the type back on
their outputs.  Zones: none, UTC and fixed offsets `+HH:MM` / `-HH:MM`.
"""
import re

import numpy as np
import pyarrow as pa

from oracle import ops

UNITS = {"s": 1, "ms": 10 ** 3, "us": 10 ** 6, "ns": 10 ** 9}
UNIT_ORDER = ["s", "ms", "us", "ns"]
PARTS = ["year", "quarter", "month", "day", "hour", "minute", "second"]
TRUNC_PARTS = ["year", "quarter", "month", "week", "day", "hour", "minute", "second"]
_TS = re.compile(r"Timestamp\((s|ms|us|ns)(?:,\s*(.+))?\)")


def parse_ts(t):
    """(unit, zone) of a Timestamp type string, or None"""
    m = _TS.fullmatch(t) if isinstance(t, str) else None
    return (m.group(1), m.group(2) or "") if m else None


def ts_type(unit: str, tz: str = "") -> str:
    return f"Timestamp({unit}, {tz})" if tz else f"Timestamp({unit})"


def arrow_type(t: str):
    unit, tz = parse_ts(t)
    return pa.timestamp(unit, tz=tz or None)


def zone_seconds(tz: str) -> int:
    if tz in ("", "UTC"):
        return 0
    m = re.fullmatch(r"([+-])(\d\d):(\d\d)", tz)
    if not m:
        raise ValueError(f"zone {tz} needs a time-zone database")
    s = int(m.group(2)) * 3600 + int(m.group(3)) * 60
    return -s if m.group(1) == "-" else s


def _local(v, unit, tz):
    ups = UNITS[unit]
    local = np.asarray(v, dtype=np.int64) + np.int64(zone_seconds(tz) * ups)
    days = np.floor_divide(local, 86400 * ups)
    return ups, local, days, local - days * (86400 * ups)


def days_from_civil(y, m, d):
    y = np.where(m <= 2, y - 1, y).astype(np.int64)
    era = np.floor_divide(y, 400)
    yoe = y - era * 400
    doy = (153 * np.where(m > 2, m - 3, m + 9) + 2) // 5 + d - 1
    doe = yoe * 365 + yoe // 4 - yoe // 100 + doy
    return era * 146097 + doe - 719468


def date_part(v, part: str, unit: str, tz: str):
    """-> (result type, values): Int32 parts, second as the unscaled Decimal128(8,6) microsecond within the minute"""
    ups, local, days, tod = _local(v, unit, tz)
    if part == "second":
        r = tod % (60 * ups)
        us = r * (10 ** 6 // ups) if ups <= 10 ** 6 else r // (ups // 10 ** 6)
        return "Decimal128(8,6)", us
    if part == "hour":
        return "Int32", (tod // (3600 * ups)).astype(np.int32)
    if part == "minute":
        return "Int32", (tod // (60 * ups) % 60).astype(np.int32)
    y, m, d = ops.civil_from_days(days)
    out = {"year": y, "quarter": (m - 1) // 3 + 1, "month": m, "day": d}[part]
    return "Int32", np.asarray(out).astype(np.int32)


def date_trunc(v, part: str, unit: str, tz: str):
    ups, local, days, tod = _local(v, unit, tz)
    day = 86400 * ups
    if part in ("second", "minute", "hour"):
        t = local - tod % ({"second": 1, "minute": 60, "hour": 3600}[part] * ups)
    elif part == "day":
        t = days * day
    elif part == "week":                      # ISO weeks start on Monday; 1970-01-01 was a Thursday
        t = (days - np.mod(days + 3, 7)) * day
    else:
        y, m, _ = ops.civil_from_days(days)
        m = np.ones_like(m) if part == "year" else ((m - 1) // 3 * 3 + 1 if part == "quarter" else m)
        t = days_from_civil(y, m, np.ones_like(m)) * day
    return t - np.int64(zone_seconds(tz) * ups)


def cast_to_date(v, unit: str, tz: str):
    return _local(v, unit, tz)[2].astype(np.int32)


# ---- lowering onto the oracle ---------------------------------------------------------------------------------------------
def _obj(vals):
    a = np.empty(len(vals), dtype=object)
    for i, x in enumerate(vals):
        a[i] = int(x)
    return a


def _append(b: ops.Batch, c: ops.Col) -> dict:
    b.cols.append(c)
    b.names.append(f"__ts{len(b.cols)}")
    return {"col": len(b.cols) - 1}


def _eval(b, e) -> ops.Col:
    return ops.eval_expr(b, lower(b, e))


def _cast(x: ops.Col, to: str) -> ops.Col:
    f, t = parse_ts(x.type), parse_ts(to)
    if f and t:
        return ops.Col(to, np.asarray(x.data, np.int64) * np.int64(UNITS[t[0]] // UNITS[f[0]]), x.valid)
    if f and to == "Date32":
        return ops.Col("Date32", cast_to_date(x.data, *f), x.valid)
    assert (f and to == "Int64") or (t and x.type == "Int64"), (x.type, to)
    return ops.Col(to, np.asarray(x.data, np.int64), x.valid)


def lower(b: ops.Batch, e):
    """`e` with its timestamp-only nodes replaced by columns appended to `b`"""
    if isinstance(e, list):
        return [lower(b, x) for x in e]
    if not isinstance(e, dict):
        return e
    if "lit" in e and parse_ts(e.get("type")):
        n = b.num_rows
        if e["lit"] is None:
            return _append(b, ops.Col(e["type"], np.zeros(n, np.int64), np.zeros(n, bool)))
        return _append(b, ops.Col(e["type"], np.full(n, int(e["lit"]), np.int64)))
    if "in" in e:
        return {**e, "in": lower(b, e["in"]), "set": [{"lit": s["lit"], "type": "Int64"} if parse_ts(s["type"]) else s for s in e["set"]]}
    if "cast" in e:
        x = _eval(b, e["cast"])
        if parse_ts(x.type) or parse_ts(e["to"]):
            return _append(b, _cast(x, e["to"]))
    if e.get("fn") in ("date_part", "date_trunc"):
        x = _eval(b, e["args"][0])
        ts = parse_ts(x.type)
        if ts:
            part = e["part"].lower()
            if e["fn"] == "date_trunc":
                return _append(b, ops.Col(x.type, date_trunc(x.data, part, *ts), x.valid))
            t, v = date_part(x.data, part, *ts)
            return _append(b, ops.Col(t, _obj(v) if ops.is_decimal(t) else v, x.valid))
    return {k: lower(b, v) for k, v in e.items()}


def _as_int64(b: ops.Batch) -> ops.Batch:
    return ops.Batch(list(b.names), [ops.Col("Int64", c.data, c.valid) if parse_ts(c.type) else c for c in b.cols])


def _retype(b: ops.Batch, types) -> ops.Batch:
    return ops.Batch(list(b.names), [ops.Col(t, c.data, c.valid) if parse_ts(t) else c for c, t in zip(b.cols, types)])


def _aggregate(b: ops.Batch, spec: dict) -> ops.Batch:
    s = dict(spec)
    s["group_by"] = [{**g, "expr": lower(b, g["expr"])} for g in spec["group_by"]]
    s["aggs"] = [{**a, "args": lower(b, a["args"])} if a.get("args") else dict(a) for a in spec["aggs"]]
    types = [ops.eval_expr(b, g["expr"]).type for g in s["group_by"]]
    merging = spec["mode"] in ("final", "final_partitioned")
    for a in s["aggs"]:
        in_t = a.get("input_type") if merging else (ops.eval_expr(b, a["args"][0]).type if a.get("args") else None)
        assert not (parse_ts(in_t) and a["fn"] in ("sum", "avg")), "sum / avg over timestamps"
        n_out = 2 if a["fn"] == "avg" and spec["mode"] == "partial" else 1
        types += [in_t if a["fn"] in ("min", "max") else None] * n_out
        if parse_ts(a.get("input_type")):
            a["input_type"] = "Int64"
    return _retype(ops.op_aggregate(_as_int64(b), s), types)


def run_op(spec: dict, *inputs: ops.Batch):
    """oracle.ops.run_op for specs whose columns, literals or expressions may be timestamps"""
    bs = [ops.Batch(list(x.names), list(x.cols)) for x in inputs]
    width = [len(x.cols) for x in bs]
    kind = spec["op"]
    if kind == "aggregate":
        return _aggregate(bs[0], spec)
    if kind in ("hash_join", "nested_loop_join", "sort_preserving_merge"):
        assert spec.get("filter") is None, "join filters over timestamps are not restated here"
        types = [c.type for x in bs for c in x.cols]
        if spec.get("projection") is not None and kind != "sort_preserving_merge":
            types = [types[i] for i in spec["projection"]]
        if kind == "sort_preserving_merge":
            types = [c.type for c in bs[0].cols]
        out = ops.run_op(spec, *[_as_int64(x) for x in bs])
        if spec.get("join_type") in ("left_semi", "left_anti"):
            types = [c.type for c in bs[0].cols]
        elif spec.get("join_type") in ("right_semi", "right_anti"):
            types = [c.type for c in bs[1].cols]
        return _retype(out, types)
    b = bs[0]
    s = dict(spec)
    keep = list(range(width[0]))
    if kind == "filter":
        s["predicate"] = lower(b, spec["predicate"])
        s["projection"] = spec.get("projection") if spec.get("projection") is not None else keep
        return ops.op_filter(b, s)
    if kind == "projection":
        s["exprs"] = [{**it, "expr": lower(b, it["expr"])} for it in spec["exprs"]]
        return ops.op_projection(b, s)
    if kind == "sort":
        s["keys"] = [{**k, "expr": lower(b, k["expr"])} for k in spec["keys"]]
        return ops.op_sort(b, s).select(keep)
    if kind == "repartition":
        s["exprs"] = lower(b, spec.get("exprs", []))
        return [p.select(keep) for p in ops.op_repartition(b, s)]
    raise ValueError(kind)


# ---- arrow bridge ---------------------------------------------------------------------------------------------------------
def batch_from_arrow(tbl) -> ops.Batch:
    if isinstance(tbl, pa.RecordBatch):
        tbl = pa.Table.from_batches([tbl])
    types = [ts_type(f.type.unit, f.type.tz or "") if pa.types.is_timestamp(f.type) else None for f in tbl.schema]
    plain = pa.table([c.cast(pa.int64()) if t else c for c, t in zip(tbl.columns, types)], names=tbl.schema.names)
    b = ops.batch_from_arrow(plain)
    return _retype(b, types)


def batch_to_arrow(b: ops.Batch) -> pa.Table:
    cols = []
    for c in b.cols:
        if parse_ts(c.type):
            cols.append(ops.col_to_arrow(ops.Col("Int64", np.asarray(c.data, np.int64), c.valid)).cast(arrow_type(c.type)))
        else:
            cols.append(ops.col_to_arrow(c))
    return pa.table(cols, names=list(b.names))


def ref_op(spec, *tables):
    """tests.util.oracle_op with timestamps"""
    out = run_op(spec, *[batch_from_arrow(t) for t in tables])
    if isinstance(out, list):
        return [batch_to_arrow(x) for x in out]
    return batch_to_arrow(out)
