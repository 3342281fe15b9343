"""TEST INFRASTRUCTURE.  The variance family (stddev, stddev_pop, var, var_pop) for aggregate specs, in exact arithmetic.

`ref_op` evaluates an aggregate spec whose group keys are plain columns.  Its other aggregates go to the numpy oracle
(oracle/ops.py) as they are; every variance aggregate is computed here and put in its place.  Each argument value is first
converted to Float64 as the engine converts it (integers rounded once, Decimal128 as its unscaled value over 10^scale), then
every sum, mean and sum of squared deviations is a `fractions.Fraction` rounded once at the end:

- single: var_pop = m2 / n (n >= 1), var = m2 / (n - 1) (n >= 2), else NULL; stddev and stddev_pop are the square roots;
- partial: the state columns name[count] (UInt64), name[mean] and name[m2] (Float64); a group without values has 0, 0.0, 0.0;
- final / final_partitioned: the state rows of a group merged exactly: n = sum n_i, S = sum n_i mean_i,
  m2 = sum (m2_i + n_i mean_i^2) - S^2 / n.

A group with a NaN or an infinite value gives NaN (every output of the family, the partial mean and m2 included).
"""
import math
from fractions import Fraction

import pyarrow as pa

from oracle import ops

VARIANCE = ("stddev", "stddev_pop", "var", "var_pop")


def oracle_op(spec, *tables):
    return ops.batch_to_arrow(ops.run_op(spec, *[ops.batch_from_arrow(t) for t in tables]))


def as_float(v, t: pa.DataType):
    """the engine's conversion of one argument value to Float64"""
    if v is None:
        return None
    if pa.types.is_decimal(t):
        unscaled = int(v.scaleb(t.scale))
        return float(unscaled) / 10.0 ** t.scale if t.scale > 0 else float(unscaled)
    return float(v)


def moments(xs):
    """(n, mean, m2) of the non-null floats xs as exact Fractions; None for mean / m2 when a value is not finite"""
    xs = [x for x in xs if x is not None]
    if any(not math.isfinite(x) for x in xs):
        return len(xs), None, None
    if not xs:
        return 0, Fraction(0), Fraction(0)
    fx = [Fraction(x) for x in xs]
    s = sum(fx)
    mean = s / len(fx)
    return len(fx), mean, sum((x - mean) ** 2 for x in fx)


def merge_states(rows):
    """(n, mean, m2) of state rows [(count, mean, m2)] merged exactly"""
    n, s, q, bad = 0, Fraction(0), Fraction(0), False
    for c, mean, m2 in rows:
        n += c
        if not (math.isfinite(mean) and math.isfinite(m2)):
            bad = True
            continue
        s += c * Fraction(mean)
        q += Fraction(m2) + c * Fraction(mean) ** 2
    if bad:
        return n, None, None
    if n == 0:
        return 0, Fraction(0), Fraction(0)
    return n, s / n, q - s * s / n


def final_value(fn, n, m2):
    pop = fn.endswith("_pop")
    if n < (1 if pop else 2):
        return None
    if m2 is None:
        return math.nan
    v = m2 / (n if pop else n - 1)
    return math.sqrt(v) if fn.startswith("stddev") else float(v)


def _rounded(x):
    return math.nan if x is None else float(x)


def ref_op(spec, table: pa.Table) -> pa.Table:
    mode = spec.get("mode", "single")
    keys = [g["expr"]["col"] for g in spec["group_by"]]
    merging = mode in ("final", "final_partitioned")
    var_aggs = [a for a in spec["aggs"] if a["fn"] in VARIANCE]
    plain = [a for a in spec["aggs"] if a["fn"] not in VARIANCE]
    key_rows = list(zip(*[table.column(k).to_pylist() for k in keys])) if keys else [()] * table.num_rows
    order = list(dict.fromkeys(key_rows)) if keys else [()]

    # the oracle's output for the other aggregates, reordered into `order`
    cols = {}
    if merging:
        assert not plain, "final mode with aggregates other than the variance family"
        for i, k in enumerate(keys):
            cols[spec["group_by"][i]["name"]] = pa.array([o[i] for o in order], table.schema.field(k).type)
    elif plain or keys:
        base = oracle_op({**spec, "aggs": plain}, table)
        base_keys = list(zip(*[base.column(i).to_pylist() for i in range(len(keys))])) if keys else [()]
        pos = {k: i for i, k in enumerate(base_keys)}
        idx = pa.array([pos[k] for k in order], pa.int64())
        for name in base.schema.names:
            c = base.column(name)
            view = pa.types.is_string_view(c.type)           # (pyarrow's take has no string_view kernel)
            c = (c.cast(pa.string()) if view else c).take(idx)
            cols[name] = c.cast(pa.string_view()) if view else c

    # the variance aggregates: per group, the moments of its values (or its merged state rows)
    state_col = len(keys)
    for a in var_aggs:
        groups = {k: [] for k in order}
        if merging:
            c, m, q = (table.column(state_col + i).to_pylist() for i in range(3))
            for k, row in zip(key_rows, zip(c, m, q)):
                groups[k].append(row)
            state_col += 3
            mom = {k: merge_states(v) for k, v in groups.items()}
        else:
            col = a["args"][0]["col"]
            t = table.schema.field(col).type
            for k, v in zip(key_rows, table.column(col).to_pylist()):
                groups[k].append(as_float(v, t))
            mom = {k: moments(v) for k, v in groups.items()}
        if mode == "partial":
            cols[a["name"] + "[count]"] = pa.array([mom[k][0] for k in order], pa.uint64())
            cols[a["name"] + "[mean]"] = pa.array([_rounded(mom[k][1]) for k in order], pa.float64())
            cols[a["name"] + "[m2]"] = pa.array([_rounded(mom[k][2]) for k in order], pa.float64())
        else:
            cols[a["name"]] = pa.array([final_value(a["fn"], mom[k][0], mom[k][2]) for k in order], pa.float64())

    names = [g["name"] for g in spec["group_by"]]
    for a in spec["aggs"]:
        if mode == "partial" and a["fn"] in VARIANCE:
            names += [a["name"] + "[count]", a["name"] + "[mean]", a["name"] + "[m2]"]
        elif mode == "partial" and a["fn"] == "avg":
            names += [a["name"] + "[count]", a["name"] + "[sum]"]
        elif mode == "partial":
            names += [a["name"] + f"[{a['fn']}]"]
        else:
            names.append(a["name"])
    return pa.table([cols[n] for n in names], names=names)


def compare(got: pa.Table, want: pa.Table, n_keys: int, rel=1e-10):
    """rows matched on their keys; Float64 columns within `rel` relative (exact 0.0 and NaN must match exactly), others equal"""
    assert got.schema.names == want.schema.names, (got.schema.names, want.schema.names)
    assert [f.type for f in got.schema] == [f.type for f in want.schema], (got.schema, want.schema)
    assert got.num_rows == want.num_rows, (got.num_rows, want.num_rows)
    key = lambda t: list(zip(*[t.column(i).to_pylist() for i in range(n_keys)])) if n_keys else [()] * t.num_rows
    wrows = dict(zip(key(want), zip(*[c.to_pylist() for c in want.columns])))
    for k, row in zip(key(got), zip(*[c.to_pylist() for c in got.columns])):
        w = wrows[k]
        for name, x, y, f in zip(got.schema.names, row, w, got.schema):
            if pa.types.is_floating(f.type) and x is not None and y is not None:
                if math.isnan(y) or y == 0.0:
                    assert (math.isnan(x) if math.isnan(y) else x == 0.0), (name, k, x, y)
                else:
                    assert abs(x - y) <= rel * abs(y), (name, k, x, y, abs(x - y) / abs(y))
            else:
                assert x == y, (name, k, x, y)
