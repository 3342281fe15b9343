"""TEST INFRASTRUCTURE.  An exact reference for integers and decimals at the full width of their types.

The numpy oracle (oracle/ops.py) keeps Int64 values in numpy and raises where a sum or a quotient wraps, and it does not model the
i128 rescale of a decimal division.  This module restates the operations the GPU path computes on Int32 / Int64 / Decimal128 with
Python integers, with every wrap and every error stated explicitly (DataFusion 53 / arrow-rs 58 with the default
`fail_on_overflow = false`):

- `+ - *` wrap: Int32 / Int64 mod 2^32 / 2^64, Decimal128 mod 2^128 at the arrow-arith result type (SURVEY.md, Appendix A).
- `/ %` are checked: division by zero, `MIN / -1`, `MIN % -1` and a decimal rescale whose product leaves i128 are errors
  (`ERR`); otherwise the quotient truncates toward zero and the remainder takes the dividend's sign.
- Decimal casts: a rescale down rounds half away from zero; a cast to an integer truncates toward zero.  A value that does not fit
  the target (precision or integer range) is an error, as arrow's cast reports it.
- Aggregates: `sum` wraps (Int64 mod 2^64, decimals mod 2^128), `min` / `max` are exact, `count` counts non-null values and
  `avg(Decimal)` is `(sum * 10^(s_out - s_in)) // count` truncating toward zero, an error when that product leaves i128.
- Ordering: Python comparison of the exact values, per-key `asc` and `nulls_first`, stable.

Values are unscaled Python ints (None = NULL); types are the spec strings (`Int64`, `Decimal128(38,10)`).
"""
import functools
import re

import numpy as np
import pyarrow as pa

ERR = "ERR"     # the error marker: the operation raises ArithmeticOverflow / DivideByZero for this row
I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1
I128_MIN, I128_MAX = -2 ** 127, 2 ** 127 - 1
INT_BITS = {"Int32": 32, "Int64": 64}
_DEC = re.compile(r"Decimal128\((\d+),\s*(\d+)\)")


def dec(p: int, s: int) -> str:
    return f"Decimal128({p},{s})"


def parse_dec(t: str):
    """(precision, scale) of a Decimal128 type string, or None"""
    m = _DEC.fullmatch(t)
    return (int(m.group(1)), int(m.group(2))) if m else None


def wrap(v: int, bits: int) -> int:
    """two's-complement wrap of v to `bits` bits"""
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def fits(v: int, bits: int) -> bool:
    return -(1 << (bits - 1)) <= v < (1 << (bits - 1))


def trunc_div(a: int, b: int) -> int:
    """a / b truncating toward zero (Python's // floors)"""
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def trunc_rem(a: int, b: int) -> int:
    return a - b * trunc_div(a, b)


# ---- types -------------------------------------------------------------------------------------------------------------
def result_type(op: str, ta: str, tb: str) -> str:
    """arrow-arith result type of `ta op tb`; integer operands of one type keep it"""
    da, db = parse_dec(ta), parse_dec(tb)
    if da is None and db is None:
        assert ta == tb, (ta, tb)
        return ta
    (p1, s1), (p2, s2) = da, db
    if op in ("+", "-"):
        s = max(s1, s2)
        return dec(min(38, max(p1 - s1, p2 - s2) + s + 1), s)
    if op == "*":
        return dec(min(38, p1 + p2 + 1), s1 + s2)
    if op == "/":
        s = min(38, s1 + 4)
        return dec(min(38, p1 - s1 + s2 + s), s)
    if op == "%":
        s = max(s1, s2)
        return dec(min(38, min(p1 - s1, p2 - s2) + s), s)
    raise ValueError(op)


def compare_type(ta: str, tb: str) -> str:
    """the common decimal type two decimals are compared at: the wider scale and the wider integer-digit count"""
    (p1, s1), (p2, s2) = parse_dec(ta), parse_dec(tb)
    s = max(s1, s2)
    return dec(min(38, max(p1 - s1, p2 - s2) + s), s)


# ---- scalar operations -------------------------------------------------------------------------------------------------
def arith(op: str, a, ta: str, b, tb: str):
    """`a op b` for operands of types ta / tb (unscaled ints or None): an int, None (NULL) or ERR"""
    if a is None or b is None:
        return None
    if ta in INT_BITS:
        bits = INT_BITS[ta]
        if op in ("+", "-", "*"):
            return wrap(a + b if op == "+" else a - b if op == "-" else a * b, bits)
        if b == 0 or (b == -1 and a == -(1 << (bits - 1))):
            return ERR
        return trunc_div(a, b) if op == "/" else trunc_rem(a, b)
    (_, s1), (_, s2) = parse_dec(ta), parse_dec(tb)
    _, s = parse_dec(result_type(op, ta, tb))
    if op in ("+", "-"):
        x, y = a * 10 ** (s - s1), b * 10 ** (s - s2)
        return wrap(x + y if op == "+" else x - y, 128)
    if op == "*":
        return wrap(a * b, 128)
    if op == "/":
        k = s - s1 + s2
        x, y = (a * 10 ** k, b) if k >= 0 else (a, b * 10 ** -k)
    else:
        x, y = a * 10 ** (s - s1), b * 10 ** (s - s2)
    if not fits(x, 128) or not fits(y, 128) or y == 0:        # arrow-rs: mul_checked, then div_checked / mod_checked
        return ERR
    q = trunc_div(x, y) if op == "/" else trunc_rem(x, y)
    return q if fits(q, 128) else ERR


def compare(op: str, a, ta: str, b, tb: str):
    """comparison of two decimals (or two integers) of possibly different types: True / False / None"""
    if a is None or b is None:
        return None
    if parse_dec(ta):
        (_, s1), (_, s2) = parse_dec(ta), parse_dec(tb)
        s = max(s1, s2)
        a, b = a * 10 ** (s - s1), b * 10 ** (s - s2)
    return {"=": a == b, "!=": a != b, "<": a < b, "<=": a <= b, ">": a > b, ">=": a >= b}[op]


def cast(v, frm: str, to: str):
    """cast between Int32 / Int64 / Decimal128 types: an int, None or ERR"""
    if v is None:
        return None
    df, dt = parse_dec(frm), parse_dec(to)
    if df and dt:
        (_, s1), (p2, s2) = df, dt
        if s2 >= s1:
            r = v * 10 ** (s2 - s1)
        else:
            d = 10 ** (s1 - s2)
            r = trunc_div(v, d)
            if 2 * abs(v - r * d) >= d:          # half away from zero
                r += 1 if v > 0 else -1
        return r if abs(r) < 10 ** p2 else ERR
    if df:                                      # decimal -> integer: truncate toward zero
        r = trunc_div(v, 10 ** df[1])
        return r if fits(r, INT_BITS[to]) else ERR
    if dt:                                      # integer -> decimal
        r = v * 10 ** dt[1]
        return r if abs(r) < 10 ** dt[0] else ERR
    return v if fits(v, INT_BITS[to]) else ERR


def case(conds, thens, otherwise):
    """CASE WHEN conds[0] THEN thens[0] ... ELSE otherwise, row values already brought to the result type"""
    for c, t in zip(conds, thens):
        if c is True:
            return t
    return otherwise


# ---- aggregates --------------------------------------------------------------------------------------------------------
def agg_type(fn: str, t: str) -> str:
    d = parse_dec(t)
    if fn == "count":
        return "Int64"
    if fn in ("min", "max"):
        return t
    if fn == "sum":
        return dec(min(38, d[0] + 10), d[1]) if d else "Int64"
    if fn == "avg":
        assert d, "avg(Int) is Float64: not restated here"
        return dec(min(38, d[0] + 4), min(38, d[1] + 4))
    raise ValueError(fn)


def aggregate(fn: str, values, t: str):
    """one group's aggregate over `values` of type t"""
    vals = [v for v in values if v is not None]
    if fn == "count":
        return len(vals)
    if not vals:
        return None
    if fn == "min":
        return min(vals)
    if fn == "max":
        return max(vals)
    total = wrap(sum(vals), 128 if parse_dec(t) else 64)
    if fn == "sum":
        return total
    _, s = parse_dec(t)
    x = total * 10 ** (parse_dec(agg_type("avg", t))[1] - s)
    return trunc_div(x, len(vals)) if fits(x, 128) else ERR


def group_by(keys, cols, aggs):
    """{key tuple: [aggregate per (fn, column index, type)]} over rows; NULL keys group together"""
    groups = {}
    for i, k in enumerate(zip(*keys)):
        groups.setdefault(k, []).append(i)
    return {k: [aggregate(fn, [cols[c][i] for i in rows], t) for fn, c, t in aggs] for k, rows in groups.items()}


# ---- ordering ----------------------------------------------------------------------------------------------------------
def sort_indices(keys):
    """stable ORDER BY over `keys` = [(values, asc, nulls_first)]: the row indices in output order"""
    n = len(keys[0][0]) if keys else 0

    def cmp(i, j):
        for vals, asc, nulls_first in keys:
            a, b = vals[i], vals[j]
            if a is None or b is None:
                if a is None and b is None:
                    continue
                return (-1 if a is None else 1) * (1 if nulls_first else -1)
            if a != b:
                return (-1 if a < b else 1) * (1 if asc else -1)
        return 0
    return sorted(range(n), key=functools.cmp_to_key(cmp))


# ---- Arrow columns <-> exact values ------------------------------------------------------------------------------------
def type_str(t: pa.DataType) -> str:
    if pa.types.is_decimal(t):
        return dec(t.precision, t.scale)
    return {pa.int32(): "Int32", pa.int64(): "Int64"}[t]


def arrow_type(t: str) -> pa.DataType:
    d = parse_dec(t)
    return pa.decimal128(*d) if d else {"Int32": pa.int32(), "Int64": pa.int64()}[t]


def values(arr) -> list:
    """unscaled Python ints (None for NULL) of an Int32 / Int64 / Decimal128 column, read from its buffers"""
    if isinstance(arr, pa.ChunkedArray):
        return [v for c in arr.chunks for v in values(c)]
    valid = arr.is_valid().to_numpy(zero_copy_only=False)
    if pa.types.is_decimal(arr.type):
        w = np.frombuffer(arr.buffers()[1], dtype="<u8")[2 * arr.offset: 2 * (arr.offset + len(arr))].reshape(-1, 2)
        out = [wrap(int(lo) | (int(hi) << 64), 128) for lo, hi in w]
    else:
        out = arr.to_numpy(zero_copy_only=False).tolist() if arr.null_count == 0 else arr.fill_null(0).to_numpy().tolist()
    return [int(v) if ok else None for v, ok in zip(out, valid)]


def array(vals, t: str) -> pa.Array:
    """an Arrow column of type t from unscaled ints / None (decimals are written as their 16 little-endian bytes, unchecked)"""
    d = parse_dec(t)
    mask = np.array([v is None for v in vals], dtype=bool)
    if not d:
        return pa.array(np.array([0 if v is None else v for v in vals], dtype=np.int64 if t == "Int64" else np.int32),
                        mask=mask if mask.any() else None)
    data = b"".join(((0 if v is None else v) & ((1 << 128) - 1)).to_bytes(16, "little") for v in vals)
    validity = pa.py_buffer(np.packbits(~mask, bitorder="little").tobytes()) if mask.any() else None
    return pa.Array.from_buffers(pa.decimal128(*d), len(vals), [validity, pa.py_buffer(data)], null_count=int(mask.sum()))
