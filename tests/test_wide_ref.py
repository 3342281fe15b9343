"""The wide-value reference (tests/wide_ref.py) against independent sources: Python's `decimal` at 100 digits for in-range decimal
arithmetic and cast rounding, pyarrow compute for the result types and values of `+ - *`, and numpy's own wrapping for Int64."""
import decimal
import random

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from tests import wide_ref as W

CTX = decimal.Context(prec=100, rounding=decimal.ROUND_DOWN, traps=[decimal.InvalidOperation, decimal.DivisionByZero])
TYPES = [W.dec(15, 2), W.dec(18, 0), W.dec(18, 6), W.dec(20, 4), W.dec(38, 2), W.dec(38, 10), W.dec(30, 0)]


def sample(t: str, rng: random.Random, n: int):
    """values of type t: the extremes of its precision, +-1, 0 and random magnitudes"""
    p, _ = W.parse_dec(t)
    top = 10 ** p - 1
    out = [0, 1, -1, top, -top, top // 7, -(top // 3)]
    out += [rng.randrange(-top, top + 1) // 10 ** rng.randrange(0, p) for _ in range(n)]
    return out


def as_decimal(v: int, t: str) -> decimal.Decimal:
    return decimal.Decimal(v).scaleb(-W.parse_dec(t)[1], CTX)


def unscaled(d: decimal.Decimal, s: int) -> int:
    return int(d.scaleb(s, CTX).to_integral_value(rounding=decimal.ROUND_DOWN, context=CTX))


@pytest.mark.parametrize("ta", TYPES)
@pytest.mark.parametrize("tb", TYPES)
@pytest.mark.parametrize("op", ["+", "-", "*", "/", "%"])
def test_decimal_arithmetic_matches_python_decimal(op, ta, tb):
    """in-range results equal exact decimal arithmetic at 100 digits (quotients truncated at the result scale); results that
    leave i128 are wrapped for + - * and errors for / %"""
    rng = random.Random(f"{op}{ta}{tb}")
    rt = W.result_type(op, ta, tb)
    _, s = W.parse_dec(rt)
    for a, b in zip(sample(ta, rng, 40), sample(tb, rng, 40)[::-1]):
        got = W.arith(op, a, ta, b, tb)
        x, y = as_decimal(a, ta), as_decimal(b, tb)
        if op in ("/", "%") and b == 0:
            assert got == W.ERR
            continue
        exact = {"+": CTX.add, "-": CTX.subtract, "*": CTX.multiply, "/": CTX.divide, "%": CTX.remainder}[op](x, y)
        want = unscaled(exact, s)
        if op in ("+", "-", "*"):
            assert got == W.wrap(want, 128), (a, b)
            continue
        # the operands as arrow-rs rescales them before dividing
        (_, s1), (_, s2) = W.parse_dec(ta), W.parse_dec(tb)
        if op == "/":
            k = s - s1 + s2
            x, y = (a * 10 ** k, b) if k >= 0 else (a, b * 10 ** -k)
        else:
            x, y = a * 10 ** (s - s1), b * 10 ** (s - s2)
        assert got == (want if W.fits(x, 128) and W.fits(y, 128) else W.ERR), (a, b)


def test_division_errors():
    assert W.arith("/", W.I64_MIN, "Int64", -1, "Int64") == W.ERR
    assert W.arith("%", W.I64_MIN, "Int64", -1, "Int64") == W.ERR
    assert W.arith("/", -2 ** 31, "Int32", -1, "Int32") == W.ERR
    assert W.arith("/", W.I64_MIN + 1, "Int64", -1, "Int64") == W.I64_MAX
    assert W.arith("%", W.I64_MIN, "Int64", 1, "Int64") == 0
    assert W.arith("/", 7, "Int64", 0, "Int64") == W.ERR
    assert W.arith("/", -7, "Int64", 2, "Int64") == -3 and W.arith("%", -7, "Int64", 2, "Int64") == -1
    assert W.arith("/", None, "Int64", 0, "Int64") is None
    # Decimal128(38,2) / Decimal128(38,10): the dividend is rescaled by 10^14 first
    big = 10 ** 30
    assert W.arith("/", big, W.dec(38, 2), 10 ** 10, W.dec(38, 10)) == W.ERR
    assert W.arith("/", 10 ** 20, W.dec(38, 2), 10 ** 10, W.dec(38, 10)) == 10 ** 24


@pytest.mark.parametrize("frm,to", [(W.dec(38, 10), W.dec(38, 2)), (W.dec(18, 6), W.dec(18, 2)), (W.dec(20, 3), W.dec(10, 0)),
                                    (W.dec(15, 2), W.dec(38, 12)), (W.dec(38, 4), "Int64"), (W.dec(18, 3), "Int64"), ("Int64", W.dec(38, 10))])
def test_casts_match_python_decimal(frm, to):
    """a rescale down rounds half away from zero (ROUND_HALF_UP in Python's decimal), ties and negative values included; a cast
    to an integer truncates"""
    rng = random.Random(frm + to)
    if frm == "Int64":
        vals = [0, 1, -1, W.I64_MAX, W.I64_MIN] + [rng.randrange(W.I64_MIN, W.I64_MAX) for _ in range(200)]
    else:
        _, s = W.parse_dec(frm)
        vals = sample(frm, rng, 200)
        vals += [sign * (m * 10 ** s + 5 * 10 ** (s - 1)) for sign in (1, -1) for m in (0, 1, 2, 12345) if s] + [10 ** s // 2 - 1, -(10 ** s // 2) + 1]
    for v in vals:
        got = W.cast(v, frm, to)
        if frm == "Int64":
            want = v * 10 ** W.parse_dec(to)[1]
        elif to == "Int64":
            want = unscaled(as_decimal(v, frm), 0)
        else:
            want = int(as_decimal(v, frm).quantize(decimal.Decimal(1).scaleb(-W.parse_dec(to)[1]), rounding=decimal.ROUND_HALF_UP, context=CTX).scaleb(W.parse_dec(to)[1], CTX))
        p = W.parse_dec(to)[0] if W.parse_dec(to) else None
        if (p is not None and abs(want) >= 10 ** p) or (to == "Int64" and not W.fits(want, 64)):
            assert got == W.ERR, v
        else:
            assert got == want, v
    assert W.cast(25, W.dec(10, 1), W.dec(10, 0)) == 3 and W.cast(-25, W.dec(10, 1), W.dec(10, 0)) == -3
    assert W.cast(-24, W.dec(10, 1), W.dec(10, 0)) == -2 and W.cast(-29, W.dec(10, 1), "Int64") == -2


@pytest.mark.parametrize("ta,tb", [(W.dec(15, 2), W.dec(16, 2)), (W.dec(18, 0), W.dec(18, 4)), (W.dec(20, 2), W.dec(17, 3)),
                                   (W.dec(12, 0), W.dec(25, 10)), (W.dec(30, 5), W.dec(7, 2))])
@pytest.mark.parametrize("op,fn", [("+", pc.add), ("-", pc.subtract), ("*", pc.multiply)])
def test_add_sub_mul_match_pyarrow(op, fn, ta, tb):
    """pyarrow's kernels agree with arrow-rs on + - * where the result precision stays within 38"""
    rt = W.result_type(op, ta, tb)
    rng = random.Random(op + ta + tb)
    pa_, pb_ = W.parse_dec(ta)[0], W.parse_dec(tb)[0]
    rp = W.parse_dec(rt)[0]
    a = [rng.randrange(-10 ** pa_ + 1, 10 ** pa_) for _ in range(300)] + [10 ** pa_ - 1, -(10 ** pa_ - 1), 0, None]
    b = [rng.randrange(-10 ** pb_ + 1, 10 ** pb_) for _ in range(300)] + [-(10 ** pb_ - 1), 10 ** pb_ - 1, 5, 7]
    got = fn(W.array(a, ta), W.array(b, tb))
    assert W.type_str(got.type) == rt
    want = [W.arith(op, x, ta, y, tb) for x, y in zip(a, b)]
    assert all(w is None or abs(w) < 10 ** rp for w in want)
    assert W.values(got) == want


@pytest.mark.parametrize("op", ["+", "-", "*"])
def test_int64_wraps_like_numpy(op):
    rng = np.random.default_rng(3)
    edge = np.array([0, 1, -1, 2 ** 55 - 1, 2 ** 55, -2 ** 55, W.I64_MAX, W.I64_MIN, 10 ** 18 - 1], dtype=np.int64)
    a = np.concatenate([edge, rng.integers(W.I64_MIN, W.I64_MAX, 500, dtype=np.int64, endpoint=True)])
    b = np.concatenate([edge[::-1], rng.integers(W.I64_MIN, W.I64_MAX, 500, dtype=np.int64, endpoint=True)])
    with np.errstate(over="ignore"):
        want = {"+": np.add, "-": np.subtract, "*": np.multiply}[op](a, b)
    assert [W.arith(op, int(x), "Int64", int(y), "Int64") for x, y in zip(a, b)] == want.tolist()


def test_aggregates():
    big = [W.I64_MAX, W.I64_MAX, 5, None]
    assert W.aggregate("sum", big, "Int64") == W.wrap(2 * W.I64_MAX + 5, 64)
    assert W.aggregate("count", big, "Int64") == 3
    assert W.aggregate("min", [W.I64_MIN, None, 3], "Int64") == W.I64_MIN
    assert W.aggregate("sum", [None], "Int64") is None and W.aggregate("count", [None], "Int64") == 0
    top = 10 ** 38 - 1
    assert W.aggregate("sum", [top, top], W.dec(38, 0)) == W.wrap(2 * top, 128)
    # avg(Decimal128(38,0)) -> Decimal128(38,4): sum * 10^4 must stay in i128
    assert W.aggregate("avg", [10 ** 30, 10 ** 30], W.dec(38, 0)) == 10 ** 34
    assert W.aggregate("avg", [top], W.dec(38, 0)) == W.ERR
    assert W.aggregate("avg", [-7, 0, 0], W.dec(10, 2)) == -23333          # -0.07 / 3 = -0.023333.. at scale 6: truncated
    assert W.agg_type("avg", W.dec(10, 2)) == W.dec(14, 6) and W.agg_type("sum", W.dec(30, 2)) == W.dec(38, 2)
    # avg equals the exact quotient truncated at the result scale
    vals = [12345, -99999, 7, 10 ** 17]
    exact = CTX.divide(sum(as_decimal(v, W.dec(18, 3)) for v in vals), decimal.Decimal(len(vals)))
    assert W.aggregate("avg", vals, W.dec(18, 3)) == unscaled(exact, 7)


def test_sort_indices_orders_exact_values():
    # -1 against 2^64: their low words order the other way round
    v = [2 ** 64, -1, None, 0, -(2 ** 64), 2 ** 64 + 1, -1]
    assert W.sort_indices([(v, True, True)]) == [2, 4, 1, 6, 3, 0, 5]
    assert W.sort_indices([(v, False, False)]) == [5, 0, 3, 1, 6, 4, 2]
    assert W.sort_indices([(v, True, False)]) == [4, 1, 6, 3, 0, 5, 2]


def test_arrow_round_trip_keeps_every_bit():
    vals = [0, 1, -1, W.I128_MAX, W.I128_MIN, 2 ** 64, -(2 ** 64), 2 ** 64 - 1, None, 10 ** 38 - 1, -(10 ** 38 - 1)]
    arr = W.array(vals, W.dec(38, 0))
    assert W.values(arr) == vals and W.values(arr.slice(3, 5)) == vals[3:8]
    in_range = [v for v in vals if v is None or abs(v) < 10 ** 38]
    assert W.values(pa.array([None if v is None else decimal.Decimal(v) for v in in_range], pa.decimal128(38, 0))) == in_range
    ints = [W.I64_MIN, W.I64_MAX, None, -1]
    assert W.values(W.array(ints, "Int64")) == ints
