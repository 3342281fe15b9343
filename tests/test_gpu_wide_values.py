"""GPU parity at the full width of the integer and decimal types, against the exact reference in tests/wide_ref.py.

Values sit on the boundaries where the kernels branch: the 2^55 limit of the aggregate's register and hot paths, the Int64 range,
the widest 18-digit decimal (the last one stored as one 64-bit word), the widest Decimal128(38), values that differ only in their
high word and values whose low words order opposite to their full values.  Projection, filter, aggregate and the overflow errors
run once in the interpreted pipeline kernel and once in the specialised (NVRTC) kernel; sort, TopK, hash join and hash
repartition run in their own kernels."""
import random

import numpy as np
import pyarrow as pa
import pytest

from tests import wide_ref as W
from tests.test_gpu_relational import pull_partition_to_host

pytestmark = pytest.mark.gpu

ERR_ARITHMETIC = 4     # sailgpu.h: SAILGPU_ERR_ARITHMETIC
D18, D17, D38 = W.dec(18, 2), W.dec(17, 0), W.dec(38, 4)


@pytest.fixture(params=["interpreted", "specialised"])
def kernel(request, monkeypatch):
    """interpreted: the tile VM with the specialiser off; specialised: the NVRTC kernel from the first row on, a kernel that
    fails to build being an error"""
    if request.param == "specialised":
        monkeypatch.delenv("SAILGPU_JIT", raising=False)
        monkeypatch.setenv("SAILGPU_JIT_MIN_ROWS", "0")
        monkeypatch.setenv("SAILGPU_JIT_STRICT", "1")
    else:
        monkeypatch.setenv("SAILGPU_JIT", "0")
    return request.param


# ---- values ------------------------------------------------------------------------------------------------------------
def edges(t: str):
    """the boundary values of type t that it can hold"""
    d = W.parse_dec(t)
    top = 10 ** d[0] - 1 if d else W.I64_MAX
    v = [0, 1, -1, 2 ** 55 - 1, -(2 ** 55 - 1), 2 ** 55, -(2 ** 55), W.I64_MAX, -W.I64_MAX, W.I64_MIN, 10 ** 18 - 1, -(10 ** 18 - 1),
         top, -top, 7, 7 + 2 ** 64, 7 - 2 ** 64, 2 ** 64, -(2 ** 64), 2 ** 64 - 1]
    lo, hi = (-top, top) if d else (W.I64_MIN, W.I64_MAX)
    return sorted({x for x in v if lo <= x <= hi})


def column(t: str, n: int, seed, nulls=False, limit=None):
    """n values of type t: every edge value, then random magnitudes over the whole width (or below `limit`); 5 % NULL if asked"""
    rng = random.Random(f"{t}/{seed}")
    d = W.parse_dec(t)
    top = min(10 ** d[0] - 1 if d else W.I64_MAX, limit or 1 << 200)
    ev = [x for x in edges(t) if abs(x) <= top]
    digits = len(str(top))
    out = [ev[i] if i < len(ev) else rng.randrange(-top, top + 1) // 10 ** rng.randrange(0, digits) for i in range(n)]
    rng.shuffle(out)
    if nulls:
        out = [None if rng.random() < 0.05 else x for x in out]
    return out


def table(**cols):
    """pa.table from name -> (values, type)"""
    return pa.table({k: W.array(v, t) for k, (v, t) in cols.items()})


def check(got: pa.Table, name: str, want, want_type: str):
    assert W.type_str(got.schema.field(name).type) == want_type, (name, got.schema.field(name).type, want_type)
    g = W.values(got.column(name))
    assert len(g) == len(want), (len(g), len(want))
    bad = [i for i, (a, b) in enumerate(zip(g, want)) if a != b]
    assert not bad, f"{name}: {len(bad)} rows differ, first at {bad[0]}: got {g[bad[0]]} want {want[bad[0]]}"


def run(spec, t, kernel_mode=None, batch=None):
    """the operator over t (in batches of `batch` rows), and whether the specialised kernel ran"""
    from sail_b200 import engine
    op = engine.GpuExec(spec, [t.schema])
    try:
        for o in range(0, max(t.num_rows, 1), batch or max(t.num_rows, 1)):
            op.push(t.slice(o, batch or t.num_rows))
        op.finish()
        out = op.collect()
        m = op.metrics()
    finally:
        op.close()
    if kernel_mode is not None:
        assert (m.get("gpu.jit_launches", 0) > 0) == (kernel_mode == "specialised"), m
    return out


def col(i):
    return {"col": i}


def binop(op, l, r):
    return {"op": op, "l": l, "r": r}


def project(exprs):
    return {"op": "projection", "exprs": [{"expr": e, "name": n} for n, e in exprs]}


# ---- projection and filter ---------------------------------------------------------------------------------------------
# (left type, right type): Int64; p <= 18 both sides (K_I64 and OP_MULW); one side wider than 18 digits in both operand orders
# (OP_MUL128_64, whose 64-bit side is negative half of the time); both wider (OP_MUL at 128 bits)
ARITH_TYPES = [("Int64", "Int64"), (W.dec(18, 2), W.dec(18, 0)), (W.dec(9, 2), W.dec(8, 3)), (W.dec(18, 4), W.dec(38, 2)),
               (W.dec(38, 2), W.dec(17, 1)), (W.dec(38, 0), W.dec(38, 10)), (W.dec(30, 5), W.dec(25, 0))]
N_SIZES = [255, 513, 5 * 256 + 7]


@pytest.mark.parametrize("n", N_SIZES)
@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("ta,tb", ARITH_TYPES)
def test_add_sub_mul_wrap_exactly(ta, tb, nulls, n, kernel):
    """+ - * bit-exact against the reference: wrapping mod 2^64 for Int64, mod 2^128 for decimals"""
    a, b = column(ta, n, 1, nulls), column(tb, n, 2, nulls)
    t = table(a=(a, ta), b=(b, tb))
    ops = ["+", "-", "*"]
    got = run(project([(f"r{i}", binop(op, col(0), col(1))) for i, op in enumerate(ops)]), t, kernel)
    for i, op in enumerate(ops):
        check(got, f"r{i}", [W.arith(op, x, ta, y, tb) for x, y in zip(a, b)], W.result_type(op, ta, tb))


# dividend / divisor types whose rescale stays inside i128 for every value, and (38,2) / (38,10) whose rescale by 10^14 is checked
DIV_TYPES = [("Int64", "Int64"), (W.dec(18, 2), W.dec(18, 6)), (W.dec(10, 2), W.dec(5, 2)), (W.dec(38, 10), W.dec(18, 2)),
             (W.dec(20, 0), W.dec(38, 4)), (W.dec(38, 2), W.dec(38, 10))]


@pytest.mark.parametrize("n", N_SIZES)
@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("ta,tb", DIV_TYPES)
def test_div_rem_truncate_exactly(ta, tb, nulls, n, kernel):
    """/ and % truncate toward zero at I64 and I128 (divisors of zero and MIN / -1 are left out: those are errors, below)"""
    limit = None
    if W.parse_dec(ta):       # a dividend whose rescale is checked (p1 + k > 38) stays below 10^(38 - k): the check passes
        (p1, s1), (_, s2) = W.parse_dec(ta), W.parse_dec(tb)
        k = max(W.parse_dec(W.result_type("/", ta, tb))[1] - s1 + s2, W.parse_dec(W.result_type("%", ta, tb))[1] - s1)
        limit = 10 ** (38 - k) - 1 if p1 + k > 38 else None
    a, b = column(ta, n, 3, nulls, limit=limit), column(tb, n, 4, nulls)
    b = [1 if y == 0 else y for y in b]
    a = [x + 1 if (x == W.I64_MIN and ta == "Int64") else x for x in a]
    t = table(a=(a, ta), b=(b, tb))
    got = run(project([("q", binop("/", col(0), col(1))), ("m", binop("%", col(0), col(1)))]), t, kernel)
    for name, op in (("q", "/"), ("m", "%")):
        want = [W.arith(op, x, ta, y, tb) for x, y in zip(a, b)]
        assert W.ERR not in want
        rt = W.result_type(op, ta, tb)
        rp = W.parse_dec(rt)
        if rp and rp[0] <= 18:       # stored in 64 bits: the quotient has to fit the result type
            assert all(w is None or abs(w) < 10 ** 18 for w in want), "test values leave the result type"
        check(got, name, want, rt)


CASTS = [(W.dec(38, 10), W.dec(38, 2)), (W.dec(18, 6), W.dec(18, 2)), (W.dec(15, 2), W.dec(38, 12)), (W.dec(18, 4), W.dec(38, 4)),
         (W.dec(22, 4), "Int64"), (W.dec(18, 3), "Int64"), ("Int64", W.dec(38, 10)), ("Int64", W.dec(20, 0)), (W.dec(38, 6), W.dec(30, 3))]


@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("frm,to", CASTS)
def test_casts(frm, to, nulls, kernel):
    """decimal -> decimal both ways (rescale down rounds half away from zero, at I64 and I128), decimal -> Int64 truncates,
    Int64 -> decimal; ties (x.5) in both signs are among the values"""
    n = 1031
    vals = column(frm, n, 5, nulls, limit=10 ** 33 if to == W.dec(30, 3) else None)
    d = W.parse_dec(frm)
    if d and d[1]:
        half = 5 * 10 ** (d[1] - 1)
        vals[:8] = [half, -half, 10 ** d[1] + half, -(10 ** d[1] + half), 3 * 10 ** d[1] - half, half - 1, -(half - 1), 0]
    t = table(a=(vals, frm))
    got = run(project([("c", {"cast": col(0), "to": to})]), t, kernel)
    want = [W.cast(v, frm, to) for v in vals]
    assert W.ERR not in want
    check(got, "c", want, to)


CMP_TYPES = [("Int64", "Int64"), (W.dec(18, 2), W.dec(38, 10)), (W.dec(20, 0), W.dec(17, 3)), (W.dec(38, 4), W.dec(38, 4)), (W.dec(18, 0), W.dec(18, 0))]


@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("ta,tb", CMP_TYPES)
def test_comparisons_and_filters(ta, tb, nulls, kernel):
    """comparisons between decimals of different precision and scale, as projected booleans and as filters"""
    n = 2 * 256 + 9
    a = column(ta, n, 6, nulls)
    b = column(tb, n, 7, nulls)
    for i in range(n // 3):                                          # equal values
        c = None if a[i] is None else W.cast(a[i], ta, tb)
        if c not in (None, W.ERR):
            b[i] = c
    if ta == tb and W.parse_dec(ta) and W.parse_dec(ta)[0] > 20:    # equal low words; low words ordered against the values
        a[n // 3: n // 3 + 4], b[n // 3: n // 3 + 4] = [7 + 2 ** 64, 7, 2 ** 64, -1], [7, 7 + 2 ** 64, -1, 2 ** 64]
    t = table(a=(a, ta), b=(b, tb), i=(list(range(n)), "Int64"))
    ops = ["=", "!=", "<", "<=", ">", ">="]
    got = run(project([(f"c{k}", binop(op, col(0), col(1))) for k, op in enumerate(ops)]), t, kernel)
    for k, op in enumerate(ops):
        want = [W.compare(op, x, ta, y, tb) for x, y in zip(a, b)]
        assert got.column(f"c{k}").to_pylist() == want, op
        kept = run({"op": "filter", "predicate": binop(op, col(0), col(1)), "projection": None}, t, kernel)
        assert W.values(kept.column("i")) == [i for i, w in enumerate(want) if w is True], op
        check(kept, "a", [a[i] for i, w in enumerate(want) if w is True], ta)


@pytest.mark.parametrize("nulls", [False, True])
def test_case_mixes_64_and_128_bit_branches(nulls, kernel):
    """CASE with a Decimal(18) branch and a Decimal(38) branch: the 64-bit branch is sign-extended into the 128-bit result"""
    n = 777
    a, b = column(W.dec(18, 2), n, 8, nulls), column(W.dec(38, 4), n, 9, nulls, limit=10 ** 35)
    t = table(a=(a, W.dec(18, 2)), b=(b, W.dec(38, 4)))
    zero = {"lit": "0", "type": W.dec(18, 2)}
    spec = project([("x", {"case": [[binop("<", col(0), zero), col(0)]], "else": col(1)}),
                    ("y", {"case": [[binop(">=", col(0), zero), col(1)]], "else": col(0)})])
    got = run(spec, t, kernel)
    rt = W.dec(38, 4)
    up = [W.cast(x, W.dec(18, 2), rt) for x in a]
    neg = [W.compare("<", x, W.dec(18, 2), 0, W.dec(18, 2)) for x in a]
    check(got, "x", [W.case([c], [u], y) for c, u, y in zip(neg, up, b)], rt)
    check(got, "y", [W.case([None if c is None else not c], [y], u) for c, u, y in zip(neg, up, b)], rt)


# ---- aggregates --------------------------------------------------------------------------------------------------------
def agg_spec(keys, aggs, mode="single"):
    """keys: column indices; aggs: (fn, column index or None, name)"""
    return {"op": "aggregate", "mode": mode, "group_by": [{"expr": col(k), "name": f"k{j}"} for j, k in enumerate(keys)],
            "aggs": [{"fn": fn, "args": [] if c is None else [col(c)], "name": name} for fn, c, name in aggs]}


def check_groups(got, key_types, aggs, want):
    """got: the aggregate's output (keys k0.., then the aggregates by name); want: {key tuple: [values]}"""
    keys = list(zip(*[W.values(got.column(f"k{j}")) for j in range(len(key_types))]))
    assert sorted(keys, key=repr) == sorted(want, key=repr), (len(keys), len(want))
    for j, t in enumerate(key_types):
        assert W.type_str(got.schema.field(f"k{j}").type) == t
    for a, (fn, t, name) in enumerate(aggs):
        vals = W.values(got.column(name))
        assert W.type_str(got.schema.field(name).type) == W.agg_type(fn, t), name
        bad = [(k, v, want[k][a]) for k, v in zip(keys, vals) if v != want[k][a]]
        assert not bad, f"{name}: {len(bad)} groups differ, e.g. key {bad[0][0]}: got {bad[0][1]} want {bad[0][2]}"


def agg_case(n, n_groups, nulls, seed, key_type="Int64"):
    """a table k, i64, d18, d17, d38 and a38: a Decimal(38,2) below 10^28 (avg's sum * 10^4 has to stay inside i128)"""
    rng = random.Random(seed)
    kv = edges(key_type)[:n_groups] if n_groups <= len(edges(key_type)) else None
    k = [kv[rng.randrange(len(kv))] for _ in range(n)] if kv else [rng.randrange(n_groups) * (2 ** 64 + 3) % (2 ** 62) - 2 ** 61 for _ in range(n)]
    cols = {"k": (k, key_type), "i64": (column("Int64", n, seed, nulls), "Int64"), "d18": (column(D18, n, seed, nulls), D18),
            "d17": (column(D17, n, seed, nulls), D17), "d38": (column(D38, n, seed, nulls), D38),
            "a38": (column(W.dec(38, 2), n, seed, nulls, limit=10 ** 28), W.dec(38, 2))}
    return table(**cols), cols


# every accumulator kind over every width (16 accumulators: the most one aggregate holds), then avg over three decimal widths
FULL_AGGS = [(fn, c) for c in ("i64", "d18", "d17", "d38") for fn in ("sum", "min", "max", "count")]
AVG_AGGS = [("avg", "d18"), ("avg", "d17"), ("avg", "a38"), ("count", None), ("sum", "a38")]
NAMES = ["k", "i64", "d18", "d17", "d38", "a38"]


def run_agg_case(t, cols, aggs, kernel, batch=None, key_type="Int64"):
    """aggs: (fn, column name or None for count(*)); grouped by column k"""
    spec = agg_spec([0], [(fn, None if c is None else NAMES.index(c), f"{fn}_{c}") for fn, c in aggs])
    got = run(spec, t, kernel, batch=batch)
    vals = [cols[c][0] for c in NAMES]
    ref = [(fn, 0, key_type) if c is None else (fn, NAMES.index(c), cols[c][1]) for fn, c in aggs]     # count(*): the never-null key
    want = W.group_by([vals[0]], vals, ref)
    for g in want.values():
        assert W.ERR not in g
    check_groups(got, [key_type], [(fn, "Int64" if c is None else cols[c][1], f"{fn}_{c}") for fn, c in aggs], want)


@pytest.mark.parametrize("col_", ["i64", "d17", "d18", "d38"])
@pytest.mark.parametrize("n", [513, 200_003])
def test_register_path_sum_before_count(col_, n, kernel):
    """the register fast path (at most 4 groups, non-null arguments, only sums and counts): a sum over values of 2^55 and more
    takes the path's rare branch straight to the table entry; the count behind it has to stay exact"""
    t, cols = agg_case(n, 4, False, 11)
    run_agg_case(t, cols, [("sum", col_), ("count", None)], kernel)


@pytest.mark.parametrize("col_", ["i64", "d17", "d38"])
def test_register_path_sum_as_last_accumulator(col_, kernel):
    """the wide sum as the entry's last accumulator: its rare branch must not write past its own words"""
    t, cols = agg_case(200_003, 4, False, 12)
    run_agg_case(t, cols, [("count", None), ("sum", "d18"), ("sum", col_)], kernel)


@pytest.mark.parametrize("no_regpath", [False, True])
@pytest.mark.parametrize("nulls", [False, True])
def test_hot_path_every_aggregate(nulls, no_regpath, kernel, monkeypatch):
    """few groups, every aggregate over Int64, Decimal(17), Decimal(18) and Decimal(38); with NULL arguments the hot path keeps
    seen bits; SAILGPU_NO_REGPATH is the A/B of the register path on the same input"""
    if no_regpath:
        monkeypatch.setenv("SAILGPU_NO_REGPATH", "1")
    t, cols = agg_case(100_003, 3, nulls, 13)
    run_agg_case(t, cols, FULL_AGGS, kernel)
    run_agg_case(t, cols, AVG_AGGS, kernel)


@pytest.mark.parametrize("mode", ["many_groups", "first_limit_0", "extreme_keys"])
def test_cold_path_every_aggregate(mode, kernel, monkeypatch):
    """the global table: many groups over several batches (the table grows while streaming), a forced hand-back after the first
    pass, and a never-null Int64 key with INT64_MIN, INT64_MAX and -1 among the keys"""
    if mode == "first_limit_0":
        monkeypatch.setenv("SAILGPU_AGG_FIRST_LIMIT", "0")
    t, cols = agg_case(60_007, 20_000, mode != "extreme_keys", 14)
    if mode == "extreme_keys":
        k = cols["k"][0]
        k[:3] = [W.I64_MIN, W.I64_MAX, -1]
        t = t.set_column(0, "k", W.array(k, "Int64"))
    run_agg_case(t, cols, FULL_AGGS, kernel, batch=16_411)
    run_agg_case(t, cols, AVG_AGGS, kernel, batch=16_411)


@pytest.mark.parametrize("n_groups", [4, 9, 3000])
def test_decimal38_group_keys_that_differ_in_the_high_word(n_groups, kernel):
    """Decimal(38) group keys 7, 7 + 2^64, 7 - 2^64, -1, 2^64 ...: equal low words, different groups"""
    rng = random.Random(n_groups)
    base = [7, 7 + 2 ** 64, 7 - 2 ** 64, -1, 2 ** 64 - 1, 2 ** 64, -(2 ** 64), 0, 10 ** 38 - 1]
    kv = base[:n_groups] if n_groups <= len(base) else base + [rng.randrange(-2 ** 100, 2 ** 100) for _ in range(n_groups - len(base))]
    n = 50_021
    k = [kv[rng.randrange(len(kv))] for _ in range(n)]
    t, cols = agg_case(n, 4, False, 15)
    cols["k"] = (k, W.dec(38, 0))
    t = t.set_column(0, "k", W.array(k, W.dec(38, 0)))
    run_agg_case(t, cols, [("sum", "i64"), ("count", None), ("sum", "d38"), ("max", "d38")], kernel, key_type=W.dec(38, 0))


def test_partial_final_merge_of_decimal38_states(kernel):
    """partial aggregates of two halves, merged by a final aggregate: sum / min / max / avg states of Decimal(38) and Int64"""
    t, cols = agg_case(40_009, 50, True, 16)
    aggs = [("sum", 4, "s38"), ("min", 4, "mn"), ("max", 4, "mx"), ("avg", 5, "av"), ("avg", 2, "a18"), ("sum", 1, "si"), ("count", None, "c")]
    partial = agg_spec([0], aggs, "partial")
    halves = [run(partial, t.slice(0, 17_000), kernel), run(partial, t.slice(17_000), kernel)]
    states = pa.concat_tables(halves)
    final = {"op": "aggregate", "mode": "final", "group_by": [{"expr": col(0), "name": "k0"}],
             "aggs": [{"fn": fn, "name": nm, "input_type": ("Int64" if c in (1, None) else cols[NAMES[c]][1])} for fn, c, nm in aggs]}
    got = run(final, states, kernel)
    vals = [cols[c][0] for c in NAMES]
    ref = [(fn, c if c is not None else 1, "Int64" if c is None else cols[NAMES[c]][1]) for fn, c, _ in aggs]
    want = W.group_by([vals[0]], vals, [(fn, c, tt) if fn != "count" else ("count", 0, "Int64") for fn, c, tt in ref])
    check_groups(got, ["Int64"], [(fn, tt, nm) for (fn, _, tt), (_, _, nm) in zip(ref, aggs)], want)


# ---- sort and TopK -----------------------------------------------------------------------------------------------------
def sort_table(n, seed):
    a = column("Int64", n, seed, True)
    d = column(W.dec(38, 0), n, seed + 1, True)
    rng = random.Random(seed)
    for i in range(0, n, 97):                                        # v and v + 2^64, -1 against 2^64, repeated
        d[i] = rng.choice([7, 7 + 2 ** 64, -1, 2 ** 64, -(2 ** 64), 10 ** 38 - 1])
    return a, d, table(a=(a, "Int64"), d=(d, W.dec(38, 0)), i=(list(range(n)), "Int64"))


@pytest.mark.parametrize("fetch", [None, 10, 1000])
@pytest.mark.parametrize("key", ["a", "d"])
@pytest.mark.parametrize("asc,nulls_first", [(True, True), (True, False), (False, True), (False, False)])
def test_sort_and_topk_over_the_full_range(key, asc, nulls_first, fetch, monkeypatch):
    """Int64 and Decimal(38) keys ascending and descending with both NULL placements; with a fetch the radix select of TopK
    (threshold lowered) decides on bytes of the high word"""
    from sail_b200 import engine
    monkeypatch.setenv("SAILGPU_TOPK_MIN_ROWS", "1000")
    n = 50_021
    a, d, t = sort_table(n, 21)
    kc = 0 if key == "a" else 1
    spec = {"op": "sort", "fetch": fetch, "keys": [{"expr": col(kc), "asc": asc, "nulls_first": nulls_first},
                                                   {"expr": col(2), "asc": True, "nulls_first": True}]}
    got = engine.run_op(spec, t)
    order = W.sort_indices([(a if key == "a" else d, asc, nulls_first), (list(range(n)), True, True)])[:fetch]
    assert W.values(got.column("i")) == order
    check(got, "d", [d[i] for i in order], W.dec(38, 0))


# ---- hash join ---------------------------------------------------------------------------------------------------------
def join_ref(build, probe, jt):
    """rows of build JOIN probe on column 0 (NULL matches nothing): inner = build ++ probe, left = inner + unmatched build rows
    with NULLs, left_semi / left_anti = build rows with / without a match"""
    out = []
    matched = [False] * len(build)
    for r in probe:
        for i, l in enumerate(build):
            if l[0] is not None and l[0] == r[0]:
                matched[i] = True
                if jt in ("inner", "left"):
                    out.append(tuple(l) + tuple(r))
    if jt == "left":
        out += [tuple(l) + (None,) * len(probe[0]) for l, m in zip(build, matched) if not m]
    if jt in ("left_semi", "left_anti"):
        out = [tuple(l) for l, m in zip(build, matched) if m == (jt == "left_semi")]
    return sorted(out, key=repr)


@pytest.mark.parametrize("jt", ["inner", "left", "left_semi", "left_anti"])
@pytest.mark.parametrize("dups", [False, True])
@pytest.mark.parametrize("kt", [W.dec(38, 0), W.dec(18, 2)])
def test_hash_join_on_wide_keys(kt, dups, jt):
    """Decimal(38) keys that differ only in the high word must not match; Decimal(18) keys (compared on their low 8 bytes) are
    mostly negative; unique and duplicate build keys"""
    from sail_b200 import engine
    rng = random.Random(f"{kt}{dups}")
    if W.parse_dec(kt)[0] > 18:
        base = [7, 7 + 2 ** 64, 7 - 2 ** 64, -1, 2 ** 64 - 1, 2 ** 64, -(2 ** 64), 10 ** 38 - 1, -(10 ** 38 - 1)]
        base += [rng.randrange(-10 ** 37, 10 ** 37) for _ in range(300)]
    else:
        base = [-1, -(10 ** 18 - 1), 10 ** 18 - 1, 1, 0, -(2 ** 55)] + [-rng.randrange(1, 10 ** 18) for _ in range(300)]
    bkeys = [base[rng.randrange(len(base))] for _ in range(700)] if dups else list(base)
    bkeys[:2] = [None, base[0]] if dups else [None, bkeys[1]]
    pkeys = [base[rng.randrange(len(base))] for _ in range(3000)] + [7 + 2 ** 65, None, -2]
    build = [(k, i) for i, k in enumerate(bkeys)]
    probe = [(k, 10_000 + i) for i, k in enumerate(pkeys)]
    lt = table(lk=(bkeys, kt), lv=(list(range(len(bkeys))), "Int64"))
    rt = table(rk=(pkeys, kt), rv=([10_000 + i for i in range(len(pkeys))], "Int64"))
    spec = {"op": "hash_join", "join_type": jt, "on": [[0, 0]], "filter": None, "projection": None}
    got = engine.run_op(spec, lt, rt)
    rows = sorted(zip(*[W.values(got.column(i)) for i in range(got.num_columns)]), key=repr)
    assert rows == join_ref(build, probe, jt)


# ---- hash repartition --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kt", ["Int64", W.dec(38, 0)])
@pytest.mark.parametrize("n_parts", [3, 8])
def test_hash_repartition_on_wide_keys(kt, n_parts):
    """every row comes out exactly once, and rows with equal keys share a partition"""
    from sail_b200 import engine
    n = 20_011
    k = column(kt, n, 31, True)
    rng = random.Random(32)
    for i in range(0, n, 13):
        k[i] = rng.choice([7, 7 + 2 ** 64, -1, 2 ** 64, W.I64_MIN]) if kt != "Int64" else rng.choice([W.I64_MIN, W.I64_MAX, -1, 0])
    t = table(k=(k, kt), i=(list(range(n)), "Int64"))
    op = engine.GpuExec({"op": "repartition", "scheme": "hash", "exprs": [col(0)], "n": n_parts}, [t.schema])
    op.push(t)
    op.finish()
    where = {}
    seen = []
    for p in range(n_parts):
        got = pull_partition_to_host(op, p, t.schema)
        for key, i in zip(W.values(got.column("k")), W.values(got.column("i"))):
            assert k[i] == key
            assert where.setdefault(repr(key), p) == p, f"key {key} in partitions {where[repr(key)]} and {p}"
            seen.append(i)
    op.close()
    assert sorted(seen) == list(range(n))


# ---- overflow errors ---------------------------------------------------------------------------------------------------
def raises_arithmetic(spec, t, kernel):
    from sail_b200 import engine
    with pytest.raises(engine.SailGpuError) as e:
        run(spec, t)
    assert e.value.code == ERR_ARITHMETIC, e.value


def int_column_with_hidden_value(vals, hidden, t="Int64"):
    """an Int column whose NULL rows hold `hidden` in their value slot"""
    data = np.array([hidden if v is None else v for v in vals], dtype=np.int64 if t == "Int64" else np.int32)
    valid = np.packbits(np.array([v is not None for v in vals]), bitorder="little").tobytes()
    return pa.Array.from_buffers(W.arrow_type(t), len(vals), [pa.py_buffer(valid), pa.py_buffer(data.tobytes())], null_count=sum(v is None for v in vals))


@pytest.mark.parametrize("op", ["/", "%"])
@pytest.mark.parametrize("t", ["Int64", "Int32"])
def test_integer_min_by_minus_one_is_an_overflow(t, op, kernel):
    mn = W.I64_MIN if t == "Int64" else -2 ** 31
    n = 1000
    at = 618                                                          # MIN / -1 in this row only
    a = [mn if i == at else i - 500 for i in range(n)]
    b = [-1 if i % 3 == 0 else 7 for i in range(n)]
    assert [W.arith(op, x, t, y, t) for x, y in zip(a, b)].count(W.ERR) == 1
    tab = table(a=(a, t), b=(b, t))
    spec = project([("q", binop(op, col(0), col(1)))])
    raises_arithmetic(spec, tab, kernel)
    # the same row with its divisor NULL (the value slot under the NULL holds -1), or removed by a fused filter, raises nothing
    nb = [None if i == at else y for i, y in enumerate(b)]
    tab2 = pa.table({"a": W.array(a, t), "b": int_column_with_hidden_value(nb, -1, t)})
    got = run(spec, tab2, kernel)
    check(got, "q", [W.arith(op, x, t, y, t) for x, y in zip(a, nb)], t)
    flt = {"op": "filter", "predicate": binop("!=", col(0), {"lit": str(mn), "type": t}), "projection": None}
    got = run({"op": "pipeline", "stages": [flt, spec]}, tab, kernel)
    check(got, "q", [W.arith(op, x, t, y, t) for x, y in zip(a, b) if x != mn], t)


@pytest.mark.parametrize("ta,tb,op", [(W.dec(38, 2), W.dec(38, 10), "/"), (W.dec(38, 0), W.dec(18, 10), "%")])
def test_decimal_rescale_that_leaves_i128_is_an_overflow(ta, tb, op, kernel):
    """the dividend rescaled by 10^(s_out - s1 + s2) (or to the common scale for %) leaves i128 for one large row"""
    n = 600
    a = [10 ** 20 + i for i in range(n)]
    a[333] = 10 ** 37
    b = [10 ** 10 + 7 * i for i in range(n)]
    assert W.arith(op, a[333], ta, b[333], tb) == W.ERR and all(W.arith(op, x, ta, y, tb) != W.ERR for x, y in zip(a[:333], b))
    spec = project([("q", binop(op, col(0), col(1)))])
    raises_arithmetic(spec, table(a=(a, ta), b=(b, tb)), kernel)
    nb = [None if i == 333 else y for i, y in enumerate(b)]
    t2 = table(a=(a, ta), b=(nb, tb))
    check(run(spec, t2, kernel), "q", [W.arith(op, x, ta, y, tb) for x, y in zip(a, nb)], W.result_type(op, ta, tb))
    flt = {"op": "filter", "predicate": binop("<", col(0), {"lit": str(10 ** 30), "type": ta}), "projection": None}
    got = run({"op": "pipeline", "stages": [flt, spec]}, table(a=(a, ta), b=(b, tb)), kernel)
    check(got, "q", [W.arith(op, x, ta, y, tb) for x, y in zip(a, b) if x < 10 ** 30], W.result_type(op, ta, tb))


def test_avg_decimal_that_leaves_i128_is_an_overflow(kernel):
    """avg(Decimal128(38,0)) -> Decimal128(38,4): sum * 10^4 leaves i128 in one group"""
    n = 3000
    k = [i % 3 for i in range(n)]
    v = [(10 ** 37 if i == 1 else i) for i in range(n)]
    t = table(k=(k, "Int64"), v=(v, W.dec(38, 0)))
    spec = agg_spec([0], [("avg", 1, "a")])
    raises_arithmetic(spec, t, kernel)
    ok = t.filter(pa.array([x != 1 for x in k]))
    got = run(spec, ok, kernel)
    want = W.group_by([[x for x in k if x != 1]], [None, [y for x, y in zip(k, v) if x != 1]], [("avg", 1, W.dec(38, 0))])
    check_groups(got, ["Int64"], [("avg", W.dec(38, 0), "a")], want)
