"""The variance family on the GPU: stddev, stddev_pop, var and var_pop against the exact reference of tests/variance_ref.py, in
the interpreted and the specialised pipeline kernel, in modes single, partial -> final and partial -> final_partitioned, on
every path of the hash aggregate (no key, a few groups held in the CTA dictionary, many groups in the global table, a key too
wide for the table that goes to the sort-based WideAggOp, and partitioned mode under a lowered slot ceiling), over groups of
0, 1 and 2 values, all-null groups, constant groups, NaN and infinities, every argument type, data with mean 1e8 and standard
deviation 1, and a describe()-shaped aggregate over TPC-H lineitem."""
import decimal
import math

import numpy as np
import pyarrow as pa
import pytest

from tests import variance_ref as ref

pytestmark = pytest.mark.gpu

FNS = ["stddev", "stddev_pop", "var", "var_pop"]


@pytest.fixture(params=["interpreted", "specialised"])
def kernel(request, monkeypatch):
    if request.param == "interpreted":
        monkeypatch.setenv("SAILGPU_JIT", "0")
    else:
        monkeypatch.setenv("SAILGPU_JIT", "1")
        monkeypatch.setenv("SAILGPU_JIT_MIN_ROWS", "0")
    return request.param


def run(spec, batches):
    from sail_b200 import engine
    op = engine.GpuExec(spec, [batches[0].schema])
    try:
        for t in batches:
            op.push(t)
        op.finish()
        return op.collect(), op.metrics()
    finally:
        op.close()


def batches_of(t: pa.Table, n):
    step = max(1, -(-t.num_rows // n))
    return [t.slice(i, step) for i in range(0, t.num_rows, step)]


def agg(aggs, keys, mode="single"):
    return {"op": "aggregate", "mode": mode, "group_by": [{"expr": {"col": k}, "name": f"k{k}"} for k in keys], "aggs": aggs}


def var_aggs(col, mode="single", extra=()):
    out = [{"fn": fn, "name": fn, "args": [{"col": col}]} for fn in FNS]
    return out + list(extra)


def final_aggs(input_type):
    return [{"fn": fn, "name": fn, "input_type": input_type} for fn in FNS]


def check_all_modes(t: pa.Table, keys, col, kernel, n_batches=3, rel=1e-10, check_jit=True):
    """single, partial and partial -> final / final_partitioned; returns the metrics of the single-mode run"""
    parts = batches_of(t, n_batches)
    spec = agg(var_aggs(col), keys)
    got, m = run(spec, parts)
    ref.compare(got, ref.ref_op(spec, t), len(keys), rel)
    if check_jit and keys and len(keys) <= 6:
        assert (m.get("gpu.jit_launches", 0) > 0) == (kernel == "specialised"), m
    # partial: the state columns; each batch its own partial operator, as DataFusion runs one per input partition
    pspec = agg(var_aggs(col), keys, mode="partial")
    states = []
    for p in parts:
        s, _ = run(pspec, [p])
        ref.compare(s, ref.ref_op(pspec, p), len(keys), rel)
        states.append(s)
    st = pa.concat_tables(states)
    n_keys = len(keys)
    # final modes over the state rows: four aggregates, each reading its own (count, mean, m2) triple
    for mode in ("final", "final_partitioned"):
        fspec = agg(final_aggs("Float64"), list(range(n_keys)), mode=mode)
        fgot, _ = run(fspec, batches_of(st, 2))
        ref.compare(fgot, ref.ref_op(fspec, st), n_keys, rel)
    return m


# ---- paths ------------------------------------------------------------------------------------------------

def data(n, n_groups, seed=1, nulls=0.1, n_keys=1):
    rng = np.random.default_rng(seed)
    x = rng.normal(50.0, 20.0, n)
    cols = [pa.array(rng.integers(0, n_groups, n).astype(np.int32) * (i + 1)) for i in range(n_keys)]
    return pa.table(cols + [pa.array(x, mask=rng.random(n) < nulls)], names=[f"k{i}" for i in range(n_keys)] + ["x"])


def test_keyless(kernel):
    t = data(100_000, 1)
    check_all_modes(t.select(["x"]), [], 0, kernel)


def test_few_groups_hot_path(kernel):
    check_all_modes(data(300_000, 4), [0], 1, kernel)


def test_many_groups_cold_path(kernel):
    check_all_modes(data(150_000, 30_000), [0], 1, kernel)


def test_wide_key_goes_to_the_sort_based_aggregate(kernel):
    t = data(60_000, 50, n_keys=7)
    spec = agg(var_aggs(7), list(range(7)))
    got, m = run(spec, batches_of(t, 2))
    ref.compare(got, ref.ref_op(spec, t), 7)
    pspec = agg(var_aggs(7), list(range(7)), mode="partial")
    s, _ = run(pspec, [t])
    ref.compare(s, ref.ref_op(pspec, t), 7)
    fspec = agg(final_aggs("Float64"), list(range(7)), mode="final")
    f, _ = run(fspec, [s])
    ref.compare(f, ref.ref_op(fspec, s), 7)


def sized(t: pa.Table, sizes):
    out, at = [], 0
    for n in sizes:
        out.append(t.slice(at, n))
        at += n
    return [b for b in out if b.num_rows]


def test_partitioned_mode(kernel, monkeypatch):
    """a table of 2^17 slots: a batch of 50 K rows of mostly new groups in the middle of the stream overflows it"""
    monkeypatch.setenv("SAILGPU_AGG_MAX_CAPACITY", str(1 << 17))
    t = data(110_000, 1_000_000)
    spec = agg(var_aggs(1, extra=[{"fn": "count", "name": "c", "args": [{"col": 1}]}]), [0])
    got, m = run(spec, sized(t, [20_000, 20_000, 50_000, 20_000]))
    assert m["gpu.agg_spills"] >= 1 and m["gpu.agg_partitions"] >= 2, m
    ref.compare(got, ref.ref_op(spec, t), 1)
    # a final aggregate in partitioned mode spills and re-merges the three state columns
    s, _ = run(agg(var_aggs(1), [0], mode="partial"), [t])
    fspec = agg(final_aggs("Float64"), [0], mode="final_partitioned")
    f, fm = run(fspec, sized(s, [20_000, 20_000, 50_000, 20_000]))
    assert fm["gpu.agg_spills"] >= 1, fm
    ref.compare(f, ref.ref_op(fspec, s), 1)


# ---- edge groups ------------------------------------------------------------------------------------------

def edge_table():
    groups = {
        0: [],                                     # no rows at all is not a group; kept for the layout below
        1: [3.25],                                 # n = 1: var NULL, var_pop 0
        2: [1.0, 4.0],                             # n = 2
        3: [None, None, None],                     # all null: everything NULL
        4: [0.1] * 1000,                           # constant: exactly 0
        5: [-7.0] * 3 + [None],
        6: [1.0, float("nan"), 2.0],               # NaN
        7: [1.0, float("inf")],                    # +inf
        8: [float("-inf")],                        # a single -inf
        9: [5.0, None],                            # n = 1 after nulls
        10: [1e8 + 0.5, 1e8 - 0.5] * 50,
    }
    k, x = [], []
    for g, xs in groups.items():
        k += [g] * len(xs)
        x += xs
    return pa.table({"k": pa.array(k, pa.int32()), "x": pa.array(x, pa.float64())})


def test_edge_groups(kernel):
    t = edge_table()
    check_all_modes(t, [0], 1, kernel, n_batches=1)
    got, _ = run(agg(var_aggs(1), [0]), [t])
    rows = {r["k0"]: r for r in got.to_pylist()}
    assert rows[1]["var"] is None and rows[1]["var_pop"] == 0.0 and rows[1]["stddev_pop"] == 0.0
    assert rows[3]["var_pop"] is None and rows[3]["stddev"] is None
    assert all(rows[4][f] == 0.0 for f in FNS) and all(rows[5][f] == 0.0 for f in FNS)
    assert all(math.isnan(rows[6][f]) for f in FNS) and all(math.isnan(rows[7][f]) for f in FNS)
    # one non-finite value: NaN (DataFusion's ungrouped accumulator reports 0.0 here; sailgpu.h documents the difference)
    assert math.isnan(rows[8]["var_pop"]) and rows[8]["var"] is None


def test_keyless_over_no_rows(kernel):
    t = pa.table({"x": pa.array([], pa.float64())})
    got, _ = run(agg(var_aggs(0), []), [pa.table({"x": pa.array([1.0])}).slice(0, 0)])
    assert got.to_pylist() == [{f: None for f in FNS}]
    s, _ = run(agg(var_aggs(0), [], mode="partial"), [t])
    assert s.to_pylist()[0]["stddev[count]"] == 0 and s.to_pylist()[0]["stddev[m2]"] == 0.0


# ---- argument types ---------------------------------------------------------------------------------------

def typed(kind, rng, n):
    v = rng.integers(-100, 100, n)
    if kind == "int8":
        return pa.array(v.astype(np.int8))
    if kind == "int64":
        return pa.array(v.astype(np.int64) * 1_000_000_007 + 2**61)
    if kind == "uint64":
        return pa.array((v + 100).astype(np.uint64) * np.uint64(3_000_000_000_000_017) + np.uint64(2**63))
    if kind == "dec15":
        return pa.array([decimal.Decimal(int(a) * 12345 + 7) / 100 for a in v], pa.decimal128(15, 2))
    if kind == "dec38":
        return pa.array([decimal.Decimal((int(a) * 10**20 + 3)) / 10**4 for a in v], pa.decimal128(38, 4))
    if kind == "float32":
        return pa.array((v * 0.37).astype(np.float32))
    return pa.array(v * 0.37 + 1e3)


@pytest.mark.parametrize("kind", ["int8", "int64", "uint64", "dec15", "dec38", "float32", "float64"])
def test_argument_types(kind, kernel):
    rng = np.random.default_rng(7)
    n = 50_000
    x = typed(kind, rng, n)
    x = pa.array(x.to_pylist(), x.type, mask=rng.random(n) < 0.1)
    t = pa.table({"k": pa.array(rng.integers(0, 5, n).astype(np.int32)), "x": x})
    check_all_modes(t, [0], 1, kernel)


# ---- accuracy ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("groups", [3, 10_000])
def test_large_mean_small_spread(groups, kernel):
    """mean 1e8, standard deviation 1: Sum(x^2) - Sum(x)^2 / n in doubles would lose every digit"""
    rng = np.random.default_rng(11)
    n = 100_000
    # every group gets n / groups values: a group of two or three draws could sit far closer together than std 1, and past
    # |mean| / std = 1e8 the double-double sums no longer promise 1e-10 (include/sailgpu.h)
    k = rng.permutation(np.arange(n) % groups).astype(np.int32)
    t = pa.table({"k": pa.array(k), "x": pa.array(1e8 + rng.normal(0.0, 1.0, n))})
    check_all_modes(t, [0], 1, kernel, n_batches=4 if groups < 100 else 1, rel=1e-10)


# ---- a describe() / q17-shaped aggregate over TPC-H lineitem ------------------------------------------------

def test_lineitem_describe_shape(kernel):
    from datagen import tpch
    li = tpch.lineitem(0.1, columns=["l_returnflag", "l_linestatus", "l_quantity", "l_extendedprice"])
    t = pa.table({"f": li.column("l_returnflag"), "s": li.column("l_linestatus"), "q": li.column("l_quantity")})
    aggs = [{"fn": "count", "name": "cnt", "args": [{"col": 2}]}, {"fn": "avg", "name": "mean", "args": [{"col": 2}]},
            {"fn": "stddev", "name": "sd", "args": [{"col": 2}]}, {"fn": "var_pop", "name": "vp", "args": [{"col": 2}]},
            {"fn": "min", "name": "lo", "args": [{"col": 2}]}, {"fn": "max", "name": "hi", "args": [{"col": 2}]}]
    spec = agg(aggs, [0, 1])
    got, m = run(spec, batches_of(t, 4))
    want = ref.ref_op(spec, t)
    # avg is a Decimal128 here (exact): compare as the reference gives it; stddev / var_pop within 1e-10
    ref.compare(got, want, 2)
    assert (m.get("gpu.jit_launches", 0) > 0) == (kernel == "specialised"), m
    pspec = agg(aggs, [0, 1], mode="partial")
    s, _ = run(pspec, [t])
    ref.compare(s, ref.ref_op(pspec, t), 2)
