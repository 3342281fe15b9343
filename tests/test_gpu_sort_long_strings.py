"""Sort, TopK, merge and sort-based grouping over string keys of any length.  String keys of the encoded paths (sorts above
1024 rows, TopK candidates, merges, WideAggOp's full-sort fallback) are ranked on the device, so values past 256 bytes, long
shared prefixes, prefixes of other values, embedded NUL bytes and multi-byte UTF-8 order exactly as the oracle orders them,
and ties keep their input order (sort, TopK) or go to the earlier run (merge)."""
import numpy as np
import pyarrow as pa
import pytest

from sail_b200 import clickbench as cb
from sail_b200 import plans
from tests.util import assert_same, gpu_op, oracle_op

pytestmark = pytest.mark.gpu


def special_words():
    """the cases the ranking has to get right: window bounds, long shared prefixes, prefixes, NUL bytes, multi-byte UTF-8"""
    w = ["", "a", "ab", "ab\x00", "ab\x00c", "ab\x00\x00", "\x00", "é", "éa", "日本語", "日本", "🙂x", "🙂"]
    w += ["x" * 12, "x" * 13, "y" * 255, "y" * 256, "y" * 257, "y" * 256 + "\x00"]
    for k in (8, 16, 64, 1024):                              # multiples of the 8-byte window, and one off on either side
        w += ["w" * (k - 1), "w" * k, "w" * (k + 1)]
    base = "p" * 1500
    w += [base, base[:-1], base + "a", base + "b", base + "\x00", base[:-1] + "q"]     # 1.5 KB shared prefix, last byte differs
    w += ["q" * 2000 + "é", "q" * 2000 + "日", "q" * 2000]
    w += ["z" * 10000, "z" * 9999 + "a", "z" * 9999]
    return w


def strings(rng, n, p_special=0.3):
    """short strings over a small alphabet (many ties and shared prefixes) mixed with the special words"""
    sp = special_words()
    alpha = np.array(list("ab\x00é"))
    out = []
    pick = rng.random(n) < p_special
    which = rng.integers(0, len(sp), n)
    lens = rng.integers(0, 20, n)
    for i in range(n):
        out.append(sp[which[i]] if pick[i] else "".join(rng.choice(alpha, lens[i])))
    return out


def table(n, seed, nulls=0.05):
    rng = np.random.default_rng(seed)
    return pa.table({"s": pa.array(strings(rng, n), type=pa.string_view(), mask=rng.random(n) < nulls),
                     "i": pa.array(rng.integers(-3, 3, n).astype(np.int64), mask=rng.random(n) < nulls),
                     "t": pa.array(strings(rng, n), type=pa.string_view()),
                     "p": pa.array(np.arange(n, dtype=np.int64))})


def sort_spec(keys, fetch=None):
    spec = {"op": "sort", "keys": [{"expr": {"col": c}, "asc": a, "nulls_first": nf} for c, a, nf in keys]}
    if fetch is not None:
        spec["fetch"] = fetch
    return spec


ORDERS = [(True, True), (True, False), (False, True), (False, False)]


@pytest.mark.parametrize("n", [1025, 70001, 300003])
@pytest.mark.parametrize("asc,nulls_first", ORDERS)
def test_full_sort_by_long_strings(n, asc, nulls_first):
    """one string key up to 10 000 bytes; ties come out in input order (the row-number payload shows it)"""
    t = table(n, n)
    spec = sort_spec([(0, asc, nulls_first)])
    assert_same(gpu_op(spec, t), oracle_op(spec, t), ordered=True)


@pytest.mark.parametrize("keys", [[(0, True, False), (1, False, True)], [(0, False, False), (2, True, True)], [(2, True, True), (0, True, True), (1, True, False)]],
                         ids=["long_then_int64", "two_long", "long_long_int64"])
def test_sort_by_long_string_and_more_keys(keys):
    t = table(70001, 11)
    spec = sort_spec(keys)
    assert_same(gpu_op(spec, t), oracle_op(spec, t), ordered=True)


@pytest.mark.parametrize("asc", [True, False])
def test_many_copies_of_few_long_strings(asc):
    """a few 2-4 KB strings that share their first 1000 bytes, each repeated thousands of times: their groups stay open for
    every window, and the row numbers show that ties keep their input order"""
    rng = np.random.default_rng(4)
    n = 100_000
    head = "h" * 1000
    words = [head + c * k for c, k in zip("abcab", (1000, 2000, 3000, 3001, 1000))] + [head + "a" * 1000 + "\x00"]
    t = pa.table({"s": pa.array([words[i] for i in rng.integers(0, len(words), n)], type=pa.string_view()),
                  "p": pa.array(np.arange(n, dtype=np.int64))})
    spec = sort_spec([(0, asc, True)])
    assert_same(gpu_op(spec, t), oracle_op(spec, t), ordered=True)


@pytest.fixture
def topk(monkeypatch):
    monkeypatch.setenv("SAILGPU_TOPK_MIN_ROWS", "1000")


@pytest.mark.parametrize("fetch", [1, 10, 1000])
@pytest.mark.parametrize("asc,nulls_first", ORDERS)
def test_topk_by_long_strings(topk, fetch, asc, nulls_first):
    t = table(70001, 21)
    spec = sort_spec([(0, asc, nulls_first), (1, True, True)], fetch)
    assert_same(gpu_op(spec, t), oracle_op(spec, t), ordered=True)


@pytest.mark.parametrize("fetch", [1, 10, 1000])
def test_topk_with_a_constant_leading_16_bytes(topk, fetch):
    """every value starts with the same 16 bytes: the selection word cannot narrow the input, and the operator sorts everything"""
    rng = np.random.default_rng(fetch)
    n = 70001
    s = ["c" * 16 + v for v in strings(rng, n)]
    t = pa.table({"s": pa.array(s, type=pa.string_view()), "p": pa.array(np.arange(n, dtype=np.int64))})
    for asc in (True, False):
        spec = sort_spec([(0, asc, True)], fetch)
        assert_same(gpu_op(spec, t), oracle_op(spec, t), ordered=True)


def run_merge(spec, runs):
    from sail_b200 import engine
    op = engine.GpuExec(spec, [runs[0].schema])
    try:
        for r in runs:
            op.push(r)
        op.finish()
        return op.collect()
    finally:
        op.close()


@pytest.mark.parametrize("n_runs", [1, 2, 5])
@pytest.mark.parametrize("fetch", [None, 100])
def test_merge_of_runs_sorted_by_long_strings(n_runs, fetch):
    """runs='batches': every pushed batch is a sorted run; ties go to the earlier run, which is the stable sort of the runs
    laid end to end"""
    keys = [(0, True, False), (1, False, True)]
    runs = []
    for r in range(n_runs):
        t = table(9000 + 1000 * r, 100 + r)
        runs.append(oracle_op(sort_spec(keys), t))
    spec = {"op": "sort_preserving_merge", "keys": sort_spec(keys)["keys"], "runs": "batches"}
    if fetch is not None:
        spec["fetch"] = fetch
    want = oracle_op(sort_spec(keys, fetch), pa.concat_tables(runs))
    assert_same(run_merge(spec, runs), want, ordered=True)


@pytest.mark.parametrize("mode", ["single", "two_phase"])
@pytest.mark.parametrize("full_sort", [False, True])
def test_grouping_by_strings_that_differ_after_byte_1000(mode, full_sort, monkeypatch):
    """seven group keys (sort-based grouping), two of them strings longer than 256 bytes that differ only after byte 1000"""
    if full_sort:
        monkeypatch.setenv("SAILGPU_WIDEAGG_FULL_SORT", "1")
    rng = np.random.default_rng(9)
    n = 40000
    long_a = ["L" * 1001 + f"{v:03d}" + "t" * (v % 7) for v in range(40)]
    long_b = ["M" * 300 + "\x00" * 700 + c for c in ["", "a", "b", "é", "\x00"]]
    mask = rng.random(n) < 0.05
    t = pa.table({
        "k0": pa.array([long_a[v] for v in rng.integers(0, len(long_a), n)], type=pa.string_view(), mask=mask),
        "k1": pa.array([long_b[v] for v in rng.integers(0, len(long_b), n)], type=pa.string_view()),
        "k2": pa.array(rng.integers(0, 3, n).astype(np.int64)),
        "k3": pa.array(rng.integers(0, 2, n).astype(np.int32), mask=rng.random(n) < 0.05),
        "k4": pa.array(rng.integers(-300, -298, n).astype(np.int16)),
        "k5": pa.array([["x", "y"][v] for v in rng.integers(0, 2, n)], type=pa.string_view()),
        "k6": pa.array(rng.integers(0, 2, n).astype(np.int64)),
        "v": pa.array(rng.integers(-1000, 1000, n).astype(np.int64)),
    })
    keys = [f"k{i}" for i in range(7)]
    aggs = [("sum", plans.col("v"), "sv", "Int64"), ("count", None, "c", None), ("min", plans.col("v"), "mn", "Int64")]
    scan = plans.scan("t", t.schema.names)
    node = plans.aggregate(scan, "single", keys, aggs) if mode == "single" else plans.two_phase(scan, keys, aggs)
    got = plans.execute(node, {"t": t}, gpu_op)
    want = plans.execute(node, {"t": t}, oracle_op)
    assert got.num_rows == want.num_rows and got.num_rows > 1000
    assert_same(got, want)


@pytest.fixture(scope="module")
def long_phrase_hits():
    """300 k hits rows in which about 2 % of the non-empty SearchPhrase values are 300-5000-byte phrases"""
    from datagen import hits as gen
    t = gen.hits(300_000, seed=7)
    rng = np.random.default_rng(8)
    sp = t.column("SearchPhrase").to_pylist()
    for i in np.nonzero(rng.random(len(sp)) < 0.02)[0]:
        v = sp[i]
        if v:
            k = int(rng.integers(300, 5001))
            sp[i] = ((v + " ") * (k // (len(v) + 1) + 1))[:k]
    assert max(len(v.encode()) for v in sp if v) >= 300
    i = t.schema.get_field_index("SearchPhrase")
    return t.set_column(i, t.schema.field(i), pa.array(sp, type=t.schema.field(i).type))


@pytest.mark.parametrize("name", ["c25", "c26"])
@pytest.mark.parametrize("topk_min", [None, "1000"])
def test_clickbench_top_search_phrases_with_long_phrases(name, topk_min, long_phrase_hits, monkeypatch):
    from tests import clickbench_sql as sql
    from tests.test_clickbench import check
    if topk_min is not None:
        monkeypatch.setenv("SAILGPU_TOPK_MIN_ROWS", topk_min)
    assert cb.QUERIES[name].sql in (25, 26)
    check(name, sql.frame(long_phrase_hits), {"hits": long_phrase_hits}, gpu_op)
