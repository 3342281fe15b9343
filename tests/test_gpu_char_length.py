"""character_length on the GPU, in the interpreted and the specialised kernel: projections against pyarrow's utf8_length over
inline and long strings of every alignment, the function inside filters and aggregates against the reference of
tests/char_length_ref.py, and ClickBench [27] against its SQL restated in pandas, resident and from Parquet."""
import io

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from sail_b200 import clickbench as cb, engine, plans
from tests import char_length_ref as ref
from tests.util import assert_same, assert_topk

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["interpreted", "specialised"])
def kernel(request, monkeypatch):
    if request.param == "interpreted":
        monkeypatch.setenv("SAILGPU_JIT", "0")
    else:
        monkeypatch.delenv("SAILGPU_JIT", raising=False)
        monkeypatch.setenv("SAILGPU_JIT_MIN_ROWS", "0")
        monkeypatch.setenv("SAILGPU_JIT_STRICT", "1")
    return request.param


def run(spec, *tables):
    op = engine.GpuExec(spec, [t.schema for t in tables])
    try:
        for i, t in enumerate(tables):
            op.push(t, i)
            op.finish(i)
        return op.collect(), op.metrics()
    finally:
        op.close()


def length(e):
    return plans.char_length(e)


def col(i):
    return {"col": i}


CHARS = ["a", "ж", "€", "𝄞"]        # 1-, 2-, 3- and 4-byte UTF-8


def edge_strings():
    """empty and null values; each character width; byte lengths 11, 12 and 13 with a multibyte character across byte 12 and one
    across the 4-byte boundary of an inline view; long strings of 16k + 1 bytes, so that consecutive ones start at every offset
    mod 16 of the heap, up to several KiB"""
    rng = np.random.default_rng(11)
    out = ["", None, "a", "ж", "€", "𝄞", "abc𝄞", "ab€€€", "a" * 11, "a" * 12, "a" * 13, "a" * 10 + "ж", "a" * 9 + "€",
           "a" * 11 + "ж", "a" * 10 + "€", "a" * 9 + "𝄞", "a" * 11 + "𝄞", "ж" * 6, "ж" * 7, "€" * 4, "𝄞" * 3, "𝄞" * 4]
    for k in range(48):
        n = 16 * int(rng.integers(1, 300 if k % 8 else 8)) + 1
        s = "".join(rng.choice(CHARS, n)).encode()[:n].decode(errors="ignore")
        out.append(s + "b" * (n - len(s.encode())))          # exactly n bytes, characters kept whole
    out += ["".join(rng.choice(CHARS, int(m))) for m in rng.integers(0, 40, 300)]
    out += [None if i % 7 == 0 else "".join(rng.choice(CHARS, int(m))) for i, m in enumerate(rng.integers(10, 3000, 60))]
    return out


@pytest.mark.parametrize("t", [pa.string(), pa.string_view()])
@pytest.mark.parametrize("offset", [0, 7])
def test_projection_equals_pyarrow_utf8_length(kernel, t, offset):
    vals = edge_strings()
    tbl = pa.table({"s": pa.array(vals, type=t)}).slice(offset)
    assert any(len(v.encode()) >= 4096 for v in vals[offset:] if v)
    spec = {"op": "projection", "exprs": [{"expr": length(col(0)), "name": "n"}]}
    got, m = run(spec, tbl)
    want = pc.utf8_length(tbl.column("s").cast(pa.string()).combine_chunks())
    assert got.column("n").type == pa.int32()
    assert got.column("n").combine_chunks().equals(want)
    if kernel == "specialised":
        assert m["gpu.jit_launches"] >= 1


def random_table(n, seed, nulls=True):
    rng = np.random.default_rng(seed)
    words = ["".join(rng.choice(CHARS, int(m))) for m in rng.integers(0, 60, 500)]
    s = pa.array(rng.choice(words, n), type=pa.string_view(), mask=(rng.random(n) < 0.05) if nulls else None)
    return pa.table({"k": pa.array(rng.integers(0, 50, n).astype(np.int32)), "s": s})


def test_filter_on_character_length(kernel):
    t = random_table(100_000, 1)
    spec = {"op": "filter", "predicate": {"op": ">", "l": length(col(1)), "r": {"lit": 20, "type": "Int32"}}}
    got, m = run(spec, t)
    assert 0 < got.num_rows < t.num_rows
    assert_same(got, ref.ref_op(spec, t))
    if kernel == "specialised":
        assert m["gpu.jit_launches"] >= 1


def test_character_length_as_a_group_key(kernel):
    t = random_table(100_000, 2)
    spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": length(col(1)), "name": "n"}],
            "aggs": [{"fn": "count", "args": [], "name": "c", "input_type": None}]}
    got, _ = run(spec, t)
    assert got.num_rows > 50
    assert_same(got, ref.ref_op(spec, t))


def test_sum_and_avg_of_character_length_partial_then_final(kernel):
    t = random_table(120_000, 3)
    aggs = [{"fn": "sum", "args": [length(col(1))], "name": "s", "input_type": "Int32"},
            {"fn": "avg", "args": [length(col(1))], "name": "a", "input_type": "Int32"},
            {"fn": "count", "args": [], "name": "c", "input_type": None}]
    partial = {"op": "aggregate", "mode": "partial", "group_by": [{"expr": col(0), "name": "k"}], "aggs": aggs}
    final = {"op": "aggregate", "mode": "final_partitioned", "group_by": [{"expr": col(0), "name": "k"}],
             "aggs": [{k: v for k, v in a.items() if k != "args"} for a in aggs]}
    halves = [t.slice(0, 60_000), t.slice(60_000)]
    got_partial = [run(partial, h)[0] for h in halves]
    want_partial = [ref.ref_op(partial, h) for h in halves]
    for g, w in zip(got_partial, want_partial):
        assert_same(g, w, float_cols=(3,))
    got, _ = run(final, pa.concat_tables(got_partial))
    assert_same(got, ref.ref_op(final, pa.concat_tables(want_partial)), float_cols=(2,))


# ---- ClickBench [27] -------------------------------------------------------------------------------------------------------------
def multibyte_urls(t: pa.Table) -> pa.Table:
    """`t` with every distinct URL mapped to a string that mixes ASCII with Cyrillic (2-byte) and 4-byte characters; the empty
    URL stays empty, so [27]'s filter keeps the same rows"""
    d = pc.dictionary_encode(t.column("URL").combine_chunks())
    table = str.maketrans({"a": "а", "e": "е", "o": "о", "p": "р", "c": "с", "x": "х"})       # Cyrillic look-alikes

    def remap(i, u):
        if not u:
            return u
        u = u.translate(table) if i % 3 else u
        return u + "🦀" * (i % 4)
    vocab = pa.array([remap(i, u) for i, u in enumerate(d.dictionary.to_pylist())], type=pa.string())
    url = pc.take(vocab, d.indices).cast(t.schema.field("URL").type)
    return t.set_column(t.schema.get_field_index("URL"), "URL", url)


@pytest.fixture(scope="module")
def hits_table():
    from datagen import hits as gen
    return multibyte_urls(gen.hits(100_000, seed=7))


@pytest.fixture(scope="module")
def frame(hits_table):
    from tests import clickbench_sql as sql
    return sql.frame(hits_table)


def check27(got, frame, min_count):
    from tests.test_clickbench import as_table
    q = cb.LENGTH_QUERIES["c27"]
    assert got.num_rows >= 10
    assert_topk(got, as_table(ref.q27(frame, min_count), got.schema), list(q.order), cb.top_sort(q.plan()).spec["fetch"], float_cols=q.floats)


def test_remapped_urls_have_multibyte_characters(frame):
    u = frame.URL[frame.URL != ""]
    assert (u.str.len() < u.str.encode("utf-8").str.len()).mean() > 0.5


def test_clickbench_27_resident(kernel, hits_table, frame):
    min_count = ref.q27_min_count(frame)
    node = cb.top_sort(cb.LENGTH_QUERIES["c27"].plan(min_count=min_count))
    launches = []

    def gpu(spec, *ts):
        out, m = run(spec, *ts)
        launches.append(m.get("gpu.jit_launches", 0))
        return out
    got = plans.execute(node, {"hits": hits_table}, gpu)
    check27(got, frame, min_count)
    if kernel == "specialised":
        assert sum(launches) >= 1


def test_clickbench_27_from_parquet(kernel, hits_table, frame):
    from datagen import hits as gen
    from tests.test_gpu_parquet_clickbench import run_gpu
    buf = io.BytesIO()
    pq.write_table(gen.stored(hits_table.select(["CounterID", "URL"])), buf, compression="zstd", compression_level=3, row_group_size=30_000)
    raw = buf.getvalue()
    n_groups = pq.ParquetFile(io.BytesIO(raw)).metadata.num_row_groups
    assert n_groups > 1
    parts = [engine.parquet_decode(raw, row_group=g, binary_as_string=True) for g in range(n_groups)]
    min_count = ref.q27_min_count(frame)
    got = run_gpu(cb.over_view(cb.top_sort(cb.LENGTH_QUERIES["c27"].plan(min_count=min_count))), {"hits": (parts, parts[0].schema.names)})
    check27(got, frame, min_count)
