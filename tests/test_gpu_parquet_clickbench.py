"""ClickBench's hits table scanned from Parquet on the device (sail_b200/csrc/parquet.cu), the way the reference stores it
(test_clickbench.py:11-119): Int16 columns as INT32 annotated INT(16, signed), EventDate as INT32 annotated INT(16, unsigned),
strings as BYTE_ARRAY without a UTF8 annotation, read with `binary_as_string`.

- 8- and 16-bit integer columns and binary columns decode bit for bit like pyarrow's reader: extremes, odd row counts, nulls,
  data pages V1 / V2, dictionary and plain pages and the writer's dictionary fallback, uncompressed and ZSTD files;
- a stored hits table of several ZSTD row groups, decoded row group by row group and read through the reference's view
  (sail_b200.clickbench.over_view), equals the generator's table, and every one of the 37 planned queries over those device
  batches equals its SQL restated in pandas (the comparisons of tests/test_clickbench.py::check)."""
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from sail_b200 import clickbench as cb

pytestmark = pytest.mark.gpu

WORDS = ["", "yandex", "купить цена", "x" * 13, "twelve bytes", "http://www.google.com/maps/search/a-considerably-longer-value"]
LAYOUTS = [("1.0", True, 1 << 20), ("1.0", False, 4096), ("2.0", True, 8192), ("2.0", False, 1 << 20)]
CODECS = [("none", None), ("zstd", 1), ("zstd", 19)]


def narrow_table(n, seed, nulls):
    """Int8 / Int16 / UInt8 / UInt16 columns over their whole range (the extremes at fixed rows, never null), a low-cardinality
    Int16 and UInt16 that stay in the dictionary, and binary columns that do (`b`) and that outgrow it (`bu`)"""
    rng = np.random.default_rng(seed)

    def mask(p):
        if not nulls:
            return None
        m = rng.random(n) < p
        m[: min(n, 2)] = False
        m[max(0, n - 2):] = False
        return m

    def full_range(dtype):
        lo, hi = np.iinfo(dtype).min, np.iinfo(dtype).max
        v = rng.integers(lo, int(hi) + 1, n).astype(dtype)
        ends = np.array([lo, hi], dtype=dtype)
        v[: min(n, 2)] = ends[: min(n, 2)]
        if n > 2:
            v[-2:] = ends[::-1]
        return v
    return pa.table({
        "i8": pa.array(full_range(np.int8), mask=mask(0.1)),
        "i16": pa.array(full_range(np.int16), mask=mask(0.2)),
        "u8": pa.array(full_range(np.uint8), mask=mask(0.05)),
        "u16": pa.array(full_range(np.uint16), mask=mask(0.1)),
        "flag": pa.array(rng.integers(-1, 10, n).astype(np.int16), mask=mask(0.1)),
        "day": pa.array((15887 + rng.integers(0, 31, n)).astype(np.uint16)),
        "b": pa.array([WORDS[i].encode() for i in rng.integers(0, len(WORDS), n)], type=pa.binary(), mask=mask(0.1)),
        "bu": pa.array([f"http://e1.ru/{i:08d}/{'q' * (i % 9)}".encode() for i in rng.permutation(n)], type=pa.binary()),
    })


def write(t, version, use_dict, page, codec, level, **kw):
    buf = io.BytesIO()
    pq.write_table(t, buf, compression=codec, compression_level=level, use_dictionary=use_dict, data_page_version=version, data_page_size=page,
                   dictionary_pagesize_limit=1 << 14, **kw)
    return buf.getvalue()


def host(batches, schema=None):
    """device batches (Arrow arrays or this library's handles) -> one host table, through an identity projection"""
    from sail_b200 import engine
    schema = schema or batches[0].schema
    spec = {"op": "projection", "exprs": [{"expr": {"col": i}, "name": n} for i, n in enumerate(schema.names)]}
    op = engine.GpuExec(spec, [schema])
    for b in batches:
        op.push(b)
    op.finish()
    t = op.collect()
    op.close()
    return t


def as_view(col):
    return col.cast(pa.string_view()) if pa.types.is_binary(col.type) else col


@pytest.mark.parametrize("n", [1, 3, 70001])
@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("version,use_dict,page", LAYOUTS)
@pytest.mark.parametrize("codec,level", CODECS)
def test_narrow_and_binary_columns_decode_like_pyarrow(n, nulls, version, use_dict, page, codec, level):
    from sail_b200 import engine
    t = narrow_table(n, 11 + n, nulls)
    raw = write(t, version, use_dict, page, codec, level)
    want = pq.read_table(io.BytesIO(raw))
    got = host([engine.parquet_decode(raw, binary_as_string=True)])
    assert got.num_rows == n
    for name in want.schema.names:
        w = as_view(want.column(name).combine_chunks())
        g = got.column(name).combine_chunks()
        assert g.type == w.type, (name, g.type, w.type)
        assert g.equals(w), name


def test_binary_bytes_pass_through_unvalidated():
    """the decoder does not look at the bytes of a binary column: a value that is not UTF-8 arrives unchanged"""
    from sail_b200 import engine
    vals = [b"\xff\xfe", b"", b"ok", b"\x00" * 20 + b"\xc3", None]
    t = pa.table({"b": pa.array(vals * 40, type=pa.binary())})
    for use_dict in (True, False):
        raw = write(t, "2.0", use_dict, 1 << 20, "zstd", 3)
        got = host([engine.parquet_decode(raw, binary_as_string=True)])
        assert got.column("b").combine_chunks().cast(pa.binary()).to_pylist() == vals * 40


# ---- the stored hits table through the view and the 37 queries ---------------------------------------------------------------
N_HITS = 100_000


@pytest.fixture(scope="module")
def stored_file():
    from datagen import hits as gen
    table = gen.hits(N_HITS, seed=7)
    buf = io.BytesIO()
    pq.write_table(gen.stored(table), buf, compression="zstd", compression_level=3, row_group_size=30_000)
    return table, buf.getvalue()


@pytest.fixture(scope="module")
def dev_hits(stored_file):
    """every row group decoded on the device, as stored: {"hits": (device batches, names)}; plans read it through the view"""
    from sail_b200 import engine
    _, raw = stored_file
    md = pq.ParquetFile(io.BytesIO(raw)).metadata
    assert md.num_row_groups > 1
    parts = [engine.parquet_decode(raw, row_group=g, binary_as_string=True) for g in range(md.num_row_groups)]
    return {"hits": (parts, parts[0].schema.names)}


def test_stored_hits_decode_and_view_equal_the_generated_table(stored_file, dev_hits):
    from sail_b200 import plans
    table, _ = stored_file
    _, names = dev_hits["hits"]
    assert names == table.schema.names
    for cols in (names[:12], names[12:]):                     # a projection has at most 24 outputs
        got = run_gpu(cb.over_view(plans.scan("hits", cols)), dev_hits)
        assert got.schema.names == cols
        for name in cols:
            g, w = got.column(name).combine_chunks(), table.column(name).combine_chunks()
            assert g.type == w.type, (name, g.type, w.type)
            assert g.equals(w), name


@pytest.fixture(scope="module")
def frame(stored_file):
    from tests import clickbench_sql as sql
    return sql.frame(stored_file[0])


def run_gpu(node, dev):
    """`node` over the stored table -> host table"""
    from sail_b200 import plans
    out = plans.execute_gpu(node, dev)
    return host(out, out[0].schema)


@pytest.mark.parametrize("name", list(cb.QUERIES))
def test_clickbench_query_from_parquet_equals_its_sql(name, dev_hits, frame):
    """tests/test_clickbench.py::check, with every scan fed by the device batches decoded from Parquet"""
    from tests.test_clickbench import as_table, sql_params, sql_result
    from tests.util import assert_same, assert_topk, gpu_op
    q = cb.QUERIES[name]
    params = sql_params(frame)
    kw = {p: params[p] for p in q.params}
    if q.parts > 1:
        parts = [run_gpu(cb.over_view(q.plan(part=i, **kw)), dev_hits) for i in range(q.parts)]
        got = pa.table([c for t in parts for c in t.columns], names=[n for t in parts for n in t.schema.names])
        assert_same(got, as_table(sql_result(name, frame, params), got.schema))
        return
    plan = q.plan(**kw)
    node = cb.top_sort(plan) or plan
    got = run_gpu(cb.over_view(node), dev_hits)
    full = as_table(sql_result(name, frame, params), got.schema)
    if node.spec["op"] == "sort":
        assert_topk(got, full, list(q.order), node.spec["fetch"], float_cols=q.floats)
    else:
        assert_same(got, full, float_cols=q.floats)
    assert got.num_rows > 0
    if node is not plan:           # [24], [26]: the projection above the TopK keeps the payload column only
        out = gpu_op(plan.spec, got)
        assert out.schema.names == plan.names and out.column(0).to_pylist() == got.column(plan.names[0]).to_pylist()

