"""Parquet pages in the DELTA_BINARY_PACKED, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY and BYTE_STREAM_SPLIT encodings decoded on
the device (sail_b200/csrc/parquet.cu), bit for bit like pyarrow's reader: every encoding with every physical type and target type
it covers, INT32 / INT64 extremes whose deltas wrap, strings that are empty, 12 or 13 bytes long or share long prefixes, DOUBLE NaN
and -0.0, nulls, data pages V1 and V2, uncompressed and ZSTD; a chunk that falls back from its dictionary to DELTA pages; a
DELTA_BYTE_ARRAY prefix longer than the value before it, refused as invalid; ClickBench's 37 queries over a hits table stored
with DELTA encodings; and TPC-H Q1 over a DELTA-encoded lineitem row group."""
import ctypes
import decimal
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from sail_b200 import clickbench as cb
from tests import test_gpu_parquet_clickbench as cbp
from tests.test_parquet_delta_plan import ENCODINGS, chunk_bytes, delta_table, spliced, varint, with_chunk, write

pytestmark = pytest.mark.gpu


def same_bits(g: pa.Array, w: pa.Array, name):
    """equal values and validity; floating point compared by bit pattern (NaN payloads, -0.0)"""
    if pa.types.is_string(w.type) or pa.types.is_binary(w.type):
        w = w.cast(pa.string_view())
    assert g.type == w.type, (name, g.type, w.type)
    if pa.types.is_floating(w.type):
        assert g.is_null().equals(w.is_null()), name
        gv, wv = g.fill_null(0.0).to_numpy(zero_copy_only=False), w.fill_null(0.0).to_numpy(zero_copy_only=False)
        assert np.array_equal(gv.view(np.int64), wv.view(np.int64)), name
    else:
        assert g.equals(w), name


def check(raw):
    from sail_b200 import engine
    want = pq.read_table(io.BytesIO(raw))
    got = cbp.host([engine.parquet_decode(raw, binary_as_string=True)])
    assert got.num_rows == want.num_rows
    for name in want.schema.names:
        same_bits(got.column(name).combine_chunks(), want.column(name).combine_chunks(), name)


@pytest.mark.parametrize("n", [1, 33, 129, 70001])
@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("codec,level", [("none", None), ("zstd", 3)])
@pytest.mark.parametrize("encoding", list(ENCODINGS))
def test_decodes_like_pyarrow(n, nulls, version, codec, level, encoding):
    check(write(delta_table(n, 5 + n, nulls), encoding, version, 8192, codec, level))


def narrow_and_decimal_table(n, seed):
    """the other targets of INT32 / INT64: Date32, Int8, UInt8, UInt16, and decimals stored as integers"""
    rng = np.random.default_rng(seed)
    return pa.table({
        "dt": pa.array(rng.integers(-5000, 30000, n).astype(np.int32)).cast(pa.date32()),
        "i8": pa.array(rng.integers(-128, 128, n).astype(np.int8)),
        "u8": pa.array(rng.integers(0, 256, n).astype(np.uint8)),
        "u16": pa.array(rng.integers(0, 65536, n).astype(np.uint16)),
        "d9": pa.array([decimal.Decimal(int(x)) / 100 for x in rng.integers(-10**9 + 1, 10**9, n)], type=pa.decimal128(9, 2)),
        "d18": pa.array([decimal.Decimal(int(x)) / 100 for x in rng.integers(-10**18 + 1, 10**18, n)], type=pa.decimal128(18, 2)),
    })


@pytest.mark.parametrize("encoding", ["DELTA_BINARY_PACKED", "BYTE_STREAM_SPLIT"])
@pytest.mark.parametrize("version", ["1.0", "2.0"])
def test_every_integer_and_decimal_target(encoding, version):
    t = narrow_and_decimal_table(20001, 4)
    buf = io.BytesIO()
    pq.write_table(t, buf, compression="none", use_dictionary=False, column_encoding={c: encoding for c in t.schema.names}, data_page_version=version,
                   data_page_size=8192, store_decimal_as_integer=True)
    md = pq.ParquetFile(io.BytesIO(buf.getvalue())).metadata.row_group(0)
    assert [md.column(i).physical_type for i in range(len(t.schema))] == ["INT32"] * 5 + ["INT64"]
    check(buf.getvalue())


# ---- a chunk that falls back from its dictionary to DELTA pages --------------------------------------------------------------------
def decode_raw(raw, mutate):
    """sailgpu_parquet_decode on descriptors the test changes first -> (code, host table or message)"""
    from sail_b200 import engine
    ctx = engine.default_context()
    buf, schema, cols, n_rows = engine._parquet_descriptors(raw, 0, None, True)
    mutate(cols)
    cschema = engine._export_schema(schema)
    d = engine.DeviceBatch(schema)
    rc = engine.lib().sailgpu_parquet_decode(ctx._h, ctypes.addressof(cschema), ctypes.addressof(cols), len(cols), n_rows, ctypes.addressof(d.c))
    engine._release_schema(cschema)
    del buf
    if rc != 0:
        return rc, engine.lib().sailgpu_ctx_last_error(None).decode()
    d._live = True
    return 0, cbp.host([d])


@pytest.mark.parametrize("name", ["i64", "i32", "s", "b", "fl"])
@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("codec", ["none", "zstd"])
def test_dictionary_then_delta_pages_in_one_chunk(name, version, codec):
    t = delta_table(20000, 9, True)
    chunk, whole = spliced(t, name, 7000, version, codec)
    rc, got = decode_raw(whole, with_chunk(chunk))
    assert rc == 0, got
    same_bits(got.column(name).combine_chunks(), t.column(name).combine_chunks(), name)


def test_prefix_longer_than_the_value_before_it_is_invalid():
    n = 500
    t = pa.table({"s": pa.array([f"value-{i:05d}-{'z' * (i % 17)}" for i in range(n)])}, schema=pa.schema([pa.field("s", pa.string(), nullable=False)]))
    raw = write(t, "DELTA_BYTE_ARRAY", "1.0", 1 << 20)
    chunk = bytearray(chunk_bytes(raw))
    # the page body starts with the prefix-length stream: the writer's block size 128, 4 miniblocks, n values, first value 0 -- the
    # first value of a page has no value before it, so a first prefix of 5 is longer than the value before it
    header = b"\x80\x01\x04" + varint(n) + b"\x00"
    at = chunk.index(header) + len(header) - 1
    assert rc_ok(raw, chunk)
    chunk[at] = 10                               # zigzag(5)
    rc, msg = decode_raw(raw, with_chunk(bytes(chunk)))
    assert rc == 1 and "column 's'" in msg and "prefix" in msg, msg


def rc_ok(raw, chunk):
    rc, got = decode_raw(raw, with_chunk(bytes(chunk)))
    return rc == 0 and got.column("s").to_pylist() == pq.read_table(io.BytesIO(raw)).column("s").to_pylist()


# ---- ClickBench over a hits table stored with DELTA encodings --------------------------------------------------------------------
@pytest.fixture(scope="module")
def stored_file():
    from datagen import hits as gen
    table = gen.hits(cbp.N_HITS, seed=7)
    s = gen.stored(table)
    buf = io.BytesIO()
    pq.write_table(s, buf, compression="zstd", compression_level=3, row_group_size=30_000, use_dictionary=False, data_page_version="2.0",
                   column_encoding=gen.delta_encoding(s.schema))
    return table, buf.getvalue()


@pytest.fixture(scope="module")
def dev_hits(stored_file):
    from sail_b200 import engine
    _, raw = stored_file
    md = pq.ParquetFile(io.BytesIO(raw)).metadata
    assert md.num_row_groups > 1
    encodings = {md.row_group(0).column(i).encodings[-1] for i in range(md.num_columns)}
    assert encodings == {"DELTA_BINARY_PACKED", "DELTA_BYTE_ARRAY"}, encodings
    parts = [engine.parquet_decode(raw, row_group=g, binary_as_string=True) for g in range(md.num_row_groups)]
    return {"hits": (parts, parts[0].schema.names)}


@pytest.fixture(scope="module")
def frame(stored_file):
    from tests import clickbench_sql as sql
    return sql.frame(stored_file[0])


def test_delta_hits_decode_and_view_equal_the_generated_table(stored_file, dev_hits):
    cbp.test_stored_hits_decode_and_view_equal_the_generated_table(stored_file, dev_hits)


@pytest.mark.parametrize("name", list(cb.QUERIES))
def test_clickbench_query_from_delta_parquet_equals_its_sql(name, dev_hits, frame):
    cbp.test_clickbench_query_from_parquet_equals_its_sql(name, dev_hits, frame)


# ---- TPC-H Q1 over a DELTA-encoded lineitem row group ------------------------------------------------------------------------------
def test_q1_over_delta_lineitem_equals_q1_over_plain():
    from bench import Q1_COLS
    from datagen import tpch
    from oracle import render
    from sail_b200 import engine, plans
    li = tpch.lineitem(0.05).select(Q1_COLS)
    enc = {c: "DELTA_BINARY_PACKED" for c in Q1_COLS if c not in ("l_returnflag", "l_linestatus")}
    enc.update({"l_returnflag": "DELTA_BYTE_ARRAY", "l_linestatus": "DELTA_LENGTH_BYTE_ARRAY"})
    results = []
    for kw in (dict(), dict(use_dictionary=False, column_encoding=enc)):
        buf = io.BytesIO()
        pq.write_table(li, buf, compression="none", store_decimal_as_integer=True, row_group_size=len(li), **kw)
        md = pq.ParquetFile(io.BytesIO(buf.getvalue())).metadata.row_group(0)
        if kw:
            assert md.column(0).physical_type == "INT64" and md.column(0).encodings[-1] == "DELTA_BINARY_PACKED"
        dev = engine.parquet_decode(buf.getvalue())
        out = plans.execute_gpu(plans.q1(), {"lineitem": ([dev], Q1_COLS)})
        results.append(sorted(render.rows(cbp.host(out, out[0].schema))))
    assert results[0] == results[1] and len(results[0]) == 4
