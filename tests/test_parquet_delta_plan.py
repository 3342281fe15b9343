"""CPU test of the host walk of Parquet's DELTA_BINARY_PACKED, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY and BYTE_STREAM_SPLIT
pages (sail_b200/csrc/parquet.cu): every value of every page is accounted for, in data pages V1 and V2, with and without nulls,
uncompressed and ZSTD; a chunk that falls back from its dictionary to DELTA pages counts both kinds of page; and corrupt DELTA
streams are refused as invalid, naming the column and the page, without a crash."""
import ctypes
import decimal
import io
import json

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from sail_b200 import engine

# column -> the encodings a writer may give it
ENCODINGS = {
    "DELTA_BINARY_PACKED": ["i32", "i64", "i16", "ts"],
    "DELTA_LENGTH_BYTE_ARRAY": ["s", "b"],
    "DELTA_BYTE_ARRAY": ["s", "b", "fl"],
    "BYTE_STREAM_SPLIT": ["i32", "i64", "d", "fl"],
}
NEW_KEYS = ["delta_pages", "delta_values", "bss_pages", "bss_values"]
KEYS = ["pages", "dense", "dict_count", "level_values", "index_values", "level_runs", "index_runs", "plain_strings", "dict_pages",
        "plain_pages", "body_bytes", "body_fnv1a"] + NEW_KEYS
I32, I64 = np.iinfo(np.int32), np.iinfo(np.int64)


def delta_table(n, seed, nulls):
    """extremes of INT32 / INT64 next to each other (so the deltas wrap), Int16 and Timestamp columns, DOUBLE bit patterns with
    NaN and -0.0, strings that are empty, 12 and 13 bytes long or share long prefixes, and a FIXED_LEN_BYTE_ARRAY decimal"""
    rng = np.random.default_rng(seed)

    def mask(p):
        if not nulls:
            return None
        m = rng.random(n) < p
        m[: min(n, 3)] = False
        return m

    def extremes(info, dtype):
        v = rng.integers(info.min, int(info.max) + 1, n, dtype=dtype)
        ends = np.array([info.max, info.min, info.max, 0, info.min, -1], dtype=dtype)
        k = min(n, len(ends))
        v[:k] = ends[:k]
        v[n // 2: n // 2 + k] = ends[:k][: n - n // 2]
        return v
    d = rng.normal(size=n) * 1e6
    specials = np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, 5e-324], dtype=np.float64)
    d[: min(n, 6)] = specials[: min(n, 6)]
    prefix = "http://example.com/some/long/shared/path/"
    words = ["", "twelve bytes", "x" * 13, prefix, prefix + "a", prefix + "ab", prefix + "b" * 40, "short"]
    strs = [words[i] if i < len(words) else f"{prefix}{j:06d}" for i, j in zip(rng.integers(0, 2 * len(words), n), rng.integers(0, 999, n))]
    return pa.table({
        "i32": pa.array(extremes(I32, np.int32), mask=mask(0.1)),
        "i64": pa.array(extremes(I64, np.int64), mask=mask(0.2)),
        "i16": pa.array(rng.integers(-32768, 32768, n).astype(np.int16), mask=mask(0.1)),
        "ts": pa.array(np.cumsum(rng.integers(0, 10**9, n)) + 1_600_000_000_000_000, type=pa.timestamp("us", tz="UTC"), mask=mask(0.1)),
        "d": pa.array(d, mask=mask(0.1)),
        "s": pa.array(strs, type=pa.string(), mask=mask(0.1)),
        "b": pa.array([s.encode() for s in strs], type=pa.binary()),
        "fl": pa.array([decimal.Decimal(int(x)) / 100 for x in rng.integers(-10**17, 10**17, n)], type=pa.decimal128(20, 2), mask=mask(0.2)),
    })


def write(t, encoding, version, page, codec="none", level=None, **kw):
    """the columns of `t` that `encoding` covers, all written with it (no dictionary)"""
    cols = [c for c in ENCODINGS[encoding] if c in t.schema.names]
    buf = io.BytesIO()
    pq.write_table(t.select(cols), buf, compression=codec, compression_level=level, use_dictionary=False, column_encoding={c: encoding for c in cols},
                   data_page_version=version, data_page_size=page, **kw)
    return buf.getvalue()


def walk(raw):
    names = pq.ParquetFile(io.BytesIO(raw)).schema_arrow.names
    return {name: engine.parquet_inspect(raw, i, binary_as_string=True) for i, name in enumerate(names)}


@pytest.mark.parametrize("n", [1, 31, 32, 33, 127, 128, 129, 70001])
@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("page", [1 << 20, 4096])
@pytest.mark.parametrize("encoding", list(ENCODINGS))
def test_walk_accounts_for_every_value(n, nulls, version, page, encoding):
    t = delta_table(n, 5 + n, nulls)
    raw = write(t, encoding, version, page)
    md = pq.ParquetFile(io.BytesIO(raw)).metadata.row_group(0)
    bss = encoding == "BYTE_STREAM_SPLIT"
    for i, (name, info) in enumerate(walk(raw).items()):
        cm = md.column(i)
        assert cm.encodings[-1] == encoding and not cm.has_dictionary_page, (name, cm.encodings)
        dense = n - t.column(name).null_count
        assert info["dense"] == dense == cm.statistics.num_values, (name, info)
        assert info["level_values"] == (n if cm.statistics.null_count or t.schema.field(name).nullable else 0), (name, info)
        assert info[("bss" if bss else "delta") + "_pages"] == info["pages"] >= 1, (name, info)
        assert info[("bss" if bss else "delta") + "_values"] == dense, (name, info)
        assert info[("delta" if bss else "bss") + "_pages"] == info[("delta" if bss else "bss") + "_values"] == 0, (name, info)
        assert info["dict_pages"] == info["plain_pages"] == info["index_values"] == info["plain_strings"] == 0, (name, info)
        if n == 70001 and page == 4096:
            assert info["pages"] > 1, (name, info)


@pytest.mark.parametrize("encoding", list(ENCODINGS))
@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("level", [1, 19])
def test_zstd_walk_equals_uncompressed_walk(encoding, version, level):
    t = delta_table(70001, 3, True)
    plain, packed = write(t, encoding, version, 8192), write(t, encoding, version, 8192, "zstd", level)
    assert pq.ParquetFile(io.BytesIO(packed)).metadata.row_group(0).column(0).compression == "ZSTD"
    a, b = walk(plain), walk(packed)
    for name in a:
        assert {k: b[name][k] for k in KEYS} == {k: a[name][k] for k in KEYS}, (name, a[name], b[name])


def test_float_and_boolean_stay_refused_under_byte_stream_split():
    t = pa.table({"f": pa.array(np.arange(100, dtype=np.float32))})
    buf = io.BytesIO()
    pq.write_table(t, buf, compression="none", use_dictionary=False, column_encoding={"f": "BYTE_STREAM_SPLIT"})
    with pytest.raises(engine.SailGpuError) as e:
        engine.parquet_inspect(buf.getvalue(), 0)
    assert e.value.code == 2


# ---- a chunk that falls back from its dictionary to DELTA pages --------------------------------------------------------------------
def chunk_bytes(raw, column=0):
    cm = pq.ParquetFile(io.BytesIO(raw)).metadata.row_group(0).column(column)
    start = cm.data_page_offset if cm.dictionary_page_offset is None else min(cm.data_page_offset, cm.dictionary_page_offset)
    return raw[start: start + cm.total_compressed_size]


def spliced(t, name, a, version, codec="none"):
    """column `name` of `t` as one chunk: the dictionary-encoded chunk of rows [0, a), then the DELTA data pages of rows [a, n)
    (what a V2 writer emits when the column outgrows its dictionary).  Returns the chunk and a file of the whole column, whose
    descriptors the chunk replaces."""
    col = t.select([name])
    enc = "DELTA_BINARY_PACKED" if name in ENCODINGS["DELTA_BINARY_PACKED"] else "DELTA_BYTE_ARRAY"
    buf = io.BytesIO()
    pq.write_table(col.slice(0, a), buf, compression=codec, use_dictionary=True, data_page_version=version, data_page_size=4096)
    head = chunk_bytes(buf.getvalue())
    tail = chunk_bytes(write(col.slice(a), enc, version, 4096, codec))
    buf = io.BytesIO()
    pq.write_table(col, buf, compression=codec, use_dictionary=False, data_page_version=version)
    return head + tail, buf.getvalue()


def with_chunk(chunk):
    keep = ctypes.create_string_buffer(chunk, len(chunk))

    def mutate(cols):
        cols[0].chunk = ctypes.addressof(keep)
        cols[0].chunk_len = len(chunk)
    mutate.keep = keep
    return mutate


def inspect_raw(raw, column, mutate):
    """sailgpu_parquet_inspect on descriptors the test changes first"""
    buf, schema, cols, n_rows = engine._parquet_descriptors(raw, 0, None, True)
    mutate(cols)
    cschema = engine._export_schema(schema)
    out = ctypes.create_string_buffer(1024)
    rc = engine.lib().sailgpu_parquet_inspect(ctypes.addressof(cschema), ctypes.addressof(cols), len(cols), n_rows, column, out, 1024)
    engine._release_schema(cschema)
    del buf
    return rc, out.value.decode()


@pytest.mark.parametrize("name", ["i64", "i32", "s", "fl"])
@pytest.mark.parametrize("version", ["1.0", "2.0"])
def test_dictionary_then_delta_pages_in_one_chunk(name, version):
    n, a = 20000, 7000
    t = delta_table(n, 9, True)
    chunk, whole = spliced(t, name, a, version)
    rc, msg = inspect_raw(whole, 0, with_chunk(chunk))
    assert rc == 0, msg
    info = json.loads(msg)
    col = t.column(name)
    assert info["dense"] == n - col.null_count
    assert info["dict_pages"] == 1 and info["delta_pages"] >= 1 and info["plain_pages"] == 0
    assert info["index_values"] == a - col.slice(0, a).null_count
    assert info["delta_values"] == (n - a) - col.slice(a).null_count


# ---- corrupt DELTA_BINARY_PACKED streams ------------------------------------------------------------------------------------------
def varint(v):
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


N_CORRUPT = 200                 # one block of the writer's 256 values: a corrupt width changes nothing else


def corrupt_case():
    """a required INT64 column of N_CORRUPT values in one DELTA_BINARY_PACKED page V1 (no levels: the page body is the stream),
    and where in its chunk the stream's header and first block's bit widths are"""
    v = np.random.default_rng(1).integers(0, 1 << 20, N_CORRUPT)
    t = pa.table({"v": pa.array(v)}, schema=pa.schema([pa.field("v", pa.int64(), nullable=False)]))
    raw = write(t.rename_columns(["i64"]), "DELTA_BINARY_PACKED", "1.0", 1 << 20)
    chunk = bytearray(chunk_bytes(raw))
    header = b"\x80\x02\x04" + varint(N_CORRUPT)                 # the writer's block size 256, 4 miniblocks, total count
    at = chunk.index(header)
    p = at + len(header)
    for _ in range(2):                                           # first value, then the first block's min delta
        while chunk[p] & 0x80:
            p += 1
        p += 1
    return raw, chunk, at, p


def refused(raw, chunk):
    rc, msg = inspect_raw(raw, 0, with_chunk(bytes(chunk)))
    assert rc == 1, msg
    assert "column 'i64'" in msg and "page 0" in msg, msg
    return msg


def test_the_uncorrupted_stream_is_accepted():
    raw, chunk, _, _ = corrupt_case()
    rc, msg = inspect_raw(raw, 0, with_chunk(bytes(chunk)))
    assert rc == 0 and json.loads(msg)["delta_values"] == N_CORRUPT, msg


def test_bit_width_above_64():
    raw, chunk, _, widths = corrupt_case()
    chunk[widths] = 65
    assert "bit width 65" in refused(raw, chunk)


@pytest.mark.parametrize("block,minis,what", [(b"\xc0\x02", b"\x04", "block size"), (b"\x80\x02", b"\x10", "multiple of 32"), (b"\x80\x02", b"\x03", "multiple of 32")])
def test_bad_block_layout(block, minis, what):
    raw, chunk, at, _ = corrupt_case()
    chunk[at: at + 3] = block + minis
    assert what in refused(raw, chunk)


@pytest.mark.parametrize("total", [N_CORRUPT - 1, N_CORRUPT + 1])
def test_total_count_other_than_the_non_null_count(total):
    raw, chunk, at, _ = corrupt_case()
    assert len(varint(total)) == len(varint(N_CORRUPT))
    chunk[at + 3: at + 3 + len(varint(total))] = varint(total)
    assert "values, the page" in refused(raw, chunk)


def test_miniblocks_that_overrun_their_page():
    raw, chunk, _, widths = corrupt_case()
    chunk[widths: widths + 4] = bytes([64] * 4)
    assert "overruns its page" in refused(raw, chunk)


def test_stream_that_ends_before_its_page():
    raw, chunk, _, widths = corrupt_case()
    w = chunk[widths]
    assert 0 < w < 64
    chunk[widths] = w - 8 if w > 8 else 0          # a narrower first miniblock: the stream ends bytes before the page does
    assert "ends" in refused(raw, chunk)


@pytest.mark.parametrize("cut", [1, 7, 100, 2000])
@pytest.mark.parametrize("encoding", list(ENCODINGS))
def test_truncated_chunks_are_invalid(cut, encoding):
    raw = write(delta_table(5000, 1, True), encoding, "2.0", 1 << 20)

    def shorten(cols):
        cols[0].chunk_len -= cut
    rc, msg = inspect_raw(raw, 0, shorten)
    assert rc == 1, msg
