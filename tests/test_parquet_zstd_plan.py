"""CPU test of ZSTD-compressed Parquet chunks (sail_b200/csrc/zstd.cuh, parquet.cu): sailgpu_parquet_inspect decompresses a
ZSTD chunk on the host with the decoder the device runs and walks the decompressed image.  The walk and the decompressed
page bodies must equal those of the uncompressed file of the same table; other codecs, dictionaries and corrupt pages are
refused with the right code and no crash."""
import ctypes
import io
import json

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from sail_b200 import engine
from tests.test_gpu_parquet import table

KEYS = ["pages", "dense", "dict_count", "level_values", "index_values", "level_runs", "index_runs", "plain_strings", "dict_pages",
        "plain_pages", "body_bytes", "body_fnv1a"]
ZSTD_MAGIC = b"\x28\xb5\x2f\xfd"


def write(t, compression, **kw):
    buf = io.BytesIO()
    pq.write_table(t, buf, compression=compression, **kw)
    return buf.getvalue()


def same_walk(t, level, **kw):
    plain = write(t, "none", **kw)
    packed = write(t, "zstd", compression_level=level, **kw)
    md = pq.ParquetFile(io.BytesIO(packed)).metadata.row_group(0)
    for i in range(t.num_columns):
        assert md.column(i).compression == "ZSTD"
        want, got = engine.parquet_inspect(plain, i), engine.parquet_inspect(packed, i)
        assert {k: got[k] for k in KEYS} == {k: want[k] for k in KEYS}, (t.schema.names[i], want, got)
    return packed


def page_sizes(raw):
    """(values, total_uncompressed_size) of every column chunk of row group 0, from pyarrow's metadata"""
    f = pq.ParquetFile(io.BytesIO(raw))
    return [(c.num_values, c.total_uncompressed_size) for c in [f.metadata.row_group(0).column(j) for j in range(f.metadata.num_columns)]]


def test_page_boundaries_coincide_with_the_uncompressed_file():
    t = table(70001, 5, True)
    kw = dict(use_dictionary=True, data_page_size=8192, dictionary_pagesize_limit=1 << 14)
    plain, packed = write(t, "none", **kw), write(t, "zstd", **kw)
    for i, ((nv_a, un_a), (nv_b, un_b)) in enumerate(zip(page_sizes(plain), page_sizes(packed))):
        a, b = engine.parquet_inspect(plain, i), engine.parquet_inspect(packed, i)
        assert nv_a == nv_b and a["pages"] == b["pages"] and a["body_bytes"] == b["body_bytes"]
        # the sizes count page headers too, which differ only in the varint of their compressed size: a byte or so per page
        assert abs(un_a - un_b) <= a["pages"] + a["dict_pages"]


@pytest.mark.parametrize("level", [1, 3, 9, 19])
@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("version,use_dict,page", [("1.0", True, 1 << 20), ("1.0", False, 4096), ("2.0", True, 8192), ("2.0", False, 1 << 20),
                                                   ("2.0", False, 65536)])
def test_zstd_walk_equals_uncompressed_walk(level, nulls, version, use_dict, page):
    n = 70001
    same_walk(table(n, 11 + level, nulls), level, use_dictionary=use_dict, data_page_version=version, data_page_size=page, dictionary_pagesize_limit=1 << 14)


@pytest.mark.parametrize("n", [0, 1])
def test_tiny_row_groups(n):
    for use_dict in (True, False):
        same_walk(table(n, 2, True), 3, use_dictionary=use_dict)


def block_kinds_table(n=300000):
    rng = np.random.default_rng(3)
    return pa.table({
        "random": pa.array(rng.integers(-(1 << 62), 1 << 62, n), type=pa.int64()),                 # Raw blocks / Raw literals
        "constant": pa.array(np.full(n, 42, dtype=np.int64)),                                      # RLE
        "period3": pa.array(np.tile(np.array([7, 1 << 40, -3], dtype=np.int64), n // 3 + 1)[:n]),  # matches overlapping their output
        "text": pa.array([f"row {i % 977} of {i % 13}" for i in range(n)], type=pa.string()),
        "unique": pa.array([f"u{i:08d}-{'z' * (i % 5)}" for i in rng.permutation(n)], type=pa.string()),  # outgrows its dictionary
    })


@pytest.mark.parametrize("level", [1, 3, 19])
@pytest.mark.parametrize("version", ["1.0", "2.0"])
def test_every_block_and_literal_kind(level, version):
    t = block_kinds_table()
    # 1 MiB pages: every page of the int64 columns is larger than a 128 KiB block, so frames hold several blocks
    same_walk(t, level, use_dictionary=["text", "unique"], data_page_version=version, data_page_size=1 << 20, dictionary_pagesize_limit=1 << 16)
    raw = write(t, "none", use_dictionary=["text", "unique"], data_page_version=version, data_page_size=1 << 20, dictionary_pagesize_limit=1 << 16)
    assert engine.parquet_inspect(raw, 4)["plain_pages"] == 1 and engine.parquet_inspect(raw, 4)["dict_pages"] == 1   # the fallback happened


@pytest.mark.parametrize("codec", ["gzip", "lz4", "brotli"])
def test_other_codecs_are_refused(codec):
    raw = write(table(100, 1, False), codec)
    with pytest.raises(engine.SailGpuError) as e:
        engine.parquet_inspect(raw, 0)
    assert e.value.code == 2


def first_frame(raw, column):
    cm = pq.ParquetFile(io.BytesIO(raw)).metadata.row_group(0).column(column)
    start = min(x for x in (cm.dictionary_page_offset, cm.data_page_offset) if x is not None)
    at = raw.index(ZSTD_MAGIC, start)
    assert at < start + cm.total_compressed_size
    return at


def test_dictionary_frames_are_refused_at_plan_time():
    raw = bytearray(write(table(5000, 2, False), "zstd"))
    at = first_frame(bytes(raw), 0)
    raw[at + 4] |= 0x03                           # Dictionary_ID_flag: a 4-byte dictionary id follows the descriptor
    with pytest.raises(engine.SailGpuError) as e:
        engine.parquet_inspect(bytes(raw), 0)
    assert e.value.code == 2


def first_block(raw, at):
    """offset and (type, size) of the first block of the frame at `at`"""
    fhd = raw[at + 4]
    single = (fhd >> 5) & 1
    fcs = [1 if single else 0, 2, 4, 8][fhd >> 6]
    h = at + 5 + (0 if single else 1) + fcs
    bh = int.from_bytes(raw[h:h + 3], "little")
    return h + 3, (bh >> 1) & 3, bh >> 3


@pytest.mark.parametrize("column", [1, 4, 5])
def test_flipped_bytes_inside_a_block_are_corrupt(column):
    raw = bytearray(write(table(20000, 4, False), "zstd", use_dictionary=False))
    start, kind, size = first_block(raw, first_frame(bytes(raw), column))
    assert kind == 2 and size > 64              # a Compressed block: Huffman literals and FSE sequences
    for k in range(size // 2, size // 2 + 8):
        raw[start + k] ^= 0xA5
    with pytest.raises(engine.SailGpuError) as e:
        engine.parquet_inspect(bytes(raw), column)
    assert e.value.code == 1
    assert "ZSTD page" in str(e.value) and f"column '{table(1, 0, False).schema.names[column]}'" in str(e.value)


def inspect_raw(raw, column, mutate):
    """sailgpu_parquet_inspect on descriptors the test changes first"""
    buf, schema, cols, n_rows = engine._parquet_descriptors(raw, 0, None)
    mutate(cols)
    cschema = engine._export_schema(schema)
    out = ctypes.create_string_buffer(1024)
    rc = engine.lib().sailgpu_parquet_inspect(ctypes.addressof(cschema), ctypes.addressof(cols), len(cols), n_rows, column, out, 1024)
    engine._release_schema(cschema)
    del buf
    return rc, out.value.decode()


@pytest.mark.parametrize("cut", [1, 7, 100, 5000])
def test_truncated_chunks_are_invalid(cut):
    raw = write(table(20000, 6, False), "zstd", use_dictionary=False, data_page_size=1 << 20)

    def shorten(cols):
        cols[0].chunk_len -= cut
    rc, msg = inspect_raw(raw, 0, shorten)
    assert rc == 1, msg


def thrift_page_header(uncompressed, compressed, num_values):
    """a compact-protocol PageHeader of a data page V1, PLAIN values, RLE levels"""
    def varint(v):
        out = bytearray()
        while True:
            b = v & 0x7F
            v >>= 7
            out.append(b | (0x80 if v else 0))
            if not v:
                return bytes(out)

    def i32(delta, v):
        return bytes([(delta << 4) | 5]) + varint((v << 1) ^ (v >> 31))
    inner = i32(1, num_values) + i32(1, 0) + i32(1, 3) + i32(1, 3) + b"\x00"
    return i32(1, 0) + i32(1, uncompressed) + i32(1, compressed) + bytes([(2 << 4) | 12]) + inner + b"\x00"


def test_page_of_several_concatenated_frames():
    n = 50000
    t = pa.table({"v": pa.array(np.arange(n, dtype=np.int64) * 7 % 1000, type=pa.int64())}, schema=pa.schema([pa.field("v", pa.int64(), nullable=False)]))
    plain = write(t, "none", use_dictionary=False, data_page_size=1 << 22)
    body = t.column(0).to_numpy().tobytes()
    codec = pa.Codec("zstd", compression_level=3)
    frames = b"".join(codec.compress(body[a:b], asbytes=True) for a, b in [(0, 1000), (1000, 200000), (200000, len(body))])
    chunk = thrift_page_header(len(body), len(frames), n) + frames
    keep = ctypes.create_string_buffer(chunk, len(chunk))

    def point_at_frames(cols):
        cols[0].chunk = ctypes.addressof(keep)
        cols[0].chunk_len = len(chunk)
        cols[0].codec = 6
    rc, msg = inspect_raw(plain, 0, point_at_frames)
    assert rc == 0, msg
    got, want = json.loads(msg), engine.parquet_inspect(plain, 0)
    assert got["body_bytes"] == want["body_bytes"] == len(body) and got["body_fnv1a"] == want["body_fnv1a"]
