"""ZSTD-compressed Parquet chunks decoded on the device (parquet_zstd_decompress_kernel, then the uncompressed path over the
decompressed image) against pyarrow's reader, bit-exact: the page grid of test_gpu_parquet.py at levels 1 and 19, one call
with hundreds of compressed pages, ZSTD and uncompressed columns in one row group, and Q1 over a ZSTD lineitem row group."""
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from tests.test_gpu_parquet import host, table

pytestmark = pytest.mark.gpu


def assert_same(got, want):
    assert got.num_rows == want.num_rows
    for name in want.schema.names:
        w = want.column(name).combine_chunks()
        g = got.column(name).combine_chunks()
        if pa.types.is_string(w.type):
            g = g.cast(pa.string())
        assert g.equals(w), name


@pytest.mark.parametrize("level", [1, 19])
@pytest.mark.parametrize("n", [0, 1, 1000, 70001])
@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("version,use_dict,page", [("1.0", True, 1 << 20), ("1.0", False, 4096), ("2.0", True, 8192), ("2.0", False, 1 << 20)])
def test_zstd_decode_matches_pyarrow(level, n, nulls, version, use_dict, page):
    from sail_b200 import engine
    t = table(n, 7 + n, nulls)
    buf = io.BytesIO()
    pq.write_table(t, buf, compression="zstd", compression_level=level, use_dictionary=use_dict, data_page_version=version, data_page_size=page,
                   dictionary_pagesize_limit=1 << 14)
    raw = buf.getvalue()
    assert_same(host(engine.parquet_decode(raw)), pq.read_table(io.BytesIO(raw)))


def wide_table(n):
    rng = np.random.default_rng(17)
    return pa.table({
        "a": pa.array(rng.integers(0, 1 << 50, n), type=pa.int64()),
        "b": pa.array(rng.integers(0, 1000, n), type=pa.int64(), mask=rng.random(n) < 0.1),
        "c": pa.array(np.arange(n, dtype=np.int64) // 7),
        "d": pa.array(rng.integers(0, 1 << 30, n).astype(np.int32)),
        "e": pa.array(rng.integers(0, 20, n).astype(np.int32)),
        "f": pa.array(rng.normal(size=n)),
        "g": pa.array(np.round(rng.random(n) * 100, 2)),
        "h": pa.array(np.array(["R", "A", "N", "longer than twelve bytes"])[rng.integers(0, 4, n)], type=pa.string()),
    })


def test_one_call_decompresses_hundreds_of_pages():
    from sail_b200 import engine
    t = wide_table(2_000_000)
    buf = io.BytesIO()
    pq.write_table(t, buf, compression="zstd", compression_level=3, row_group_size=t.num_rows, data_page_size=1 << 20)
    raw = buf.getvalue()
    ctx = engine.default_context()
    dev = engine.parquet_decode(raw, ctx=ctx)
    stats = engine.parquet_stats(ctx)
    assert stats["zstd_pages"] >= 200, stats
    assert stats["zstd_out_bytes"] > 0 and stats["decompress_ms"] > 0, stats
    assert_same(host(dev), pq.read_table(io.BytesIO(raw)))


def test_zstd_and_uncompressed_columns_in_one_row_group():
    from sail_b200 import engine
    t = table(70001, 9, True)
    codecs = {name: ("zstd" if i % 2 == 0 else "none") for i, name in enumerate(t.schema.names)}
    buf = io.BytesIO()
    pq.write_table(t, buf, compression=codecs, data_page_size=8192, dictionary_pagesize_limit=1 << 14)
    raw = buf.getvalue()
    md = pq.ParquetFile(io.BytesIO(raw)).metadata.row_group(0)
    assert {md.column(i).compression for i in range(md.num_columns)} == {"ZSTD", "UNCOMPRESSED"}
    ctx = engine.default_context()
    got = host(engine.parquet_decode(raw, ctx=ctx))
    assert engine.parquet_stats(ctx)["zstd_pages"] > 0
    assert_same(got, pq.read_table(io.BytesIO(raw)))
    # projection of the uncompressed columns only: no ZSTD work at all
    engine.parquet_decode(raw, columns=["small", "wide"], ctx=ctx)
    assert engine.parquet_stats(ctx)["zstd_pages"] == 0


def test_q1_over_a_zstd_lineitem_row_group():
    import bench
    from datagen import tpch
    from sail_b200 import engine
    t = tpch.lineitem(0.05, bench.Q1_COLS, strings="utf8").combine_chunks()
    ctx = engine.default_context()
    outs = []
    for codec in ("none", "zstd"):
        buf = io.BytesIO()
        pq.write_table(t, buf, compression=codec, compression_level=3 if codec == "zstd" else None, row_group_size=t.num_rows, use_dictionary=True,
                       data_page_size=1 << 20)
        dev = engine.parquet_decode(buf.getvalue(), ctx=ctx)
        out, *_ = bench.run_query(ctx, bench.q1_specs(), [dev], dev.schema)
        outs.append(sorted(map(tuple, [list(r.values()) for r in out.to_pylist()])))
    assert engine.parquet_stats(ctx)["zstd_pages"] > 0
    assert outs[0] == outs[1] and len(outs[0]) == 4
