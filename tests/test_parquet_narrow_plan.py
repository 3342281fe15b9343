"""CPU test of the host half of the Parquet decoder (sail_b200/csrc/parquet.cu) on the column kinds ClickBench's hits table is
stored as: INT32 columns annotated INT(8|16, signed|unsigned), decoded to Int8 / Int16 / UInt8 / UInt16, and BYTE_ARRAY columns
without a UTF8 annotation, read with `binary_as_string`.  The page and run walk must account for every value pyarrow's metadata
reports, in uncompressed and ZSTD files alike; what stays out of the GPU path stays refused; and the reference's view over the
stored hits table validates to the schema of datagen/hits.py."""
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from sail_b200 import clickbench as cb, engine
from tests.test_gpu_parquet_clickbench import CODECS, LAYOUTS, narrow_table, write
from tests.util import oracle_op


def walk(raw):
    names = pq.ParquetFile(io.BytesIO(raw)).schema_arrow.names
    return {name: engine.parquet_inspect(raw, i, binary_as_string=True) for i, name in enumerate(names)}


@pytest.mark.parametrize("n", [1, 3, 70001])
@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("version,use_dict,page", LAYOUTS)
@pytest.mark.parametrize("codec,level", CODECS)
def test_page_and_run_walk_accounts_for_every_value(n, nulls, version, use_dict, page, codec, level):
    t = narrow_table(n, 11 + n, nulls)
    raw = write(t, version, use_dict, page, codec, level)
    infos = walk(raw)
    for name, info in infos.items():
        col = t.column(name)
        assert info["dense"] == n - col.null_count, (name, info)
        assert info["level_values"] == n, (name, info)            # every column is `optional`: one definition level per row
        if not use_dict:
            assert info["dict_pages"] == 0 and info["index_values"] == 0, (name, info)
        else:
            assert info["index_values"] <= info["dense"], (name, info)
            if not info["plain_pages"]:
                assert info["index_values"] == info["dense"] and info["dict_count"] == len(set(col.drop_null().to_pylist())), (name, info)
        if pa.types.is_binary(col.type) and info["plain_pages"] and not info["dict_pages"]:
            assert info["plain_strings"] == info["dense"], (name, info)
    if codec == "zstd":
        # the decompressed pages are the pages of the uncompressed file: same walk, same bodies
        assert infos == walk(write(t, version, use_dict, page, "none", None)), "ZSTD walk differs from the uncompressed one"


def test_the_grid_reaches_dictionary_fallback_and_both_page_kinds():
    t = narrow_table(70001, 11 + 70001, True)
    dict_file = walk(write(t, "1.0", True, 1 << 20, "none", None))
    assert dict_file["bu"]["dict_pages"] and dict_file["bu"]["plain_pages"], dict_file["bu"]      # outgrows its dictionary
    assert dict_file["u16"]["dict_pages"] and dict_file["u16"]["plain_pages"], dict_file["u16"]
    assert dict_file["flag"]["dict_pages"] and not dict_file["flag"]["plain_pages"], dict_file["flag"]
    assert dict_file["b"]["dict_pages"] and not dict_file["b"]["plain_pages"], dict_file["b"]
    plain_file = walk(write(t, "2.0", False, 4096, "none", None))
    assert all(info["pages"] > 1 and info["plain_pages"] for info in plain_file.values()), plain_file


def test_binary_without_binary_as_string_is_refused():
    raw = write(narrow_table(100, 1, False).select(["i16", "b"]), "1.0", True, 1 << 20, "none", None)
    assert engine.parquet_inspect(raw, 0, columns=["i16"])["dense"] == 100          # the Int16 column needs no flag
    with pytest.raises(engine.SailGpuError) as e:
        engine.parquet_inspect(raw, 0, columns=["b"])
    assert e.value.code == 2
    assert engine.parquet_inspect(raw, 0, columns=["b"], binary_as_string=True)["dense"] == 100


def _inspect_as(raw, column: int, arrow_type):
    """the walk of `column` with the Arrow target replaced by `arrow_type` (what a caller could ask the C ABI for)"""
    import ctypes
    buf, schema, cols, n_rows = engine._parquet_descriptors(raw, 0, None, True)
    schema = schema.set(column, pa.field(schema.field(column).name, arrow_type))
    cschema = engine._export_schema(schema)
    out = ctypes.create_string_buffer(1024)
    rc = engine.lib().sailgpu_parquet_inspect(ctypes.addressof(cschema), ctypes.addressof(cols), len(cols), n_rows, column, out, 1024)
    engine._release_schema(cschema)
    del buf
    return rc, out.value.decode()


@pytest.mark.parametrize("target", [pa.int8(), pa.int16(), pa.uint8(), pa.uint16()])
def test_int64_to_a_narrow_type_is_refused(target):
    raw = write(pa.table({"k": pa.array(np.arange(50, dtype=np.int64))}), "1.0", True, 1 << 20, "none", None)
    rc, msg = _inspect_as(raw, 0, target)
    assert rc == 2, msg
    assert _inspect_as(raw, 0, pa.int64())[0] == 0


def test_int32_narrow_targets_are_accepted_and_bool_is_not():
    raw = write(pa.table({"k": pa.array(np.arange(50, dtype=np.int32))}), "1.0", True, 1 << 20, "none", None)
    for target in (pa.int8(), pa.int16(), pa.uint8(), pa.uint16(), pa.int32(), pa.date32()):
        rc, msg = _inspect_as(raw, 0, target)
        assert rc == 0, (target, msg)
    assert _inspect_as(raw, 0, pa.bool_())[0] == 2


@pytest.mark.parametrize("col", [pa.array([True, False, None] * 10), pa.array(np.arange(30, dtype=np.float32))], ids=["BOOLEAN", "FLOAT"])
def test_boolean_and_float_columns_stay_refused(col):
    raw = write(pa.table({"c": col}), "1.0", True, 1 << 20, "none", None)
    with pytest.raises(engine.SailGpuError) as e:
        engine.parquet_inspect(raw, 0)
    assert e.value.code == 2


def test_int96_columns_stay_refused():
    t = pa.table({"ts": pa.array(np.arange(30, dtype=np.int64) * 10**9, type=pa.timestamp("ns"))})
    buf = io.BytesIO()
    pq.write_table(t, buf, use_deprecated_int96_timestamps=True, compression="none")
    assert pq.ParquetFile(io.BytesIO(buf.getvalue())).metadata.row_group(0).column(0).physical_type == "INT96"
    rc, msg = _inspect_as(buf.getvalue(), 0, pa.int64())
    assert rc == 2, msg


# ---- the reference's view over the stored hits table ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def stored():
    from datagen import hits as gen
    table = gen.hits(3000, seed=7)
    buf = io.BytesIO()
    pq.write_table(gen.stored(table), buf, compression="zstd", compression_level=3, row_group_size=1000)
    return table, buf.getvalue()


def test_stored_types_are_the_reference_schema(stored):
    _, raw = stored
    f = pq.ParquetFile(io.BytesIO(raw))
    s = f.schema_arrow
    assert s.field("EventDate").type == pa.uint16() and s.field("URL").type == pa.binary() and s.field("IsRefresh").type == pa.int16()
    col = {f.schema.column(i).name: f.schema.column(i) for i in range(len(s))}
    assert col["EventDate"].physical_type == "INT32" and col["EventDate"].logical_type.to_json() == '{"Type": "Int", "bitWidth": 16, "isSigned": false}'
    assert col["IsRefresh"].physical_type == "INT32" and col["IsRefresh"].logical_type.to_json() == '{"Type": "Int", "bitWidth": 16, "isSigned": true}'
    assert col["URL"].physical_type == "BYTE_ARRAY" and col["URL"].logical_type.type == "NONE"


def test_view_over_the_stored_table_validates_to_the_generator_schema(stored):
    table, raw = stored
    _, scanned, _, _ = engine._parquet_descriptors(raw, 0, None, True)      # the schema the GPU scan decodes to
    read = pq.read_table(io.BytesIO(raw))
    read = pa.table([c.cast(pa.string_view()) if pa.types.is_binary(c.type) else c for c in read.columns], names=read.schema.names)
    assert read.schema.names == scanned.names and [f.type for f in read.schema] == [f.type for f in scanned]
    names = scanned.names
    for cols in (names[:12], names[12:]):                     # a projection has at most 24 outputs
        spec = cb.view(cols)
        got = engine.validate(spec, [pa.schema([scanned.field(c) for c in cols])])
        want = table.schema
        assert got.names == cols
        assert [str(f.type) for f in got] == [str(want.field(c).type) for c in cols]
        # the oracle agrees on the types, and on the values: the view over the stored file is the generated table
        out = oracle_op(spec, read.select(cols))
        assert [str(f.type) for f in out.schema] == [str(f.type) for f in got]
        for name in cols:
            assert out.column(name).combine_chunks().equals(table.column(name).combine_chunks()), name


@pytest.mark.parametrize("name", list(cb.QUERIES))
def test_every_plan_over_the_view_is_accepted_with_the_oracle_schema(name, stored):
    """tests/test_clickbench.py's plan-time check, with every scan reading the stored table through the view"""
    _, raw = stored
    read = pq.read_table(io.BytesIO(raw))
    read = pa.table([c.cast(pa.string_view()) if pa.types.is_binary(c.type) else c for c in read.columns], names=read.schema.names)
    seen = []

    def walk(node):
        if node.spec["op"] == "scan":
            return read.select(node.spec["columns"]).slice(0, 2000)
        ins = [walk(c) for c in node.inputs]
        out = oracle_op(node.spec, *ins)
        got = engine.validate(node.spec, [t.schema for t in ins])
        assert got.names == out.schema.names and [str(f.type) for f in got] == [str(f.type) for f in out.schema], (node.spec["op"], got, out.schema)
        seen.append(node.spec["op"])
        return out
    q = cb.QUERIES[name]
    for i in range(q.parts):
        walk(cb.over_view(q.plan(part=i) if q.parts > 1 else q.plan()))
    assert seen.count("projection") >= 1


def test_every_walk_of_the_stored_table_is_accepted(stored):
    table, raw = stored
    md = pq.ParquetFile(io.BytesIO(raw)).metadata
    assert md.num_row_groups == 3
    for g in range(md.num_row_groups):
        for i, name in enumerate(table.schema.names):
            info = engine.parquet_inspect(raw, i, row_group=g, binary_as_string=True)
            assert info["dense"] == md.row_group(g).num_rows, (g, name, info)
