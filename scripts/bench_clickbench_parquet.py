"""ClickBench fed by the Parquet scan: the synthetic hits table (datagen/hits.py) stored the way the reference stores it (Int16
columns, EventDate as UInt16, strings as binary; datagen/hits.py:stored), in row groups of 1 Mi rows, ZSTD level 3 (Sail's writer
default) or uncompressed, then two legs over the columns the 37 planned queries read:
  (a) sailgpu_parquet_decode of every row group (`binary_as_string`) -> the 37 queries, each scan read through the reference's
      view (sail_b200.clickbench.over_view), every intermediate in HBM;
  (b) pyarrow's CPU reader (all host threads), binary cast to string_view -> packed host ingest (sailgpu_op_push) -> the same
      37 queries through the same view.
Leg (a) must give leg (b)'s result on every query (ORDER BY .. LIMIT up to ties cut by the LIMIT, Float64 AVG within 1e-6).
Reported: the best of `reps` runs after one warm-up, for the decode (up to resident device batches) and for the 37 queries separately; with
zstd, the decompression launch and the image read-back of that best decode, summed over its row groups (engine.parquet_stats).
Runs the interpreted pipelines (SAILGPU_JIT=0), as bench.py's ClickBench leg does: the specialised Int16 kernels have not been
parity-checked on these queries.
Layout `plain` (the default) writes what pyarrow writes by default: dictionary pages, falling back to PLAIN.  `delta` writes data
pages V2 without dictionaries, integer columns as DELTA_BINARY_PACKED and strings as DELTA_BYTE_ARRAY (datagen/hits.py:delta_encoding).
usage: python scripts/bench_clickbench_parquet.py [rows] [reps] [none|zstd] [plain|delta]"""
import collections
import io
import json
import os
import subprocess
import sys
import time

os.environ["SAILGPU_JIT"] = "0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pyarrow as pa  # noqa: E402
import pyarrow.parquet as pq  # noqa: E402
import bench  # noqa: E402
from datagen import hits as gen  # noqa: E402
from oracle import render  # noqa: E402
from sail_b200 import clickbench as cb, engine, plans  # noqa: E402
from tests import clickbench_sql as sql  # noqa: E402
from tests.test_clickbench import sql_params  # noqa: E402
from tests.util import assert_same  # noqa: E402

ROW_GROUP = 1 << 20


def card():
    """name and power limit of the card, read-only"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as e:                 # noqa: BLE001 -- reported, not fatal
        return {"error": f"{type(e).__name__}: {e}"[:200]}


def scanned_columns():
    cols = set()

    def walk(node):
        if node.spec["op"] == "scan":
            cols.update(node.spec["columns"])
        for c in node.inputs:
            walk(c)
    for q in cb.QUERIES.values():
        for i in range(q.parts):
            walk(q.plan(part=i) if q.parts > 1 else q.plan())
    return [c for c in gen.COLUMNS if c in cols]


def resident(op):
    """an operator's output as device batches the queries' scans can borrow"""
    op.finish()
    out = op.collect_device()
    for d in out:
        d.schema = op.schema
    op.close()
    return out


def as_string_view(col: pa.ChunkedArray) -> pa.ChunkedArray:
    """binary -> string_view as pyarrow casts it.  When every value of a chunk is inline (at most 12 bytes) the cast leaves a
    None data buffer behind, which pyarrow 24's C-data export dereferences; such a chunk is rebuilt without it."""
    out = []
    for a in col.cast(pa.string_view()).chunks:
        b = a.buffers()
        if any(x is None for x in b[2:]):
            a = pa.Array.from_buffers(a.type, len(a), b[:2], null_count=a.null_count, offset=a.offset)
        out.append(a)
    return pa.chunked_array(out, type=pa.string_view())


def to_host(batches, ctx):
    schema = batches[0].schema
    op = engine.GpuExec({"op": "projection", "exprs": [{"expr": {"col": i}, "name": n} for i, n in enumerate(schema.names)]}, [schema], ctx)
    for b in batches:
        op.push(b)
    op.finish()
    t = op.collect()
    op.close()
    return t


def same_up_to_ties(a: pa.Table, b: pa.Table, keys, floats):
    """two ORDER BY keys LIMIT k results: the keys agree row by row, and every tie group but the last (which the LIMIT may cut
    differently) holds the same rows; Float64 columns within 1e-6 relative"""
    assert a.schema.names == b.schema.names and a.num_rows == b.num_rows, (a.schema, b.schema, a.num_rows, b.num_rows)
    ga, gb = render.rows(a), render.rows(b)
    ki = [a.schema.names.index(k) for k in keys]
    assert [tuple(r[i] for i in ki) for r in ga] == [tuple(r[i] for i in ki) for r in gb], "ORDER BY keys differ"
    groups_a, groups_b = collections.OrderedDict(), collections.OrderedDict()
    for r in ga:
        groups_a.setdefault(tuple(r[i] for i in ki), []).append(r)
    for r in gb:
        groups_b.setdefault(tuple(r[i] for i in ki), []).append(r)
    exact = [i for i in range(a.num_columns) if i not in floats]
    for k in list(groups_a)[:-1]:
        ra = sorted(groups_a[k], key=lambda r: tuple(r[i] for i in exact))
        rb = sorted(groups_b[k], key=lambda r: tuple(r[i] for i in exact))
        for x, y in zip(ra, rb):
            for i in range(a.num_columns):
                if i in floats and x[i] != "NULL" and y[i] != "NULL":
                    assert abs(float(x[i]) - float(y[i])) <= 1e-6 * max(1.0, abs(float(y[i]))), (x, y)
                else:
                    assert x[i] == y[i], (x, y)


def main():
    rows = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    codec = sys.argv[3] if len(sys.argv) > 3 else "zstd"
    layout = sys.argv[4] if len(sys.argv) > 4 else "plain"
    assert codec in ("none", "zstd"), codec
    assert layout in ("plain", "delta"), layout
    res = {"rows": rows, "codec": codec, "row_group_rows": ROW_GROUP, "card": card()}
    if layout == "delta":
        res["layout"] = layout
    print("card", json.dumps(res["card"]), flush=True)
    cols = scanned_columns()
    t0 = time.perf_counter()
    table = gen.hits(rows, seed=11, columns=cols)
    params = sql_params(sql.frame(table.select(["CounterID", "EventDate", "IsRefresh", "TraficSourceID", "DontCountHits", "UserID", "RefererHash", "URLHash"])))
    buf = io.BytesIO()
    stored = gen.stored(table)
    kw = dict(use_dictionary=False, data_page_version="2.0", column_encoding=gen.delta_encoding(stored.schema)) if layout == "delta" else {}
    pq.write_table(stored, buf, compression=codec, compression_level=3 if codec == "zstd" else None, row_group_size=ROW_GROUP, **kw)
    del stored
    raw = buf.getvalue()
    del table
    n_groups = pq.ParquetFile(io.BytesIO(raw)).metadata.num_row_groups
    res.update({"columns": len(cols), "row_groups": n_groups, "parquet_bytes": len(raw), "prep_s": round(time.perf_counter() - t0, 1)})
    print("parquet_file", json.dumps({k: res[k] for k in ("columns", "row_groups", "parquet_bytes", "prep_s")}), flush=True)
    ctx = engine.default_context()
    pa.set_cpu_count(bench.host_cores())

    def decode_gpu():
        out, stats = [], []
        for g in range(n_groups):                  # row group by row group
            out.append(engine.parquet_decode(raw, row_group=g, ctx=ctx, binary_as_string=True))
            stats.append(engine.parquet_stats(ctx))
        return out, stats

    def decode_cpu():
        tab = pq.read_table(io.BytesIO(raw)).combine_chunks()
        tab = pa.table([as_string_view(c) if pa.types.is_binary(c.type) else c for c in tab.columns], names=tab.schema.names)
        op = engine.GpuExec({"op": "projection", "exprs": [{"expr": {"col": i}, "name": n} for i, n in enumerate(tab.schema.names)]}, [tab.schema], ctx)
        op.push(tab)
        return resident(op), []

    def plans_of(q, node_for_parity=False):
        kw = {p: params[p] for p in q.params}
        parts = [q.plan(part=i, **kw) for i in range(q.parts)] if q.parts > 1 else [q.plan(**kw)]
        return [cb.over_view((cb.top_sort(p) or p) if node_for_parity else p) for p in parts]

    def queries(dev):
        tables = {"hits": (dev, dev[0].schema.names)}
        return {name: [plans.execute_gpu(p, tables, ctx) for p in plans_of(q)] for name, q in cb.QUERIES.items()}

    def parity_results(dev):
        """per query, what tests/test_clickbench.py::check compares: the TopK node under [24]'s / [26]'s projection"""
        tables = {"hits": (dev, dev[0].schema.names)}
        return {name: [to_host(plans.execute_gpu(p, tables, ctx), ctx) for p in plans_of(q, True)] for name, q in cb.QUERIES.items()}

    results = {}
    for leg, decode in (("gpu_parquet_decode", decode_gpu), ("cpu_reader_plus_packed_ingest", decode_cpu)):
        dec_ms, q_ms, zs = [], [], []
        for r in range(reps + 1):
            ctx.synchronize()
            t0 = time.perf_counter()
            dev, stats = decode(); ctx.synchronize()
            t1 = time.perf_counter()
            out = queries(dev); ctx.synchronize()
            t2 = time.perf_counter()
            dec_ms.append((t1 - t0) * 1e3)
            q_ms.append((t2 - t1) * 1e3)
            zs.append(stats)
            if r == reps:
                results[leg] = parity_results(dev)
            del dev, out
        best = min(dec_ms[1:])
        k = 1 + dec_ms[1:].index(best)
        rec = {"decode_ms": round(best, 2), "queries_ms": round(min(q_ms[1:]), 2), "decode_runs_ms": [round(x, 1) for x in dec_ms[1:]],
               "queries_runs_ms": [round(x, 1) for x in q_ms[1:]]}
        if leg == "gpu_parquet_decode" and codec == "zstd":
            z = zs[k]
            dm, rm = sum(s["decompress_ms"] for s in z), sum(s["readback_ms"] for s in z)
            rec.update({"zstd_pages": sum(s["zstd_pages"] for s in z), "decompress_ms": round(dm, 2),
                        "decompressed_GBps": round(sum(s["zstd_out_bytes"] for s in z) / (dm * 1e-3) / 1e9, 3) if dm else None,
                        "image_bytes": sum(s["image_bytes"] for s in z), "readback_ms": round(rm, 2), "rest_ms": round(best - dm - rm, 2),
                        "per_row_group": [{"decompress_ms": round(s["decompress_ms"], 3), "readback_ms": round(s["readback_ms"], 3)} for s in z]})
        res[leg] = rec
        print(leg, json.dumps(rec), flush=True)

    parity = {}
    for name, q in cb.QUERIES.items():
        try:
            for a, b in zip(results["gpu_parquet_decode"][name], results["cpu_reader_plus_packed_ingest"][name]):
                if q.order and q.parts == 1 and cb.top_sort(q.plan()) is not None:
                    same_up_to_ties(a, b, list(q.order), q.floats)
                else:
                    assert_same(a, b, float_cols=q.floats)
            parity[name] = "ok"
        except AssertionError as e:
            parity[name] = f"FAILED: {e}"[:300]
    res["parity"] = parity
    res["parity_ok"] = sum(v == "ok" for v in parity.values())
    print(json.dumps(res), flush=True)
    if res["parity_ok"] != len(cb.QUERIES):
        sys.exit(1)


if __name__ == "__main__":
    main()
