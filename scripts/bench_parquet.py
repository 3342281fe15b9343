"""The scan in front of the path (SURVEY.md section 8 f2): one Parquet row group of TPC-H lineitem (the seven Q1 columns),
uncompressed or ZSTD level 3 (Sail's writer default) -> Arrow batch in HBM -> Q1, three ways:
  (a) sailgpu_parquet_decode: the column chunks cross PCIe as stored, ZSTD pages are decompressed and pages / dictionaries /
      RLE runs are decoded on the GPU;
  (b) pyarrow's CPU reader (all host threads) -> Arrow table -> packed host ingest (sailgpu_op_push);
  (c) (b) without the GPU: pyarrow reader + the C port of Q1 on the host cores.
All three must give the same Q1 result.  With zstd, leg (a) is split into the decompression launch and the image read-back
(CUDA events inside the library, best run) and the rest.
usage: python scripts/bench_parquet.py [sf] [reps] [none|zstd]"""
import io
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pyarrow as pa  # noqa: E402
import pyarrow.parquet as pq  # noqa: E402
import bench  # noqa: E402
from datagen import tpch  # noqa: E402
from sail_b200 import engine, plans  # noqa: E402


def main():
    sf = float(sys.argv[1]) if len(sys.argv) > 1 else 2.0
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    codec = sys.argv[3] if len(sys.argv) > 3 else "none"
    assert codec in ("none", "zstd"), codec
    t = tpch.lineitem(sf, bench.Q1_COLS, strings="utf8").combine_chunks()
    files = {}
    for c in sorted({"none", codec}):
        buf = io.BytesIO()
        pq.write_table(t, buf, compression=c, compression_level=3 if c == "zstd" else None, row_group_size=t.num_rows, use_dictionary=True,
                       data_page_size=1 << 20)
        files[c] = buf.getvalue()
        print("parquet_file", json.dumps({"codec": c, "bytes": len(files[c])}), flush=True)
    raw = files[codec]
    ctx = engine.default_context()
    specs = bench.q1_specs()
    pa.set_cpu_count(bench.host_cores())

    def q1_dev(dev):
        out, *_ = bench.run_query(ctx, specs, [dev], dev.schema)
        return out

    def leg_gpu_decode():
        dev = engine.parquet_decode(raw, ctx=ctx)
        return q1_dev(dev)

    def leg_cpu_decode():
        tab = pq.read_table(io.BytesIO(raw), read_dictionary=[]).combine_chunks()      # Utf8 strings, as the reader delivers them
        out, *_ = bench.run_query(ctx, specs, None, tab.schema, host_chunks=[tab.to_batches()[0]])
        return out

    def leg_cpu_only():
        tab = pq.read_table(io.BytesIO(raw)).combine_chunks()
        from oracle import cpipelines
        return cpipelines.q1(tab.cast(pa.schema([pa.field(f.name, pa.string_view() if pa.types.is_string(f.type) else f.type) for f in tab.schema])), plans.days("1998-09-24"), bench.host_cores())

    res = {"sf": sf, "rows": t.num_rows, "codec": codec, "parquet_bytes": len(raw), "arrow_bytes": t.nbytes}
    outs = {}
    for name, fn in (("gpu_page_decode", leg_gpu_decode), ("cpu_reader_plus_packed_ingest", leg_cpu_decode), ("cpu_reader_plus_cpu_q1", leg_cpu_only)):
        ts, zs = [], []
        for r in range(reps + 1):
            ctx.synchronize()
            t0 = time.perf_counter()
            outs[name] = fn()
            ctx.synchronize()
            ts.append(time.perf_counter() - t0)
            if name == "gpu_page_decode":
                zs.append(engine.parquet_stats(ctx))
        best = min(ts[1:])
        res[name] = {"ms": round(best * 1e3, 2), "rows_per_s": t.num_rows / best, "parquet_GBps": len(raw) / best / 1e9}
        if name == "gpu_page_decode" and codec == "zstd":
            k = 1 + ts[1:].index(best)
            z = zs[k]
            res[name].update({"zstd_pages": z["zstd_pages"], "decompress_ms": round(z["decompress_ms"], 3),
                              "decompressed_GBps": z["zstd_out_bytes"] / (z["decompress_ms"] * 1e-3) / 1e9 if z["decompress_ms"] else None,
                              "image_bytes": z["image_bytes"], "readback_ms": round(z["readback_ms"], 3),
                              "rest_ms": round(best * 1e3 - z["decompress_ms"] - z["readback_ms"], 2)})
        print(name, json.dumps(res[name]), flush=True)
    a = sorted(map(tuple, [list(r.values()) for r in outs["gpu_page_decode"].to_pylist()]))
    b = sorted(map(tuple, [list(r.values()) for r in outs["cpu_reader_plus_packed_ingest"].to_pylist()]))
    assert a == b, "Q1 over the GPU-decoded row group differs from Q1 over pyarrow's decode"
    bench.check_result(outs["gpu_page_decode"], bench.merge_q1_rows([outs["cpu_reader_plus_cpu_q1"]]))
    res["parity"] = "ok: Q1 over the GPU-decoded row group == Q1 over pyarrow's decode == the C port"
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
