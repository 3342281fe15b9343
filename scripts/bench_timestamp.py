"""Timestamps on the GPU: the wall-clock functions' projection over resident microsecond timestamps, interpreted and specialised,
against the card's streaming read, and ClickBench [18] / [42] over resident hits rows with parity against their SQL in pandas.

    python scripts/bench_timestamp.py [rows=200000000] [hits_rows=10000000]

Prints one JSON object per measurement.  The projection is date_trunc('minute', ts), date_part('minute', ts), date_part('hour', ts):
the algorithm needs 8 B in and 8 + 4 + 4 B out per row.  Its time is the operator's (push of a resident batch, the pipeline kernel,
the hand-off of the device result) by CUDA events on the library's stream, best of five after a warm-up."""
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    """name and power limit of the card, read-only"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as e:                 # noqa: BLE001 -- reported, not fatal
        return {"error": f"{type(e).__name__}: {e}"[:200]}


def stream_read():
    with tempfile.TemporaryDirectory(prefix="sailgpu_stream_") as d:
        exe = os.path.join(d, "stream_read")
        subprocess.run(["/usr/local/cuda/bin/nvcc", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, os.path.join(ROOT, "scripts", "stream_read.cu")], check=True)
        rows = [json.loads(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines() if x.startswith("{")]
    return max(r["GBps"] for r in rows)


def projection(n):
    import pyarrow as pa
    import torch
    from sail_b200 import engine
    ctx = engine.default_context()
    stream = torch.cuda.ExternalStream(ctx.stream())
    g = torch.Generator(device="cuda").manual_seed(1)
    ts = torch.randint(1_300_000_000_000_000, 1_400_000_000_000_000, (n,), dtype=torch.int64, device="cuda", generator=g)
    schema = pa.schema([pa.field("t", pa.timestamp("us", tz="UTC"), nullable=False)])
    dev = engine.device_batch_from_buffers(schema, n, [ts], ctx)
    arg = {"col": 0}
    spec = {"op": "projection", "exprs": [{"expr": {"fn": "date_trunc", "part": "minute", "args": [arg]}, "name": "m"},
                                          {"expr": {"fn": "date_part", "part": "minute", "args": [arg]}, "name": "pm"},
                                          {"expr": {"fn": "date_part", "part": "hour", "args": [arg]}, "name": "ph"}]}
    # the same bytes in and out without the timestamp ops: what the kernel costs when the arithmetic is a copy and two narrowings
    i64 = {"cast": arg, "to": "Int64"}
    plain = {"op": "projection", "exprs": [{"expr": i64, "name": "m"}, {"expr": {"cast": i64, "to": "Int32"}, "name": "pm"},
                                           {"expr": {"cast": {"op": "+", "l": i64, "r": {"lit": 1, "type": "Int64"}}, "to": "Int32"}, "name": "ph"}]}
    out = {}
    for kernel in ("interpreted", "specialised"):
        for label, sp in ((kernel, spec), (kernel + "_same_width_without_timestamp_ops", plain)):
            if kernel == "interpreted":
                os.environ["SAILGPU_JIT"] = "0"
            else:
                os.environ.pop("SAILGPU_JIT", None)
                os.environ["SAILGPU_JIT_MIN_ROWS"] = "0"
            best, jit = 1e30, 0
            for rep in range(6):
                op = engine.GpuExec(sp, [schema], ctx)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ctx.synchronize()
                a.record(stream)
                op.push(dev.borrow())
                op.finish()
                res = op.collect_device(handle=True)
                b.record(stream)
                b.synchronize()
                jit = op.metrics().get("gpu.jit_launches", 0)
                op.close()
                del res
                if rep:                                  # the first run warms up (and, specialised, compiles the kernel)
                    best = min(best, a.elapsed_time(b))
            gbps = n * (8 + 8 + 4 + 4) / best / 1e6
            out[label] = {"ms": round(best, 3), "GBps": round(gbps, 1), "jit_launches": jit}
    return out


def clickbench(n):
    import pyarrow as pa
    from datagen import hits as gen
    from sail_b200 import clickbench as cb, engine, plans
    from tests import clickbench_sql as sql
    from tests.test_clickbench import as_table
    from tests.test_gpu_parquet_clickbench import host
    from tests.test_gpu_timestamp import sql18, sql42
    from tests.util import assert_topk
    table = gen.hits(n, seed=7)
    frame = sql.frame(table)
    res = {}
    for name, q in cb.TIMESTAMP_QUERIES.items():
        node = cb.top_sort(q.plan())
        cols = sorted({c for s in _scans(node) for c in s})
        dev = engine.to_device(table.select(cols))
        tables = {"hits": (dev, cols)}
        times = []
        for _ in range(4):
            engine.default_context().synchronize()
            t0 = time.perf_counter()
            out = plans.execute_gpu(node, tables)
            engine.default_context().synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
        got = host(out, out[0].schema)
        try:
            assert_topk(got, as_table({"c18": sql18, "c42": sql42}[name](frame), got.schema), list(q.order), node.spec["fetch"])
            parity = "ok" if got.slice(q.skip).num_rows > 0 else "empty after OFFSET"
        except AssertionError as e:
            parity = f"MISMATCH: {str(e)[:200]}"
        res[name] = {"rows": n, "ms_best": round(min(times[1:]), 2), "parity": parity}
    return res


def _scans(node):
    if node.spec["op"] == "scan":
        return [node.spec["columns"]]
    return [c for i in node.inputs for c in _scans(i)]


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 200_000_000
    hits_rows = int(sys.argv[2]) if len(sys.argv) > 2 else 10_000_000
    print(json.dumps({"card": card()}), flush=True)
    sr = stream_read()
    proj = projection(n)
    for k, v in proj.items():
        v["of_stream_read"] = round(v["GBps"] / sr, 3)
    print(json.dumps({"projection_rows": n, "stream_read_GBps": sr, **proj}), flush=True)
    print(json.dumps({"clickbench": clickbench(hits_rows)}), flush=True)


if __name__ == "__main__":
    main()
