"""Where the device waits during a resident Q1 step.

Takes a torch.profiler trace (CUDA activities) of three resident Q1 steps exactly as bench.py runs them and prints, per step:
the gaps between the fused launches (the kernels longer than 1 ms), the device-idle time inside the step and the stream drains
the library made (gpu.host_syncs).  A step's window is its host-side duration: it begins when the operator chain is created
and ends when the result is on the host, so host work before the first launch counts as idle time.

  python scripts/step_idle.py [--sf 50] [--chunk-sf 10] [--steps 3] [--trace DIR]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def busy_in(intervals, lo, hi):
    """length of the union of [s, e) intervals clipped to [lo, hi)"""
    total, cur_s, cur_e = 0.0, None, None
    for s, e in sorted((max(s, lo), min(e, hi)) for s, e in intervals if e > lo and s < hi):
        if cur_e is None or s > cur_e:
            if cur_e is not None:
                total += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    if cur_e is not None:
        total += cur_e - cur_s
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=50.0)
    ap.add_argument("--chunk-sf", type=float, default=10.0)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--trace", default=None, help="directory for the Chrome trace (default: a temporary directory)")
    args = ap.parse_args()

    import tempfile
    import bench
    bench.private_jit_cache()
    import torch
    from torch.profiler import ProfilerActivity, profile, record_function
    from datagen import tpch_gpu
    from sail_b200 import engine

    ctx = engine.Context(0)
    total_sf, chunks = bench.shard_chunks(args.sf, args.chunk_sf, 0, 1)
    gens = [tpch_gpu.generate_buffers(total_sf, f, n, (), bench.Q1_COLS, 0)[1] for f, n in chunks]
    devs = [g.device_batch(ctx) for g in gens]
    schema = gens[0].schema
    specs = bench.q1_specs()
    for _ in range(args.warmup):
        bench.run_query(ctx, specs, devs, schema)
    ctx.synchronize()
    torch.cuda.synchronize()

    syncs = []
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            with record_function(f"q1_step_{i}"):
                bench.run_query(ctx, specs, devs, schema)
            syncs.append(bench.LAST_METRICS.get("gpu.host_syncs"))
        ctx.synchronize()
    out_dir = args.trace or tempfile.mkdtemp(prefix="step_idle_")
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "q1_steps.json")
    prof.export_chrome_trace(path)
    events = json.load(open(path))["traceEvents"]

    steps = sorted((e["ts"], e["ts"] + e["dur"]) for e in events
                   if e.get("ph") == "X" and e.get("cat") == "user_annotation" and str(e.get("name", "")).startswith("q1_step_"))
    dev = [e for e in events if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    busy = [(e["ts"], e["ts"] + e["dur"]) for e in dev]
    rows = []
    for i, (lo, hi) in enumerate(steps):
        fused = sorted((e["ts"], e["ts"] + e["dur"]) for e in dev if e.get("cat") == "kernel" and e["dur"] > 1000 and lo <= e["ts"] < hi)
        gaps = [round(fused[j + 1][0] - fused[j][1], 1) for j in range(len(fused) - 1)]
        b = busy_in(busy, lo, hi)
        row = {"step": i, "step_ms": round((hi - lo) / 1e3, 3), "device_busy_ms": round(b / 1e3, 3), "device_idle_ms": round((hi - lo - b) / 1e3, 3),
               "fused_launches": len(fused), "fused_gaps_us": gaps,
               "tail_idle_ms": round(((hi - lo - b) - sum(gaps)) / 1e3, 3), "host_syncs": syncs[i]}
        rows.append(row)
        print(json.dumps(row))
    print(json.dumps({"device": torch.cuda.get_device_name(0), "trace": path,
                      "mean_device_idle_ms": round(sum(r["device_idle_ms"] for r in rows) / max(1, len(rows)), 3)}))


if __name__ == "__main__":
    main()
