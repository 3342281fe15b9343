"""Partitioned mode of the hash aggregate (engine.cu, PipelineOp) on one GPU.

  python scripts/bench_agg_overflow.py [--sf100-orders N] [--reps R] [--baseline-tree DIR] [--out DIR]

1. GROUP BY l_orderkey with sum and count over SF100-sized lineitem keys: 150 M orders, 1-7 rows each as dbgen makes them
   (sorted by order key, about 600 M rows), resident in HBM as batches of 50 M rows.  Past 2^28 slots: time and partitions.
2. The same at SF10 (15 M groups): the monolithic table against partitioned mode forced by SAILGPU_AGG_MAX_CAPACITY, alternated.
3. With --baseline-tree: Q1 of bench.py (--skip-cpu --skip-e2e --skip-joins --skip-suites) from this tree and from the given
   one, alternated; their --dump-outputs files are compared byte for byte.

Prints the card's name and power limit with the numbers, and one JSON line at the end (also written to DIR/agg_overflow.json)."""
import argparse
import filecmp
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import pyarrow as pa

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    return out.stdout.strip().splitlines()[0]


def lineitem_keys(n_orders, batch_rows, seed=1):
    """dbgen's l_orderkey: order o (0-based) has key (o // 8) * 32 + o % 8 + 1 and 1..7 lines; l_quantity 1..50"""
    rng = np.random.default_rng(seed)
    lines = rng.integers(1, 8, n_orders).astype(np.int64)
    o = 0
    while o < n_orders:
        c = np.cumsum(lines[o:])
        take = int(np.searchsorted(c, batch_rows, side="right")) or 1
        orders = np.arange(o, o + take, dtype=np.int64)
        keys = np.repeat((orders // 8) * 32 + orders % 8 + 1, lines[o:o + take])
        qty = rng.integers(1, 51, len(keys)).astype(np.int64)
        yield pa.table({"l_orderkey": pa.array(keys), "l_quantity": pa.array(qty)})
        o += take


SPEC = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": 0}, "name": "l_orderkey"}],
        "aggs": [{"fn": "sum", "args": [{"col": 1}], "name": "sum_qty"}, {"fn": "count", "args": [], "name": "n"}]}


def run_once(devs, schema, ctx):
    from sail_b200 import engine
    ctx.synchronize()
    t0 = time.perf_counter()
    op = engine.GpuExec(SPEC, [schema], ctx)
    for d in devs:
        op.push(d.borrow())
    op.finish()
    out = op.collect_device(handle=True)
    ctx.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    m = op.metrics()
    op.close()
    rows = sum(d.num_rows for d in out)
    del out
    return ms, rows, m


def leg(n_orders, batch_rows, reps, forced_ceiling=None):
    """-> {"orders", "rows", "default_ms": [...], "forced_ms": [...], partitions and spills of each}; the variants alternated"""
    from sail_b200 import engine
    ctx = engine.default_context()
    devs, rows, schema = [], 0, None
    for t in lineitem_keys(n_orders, batch_rows):
        schema = t.schema
        devs.append(engine.to_device(t, ctx))
        rows += t.num_rows
    res = {"orders": n_orders, "rows": rows}
    variants = [("default", None)] + ([("forced", forced_ceiling)] if forced_ceiling else [])
    for r in range(reps + 1):                     # the first round warms up every shape
        for name, ceil in variants:
            if ceil:
                os.environ["SAILGPU_AGG_MAX_CAPACITY"] = str(ceil)
            else:
                os.environ.pop("SAILGPU_AGG_MAX_CAPACITY", None)
            ms, groups, m = run_once(devs, schema, ctx)
            assert groups == n_orders, (groups, n_orders)
            if r:
                res.setdefault(name + "_ms", []).append(round(ms, 1))
                res[name + "_partitions"] = m.get("gpu.agg_partitions", 0)
                res[name + "_spills"] = m.get("gpu.agg_spills", 0)
                if m.get("gpu.agg_partition_groups"):
                    g = m["gpu.agg_partition_groups"]
                    res[name + "_partition_groups_min_max"] = [min(g), max(g)]
    os.environ.pop("SAILGPU_AGG_MAX_CAPACITY", None)
    return res


def q1_alternated(baseline, reps, out_dir):
    """bench.py's Q1 leg from this tree and from `baseline`, alternated; kernel time and dumped outputs of both"""
    res = {"new_step_ms": [], "old_step_ms": [], "new_kernel_ms": [], "old_kernel_ms": []}
    dumps = {}
    for r in range(reps):
        for tag, tree in (("new", ROOT), ("old", baseline)):
            d = os.path.abspath(os.path.join(out_dir, f"q1_dump_{tag}"))
            os.makedirs(d, exist_ok=True)
            cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", "20", "--warmup", "3", "--skip-cpu", "--skip-e2e",
                   "--skip-joins", "--skip-suites", "--dump-outputs", d]
            p = subprocess.run(cmd, cwd=tree, capture_output=True, text=True)
            assert p.returncode == 0, p.stderr[-3000:]
            line = [x for x in p.stdout.splitlines() if x.startswith("{")][-1]
            j = json.loads(line)
            res[f"{tag}_raw"] = j
            res[f"{tag}_step_ms"].append(round(j["ms_per_step"], 3))
            res[f"{tag}_kernel_ms"].append(round(j["roofline"]["kernel_ms"], 3))
            dumps[tag] = d
    a, b = dumps["new"], dumps["old"]
    names = sorted(os.listdir(a))
    res["dump_files"] = names
    res["dumps_identical"] = names == sorted(os.listdir(b)) and all(filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False) for f in names)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf100-orders", type=int, default=150_000_000)
    ap.add_argument("--sf10-orders", type=int, default=15_000_000)
    ap.add_argument("--batch-rows", type=int, default=50_000_000)
    ap.add_argument("--forced-ceiling", type=int, default=1 << 23)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--baseline-tree", default=None)
    ap.add_argument("--skip-sf100", action="store_true")
    ap.add_argument("--out", default=tempfile.mkdtemp(prefix="agg_overflow_"))
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    res = {"card": card()}
    print("card, power limit:", res["card"], flush=True)
    if a.baseline_tree:
        res["q1"] = q1_alternated(a.baseline_tree, a.reps, a.out)
        print("q1:", json.dumps(res["q1"]), flush=True)
    res["sf10"] = leg(a.sf10_orders, a.batch_rows, a.reps, a.forced_ceiling)
    print("sf10:", json.dumps(res["sf10"]), flush=True)
    if not a.skip_sf100:
        res["sf100"] = leg(a.sf100_orders, a.batch_rows, max(1, a.reps - 1))
        print("sf100:", json.dumps(res["sf100"]), flush=True)
    res["card_after"] = card()
    with open(os.path.join(a.out, "agg_overflow.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
