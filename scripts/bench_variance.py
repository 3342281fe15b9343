"""Grouped stddev(x) against avg(x) over the same resident Float64 column, in the interpreted and the specialised pipeline kernel.

    python scripts/bench_variance.py [rows=200000000]

x is normal around 1e3; k takes 4 values (the CTA-dictionary path) or about 10 M values (the global table).  avg(x) is a count
and a Float64 sum per group; stddev(x) is the same count plus two double-double sums, whose table updates are 16-byte
compare-and-swap loops.  Times are host clocks around one single-mode aggregate over resident input, ending in a device
synchronise, best of four after a warm-up.  Prints the card's name and power limit, then one JSON object per measurement with
the parity of stddev on a few groups against a two-pass Float64 computation."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.bench_timestamp import card  # noqa: E402


def timed(node, tables, reps=5):
    from sail_b200 import engine, plans
    times = []
    out = None
    for _ in range(reps):
        engine.default_context().synchronize()
        t0 = time.perf_counter()
        out = plans.execute_gpu(node, tables)
        engine.default_context().synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return round(min(times[1:]), 2), out


def host(out):
    import pyarrow as pa
    from tests.test_gpu_parquet_clickbench import host as h
    return h(out, out[0].schema) if isinstance(out, list) else pa.table(out)


def parity(got, k, x, n_check=3):
    """stddev of the first few groups against a two-pass Float64 computation (good to about 1e-12 for this data)"""
    for r in got.to_pylist()[:n_check]:
        xs = x[k == r["k"]]
        want = float(np.sqrt(np.sum((xs - xs.mean()) ** 2) / (len(xs) - 1))) if len(xs) > 1 else None
        if want is None or abs(r["sd"] - want) > 1e-9 * abs(want):
            return f"MISMATCH k={r['k']}: {r['sd']} vs {want}"
    return "ok"


def main():
    import pyarrow as pa
    from sail_b200 import engine, plans
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 200_000_000
    print(json.dumps({"card": card(), "rows": n}), flush=True)
    rng = np.random.default_rng(5)
    x = rng.normal(1e3, 25.0, n)
    t = plans.scan("t", ["k", "x"])
    avg = plans.aggregate(t, "single", ["k"], [("avg", plans.col("x"), "m", "Float64")])
    sd = plans.aggregate(t, "single", ["k"], [("stddev", plans.col("x"), "sd", "Float64")])
    for groups in (4, 10_000_000):
        k = (rng.integers(0, groups, n)).astype(np.int32)
        tables = {"t": (engine.to_device(pa.table({"k": k, "x": x})), ["k", "x"])}
        for kernel, env in (("interpreted", "0"), ("specialised", "1")):
            os.environ["SAILGPU_JIT"] = env
            ms_avg, _ = timed(avg, tables)
            ms_sd, out = timed(sd, tables)
            got = host(out)
            print(json.dumps({"groups": groups, "kernel": kernel, "avg_ms": ms_avg, "stddev_ms": ms_sd,
                              "stddev_over_avg": round(ms_sd / ms_avg, 3), "out_groups": got.num_rows,
                              "parity": parity(got, k, x)}), flush=True)
        del tables


if __name__ == "__main__":
    main()
