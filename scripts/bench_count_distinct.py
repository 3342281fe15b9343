"""count(DISTINCT) next to other aggregates on the GPU: ClickBench [09] in the reference's shape (one single-mode aggregate with a
gated count(DISTINCT UserID), `clickbench.DISTINCT_QUERIES['c9_single']`) against the two-level rewrite `c9`, and a cardinality
sweep of `count(DISTINCT x) GROUP BY k`, fused against the two stacked aggregates, with parity between the two in the same run.

    python scripts/bench_count_distinct.py [hits_rows=10000000] [sweep_rows=100000000]

Prints one JSON object per measurement.  [09] runs over `hits_rows` resident synthetic rows and over ten copies of them (the
copies repeat every (RegionID, UserID) pair, so the DISTINCT count is that of the first copy).  The sweep keeps `sweep_rows`
rows resident (k Int32, x Int64) and varies the number of distinct pairs from 10^3 to 10^8 (x = i * 2654435761 mod P takes every
value below P once per P rows; k = x mod 1000).  Times are host clocks around the whole plan over resident input, ending in a
device synchronise, best of four after a warm-up.  Both plans run interpreted (SAILGPU_JIT=0): the gated pipeline is never
specialised, and so the two-level plan is timed on the same kernel."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.bench_timestamp import _scans, card  # noqa: E402


def timed(node, tables, reps=5):
    from sail_b200 import engine, plans
    from tests.test_gpu_parquet_clickbench import host
    times = []
    for _ in range(reps):
        engine.default_context().synchronize()
        t0 = time.perf_counter()
        out = plans.execute_gpu(node, tables)
        engine.default_context().synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return round(min(times[1:]), 2), host(out, out[0].schema)


def same(a, b, float_cols=()):
    from tests.util import assert_same
    try:
        assert_same(a, b, float_cols=float_cols)
        return "ok"
    except AssertionError as e:
        return f"MISMATCH: {str(e)[:200]}"


def c9(n):
    import pyarrow as pa
    from datagen import hits as gen
    from sail_b200 import clickbench as cb, engine
    q = cb.DISTINCT_QUERIES["c9_single"]
    cols = sorted({c for s in _scans(q.plan()) for c in s})
    table = gen.hits(n, seed=7).select(cols)
    out = {}
    for copies in (1, 10):
        t = pa.concat_tables([table] * copies) if copies > 1 else table
        tables = {"hits": (engine.to_device(t), cols)}
        ms_single, got = timed(cb.without_limit(q.plan()), tables)
        ms_two, want = timed(cb.without_limit(cb.c9()), tables)
        out[f"rows_{t.num_rows}"] = {"c9_single_ms": ms_single, "c9_two_level_ms": ms_two, "groups": got.num_rows, "parity": same(got, want, q.floats)}
        del tables
    return out


def sweep(n):
    import pyarrow as pa
    from sail_b200 import engine, plans
    i = np.arange(n, dtype=np.uint64)
    t = plans.scan("t", ["k", "x"])
    fused = plans.aggregate(t, "single", ["k"], [("count", plans.col("x"), "n", "Int64", True)])
    inner = plans.aggregate(t, "single", ["k", "x"], [])
    two_level = plans.aggregate(inner, "single", ["k"], [("count", plans.col("x"), "n", "Int64")])
    out = {}
    for p in (10**3, 10**4, 10**5, 10**6, 10**7, 10**8):
        x = ((i * np.uint64(2654435761)) % np.uint64(p)).astype(np.int64)
        tbl = pa.table({"k": (x % 1000).astype(np.int32), "x": x})
        tables = {"t": (engine.to_device(tbl), ["k", "x"])}
        ms_f, got = timed(fused, tables)
        ms_t, want = timed(two_level, tables)
        out[f"pairs_{min(p, n)}"] = {"fused_ms": ms_f, "two_level_ms": ms_t, "fused_over_two_level": round(ms_f / ms_t, 3), "parity": same(got, want)}
        print(json.dumps({"sweep_rows": n, **{k: v for k, v in out.items() if k == f"pairs_{min(p, n)}"}}), flush=True)
        del tables
    return out


def main():
    hits_rows = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
    sweep_rows = int(sys.argv[2]) if len(sys.argv) > 2 else 100_000_000
    os.environ["SAILGPU_JIT"] = "0"          # both plans interpreted: the gated pipeline is never specialised
    print(json.dumps({"card": card()}), flush=True)
    print(json.dumps({"c9": c9(hits_rows)}), flush=True)
    sweep(sweep_rows)


if __name__ == "__main__":
    main()
