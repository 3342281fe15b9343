"""Where does the first run of a high-cardinality aggregate spend its time?  ClickBench [04] (count(DISTINCT UserID)) on 3 M rows was
far slower on its first run than afterwards.  Prints per-operator wall time of the first runs.

    SAILGPU_JIT_VERBOSE=1 python scripts/first_run_probe.py [rows]
"""
import os
import sys
import time

import numpy as np
import pyarrow as pa

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sail_b200 import clickbench as cb, engine, plans   # noqa: E402


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 3_000_000
    rng = np.random.default_rng(1)
    users = rng.integers(1 << 40, 1 << 62, n // 6, dtype=np.int64)
    w = 1.0 / np.power(np.arange(1, len(users) + 1, dtype=np.float64), 1.15)
    cdf = np.cumsum(w) / w.sum()
    table = pa.table({"UserID": users[np.searchsorted(cdf, rng.random(n)).clip(0, len(users) - 1)]})
    ctx = engine.default_context()
    t0 = time.perf_counter()
    dev = {"hits": (engine.to_device(table), table.schema.names)}
    ctx.synchronize()
    print(f"to_device {1e3 * (time.perf_counter() - t0):.1f} ms", flush=True)
    for name in ("c15", "c4", "c4"):
        stats = {}
        t0 = time.perf_counter()
        out = plans.execute_gpu(cb.QUERIES[name].plan(), dev, ctx, stats)
        ctx.synchronize()
        print(f"{name}: {1e3 * (time.perf_counter() - t0):.1f} ms, rows {sum(b.num_rows for b in out)}", flush=True)
        for k, v in stats.items():
            print("   ", k, v, flush=True)


if __name__ == "__main__":
    main()
