"""ClickBench on one H100: every query of sail_b200/clickbench.py through the C ABI, (1) checked against the SQL restated in pandas
(tests/clickbench_sql.py) on a small synthetic hits table, (2) timed on a larger one resident in HBM.  One JSON line per query and
leg is appended to --out as soon as it is known, and a query is marked "started" before it runs, so that a crash costs one
query: run again with the same --out and the finished (or crashed) ones are skipped.

    python scripts/clickbench_gpu.py --out gpurun_out/clickbench.jsonl [--parity-rows 200000] [--timing-rows 3000000]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--parity-rows", type=int, default=200_000)
    ap.add_argument("--timing-rows", type=int, default=3_000_000)
    ap.add_argument("--budget-s", type=float, default=1e9, help="stop starting new work after this many seconds")
    a = ap.parse_args()
    t_start = time.time()
    done = {}
    if os.path.exists(a.out):
        for line in open(a.out):
            r = json.loads(line)
            done[(r["leg"], r["query"])] = r["status"]
    out = open(a.out, "a")

    def emit(**kw):
        out.write(json.dumps(kw) + "\n")
        out.flush()
        os.fsync(out.fileno())

    from datagen import hits as gen
    from sail_b200 import clickbench as cb, engine, plans
    from tests import clickbench_sql as sql
    from tests import test_clickbench as T
    from tests.util import gpu_op

    names = list(cb.QUERIES)
    todo = [n for n in names if ("parity", n) not in done]
    if todo:
        table = gen.hits(a.parity_rows, seed=7)
        frame = sql.frame(table)
        for n in todo:
            if time.time() - t_start > a.budget_s:
                return
            emit(leg="parity", query=n, status="started")
            t0 = time.time()
            try:
                got = T.check(n, frame, {"hits": table}, gpu_op)
                emit(leg="parity", query=n, status="ok", rows=got.num_rows, input_rows=a.parity_rows, s=round(time.time() - t0, 3))
            except Exception as e:                                  # noqa: BLE001 -- every failure is a result here
                emit(leg="parity", query=n, status="FAILED", error=f"{type(e).__name__}: {e}"[:600], s=round(time.time() - t0, 3))

    todo = [n for n in names if ("timing", n) not in done and done.get(("parity", n), "ok") != "started"]
    if todo and a.timing_rows > 0:
        table = gen.hits(a.timing_rows, seed=11).combine_chunks()
        frame_params = T.sql_params(sql.frame(table.select(["CounterID", "EventDate", "IsRefresh", "TraficSourceID", "DontCountHits", "UserID", "RefererHash", "URLHash"])))
        ctx = engine.default_context()
        dev = {"hits": (engine.to_device(table), table.schema.names)}
        ctx.synchronize()
        for n in todo:
            if time.time() - t_start > a.budget_s:
                return
            q = cb.QUERIES[n]
            kw = {p: frame_params[p] for p in q.params}
            parts = [q.plan(part=i, **kw) for i in range(q.parts)] if q.parts > 1 else [q.plan(**kw)]
            emit(leg="timing", query=n, status="started")
            try:
                ms = []
                for _ in range(3):
                    ctx.synchronize()
                    t0 = time.perf_counter()
                    rows = 0
                    for plan in parts:
                        res = plans.execute_gpu(plan, dev, ctx)
                        rows = max(rows, sum(b.num_rows for b in res))
                        del res
                    ctx.synchronize()
                    ms.append((time.perf_counter() - t0) * 1e3)
                emit(leg="timing", query=n, status="ok", rows=rows, input_rows=a.timing_rows, ms_first=round(ms[0], 3), ms=round(min(ms[1:]), 3))
            except Exception as e:                                  # noqa: BLE001
                emit(leg="timing", query=n, status="FAILED", error=f"{type(e).__name__}: {e}"[:600])
    emit(leg="end", query="-", status="ok", s=round(time.time() - t_start, 1))


if __name__ == "__main__":
    main()
