"""Per-operator throughput on one H100 (inputs resident in HBM), with the algorithmic-bytes formulas of SURVEY.md
section 8(d) and the measured HBM peak: FilterExec, ProjectionExec, AggregateExec (low / high cardinality), HashJoinExec
(build + probe), SortExec, hash RepartitionExec.  Times are CUDA-synchronised wall clock around push/finish/pull_device
of ONE operator (device hand-off on both sides), best of `reps`."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["SAILGPU_TIMING"] = "1"
from datagen import tpch  # noqa: E402
from sail_b200 import engine, plans  # noqa: E402

W = {"l_orderkey": 8, "l_suppkey": 8, "l_quantity": 16, "l_extendedprice": 16, "l_discount": 16, "l_tax": 16, "l_returnflag": 16,
     "l_linestatus": 16, "l_shipdate": 4, "o_orderkey": 8, "o_custkey": 8, "o_orderdate": 4, "o_shippriority": 4}


ONLY = os.environ.get("OPS_ONLY", "")          # substring of the operator label: run just those (profiling)
REPS = os.environ.get("OPS_REPS")


def want(label):
    return ONLY == "" or ONLY.lower() in label.lower()


def run(ctx, spec, inputs, reps=3):
    """inputs: list of (DeviceBatch) per operator input.  returns (best ms, out rows, kernel ms)"""
    best, rows, kms = 1e30, 0, 0.0
    if REPS is not None:
        reps = int(REPS)
    for _ in range(reps + 1):
        op = engine.GpuExec(spec, [i.schema for i in inputs], ctx)
        ctx.synchronize()
        t0 = time.perf_counter()
        for k, d in enumerate(inputs):
            op.push(d.borrow(), k)
            op.finish(k)
        out = op.collect_device()
        ctx.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        m = op.metrics()
        if os.environ.get("OPS_METRICS"):
            print("  metrics:", {k_: v for k_, v in m.items() if v}, file=sys.stderr)
        op.close()
        if ms < best:
            best, rows, kms = ms, sum(d.num_rows for d in out), m["gpu.pipeline_kernel_ns"] / 1e6
        for d in out:
            d.release()
    return best, rows, kms


def main():
    sf = float(sys.argv[1]) if len(sys.argv) > 1 else 10.0
    peak = 3350.0       # H100 SXM data sheet (HBM3), used when no measured peak is present
    pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pk):
        peak = float(json.load(open(pk))["hbm_gbs"])
    ctx = engine.Context(0)
    li_cols = ["l_orderkey", "l_quantity", "l_extendedprice", "l_discount", "l_tax", "l_returnflag", "l_linestatus", "l_shipdate"]
    li = tpch.lineitem(sf, li_cols).combine_chunks()
    od = tpch.orders(sf, ["o_orderkey", "o_custkey", "o_orderdate", "o_shippriority"]).combine_chunks()
    N, NO = li.num_rows, od.num_rows
    dli, dod = engine.to_device(li, ctx), engine.to_device(od, ctx)
    names = li.schema.names
    C = lambda n: {"col": names.index(n)}  # noqa: E731
    res = {}

    def rec(name, ms, rows_in, rows_out, algo_bytes, kms=None):
        res[name] = {"ms": round(ms, 3), "rows_in": rows_in, "rows_out": rows_out, "rows_per_s": rows_in / (ms / 1e3),
                     "algorithmic_GB": round(algo_bytes / 1e9, 3), "GBps": round(algo_bytes / (ms / 1e3) / 1e9, 1),
                     "frac_of_hbm_peak": round(algo_bytes / (ms / 1e3) / 1e9 / peak, 3)}
        if kms:
            res[name]["kernel_ms"] = round(kms, 3)
        print(name, json.dumps(res[name]), flush=True)

    # FilterExec (Q1 predicate, 98.9 % pass) with projection of 6 columns: N*(4 + 96) in, sel*N*96 out
    proj = ["l_quantity", "l_extendedprice", "l_discount", "l_tax", "l_returnflag", "l_linestatus"]
    f = {"op": "filter", "predicate": plans.binop("<=", C("l_shipdate"), plans.date("1998-09-24")), "projection": [names.index(c) for c in proj]}
    if want("FilterExec q1 (sel 0.99, 6 cols out)"):
        ms, out, k = run(ctx, f, [dli])
        rec("FilterExec q1 (sel 0.99, 6 cols out)", ms, N, out, N * 100 + out * 96, k)
    # FilterExec (Q6 predicate, ~1.9 % pass): N*52 in, out*32
    pred = plans.and_(plans.binop(">=", C("l_shipdate"), plans.date("1994-01-01")), plans.binop("<", C("l_shipdate"), plans.date("1995-01-01")),
                      plans.binop(">=", C("l_discount"), plans.dec(5, 15, 2)), plans.binop("<=", C("l_discount"), plans.dec(7, 15, 2)),
                      plans.binop("<", C("l_quantity"), plans.dec(2400, 15, 2)))
    f6 = {"op": "filter", "predicate": pred, "projection": [names.index("l_extendedprice"), names.index("l_discount")]}
    if want("FilterExec q6 (sel 0.02, 2 cols out)"):
        ms, out, k = run(ctx, f6, [dli])
        rec("FilterExec q6 (sel 0.02, 2 cols out)", ms, N, out, N * 52 + out * 32, k)
    # ProjectionExec: price*(1-disc): 32 B in + 16 B out per row (pass-through columns are zero-copy in DataFusion; here 0 too)
    p = {"op": "projection", "exprs": [{"expr": plans.binop("*", C("l_extendedprice"), plans.binop("-", plans.dec(1, 10, 0), C("l_discount"))), "name": "x"}]}
    if want("ProjectionExec price*(1-disc)"):
        ms, out, k = run(ctx, p, [dli])
        rec("ProjectionExec price*(1-disc)", ms, N, out, N * 48, k)
    # AggregateExec low cardinality: group by (returnflag, linestatus): 2*16 keys + sum(qty)+sum(price) 32 B
    a = {"op": "aggregate", "mode": "single", "group_by": [{"expr": C("l_returnflag"), "name": "rf"}, {"expr": C("l_linestatus"), "name": "ls"}],
         "aggs": [{"fn": "sum", "args": [C("l_quantity")], "name": "sq"}, {"fn": "sum", "args": [C("l_extendedprice")], "name": "sp"}, {"fn": "count", "args": [], "name": "c"}]}
    if want("AggregateExec 4 groups (2 view keys, 2 sums, count)"):
        ms, out, k = run(ctx, a, [dli])
        rec("AggregateExec 4 groups (2 view keys, 2 sums, count)", ms, N, out, N * 64, k)
    # AggregateExec high cardinality: group by l_orderkey (15 M groups at SF10): 8 B key + 16 B value, + groups * 32 B state
    ah = {"op": "aggregate", "mode": "single", "group_by": [{"expr": C("l_orderkey"), "name": "k"}], "aggs": [{"fn": "sum", "args": [C("l_quantity")], "name": "sq"}]}
    if want("AggregateExec high cardinality (l_orderkey)"):
        ms, out, k = run(ctx, ah, [dli])
        rec("AggregateExec high cardinality (l_orderkey)", ms, N, out, N * 24 + out * 24, k)
    # HashJoinExec inner: build orders(o_orderkey,o_orderdate,o_shippriority) probe lineitem(l_orderkey, price, disc): B*(8+8) + P*(8+32) + M*48
    jb = engine.to_device(od.select(["o_orderkey", "o_orderdate", "o_shippriority"]), ctx)
    jp = engine.to_device(li.select(["l_orderkey", "l_extendedprice", "l_discount"]), ctx)
    j = {"op": "hash_join", "join_type": "inner", "on": [[0, 0]], "filter": None, "projection": [1, 2, 3, 4, 5]}
    if want("HashJoinExec inner orders(15M) x lineitem(60M)"):
        ms, out, k = run(ctx, j, [jb, jp])
        rec("HashJoinExec inner orders(15M) x lineitem(60M)", ms, NO + N, out, NO * 16 + N * 40 + out * 48, k)
    # SortExec on (l_orderkey desc) with 2 payload columns: 2 * N * 40 B ; run on a 1/4 slice to bound time
    sl = li.select(["l_orderkey", "l_extendedprice", "l_discount"]).slice(0, N // 4).combine_chunks()
    ds = engine.to_device(sl, ctx)
    s = {"op": "sort", "keys": [{"expr": {"col": 0}, "asc": False, "nulls_first": False}], "fetch": None}
    if want("SortExec by int64 key (N/4 rows, 40 B rows)"):
        ms, out, k = run(ctx, s, [ds], reps=1)
        rec("SortExec by int64 key (N/4 rows, 40 B rows)", ms, sl.num_rows, out, 2 * sl.num_rows * 40)
    # RepartitionExec Hash(l_orderkey, 8): 2 * N * 40 B
    r = {"op": "repartition", "scheme": "hash", "exprs": [{"col": 0}], "n": 8}
    if want("RepartitionExec Hash(l_orderkey, 8)"):
        ms, out, k = run(ctx, r, [jp])
        rec("RepartitionExec Hash(l_orderkey, 8)", ms, N, out, 2 * N * 40, k)
    print(json.dumps({"sf": sf, "hbm_peak_GBps": peak, "operators": res}))
    for d in (dli, dod, jb, jp, ds):
        d.release()
    ctx.synchronize()


if __name__ == "__main__":
    main()
