"""All 22 TPC-H queries on one H100 with the referenced columns resident in HBM: wall-clock per query through the C ABI (every
intermediate stays on the device), rows/s over the scanned rows, per-operator times, and the total of the 22 (SURVEY.md section 8d:
"total 22-query wall-clock").  Result parity of every plan is the test-suite's job (golden snapshot at SF0.001, oracle at SF0.1).
Usage: python scripts/bench_tpch.py [SF] [reps]"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from datagen import tpch  # noqa: E402
from sail_b200 import engine, plans  # noqa: E402

NEEDED = {
    "lineitem": ["l_orderkey", "l_partkey", "l_suppkey", "l_quantity", "l_extendedprice", "l_discount", "l_tax", "l_returnflag", "l_linestatus",
                 "l_shipdate", "l_commitdate", "l_receiptdate", "l_shipinstruct", "l_shipmode"],
    "orders": ["o_orderkey", "o_custkey", "o_orderstatus", "o_totalprice", "o_orderdate", "o_orderpriority", "o_shippriority", "o_comment"],
    "customer": ["c_custkey", "c_nationkey", "c_acctbal", "c_mktsegment", "c_name", "c_phone", "c_address", "c_comment"],
    "supplier": ["s_suppkey", "s_nationkey", "s_acctbal", "s_name", "s_phone", "s_address", "s_comment"],
    "part": ["p_partkey", "p_brand", "p_type", "p_size", "p_container", "p_name", "p_mfgr"],
}
QUERIES = [f"q{i}" for i in range(1, 23)]


def load(sf):
    t = {"lineitem": tpch.lineitem(sf, NEEDED["lineitem"]), "orders": tpch.orders(sf, NEEDED["orders"]),
         "customer": tpch.customer(sf, NEEDED["customer"]), "supplier": tpch.supplier(sf, NEEDED["supplier"]), "part": tpch.part(sf, NEEDED["part"]),
         "partsupp": tpch.partsupp(sf), "nation": tpch.nation(), "region": tpch.region()}
    return {k: v.combine_chunks() for k, v in t.items()}


def scanned_rows(node, tables):
    if node.spec["op"] == "scan":
        return tables[node.spec["table"]].num_rows
    return sum(scanned_rows(c, tables) for c in node.inputs)


def main():
    sf = float(sys.argv[1]) if len(sys.argv) > 1 else 10.0
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    ctx = engine.Context(0)
    t0 = time.time()
    tables = load(sf)
    print(f"generated SF{sf:g} in {time.time() - t0:.1f}s: " + ", ".join(f"{k}={v.num_rows}" for k, v in tables.items()), flush=True)
    dev = {k: (engine.to_device(v, ctx), v.schema.names) for k, v in tables.items()}
    hbm = sum(v.nbytes for v in tables.values())
    results = {}
    for q in QUERIES:
        plan = plans.TPCH[q]()
        try:
            times, stats = [], {}
            for r in range(reps + 1):
                ctx.synchronize()
                t1 = time.perf_counter()
                st = {} if r == reps else None
                out = plans.execute_gpu(plan, dev, ctx, st)
                ctx.synchronize()
                times.append((time.perf_counter() - t1) * 1e3)
                if st is not None:
                    stats = st
            ms = min(times[1:])
            rows = scanned_rows(plan, tables)
            results[q] = {"ms": round(ms, 3), "scanned_rows": rows, "rows_per_s": rows / (ms / 1e3), "out_rows": sum(d.num_rows for d in out),
                          "operators": stats}
            print(q, json.dumps(results[q]), flush=True)
        except engine.SailGpuError as e:
            print(q, "FAILED", e, flush=True)
    total = sum(v["ms"] for v in results.values())
    print(f"total of {len(results)} queries: {total:.1f} ms", flush=True)
    print(json.dumps({"sf": sf, "hbm_bytes": hbm, "n_queries": len(results), "total_ms": round(total, 2), "queries": {k: {kk: vv for kk, vv in v.items() if kk != "operators"} for k, v in results.items()}}))
    del dev
    ctx.synchronize()


if __name__ == "__main__":
    main()
