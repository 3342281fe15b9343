"""Physical plans of the BASELINE.json workloads, written as trees of operator specs.

Each node is the JSON object a Rust `ExecutionPlan` shim would hand to `sailgpu_op_create`
(include/sailgpu.h) for the DataFusion operator it replaces.  The shapes follow the reference's
plan snapshots (python/pysail/tests/spark/__snapshots__/test_tpch.plan.yaml): Q1 `:3-19`,
Q3 `:72-97`, Q4 `:99-118`, Q5 `:120-156`, Q6, Q7 `:172-209`, Q12, Q14 `:409-425`, Q18 `:529-557`, Q19 `:559-575` -- minus the rename-only ProjectionExecs and
the RoundRobinBatch fan-out that pre-sharded tables make unnecessary (SURVEY.md Appendix D).

The tree is engine-agnostic: `execute(plan, tables, run_op)` drives it with any callable that maps
(spec, *input tables) -> table.  tests/ drive it with the oracle and with the CUDA engine and diff
the two.
"""
from __future__ import annotations

import datetime
from dataclasses import dataclass, field


def days(iso: str) -> int:
    return (datetime.date.fromisoformat(iso) - datetime.date(1970, 1, 1)).days


# ---- expression helpers (column refs by NAME here; resolved to indices when the node is built) ----
def col(name):
    return {"col": name}


def lit(value, type_):
    return {"lit": value, "type": type_}


def dec(unscaled: int, p: int, s: int):
    return {"lit": str(int(unscaled)), "type": f"Decimal128({p},{s})"}


def date(iso: str):
    return {"lit": days(iso), "type": "Date32"}


def string(v: str, type_="Utf8View"):
    return {"lit": v, "type": type_}


def binop(op, l, r):
    return {"op": op, "l": l, "r": r}


def and_(*xs):
    out = xs[0]
    for x in xs[1:]:
        out = binop("and", out, x)
    return out


def or_(*xs):
    out = xs[0]
    for x in xs[1:]:
        out = binop("or", out, x)
    return out


def resolve(e, names):
    """replace {"col": "name"} by {"col": index}"""
    if isinstance(e, dict):
        if "col" in e and isinstance(e["col"], str):
            return {"col": names.index(e["col"])}
        return {k: resolve(v, names) for k, v in e.items()}
    if isinstance(e, list):
        return [resolve(x, names) for x in e]
    return e


@dataclass
class Node:
    spec: dict
    inputs: list = field(default_factory=list)
    names: list = field(default_factory=list)


def scan(table: str, columns: list) -> Node:
    return Node({"op": "scan", "table": table, "columns": list(columns)}, [], list(columns))


def filter_(child: Node, predicate, projection=None) -> Node:
    proj = None if projection is None else [child.names.index(c) for c in projection]
    names = child.names if proj is None else list(projection)
    return Node({"op": "filter", "predicate": resolve(predicate, child.names), "projection": proj}, [child], list(names))


def project(child: Node, exprs: list) -> Node:
    """exprs: list of (expr, name) or column names"""
    items = []
    for e in exprs:
        if isinstance(e, str):
            e = (col(e), e)
        items.append({"expr": resolve(e[0], child.names), "name": e[1]})
    return Node({"op": "projection", "exprs": items}, [child], [i["name"] for i in items])


def aggregate(child: Node, mode: str, group_by: list, aggs: list) -> Node:
    """group_by: column names or (expr, name); aggs: (fn, arg_expr|None, name, input_type), or (fn, arg, name, input_type, True)
    for fn(DISTINCT arg)"""
    gb = []
    for g in group_by:
        if isinstance(g, str):
            g = (col(g), g)
        gb.append({"expr": resolve(g[0], child.names), "name": g[1]})
    merging = mode in ("final", "final_partitioned")
    specs, names = [], [g["name"] for g in gb]
    for fn, arg, name, in_type, *distinct in aggs:
        a = {"fn": fn, "name": name, "input_type": in_type}
        if not merging:
            a["args"] = [] if arg is None else [resolve(arg, child.names)]
        if distinct and distinct[0]:
            a["distinct"] = True
        specs.append(a)
        if mode == "partial":
            names += [f"{name}[count]", f"{name}[sum]"] if fn == "avg" else [f"{name}[{fn}]"]
        else:
            names.append(name)
    return Node({"op": "aggregate", "mode": mode, "group_by": gb, "aggs": specs}, [child], names)


def two_phase(child: Node, group_by: list, aggs: list) -> Node:
    """AggregateExec Partial -> [RepartitionExec Hash(group keys)] -> FinalPartitioned"""
    part = aggregate(child, "partial", group_by, aggs)
    gnames = [g if isinstance(g, str) else g[1] for g in group_by]
    return aggregate(part, "final_partitioned" if gnames else "final", gnames, aggs)


def hash_join(build: Node, probe: Node, on: list, join_type="inner", projection=None, filter=None) -> Node:
    names = {"left_semi": build.names, "left_anti": build.names,
             "right_semi": probe.names, "right_anti": probe.names}.get(join_type, build.names + probe.names)
    spec = {"op": "hash_join", "join_type": join_type, "mode": "collect_left",
            "on": [[build.names.index(a), probe.names.index(b)] for a, b in on],
            "filter": None if filter is None else resolve(filter, build.names + probe.names),
            "projection": None if projection is None else [names.index(c) for c in projection]}
    return Node(spec, [build, probe], list(names if projection is None else projection))


def nested_loop_join(build: Node, probe: Node, filter=None, projection=None) -> Node:
    """NestedLoopJoinExec, inner: build = left child (the one-row scalar subquery in TPC-H Q11 / Q22)"""
    names = build.names + probe.names
    spec = {"op": "nested_loop_join", "join_type": "inner",
            "filter": None if filter is None else resolve(filter, names),
            "projection": None if projection is None else [names.index(c) for c in projection]}
    return Node(spec, [build, probe], list(names if projection is None else projection))


def substr(e, start: int, length: int | None = None):
    return {"fn": "substr", "args": [e], "start": start, "length": length}


def char_length(e):
    return {"fn": "character_length", "args": [e]}


def sort(child: Node, keys: list, fetch=None) -> Node:
    """keys: (column name, asc) -- Spark default null ordering: ASC NULLS FIRST / DESC NULLS LAST"""
    ks = [{"expr": resolve(col(k), child.names), "asc": asc, "nulls_first": asc} for k, asc in keys]
    return Node({"op": "sort", "keys": ks, "fetch": fetch}, [child], list(child.names))


def execute(node: Node, tables: dict, run_op):
    if node.spec["op"] == "scan":
        return tables[node.spec["table"]].select(node.spec["columns"])
    ins = [execute(c, tables, run_op) for c in node.inputs]
    return run_op(node.spec, *ins)


def execute_gpu(node: Node, dev_tables: dict, ctx=None, stats: dict | None = None):
    """Runs the plan through libsailgpu with every intermediate batch staying in HBM (device hand-off between
    operators).  dev_tables: {table: (DeviceBatch or a list of them, schema names)} resident inputs; returns a list of DeviceBatch.
    stats (optional) collects per-operator metrics keyed by a running node number."""
    from . import engine
    if node.spec["op"] == "scan":
        dev, names = dev_tables[node.spec["table"]]
        idx = [names.index(c) for c in node.spec["columns"]]
        spec = {"op": "projection", "exprs": [{"expr": {"col": i}, "name": names[i]} for i in idx]}
        devs = dev if isinstance(dev, (list, tuple)) else [dev]          # a table may be resident as several batches
        op = engine.GpuExec(spec, [devs[0].schema], ctx)
        for d in devs:
            op.push(d.borrow())
        op.finish()
        out = op.collect_device(handle=True)
        for d in out:
            d.schema = op.schema
        op.close()
        return out
    ins = [execute_gpu(c, dev_tables, ctx, stats) for c in node.inputs]
    if stats is not None:
        import time
        (ctx or engine.default_context()).synchronize()
        t0 = time.perf_counter()
    op = engine.GpuExec(node.spec, [i[0].schema for i in ins], ctx)
    for k, batches in enumerate(ins):
        for b in batches:
            op.push(b, k)
        op.finish(k)
    out = op.collect_device(handle=True)      # GpuExec -> GpuExec: the batch is handed on in its internal form
    for d in out:
        d.schema = op.schema
    if stats is not None:
        m = op.metrics()
        (ctx or engine.default_context()).synchronize()
        stats[f"{len(stats):02d} {op.name()}"] = {"in": m["input_rows"] + m.get("build_input_rows", 0), "out": m["output_rows"],
                                               "launches": m["gpu.kernel_launches"], "ms": round((time.perf_counter() - t0) * 1e3, 3)}
    op.close()
    return out


# ---- TPC-H ------------------------------------------------------------------------------------------
ONE = dec(1, 10, 0)     # `Int32(1)` coerced by DataFusion to Decimal128(10,0): test_tpch.plan.yaml:15
D152 = "Decimal128(15,2)"
DISC_PRICE = binop("*", col("l_extendedprice"), binop("-", ONE, col("l_discount")))   # Decimal128(32,4)


def q1(strings="Utf8View") -> Node:
    li = scan("lineitem", ["l_quantity", "l_extendedprice", "l_discount", "l_tax", "l_returnflag",
                           "l_linestatus", "l_shipdate"])
    f = filter_(li, binop("<=", col("l_shipdate"), date("1998-09-24")),
                ["l_quantity", "l_extendedprice", "l_discount", "l_tax", "l_returnflag", "l_linestatus"])
    p = project(f, [(DISC_PRICE, "__common_expr_1"), "l_quantity", "l_extendedprice", "l_discount", "l_tax",
                    "l_returnflag", "l_linestatus"])
    charge = binop("*", col("__common_expr_1"), binop("+", ONE, col("l_tax")))
    aggs = [("sum", col("l_quantity"), "sum_qty", D152),
            ("sum", col("l_extendedprice"), "sum_base_price", D152),
            ("sum", col("__common_expr_1"), "sum_disc_price", "Decimal128(32,4)"),
            ("sum", charge, "sum_charge", "Decimal128(38,6)"),
            ("avg", col("l_quantity"), "avg_qty", D152),
            ("avg", col("l_extendedprice"), "avg_price", D152),
            ("avg", col("l_discount"), "avg_disc", D152),
            ("count", None, "count_order", None)]
    a = two_phase(p, ["l_returnflag", "l_linestatus"], aggs)
    return sort(a, [("l_returnflag", True), ("l_linestatus", True)])


def q6() -> Node:
    li = scan("lineitem", ["l_quantity", "l_extendedprice", "l_discount", "l_shipdate"])
    pred = and_(binop(">=", col("l_shipdate"), date("1994-01-01")),
                binop("<", col("l_shipdate"), date("1995-01-01")),
                binop(">=", col("l_discount"), dec(3, 15, 2)),
                binop("<=", col("l_discount"), dec(5, 15, 2)),
                binop("<", col("l_quantity"), dec(2400, 15, 2)))
    f = filter_(li, pred, ["l_extendedprice", "l_discount"])
    p = project(f, [(binop("*", col("l_extendedprice"), col("l_discount")), "rev")])
    return two_phase(p, [], [("sum", col("rev"), "revenue", "Decimal128(31,4)")])


def q3(strings="Utf8View") -> Node:
    cust = filter_(scan("customer", ["c_custkey", "c_mktsegment"]),
                   binop("=", col("c_mktsegment"), string("BUILDING", strings)), ["c_custkey"])
    ords = filter_(scan("orders", ["o_orderkey", "o_custkey", "o_orderdate", "o_shippriority"]),
                   binop("<", col("o_orderdate"), date("1995-03-15")))
    j1 = hash_join(cust, ords, [("c_custkey", "o_custkey")], projection=["o_orderkey", "o_orderdate", "o_shippriority"])
    li = filter_(scan("lineitem", ["l_orderkey", "l_extendedprice", "l_discount", "l_shipdate"]),
                 binop(">", col("l_shipdate"), date("1995-03-15")), ["l_orderkey", "l_extendedprice", "l_discount"])
    j2 = hash_join(j1, li, [("o_orderkey", "l_orderkey")],
                   projection=["o_orderdate", "o_shippriority", "l_orderkey", "l_extendedprice", "l_discount"])
    a = two_phase(j2, ["l_orderkey", "o_orderdate", "o_shippriority"],
                  [("sum", DISC_PRICE, "revenue", "Decimal128(32,4)")])
    p = project(a, ["l_orderkey", "revenue", "o_orderdate", "o_shippriority"])
    return sort(p, [("revenue", False), ("o_orderdate", True)], fetch=10)


def q4(strings="Utf8View") -> Node:
    li = filter_(scan("lineitem", ["l_orderkey", "l_commitdate", "l_receiptdate"]),
                 binop(">", col("l_receiptdate"), col("l_commitdate")), ["l_orderkey"])
    ords = filter_(scan("orders", ["o_orderkey", "o_orderdate", "o_orderpriority"]),
                   and_(binop(">=", col("o_orderdate"), date("1995-04-01")),
                        binop("<", col("o_orderdate"), date("1995-07-01"))), ["o_orderkey", "o_orderpriority"])
    j = hash_join(li, ords, [("l_orderkey", "o_orderkey")], join_type="right_semi", projection=["o_orderpriority"])
    a = two_phase(j, ["o_orderpriority"], [("count", None, "order_count", None)])
    return sort(a, [("o_orderpriority", True)])


def q5(strings="Utf8View") -> Node:
    cust = scan("customer", ["c_custkey", "c_nationkey"])
    ords = filter_(scan("orders", ["o_orderkey", "o_custkey", "o_orderdate"]),
                   and_(binop(">=", col("o_orderdate"), date("1994-01-01")),
                        binop("<", col("o_orderdate"), date("1995-01-01"))), ["o_orderkey", "o_custkey"])
    j1 = hash_join(cust, ords, [("c_custkey", "o_custkey")], projection=["c_nationkey", "o_orderkey"])
    li = scan("lineitem", ["l_orderkey", "l_suppkey", "l_extendedprice", "l_discount"])
    j2 = hash_join(j1, li, [("o_orderkey", "l_orderkey")],
                   projection=["c_nationkey", "l_suppkey", "l_extendedprice", "l_discount"])
    supp = scan("supplier", ["s_suppkey", "s_nationkey"])
    j3 = hash_join(supp, j2, [("s_suppkey", "l_suppkey"), ("s_nationkey", "c_nationkey")],
                   projection=["s_nationkey", "l_extendedprice", "l_discount"])
    nat = scan("nation", ["n_nationkey", "n_name", "n_regionkey"])
    j4 = hash_join(j3, nat, [("s_nationkey", "n_nationkey")],
                   projection=["l_extendedprice", "l_discount", "n_name", "n_regionkey"])
    reg = filter_(scan("region", ["r_regionkey", "r_name"]),
                  binop("=", col("r_name"), string("AFRICA", strings)), ["r_regionkey"])
    j5 = hash_join(reg, j4, [("r_regionkey", "n_regionkey")], projection=["l_extendedprice", "l_discount", "n_name"])
    a = two_phase(j5, ["n_name"], [("sum", DISC_PRICE, "revenue", "Decimal128(32,4)")])
    return sort(a, [("revenue", False)])


def q8(strings="Utf8View") -> Node:
    """test_tpch.plan.yaml:211-258: seven joins (part -> lineitem -> supplier -> orders -> customer -> nation n1 -> nation n2 ->
    region), market share = ratio of two sums per order year."""
    pt = filter_(scan("part", ["p_partkey", "p_type"]), binop("=", col("p_type"), string("LARGE PLATED STEEL", strings)), ["p_partkey"])
    li = scan("lineitem", ["l_orderkey", "l_partkey", "l_suppkey", "l_extendedprice", "l_discount"])
    ja = hash_join(pt, li, [("p_partkey", "l_partkey")], projection=["l_orderkey", "l_suppkey", "l_extendedprice", "l_discount"])
    supp = scan("supplier", ["s_suppkey", "s_nationkey"])
    jb = hash_join(supp, ja, [("s_suppkey", "l_suppkey")], projection=["s_nationkey", "l_orderkey", "l_extendedprice", "l_discount"])
    jb = project(jb, ["l_orderkey", "l_extendedprice", "l_discount", "s_nationkey"])
    ords = filter_(scan("orders", ["o_orderkey", "o_custkey", "o_orderdate"]),
                   and_(binop(">=", col("o_orderdate"), date("1995-01-01")), binop("<=", col("o_orderdate"), date("1996-12-31"))))
    jc = hash_join(jb, ords, [("l_orderkey", "o_orderkey")],
                   projection=["l_extendedprice", "l_discount", "s_nationkey", "o_custkey", "o_orderdate"])
    cust = scan("customer", ["c_custkey", "c_nationkey"])
    jd = hash_join(jc, cust, [("o_custkey", "c_custkey")],
                   projection=["l_extendedprice", "l_discount", "s_nationkey", "o_orderdate", "c_nationkey"])
    n1 = project(scan("nation", ["n_nationkey", "n_regionkey"]), [(col("n_nationkey"), "n1_key"), (col("n_regionkey"), "n1_region")])
    je = hash_join(n1, jd, [("n1_key", "c_nationkey")],
                   projection=["n1_region", "l_extendedprice", "l_discount", "s_nationkey", "o_orderdate"])
    je = project(je, ["l_extendedprice", "l_discount", "s_nationkey", "o_orderdate", "n1_region"])
    n2 = project(scan("nation", ["n_nationkey", "n_name"]), [(col("n_nationkey"), "n2_key"), (col("n_name"), "n2_name")])
    jf = hash_join(je, n2, [("s_nationkey", "n2_key")], projection=["l_extendedprice", "l_discount", "o_orderdate", "n1_region", "n2_name"])
    reg = filter_(scan("region", ["r_regionkey", "r_name"]), binop("=", col("r_name"), string("MIDDLE EAST", strings)), ["r_regionkey"])
    jg = hash_join(reg, jf, [("r_regionkey", "n1_region")], projection=["l_extendedprice", "l_discount", "o_orderdate", "n2_name"])
    p = project(jg, [({"fn": "date_part", "part": "year", "args": [col("o_orderdate")]}, "o_year"), (DISC_PRICE, "volume"), (col("n2_name"), "nation")])
    iraq = {"case": [[binop("=", col("nation"), string("IRAQ", strings)), col("volume")]], "else": lit(0, "Int32")}
    a = two_phase(p, ["o_year"], [("sum", iraq, "iraq", "Decimal128(32,4)"), ("sum", col("volume"), "total", "Decimal128(32,4)")])
    r = project(a, ["o_year", (binop("/", col("iraq"), col("total")), "mkt_share")])
    return sort(r, [("o_year", True)])


def q12(strings="Utf8View") -> Node:
    li = filter_(scan("lineitem", ["l_orderkey", "l_shipdate", "l_commitdate", "l_receiptdate", "l_shipmode"]),
                 and_(or_(binop("=", col("l_shipmode"), string("FOB", strings)),
                          binop("=", col("l_shipmode"), string("SHIP", strings))),
                      binop(">", col("l_receiptdate"), col("l_commitdate")),
                      binop("<", col("l_shipdate"), col("l_commitdate")),
                      binop(">=", col("l_receiptdate"), date("1995-01-01")),
                      binop("<", col("l_receiptdate"), date("1996-01-01"))), ["l_orderkey", "l_shipmode"])
    ords = scan("orders", ["o_orderkey", "o_orderpriority"])
    j = hash_join(li, ords, [("l_orderkey", "o_orderkey")], projection=["l_shipmode", "o_orderpriority"])
    urgent = or_(binop("=", col("o_orderpriority"), string("1-URGENT", strings)),
                 binop("=", col("o_orderpriority"), string("2-HIGH", strings)))
    other = and_(binop("!=", col("o_orderpriority"), string("1-URGENT", strings)),
                 binop("!=", col("o_orderpriority"), string("2-HIGH", strings)))
    one, zero = lit(1, "Int64"), lit(0, "Int64")
    a = two_phase(j, ["l_shipmode"],
                  [("sum", {"case": [[urgent, one]], "else": zero}, "high_line_count", "Int64"),
                   ("sum", {"case": [[other, one]], "else": zero}, "low_line_count", "Int64")])
    return sort(a, [("l_shipmode", True)])


def q7(strings="Utf8View") -> Node:
    """test_tpch.plan.yaml:172-209: five CollectLeft joins (the growing intermediate is always the build side), the
    nation-pair predicate as the residual filter of the last join, date_part in the projection."""
    supp = scan("supplier", ["s_suppkey", "s_nationkey"])
    li = filter_(scan("lineitem", ["l_orderkey", "l_suppkey", "l_extendedprice", "l_discount", "l_shipdate"]),
                 and_(binop(">=", col("l_shipdate"), date("1995-01-01")), binop("<=", col("l_shipdate"), date("1996-12-31"))))
    j1 = hash_join(supp, li, [("s_suppkey", "l_suppkey")],
                   projection=["s_nationkey", "l_orderkey", "l_extendedprice", "l_discount", "l_shipdate"])
    ords = scan("orders", ["o_orderkey", "o_custkey"])
    j2 = hash_join(j1, ords, [("l_orderkey", "o_orderkey")],
                   projection=["s_nationkey", "l_extendedprice", "l_discount", "l_shipdate", "o_custkey"])
    cust = scan("customer", ["c_custkey", "c_nationkey"])
    j3 = hash_join(j2, cust, [("o_custkey", "c_custkey")],
                   projection=["s_nationkey", "l_extendedprice", "l_discount", "l_shipdate", "c_nationkey"])
    pair = or_(binop("=", col("n_name"), string("GERMANY", strings)), binop("=", col("n_name"), string("IRAQ", strings)))
    n1 = project(filter_(scan("nation", ["n_nationkey", "n_name"]), pair), [(col("n_nationkey"), "n1_key"), (col("n_name"), "n1_name")])
    j4 = hash_join(j3, n1, [("s_nationkey", "n1_key")],
                   projection=["l_extendedprice", "l_discount", "l_shipdate", "c_nationkey", "n1_name"])
    n2 = project(filter_(scan("nation", ["n_nationkey", "n_name"]), pair), [(col("n_nationkey"), "n2_key"), (col("n_name"), "n2_name")])
    cross = or_(and_(binop("=", col("n1_name"), string("GERMANY", strings)), binop("=", col("n2_name"), string("IRAQ", strings))),
                and_(binop("=", col("n1_name"), string("IRAQ", strings)), binop("=", col("n2_name"), string("GERMANY", strings))))
    j5 = hash_join(j4, n2, [("c_nationkey", "n2_key")], filter=cross,
                   projection=["l_extendedprice", "l_discount", "l_shipdate", "n1_name", "n2_name"])
    p = project(j5, [(col("n1_name"), "supp_nation"), (col("n2_name"), "cust_nation"),
                     ({"fn": "date_part", "part": "year", "args": [col("l_shipdate")]}, "l_year"), (DISC_PRICE, "volume")])
    a = two_phase(p, ["supp_nation", "cust_nation", "l_year"], [("sum", col("volume"), "revenue", "Decimal128(32,4)")])
    return sort(a, [("supp_nation", True), ("cust_nation", True), ("l_year", True)])


def q14(strings="Utf8View") -> Node:
    """test_tpch.plan.yaml:409-425: the filtered lineitem rows are the build side, part the probe side; the promo ratio is
    a decimal division of the two final sums (the reference guards the divisor with raise_error; division by zero is an
    error on both paths)."""
    li = filter_(scan("lineitem", ["l_partkey", "l_extendedprice", "l_discount", "l_shipdate"]),
                 and_(binop(">=", col("l_shipdate"), date("1995-02-01")), binop("<", col("l_shipdate"), date("1995-03-01"))),
                 ["l_partkey", "l_extendedprice", "l_discount"])
    pt = scan("part", ["p_partkey", "p_type"])
    j = hash_join(li, pt, [("l_partkey", "p_partkey")], projection=["l_extendedprice", "l_discount", "p_type"])
    p = project(j, [(DISC_PRICE, "__common_expr_1"), "p_type"])
    promo = {"case": [[{"like": col("p_type"), "pattern": "PROMO%"}, col("__common_expr_1")]], "else": lit(0, "Int32")}
    a = two_phase(p, [], [("sum", promo, "promo", "Decimal128(32,4)"), ("sum", col("__common_expr_1"), "total", "Decimal128(32,4)")])
    ratio = binop("/", binop("*", dec(10000, 5, 2), col("promo")), col("total"))
    return project(a, [(ratio, "promo_revenue")])


def q19(strings="Utf8View") -> Node:
    """test_tpch.plan.yaml:559-575: filtered part is the build side, filtered lineitem the probe side; the three
    brand/container/quantity/size alternatives are the residual filter of the join (IN lists, decimal ranges)."""
    def S(v):
        return string(v, strings)

    def alt(brand, containers, qlo, qhi, size_hi, with_qty):
        xs = [binop("=", col("p_brand"), S(brand)), {"in": col("p_container"), "set": [S(c) for c in containers]}]
        if with_qty:
            xs += [binop(">=", col("l_quantity"), dec(qlo * 100, 15, 2)), binop("<=", col("l_quantity"), dec(qhi * 100, 15, 2))]
        xs.append(binop("<=", col("p_size"), lit(size_hi, "Int32")))
        return and_(*xs)

    alts = [("Brand#21", ["SM CASE", "SM BOX", "SM PACK", "SM PKG"], 8, 18, 5),
            ("Brand#13", ["MED BAG", "MED BOX", "MED PKG", "MED PACK"], 20, 30, 10),
            ("Brand#52", ["LG CASE", "LG BOX", "LG PACK", "LG PKG"], 30, 40, 15)]
    pt = filter_(scan("part", ["p_partkey", "p_brand", "p_size", "p_container"]),
                 and_(or_(*[alt(*a, False) for a in alts]), binop(">=", col("p_size"), lit(1, "Int32"))))
    qty = or_(*[and_(binop(">=", col("l_quantity"), dec(lo * 100, 15, 2)), binop("<=", col("l_quantity"), dec(hi * 100, 15, 2)))
                for _, _, lo, hi, _ in alts])
    li = filter_(scan("lineitem", ["l_partkey", "l_quantity", "l_extendedprice", "l_discount", "l_shipinstruct", "l_shipmode"]),
                 and_(qty, or_(binop("=", col("l_shipmode"), S("AIR")), binop("=", col("l_shipmode"), S("AIR REG"))),
                      binop("=", col("l_shipinstruct"), S("DELIVER IN PERSON"))),
                 ["l_partkey", "l_quantity", "l_extendedprice", "l_discount"])
    j = hash_join(pt, li, [("p_partkey", "l_partkey")], filter=or_(*[alt(*a, True) for a in alts]),
                  projection=["l_extendedprice", "l_discount"])
    return two_phase(j, [], [("sum", DISC_PRICE, "revenue", "Decimal128(32,4)")])


def q18(strings="Utf8View", min_qty=313) -> Node:
    """test_tpch.plan.yaml:529-557: orders x customer x lineitem, LeftSemi against the orders whose quantity sums exceed
    313 (a grouped aggregate + filter on the probe side), five group keys including an 18-byte name, TopK 100."""
    del strings
    ords = scan("orders", ["o_orderkey", "o_custkey", "o_totalprice", "o_orderdate"])
    cust = scan("customer", ["c_custkey", "c_name"])
    j1 = hash_join(ords, cust, [("o_custkey", "c_custkey")], projection=["o_orderkey", "o_totalprice", "o_orderdate", "c_custkey", "c_name"])
    j1 = project(j1, ["c_custkey", "c_name", "o_orderkey", "o_totalprice", "o_orderdate"])
    li = scan("lineitem", ["l_orderkey", "l_quantity"])
    j2 = hash_join(j1, li, [("o_orderkey", "l_orderkey")],
                   projection=["c_custkey", "c_name", "o_orderkey", "o_totalprice", "o_orderdate", "l_quantity"])
    big = two_phase(scan("lineitem", ["l_orderkey", "l_quantity"]), ["l_orderkey"], [("sum", col("l_quantity"), "q", D152)])
    big = filter_(big, binop(">", col("q"), dec(min_qty * 100, 14, 2)), ["l_orderkey"])
    j3 = hash_join(j2, big, [("o_orderkey", "l_orderkey")], join_type="left_semi")
    a = two_phase(j3, ["c_name", "c_custkey", "o_orderkey", "o_orderdate", "o_totalprice"], [("sum", col("l_quantity"), "sum(l_quantity)", D152)])
    return sort(a, [("o_totalprice", False), ("o_orderdate", True)], fetch=100)


def q11(strings="Utf8View", nation="ALGERIA") -> Node:
    """test_tpch.plan.yaml:324-363: the HAVING threshold is a scalar subquery -> NestedLoopJoinExec against a one-row aggregate"""
    def joined():
        nat = filter_(scan("nation", ["n_nationkey", "n_name"]), binop("=", col("n_name"), string(nation, strings)), ["n_nationkey"])
        sp = hash_join(scan("supplier", ["s_suppkey", "s_nationkey"]), scan("partsupp", ["ps_partkey", "ps_suppkey", "ps_availqty", "ps_supplycost"]),
                       [("s_suppkey", "ps_suppkey")], projection=["s_nationkey", "ps_partkey", "ps_availqty", "ps_supplycost"])
        return hash_join(nat, sp, [("n_nationkey", "s_nationkey")], projection=["ps_partkey", "ps_availqty", "ps_supplycost"])
    value = binop("*", col("ps_supplycost"), col("ps_availqty"))
    total = two_phase(joined(), [], [("sum", value, "total", "Decimal128(26,2)")])
    thr = project(total, [(binop("*", col("total"), dec(1000000, 10, 10)), "threshold")])
    per = two_phase(joined(), ["ps_partkey"], [("sum", value, "value", "Decimal128(26,2)")])
    per = project(per, ["ps_partkey", "value", ({"cast": col("value"), "to": "Decimal128(38,12)"}, "value_cmp")])
    j = nested_loop_join(thr, per, binop(">", col("value_cmp"), col("threshold")), ["ps_partkey", "value"])
    return sort(j, [("value", False)])


def q17(strings="Utf8View", brand="Brand#42", container="LG BAG") -> Node:
    """test_tpch.plan.yaml:504-527: the correlated avg() is decorrelated into a grouped aggregate joined back with a residual filter"""
    pt = filter_(scan("part", ["p_partkey", "p_brand", "p_container"]),
                 and_(binop("=", col("p_brand"), string(brand, strings)), binop("=", col("p_container"), string(container, strings))), ["p_partkey"])
    j1 = hash_join(pt, scan("lineitem", ["l_partkey", "l_quantity", "l_extendedprice"]), [("p_partkey", "l_partkey")],
                   projection=["p_partkey", "l_quantity", "l_extendedprice"])
    j1 = project(j1, ["l_quantity", "l_extendedprice", "p_partkey"])
    avgq = two_phase(project(scan("lineitem", ["l_partkey", "l_quantity"]), [(col("l_partkey"), "k"), (col("l_quantity"), "q")]),
                     ["k"], [("avg", col("q"), "avg_q", D152)])
    thr = project(avgq, [(binop("*", dec(2, 1, 1), col("avg_q")), "limit_q"), "k"])
    j2 = hash_join(j1, thr, [("p_partkey", "k")], filter=binop("<", col("l_quantity"), col("limit_q")), projection=["l_extendedprice"])
    a = two_phase(j2, [], [("sum", col("l_extendedprice"), "s", D152)])
    return project(a, [(binop("/", col("s"), dec(70, 2, 1)), "avg_yearly")])


def q21(strings="Utf8View", nation="ARGENTINA") -> Node:
    """test_tpch.plan.yaml:608-645: EXISTS / NOT EXISTS with `l_suppkey <>` become LeftSemi / LeftAnti joins with a residual filter"""
    late = binop(">", col("l_receiptdate"), col("l_commitdate"))
    nat = filter_(scan("nation", ["n_nationkey", "n_name"]), binop("=", col("n_name"), string(nation, strings)), ["n_nationkey"])
    l1 = filter_(scan("lineitem", ["l_orderkey", "l_suppkey", "l_commitdate", "l_receiptdate"]), late, ["l_orderkey", "l_suppkey"])
    ja = hash_join(scan("supplier", ["s_suppkey", "s_name", "s_nationkey"]), l1, [("s_suppkey", "l_suppkey")],
                   projection=["s_name", "s_nationkey", "l_orderkey", "l_suppkey"])
    of = filter_(scan("orders", ["o_orderkey", "o_orderstatus"]), binop("=", col("o_orderstatus"), string("F", strings)), ["o_orderkey"])
    jb = hash_join(ja, of, [("l_orderkey", "o_orderkey")], projection=["s_name", "s_nationkey", "l_orderkey", "l_suppkey"])
    jc = hash_join(nat, jb, [("n_nationkey", "s_nationkey")], projection=["s_name", "l_orderkey", "l_suppkey"])
    l2 = project(scan("lineitem", ["l_orderkey", "l_suppkey"]), [(col("l_orderkey"), "l2_orderkey"), (col("l_suppkey"), "l2_suppkey")])
    semi = hash_join(jc, l2, [("l_orderkey", "l2_orderkey")], join_type="left_semi", filter=binop("!=", col("l2_suppkey"), col("l_suppkey")))
    l3 = project(filter_(scan("lineitem", ["l_orderkey", "l_suppkey", "l_commitdate", "l_receiptdate"]), late, ["l_orderkey", "l_suppkey"]),
                 [(col("l_orderkey"), "l3_orderkey"), (col("l_suppkey"), "l3_suppkey")])
    anti = hash_join(semi, l3, [("l_orderkey", "l3_orderkey")], join_type="left_anti", filter=binop("!=", col("l3_suppkey"), col("l_suppkey")),
                     projection=["s_name"])
    a = two_phase(anti, ["s_name"], [("count", None, "numwait", None)])
    return sort(a, [("numwait", False), ("s_name", True)], fetch=100)


def q22(strings="Utf8View", codes=("24", "34", "16", "30", "33", "14", "13")) -> Node:
    """test_tpch.plan.yaml:647-680: substr() country codes, NOT EXISTS as RightAnti, avg() threshold as a NestedLoopJoinExec"""
    code = substr(col("c_phone"), 1, 2)
    in_codes = {"in": code, "set": [string(c, strings) for c in codes], "negated": False}
    cust = filter_(scan("customer", ["c_custkey", "c_phone", "c_acctbal"]), in_codes)
    anti = hash_join(scan("orders", ["o_custkey"]), cust, [("o_custkey", "c_custkey")], join_type="right_anti", projection=["c_phone", "c_acctbal"])
    right = project(anti, ["c_phone", "c_acctbal", ({"cast": col("c_acctbal"), "to": "Decimal128(19,6)"}, "bal_cmp")])
    pos = filter_(scan("customer", ["c_phone", "c_acctbal"]), and_(binop(">", col("c_acctbal"), dec(0, 15, 2)), in_codes), ["c_acctbal"])
    avgb = two_phase(pos, [], [("avg", col("c_acctbal"), "avg_bal", D152)])
    j = nested_loop_join(avgb, right, binop(">", col("bal_cmp"), col("avg_bal")), ["c_phone", "c_acctbal"])
    p = project(j, [(code, "cntrycode"), "c_acctbal"])
    a = two_phase(p, ["cntrycode"], [("count", None, "numcust", None), ("sum", col("c_acctbal"), "totacctbal", D152)])
    return sort(a, [("cntrycode", True)])


def like(e, pattern: str, negated=False):
    return {"like": e, "pattern": pattern, "negated": negated}


def q2(strings="Utf8View", size=48, type_suffix="%TIN", region="ASIA") -> Node:
    """test_tpch.plan.yaml [02]: the correlated min(ps_supplycost) is decorrelated into a grouped aggregate over the same
    region's suppliers, joined back on (partkey, cost); eight output columns, four of them long strings; TopK 100 on four keys."""
    def region_keys():
        return filter_(scan("region", ["r_regionkey", "r_name"]), binop("=", col("r_name"), string(region, strings)), ["r_regionkey"])
    pt = filter_(scan("part", ["p_partkey", "p_mfgr", "p_type", "p_size"]),
                 and_(binop("=", col("p_size"), lit(size, "Int32")), like(col("p_type"), type_suffix)), ["p_partkey", "p_mfgr"])
    j1 = hash_join(scan("partsupp", ["ps_partkey", "ps_suppkey", "ps_supplycost"]), pt, [("ps_partkey", "p_partkey")],
                   projection=["ps_suppkey", "ps_supplycost", "p_partkey", "p_mfgr"])
    j1 = project(j1, ["p_partkey", "p_mfgr", "ps_suppkey", "ps_supplycost"])
    sup = scan("supplier", ["s_suppkey", "s_name", "s_address", "s_nationkey", "s_phone", "s_acctbal", "s_comment"])
    j2 = hash_join(sup, j1, [("s_suppkey", "ps_suppkey")],
                   projection=["s_name", "s_address", "s_nationkey", "s_phone", "s_acctbal", "s_comment", "p_partkey", "p_mfgr", "ps_supplycost"])
    j2 = project(j2, ["p_partkey", "p_mfgr", "s_name", "s_address", "s_nationkey", "s_phone", "s_acctbal", "s_comment", "ps_supplycost"])
    j3 = hash_join(j2, scan("nation", ["n_nationkey", "n_name", "n_regionkey"]), [("s_nationkey", "n_nationkey")],
                   projection=["p_partkey", "p_mfgr", "s_name", "s_address", "s_phone", "s_acctbal", "s_comment", "ps_supplycost", "n_name", "n_regionkey"])
    j4 = hash_join(region_keys(), j3, [("r_regionkey", "n_regionkey")],
                   projection=["p_partkey", "p_mfgr", "s_name", "s_address", "s_phone", "s_acctbal", "s_comment", "ps_supplycost", "n_name"])
    k1 = hash_join(scan("supplier", ["s_suppkey", "s_nationkey"]),
                   project(scan("partsupp", ["ps_partkey", "ps_suppkey", "ps_supplycost"]), [(col("ps_partkey"), "k_partkey"), (col("ps_suppkey"), "k_suppkey"), (col("ps_supplycost"), "k_cost")]),
                   [("s_suppkey", "k_suppkey")], projection=["s_nationkey", "k_partkey", "k_cost"])
    k1 = project(k1, ["k_partkey", "k_cost", "s_nationkey"])
    k2 = hash_join(scan("nation", ["n_nationkey", "n_regionkey"]), k1, [("n_nationkey", "s_nationkey")], projection=["n_regionkey", "k_partkey", "k_cost"])
    k2 = project(k2, ["k_partkey", "k_cost", "n_regionkey"])
    k3 = hash_join(region_keys(), k2, [("r_regionkey", "n_regionkey")], projection=["k_partkey", "k_cost"])
    mn = two_phase(k3, ["k_partkey"], [("min", col("k_cost"), "min_cost", D152)])
    mn = project(mn, ["min_cost", "k_partkey"])
    j5 = hash_join(j4, mn, [("p_partkey", "k_partkey"), ("ps_supplycost", "min_cost")],
                   projection=["p_partkey", "p_mfgr", "s_name", "s_address", "s_phone", "s_acctbal", "s_comment", "n_name"])
    p = project(j5, ["s_acctbal", "s_name", "n_name", "p_partkey", "p_mfgr", "s_address", "s_phone", "s_comment"])
    return sort(p, [("s_acctbal", False), ("n_name", True), ("s_name", True), ("p_partkey", True)], fetch=100)


def q9(strings="Utf8View", colour="moccasin") -> Node:
    """test_tpch.plan.yaml [09]: p_name LIKE '%colour%' on a 5-word string, five inner joins (one on two keys against a
    duplicate-key build side), profit = price * (1 - discount) - cost * quantity grouped by nation and order year."""
    del strings
    pt = filter_(scan("part", ["p_partkey", "p_name"]), like(col("p_name"), f"%{colour}%"), ["p_partkey"])
    LI = ["l_orderkey", "l_partkey", "l_suppkey", "l_quantity", "l_extendedprice", "l_discount"]
    j1 = hash_join(pt, scan("lineitem", LI), [("p_partkey", "l_partkey")], projection=LI)
    j2 = hash_join(scan("supplier", ["s_suppkey", "s_nationkey"]), j1, [("s_suppkey", "l_suppkey")], projection=["s_nationkey"] + LI)
    j2 = project(j2, LI + ["s_nationkey"])
    j3 = hash_join(j2, scan("partsupp", ["ps_partkey", "ps_suppkey", "ps_supplycost"]), [("l_suppkey", "ps_suppkey"), ("l_partkey", "ps_partkey")],
                   projection=["l_orderkey", "l_quantity", "l_extendedprice", "l_discount", "s_nationkey", "ps_supplycost"])
    j4 = hash_join(j3, scan("orders", ["o_orderkey", "o_orderdate"]), [("l_orderkey", "o_orderkey")],
                   projection=["l_quantity", "l_extendedprice", "l_discount", "s_nationkey", "ps_supplycost", "o_orderdate"])
    j5 = hash_join(j4, scan("nation", ["n_nationkey", "n_name"]), [("s_nationkey", "n_nationkey")])
    amount = binop("-", DISC_PRICE, binop("*", col("ps_supplycost"), col("l_quantity")))          # Decimal128(33,4)
    p = project(j5, [(col("n_name"), "nation"), ({"fn": "date_part", "part": "year", "args": [col("o_orderdate")]}, "o_year"), (amount, "amount")])
    a = two_phase(p, ["nation", "o_year"], [("sum", col("amount"), "sum_profit", "Decimal128(33,4)")])
    return sort(a, [("nation", True), ("o_year", False)])


def q10(strings="Utf8View", first="1993-07-01", last="1993-10-01") -> Node:
    """test_tpch.plan.yaml [10]: three inner joins, then an aggregate on SEVEN group keys (four of them strings, three longer
    than a view's inline 12 bytes), TopK 20 on the sum."""
    ords = filter_(scan("orders", ["o_orderkey", "o_custkey", "o_orderdate"]),
                   and_(binop(">=", col("o_orderdate"), date(first)), binop("<", col("o_orderdate"), date(last))), ["o_orderkey", "o_custkey"])
    C = ["c_custkey", "c_name", "c_address", "c_nationkey", "c_phone", "c_acctbal", "c_comment"]
    j1 = hash_join(ords, scan("customer", C), [("o_custkey", "c_custkey")], projection=["o_orderkey"] + C)
    j1 = project(j1, C + ["o_orderkey"])
    li = filter_(scan("lineitem", ["l_orderkey", "l_extendedprice", "l_discount", "l_returnflag"]),
                 binop("=", col("l_returnflag"), string("R", strings)), ["l_orderkey", "l_extendedprice", "l_discount"])
    j2 = hash_join(j1, li, [("o_orderkey", "l_orderkey")], projection=C + ["l_extendedprice", "l_discount"])
    j3 = hash_join(scan("nation", ["n_nationkey", "n_name"]), j2, [("n_nationkey", "c_nationkey")],
                   projection=["n_name", "c_custkey", "c_name", "c_address", "c_phone", "c_acctbal", "c_comment", "l_extendedprice", "l_discount"])
    j3 = project(j3, ["c_custkey", "c_name", "c_address", "c_phone", "c_acctbal", "c_comment", "l_extendedprice", "l_discount", "n_name"])
    a = two_phase(j3, ["c_custkey", "c_name", "c_acctbal", "c_phone", "n_name", "c_address", "c_comment"],
                  [("sum", DISC_PRICE, "revenue", "Decimal128(32,4)")])
    p = project(a, ["c_custkey", "c_name", "revenue", "c_acctbal", "n_name", "c_address", "c_phone", "c_comment"])
    return sort(p, [("revenue", False)], fetch=20)


def q13(strings="Utf8View", w1="express", w2="requests") -> Node:
    """test_tpch.plan.yaml [13]: LEFT join (customers without orders keep a NULL order key), count(o_orderkey) skips the NULLs,
    then a second aggregate over the counts; the filter is NOT LIKE on a long comment column."""
    del strings
    ords = filter_(scan("orders", ["o_orderkey", "o_custkey", "o_comment"]), like(col("o_comment"), f"%{w1}%{w2}%", True), ["o_orderkey", "o_custkey"])
    j = hash_join(scan("customer", ["c_custkey"]), ords, [("c_custkey", "o_custkey")], join_type="left", projection=["c_custkey", "o_orderkey"])
    a1 = two_phase(j, ["c_custkey"], [("count", col("o_orderkey"), "c_count", "Int64")])
    a2 = two_phase(project(a1, ["c_count"]), ["c_count"], [("count", None, "custdist", None)])
    return sort(a2, [("custdist", False), ("c_count", False)])


def q15(strings="Utf8View", first="1996-08-01", last="1996-11-01") -> Node:
    """test_tpch.plan.yaml [15].1: the revenue view is planned twice -- once under max() (a keyless aggregate over a grouped
    one), once joined to supplier -- and the two meet in a join on the Decimal128(38,4) revenue itself."""
    del strings

    def revenue():
        li = filter_(scan("lineitem", ["l_suppkey", "l_extendedprice", "l_discount", "l_shipdate"]),
                     and_(binop(">=", col("l_shipdate"), date(first)), binop("<", col("l_shipdate"), date(last))), ["l_suppkey", "l_extendedprice", "l_discount"])
        return two_phase(li, ["l_suppkey"], [("sum", DISC_PRICE, "total_revenue", "Decimal128(32,4)")])
    mx = two_phase(project(revenue(), ["total_revenue"]), [], [("max", col("total_revenue"), "max_revenue", "Decimal128(38,4)")])
    sup = scan("supplier", ["s_suppkey", "s_name", "s_address", "s_phone"])
    j1 = hash_join(sup, project(revenue(), [(col("l_suppkey"), "supplier_no"), "total_revenue"]), [("s_suppkey", "supplier_no")],
                   projection=["s_suppkey", "s_name", "s_address", "s_phone", "total_revenue"])
    j2 = hash_join(mx, j1, [("max_revenue", "total_revenue")], projection=["s_suppkey", "s_name", "s_address", "s_phone", "total_revenue"])
    return sort(j2, [("s_suppkey", True)])


def q16(strings="Utf8View", brand="Brand#14", type_prefix="SMALL PLATED%", sizes=(14, 6, 5, 31, 49, 15, 41, 47)) -> Node:
    """test_tpch.plan.yaml [16]: NOT IN (subquery) as LeftAnti, count(DISTINCT) as two stacked aggregates (the inner one has
    group keys only), != / NOT LIKE / IN-list filter."""
    pt = filter_(scan("part", ["p_partkey", "p_brand", "p_type", "p_size"]),
                 and_(binop("!=", col("p_brand"), string(brand, strings)), like(col("p_type"), type_prefix, True),
                      {"in": col("p_size"), "set": [lit(v, "Int32") for v in sizes], "negated": False}))
    j1 = hash_join(scan("partsupp", ["ps_partkey", "ps_suppkey"]), pt, [("ps_partkey", "p_partkey")], projection=["ps_suppkey", "p_brand", "p_type", "p_size"])
    bad = filter_(scan("supplier", ["s_suppkey", "s_comment"]), like(col("s_comment"), "%Customer%Complaints%"), ["s_suppkey"])
    anti = hash_join(j1, bad, [("ps_suppkey", "s_suppkey")], join_type="left_anti")
    d = two_phase(anti, ["p_brand", "p_type", "p_size", (col("ps_suppkey"), "alias1")], [])
    c = two_phase(d, ["p_brand", "p_type", "p_size"], [("count", col("alias1"), "supplier_cnt", "Int64")])
    return sort(c, [("supplier_cnt", False), ("p_brand", True), ("p_type", True), ("p_size", True)])


def q20(strings="Utf8View", colour="blanched", nation="KENYA", first="1993-01-01", last="1994-01-01") -> Node:
    """test_tpch.plan.yaml [20]: IN (subquery) chains become RightSemi / LeftSemi joins; the correlated 0.5 * sum(l_quantity)
    is a grouped aggregate joined on two keys with a residual `availqty > half` filter in Decimal128(23,3)."""
    nat = filter_(scan("nation", ["n_nationkey", "n_name"]), binop("=", col("n_name"), string(nation, strings)), ["n_nationkey"])
    j1 = hash_join(nat, scan("supplier", ["s_suppkey", "s_name", "s_address", "s_nationkey"]), [("n_nationkey", "s_nationkey")],
                   projection=["s_suppkey", "s_name", "s_address"])
    pt = filter_(scan("part", ["p_partkey", "p_name"]), like(col("p_name"), f"{colour}%"), ["p_partkey"])
    rs = hash_join(pt, scan("partsupp", ["ps_partkey", "ps_suppkey", "ps_availqty"]), [("p_partkey", "ps_partkey")], join_type="right_semi")
    li = filter_(scan("lineitem", ["l_partkey", "l_suppkey", "l_quantity", "l_shipdate"]),
                 and_(binop(">=", col("l_shipdate"), date(first)), binop("<", col("l_shipdate"), date(last))), ["l_partkey", "l_suppkey", "l_quantity"])
    ag = two_phase(li, ["l_partkey", "l_suppkey"], [("sum", col("l_quantity"), "sum_qty", D152)])
    half = {"cast": binop("*", dec(5, 1, 1), col("sum_qty")), "to": "Decimal128(23,3)"}
    thr = project(ag, [(half, "half_qty"), "l_partkey", "l_suppkey"])
    j2 = hash_join(rs, thr, [("ps_partkey", "l_partkey"), ("ps_suppkey", "l_suppkey")],
                   filter=binop(">", {"cast": col("ps_availqty"), "to": "Decimal128(23,3)"}, col("half_qty")), projection=["ps_suppkey"])
    semi = hash_join(j1, j2, [("s_suppkey", "ps_suppkey")], join_type="left_semi", projection=["s_name", "s_address"])
    return sort(semi, [("s_name", True)])


TPCH = {"q1": q1, "q3": q3, "q4": q4, "q5": q5, "q6": q6, "q7": q7, "q8": q8, "q11": q11, "q12": q12, "q14": q14, "q17": q17, "q18": q18, "q19": q19,
        "q21": q21, "q22": q22, "q2": q2, "q9": q9, "q10": q10, "q13": q13, "q15": q15, "q16": q16, "q20": q20}
