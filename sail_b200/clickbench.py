"""ClickBench (BASELINE.json configs[4]) as trees of operator specs, numbered like the reference's 0-based query ids
(python/pysail/data/clickbench/queries.sql, one query per line; python/pysail/tests/spark/test_clickbench.py:150-158).

The shapes follow the reference's plan snapshot (python/pysail/tests/spark/__snapshots__/test_clickbench.plan.yaml):
COUNT(DISTINCT x) is two stacked aggregates, the inner one with group keys only ([04], [08], [10]); grouped queries are
Partial -> Hash repartition -> FinalPartitioned ([07], [12]); ORDER BY .. LIMIT k is `SortExec: TopK(fetch=k)` ([08]..[17]).
`OFFSET m` queries keep `TopK(fetch=m+k)` on the GPU and leave the final GlobalLimitExec(skip=m) -- a slice of at most
m+k rows -- to the caller: `QUERIES[id].skip`.

37 of the 43 queries run.  What does NOT, and why (the library rejects such specs at plan time with SAILGPU_ERR_UNSUPPORTED,
nothing falls back):
  18, 42  extract(minute ..) / date_trunc('minute', ..) on a Timestamp: planned in TIMESTAMP_QUERIES (over the Int64 EventTime of
          the view, cast to Timestamp(us, UTC) as the reference's scan projection does)
  21, 22  MIN(URL) / MIN(Title): min/max over strings (planned below as REJECTED, the tests pin the plan-time error)
  27      length(URL): character_length, planned in LENGTH_QUERIES
  28      regexp_replace(): a scalar string function outside {substr, like, character_length}
[09] runs in QUERIES as the two-level rewrite c9; DISTINCT_QUERIES['c9_single'] is the reference's own shape, one single-mode
aggregate with count(DISTINCT UserID) next to the plain aggregates.
Strings are Utf8View and EventTime is Int64 seconds (see datagen/hits.py); [23] `SELECT *` selects ten columns, [29] runs as six aggregates.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable

from .plans import Node, aggregate, and_, binop, char_length, col, date, filter_, like, lit, project, scan, sort, string, two_phase

I16, I32, I64 = "Int16", "Int32", "Int64"
COUNT_STAR = ("count", None, "c", None)


def hits(columns):
    return scan("hits", columns)


def view(columns: list) -> dict:
    """The reference's view over hits.parquet (test_clickbench.py:134-136) as a projection spec over the stored `columns`
    (datagen/hits.py:stored): EventDate, stored as UInt16 days since the epoch, becomes Date32 -- what
    `date_add('1970-01-01', EventDate)` gives -- and every other column is passed through.  The binary strings are already
    Utf8View when the scan reads them with `binary_as_string`; EventTime stays Int64 (see datagen/hits.py).  A projection
    has at most 24 outputs, so the view is applied per scan, over the columns it reads (over_view), as DataFusion pushes the
    view's projection into each scan."""
    def expr(i, name):
        return {"cast": {"col": i}, "to": "Date32"} if name == "EventDate" else {"col": i}
    return {"op": "projection", "exprs": [{"expr": expr(i, n), "name": n} for i, n in enumerate(columns)]}


def over_view(plan: Node) -> Node:
    """`plan` with every scan of hits read through the view: the plan to run over the stored table (datagen/hits.py:stored)"""
    if plan.spec["op"] == "scan":
        return Node(view(plan.names), [plan], list(plan.names))
    return Node(plan.spec, [over_view(c) for c in plan.inputs], list(plan.names))


def ne_empty(c):
    return binop("!=", col(c), string(""))


def count_distinct(child: Node, keys: list, what: str, name: str, extra: list | None = None) -> Node:
    """count(DISTINCT what) GROUP BY keys: the inner aggregate groups by (keys, what) and keeps nothing else, the outer one
    counts rows per key (test_clickbench.plan.yaml [04], [08], [10])"""
    inner = two_phase(child, list(keys) + [(col(what), "alias1")], [])
    return two_phase(inner, list(keys), [("count", col("alias1"), name, I64)] + (extra or []))


def c0():
    return two_phase(hits(["AdvEngineID"]), [], [("count", None, "count(*)", None)])


def c1():
    f = filter_(hits(["AdvEngineID"]), binop("!=", col("AdvEngineID"), lit(0, I16)))
    return two_phase(f, [], [("count", None, "count(*)", None)])


def c2():
    return two_phase(hits(["AdvEngineID", "ResolutionWidth"]), [],
                     [("sum", col("AdvEngineID"), "sum(AdvEngineID)", I16), ("count", None, "count(*)", None), ("avg", col("ResolutionWidth"), "avg(ResolutionWidth)", I16)])


def c3():
    return two_phase(hits(["UserID"]), [], [("avg", col("UserID"), "avg(UserID)", I64)])


def c4():
    return count_distinct(hits(["UserID"]), [], "UserID", "count(DISTINCT UserID)")


def c5():
    return count_distinct(hits(["SearchPhrase"]), [], "SearchPhrase", "count(DISTINCT SearchPhrase)")


def c6():
    return two_phase(hits(["EventDate"]), [], [("min", col("EventDate"), "min(EventDate)", "Date32"), ("max", col("EventDate"), "max(EventDate)", "Date32")])


def c7():
    f = filter_(hits(["AdvEngineID"]), binop("!=", col("AdvEngineID"), lit(0, I16)))
    return sort(two_phase(f, ["AdvEngineID"], [("count", None, "count(*)", None)]), [("count(*)", False)])


def c8():
    return sort(count_distinct(hits(["RegionID", "UserID"]), ["RegionID"], "UserID", "u"), [("u", False)], fetch=10)


def c9():
    """one DISTINCT next to plain aggregates: grouped once by (RegionID, UserID) with the plain aggregates as per-pair partial
    results, then by RegionID -- sum of sums, sum of counts, avg = sum / count in Float64 (exact: the Int16 sums stay far below
    2^53), count of pairs = count(DISTINCT UserID).  DataFusion's SingleDistinctToGroupBy does this rewrite for sum/count/min/max;
    the reference's [09] keeps one AggregateExec with a distinct accumulator instead, which has no GPU counterpart."""
    inner = two_phase(hits(["RegionID", "UserID", "AdvEngineID", "ResolutionWidth"]), ["RegionID", (col("UserID"), "alias1")],
                      [("sum", col("AdvEngineID"), "s", I16), ("count", None, "n", None), ("sum", col("ResolutionWidth"), "rs", I16), ("count", col("ResolutionWidth"), "rn", I16)])
    outer = two_phase(inner, ["RegionID"], [("sum", col("s"), "sum(AdvEngineID)", I64), ("sum", col("n"), "c", I64), ("sum", col("rs"), "rs", I64), ("sum", col("rn"), "rn", I64),
                                            ("count", col("alias1"), "count(DISTINCT UserID)", I64)])
    avg = binop("/", {"cast": col("rs"), "to": "Float64"}, {"cast": col("rn"), "to": "Float64"})
    p = project(outer, ["RegionID", "sum(AdvEngineID)", "c", (avg, "avg(ResolutionWidth)"), "count(DISTINCT UserID)"])
    return sort(p, [("c", False)], fetch=10)


def c9_single():
    """[09] in the reference's plan shape (test_clickbench.plan.yaml [09]): one single-mode aggregate by RegionID with
    count(DISTINCT UserID) next to the plain aggregates -- the DISTINCT accumulator runs behind a per-(RegionID, UserID) gate on
    the GPU -- then the projection and TopK(fetch=10) on c"""
    a = aggregate(hits(["RegionID", "UserID", "AdvEngineID", "ResolutionWidth"]), "single", ["RegionID"],
                  [("sum", col("AdvEngineID"), "sum(AdvEngineID)", I16), ("count", None, "c", None), ("avg", col("ResolutionWidth"), "avg(ResolutionWidth)", I16),
                   ("count", col("UserID"), "count(DISTINCT UserID)", I64, True)])
    p = project(a, ["RegionID", "sum(AdvEngineID)", "c", "avg(ResolutionWidth)", "count(DISTINCT UserID)"])
    return sort(p, [("c", False)], fetch=10)


def c10():
    f = filter_(hits(["UserID", "MobilePhoneModel"]), ne_empty("MobilePhoneModel"))
    return sort(count_distinct(f, ["MobilePhoneModel"], "UserID", "u"), [("u", False)], fetch=10)


def c11():
    f = filter_(hits(["UserID", "MobilePhone", "MobilePhoneModel"]), ne_empty("MobilePhoneModel"))
    return sort(count_distinct(f, ["MobilePhone", "MobilePhoneModel"], "UserID", "u"), [("u", False)], fetch=10)


def c12():
    f = filter_(hits(["SearchPhrase"]), ne_empty("SearchPhrase"))
    return sort(two_phase(f, ["SearchPhrase"], [COUNT_STAR]), [("c", False)], fetch=10)


def c13():
    f = filter_(hits(["UserID", "SearchPhrase"]), ne_empty("SearchPhrase"))
    return sort(count_distinct(f, ["SearchPhrase"], "UserID", "u"), [("u", False)], fetch=10)


def c14():
    f = filter_(hits(["SearchEngineID", "SearchPhrase"]), ne_empty("SearchPhrase"))
    return sort(two_phase(f, ["SearchEngineID", "SearchPhrase"], [COUNT_STAR]), [("c", False)], fetch=10)


def c15():
    return sort(two_phase(hits(["UserID"]), ["UserID"], [("count", None, "count(*)", None)]), [("count(*)", False)], fetch=10)


def c16():
    return sort(two_phase(hits(["UserID", "SearchPhrase"]), ["UserID", "SearchPhrase"], [("count", None, "count(*)", None)]), [("count(*)", False)], fetch=10)


def c17():
    """no ORDER BY: any ten groups are a valid answer (the reference plans a CoalescePartitionsExec with fetch=10)"""
    a = two_phase(hits(["UserID", "SearchPhrase"]), ["UserID", "SearchPhrase"], [("count", None, "count(*)", None)])
    return sort(a, [("UserID", True), ("SearchPhrase", True)], fetch=10)


def c19(user: int = 435090932899640449):
    return filter_(hits(["UserID"]), binop("=", col("UserID"), lit(user, I64)))


def c20():
    f = filter_(hits(["URL"]), like(col("URL"), "%google%"))
    return two_phase(f, [], [("count", None, "count(*)", None)])


def c21():
    f = filter_(hits(["URL", "SearchPhrase"]), and_(like(col("URL"), "%google%"), ne_empty("SearchPhrase")))
    a = two_phase(f, ["SearchPhrase"], [("min", col("URL"), "min(URL)", "Utf8View"), COUNT_STAR])
    return sort(a, [("c", False)], fetch=10)


def c22():
    """min / count / count(DISTINCT) together: the same two-level rewrite as c9 (min of mins, sum of counts, count of pairs)"""
    f = filter_(hits(["Title", "UserID", "URL", "SearchPhrase"]),
                and_(like(col("Title"), "%Google%"), like(col("URL"), "%.google.%", True), ne_empty("SearchPhrase")))
    inner = two_phase(f, ["SearchPhrase", (col("UserID"), "alias1")], [("min", col("URL"), "mu", "Utf8View"), ("min", col("Title"), "mt", "Utf8View"), ("count", None, "n", None)])
    outer = two_phase(inner, ["SearchPhrase"], [("min", col("mu"), "min(URL)", "Utf8View"), ("min", col("mt"), "min(Title)", "Utf8View"), ("sum", col("n"), "c", I64),
                                                ("count", col("alias1"), "count(DISTINCT UserID)", I64)])
    return sort(outer, [("c", False)], fetch=10)


STAR = ["WatchID", "Title", "EventTime", "EventDate", "CounterID", "ClientIP", "RegionID", "UserID", "URL", "Referer"]


def c23(columns=None):
    """`SELECT *`: ten columns -- a filter pipeline stages at most 20 column buffers per tile, validity bitmaps included (the full
    105-column row needs the filter run per column chunk against one selection vector, which the library does not do yet)"""
    f = filter_(hits(list(columns or STAR)), like(col("URL"), "%google%"))
    return sort(f, [("EventTime", True)], fetch=10)


def c24():
    f = filter_(hits(["EventTime", "SearchPhrase"]), ne_empty("SearchPhrase"))
    return project(sort(f, [("EventTime", True)], fetch=10), ["SearchPhrase"])


def c25():
    f = filter_(hits(["SearchPhrase"]), ne_empty("SearchPhrase"))
    return sort(f, [("SearchPhrase", True)], fetch=10)


def c26():
    f = filter_(hits(["EventTime", "SearchPhrase"]), ne_empty("SearchPhrase"))
    return project(sort(f, [("EventTime", True), ("SearchPhrase", True)], fetch=10), ["SearchPhrase"])


def c29(part: int = 0, n_sums: int = 90, per_pass: int = 15):
    """ninety sums of one Int16 column: an aggregate carries at most 16 accumulators, so the sums are computed fifteen at a time --
    six keyless aggregates over the same 2-byte column (`QUERIES["c29"].parts`), whose one-row results the caller puts side by
    side.  The reference plans a single AggregateExec."""
    w = {"cast": col("ResolutionWidth"), "to": I32}          # Spark widens SMALLINT + INT literal to INT before the sum
    sums = [("sum", w if i == 0 else binop("+", w, lit(i, I32)), "sum(ResolutionWidth)" if i == 0 else f"sum((ResolutionWidth + {i}))", I32) for i in range(n_sums)]
    return two_phase(hits(["ResolutionWidth"]), [], sums[part * per_pass:(part + 1) * per_pass])


def _c30(keys, filtered):
    src = hits(["SearchEngineID", "ClientIP", "WatchID", "IsRefresh", "ResolutionWidth", "SearchPhrase"])
    if filtered:
        src = filter_(src, ne_empty("SearchPhrase"), ["SearchEngineID", "ClientIP", "WatchID", "IsRefresh", "ResolutionWidth"])
    a = two_phase(src, keys, [COUNT_STAR, ("sum", col("IsRefresh"), "sum(IsRefresh)", I16), ("avg", col("ResolutionWidth"), "avg(ResolutionWidth)", I16)])
    return sort(a, [("c", False)], fetch=10)


def c30():
    return _c30(["SearchEngineID", "ClientIP"], True)


def c31():
    return _c30(["WatchID", "ClientIP"], True)


def c32():
    return _c30(["WatchID", "ClientIP"], False)


def c33():
    return sort(two_phase(hits(["URL"]), ["URL"], [COUNT_STAR]), [("c", False)], fetch=10)


def c34():
    """`SELECT 1, URL, ..GROUP BY 1, URL`: the optimiser folds the constant key away and projects it back"""
    a = two_phase(hits(["URL"]), ["URL"], [COUNT_STAR])
    return sort(project(a, [(lit(1, I32), "1"), "URL", "c"]), [("c", False)], fetch=10)


def c35():
    ip = col("ClientIP")
    keys = ["ClientIP"] + [(binop("-", ip, lit(i, I32)), f"(ClientIP - {i})") for i in (1, 2, 3)]
    return sort(two_phase(hits(["ClientIP"]), keys, [COUNT_STAR]), [("c", False)], fetch=10)


def _july(counter=62, first="2013-07-01", last="2013-07-31"):
    return [binop("=", col("CounterID"), lit(counter, I32)), binop(">=", col("EventDate"), date(first)), binop("<=", col("EventDate"), date(last))]


def zero(c):
    return binop("=", col(c), lit(0, I16))


def c36():
    f = filter_(hits(["CounterID", "EventDate", "DontCountHits", "IsRefresh", "URL"]), and_(*_july(), zero("DontCountHits"), zero("IsRefresh"), ne_empty("URL")), ["URL"])
    return sort(two_phase(f, ["URL"], [("count", None, "PageViews", None)]), [("PageViews", False)], fetch=10)


def c37():
    f = filter_(hits(["CounterID", "EventDate", "DontCountHits", "IsRefresh", "Title"]), and_(*_july(), zero("DontCountHits"), zero("IsRefresh"), ne_empty("Title")), ["Title"])
    return sort(two_phase(f, ["Title"], [("count", None, "PageViews", None)]), [("PageViews", False)], fetch=10)


def c38(skip=1000):
    f = filter_(hits(["CounterID", "EventDate", "IsRefresh", "IsLink", "IsDownload", "URL"]),
                and_(*_july(), zero("IsRefresh"), binop("!=", col("IsLink"), lit(0, I16)), zero("IsDownload")), ["URL"])
    return sort(two_phase(f, ["URL"], [("count", None, "PageViews", None)]), [("PageViews", False)], fetch=skip + 10)


def c39(skip=1000):
    f = filter_(hits(["CounterID", "EventDate", "IsRefresh", "TraficSourceID", "SearchEngineID", "AdvEngineID", "Referer", "URL"]), and_(*_july(), zero("IsRefresh")),
                ["TraficSourceID", "SearchEngineID", "AdvEngineID", "Referer", "URL"])
    src = {"case": [[and_(zero("SearchEngineID"), zero("AdvEngineID")), col("Referer")]], "else": string("")}
    a = two_phase(f, ["TraficSourceID", "SearchEngineID", "AdvEngineID", (src, "Src"), (col("URL"), "Dst")], [("count", None, "PageViews", None)])
    return sort(a, [("PageViews", False)], fetch=skip + 10)


def c40(referer_hash: int = 3594120000172545465, skip=100):
    f = filter_(hits(["CounterID", "EventDate", "IsRefresh", "TraficSourceID", "RefererHash", "URLHash"]),
                and_(*_july(), zero("IsRefresh"), {"in": col("TraficSourceID"), "set": [lit(-1, I16), lit(6, I16)], "negated": False},
                     binop("=", col("RefererHash"), lit(referer_hash, I64))), ["URLHash", "EventDate"])
    return sort(two_phase(f, ["URLHash", "EventDate"], [("count", None, "PageViews", None)]), [("PageViews", False)], fetch=skip + 10)


def c41(url_hash: int = 2868770270353813622, skip=10000):
    f = filter_(hits(["CounterID", "EventDate", "IsRefresh", "DontCountHits", "URLHash", "WindowClientWidth", "WindowClientHeight"]),
                and_(*_july(), zero("IsRefresh"), zero("DontCountHits"), binop("=", col("URLHash"), lit(url_hash, I64))), ["WindowClientWidth", "WindowClientHeight"])
    return sort(two_phase(f, ["WindowClientWidth", "WindowClientHeight"], [("count", None, "PageViews", None)]), [("PageViews", False)], fetch=skip + 10)


TS_US = "Timestamp(us, UTC)"


def event_ts():
    """the reference's scan projection `CAST(EventTime * 1000000 AS Timestamp(us, "UTC"))` (EventTime is Int64 seconds)"""
    return {"cast": binop("*", col("EventTime"), lit(1000000, I64)), "to": TS_US}


def c18():
    """extract(minute ..) as a group key of one single-partitioned aggregate (test_clickbench.plan.yaml [18])"""
    minute = {"fn": "date_part", "part": "minute", "args": [event_ts()]}
    a = aggregate(hits(["UserID", "EventTime", "SearchPhrase"]), "single", ["UserID", (minute, "m"), "SearchPhrase"], [("count", None, "count(*)", None)])
    return sort(a, [("count(*)", False)], fetch=10)


def c42(skip=1000):
    """date_trunc('minute', ..) as the key of Partial -> Hash -> FinalPartitioned under TopK(fetch=skip+10) ascending on the Timestamp"""
    f = filter_(hits(["CounterID", "EventDate", "IsRefresh", "DontCountHits", "EventTime"]),
                and_(*_july(first="2013-07-14", last="2013-07-15"), zero("IsRefresh"), zero("DontCountHits")), ["EventTime"])
    a = two_phase(f, [({"fn": "date_trunc", "part": "minute", "args": [event_ts()]}, "M")], [("count", None, "PageViews", None)])
    return sort(a, [("M", True)], fetch=skip + 10)


def c27(min_count: int = 100000):
    """avg(length(URL)) per CounterID: Spark's `length` is DataFusion's `character_length` in both the Partial and the
    FinalPartitioned aggregate (test_clickbench.plan.yaml [27]); HAVING is a filter on the final count"""
    f = filter_(hits(["CounterID", "URL"]), ne_empty("URL"))
    a = two_phase(f, ["CounterID"], [("avg", char_length(col("URL")), "l", I32), COUNT_STAR])
    return sort(filter_(a, binop(">", col("c"), lit(min_count, I64))), [("l", False)], fetch=25)


@dataclass
class Query:
    plan: Callable[..., Node]
    sql: int                       # 0-based line of queries.sql
    order: tuple = ()              # ORDER BY columns of the result, in order (the rest of a row is only determined up to ties)
    skip: int = 0                  # OFFSET applied by the caller (GlobalLimitExec) to the TopK(fetch=skip+k) result
    floats: tuple = ()             # Float64 result columns (compared within 1e-6 relative)
    params: tuple = ()             # literals of the SQL text that a synthetic table has to supply (plan(**{name: value}))
    parts: int = 1                 # the result is plan(part=0) .. plan(part=parts-1) side by side ([29])
    note: str = ""


def top_sort(plan: Node):
    """the ORDER BY [.. LIMIT] node of a plan: the root, or the child of a root projection ([24], [26]); None if there is none"""
    if plan.spec["op"] == "sort":
        return plan
    if plan.spec["op"] == "projection" and plan.inputs[0].spec["op"] == "sort":
        return plan.inputs[0]
    return None


def without_limit(sort_node: Node) -> Node:
    return Node({**sort_node.spec, "fetch": None}, sort_node.inputs, sort_node.names)


QUERIES = {
    "c0": Query(c0, 0), "c1": Query(c1, 1), "c2": Query(c2, 2, floats=(2,)), "c3": Query(c3, 3, floats=(0,)), "c4": Query(c4, 4), "c5": Query(c5, 5), "c6": Query(c6, 6),
    "c7": Query(c7, 7, order=("count(*)",)), "c8": Query(c8, 8, order=("u",)),
    "c9": Query(c9, 9, order=("c",), floats=(3,)),
    "c10": Query(c10, 10, order=("u",)), "c11": Query(c11, 11, order=("u",)), "c12": Query(c12, 12, order=("c",)), "c13": Query(c13, 13, order=("u",)),
    "c14": Query(c14, 14, order=("c",)), "c15": Query(c15, 15, order=("count(*)",)), "c16": Query(c16, 16, order=("count(*)",)),
    "c17": Query(c17, 17, order=("UserID", "SearchPhrase"), note="LIMIT without ORDER BY: the plan orders by the keys to make the ten rows deterministic"),
    "c19": Query(c19, 19, params=("user",)), "c20": Query(c20, 20),
    "c23": Query(c23, 23, order=("EventTime",)), "c24": Query(c24, 24, order=("EventTime",)), "c25": Query(c25, 25, order=("SearchPhrase",)), "c26": Query(c26, 26, order=("EventTime", "SearchPhrase")),
    "c29": Query(c29, 29, parts=6), "c30": Query(c30, 30, order=("c",), floats=(4,)), "c31": Query(c31, 31, order=("c",), floats=(4,)), "c32": Query(c32, 32, order=("c",), floats=(4,)),
    "c33": Query(c33, 33, order=("c",)), "c34": Query(c34, 34, order=("c",)), "c35": Query(c35, 35, order=("c",)),
    "c36": Query(c36, 36, order=("PageViews",)), "c37": Query(c37, 37, order=("PageViews",)),
    "c38": Query(c38, 38, order=("PageViews",), skip=1000), "c39": Query(c39, 39, order=("PageViews",), skip=1000),
    "c40": Query(c40, 40, order=("PageViews",), skip=100, params=("referer_hash",)), "c41": Query(c41, 41, order=("PageViews",), skip=10000, params=("url_hash",)),
}
# planned, but rejected by the library at plan time (SAILGPU_ERR_UNSUPPORTED: min/max over strings) -- kept so that the tests pin the rejection
REJECTED = {"c21": Query(c21, 21, order=("c",)), "c22": Query(c22, 22, order=("c",))}
# the two queries that need the Timestamp type: planned here, outside QUERIES, so that the split above stays as the tests pin it
TIMESTAMP_QUERIES = {"c18": Query(c18, 18, order=("count(*)",)), "c42": Query(c42, 42, order=("M",), skip=1000)}
# [27] needs character_length: planned outside QUERIES as well
LENGTH_QUERIES = {"c27": Query(c27, 27, order=("l",), floats=(1,), params=("min_count",))}
# [09] as the reference plans it (a DISTINCT aggregate next to plain ones, mode single); QUERIES keeps the two-level rewrite c9
DISTINCT_QUERIES = {"c9_single": Query(c9_single, 9, order=("c",), floats=(3,))}
NOT_PLANNED = {18: "extract(minute FROM Timestamp): TIMESTAMP_QUERIES['c18']", 27: "length(URL): LENGTH_QUERIES['c27']", 28: "regexp_replace(Referer, ..)",
               42: "date_trunc('minute', Timestamp): TIMESTAMP_QUERIES['c42']"}
