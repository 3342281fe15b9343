"""Operators ordered or grouped by string keys, over resident input: a full sort, TopK, a k-way merge, a sort-based aggregate.
String keys of these operators are encoded as their dense rank (string_ranks, relational.cu); this script times them and
prints a digest of every output, so that two builds of the library can be compared on the same inputs.

    python scripts/bench_sort_strings.py [--lib path/to/libsailgpu.so] [--scale 1.0] [--only name,name]

Workloads (row counts times --scale):
  sort_urls       50 M URL-like rows (84 B on average, about 3 % longer than 256 B) with an Int64 payload, ORDER BY url
  sort_urls_200   the same rows cut to 200 B
  topk_phrases    TopK 10 over 100 M SearchPhrase-like rows (a third empty, the rest 2-60 B)
  merge_8_runs    a merge of 8 sorted runs of 5 M URL-like rows
  q10_agg         a Q10-shaped sort-based aggregate: 10 M rows, seven group keys of which four are strings, ~1 M groups
  few_long        the worst case of the ranking: 10 M rows over 100 distinct 2 KB strings that share their first 1000 bytes
Strings are views into a small vocabulary, so the host never materialises the column.  Each workload runs four times; the
best of the last three is reported with gpu.host_syncs of that run and the growth of the device memory the library holds
(its size-class cache keeps what the operator allocated) after the first run.  A build that refuses a workload reports the
error instead.  Prints one JSON object per workload; the first line names the card and its power limit."""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np
import pyarrow as pa

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.bench_timestamp import card  # noqa: E402


def views_of(vocab, idx, nulls=None):
    """a Utf8View array whose row i is vocab[idx[i]], built from one data buffer holding the vocabulary once"""
    enc = [v.encode() for v in vocab]
    lens = np.array([len(b) for b in enc], dtype=np.uint32)
    offs = np.zeros(len(enc), dtype=np.uint64)
    offs[1:] = np.cumsum(lens[:-1], dtype=np.uint64)
    data = b"".join(enc)
    rec = np.zeros((len(enc), 16), dtype=np.uint8)
    for i, b in enumerate(enc):
        rec[i, 0:4] = np.frombuffer(np.uint32(len(b)).tobytes(), dtype=np.uint8)
        if len(b) <= 12:
            rec[i, 4:4 + len(b)] = np.frombuffer(b, dtype=np.uint8)
        else:
            rec[i, 4:8] = np.frombuffer(b[:4], dtype=np.uint8)
            rec[i, 12:16] = np.frombuffer(np.uint32(offs[i]).tobytes(), dtype=np.uint8)
    views = rec[idx]
    validity = None
    if nulls is not None:
        validity = pa.py_buffer(np.packbits(~nulls, bitorder="little").tobytes())
    return pa.Array.from_buffers(pa.string_view(), len(idx), [validity, pa.py_buffer(views.tobytes()), pa.py_buffer(data)],
                                 null_count=-1 if nulls is not None else 0)


def url_vocab(rng, n, cap=None):
    doms = ["example.com", "news.site.ru", "shop.example.org", "video.host.net", "maps.mirror.io"]
    out = []
    for i in range(n):
        k = int(rng.integers(20, 140)) if rng.random() > 0.03 else int(rng.integers(257, 1200))
        u = f"http://{doms[i % len(doms)]}/{i * 2654435761 % 10**9:09d}/" + "seg/" * (k // 4)
        u = u[:k]
        out.append(u[:cap] if cap else u)
    return sorted(set(out))


def phrase_vocab(rng, n):
    words = ["buy", "cheap", "car", "weather", "moscow", "news", "film", "online", "free", "download", "music", "tv"]
    out = [""]
    for _ in range(n):
        out.append(" ".join(words[j] for j in rng.integers(0, len(words), int(rng.integers(1, 8))))[: int(rng.integers(2, 61))])
    return sorted(set(out))


def sort_spec(cols, fetch=None):
    s = {"op": "sort", "keys": [{"expr": {"col": c}, "asc": True, "nulls_first": True} for c in cols]}
    if fetch is not None:
        s["fetch"] = fetch
    return s


def workloads(scale, rng):
    n = lambda x: max(2048, int(x * scale))       # noqa: E731
    urls = url_vocab(rng, 1_000_000)
    urls200 = sorted(set(u[:200] for u in urls))
    phrases = phrase_vocab(rng, 300_000)

    def sort_of(vocab, rows):
        def make():
            t = pa.table({"url": views_of(vocab, rng.integers(0, len(vocab), rows)), "p": pa.array(np.arange(rows, dtype=np.int64))})
            return sort_spec([0]), [[t]]
        return make

    def topk():
        rows = n(100e6)
        idx = np.where(rng.random(rows) < 0.33, 0, rng.integers(0, len(phrases), rows))
        t = pa.table({"SearchPhrase": views_of(phrases, idx), "p": pa.array(np.arange(rows, dtype=np.int64))})
        return sort_spec([0], fetch=10), [[t]]

    def merge():
        rows = n(5e6)
        runs = [pa.table({"url": views_of(urls, np.sort(rng.integers(0, len(urls), rows))), "p": pa.array(np.arange(rows, dtype=np.int64))}) for _ in range(8)]
        spec = {"op": "sort_preserving_merge", "keys": sort_spec([0])["keys"], "runs": "batches"}
        return spec, [runs]

    def q10():
        rows = n(10e6)
        cust = rng.integers(0, max(1, rows // 10), rows)
        names = [f"Customer#{i:09d}" for i in range(max(1, rows // 10))]
        addrs = ["".join(chr(97 + (i * 7 + j) % 26) for j in range(10 + i % 30)) for i in range(997)]
        nations = ["ALGERIA", "ARGENTINA", "BRAZIL", "CANADA", "EGYPT", "UNITED KINGDOM", "UNITED STATES"]
        comments = [("carefully final deposits detect slyly agai " * 4)[: 29 + i % 88] + str(i) for i in range(991)]
        t = pa.table({"c_custkey": pa.array(cust.astype(np.int64)), "c_name": views_of(names, cust),
                      "c_acctbal": pa.array((cust * 37 % 1000000).astype(np.int64)), "c_phone": views_of([f"{10 + i % 25}-{i:03d}-555-0100" for i in range(1000)], cust % 1000),
                      "n_name": views_of(nations, cust % len(nations)), "c_address": views_of(addrs, cust % len(addrs)),
                      "c_comment": views_of(comments, cust % len(comments)), "rev": pa.array(rng.integers(0, 10**6, rows).astype(np.int64))})
        spec = {"op": "aggregate", "mode": "single", "group_by": [{"expr": {"col": i}, "name": t.schema.names[i]} for i in range(7)],
                "aggs": [{"fn": "sum", "args": [{"col": 7}], "name": "revenue", "input_type": "Int64"}]}
        return spec, [[t]]

    def few_long():
        rows = n(10e6)
        head = "h" * 1000
        vocab = sorted(head + f"{i:04d}" + chr(97 + i % 26) * 1044 for i in range(100))
        t = pa.table({"s": views_of(vocab, rng.integers(0, len(vocab), rows)), "p": pa.array(np.arange(rows, dtype=np.int64))})
        return sort_spec([0]), [[t.slice(o, 500_000) for o in range(0, rows, 500_000)]]      # one batch holds at most 2 GiB of string bytes

    return {"sort_urls": sort_of(urls, n(50e6)), "sort_urls_200": sort_of(urls200, n(50e6)), "topk_phrases": topk, "merge_8_runs": merge,
            "q10_agg": q10, "few_long": few_long}


def digest(t):
    """sha256 over every column's values and validity, in row order"""
    h = hashlib.sha256()
    for c in t.columns:
        a = c.combine_chunks()
        h.update(np.packbits(a.is_valid().to_numpy(zero_copy_only=False)).tobytes())
        if pa.types.is_string_view(a.type) or pa.types.is_binary_view(a.type) or pa.types.is_string(a.type) or pa.types.is_large_string(a.type):
            a = a.cast(pa.large_string())
            h.update(a.buffers()[1]); h.update(a.buffers()[2] or b"")
        else:
            h.update(a.fill_null(0).to_numpy(zero_copy_only=False).tobytes())
    return h.hexdigest()[:16]


def run_once(spec, inputs, devs, ctx, engine):
    op = engine.GpuExec(spec, [d[0].schema for d in devs], ctx)
    try:
        ctx.synchronize()
        t0 = time.perf_counter()
        for k, batches in enumerate(devs):
            for d in batches:
                op.push(d.borrow(), k)
            op.finish(k)
        out = op.collect_device(handle=True)
        ctx.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        return ms, op.metrics(), out
    finally:
        op.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    from sail_b200 import engine
    if a.lib:
        engine.LIB_PATH = os.path.abspath(a.lib)
    import torch
    print(json.dumps({"card": card(), "lib": engine.LIB_PATH, "scale": a.scale}), flush=True)
    ctx = engine.default_context()
    wl = workloads(a.scale, np.random.default_rng(1))
    for name, make in wl.items():
        if a.only and name not in a.only.split(","):
            continue
        spec, inputs = make()
        devs = [[engine.to_device(t, ctx) for t in batches] for batches in inputs]
        rows = sum(t.num_rows for b in inputs for t in b)
        res = {"workload": name, "rows": rows}
        try:
            free0 = torch.cuda.mem_get_info()[0]
            times, syncs = [], []
            for rep in range(4):
                ms, m, out = run_once(spec, inputs, devs, ctx, engine)
                if rep == 0:
                    res["held_mb_after_first_run"] = round((free0 - torch.cuda.mem_get_info()[0]) / 2**20)
                else:
                    times.append(ms)
                    syncs.append(m.get("gpu.host_syncs"))
                if rep < 3:
                    del out
            i = int(np.argmin(times))
            res.update(ms=round(times[i], 2), ms_all=[round(x, 2) for x in times], host_syncs=syncs[i])
            del out
            try:
                op = engine.GpuExec(spec, [d[0].schema for d in devs], ctx)
                for k, batches in enumerate(devs):
                    for d in batches:
                        op.push(d.borrow(), k)
                    op.finish(k)
                try:
                    host = op.collect()
                finally:
                    op.close()
                res["out_rows"] = host.num_rows
                # the aggregate's row order is unspecified: its digest is taken in key order
                if name == "q10_agg":
                    host = pa.table([c.cast(pa.large_string()) if pa.types.is_string_view(c.type) or pa.types.is_binary_view(c.type) else c for c in host.columns],
                                    names=host.schema.names)
                    host = host.sort_by([(c, "ascending") for c in host.schema.names])
                res["digest"] = digest(host)
            except engine.SailGpuError as e:        # the host export of one batch holds at most 2 GiB of string bytes
                res["digest"] = "not taken: " + str(e)[:120]
        except engine.SailGpuError as e:
            res["error"] = str(e)[:200]
        print(json.dumps(res), flush=True)
        del devs


if __name__ == "__main__":
    main()
