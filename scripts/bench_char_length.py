"""character_length on the GPU: a projection over resident URL-like Utf8View values, interpreted and specialised, against the same
projection without the function and the card's streaming read, and ClickBench [27] over resident hits rows with parity against
its SQL in pandas.

    python scripts/bench_char_length.py [rows=200000000] [hits_rows=10000000]

Prints one JSON object per measurement.  The strings are 8 to 159 bytes (84 on average; the 3 % of at most 12 bytes are inline
views) of mostly ASCII text with 2-, 3- and 4-byte characters, cut at character boundaries.  20 M distinct strings (1.7 GB of heap,
far more than L2) repeat in row order up to `rows`, so every row reads its bytes from HBM.  Bytes moved per row: the 16-byte view,
the heap bytes of a string longer than 12 bytes, and the 4-byte Int32 result.  The projection without the function is
`CASE WHEN s = '' THEN 0 ELSE 1 END`: the same view read and Int32 write, no heap bytes.  Times are the operator's (push of a
resident batch in the library's own form, the pipeline kernel, the hand-off of the device result) by CUDA events on the library's
stream, best of five after a warm-up."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.bench_timestamp import _scans, card, stream_read  # noqa: E402

DISTINCT = 20_000_000


def text_block(rng, size=1 << 20):
    """valid UTF-8: 80 % ASCII, the rest 2-, 3- and 4-byte characters"""
    chars = [c.encode() for c in "abcdefghijklmnopqrstuvwxyz0123456789/.-_?=&"] * 8 + [c.encode() for c in "жпрвёщ€→🦀𝄞"]
    out = bytearray()
    while len(out) < size:
        out += b"".join(chars[i] for i in rng.integers(0, len(chars), 4096))
    return np.frombuffer(bytes(out), dtype=np.uint8)


def url_views(n, seed=1):
    """-> (pyarrow Utf8View array of n rows, heap bytes one pass over the rows reads, character count of every distinct string)"""
    import pyarrow as pa
    rng = np.random.default_rng(seed)
    block = text_block(rng)
    b = len(block)
    starts_in_block = np.flatnonzero((block & 0xC0) != 0x80)
    next_start = starts_in_block[np.minimum(np.searchsorted(starts_in_block, np.arange(b + 1)), len(starts_in_block) - 1)]
    next_start[np.arange(b + 1) > starts_in_block[-1]] = b             # past the last start: the next block's first byte
    d = min(DISTINCT, n)
    ends = np.cumsum(rng.integers(8, 160, d).astype(np.int64))
    ends = ends // b * b + next_start[ends % b]                        # snap every boundary to a character start
    starts = np.concatenate([[0], ends[:-1]])
    lens = (ends - starts).astype(np.int64)
    heap = np.tile(block, int(ends[-1] // b) + 1)[: int(ends[-1])]
    assert len(heap) < 2 ** 31 and lens.min() > 0
    v = np.zeros((d, 16), dtype=np.uint8)
    v[:, :4] = lens.astype("<u4").view(np.uint8).reshape(-1, 4)
    k = np.arange(12)
    inline = lens <= 12
    data = heap[np.minimum(starts[:, None] + k, len(heap) - 1)] * (k < lens[:, None])
    v[:, 4:16] = np.where(inline[:, None], data, 0)
    v[~inline, 4:8] = data[~inline, :4]
    v[~inline, 12:16] = starts[~inline].astype("<u4").view(np.uint8).reshape(-1, 4)      # buffer 0, offset
    chars = np.add.reduceat((heap & 0xC0) != 0x80, starts, dtype=np.int32)
    reps = -(-n // d)
    views = np.tile(v, (reps, 1))[:n]
    arr = pa.Array.from_buffers(pa.string_view(), n, [None, pa.py_buffer(views), pa.py_buffer(heap)])
    long_lens = np.where(inline, 0, lens)
    long_bytes = int(long_lens.sum()) * (n // d) + int(long_lens[: n % d].sum())
    return arr, long_bytes, chars


def projection(n):
    import pyarrow as pa
    import torch
    from sail_b200 import engine
    ctx = engine.default_context()
    stream = torch.cuda.ExternalStream(ctx.stream())
    arr, long_bytes, chars = url_views(n)
    schema = pa.schema([pa.field("s", pa.string_view(), nullable=False)])
    table = pa.table([arr], schema=schema)

    def resident():
        """the batch in HBM in the library's own form, as one operator hands it to the next (uploaded through an identity
        projection, not timed: a batch whose rows repeat heap bytes cannot be exported as one Arrow batch under 2 GiB of heap)"""
        up = engine.GpuExec({"op": "projection", "exprs": [{"expr": {"col": 0}, "name": "s"}]}, [schema], ctx)
        up.push(table)
        up.finish()
        h = up.collect_device(handle=True)
        up.close()
        assert len(h) == 1
        return h[0]
    s = {"col": 0}
    spec = {"op": "projection", "exprs": [{"expr": {"fn": "character_length", "args": [s]}, "name": "n"}]}
    plain = {"op": "projection", "exprs": [{"expr": {"case": [[{"op": "=", "l": s, "r": {"lit": "", "type": "Utf8View"}}, {"lit": 0, "type": "Int32"}]],
                                                     "else": {"lit": 1, "type": "Int32"}}, "name": "n"}]}
    out, parity = {}, None
    for kernel in ("interpreted", "specialised"):
        for label, sp in ((kernel, spec), (kernel + "_same_width_without_character_length", plain)):
            if kernel == "interpreted":
                os.environ["SAILGPU_JIT"] = "0"
            else:
                os.environ.pop("SAILGPU_JIT", None)
                os.environ["SAILGPU_JIT_MIN_ROWS"] = "0"
            best, jit = 1e30, 0
            for rep in range(6):
                h = resident()
                op = engine.GpuExec(sp, [schema], ctx)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ctx.synchronize()
                a.record(stream)
                op.push(h)
                op.finish()
                res = op.collect_device(handle=True)
                b.record(stream)
                b.synchronize()
                jit = op.metrics().get("gpu.jit_launches", 0)
                op.close()
                if rep == 5 and sp is spec:                # the result of the last run against the counts of the host
                    from tests.test_gpu_parquet_clickbench import host
                    got = host(res, res[0].schema).column("n").to_numpy()
                    want = np.resize(chars, n)
                    ok = bool(np.array_equal(got, want))
                    parity = ok if parity is None else parity and ok
                del res
                if rep:                                    # the first run warms up (and, specialised, compiles the kernel)
                    best = min(best, a.elapsed_time(b))
            moved = n * (16 + 4) + (long_bytes if sp is spec else 0)
            out[label] = {"ms": round(best, 3), "GB_moved": round(moved / 1e9, 2), "GBps": round(moved / best / 1e6, 1), "jit_launches": jit}
    out["parity"] = "ok" if parity else "MISMATCH"
    return out


def clickbench(n):
    from datagen import hits as gen
    from sail_b200 import clickbench as cb, engine, plans
    from tests import char_length_ref as ref, clickbench_sql as sql
    from tests.test_clickbench import as_table
    from tests.test_gpu_parquet_clickbench import host
    from tests.util import assert_topk
    table = gen.hits(n, seed=7)
    frame = sql.frame(table)
    q = cb.LENGTH_QUERIES["c27"]
    min_count = ref.q27_min_count(frame)
    node = cb.top_sort(q.plan(min_count=min_count))
    cols = sorted({c for s in _scans(node) for c in s})
    tables = {"hits": (engine.to_device(table.select(cols)), cols)}
    times = []
    for _ in range(4):
        engine.default_context().synchronize()
        t0 = time.perf_counter()
        out = plans.execute_gpu(node, tables)
        engine.default_context().synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    got = host(out, out[0].schema)
    try:
        assert_topk(got, as_table(ref.q27(frame, min_count), got.schema), list(q.order), node.spec["fetch"], float_cols=q.floats)
        parity = "ok" if got.num_rows else "empty"
    except AssertionError as e:
        parity = f"MISMATCH: {str(e)[:200]}"
    return {"c27": {"rows": n, "min_count": min_count, "groups": got.num_rows, "ms_best": round(min(times[1:]), 2), "parity": parity}}


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 200_000_000
    hits_rows = int(sys.argv[2]) if len(sys.argv) > 2 else 10_000_000
    print(json.dumps({"card": card()}), flush=True)
    sr = stream_read()
    proj = projection(n)
    for v in proj.values():
        if isinstance(v, dict):
            v["of_stream_read"] = round(v["GBps"] / sr, 3)
    print(json.dumps({"projection_rows": n, "stream_read_GBps": sr, **proj}), flush=True)
    print(json.dumps({"clickbench": clickbench(hits_rows)}), flush=True)


if __name__ == "__main__":
    main()
