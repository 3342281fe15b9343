"""NVRTC-compiles the specialised kernel of every Filter / Projection / Aggregate node of the ClickBench (and, with --tpch, the
TPC-H) plans for sm_90a -- no GPU needed -- into a SCRATCH cache (never the shipped one: a cached cubin is used from the first
batch on, and only the bench pipelines' kernels are parity-checked at that size), and prints one line per kernel with its
resource usage.  What `sailgpu_jit_precompile(.., SAILGPU_JIT_COMPILE)` would do for a rewrite pass at plan time.

    python scripts/jit_compile_all.py [--tpch]
"""
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SCRATCH = tempfile.mkdtemp(prefix="sailgpu_jit_")
os.environ["SAILGPU_JIT_CACHE"] = SCRATCH          # before the library is loaded: the cache directory is read once

from sail_b200 import clickbench as cb, engine, plans   # noqa: E402
from tests.util import oracle_op                        # noqa: E402


def usage(before):
    new = sorted(set(os.listdir(SCRATCH)) - before)
    if not new:
        return "(cached)"
    f = os.path.join(SCRATCH, new[-1])
    res = subprocess.run(["cuobjdump", "--dump-resource-usage", f], capture_output=True, text=True).stdout
    m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+)", res)
    sass = subprocess.run(["cuobjdump", "-sass", f], capture_output=True, text=True).stdout
    return f"{os.path.getsize(f)} B  " + (f"REG:{m.group(1)} STACK:{m.group(2)} SHARED:{m.group(3)}" if m else "?") + f"  UBLKCP={sass.count('UBLKCP')} SYNCS={sass.count('SYNCS')}"


def main():
    from datagen import hits, tpch
    work = [(n, (q.plan() if q.parts == 1 else q.plan(part=0)), "hits") for n, q in cb.QUERIES.items()]
    tables = {"hits": hits.hits(2000, seed=3)}
    if "--tpch" in sys.argv:
        tables.update(tpch.tables(0.001))
        work += [(q, plans.TPCH[q](), None) for q in sorted(plans.TPCH, key=lambda s: int(s[1:]))]
    seen, ok, refused, t0 = set(), 0, 0, time.time()

    def walk(node, qname):
        nonlocal ok, refused
        if node.spec["op"] == "scan":
            return tables[node.spec["table"]].select(node.spec["columns"])
        ins = [walk(c, qname) for c in node.inputs]
        out = oracle_op(node.spec, *ins)
        key = json.dumps(node.spec, sort_keys=True) + str(ins[0].schema)
        if node.spec["op"] in ("filter", "projection", "aggregate", "pipeline") and key not in seen:
            seen.add(key)
            for variant, flags in (("dictionary", 0), ("global table", engine.JIT_COLD_VARIANT)):
                if variant != "dictionary" and node.spec["op"] != "aggregate":
                    continue
                before = set(os.listdir(SCRATCH))
                try:
                    engine.jit_precompile(node.spec, [ins[0].schema], 0, flags | engine.JIT_COMPILE)
                    ok += 1
                    print(f"{qname:5s} {node.spec['op']:10s} {variant:12s} {usage(before)}", flush=True)
                except engine.SailGpuError as e:
                    refused += 1
                    print(f"{qname:5s} {node.spec['op']:10s} {variant:12s} interpreted: {e}", flush=True)
        return out
    for name, plan, _ in work:
        walk(plan, name)
    print(f"# {ok} kernels compiled for sm_90a, {refused} pipelines stay interpreted, {time.time() - t0:.0f} s on the CPU (NVRTC)")


if __name__ == "__main__":
    main()
