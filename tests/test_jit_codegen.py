"""The kernel specialiser's code generator on the CPU: for every Filter / Projection / Aggregate node of the 22 TPC-H and the 37
ClickBench plans `sailgpu_jit_precompile` (no device, no NVRTC: source only, nothing is written to the kernel cache) either
emits the CUDA source of the specialised kernel or says why the pipeline stays interpreted (SAILGPU_ERR_UNSUPPORTED).
NVRTC-compiling all of them for sm_90a takes a minute and is what `__graft_entry__.build()` does for the bench pipelines;
`scripts/jit_compile_all.py` does it for every ClickBench pipeline into a scratch cache."""
import json

import pytest

from sail_b200 import clickbench as cb, engine, plans
from tests.util import oracle_op

PIPELINE_OPS = ("filter", "projection", "aggregate", "pipeline")


def generate(plan, tables):
    """-> [(op, variant, outcome)] over the plan's pipeline nodes; outcome = source length or the refusal"""
    out, seen = [], set()

    def walk(node):
        if node.spec["op"] == "scan":
            return tables[node.spec["table"]].select(node.spec["columns"])
        ins = [walk(c) for c in node.inputs]
        res = oracle_op(node.spec, *ins)
        key = json.dumps(node.spec, sort_keys=True) + str(ins[0].schema)
        if node.spec["op"] in PIPELINE_OPS and key not in seen:
            seen.add(key)
            for variant, flags in (("dictionary", 0), ("global table", engine.JIT_COLD_VARIANT)):
                if variant == "global table" and node.spec["op"] != "aggregate":
                    continue
                try:
                    n, src = engine.jit_precompile(node.spec, [ins[0].schema], 0, flags)
                    assert n == len(src) > 1000 and "struct G" in src
                    out.append((node.spec["op"], variant, n))
                except engine.SailGpuError as e:
                    assert e.code == 2, (node.spec, e)          # "not covered" is the only legal refusal
                    out.append((node.spec["op"], variant, str(e)))
        return res
    walk(plan)
    return out


@pytest.fixture(scope="module")
def hits_small():
    from datagen import hits
    return {"hits": hits.hits(2000, seed=3)}


@pytest.mark.parametrize("name", list(cb.QUERIES))
def test_clickbench_pipelines_generate(name, hits_small):
    q = cb.QUERIES[name]
    res = generate(q.plan() if q.parts == 1 else q.plan(part=0), hits_small)
    assert res
    refused = [r for r in res if isinstance(r[2], str)]
    assert all("reads no column" in r[2] for r in refused), refused     # count(*) over nothing: nothing to stage, stays interpreted


@pytest.mark.parametrize("q", sorted(plans.TPCH, key=lambda s: int(s[1:])))
def test_tpch_pipelines_generate(q, tpch_tiny):
    res = generate(plans.TPCH[q](), tpch_tiny)
    assert any(isinstance(r[2], int) for r in res)
