"""The specialised kernels of the bench pipelines keep every group key in registers: NVRTC-compiled for sm_90a (no GPU
needed) into a scratch kernel cache, each reports a zero stack frame and has no local loads or stores in its SASS.  Local
traffic there would share the L1 / shared-memory pipe with the reads of the TMA stages on every tile."""
import os
import re
import shutil
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r"""
import os, sys
sys.path.insert(0, sys.argv[1])
from sail_b200 import engine, jit_warm
for name, spec, schema, mask, flags in jit_warm.pipelines():
    before = set(os.listdir(os.environ["SAILGPU_JIT_CACHE"]))
    engine.jit_precompile(spec, [schema], mask, flags | engine.JIT_COMPILE)
    new = sorted(set(os.listdir(os.environ["SAILGPU_JIT_CACHE"])) - before)
    print(name + "\t" + (new[-1] if new else ""))
"""


@pytest.mark.skipif(shutil.which("cuobjdump") is None and not os.path.exists("/usr/local/cuda/bin/cuobjdump"), reason="cuobjdump not installed")
def test_bench_kernels_use_no_local_memory():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    with tempfile.TemporaryDirectory(prefix="sailgpu_jit_") as cache:
        env = dict(os.environ, SAILGPU_JIT_CACHE=cache)
        out = subprocess.run([sys.executable, "-c", SCRIPT, ROOT], env=env, capture_output=True, text=True, check=True).stdout
        kernels = [line.split("\t") for line in out.strip().splitlines()]
        assert any(name.startswith("q1") for name, _ in kernels)
        for name, f in kernels:
            assert f, f"{name}: no kernel compiled"
            path = os.path.join(cache, f)
            res = subprocess.run([cuobjdump, "--dump-resource-usage", path], capture_output=True, text=True, check=True).stdout
            m = re.search(r"REG:(\d+) STACK:(\d+)", res)
            assert m and int(m.group(2)) == 0, f"{name}: {res}"
            sass = subprocess.run([cuobjdump, "-sass", path], capture_output=True, text=True, check=True).stdout
            assert not re.search(r"\b(STL|LDL)\b", sass), f"{name}: local loads or stores in the SASS"
