"""The variance family on the CPU: plan-time names, types and nullability of stddev, stddev_pop, var and var_pop in every
aggregate mode and over every argument type, the refusals, the exact reference of tests/variance_ref.py against Python's
statistics module, and the specialised kernel generated and compiled for an aggregate with stddev without local memory."""
import decimal
import math
import os
import re
import shutil
import statistics
import subprocess
import tempfile

import pyarrow as pa
import pytest

from sail_b200 import engine
from tests import variance_ref as ref

UNSUPPORTED, INVALID = 2, 1
FNS = ["stddev", "stddev_pop", "var", "var_pop"]
ARG_TYPES = [pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.uint8(), pa.uint32(), pa.uint64(), pa.decimal128(15, 2),
             pa.decimal128(38, 4), pa.float32(), pa.float64()]


def agg(aggs, keys=(0,), mode="single"):
    return {"op": "aggregate", "mode": mode, "group_by": [{"expr": {"col": k}, "name": f"k{k}"} for k in keys], "aggs": aggs}


def a(fn, arg=1, name="r", **kw):
    return {"fn": fn, "name": name, "args": [] if arg is None else [{"col": arg}], **kw}


def schema(x_type, nullable=True):
    return [pa.schema([pa.field("k", pa.int32()), pa.field("x", x_type, nullable=nullable)])]


def state_schema(t=pa.uint64()):
    return [pa.schema([pa.field("k", pa.int32()), pa.field("c", t, False), pa.field("m", pa.float64()), pa.field("q", pa.float64())])]


@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("t", ARG_TYPES, ids=str)
@pytest.mark.parametrize("nullable", [False, True])
def test_single_is_nullable_float64(fn, t, nullable):
    out = engine.validate(agg([a(fn)]), schema(t, nullable))
    assert out.field("r").type == pa.float64() and out.field("r").nullable


@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("t", ARG_TYPES, ids=str)
def test_partial_states_are_datafusions(fn, t):
    out = engine.validate(agg([a(fn)], mode="partial"), schema(t))
    assert out.names == ["k0", "r[count]", "r[mean]", "r[m2]"]
    assert [f.type for f in out][1:] == [pa.uint64(), pa.float64(), pa.float64()]


@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("mode", ["final", "final_partitioned"])
@pytest.mark.parametrize("count_type", [pa.uint64(), pa.int64()])
def test_final_reads_three_state_columns(fn, mode, count_type):
    out = engine.validate(agg([{"fn": fn, "name": "r", "input_type": "Int64"}], mode=mode), state_schema(count_type))
    assert out.names == ["k0", "r"] and out.field("r").type == pa.float64() and out.field("r").nullable


@pytest.mark.parametrize("mode", ["single", "partial"])
def test_next_to_count_avg_min_max(mode):
    aggs = [a("count", name="c"), a("avg", name="m"), a("stddev", name="s"), a("var_pop", name="v"), a("min", name="lo"), a("max", name="hi")]
    out = engine.validate(agg(aggs, mode=mode), schema(pa.float64()))
    if mode == "single":
        assert out.names == ["k0", "c", "m", "s", "v", "lo", "hi"]
    else:
        assert out.names == ["k0", "c[count]", "m[count]", "m[sum]", "s[count]", "s[mean]", "s[m2]", "v[count]", "v[mean]", "v[m2]", "lo[min]", "hi[max]"]


def refused(spec, s):
    with pytest.raises(engine.SailGpuError) as e:
        engine.validate(spec, s)
    return e.value


@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("t", [pa.string(), pa.string_view(), pa.bool_(), pa.date32()], ids=str)
def test_non_numeric_arguments_are_invalid(fn, t):
    assert refused(agg([a(fn)]), schema(t)).code == INVALID


@pytest.mark.parametrize("fn", FNS)
def test_timestamp_argument_is_unsupported(fn):
    assert refused(agg([a(fn)]), schema(pa.timestamp("us", tz="UTC"))).code == UNSUPPORTED


@pytest.mark.parametrize("fn", ["stddev_samp", "variance", "var_samp", "std", "covar_pop", "corr"])
def test_aliases_and_other_statistics_are_unsupported(fn):
    assert refused(agg([a(fn)]), schema(pa.float64())).code == UNSUPPORTED


@pytest.mark.parametrize("fn", FNS)
def test_distinct_is_unsupported(fn):
    assert refused(agg([a(fn, distinct=True)]), schema(pa.float64())).code == UNSUPPORTED


def test_final_with_wrong_state_types_is_invalid():
    s = [pa.schema([pa.field("k", pa.int32()), pa.field("c", pa.uint64()), pa.field("m", pa.float64()), pa.field("q", pa.int64())])]
    assert refused(agg([{"fn": "stddev", "name": "r", "input_type": "Int64"}], mode="final"), s).code == INVALID
    assert refused(agg([{"fn": "stddev", "name": "r", "input_type": "Int64"}], mode="final"), [s[0].remove(3)]).code == INVALID


def test_no_argument_is_invalid():
    assert refused(agg([a("var", arg=None)]), schema(pa.float64())).code == INVALID


# ---- the reference ----------------------------------------------------------------------------------------

SAMPLES = [[1.0, 2.0, 4.0, 7.0], [0.1] * 9, [3.5, -2.25], [1e8 + 0.5, 1e8 - 1.25, 1e8 + 3.0, 1e8], [2.0 ** -30, 5.0, -7.5, 11.0, 0.3]]


@pytest.mark.parametrize("xs", SAMPLES)
def test_reference_against_statistics(xs):
    t = pa.table({"k": pa.array([0] * len(xs), pa.int32()), "x": pa.array(xs, pa.float64())})
    spec = agg([a("var", name="v"), a("var_pop", name="vp"), a("stddev", name="s"), a("stddev_pop", name="sp")])
    got = ref.ref_op(spec, t).to_pylist()[0]
    for name, want in [("v", statistics.variance(xs)), ("vp", statistics.pvariance(xs)), ("s", statistics.stdev(xs)), ("sp", statistics.pstdev(xs))]:
        assert got[name] == pytest.approx(want, rel=1e-15, abs=0.0), name


def test_reference_small_groups_and_partial_states():
    t = pa.table({"k": pa.array([0, 1, 1, 2, 2, 2, 3], pa.int32()), "x": pa.array([5.0, 1.0, 3.0, None, None, None, math.inf])})
    got = {r["k0"]: r for r in ref.ref_op(agg([a("var", name="v"), a("var_pop", name="vp")]), t).to_pylist()}
    assert got[0]["v"] is None and got[0]["vp"] == 0.0
    assert got[1]["v"] == 2.0 and got[1]["vp"] == 1.0
    assert got[2]["v"] is None and got[2]["vp"] is None
    assert math.isnan(got[3]["vp"]) and got[3]["v"] is None
    part = {r["k0"]: r for r in ref.ref_op(agg([a("stddev", name="s")], mode="partial"), t).to_pylist()}
    assert (part[1]["s[count]"], part[1]["s[mean]"], part[1]["s[m2]"]) == (2, 2.0, 2.0)
    assert (part[2]["s[count]"], part[2]["s[mean]"], part[2]["s[m2]"]) == (0, 0.0, 0.0)


def test_reference_merge_of_states_is_the_whole():
    xs = [1.5, 2.5, 10.0, -4.0, 7.25, 3.0]
    whole = ref.moments(xs)
    parts = [ref.moments(xs[:2]), ref.moments(xs[2:5]), ref.moments(xs[5:])]
    merged = ref.merge_states([(n, float(m), float(q)) for n, m, q in parts])
    assert merged[0] == whole[0] and float(merged[2]) == pytest.approx(float(whole[2]), rel=1e-15)


def test_reference_converts_decimals_like_the_engine():
    assert ref.as_float(decimal.Decimal("12.34"), pa.decimal128(15, 2)) == 1234.0 / 100.0
    assert ref.as_float(2**64 - 1, pa.uint64()) == 2.0 ** 64


# ---- the specialised kernel -------------------------------------------------------------------------------

def describe_spec():
    return agg([a("count", name="c"), a("avg", name="m"), a("stddev", name="s"), a("var_pop", name="v"), a("min", name="lo"), a("max", name="hi")])


@pytest.mark.parametrize("mode", ["single", "partial", "final"])
def test_specialiser_generates_variance_pipelines(mode):
    if mode == "final":
        spec, s = agg([{"fn": "stddev", "name": "s", "input_type": "Float64"}], mode="final"), state_schema()
    else:
        spec, s = ({**describe_spec(), "mode": mode}), schema(pa.float64())
    n, src = engine.jit_precompile(spec, s, 0, 0)
    assert n > 0 and "dd_term(" in src


SCRIPT = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import pyarrow as pa
from sail_b200 import engine
spec = json.loads(sys.argv[2])
s = [pa.schema([pa.field("k", pa.int32()), pa.field("x", pa.float64())])]
for flags in (engine.JIT_COMPILE, engine.JIT_COMPILE | engine.JIT_COLD_VARIANT):
    engine.jit_precompile(spec, s, 0, flags)
"""


@pytest.mark.skipif(shutil.which("cuobjdump") is None and not os.path.exists("/usr/local/cuda/bin/cuobjdump"), reason="cuobjdump not installed")
def test_specialised_variance_kernels_use_no_local_memory():
    """the dictionary and the many-groups variants of a describe()-shaped aggregate, compiled by NVRTC for sm_90a"""
    import json
    import sys
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with tempfile.TemporaryDirectory(prefix="sailgpu_jit_") as cache:
        env = dict(os.environ, SAILGPU_JIT_CACHE=cache)
        subprocess.run([sys.executable, "-c", SCRIPT, root, json.dumps(describe_spec())], env=env, check=True)
        files = os.listdir(cache)
        assert len(files) == 2, files
        for f in files:
            path = os.path.join(cache, f)
            res = subprocess.run([cuobjdump, "--dump-resource-usage", path], capture_output=True, text=True, check=True).stdout
            m = re.search(r"REG:(\d+) STACK:(\d+)", res)
            assert m and int(m.group(2)) == 0, res
            sass = subprocess.run([cuobjdump, "-sass", path], capture_output=True, text=True, check=True).stdout
            assert not re.search(r"\b(STL|LDL)\b", sass), "local loads or stores in the SASS"
