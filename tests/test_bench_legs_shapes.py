"""The shapes tests/test_gpu_bench_legs.py checks are the shapes bench.py times.

bench.py is read as source (ast), never imported: importing it sets MXB_PATCH_CACHE for the whole process and registers an exit
handler. When a workload in bench.py changes size or chain, this test fails until the GPU module follows it.
"""
import ast
import operator
import os

import test_gpu_bench_legs as L

BENCH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "bench.py")
# the keys that decide which kernels run and at what shape; descriptions and byte counts are bench.py's own business
KEYS = ("voices", "osc", "filt", "env", "delay", "channels", "fft", "hop", "hops_per_step", "filters", "coeffs")
OPS = {ast.LShift: operator.lshift, ast.Mult: operator.mul, ast.Add: operator.add}


def _eval(node):
    """literals combined with <<, * and +"""
    if isinstance(node, ast.Constant):
        return node.value
    if isinstance(node, ast.BinOp) and type(node.op) in OPS:
        return OPS[type(node.op)](_eval(node.left), _eval(node.right))
    raise ValueError(f"bench.py:{node.lineno}: not a literal expression: {ast.unparse(node)}")


def _shape(call):
    """the KEYS of a dict(...) call"""
    assert isinstance(call, ast.Call) and call.func.id == "dict", ast.unparse(call)
    return {kw.arg: _eval(kw.value) for kw in call.keywords if kw.arg in KEYS}


def bench_shapes(path=BENCH):
    """BLOCK, SR, WORKLOADS, MFCC_WL, PATCH_WL and SPEC_WL as bench.py assigns them at module level"""
    tree = ast.parse(open(path).read(), path)
    found = {}
    for node in tree.body:
        if not (isinstance(node, ast.Assign) and len(node.targets) == 1 and isinstance(node.targets[0], ast.Name)):
            continue
        name = node.targets[0].id
        if name in ("BLOCK", "SR"):
            found[name] = _eval(node.value)
        elif name == "WORKLOADS":
            found[name] = {_eval(k): _shape(v) for k, v in zip(node.value.keys, node.value.values)}
        elif name in ("MFCC_WL", "PATCH_WL", "SPEC_WL"):
            found[name] = _shape(node.value)
    missing = {"BLOCK", "SR", "WORKLOADS", "MFCC_WL", "PATCH_WL", "SPEC_WL"} - set(found)
    assert not missing, f"bench.py no longer assigns {sorted(missing)} at module level"
    return found


def test_gpu_module_runs_the_benchmark_shapes():
    b = bench_shapes()
    assert (b["BLOCK"], b["SR"]) == (L.BLOCK, L.SR)
    assert b["WORKLOADS"] == L.BANK_WL
    assert b["MFCC_WL"] == L.MFCC
    assert b["PATCH_WL"] == L.PATCH
    assert b["SPEC_WL"] == L.SPEC


def test_a_moved_shape_is_seen(tmp_path):
    """the reader sees a change of one shape in a copy of bench.py (here: the headline bank at half its voices)"""
    src = open(BENCH).read()
    assert src.count('"svf": dict(voices=1 << 20,') == 1
    moved = tmp_path / "bench.py"
    moved.write_text(src.replace('"svf": dict(voices=1 << 20,', '"svf": dict(voices=1 << 19,'))
    assert bench_shapes(str(moved))["WORKLOADS"]["svf"]["voices"] == 1 << 19 != L.BANK_WL["svf"]["voices"]
