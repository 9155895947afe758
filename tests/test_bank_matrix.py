"""The bank matrix's table (tests/bank_matrix.py) covers every kernel the library holds and every runtime branch it means to reach.
CPU only: the kernels are read from the built library's symbols."""
import os
import shutil
import subprocess

import pytest

import bank_matrix as M
from maximilian_b200 import build, capi


def _table_keys(family):
    return {b.key for g in M.GROUPS if g.family == family for b in g.blocks}


def test_table_keys_are_the_template_domains():
    assert len(M.K1_KEYS) == len(set(M.K1_KEYS)) == 480
    assert len(M.K2_KEYS) == len(set(M.K2_KEYS)) == 240
    assert _table_keys("k1") == set(M.K1_KEYS)
    assert _table_keys("k2") == set(M.K2_KEYS)
    assert len(M.K1_GROUPS) == 48 and len(M.K2_GROUPS) == 24


def test_every_block_runs_another_instantiation_than_the_one_before():
    for g in M.GROUPS:
        keys = [b.key for b in g.blocks]
        assert all(a != b for a, b in zip(keys, keys[1:])), g.name
        assert len({b.n for b in g.blocks}) > 1, g.name
        last = g.blocks[-1]
        assert not (last.fm or last.cm or last.size_tv), f"{g.name}: the last block runs on the block-constant parameters"


def _library_kernels():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    filt = shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
    sources = [capi.LIB_PATH]
    names = subprocess.run([tool, "-symbols", capi.LIB_PATH], capture_output=True, text=True)
    if names.returncode != 0 or "bank_kernel" not in names.stdout:       # the tool does not read the .so: read the objects
        sources = [os.path.join(build.OBJ, f) for f in sorted(os.listdir(build.OBJ)) if f.endswith(".o")]
        names = subprocess.run([tool, "-symbols"] + sources, capture_output=True, text=True, check=True)
    mangled = sorted({w for w in names.stdout.split() if w.startswith("_Z") and "bank_kernel" in w})
    demangled = subprocess.run([filt], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.splitlines()
    return [M.kernel_key(s) for s in demangled]


@pytest.mark.skipif(not os.path.exists(capi.LIB_PATH), reason="the library has not been built (python -m maximilian_b200.build)")
def test_table_keys_are_the_kernels_in_the_library():
    """A new instantiation fails here until the table covers it."""
    keys = _library_kernels()
    assert None not in keys
    assert {k for f, k in keys if f == "k1"} == set(M.K1_KEYS)
    assert {k for f, k in keys if f == "k2"} == set(M.K2_KEYS)
    assert len(keys) == 720


@pytest.mark.parametrize("family", ["k1", "k2"])
def test_every_branch_occurs_in_each_family(family):
    seen = set().union(*(b.tags for g in M.GROUPS if g.family == family for b in g.blocks))
    assert M.required_tags(family) <= seen, sorted(M.required_tags(family) - seen)
    types = {g.desc["biquad_type"] for g in M.GROUPS if g.desc["filt"] == "biquad"}
    assert types == set(M.BIQUADS)


def test_key_of_restates_the_dispatch():
    d = dict(osc="pulse", filt="svf", env="ar", delay=False, svf_mix=(1.0, -0.0, 0.0, 0.0))
    call = dict(out=True, mix=False, f32=True, freq_tv=True, cutoff_tv=True)
    assert M.key_of(d, call) == ("k1", ("svf_lp", "generic", 1, True, False, 3))
    assert M.key_of(dict(d, svf_mix=(1.0, 0.0, 0.0, 0.5)), call)[1][0] == "svf"
    assert M.key_of(dict(d, osc="sinewave"), dict(call, cutoff_tv=False))[1] == ("svf_lp", "sine", 1, True, False, 1)
    k2 = dict(d, delay="position", osc="sinewave")
    assert M.key_of(k2, call) == ("k2", ("svf_lp", "generic", 1, "f32", False, 1))
    assert M.key_of(dict(k2, osc="saw"), dict(call, out=False, freq_tv=False)) == ("k2", ("svf_lp", "saw", 1, "none", True, 1))
    assert M.key_of(dict(k2, env=False), dict(call, f32=False, freq_tv=False, cutoff_tv=False))[1] == \
        ("svf_lp", "generic", 0, "f64", False, 0)
    with pytest.raises(AssertionError):
        M.key_of(dict(d, filt="biquad"), call)
