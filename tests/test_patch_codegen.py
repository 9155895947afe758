"""Host-side checks of the patch code generator (maximilian_b200/csrc/patch_fuse.cu): no device needed -- the source is generated
and compiled for sm_90a by NVRTC exactly as a fused patch's first launch does, only the loading step is left out."""
import re

import numpy as np

import pytest

import patch_cases as PC
from maximilian_b200 import capi
from maximilian_b200.patchdef import PatchDef, R
from patch_checks import BAD_KINDS, bad_kind_patch


@pytest.mark.parametrize("case", PC.cases() + [PC.chorus(False), PC.chorus(True)], ids=lambda c: c[0])
def test_generated_kernel_compiles_for_sm90a(case):
    name, d, params, inputs, exact, taps = case
    src = capi.patch_codegen(d, compile=True)
    assert 'extern "C" __global__' in src and "mxb_fused_patch" in src
    # one body per stage, in order
    assert [int(x) for x in re.findall(r"// stage (\d+):", src)] == list(range(len(d.stages)))
    # every constant arrives as a bit-exact literal
    assert len(re.findall(r"__longlong_as_double\(0x[0-9a-f]{16}LL\)", src)) == len(d.consts)


def test_block_constant_arguments_are_designed_once():
    d = PatchDef()
    d.stage("osc", d.P("f"), kind="saw", dst=R(0))
    d.stage("filter", R(0), d.P("cut"), d.K(3.0), kind="lores", dst=R(1))
    d.stage("filter", R(1), R(0), d.K(3.0), kind="hires", dst=R(2))              # cutoff from a register: per sample
    d.stage("out", R(2))
    src = capi.patch_codegen(d, compile=True)
    head, loop = src.split("for (int t = 0", 1)
    assert "filt_design<FILT_T_LORES>(f1, p1, c0, sr);" in head and "const double inc0" in head
    assert "filt_design<FILT_T_LORES>(f2, r0, c0, sr);" in loop


def test_input_element_types_are_part_of_the_program():
    from maximilian_b200 import workloads as W
    srcs = {ty: capi.patch_codegen(W.polysynth_patch(ty), compile=True) for ty in ("f64", "u8", "bits")}
    assert "(const double*)a.inputs[0]" in srcs["f64"] and "(const unsigned char*)a.inputs[0]" in srcs["u8"] and "(const unsigned*)a.inputs[0]" in srcs["bits"]
    assert len({*srcs.values()}) == 3
    x = (np.arange(3 * 70).reshape(3, 70) % 3 == 0)
    w = capi.pack_bits(x)
    assert w.shape == (3, 3) and w.dtype == np.uint32
    for v in range(70):
        assert np.array_equal((w[:, v // 32] >> np.uint32(v % 32)) & 1, x[:, v].astype(np.uint32))


def test_compiled_kernels_are_cached_on_disk(tmp_path, monkeypatch):
    """the second compilation of a program (here: in the same process; in practice: the next process) reads the cubin file"""
    import os
    import time
    monkeypatch.setenv("MXB_PATCH_CACHE", str(tmp_path / "cache" / "nested"))
    d = PatchDef()
    d.stage("osc", d.P("f"), kind="triangle", dst=R(0))
    d.stage("filter", R(0), d.K(1234.5 + (os.getpid() % 97)), d.K(2.0), kind="hires", dst=R(1))     # a program no earlier run compiled
    d.stage("out", R(1))
    t0 = time.perf_counter(); capi.patch_codegen(d, compile=True); t_cold = time.perf_counter() - t0
    files = list((tmp_path / "cache" / "nested").glob("patch_*.cubin"))
    assert len(files) == 1 and files[0].read_bytes()[:4] == b"\x7fELF"
    stamp = files[0].stat().st_mtime_ns
    t0 = time.perf_counter(); capi.patch_codegen(d, compile=True); t_warm = time.perf_counter() - t0
    assert files[0].stat().st_mtime_ns == stamp and t_warm < t_cold
    files[0].write_bytes(b"garbage")                        # a damaged file is ignored and replaced
    capi.patch_codegen(d, compile=True)
    assert files[0].read_bytes()[:4] == b"\x7fELF"
    monkeypatch.setenv("MXB_PATCH_CACHE", "0")
    capi.patch_codegen(d, compile=True)                     # and the cache can be switched off


def test_a_program_the_generator_rejects_is_an_error_not_a_crash():
    d = PatchDef(); d.stages.append((99, 0, -1, [-1] * 8))
    with pytest.raises(capi.MxbError):
        capi.patch_codegen(d)
    d = PatchDef(); d.stage("add", 0x100 + 5, 0x200 + 7, dst=R(0))                 # parameter / constant that do not exist
    with pytest.raises(capi.MxbError):
        capi.patch_codegen(d)


@pytest.mark.parametrize("op,kind", BAD_KINDS)
def test_the_generator_refuses_what_patch_create_refuses(op, kind):
    with pytest.raises(capi.MxbError):
        capi.patch_codegen(bad_kind_patch(op, kind))
    ok = bad_kind_patch(op, 0 if op != "filter" else 1)
    assert "mxb_fused_patch" in capi.patch_codegen(ok)
