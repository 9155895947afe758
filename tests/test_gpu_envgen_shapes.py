"""Voice patches with several maxiEnvGen shapes (mxb_patch_create2) on the GPU: the generated kernel (K8f) and the interpreter (K8)
against the C oracle, against each other, and a one-shape patch through mxb_patch_create2 against the same patch through
mxb_patch_create. Plus the checks mxb_patch_create2 makes of its arguments."""
import ctypes as C

import numpy as np
import pytest

from maximilian_b200 import capi
from maximilian_b200.patchdef import PatchDef, R, ENVGEN_HOLD
import envgen_cases as EC

MODES = ["fused", "interpret"]
BLOCKS = [1, 17, 1024]
INT_SLOTS = [1, 2, 3, 4, 6, 7, 8, 9, 10, 11]      # segment, play state, nxcHappened, counter, the three maxiTrigger detectors


def create2(defn, V, n_shapes=None, shapes=None, max_frames=1024, mode=None, eg_stages=0):
    """A capi.Patch made by mxb_patch_create2 with the PatchDef's shapes (or the given ones); returns (rc, patch or None)."""
    d, keep = capi._patch_desc(defn, V, max_frames, 0)
    d.eg_stages = eg_stages
    arr, keep2 = capi.envgen_shapes(defn.shapes if shapes is None else shapes)
    n = len(defn.shapes) if n_shapes is None else n_shapes
    p = capi.Patch.__new__(capi.Patch)
    p.ctx, p.defn, p.V, p.max_frames, p.h = capi.default_context(), defn, V, max_frames, C.c_void_p()
    rc = capi.lib().mxb_patch_create2(p.ctx.h, C.byref(d), n, arr, C.byref(p.h))
    if rc != 0:
        p.h = None
        return rc, None
    if mode is not None:
        p.set_mode(mode)
    return rc, p


def _blocks(ins):
    t = 0
    for n in BLOCKS:
        yield n, {k: np.ascontiguousarray(a[t:t + n]) for k, a in ins.items()}
        t += n


def _envgen_stages(d):
    return [si for si, st in enumerate(d.stages) if st[0] == 4]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", EC.cases(), ids=lambda c: c[0])
def test_envgen_shapes_match_oracle(port, case, mode):
    name, d, params, inputs = case
    V = 333                                                # a partial last warp
    ins = inputs(V, sum(BLOCKS), 21)
    g = capi.Patch(d, V, max_frames=1024, mode=mode)
    o = port.Patch(d, V, kind="port")
    for k, v in params(V, 4).items():
        g.set(k, v); o.set(k, v)
    for n, x in _blocks(ins):
        og, mg = g.process(n, x, want_mix=True)
        oo, mo = o.process(n, x, want_mix=True)
        np.testing.assert_allclose(og, oo, rtol=1e-9, atol=1e-12, err_msg=f"{name} {mode} out, block of {n}")
        np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-10, err_msg=f"{name} {mode} bus, block of {n}")
        for si in _envgen_stages(d):
            for sl in INT_SLOTS:
                assert np.array_equal(g.get_state(si, sl), o.get_state(si, sl)), (name, mode, n, si, sl)
            for sl in (0, 5):
                np.testing.assert_allclose(g.get_state(si, sl), o.get_state(si, sl), rtol=1e-9, atol=1e-12)
    assert np.abs(og).max() > 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("case", EC.cases(), ids=lambda c: c[0])
def test_fused_equals_interpreted_also_when_switched_mid_stream(case):
    name, d, params, inputs = case
    V = 1000
    ins = inputs(V, 4 * sum(BLOCKS), 8)
    pf = capi.Patch(d, V, mode="fused"); pi = capi.Patch(d, V, mode="interpret"); ps = capi.Patch(d, V, mode="interpret")
    for k, v in params(V, 6).items():
        for p in (pf, pi, ps):
            p.set(k, v)
    t = 0
    for rep in range(4):
        for n in BLOCKS:
            x = {k: np.ascontiguousarray(a[t:t + n]) for k, a in ins.items()}
            t += n
            ps.set_mode(MODES[(rep + n) % 2])             # the switched patch alternates between the two kernels
            of, mf = pf.process(n, x, want_mix=True); oi, mi = pi.process(n, x, want_mix=True); os_, ms = ps.process(n, x, want_mix=True)
            assert np.array_equal(of, oi) and np.array_equal(mf, mi), (name, rep, n)
            assert np.array_equal(of, os_) and np.array_equal(mf, ms), (name, rep, n)
    for si in range(len(d.stages)):
        for sl in range(EC.SLOTS if d.stages[si][0] == 4 else 0):
            a = pf.get_state(si, sl)
            assert np.array_equal(a, pi.get_state(si, sl)) and np.array_equal(a, ps.get_state(si, sl)), (name, si, sl)


def _one_shape():
    d = PatchDef()
    d.envgen([0.0, 1.0, 0.5, 0.5, 0.0], [0.9, 0.6, ENVGEN_HOLD, 1.1], [1.0, 2.0, 1.0, 0.5], retrigger=True)
    d.stage("envgen", d.IN("gate"), dst=R(0))
    d.stage("envgen", d.IN("gate2"), dst=R(1))
    d.stage("osc", d.P("freq"), kind="triangle", dst=R(2))
    d.stage("mul", R(2), R(0), dst=R(3))
    d.stage("add", R(3), R(1), dst=R(3))
    d.stage("out", R(3))
    d.stage("mix_stereo", R(3), d.P("pan"))
    return d


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_one_shape_through_create2_equals_create(mode):
    """mxb_patch_create is mxb_patch_create2 with the descriptor's shape as shape 0: same outputs, bus and state, bit for bit."""
    d = _one_shape()
    V = 500
    _, _, _, inputs = EC.four_shapes()
    ins = inputs(V, sum(BLOCKS), 2)
    a = capi.Patch(d, V, mode=mode)
    rc, b = create2(d, V, mode=mode)
    assert rc == 0
    rng = np.random.default_rng(1)
    for k, v in dict(freq=100.0 + 900.0 * rng.random(V), pan=rng.random(V)).items():
        a.set(k, v); b.set(k, v)
    for n, x in _blocks(ins):
        oa, ma = a.process(n, x, want_mix=True); ob, mb = b.process(n, x, want_mix=True)
        assert np.array_equal(oa, ob) and np.array_equal(ma, mb), n
    for si in (0, 1):
        for sl in range(EC.SLOTS):
            assert np.array_equal(a.get_state(si, sl), b.get_state(si, sl)), (si, sl)
    assert np.abs(oa).max() > 1e-3


@pytest.mark.gpu
def test_create2_rejects_invalid_shapes():
    name, d, _, _ = EC.four_shapes()
    V, INVALID = 64, -1
    good = d.shapes
    assert create2(d, V)[0] == 0
    hold2 = ([0.0, 1.0, 1.0, 0.0], [1.0, ENVGEN_HOLD, ENVGEN_HOLD], [1.0, 1.0, 1.0], False, False)
    assert create2(d, V, shapes=good[:3] + [hold2])[0] == INVALID                      # two HOLD segments
    assert create2(d, V, n_shapes=5, shapes=good + [good[0]])[0] == INVALID             # n_shapes > 4
    assert create2(d, V, n_shapes=-1)[0] == INVALID
    assert create2(d, V, n_shapes=3)[0] == INVALID                                     # a stage plays shape 3
    assert create2(d, V, eg_stages=2)[0] == INVALID                                    # the descriptor's eg_* must be empty
    long_shape = ([0.0] * 18, [1.0] * 17, [1.0] * 17, False, False)
    assert create2(d, V, shapes=good[:3] + [long_shape])[0] == INVALID                  # 17 segments > 16
    # NULL arrays / NULL shape list / negative stages, built by hand
    dd, keep = capi._patch_desc(d, V, 1024, 0)
    dd.eg_stages = 0
    arr, keep2 = capi.envgen_shapes(good)
    ctx = capi.default_context()
    h = C.c_void_p()
    assert capi.lib().mxb_patch_create2(ctx.h, C.byref(dd), 4, None, C.byref(h)) == INVALID
    arr[1].times = C.POINTER(C.c_double)()
    assert capi.lib().mxb_patch_create2(ctx.h, C.byref(dd), 4, arr, C.byref(h)) == INVALID
    arr, keep2 = capi.envgen_shapes(good)
    arr[0].stages = -1
    assert capi.lib().mxb_patch_create2(ctx.h, C.byref(dd), 4, arr, C.byref(h)) == INVALID
    # a stage kind outside the shape list, and mxb_patch_create: an ENVGEN stage plays shape 0
    bad = PatchDef()
    bad.envgen([0.0, 1.0], [1.0], [1.0])
    bad.stage("envgen", bad.K(1.0), kind=-1, dst=R(0))
    bad.stage("out", R(0))
    assert create2(bad, V)[0] == INVALID
    bad.stages[0] = (4, 1, 0, bad.stages[0][3])
    assert create2(bad, V)[0] == INVALID
    with pytest.raises(capi.MxbError, match="shape 1"):
        capi.Patch(bad, V)


def test_generated_kernel_takes_the_shape_index_as_a_literal():
    """The generated source names shape k as a.eg[k]: the segment tables stay kernel arguments, so the program (and its cubin) is the
    same for every set of shapes. Kinds 0..3 are accepted, 4 is not."""
    name, d, _, _ = EC.four_shapes()
    src = capi.patch_codegen(d)
    for k in range(4):
        assert f"a.eg[{k}], a.eg_n[{k}], a.eg_loop[{k}], a.eg_retrigger[{k}]" in src
    other = PatchDef()
    for lv in d.shapes:
        other.envgen([x * 0.5 for x in lv[0]], lv[1], lv[2], lv[3], lv[4])
    other.stages, other.consts, other.params, other.inputs = d.stages, d.consts, d.params, d.inputs
    assert capi.patch_codegen(other) == src
    d.stages[0] = (4, 4, d.stages[0][2], d.stages[0][3])
    with pytest.raises(capi.MxbError):
        capi.patch_codegen(d)
