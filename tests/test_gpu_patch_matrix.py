"""The voice-patch matrix (tests/patch_matrix.py) and random stage lists on the GPU, both ways a patch runs -- the kernel generated for
its stage list (K8f, patch_fuse.cu) and the interpreting kernel (K8, patch.cu) -- against the plain-C oracle, at the voice counts,
block lengths and descriptor limits where the kernels change shape, and through the API paths the other patch tests do not take.

Bars (as in test_gpu_patch.py): exact cases bit for bit; a case with a libm stage 1e-9 relative + 1e-12; integral state slots exact
in both; the bus 1e-9 (another fixed summation order). Fused and interpreted: bit for bit, outputs, bus, every state slot, the rings."""
import ctypes as C

import numpy as np
import pytest

import patch_matrix as PM
from patch_checks import BAD_KINDS, INT_SLOTS, bad_kind_patch, cmp as _cmp, ring_stages as _ring_stages, set_tables
from maximilian_b200 import capi
from maximilian_b200.patchdef import PatchDef, R, OP, BIQUAD, ENVGEN_HOLD, STATE_SLOTS as SLOTS

pytestmark = pytest.mark.gpu

MODES = ["fused", "interpret"]


@pytest.fixture(autouse=True)
def _tables(port):
    set_tables(port)


def _state(p, d, taps, voices):
    """every state slot and the rings of `voices`"""
    s = {(si, sl): p.get_state(si, sl) for si, (op, *_) in enumerate(d.stages) for sl in range(SLOTS.get(op, 0))}
    for si, n in _ring_stages(d):
        for v in voices:
            s[(si, "ring", v)] = p.ring(si, v, n * taps)
    return s


def _same_state(a, b, what):
    for k in a:
        assert np.array_equal(a[k], b[k], equal_nan=True), f"{what}: {k}"


def _vs_port(g, o, d, taps, voices, exact, what):
    for si, (op, kind, dst, src) in enumerate(d.stages):
        for sl in range(SLOTS.get(op, 0)):
            if op == OP["envgen"] and sl == 3:
                continue
            _cmp(g.get_state(si, sl), o.get_state(si, sl), exact or sl in INT_SLOTS.get(op, ()), f"{what} stage {si} slot {sl}")
    for si, n in _ring_stages(d):
        for v in voices:
            _cmp(g.ring(si, v, n * taps), o.ring(si, v, n * taps), exact, f"{what} ring {si}/{v}")


@pytest.mark.parametrize("case", PM.cases(), ids=lambda c: c[0])
def test_matrix_both_modes_vs_port(port, case):
    """each case in both modes against the port (exact cases bit for bit), and fused against interpreted bit for bit"""
    name, d, params, inputs, exact, taps = case
    V, B, NB = 333, 257, 3
    gs = {m: capi.Patch(d, V, max_frames=B, delay_taps=taps, mode=m) for m in MODES}
    o = port.Patch(d, V, delay_taps=taps, kind="port")
    for k, v in params(V, 21).items():
        o.set(k, v)
        for g in gs.values():
            g.set(k, v)
    for blk in range(NB):
        ins = inputs(V, B, blk, 9)
        oo, mo = o.process(B, ins, want_mix=True)
        res = {m: g.process(B, ins, want_mix=True) for m, g in gs.items()}
        for m, (og, mg) in res.items():
            _cmp(og, oo, exact, f"{name} {m} blk{blk}")
            np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-10, err_msg=f"{name} {m} bus blk{blk}")
        assert np.array_equal(res["fused"][0], res["interpret"][0], equal_nan=True), f"{name} blk{blk}: fused and interpreted outputs differ"
        assert np.array_equal(res["fused"][1], res["interpret"][1], equal_nan=True), f"{name} blk{blk}: fused and interpreted buses differ"
    voices = range(0, V, 37)
    for m, g in gs.items():
        _vs_port(g, o, d, taps, voices, exact, f"{name} {m}")
    _same_state(_state(gs["fused"], d, taps, voices), _state(gs["interpret"], d, taps, voices), f"{name} fused vs interpreted")


def test_holdtime_beyond_32_bits_holds_like_the_reference(port):
    """maxiEnv's holdtime and holdcount are `long`: 2^32 + 3 holds for 2^32 + 3 samples (not 3), 2^31 - 1 and 0 / 1 as given"""
    d = PatchDef()
    d.stage("env_adsr", d.K(1.0), d.IN("gate", "u8"), d.K(0.5), d.K(0.9), d.K(0.5), d.K(0.9), d.P("ht"), dst=R(0))
    d.stage("env_ar", d.K(1.0), d.IN("gate", "u8"), d.K(0.5), d.K(0.9), d.P("ht"), dst=R(1))
    d.stage("add", R(0), R(1), dst=R(2)); d.stage("out", R(2))
    V, B = 4, 64
    ht = np.array(PM.HOLDTIMES)
    gate = np.zeros((B, V), dtype=np.uint8); gate[:8] = 1                      # open for 8 samples, then closed
    o = port.Patch(d, V, kind="port"); o.set("ht", ht)
    oo, _ = o.process(B, {"gate": gate})
    assert np.array_equal(oo[:, 2], oo[:, 3]) and not np.array_equal(oo[:, 1], oo[:, 3])     # 2^31 - 1 and 2^32 + 3 both still hold
    for m in MODES:
        g = capi.Patch(d, V, max_frames=B, mode=m); g.set("ht", ht)
        og, _ = g.process(B, {"gate": gate})
        assert np.array_equal(og, oo), m
        for si in (0, 1):
            assert np.array_equal(g.get_state(si, 2), o.get_state(si, 2)), (m, si)


# ---------------------------------------------------------------------------------------------------------------------- shapes
def _shape_patches():
    """an exact patch (saw, ADSR on a packed-bit trigger, delay line, mix) and a libm one (sine, lores swept per sample, ADSR on bits)"""
    c = PM.Case("shape_exact", True, 64)
    d = c.d
    d.stage("osc", c.ctrl("P", "f", 40.0, 3000.0, PM.FREQ_CORNERS), kind="saw", dst=R(0))
    d.stage("env_adsr", R(0), c.trig("I", "gate", "bits"), d.K(0.3), d.K(0.95), d.K(0.5), c.ctrl("P", "rel", 0.9, 0.999), c.ctrl("P", "ht", 0.0, 9.0, integral=True), dst=R(1))
    d.stage("delay", R(1), c.ctrl("P", "size", 1.0, 64.0, (1.0, 64.0), integral=True), d.K(0.7), kind="dl", dst=R(2))
    c.nreg = 3
    exact = c.finish([R(1), R(2)])
    c = PM.Case("shape_libm", False)
    d = c.d
    d.stage("osc", c.ctrl("P", "f", 40.0, 3000.0), kind="sinewave", dst=R(0))
    c.nreg = 1
    cut = c.ctrl("R", "cut", 100.0, 8000.0)
    d.stage("filter", R(0), cut, d.K(2.0), kind="lores", dst=R(5))
    d.stage("env_ar", R(5), c.trig("I", "gate", "bits"), d.K(0.2), c.ctrl("P", "rel", 0.9, 0.999), d.K(3.0), dst=R(6))
    c.nreg = 7
    return [exact, c.finish([R(6)])]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("which", [0, 1], ids=["exact", "libm"])
@pytest.mark.parametrize("V", [1, 31, 32, 33, 127, 128, 129, 4097])
def test_shapes_vs_port(port, V, which, mode):
    """blocks of 1 frame and of max_frames, and a 0-frame call that leaves every state slot and the rings as they were"""
    name, d, params, inputs, exact, taps = _shape_patches()[which]
    MF = 300
    g = capi.Patch(d, V, max_frames=MF, delay_taps=taps, mode=mode); o = port.Patch(d, V, delay_taps=taps, kind="port")
    for k, v in params(V, 4).items():
        g.set(k, v); o.set(k, v)
    voices = sorted({0, V // 2, V - 1})
    for blk, B in enumerate((1, MF, 0, 1, MF)):
        ins = inputs(V, B, blk, 5)
        if B == 0:
            before = _state(g, d, taps, voices)
            og, mg = g.process(0, ins, want_mix=True)
            assert og.shape == (0, V) and mg.shape == (0, 2)
            _same_state(_state(g, d, taps, voices), before, f"{name} V={V}: a 0-frame call changed the state")
            continue
        og, mg = g.process(B, ins, want_mix=True); oo, mo = o.process(B, ins, want_mix=True)
        _cmp(og, oo, exact, f"{name} V={V} blk{blk} ({B} frames)")
        np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-10)
    _vs_port(g, o, d, taps, voices, exact, f"{name} V={V}")


# ---------------------------------------------------------------------------------------------------------------------- limits
def _full_descriptor():
    """64 stages over all 16 registers, 32 parameters, 64 constants and 8 input streams (f64, u8 and bits), exact stages only"""
    c = PM.Case("limits", True)
    d = c.d
    types = ["f64", "u8", "bits", "f64", "u8", "bits", "f64", "f64"]
    ins = []
    for k, ty in enumerate(types):
        if ty == "f64":
            c.ispec[f"in{k}"] = ("uniform", 0.0, 1.0, (0.0, 1.0), False)
        else:
            c.ispec[f"in{k}"] = ("gate", ty)
        ins.append(d.IN(f"in{k}", ty))
    prm = [c.ctrl("P", f"p{j}", 0.1, 0.9, (0.1, 0.9)) for j in range(32)]
    ks = [d.K(0.01 * (j + 1)) for j in range(64)]
    kj = iter(ks)
    pj = iter(prm)
    for k in range(16):                                   # 16 oscillators and envelopes, one per register
        if k % 2 == 0:
            d.stage("osc", next(pj), kind=["phasor", "saw", "triangle", "square"][k // 2 % 4], dst=R(k))
        else:
            d.stage("env_ar", R(k - 1), ins[k // 2], next(pj), next(pj), next(kj), dst=R(k))
    for k in range(16, 62):                               # 46 arithmetic / filter stages mixing every operand class
        a, b = R(k % 16), R((k * 7 + 3) % 16)
        op = ["add", "sub", "mul", "filter"][k % 4]
        if op == "filter":
            d.stage("filter", a, next(pj, ks[k]), kind="lopass", dst=R((k * 5) % 16))
        else:
            d.stage(op, a, ins[k % 8] if k % 3 == 0 else next(kj, b), dst=R((k * 5) % 16))
    for j in range(len(d.consts), 64):
        d.K(1000.0 + j)
    rest = [x for x in kj]
    d.stage("add", R(3), rest[0] if rest else d.K(3.0), dst=R(0))
    d.stage("out", R(0))
    assert len(d.stages) == 64 and len(d.params) == 32 and len(d.consts) == 64 and len(d.inputs) == 8
    return (c.name, d, c.params, c.inputs, True, 0)


@pytest.mark.parametrize("mode", MODES)
def test_descriptor_limits_vs_port(port, mode):
    name, d, params, inputs, exact, taps = _full_descriptor()
    V, B = 500, 200
    g = capi.Patch(d, V, max_frames=B, mode=mode); o = port.Patch(d, V, kind="port")
    for k, v in params(V, 8).items():
        g.set(k, v); o.set(k, v)
    for blk in range(2):
        ins = inputs(V, B, blk, 8)
        og, _ = g.process(B, ins); oo, _ = o.process(B, ins)
        _cmp(og, oo, True, f"limits {mode} blk{blk}")
    _vs_port(g, o, d, 0, (), True, f"limits {mode}")


def _smem_patch(extra):
    """16 registers + n_params + n_state = 200 + extra doubles per voice: 31 (+ extra) parameters, 153 state words"""
    d = PatchDef()
    d.stage("osc", d.P("p0"), kind="saw", dst=R(0))                                    # 2 state words
    for k in range(37):                                                                # 37 x 4
        d.stage("env_adsr", R(k % 2), d.IN("gate", "u8"), d.P(f"p{1 + k % 30}"), d.K(0.95), d.K(0.5), d.P("p30"), d.K(3.0), dst=R((k + 1) % 2))
    d.stage("filter", R(1), d.K(0.3), kind="lopass", dst=R(2))                          # 2
    d.stage("delay", R(2), d.K(16.0), d.K(0.5), kind="dl", dst=R(3))                    # 1
    for j in range(extra):
        d.stage("add", R(3), d.P(f"x{j}"), dst=R(3))
    d.stage("out", R(3))
    return d


@pytest.mark.parametrize("mode", MODES)
def test_interpreter_shared_memory_budget(port, mode):
    """exactly 200 doubles of registers, parameters and state per voice run (the interpreter holds them in 200 KiB of shared memory, the
    generated kernel in registers and spills) and match the port; one more is refused at create with MXB_ERR_UNSUPPORTED"""
    d = _smem_patch(0)
    assert 16 + len(d.params) + 2 + 37 * 4 + 2 + 1 == 200
    V, B = 300, 128
    g = capi.Patch(d, V, max_frames=B, delay_taps=16, mode=mode); o = port.Patch(d, V, delay_taps=16, kind="port")
    rng = np.random.default_rng(3)
    for k in d.params:
        x = rng.uniform(40.0, 900.0, V) if k == "p0" else rng.uniform(0.01, 0.99, V)
        g.set(k, x); o.set(k, x)
    for blk in range(2):
        gate = (rng.random((B, V)) < 0.3).astype(np.uint8)
        og, _ = g.process(B, {"gate": gate}); oo, _ = o.process(B, {"gate": gate})
        _cmp(og, oo, True, f"200 doubles {mode} blk{blk}")
    _vs_port(g, o, d, 16, range(0, V, 29), True, f"200 doubles {mode}")
    with pytest.raises(capi.MxbError, match=r"-> -4:"):
        capi.Patch(_smem_patch(1), V, max_frames=B, delay_taps=16, mode=mode)


# ---------------------------------------------------------------------------------------------------------------------- random programs
EXACT_STAGES = [("osc", k) for k in ("phasor", "saw", "square", "pulse", "impulse", "triangle", "phasorbetween", "sinebuf", "sinebuf4", "sawn")] + \
    [("env_adsr", 0), ("env_ar", 0), ("filter", "lopass"), ("filter", "hipass"), ("dcblock", 0), ("nonlin", "fastatan"), ("nonlin", "fastatandist"),
     ("nonlin", "hardclip"), ("delay", "dl"), ("delay", "position"), ("flanger", 0), ("add", 0), ("sub", 0), ("mul", 0), ("div", 0), ("out", 0), ("mix_stereo", 0)]
LIBM_STAGES = [("osc", "sinewave"), ("osc", "coswave"), ("filter", "lores"), ("filter", "hires"), ("filter", "bandpass"), ("svf", 0), ("envgen", 0)] + \
    [("biquad", k) for k in BIQUAD] + [("nonlin", k) for k in ("atandist", "softclip", "asymclip")]
RTAPS = 48


def random_program(seed, libm=False):
    """4-20 stages drawn at random. Operands of any class -- registers included, also ones written later in the sample or never -- except
    where the reference converts to an integer or indexes a table (triggers, holdtime, delay size / position, flanger delay, table
    oscillator frequency): those come from parameters, constants and input streams inside the operand domain."""
    rng = np.random.default_rng(seed)
    c = PM.Case(f"random{seed}", not libm, RTAPS)
    d = c.d
    n_in = [0]

    def stream(tag, lo, hi, integral=False):
        if n_in[0] >= 8:
            return c.ctrl("P", tag, lo, hi, integral=integral)
        n_in[0] += 1
        ty = rng.choice(["f64", "u8", "bits"]) if lo >= 0 and hi >= 1 and integral else "f64"
        if ty == "f64":
            return c.ctrl("I", tag, lo, hi, integral=integral)
        c.ispec[tag] = ("gate", ty)
        return d.IN(tag, ty)

    def safe(tag, lo, hi, integral=False):
        cls = rng.choice(["K", "P", "I"])
        if cls == "I":
            return stream(tag, lo, hi, integral)
        v = float(rng.uniform(lo, hi))
        return c.ctrl(cls, tag, lo, hi, const=float(np.floor(v)) if integral else v, integral=integral)

    def free(tag, lo, hi):
        cls = rng.choice(["R", "R", "K", "P", "I"])
        if cls == "R":
            return R(int(rng.integers(0, 16)))
        if cls == "I":
            return stream(tag, lo, hi)
        return c.ctrl(cls, tag, lo, hi, const=float(rng.uniform(lo, hi)))

    def trig(tag):
        cls = rng.choice(["K", "P", "I"])
        if cls == "I" and n_in[0] < 8:
            n_in[0] += 1
            return c.trig("I", tag, str(rng.choice(["f64", "u8", "bits"])))
        return c.trig("K" if cls == "K" else "P", tag)

    pool = EXACT_STAGES + (LIBM_STAGES if libm else [])
    if libm:
        d.envgen([0.0, 1.0, 0.3, 0.0], [1.0, ENVGEN_HOLD, 2.0], [1.5, 1.0, 0.7], loop=bool(rng.integers(0, 2)), retrigger=True)
    n = int(rng.integers(4, 21))
    for i in range(n):
        op, kind = pool[int(rng.integers(0, len(pool)))]
        t = f"s{i}_"
        dst = R(int(rng.integers(0, 16))) if op not in ("out", "mix_stereo") or rng.random() < 0.3 else -1
        if op == "osc":
            if kind in PM.TABLE_OSC:
                src = [safe(t + "f", 0.5 if kind == "sawn" else 0.0, 20000.0)]
            else:
                src = [free(t + "f", -100.0, 5000.0), free(t + "a", -0.2, 1.2), free(t + "b", 0.0, 1.3)]
        elif op in ("env_adsr", "env_ar"):
            rates = [free(t + "att", 0.01, 0.5), free(t + "rel", 0.9, 0.999)]
            if op == "env_adsr":
                rates = [rates[0], free(t + "dec", 0.9, 0.99), free(t + "sus", 0.1, 0.9), rates[1]]
            src = [free(t + "x", -1.0, 1.0), trig(t + "tr")] + rates + [safe(t + "ht", 0.0, 12.0, integral=True)]
        elif op == "filter":
            src = [free(t + "x", -1.0, 1.0), free(t + "c", 0.0, 1.0) if kind in ("lopass", "hipass") else free(t + "c", 10.0, 20000.0),
                   free(t + "r", 0.0, 4.0)]
        elif op == "svf":
            src = [free(t + "x", -1.0, 1.0), free(t + "c", 10.0, 20000.0), free(t + "r", 0.0, 4.0)] + [free(t + f"m{k}", -1.0, 1.0) for k in range(4)]
        elif op == "biquad":
            src = [free(t + "x", -1.0, 1.0), free(t + "c", 10.0, 20000.0), free(t + "q", 0.3, 8.0), free(t + "g", -20.0, 20.0)]
        elif op == "dcblock":
            src = [free(t + "x", -1.0, 1.0), free(t + "R", 0.9, 0.999)]
        elif op == "nonlin":
            src = [free(t + "x", -2.0, 2.0), free(t + "a", 0.5, 6.0), free(t + "b", 0.5, 3.0)]
        elif op == "delay":
            src = [free(t + "x", -1.0, 1.0), safe(t + "size", 1.0, RTAPS, integral=True), free(t + "fb", 0.0, 1.2)]
            if kind == "position":
                src.append(safe(t + "pos", 0.0, RTAPS + 10.0, integral=True))
        elif op == "flanger":
            src = [free(t + "x", -1.0, 1.0), safe(t + "dl", 1.0, 20.0, integral=True), free(t + "fb", 0.0, 1.0), safe(t + "sp", 0.0, 100.0),
                   safe(t + "dp", 0.0, 1.0)]
        elif op == "envgen":
            src = [free(t + "tr", -1.0, 1.0)]
        elif op == "mix_stereo":
            src = [free(t + "x", -1.0, 1.0), free(t + "pan", -0.5, 1.5)]
        elif op == "out":
            src = [free(t + "x", -1.0, 1.0)]
        else:
            src = [free(t + "a", -2.0, 2.0), free(t + "b", -2.0, 2.0)]
        d.stage(op, *src, kind=kind, dst=dst)
    d.stage("out", R(int(rng.integers(0, 16))))
    d.stage("mix_stereo", R(int(rng.integers(0, 16))), c.ctrl("P", "pan", 0.0, 1.0, PM.PANS))
    return (c.name, d, c.params, c.inputs, c.exact, c.taps)


@pytest.mark.parametrize("seed", range(40))
def test_random_exact_programs_both_modes_vs_port(port, seed):
    """bit for bit against the port in both modes: outputs, every state slot, the rings; the two buses bit for bit to each other"""
    name, d, params, inputs, exact, taps = random_program(1000 + seed)
    rng = np.random.default_rng(seed)
    V = int(rng.choice([1, 7, 32, 33, 100, 129, 640, 1500]))
    MF = 300
    gs = {m: capi.Patch(d, V, max_frames=MF, delay_taps=taps, mode=m) for m in MODES}
    o = port.Patch(d, V, delay_taps=taps, kind="port")
    for k, v in params(V, seed).items():
        o.set(k, v)
        for g in gs.values():
            g.set(k, v)
    for blk in range(3):
        B = int(rng.integers(1, MF + 1))
        ins = inputs(V, B, blk, seed)
        oo, _ = o.process(B, ins)
        res = {m: g.process(B, ins, want_mix=True) for m, g in gs.items()}
        for m, (og, _) in res.items():
            _cmp(og, oo, True, f"{name} {m} blk{blk} V={V} B={B}")
        assert np.array_equal(res["fused"][1], res["interpret"][1], equal_nan=True), f"{name} blk{blk}: buses differ"
    voices = sorted({0, V // 3, V - 1})
    for m, g in gs.items():
        _vs_port(g, o, d, taps, voices, True, f"{name} {m}")


@pytest.mark.parametrize("seed", range(20))
def test_random_libm_programs_fused_equals_interpreted(seed):
    name, d, params, inputs, exact, taps = random_program(5000 + seed, libm=True)
    rng = np.random.default_rng(seed)
    V = int(rng.choice([1, 33, 129, 700, 2049]))
    MF = 256
    gs = {m: capi.Patch(d, V, max_frames=MF, delay_taps=taps, mode=m) for m in MODES}
    for k, v in params(V, seed).items():
        for g in gs.values():
            g.set(k, v)
    for blk in range(3):
        B = int(rng.integers(1, MF + 1))
        ins = inputs(V, B, blk, seed)
        (oa, ma), (ob, mb) = [g.process(B, ins, want_mix=True) for g in gs.values()]
        assert np.array_equal(oa, ob, equal_nan=True) and np.array_equal(ma, mb, equal_nan=True), f"{name} blk{blk} V={V} B={B}"
    voices = sorted({0, V // 2, V - 1})
    _same_state(_state(gs["fused"], d, taps, voices), _state(gs["interpret"], d, taps, voices), name)


# ---------------------------------------------------------------------------------------------------------------------- API paths
def _api_patch():
    """a patch with a ring-free state, every input element type, out and the bus"""
    c = PM.Case("api", True)
    d = c.d
    d.stage("osc", c.ctrl("I", "f", 40.0, 3000.0), kind="saw", dst=R(0))
    d.stage("env_adsr", R(0), c.trig("I", "gate", "u8"), c.ctrl("P", "att", 0.01, 0.5), d.K(0.95), d.K(0.5), c.ctrl("P", "rel", 0.9, 0.999),
            d.K(5.0), dst=R(1))
    d.stage("env_ar", R(1), c.trig("I", "tr", "bits"), d.K(0.3), d.K(0.99), d.K(2.0), dst=R(2))
    d.stage("filter", R(2), c.ctrl("P", "c", 0.05, 0.9), kind="lopass", dst=R(3))
    c.nreg = 4
    return c.finish([R(3)])


def _device_inputs(torch, d, ins):
    ts = []
    for n in d.inputs:
        ty = d.input_types.get(n)
        a = capi.pack_bits(ins[n]).view(np.int32) if ty == "bits" else np.ascontiguousarray(ins[n], dtype=np.uint8 if ty == "u8" else np.float64)
        ts.append(torch.from_numpy(a).cuda())
    return ts


@pytest.mark.parametrize("mode", MODES)
def test_process_device_on_a_stream_equals_host(mode):
    torch = pytest.importorskip("torch")
    name, d, params, inputs, exact, taps = _api_patch()
    V, B = 777, 200
    a = capi.Patch(d, V, max_frames=B, mode=mode); b = capi.Patch(d, V, max_frames=B, mode=mode)
    for k, v in params(V, 2).items():
        a.set(k, v); b.set(k, v)
    s = torch.cuda.Stream()                                   # PyTorch's streams do not synchronise with the legacy default stream
    for blk in range(3):
        ins = inputs(V, B, blk, 2)
        oh, mh = a.process(B, ins, want_mix=True)
        dev = _device_inputs(torch, d, ins)
        out = torch.full((B, V), float("nan"), dtype=torch.float64, device="cuda"); mix = torch.full((B, 2), float("nan"), dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        b.process_device(B, [t.data_ptr() for t in dev], out.data_ptr(), mix.data_ptr(), stream=s.cuda_stream)
        s.synchronize()
        assert np.array_equal(out.cpu().numpy(), oh) and np.array_equal(mix.cpu().numpy(), mh), blk


@pytest.mark.parametrize("mode", MODES)
def test_mix_only_call_equals_the_bus_of_out_and_mix(mode):
    name, d, params, inputs, exact, taps = _api_patch()
    V, B = 1029, 160
    a = capi.Patch(d, V, max_frames=B, mode=mode); b = capi.Patch(d, V, max_frames=B, mode=mode)
    for k, v in params(V, 3).items():
        a.set(k, v); b.set(k, v)
    for blk in range(3):
        ins = inputs(V, B, blk, 3)
        _, ma = a.process(B, ins, want_mix=True)
        ob, mb = b.process(B, ins, want_out=False, want_mix=True)
        assert ob is None and np.array_equal(ma, mb), blk


@pytest.mark.parametrize("mode", MODES)
def test_parameters_from_device_memory(mode):
    torch = pytest.importorskip("torch")
    name, d, params, inputs, exact, taps = _api_patch()
    V, B = 300, 128
    a = capi.Patch(d, V, max_frames=B, mode=mode); b = capi.Patch(d, V, max_frames=B, mode=mode)
    keep = []
    for k, v in params(V, 4).items():
        a.set(k, v)
        t = torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).cuda(); keep.append(t)
        torch.cuda.synchronize()
        capi.check(capi.lib().mxb_patch_set_param(b.h, d.params.index(k), C.c_void_p(t.data_ptr()), capi.MEM_DEVICE), "mxb_patch_set_param")
    for blk in range(2):
        ins = inputs(V, B, blk, 4)
        oa, ma = a.process(B, ins, want_mix=True); ob, mb = b.process(B, ins, want_mix=True)
        assert np.array_equal(oa, ob) and np.array_equal(ma, mb), blk


@pytest.mark.parametrize("mode", MODES)
def test_set_state_resumes_a_patch_mid_stream(mode):
    """every state slot of a ring-free patch copied into a fresh patch after one block: its next blocks equal the uninterrupted patch's"""
    name, d, params, inputs, exact, taps = PM.env_case("env_ar")
    assert not _ring_stages(d)
    V, B = 555, 150
    a = capi.Patch(d, V, max_frames=B, mode=mode); b = capi.Patch(d, V, max_frames=B, mode=mode)
    prm = params(V, 5)
    for k, v in prm.items():
        a.set(k, v); b.set(k, v)
    a.process(B, inputs(V, B, 0, 5)); b.process(B, inputs(V, B, 0, 5))
    c = capi.Patch(d, V, max_frames=B, mode=mode)
    for k, v in prm.items():
        c.set(k, v)
    for si, (op, *_) in enumerate(d.stages):
        for sl in range(SLOTS.get(op, 0)):
            c.set_state(si, sl, b.get_state(si, sl))
    del b
    for blk in (1, 2):
        ins = inputs(V, B, blk, 5)
        oa, ma = a.process(B, ins, want_mix=True); oc, mc = c.process(B, ins, want_mix=True)
        assert np.array_equal(oa, oc) and np.array_equal(ma, mc), blk
    _same_state(_state(a, d, 0, ()), _state(c, d, 0, ()), "resumed")


def test_state_slots_table_is_the_librarys():
    """patchdef.STATE_SLOTS against mxb_patch_get_state: a stage has exactly that many state words, every op of the matrix"""
    seen = set()
    for name, d, params, inputs, exact, taps in PM.cases():
        p = capi.Patch(d, 40, max_frames=8, delay_taps=taps, mode="interpret")
        for si, (op, *_) in enumerate(d.stages):
            n = SLOTS.get(op, 0)
            with pytest.raises(capi.MxbError):
                p.get_state(si, n)
            if n:
                assert p.get_state(si, n - 1).shape == (40,)
            seen.add(op)
    assert seen == set(OP.values())


def test_patch_create_refuses_the_kinds_the_generator_refuses():
    for op, kind in BAD_KINDS:
        with pytest.raises(capi.MxbError):
            capi.Patch(bad_kind_patch(op, kind), 40, max_frames=8, mode="interpret")
