"""GPU parity of voice patches through the C ABI against the plain-C oracle and the golden fixture made by the compiled reference,
both ways a patch runs: the kernel generated and compiled for its stage list (K8f, maximilian_b200/csrc/patch_fuse.cu) and the
interpreting kernel (K8, patch.cu). The two must also agree with each other BIT FOR BIT on every patch (same stage bodies, same
libdevice routines, same arguments: hoisting a coefficient design out of the sample loop does not change its result).

Bars: patches whose stages are table look-ups and + - * / only are BIT-IDENTICAL; a patch with a stage that designs
coefficients or calls pow / atan / tan / cos on every sample (libdevice where the reference calls glibc) is asserted at
1e-9 relative + 1e-12 (north_star: 1e-5). Integer state (envelope flags, hold counts, delay ring indices, maxiEnvGen segment
and counters) is exact in both. The stereo bus sums voices in another (fixed) order: 1e-9 relative."""
import numpy as np
import pytest

import golden_checks as G
import patch_cases as PC
from patch_checks import INT_SLOTS, cmp as _cmp, set_tables as _tables
from maximilian_b200 import capi
from maximilian_b200 import workloads as W
from maximilian_b200.patchdef import STATE_SLOTS as SLOTS

pytestmark = pytest.mark.gpu

MODES = ["fused", "interpret"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("V,B", [(333, 257), (4100, 64)])
@pytest.mark.parametrize("case", PC.cases(), ids=lambda c: c[0])
def test_patch_vs_oracle(port, case, V, B, mode):
    name, d, params, inputs, exact, taps = case
    _tables(port)
    g = capi.Patch(d, V, max_frames=B, delay_taps=taps, mode=mode); o = port.Patch(d, V, delay_taps=taps, kind="port")
    assert g.mode == mode
    for k, v in params(V, 21).items():
        g.set(k, v); o.set(k, v)
    for blk in range(3):
        ins = inputs(V, B, blk, 9)
        og, mg = g.process(B, ins, want_mix=True); oo, mo = o.process(B, ins, want_mix=True)
        _cmp(og, oo, exact, f"{name} blk{blk}")
        np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-10)
    for si, (op, kind, dst, src) in enumerate(d.stages):
        for sl in range(SLOTS.get(op, 0)):
            if op == 4 and sl == 3:
                continue
            _cmp(g.get_state(si, sl), o.get_state(si, sl), exact or sl in INT_SLOTS.get(op, ()), f"{name} stage {si} slot {sl}")
        if op in (10, 11):
            for v in range(0, V, 37):
                _cmp(g.ring(si, v, taps), o.ring(si, v, taps), exact, f"{name} ring {si}/{v}")


@pytest.mark.parametrize("case", PC.cases(), ids=lambda c: c[0])
def test_fused_equals_interpreted_bit_for_bit(port, case):
    """the generated kernel against the interpreter: outputs, bus, every state word and the rings, three blocks, switching the
    SAME patch object between the modes in the last block (identical state layout)"""
    name, d, params, inputs, exact, taps = case
    _tables(port)
    V, B = 1500, 200
    a = capi.Patch(d, V, max_frames=B, delay_taps=taps, mode="fused"); b = capi.Patch(d, V, max_frames=B, delay_taps=taps, mode="interpret")
    for k, v in params(V, 5).items():
        a.set(k, v); b.set(k, v)
    for blk in range(3):
        if blk == 2:
            a.set_mode("interpret"); b.set_mode("fused")
        ins = inputs(V, B, blk, 4)
        oa, ma = a.process(B, ins, want_mix=True); ob, mb = b.process(B, ins, want_mix=True)
        assert np.array_equal(oa, ob, equal_nan=True), f"{name} blk{blk}: fused and interpreted outputs differ"
        assert np.array_equal(ma, mb, equal_nan=True), f"{name} blk{blk}: fused and interpreted buses differ"
    for si, (op, kind, dst, src) in enumerate(d.stages):
        for sl in range(SLOTS.get(op, 0)):
            assert np.array_equal(a.get_state(si, sl), b.get_state(si, sl), equal_nan=True), f"{name} stage {si} slot {sl}"
        if op in (10, 11):
            for v in range(0, V, 101):
                assert np.array_equal(a.ring(si, v, taps), b.ring(si, v, taps), equal_nan=True)


def test_fused_hoists_block_constant_designs(port):
    """a patch whose filter / oscillator arguments are parameters and constants only (designs emitted before the sample loop)
    against the oracle, which designs on every sample like the reference"""
    from maximilian_b200.patchdef import PatchDef, R
    d = PatchDef()
    d.stage("osc", d.P("f"), kind="saw", dst=R(0))
    d.stage("filter", R(0), d.P("cut"), d.K(3.0), kind="lores", dst=R(1))
    d.stage("svf", R(1), d.P("cut"), d.K(2.0), d.K(1.0), d.K(0.25), d.K(0.0), d.K(0.5), dst=R(2))
    d.stage("biquad", R(2), d.P("cut"), d.K(0.9), d.K(3.0), kind="peak", dst=R(3))
    d.stage("filter", R(3), d.P("cut"), d.K(0.4), kind="bandpass", dst=R(4))
    d.stage("out", R(4)); d.stage("mix_stereo", R(4), d.K(0.3))
    src = capi.patch_codegen(d)
    head = src[:src.index("for (int t = 0")]
    for fn in ("filt_design<FILT_T_LORES>", "filt_design<FILT_T_SVF>", "design_biquad_one", "design_bandpass", "const double inc0"):
        assert fn in head, f"{fn} was not hoisted out of the sample loop"
    V, B = 777, 300
    rng = np.random.default_rng(3)
    prm = dict(f=rng.uniform(30, 2000, V), cut=rng.uniform(100, 8000, V))
    g = capi.Patch(d, V, max_frames=B, mode="fused"); o = port.Patch(d, V, kind="port")
    for k, v in prm.items():
        g.set(k, v); o.set(k, v)
    for blk in range(2):
        og, mg = g.process(B, want_mix=True); oo, mo = o.process(B, want_mix=True)
        _cmp(og, oo, False, f"hoisted blk{blk}")
        np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-10)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", PC.cases(), ids=lambda c: c[0])
def test_patch_golden(port, case, mode):
    name, d, params, inputs, exact, taps = case
    _tables(port)
    gl = G.load("patches")
    V, B, NB = int(gl["V"]), int(gl["B"]), int(gl["NB"])
    p = capi.Patch(d, V, max_frames=B, delay_taps=taps, mode=mode)
    for k, v in params(V, 2468).items():
        p.set(k, v)
    for blk in range(NB):
        ins = {k: gl[f"{name}/in/{k}/{blk}"] for k in d.inputs}
        o, m = p.process(B, ins, want_mix=True)
        _cmp(o, gl[name + "/out"][blk], exact, f"{name} blk{blk}")
        np.testing.assert_allclose(m, gl[name + "/mix"][blk], rtol=1e-9, atol=1e-12)


def test_full_size_polysynth_256k_voices_vs_oracle_slices(port):
    """The bench's patch leg at its own size (262 144 voices x 1024 frames, trigger bytes, the generated kernel), two blocks: a
    1536-voice slice -- first, middle and last warps -- against the oracle run on those voices (outputs 1e-9, envelope flags / hold
    counts exact), the bus against the pan-weighted sum of the GPU's own output, and the interpreter on the slice bit for bit."""
    V, B = 262144, 1024
    _tables(port)
    d = W.polysynth_patch("u8")
    prm = W.polysynth_params(V, seed=31); pat = W.note_pattern(V, seed=31)
    sl = np.concatenate([np.arange(0, 512), np.arange(V // 2 - 256, V // 2 + 256), np.arange(V - 512, V)])
    g = capi.Patch(d, V, max_frames=B, mode="fused")
    o = port.Patch(d, sl.size, kind="port"); gi = capi.Patch(d, sl.size, max_frames=B, mode="interpret")
    for k, v in prm.items():
        g.set(k, v); o.set(k, v[sl]); gi.set(k, v[sl])
    pan = np.clip(prm["pan"], 0.0, 1.0)
    for blk in range(2):
        tr = W.note_triggers(pat, B, blk)
        og, mg = g.process(B, {"trigger": tr}, want_mix=True)
        oo, _ = o.process(B, {"trigger": tr[:, sl].astype(np.float64)})
        oi, _ = gi.process(B, {"trigger": np.ascontiguousarray(tr[:, sl])})
        np.testing.assert_allclose(og[:, sl], oo, rtol=1e-9, atol=1e-12)
        assert np.array_equal(og[:, sl], oi)
        bus = np.stack([og @ np.sqrt(1.0 - pan), og @ np.sqrt(pan)], axis=1)
        np.testing.assert_allclose(mg, bus, rtol=1e-9, atol=1e-9)
    for slot in (2, 3):                                        # holdcount, flags of the ADSR (stage 0)
        assert np.array_equal(g.get_state(0, slot)[sl], o.get_state(0, slot))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("V", [96, 1000, 4099])
def test_trigger_streams_as_bytes_and_as_packed_bits(mode, V):
    """the three element types of an input stream (doubles, bytes, one bit per voice-sample) give the same bits out; voice counts that
    are not multiples of 32 end in a partly used word"""
    B = 160
    prm = W.polysynth_params(V, seed=9); pat = W.note_pattern(V, seed=9)
    ps = {ty: capi.Patch(W.polysynth_patch(ty), V, max_frames=B, mode=mode) for ty in ("f64", "u8", "bits")}
    for p in ps.values():
        for k, v in prm.items():
            p.set(k, v)
    for blk in range(2):
        tr = W.note_triggers(pat, B, blk)
        ref = None
        for ty, p in ps.items():
            o, m = p.process(B, {"trigger": tr.astype(np.float64) if ty == "f64" else tr}, want_mix=True)
            if ref is None:
                ref = (o, m)
            else:
                assert np.array_equal(o, ref[0]) and np.array_equal(m, ref[1]), (ty, blk)


@pytest.mark.parametrize("mode", MODES)
def test_host_staging_grows_with_the_block(port, mode):
    """Host-memory blocks of 16, 300, 40 and 512 frames through one patch that reads a byte stream (trigger) and a double stream
    (frequency) and writes out and the bus: the staging buffers of both inputs and of out grow between blocks. Bit-identical to
    the oracle (saw, ADSR, * only), the bus within 1e-9."""
    from maximilian_b200.patchdef import PatchDef, R
    d = PatchDef()
    d.stage("env_adsr", d.K(1.0), d.IN("trigger", "u8"), d.P("attack"), d.P("decay"), d.P("sustain"), d.P("release"), d.K(1.0), dst=R(0))
    d.stage("osc", d.IN("freq"), kind="saw", dst=R(1))
    d.stage("mul", R(1), R(0), dst=R(2))
    d.stage("out", R(2)); d.stage("mix_stereo", R(2), d.P("pan"))
    V = 333
    prm = W.polysynth_params(V, seed=12); pat = W.note_pattern(V, seed=12)
    g = capi.Patch(d, V, max_frames=512, mode=mode); o = port.Patch(d, V, kind="port")
    for k in ("attack", "decay", "sustain", "release", "pan"):
        g.set(k, prm[k]); o.set(k, prm[k])
    rng = np.random.default_rng(12)
    for blk, B in enumerate((16, 300, 40, 512)):
        ins = {"trigger": W.note_triggers(pat, B, blk), "freq": rng.uniform(30.0, 3000.0, (B, V))}
        og, mg = g.process(B, ins, want_mix=True); oo, mo = o.process(B, ins, want_mix=True)
        _cmp(og, oo, True, f"blk{blk} ({B} frames)")
        np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-10, err_msg=f"blk{blk} ({B} frames)")
    for sl in range(SLOTS[2]):
        _cmp(g.get_state(0, sl), o.get_state(0, sl), True, f"ADSR slot {sl}")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("modulated", [False, True])
def test_chorus_vs_oracle(port, mode, modulated):
    """maxiChorus as a stage (the noise it draws is an input stream): outputs 1e-9 (cos / sqrt of the per-sample or hoisted lores design
    are libdevice's), both delay-line indices exact, both rings and the lores state 1e-9; three blocks, odd voice count."""
    name, d, params, _, exact, taps = PC.chorus(modulated)
    V, B, NB = 333, 180, 3
    noise = port.noise_fill(31, NB * B * V, "port").reshape(NB, B, V)
    g = capi.Patch(d, V, max_frames=B, delay_taps=taps, mode=mode); o = port.Patch(d, V, delay_taps=taps, kind="port")
    if not modulated and mode == "fused":
        src = capi.patch_codegen(d)
        assert "filt_design<FILT_T_LORES>" in src[:src.index("for (int t = 0")]           # constant speed: designed once per block
    for k, v in params(V, 6).items():
        g.set(k, v); o.set(k, v)
    for blk in range(NB):
        og, mg = g.process(B, {"noise": noise[blk]}, want_mix=True); oo, mo = o.process(B, {"noise": noise[blk]}, want_mix=True)
        _cmp(og, oo, False, f"{name} blk{blk}")
        np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-10)
    si = [i for i, st in enumerate(d.stages) if st[0] == 18][0]
    for sl in range(4):
        _cmp(g.get_state(si, sl), o.get_state(si, sl), sl < 2, f"{name} slot {sl}")
    for v in range(0, V, 41):
        _cmp(g.ring(si, v, 2 * taps), o.ring(si, v, 2 * taps), False, f"{name} rings of voice {v}")


def test_chorus_golden_and_modes_agree(port):
    """tests/golden/chorus.npz (the compiled reference drawing its own rand()) replayed on the GPU both ways; fused == interpreted bit for bit"""
    gl = G.load("chorus")
    name, d, params, _, exact, taps = PC.chorus()
    V, B, NB = int(gl["V"]), int(gl["B"]), int(gl["NB"])
    ps = {m: capi.Patch(d, V, max_frames=B, delay_taps=taps, mode=m) for m in MODES}
    for p in ps.values():
        for k, v in params(V, 99).items():
            p.set(k, v)
    for blk in range(NB):
        res = {m: p.process(B, {"noise": gl["noise"][blk]}, want_mix=True) for m, p in ps.items()}
        _cmp(res["fused"][0], gl["out"][blk], False, f"chorus golden blk{blk}")
        np.testing.assert_allclose(res["fused"][1], gl["mix"][blk], rtol=1e-9, atol=1e-12)
        assert np.array_equal(res["fused"][0], res["interpret"][0]) and np.array_equal(res["fused"][1], res["interpret"][1])


def test_patch_rejects_bad_programs():
    from maximilian_b200.patchdef import PatchDef, R
    d = PatchDef(); d.stage("osc", d.K(100.0), kind="sinebuf", dst=R(0)); d.stage("out", R(0))
    ctx = capi.Context(0, 44100)                                    # a context that was never given the tables
    with pytest.raises(capi.MxbError):
        capi.Patch(d, 8, ctx=ctx, sample_rate=44100)
    d = PatchDef(); d.stage("delay", d.K(1.0), d.K(4.0), d.K(0.5), kind="dl", dst=R(0)); d.stage("out", R(0))
    with pytest.raises(capi.MxbError):
        capi.Patch(d, 8, delay_taps=0)
    d = PatchDef(); d.stages.append((99, 0, -1, [-1] * 8))
    with pytest.raises(capi.MxbError):
        capi.Patch(d, 8)
