"""GPU parity of the voice-bank kernels (K1 osc/env/filter, K2 delay line, K3 mix), through the C ABI
(host buffers in, host buffers out) against the plain-C oracle and the committed golden vectors.

Bars (SURVEY.md 8c / north_star):
  * integer state (delay ring index, envelope flags/holdcount): exact
  * fp64 sample values: within 1e-5 relative (north_star). What we actually assert is stronger: chains
    without sin/cos are BIT-IDENTICAL to the reference (no FMA contraction, host-designed coefficients);
    sinewave/coswave differ only by libdevice-vs-glibc sin (<= 2 ulp), asserted at 1e-12 absolute.
  * stereo mix: sum over voices in a different (fixed) order: 1e-9 relative.
"""
import itertools

import numpy as np
import pytest

import golden_checks as G
from maximilian_b200 import capi
from maximilian_b200 import workloads as W

pytestmark = pytest.mark.gpu

OSCS = ["sinewave", "coswave", "phasor", "saw", "square", "pulse", "impulse", "triangle", "phasorbetween"]
FILTS = ["none", "lores", "hires", "svf", "biquad"]
TRIG = {"sinewave", "coswave"}


def gpu_bank(V, **kw):
    return capi.Bank(V, **kw)


def _close(got, ref, trig, what=""):
    if trig:
        assert np.array_equal(np.isnan(got), np.isnan(ref)), what
        np.testing.assert_allclose(got, ref, rtol=1e-9, atol=1e-12, err_msg=what)
    else:
        assert np.array_equal(got, ref, equal_nan=True), f"{what}: not bit-identical, max abs err {np.nanmax(np.abs(got - ref))}"


@pytest.mark.parametrize("case", G.chain_cases(), ids=lambda c: c[0])
def test_golden_chains(case):
    trig = case[1] in TRIG
    G.run_chain_case(gpu_bank, case, exact=not trig, exact_mix=False)


@pytest.mark.parametrize("case", G.mod_cases(), ids=lambda c: c[0])
def test_golden_modulated(case):
    """tests/golden/mods.npz (from the compiled reference): bit-identical unless the cutoff is swept, where the coefficient
    design runs on the device (libdevice cos/sqrt/pow/tan): 1e-9 relative."""
    G.run_mod_case(gpu_bank, case, exact="cutoff" not in case[5])


@pytest.mark.parametrize("osc,filt", list(itertools.product(OSCS, FILTS)))
def test_every_osc_filter_pair_vs_oracle(port, osc, filt):
    V, B = 333, 129
    p = W.voice_params(V, seed=21)
    g = gpu_bank(V, osc=osc, filt=filt, max_frames=B); o = port.Bank(V, osc=osc, filt=filt)
    W.configure_bank(g, filt, p); W.configure_bank(o, filt, p)
    for blk in range(3):
        og, mg = g.process(B, want_mix=True); oo, mo = o.process(B, want_mix=True)
        _close(og, oo, osc in TRIG, f"{osc}->{filt} blk{blk}")
        np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-11)
    for s in ("phase", "filt0", "filt1", "filt2", "osc_output"):      # maxiOsc::output: assigned by every method but impulse
        _close(g.get(s), o.get(s), osc in TRIG, s)


@pytest.mark.parametrize("V", [1, 2, 33, 4096, 4097])
@pytest.mark.parametrize("B", [1, 17, 512, 1024])
def test_shapes_saw_svf(port, V, B):
    p = W.voice_params(V, seed=V + B)
    g = gpu_bank(V, osc="saw", filt="svf", max_frames=B); o = port.Bank(V, osc="saw", filt="svf")
    W.configure_bank(g, "svf", p); W.configure_bank(o, "svf", p)
    for blk in range(2):
        og, _ = g.process(B); oo, _ = o.process(B)
        _close(og, oo, False, f"V{V} B{B} blk{blk}")


def test_config1_plumbing_one_voice_sine_lores(port):
    # BASELINE.json configs[0]: 1 voice sinewave -> lores, 48 kHz, 512-sample blocks
    g = gpu_bank(1, osc="sinewave", filt="lores", max_frames=512); o = port.Bank(1, osc="sinewave", filt="lores")
    for b in (g, o):
        b.set("freq", 440.0); b.set("cutoff", 1000.0); b.set("resonance", 2.0)
    for blk in range(8):
        og, _ = g.process(512); oo, _ = o.process(512)
        np.testing.assert_allclose(og, oo, rtol=1e-9, atol=1e-12)


@pytest.mark.parametrize("btype", ["lowpass", "highpass", "bandpass", "notch", "peak", "lowshelf", "highshelf"])
def test_biquad_types(port, btype):
    V, B = 64, 256
    p = W.voice_params(V, seed=5)
    p["gain"] = np.linspace(-12, 12, V)
    g = gpu_bank(V, osc="saw", filt="biquad", biquad_type=btype, max_frames=B); o = port.Bank(V, osc="saw", filt="biquad", biquad_type=btype)
    W.configure_bank(g, "biquad", p); W.configure_bank(o, "biquad", p)
    og, _ = g.process(B); oo, _ = o.process(B)
    _close(og, oo, False, btype)


@pytest.mark.parametrize("mix", [(1, 0, 0, 0), (0, 1, 0, 0), (0, 0, 1, 0), (0, 0, 0, 1), (0.3, 0.2, 0.4, 0.1)])
def test_svf_mix_weights(port, mix):
    V, B = 64, 256
    mix = tuple(float(m) for m in mix)
    p = W.voice_params(V, seed=6); p["res_svf"][0] = 0.0
    g = gpu_bank(V, osc="saw", filt="svf", svf_mix=mix, max_frames=B); o = port.Bank(V, osc="saw", filt="svf", svf_mix=mix)
    W.configure_bank(g, "svf", p); W.configure_bank(o, "svf", p)
    og, _ = g.process(B); oo, _ = o.process(B)
    _close(og, oo, False, str(mix))


def test_lores_clamps_and_nan(port):
    V, B = 6, 64
    p = W.voice_params(V, seed=2)
    p["cutoff"] = np.array([1.0, 9.999, 10.0, 47999.0, 48000.0, 96000.0])
    p["q_lores"] = np.array([0.0, 0.5, 1.0, 1.5, 2.0, 3.0])
    for filt in ("lores", "hires"):
        g = gpu_bank(V, osc="saw", filt=filt, max_frames=B); o = port.Bank(V, osc="saw", filt=filt)
        W.configure_bank(g, filt, p); W.configure_bank(o, filt, p)
        og, _ = g.process(B); oo, _ = o.process(B)
        _close(og, oo, False, filt)
        assert np.isnan(og[-1, 4])


def test_lores_without_parameters_is_an_error():
    g = gpu_bank(4, osc="saw", filt="lores", max_frames=8)
    with pytest.raises(capi.MxbError):
        g.process(8)


@pytest.mark.parametrize("filt", ["none", "lores", "biquad"])
def test_envelope_state_machine(port, filt):
    V, B = 256, 512
    p = W.voice_params(V, seed=9)
    p["env_holdtime"] = np.array([1, 1, 0, 5, 100, 1000, 1, 3] * (V // 8), dtype=np.float64)
    g = gpu_bank(V, osc="saw", filt=filt, env=True, max_frames=B); o = port.Bank(V, osc="saw", filt=filt, env=True)
    W.configure_bank(g, filt, p, env=True); W.configure_bank(o, filt, p, env=True)
    for blk in range(8):
        on, off = W.gate(V, B, blk)
        if blk == 5:
            on[:] = 0; off[:] = B
        og, _ = g.process(B, on, off); oo, _ = o.process(B, on, off)
        _close(og, oo, False, f"env blk{blk}")
        for s in ("env_holdcount", "env_flags"):
            assert np.array_equal(g.get(s), o.get(s)), (blk, s)           # integer state: exact
        for s in ("env_amplitude", "env_output"):
            _close(g.get(s), o.get(s), False, s)


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("B", [1024, 700, 37])
def test_delayline_index_exact(port, ragged, B):
    V, cap = 200, 512
    p = W.voice_params(V, seed=4, delay_size=cap, ragged_delay=ragged)
    if ragged:
        p["delay_size"][:8] = [1, 2, 3, 63, 64, 65, 96, cap]      # literal path below 64 slots, staged path from 64
    g = gpu_bank(V, osc="saw", env=True, delay=True, delay_capacity=cap, max_frames=B)
    o = port.Bank(V, osc="saw", env=True, delay=True, delay_capacity=cap)
    W.configure_bank(g, "none", p, env=True, delay=True); W.configure_bank(o, "none", p, env=True, delay=True)
    for blk in range(4):
        on, off = W.gate(V, B, blk)
        if blk == 2:       # ring shrinks between blocks: `phase >= size -> 0` on the next access (SURVEY.md A6)
            p["delay_size"] = np.maximum(1, p["delay_size"] // 2)
            g.set("delay_size", p["delay_size"]); o.set("delay_size", p["delay_size"])
        og, mg = g.process(B, on, off, want_mix=True); oo, mo = o.process(B, on, off, want_mix=True)
        _close(og, oo, False, f"delay blk{blk}")
        np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-11)
        assert np.array_equal(g.get("delay_phase"), o.get("delay_phase")), blk     # int ring index: exact
    for v in range(0, V, 17):
        assert np.array_equal(g.ring(v, cap), o.ring(v, cap)), v


@pytest.mark.parametrize("filt", ["none", "svf"])
def test_delay_envelope_steady_windows(port, filt):
    """K2 runs whole windows in which every voice of a warp sits in the sustain or the release state of maxiEnv::adsr
    through two-statement shortcuts: gates held over whole blocks, releases that last for blocks, amplitudes that
    underflow to exactly 0 (release 0.5 and 0.0), mixed with warps that are mid-attack -- all bit-identical."""
    V, B, cap = 160, 256, 128
    p = W.voice_params(V, seed=12, delay_size=cap)
    g = gpu_bank(V, osc="saw", filt=filt, env=True, delay=True, delay_capacity=cap, max_frames=B)
    o = port.Bank(V, osc="saw", filt=filt, env=True, delay=True, delay_capacity=cap)
    W.configure_bank(g, filt, p, env=True, delay=True); W.configure_bank(o, filt, p, env=True, delay=True)
    rng = np.random.default_rng(12)
    att = np.where(np.arange(V) < 128, 0.5, 0.001)                 # warps 0-3 reach hold within a few steps, warp 4 never
    dec = np.full(V, 0.5); sus = np.full(V, 0.3)
    rel = np.choose(np.arange(V) % 4, [0.999, 0.5, 0.0, 0.9])
    hold = np.choose(np.arange(V) % 3, [1.0, 5.0, 40.0])
    for b in (g, o):
        b.set("env_attack", att); b.set("env_decay", dec); b.set("env_sustain", sus); b.set("env_release", rel)
        b.set("env_holdtime", hold)
    t_on = rng.integers(0, 20, V).astype(np.int32); t_mid = rng.integers(40, 200, V).astype(np.int32)
    zeros, full = np.zeros(V, np.int32), np.full(V, B, np.int32)
    gates = [(t_on, full), (zeros, full), (zeros, full), (zeros, t_mid)] + [(zeros, zeros)] * 8
    for blk, (on, off) in enumerate(gates):
        og, _ = g.process(B, on, off); oo, _ = o.process(B, on, off)
        _close(og, oo, False, f"steady blk{blk}")
        for s in ("env_holdcount", "env_flags", "delay_phase"):
            assert np.array_equal(g.get(s), o.get(s)), (blk, s)
        for s in ("env_amplitude", "env_output"):
            _close(g.get(s), o.get(s), False, s)
    assert np.count_nonzero(g.get("env_amplitude") == 0.0) >= V // 4      # the release-to-zero case was reached


@pytest.mark.parametrize("delay", ["dl", "position"])
def test_per_sample_delay_size(port, delay):
    """SURVEY.md 8(f) rank 4: the `size` argument of dl()/dlFromPosition() changing on every call (flanger / chorus):
    ring indices and samples bit-identical, block after block, then back to the block-constant size."""
    from test_oracle_vs_reference import flanger_sizes
    V, B, cap = 100, 300, 256
    p = W.voice_params(V, seed=41, delay_size=cap, ragged_delay=True)
    g = gpu_bank(V, osc="saw", filt="lores", env=True, delay=delay, delay_capacity=cap, max_frames=B)
    o = port.Bank(V, osc="saw", filt="lores", env=True, delay=delay, delay_capacity=cap)
    W.configure_bank(g, "lores", p, env=True, delay=True); W.configure_bank(o, "lores", p, env=True, delay=True)
    if delay == "position":
        pos = (np.arange(V) % 40).astype(np.float64) * 3.0
        g.set("delay_position", pos); o.set("delay_position", pos)
    for blk in range(3):
        on, off = W.gate(V, B, blk); sz = flanger_sizes(V, B, blk, cap)
        og, mg = g.process(B, on, off, delay_size_tv=sz, want_mix=True); oo, mo = o.process(B, on, off, delay_size_tv=sz, want_mix=True)
        _close(og, oo, False, f"swept size blk{blk}")
        np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-11)
        assert np.array_equal(g.get("delay_phase"), o.get("delay_phase")), blk
    og, _ = g.process(B); oo, _ = o.process(B)
    _close(og, oo, False, "back to the block-constant size")
    for v in range(0, V, 9):
        assert np.array_equal(g.ring(v, cap), o.ring(v, cap)), v
    nd = gpu_bank(8, osc="saw", max_frames=16)
    with pytest.raises(capi.MxbError):
        nd.process(16, delay_size_tv=np.full((16, 8), 4.0))


def test_clone_and_state_restore(port):
    """The reference's voices are value objects: copying one forks it, assigning its members restores it. mxb_bank_clone is
    the copy; get_state/get_ring -> set_state/set_ring into a freshly configured bank is the member-wise restore. Both
    continue bit-identically (and identically to the oracle, which never stopped)."""
    V, B, cap = 70, 128, 64
    p = W.voice_params(V, seed=17, delay_size=cap, ragged_delay=True)
    mk = lambda: gpu_bank(V, osc="pulse", filt="svf", env=True, delay=True, delay_capacity=cap, max_frames=B)
    g = mk(); o = port.Bank(V, osc="pulse", filt="svf", env=True, delay=True, delay_capacity=cap)
    W.configure_bank(g, "svf", p, env=True, delay=True); W.configure_bank(o, "svf", p, env=True, delay=True)
    for blk in range(2):
        on, off = W.gate(V, B, blk)
        g.process(B, on, off); o.process(B, on, off)
    c = g.clone()                                                   # fork
    r = mk(); W.configure_bank(r, "svf", p, env=True, delay=True)   # member-wise restore into a fresh bank
    r.set("phase", g.get("phase"))
    for s in ("osc_output", "filt0", "filt1", "filt2", "env_amplitude", "env_output", "env_holdcount", "env_flags", "delay_phase"):
        r.set_state(s, g.get(s))
    for v in range(V):
        r.set_ring(v, g.ring(v, cap))
    for blk in range(2, 4):
        on, off = W.gate(V, B, blk)
        og, _ = g.process(B, on, off); oc, _ = c.process(B, on, off); orr, _ = r.process(B, on, off); oo, _ = o.process(B, on, off)
        assert np.array_equal(og, oo) and np.array_equal(oc, oo) and np.array_equal(orr, oo), blk
    c.set("freq", 2.0 * p["freq"])                                  # the copies are independent of each other
    oc, _ = c.process(B); og, _ = g.process(B)
    assert not np.array_equal(oc, og)
    with pytest.raises(capi.MxbError):
        g.set_state("freq", p["freq"])                              # parameters go through set_param


@pytest.mark.parametrize("osc", ["triangle", "phasorbetween"])
def test_delay_with_filter_and_nonpositive_size(port, osc):
    V, B, cap = 40, 130, 128
    p = W.voice_params(V, seed=8, delay_size=cap, ragged_delay=True)
    p["delay_size"][:3] = [0.0, -3.0, 1.0]
    g = gpu_bank(V, osc=osc, filt="svf", delay=True, delay_capacity=cap, max_frames=B)
    o = port.Bank(V, osc=osc, filt="svf", delay=True, delay_capacity=cap)
    W.configure_bank(g, "svf", p, delay=True); W.configure_bank(o, "svf", p, delay=True)
    for blk in range(3):
        og, _ = g.process(B); oo, _ = o.process(B)
        _close(og, oo, False, f"blk{blk}")
        assert np.array_equal(g.get("delay_phase"), o.get("delay_phase"))


@pytest.mark.parametrize("osc,filt,env,ragged,cm,dsz", [("saw", "none", True, False, False, False), ("saw", "lores", True, True, True, False),
                                                        ("pulse", "svf", False, False, True, False), ("phasorbetween", "biquad", True, True, False, False),
                                                        ("sinewave", "hires", False, False, True, True)])
def test_modulated_frequency_and_cutoff_with_a_delay_line(port, osc, filt, env, ragged, cm, dsz):
    """VERDICT r1 next #5: per-sample frequency / cutoff on a chain WITH a delay line run on the staged-window kernel (K2), uniform and
    generic schedules, with the envelope's per-sample trigger and (last case) a per-sample delay size on top. Ring contents and the
    ring index are compared too."""
    from test_oracle_vs_reference import cutoff_sweeps, fm_frequencies
    V, B, cap = 173, 200, 128
    p = W.voice_params(V, seed=61, delay_size=cap, ragged_delay=ragged)
    g = gpu_bank(V, osc=osc, filt=filt, env=env, delay=True, delay_capacity=cap, max_frames=B)
    o = port.Bank(V, osc=osc, filt=filt, env=env, delay=True, delay_capacity=cap)
    W.configure_bank(g, filt, p, env, True); W.configure_bank(o, filt, p, env, True)
    exact = not cm and osc not in TRIG
    for blk in range(3):
        f = fm_frequencies(V, B, blk); cu = cutoff_sweeps(V, B, blk) if cm else None
        tv = trigger_bytes(V, B, blk, seed=7) if env else None
        sz = None
        if dsz:
            sz = np.floor(1 + (cap - 1) * np.random.default_rng(90 + blk).random((B, V)))
        og, mg = g.process(B, freq_tv=f, cutoff_tv=cu, trig_tv=tv, delay_size_tv=sz, want_mix=True)
        oo, mo = o.process(B, freq_tv=f, cutoff_tv=cu, trig_tv=tv, delay_size_tv=sz, want_mix=True)
        if exact:
            assert np.array_equal(og, oo), f"blk{blk}"
        else:
            np.testing.assert_allclose(og, oo, rtol=1e-9, atol=1e-12, err_msg=f"blk{blk}")
        np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-11)
        assert np.array_equal(g.get("delay_phase"), o.get("delay_phase")), blk
    on, off = (W.gate(V, B, 3) if env else (None, None))
    og, _ = g.process(B, on, off); oo, _ = o.process(B, on, off)      # block-constant parameters are in force again
    if exact:
        assert np.array_equal(og, oo)
    else:
        np.testing.assert_allclose(og, oo, rtol=1e-9, atol=1e-12)
    for v in (0, 1, 31, 32, V // 2, V - 1):
        rg, ro = g.ring(v, cap), o.ring(v, cap)
        if exact:
            assert np.array_equal(rg, ro), v
        else:
            np.testing.assert_allclose(rg, ro, rtol=1e-9, atol=1e-12, err_msg=f"ring of voice {v}")


def trigger_bytes(V, B, blk, seed=0):
    """maxiEnv::trigger written by the patch on every sample: notes that start and stop anywhere, several per block."""
    rng = np.random.default_rng(1000 * seed + blk)
    t = np.zeros((B, V), dtype=np.uint8)
    for v in range(V):
        pos = int(rng.integers(0, 200))
        while pos < B:
            ln = int(rng.integers(1, 180))
            t[pos:pos + ln, v] = 1
            pos += ln + int(rng.integers(1, 260))
    t[:, 0] = 0; t[:, 1 % V] = 1; t[::2, 2 % V] = 1           # never, always, every other sample
    return t


@pytest.mark.parametrize("filt,delay,env", [("none", False, "adsr"), ("lores", False, "adsr"), ("svf", False, "ar"), ("none", True, "adsr"),
                                            ("biquad", True, "adsr")])
def test_per_sample_trigger(port, filt, delay, env):
    """VERDICT r1 weak #4: the trigger is a public int a patch writes on any sample (src/maximilian.h:913,
    maximilian_examples/10.Filters/main.cpp:27-36): several notes inside one block, on K1 and on K2 -- bit-identical."""
    V, B, cap = 300, 700, 128
    p = W.voice_params(V, seed=51, delay_size=cap, ragged_delay=True)
    g = gpu_bank(V, osc="saw", filt=filt, env=env, delay=delay, delay_capacity=cap, max_frames=B)
    o = port.Bank(V, osc="saw", filt=filt, env=env, delay=delay, delay_capacity=cap)
    W.configure_bank(g, filt, p, env=True, delay=delay); W.configure_bank(o, filt, p, env=True, delay=delay)
    for blk in range(3):
        tv = trigger_bytes(V, B, blk)
        og, mg = g.process(B, trig_tv=tv, want_mix=True); oo, mo = o.process(B, trig_tv=tv, want_mix=True)
        _close(og, oo, False, f"trig_tv blk{blk}")
        np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-11)
        for s_ in ("env_holdcount", "env_flags"):
            assert np.array_equal(g.get(s_), o.get(s_)), (blk, s_)
    on, off = W.gate(V, B, 0)
    og, _ = g.process(B, on, off); oo, _ = o.process(B, on, off)         # and back to the interval gate
    _close(og, oo, False, "interval gate after per-sample triggers")
    with pytest.raises(capi.MxbError):
        g.process(B, on, off, trig_tv=trigger_bytes(V, B, 0))            # one or the other


@pytest.mark.parametrize("filt", ["lores", "svf"])
def test_modulated_frequency_and_cutoff_with_envelope(port, filt):
    """The combination real patches use (VERDICT r1 weak #4): FM + swept cutoff + ADSR with per-sample triggers in one chain."""
    from test_oracle_vs_reference import cutoff_sweeps, fm_frequencies
    V, B = 150, 300
    p = W.voice_params(V, seed=52)
    g = gpu_bank(V, osc="saw", filt=filt, env=True, max_frames=B); o = port.Bank(V, osc="saw", filt=filt, env=True)
    W.configure_bank(g, filt, p, env=True); W.configure_bank(o, filt, p, env=True)
    for blk in range(3):
        f = fm_frequencies(V, B, blk); cu = cutoff_sweeps(V, B, blk); tv = trigger_bytes(V, B, blk, seed=3)
        og, _ = g.process(B, freq_tv=f, cutoff_tv=cu, trig_tv=tv); oo, _ = o.process(B, freq_tv=f, cutoff_tv=cu, trig_tv=tv)
        np.testing.assert_allclose(og, oo, rtol=1e-9, atol=1e-12, err_msg=f"blk{blk}")
        og, _ = g.process(B, freq_tv=f, trig_tv=tv); oo, _ = o.process(B, freq_tv=f, trig_tv=tv)      # FM alone: no device libm
        np.testing.assert_allclose(og, oo, rtol=1e-9, atol=1e-12)


def test_host_staging_grows_with_the_block(port):
    """Host-memory blocks of 16, 300, 40 and 512 frames through one bank (ADSR, lores, delay line) with every per-sample stream
    (frequency, cutoff, trigger bytes, delay size), out and the bus: each staging buffer grows between blocks, and an fp32 block
    followed by an fp64 block of the same length grows the output's by element size. Against the oracle at the bars of the
    modulated tests (the swept cutoff is designed with libdevice: 1e-9); fp32 blocks are the oracle's output rounded to float32."""
    from test_oracle_vs_reference import cutoff_sweeps, fm_frequencies
    V, cap = 173, 128
    p = W.voice_params(V, seed=71, delay_size=cap)
    g = gpu_bank(V, osc="saw", filt="lores", env=True, delay=True, delay_capacity=cap, max_frames=512)
    o = port.Bank(V, osc="saw", filt="lores", env=True, delay=True, delay_capacity=cap)
    W.configure_bank(g, "lores", p, env=True, delay=True); W.configure_bank(o, "lores", p, env=True, delay=True)
    blocks = [(16, np.float64), (300, np.float64), (40, np.float64), (512, np.float32), (512, np.float64)]
    for blk, (B, dt) in enumerate(blocks):
        f = fm_frequencies(V, B, blk); cu = cutoff_sweeps(V, B, blk); tv = trigger_bytes(V, B, blk, seed=11)
        sz = np.floor(1 + (cap - 1) * np.random.default_rng(70 + blk).random((B, V)))
        og, mg = g.process(B, freq_tv=f, cutoff_tv=cu, trig_tv=tv, delay_size_tv=sz, want_mix=True, out_dtype=dt)
        oo, mo = o.process(B, freq_tv=f, cutoff_tv=cu, trig_tv=tv, delay_size_tv=sz, want_mix=True)
        assert og.dtype == dt
        # fp32: rounding to float32 (2^-24 relative) on top of the 1e-9 of the cutoff design
        np.testing.assert_allclose(og, oo, rtol=1e-9 if dt == np.float64 else 2.0 ** -24 + 1e-9, atol=1e-12, err_msg=f"blk{blk} ({B} frames)")
        np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-11, err_msg=f"blk{blk} ({B} frames)")
        for s_ in ("delay_phase", "env_holdcount", "env_flags"):
            assert np.array_equal(g.get(s_), o.get(s_)), (blk, s_)
    for v in (0, 1, 31, 32, V // 2, V - 1):
        np.testing.assert_allclose(g.ring(v, cap), o.ring(v, cap), rtol=1e-9, atol=1e-12, err_msg=f"ring of voice {v}")


def test_play_block_is_the_interleaved_bus(port):
    """mxb_play_block = routing() of cpp/commandline/player.cpp:25-44: the interleaved RTAUDIO_FLOAT64 buffer of the next block."""
    V, B = 500, 256
    p = W.voice_params(V, seed=53)
    g = gpu_bank(V, osc="saw", filt="svf", max_frames=B); g6 = gpu_bank(V, osc="saw", filt="svf", max_frames=B); o = port.Bank(V, osc="saw", filt="svf")
    for k in (g, g6, o):
        W.configure_bank(k, "svf", p)
    for blk in range(2):
        buf = g.play_block(B, 2); buf6 = g6.play_block(B, 6); _, mo = o.process(B, want_out=False, want_mix=True)
        np.testing.assert_allclose(buf, mo, rtol=1e-9, atol=1e-11)
        assert np.array_equal(buf6[:, :2], buf) and np.all(buf6[:, 2:] == 0.0)


@pytest.mark.parametrize("osc,filt,delay", [("sinewave", "none", False), ("saw", "svf", False), ("phasor", "biquad", False),
                                            ("triangle", "lores", False), ("phasorbetween", "hires", False)])
def test_per_sample_frequency_fm(port, osc, filt, delay):
    """SURVEY.md 8(f) rank 1: audio-rate modulated oscillator frequency, mxb_bank_process_fm."""
    from test_oracle_vs_reference import fm_frequencies
    V, B, cap = 130, 200, 128
    p = W.voice_params(V, seed=31, delay_size=cap)
    g = gpu_bank(V, osc=osc, filt=filt, delay=delay, delay_capacity=cap, max_frames=B)
    o = port.Bank(V, osc=osc, filt=filt, delay=delay, delay_capacity=cap)
    W.configure_bank(g, filt, p, False, delay); W.configure_bank(o, filt, p, False, delay)
    for blk in range(3):
        f = fm_frequencies(V, B, blk)
        og, mg = g.process(B, freq_tv=f, want_mix=True); oo, mo = o.process(B, freq_tv=f, want_mix=True)
        _close(og, oo, osc in TRIG, f"fm {osc} blk{blk}")
        np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-11)
    og, _ = g.process(B); oo, _ = o.process(B)
    _close(og, oo, osc in TRIG, "back to block-constant frequency")


@pytest.mark.parametrize("osc,filt,fm", [("saw", "svf", False), ("saw", "lores", False), ("phasor", "hires", True), ("square", "svf", True)])
def test_per_sample_cutoff(port, osc, filt, fm):
    """SURVEY.md 8(f) rank 1 / A6b: a filter cutoff that changes every sample (lores/hires call argument; maxiSVF::setCutoff
    before every play()). The coefficient design runs per sample with libdevice's cos/sqrt/pow/tan instead of glibc's:
    not bit-identical any more -- 1e-9 relative + 1e-12 (north_star's bar is 1e-5)."""
    from test_oracle_vs_reference import cutoff_sweeps, fm_frequencies
    V, B = 133, 192
    p = W.voice_params(V, seed=33)
    g = gpu_bank(V, osc=osc, filt=filt, max_frames=B); o = port.Bank(V, osc=osc, filt=filt)
    W.configure_bank(g, filt, p); W.configure_bank(o, filt, p)
    for blk in range(3):
        cu = cutoff_sweeps(V, B, blk); f = fm_frequencies(V, B, blk) if fm else None
        og, mg = g.process(B, freq_tv=f, cutoff_tv=cu, want_mix=True); oo, mo = o.process(B, freq_tv=f, cutoff_tv=cu, want_mix=True)
        np.testing.assert_allclose(og, oo, rtol=1e-9, atol=1e-12, err_msg=f"swept {filt} blk{blk}")
        np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-11)
    og, _ = g.process(B); oo, _ = o.process(B)        # the block-constant MXB_P_CUTOFF is in force again
    np.testing.assert_allclose(og, oo, rtol=1e-9, atol=1e-12)


def test_per_sample_cutoff_refused_where_not_built():
    g = gpu_bank(8, osc="saw", filt="biquad", max_frames=16)
    g.set("cutoff", 500.0); g.set("resonance", 1.0); g.set("gain", 0.0)
    with pytest.raises(capi.MxbError):
        g.process(16, cutoff_tv=np.full((16, 8), 300.0))
    g = gpu_bank(8, osc="saw", filt="biquad", delay=True, delay_capacity=64, max_frames=16)
    g.set("cutoff", 500.0); g.set("resonance", 1.0); g.set("gain", 0.0); g.set("delay_size", 32.0)
    with pytest.raises(capi.MxbError):
        g.process(16, cutoff_tv=np.full((16, 8), 300.0))


def test_env_ar(port):
    # maxiEnv::ar, src/maximilian.cpp:1319-1358 (output = input in the hold states; clamp test on every call)
    V, B = 200, 400
    p = W.voice_params(V, seed=19)
    att, dec, rel = W.env_coeffs(p)
    hold = np.array([1, 0, 5, 50, 300, 1, 2, 1000] * (V // 8), dtype=np.float64)
    g = gpu_bank(V, osc="saw", filt="lores", env="ar", max_frames=B); o = port.Bank(V, osc="saw", filt="lores", env="ar")
    for k in (g, o):
        W.configure_bank(k, "lores", p)
        k.set("env_attack", att); k.set("env_release", rel); k.set("env_holdtime", hold)
    for blk in range(6):
        on, off = W.gate(V, B, blk)
        if blk == 3:
            on[:] = 0; off[:] = B
        og, _ = g.process(B, on, off); oo, _ = o.process(B, on, off)
        _close(og, oo, False, f"ar blk{blk}")
        for s in ("env_holdcount", "env_flags"):
            assert np.array_equal(g.get(s), o.get(s)), (blk, s)


def test_dl_from_position(port):
    # maxiDelayline::dlFromPosition, src/maximilian.cpp:431-439
    V, B, cap = 70, 300, 256
    p = W.voice_params(V, seed=23, delay_size=cap, ragged_delay=True)
    pos = np.random.default_rng(1).integers(0, 300, V).astype(np.float64)      # some >= size -> 0
    g = gpu_bank(V, osc="saw", delay="position", delay_capacity=cap, max_frames=B)
    o = port.Bank(V, osc="saw", delay="position", delay_capacity=cap)
    for k in (g, o):
        W.configure_bank(k, "none", p, False, True)
        k.set("delay_position", pos)
    for blk in range(3):
        og, _ = g.process(B); oo, _ = o.process(B)
        _close(og, oo, False, f"dlFromPosition blk{blk}")
        assert np.array_equal(g.get("delay_phase"), o.get("delay_phase"))
    for v in range(0, V, 9):
        assert np.array_equal(g.ring(v, cap), o.ring(v, cap)), v


def test_delay_size_above_capacity_rejected():
    g = gpu_bank(4, osc="saw", delay=True, delay_capacity=64, max_frames=8)
    with pytest.raises(capi.MxbError):
        g.set("delay_size", 65.0)


@pytest.mark.parametrize("mix", [False, True], ids=["out", "out+mix"])
@pytest.mark.parametrize("lead", ["none", "1", "16", "17", "last", "size"])
@pytest.mark.parametrize("size", [32, 48, 64, 112, 128, 144, 160])
def test_uniform_schedule_ring_sweep(port, size, lead, mix):
    """K2's uniform schedule (one bulk copy per window each way) on rings of 2 to 10 chunks: how long a window's request waits
    for older write-backs depends on the chunk count (all of them below 9 chunks, all but the latest seven from 9 on). Every
    1024-frame block wraps the ring many times. A first block of `lead` frames sets where the next block starts: slot 16
    (a warp that starts at chunk 1), the last chunk, or exactly `size` (the index goes back to 0 before the next access);
    lengths 1, 16 and 17 also end in a short window that writes a whole chunk back. 100 voices: the last warp is partial.
    Four blocks, then one with a per-sample frequency (the modulated kernel); output, bus, ring index and every ring
    bit-exact against the oracle."""
    from test_oracle_vs_reference import fm_frequencies
    V, B, cap = 100, 1024, 160
    n0 = {"none": 0, "1": 1, "16": 16, "17": 17, "last": size - 16, "size": size}[lead]
    p = W.voice_params(V, seed=size, delay_size=size)
    g = gpu_bank(V, osc="saw", delay=True, delay_capacity=cap, max_frames=B)
    o = port.Bank(V, osc="saw", delay=True, delay_capacity=cap)
    W.configure_bank(g, "none", p, delay=True); W.configure_bank(o, "none", p, delay=True)
    blocks = ([(n0, None)] if n0 else []) + [(B, None)] * 4 + [(B, fm_frequencies(V, B, 0))]
    for i, (n, f) in enumerate(blocks):
        og, mg = g.process(n, want_mix=mix, freq_tv=f); oo, mo = o.process(n, want_mix=mix, freq_tv=f)
        _close(og, oo, False, f"block {i} ({n} frames)")
        if mix:
            np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-11, err_msg=f"block {i}")
        assert np.array_equal(g.get("delay_phase"), o.get("delay_phase")), f"block {i}: ring index"
    for v in range(V):
        assert np.array_equal(g.ring(v, cap), o.ring(v, cap)), f"ring of voice {v}"


def test_fp32_output_storage(port):
    V, B = 512, 256
    p = W.voice_params(V, seed=12)
    g = gpu_bank(V, osc="saw", filt="biquad", max_frames=B); o = port.Bank(V, osc="saw", filt="biquad")
    W.configure_bank(g, "biquad", p); W.configure_bank(o, "biquad", p)
    og, _ = g.process(B, out_dtype=np.float32); oo, _ = o.process(B)
    assert og.dtype == np.float32
    assert np.array_equal(og, oo.astype(np.float32))          # state stays fp64; only the stored sample is rounded


# (K1 voices, filter, mix) | (K2 voices, ring sizes, mix, per-sample frequency)
FP32_CASES = {
    "k1_even": ("k1", 512, "biquad", False), "k1_even_mix": ("k1", 512, "biquad", True),
    "k1_odd": ("k1", 513, "biquad", False), "k1_odd_mix": ("k1", 513, "svf", True),
    "k2_uniform": ("k2", 161, "uniform", False), "k2_uniform_mix": ("k2", 161, "uniform", True),
    "k2_generic_mix": ("k2", 161, "generic", True), "k2_literal": ("k2", 161, "literal", False),
    "k2_modulated_mix": ("k2", 161, "modulated", True),
}


@pytest.mark.parametrize("case", list(FP32_CASES))
def test_fp32_output_storage_paths(port, case):
    """fp32 storage rounds only the stored sample: the output is the oracle's rounded to float32, bit for bit, and the fp64
    state, rings and bus are those of an identical bank that stores fp64. K1: the paired store (even V), the scalar store
    (odd V), each with and without the bus. K2: uniform, generic and literal (< 32 slots) rings and the modulated kernel."""
    from test_oracle_vs_reference import fm_frequencies
    kern, V, kind, mix = FP32_CASES[case]
    B, cap = 256, 128
    k2 = kern == "k2"
    filt = "svf" if k2 else kind
    p = W.voice_params(V, seed=12, delay_size=cap, ragged_delay=kind == "generic")
    if kind == "literal":
        p["delay_size"] = 1.0 + np.arange(V) % 31
    kw = dict(osc="saw", filt=filt, env=k2, delay=k2, delay_capacity=cap)
    g32 = gpu_bank(V, max_frames=B, **kw); g64 = gpu_bank(V, max_frames=B, **kw); o = port.Bank(V, **kw)
    for b in (g32, g64, o):
        W.configure_bank(b, filt, p, env=k2, delay=k2)
    for blk in range(3):
        on, off = W.gate(V, B, blk) if k2 else (None, None)
        f = fm_frequencies(V, B, blk) if kind == "modulated" else None
        o32, m32 = g32.process(B, on, off, want_mix=mix, out_dtype=np.float32, freq_tv=f)
        o64, m64 = g64.process(B, on, off, want_mix=mix, freq_tv=f)
        oo, mo = o.process(B, on, off, want_mix=mix, freq_tv=f)
        assert o32.dtype == np.float32
        assert np.array_equal(o32, oo.astype(np.float32)), f"blk{blk}: fp32 output is not the oracle's, rounded"
        assert np.array_equal(o64, oo), f"blk{blk}"
        if mix:
            assert np.array_equal(m32, m64), f"blk{blk}: the bus depends on the output's storage type"
            np.testing.assert_allclose(m32, mo, rtol=1e-9, atol=1e-11)
    names = ["phase", "osc_output", "filt0", "filt1"] + (["filt2"] if filt == "svf" else [])
    names += ["env_amplitude", "env_output", "env_holdcount", "env_flags", "delay_phase"] if k2 else []
    for name in names:
        assert np.array_equal(g32.get(name), g64.get(name)), name
    if k2:
        for v in range(V):
            assert np.array_equal(g32.ring(v, cap), g64.ring(v, cap)), f"ring of voice {v}"


def test_mix_only_and_determinism(port):
    V, B = 5000, 256
    p = W.voice_params(V, seed=13)
    runs = []
    for _ in range(2):
        g = gpu_bank(V, osc="saw", filt="biquad", max_frames=B)
        W.configure_bank(g, "biquad", p)
        _, m = g.process(B, want_out=False, want_mix=True)
        runs.append(m)
    assert np.array_equal(runs[0], runs[1])                     # fixed summation order
    o = port.Bank(V, osc="saw", filt="biquad"); W.configure_bank(o, "biquad", p)
    _, mo = o.process(B, want_out=False, want_mix=True)
    np.testing.assert_allclose(runs[0], mo, rtol=1e-9, atol=1e-10)


@pytest.mark.parametrize("chain", ["k1_biquad", "k2_uniform"])
def test_mix_only_bus_is_the_out_mix_bus(port, chain):
    """The bus of a mix-only bank is the bus of an identical bank that also writes `out`, bit for bit, and a second mix-only
    run reproduces it (fixed summation order); within fp64 reassociation of the oracle's bus. K2: uniform 128-slot rings,
    ADSR notes, a partial last warp."""
    V, B, NB, cap = 5000, 256, 3, 128
    k2 = chain.startswith("k2")
    filt = "none" if k2 else "biquad"
    p = W.voice_params(V, seed=13, delay_size=cap)
    kw = dict(osc="saw", filt=filt, env=k2, delay=k2, delay_capacity=cap)
    gates = [W.gate(V, B, 4 * blk) if k2 else (None, None) for blk in range(NB)]
    runs = []
    for want_out in (False, False, True):
        g = gpu_bank(V, max_frames=B, **kw)
        W.configure_bank(g, filt, p, env=k2, delay=k2)
        runs.append([g.process(B, on, off, want_out=want_out, want_mix=True)[1] for on, off in gates])
    o = port.Bank(V, **kw); W.configure_bank(o, filt, p, env=k2, delay=k2)
    for blk, (on, off) in enumerate(gates):
        assert np.array_equal(runs[0][blk], runs[1][blk]), f"blk{blk}: mix-only runs differ"
        assert np.array_equal(runs[0][blk], runs[2][blk]), f"blk{blk}: mix-only bus != out+mix bus"
        _, mo = o.process(B, on, off, want_out=False, want_mix=True)
        np.testing.assert_allclose(runs[0][blk], mo, rtol=1e-9, atol=1e-10)


@pytest.mark.parametrize("f32", [False, True], ids=["f64", "f32"])
def test_misaligned_device_output(port, f32):
    """K1 picks its store flavour once per block: `out` one element past an aligned address (8 bytes for fp64, 4 for fp32) on an
    even bank, which would otherwise take the paired stores, must take the scalar ones -- the same bits as an aligned `out`,
    and nothing written outside it."""
    import torch
    V, B = 1024, 200
    dev = torch.device("cuda", 0)
    dt = torch.float32 if f32 else torch.float64
    p = W.voice_params(V, seed=14)
    banks = [gpu_bank(V, osc="saw", filt="svf", max_frames=B) for _ in range(2)]
    o = port.Bank(V, osc="saw", filt="svf")
    for b in banks + [o]:
        W.configure_bank(b, "svf", p)
    bufs = [torch.full((B * V + 2,), -7.0, dtype=dt, device=dev) for _ in range(2)]
    views = [bufs[0][:B * V], bufs[1][1:1 + B * V]]
    assert views[0].data_ptr() % 16 == 0 and views[1].data_ptr() % 16 == (4 if f32 else 8)
    for blk in range(2):
        for b, v in zip(banks, views):
            b.process_device(B, out_ptr=v.data_ptr(), f32=f32)
        torch.cuda.synchronize()
        oo, _ = o.process(B)
        ref = oo.astype(np.float32) if f32 else oo
        got = [v.cpu().numpy().reshape(B, V) for v in views]
        assert np.array_equal(got[0], ref), f"blk{blk}: aligned out differs from the oracle"
        assert np.array_equal(got[1], got[0]), f"blk{blk}: misaligned out differs from aligned out"
    assert bufs[1][0].item() == -7.0 and bufs[1][-1].item() == -7.0 and bufs[0][-2:].eq(-7.0).all().item()


def _slice_indices(V, n_each=704, mid=640):
    """2048 voices: the first and last warps of the bank and a run in the middle (CTA- and warp-boundary crossing)."""
    return np.concatenate([np.arange(0, n_each), np.arange(V // 2 - mid // 2, V // 2 + mid // 2), np.arange(V - n_each, V)])


def test_full_size_1m_voices_vs_oracle_slices(port):
    """BASELINE.json configs[1] at its own size (1 Mi voices, saw -> SVF low-pass, 1024-frame blocks, device buffers as in
    bench.py), three consecutive blocks: a 2048-voice slice (first / middle / last warps of the grid) of the materialised
    output is compared BIT FOR BIT with the CPU oracle run on those voices, the filter state and phases of the slice
    likewise; the stereo bus equals the pan-weighted sum of the materialised output (fp64 reassociation only) and a
    second identical bank reproduces it bit for bit (fixed summation order)."""
    import torch
    V, B = 1 << 20, 1024
    dev = torch.device("cuda", 0)
    p = W.voice_params(V, seed=W.SEED)
    idx = _slice_indices(V)
    big = gpu_bank(V, osc="saw", filt="svf", max_frames=B)
    W.configure_bank(big, "svf", p)
    o = port.Bank(idx.size, osc="saw", filt="svf"); W.configure_bank(o, "svf", {k: v[idx] for k, v in p.items()})
    out = torch.empty((B, V), dtype=torch.float64, device=dev)
    mix = torch.empty((B, 2), dtype=torch.float64, device=dev)
    tidx = torch.from_numpy(idx).to(dev)
    pan = torch.from_numpy(np.clip(p["pan"], 0, 1)).to(dev)
    for blk in range(3):
        big.process_device(B, out_ptr=out.data_ptr(), mix_ptr=mix.data_ptr())
        torch.cuda.synchronize()
        oo, _ = o.process(B)
        got = out[:, tidx].cpu().numpy()
        assert np.array_equal(got, oo), f"blk{blk}: slice differs from the oracle, max {np.abs(got - oo).max()}"
        ref_mix = torch.stack([out @ torch.sqrt(1 - pan), out @ torch.sqrt(pan)], dim=1)
        torch.testing.assert_close(mix, ref_mix, rtol=1e-9, atol=1e-7)
    for s_ in ("phase", "filt0", "filt1", "filt2", "osc_output"):
        assert np.array_equal(big.get(s_)[idx], o.get(s_)), s_
    mix1 = mix.cpu().numpy()
    del out
    big2 = gpu_bank(V, osc="saw", filt="svf", max_frames=B)
    W.configure_bank(big2, "svf", p)
    for blk in range(3):
        big2.process_device(B, out_ptr=None, mix_ptr=mix.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(mix.cpu().numpy(), mix1)           # mix-only kernel == out+mix kernel, run to run


@pytest.mark.parametrize("ragged", [False, True])
def test_full_size_config2_delay_256k_voices_4096_taps_vs_oracle_slices(port, ragged):
    """BASELINE.json configs[2] at its own parameters: 262 144 voices, saw -> maxiEnv::adsr -> maxiDelayline::dl with a
    4096-slot ring per voice (8 GiB of rings, 64-bit slot arithmetic), 1024-frame blocks, 5 consecutive blocks with
    note gates (so the ring index wraps: 5 * 1024 > 4096) -- the uniform 4 KB-run schedule (ragged=False) and the
    per-voice schedule (ragged sizes in [1024, 4096]). A 2048-voice slice (first / middle / last warps) of the output,
    the int ring index, the envelope state and the FULL ring contents of 24 of those voices are compared bit for bit with
    the CPU oracle run on those voices; shard invariance: the first 4096 voices as their own bank give the same bits."""
    import torch
    V, B, cap, NB = 1 << 18, 1024, 4096, 5
    dev = torch.device("cuda", 0)
    p = W.voice_params(V, seed=W.SEED + 2, delay_size=cap, ragged_delay=ragged)
    idx = _slice_indices(V)
    big = gpu_bank(V, osc="saw", env=True, delay=True, delay_capacity=cap, max_frames=B)
    W.configure_bank(big, "none", p, env=True, delay=True)
    o = port.Bank(idx.size, osc="saw", env=True, delay=True, delay_capacity=cap)
    W.configure_bank(o, "none", {k: v[idx] for k, v in p.items()}, env=True, delay=True)
    S = 4096
    small = gpu_bank(S, osc="saw", env=True, delay=True, delay_capacity=cap, max_frames=B)
    W.configure_bank(small, "none", {k: v[:S] for k, v in p.items()}, env=True, delay=True)
    out = torch.empty((B, V), dtype=torch.float64, device=dev)
    tidx = torch.from_numpy(idx).to(dev)
    for blk in range(NB):
        on, off = W.gate(V, B, 4 * (blk // 2) if blk % 2 == 0 else 1, seed=W.SEED + blk)
        d_on, d_off = torch.from_numpy(on).to(dev), torch.from_numpy(off).to(dev)
        big.process_device(B, out_ptr=out.data_ptr(), trig_on_ptr=d_on.data_ptr(), trig_off_ptr=d_off.data_ptr())
        torch.cuda.synchronize()
        oo, _ = o.process(B, on[idx], off[idx])
        got = out[:, tidx].cpu().numpy()
        assert np.array_equal(got, oo), f"blk{blk}: slice differs from the oracle, max {np.abs(got - oo).max()}"
        os_, _ = small.process(B, on[:S], off[:S])
        assert np.array_equal(out[:, :S].cpu().numpy(), os_), f"blk{blk}: shard invariance"
        assert np.array_equal(big.get("delay_phase")[idx], o.get("delay_phase")), blk          # int ring index: exact
    for s_ in ("env_holdcount", "env_flags", "env_amplitude", "env_output", "phase"):
        assert np.array_equal(big.get(s_)[idx], o.get(s_)), s_
    for k in range(0, idx.size, idx.size // 24):
        assert np.array_equal(big.ring(int(idx[k]), cap), o.ring(k, cap)), f"ring of voice {idx[k]}"
