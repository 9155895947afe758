"""Pins the plain-C oracle (oracle/maxi_oracle.c) BIT-FOR-BIT against the unmodified reference
compiled by oracle/Makefile (oracle/_ref/libmaxiref.so), through the calls and results recorded from it (oracle/replay.py).

CPU only. Tolerance: none. fp64 and fp32 values are compared with ==, integer state exactly.
"""
import itertools

import numpy as np
import pytest

from maximilian_b200 import workloads as W
from oracle.replay import same

OSCS = ["sinewave", "coswave", "phasor", "saw", "square", "pulse", "impulse", "triangle", "phasorbetween"]
FILTS = ["none", "lores", "hires", "svf", "biquad"]


_configure = W.configure_bank


def _pair(port, reference, V, **kw):
    return port.Bank(V, kind="port", **kw), reference.Bank(V, kind="reference", **kw)


def _same(a, b):
    return same(a, b)


@pytest.mark.parametrize("osc,filt", list(itertools.product(OSCS, FILTS)))
def test_osc_filter_chains_bit_exact(port, reference, osc, filt):
    V, B = 37, 257
    p = W.voice_params(V, seed=11)
    a, b = _pair(port, reference, V, osc=osc, filt=filt)
    _configure(a, filt, p, False, False); _configure(b, filt, p, False, False)
    for _ in range(3):                        # state carried over consecutive blocks
        oa, ma = a.process(B, want_mix=True)
        ob, mb = b.process(B, want_mix=True)
        assert _same(oa, ob)
        assert _same(ma, mb)
    for s in ("phase", "filt0", "filt1", "filt2"):
        assert _same(a.get(s), b.get(s)), s


@pytest.mark.parametrize("btype", ["lowpass", "highpass", "bandpass", "notch", "peak", "lowshelf", "highshelf"])
@pytest.mark.parametrize("gain_sign", [1.0, -1.0])
def test_biquad_types_bit_exact(port, reference, btype, gain_sign):
    V, B = 16, 300
    p = W.voice_params(V, seed=5)
    p["gain"] = gain_sign * (0.5 + 11.5 * np.random.default_rng(3).random(V))
    a, b = _pair(port, reference, V, osc="saw", filt="biquad", biquad_type=btype)
    _configure(a, "biquad", p, False, False); _configure(b, "biquad", p, False, False)
    oa, _ = a.process(B); ob, _ = b.process(B)
    assert _same(oa, ob)


@pytest.mark.parametrize("mix", [(1, 0, 0, 0), (0, 1, 0, 0), (0, 0, 1, 0), (0, 0, 0, 1), (0.3, 0.2, 0.4, 0.1)])
def test_svf_mixes_bit_exact(port, reference, mix):
    V, B = 16, 300
    p = W.voice_params(V, seed=6)
    p["res_svf"][0] = 0.0                     # res == 0 -> damping 0 branch (src/maximilian.h:1327)
    a, b = _pair(port, reference, V, osc="saw", filt="svf", svf_mix=tuple(float(m) for m in mix))
    _configure(a, "svf", p, False, False); _configure(b, "svf", p, False, False)
    oa, _ = a.process(B); ob, _ = b.process(B)
    assert _same(oa, ob)


def test_lores_clamps_bit_exact(port, reference):
    # cutoff < 10 -> 10, cutoff > sr -> sr (NaN: z == 1 gives 0/0), resonance < 1 -> 1  (SURVEY.md A3)
    V, B = 6, 64
    p = W.voice_params(V, seed=2)
    p["cutoff"] = np.array([1.0, 9.999, 10.0, 47999.0, 48000.0, 96000.0])
    p["q_lores"] = np.array([0.0, 0.5, 1.0, 1.5, 2.0, 3.0])
    for filt in ("lores", "hires"):
        a, b = _pair(port, reference, V, osc="saw", filt=filt)
        _configure(a, filt, p, False, False); _configure(b, filt, p, False, False)
        oa, _ = a.process(B); ob, _ = b.process(B)
        assert _same(oa, ob)
        assert np.isnan(oa[-1, 4]) and np.isnan(oa[-1, 5])


def test_sample_rates(port, reference):
    for sr in (44100, 48000, 96000):
        V, B = 8, 200
        p = W.voice_params(V, seed=sr)
        a, b = _pair(port, reference, V, osc="sinewave", filt="svf", sample_rate=sr)
        _configure(a, "svf", p, False, False); _configure(b, "svf", p, False, False)
        oa, _ = a.process(B); ob, _ = b.process(B)
        assert _same(oa, ob)


@pytest.mark.parametrize("filt", ["none", "lores"])
def test_env_state_machine_bit_exact(port, reference, filt):
    V, B = 64, 512
    p = W.voice_params(V, seed=9)
    p["env_holdtime"] = np.array([1, 1, 0, 5, 100, 1000, 1, 3] * (V // 8), dtype=np.float64)
    a, b = _pair(port, reference, V, osc="saw", filt=filt, env=True)
    _configure(a, filt, p, True, False); _configure(b, filt, p, True, False)
    for blk in range(8):
        on, off = W.gate(V, B, blk)
        if blk == 5:                          # retrigger while still releasing, gate across the whole block
            on[:] = 0; off[:] = B
        oa, _ = a.process(B, on, off); ob, _ = b.process(B, on, off)
        assert _same(oa, ob), blk
        for s in ("env_amplitude", "env_output", "env_holdcount", "env_flags"):
            assert _same(a.get(s), b.get(s)), (blk, s)


def test_env_setters(port, reference):
    la, lb = port.load("port"), reference.load("reference")
    for ms in (0.5, 1.0, 2.0, 17.3, 500.0):
        for sr in (44100, 48000):
            assert la.mxo_env_attack_coeff(ms, sr) == lb.mxo_env_attack_coeff(ms, sr)
            assert la.mxo_env_attack_ms_coeff(ms, sr) == lb.mxo_env_attack_ms_coeff(ms, sr)
            assert la.mxo_env_decay_coeff(ms, sr) == lb.mxo_env_decay_coeff(ms, sr)
    p = W.voice_params(8, seed=1)
    att, dec, rel = W.env_coeffs(p)           # math.pow == libm pow
    for i in range(8):
        assert att[i] == lb.mxo_env_attack_coeff(p["attack_ms"][i], 48000)
        assert dec[i] == lb.mxo_env_decay_coeff(p["decay_ms"][i], 48000)
        assert rel[i] == lb.mxo_env_decay_coeff(p["release_ms"][i], 48000)


def test_delayline_indices_and_ring_bit_exact(port, reference):
    # small V: every reference maxiDelayline is a 5.6 MB object (src/maximilian.h:273)
    V, B, cap = 12, 700, 512
    p = W.voice_params(V, seed=4, delay_size=cap, ragged_delay=True)
    p["delay_size"][:4] = [1, 2, 3, cap]
    a, b = _pair(port, reference, V, osc="saw", env=True, delay=True, delay_capacity=cap)
    _configure(a, "none", p, True, True); _configure(b, "none", p, True, True)
    for blk in range(4):
        on, off = W.gate(V, B, blk)
        if blk == 2:                          # size shrinks mid-stream: phase >= size -> 0 on the next call (A6)
            p["delay_size"] = np.maximum(1, p["delay_size"] // 2)
            a.set("delay_size", p["delay_size"]); b.set("delay_size", p["delay_size"])
        oa, _ = a.process(B, on, off); ob, _ = b.process(B, on, off)
        assert _same(oa, ob), blk
        assert same(a.get("delay_phase"), b.get("delay_phase"), equal_nan=False)     # integer index: exact
    for v in range(V):
        assert _same(a.ring(v, cap), b.ring(v, cap)), v


def fm_frequencies(V, B, blk, seed=5):
    """freq[t][v] = carrier + depth * sin(2*pi*rate*t/sr): what 5.FM1's play() feeds its carrier (main.cpp:29)."""
    rng = np.random.default_rng(seed)
    carrier = 110.0 * np.exp2(3.0 * rng.random(V)); depth = 50.0 * rng.random(V); rate = 0.5 + 8.0 * rng.random(V)
    t = (blk * B + np.arange(B))[:, None] / 48000.0
    return carrier[None, :] + depth[None, :] * np.sin(2 * np.pi * rate[None, :] * t)


@pytest.mark.parametrize("osc,filt", [("sinewave", "none"), ("saw", "svf"), ("triangle", "lores")])
def test_per_sample_frequency_bit_exact(port, reference, osc, filt):
    V, B = 21, 200
    p = W.voice_params(V, seed=31)
    a, b = _pair(port, reference, V, osc=osc, filt=filt)
    _configure(a, filt, p); _configure(b, filt, p)
    for blk in range(3):
        f = fm_frequencies(V, B, blk)
        oa, _ = a.process(B, freq_tv=f); ob, _ = b.process(B, freq_tv=f)
        assert _same(oa, ob), blk
    oa, _ = a.process(B); ob, _ = b.process(B)          # back to the block-constant frequency
    assert _same(oa, ob)


def cutoff_sweeps(V, B, blk, seed=6):
    """cutoff[t][v] = centre * 2^(depth * sin(2*pi*rate*t/sr)): an LFO-swept filter, 60 Hz .. 12 kHz."""
    rng = np.random.default_rng(seed)
    centre = 200.0 * np.exp2(4.0 * rng.random(V)); depth = 1.5 * rng.random(V); rate = 0.2 + 6.0 * rng.random(V)
    t = (blk * B + np.arange(B))[:, None] / 48000.0
    return centre[None, :] * np.exp2(depth[None, :] * np.sin(2 * np.pi * rate[None, :] * t))


@pytest.mark.parametrize("osc,filt,fm", [("saw", "svf", False), ("saw", "lores", False), ("phasor", "hires", True), ("square", "svf", True)])
def test_per_sample_cutoff_bit_exact(port, reference, osc, filt, fm):
    # lores/hires take the cutoff per call; the SVF patch calls setCutoff() per sample (src/maximilian.h:1287-1290)
    V, B = 19, 160
    p = W.voice_params(V, seed=33)
    a, b = _pair(port, reference, V, osc=osc, filt=filt)
    _configure(a, filt, p); _configure(b, filt, p)
    for blk in range(3):
        cu = cutoff_sweeps(V, B, blk); f = fm_frequencies(V, B, blk) if fm else None
        oa, ma = a.process(B, freq_tv=f, cutoff_tv=cu, want_mix=True); ob, mb = b.process(B, freq_tv=f, cutoff_tv=cu, want_mix=True)
        assert _same(oa, ob) and _same(ma, mb), blk
    oa, _ = a.process(B); ob, _ = b.process(B)          # the block-constant cutoff is in force again
    assert _same(oa, ob)
    for s in ("filt0", "filt1"):
        assert _same(a.get(s), b.get(s)), s


def test_per_sample_cutoff_not_for_biquad(port, reference):
    for lib in (port, reference):
        bq = lib.Bank(4, osc="saw", filt="biquad")
        bq.set("cutoff", 800.0); bq.set("resonance", 1.0); bq.set("gain", 0.0)
        with pytest.raises(RuntimeError):
            bq.process(8, cutoff_tv=np.full((8, 4), 500.0))


def flanger_sizes(V, B, blk, cap, seed=7):
    """size[t][v] = delay + triangle-ish LFO * depth * delay + 1, like maxiFlanger::flange feeds dl() (src/maximilian.h:1144-1180);
    some voices sweep down to 1 slot, some stay constant; every value <= cap."""
    rng = np.random.default_rng(seed)
    delay = rng.integers(8, cap // 2, V).astype(np.float64); depth = rng.random(V); rate = 0.5 + 20.0 * rng.random(V)
    depth[::5] = 0.0
    t = (blk * B + np.arange(B))[:, None] / 48000.0
    lfo = 2.0 * np.abs(2.0 * ((rate[None, :] * t) % 1.0) - 1.0) - 1.0
    return np.clip(np.floor(delay[None, :] + lfo * depth[None, :] * delay[None, :] + 1.0), 1, cap)


@pytest.mark.parametrize("delay", ["dl", "position"])
def test_per_sample_delay_size_bit_exact(port, reference, delay):
    V, B, cap = 10, 300, 256            # small V: every reference maxiDelayline is a 5.6 MB object
    p = W.voice_params(V, seed=41, delay_size=cap, ragged_delay=True)
    a, b = _pair(port, reference, V, osc="saw", filt="lores", env=True, delay=delay, delay_capacity=cap)
    _configure(a, "lores", p, True, True); _configure(b, "lores", p, True, True)
    if delay == "position":
        pos = np.arange(V, dtype=np.float64) * 3.0
        a.set("delay_position", pos); b.set("delay_position", pos)
    for blk in range(3):
        on, off = W.gate(V, B, blk); sz = flanger_sizes(V, B, blk, cap)
        oa, _ = a.process(B, on, off, delay_size_tv=sz); ob, _ = b.process(B, on, off, delay_size_tv=sz)
        assert _same(oa, ob), blk
        assert same(a.get("delay_phase"), b.get("delay_phase"), equal_nan=False)
    oa, _ = a.process(B); ob, _ = b.process(B)          # back to the block-constant size
    assert _same(oa, ob)
    for v in range(V):
        assert _same(a.ring(v, cap), b.ring(v, cap)), v


def test_env_ar_bit_exact(port, reference):
    # maxiEnv::ar(input, attack, release, holdtime, trigger), src/maximilian.cpp:1319-1358
    V, B = 48, 400
    p = W.voice_params(V, seed=19)
    att, dec, rel = W.env_coeffs(p)
    hold = np.array([1, 0, 5, 50, 300, 1, 2, 1000] * (V // 8), dtype=np.float64)
    a, b = _pair(port, reference, V, osc="saw", filt="lores", env="ar")
    for k in (a, b):
        _configure(k, "lores", p)
        k.set("env_attack", att); k.set("env_release", rel); k.set("env_holdtime", hold)
    for blk in range(6):
        on, off = W.gate(V, B, blk)
        if blk == 3:
            on[:] = 0; off[:] = B
        oa, _ = a.process(B, on, off); ob, _ = b.process(B, on, off)
        assert _same(oa, ob), blk
        for s in ("env_amplitude", "env_output", "env_holdcount", "env_flags"):
            assert _same(a.get(s), b.get(s)), (blk, s)


def test_dl_from_position_bit_exact(port, reference):
    # maxiDelayline::dlFromPosition, src/maximilian.cpp:431-439
    V, B, cap = 10, 300, 256
    p = W.voice_params(V, seed=23, delay_size=cap, ragged_delay=True)
    pos = np.array([0, 1, 5, 63, 64, 100, 200, 255, 300, 17], dtype=np.float64)     # 300 >= size -> 0
    a, b = _pair(port, reference, V, osc="saw", delay="position", delay_capacity=cap)
    for k in (a, b):
        _configure(k, "none", p, False, True)
        k.set("delay_position", pos)
    for blk in range(3):
        oa, _ = a.process(B); ob, _ = b.process(B)
        assert _same(oa, ob), blk
        assert same(a.get("delay_phase"), b.get("delay_phase"), equal_nan=False)
    for v in range(V):
        assert _same(a.ring(v, cap), b.ring(v, cap)), v


def test_delay_size_nonpositive(port, reference):
    V, B = 3, 20
    a, b = _pair(port, reference, V, osc="saw", delay=True, delay_capacity=16)
    for k in (a, b):
        k.set("freq", [100.0, 200.0, 300.0]); k.set("delay_size", [0.0, -3.0, 1.0]); k.set("delay_feedback", 0.7)
    oa, _ = a.process(B); ob, _ = b.process(B)
    assert _same(oa, ob)
    assert same(a.get("delay_phase"), b.get("delay_phase"), equal_nan=False)


def test_threaded_partition_matches_serial(port):
    V, B = 64, 128
    p = W.voice_params(V, seed=3)
    a = port.Bank(V, osc="saw", filt="biquad"); b = port.Bank(V, osc="saw", filt="biquad")
    _configure(a, "biquad", p, False, False); _configure(b, "biquad", p, False, False)
    oa, ma = a.process(B, want_mix=True, threads=1)
    ob, mb = b.process(B, want_mix=True, threads=4)
    assert _same(oa, ob)
    np.testing.assert_allclose(ma, mb, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------ spectral

@pytest.mark.parametrize("n,hop", [(1024, 512), (1024, 256), (512, 128), (256, 256), (64, 16)])
def test_stft_bit_exact(port, reference, n, hop):
    C = 5
    x = W.channel_streams(C, 6 * n + 37, seed=n + hop)
    x[1] *= 1000.0
    x[2] = 0.0
    a = port.Stft(C, n, hop, kind="port"); b = reference.Stft(C, n, hop, kind="reference")
    assert _same(a.window(), b.window())
    # feed in uneven chunks: the frame schedule (integer pos) must agree exactly
    cuts = [0, 3, hop - 1, hop, 2 * n + 5, x.shape[1]]
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        ra = a.process(x[:, lo:hi]); rb = b.process(x[:, lo:hi])
        assert ra["mags"].shape == rb["mags"].shape
        for k in ("re", "im", "mags", "phases"):
            assert _same(ra[k], rb[k]), (k, lo, hi)


def test_stft_frame_schedule(port):
    # first frame after hop samples; 93 frames in 48000 samples at hop 512 (SURVEY.md section 4, item 4)
    s = port.Stft(1, 1024, 512)
    r = s.process(np.zeros((1, 48000), dtype=np.float32))
    assert r["mags"].shape[1] == 93
    s = port.Stft(1, 1024, 512)
    assert s.process(np.zeros((1, 511), dtype=np.float32))["mags"].shape[1] == 0
    assert s.process(np.zeros((1, 1), dtype=np.float32))["mags"].shape[1] == 1


# the shapes the GPU's fused paths are checked at (tests/test_gpu_spectral_epilogues.py): filter / coefficient counts that change the
# tensor-core tiling, band limits that move the bank's last bin, the 64 / 128 / 1024-bin banks of 128 / 256 / 2048-point transforms
MFCC_SHAPES = [(512, 42, 40, 20.0, 20000.0, 48000), (512, 42, 13, 20.0, 20000.0, 44100),
               (512, 256, 13, 20.0, 20000.0, 48000), (256, 20, 12, 100.0, 8000.0, 48000),
               (512, 40, 13, 20.0, 20000.0, 48000), (512, 32, 32, 20.0, 20000.0, 48000), (512, 24, 30, 300.0, 24000.0, 48000),
               (512, 3, 5, 20.0, 20000.0, 48000), (512, 1, 1, 20.0, 20000.0, 48000), (512, 26, 13, 2000.0, 8000.0, 16000),
               (512, 64, 20, 0.0, 24000.0, 48000), (512, 520, 13, 20.0, 20000.0, 48000),
               (64, 16, 13, 20.0, 20000.0, 48000), (128, 26, 13, 20.0, 20000.0, 44100), (1024, 42, 40, 20.0, 20000.0, 48000)]


def mfcc_bad_bins(cfg):
    """Bins for the non-finite rows of an MFCC test: one inside the bank's bands (the middle of its frequency range; the reference's
    bin spacing is sr / numBins) and the top bin, where no band has weight."""
    bins, _, _, fmin, fmax, sr = cfg
    return int((fmin + min(fmax, sr / 2)) / 2 / (sr / bins)), bins - 1


@pytest.mark.parametrize("cfg", MFCC_SHAPES)
def test_mfcc_bit_exact(port, reference, cfg):
    bins = cfg[0]
    st = port.Stft(3, 2 * bins, bins)
    mags = st.process(W.channel_streams(3, 2 * bins * 8, seed=bins))["mags"]
    mags[0, 0] = 0.0                                   # silent frame: log gate (> 1e-6) takes the 0 branch
    # non-finite magnitudes: the reference sums weight * magnitude over every bin, so 0 * NaN and 0 * inf make a band NaN (-> 0)
    inside, above = mfcc_bad_bins(cfg)
    mags[2, 0, 5] = np.nan
    mags[2, 1, inside] = np.inf
    mags[2, 2, above] = np.inf
    a = port.Mfcc(*cfg, kind="port"); b = reference.Mfcc(*cfg, kind="reference")
    ca, ma = a.process(mags); cb, mb = b.process(mags)
    assert _same(ma, mb)
    assert _same(ca, cb)
    assert np.all(ma[..., 0] == 0.0)                   # filter 0 is never initialised by the reference (A13)


def test_spectral_features_bit_exact(port, reference):
    # maxiFFT::magsToDB / spectralFlatness / spectralCentroid, src/libs/maxiFFT.cpp:101-132, at three transform sizes
    for n in (1024, 256, 2048):
        mags = port.Stft(3, n, n // 2).process(W.channel_streams(3, 8 * n, seed=8))["mags"]
        mags[0, 0] = 0.0                              # all-zero frame: both features return 0
        mags[1, 1, :7] = 0.0                          # zeros are skipped by the geometric mean
        for sr in (44100, 48000):
            a = port.spectral_features(mags, n, sr, kind="port")
            b = reference.spectral_features(mags, n, sr, kind="reference")
            for x, y in zip(a, b):
                assert _same(x, y)


@pytest.mark.parametrize("n,hop", [(1024, 512), (1024, 256), (256, 64)])
def test_istft_bit_exact(port, reference, n, hop):
    C = 3
    x = W.channel_streams(C, 10 * n, seed=77)
    r = port.Stft(C, n, hop).process(x)
    a = port.Istft(C, n, hop, kind="port"); b = reference.Istft(C, n, hop, kind="reference")
    F = r["mags"].shape[1]
    for lo, hi in ((0, 3), (3, F)):
        ya = a.process(r["mags"][:, lo:hi], r["phases"][:, lo:hi])
        yb = b.process(r["mags"][:, lo:hi], r["phases"][:, lo:hi])
        assert _same(ya, yb)


# ---- maxiFFTOctaveAnalyzer / maxiBark (SURVEY.md 8f-3) ------------------------------------------------------------------------

@pytest.mark.parametrize("per_octave,sr", [(1, 48000), (3, 48000), (3, 44100), (6, 48000), (0, 48000), (12, 48000)])
def test_octave_analyser_port_equals_reference(port, reference, per_octave, sr):
    """maxiFFTOctaveAnalyzer::setup + calculate per channel (float sums in bin order, peak hold / decay carried across frames and
    calls), with the public members changed from their defaults: averages and peaks bit for bit."""
    x = W.channel_streams(3, 1024 * 9, seed=5)
    mags = port.Stft(3, 1024, 512, kind="port").process(x)["mags"]
    a = port.Octave(3, sr, 512, per_octave, kind="port"); b = reference.Octave(3, sr, 512, per_octave, kind="reference")
    assert a.n_averages == b.n_averages > 0
    a.config(2, 0.8, 1.0, 0.01); b.config(2, 0.8, 1.0, 0.01)
    for lo, hi in ((0, 5), (5, mags.shape[1])):
        ra = a.process(mags[:, lo:hi]); rb = b.process(mags[:, lo:hi])
        assert same(ra[0], rb[0], equal_nan=False) and same(ra[1], rb[1], equal_nan=False), (lo, hi)


@pytest.mark.parametrize("sr,bs", [(48000, 1024), (44100, 1024), (48000, 512), (22050, 256)])
def test_bark_port_equals_reference(port, reference, sr, bs):
    """maxiBarkScaleAnalyser: integer binToHz, int band ends, the 25th band limit written behind bbLimits[24] -- specific, relative and
    total loudness bit for bit (the reference class is compiled at -O0 inside the shim: its setup() is undefined behaviour that -O2
    turns into a crash)."""
    x = W.channel_streams(3, 1024 * 9, seed=6)
    mags = np.ascontiguousarray(port.Stft(3, 1024, 512, kind="port").process(x)["mags"][..., :bs // 2])
    pa = port.bark(mags, sr, bs, "port"); pb = reference.bark(mags, sr, bs, "reference")
    for u, v in zip(pa, pb):
        assert _same(u, v)
    assert np.all(pa[1].max(axis=-1) == 1.0)


@pytest.mark.parametrize("filt,delay,env", [("none", False, "adsr"), ("lores", False, "ar"), ("svf", True, "adsr")])
def test_per_sample_trigger_port_equals_reference(port, reference, filt, delay, env):
    """maxiEnv::trigger written on every sample (mxo_bank_process_mod2): several notes per block, both envelope kinds."""
    rng = np.random.default_rng(5)
    V, B, cap = 12, 400, 64
    p = W.voice_params(V, seed=61, delay_size=cap, ragged_delay=True)
    a = port.Bank(V, osc="saw", filt=filt, env=env, delay=delay, delay_capacity=cap, kind="port")
    b = reference.Bank(V, osc="saw", filt=filt, env=env, delay=delay, delay_capacity=cap, kind="reference")
    W.configure_bank(a, filt, p, env=True, delay=delay); W.configure_bank(b, filt, p, env=True, delay=delay)
    for blk in range(3):
        tv = (rng.random((B, V)) < 0.5).astype(np.uint8)
        tv[:, 0] = 0; tv[:, 1] = 1
        tv[100:250, 2:6] = 1; tv[250:260, 2:6] = 0; tv[260:300, 2:6] = 1
        oa, ma = a.process(B, trig_tv=tv, want_mix=True); ob, mb = b.process(B, trig_tv=tv, want_mix=True)
        assert same(oa, ob, equal_nan=False) and same(ma, mb, equal_nan=False), blk
        for s_ in ("env_holdcount", "env_flags", "env_amplitude", "env_output"):
            assert same(a.get(s_), b.get(s_), equal_nan=False), (blk, s_)


@pytest.mark.parametrize("osc,filt,env,cm,dsz", [("saw", "none", True, False, False), ("saw", "lores", True, True, False), ("pulse", "svf", False, True, False),
                                                 ("phasorbetween", "biquad", True, False, False), ("sinewave", "hires", False, True, True)])
def test_modulated_chain_with_a_delay_line_port_equals_reference(port, reference, osc, filt, env, cm, dsz):
    """Per-sample frequency / cutoff (/ delay size / trigger) on a chain that ends in maxiDelayline::dl -- the combinations the modulated
    instantiation of K2 is tested against (tests/test_gpu_bank.py::test_modulated_frequency_and_cutoff_with_a_delay_line compares it
    with the port): the port itself against the compiled reference, samples, ring index and ring contents bit for bit."""
    V, B, cap = 23, 150, 96
    p = W.voice_params(V, seed=61, delay_size=cap, ragged_delay=True)
    a, b = _pair(port, reference, V, osc=osc, filt=filt, env=env, delay=True, delay_capacity=cap)
    _configure(a, filt, p, env, True); _configure(b, filt, p, env, True)
    rng = np.random.default_rng(8)
    for blk in range(3):
        f = fm_frequencies(V, B, blk); cu = cutoff_sweeps(V, B, blk) if cm else None
        tv = (rng.random((B, V)) < 0.4).astype(np.uint8) if env else None
        sz = np.floor(1 + (cap - 1) * rng.random((B, V))) if dsz else None
        oa, ma = a.process(B, freq_tv=f, cutoff_tv=cu, trig_tv=tv, delay_size_tv=sz, want_mix=True)
        ob, mb = b.process(B, freq_tv=f, cutoff_tv=cu, trig_tv=tv, delay_size_tv=sz, want_mix=True)
        assert _same(oa, ob) and _same(ma, mb), blk
        assert same(a.get("delay_phase"), b.get("delay_phase"), equal_nan=False), blk
    on, off = (W.gate(V, B, 3) if env else (None, None))
    oa, _ = a.process(B, on, off); ob, _ = b.process(B, on, off)
    assert _same(oa, ob)
    for v in (0, V // 2, V - 1):
        assert _same(a.ring(v, cap), b.ring(v, cap)), v


def test_per_sample_analysis_resynthesis_idiom(port, reference):
    """`if (fft.process(sample)) ...; out = ifft.process(fft.getMagnitudes(), fft.getPhases())` on every sample, run by the compiled
    reference (ref_shim: mxo_ref_per_sample_roundtrip), equals the block functions composed the way the C++ layer's per-sample signatures
    compose them (tests/test_cpp_dropin.py::test_per_sample_feature_extractor_matches_oracle): a frame fires on the last sample of every
    hop; the resynthesis reads zeros during the first hop and frame k - 1 during hop k. Bit for bit."""
    N, n, hop, bins = 6 * 1024 + 300, 1024, 512, 512
    x = W.channel_streams(1, N, seed=45)
    F, y, fired = reference.per_sample_roundtrip(x, n, hop, "reference")
    every_hop = np.zeros(N, dtype=np.uint8); every_hop[hop * np.arange(1, N // hop + 1) - 1] = 1
    assert F == N // hop and same(fired, every_hop, equal_nan=False)
    o = port.Stft(1, n, hop, kind="port").process(x)
    K = (N + hop - 1) // hop
    z = np.zeros((1, 1, bins), dtype=np.float32)
    oy = port.Istft(1, n, hop, kind="port").process(np.concatenate([z, o["mags"][:, :K - 1]], axis=1), np.concatenate([z, o["phases"][:, :K - 1]], axis=1))
    assert same(y, np.ascontiguousarray(oy[0, :N]), equal_nan=False)


# The corners the bank matrix (tests/bank_matrix.py) feeds the GPU banks, with the port pinned to the reference there first.
FM_OUTSIDE_AUDIO = (0.0, -300.0, 2.0 ** -70, 2.0 ** 61, 72000.0, np.inf, np.nan)


def _fm_outside_audio(V, B, blk, moderate=False):
    """fm_frequencies() with, on chosen samples, every frequency outside the audio range (moderate: only those that keep a
    sinewave's phase finite and small), on single voices and on all voices at once"""
    f = fm_frequencies(V, B, blk)
    vals = FM_OUTSIDE_AUDIO[:2] + FM_OUTSIDE_AUDIO[2:3] + FM_OUTSIDE_AUDIO[4:5] if moderate else FM_OUTSIDE_AUDIO
    for k, c in enumerate(vals):
        f[7 * k + 3, k % V] = c
        f[7 * k + 5, (k + 1) % V] = c
    f[B // 2, :] = 0.0
    return f


@pytest.mark.parametrize("osc", ["saw", "phasor", "square", "pulse", "impulse", "triangle", "phasorbetween", "sinewave", "coswave"])
def test_fm_outside_the_audio_range_bit_exact(port, reference, osc):
    V, B = 9, 64
    p = W.voice_params(V, seed=35)
    a, b = _pair(port, reference, V, osc=osc, filt="none")
    _configure(a, "none", p); _configure(b, "none", p)
    for blk in range(2):
        f = _fm_outside_audio(V, B, blk, moderate=osc in ("sinewave", "coswave"))
        oa, ma = a.process(B, freq_tv=f, want_mix=True); ob, mb = b.process(B, freq_tv=f, want_mix=True)
        assert _same(oa, ob) and _same(ma, mb), blk
        for s in ("phase", "osc_output"):
            assert _same(a.get(s), b.get(s)), (blk, s)


@pytest.mark.parametrize("filt", ["lores", "hires", "svf"])
def test_cutoff_outside_the_clamp_bit_exact(port, reference, filt):
    """per-sample cutoffs below the lores / hires clamp of 10 Hz, at and above the sample rate (lores / hires: clamped to sr, where
    the design divides 0 by 0), SVF cutoffs at and above Nyquist and above the sample rate; resonances below 1"""
    V, B = 8, 96
    p = W.voice_params(V, seed=36)
    p["q_lores"][:2] = (0.5, 0.0)
    a, b = _pair(port, reference, V, osc="saw", filt=filt)
    _configure(a, filt, p); _configure(b, filt, p)
    for blk in range(2):
        cu = cutoff_sweeps(V, B, blk)
        cu[3, :4] = (5.0, 0.0, -100.0, 9.999)
        cu[40, 4], cu[41, 5] = 24000.0, 30000.0
        cu[60, 6] = 60000.0
        if blk == 1:
            cu[B - 1, 6], cu[B - 1, 7] = 48000.0, 96000.0
        oa, ma = a.process(B, cutoff_tv=cu, want_mix=True); ob, mb = b.process(B, cutoff_tv=cu, want_mix=True)
        assert _same(oa, ob) and _same(ma, mb), blk
        for s in ("filt0", "filt1", "filt2"):
            assert _same(a.get(s), b.get(s)), (blk, s)


@pytest.mark.parametrize("delay", [False, True])
def test_ar_with_per_sample_triggers_under_fm_bit_exact(port, reference, delay):
    V, B, cap = 10, 200, 64
    rng = np.random.default_rng(37)
    p = W.voice_params(V, seed=37, delay_size=cap, ragged_delay=True)
    att, _, rel = W.env_coeffs(p)
    a, b = _pair(port, reference, V, osc="pulse", filt="lores", env="ar", delay=delay, delay_capacity=cap)
    for k in (a, b):
        _configure(k, "lores", p, delay=delay)
        k.set("env_attack", att * 20.0); k.set("env_release", rel); k.set("env_holdtime", np.resize([1.0, 0.0, 3.0, 40.0], V))
    for blk in range(3):
        tv = (rng.random((B, V)) < 0.3).astype(np.uint8)
        tv[:, 0] = 0; tv[:, 1] = 1; tv[::2, 2] = 1; tv[1::2, 2] = 0
        f = _fm_outside_audio(V, B, blk)
        oa, ma = a.process(B, freq_tv=f, trig_tv=tv, want_mix=True); ob, mb = b.process(B, freq_tv=f, trig_tv=tv, want_mix=True)
        assert _same(oa, ob) and _same(ma, mb), blk
        for s in ("env_amplitude", "env_output", "env_holdcount", "env_flags"):
            assert _same(a.get(s), b.get(s)), (blk, s)


def test_dl_from_position_with_fm_and_a_swept_cutoff_bit_exact(port, reference):
    V, B, cap = 10, 150, 96
    p = W.voice_params(V, seed=38, delay_size=cap, ragged_delay=True)
    pos = np.array([0, 1, 5, 63, 95, 100, 200, 17, 40, 90], dtype=np.float64)     # >= size -> 0
    a, b = _pair(port, reference, V, osc="phasorbetween", filt="svf", env=True, delay="position", delay_capacity=cap)
    for k in (a, b):
        _configure(k, "svf", p, env=True, delay=True)
        k.set("delay_position", pos)
    for blk in range(3):
        f = _fm_outside_audio(V, B, blk); cu = cutoff_sweeps(V, B, blk)
        on, off = W.gate(V, B, 4 * blk)
        oa, ma = a.process(B, on, off, freq_tv=f, cutoff_tv=cu, want_mix=True); ob, mb = b.process(B, on, off, freq_tv=f, cutoff_tv=cu, want_mix=True)
        assert _same(oa, ob) and _same(ma, mb), blk
        assert same(a.get("delay_phase"), b.get("delay_phase"), equal_nan=False), blk
    for v in range(V):
        assert _same(a.ring(v, cap), b.ring(v, cap)), v
