"""The C++ host layer (include/maximilian_b200.hpp): a reference-style patch compiles against it (CPU check) and,
on the GPU, its audio-callback output equals the oracle running the same chain per sample."""
import os
import subprocess

import numpy as np
import pytest

from maximilian_b200 import build
from maximilian_b200 import workloads as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "patch_poly.cpp")


@pytest.fixture(scope="module")
def bindir(tmp_path_factory):
    """The compiled patches are build products: they go to a temporary directory, so that the suite also runs from a read-only
    checkout."""
    return tmp_path_factory.mktemp("dropin")


def compile_patch(bindir, src=SRC):
    # the library is built by __graft_entry__.build() / python -m maximilian_b200.build; a test session only links against it (on the GPU box
    # the object directory does not travel: build.build() there would recompile every kernel, minutes of GPU-box time)
    lib = build.LIB if os.path.exists(build.LIB) else build.build()
    libdir = os.path.dirname(lib)
    exe = os.path.join(str(bindir), os.path.splitext(os.path.basename(src))[0])
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
           "-L", libdir, "-lmaxib200", "-Wl,-rpath," + libdir]
    subprocess.check_call(cmd)
    return exe


SRC_SPEC = os.path.join(ROOT, "tests", "cpp", "patch_spectral.cpp")


def test_spectral_patch_compiles_against_the_dropin_header(bindir):
    exe = compile_patch(bindir, SRC_SPEC)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr


@pytest.mark.gpu
def test_spectral_patch_matches_oracle(port, tmp_path, bindir):
    """maxiFFT / maxiMFCC / maxiIFFT of the C++ layer, fed in ragged chunks, against the oracle fed sample by sample."""
    exe = compile_patch(bindir, SRC_SPEC)
    C, N, bins, hop, nc = 5, 7 * 1024 + 100, 512, 512, 13
    x = W.channel_streams(C, N, seed=44)
    x.tofile(tmp_path / "in.bin")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(C), str(N)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = open(tmp_path / "out.bin", "rb").read()
    F = int(np.frombuffer(raw, dtype=np.int32, count=1)[0]); off = 4

    def take(dtype, shape):
        nonlocal off
        n = int(np.prod(shape)); a = np.frombuffer(raw, dtype=dtype, count=n, offset=off).reshape(shape)
        off += a.nbytes
        return a
    mags, phases, db = take(np.float32, (C, F, bins)), take(np.float32, (C, F, bins)), take(np.float32, (C, F, bins))
    flat, cent = take(np.float32, (C, F)), take(np.float32, (C, F))
    co, y = take(np.float64, (C, F, nc)), take(np.float32, (C, F * hop))
    assert off == len(raw)

    o = port.Stft(C, 1024, hop).process(x)
    assert o["mags"].shape == (C, F, bins)                        # frame schedule
    assert np.array_equal(mags, o["mags"])                        # bit-identical magnitudes
    d = np.angle(np.exp(1j * (phases.astype(np.float64) - o["phases"])))
    assert np.abs(d[o["mags"] > 1e-3 * o["mags"].max(axis=-1, keepdims=True)]).max() <= 1e-4
    odb, ofl, oce = port.spectral_features(o["mags"], 1024, 48000)
    np.testing.assert_allclose(db, odb, rtol=2e-6, atol=1e-6)
    np.testing.assert_allclose(flat, ofl, rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(cent, oce, rtol=1e-4, atol=1e-3)
    oc, _ = port.Mfcc(bins, 42, nc, 20.0, 20000.0, 48000).process(o["mags"])
    np.testing.assert_allclose(co, oc, rtol=1e-9, atol=1e-12)
    oy = port.Istft(C, 1024, hop).process(o["mags"], o["phases"])
    # the resynthesis starts from this side's own phases (atan2f ulps away from the oracle's) and adds cosf/sinf ulps
    assert np.abs(y - oy).max() <= 2e-5 * np.abs(oy).max()


def test_patch_compiles_against_the_dropin_header(bindir):
    exe = compile_patch(bindir)
    assert os.path.exists(exe)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr


@pytest.mark.gpu
def test_patch_through_routing_matches_oracle(port, tmp_path, bindir):
    exe = compile_patch(bindir)
    V, B, NB, cap = 300, 256, 3, 512
    p = W.voice_params(V, seed=31, delay_size=cap, ragged_delay=True)
    gates = [W.gate(V, B, 4 * k) for k in range(NB + 1)]
    with open(tmp_path / "params.bin", "wb") as f:
        for k in ("freq", "phase", "cutoff", "res_svf", "attack_ms", "decay_ms", "env_sustain", "release_ms",
                  "delay_size", "delay_feedback", "pan", "gain"):
            f.write(np.ascontiguousarray(p[k], dtype=np.float64).tobytes())
        for on, off in gates:
            f.write(on.astype(np.int32).tobytes()); f.write(off.astype(np.int32).tobytes())
    r = subprocess.run([exe, str(tmp_path / "params.bin"), str(tmp_path / "out.bin"), str(V), str(B), str(NB)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = np.fromfile(tmp_path / "out.bin", dtype=np.float64)
    mix = raw[:NB * B * 2].reshape(NB, B, 2)
    voices = raw[NB * B * 2:].reshape(B, V)

    o = port.Bank(V, osc="saw", filt="svf", env=True, delay=True, delay_capacity=cap)
    W.configure_bank(o, "svf", p, env=True, delay=True)
    for k in range(NB):
        _, mo = o.process(B, gates[k][0], gates[k][1], want_out=False, want_mix=True)
        np.testing.assert_allclose(mix[k], mo, rtol=1e-9, atol=1e-11)
    oo, _ = o.process(B, gates[NB][0], gates[NB][1])
    assert np.array_equal(voices, oo)


SRC_POLY = os.path.join(ROOT, "tests", "cpp", "patch_polysynth.cpp")


def test_polysynth_port_compiles_against_the_dropin_header(bindir):
    """cpp/commandline/maximilian_examples/15.polysynth/main.cpp ported to the block-rate classes: same objects, same expressions."""
    exe = compile_patch(bindir, SRC_POLY)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr


@pytest.mark.gpu
def test_polysynth_port_matches_oracle(port, tmp_path, bindir):
    """The polysynth example (two pulse VCOs summed into a lores VCF, sinebuf LFO on frequency and cutoff, ADSR applied after the filter,
    notes triggered on single samples by a metronome) through the C++ layer -> patch interpreter, against the same graph
    (tests/patch_cases.py) run by the C oracle with the trigger stream the C++ control code produced: 1e-9 relative (lores designs its
    coefficients on every sample: libdevice cos / sqrt / pow)."""
    import golden_checks as G
    import patch_cases as PC
    exe = compile_patch(bindir, SRC_POLY)
    g = G.load("tables")
    np.concatenate([g["sine"], g["transition"], [float(g["sine_before"])]]).astype(np.float64).tofile(tmp_path / "tables.bin")
    NB, B, V = 40, 512, 6
    r = subprocess.run([exe, str(tmp_path / "tables.bin"), str(tmp_path / "out.bin"), str(NB), str(B)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = np.fromfile(tmp_path / "out.bin", dtype=np.float64)
    trig = raw[:NB * B * V].reshape(NB, B, V); out = raw[NB * B * V:].reshape(NB, B, 2)
    assert 2 <= trig.sum() <= 4 and abs(trig.sum() - NB * B * 8 / 44100) <= 1        # the 8 Hz metronome fired
    name, d, params, inputs, exact, taps = PC.polysynth()
    port.set_tables(g["sine"], g["transition"], float(g["sine_before"]), "port")
    o = port.Patch(d, V, sample_rate=44100, kind="port")
    pitch = np.arange(1.0, 7.0)
    lib = port.load("port")
    vals = dict(attack=lib.mxo_env_attack_coeff(0.0, 44100), decay=lib.mxo_env_decay_coeff(200.0, 44100), sustain=0.2,
                release=lib.mxo_env_decay_coeff(2000.0, 44100), f1=55.0 * pitch, f2=110.0 * pitch, pitch=pitch, pan=0.5)
    for k, v in vals.items():
        o.set(k, v)
    for blk in range(NB):
        oo, _ = o.process(B, dict(trigger=trig[blk]))
        ref = oo.sum(axis=1) * 0.5                                     # mix += VCFout*ADSRout/6 over the six voices; output = mix*0.5
        np.testing.assert_allclose(out[blk, :, 0], ref, rtol=1e-9, atol=1e-12, err_msg=f"blk{blk}")
        assert np.array_equal(out[blk, :, 0], out[blk, :, 1])
    assert np.abs(out).max() > 1e-3


SRC_FX = os.path.join(ROOT, "tests", "cpp", "patch_featurex.cpp")


def test_per_sample_feature_extractor_compiles_against_the_dropin_header(bindir):
    exe = compile_patch(bindir, SRC_FX)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr


@pytest.mark.gpu
def test_per_sample_feature_extractor_matches_oracle(port, tmp_path, bindir):
    """The reference's per-sample idiom (`if (fft.process(x)) {...}`, `y = ifft.process(mags, phases)` every sample; maxiFFTOctaveAnalyzer /
    maxiBark / maxiMFCC on the fired frame) through the C++ layer's scalar signatures, against the oracle: frame schedule exact, magnitudes
    and octave averages / peaks bit-identical, Bark 1e-12, MFCC 1e-9, resynthesis 2e-5 of max (atan2f / cosf / sinf ulps)."""
    exe = compile_patch(bindir, SRC_FX)
    N, bins, hop, nc = 6 * 1024 + 300, 512, 512, 13
    x = W.channel_streams(1, N, seed=45)
    x.tofile(tmp_path / "in.bin")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(N)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = open(tmp_path / "out.bin", "rb").read()
    F, nA = (int(v) for v in np.frombuffer(raw, dtype=np.int32, count=2)); off = 8

    def take(dtype, shape):
        nonlocal off
        n = int(np.prod(shape)); a = np.frombuffer(raw, dtype=dtype, count=n, offset=off).reshape(shape)
        off += a.nbytes
        return a
    fired, mags = take(np.float32, (N,)), take(np.float32, (1, F, bins))
    avs, pks = take(np.float32, (1, F, nA)), take(np.float32, (1, F, nA))
    spec, rel, tot = take(np.float64, (1, F, 24)), take(np.float64, (1, F, 24)), take(np.float64, (1, F))
    co, y = take(np.float64, (1, F, nc)), take(np.float32, (N,))
    assert off == len(raw)

    assert F == N // hop and np.array_equal(np.nonzero(fired)[0], hop * np.arange(1, F + 1) - 1)   # true on the sample that completes a frame
    o = port.Stft(1, 1024, hop).process(x)
    assert np.array_equal(mags, o["mags"][:, :F])
    ooc = port.Octave(1, 48000, bins, 3); ooc.config(2, 0.8, 0.9, 0.01)
    assert ooc.n_averages == nA
    oav, opk = ooc.process(o["mags"][:, :F])
    assert np.array_equal(avs, oav) and np.array_equal(pks, opk)
    sp, rl, tt = port.bark(o["mags"][:, :F], 48000, 1024)
    np.testing.assert_allclose(spec, sp, rtol=1e-12, atol=0)
    np.testing.assert_allclose(rel, rl, rtol=1e-12, atol=0)
    np.testing.assert_allclose(tot, tt, rtol=1e-12, atol=0)
    oc, _ = port.Mfcc(bins, 42, nc, 20.0, 20000.0, 48000).process(o["mags"][:, :F])
    np.testing.assert_allclose(co, oc, rtol=1e-9, atol=1e-12)
    # maxiIFFT::process reads the spectrum on the first sample of every hop: zeros before the first frame, then frame k - 1 during hop k
    K = (N + hop - 1) // hop
    zm = np.zeros((1, 1, bins), dtype=np.float32)
    oy = port.Istft(1, 1024, hop).process(np.concatenate([zm, o["mags"][:, :K - 1]], axis=1), np.concatenate([zm, o["phases"][:, :K - 1]], axis=1))
    assert np.abs(y - oy[0, :N]).max() <= 2e-5 * np.abs(oy).max()
    assert np.abs(y[hop:]).max() > 1e-3
