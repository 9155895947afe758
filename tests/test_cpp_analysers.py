"""The octave analyser and maxiBark of the C++ layer at transform sizes other than 1024 (tests/cpp/featurex_sizes.cpp): attached to a
maxiFFT fed one sample per call, and not attached, handed a spectrum the program makes. It compiles against
include/maximilian_b200.hpp (CPU check) and, on the GPU, equals the port: averages / peaks bit for bit, Bark 1e-12."""
import os
import subprocess

import numpy as np
import pytest

from maximilian_b200 import workloads as W
from test_cpp_dropin import ROOT, compile_patch

SRC = os.path.join(ROOT, "tests", "cpp", "featurex_sizes.cpp")


@pytest.fixture(scope="module")
def bindir(tmp_path_factory):
    return tmp_path_factory.mktemp("analysers")


def test_featurex_sizes_compiles_against_the_dropin_header(bindir):
    exe = compile_patch(bindir, SRC)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("fft_size", [512, 2048])
def test_featurex_sizes_matches_port(port, tmp_path, bindir, fft_size):
    exe = compile_patch(bindir, SRC)
    hop, bins = fft_size // 2, fft_size // 2
    N = 9 * hop + 123
    x = W.channel_streams(1, N, seed=fft_size)
    x.tofile(tmp_path / "in.bin")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(N), str(fft_size)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = open(tmp_path / "out.bin", "rb").read()
    F, nA = (int(v) for v in np.frombuffer(raw, dtype=np.int32, count=2)); off = 8

    def take(dtype, shape):
        nonlocal off
        n = int(np.prod(shape)); a = np.frombuffer(raw, dtype=dtype, count=n, offset=off).reshape(shape)
        off += a.nbytes
        return a
    fired, mags = take(np.float32, (N,)), take(np.float32, (1, F, bins))
    att = (take(np.float32, (1, F, nA)), take(np.float32, (1, F, nA)), take(np.float64, (1, F, 24)), take(np.float64, (1, F, 24)),
           take(np.float64, (1, F)))
    alone = (take(np.float32, (1, F, nA)), take(np.float32, (1, F, nA)), take(np.float64, (1, F, 24)), take(np.float64, (1, F, 24)),
             take(np.float64, (1, F)))
    assert off == len(raw)

    assert F == N // hop and np.array_equal(np.nonzero(fired)[0], hop * np.arange(1, F + 1) - 1)
    o = port.Stft(1, fft_size, hop).process(x)
    assert np.array_equal(mags, o["mags"][:, :F])
    for what, m, out in (("attached", o["mags"][:, :F], att), ("not attached", o["mags"][:, :F] / np.float32(fft_size), alone)):
        ooc = port.Octave(1, 48000, bins, 3); ooc.config(2, 0.8, 0.9, 0.01)
        assert ooc.n_averages == nA
        oav, opk = ooc.process(m)
        assert np.array_equal(out[0], oav) and np.array_equal(out[1], opk), what
        for got, exp in zip(out[2:], port.bark(m, 48000, fft_size)):
            np.testing.assert_allclose(got, exp, rtol=1e-12, atol=0, err_msg=what)
    assert np.abs(att[0]).max() > 0 and np.abs(alone[2]).max() > 0


SRC_BLOCK = os.path.join(ROOT, "tests", "cpp", "featurex_block.cpp")


def test_featurex_block_compiles_against_the_dropin_header(bindir):
    exe = compile_patch(bindir, SRC_BLOCK)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("fft_size", [512, 2048])
def test_featurex_block_matches_port(port, tmp_path, bindir, fft_size):
    """Attached analysers on a 3-channel block transform fed in ragged calls of several frames each: every channel's frames against the
    port (averages / peaks bit for bit, Bark 1e-12); an attached analyser whose band count is not the transform's bin count (larger:
    the reference's `oct.setup(sr, fftSize, ...)` next to `fft.setup(fftSize, ...)`; smaller) is refused with MXB_ERR_INVALID, and the
    transform carries on."""
    exe = compile_patch(bindir, SRC_BLOCK)
    C, hop, bins = 3, fft_size // 2, fft_size // 2
    N = 12 * hop + 50
    x = W.channel_streams(C, N, seed=fft_size + 1)
    x[1] = 0.0                                                      # a silent channel
    x.tofile(tmp_path / "in.bin")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(C), str(N), str(fft_size)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = open(tmp_path / "out.bin", "rb").read()
    F, nA, code_big, code_small, after = (int(v) for v in np.frombuffer(raw, dtype=np.int32, count=5)); off = 20

    def take(dtype, shape):
        nonlocal off
        n = int(np.prod(shape)); a = np.frombuffer(raw, dtype=dtype, count=n, offset=off).reshape(shape)
        off += a.nbytes
        return a
    mags, avs, pks = take(np.float32, (C, F, bins)), take(np.float32, (C, F, nA)), take(np.float32, (C, F, nA))
    spec, rel, tot = take(np.float64, (C, F, 24)), take(np.float64, (C, F, 24)), take(np.float64, (C, F))
    assert off == len(raw)
    assert code_big == -1 and code_small == -1 and after == 2           # MXB_ERR_INVALID
    o = port.Stft(C, fft_size, hop).process(x)
    assert F == o["mags"].shape[1] and np.array_equal(mags, o["mags"])
    ooc = port.Octave(C, 48000, bins, 6); ooc.config(3, 0.85, 1.1, 0.002)
    assert ooc.n_averages == nA
    oav, opk = ooc.process(o["mags"])
    assert np.array_equal(avs, oav, equal_nan=True) and np.array_equal(pks, opk, equal_nan=True)
    sp, rl, tt = port.bark(o["mags"], 48000, fft_size)
    for got, exp in ((spec, sp), (rel, rl), (tot, tt)):
        assert np.array_equal(np.isnan(got), np.isnan(exp))
        np.testing.assert_allclose(got, exp, rtol=1e-12, atol=0)
    assert np.isnan(rel[1]).all() and np.abs(avs[0]).max() > 0
