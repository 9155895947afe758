"""9.Envelopes2 through the C++ layer (tests/cpp/patch_envelopes.cpp): three maxiEnvGen objects, each with its own setup(), in one play().
It compiles against include/maximilian_b200.hpp (CPU check) and, on the GPU, its output equals the C oracle running the same graph with
the three shapes (tests/envgen_cases.py), in both ways a patch runs."""
import os
import subprocess

import numpy as np
import pytest

import envgen_cases as EC
from test_cpp_dropin import ROOT, compile_patch

SRC = os.path.join(ROOT, "tests", "cpp", "patch_envelopes.cpp")


@pytest.fixture(scope="module")
def bindir(tmp_path_factory):
    return tmp_path_factory.mktemp("envelopes")


def test_envelopes_port_compiles_against_the_dropin_header(bindir):
    exe = compile_patch(bindir, SRC)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fused", "interpret"])
def test_envelopes_port_matches_oracle(port, tmp_path, bindir, mode):
    """2.5 s of the example at 44.1 kHz: the slow envelope widens the 1 Hz pulse, whose edges start and end the HOLD of the amp envelope,
    while the third envelope sweeps the lowpass from 2 kHz down. 1e-9 of the signal's peak (maxiEnvGen curves and the biquad design run
    libdevice pow / tan on the GPU, glibc in the oracle)."""
    exe = compile_patch(bindir, SRC)
    NB, B, V = 108, 1024, 2
    env = dict(os.environ, MXB_PATCH_MODE=mode)
    r = subprocess.run([exe, str(tmp_path / "out.bin"), str(NB), str(B)], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    out = np.fromfile(tmp_path / "out.bin", dtype=np.float64).reshape(NB * B, V)
    o = port.Patch(EC.envelopes2(), V, sample_rate=44100, kind="port")
    oo, _ = o.process(NB * B)
    peak = np.abs(oo).max()
    assert peak > 1e-2
    np.testing.assert_allclose(out, oo, rtol=1e-9, atol=1e-9 * peak)
    assert np.array_equal(out[:, 0], out[:, 1])
    # the silent failure this guards against: every maxiEnvGen playing the shape of the last setup() (myEnv3) sounds far from it
    d = EC.envelopes2()
    d.stages = [(op, 2 if op == 4 else k, dst, src) for op, k, dst, src in d.stages]
    ow, _ = port.Patch(d, V, sample_rate=44100, kind="port").process(NB * B)
    assert np.abs(ow - out).max() > 0.1 * peak
