"""16.Replicant's play() through the C++ layer with its control values as maxiEvents (tests/cpp/patch_events.cpp): it compiles against
include/maximilian_b200.hpp (CPU check) and, on the GPU, the events run gives the same bits as the same program fed dense maxiStreams,
in both ways a patch runs, and both match the port running the same graph on the dense streams."""
import os
import subprocess

import numpy as np
import pytest

from patch_checks import set_tables
from test_cpp_dropin import ROOT, compile_patch
import golden_checks as G
from maximilian_b200.patchdef import PatchDef, R

SRC = os.path.join(ROOT, "tests", "cpp", "patch_events.cpp")


@pytest.fixture(scope="module")
def bindir(tmp_path_factory):
    return tmp_path_factory.mktemp("events")


def replicant():
    """the graph Replicant::play records (inputs: currentPitch, leadPitch, trigger, trigger2), stage for stage"""
    d = PatchDef()
    cp, lp = d.IN("currentPitch"), d.IN("leadPitch")
    d.stage("mul", cp, d.K(0.5), dst=R(0))                                              # half = cp * 0.5
    d.stage("osc", R(0), kind="saw", dst=R(1))                                          # bass.saw(half)
    d.stage("osc", d.K(1.0), kind="phasor", dst=R(2))                                   # mod.phasor(1)
    d.stage("osc", R(0), R(2), kind="pulse", dst=R(3))                                  # sound.pulse(half, m)
    d.stage("add", R(1), R(3), dst=R(4))
    d.stage("env_adsr", R(4), d.IN("trigger"), d.K(1.0), d.K(0.9995), d.K(0.25), d.K(0.9995), d.K(1.0), dst=R(5))
    d.stage("filter", R(5), d.K(9250.0), d.K(2.0), kind="lores", dst=R(6))             # bassout
    d.stage("mul", lp, d.K(4.0), dst=R(7))
    d.stage("osc", R(7), kind="saw", dst=R(8))                                          # lead2.saw(lp * 4)
    d.stage("osc", d.K(1.9), kind="sinebuf", dst=R(9))                                  # leadmod.sinebuf(1.9)
    d.stage("mul", R(9), d.K(1.5), dst=R(10))
    d.stage("add", lp, R(10), dst=R(11))
    d.stage("osc", R(11), d.K(0.6), kind="pulse", dst=R(12))                            # lead.pulse(lp + lm * 1.5, 0.6)
    d.stage("add", R(8), R(12), dst=R(13))
    d.stage("env_ar", R(13), d.IN("trigger2"), d.K(0.00005), d.K(0.999975), d.K(50000.0), dst=R(14))
    d.stage("filter", R(14), d.K(5900.0), d.K(10.0), kind="lores", dst=R(15))          # leadout
    d.stage("out", R(6))
    d.stage("mix_stereo", R(15), d.K(0.5))
    return d


def test_events_port_compiles_against_the_dropin_header(bindir):
    exe = compile_patch(bindir, SRC)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fused", "interpret"])
def test_events_equal_dense_streams_and_the_port(port, tmp_path, bindir, mode):
    """40 voices at tempos from 9 to 106.5 ticks per second, 24 blocks of 1000 frames at 44.1 kHz: every tick is an event of currentPitch and
    two of trigger (1, then 0 on the next sample, across block edges too), some ticks move leadPitch and trigger2. The events run equals the
    dense run bit for bit; both match the port within 1e-9 of the peak (lores designs libdevice tan / cos on the GPU, glibc in the port)."""
    exe = compile_patch(bindir, SRC)
    V, NB, B = 40, 24, 1000
    g = G.load("tables")
    np.concatenate([g["sine"], g["transition"], [float(g["sine_before"])]]).astype(np.float64).tofile(tmp_path / "tables.bin")
    r = subprocess.run([exe, str(tmp_path / "tables.bin"), str(tmp_path / "out.bin"), str(V), str(NB), str(B)], capture_output=True, text=True,
                       env=dict(os.environ, MXB_PATCH_MODE=mode))
    assert r.returncode == 0, r.stderr
    T = NB * B
    x = np.fromfile(tmp_path / "out.bin", dtype=np.float64)
    sizes = [T * V] * 4 + [T * V, T * 2, T * V, T * 2]
    assert x.size == sum(sizes)
    parts = np.split(x, np.cumsum(sizes)[:-1])
    cp, lp, tr, tr2 = (a.reshape(T, V) for a in parts[:4])
    out_e, bus_e, out_d, bus_d = parts[4].reshape(T, V), parts[5].reshape(T, 2), parts[6].reshape(T, V), parts[7].reshape(T, 2)
    assert np.array_equal(out_e, out_d) and np.array_equal(bus_e, bus_d), "events and dense streams differ"
    assert (np.diff(tr, axis=0) > 0).sum() > 10 * V and (np.diff(lp, axis=0) != 0).sum() > V      # the control code did move them
    set_tables(port)
    o = port.Patch(replicant(), V, sample_rate=44100, kind="port")
    oo, mo = o.process(T, {"currentPitch": cp, "leadPitch": lp, "trigger": tr, "trigger2": tr2}, want_mix=True)
    peak = np.abs(oo).max()
    assert peak > 1e-2
    np.testing.assert_allclose(out_e, oo / 2, rtol=1e-9, atol=1e-9 * peak)
    np.testing.assert_allclose(bus_e, mo, rtol=1e-9, atol=1e-9 * np.abs(mo).max())
