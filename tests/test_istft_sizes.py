"""tests/golden/istft_sizes.npz (the compiled reference's maxiIFFT at 2048 points and at hops that do not divide the frame, written by
tests/golden/make_istft_golden.py) replayed through the plain-C port: bit for bit, NaN included, in the same ragged calls. The GPU tests
(test_gpu_istft_sizes.py) compare the device resynthesis with this port and with the file. The per-sample C++ program they run compiles
against the drop-in header here."""
import importlib.util
import os
import subprocess

import numpy as np
import pytest

import golden_checks as G


def _maker():
    spec = importlib.util.spec_from_file_location("make_istft_golden", os.path.join(G.GOLD, "make_istft_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


M = _maker()


@pytest.mark.parametrize("n,hop", M.PAIRS)
def test_istft_port_replays_reference(port, n, hop):
    g = G.load("istft_sizes")
    y = M.resynthesise(port.Istft(M.C, n, hop, kind="port"), g[f"{n}/mags"], g[f"{n}/phases"])
    ref = g[f"{n}/{hop}/out"]
    assert y.shape == ref.shape == (M.C, M.F * hop)
    assert np.array_equal(y, ref, equal_nan=True), (n, hop)
    assert np.isnan(ref[1]).any() and not np.isnan(ref[[0, 2]]).any()      # the NaN frame reached the output of its channel only


def test_resynthesis_sizes_program_compiles_against_the_dropin_header(tmp_path):
    from test_cpp_dropin import compile_patch
    exe = compile_patch(tmp_path, os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "resynth_sizes.cpp"))
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr
