"""tests/golden/analysers.npz (the compiled reference's maxiFFTOctaveAnalyzer and maxiBark on spectra of every size the stand-alone
analysers take, written by tests/golden/make_analysers_golden.py) replayed through the plain-C port: bit for bit, NaN included. The GPU
tests compare the device analysers with this port."""
import importlib.util
import os

import numpy as np
import pytest

import golden_checks as G


def _maker():
    spec = importlib.util.spec_from_file_location("make_analysers_golden", os.path.join(G.GOLD, "make_analysers_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


M = _maker()


@pytest.mark.parametrize("n_bands", M.OCT_BANDS)
def test_octave_port_replays_reference(port, n_bands):
    g = G.load("analysers")
    mags = g[f"oct/{n_bands}/mags"]
    for po in M.OCT_PER_OCTAVE:
        for sr in M.OCT_RATES:
            o = port.Octave(M.OCT_C, sr, n_bands, po, kind="port")
            o.config(M.OCT_HOLD, M.OCT_DECAY, M.OCT_ICPT, M.oct_slope(n_bands))
            av, pk = o.process(mags)
            assert np.array_equal(av, g[f"oct/{n_bands}/{po}/{sr}/averages"], equal_nan=True), (n_bands, po, sr)
            assert np.array_equal(pk, g[f"oct/{n_bands}/{po}/{sr}/peaks"], equal_nan=True), (n_bands, po, sr)


@pytest.mark.parametrize("buffer_size", M.BARK_SIZES)
def test_bark_port_replays_reference(port, buffer_size):
    g = G.load("analysers")
    s = g[f"bark/{buffer_size}/spectrum"]
    for sr in M.BARK_RATES:
        sp, rl, tt = port.bark(s, sr, buffer_size, kind="port")
        for name, a in (("specific", sp), ("relative", rl), ("total", tt)):
            assert np.array_equal(a, g[f"bark/{buffer_size}/{sr}/{name}"], equal_nan=True), (buffer_size, sr, name)
