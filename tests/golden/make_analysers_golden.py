"""Generates tests/golden/analysers.npz from the UNMODIFIED reference (oracle/_ref/libmaxiref.so, built by oracle/Makefile): the
reference's maxiFFTOctaveAnalyzer::calculate and maxiBark (specificLoudness / relativeLoudness / totalLoudness) on spectra of every
size the stand-alone analysers take, including silent frames, NaN, inf and negative bins. Inputs are stored beside the outputs. Run
where the reference is built:

    python tests/golden/make_analysers_golden.py

  octave  n_bands 64 .. 1024 x 1 / 3 / 6 / 12 per octave x 44.1 / 48 kHz, 2 channels x 6 consecutive frames in one call, peak hold 3,
          decay 0.85, linear EQ 0.9 + b * 0.5 / n_bands
  bark    buffer sizes 128 .. 4096 x 22.05 / 44.1 / 48 / 96 kHz, 5 frames
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import oracle_py as O          # noqa: E402

OCT_BANDS = (64, 128, 256, 512, 1024)
OCT_PER_OCTAVE = (1, 3, 6, 12)
OCT_RATES = (44100, 48000)
OCT_C, OCT_F = 2, 6
OCT_HOLD, OCT_DECAY, OCT_ICPT = 3, 0.85, 0.9
BARK_SIZES = (128, 256, 512, 1024, 2048, 4096)
BARK_RATES = (22050, 44100, 48000, 96000)
BARK_F = 5


def oct_slope(n_bands):
    return 0.5 / n_bands


def octave_mags(n_bands, seed):
    """[C][F][n_bands]: magnitude-like values; channel 1 frame 2 silent, channel 0 frame 3 with NaN and inf bins, channel 1 frame 4 with
    a negative bin and an inf."""
    r = np.random.default_rng(seed)
    m = (r.exponential(1.0, (OCT_C, OCT_F, n_bands)) * np.linspace(4.0, 0.2, n_bands)).astype(np.float32)
    m[1, 2] = 0.0
    m[0, 3, n_bands // 3] = np.nan; m[0, 3, n_bands - 2] = np.inf
    m[1, 4, 5] = -3.0; m[1, 4, n_bands // 2] = np.inf
    return m


def bark_spectra(buffer_size, seed):
    """[F][buffer_size / 2]: frame 1 silent, frame 2 NaN and inf bins, frame 3 negative bins, frame 4 an inf."""
    r = np.random.default_rng(seed)
    spec = buffer_size // 2
    s = (r.exponential(0.05, (BARK_F, spec)) * np.linspace(2.0, 0.1, spec)).astype(np.float32)
    s[1] = 0.0
    s[2, spec // 5] = np.nan; s[2, spec // 2] = np.inf
    s[3, 1::7] *= -1.0
    s[4, spec // 3] = np.inf
    return s


def main():
    O.build("reference")
    out = {}
    for nb in OCT_BANDS:
        m = octave_mags(nb, seed=nb)
        out[f"oct/{nb}/mags"] = m
        for po in OCT_PER_OCTAVE:
            for sr in OCT_RATES:
                o = O.Octave(OCT_C, sr, nb, po, kind="reference")
                o.config(OCT_HOLD, OCT_DECAY, OCT_ICPT, oct_slope(nb))
                av, pk = o.process(m)
                out[f"oct/{nb}/{po}/{sr}/averages"] = av
                out[f"oct/{nb}/{po}/{sr}/peaks"] = pk
    for bs in BARK_SIZES:
        s = bark_spectra(bs, seed=bs + 1)
        out[f"bark/{bs}/spectrum"] = s
        for sr in BARK_RATES:
            sp, rl, tt = O.bark(s, sr, bs, kind="reference")
            out[f"bark/{bs}/{sr}/specific"] = sp
            out[f"bark/{bs}/{sr}/relative"] = rl
            out[f"bark/{bs}/{sr}/total"] = tt
    np.savez_compressed(os.path.join(HERE, "analysers.npz"), **out)


if __name__ == "__main__":
    main()
