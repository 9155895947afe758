"""Generates tests/golden/istft_sizes.npz from the UNMODIFIED reference (oracle/_ref/libmaxiref.so, built by oracle/Makefile): the
reference's maxiIFFT::process (SPECTRUM) at 2048 points and at hops that do not divide the frame, next to a few sizes the resynthesis
already took. Inputs are stored beside the outputs. Run where the reference is built:

    python tests/golden/make_istft_golden.py

  spectra  per fft size n: the reference's maxiFFT (at max(n, 128) points, hop n / 2, the first n / 2 bins kept) of
           workloads.channel_streams, 3 channels x 8 frames; channel 1 frame 4 has a NaN magnitude, channel 2 frame 2 is silent
  pairs    (n, hop) in PAIRS, each fed in the ragged calls of CALLS (1 frame, 2 frames, the rest) so that the carried buffer is used
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from maximilian_b200 import workloads as W  # noqa: E402
from oracle import oracle_py as O          # noqa: E402

PAIRS = ((2048, 1024), (2048, 441), (2048, 2048), (2048, 1), (1024, 441), (1024, 1023), (512, 100), (64, 48))
C, F = 3, 8
CALLS = ((0, 1), (1, 3), (3, F))


def spectra(n, kind="reference"):
    """(mags, phases) float32 [C][F][n / 2]."""
    fwd = max(n, 128)
    x = W.channel_streams(C, (F + 1) * (fwd // 2), seed=n)
    r = O.Stft(C, fwd, fwd // 2, kind=kind).process(x, want=("mags", "phases"))
    mags = np.ascontiguousarray(r["mags"][:, :F, :n // 2])
    phases = np.ascontiguousarray(r["phases"][:, :F, :n // 2])
    assert mags.shape == (C, F, n // 2)
    mags[1, 4, n // 8] = np.nan
    mags[2, 2] = 0.0
    phases[2, 2] = 0.0
    return mags, phases


def resynthesise(istft, mags, phases):
    """The calls of CALLS on one maxiIFFT object per channel: float32 [C][F * hop]."""
    return np.concatenate([istft.process(mags[:, lo:hi], phases[:, lo:hi]) for lo, hi in CALLS], axis=1)


def main():
    O.build("reference")
    out = {}
    for n in sorted({n for n, _ in PAIRS}):
        out[f"{n}/mags"], out[f"{n}/phases"] = spectra(n)
    for n, hop in PAIRS:
        out[f"{n}/{hop}/out"] = resynthesise(O.Istft(C, n, hop, kind="reference"), out[f"{n}/mags"], out[f"{n}/phases"])
    np.savez_compressed(os.path.join(HERE, "istft_sizes.npz"), **out)


if __name__ == "__main__":
    main()
