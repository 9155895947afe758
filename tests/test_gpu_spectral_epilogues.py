"""The transform's fused epilogues -- MFCC, dB / flatness / centroid, octave analyser, Bark -- at the sizes, shapes and schedules
they accept, against the CPU oracle fed the same samples over several calls (carried state used, ragged first cuts).

Bars (DESIGN.md section 2): magnitudes bit for bit; MFCC 1e-9 relative + 1e-12; octave averages / peaks bit for bit; Bark 1e-12
relative; dB 2e-6; flatness / centroid 1e-4.

  A  the r01 kernel (stft_kernel<P>: fft sizes 128, 256, 512, 2048) with its fused MFCC in both variants (compact row: MFCC only;
     padded: spectra written), with dB / flatness / centroid, a silent channel, 9 channels (not a multiple of a CTA's 8 warps)
  B  the 1024-point streaming kernel's tensor-core MFCC (K4s) across bank shapes, MFCC-only and spectra-written
  C  octave analyser configurations that wrap the 32-lane loops, Bark at 44.1 kHz
  D  every output in one call on the sliced host pipeline
  E  device-memory inputs and outputs (planar and time-major), odd hops
  F  non-finite magnitudes (the reference's band sum runs over every bin: 0 * NaN and 0 * inf poison a band)
  G  fused MFCC tables beyond the device's shared memory: MXB_ERR_UNSUPPORTED, handle still usable
"""
import ctypes as C

import numpy as np
import pytest

from maximilian_b200 import capi
from maximilian_b200 import workloads as W

pytestmark = pytest.mark.gpu

ERR_UNSUPPORTED = -4


# ---------------------------------------------------------------------------------------------------------------- helpers

def _ptr(a):
    return None if a is None else a.ctypes.data


def run3(st, x, mags=True, feats=False, mfcc=None, octave=None, bark=False):
    """One mxb_stft_process3 call on planar host samples with any set of outputs -> dict of the frames that fired."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    nch, N = x.shape
    maxf = max(1, N // st.hop + 2)
    z = lambda *s: np.zeros(s, dtype=np.float32)                       # noqa: E731
    out = dict(mags=z(nch, maxf, st.bins) if mags else None,
               mags_db=z(nch, maxf, st.bins) if feats else None,
               flatness=z(nch, maxf) if feats else None, centroid=z(nch, maxf) if feats else None,
               mfcc=np.zeros((nch, maxf, mfcc.coeffs)) if mfcc is not None else None,
               averages=z(nch, maxf, octave.n_averages) if octave is not None else None,
               peaks=z(nch, maxf, octave.n_averages) if octave is not None else None,
               bark_specific=np.zeros((nch, maxf, 24)) if bark else None, bark_relative=np.zeros((nch, maxf, 24)) if bark else None,
               bark_total=np.zeros((nch, maxf)) if bark else None)
    o = capi.StftOutputs(_ptr(out["mags"]), None, None, None, _ptr(out["mags_db"]), _ptr(out["flatness"]), _ptr(out["centroid"]),
                         _ptr(out["mfcc"]))
    post = None
    if octave is not None or bark:
        post = capi.StftPost(octave.h if octave is not None else None, _ptr(out["averages"]), _ptr(out["peaks"]), 1 if bark else 0,
                             _ptr(out["bark_specific"]), _ptr(out["bark_relative"]), _ptr(out["bark_total"]))
    nf = C.c_int32(0)
    capi.check(capi.lib().mxb_stft_process3(st.h, x.ctypes.data, N, 1, N, maxf, C.byref(o), C.byref(post) if post is not None else None,
                                            mfcc.h if mfcc is not None else None, C.byref(nf), capi.MEM_HOST, None), "mxb_stft_process3")
    return {k: np.ascontiguousarray(v[:, :nf.value]) for k, v in out.items() if v is not None}


def expected(port, om, n, sr, omf=None, feats=False, ooc=None, bark=False):
    """The oracle's epilogues of the oracle's magnitudes om [C][F][bins]."""
    e = dict(mags=om)
    if omf is not None:
        e["mfcc"], e["melbands"] = omf.process(om)
    if feats:
        e["mags_db"], e["flatness"], e["centroid"] = port.spectral_features(om, n, sr)
    if ooc is not None:
        e["averages"], e["peaks"] = ooc.process(om)
    if bark:
        e["bark_specific"], e["bark_relative"], e["bark_total"] = port.bark(om, sr, n)
    return e


def mfcc_atol(e):
    """1e-12, or for big banks 1e-12 of the DCT's term scale sum_j |dct_ij * mel_j| / numCoeffs (|dct_ij| <= sqrt(2 / filters)):
    a coefficient that cancels to near 0 keeps the fp64 reassociation error of its terms. The relative bar stays 1e-9."""
    mel = e["melbands"]
    nfil, nc = mel.shape[-1], e["mfcc"].shape[-1]
    if nfil < 256:
        return 1e-12
    return 1e-12 * max(1.0, float(np.sqrt(2.0 / nfil) * np.abs(mel).sum(axis=-1).max() / nc))


def check(r, e, what, keys=None):
    """Every output of r that e has, at its bar."""
    for k in keys or r:
        if k not in e:
            continue
        g, o = r[k], e[k]
        assert g.shape == o.shape, (what, k, g.shape, o.shape)
        if g.size == 0:
            continue
        if k in ("mags", "averages", "peaks"):
            assert np.array_equal(g, o, equal_nan=True), (what, k, np.nanmax(np.abs(g - o)))
        elif k == "mfcc":
            np.testing.assert_allclose(g, o, rtol=1e-9, atol=mfcc_atol(e), equal_nan=True, err_msg=f"{what} {k}")
        elif k == "mags_db":
            np.testing.assert_allclose(g, o, rtol=2e-6, atol=1e-6, err_msg=f"{what} {k}")
        elif k == "flatness":
            np.testing.assert_allclose(g, o, rtol=1e-4, atol=1e-7, err_msg=f"{what} {k}")
        elif k == "centroid":
            np.testing.assert_allclose(g, o, rtol=1e-4, atol=1e-3, err_msg=f"{what} {k}")
        elif k == "bark_relative":                                     # 0 / 0 on a silent frame, like the reference
            assert np.array_equal(np.isnan(g), np.isnan(o)), what
            np.testing.assert_allclose(np.nan_to_num(g), np.nan_to_num(o), rtol=1e-12, atol=0, err_msg=f"{what} {k}")
        elif k.startswith("bark"):
            np.testing.assert_allclose(g, o, rtol=1e-12, atol=0, err_msg=f"{what} {k}")


def same_bits(r, s, what):
    for k in s:
        assert np.array_equal(r[k], s[k], equal_nan=True), (what, k)


def slices(total, cuts):
    cuts = [0] + list(cuts) + [total]
    return list(zip(cuts[:-1], cuts[1:]))


# ------------------------------------------------------------------------------------ A. the r01 kernel (128 / 256 / 512 / 2048)

R01 = [(128, 64, (64, 16, 13, 20.0, 20000.0, 48000)), (256, 96, (128, 26, 13, 20.0, 20000.0, 44100)),
       (512, 256, (256, 20, 12, 100.0, 8000.0, 48000)), (2048, 512, (1024, 42, 40, 20.0, 20000.0, 48000))]


@pytest.mark.parametrize("n,hop,cfg", R01, ids=[str(c[0]) for c in R01])
def test_r01_fused_mfcc_and_features(port, n, hop, cfg):
    """stft_kernel<P> with its epilogues: MFCC only (compact magnitude row), MFCC with magnitudes written (padded spectrum), and
    MFCC + dB + flatness + centroid in one call, on 9 channels with a silent one, over three calls with a 3-sample first cut.
    Both MFCC variants give the same bits (same sums, same tensor-core DCT) and equal the standalone mxb_mfcc_process on the
    returned magnitudes to fp64 reassociation."""
    bins, nfil, nc, fmin, fmax, sr = cfg
    nch = 9
    x = W.channel_streams(nch, 6 * n + 37, seed=n)
    x[1] *= 100.0
    x[4] = 0.0                                                          # silent: MFCCs, flatness and centroid are 0
    mf = capi.Mfcc(bins, nfil, nc, fmin, fmax, sample_rate=sr)
    omf = port.Mfcc(bins, nfil, nc, fmin, fmax, sr)
    compact, padded, feat = (capi.Stft(nch, n, hop, sample_rate=sr) for _ in range(3))
    ost = port.Stft(nch, n, hop)
    fired = 0
    for lo, hi in slices(x.shape[1], (3, 2 * n + hop // 2 + 1)):
        xs = x[:, lo:hi]
        e = expected(port, ost.process(xs, want=("mags",))["mags"], n, sr, omf=omf, feats=True)
        rc = run3(compact, xs, mags=False, mfcc=mf)
        rp = run3(padded, xs, mfcc=mf)
        rf = run3(feat, xs, feats=True, mfcc=mf)
        check(rc, e, ("compact", lo)); check(rp, e, ("padded", lo)); check(rf, e, ("features", lo))
        assert np.array_equal(rc["mfcc"], rp["mfcc"]) and np.array_equal(rp["mfcc"], rf["mfcc"]), lo
        fired += e["mags"].shape[1]
        if e["mags"].shape[1]:
            cs, _ = mf.process(rp["mags"])
            np.testing.assert_allclose(cs, rp["mfcc"], rtol=1e-12, atol=1e-13)
            assert np.all(rf["mfcc"][4] == 0.0) and np.all(rf["flatness"][4] == 0.0) and np.all(rf["centroid"][4] == 0.0)
    assert fired >= 4


# ------------------------------------------------------------------------------------ B. K4s tensor-core MFCC across bank shapes

# Layouts of mxb_mfcc_create's mel tiles at 512 bins (1024-point frames), computed from its tile code:
#
# | filters, coeffs, fmin-fmax, sr     | mel tiles (&3) | branch                                                    |
# |------------------------------------|----------------|-----------------------------------------------------------|
# | 42, 13, 20-20000, 44100 (pinned)   | 6 (2)          | halves, 13 coeffs: partial DCT tile                       |
# | 40, 13, 20-20000, 48000            | 5 (1)          | halves, one tile                                          |
# | 32, 32, 20-20000, 48000            | 4 (0)          | no halves                                                 |
# | 24, 30, 300-24000, 48000           | 3 (3)          | warp 3 has no mel tile; coeffs > filters                  |
# | 3, 5, 20-20000, 48000              | 1 (1)          | fewer filters than a tile                                 |
# | 1, 1, 20-20000, 48000              | 1 (1)          | empty bank (maxbin 0), every band 0                       |
# | 26, 13, 2000-8000, 16000           | 4 (0)          | maxbin 260 > 256: MFCC-only call forced onto FULL = true  |
# | 64, 20, 0-24000, 48000             | 8 (0)          | maxbin exactly 256: stays FULL = false                    |
# | 256, 13, 20-20000, 48000 (pinned)  | 32 (0)         | 149 KB shared memory                                      |
# | 520, 13, 20-20000, 48000           | 65 (1)         | 217 KB, the last shape that fits; one CTA per SM          |
# | 600, 13, 20-20000, 48000           | -              | 237 KB: MXB_ERR_UNSUPPORTED                               |
K4S = [(42, 13, 20.0, 20000.0, 44100), (40, 13, 20.0, 20000.0, 48000), (32, 32, 20.0, 20000.0, 48000), (24, 30, 300.0, 24000.0, 48000),
       (3, 5, 20.0, 20000.0, 48000), (1, 1, 20.0, 20000.0, 48000), (26, 13, 2000.0, 8000.0, 16000), (64, 20, 0.0, 24000.0, 48000),
       (256, 13, 20.0, 20000.0, 48000), (520, 13, 20.0, 20000.0, 48000)]


@pytest.mark.parametrize("shape", K4S, ids=[f"{s[0]}x{s[1]}@{s[4]}" for s in K4S])
def test_stream_kernel_mfcc_shapes(port, shape):
    """The packed two-channel kernel's fused MFCC at every bank shape of the table above, MFCC-only and with magnitudes written,
    7 channels (a pair with one channel) and a silent one, three calls with a ragged first cut; the coefficients also equal the
    standalone kernel's on the oracle's magnitudes to fp64 reassociation (sequential vs tensor-core mel sums)."""
    nfil, nc, fmin, fmax, sr = shape
    nch, n, hop = 7, 1024, 512
    x = W.channel_streams(nch, 9 * hop + 100, seed=nfil)
    x[3] = 0.0
    mf = capi.Mfcc(512, nfil, nc, fmin, fmax, sample_rate=sr)
    omf = port.Mfcc(512, nfil, nc, fmin, fmax, sr)
    only, spectra = capi.Stft(nch, n, hop, sample_rate=sr), capi.Stft(nch, n, hop, sample_rate=sr)
    ost = port.Stft(nch, n, hop)
    for lo, hi in slices(x.shape[1], (3 * hop + 5, 4 * hop + 5)):
        xs = x[:, lo:hi]
        e = expected(port, ost.process(xs, want=("mags",))["mags"], n, sr, omf=omf)
        ra = only.process(xs, want=(), mfcc=mf)
        rb = spectra.process(xs, want=("mags",), mfcc=mf)
        check(ra, e, ("mfcc only", lo)); check(rb, e, ("spectra", lo))
        cs, _ = mf.process(e["mags"])
        np.testing.assert_allclose(cs, rb["mfcc"], rtol=1e-12, atol=1e-13 * max(1.0, mfcc_atol(e) / 1e-12))
        assert np.all(ra["mfcc"][3] == 0.0)
        if nfil == 1:
            assert np.all(ra["mfcc"] == 0.0)                              # filter 0 has no weights: every band 0


def test_stream_kernel_refuses_a_bank_beyond_shared_memory(port):
    """600 filters need 237 KB of shared memory in the fused kernel: MXB_ERR_UNSUPPORTED before any launch, and the stream stays
    where it was -- the next call, without the MFCC, continues the oracle's frame schedule exactly."""
    nch, n, hop = 5, 1024, 512
    x = W.channel_streams(nch, 5000, seed=600)
    st, ost = capi.Stft(nch, n, hop), port.Stft(nch, n, hop)
    big = capi.Mfcc(512, 600, 13, 20.0, 20000.0)
    assert np.array_equal(st.process(x[:, :1000], want=("mags",))["mags"], ost.process(x[:, :1000], want=("mags",))["mags"])
    for want in ((), ("mags",)):
        with pytest.raises(capi.MxbError, match=f"-> {ERR_UNSUPPORTED}:"):
            st.process(x[:, 1000:2500], want=want, mfcc=big)
    r, ro = st.process(x[:, 1000:], want=("mags",)), ost.process(x[:, 1000:], want=("mags",))
    assert r["mags"].shape == ro["mags"].shape and np.array_equal(r["mags"], ro["mags"])


# ------------------------------------------------------------------------------------------------ C. octave analyser and Bark

@pytest.mark.parametrize("per_octave,sr", [(1, 48000), (6, 48000), (3, 44100), (12, 48000)])
def test_octave_and_bark_configs(port, per_octave, sr):
    """maxiFFTOctaveAnalyzer at configurations beyond the default (6 and 12 per octave: more than 32 bands and runs, the lane loops
    wrap), with a peak hold longer than one call so that hold counters cross calls; Bark on a transform whose context runs at `sr`."""
    nch, n, hop = 5, 1024, 512
    x = W.channel_streams(nch, 14 * hop + 77, seed=per_octave)
    x[2] = 0.0
    x[4, 6 * hop:] *= 0.05                                               # a drop in level: peaks decay after their hold
    st = capi.Stft(nch, n, hop, sample_rate=sr)
    oc, ooc = capi.Octave(nch, sr, 512, per_octave), port.Octave(nch, sr, 512, per_octave)
    assert oc.n_averages == ooc.n_averages
    if per_octave >= 6:
        assert oc.n_averages > 32
    oc.config(6, 0.7, 0.5, 0.02); ooc.config(6, 0.7, 0.5, 0.02)
    ost = port.Stft(nch, n, hop)
    for lo, hi in slices(x.shape[1], (4 * hop + 3, 9 * hop)):
        xs = x[:, lo:hi]
        e = expected(port, ost.process(xs, want=("mags",))["mags"], n, sr, ooc=ooc, bark=True)
        check(run3(st, xs, octave=oc, bark=True), e, (per_octave, sr, lo))


# ------------------------------------------------------------------------------------------------------ D. everything at once

def test_everything_in_one_sliced_call(port):
    """mags, dB, flatness, centroid, octave, Bark and a fused MFCC (13 coefficients, 44.1 kHz) in ONE mxb_stft_process3 call on 1030
    channels x 4096 samples: the 4-slice host pipeline (slices of 257 / 258 channels), two calls, so octave peaks and hold counters
    cross slice and call boundaries. 96 channels (first, last, both sides of each slice boundary, random) against the oracle; every
    channel bit for bit against the same transform asked for fewer outputs."""
    nch, n, hop, N, sr = 1030, 1024, 512, 4096, 44100
    rng = np.random.default_rng(1030)
    x = W.channel_streams(nch, 2 * N, seed=41)
    x[513] = 0.0
    edges = [c for b in (257, 515, 772) for c in (b - 2, b - 1, b, b + 1)]
    rest = np.setdiff1d(np.arange(16, nch - 16), edges)
    pick = np.sort(np.concatenate([np.arange(16), np.arange(nch - 16, nch), edges, rng.choice(rest, 96 - 44, replace=False)]))
    assert pick.size == 96 and np.unique(pick).size == 96
    mf = capi.Mfcc(512, 42, 13, 20.0, 20000.0, sample_rate=sr)
    omf = port.Mfcc(512, 42, 13, 20.0, 20000.0, sr)
    octs = [capi.Octave(nch, sr, 512, 6) for _ in range(2)]
    ooc = port.Octave(pick.size, sr, 512, 6)
    for o in octs + [ooc]:
        o.config(10, 0.8, 1.0, 0.01)
    everything, mags_mfcc, features, post = (capi.Stft(nch, n, hop, sample_rate=sr) for _ in range(4))
    ost = port.Stft(pick.size, n, hop)
    for lo, hi in ((0, N), (N, 2 * N)):
        xs = x[:, lo:hi]
        r = run3(everything, xs, feats=True, mfcc=mf, octave=octs[0], bark=True)
        assert r["mags"].shape == (nch, N // hop, 512)
        e = expected(port, ost.process(xs[pick], want=("mags",))["mags"], n, sr, omf=omf, feats=True, ooc=ooc, bark=True)
        check({k: v[pick] for k, v in r.items()}, e, ("oracle", lo))
        same_bits(r, run3(mags_mfcc, xs, mfcc=mf), ("mags + mfcc", lo))
        same_bits(r, run3(features, xs, feats=True), ("features", lo))
        same_bits(r, run3(post, xs, octave=octs[1], bark=True), ("octave + bark", lo))


# ------------------------------------------------------------------------------------------ E. device memory and odd hops

DEV_MFCC = {512: (256, 20, 12, 100.0, 8000.0, 48000), 1024: (512, 42, 40, 20.0, 20000.0, 48000)}


@pytest.mark.parametrize("layout", ["planar", "time_major"])
@pytest.mark.parametrize("n", [512, 1024])
def test_device_memory_matches_host_and_oracle(port, n, layout):
    """MXB_MEM_DEVICE input and outputs (torch tensors): mxb_stft_process2 with magnitudes, features and MFCC, and mxb_stft_process with
    MFCC alone, fed planar or time-major samples (stride_c = 1, stride_t = C) in ragged calls: bit for bit the host path, and the
    oracle's values."""
    import torch
    dev = torch.device("cuda:0")
    nch, hop = 12, n // 2
    bins, nfil, nc, fmin, fmax, sr = DEV_MFCC[n]
    x = W.channel_streams(nch, 6 * n + 37, seed=n + 7)
    mf = capi.Mfcc(bins, nfil, nc, fmin, fmax, sample_rate=sr)
    omf = port.Mfcc(bins, nfil, nc, fmin, fmax, sr)
    d_full, d_only, h_full, h_only = (capi.Stft(nch, n, hop, sample_rate=sr) for _ in range(4))
    ost = port.Stft(nch, n, hop)
    for lo, hi in slices(x.shape[1], (3, hop + 5, 4 * n + 1)):
        xs = x[:, lo:hi]
        N = hi - lo
        if layout == "planar":
            xt, sc, stt = torch.from_numpy(np.ascontiguousarray(xs)).to(dev), N, 1
        else:
            xt, sc, stt = torch.from_numpy(np.ascontiguousarray(xs.T)).to(dev), 1, nch
        maxf = N // hop + 2
        t = dict(mags=torch.zeros(nch, maxf, bins, device=dev), mags_db=torch.zeros(nch, maxf, bins, device=dev),
                 flatness=torch.zeros(nch, maxf, device=dev), centroid=torch.zeros(nch, maxf, device=dev),
                 mfcc=torch.zeros(nch, maxf, nc, dtype=torch.float64, device=dev))
        o = capi.StftOutputs(t["mags"].data_ptr(), None, None, None, t["mags_db"].data_ptr(), t["flatness"].data_ptr(),
                             t["centroid"].data_ptr(), t["mfcc"].data_ptr())
        nf = C.c_int32(0)
        capi.check(capi.lib().mxb_stft_process2(d_full.h, xt.data_ptr(), sc, stt, N, maxf, C.byref(o), mf.h, C.byref(nf),
                                                capi.MEM_DEVICE, None), "mxb_stft_process2")
        co_only = torch.zeros(nch, maxf, nc, dtype=torch.float64, device=dev)
        f_only = d_only.process_device(xt.data_ptr(), sc, stt, N, maxf, mfcc=mf, coeffs=co_only.data_ptr())
        torch.cuda.synchronize()
        rd = {k: v[:, :nf.value].cpu().numpy() for k, v in t.items()}
        assert f_only == nf.value
        e = expected(port, ost.process(xs, want=("mags",))["mags"], n, sr, omf=omf, feats=True)
        same_bits(rd, run3(h_full, xs, feats=True, mfcc=mf), ("device vs host", lo))
        ro = h_only.process(xs, want=(), mfcc=mf)
        assert np.array_equal(co_only[:, :f_only].cpu().numpy(), ro["mfcc"]), lo
        check(rd, e, ("device", lo)); check(ro, e, ("host mfcc only", lo))


@pytest.mark.parametrize("n,hop", [(1024, 441), (1024, 333), (1024, 1023), (1024, 1), (512, 100)])
def test_odd_hops_with_mfcc_and_features(port, n, hop):
    """Hops that are not multiples of 32 (441 = 10 ms at 44.1 kHz), with the fused MFCC and the features on, and an MFCC-only
    transform beside them: the vector-load, fused-tail and buffer-boundary tests all take their other branches. First call: 3 samples."""
    nch = 5
    bins, nfil, nc, fmin, fmax, sr = (512, 42, 13, 20.0, 20000.0, 44100) if n == 1024 else DEV_MFCC[512]
    total = 3 + 250 if hop == 1 else 9 * hop + n + 51
    x = W.channel_streams(nch, total, seed=hop)
    mf = capi.Mfcc(bins, nfil, nc, fmin, fmax, sample_rate=sr)
    omf = port.Mfcc(bins, nfil, nc, fmin, fmax, sr)
    full, only = capi.Stft(nch, n, hop, sample_rate=sr), capi.Stft(nch, n, hop, sample_rate=sr)
    ost = port.Stft(nch, n, hop)
    fired = 0
    for lo, hi in slices(total, (3, 3 + (120 if hop == 1 else 3 * hop + 17))):
        xs = x[:, lo:hi]
        e = expected(port, ost.process(xs, want=("mags",))["mags"], n, sr, omf=omf, feats=True)
        check(run3(full, xs, feats=True, mfcc=mf), e, ("full", hop, lo))
        check(only.process(xs, want=(), mfcc=mf), e, ("mfcc only", hop, lo))
        fired += e["mags"].shape[1]
    assert fired >= 8


# ---------------------------------------------------------------------------------------------- F. non-finite magnitudes

def bad_bins(bins, fmin, fmax, sr):
    """One bin inside the bank's bands (the middle of its range; the reference's bin spacing is sr / numBins) and the top bin,
    where no band has weight."""
    return int((fmin + min(fmax, sr / 2)) / 2 / (sr / bins)), bins - 1


@pytest.mark.parametrize("cfg", [(512, 42, 40, 20.0, 20000.0, 48000), (512, 42, 13, 20.0, 20000.0, 44100), (256, 20, 12, 100.0, 8000.0, 48000),
                                 (1024, 42, 40, 20.0, 20000.0, 48000), (512, 1, 1, 20.0, 20000.0, 48000)])
def test_mfcc_process_non_finite_magnitudes(port, cfg):
    """mxb_mfcc_process on rows with one NaN bin, one +inf bin inside the bands, one +inf bin above the last band: the oracle's
    values (pinned to the reference), its zeros, infs and NaNs included. A NaN anywhere or an inf where no band has weight makes
    every band 0 -- all-zero coefficients; an inf inside bands gives those bands +inf and the others 0."""
    bins, nfil, nc, fmin, fmax, sr = cfg
    mags = port.Stft(3, 2 * bins, bins).process(W.channel_streams(3, 2 * bins * 8, seed=bins))["mags"]
    inside, above = bad_bins(bins, fmin, fmax, sr)
    mags[2, 0, 5] = np.nan
    mags[2, 1, inside] = np.inf
    mags[2, 2, above] = np.inf
    mags[2, 3, :] = np.nan
    g = capi.Mfcc(bins, nfil, nc, fmin, fmax, sample_rate=sr)
    cg, mg = g.process(mags)
    co, mo = port.Mfcc(bins, nfil, nc, fmin, fmax, sr).process(mags)
    np.testing.assert_allclose(mg, mo, rtol=1e-9, atol=1e-12, equal_nan=True)
    np.testing.assert_allclose(cg, co, rtol=1e-9, atol=1e-12, equal_nan=True)
    for f in (0, 2, 3):
        assert np.all(mo[2, f] == 0.0) and np.all(co[2, f] == 0.0), f
    if nfil > 1:
        assert np.isinf(mo[2, 1]).any() and not np.isnan(mo[2, 1]).any()


@pytest.mark.parametrize("n", [256, 2048, 1024])
def test_nan_input_sample(port, n):
    """A NaN input sample makes every bin of the frames that hold it NaN, and the oracle's MFCCs 0 there. On both kernels (r01 at
    256 / 2048, K4s at 1024), MFCC-only and spectra-written: the bad channel's values are the oracle's, and every other channel --
    sharing the 8-frame tensor-core tiles with it -- is bit for bit the same transform of clean samples."""
    nch, hop = 11, n // 2
    cfg ={256: (128, 26, 13, 20.0, 20000.0, 48000), 2048: (1024, 42, 40, 20.0, 20000.0, 48000), 1024: (512, 42, 40, 20.0, 20000.0, 48000)}[n]
    x = W.channel_streams(nch, 5 * n, seed=n + 3)
    xb = x.copy()
    xb[5, 2 * n + 7] = np.nan
    mf = capi.Mfcc(*cfg[:5])
    omf = port.Mfcc(*cfg)
    e = expected(port, port.Stft(nch, n, hop).process(xb, want=("mags",))["mags"], n, 48000, omf=omf)
    bad = np.isnan(e["mags"][5]).all(axis=-1)
    assert bad.any() and np.all(e["mfcc"][5][bad] == 0.0)
    others = np.arange(nch) != 5
    for want in ((), ("mags",)):
        r = capi.Stft(nch, n, hop).process(xb, want=want, mfcc=mf)
        clean = capi.Stft(nch, n, hop).process(x, want=want, mfcc=mf)
        check(r, e, ("nan sample", want))
        for k in r:
            assert np.array_equal(r[k][others], clean[k][others]), (want, k)


# ------------------------------------------------------------------------------------ G. fused tables beyond shared memory

def test_r01_refuses_tables_beyond_shared_memory(port):
    """2048-point frames with a 512-filter x 40-coefficient MFCC need ~300 KB of shared memory per CTA: MXB_ERR_UNSUPPORTED with a
    message, not a CUDA error; the transform then goes on with a bank that fits, continuing the oracle's schedule."""
    nch, n, hop = 3, 2048, 1024
    x = W.channel_streams(nch, 6 * n, seed=2048)
    st = capi.Stft(nch, n, hop)
    with pytest.raises(capi.MxbError, match=f"-> {ERR_UNSUPPORTED}:.*shared memory"):
        st.process(x[:, :3 * n], want=(), mfcc=capi.Mfcc(1024, 512, 40))
    cfg = (1024, 42, 40, 20.0, 20000.0, 48000)
    mf, omf, ost = capi.Mfcc(*cfg[:5]), port.Mfcc(*cfg), port.Stft(nch, n, hop)
    for lo, hi in ((0, 3 * n), (3 * n, 6 * n)):
        e = expected(port, ost.process(x[:, lo:hi], want=("mags",))["mags"], n, 48000, omf=omf)
        check(st.process(x[:, lo:hi], want=("mags",), mfcc=mf), e, lo)


def test_mfcc_process_refuses_tables_beyond_shared_memory(port):
    """8192 bins need 8 x 33 KB of shared memory in the standalone kernel: MXB_ERR_UNSUPPORTED with a message; the library goes on."""
    big = capi.Mfcc(8192, 40, 13)
    with pytest.raises(capi.MxbError, match=f"-> {ERR_UNSUPPORTED}:.*shared memory"):
        big.process(np.ones((2, 8192), dtype=np.float32))
    mags = port.Stft(2, 1024, 512).process(W.channel_streams(2, 4096, seed=9))["mags"]
    cg, _ = capi.Mfcc(512, 42, 40).process(mags)
    np.testing.assert_allclose(cg, port.Mfcc(512, 42, 40).process(mags)[0], rtol=1e-9, atol=1e-12)
