"""The stand-alone octave analyser and Bark loudness (mxb_octave_process / mxb_bark_process) on caller-supplied spectra, at every size.

Bars (DESIGN.md section 2): octave averages and peaks bit for bit, NaN included; Bark 1e-12 relative, with the same NaN positions.

  1  octave against the port at 64 .. 1024 bins, magnitudes from the transform at the matching size, 1 / 5 / 9 / 33 channels (one
     silent), several calls with a hold longer than one call, configurations with more than 32 runs and bands
  2  both against the compiled reference's outputs (tests/golden/analysers.npz): silent frames, NaN, inf and negative bins
  3  stand-alone equals fused at 1024 bins; one octave handle switched between the two paths mid-stream follows the port
  4  host memory and device memory (torch tensors, a non-default stream) give the same bits
  5  64 Ki channels x 8 frames of 2048-point spectra
  6  every refusal, and the handle still usable after it
  7  frames the 16-byte copies cannot take: bin counts not a multiple of 4, device rows off a 16-byte boundary
"""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest

import golden_checks as G
from maximilian_b200 import capi
from maximilian_b200 import workloads as W

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_UNSUPPORTED = -1, -4


def _maker():
    spec = importlib.util.spec_from_file_location("make_analysers_golden", os.path.join(G.GOLD, "make_analysers_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


M = _maker()


def bark_close(got, exp, what=""):
    for g, e, name in zip(got, exp, ("specific", "relative", "total")):
        assert g.shape == e.shape, (what, name)
        assert np.array_equal(np.isnan(g), np.isnan(e)), (what, name)
        np.testing.assert_allclose(g, e, rtol=1e-12, atol=0, err_msg=f"{what} {name}")


def same_bits(a, b, what=""):
    for x, y in zip(a, b):
        assert np.array_equal(x, y, equal_nan=True), what


def transform_mags(n, C, N, seed, silent=None):
    """Magnitudes of the fft_size-n transform (hop n / 2) of C channels of N samples -> float32 [C][frames][n / 2]."""
    x = W.channel_streams(C, N, seed=seed)
    if silent is not None:
        x[silent] = 0.0
    return capi.Stft(C, n, n // 2).process(x, want=("mags",))["mags"]


# ------------------------------------------------------------------------------------------------ 1. octave against the port

@pytest.mark.parametrize("n_bands", [64, 128, 256, 512, 1024])
def test_octave_against_port(port, n_bands):
    n = 2 * n_bands
    for k, nch in enumerate((1, 5, 9, 33)):
        per_octave = (3, 12, 6, 12)[k]             # 12 per octave: more than 32 bands and runs from 256 bins on
        sr = 44100 if k % 2 else 48000
        mags = transform_mags(n, nch, 13 * (n // 2) + 17, seed=n_bands + k, silent=nch // 2 if nch > 1 else None)
        oc, ooc = capi.Octave(nch, sr, n_bands, per_octave), port.Octave(nch, sr, n_bands, per_octave)
        assert oc.n_averages == ooc.n_averages
        for h in (oc, ooc):
            h.config(5, 0.8, 0.95, 0.002)              # hold 5 frames: longer than one of the calls below
        for lo, hi in ((0, 4), (4, 5), (5, mags.shape[1])):
            got, exp = oc.process(mags[:, lo:hi]), ooc.process(mags[:, lo:hi])
            same_bits(got, exp, (n_bands, nch, lo))
        if nch > 1:
            assert not got[0][nch // 2].any()              # the silent channel


# ------------------------------------------------------------------------------------------------ 2. against the reference's outputs

@pytest.mark.parametrize("n_bands", M.OCT_BANDS)
def test_octave_golden(n_bands):
    g = G.load("analysers")
    mags = g[f"oct/{n_bands}/mags"]
    for po in M.OCT_PER_OCTAVE:
        for sr in M.OCT_RATES:
            o = capi.Octave(M.OCT_C, sr, n_bands, po)
            o.config(M.OCT_HOLD, M.OCT_DECAY, M.OCT_ICPT, M.oct_slope(n_bands))
            av, pk = o.process(mags)
            assert np.isnan(av).any()
            same_bits((av, pk), (g[f"oct/{n_bands}/{po}/{sr}/averages"], g[f"oct/{n_bands}/{po}/{sr}/peaks"]), (n_bands, po, sr))


@pytest.mark.parametrize("buffer_size", M.BARK_SIZES)
def test_bark_golden(port, buffer_size):
    g = G.load("analysers")
    s = g[f"bark/{buffer_size}/spectrum"]
    for sr in M.BARK_RATES:
        got = capi.Bark(sr, buffer_size).process(s)
        exp = tuple(g[f"bark/{buffer_size}/{sr}/{k}"] for k in ("specific", "relative", "total"))
        bark_close(got, exp, (buffer_size, sr))
        assert np.isnan(got[1][1]).all()                   # the silent frame: 0 / 0, like the reference
        bark_close(got, port.bark(s, sr, buffer_size), (buffer_size, sr, "port"))


@pytest.mark.parametrize("buffer_size", [s for s in M.BARK_SIZES if s <= 2048])       # the transform's sizes
def test_bark_on_transform_magnitudes(port, buffer_size):
    """Bark on the transform's own magnitudes (a channel silent), every rate, frames laid out [C][frames][bins]."""
    mags = transform_mags(buffer_size, 3, 9 * buffer_size // 2, seed=buffer_size, silent=1)
    for sr in M.BARK_RATES:
        bark_close(capi.Bark(sr, buffer_size).process(mags), port.bark(mags, sr, buffer_size), (buffer_size, sr))


# ------------------------------------------------------------------------------------------------ 3. stand-alone equals fused

def fused_call(st, x, oc):
    """mxb_stft_process3 with the magnitudes, the octave analyser and Bark: host arrays of the frames that fired."""
    nch, N = x.shape
    maxf = N // st.hop + 2
    mags = np.zeros((nch, maxf, st.bins), dtype=np.float32)
    av = np.zeros((nch, maxf, oc.n_averages), dtype=np.float32); pk = np.zeros_like(av)
    bs = np.zeros((nch, maxf, 24)); br = np.zeros_like(bs); bt = np.zeros((nch, maxf))
    o = capi.StftOutputs(mags.ctypes.data, None, None, None, None, None, None, None)
    post = capi.StftPost(oc.h, av.ctypes.data, pk.ctypes.data, 1, bs.ctypes.data, br.ctypes.data, bt.ctypes.data)
    nf = C.c_int32(0)
    xs = np.ascontiguousarray(x, dtype=np.float32)
    capi.check(capi.lib().mxb_stft_process3(st.h, xs.ctypes.data, N, 1, N, maxf, C.byref(o), C.byref(post), None, C.byref(nf),
                                            capi.MEM_HOST, None), "mxb_stft_process3")
    f = nf.value
    return mags[:, :f].copy(), av[:, :f].copy(), pk[:, :f].copy(), bs[:, :f].copy(), br[:, :f].copy(), bt[:, :f].copy()


def test_standalone_equals_fused_at_1024(port):
    nch, N = 11, 9 * 512 + 100
    x = W.channel_streams(nch, N, seed=77)
    x[4] = 0.0
    st = capi.Stft(nch, 1024, 512)
    fused, alone = capi.Octave(nch, 48000, 512, 6), capi.Octave(nch, 48000, 512, 6)
    for h in (fused, alone):
        h.config(3, 0.85, 0.9, 0.01)
    bk = capi.Bark(48000, 1024)
    for lo, hi in ((0, 3000), (3000, N)):
        mags, av, pk, bs, br, bt = fused_call(st, x[:, lo:hi], fused)
        same_bits(alone.process(mags), (av, pk), ("octave", lo))
        same_bits(bk.process(mags), (bs, br, bt), ("bark", lo))


def test_one_octave_handle_switches_paths_midstream(port):
    nch, hop = 6, 512
    x = W.channel_streams(nch, 16 * hop, seed=78)
    st = capi.Stft(nch, 1024, hop)
    oc, ooc = capi.Octave(nch, 44100, 512, 12), port.Octave(nch, 44100, 512, 12)
    for h in (oc, ooc):
        h.config(4, 0.7, 1.0, 0.0)
    ost = port.Stft(nch, 1024, hop)
    cuts = [0, 3 * hop, 7 * hop, 11 * hop, 16 * hop]
    for k in range(len(cuts) - 1):
        xs = x[:, cuts[k]:cuts[k + 1]]
        om = ost.process(xs, want=("mags",))["mags"]
        if k % 2 == 0:
            mags, av, pk = fused_call(st, xs, oc)[:3]
            assert np.array_equal(mags, om)
        else:
            st.process(xs, want=("mags",))                  # the transform advances; the analyser runs on the magnitudes alone
            av, pk = oc.process(om)
        same_bits((av, pk), ooc.process(om), ("switch", k))


# ------------------------------------------------------------------------------------------------ 4. host memory == device memory

def test_host_and_device_memory_agree():
    import torch
    nch, F, nb = 7, 5, 1024
    r = np.random.default_rng(5)
    mags = r.exponential(1.0, (nch, F + 2, nb)).astype(np.float32)          # max_frames F + 2: rows past `frames` are not read
    mags[2, 1, 17] = np.nan
    host, dev = capi.Octave(nch, 48000, nb, 6), capi.Octave(nch, 48000, nb, 6)
    ha, hp = host.process(mags[:, :F])
    s = torch.cuda.Stream()
    dm = torch.from_numpy(mags).cuda()
    da = torch.full((nch, F + 2, dev.n_averages), -1.0, dtype=torch.float32, device="cuda"); dp = torch.full_like(da, -1.0)
    dev.process_device(dm.data_ptr(), F, F + 2, da.data_ptr(), dp.data_ptr(), stream=s.cuda_stream)
    s.synchronize()
    same_bits((da[:, :F].cpu().numpy(), dp[:, :F].cpu().numpy()), (ha, hp), "octave")
    assert (da[:, F:] == -1.0).all()
    spec = r.exponential(0.1, (13, 1024)).astype(np.float32)
    spec[3] = 0.0; spec[4, 9] = np.inf
    bk = capi.Bark(44100, 2048)
    hb = bk.process(spec)
    ds = torch.from_numpy(spec).cuda()
    out = [torch.empty((13, 24), dtype=torch.float64, device="cuda"), torch.empty((13, 24), dtype=torch.float64, device="cuda"),
           torch.empty(13, dtype=torch.float64, device="cuda")]
    bk.process_device(ds.data_ptr(), 13, *[o.data_ptr() for o in out], stream=s.cuda_stream)
    s.synchronize()
    same_bits([o.cpu().numpy() for o in out], hb, "bark")


# ------------------------------------------------------------------------------------------------ 5. full size

def test_full_size_64k_channels(port):
    """64 Ki channels x 8 frames of 1024-bin spectra in one call: 96 channels (first, last, random) against the port, the rest bit for bit
    against a second call on its own handle that asks for fewer outputs."""
    import torch
    nch, F, nb = 65536, 8, 1024
    g = torch.Generator(device="cuda").manual_seed(9)
    mags = torch.rand((nch, F, nb), generator=g, device="cuda", dtype=torch.float32).mul_(3.0)
    mags[123] = 0.0
    a1, a2 = capi.Octave(nch, 48000, nb, 6), capi.Octave(nch, 48000, nb, 6)
    for h in (a1, a2):
        h.config(2, 0.9, 1.0, 0.001)
    nA = a1.n_averages
    av = torch.empty((nch, F, nA), dtype=torch.float32, device="cuda"); pk = torch.empty_like(av); av2 = torch.empty_like(av)
    a1.process_device(mags.data_ptr(), F, F, av.data_ptr(), pk.data_ptr())
    a2.process_device(mags.data_ptr(), F, F, av2.data_ptr(), None)
    bk = capi.Bark(48000, 2048)
    n = nch * F
    bs = torch.empty((n, 24), dtype=torch.float64, device="cuda"); br = torch.empty_like(bs); bt = torch.empty(n, dtype=torch.float64, device="cuda")
    bs2 = torch.empty_like(bs)
    bk.process_device(mags.data_ptr(), n, bs.data_ptr(), br.data_ptr(), bt.data_ptr())
    bk.process_device(mags.data_ptr(), n, bs2.data_ptr(), None, None)
    torch.cuda.synchronize()
    assert torch.equal(av, av2) and torch.equal(bs, bs2)
    pick = np.unique(np.concatenate([[0, 123, nch - 1], np.random.default_rng(3).choice(nch, 93, replace=False)]))
    idx = torch.from_numpy(pick).cuda()
    m = mags[idx].cpu().numpy()
    ooc = port.Octave(pick.size, 48000, nb, 6); ooc.config(2, 0.9, 1.0, 0.001)
    same_bits((av[idx].cpu().numpy(), pk[idx].cpu().numpy()), ooc.process(m), "octave")
    sel = lambda t: t.view(nch, F, *t.shape[1:])[idx].cpu().numpy()            # noqa: E731
    bark_close((sel(bs), sel(br), sel(bt)), port.bark(m, 48000, 2048), "bark")


# ------------------------------------------------------------------------------------------------ 6. refusals

def test_refusals_leave_handles_usable(port):
    L = capi.lib()
    ctx = capi.default_context()
    oc, ooc = capi.Octave(2, 48000, 256, 3), port.Octave(2, 48000, 256, 3)
    mags = transform_mags(512, 2, 6 * 256, seed=4)
    F = mags.shape[1]
    a = np.zeros((2, F, oc.n_averages), dtype=np.float32)
    P = lambda x: C.c_void_p(x.ctypes.data)                                  # noqa: E731
    assert L.mxb_octave_process(None, P(mags), F, F, P(a), P(a), 0, None) == ERR_INVALID
    assert L.mxb_octave_process(oc.h, None, F, F, P(a), P(a), 0, None) == ERR_INVALID
    assert L.mxb_octave_process(oc.h, P(mags), -1, F, P(a), P(a), 0, None) == ERR_INVALID
    assert L.mxb_octave_process(oc.h, P(mags), F, F - 1, P(a), P(a), 0, None) == ERR_INVALID
    assert L.mxb_octave_process(oc.h, P(mags), F, F, P(a), P(a), 7, None) == ERR_INVALID
    assert L.mxb_octave_process(oc.h, P(mags), 0, 0, P(a), P(a), 0, None) == 0 and not a.any()      # frames == 0: nothing
    same_bits(oc.process(mags), ooc.process(mags), "octave after refusals")
    b = C.c_void_p()
    for sr, bs in ((48000, 1), (48000, 4097), (48000, 0), (0, 1024), (-44100, 1024), (2 ** 31 - 1, 1024), (8_500_000, 1024)):
        assert L.mxb_bark_create(ctx.h, sr, bs, C.byref(b)) == ERR_INVALID, (sr, bs)
        assert not b.value
    assert L.mxb_bark_create(ctx.h, 8_400_000, 1024, C.byref(b)) == 0          # 511 * 8.4e6 < 2^32
    L.mxb_bark_destroy(b)
    assert L.mxb_bark_create(None, 48000, 1024, C.byref(b)) == ERR_INVALID
    bk = capi.Bark(48000, 1024)
    sp = np.zeros((4, 24)); s512 = np.abs(np.random.default_rng(1).standard_normal((4, 512))).astype(np.float32)
    assert L.mxb_bark_process(None, P(s512), 4, P(sp), None, None, 0, None) == ERR_INVALID
    assert L.mxb_bark_process(bk.h, None, 4, P(sp), None, None, 0, None) == ERR_INVALID
    assert L.mxb_bark_process(bk.h, P(s512), -1, P(sp), None, None, 0, None) == ERR_INVALID
    assert L.mxb_bark_process(bk.h, P(s512), 4, P(sp), None, None, 3, None) == ERR_INVALID
    assert L.mxb_bark_process(bk.h, P(s512), 0, P(sp), None, None, 0, None) == 0 and not sp.any()
    bark_close(bk.process(s512), port.bark(s512, 48000, 1024), "bark after refusals")
    # the fused entry point still refuses the analysers at sizes other than 1024, and names the stand-alone ones
    with pytest.raises(capi.MxbError, match="mxb_octave_process"):
        capi.stft_process_post(capi.Stft(2, 512, 128), W.channel_streams(2, 1024, seed=1), octave=capi.Octave(2, 48000, 256, 3))
    with pytest.raises(capi.MxbError):
        capi.stft_process_post(capi.Stft(2, 2048, 1024), W.channel_streams(2, 4096, seed=1), bark=True)


# ------------------------------------------------------------------------------------------------ 7. rows the 16-byte copies cannot take

def test_unaligned_rows_and_odd_bin_counts(port):
    """Frames staged with plain loads: a bin count that is not a multiple of 4 (octave 102 bins, Bark buffer_size 1022: 511 bins), and
    device rows 4 bytes off a 16-byte boundary."""
    import torch
    r = np.random.default_rng(11)
    m = r.exponential(1.0, (3, 5, 102)).astype(np.float32)
    m[2, 3, 40] = np.nan
    oc, ooc = capi.Octave(3, 44100, 102, 6), port.Octave(3, 44100, 102, 6)
    for h in (oc, ooc):
        h.config(2, 0.9, 1.0, 0.01)
    same_bits(oc.process(m), ooc.process(m), "octave, 102 bins")
    s = r.exponential(0.1, (7, 511)).astype(np.float32)
    s[2] = 0.0; s[4, 100] = np.inf
    bark_close(capi.Bark(48000, 1022).process(s), port.bark(s, 48000, 1022), "bark, 511 bins")
    # device rows 4 bytes past a 16-byte boundary, 1024 bins
    nch, F, nb = 4, 3, 1024
    mm = r.exponential(1.0, (nch, F, nb)).astype(np.float32)
    buf = torch.zeros(nch * F * nb + 1, dtype=torch.float32, device="cuda")
    buf[1:] = torch.from_numpy(mm.ravel()).cuda()
    ptr = buf.data_ptr() + 4
    assert ptr % 16 == 4
    oc, ooc = capi.Octave(nch, 48000, nb, 3), port.Octave(nch, 48000, nb, 3)
    av = torch.empty((nch, F, oc.n_averages), dtype=torch.float32, device="cuda"); pk = torch.empty_like(av)
    oc.process_device(ptr, F, F, av.data_ptr(), pk.data_ptr())
    bk = capi.Bark(48000, 2048)
    out = [torch.empty((nch * F, 24), dtype=torch.float64, device="cuda"), torch.empty((nch * F, 24), dtype=torch.float64, device="cuda"),
           torch.empty(nch * F, dtype=torch.float64, device="cuda")]
    bk.process_device(ptr, nch * F, *[o.data_ptr() for o in out])
    torch.cuda.synchronize()
    same_bits((av.cpu().numpy(), pk.cpu().numpy()), ooc.process(mm), "octave, unaligned rows")
    bark_close([o.cpu().numpy() for o in out], [a.reshape(nch * F, *a.shape[2:]) for a in port.bark(mm, 48000, 2048)], "bark, unaligned rows")
