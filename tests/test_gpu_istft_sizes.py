"""maxiIFFT at 2048 points and at any hop (mxb_istft_*): the one-kernel resynthesis at 1024 and 2048 points (istft1024_kernel /
istft2048_kernel) and the two-kernel path below 1024, at hops that do not divide the frame, against the plain-C oracle and the compiled
reference's golden vectors (tests/golden/istft_sizes.npz).

Bar (DESIGN.md): |d| <= 1e-5 * max|out| (the device's sincosf against glibc's cosf / sinf), NaN at the same positions. Where the same
kernels run on the same inputs -- host against device staging, one call against several -- the outputs are bit-identical."""
import ctypes as C_
import os
import subprocess

import numpy as np
import pytest

import golden_checks as G
from maximilian_b200 import capi
from maximilian_b200 import workloads as W
from test_cpp_dropin import compile_patch
from test_istft_sizes import M

pytestmark = pytest.mark.gpu

PAIRS = M.PAIRS + ((256, 100), (1024, 1))


def _close(y, yo, what=""):
    assert y.shape == yo.shape, (what, y.shape, yo.shape)
    nan = np.isnan(yo)
    assert np.array_equal(np.isnan(y), nan), what
    scale = max(np.abs(yo[~nan]).max(), 1e-6)
    d = np.abs(y[~nan] - yo[~nan]).max()
    assert d <= 1e-5 * scale, (what, d, scale)


def _spectra(port, C, n, F, seed):
    """(mags, phases) [C][F][n / 2] from the oracle's forward transform; channel 3 frame 4 has a NaN magnitude, channel 5 frame 2 is silent"""
    fwd = max(n, 128)
    x = W.channel_streams(C, (F + 1) * (fwd // 2), seed=seed)
    r = port.Stft(C, fwd, fwd // 2).process(x, want=("mags", "phases"))
    mags, phases = np.ascontiguousarray(r["mags"][:, :F, :n // 2]), np.ascontiguousarray(r["phases"][:, :F, :n // 2])
    mags[3, 4, n // 8] = np.nan
    mags[5, 2] = 0.0
    return mags, phases


@pytest.mark.parametrize("n,hop", PAIRS)
def test_istft_sizes_vs_oracle(port, n, hop):
    """37 channels (more than one CTA's warps, not a multiple of them) in ragged calls, so that the carried buffer is used."""
    C, F = 37, 10
    mags, phases = _spectra(port, C, n, F, seed=n + hop)
    g = capi.Istft(C, n, hop); o = port.Istft(C, n, hop)
    for lo, hi in ((0, 1), (1, 4), (4, F)):
        y = g.process(mags[:, lo:hi], phases[:, lo:hi]); yo = o.process(mags[:, lo:hi], phases[:, lo:hi])
        assert y.shape == (C, (hi - lo) * hop)
        _close(y, yo, (n, hop, lo, hi))
    if F * hop >= n // 2:                   # past the windows' silent edges: the outputs are not trivially small
        assert np.abs(y[0]).max() > 1e-3


@pytest.mark.parametrize("n,hop", M.PAIRS)
def test_istft_sizes_golden(n, hop):
    g = G.load("istft_sizes")
    y = M.resynthesise(capi.Istft(M.C, n, hop), g[f"{n}/mags"], g[f"{n}/phases"])
    _close(y, g[f"{n}/{hop}/out"], (n, hop))


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("hop", [1024, 441, 2048, 1])
def test_istft_2048_host_staging_equals_device_memory(hop):
    import torch
    C, n, bins = 40, 2048, 1024
    twins = [capi.Istft(C, n, hop) for _ in range(2)]
    rng = np.random.default_rng(hop)
    L = capi.lib()
    for k, F in enumerate([1, 7, 3]):
        mags = rng.random((C, F, bins), dtype=np.float32)
        ph = (rng.random((C, F, bins), dtype=np.float32) - 0.5) * 6.0
        oh = np.full((C, F * hop), np.nan, dtype=np.float32)
        od = torch.full((C, F * hop), float("nan"), dtype=torch.float32, device="cuda")
        capi.check(L.mxb_istft_process(twins[0].h, mags.ctypes.data, ph.ctypes.data, F, oh.ctypes.data, capi.MEM_HOST, None), "host twin")
        dm, dp = _dev(mags), _dev(ph)
        capi.check(L.mxb_istft_process(twins[1].h, C_.c_void_p(dm.data_ptr()), C_.c_void_p(dp.data_ptr()), F, C_.c_void_p(od.data_ptr()),
                                       capi.MEM_DEVICE, None), "device twin")
        torch.cuda.synchronize()
        assert np.array_equal(oh, od.cpu().numpy()), (hop, k)


@pytest.mark.parametrize("n,hop", [(2048, 441), (2048, 1), (2048, 2048), (1024, 441), (512, 100), (64, 48)])
def test_istft_one_call_equals_split_calls(port, n, hop):
    C, F = 9, 11
    mags, phases = _spectra(port, C, n, F, seed=3 * n + hop)
    whole = capi.Istft(C, n, hop).process(mags, phases)
    s = capi.Istft(C, n, hop)
    parts = np.concatenate([s.process(mags[:, lo:hi], phases[:, lo:hi]) for lo, hi in ((0, 1), (1, 3), (3, 4), (4, F))], axis=1)
    assert np.array_equal(whole, parts, equal_nan=True)


def test_istft_2048_hop441_16k_channels_vs_oracle_slices(port):
    """2048 / 441 at 16 Ki channels, spectra from the device's own 2048-point analysis, two calls of 8 frames: 80 channels (first, random,
    last) against the oracle fed the same spectra."""
    import torch
    C, n, hop, H = 16384, 2048, 441, 8
    bins = n // 2
    rng = np.random.default_rng(9)
    N = 2 * H * hop
    base = torch.from_numpy(W.channel_streams(256, N, seed=29)).cuda()
    x = (base.repeat(C // 256, 1) * torch.from_numpy((1.0 + 0.001 * rng.random((C, 1))).astype(np.float32)).cuda()).contiguous()
    pick = np.concatenate([np.arange(24), np.sort(rng.choice(np.arange(24, C - 24), 32, replace=False)), np.arange(C - 24, C)])
    st = capi.Stft(C, n, hop); ist = capi.Istft(C, n, hop); oist = port.Istft(pick.size, n, hop)
    maxf = N // hop + 2
    mags = torch.empty((C, maxf, bins), dtype=torch.float32, device="cuda"); phases = torch.empty_like(mags)
    assert st.process_device(x.data_ptr(), N, 1, N, maxf, mags=mags.data_ptr(), phases=phases.data_ptr()) == 2 * H
    idx = torch.from_numpy(pick).cuda()
    L = capi.lib()
    for k in range(2):
        m = mags[:, k * H:(k + 1) * H].contiguous(); p = phases[:, k * H:(k + 1) * H].contiguous()
        y = torch.empty((C, H * hop), dtype=torch.float32, device="cuda")
        capi.check(L.mxb_istft_process(ist.h, C_.c_void_p(m.data_ptr()), C_.c_void_p(p.data_ptr()), H, C_.c_void_p(y.data_ptr()),
                                       capi.MEM_DEVICE, None), "mxb_istft_process")
        torch.cuda.synchronize()
        yo = oist.process(m[idx].cpu().numpy(), p[idx].cpu().numpy())
        _close(y[idx].cpu().numpy(), yo, k)
        assert np.abs(yo).max() > 1e-3


def test_istft_rejects_bad_sizes_and_goes_on(port):
    for n, hop in ((4096, 1024), (32, 16), (1000, 500), (2048, 0), (2048, 2049), (1024, 1025), (64, 65)):
        with pytest.raises(capi.MxbError):
            capi.Istft(1, n, hop)
    mags, phases = _spectra(port, 6, 2048, 6, seed=1)
    _close(capi.Istft(6, 2048, 441).process(mags, phases), port.Istft(6, 2048, 441).process(mags, phases))


@pytest.mark.parametrize("n,hop", [(2048, 1024), (2048, 441), (1024, 441), (512, 100)])
def test_per_sample_resynthesis_at_any_size_matches_oracle(port, tmp_path_factory, n, hop):
    """tests/cpp/resynth_sizes.cpp: the reference's per-sample idiom through the C++ layer's scalar signatures, against the oracle: frames
    fire on the reference's sample, resynthesis within 2e-5 of max (the analysis' atan2f ulps feed the resynthesis' sincosf ulps)."""
    tmp = tmp_path_factory.mktemp(f"resynth_{n}_{hop}")
    exe = compile_patch(tmp, os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "resynth_sizes.cpp"))
    N = 5 * n + 3 * hop + 17
    x = W.channel_streams(1, N, seed=n + hop)
    x.tofile(tmp / "in.bin")
    r = subprocess.run([exe, str(tmp / "in.bin"), str(tmp / "out.bin"), str(N), str(n), str(hop)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = open(tmp / "out.bin", "rb").read()
    F = int(np.frombuffer(raw, dtype=np.int32, count=1)[0])
    fired = np.frombuffer(raw, dtype=np.float32, count=N, offset=4)
    y = np.frombuffer(raw, dtype=np.float32, count=N, offset=4 + 4 * N)
    assert 4 + 8 * N == len(raw)
    assert F == N // hop and np.array_equal(np.nonzero(fired)[0], hop * np.arange(1, F + 1) - 1)   # true on the sample that completes a frame
    o = port.Stft(1, n, hop).process(x)
    assert o["mags"].shape[1] == F
    # maxiIFFT::process reads the spectrum on the first sample of every hop: zeros before the first frame, then frame k - 1 during hop k
    K = (N + hop - 1) // hop
    z = np.zeros((1, 1, n // 2), dtype=np.float32)
    oy = port.Istft(1, n, hop).process(np.concatenate([z, o["mags"][:, :K - 1]], axis=1), np.concatenate([z, o["phases"][:, :K - 1]], axis=1))
    assert np.abs(y - oy[0, :N]).max() <= 2e-5 * np.abs(oy).max()
    assert np.abs(y[hop:]).max() > 1e-3
