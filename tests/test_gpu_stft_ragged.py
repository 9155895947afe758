"""Channels that advance independently: mxb_stft_process_ragged / mxb_istft_process_ragged, every channel against a one-channel oracle
Stft / Istft fed that channel's samples only (the reference's separate maxiFFT / maxiIFFT objects).

Bars (DESIGN.md): magnitudes, real, imaginary, octave averages / peaks bit for bit; phases 1e-4 rad; MFCC 1e-9 relative; Bark 1e-12
relative; dB, flatness and centroid as in test_gpu_spectral_epilogues; resynthesis 1e-5 of the maximum.
"""
import ctypes as C

import ctypes as C_
import os
import subprocess

import numpy as np
import pytest

from maximilian_b200 import capi
from maximilian_b200 import workloads as W

pytestmark = pytest.mark.gpu


def _phase_close(pg, po, mags):
    if mags.size == 0:
        return
    d = np.angle(np.exp(1j * (pg.astype(np.float64) - po.astype(np.float64))))
    sel = mags > 1e-3 * mags.max(axis=-1, keepdims=True)
    assert np.abs(d[sel]).max(initial=0.0) <= 1e-4


def _counts(rng, C, hop, calls):
    """Per call and channel: 0, 1, hop - 1, exactly one hop, several hops, or random; some channels idle for several calls."""
    pick = np.array([0, 1, hop - 1, hop, 3 * hop + 5, 2 * hop])
    out = []
    for k in range(calls):
        c = pick[rng.integers(0, len(pick), C)]
        c = np.where(rng.random(C) < 0.3, rng.integers(0, 4 * hop, C), c)
        c[:: 5] = 0 if k < 2 else c[:: 5]                  # every fifth channel idle for the first two calls
        out.append(c.astype(np.int32))
    return out


class Streams:
    """The device handle and one oracle Stft per channel, fed the same per-channel cuts of one long stream each."""

    def __init__(self, port, C, n, hop, seed, length):
        self.C, self.n, self.hop = C, n, hop
        self.x = W.channel_streams(C, length, seed=seed)
        self.off = np.zeros(C, dtype=np.int64)
        self.oracles = [port.Stft(1, n, hop) for _ in range(C)]
        self.pos = np.full(C, n - hop)

    def cut(self, counts):
        m = max(1, int(counts.max()))
        buf = np.zeros((self.C, m), dtype=np.float32)
        for c in range(self.C):
            buf[c, :counts[c]] = self.x[c, self.off[c]:self.off[c] + counts[c]]
        return buf

    def oracle(self, counts, want):
        res = []
        for c in range(self.C):
            seg = self.x[c:c + 1, self.off[c]:self.off[c] + counts[c]]
            res.append(self.oracles[c].process(seg, want=want))
            a = self.pos[c] + counts[c]
            f = (a - self.n) // self.hop + 1 if a >= self.n else 0
            self.pos[c] = a - f * self.hop
        self.off += counts
        return res


def _check_spectra(fr, r, ro):
    for c, o in enumerate(ro):
        f = o["mags"].shape[1]
        assert fr[c] == f, (c, fr[c], f)
        for k in ("re", "im", "mags"):
            if k in r:
                assert np.array_equal(r[k][c, :f], o[k][0]), (k, c)
        if "phases" in r:
            _phase_close(r["phases"][c, :f], o["phases"][0], o["mags"][0])


@pytest.mark.parametrize("n,hop", [(128, 32), (256, 256), (512, 100), (512, 128), (1024, 441), (1024, 512), (2048, 441), (2048, 512)])
def test_ragged_spectra_every_size(port, n, hop):
    C, calls = 37, 5
    rng = np.random.default_rng(n + hop)
    cs = _counts(rng, C, hop, calls)
    s = Streams(port, C, n, hop, seed=n * 7 + hop, length=int(sum(c.max() for c in cs)) + 1)
    st = capi.Stft(C, n, hop)
    for counts in cs:
        fr, r = st.process_ragged(s.cut(counts), counts)
        _check_spectra(fr, r, s.oracle(counts, ("mags", "phases", "re", "im")))
        assert np.array_equal(st.positions(), s.pos)


@pytest.mark.parametrize("n,hop", [(1024, 512), (512, 128)])
def test_ragged_many_channels_sliced(port, n, hop):
    """1030 channels: many CTAs, and enough samples per call for the sliced host pipeline (C x most samples >= 4 Mi)."""
    C = 1030
    rng = np.random.default_rng(3)
    cs = [rng.integers(0, 4200, C).astype(np.int32) for _ in range(4)]
    cs[0][0] = 4100                                           # the largest count of a call decides the slicing
    for c in cs:
        c[rng.random(C) < 0.2] = 0
    s = Streams(port, C, n, hop, seed=11, length=int(sum(c.max() for c in cs)) + 1)
    st = capi.Stft(C, n, hop)
    for counts in cs:
        fr, r = st.process_ragged(s.cut(counts), counts, want=("mags", "re"))
        _check_spectra(fr, r, s.oracle(counts, ("mags", "re")))


def test_ragged_pairs_one_half_idle(port):
    """The 1024-point kernel packs channels 2k, 2k+1 into one warp: one half with frames, the other with none or fewer."""
    C, n, hop = 9, 1024, 512
    cs = [np.array([3000, 0, 0, 3000, 700, 2600, 1, 0, 5000], dtype=np.int32),
          np.array([0, 2100, 1500, 0, 0, 0, 4000, 512, 0], dtype=np.int32),
          np.array([513, 511, 0, 0, 2048, 1, 1, 1, 900], dtype=np.int32),
          np.array([1024, 0, 1024, 0, 1024, 0, 1024, 0, 1024], dtype=np.int32)]
    s = Streams(port, C, n, hop, seed=2, length=int(sum(c.max() for c in cs)) + 1)
    st = capi.Stft(C, n, hop)
    for counts in cs:
        fr, r = st.process_ragged(s.cut(counts), counts, features=True)
        ro = s.oracle(counts, ("mags", "phases", "re", "im"))
        _check_spectra(fr, r, ro)
        for c, o in enumerate(ro):
            f = fr[c]
            if f == 0:
                continue
            db, fl, ce = port.spectral_features(o["mags"][0], n)
            np.testing.assert_allclose(r["mags_db"][c, :f], db, rtol=1e-6, atol=1e-5)
            np.testing.assert_allclose(r["flatness"][c, :f], fl, rtol=1e-4, atol=1e-7)
            np.testing.assert_allclose(r["centroid"][c, :f], ce, rtol=1e-4, atol=1e-3)


def test_ragged_fused_octave_bark_hold(port):
    """Octave (peak hold longer than one call) and Bark fused at 1024 points: a channel that fires nothing keeps its averages, peaks
    and hold counters -- its next frames match the oracle's analyser fed only that channel's frames."""
    C, n, hop = 6, 1024, 512
    cs = [np.array([4096, 0, 2048, 100, 0, 3000], dtype=np.int32),
          np.array([0, 3000, 0, 1500, 0, 600], dtype=np.int32),
          np.array([2048, 512, 0, 0, 0, 2000], dtype=np.int32),
          np.array([512, 1024, 4096, 2048, 0, 0], dtype=np.int32)]
    s = Streams(port, C, n, hop, seed=5, length=int(sum(c.max() for c in cs)) + 1)
    st = capi.Stft(C, n, hop)
    oc = capi.Octave(C, 48000.0, n // 2, 3)
    oc.config(peak_hold_time=5, peak_decay_rate=0.8)
    oo = [port.Octave(1, 48000.0, n // 2, 3) for _ in range(C)]
    for o in oo:
        o.config(peak_hold_time=5, peak_decay_rate=0.8)
    for counts in cs:
        fr, r = st.process_ragged(s.cut(counts), counts, want=("mags",), octave=oc, bark=True)
        ro = s.oracle(counts, ("mags",))
        _check_spectra(fr, r, ro)
        for c in range(C):
            f = fr[c]
            if f == 0:
                continue
            av, pk = oo[c].process(ro[c]["mags"])
            assert np.array_equal(r["averages"][c, :f], av[0]) and np.array_equal(r["peaks"][c, :f], pk[0]), c
            sp, rl, tt = port.bark(ro[c]["mags"][0], 48000, n)
            np.testing.assert_allclose(r["bark_specific"][c, :f], sp, rtol=1e-12, atol=0)
            np.testing.assert_allclose(r["bark_relative"][c, :f], rl, rtol=1e-12, atol=0)
            np.testing.assert_allclose(r["bark_total"][c, :f], tt, rtol=1e-12, atol=0)


@pytest.mark.parametrize("n,hop,spectra", [(1024, 512, False), (1024, 441, True), (512, 128, False), (512, 100, True)])
def test_ragged_fused_mfcc(port, n, hop, spectra):
    C = 11
    rng = np.random.default_rng(n + hop)
    cs = _counts(rng, C, hop, 4)
    s = Streams(port, C, n, hop, seed=n + 3 * hop, length=int(sum(c.max() for c in cs)) + 1)
    st = capi.Stft(C, n, hop)
    mf = capi.Mfcc(n // 2, 42, 13 if n == 512 else 40, 20.0, 20000.0)
    omf = port.Mfcc(n // 2, 42, 13 if n == 512 else 40, 20.0, 20000.0, 48000)
    for counts in cs:
        fr, r = st.process_ragged(s.cut(counts), counts, want=("mags",) if spectra else (), mfcc=mf)
        ro = s.oracle(counts, ("mags",))
        for c, o in enumerate(ro):
            f = o["mags"].shape[1]
            assert fr[c] == f
            if f:
                co, _ = omf.process(o["mags"][0])
                np.testing.assert_allclose(r["mfcc"][c, :f], co, rtol=1e-9, atol=1e-12)


def _device(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("n,hop,layout", [(1024, 512, "planar"), (1024, 441, "time"), (2048, 441, "planar"), (256, 64, "time")])
def test_ragged_device_memory(port, n, hop, layout):
    import torch
    C = 21
    rng = np.random.default_rng(n + hop + len(layout))
    cs = _counts(rng, C, hop, 4)
    s = Streams(port, C, n, hop, seed=9, length=int(sum(c.max() for c in cs)) + 1)
    st = capi.Stft(C, n, hop)
    maxf = 16
    for counts in cs:
        buf = s.cut(counts)
        if layout == "planar":
            d_in = _device(buf); sc, stt = buf.shape[1], 1
        else:
            d_in = _device(buf.T); sc, stt = 1, C
        d_m = torch.zeros((C, maxf, n // 2), dtype=torch.float32, device="cuda")
        d_r = torch.zeros_like(d_m)
        fr = st.process_ragged_device(d_in.data_ptr(), sc, stt, counts, maxf, mags=d_m.data_ptr(), re=d_r.data_ptr())
        torch.cuda.synchronize()
        mags, re = d_m.cpu().numpy(), d_r.cpu().numpy()
        _check_spectra(fr, dict(mags=mags, re=re), s.oracle(counts, ("mags", "re")))
        for c in range(C):                                        # a channel (or a K4s half) past its last frame stores nothing
            assert not mags[c, fr[c]:].any() and not re[c, fr[c]:].any(), c


@pytest.mark.parametrize("n,hop", [(1024, 441), (512, 128)])
def test_ragged_host_time_major(port, n, hop):
    """Host memory, input [t][c] (the layout a voice bank writes): stride_c = 1, stride_t = C."""
    C = 15
    rng = np.random.default_rng(n)
    cs = _counts(rng, C, hop, 4)
    s = Streams(port, C, n, hop, seed=21, length=int(sum(c.max() for c in cs)) + 1)
    st = capi.Stft(C, n, hop)
    L = capi.lib()
    for counts in cs:
        xt = np.ascontiguousarray(s.cut(counts).T)
        maxf = 16
        mags = np.zeros((C, maxf, n // 2), dtype=np.float32); re = np.zeros_like(mags)
        o = capi.StftOutputs(mags.ctypes.data, None, re.ctypes.data, None, None, None, None, None)
        fr = np.zeros(C, dtype=np.int32)
        capi.check(L.mxb_stft_process_ragged(st.h, xt.ctypes.data, 1, C, counts.ctypes.data, maxf, C_.byref(o), None, None, fr.ctypes.data,
                                             capi.MEM_HOST, None), "mxb_stft_process_ragged")
        _check_spectra(fr, dict(mags=mags, re=re), s.oracle(counts, ("mags", "re")))


@pytest.mark.parametrize("n,hop", [(1024, 512), (512, 100)])
def test_ragged_streams_cpp_program(port, tmp_path, n, hop):
    """tests/cpp/ragged_streams.cpp: ragged analysis and resynthesis through the C++ layer (an octave analyser attached at 1024, a Bark
    analyser at 512), every channel against one-channel oracle objects fed only its samples / frames."""
    from test_cpp_dropin import compile_patch
    exe = compile_patch(tmp_path, os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "ragged_streams.cpp"))
    C, calls, bins = 7, 5, n // 2
    rng = np.random.default_rng(n + hop)
    cs = np.stack(_counts(rng, C, hop, calls))
    N = int(cs.sum(axis=0).max()) + 1
    x = W.channel_streams(C, N, seed=17)
    x.tofile(tmp_path / "in.bin"); cs.astype(np.int32).tofile(tmp_path / "counts.bin")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "counts.bin"), str(tmp_path / "out.bin"), str(C), str(N), str(calls),
                        str(n), str(hop)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = open(tmp_path / "out.bin", "rb").read()
    nA = int(np.frombuffer(raw, dtype=np.int32, count=1)[0])
    at = 4

    def take(dtype, count):
        nonlocal at
        a = np.frombuffer(raw, dtype=dtype, count=count, offset=at)
        at += a.nbytes
        return a
    ost = [port.Stft(1, n, hop) for _ in range(C)]
    ois = [port.Istft(1, n, hop) for _ in range(C)]
    ooc = [port.Octave(1, 44100.0, bins, 3) for _ in range(C)] if nA else None
    for o in ooc or ():
        o.config(peak_hold_time=3, peak_decay_rate=0.85)
    off = np.zeros(C, dtype=np.int64)
    for k in range(calls):
        for c in range(C):
            f = int(take(np.int32, 1)[0])
            ro = ost[c].process(x[c:c + 1, off[c]:off[c] + cs[k, c]], want=("mags", "phases"))
            off[c] += cs[k, c]
            assert f == ro["mags"].shape[1], (k, c)
            assert np.array_equal(take(np.float32, f * bins).reshape(f, bins), ro["mags"][0]), (k, c)
            if nA:
                av, pk = (ooc[c].process(ro["mags"]) if f else (np.zeros((1, 0, nA), np.float32),) * 2)
                assert np.array_equal(take(np.float32, f * nA).reshape(f, nA), av[0]) and np.array_equal(take(np.float32, f * nA).reshape(f, nA), pk[0])
            else:
                tt = take(np.float64, f)
                if f:
                    np.testing.assert_allclose(tt, port.bark(ro["mags"][0], 44100, n)[2], rtol=1e-12, atol=0)
            y = take(np.float32, f * hop)
            if f:
                oy = ois[c].process(ro["mags"], ro["phases"])[0]
                assert np.abs(y - oy).max() <= 2e-5 * max(1.0, float(np.abs(oy).max())), (k, c)
    assert at == len(raw)


@pytest.mark.parametrize("n,hop", [(1024, 512), (512, 128), (2048, 441)])
def test_ragged_equal_counts_match_uniform_twin(n, hop):
    """All counts equal: the ragged call gives the bits of mxb_stft_process3 on a twin handle, and the positions stay uniform."""
    C = 13
    x = W.channel_streams(C, 6 * n, seed=n)
    a, b = capi.Stft(C, n, hop), capi.Stft(C, n, hop)
    for lo, hi in ((0, 5), (5, 5 + hop), (5 + hop, 3 * n), (3 * n, 6 * n)):
        ra = a.process(x[:, lo:hi])
        fr, rb = b.process_ragged(np.ascontiguousarray(x[:, lo:hi]), np.full(C, hi - lo, dtype=np.int32))
        f = ra["mags"].shape[1]
        assert np.all(fr == f)
        for k in ("mags", "phases", "re", "im"):
            assert np.array_equal(rb[k][:, :f], ra[k]), k
        assert np.array_equal(a.positions(), b.positions())


def test_uniform_after_ragged_is_a_state_error(port):
    C, n, hop = 4, 512, 128
    s = Streams(port, C, n, hop, seed=1, length=8192)
    st = capi.Stft(C, n, hop)
    counts = np.array([300, 0, 17, 300], dtype=np.int32)
    _check_spectra(*st.process_ragged(s.cut(counts), counts), s.oracle(counts, ("mags", "phases", "re", "im")))
    with pytest.raises(capi.MxbError, match="mxb_stft_process_ragged") as e:
        st.process(np.zeros((C, 128), dtype=np.float32))
    assert "-5" in str(e.value)                                # MXB_ERR_STATE
    assert np.array_equal(st.positions(), s.pos)               # the refused call moved nothing
    # bring every channel to the same position: the uniform calls work again, and match the oracle
    fill = (s.pos.max() - s.pos).astype(np.int32)
    _check_spectra(*st.process_ragged(s.cut(fill), fill), s.oracle(fill, ("mags", "phases", "re", "im")))
    assert len(set(st.positions().tolist())) == 1
    for k in (128, 700, 33):
        counts = np.full(C, k, dtype=np.int32)
        r = st.process(s.cut(counts))
        ro = s.oracle(counts, ("mags", "phases", "re", "im"))
        _check_spectra(np.full(C, r["mags"].shape[1]), r, ro)


def test_invalid_calls_change_nothing(port):
    C, n, hop = 5, 1024, 512
    s = Streams(port, C, n, hop, seed=4, length=20000)
    st = capi.Stft(C, n, hop)
    counts = np.array([600, 0, 2000, 1, 1500], dtype=np.int32)
    fr, r = st.process_ragged(s.cut(counts), counts)
    _check_spectra(fr, r, s.oracle(counts, ("mags", "phases", "re", "im")))
    pos = st.positions()
    bad = np.array([10, -1, 10, 10, 10], dtype=np.int32)
    with pytest.raises(capi.MxbError, match="-1"):
        st.process_ragged(np.zeros((C, 10), dtype=np.float32), bad)
    big = np.array([10, 10, 9000, 10, 10], dtype=np.int32)
    with pytest.raises(capi.MxbError, match="max_frames"):
        st.process_ragged(np.zeros((C, 9000), dtype=np.float32), big, max_frames=4)
    assert np.array_equal(st.positions(), pos)
    counts = np.array([3000, 700, 0, 1023, 5000], dtype=np.int32)
    fr, r = st.process_ragged(s.cut(counts), counts)
    _check_spectra(fr, r, s.oracle(counts, ("mags", "phases", "re", "im")))


@pytest.mark.parametrize("n,hop", [(64, 16), (512, 100), (1024, 256), (1024, 441), (2048, 512)])
def test_istft_ragged(port, n, hop):
    C, bins = 19, n // 2
    rng = np.random.default_rng(n + hop)
    g = capi.Istft(C, n, hop)
    oo = [port.Istft(1, n, hop) for _ in range(C)]
    for call in range(4):
        fr = rng.integers(0, 6, C).astype(np.int32)
        fr[::4] = 0 if call % 2 == 0 else fr[::4]                 # channels with no frame keep their overlap-add buffer
        maxf = int(fr.max()) + 1
        m = (rng.random((C, maxf, bins)) * 4).astype(np.float32)
        p = ((rng.random((C, maxf, bins)) - 0.5) * 6.2).astype(np.float32)
        out = g.process_ragged(m, p, fr)
        for c in range(C):
            f = fr[c]
            ref = oo[c].process(m[c:c + 1, :f], p[c:c + 1, :f])[0] if f else np.zeros(0, dtype=np.float32)
            got = out[c, :f * hop]
            scale = max(1.0, float(np.abs(ref).max(initial=0.0)))
            assert np.abs(got - ref).max(initial=0.0) <= 1e-5 * scale, (c, call)


def test_round_trip_16k_channels_device(port):
    """16 Ki channels, device analysis then device resynthesis with per-channel counts from a seeded RNG; 80 channels checked."""
    import torch
    C, n, hop, calls = 16384, 1024, 512, 4
    rng = np.random.default_rng(16384)
    cs = [rng.integers(0, 3 * hop, C).astype(np.int32) for _ in range(calls)]
    check = np.unique(np.concatenate([[0, C - 1], rng.integers(0, C, 78)]))
    st, ist = capi.Stft(C, n, hop), capi.Istft(C, n, hop)
    length = int(sum(c.max() for c in cs)) + 1
    x = np.zeros((C, length), dtype=np.float32)
    x[check] = W.channel_streams(len(check), length, seed=3)
    rest = np.setdiff1d(np.arange(C), check)
    x[rest] = np.sin(np.arange(length, dtype=np.float32)[None, :] * 0.01 * (1 + rest[:, None] % 7)).astype(np.float32)
    ost = {int(c): port.Stft(1, n, hop) for c in check}
    ois = {int(c): port.Istft(1, n, hop) for c in check}
    off = np.zeros(C, dtype=np.int64)
    maxf = 4
    for counts in cs:
        m = int(counts.max())
        buf = np.zeros((C, m), dtype=np.float32)
        for c in range(C):
            buf[c, :counts[c]] = x[c, off[c]:off[c] + counts[c]]
        d_in = _device(buf)
        d_m = torch.zeros((C, maxf, n // 2), dtype=torch.float32, device="cuda"); d_p = torch.zeros_like(d_m)
        fr = st.process_ragged_device(d_in.data_ptr(), m, 1, counts, maxf, mags=d_m.data_ptr(), phases=d_p.data_ptr())
        d_o = torch.zeros((C, maxf * hop), dtype=torch.float32, device="cuda")
        ist.process_ragged_device(d_m.data_ptr(), d_p.data_ptr(), fr, maxf, d_o.data_ptr())
        torch.cuda.synchronize()
        idx = torch.from_numpy(check).cuda()
        mags, phases, out = d_m[idx].cpu().numpy(), d_p[idx].cpu().numpy(), d_o[idx].cpu().numpy()
        for j, c in enumerate(check):
            ro = ost[int(c)].process(x[c:c + 1, off[c]:off[c] + counts[c]], want=("mags", "phases"))
            f = ro["mags"].shape[1]
            assert fr[c] == f
            assert np.array_equal(mags[j, :f], ro["mags"][0])
            _phase_close(phases[j, :f], ro["phases"][0], ro["mags"][0])
            if f:
                ref = ois[int(c)].process(mags[j:j + 1, :f], phases[j:j + 1, :f])[0]      # the resynthesis of the device's own spectra
                assert np.abs(out[j, :f * hop] - ref).max() <= 1e-5 * max(1.0, float(np.abs(ref).max()))
        off += counts
