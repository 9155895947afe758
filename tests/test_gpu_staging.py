"""Host staging over the life of a handle. Every handle of the library is driven as two twins with the same seeded inputs: one
with its data in host memory, so that each call goes through the handle's staging buffers, the other with its data in device
memory. The calls' sizes rise and then fall, and inputs and outputs are switched on and off between calls, so the staging
buffers grow, are reused while larger than needed, and serve outputs that were absent on the call before. Outputs and state
must be bit-identical after every call.

Output arrays start filled with a sentinel on both twins: rows a call does not write (frames that did not fire, pitch rows
past `frames`) must stay untouched in both."""
import ctypes as C

import numpy as np
import pytest

from maximilian_b200 import capi
from maximilian_b200 import workloads as W

pytestmark = pytest.mark.gpu

L = capi.lib
SENTINEL = -7.25


def _torch():
    import torch
    return torch


def _dev(a):
    """numpy -> a CUDA tensor holding the same bytes (None stays None). Keep the tensor referenced until the call that reads it
    has run: a temporary's memory goes back to torch's allocator at once and may back the next tensor."""
    return None if a is None else _torch().from_numpy(np.ascontiguousarray(a)).cuda()


def _pair(shape, dtype, on=True):
    """one output array per twin, both filled with the sentinel: (numpy host array, CUDA tensor), or (None, None)"""
    if not on:
        return None, None
    h = np.full(shape, SENTINEL, dtype=dtype)
    return h, _dev(h)


def _p(x):
    """host pointer of a numpy array, device pointer of a tensor, NULL for None"""
    if x is None:
        return None
    return C.c_void_p(x.ctypes.data) if isinstance(x, np.ndarray) else C.c_void_p(x.data_ptr())


def _same(h, d, what):
    """the host twin's array (numpy or tensor) against the device twin's tensor, bit for bit"""
    if h is None and d is None:
        return
    _torch().cuda.synchronize()
    hb = h.cpu().numpy() if not isinstance(h, np.ndarray) else h
    assert hb.tobytes() == d.cpu().numpy().tobytes(), what


# ------------------------------------------------------------------------------------------------ bank

# (frames, host mode, out dtype or None, mix, gates, freq_tv, cutoff_tv, delay_size_tv, trig_tv)
BANK_CALLS = [
    (16, "host", np.float64, False, True, False, False, False, False),
    (96, "split_async", np.float32, True, True, True, False, False, False),
    (256, "host", np.float64, True, False, True, True, True, True),
    (200, "split_async", np.float64, True, False, True, True, True, True),
    (64, "host", None, True, True, False, True, False, False),
    (8, "split_async", np.float32, False, False, False, False, True, False),
    (1, "host", np.float32, True, True, True, False, False, False),
]


def test_bank_host_and_split_async_staging_match_device_memory():
    V, cap = 777, 128
    p = W.voice_params(V, seed=5, delay_size=cap, ragged_delay=True)
    twins = [capi.Bank(V, osc="saw", filt="lores", env=True, delay=True, delay_capacity=cap, max_frames=256) for _ in range(2)]
    for b in twins:
        W.configure_bank(b, "lores", p, env=True, delay=True)
    hb, db = twins
    rng = np.random.default_rng(11)
    for k, (B, mode, odt, want_mix, gates, fm, cm, ds, tv) in enumerate(BANK_CALLS):
        on, off = W.gate(V, B, k) if gates else (None, None)
        on = None if on is None else np.ascontiguousarray(on, dtype=np.int32)
        off = None if off is None else np.ascontiguousarray(off, dtype=np.int32)
        f = rng.uniform(30.0, 3000.0, (B, V)) if fm else None
        cu = rng.uniform(200.0, 8000.0, (B, V)) if cm else None
        sz = np.floor(1 + (cap - 1) * rng.random((B, V))) if ds else None
        trig = (rng.random((B, V)) < 0.02).astype(np.uint8) if tv else None
        out_h, out_d = _pair((B, V), odt, odt is not None)
        mix_h, mix_d = _pair((B, 2), np.float64, want_mix)
        f32 = capi.F32 if odt == np.float32 else capi.F64
        if mode == "host":
            mem, out_arg = capi.MEM_HOST, out_h
        else:            # gates, per-sample arrays and the bus in host memory, out on the device; the call does not wait
            mem, out_arg = capi.MEM_SPLIT | capi.MEM_ASYNC, (None if out_h is None else _dev(out_h))
        mod = capi.Modulation(_p(f), _p(cu), _p(sz), _p(trig))
        capi.check(L().mxb_bank_process_mod(hb.h, B, C.byref(mod), _p(on), _p(off), _p(out_arg), f32, _p(mix_h), mem, None), "host twin")
        dev_in = [_dev(a) for a in (f, cu, sz, trig, on, off)]
        dmod = capi.Modulation(*[_p(a) for a in dev_in[:4]])
        capi.check(L().mxb_bank_process_mod(db.h, B, C.byref(dmod), _p(dev_in[4]), _p(dev_in[5]), _p(out_d), f32, _p(mix_d),
                                            capi.MEM_DEVICE, None), "device twin")
        capi.check(L().mxb_ctx_synchronize(hb.ctx.h), "sync")
        _same(out_arg, out_d, f"bank out, call {k}")
        _same(mix_h, mix_d, f"bank mix, call {k}")
        for name in ("filt0", "filt1", "env_amplitude", "env_output", "env_holdcount", "env_flags", "delay_phase", "osc_output"):
            assert hb.get(name).tobytes() == db.get(name).tobytes(), (name, k)
        for v in (0, V // 2, V - 1):
            assert hb.ring(v, cap).tobytes() == db.ring(v, cap).tobytes(), (v, k)


# ------------------------------------------------------------------------------------------------ patch

def test_patch_staging_matches_device_memory():
    from maximilian_b200.patchdef import PatchDef, R, STATE_SLOTS
    d = PatchDef()
    d.stage("env_adsr", d.K(1.0), d.IN("trigger", "u8"), d.P("attack"), d.P("decay"), d.P("sustain"), d.P("release"), d.K(1.0), dst=R(0))
    d.stage("osc", d.IN("freq"), kind="saw", dst=R(1))
    d.stage("filter", R(1), d.IN("cutoff"), d.K(2.0), kind="lores", dst=R(2))
    d.stage("mul", R(2), R(0), dst=R(3))
    d.stage("out", R(3)); d.stage("mix_stereo", R(3), d.P("pan"))
    V = 333
    prm = W.polysynth_params(V, seed=4)
    twins = [capi.Patch(d, V, max_frames=512, mode="interpret") for _ in range(2)]
    for p in twins:
        for k in d.params:
            p.set(k, prm[k])
    hp, dp = twins
    rng = np.random.default_rng(12)
    for k, (B, want_out, want_mix) in enumerate([(16, True, False), (300, True, True), (512, False, True), (40, True, True), (3, True, False)]):
        ins = [(rng.random((B, V)) < 0.05).astype(np.uint8), rng.uniform(40.0, 2000.0, (B, V)), rng.uniform(100.0, 6000.0, (B, V))]
        out_h, out_d = _pair((B, V), np.float64, want_out)
        mix_h, mix_d = _pair((B, 2), np.float64, want_mix)
        ptrs = (C.c_void_p * 3)(*[a.ctypes.data for a in ins])
        capi.check(L().mxb_patch_process(hp.h, B, ptrs, _p(out_h), _p(mix_h), capi.MEM_HOST, None), "host twin")
        dev_in = [_dev(a) for a in ins]
        dptrs = (C.c_void_p * 3)(*[a.data_ptr() for a in dev_in])
        capi.check(L().mxb_patch_process(dp.h, B, dptrs, _p(out_d), _p(mix_d), capi.MEM_DEVICE, None), "device twin")
        _same(out_h, out_d, f"patch out, call {k}")
        _same(mix_h, mix_d, f"patch mix, call {k}")
        for si, (op, *_rest) in enumerate(d.stages):
            for slot in range(STATE_SLOTS.get(op, 0)):
                assert hp.get_state(si, slot).tobytes() == dp.get_state(si, slot).tobytes(), (si, slot, k)


# ------------------------------------------------------------------------------------------------ STFT (+ fused MFCC / octave / Bark)

# (samples, interleaved input, outputs, mfcc, octave, bark). With 1024 channels, 4096 planar samples are 4 Mi samples: the host twin
# takes the sliced three-stream pipeline there.
STFT_CALLS = [
    (300, False, ("mags",), False, False, False),
    (1500, False, ("mags", "phases", "re", "im"), True, False, False),
    (4096, False, ("mags", "mags_db", "flatness", "centroid"), True, True, True),
    (2000, True, ("re", "im", "flatness"), False, True, False),
    (100, False, ("mags",), False, False, True),
    (700, False, ("phases", "centroid"), True, False, True),
]
STFT_FIELDS = ("mags", "phases", "re", "im", "mags_db", "flatness", "centroid")


def test_stft_staging_matches_device_memory_through_the_sliced_pipeline():
    nch, n, hop = 1024, 1024, 512
    bins = n // 2
    twins = [capi.Stft(nch, n, hop) for _ in range(2)]
    octs = [capi.Octave(nch, 48000.0, bins, 3) for _ in range(2)]
    mf = capi.Mfcc(bins, 42, 13)                 # tables only: one handle serves both twins
    nA = octs[0].n_averages
    rng = np.random.default_rng(13)
    for k, (ns, inter, outs, use_mfcc, use_oct, use_bark) in enumerate(STFT_CALLS):
        x = rng.standard_normal((nch, ns)).astype(np.float32)
        if inter:
            x = np.ascontiguousarray(x.T)        # [samples][channels]
        sc, stt = (1, nch) if inter else (ns, 1)
        maxf = ns // hop + 3
        res = []
        for t, mem in enumerate((capi.MEM_HOST, capi.MEM_DEVICE)):
            host = mem == capi.MEM_HOST
            pick = lambda shape, dt, on: _pair(shape, dt, on)[0 if host else 1]
            o = {f: pick((nch, maxf, bins) if f not in ("flatness", "centroid") else (nch, maxf), np.float32, f in outs) for f in STFT_FIELDS}
            co = pick((nch, maxf, mf.coeffs), np.float64, use_mfcc)
            av = pick((nch, maxf, nA), np.float32, use_oct); pk = pick((nch, maxf, nA), np.float32, use_oct and k % 2 == 0)
            bs = pick((nch, maxf, 24), np.float64, use_bark); br = pick((nch, maxf, 24), np.float64, use_bark and k != 4)
            bt = pick((nch, maxf), np.float64, use_bark)
            xin = x if host else _dev(x)
            so = capi.StftOutputs(*[_p(o[f]) for f in STFT_FIELDS], _p(co))
            post = capi.StftPost(octs[t].h if use_oct else None, _p(av), _p(pk), 1 if use_bark else 0, _p(bs), _p(br), _p(bt))
            nf = C.c_int32(0)
            capi.check(L().mxb_stft_process3(twins[t].h, _p(xin), sc, stt, ns, maxf, C.byref(so), C.byref(post),
                                             mf.h if use_mfcc else None, C.byref(nf), mem, None), f"stft twin {t}")
            res.append((nf.value, [o[f] for f in STFT_FIELDS] + [co, av, pk, bs, br, bt]))
        assert res[0][0] == res[1][0], k
        for i, (h, dv) in enumerate(zip(res[0][1], res[1][1])):
            _same(h, dv, f"stft output {i}, call {k}")


# ------------------------------------------------------------------------------------------------ octave analyser, Bark, MFCC

def test_octave_staging_matches_device_memory():
    nch, bands = 96, 512
    twins = [capi.Octave(nch, 44100.0, bands, 3) for _ in range(2)]
    for o in twins:
        o.config(peak_hold_time=3, peak_decay_rate=0.8)
    nA = twins[0].n_averages
    rng = np.random.default_rng(14)
    for k, (F, maxf, want_av, want_pk) in enumerate([(2, 3, True, False), (9, 12, True, True), (30, 30, False, True), (5, 40, True, True),
                                                     (1, 1, True, False)]):
        m = rng.random((nch, maxf, bands), dtype=np.float32) * 3.0      # rows past F (the pitch) are not read
        (ah, ad), (ph, pd) = _pair((nch, maxf, nA), np.float32, want_av), _pair((nch, maxf, nA), np.float32, want_pk)
        capi.check(L().mxb_octave_process(twins[0].h, _p(m), F, maxf, _p(ah), _p(ph), capi.MEM_HOST, None), "host twin")
        dm = _dev(m)
        capi.check(L().mxb_octave_process(twins[1].h, _p(dm), F, maxf, _p(ad), _p(pd), capi.MEM_DEVICE, None), "device twin")
        _same(ah, ad, f"octave averages, call {k}")
        _same(ph, pd, f"octave peaks, call {k}")


def test_bark_staging_matches_device_memory():
    twins = [capi.Bark(44100, 1024) for _ in range(2)]
    rng = np.random.default_rng(15)
    for k, (n, outs) in enumerate([(3, (1, 0, 0)), (500, (1, 1, 1)), (2000, (0, 1, 1)), (40, (1, 0, 1)), (1, (1, 1, 1))]):
        sp = rng.random((n, 512), dtype=np.float32) * 2.0
        pairs = [_pair((n, 24) if i < 2 else (n,), np.float64, on) for i, on in enumerate(outs)]
        capi.check(L().mxb_bark_process(twins[0].h, _p(sp), n, *[_p(h) for h, _ in pairs], capi.MEM_HOST, None), "host twin")
        dsp = _dev(sp)
        capi.check(L().mxb_bark_process(twins[1].h, _p(dsp), n, *[_p(dv) for _, dv in pairs], capi.MEM_DEVICE, None), "device twin")
        for i, (h, dv) in enumerate(pairs):
            _same(h, dv, f"bark output {i}, call {k}")


def test_mfcc_staging_matches_device_memory():
    twins = [capi.Mfcc(512, 42, 13) for _ in range(2)]
    rng = np.random.default_rng(16)
    for k, (n, want_mb) in enumerate([(4, False), (700, True), (3000, True), (64, False), (1, True)]):
        mags = rng.random((n, 512), dtype=np.float32) * 4.0
        (ch, cd), (bh, bd) = _pair((n, 13), np.float64), _pair((n, 42), np.float64, want_mb)
        capi.check(L().mxb_mfcc_process(twins[0].h, _p(mags), n, _p(ch), _p(bh), capi.MEM_HOST, None), "host twin")
        dmags = _dev(mags)
        capi.check(L().mxb_mfcc_process(twins[1].h, _p(dmags), n, _p(cd), _p(bd), capi.MEM_DEVICE, None), "device twin")
        _same(ch, cd, f"mfcc coefficients, call {k}")
        _same(bh, bd, f"mfcc mel bands, call {k}")


# ------------------------------------------------------------------------------------------------ ISTFT

@pytest.mark.parametrize("fft_size", [512, 1024])      # the two-kernel path with its scratch buffer, and the one-kernel K7s
def test_istft_staging_matches_device_memory(fft_size):
    nch, hop = 40, fft_size // 4
    bins = fft_size // 2
    twins = [capi.Istft(nch, fft_size, hop) for _ in range(2)]
    rng = np.random.default_rng(17)
    for k, F in enumerate([1, 7, 30, 12, 2]):
        mags = rng.random((nch, F, bins), dtype=np.float32)
        ph = (rng.random((nch, F, bins), dtype=np.float32) - 0.5) * 6.0
        oh, od = _pair((nch, F * hop), np.float32)
        capi.check(L().mxb_istft_process(twins[0].h, _p(mags), _p(ph), F, _p(oh), capi.MEM_HOST, None), "host twin")
        dmags, dph = _dev(mags), _dev(ph)
        capi.check(L().mxb_istft_process(twins[1].h, _p(dmags), _p(dph), F, _p(od), capi.MEM_DEVICE, None), "device twin")
        _same(oh, od, f"istft out, call {k}")
