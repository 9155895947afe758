"""Every leg bench.py times, at the benchmark's own shape and with the benchmark's own inputs, against the oracle.

The small-bank matrices check every instantiation and branch of the kernels; what changes between them and the benchmark is the
shape: persistent loops that walk many batches per CTA, 64-bit offsets past 2^32 bytes, look-ahead prefetches into multi-GiB
streams, grids and partial counts in the millions. Each test here builds one leg's inputs the way bench.py builds them (its
formulas are restated and cited by line: importing bench.py would set MXB_PATCH_CACHE for the whole process and register an
exit handler), runs the launch path the benchmark times, and checks it at the bars of DESIGN.md §2:

  * a slice of voices or channels -- first, middle and last warps or pair batches -- against the CPU oracle fed the same data;
  * where the inputs are tiled copies of a smaller set (the spectral legs), every channel against its twin, bit for bit, which
    covers every CTA and batch of the grid at no cost; twins cannot see a channel that reads its twin's data, the slices can.

Nothing is timed. Each test frees its device memory before the next one starts; the largest leg (fm_svf: an 8 GiB output and an
8 GiB per-sample frequency stream) sets the module's peak. tests/test_bench_legs_shapes.py keeps the shapes below equal to
bench.py's.
"""
import gc
import math

import numpy as np
import pytest

from maximilian_b200 import capi
from maximilian_b200 import workloads as W
from maximilian_b200.patchdef import STATE_SLOTS as SLOTS
from patch_checks import INT_SLOTS, cmp as _cmp, set_tables as _tables
from test_gpu_bank import _slice_indices

pytestmark = pytest.mark.gpu

# bench.py's shapes (BLOCK, SR, WORKLOADS, MFCC_WL, PATCH_WL, SPEC_WL): the keys that decide what the kernels run
BLOCK = 1024
SR = 48000
BANK_WL = {"svf": dict(voices=1 << 20, osc="saw", filt="svf", env=False, delay=0),
           "biquad": dict(voices=1 << 20, osc="saw", filt="biquad", env=False, delay=0),
           "delay": dict(voices=1 << 18, osc="saw", filt="none", env=True, delay=4096)}
MFCC = dict(channels=65536, fft=1024, hop=512, filters=42, coeffs=40, hops_per_step=8)
PATCH = dict(voices=1 << 18)
SPEC = dict(channels=1 << 14, fft=1024, hop=512, hops_per_step=8)
PAIR_BATCH = 16          # channels one CTA of the streaming transform takes per batch (8 warps, a channel pair each)


@pytest.fixture(autouse=True)
def _free_device_memory():
    """what a test allocated is released before the next one starts (the legs take up to 16 GiB each)"""
    import torch
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _bits(t):
    """the same storage as integers: torch.equal on these is bit equality, NaN included"""
    import torch
    return t.view({8: torch.int64, 4: torch.int32}[t.element_size()])


def _bit_equal(a, b):
    import torch
    return torch.equal(_bits(a), _bits(b))


def _assert_twins(a, period, what):
    """a[c] == a[c % period] bit for bit, for every channel c (the inputs are np.tile copies of `period` channels)"""
    import torch
    v = _bits(a.contiguous()).view(a.shape[0] // period, period, -1)
    bad = (v != v[:1]).any(dim=2)
    if bool(bad.any()):
        first = int(bad.flatten().nonzero()[0, 0])
        raise AssertionError(f"{what}: {int(bad.sum())} channels differ from their twins, the first is channel {first}")
    del v, bad
    torch.cuda.synchronize()


def _vibrato(V, freq, dev):
    """freq_tv[t][v] = f_v * (1 + 0.02 sin(2 pi 5 t / sr + v)), built in place on the device exactly as bench.py's modulated_leg
    builds it (bench.py:1045-1047)"""
    import torch
    ft = torch.arange(BLOCK, dtype=torch.float64, device=dev).mul_(2.0 * math.pi * 5.0 / SR)[:, None].expand(BLOCK, V).contiguous()
    ft.add_(torch.arange(V, dtype=torch.float64, device=dev)[None, :]).sin_().mul_(0.02).add_(1.0)
    ft.mul_(torch.from_numpy(freq).to(dev)[None, :])
    return ft


def _bank(wl, **kw):
    return capi.Bank(wl["voices"], osc=wl["osc"], filt=wl["filt"], env=wl["env"], delay=wl["delay"] > 0,
                     delay_capacity=max(wl["delay"], 1), max_frames=BLOCK, sample_rate=SR, **kw)


def _port_bank(port, wl, n, p, idx):
    o = port.Bank(n, osc=wl["osc"], filt=wl["filt"], env=wl["env"], delay=wl["delay"] > 0, delay_capacity=max(wl["delay"], 1))
    W.configure_bank(o, wl["filt"], {k: v[idx] for k, v in p.items()}, wl["env"], wl["delay"] > 0)
    return o


def test_fm_svf_1m_voices_device_vibrato_vs_oracle_slices(port):
    """bench `modulated.fm_svf`: K1's MOD = 1 instantiation, 1 Mi voices of saw -> SVF with the 5 Hz vibrato built on the device
    (8 GiB of freq_tv: its byte offsets pass 2^32 from frame 512 on), three blocks enqueued on one non-blocking stream with one
    synchronisation. The 2048-voice slice of every block, the phases and the filter state bit for bit against the oracle fed
    the same frequencies."""
    import torch
    wl = BANK_WL["svf"]
    V, B, NB = wl["voices"], BLOCK, 3
    dev = torch.device("cuda", 0)
    p = W.voice_params(V, seed=W.SEED, delay_size=wl["delay"] or 4096)          # bench.py:1039 (rank 0)
    idx = _slice_indices(V)
    tidx = torch.from_numpy(idx).to(dev)
    g = _bank(wl)
    W.configure_bank(g, wl["filt"], p, wl["env"], wl["delay"] > 0)
    out = torch.empty((B, V), dtype=torch.float64, device=dev)
    ft = _vibrato(V, p["freq"], dev)
    st = torch.cuda.Stream()                       # cudaStreamNonBlocking
    torch.cuda.synchronize()
    got = []
    with torch.cuda.stream(st):
        for _ in range(NB):
            g.process_mod_device(B, out_ptr=out.data_ptr(), freq_tv_ptr=ft.data_ptr(), stream=st.cuda_stream)
            got.append(out.index_select(1, tidx))
    st.synchronize()
    fts = ft[:, tidx].cpu().numpy()
    o = _port_bank(port, wl, idx.size, p, idx)
    for blk in range(NB):
        oo, _ = o.process(B, freq_tv=fts)
        gb = got[blk].cpu().numpy()
        assert np.array_equal(gb, oo), f"blk{blk}: slice differs from the oracle in {np.count_nonzero(gb != oo)} samples"
    for name in ("phase", "osc_output", "filt0", "filt1", "filt2"):
        assert np.array_equal(g.get(name)[idx], o.get(name)), name
    del g, out, ft, got


def test_fm_delay_256k_voices_4096_taps_vs_oracle_slices(port):
    """bench `modulated.fm_delay`: K2's modulated instantiation, 256 Ki voices of saw -> ADSR -> 4096-tap delay line (8 GiB of
    rings, uniform schedule: every window takes the modulated body), the leg's gates on every block and the device vibrato, five
    blocks so that the ring index wraps. Output slice, int ring index and envelope state bit for bit against the oracle, the
    full rings of 24 slice voices, and shard invariance: the first 4096 voices as a bank of their own give the same bits."""
    import torch
    wl = BANK_WL["delay"]
    V, B, NB, cap, S = wl["voices"], BLOCK, 5, wl["delay"], 4096
    dev = torch.device("cuda", 0)
    p = W.voice_params(V, seed=W.SEED, delay_size=cap)                           # bench.py:1039 (rank 0)
    on, off = W.gate(V, B, 0, seed=W.SEED)                                       # bench.py:1050, the same gates every block
    idx = _slice_indices(V)
    tidx = torch.from_numpy(idx).to(dev)
    g = _bank(wl)
    W.configure_bank(g, wl["filt"], p, wl["env"], True)
    small = capi.Bank(S, osc=wl["osc"], filt=wl["filt"], env=True, delay=True, delay_capacity=cap, max_frames=B)
    W.configure_bank(small, wl["filt"], {k: v[:S] for k, v in p.items()}, True, True)
    o = _port_bank(port, wl, idx.size, p, idx)
    out = torch.empty((B, V), dtype=torch.float64, device=dev)
    ft = _vibrato(V, p["freq"], dev)
    d_on, d_off = torch.from_numpy(on).to(dev), torch.from_numpy(off).to(dev)
    fts, ft_small = ft[:, tidx].cpu().numpy(), ft[:, :S].cpu().numpy()
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for blk in range(NB):
        g.process_mod_device(B, out_ptr=out.data_ptr(), freq_tv_ptr=ft.data_ptr(), trig_on_ptr=d_on.data_ptr(), trig_off_ptr=d_off.data_ptr(),
                             stream=st.cuda_stream)
        st.synchronize()
        oo, _ = o.process(B, on[idx], off[idx], freq_tv=fts)
        gb = out[:, tidx].cpu().numpy()
        assert np.array_equal(gb, oo), f"blk{blk}: slice differs from the oracle in {np.count_nonzero(gb != oo)} samples"
        os_, _ = small.process(B, on[:S], off[:S], freq_tv=ft_small)
        assert np.array_equal(out[:, :S].cpu().numpy(), os_), f"blk{blk}: shard invariance"
        assert np.array_equal(g.get("delay_phase")[idx], o.get("delay_phase")), f"blk{blk}: ring index"
    for name in ("env_holdcount", "env_flags", "env_amplitude", "env_output", "phase", "osc_output"):
        assert np.array_equal(g.get(name)[idx], o.get(name)), name
    for k in range(0, idx.size, idx.size // 24):
        assert np.array_equal(g.ring(int(idx[k]), cap), o.ring(k, cap)), f"ring of voice {idx[k]}"
    del g, small, out, ft, d_on, d_off


def test_biquad_bank_and_mixdown_1m_voices(port):
    """bench `biquad_bank` and `mixdown`: configs[4]'s saw -> biquad bank at 1 Mi voices with the mixdown leg's parameters
    (bench.py:589), three blocks. With out + bus the output slice is the oracle's bit for bit and the bus is the pan-weighted sum
    of the GPU's own output (fp64 reassociation); the mix-only bank (out = NULL: the kernel bench.py times as `mixdown`, and the
    mix-reduce kernel over its partials) gives the same bus bit for bit, block after block, and the same state."""
    import torch
    wl = BANK_WL["biquad"]
    V, B, NB = wl["voices"], BLOCK, 3
    dev = torch.device("cuda", 0)
    p = W.voice_params(V, seed=W.SEED + 100)
    idx = _slice_indices(V)
    tidx = torch.from_numpy(idx).to(dev)
    g = _bank(wl); m = _bank(wl)
    for b in (g, m):
        W.configure_bank(b, wl["filt"], p, False, False)
    o = _port_bank(port, wl, idx.size, p, idx)
    out = torch.empty((B, V), dtype=torch.float64, device=dev)
    mix = torch.zeros((B, 2), dtype=torch.float64, device=dev)
    mix_only = torch.zeros_like(mix)
    pan = torch.from_numpy(np.clip(p["pan"], 0.0, 1.0)).to(dev)
    gl, gr = torch.sqrt(1.0 - pan), torch.sqrt(pan)
    for blk in range(NB):
        g.process_device(B, out_ptr=out.data_ptr(), mix_ptr=mix.data_ptr())
        m.process_device(B, out_ptr=None, mix_ptr=mix_only.data_ptr())
        torch.cuda.synchronize()
        oo, _ = o.process(B)
        gb = out[:, tidx].cpu().numpy()
        assert np.array_equal(gb, oo), f"blk{blk}: slice differs from the oracle in {np.count_nonzero(gb != oo)} samples"
        torch.testing.assert_close(mix, torch.stack([out @ gl, out @ gr], dim=1), rtol=1e-9, atol=1e-7)
        assert torch.equal(mix_only, mix), f"blk{blk}: the mix-only bus is not the out + mix bus"
    for name in ("phase", "osc_output", "filt0", "filt1"):
        ga = g.get(name)
        assert np.array_equal(ga[idx], o.get(name)), name
        assert np.array_equal(m.get(name), ga), f"{name}: mix-only bank != out + mix bank"
    del g, m, out


def test_headline_f32_out_1m_voices_vs_oracle_slices(port):
    """bench with --f32-out: the headline saw -> SVF bank at 1 Mi voices storing fp32 (K1's paired fp32 stores), three blocks: the
    slice is the oracle's fp64 output rounded to float32, bit for bit, and the fp64 state is the oracle's."""
    import torch
    wl = BANK_WL["svf"]
    V, B, NB = wl["voices"], BLOCK, 3
    dev = torch.device("cuda", 0)
    p = W.voice_params(V, seed=W.SEED)                                             # bench.py:425 (rank 0)
    idx = _slice_indices(V)
    tidx = torch.from_numpy(idx).to(dev)
    g = _bank(wl)
    W.configure_bank(g, wl["filt"], p, False, False)
    o = _port_bank(port, wl, idx.size, p, idx)
    out = torch.empty((B, V), dtype=torch.float32, device=dev)
    assert out.data_ptr() % 16 == 0 and V % 2 == 0                                # the paired-store flavour
    for blk in range(NB):
        g.process_device(B, out_ptr=out.data_ptr(), f32=True)
        torch.cuda.synchronize()
        oo, _ = o.process(B)
        gb = out[:, tidx].cpu().numpy()
        assert np.array_equal(gb, oo.astype(np.float32)), f"blk{blk}: slice is not the oracle's, rounded"
    for name in ("phase", "osc_output", "filt0", "filt1", "filt2"):
        assert np.array_equal(g.get(name)[idx], o.get(name)), name
    del g, out


def _device_triggers(pat, block_index, V, dev):
    """bench.py's patch_leg trigger words (bench.py:918-924): workloads.note_triggers' formula evaluated on the device for every
    voice, packed one bit per voice-sample (voice v = bit v % 32 of word v / 32)"""
    import torch
    weights = torch.ones(32, dtype=torch.int64, device=dev) << torch.arange(32, dtype=torch.int64, device=dev)
    t = (torch.arange(BLOCK, dtype=torch.int64, device=dev) + BLOCK * block_index)[:, None]
    on = (((t + pat[1][None, :]) % pat[0][None, :]) < pat[2][None, :]).to(torch.int64)
    return (on.view(BLOCK, V // 32, 32) * weights).sum(-1).to(torch.int32).contiguous()


def test_patch_bits_256k_voices_fused_and_interpreted(port):
    """bench `patch`: the polysynth with its trigger as packed bits built on the device (first checked against capi.pack_bits of
    workloads.note_triggers: the benchmark's input is the one being checked), on 256 Ki voices, two blocks, on both the generated
    kernel (K8f) and the interpreter (K8). The two agree over all voices on outputs, buses and every state slot, bit for bit;
    a 1536-voice slice -- first, middle and last warps -- matches the oracle at 1e-9 + 1e-12 with the ADSR hold counts and flags
    exact; the bus is the pan-weighted sum of the output."""
    import torch
    V, B = PATCH["voices"], BLOCK
    dev = torch.device("cuda", 0)
    _tables(port)
    d = W.polysynth_patch("bits")
    prm = W.polysynth_params(V, seed=W.SEED)                                        # bench.py:917 (rank 0)
    pat = W.note_pattern(V, seed=W.SEED)
    dpat = tuple(torch.from_numpy(a).to(dev) for a in pat)
    trig = [_device_triggers(dpat, b, V, dev) for b in range(2)]
    chunk = 1 << 15
    for b in range(2):
        ref = np.concatenate([capi.pack_bits(W.note_triggers(pat, B, b, lo, lo + chunk)) for lo in range(0, V, chunk)], axis=1)
        assert np.array_equal(trig[b].cpu().numpy().view(np.uint32), ref), f"blk{b}: device trigger words != pack_bits(note_triggers)"
    sl = np.concatenate([np.arange(0, 512), np.arange(V // 2 - 256, V // 2 + 256), np.arange(V - 512, V)])
    tsl = torch.from_numpy(sl).to(dev)
    modes = ("fused", "interpret")
    pts = {md: capi.Patch(d, V, max_frames=B, sample_rate=SR, mode=md) for md in modes}
    for pt in pts.values():
        for k, v in prm.items():
            pt.set(k, v)
    o = port.Patch(d, sl.size, kind="port")
    for k, v in prm.items():
        o.set(k, v[sl])
    out = {md: torch.empty((B, V), dtype=torch.float64, device=dev) for md in modes}
    mix = {md: torch.zeros((B, 2), dtype=torch.float64, device=dev) for md in modes}
    pan = torch.from_numpy(np.clip(prm["pan"], 0.0, 1.0)).to(dev)
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    pat_sl = tuple(a[sl] for a in pat)
    for blk in range(2):
        for md in modes:
            pts[md].process_device(B, [trig[blk].data_ptr()], out[md].data_ptr(), mix[md].data_ptr(), stream=st.cuda_stream)
        st.synchronize()
        assert _bit_equal(out["fused"], out["interpret"]), f"blk{blk}: fused and interpreted outputs differ"
        assert _bit_equal(mix["fused"], mix["interpret"]), f"blk{blk}: fused and interpreted buses differ"
        ref_mix = torch.stack([out["fused"] @ torch.sqrt(1.0 - pan), out["fused"] @ torch.sqrt(pan)], dim=1)
        torch.testing.assert_close(mix["fused"], ref_mix, rtol=1e-9, atol=1e-9)
        oo, _ = o.process(B, {"trigger": W.note_triggers(pat_sl, B, blk, dtype=np.float64)})
        _cmp(out["fused"][:, tsl].cpu().numpy(), oo, False, f"blk{blk}: slice")
    for si, (op, kind, dst, src) in enumerate(d.stages):
        for s_ in range(SLOTS.get(op, 0)):
            gf = pts["fused"].get_state(si, s_)
            assert np.array_equal(gf, pts["interpret"].get_state(si, s_), equal_nan=True), f"stage {si} slot {s_}: fused != interpreted"
            _cmp(gf[sl], o.get_state(si, s_), s_ in INT_SLOTS.get(op, ()), f"stage {si} slot {s_}")
    del pts, out, mix, trig, dpat


def _channel_pick(C, rng):
    """96 channels: the first two pair batches of the grid, 32 channels drawn from the middle, the last two pair batches"""
    e = 2 * PAIR_BATCH
    return np.concatenate([np.arange(e), np.sort(rng.choice(np.arange(e, C - e), 32, replace=False)), np.arange(C - e, C)])


def test_mfcc_leg_64k_channels_device_steps(port):
    """bench `mfcc` as timed: K4s on device memory, ONE launch over 64 Ki channels per step (4096 pair batches: 15 or 16 per CTA on a 132-SM H100), the
    same 8 hops fed three steps in a row (bench.py:760-768: each step's frames read the assembly buffer the previous step left),
    MFCC 42 -> 40. Every channel's MFCCs equal its twin's (channel c mod 1024) bit for bit at every step; 96 channels against the
    oracle fed the same three steps at 1e-9 + 1e-12. A fourth step also writes the magnitudes: bit for bit on the slice, twins
    over the whole array."""
    import torch
    wl = MFCC
    C, n, hop, H, nc = wl["channels"], wl["fft"], wl["hop"], wl["hops_per_step"], wl["coeffs"]
    dev = torch.device("cuda", 0)
    base = W.channel_streams(1024, H * hop, seed=5)                                # bench.py:760 (rank 0)
    x = torch.from_numpy(np.tile(base, (C // 1024, 1))).to(dev)                    # bench.py:761-762
    pick = _channel_pick(C, np.random.default_rng(40))
    tpick = torch.from_numpy(pick).to(dev)
    st = capi.Stft(C, n, hop); mf = capi.Mfcc(n // 2, wl["filters"], nc, 20.0, 20000.0)
    ost = port.Stft(pick.size, n, hop); omf = port.Mfcc(n // 2, wl["filters"], nc, 20.0, 20000.0, SR)
    xs = base[pick % 1024]
    coeffs = torch.empty((C, H, nc), dtype=torch.float64, device=dev)
    mags = None
    for step in range(4):
        if step == 3:
            mags = torch.empty((C, H, n // 2), dtype=torch.float32, device=dev)
        f = st.process_device(x.data_ptr(), H * hop, 1, H * hop, H, mags=mags.data_ptr() if mags is not None else None, mfcc=mf,
                              coeffs=coeffs.data_ptr())
        assert f == H
        torch.cuda.synchronize()
        _assert_twins(coeffs, 1024, f"step {step}: MFCCs")
        ro = ost.process(xs, want=("mags",))
        assert ro["mags"].shape[1] == H
        co, _ = omf.process(ro["mags"])
        np.testing.assert_allclose(coeffs[tpick].cpu().numpy(), co, rtol=1e-9, atol=1e-12, err_msg=f"step {step}: MFCCs")
        if mags is not None:
            _assert_twins(mags, 1024, f"step {step}: magnitudes")
            assert np.array_equal(mags[tpick].cpu().numpy(), ro["mags"]), f"step {step}: magnitudes"
    del st, mf, x, coeffs, mags


def test_analysis_octave_bark_16k_channels(port):
    """bench `spectral_extras.analysis_octave_bark`: the transform with the octave-analyser (3 per octave) and Bark epilogues
    fused (mxb_stft_process3 on device memory), 16 Ki channels x 8 hops, two calls on the same samples as the timed loop makes
    them (the peaks and hold counters carry). Magnitudes, octave averages and peaks bit for bit on 96 channels against the oracle,
    Bark at 1e-12 relative with the same NaN positions; every array's channels equal their twins' (c mod 1024) bit for bit."""
    import ctypes as C_
    import torch
    wl = SPEC
    C, n, hop, H = wl["channels"], wl["fft"], wl["hop"], wl["hops_per_step"]
    bins = n // 2
    dev = torch.device("cuda", 0)
    base = W.channel_streams(1024, H * hop, seed=11)                               # bench.py:1099 (rank 0)
    x = torch.from_numpy(np.tile(base, (C // 1024, 1))).to(dev)                    # bench.py:1100
    pick = _channel_pick(C, np.random.default_rng(41))
    tpick = torch.from_numpy(pick).to(dev)
    st = capi.Stft(C, n, hop); oc = capi.Octave(C, float(SR), bins, 3)
    nA = oc.n_averages
    ost = port.Stft(pick.size, n, hop); ooc = port.Octave(pick.size, float(SR), bins, 3)
    assert ooc.n_averages == nA
    xs = base[pick % 1024]
    mags = torch.empty((C, H, bins), dtype=torch.float32, device=dev)
    av = torch.empty((C, H, nA), dtype=torch.float32, device=dev); pk = torch.empty_like(av)
    bs = torch.empty((C, H, 24), dtype=torch.float64, device=dev); br = torch.empty_like(bs)
    bt = torch.empty((C, H), dtype=torch.float64, device=dev)
    o = capi.StftOutputs(mags.data_ptr(), None, None, None, None, None, None, None)
    post = capi.StftPost(oc.h, av.data_ptr(), pk.data_ptr(), 1, bs.data_ptr(), br.data_ptr(), bt.data_ptr())
    nf = C_.c_int32(0)
    for call in range(2):
        capi.check(capi.lib().mxb_stft_process3(st.h, C_.c_void_p(x.data_ptr()), H * hop, 1, H * hop, H, C_.byref(o), C_.byref(post), None,
                                                C_.byref(nf), capi.MEM_DEVICE, None), "mxb_stft_process3")
        torch.cuda.synchronize()
        assert nf.value == H
        arrays = dict(mags=mags, averages=av, peaks=pk, bark_specific=bs, bark_relative=br, bark_total=bt)
        for name, a in arrays.items():
            _assert_twins(a, 1024, f"call {call}: {name}")
        got = {name: a[tpick].cpu().numpy() for name, a in arrays.items()}
        om = ost.process(xs, want=("mags",))["mags"]
        oav, opk = ooc.process(om)
        sp, rl, tt = port.bark(om, SR, n)
        assert np.array_equal(got["mags"], om), f"call {call}: magnitudes"
        assert np.array_equal(got["averages"], oav, equal_nan=True), f"call {call}: octave averages"
        assert np.array_equal(got["peaks"], opk, equal_nan=True), f"call {call}: octave peaks"
        for name, ref in (("bark_specific", sp), ("bark_relative", rl), ("bark_total", tt)):
            assert np.array_equal(np.isnan(got[name]), np.isnan(ref)), f"call {call}: {name} NaN positions"
            np.testing.assert_allclose(np.nan_to_num(got[name]), np.nan_to_num(ref), rtol=1e-12, atol=0, err_msg=f"call {call}: {name}")
    del st, oc, x, mags, av, pk, bs, br, bt
