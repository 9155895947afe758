"""The bank's pipelined block loop, as an audio loop or bench.py's e2e legs drive it: block-rate control data uploaded with
mxb_bank_set_param_async while earlier blocks run, MXB_MEM_SPLIT / MXB_MEM_HOST with MXB_MEM_ASYNC, page-locked host memory
(mxb_host_alloc), device-resident modulation streams (process_mod_device), all on a non-blocking stream with one
synchronisation at the end.

Every block gets values of its own, and every block reads from and writes to host buffers of its own, so that no buffer is
rewritten while a copy may still read it (the contract of include/maxib200.h). The pipelined loop must give the bits of the
synchronous loop it replaces, on a twin bank driven by set() + process(), and both agree with the oracle.
"""
import ctypes as C

import numpy as np
import pytest

from maximilian_b200 import capi
from maximilian_b200 import workloads as W
from test_gpu_bank import _slice_indices, trigger_bytes

pytestmark = pytest.mark.gpu

K1_STATE = ("phase", "filt0", "filt1", "filt2", "osc_output")
K2_STATE = ("phase", "osc_output", "env_amplitude", "env_output", "env_holdcount", "env_flags", "delay_phase")


@pytest.fixture
def host():
    """Page-locked host arrays: host.alloc(shape, dtype) from mxb_host_alloc (released with mxb_host_free at teardown),
    host.pinned(shape, dtype) from torch's pinned allocator."""
    import torch

    class Host:
        def __init__(self):
            self.ctx = capi.default_context()
            self.ptrs, self.keep = [], []

        def alloc(self, shape, dtype=np.float64):
            nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
            p = C.c_void_p()
            capi.check(capi.lib().mxb_host_alloc(self.ctx.h, nbytes, C.byref(p)), "mxb_host_alloc")
            self.ptrs.append(p)
            return np.frombuffer((C.c_char * nbytes).from_address(p.value), dtype=dtype).reshape(shape)

        def pinned(self, shape, dtype=np.float64):
            t = torch.zeros(shape, dtype={np.float64: torch.float64, np.int32: torch.int32}[dtype]).pin_memory()
            self.keep.append(t)
            return t.numpy()

    h = Host()
    yield h
    torch.cuda.synchronize()
    for p in h.ptrs:
        capi.check(capi.lib().mxb_host_free(h.ctx.h, p), "mxb_host_free")


def _stream():
    import torch
    return torch.cuda.Stream()          # torch's pool streams are created with cudaStreamNonBlocking


def test_pipelined_k1_loop_is_the_synchronous_loop_1m_voices(port, host):
    """1 Mi voices of saw -> SVF, mix bus only (MXB_MEM_SPLIT | MXB_MEM_ASYNC): process(k), then the uploads of block k+1's
    frequencies and pans, then process(k+1) ... with no host synchronisation. The upload for block k+2 lands in the buffer
    block k reads; a block that has not finished when that copy runs would be computed partly with later values. The final
    phases integrate every block's increments, so a CTA that read the wrong buffer shows there as well as in the bus."""
    V, B, NB = 1 << 20, 1024, 6
    p = W.voice_params(V, seed=W.SEED)
    rng = np.random.default_rng(101)
    freq = host.alloc((NB, V)); pan = host.pinned((NB, V)); mix = host.pinned((NB, B, 2))
    freq[0], pan[0] = p["freq"], p["pan"]
    for k in range(1, NB):
        freq[k] = p["freq"] * (0.5 + rng.random(V)); pan[k] = rng.random(V)
    a = capi.Bank(V, osc="saw", filt="svf", max_frames=B); W.configure_bank(a, "svf", p)
    s = capi.Bank(V, osc="saw", filt="svf", max_frames=B); W.configure_bank(s, "svf", p)
    import torch
    st = _stream()
    torch.cuda.synchronize()
    for k in range(NB):
        if k:
            a.set_host_array("freq", freq[k], stream=st.cuda_stream)
            a.set_host_array("pan", pan[k], stream=st.cuda_stream)
        a.process_split(B, None, mix[k], stream=st.cuda_stream, wait=False)
    st.synchronize()
    idx = _slice_indices(V)
    o = port.Bank(idx.size, osc="saw", filt="svf"); W.configure_bank(o, "svf", {k_: v[idx] for k_, v in p.items()})
    for k in range(NB):
        s.set("freq", freq[k]); s.set("pan", pan[k])
        _, ms = s.process(B, want_out=False, want_mix=True)
        assert np.array_equal(mix[k], ms), f"block {k}: the pipelined bus differs from the synchronous one"
        o.set("freq", freq[k][idx]); o.set("pan", pan[k][idx])
        o.process(B, want_out=False)
    for name in K1_STATE:
        ga = a.get(name)
        assert np.array_equal(ga, s.get(name)), f"{name}: pipelined != synchronous ({np.count_nonzero(ga != s.get(name))} voices)"
        assert np.array_equal(ga[idx], o.get(name)), f"{name}: slice differs from the oracle"
    assert np.array_equal(a.get("freq"), freq[NB - 1])


def test_pipelined_k2_loop_is_the_synchronous_loop(port, host):
    """The same on the delay-line kernel: 256 Ki voices of saw -> ADSR -> maxiDelayline::dl on uniform 256-slot rings, with
    frequency, pan and feedback uploaded asynchronously for every block. Bus, ring index, envelope state and the rings of
    sampled voices are those of the synchronous loop, and a 2048-voice slice is the oracle's."""
    V, B, NB, cap = 1 << 18, 1024, 6, 256
    p = W.voice_params(V, seed=W.SEED + 5, delay_size=cap)
    rng = np.random.default_rng(102)
    names = ("freq", "pan", "delay_feedback")
    vals = {n: (host.alloc((NB, V)) if n == "delay_feedback" else host.pinned((NB, V))) for n in names}
    for n in names:
        vals[n][0] = p[n]
    for k in range(1, NB):
        vals["freq"][k] = p["freq"] * (0.5 + rng.random(V)); vals["pan"][k] = rng.random(V)
        vals["delay_feedback"][k] = 0.1 + 0.8 * rng.random(V)
    on0, off0 = W.gate(V, B, 0)
    on, off = host.pinned((V,), np.int32), host.pinned((V,), np.int32)
    on[:], off[:] = on0, off0
    mix = host.pinned((NB, B, 2))
    kw = dict(osc="saw", env=True, delay=True, delay_capacity=cap, max_frames=B)
    a = capi.Bank(V, **kw); s = capi.Bank(V, **kw)
    for b in (a, s):
        W.configure_bank(b, "none", p, env=True, delay=True)
    import torch
    st = _stream()
    torch.cuda.synchronize()
    for k in range(NB):
        if k:
            for n in names:
                a.set_host_array(n, vals[n][k], stream=st.cuda_stream)
        g = (on, off) if k == 0 else (None, None)           # one note, at block 0; the rest is the release and the echoes
        a.process_split(B, None, mix[k], *g, stream=st.cuda_stream, wait=False)
    st.synchronize()
    idx = _slice_indices(V)
    o = port.Bank(idx.size, **{k_: v for k_, v in kw.items() if k_ != "max_frames"})
    W.configure_bank(o, "none", {k_: v[idx] for k_, v in p.items()}, env=True, delay=True)
    for k in range(NB):
        for n in names:
            s.set(n, vals[n][k]); o.set(n, vals[n][k][idx])
        g = (on0, off0) if k == 0 else (None, None)
        _, ms = s.process(B, *g, want_out=False, want_mix=True)
        assert np.array_equal(mix[k], ms), f"block {k}: the pipelined bus differs from the synchronous one"
        o.process(B, *(x[idx] if x is not None else None for x in g), want_out=False)
    for name in K2_STATE:
        ga = a.get(name)
        assert np.array_equal(ga, s.get(name)), f"{name}: pipelined != synchronous ({np.count_nonzero(ga != s.get(name))} voices)"
        assert np.array_equal(ga[idx], o.get(name)), f"{name}: slice differs from the oracle"
    for j in range(0, idx.size, idx.size // 24):
        v = int(idx[j])
        assert np.array_equal(a.ring(v, cap), s.ring(v, cap)), f"ring of voice {v}: pipelined != synchronous"
        assert np.array_equal(a.ring(v, cap), o.ring(j, cap)), f"ring of voice {v} differs from the oracle"
    assert np.any(a.ring(int(idx[0]), cap) != 0.0)


@pytest.mark.parametrize("delay", [False, True], ids=["k1", "k2"])
def test_host_async_blocks_are_the_synchronous_blocks(port, host, delay):
    """MXB_MEM_HOST | MXB_MEM_ASYNC: gates in, the whole `out` and the bus out, through page-locked host buffers of their own for
    every block, the block's frequencies uploaded asynchronously, one synchronisation after the last block."""
    V, B, NB, cap = 2500, 400, 4, 128
    filt = "none" if delay else "lores"
    p = W.voice_params(V, seed=103, delay_size=cap)
    rng = np.random.default_rng(103)
    freq = host.alloc((NB, V)); on = host.pinned((NB, V), np.int32); off = host.pinned((NB, V), np.int32)
    out = host.pinned((NB, B, V)); mix = host.pinned((NB, B, 2))
    freq[0] = p["freq"]
    for k in range(NB):
        if k:
            freq[k] = p["freq"] * (0.5 + rng.random(V))
        on[k], off[k] = W.gate(V, B, 4 * k if k % 2 == 0 else 1, seed=103 + k)
    kw = dict(osc="saw", filt=filt, env=True, delay=delay, delay_capacity=cap, max_frames=B)
    a = capi.Bank(V, **kw); s = capi.Bank(V, **kw)
    o = port.Bank(V, **{k_: v for k_, v in kw.items() if k_ != "max_frames"})
    for b in (a, s, o):
        W.configure_bank(b, filt, p, env=True, delay=delay)
    import torch
    st = _stream()
    torch.cuda.synchronize()
    P = lambda x: C.c_void_p(x.ctypes.data)
    for k in range(NB):
        if k:
            a.set_host_array("freq", freq[k], stream=st.cuda_stream)
        capi.check(capi.lib().mxb_bank_process(a.h, B, P(on[k]), P(off[k]), P(out[k]), capi.F64, P(mix[k]),
                                               capi.MEM_HOST | capi.MEM_ASYNC, C.c_void_p(st.cuda_stream)), "mxb_bank_process")
    st.synchronize()
    for k in range(NB):
        for b in (s, o):
            b.set("freq", freq[k])
        os_, ms = s.process(B, on[k], off[k], want_mix=True)
        oo, mo = o.process(B, on[k], off[k], want_mix=True)
        assert np.array_equal(out[k], os_) and np.array_equal(mix[k], ms), f"block {k}: host-async != synchronous"
        assert np.array_equal(out[k], oo), f"block {k}: differs from the oracle"
        np.testing.assert_allclose(mix[k], mo, rtol=1e-9, atol=1e-11)
    for name in K2_STATE if delay else K1_STATE:
        assert np.array_equal(a.get(name), s.get(name)), name


def test_later_parameter_call_wins(host):
    """mxb_bank_set_param_async: of several calls for one parameter before a block, the later one is in force for that block,
    whatever the calls' kinds -- host upload, device copy, synchronous set_param. Each block is compared with a twin bank that
    was given the expected values synchronously; get("freq") returns them."""
    import torch
    V, B = 1000, 64
    rng = np.random.default_rng(104)
    h = host.alloc((8, V))
    h[:] = 30.0 + 3000.0 * rng.random((8, V))
    dv = torch.from_numpy(h.copy()).cuda()
    a = capi.Bank(V, osc="saw", max_frames=B); t = capi.Bank(V, osc="saw", max_frames=B)
    mix = host.pinned((B, 2))
    st = _stream()
    torch.cuda.synchronize()
    sp = st.cuda_stream

    def host_async(i):
        a.set_host_array("freq", h[i], stream=sp)

    def dev_async(i):
        capi.check(capi.lib().mxb_bank_set_param_async(a.h, capi.P["freq"], C.c_void_p(dv[i].data_ptr()), capi.MEM_DEVICE,
                                                       C.c_void_p(sp)), "mxb_bank_set_param_async")

    def block(i, what):
        a.process_split(B, None, mix, stream=sp, wait=True)
        t.set("freq", h[i]); _, mt = t.process(B, want_out=False, want_mix=True)
        assert np.array_equal(mix, mt), f"{what}: the block did not run with the values of the later call"
        assert np.array_equal(a.get("phase"), t.get("phase")), what
        assert np.array_equal(a.get("freq"), h[i]), what

    a.set("freq", h[7]); block(7, "set_param")
    host_async(0); dev_async(1); block(1, "host-async, then device-async")
    host_async(2); block(2, "a host upload after a dropped one")
    host_async(3); a.set("freq", h[4]); block(4, "host-async, then set_param")
    host_async(5); host_async(6); block(6, "two host uploads")
    dev_async(0); host_async(3); block(3, "device-async, then host-async")
    host_async(5); dev_async(2); host_async(7); block(7, "host-async, device-async, host-async")
    block(7, "no new values: the last ones stay in force")


@pytest.mark.parametrize("delay", [False, True], ids=["k1", "k2"])
def test_process_mod_device_on_a_stream_is_process(delay):
    """bench.py's `modulated` path: per-sample frequency, cutoff and trigger streams (and, with a delay line, the delay size)
    resident on the device, three blocks enqueued on a non-blocking stream with one synchronisation at the end -- the bits
    of Bank.process with the same arrays from host memory."""
    import torch
    from test_oracle_vs_reference import cutoff_sweeps, flanger_sizes, fm_frequencies
    V, B, NB, cap = 777, 300, 3, 128
    dev = torch.device("cuda", 0)
    filt = "lores" if delay else "svf"
    kw = dict(osc="saw", filt=filt, env=True, delay=delay, delay_capacity=cap, max_frames=B)
    p = W.voice_params(V, seed=105, delay_size=cap, ragged_delay=True)
    g = capi.Bank(V, **kw); h = capi.Bank(V, **kw)
    for b in (g, h):
        W.configure_bank(b, filt, p, env=True, delay=delay)
    ins = []
    for blk in range(NB):
        d = dict(freq_tv=fm_frequencies(V, B, blk), cutoff_tv=cutoff_sweeps(V, B, blk), trig_tv=trigger_bytes(V, B, blk, seed=11))
        if delay:
            d["delay_size_tv"] = flanger_sizes(V, B, blk, cap)
        ins.append(d)
    dins = [{k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in d.items()} for d in ins]
    out = torch.full((NB, B, V), np.nan, dtype=torch.float64, device=dev)
    mix = torch.full((NB, B, 2), np.nan, dtype=torch.float64, device=dev)
    st = _stream()
    torch.cuda.synchronize()
    for blk in range(NB):
        d = dins[blk]
        g.process_mod_device(B, out_ptr=out[blk].data_ptr(), mix_ptr=mix[blk].data_ptr(), freq_tv_ptr=d["freq_tv"].data_ptr(),
                             cutoff_tv_ptr=d["cutoff_tv"].data_ptr(), trig_tv_ptr=d["trig_tv"].data_ptr(),
                             delay_size_tv_ptr=d["delay_size_tv"].data_ptr() if delay else None, stream=st.cuda_stream)
    st.synchronize()
    for blk in range(NB):
        oh, mh = h.process(B, want_mix=True, **ins[blk])
        assert np.array_equal(out[blk].cpu().numpy(), oh), f"block {blk}: out"
        assert np.array_equal(mix[blk].cpu().numpy(), mh), f"block {blk}: mix"
    for name in (K2_STATE + ("filt0", "filt1")) if delay else K1_STATE + ("env_amplitude", "env_flags"):
        assert np.array_equal(g.get(name), h.get(name)), name
    if delay:
        for v in range(0, V, 37):
            assert np.array_equal(g.ring(v, cap), h.ring(v, cap)), v
