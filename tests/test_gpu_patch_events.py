"""Control events (MXB_IN_EVENTS) on the GPU, both ways a patch runs: every case is held BIT FOR BIT against the same stage list fed the
equivalent dense f64 stream (events_checks.events_to_dense) -- output, bus, every state word, the rings and the held values. The dense
path is pinned to the port and the port to the reference by the other patch tests, so this pins the events path to both."""
import ctypes as C

import numpy as np
import pytest

import events_checks as EV
from patch_checks import ring_stages, set_tables
from maximilian_b200 import capi
from maximilian_b200 import workloads as W
from maximilian_b200.patchdef import STATE_SLOTS as SLOTS, PatchDef, R

pytestmark = pytest.mark.gpu

MODES = ["fused", "interpret"]
OTHER = {"fused": "interpret", "interpret": "fused"}


def _same(a, b, what):
    assert np.array_equal(a, b, equal_nan=True), f"{what}: not bit-identical"


def _same_state(a, b, d, V, taps, what):
    for si, (op, *_) in enumerate(d.stages):
        for sl in range(SLOTS.get(op, 0)):
            _same(a.get_state(si, sl), b.get_state(si, sl), f"{what}: stage {si} slot {sl}")
    for si, nl in ring_stages(d):
        for v in sorted({0, 1, 31, 32, V // 2, V - 1} & set(range(V))):
            _same(a.ring(si, v, taps * nl), b.ring(si, v, taps * nl), f"{what}: ring {si} voice {v}")


@pytest.mark.parametrize("V", [1, 31, 300, 4096])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", EV.CASES, ids=lambda c: c[0])
def test_events_equal_the_dense_stream(case, mode, V):
    """blocks of 1 to 1024 frames over several calls, random lists (unsorted, repeated frames, frames < 0 and >= n, empty voices, a call
    without any event); the events patch switches mode after the third call, the dense twin stays in `mode`"""
    name, build, values, taps = case
    rng = np.random.default_rng(1000 + V)
    ev = capi.Patch(build("events"), V, max_frames=1024, delay_taps=taps, mode=mode)
    de = capi.Patch(build("f64"), V, max_frames=1024, delay_taps=taps, mode=mode)
    for k, x in EV._f(rng, V).items():
        if k in ev.defn.params:
            ev.set(k, x); de.set(k, x)
    held = np.zeros(V)
    for call, n in enumerate([1, 17, 1024, 5, 300, 64]):
        if call == 3:
            ev.set_mode(OTHER[mode])
        lists = [[] for _ in range(V)] if call == 4 else EV.random_events(rng, V, n, values=values)
        first, frame, value = capi.pack_events(lists)
        dense, held = EV.events_to_dense(first, frame, value, n, held)
        oe, me = ev.process(n, {"x": (first, frame, value)}, want_mix=True)
        od, md = de.process(n, {"x": dense}, want_mix=True)
        _same(oe, od, f"{name} call {call} out"); _same(me, md, f"{name} call {call} bus")
        _same(ev.get_held("x"), held, f"{name} call {call} held")
    _same_state(ev, de, ev.defn, V, taps, name)


@pytest.mark.parametrize("mode", MODES)
def test_held_values_round_trip_and_start_a_voice(mode):
    """set_held starts every voice at its own frequency without any event; get_held returns what set_held wrote and what the events left"""
    V, n = 300, 128
    rng = np.random.default_rng(5)
    ev = capi.Patch(EV._frequency("events"), V, max_frames=n, mode=mode)
    de = capi.Patch(EV._frequency("f64"), V, max_frames=n, mode=mode)
    for p in (ev, de):
        p.set("pan", 0.5)
    assert np.array_equal(ev.get_held("x"), np.zeros(V))
    start = rng.uniform(50.0, 1000.0, V)
    ev.set_held("x", start)
    _same(ev.get_held("x"), start, "set_held -> get_held")
    oe, _ = ev.process(n, {"x": [[] for _ in range(V)]})
    od, _ = de.process(n, {"x": np.broadcast_to(start, (n, V))})
    _same(oe, od, "held start")
    lists = EV.random_events(rng, V, n, values=lambda r, k: r.uniform(50.0, 1000.0, k))
    dense, held = EV.events_to_dense(*capi.pack_events(lists), n, start)
    oe, _ = ev.process(n, {"x": lists}); od, _ = de.process(n, {"x": dense})
    _same(oe, od, "after events"); _same(ev.get_held("x"), held, "held after events")
    with pytest.raises(capi.MxbError, match="-> -1"):
        capi.check(capi.lib().mxb_patch_get_held(de.h, 0, capi._np_ptr(np.empty(V)), capi.MEM_HOST), "get_held of a dense stream")
    with pytest.raises(capi.MxbError, match="-> -1"):
        capi.check(capi.lib().mxb_patch_set_held(ev.h, 1, capi._np_ptr(np.empty(V)), capi.MEM_HOST), "set_held of a stream that does not exist")


def _process_raw(p, n, descs, mem, out, mix):
    ptrs = (C.c_void_p * len(descs))(*[C.addressof(x) for x in descs])
    return capi.lib().mxb_patch_process(p.h, n, ptrs, out, mix, mem, None)


@pytest.mark.parametrize("mode", MODES)
def test_host_memory_equals_device_memory(mode):
    """the same calls with the three arrays in host memory and in device memory (no staging): the same bits. In device memory a voice
    whose first[v+1] < first[v] has no events (the host path refuses such a list)."""
    import torch
    V, taps = 1000, 64
    rng = np.random.default_rng(8)
    d = EV._delay_size("events")
    a = capi.Patch(d, V, max_frames=512, delay_taps=taps, mode=mode); b = capi.Patch(d, V, max_frames=512, delay_taps=taps, mode=mode)
    prm = EV._f(rng, V)
    for p in (a, b):
        p.set("f", prm["f"]); p.set("pan", prm["pan"])
    for call, n in enumerate([512, 3, 200]):
        lists = EV.random_events(rng, V, n, values=lambda r, k: r.integers(1, 64, k).astype(np.float64))
        first, frame, value = capi.pack_events(lists)
        if call == 2:                   # one voice with first[v+1] < first[v]: it has no events; its neighbours' ranges move with it
            v = next(v for v in range(1, V - 1) if first[v] >= 1)
            first[v + 1] = first[v] - 1
            lists = [[(int(frame[i]), float(value[i])) for i in range(first[u], first[u + 1])] for u in range(V)]
            assert lists[v] == []
        dev = [torch.from_numpy(x).cuda() for x in (first, frame, value)]
        ob = torch.empty((n, V), dtype=torch.float64, device="cuda"); mb = torch.empty((n, 2), dtype=torch.float64, device="cuda")
        desc = capi.Events(dev[0].data_ptr(), dev[1].data_ptr(), dev[2].data_ptr())
        capi.check(_process_raw(b, n, [desc], capi.MEM_DEVICE, C.c_void_p(ob.data_ptr()), C.c_void_p(mb.data_ptr())), "device process")
        torch.cuda.synchronize()
        oa, ma = a.process(n, {"x": lists}, want_mix=True)
        _same(ob.cpu().numpy(), oa, f"call {call} out"); _same(mb.cpu().numpy(), ma, f"call {call} bus")
        _same(b.get_held("x"), a.get_held("x"), f"call {call} held")
    _same_state(a, b, d, V, taps, "host vs device")


def test_malformed_descriptors_are_refused_and_change_nothing():
    V, n = 40, 32
    p = capi.Patch(EV._frequency("events"), V, max_frames=n, mode="interpret")
    p.set("pan", 0.5)
    p.set_held("x", 3.0)
    first, frame, value = capi.pack_events([[(1, 440.0)]] * V)
    out = np.empty((n, V))
    bad = {
        "NULL first": capi.Events(None, frame.ctypes.data, value.ctypes.data),
        "NULL frame": capi.Events(first.ctypes.data, None, value.ctypes.data),
        "NULL value": capi.Events(first.ctypes.data, frame.ctypes.data, None),
    }
    dec = first.copy(); dec[5] = dec[4] - 1
    neg = first - 1
    bad["decreasing first"] = capi.Events(dec.ctypes.data, frame.ctypes.data, value.ctypes.data)
    bad["negative first[0]"] = capi.Events(neg.ctypes.data, frame.ctypes.data, value.ctypes.data)
    for what, desc in bad.items():
        assert _process_raw(p, n, [desc], capi.MEM_HOST, capi._np_ptr(out), None) == -1, what
    ptrs = (C.c_void_p * 1)(None)
    assert capi.lib().mxb_patch_process(p.h, n, ptrs, capi._np_ptr(out), None, capi.MEM_HOST, None) == -1, "NULL descriptor"
    assert np.array_equal(p.get_held("x"), np.full(V, 3.0))
    assert np.array_equal(p.get_state(0, 0), np.zeros(V))                # no kernel ran
    good = capi.Events(first.ctypes.data, frame.ctypes.data, value.ctypes.data)
    assert _process_raw(p, n, [good], capi.MEM_HOST, capi._np_ptr(out), None) == 0
    assert np.array_equal(p.get_held("x"), np.full(V, 440.0))


def test_interpreter_budget_counts_events_streams():
    """200 doubles per voice fit and 201 are refused, with the 3 words of each events stream counted; the 201-double stage list over
    dense streams (no events words) fits. The 200-double patch runs on the interpreter bit for bit as the generated kernel does."""
    V, n = 200, 64
    rng = np.random.default_rng(3)
    with pytest.raises(capi.MxbError, match="-> -4"):
        capi.Patch(EV.budget_patch(True, "events"), V, max_frames=n, delay_taps=8, mode="interpret")
    capi.Patch(EV.budget_patch(True, "f64"), V, max_frames=n, delay_taps=8, mode="interpret")
    d200 = EV.budget_patch(False, "events")
    a = capi.Patch(d200, V, max_frames=n, mode="interpret"); b = capi.Patch(d200, V, max_frames=n, mode="fused")
    for p in (a, b):
        for j in range(32):
            p.set(f"p{j}", 100.0 + j)
    ins = {f"e{j}": EV.random_events(rng, V, n, values=lambda r, k: r.uniform(0.0, 500.0, k)) for j in range(8)}
    oa, _ = a.process(n, ins); ob, _ = b.process(n, ins)
    _same(oa, ob, "budget patch: interpreter vs fused")
    for j in range(8):
        _same(a.get_held(f"e{j}"), b.get_held(f"e{j}"), f"held e{j}")


def _slice(ev, sl):
    first, frame, value = ev
    idx = np.concatenate([np.arange(first[v], first[v + 1]) for v in sl])
    f2 = np.zeros(sl.size + 1, dtype=np.int32); f2[1:] = np.cumsum(first[sl + 1] - first[sl])
    return f2, frame[idx], value[idx]


def test_full_size_polysynth_256k_voices_events_vs_oracle_slices(port):
    """The polysynth at the bench's size (262 144 voices x 1024 frames) with pitch and trigger as events, the generated kernel, two
    blocks: a 1536-voice slice -- first, middle and last warps -- against the oracle fed the dense streams of those voices (1e-9, the
    envelope's flags and hold counts exact), the interpreter on the slice bit for bit, and the held values."""
    V, B = 262144, 1024
    set_tables(port)
    prm = W.polysynth_params(V, seed=31)
    prm = {k: prm[k] for k in ("attack", "decay", "sustain", "release", "pan")}
    sl = np.concatenate([np.arange(0, 512), np.arange(V // 2 - 256, V // 2 + 256), np.arange(V - 512, V)])
    g = capi.Patch(W.polysynth_pitch_patch("events", "events"), V, max_frames=B, mode="fused")
    o = port.Patch(W.polysynth_pitch_patch("f64", "f64"), sl.size, kind="port")
    gi = capi.Patch(W.polysynth_pitch_patch("events", "events"), sl.size, max_frames=B, mode="interpret")
    for k, v in prm.items():
        g.set(k, v); o.set(k, v[sl]); gi.set(k, v[sl])
    held = {"pitch": np.zeros(sl.size), "trigger": np.zeros(sl.size)}
    for blk in range(2):
        pe, te = W.note_events(V, B, blk, seed=77)
        og, _ = g.process(B, {"pitch": pe, "trigger": te})
        ps, ts = _slice(pe, sl), _slice(te, sl)
        dp, held["pitch"] = EV.events_to_dense(*ps, B, held["pitch"])
        dt, held["trigger"] = EV.events_to_dense(*ts, B, held["trigger"])
        oo, _ = o.process(B, {"pitch": dp, "trigger": dt})
        oi, _ = gi.process(B, {"pitch": ps, "trigger": ts})
        np.testing.assert_allclose(og[:, sl], oo, rtol=1e-9, atol=1e-12)
        _same(og[:, sl], oi, f"block {blk}: fused vs interpreter")
    for slot in (2, 3):
        assert np.array_equal(g.get_state(0, slot)[sl], o.get_state(0, slot))
    for k in held:
        _same(g.get_held(k)[sl], held[k], f"held {k}")
