"""Per-rank bodies of test_gpu_exchange_one_device.py: every rank of the world shares one device, owns a voice shard, and runs the handle
under test (the exchange attached) next to a twin (the same shard, the same calls, no exchange). The twin's bus is the lane the rank
contributes, so the parent can rebuild the exchanged bus bit for bit: ((0.0 + L_0) + L_1) + ... in rank order.

The children import this module by name (spawn start method): it needs no device at import time, and only S8 imports torch."""
import os
import traceback

import numpy as np

from maximilian_b200 import capi
from maximilian_b200 import workloads as W
from maximilian_b200.patchdef import STATE_SLOTS
from maximilian_b200.shard import shard_range

B = 256                         # the exchange holds 2 * B doubles: a B-frame block fills it
MAX_FRAMES = B + 1              # every handle accepts one frame more than the exchange holds (S4)
TIMEOUT_MS = "20000"            # ranks time-slice one device: a peer that is merely descheduled must not read as dead

S1_V, S1_BLOCKS = 6001, [1, 256, 7, 256, 129, 33]
S2_V, S2_BLOCKS, S2_CAP = 1000, [256, 64, 256, 100, 256], 512
S3_BLOCKS = [256, 1, 65, 256]
S4_CALLS = [64, B + 1, 256, B + 1, 1]
S5_V, S5_BLOCKS = 1500, [256, 100, 256, 37]
S6_V, S6_BLOCKS = 1200, [256, 128, 256]
S7_BANK_BLOCKS, S7_PATCH_BLOCKS = [128, 256], [256, 64]

BANK_STATE = ("phase", "filt0", "filt1", "filt2", "osc_output", "env_amplitude", "env_output", "env_holdcount", "env_flags", "delay_phase")


def slice_events(ev, lo, hi):
    """The CSR triple (first, frame, value) of voices [lo, hi) of a whole-bank events stream."""
    first, frame, value = ev
    a, b = int(first[lo]), int(first[hi])
    return (np.ascontiguousarray(first[lo:hi + 1] - first[lo], dtype=np.int32), np.ascontiguousarray(frame[a:b]),
            np.ascontiguousarray(value[a:b]))


def bank_state(b, ring=0):
    st = {}
    for k in BANK_STATE:
        try:
            st[k] = b.get(k)
        except capi.MxbError:          # a state array this bank does not have
            pass
    if ring:
        st["ring"] = np.stack([b.ring(v, ring) for v in sorted({0, b.V // 2, b.V - 1})])
    return st


def patch_state(p):
    st = {f"stage {si} slot {sl}": p.get_state(si, sl) for si, (op, *_) in enumerate(p.defn.stages) for sl in range(STATE_SLOTS.get(op, 0))}
    for n in p.defn.inputs:
        if p.defn.input_types.get(n) == "events":
            st[f"held {n}"] = p.get_held(n)
    return st


def _part(bus, twin, state, out=None, twin_out=None):
    return dict(bus=bus, twin=twin, state=state, out=out, twin_out=twin_out)


def _saw_biquad(ctx, V, rank, world, seed=3):
    lo, hi = shard_range(V, rank, world)
    p = {k: v[lo:hi] for k, v in W.voice_params(V, seed=seed).items()}
    pair = [capi.Bank(hi - lo, osc="saw", filt="biquad", max_frames=MAX_FRAMES, ctx=ctx) for _ in range(2)]
    for b in pair:
        W.configure_bank(b, "biquad", p)
    return pair


def _bus_blocks(main, twin, blocks):
    bus, tw = [], []
    for n in blocks:
        bus.append(main.process(n, want_out=False, want_mix=True)[1])
        tw.append(twin.process(n, want_out=False, want_mix=True)[1])
    return bus, tw


def s1_bank_bus(rank, world, ctx, ex):
    """saw -> biquad, uneven shards, blocks of 1 to 256 frames: a full bus, short buses, rows past one stride of the final loop"""
    main, twin = _saw_biquad(ctx, S1_V, rank, world)
    ex.attach(main)
    bus, tw = _bus_blocks(main, twin, S1_BLOCKS)
    return {"parts": {"main": _part(bus, tw, (bank_state(main), bank_state(twin)))}}


def _delay_bank(ctx, V, rank, world, seed):
    lo, hi = shard_range(V, rank, world)
    p = {k: v[lo:hi] for k, v in W.voice_params(V, seed=seed, delay_size=S2_CAP, ragged_delay=True).items()}
    main, twin = (capi.Bank(hi - lo, osc="saw", filt="none", env=True, delay=True, delay_capacity=S2_CAP, max_frames=MAX_FRAMES, ctx=ctx)
                  for _ in range(2))
    for b in (main, twin):
        W.configure_bank(b, "none", p, env=True, delay=True)
    return main, twin, lo, hi


def delay_gates(V, n, k, seed):
    """whole-bank gates of block k: every block carries a note"""
    return W.gate(V, n, 4 * k, seed=seed)


def _delay_blocks(main, twin, lo, hi, V, blocks, seed):
    bus, tw, out, tout = [], [], [], []
    for k, n in enumerate(blocks):
        on, off = delay_gates(V, n, k, seed)
        o, m = main.process(n, on[lo:hi], off[lo:hi], want_out=True, want_mix=True)
        to, t = twin.process(n, on[lo:hi], off[lo:hi], want_out=True, want_mix=True)
        bus.append(m); tw.append(t); out.append(o); tout.append(to)
    return _part(bus, tw, (bank_state(main, S2_CAP), bank_state(twin, S2_CAP)), out, tout)


def s2_delay_bank(rank, world, ctx, ex):
    """saw -> ADSR -> maxiDelayline::dl (the delay kernel and its own warp count), gates sliced from whole-bank arrays, out and bus"""
    main, twin, lo, hi = _delay_bank(ctx, S2_V, rank, world, seed=5)
    ex.attach(main)
    return {"parts": {"main": _delay_blocks(main, twin, lo, hi, S2_V, S2_BLOCKS, seed=5)}}


def s3_tiny_shards(rank, world, ctx, ex):
    """V = world + 1 (one rank with 2 voices, the others 1: one warp each), then 33 voices on every rank of a delay bank (lane = voice:
    a full warp and one lane of a second)"""
    main, twin = _saw_biquad(ctx, world + 1, rank, world, seed=13)
    ex.attach(main)
    bus, tw = _bus_blocks(main, twin, S3_BLOCKS)
    tiny = _part(bus, tw, (bank_state(main), bank_state(twin)))
    dmain, dtwin, lo, hi = _delay_bank(ctx, 33 * world, rank, world, seed=17)
    ex.attach(dmain)
    return {"parts": {"tiny": tiny, "warp33": _delay_blocks(dmain, dtwin, lo, hi, 33 * world, S3_BLOCKS, seed=17)}}


def s4_refused(rank, world, ctx, ex):
    """every rank asks for a bus of max_doubles + 2 values: refused before any kernel, state untouched; the next block exchanges"""
    main, twin = _saw_biquad(ctx, S1_V, rank, world)
    ex.attach(main)
    bus, tw, refusals = [], [], []
    for n in S4_CALLS:
        if 2 * n <= 2 * B:
            b, t = _bus_blocks(main, twin, [n])
            bus += b; tw += t
            continue
        launches, err = main.launches, None
        try:
            main.process(n, want_out=False, want_mix=True)
        except capi.MxbError as e:
            err = str(e)
        refusals.append(dict(error=err, launches=main.launches - launches, state=(bank_state(main), bank_state(twin))))
    return {"parts": {"main": _part(bus, tw, (bank_state(main), bank_state(twin)))}, "refusals": refusals}


def _polysynth(ctx, V, rank, world, mode, seed):
    lo, hi = shard_range(V, rank, world)
    pair = [capi.Patch(W.polysynth_patch("u8"), hi - lo, max_frames=MAX_FRAMES, ctx=ctx, mode=mode) for _ in range(2)]
    for k, v in W.polysynth_params(V, seed=seed).items():
        for p in pair:
            p.set(k, np.ascontiguousarray(v[lo:hi]))
    return pair + [lo, hi]


def _patch_blocks(main, twin, pat, lo, hi, blocks, first_block=0, switch_after=None):
    bus, tw, out, tout = [], [], [], []
    for k, n in enumerate(blocks):
        if k == switch_after:
            for p in (main, twin):
                p.set_mode("interpret" if p.mode == "fused" else "fused")
        ins = {"trigger": W.note_triggers(pat, n, first_block + k, lo, hi)}
        o, m = main.process(n, ins, want_mix=True)
        to, t = twin.process(n, ins, want_mix=True)
        bus.append(m); tw.append(t); out.append(o); tout.append(to)
    return _part(bus, tw, (patch_state(main), patch_state(twin)), out, tout)


def s5_voice_patch(rank, world, ctx, ex):
    """the polysynth: even ranks start fused, odd ranks interpreted, and every rank switches after the second block"""
    main, twin, lo, hi = _polysynth(ctx, S5_V, rank, world, "fused" if rank % 2 == 0 else "interpret", seed=9)
    ex.attach(main)
    pat = W.note_pattern(S5_V, seed=9)
    return {"parts": {"main": _patch_blocks(main, twin, pat, lo, hi, S5_BLOCKS, switch_after=2)}}


def s6_patch_events(rank, world, ctx, ex):
    """pitch and trigger as events streams, the whole bank's CSR lists sliced per shard"""
    lo, hi = shard_range(S6_V, rank, world)
    d = W.polysynth_pitch_patch("events", "events")
    main, twin = (capi.Patch(d, hi - lo, max_frames=MAX_FRAMES, ctx=ctx) for _ in range(2))
    prm = W.polysynth_params(S6_V, seed=31)
    for k in ("attack", "decay", "sustain", "release", "pan"):
        for p in (main, twin):
            p.set(k, np.ascontiguousarray(prm[k][lo:hi]))
    ex.attach(main)
    bus, tw, out, tout = [], [], [], []
    for k, n in enumerate(S6_BLOCKS):
        pe, te = W.note_events(S6_V, n, k, seed=77)
        ins = {"pitch": slice_events(pe, lo, hi), "trigger": slice_events(te, lo, hi)}
        o, m = main.process(n, ins, want_mix=True)
        to, t = twin.process(n, ins, want_mix=True)
        bus.append(m); tw.append(t); out.append(o); tout.append(to)
    return {"parts": {"main": _part(bus, tw, (patch_state(main), patch_state(twin)), out, tout)}}


def s7_handover(rank, world, ctx, ex):
    """one exchange on a bank, detached, then on a patch, with a 0-frame call in between: its sequence carries over"""
    bank, btwin = _saw_biquad(ctx, S1_V, rank, world)
    ex.attach(bank)
    bus, tw = _bus_blocks(bank, btwin, S7_BANK_BLOCKS)
    parts = {"bank": _part(bus, tw, (bank_state(bank), bank_state(btwin)))}
    capi.check(capi.lib().mxb_bank_set_exchange(bank.h, None), "mxb_bank_set_exchange(NULL)")
    bus, tw = _bus_blocks(bank, btwin, [64])           # detached: the local bus again
    parts["detached"] = _part(bus, tw, (bank_state(bank), bank_state(btwin)))
    main, twin, lo, hi = _polysynth(ctx, S5_V, rank, world, None, seed=9)
    ex.attach(main)
    launches = main.launches
    _, m0 = main.process(0, {"trigger": np.zeros((0, hi - lo), dtype=np.uint8)}, want_out=False, want_mix=True)
    zero = dict(launches=main.launches - launches, shape=m0.shape)
    pat = W.note_pattern(S5_V, seed=9)
    parts["patch"] = _patch_blocks(main, twin, pat, lo, hi, S7_PATCH_BLOCKS)
    return {"parts": parts, "zero": zero}


def s8_memory_modes(rank, world, ctx, ex):
    """S1's blocks with the bus in device memory on a non-blocking stream, then with MXB_MEM_SPLIT | MXB_MEM_ASYNC into page-locked
    host buffers; neither mode reads the exchange status, so the caller synchronises and reads it"""
    import torch
    dev = torch.device("cuda", ctx.device)
    stream = torch.cuda.Stream(device=dev)
    parts = {}
    main, twin = _saw_biquad(ctx, S1_V, rank, world)
    ex.attach(main)
    d = torch.zeros((len(S1_BLOCKS), B, 2), dtype=torch.float64, device=dev)
    for k, n in enumerate(S1_BLOCKS):
        main.process_device(n, mix_ptr=d[k].data_ptr(), stream=stream.cuda_stream)
    stream.synchronize()
    status = ex.status()
    bus = [d[k, :n].cpu().numpy() for k, n in enumerate(S1_BLOCKS)]
    parts["device"] = _part(bus, [twin.process(n, want_out=False, want_mix=True)[1] for n in S1_BLOCKS], (bank_state(main), bank_state(twin)))
    main, twin = _saw_biquad(ctx, S1_V, rank, world)
    ex.attach(main)
    h = torch.zeros((len(S1_BLOCKS), B, 2), dtype=torch.float64, pin_memory=True).numpy()
    for k, n in enumerate(S1_BLOCKS):
        main.process_split(n, None, h[k, :n], wait=False, stream=stream.cuda_stream)
    stream.synchronize()
    status |= ex.status()
    bus = [h[k, :n].copy() for k, n in enumerate(S1_BLOCKS)]
    parts["split"] = _part(bus, [twin.process(n, want_out=False, want_mix=True)[1] for n in S1_BLOCKS], (bank_state(main), bank_state(twin)))
    return {"parts": parts, "mode_status": status}


SCENARIOS = {"s1": s1_bank_bus, "s2": s2_delay_bank, "s3": s3_tiny_shards, "s4": s4_refused, "s5": s5_voice_patch,
             "s6": s6_patch_events, "s7": s7_handover, "s8": s8_memory_modes}


def run_scenarios(rank, world, ctx, link, names, tables):
    """shard.run_ranks body: one exchange (2 * B doubles) for the whole list, attached to each scenario's handle in turn, so its sequence
    runs on through every scenario. Returns {name: scenario result + the exchange's status mask after it, or {"error": traceback}}."""
    os.environ["MXB_EXCHANGE_TIMEOUT_MS"] = TIMEOUT_MS        # read by mxb_exchange_create
    capi.set_tables(*tables, ctx=ctx)
    ex = capi.Exchange(ctx, rank, world, max_doubles=2 * B)
    handles = link.handshake(ex.local_handle())
    if handles is None:
        return None
    ex.connect(handles)
    res = {}
    for name in names:
        try:
            res[name] = SCENARIOS[name](rank, world, ctx, ex)
            res[name]["status"] = ex.status()
        except Exception:
            res[name] = {"error": traceback.format_exc()}
    ctx.synchronize()
    ex.close()
    return res
