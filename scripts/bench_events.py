"""Host-driven notes on the polysynth patch: what it costs to hand over a new pitch and a trigger per voice per block as control events
(MXB_IN_EVENTS) instead of dense per-sample streams.

    python scripts/bench_events.py [--voices 262144] [--block 1024] [--steps 20] [--warmup 3] [--rounds 3]

The patch is workloads.polysynth_pitch_patch: 15.polysynth with the voice's pitch as a stream (both VCOs and the cutoff follow it).
Every voice plays about one note per block: a new pitch at a random frame and a one-sample trigger there (workloads.note_events).
Three ways of feeding it, on the generated kernel:
  (a) dense: the pitch as f64 [block][voices] and the trigger as packed bits, from pinned host memory;
  (b) events: pitch and trigger as events (first / frame / value), from pinned host memory;
  (c) resident: the inputs of (a) and of (b) already on the device -- the kernel alone.
For (a) and (b) each step copies the block's inputs up on a copy stream (double-buffered on the device), runs the patch and copies
the stereo bus back into pinned memory, as bench.py's e2e loop does. Kernel times are CUDA events over the steps; e2e rates are
voice-samples per second of wall time over the steps; bytes are what crosses PCIe per block. Dense and events are timed in turn, round after round, so
that the spread between rounds is visible. Prints one JSON line with the card's name and power limit read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SR = 48000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, limit = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voices", type=int, default=262144)
    ap.add_argument("--block", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    from maximilian_b200 import capi
    from maximilian_b200 import workloads as W
    import golden_checks as G

    if not torch.cuda.is_available():
        raise SystemExit("bench_events.py needs a CUDA device")
    V, B = args.voices, args.block
    assert V % 32 == 0
    g = G.load("tables")
    ctx = capi.default_context(0, SR)
    capi.set_tables(g["sine"], g["transition"], float(g["sine_before"]), ctx=ctx)
    prm = W.polysynth_params(V)
    prm = {k: prm[k] for k in ("attack", "decay", "sustain", "release", "pan")}
    dev, stream, copy_stream = torch.device("cuda:0"), torch.cuda.Stream(), torch.cuda.Stream()

    # two blocks of notes, alternated step by step; the dense form of the same notes for (a)
    blocks = [W.note_events(V, B, b) for b in range(2)]
    prev = np.zeros(V)
    dense = []
    for pe, te in blocks:
        _, t, pitch = pe                                          # one pitch event per voice, at frame t; the trigger is 1 at t only
        frames = np.arange(B)[:, None]
        dense.append((torch.from_numpy(np.where(frames >= t[None, :], pitch[None, :], prev[None, :])),
                      torch.from_numpy(capi.pack_bits(frames == t[None, :]).view(np.int32))))
        prev = pitch
    host = {"dense": [tuple(x.pin_memory() for x in d) for d in dense],
            "events": [tuple(torch.from_numpy(np.ascontiguousarray(a)).pin_memory() for a in pe + te) for pe, te in blocks]}
    resident = {k: [tuple(x.to(dev) for x in blk) for blk in v] for k, v in host.items()}
    staged = {k: [tuple(torch.empty_like(x, device=dev) for x in v[0]) for _ in range(2)] for k, v in host.items()}
    patches = {"dense": capi.Patch(W.polysynth_pitch_patch("f64", "bits"), V, max_frames=B, ctx=ctx, sample_rate=SR, mode="fused"),
               "events": capi.Patch(W.polysynth_pitch_patch("events", "events"), V, max_frames=B, ctx=ctx, sample_rate=SR, mode="fused")}
    for p in patches.values():
        for k, v in prm.items():
            p.set(k, v)
    out = torch.empty((B, V), dtype=torch.float64, device=dev)
    mix = [torch.zeros((B, 2), dtype=torch.float64, device=dev) for _ in range(2)]
    mix_host = [torch.zeros((B, 2), dtype=torch.float64).pin_memory() for _ in range(2)]

    def launch(kind, bufs, b):
        if kind == "dense":
            ptrs = [bufs[0].data_ptr(), bufs[1].data_ptr()]
            descs = []
        else:
            descs = [capi.Events(*(x.data_ptr() for x in bufs[:3])), capi.Events(*(x.data_ptr() for x in bufs[3:]))]
            ptrs = [C.addressof(x) for x in descs]
        patches[kind].process_device(B, ptrs, out.data_ptr(), mix[b].data_ptr(), stream=stream.cuda_stream)

    def kernel_ms(kind, n):
        for k in range(args.warmup):
            launch(kind, resident[kind][k & 1], k & 1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for k in range(n):
            launch(kind, resident[kind][k & 1], k & 1)
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    ev_up = [torch.cuda.Event() for _ in range(2)]
    ev_done = [torch.cuda.Event() for _ in range(2)]

    def e2e_rate(kind, n):
        def step(k):
            b = k & 1
            with torch.cuda.stream(copy_stream):
                copy_stream.wait_event(ev_done[b])
                for d, s in zip(staged[kind][b], host[kind][b]):
                    d.copy_(s, non_blocking=True)
                ev_up[b].record(copy_stream)
            stream.wait_event(ev_up[b])
            launch(kind, staged[kind][b], b)
            ev_done[b].record(stream)
            with torch.cuda.stream(stream):
                mix_host[b].copy_(mix[b], non_blocking=True)
        for k in range(args.warmup):
            step(k)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for k in range(n):
            step(k)
        torch.cuda.synchronize()
        return V * B * n / (time.perf_counter() - t0)

    runs = {f"{k}_{w}": [] for k in ("dense", "events") for w in ("kernel_ms", "e2e")}
    for _ in range(args.rounds):
        for kind in ("dense", "events"):
            runs[f"{kind}_kernel_ms"].append(kernel_ms(kind, args.steps))
            runs[f"{kind}_e2e"].append(e2e_rate(kind, args.steps))
    h2d = {k: int(sum(x.numel() * x.element_size() for x in v[0])) for k, v in host.items()}
    name, limit = card()
    res = {"card": name, "power_limit": limit, "voices": V, "block": B, "sample_rate": SR, "steps": args.steps, "rounds": args.rounds}
    for kind in ("dense", "events"):
        ms = runs[f"{kind}_kernel_ms"]
        e2e = runs[f"{kind}_e2e"]
        res[kind] = {"kernel_ms_per_block": ms, "resident_rate": [V * B / (m * 1e-3) for m in ms], "e2e_rate": e2e,
                     "e2e_frac_of_resident": [e / (V * B / (m * 1e-3)) for e, m in zip(e2e, ms)],
                     "h2d_bytes_per_block": h2d[kind], "d2h_bytes_per_block": B * 2 * 8}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
