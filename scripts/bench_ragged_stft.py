"""Throughput of channels that advance independently (mxb_stft_process_ragged) against the uniform call (mxb_stft_process3), on device
memory, magnitudes written.

    python scripts/bench_ragged_stft.py [--channels 65536] [--hops 8] [--steps 10] [--warmup 2] [--rounds 3]

Every call gives each channel about `hops` hops of samples at 1024 points, hop 512 (the fused two-channel kernel K4s) and at 512 points,
hop 128 (the one-warp-per-frame kernel). Count patterns: "equal" -- every channel `hops` hops, the ragged call against the uniform call
on a twin handle; "random" -- each channel a fixed draw, uniform within +-50 % of that; "half_idle" -- every other channel nothing, the
rest `hops` hops (so that K4s's channel pairs have one idle half). The rate is frames fired per second; ratio is against the uniform
call at the same size. The legs are timed in turn, round after round, so that the spread between rounds shows next to the differences.
Prints one JSON line with the card's name and power limit read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SR = 48000
SIZES = ((1024, 512), (512, 128))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, limit = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return name, limit


def timed(fn, steps, warmup, stream):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=65536)
    ap.add_argument("--hops", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    from maximilian_b200 import capi
    dev = torch.device("cuda:0")
    ctx = capi.default_context(0, SR)
    stream = torch.cuda.Stream()
    sp = C.c_void_p(stream.cuda_stream)
    L = capi.lib()
    Ch, H = args.channels, args.hops
    rng = np.random.default_rng(1)
    legs, frames = [], {}
    for n, hop in SIZES:
        full = H * hop
        pattern = {"equal": np.full(Ch, full, dtype=np.int32),
                   "random": rng.integers(full // 2, full + full // 2 + 1, Ch).astype(np.int32),
                   "half_idle": np.where(np.arange(Ch) % 2 == 0, full, 0).astype(np.int32)}
        most = int(max(p.max() for p in pattern.values()))
        x = (torch.rand((Ch, most), device=dev, dtype=torch.float32) - 0.5)
        maxf = most // hop + 2
        mags = torch.empty((Ch, maxf, n // 2), device=dev, dtype=torch.float32)
        out = capi.StftOutputs(mags.data_ptr(), None, None, None, None, None, None, None)
        nf1 = C.c_int32(0)
        uni = capi.Stft(Ch, n, hop, ctx=ctx)

        def uniform(uni=uni, x=x, most=most, full=full, maxf=maxf, out=out, nf1=nf1):
            capi.check(L.mxb_stft_process3(uni.h, C.c_void_p(x.data_ptr()), most, 1, full, maxf, C.byref(out), None, None, C.byref(nf1),
                                           capi.MEM_DEVICE, sp), "mxb_stft_process3")
        legs.append((f"{n}_{hop}_uniform", uniform))
        frames[f"{n}_{hop}_uniform"] = Ch * ((n - hop + full - n) // hop + 1)
        for name, cnt in pattern.items():
            st = capi.Stft(Ch, n, hop, ctx=ctx)
            nf = np.zeros(Ch, dtype=np.int32)

            def ragged(st=st, x=x, most=most, cnt=cnt, maxf=maxf, out=out, nf=nf):
                capi.check(L.mxb_stft_process_ragged(st.h, C.c_void_p(x.data_ptr()), most, 1, cnt.ctypes.data_as(C.c_void_p), maxf, C.byref(out),
                                                     None, None, nf.ctypes.data_as(C.c_void_p), capi.MEM_DEVICE, sp), "mxb_stft_process_ragged")
            ragged()
            torch.cuda.synchronize()
            frames[f"{n}_{hop}_{name}"] = int(nf.sum())          # frames of one call (the counts repeat, so does the schedule, to +-1)
            legs.append((f"{n}_{hop}_{name}", ragged))
    ms = {k: [] for k, _ in legs}
    for _ in range(args.rounds):
        for k, fn in legs:
            ms[k].append(timed(fn, args.steps, args.warmup, stream))
    res = {}
    for k, _ in legs:
        t = sorted(ms[k])
        med = t[len(t) // 2]
        res[k] = dict(ms_per_call_rounds=ms[k], ms_per_call_median=med, frames_per_call=frames[k], frames_per_s=frames[k] / (med * 1e-3),
                      frames_per_s_range=[frames[k] / (t[-1] * 1e-3), frames[k] / (t[0] * 1e-3)])
    for n, hop in SIZES:
        base = res[f"{n}_{hop}_uniform"]["frames_per_s"]
        for name in ("equal", "random", "half_idle"):
            res[f"{n}_{hop}_{name}"]["ratio_to_uniform"] = res[f"{n}_{hop}_{name}"]["frames_per_s"] / base
    name, limit = card()
    print(json.dumps(dict(workload=f"{Ch} channels x ~{H} hops per call, device memory, magnitudes", gpu=name, power_limit=limit,
                          steps=args.steps, rounds=args.rounds, **res)))


if __name__ == "__main__":
    main()
