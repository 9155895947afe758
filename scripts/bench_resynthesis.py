"""Throughput of maxiIFFT resynthesis (mxb_istft_process) on spectra in device memory, at 1024 and 2048 points and at hops that do not
divide the frame.

    python scripts/bench_resynthesis.py [--channels 16384] [--frames 8] [--steps 20] [--warmup 3] [--rounds 3]

`channels` x `frames` spectra per call. (1024, 512) is the one-kernel path bench.py times (istft1024_kernel), the anchor the others are
read against; (1024, 441) is the same kernel at a hop that does not divide the frame, (2048, 1024) and (2048, 441) run istft2048_kernel,
(512, 100) the two-kernel path of the sizes below 1024. The configurations are timed in turn, round after round, so that the spread
between rounds is visible next to the differences between configurations. Bytes per frame are what the algorithm has to move: the
magnitudes and phases read (2 x 4 B per bin) and the hop's samples written (4 B each); the fraction is of the H100 SXM's 3.35 TB/s
data-sheet HBM bandwidth. Prints one JSON line with the card's name and power limit read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SR, HBM = 48000, 3.35e12
CONFIGS = ((1024, 512), (1024, 441), (2048, 1024), (2048, 441), (512, 100))


def kernel(n):
    return {1024: "istft1024_kernel", 2048: "istft2048_kernel"}.get(n, "istft_frame_kernel + istft_ola_kernel")


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
    ap.add_argument("--channels", type=int, default=16384)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    from maximilian_b200 import capi
    dev = torch.device("cuda:0")
    ctx = capi.default_context(0, SR)
    stream = torch.cuda.Stream()
    sp = C.c_void_p(stream.cuda_stream)
    Ch, F = args.channels, args.frames
    L = capi.lib()
    g = torch.Generator(device=dev).manual_seed(1)
    spectra = {}
    for n in sorted({n for n, _ in CONFIGS}):
        mags = torch.rand((Ch, F, n // 2), generator=g, device=dev, dtype=torch.float32)
        phases = (torch.rand((Ch, F, n // 2), generator=g, device=dev, dtype=torch.float32) - 0.5) * 6.2831855
        spectra[n] = (mags, phases)
    legs = []
    for n, hop in CONFIGS:
        ist = capi.Istft(Ch, n, hop, ctx=ctx)
        y = torch.empty((Ch, F * hop), dtype=torch.float32, device=dev)
        mags, phases = spectra[n]

        def call(ist=ist, y=y, mags=mags, phases=phases):
            capi.check(L.mxb_istft_process(ist.h, C.c_void_p(mags.data_ptr()), C.c_void_p(phases.data_ptr()), F, C.c_void_p(y.data_ptr()),
                                           capi.MEM_DEVICE, sp), "mxb_istft_process")
        legs.append((n, hop, ist, y, call))
    ms = {(n, hop): [] for n, hop in CONFIGS}
    for _ in range(args.rounds):
        for n, hop, _ist, _y, call in legs:
            ms[(n, hop)].append(timed(call, args.steps, args.warmup, stream))
    res = {}
    for n, hop in CONFIGS:
        t = sorted(ms[(n, hop)])
        med = t[len(t) // 2]
        rate = Ch * F / (med * 1e-3)
        bpf = 2 * (n // 2) * 4 + hop * 4
        res[f"{n}_{hop}"] = dict(kernel=kernel(n), ms_per_call_rounds=ms[(n, hop)], ms_per_call_median=med, frames_per_s=rate,
                                 frames_per_s_range=[Ch * F / (t[-1] * 1e-3), Ch * F / (t[0] * 1e-3)],
                                 algorithmic_bytes_per_frame=bpf, hbm_fraction=rate * bpf / HBM)
    name, limit = card()
    print(json.dumps(dict(workload=f"{Ch} channels x {F} frames per call, spectra in device memory", gpu=name, power_limit=limit,
                          steps=args.steps, rounds=args.rounds, hbm_peak_bytes_per_s=HBM, **res)))


if __name__ == "__main__":
    main()
