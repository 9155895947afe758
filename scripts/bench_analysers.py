"""Throughput of the stand-alone octave analyser and Bark loudness (mxb_octave_process / mxb_bark_process) on spectra in device memory,
next to the analysers fused into the 1024-point transform.

    python scripts/bench_analysers.py [--channels 65536] [--frames 8] [--steps 20] [--warmup 3]

Stand-alone: `channels` x `frames` spectra of 512 and 1024 bins, read once per call. Bytes per frame are what the algorithm has to move:
the magnitudes read (4 B per bin), the outputs written (averages and peaks, 8 B per band; Bark 49 doubles), and for the octave analyser
the per-channel state read and written once per call, spread over the frames. The fraction is of the H100 SXM's 3.35 TB/s data-sheet
HBM bandwidth. Fused: bench.py's analysis_octave_bark configuration (16 Ki channels x 8 hops of the 1024 / 512 transform, magnitudes,
octave analyser at 3 per octave, Bark), timed the same way. Prints one JSON line with the card's name and power limit read in the same
run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

SR, HBM = 48000, 3.35e12


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


def entry(ms, frames, bytes_per_frame, what):
    rate = frames / (ms * 1e-3)
    return dict(what=what, ms_per_call=ms, frames_per_s=rate, algorithmic_bytes_per_frame=bytes_per_frame,
                hbm_fraction=rate * bytes_per_frame / HBM)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=65536)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    from maximilian_b200 import capi
    from maximilian_b200 import workloads as W
    dev = torch.device("cuda:0")
    ctx = capi.default_context(0, SR)
    stream = torch.cuda.Stream()
    sp = stream.cuda_stream
    Ch, F = args.channels, args.frames
    res = {}
    g = torch.Generator(device=dev).manual_seed(1)
    for bins in (512, 1024):
        mags = torch.rand((Ch, F, bins), generator=g, device=dev, dtype=torch.float32)
        oc = capi.Octave(Ch, SR, bins, 3, ctx=ctx)
        nA = oc.n_averages
        av = torch.empty((Ch, F, nA), dtype=torch.float32, device=dev); pk = torch.empty_like(av)
        ms = timed(lambda: oc.process_device(mags.data_ptr(), F, F, av.data_ptr(), pk.data_ptr(), stream=sp), args.steps, args.warmup, stream)
        res[f"octave_{bins}"] = entry(ms, Ch * F, 4 * bins + 8 * nA + 2 * 12 * nA / F,
                                      f"octave_kernel, {bins} bins, {nA} averages + peaks, frames in order per channel")
        oc.close()
        del av, pk
        bk = capi.Bark(SR, 2 * bins, ctx=ctx)
        n = Ch * F
        bs = torch.empty((n, 24), dtype=torch.float64, device=dev); br = torch.empty_like(bs); bt = torch.empty(n, dtype=torch.float64, device=dev)
        ms = timed(lambda: bk.process_device(mags.data_ptr(), n, bs.data_ptr(), br.data_ptr(), bt.data_ptr(), stream=sp), args.steps, args.warmup, stream)
        res[f"bark_{bins}"] = entry(ms, n, 4 * bins + 49 * 8, f"bark_kernel, {bins} bins, specific + relative + total")
        bk.close()
        del mags, bs, br, bt
        torch.cuda.empty_cache()

    # the fused path, bench.py's analysis_octave_bark configuration
    Cf, n, hop, H = 1 << 14, 1024, 512, 8
    base = W.channel_streams(1024, H * hop, seed=11)
    x = torch.from_numpy(np.tile(base, (Cf // 1024, 1))).to(dev)
    st = capi.Stft(Cf, n, hop, ctx=ctx)
    oc = capi.Octave(Cf, float(SR), n // 2, 3, ctx=ctx)
    nA = oc.n_averages
    mags = torch.empty((Cf, H, n // 2), dtype=torch.float32, device=dev)
    av = torch.empty((Cf, H, nA), dtype=torch.float32, device=dev); pk = torch.empty_like(av)
    bs = torch.empty((Cf, H, 24), dtype=torch.float64, device=dev); br = torch.empty_like(bs); bt = torch.empty((Cf, H), dtype=torch.float64, device=dev)
    o = capi.StftOutputs(mags.data_ptr(), None, None, None, None, None, None, None)
    post = capi.StftPost(oc.h, av.data_ptr(), pk.data_ptr(), 1, bs.data_ptr(), br.data_ptr(), bt.data_ptr())
    nf = C.c_int32(0)
    L = capi.lib()

    def fused():
        capi.check(L.mxb_stft_process3(st.h, C.c_void_p(x.data_ptr()), H * hop, 1, H * hop, H, C.byref(o), C.byref(post), None, C.byref(nf),
                                       capi.MEM_DEVICE, C.c_void_p(sp)), "mxb_stft_process3")
    ms = timed(fused, args.steps, args.warmup, stream)
    res["fused_1024"] = entry(ms, Cf * H, hop * 4 + (n // 2) * 4 + 2 * nA * 4 + 49 * 8,
                              "stft_stream_kernel<FULL> + octave / Bark epilogues (bench.py analysis_octave_bark): samples in, magnitudes, "
                              "averages, peaks, Bark out")
    name, limit = card()
    print(json.dumps(dict(workload=f"{Ch} channels x {F} frames per call (stand-alone); fused: {Cf} channels x {H} hops", gpu=name,
                          power_limit=limit, steps=args.steps, hbm_peak_bytes_per_s=HBM, **res)))


if __name__ == "__main__":
    main()
