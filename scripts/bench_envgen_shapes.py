"""Throughput of a voice patch with two maxiEnvGen shapes (mxb_patch_create2), on the generated kernel (K8f) and the interpreter (K8).

    python scripts/bench_envgen_shapes.py [--voices 262144] [--steps 20] [--warmup 3]

The graph is bench.py's polysynth patch (cpp/commandline/maximilian_examples/15.polysynth) with its maxiEnv::adsr replaced by a
maxiEnvGen amp envelope, plus a second maxiEnvGen shape that sweeps the filter cutoff: the usual subtractive voice. Per-sample note
triggers arrive as one bit per voice-sample, as in bench.py. Prints one JSON line: voice-samples/s of each kernel, with the card's name
and power limit read in the same run. Compiled patch kernels go to a temporary directory.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("MXB_PATCH_CACHE", tempfile.mkdtemp(prefix="mxb_envgen_bench_"))

import numpy as np  # noqa: E402

BLOCK, SR = 1024, 48000


def envgen_polysynth():
    from maximilian_b200.patchdef import PatchDef, R
    d = PatchDef()
    amp = d.envgen([0.0, 1.0, 0.3, 0.0], [8.0, 120.0, 600.0], [1.0, 2.0, 0.5], retrigger=True)
    cut = d.envgen([0.0, 1.0, 0.1], [30.0, 900.0], [0.5, 2.0], retrigger=True)
    trig = d.IN("trigger", "bits")
    d.stage("envgen", trig, kind=amp, dst=R(0))                                            # amp envelope
    d.stage("envgen", trig, kind=cut, dst=R(8))                                            # filter envelope
    d.stage("osc", d.K(0.2), kind="sinebuf", dst=R(1))                                     # LFO1out
    d.stage("osc", d.P("f1"), d.K(0.6), kind="pulse", dst=R(2))                            # VCO1out
    d.stage("add", d.P("f2"), R(1), dst=R(3))
    d.stage("osc", R(3), d.K(0.2), kind="pulse", dst=R(3))                                 # VCO2out
    d.stage("add", R(2), R(3), dst=R(4))
    d.stage("mul", R(4), d.K(0.5), dst=R(4))
    d.stage("add", d.P("pitch"), R(1), dst=R(5))
    d.stage("mul", R(5), d.K(1000.0), dst=R(5))
    d.stage("mul", R(5), R(8), dst=R(5))                                                   # the cutoff follows the filter envelope
    d.stage("add", d.K(250.0), R(5), dst=R(5))
    d.stage("filter", R(4), R(5), d.K(10.0), kind="lores", dst=R(6))                       # VCFout
    d.stage("mul", R(6), R(0), dst=R(7))
    d.stage("div", R(7), d.K(6.0), dst=R(7))
    d.stage("out", R(7))
    d.stage("mix_stereo", R(7), d.P("pan"))
    return d


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, limit = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voices", type=int, default=262144)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    from maximilian_b200 import capi
    from maximilian_b200 import workloads as W
    V = args.voices
    assert V % 32 == 0
    dev = torch.device("cuda:0")
    ctx = capi.default_context(0, SR)
    tb = np.load(os.path.join(ROOT, "tests", "golden", "tables.npz"))
    capi.set_tables(tb["sine"], tb["transition"], float(tb["sine_before"]), ctx=ctx)
    d = envgen_polysynth()
    prm = {k: v for k, v in W.polysynth_params(V, seed=W.SEED).items() if k in d.params}      # the ADSR coefficients are gone
    pat = W.note_pattern(V, seed=W.SEED)
    trig = [torch.from_numpy(capi.pack_bits(W.note_triggers(pat, BLOCK, b))).to(dev) for b in range(2)]
    out = torch.empty((BLOCK, V), dtype=torch.float64, device=dev)
    mix = torch.zeros((BLOCK, 2), dtype=torch.float64, device=dev)
    stream = torch.cuda.Stream()
    res = {}
    for mode in ("fused", "interpret"):
        pt = capi.Patch(d, V, max_frames=BLOCK, ctx=ctx, sample_rate=SR, mode=mode)
        for k, v in prm.items():
            pt.set(k, v)
        with torch.cuda.stream(stream):
            for k in range(args.warmup):
                pt.process_device(BLOCK, [trig[k & 1].data_ptr()], out.data_ptr(), mix.data_ptr(), stream=stream.cuda_stream)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for k in range(args.steps):
                pt.process_device(BLOCK, [trig[k & 1].data_ptr()], out.data_ptr(), mix.data_ptr(), stream=stream.cuda_stream)
            e1.record(stream)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        res[mode] = dict(samples_per_s=V * BLOCK / (ms * 1e-3), ms_per_block=ms)
        assert torch.isfinite(out).all() and out.abs().max().item() > 1e-3
        pt.close()
    name, limit = card()
    print(json.dumps(dict(workload=f"polysynth with two maxiEnvGen shapes, {V} voices x {BLOCK} frames, trigger bits", gpu=name,
                          power_limit=limit, steps=args.steps, K8f=res["fused"], K8=res["interpret"])))


if __name__ == "__main__":
    main()
