"""Handles driven from several host threads at once (include/maxib200.h: different handles are independent, also when they are called
from different host threads at the same time).

Every scenario builds its handles on the main thread, then runs twice: once one call after another on one thread (the twin), once with
T = 8 worker threads released together by a barrier, each driving its own handles through the same calls (ctypes drops the GIL, so the
library calls overlap). Every call must succeed, and every output, bus, state word, ring and held value must equal the twin's bit for
bit. One handle of each kind is also checked against the oracle at the bars of DESIGN §2. Each scenario runs in host memory on the NULL
stream (what the Python wrappers do) and in device memory with one stream per thread.

The handles are chosen so that threads sharing a kernel need different amounts of dynamic shared memory, some below 48 KB and some far
above it: the interpreter's four instantiations from a bare oscillator (20 KB) to the 200-double budget patch (200 KB), the streaming
transform with fused MFCC banks of 8 to 520 filters (up to 217 KB), the r01 transform, MFCC, octave and Bark kernels at several sizes.
The limit is a property of the kernel shared by all threads; a launch site that set it to its own size and then launched could have it
lowered by another thread in between, and its launch refused (tests/test_patch_cache_integrity.py scans the sources for such a site)."""
import ctypes as C
import itertools
import threading
import traceback

import numpy as np
import pytest

import envgen_cases as EG
import events_checks as EV
from patch_checks import cmp, ring_stages
from maximilian_b200 import capi
from maximilian_b200 import workloads as W
from maximilian_b200.patchdef import STATE_SLOTS as SLOTS, PatchDef, R

pytestmark = pytest.mark.gpu

T = 8
MEMS = ["host", "device"]


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _empty(shape, dtype):
    import torch
    return torch.empty(shape, dtype=dtype, device="cuda")


def _np(t):
    return t.cpu().numpy()


def _vp(stream):
    return C.c_void_p(int(stream)) if stream else None


# ------------------------------------------------------------------------------------------------ jobs: handles + a sequence of calls

class Job:
    """setup(dev) on the main thread (handles, inputs, device buffers); step(k, stream) on the worker thread (library calls only);
    results() on the main thread once every stream is idle: the arrays the twin must reproduce."""
    name = "job"
    n_calls = 0

    def run(self, stream):
        for k in range(self.n_calls):
            self.step(k, stream)


class Several(Job):
    """one thread driving several handles, call k of each in turn"""

    def __init__(self, *jobs):
        self.jobs = jobs
        self.name = "+".join(j.name for j in jobs)
        self.n_calls = max(j.n_calls for j in jobs)

    def setup(self, dev):
        for j in self.jobs:
            j.setup(dev)

    def step(self, k, stream):
        for j in self.jobs:
            if k < j.n_calls:
                j.step(k, stream)

    def results(self):
        return [a for j in self.jobs for a in j.results()]


FRAMES = [64, 1, 300, 17, 256, 128, 5, 200, 33, 300, 2, 99]


class PatchJob(Job):
    """a voice patch: `inputs(rng, V, n)` gives one call's streams (events as per-voice lists); `switch`: {call: mode} set before it"""

    def __init__(self, name, defn, V, inputs=None, params=None, mode="interpret", switch=None, taps=0, seed=0, frames=FRAMES):
        self.name, self.defn, self.V, self.mode, self.switch, self.taps, self.frames = name, defn, V, mode, switch or {}, taps, frames
        self.n_calls = len(frames)
        rng = np.random.default_rng(seed)
        self.params = params(rng, V) if params else {}
        self.ins = []
        for n in frames:
            x = inputs(rng, V, n) if inputs else {}
            self.ins.append({k: capi.pack_events(v) if defn.input_types.get(k) == "events" else v for k, v in x.items()})

    def setup(self, dev):
        import torch
        self.dev = dev
        self.p = capi.Patch(self.defn, self.V, max_frames=max(self.frames), delay_taps=self.taps, mode=self.mode)
        for k, v in self.params.items():
            self.p.set(k, v)
        self.got, self.d_calls = [], []
        if not dev:
            return
        for k, n in enumerate(self.frames):
            keep, ptrs = [], []
            for name in self.defn.inputs:
                x = self.ins[k][name]
                if self.defn.input_types.get(name) == "events":
                    t = [_dev(a) for a in x]
                    e = capi.Events(*[a.data_ptr() for a in t])
                    keep += t + [e]
                    ptrs.append(C.addressof(e))
                else:
                    t = _dev(np.asarray(x, dtype=np.float64))
                    keep.append(t)
                    ptrs.append(t.data_ptr())
            self.d_calls.append((ptrs, keep, _empty((n, self.V), torch.float64), _empty((n, 2), torch.float64)))

    def step(self, k, stream):
        if k in self.switch:
            self.p.set_mode(self.switch[k])
        n = self.frames[k]
        if self.dev:
            ptrs, _, out, mix = self.d_calls[k]
            self.p.process_device(n, ptrs, out.data_ptr(), mix.data_ptr(), stream=int(stream))
        else:
            self.got.append(self.p.process(n, self.ins[k], want_mix=True))

    def outputs(self):
        return [(_np(o), _np(m)) for _, _, o, m in self.d_calls] if self.dev else self.got

    def results(self):
        r = [a for om in self.outputs() for a in om]
        for si, (op, *_) in enumerate(self.defn.stages):
            r += [self.p.get_state(si, sl) for sl in range(SLOTS.get(op, 0))]
        for si, nl in ring_stages(self.defn):
            r += [self.p.ring(si, v, self.taps * nl) for v in sorted({0, 31, self.V // 2, self.V - 1})]
        r += [self.p.get_held(n) for n in self.defn.inputs if self.defn.input_types.get(n) == "events"]
        return r + [np.array([self.p.launches])]

    def oracle(self, port):
        """the port fed the same (dense) streams: outputs and bus at 1e-9 relative + 1e-12, every state word"""
        o = port.Patch(self.defn, self.V, delay_taps=self.taps, kind="port")
        for k, v in self.params.items():
            o.set(k, v)
        for k, (n, (out, mix)) in enumerate(zip(self.frames, self.outputs())):
            oo, om = o.process(n, self.ins[k], want_mix=True)
            cmp(out, oo, False, f"{self.name} call {k} out vs oracle")
            cmp(mix, om, False, f"{self.name} call {k} bus vs oracle")
        for si, (op, *_) in enumerate(self.defn.stages):
            for sl in range(SLOTS.get(op, 0)):
                cmp(self.p.get_state(si, sl), o.get_state(si, sl), False, f"{self.name} stage {si} slot {sl} vs oracle")


def _events_inputs(values):
    """inputs(rng, V, n) of random event lists, one per stream: values[name](rng, k)"""
    return lambda rng, V, n: {k: EV.random_events(rng, V, n, values=f) for k, f in values.items()}


def _budget(flanger, ty, V, seed, **kw):
    d = EV.budget_patch(flanger, ty)
    vals = lambda r, k: r.uniform(0.0, 500.0, k)                                     # noqa: E731
    if ty == "events":
        inputs = _events_inputs({f"e{j}": vals for j in range(8)})
    else:
        inputs = lambda rng, V, n: {f"e{j}": rng.uniform(0.0, 500.0, (n, V)) for j in range(8)}     # noqa: E731
    params = lambda rng, V: {f"p{j}": 100.0 + j + rng.uniform(0.0, 50.0, V) for j in range(32)}    # noqa: E731
    return PatchJob(f"budget_{ty}{'_flanger' if flanger else ''}", d, V, inputs, params, taps=8 if flanger else 0, seed=seed, **kw)


def _bare_saw(V, seed, **kw):
    d = PatchDef()
    d.stage("osc", d.P("f"), kind="saw", dst=R(0))
    d.stage("out", R(0)); d.stage("mix_stereo", R(0), d.P("pan"))
    return PatchJob("bare_saw", d, V, None, EV._f, seed=seed, **kw)


def _shapes_events():
    """two maxiEnvGen shapes (create2) whose gate, and an oscillator whose frequency, arrive as events"""
    d = PatchDef()
    a = d.envgen([0.0, 1.0, 0.0], [1.5, 2.5], [1.0, 1.0])
    b = d.envgen([0.1, 1.0, 0.3], [0.7, 0.9], [0.5, 3.0], loop=True, retrigger=True)
    d.stage("envgen", d.IN("gate", "events"), kind=a, dst=R(0))
    d.stage("envgen", d.IN("gate", "events"), kind=b, dst=R(1))
    d.stage("osc", d.IN("f", "events"), kind="saw", dst=R(2))
    d.stage("mul", R(2), R(0), dst=R(3)); d.stage("add", R(3), R(1), dst=R(3))
    d.stage("out", R(3)); d.stage("mix_stereo", R(3), d.P("pan"))
    return d


def _four_shapes(V, seed, **kw):
    _, d, params, inputs = EG.four_shapes()
    ctr = itertools.count()
    return PatchJob("four_shapes", d, V, lambda rng, V, n: inputs(V, n, seed + next(ctr)), lambda rng, V: params(V, seed), seed=seed, **kw)


def _events_case(i, V, seed, **kw):
    name, build, values, taps = EV.CASES[i]
    d = build("events")
    params = lambda rng, V: {k: v for k, v in EV._f(rng, V).items() if k in d.params}      # noqa: E731
    return PatchJob(name, d, V, _events_inputs({"x": values}), params, taps=taps, seed=seed, **kw)


# ------------------------------------------------------------------------------------------------ spectral jobs

CHUNKS = lambda n: [3 * n // 2 + 17, n // 2, 1, n - 18, 2 * n + 5, 700]      # noqa: E731  samples per call, ragged


class StftJob(Job):
    """a streaming transform, optionally fused with an MFCC bank (and then writing no spectrum unless `mags`)"""

    def __init__(self, C_, n, hop, mfcc=None, mags=False, seed=0):
        self.C, self.n, self.hop, self.mfcc_cfg, self.want_mags = C_, n, hop, mfcc, mags or mfcc is None
        self.name = f"stft{n}/{hop}" + (f"+mfcc{mfcc[1]}" if mfcc else "")
        chunks = CHUNKS(n)
        x = W.channel_streams(C_, sum(chunks), seed=seed)
        cuts = np.cumsum([0] + chunks)
        self.xs = [np.ascontiguousarray(x[:, cuts[k]:cuts[k + 1]]) for k in range(len(chunks))]
        self.n_calls = len(chunks)

    def setup(self, dev):
        import torch
        self.dev = dev
        self.st = capi.Stft(self.C, self.n, self.hop)
        self.mf = capi.Mfcc(*self.mfcc_cfg) if self.mfcc_cfg else None
        self.got, self.d_calls = [], []
        if dev:
            for x in self.xs:
                maxf = x.shape[1] // self.hop + 2
                mags = _empty((self.C, maxf, self.n // 2), torch.float32) if self.want_mags else None
                co = _empty((self.C, maxf, self.mf.coeffs), torch.float64) if self.mf else None
                self.d_calls.append([_dev(x), maxf, mags, co, 0])

    def step(self, k, stream):
        if self.dev:
            c = self.d_calls[k]
            x = self.xs[k]
            c[4] = self.st.process_device(c[0].data_ptr(), x.shape[1], 1, x.shape[1], c[1], mags=c[2].data_ptr() if c[2] is not None else None,
                                          mfcc=self.mf, coeffs=c[3].data_ptr() if c[3] is not None else None, stream=int(stream))
        else:
            self.got.append(self.st.process(self.xs[k], want=("mags",) if self.want_mags else (), mfcc=self.mf))

    def outputs(self):
        """per call: (magnitudes or None, coefficients or None)"""
        if not self.dev:
            return [(g.get("mags"), g.get("mfcc")) for g in self.got]
        return [(_np(m[:, :f]) if m is not None else None, _np(co[:, :f]) if co is not None else None) for _, _, m, co, f in self.d_calls]

    def results(self):
        return [a for pair in self.outputs() for a in pair if a is not None]

    def oracle(self, port):
        """magnitudes bit for bit, MFCCs 1e-9 relative + 1e-12"""
        ost = port.Stft(self.C, self.n, self.hop)
        omf = port.Mfcc(*self.mfcc_cfg) if self.mfcc_cfg else None
        for k, (x, (mags, co)) in enumerate(zip(self.xs, self.outputs())):
            om = ost.process(x, want=("mags",))["mags"]
            if mags is not None:
                assert np.array_equal(mags, om), f"{self.name} call {k}: magnitudes differ from the oracle"
            if omf is not None:
                np.testing.assert_allclose(co, omf.process(om)[0], rtol=1e-9, atol=1e-12, err_msg=f"{self.name} call {k}: MFCC vs oracle")


class PostJob(StftJob):
    """the 1024-point transform with every spectrum out: magnitudes, the octave analyser and Bark fused into it (FULL instantiation)"""

    def __init__(self, C_, seed=0):
        super().__init__(C_, 1024, 512, None, True, seed)
        self.name = "stft1024+octave+bark"

    def setup(self, dev):
        super().setup(dev)
        import torch
        self.oc = capi.Octave(self.C, 48000, 512, 6)
        self.oc.config(3, 0.85, 0.9, 0.01)
        nA = self.oc.n_averages
        if dev:
            for c in self.d_calls:
                maxf = c[1]
                c += [_empty((self.C, maxf, nA), torch.float32), _empty((self.C, maxf, nA), torch.float32),
                      _empty((self.C, maxf, 24), torch.float64), _empty((self.C, maxf, 24), torch.float64), _empty((self.C, maxf), torch.float64)]

    def step(self, k, stream):
        if not self.dev:
            self.got.append(capi.stft_process_post(self.st, self.xs[k], octave=self.oc, bark=True))
            return
        c = self.d_calls[k]
        N = self.xs[k].shape[1]
        o = capi.StftOutputs(c[2].data_ptr(), None, None, None, None, None, None, None)
        post = capi.StftPost(self.oc.h, c[5].data_ptr(), c[6].data_ptr(), 1, c[7].data_ptr(), c[8].data_ptr(), c[9].data_ptr())
        nf = C.c_int32(0)
        capi.check(capi.lib().mxb_stft_process3(self.st.h, c[0].data_ptr(), N, 1, N, c[1], C.byref(o), C.byref(post), None, C.byref(nf),
                                                capi.MEM_DEVICE, _vp(stream)), "mxb_stft_process3")
        c[4] = nf.value

    def results(self):
        if not self.dev:
            return [g[k] for g in self.got for k in ("mags", "averages", "peaks", "bark_specific", "bark_relative", "bark_total")]
        return [_np(c[i][:, :c[4]]) for c in self.d_calls for i in (2, 5, 6, 7, 8, 9)]


class MfccJob(Job):
    """the stand-alone MFCC kernel on magnitudes in memory"""

    def __init__(self, bins, filters, coeffs=13, fmax=20000.0, frames=(40, 1, 300, 77), seed=0):
        self.cfg = (bins, filters, coeffs, 20.0, fmax)
        self.name = f"mfcc{bins}x{filters}"
        r = np.random.default_rng(seed)
        self.mags = [r.exponential(1.0, (f, bins)).astype(np.float32) for f in frames]
        self.n_calls = len(frames)

    def setup(self, dev):
        import torch
        self.dev, self.mf, self.got = dev, capi.Mfcc(*self.cfg), []
        self.d_calls = [(_dev(m), _empty((m.shape[0], self.cfg[2]), torch.float64)) for m in self.mags] if dev else []

    def step(self, k, stream):
        if self.dev:
            m, co = self.d_calls[k]
            capi.check(capi.lib().mxb_mfcc_process(self.mf.h, m.data_ptr(), m.shape[0], co.data_ptr(), None, capi.MEM_DEVICE, _vp(stream)),
                       "mxb_mfcc_process")
        else:
            self.got.append(self.mf.process(self.mags[k])[0])

    def results(self):
        return [_np(co) for _, co in self.d_calls] if self.dev else self.got

    def oracle(self, port):
        omf = port.Mfcc(*self.cfg)
        for k, (m, co) in enumerate(zip(self.mags, self.results())):
            np.testing.assert_allclose(co, omf.process(m)[0], rtol=1e-9, atol=1e-12, err_msg=f"{self.name} call {k} vs oracle")


class OctaveJob(Job):
    """the stand-alone octave analyser: its averages, peaks and hold times carry from call to call"""

    def __init__(self, C_, sr, bands, per_octave, frames=(4, 1, 9, 3), seed=0):
        self.cfg = (C_, sr, bands, per_octave)
        self.name = f"octave{bands}/{per_octave}"
        r = np.random.default_rng(seed)
        self.mags = [r.exponential(1.0, (C_, f, bands)).astype(np.float32) for f in frames]
        self.n_calls = len(frames)

    def setup(self, dev):
        import torch
        self.dev, self.oc, self.got = dev, capi.Octave(*self.cfg), []
        self.oc.config(5, 0.8, 0.95, 0.002)
        nA = self.oc.n_averages
        self.d_calls = [(_dev(m), _empty((self.cfg[0], m.shape[1], nA), torch.float32), _empty((self.cfg[0], m.shape[1], nA), torch.float32))
                        for m in self.mags] if dev else []

    def step(self, k, stream):
        if self.dev:
            m, av, pk = self.d_calls[k]
            self.oc.process_device(m.data_ptr(), m.shape[1], m.shape[1], av.data_ptr(), pk.data_ptr(), stream=int(stream))
        else:
            self.got += list(self.oc.process(self.mags[k]))

    def results(self):
        return [_np(a) for _, av, pk in self.d_calls for a in (av, pk)] if self.dev else self.got

    def oracle(self, port):
        ooc = port.Octave(*self.cfg)
        ooc.config(5, 0.8, 0.95, 0.002)
        res = self.results()
        for k, m in enumerate(self.mags):
            av, pk = ooc.process(m)
            assert np.array_equal(res[2 * k], av, equal_nan=True) and np.array_equal(res[2 * k + 1], pk, equal_nan=True), \
                f"{self.name} call {k}: differs from the oracle"


class BarkJob(Job):
    def __init__(self, sr, buffer_size, counts=(200, 1, 37), seed=0):
        self.sr, self.bs = sr, buffer_size
        self.name = f"bark{buffer_size}"
        r = np.random.default_rng(seed)
        self.spec = [r.exponential(0.1, (c, buffer_size // 2)).astype(np.float32) for c in counts]
        self.n_calls = len(counts)

    def setup(self, dev):
        import torch
        self.dev, self.bk, self.got = dev, capi.Bark(self.sr, self.bs), []
        self.d_calls = [(_dev(s), _empty((s.shape[0], 24), torch.float64), _empty((s.shape[0], 24), torch.float64),
                         _empty((s.shape[0],), torch.float64)) for s in self.spec] if dev else []

    def step(self, k, stream):
        if self.dev:
            s, sp, rl, tt = self.d_calls[k]
            self.bk.process_device(s.data_ptr(), s.shape[0], sp.data_ptr(), rl.data_ptr(), tt.data_ptr(), stream=int(stream))
        else:
            self.got += list(self.bk.process(self.spec[k]))

    def results(self):
        return [_np(a) for c in self.d_calls for a in c[1:]] if self.dev else self.got

    def oracle(self, port):
        res = self.results()
        for k, s in enumerate(self.spec):
            for g, e in zip(res[3 * k:3 * k + 3], port.bark(s, self.sr, self.bs)):
                np.testing.assert_allclose(g, e, rtol=1e-12, atol=0, err_msg=f"{self.name} call {k} vs oracle")


# ------------------------------------------------------------------------------------------------ controls: fixed shared-memory footprints

class BankJob(Job):
    """K1 (saw -> SVF, out + mix bus) or K2 (saw -> ADSR -> delay line, out + mix bus)"""

    def __init__(self, V, delay, B=256, calls=6, seed=0):
        self.V, self.delay, self.B, self.n_calls, self.seed = V, delay, B, calls, seed
        self.name = "k2_delay" if delay else "k1_svf"
        self.prm = W.voice_params(V, seed=seed, delay_size=200)
        self.gates = [W.gate(V, B, k, seed=seed) for k in range(calls)]

    def _make(self, mod):
        kw = dict(osc="saw", env=True, delay=True, delay_capacity=256) if self.delay else dict(osc="saw", filt="svf")
        b = (mod.Bank(self.V, max_frames=self.B, **kw) if mod is capi else mod.Bank(self.V, kind="port", **kw))
        W.configure_bank(b, "none" if self.delay else "svf", self.prm, self.delay, self.delay)
        return b

    def setup(self, dev):
        import torch
        self.dev, self.b, self.got = dev, self._make(capi), []
        self.d_calls = [(_dev(on), _dev(off), _empty((self.B, self.V), torch.float64), _empty((self.B, 2), torch.float64))
                        for on, off in self.gates] if dev else []

    def step(self, k, stream):
        if self.dev:
            on, off, out, mix = self.d_calls[k]
            self.b.process_device(self.B, out.data_ptr(), mix.data_ptr(), on.data_ptr() if self.delay else None,
                                  off.data_ptr() if self.delay else None, stream=int(stream))
        else:
            on, off = self.gates[k]
            self.got.append(self.b.process(self.B, on if self.delay else None, off if self.delay else None, want_mix=True))

    def outputs(self):
        return [(_np(o), _np(m)) for _, _, o, m in self.d_calls] if self.dev else self.got

    def state(self, b):
        names = ("phase", "delay_phase", "env_amplitude") if self.delay else ("phase", "filt0", "filt1", "filt2")
        r = [b.get(n) for n in names]
        if self.delay:
            r += [b.ring(v, 256) for v in (0, 31, self.V // 2, self.V - 1)]
        return r

    def results(self):
        return [a for om in self.outputs() for a in om] + self.state(self.b)

    def oracle(self, port):
        o = self._make(port)
        for k, (out, mix) in enumerate(self.outputs()):
            on, off = self.gates[k]
            oo, om = o.process(self.B, on if self.delay else None, off if self.delay else None, want_mix=True)
            assert np.array_equal(out, oo), f"{self.name} block {k}: output differs from the oracle"
            np.testing.assert_allclose(mix, om, rtol=1e-9, atol=1e-10, err_msg=f"{self.name} block {k}: bus vs oracle")
        for g, e in zip(self.state(self.b), self.state(o)):
            assert np.array_equal(g, e), f"{self.name}: state differs from the oracle"


class IstftJob(Job):
    def __init__(self, C_, n, hop, frames=(3, 1, 8, 2), seed=0):
        self.C, self.n, self.hop, self.name = C_, n, hop, f"istft{n}/{hop}"
        r = np.random.default_rng(seed)
        self.ins = [(r.exponential(1.0, (C_, f, n // 2)).astype(np.float32), r.uniform(-np.pi, np.pi, (C_, f, n // 2)).astype(np.float32))
                    for f in frames]
        self.n_calls = len(frames)

    def setup(self, dev):
        import torch
        self.dev, self.s, self.got = dev, capi.Istft(self.C, self.n, self.hop), []
        self.d_calls = [(_dev(m), _dev(p), _empty((self.C, m.shape[1] * self.hop), torch.float32)) for m, p in self.ins] if dev else []

    def step(self, k, stream):
        if self.dev:
            m, p, out = self.d_calls[k]
            capi.check(capi.lib().mxb_istft_process(self.s.h, m.data_ptr(), p.data_ptr(), m.shape[1], out.data_ptr(), capi.MEM_DEVICE, _vp(stream)),
                       "mxb_istft_process")
        else:
            self.got.append(self.s.process(*self.ins[k]))

    def results(self):
        return [_np(o) for _, _, o in self.d_calls] if self.dev else self.got

    def oracle(self, port):
        o = port.Istft(self.C, self.n, self.hop)
        for k, (g, (m, p)) in enumerate(zip(self.results(), self.ins)):
            e = o.process(m, p)
            np.testing.assert_allclose(g, e, rtol=0, atol=1e-5 * float(np.abs(e).max()), err_msg=f"{self.name} call {k} vs oracle")


# ------------------------------------------------------------------------------------------------ the runner

def _run(jobs, dev, threaded):
    """setup on this thread, then every job's calls: on T threads at once, or one job after another; returns every job's results"""
    import torch
    assert len(jobs) == T
    capi.default_context()
    for j in jobs:
        j.setup(dev)
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() if dev else None for _ in jobs]
    go = threading.Barrier(T, timeout=120) if threaded else None
    errors = []

    def drive(i):
        try:
            if go is not None:
                go.wait()
            jobs[i].run(streams[i].cuda_stream if dev else 0)
            if dev:
                streams[i].synchronize()
        except Exception:             # noqa: BLE001 -- capi.check's message carries mxb_last_error() as this thread saw it
            errors.append(f"thread {i} ({jobs[i].name}):\n{traceback.format_exc()}")

    if threaded:
        threads = [threading.Thread(target=drive, args=(i,), name=f"mxb-{i}") for i in range(T)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    else:
        for i in range(T):
            drive(i)
    assert not errors, "\n".join(errors)
    torch.cuda.synchronize()
    return [j.results() for j in jobs]


def _threads_equal_twin(make_jobs, mem):
    """make_jobs() -> T fresh jobs; the single-threaded twin first, then the threaded run, compared bit for bit. Returns the threaded jobs."""
    dev = mem == "device"
    twin = _run(make_jobs(), dev, threaded=False)
    jobs = make_jobs()
    got = _run(jobs, dev, threaded=True)
    for j, a, b in zip(jobs, twin, got):
        assert len(a) == len(b), j.name
        for k, (x, y) in enumerate(zip(a, b)):
            assert x.shape == y.shape and np.array_equal(x, y, equal_nan=True), f"{j.name}: array {k} differs from the single-threaded run"
    return jobs


# ------------------------------------------------------------------------------------------------ scenarios

def _interpreted_jobs():
    shapes_ev = lambda: PatchJob("shapes_events", _shapes_events(), 1000,                                      # noqa: E731
                                 _events_inputs({"gate": lambda r, k: r.choice([-1.0, 1.0], k), "f": lambda r, k: r.uniform(50.0, 2000.0, k)}),
                                 lambda rng, V: {"pan": rng.uniform(0.0, 1.0, V)}, seed=4)
    return [
        _bare_saw(3000, seed=1),                                    # one shape, no events: 20 KB
        _budget(False, "events", 500, seed=2),                      # one shape, events: 200 doubles per voice, 200 KB
        _budget(True, "f64", 700, seed=3),                          # one shape, dense streams and a flanger: 177 doubles
        _four_shapes(300, seed=5),                                  # several shapes, no events
        shapes_ev(),                                                # several shapes, events
        _events_case(1, 2000, seed=6),                              # trigger -> maxiEnvGen, events, small
        _events_case(4, 1000, seed=7, switch={2: "fused", 5: "interpret", 9: "fused"}),    # switches kernel mid-stream
        _events_case(3, 1500, seed=8),                              # per-sample cutoff design, events
    ]


@pytest.mark.parametrize("mem", MEMS)
def test_interpreted_patches_on_eight_threads(mem, port):
    jobs = _threads_equal_twin(_interpreted_jobs, mem)
    if mem == "host":
        jobs[3].oracle(port)


_salt = itertools.count(1)


def _fused_jobs():
    """four threads make the first launch of four different programs, four the first launch of one program. A stage whose result
    nothing reads makes each call of this function compile programs no earlier run in this process compiled."""
    salts = [next(_salt) for _ in range(5)]

    def salted(job, s):
        job.defn.stage("add", job.defn.K(1e6 + s), job.defn.K(0.0), dst=R(15))
        job.mode = None                                            # the default, fused: compiled at the first process call
        return job

    different = [salted(_events_case(i, 700 + 100 * i, seed=20 + i), salts[k]) for k, i in enumerate((0, 2, 3, 5))]
    same = [salted(_four_shapes(256, seed=30 + i, frames=FRAMES[:6]), salts[4]) for i in range(4)]
    return different + same


@pytest.mark.parametrize("mem", MEMS)
def test_fused_patches_first_launch_on_eight_threads(mem, tmp_path, monkeypatch):
    monkeypatch.setenv("MXB_PATCH_CACHE", str(tmp_path / "cache"))
    monkeypatch.delenv("MXB_PATCH_MODE", raising=False)
    jobs = _threads_equal_twin(_fused_jobs, mem)
    assert all(j.p.mode == "fused" for j in jobs)
    cubins = sorted((tmp_path / "cache").glob("*"))
    assert len(cubins) == 2 * 5 and all(p.suffix == ".cubin" for p in cubins), [p.name for p in cubins]      # twin + threads, no temporaries


def _spectral_jobs():
    return [
        StftJob(16, 1024, 512, (512, 8, 8, 20.0, 8000.0), seed=1),             # K4s, FULL = false, fused MFCC tables of 8 to 128 filters
        StftJob(16, 1024, 512, (512, 42, 13, 20.0, 8000.0), seed=2),
        StftJob(16, 1024, 512, (512, 128, 13, 20.0, 8000.0), seed=3),
        StftJob(16, 1024, 512, (512, 520, 13, 20.0, 20000.0), seed=4),         # 217 KB (a bank past bin 256: FULL = true)
        PostJob(16, seed=5),                                                    # FULL = true with the octave and Bark epilogues
        Several(StftJob(8, 256, 128, (128, 20, 13), seed=6), StftJob(8, 2048, 1024, (1024, 40, 13), seed=7), BarkJob(48000, 2048, seed=8)),
        Several(StftJob(8, 512, 200, (256, 30, 13), seed=9), MfccJob(256, 26, seed=10), MfccJob(1024, 40, seed=11), BarkJob(44100, 256, seed=12)),
        Several(OctaveJob(8, 44100, 128, 3, seed=13), OctaveJob(8, 48000, 1024, 12, seed=14), OctaveJob(5, 48000, 512, 6, seed=15),
                BarkJob(48000, 1024, seed=16)),
    ]


@pytest.mark.parametrize("mem", MEMS)
def test_spectral_handles_on_eight_threads(mem, port):
    jobs = _threads_equal_twin(_spectral_jobs, mem)
    if mem == "host":
        jobs[1].oracle(port)
        jobs[5].jobs[1].oracle(port)
        jobs[5].jobs[2].oracle(port)
        jobs[6].jobs[2].oracle(port)
        jobs[7].jobs[1].oracle(port)


def _mixed_jobs():
    """the kernels with a fixed footprint (mix reducer, the delay kernel's bulk copies, both one-kernel resyntheses) beside the rest"""
    return [
        BankJob(4096, False, seed=1),
        BankJob(2048, True, seed=2),
        IstftJob(16, 1024, 256, seed=3),
        IstftJob(16, 2048, 512, seed=4),
        _budget(False, "events", 400, seed=5, frames=FRAMES[:6]),
        StftJob(16, 1024, 512, (512, 520, 13, 20.0, 20000.0), seed=6),
        BarkJob(48000, 2048, seed=7),
        _bare_saw(1000, seed=8, frames=FRAMES[:6]),
    ]


@pytest.mark.parametrize("mem", MEMS)
def test_controls_beside_the_rest_on_eight_threads(mem, port):
    jobs = _threads_equal_twin(_mixed_jobs, mem)
    if mem == "host":
        for j in jobs[:4]:
            j.oracle(port)


def test_a_refused_call_sets_the_error_of_its_own_thread_only():
    """thread A's refused call leaves thread B's last error (from B's own earlier refusal) and C's (none) as they were"""
    ctx = capi.default_context()
    p = capi.Patch(_bare_saw(64, 0).defn, 64, max_frames=32, mode="interpret")
    out = np.empty((33, 64))
    first, second = threading.Barrier(3, timeout=60), threading.Barrier(3, timeout=60)
    seen = {}

    def a():
        first.wait()
        h = C.c_void_p()
        seen["a_rc"] = capi.lib().mxb_bark_create(ctx.h, 48000, 5000, C.byref(h))
        seen["a"] = capi.lib().mxb_last_error().decode()
        second.wait()

    def b():
        seen["b_rc"] = capi.lib().mxb_patch_process(p.h, 33, None, capi._np_ptr(out), None, capi.MEM_HOST, None)
        seen["b_before"] = capi.lib().mxb_last_error().decode()
        first.wait()
        second.wait()
        seen["b_after"] = capi.lib().mxb_last_error().decode()

    def c():
        first.wait()
        second.wait()
        seen["c"] = capi.lib().mxb_last_error().decode()

    threads = [threading.Thread(target=f) for f in (a, b, c)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert seen["a_rc"] == -1 and "mxb_bark_create" in seen["a"] and "5000" in seen["a"], seen
    assert seen["b_rc"] == -1 and "mxb_patch_process" in seen["b_before"] and "33" in seen["b_before"], seen
    assert seen["b_after"] == seen["b_before"], seen
    assert seen["c"] == "", seen
    assert p.process(32)[0].shape == (32, 64)                       # the handle B was refused on still works
