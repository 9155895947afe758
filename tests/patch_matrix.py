"""The voice-patch matrix: one small patch per (op, kind) of maximilian_b200/patchdef.py, each case a tuple
(name, PatchDef, params(V, seed), inputs(V, B, blk, seed), exact, taps) like tests/patch_cases.py. CPU-importable, no device.

The stage under test is fed from an oscillator or an input stream, and each of its control operands is drawn from every class
the code generator (maximilian_b200/csrc/patch_fuse.cu) treats differently: a constant or a per-voice parameter (a design,
increment or envelope rate hoisted before the sample loop), a register modulated on every sample by a triangle LFO, and an input
stream (f64, and u8 / bits where the operand is a trigger) -- both computed per sample. Parameters and streams carry the corners
the reference defines: frequencies 0, -0, negative, above Nyquist and 1e-300; duties outside [0, 1]; cutoffs below the lores
clamp and above sr; resonance >= 1 and 0; biquad gains +, 0 and -; inputs exactly at +-1 and across the clip rails; delay sizes 1
and == taps, positions >= size, feedback 0 and > 1, sizes that shrink below the ring index; holdtime 0, 1, 2^31 - 1 and 2^32 + 3;
triggers 1.0, 0.999, 1.5 and -1; division by +0 and -0; pans outside [0, 1] and at 0 and 1.

`exact`: every stage avoids libm (all oscillators but sine and cos, the table oscillators, ADSR / AR, lopass / hipass / DC blocker,
fastatan / fastatandist / hardclip, delay / dlFromPosition / flanger, + - * /, out and the stereo mix): bit parity expected.

Left out on purpose -- the reference itself is undefined there, so no executor can be held to it:
  - double -> int conversions out of range or of a NaN: delay size and position, flanger delay, holdtime, trigger;
  - the table oscillators (sinebuf, sinebuf4, sawn) at a negative frequency or above sr, and sawn at 0 Hz: they read outside
    their tables;
  - a delay index at or beyond the ring (size or position > taps), or a negative position.
"""
import zlib

import numpy as np

from maximilian_b200.patchdef import PatchDef, R, ENVGEN_HOLD, OP, OSC, FILT, BIQUAD, NONLIN, DELAY

SR = 48000.0
CLASSES = "KPRI"                        # constant, per-voice parameter, LFO-modulated register, input stream
HOLDTIMES = (0.0, 1.0, 2.0 ** 31 - 1, 2.0 ** 32 + 3)
TRIGGERS = (1.0, 0.999, 1.5, -1.0)
PANS = (-0.5, 0.0, 1.0, 1.5, 0.5)
LIBM_OSC = ("sinewave", "coswave")
TABLE_OSC = ("sinebuf", "sinebuf4", "sawn")


def _rng(seed, *key):
    return np.random.default_rng([int(seed) & 0xffffffff] + [zlib.crc32(str(k).encode()) for k in key])


def _gates(rng, B, V, density=0.02, hold=(3, 60)):
    """[B][V] of 0 / 1: gates that open and close anywhere inside the block"""
    g = np.zeros((B, V))
    for v in range(V):
        pos = int(rng.integers(0, 8))
        while pos < B:
            ln = int(rng.integers(hold[0], hold[1]))
            g[pos:pos + ln, v] = 1.0
            pos += ln + int(rng.geometric(density))
    return g


class Case:
    """A patch under construction: its PatchDef, what its parameters and input streams hold, the registers it has used."""

    def __init__(self, name, exact, taps=0):
        self.name, self.exact, self.taps = name, exact, taps
        self.d = PatchDef()
        self.pspec, self.ispec, self.lfo = {}, {}, {}
        self.nreg = 0

    def reg(self):
        r = self.nreg
        self.nreg += 1
        return R(r)

    def ctrl(self, cls, tag, lo, hi, corners=(), const=None, integral=False, rate=None, smooth=False):
        """an operand of class cls ("K" constant `const`, "P" parameter, "R" register swept over [lo, hi] by a triangle LFO,
        "I" f64 input stream) with values in [lo, hi] and, for P and I, the corner values. smooth: the stream walks in small steps and
        holds each corner on a voice of its own, instead of a new random value on every sample (a biquad redesigned that way turns
        1-ulp differences of tan / pow into far more than 1e-9)"""
        d = self.d
        if cls == "K":
            return d.K(lo if const is None else const)
        if cls == "P":
            self.pspec[tag] = ("uniform", lo, hi, tuple(corners), integral)
            return d.P(tag)
        if cls == "I":
            self.ispec[tag] = ("walk" if smooth else "uniform", lo, hi, tuple(corners), integral)
            return d.IN(tag)
        key = (tag, lo, hi)
        if key not in self.lfo:                                        # triangle in [-1, 1] -> [lo, hi], exact arithmetic
            r = self.reg()
            d.stage("osc", d.K(rate or 5.0 + 2.0 * len(self.lfo)), kind="triangle", dst=r)
            d.stage("mul", r, d.K((hi - lo) / 2.0), dst=r)
            d.stage("add", r, d.K((hi + lo) / 2.0), dst=r)
            self.lfo[key] = r
        return self.lfo[key]

    def trig(self, cls, tag, dtype="f64"):
        """a maxiEnv trigger ((int)value == 1): constant 1, per-voice 1.0 / 0.999 / 1.5 / -1 / 0, a square LFO (+-1) in a register,
        or a gate stream -- f64 (its open samples take 1.0, 0.999, 1.5 and -1), u8 or packed bits"""
        d = self.d
        if cls == "K":
            return d.K(1.0)
        if cls == "P":
            self.pspec[tag] = ("choice", TRIGGERS + (0.0,))
            return d.P(tag)
        if cls == "R":
            r = self.reg()
            d.stage("osc", d.K(90.0), kind="square", dst=r)
            return r
        self.ispec[tag] = ("gate", dtype)
        return d.IN(tag, dtype)

    def params(self, V, seed):
        out = {}
        for tag, spec in self.pspec.items():
            rng = _rng(seed, self.name, tag)
            if spec[0] == "choice":
                x = rng.choice(np.array(spec[1]), V)
            else:
                _, lo, hi, corners, integral = spec
                x = rng.uniform(lo, hi, V)
                if integral:
                    x = np.floor(x)
                n = min(len(corners), V)
                x[:n] = corners[:n]
            out[tag] = x
        return out

    def inputs(self, V, B, blk, seed):
        out = {}
        for tag, spec in self.ispec.items():
            rng = _rng(seed, self.name, tag, blk)
            if spec[0] == "gate":
                g = _gates(rng, B, V)
                if spec[1] == "f64":
                    g = np.where(g != 0, rng.choice(np.array(TRIGGERS), (B, V), p=[0.7, 0.1, 0.1, 0.1]), 0.0)
                    out[tag] = g
                else:
                    out[tag] = g.astype(np.uint8)
            elif spec[0] == "noise":
                from oracle import oracle_py
                out[tag] = oracle_py.noise_fill(seed, (blk + 1) * B * V, "port")[blk * B * V:].reshape(B, V)
            elif spec[0] == "walk":
                _, lo, hi, corners, integral = spec
                steps = rng.uniform(-0.003, 0.003, (B, V)) * (hi - lo)
                x = np.clip(rng.uniform(lo, hi, V) + np.cumsum(steps, axis=0), lo, hi)
                n = min(len(corners), V)
                x[:, :n] = corners[:n]
                out[tag] = x
            else:
                _, lo, hi, corners, integral = spec
                x = rng.uniform(lo, hi, (B, V))
                if integral:
                    x = np.floor(x)
                for c in corners:
                    x[rng.random((B, V)) < 0.03] = c
                out[tag] = x
        return out

    def finish(self, regs, pan=True):
        """out = the sum of the stage outputs in `regs` (left to right); the stereo bus takes it at a per-voice pan"""
        d = self.d
        acc = self.reg()
        d.stage("add", regs[0], d.K(0.0), dst=acc)
        for r in regs[1:]:
            d.stage("add", acc, r, dst=acc)
        d.stage("out", acc)
        if pan:
            d.stage("mix_stereo", acc, self.ctrl("P", "pan", 0.0, 1.0, PANS))
        return (self.name, self.d, self.params, self.inputs, self.exact, self.taps)


def _source(c, tag="fin", kind="saw"):
    """the signal a filter / nonlinearity / delay under test processes: an oscillator at a per-voice frequency"""
    r = c.reg()
    c.d.stage("osc", c.ctrl("P", tag, 40.0, 3000.0), kind=kind, dst=r)
    return r


FREQ_K = (0.0, -0.0, -220.0, 30000.0, 1e-300, 440.0, 0.75 * SR, 3.0, 1000.0)
FREQ_CORNERS = (0.0, -0.0, -330.0, 30000.0, 1e-300, 0.75 * SR, 440.0, 24000.0)


def osc_case(kind):
    table = kind in TABLE_OSC
    c = Case("osc_" + kind, kind not in LIBM_OSC)
    if table:
        lo, hi = (0.5, 24000.0) if kind == "sawn" else (0.0, 24000.0)
        corners = (1e-300, 24000.0, 0.5, 23999.5) if kind == "sawn" else (0.0, 24000.0, 1e-300, 0.25)
        kconst = 220.0
    else:
        lo, hi, corners, kconst = -500.0, 30000.0, FREQ_CORNERS, FREQ_K[list(OSC).index(kind) % len(FREQ_K)]
    regs = []
    for i, cls in enumerate(CLASSES):
        f = c.ctrl(cls, "f" + cls, lo, hi, corners, const=kconst)
        a1 = a2 = None
        c2 = CLASSES[(i + 1) % 4]
        if kind == "pulse":
            a1 = c.ctrl(c2, "duty" + c2, -0.2, 1.2, (-0.5, 0.0, 1.0, 1.5), const=(-0.25, 0.3, 1.25, 0.5)[i])
        if kind == "phasorbetween":
            a1 = c.ctrl(c2, "start" + c2, -0.5, 0.8, (0.9, 0.0, -0.25, 0.5), const=(0.2, 0.9, -0.3, 0.0)[i])
            c3 = CLASSES[(i + 2) % 4]
            a2 = c.ctrl(c3, "end" + c3, 0.2, 1.5, (0.1, 1.0, 0.5, 0.2), const=(0.8, 0.1, 1.3, 1.0)[i])
        r = c.reg()
        c.d.stage("osc", *[x for x in (f, a1, a2) if x is not None], kind=kind, dst=r)
        regs.append(r)
    return c.finish(regs)


def filter_case(kind):
    c = Case("filter_" + kind, kind in ("lopass", "hipass"))
    src = _source(c)
    regs = []
    for i, cls in enumerate(CLASSES):
        c2 = CLASSES[(i + 1) % 4]
        if kind in ("lores", "hires"):
            cut = c.ctrl(cls, "cut" + cls, 0.0, 60000.0, (5.0, 10.0, -100.0, SR, 60000.0, 800.0), const=(5.0, 60000.0, 1500.0, 9.0)[i])
            res = c.ctrl(c2, "res" + c2, 0.5, 6.0, (0.5, 1.0, 0.0, 4.0), const=(0.5, 3.0, 1.0, 2.0)[i])
        elif kind == "bandpass":
            cut = c.ctrl(cls, "cut" + cls, 50.0, 30000.0, (24000.0, 30000.0, 0.0, 1000.0), const=(30000.0, 24000.0, 700.0, 5000.0)[i])
            res = c.ctrl(c2, "res" + c2, 0.0, 1.5, (0.999, 1.0, 1.5, 0.0), const=(1.0, 0.0, 1.2, 0.5)[i])
        else:
            cut = c.ctrl(cls, "cut" + cls, 0.0, 1.0, (0.0, 1.0, 0.5), const=(0.0, 1.0, 0.3, 0.05)[i])
            res = None
        r = c.reg()
        c.d.stage("filter", src, cut, *([res] if res is not None else []), kind=kind, dst=r)
        regs.append(r)
    return c.finish(regs)


def svf_case():
    c = Case("svf", False)
    src = _source(c)
    regs = []
    for i, cls in enumerate(CLASSES):
        c2 = CLASSES[(i + 1) % 4]
        cut = c.ctrl(cls, "cut" + cls, 50.0, 20000.0, (50.0, 20000.0, 1000.0), const=(300.0, 5000.0, 12000.0, 80.0)[i])
        res = c.ctrl(c2, "res" + c2, 0.0, 4.0, (0.0, 0.5, 10.0), const=(0.0, 1.0, 2.0, 0.7)[i])
        mix = [c.ctrl(CLASSES[(i + k) % 4], "mw%d" % k + CLASSES[(i + k) % 4], -1.0, 1.0, (0.0, 1.0), const=(1.0, 0.5, -0.25, 0.0)[k]) for k in range(4)]
        r = c.reg()
        c.d.stage("svf", src, cut, res, *mix, dst=r)
        regs.append(r)
    return c.finish(regs)


def biquad_case(kind):
    c = Case("biquad_" + kind, False)
    src = _source(c)
    regs = []
    for i, cls in enumerate(CLASSES):
        c2, c3 = CLASSES[(i + 1) % 4], CLASSES[(i + 2) % 4]
        cut = c.ctrl(cls, "cut" + cls, 50.0, 20000.0, (50.0, 20000.0, 1000.0), const=(300.0, 5000.0, 12000.0, 80.0)[i], smooth=True)
        q = c.ctrl(c2, "q" + c2, 0.3, 10.0, (0.3, 0.7071067811865476, 10.0), const=(0.5, 0.7071067811865476, 4.0, 2.0)[i], smooth=True)
        gain = c.ctrl(c3, "gain" + c3, -24.0, 24.0, (6.0, 0.0, -6.0, -0.0), const=(6.0, 0.0, -9.0, -0.0)[i], smooth=True)
        r = c.reg()
        c.d.stage("biquad", src, cut, q, gain, kind=kind, dst=r)
        regs.append(r)
    return c.finish(regs)


def dcblock_case():
    c = Case("dcblock", True)
    src = _source(c)
    c.d.stage("add", src, c.d.K(0.25), dst=src)                                # a DC offset to remove
    regs = []
    for cls in CLASSES:
        r = c.reg()
        c.d.stage("dcblock", src, c.ctrl(cls, "R" + cls, 0.9, 0.999, (0.995, 1.0, 0.0)), dst=r)
        regs.append(r)
    return c.finish(regs)


def nonlin_case(kind):
    c = Case("nonlin_" + kind, kind in ("fastatan", "fastatandist", "hardclip"))
    src = _source(c)
    c.d.stage("mul", src, c.d.K(1.5), dst=src)                                 # the saw crosses the clip rails
    stream = c.ctrl("I", "x", -2.0, 2.0, (1.0, -1.0, 0.0, 1.0000000000000002, -0.9999999999999999))
    regs = []
    for i, cls in enumerate(CLASSES):
        x = stream if i % 2 else src
        c2 = CLASSES[(i + 1) % 4]
        a = c.ctrl(cls, "a" + cls, 0.5, 8.0, (0.5, 1.0, 8.0), const=(0.5, 2.0, 5.0, 1.0)[i])
        b = c.ctrl(c2, "b" + c2, 0.5, 3.0, (0.5, 1.0, 3.0), const=(1.5, 0.7, 2.0, 1.0)[i])
        r = c.reg()
        c.d.stage("nonlin", x, a, b, kind=kind, dst=r)
        regs.append(r)
    return c.finish(regs)


TAPS = 64


def delay_case(kind):
    c = Case("delay_" + kind, True, TAPS)
    src = _source(c)
    pos = kind == "position"
    regs = []
    for i, cls in enumerate(CLASSES):
        c2 = CLASSES[(i + 1) % 4]
        size = c.ctrl(cls, "size" + cls, 1.0, TAPS, (1.0, TAPS, 2.0, TAPS - 1.0), const=(1.0, TAPS, 17.0, 2.0)[i], integral=True, rate=7.0)
        fb = c.ctrl(c2, "fb" + c2, 0.0, 1.2, (0.0, 1.5, 1.0), const=(0.0, 1.1, 0.5, 1.0)[i])
        args = [src, size, fb]
        if pos:
            c3 = CLASSES[(i + 2) % 4]
            args.append(c.ctrl(c3, "pos" + c3, 0.0, 80.0, (0.0, TAPS - 1.0, TAPS, 80.0), const=(0.0, 30.0, TAPS, 80.0)[i], integral=True))
        r = c.reg()
        c.d.stage("delay", *args, kind=kind, dst=r)
        regs.append(r)
    return c.finish(regs)


def flanger_case():
    c = Case("flanger", True, TAPS)
    src = _source(c)
    d = c.d
    r0, r1, r2 = c.reg(), c.reg(), c.reg()
    # 750 Hz: the LFO increment is 1/64 exactly, so the triangle reaches +1 and the sweep reaches 21 + 2 * 21 + 1 = 64 = taps
    d.stage("flanger", src, d.K(21.0), c.ctrl("P", "fbP", 0.0, 0.9, (0.0, 1.2)), d.K(750.0), d.K(2.0), dst=r0)
    d.stage("flanger", src, c.ctrl("P", "dl", 1.0, 30.0, (1.0, 30.0), integral=True), c.ctrl("R", "fbR", 0.0, 0.9),
            c.ctrl("I", "speed", 0.1, 40.0, (0.0, 750.0)), c.ctrl("P", "depth", 0.0, 1.0, (0.0, 1.0)), dst=r1)
    d.stage("flanger", src, c.ctrl("I", "dlI", 1.0, 31.0, (1.0, 31.0), integral=True), c.ctrl("I", "fbI", 0.0, 1.1, (0.0,)),
            c.ctrl("P", "speedP", 0.1, 750.0, (0.0, 750.0, 1e-300)), c.ctrl("I", "depthI", 0.0, 1.0, (1.0,)), dst=r2)
    return c.finish([r0, r1, r2])


def env_case(op):
    c = Case(op, True)
    d = c.d
    adsr = op == "env_adsr"
    src = _source(c, "fin", "triangle")
    regs = []
    trig_kinds = [("K", "f64"), ("P", "f64"), ("R", "f64"), ("I", "f64"), ("I", "u8"), ("I", "bits")]
    for i, (tcls, ty) in enumerate(trig_kinds):
        tr = c.trig(tcls, "trig%d" % i, ty)
        rc = CLASSES[i % 4]
        att = c.ctrl(rc, "att" + rc, 0.01, 0.5, (0.01, 1.0, 0.3), const=0.2)
        rel = c.ctrl(CLASSES[(i + 1) % 4], "rel" + CLASSES[(i + 1) % 4], 0.9, 0.999, (0.9, 0.999), const=0.95)
        if i in (3, 4, 5):
            ht = c.ctrl("P", "ht%d" % i, 0.0, 40.0, HOLDTIMES, integral=True)      # the gated stages see every holdtime corner
        else:
            ht = c.ctrl(CLASSES[(i + 2) % 4], "ht" + CLASSES[(i + 2) % 4], 0.0, 40.0, HOLDTIMES, const=2.0 ** 32 + 3, integral=True)
        r = c.reg()
        if adsr:
            dec = c.ctrl(CLASSES[(i + 3) % 4], "dec" + CLASSES[(i + 3) % 4], 0.9, 0.99, (0.9,), const=0.95)
            sus = c.ctrl(CLASSES[(i + 2) % 4], "sus" + CLASSES[(i + 2) % 4], 0.1, 0.9, (0.5,), const=0.5)
            d.stage("env_adsr", src if i % 2 else d.K(1.0), tr, att, dec, sus, rel, ht, dst=r)
        else:
            d.stage("env_ar", src if i % 2 else d.K(1.0), tr, att, rel, ht, dst=r)
        regs.append(r)
    return c.finish(regs)


def envgen_case():
    c = Case("envgen", False)
    d = c.d
    d.envgen([0.0, 1.0, 0.4, 0.4, 0.0], [2.0, 3.0, ENVGEN_HOLD, 4.0], [1.0, 2.5, 1.0, 0.5], loop=False, retrigger=True)
    regs = []
    for cls in ("K", "P", "R", "I"):
        tr = c.trig(cls, "egtrig" + cls)
        r = c.reg()
        d.stage("envgen", tr, dst=r)
        regs.append(r)
    return c.finish(regs)


def envgen_nan_curve_case():
    """maxiMap::linlin clamps with std::min / std::max, which let a NaN through: a NaN curve makes the segment's level NaN"""
    c = Case("envgen_nan_curve", False)
    d = c.d
    d.envgen([0.0, 1.0, 0.5, 0.0], [1.0, 2.0, 1.5], [2.0, float("nan"), 1.0], loop=True, retrigger=False)
    c.ispec["gate"] = ("gate", "f64")
    r = c.reg()
    d.stage("envgen", d.IN("gate"), dst=r)
    return c.finish([r])


def chorus_case():
    c = Case("chorus", False, 512)
    d = c.d
    src = _source(c)
    c.ispec["noise"] = ("noise",)
    r = c.reg()
    d.stage("chorus", src, d.K(120.0), c.ctrl("P", "fb", 0.0, 0.9, (0.0,)), c.ctrl("R", "speed", 20.0, 60.0), c.ctrl("P", "depth", 0.2, 0.8),
            d.IN("noise"), dst=r)
    return c.finish([r])


def arith_case(op):
    c = Case("arith_" + op, True)
    d = c.d
    regs = []
    for i, cls in enumerate(CLASSES):
        c2 = CLASSES[(i + 1) % 4]
        a = c.ctrl(cls, "a" + cls, -3.0, 3.0, (0.0, -0.0, 1.0), const=(0.5, -0.0, 3.0, -1.5)[i])
        b = c.ctrl(c2, "b" + c2, 0.5, 2.0, (0.5, 2.0, -1.0), const=(1.5, 0.25, -2.0, 3.0)[i])
        r = c.reg()
        d.stage(op, a, b, dst=r)
        regs.append(r)
    if op == "div":                                      # x / +0 and x / -0 (and 0 / 0): infinities of either sign, NaN
        x = c.ctrl("I", "x", -1.0, 1.0, (0.0, -0.0, 1.0))
        r1, r2 = c.reg(), c.reg()
        d.stage("div", x, d.K(0.0), dst=r1)
        d.stage("div", x, d.K(-0.0), dst=r2)
        d.stage("mix_stereo", r1, d.K(0.25))
        d.stage("mix_stereo", r2, d.K(0.75))
        d.stage("out", r1)                               # overridden by the sum below: the last OUT wins
    return c.finish(regs)


def special_consts_case():
    """constants with special bit patterns (-0, +-inf, NaN, subnormals) as operands"""
    c = Case("special_consts", True)
    d = c.d
    x = c.ctrl("I", "x", -1.0, 1.0, (0.0, -0.0))
    r0, r1, r2, r3 = c.reg(), c.reg(), c.reg(), c.reg()
    d.stage("add", x, d.K(-0.0), dst=r0)                                        # -0 + -0 = -0, x + -0 = x
    d.stage("mul", r0, d.K(5e-324), dst=r1)                                     # the smallest subnormal
    d.stage("add", r1, d.K(2.2250738585072009e-308), dst=r1)                    # the largest subnormal
    d.stage("mul", r1, d.K(2.0 ** 1000), dst=r1)
    d.stage("mul", x, d.K(float("inf")), dst=r2)                                # +-inf, NaN at x = 0
    d.stage("add", x, d.K(float("-inf")), dst=r3)
    d.stage("mix_stereo", r2, d.K(0.5))
    d.stage("mix_stereo", r3, d.K(float("nan")))                                # a NaN pan passes both clamps
    d.stage("mul", r0, d.K(float("nan")), dst=r2)
    d.stage("out", r2)                                                          # overridden below
    return c.finish([r1, r0], pan=False)


def placement_case():
    """OUT and MIX_STEREO with a dst (which reads 0 after them), two OUT stages (the last wins), two MIX_STEREO stages (they add up),
    a register read before the stage that writes it in this sample (0), pans at and beyond 0 and 1"""
    c = Case("placement", True)
    c.nreg = 10                                                                 # R0..R9 are named below
    d = c.d
    x = c.ctrl("I", "x", -1.0, 1.0, (0.0, 1.0, -1.0))
    d.stage("add", x, R(9), dst=R(0))                                           # R9 is written at the end of the sample
    d.stage("out", R(0), dst=R(4))
    d.stage("mix_stereo", R(0), c.ctrl("P", "pan", 0.0, 1.0, PANS), dst=R(5))
    d.stage("mix_stereo", x, c.ctrl("R", "panR", -0.5, 1.5))
    d.stage("add", R(4), R(5), dst=R(6))
    d.stage("mul", R(0), d.K(0.5), dst=R(7))
    d.stage("add", R(7), R(6), dst=R(8))
    d.stage("out", R(8))
    d.stage("add", R(8), d.K(1.0), dst=R(9))
    return (c.name, c.d, c.params, c.inputs, c.exact, c.taps)


def cases():
    out = [osc_case(k) for k in OSC]
    out += [filter_case(k) for k in FILT]
    out += [svf_case()]
    out += [biquad_case(k) for k in BIQUAD]
    out += [dcblock_case()]
    out += [nonlin_case(k) for k in NONLIN]
    out += [delay_case(k) for k in DELAY]
    out += [flanger_case(), env_case("env_adsr"), env_case("env_ar"), envgen_case(), envgen_nan_curve_case(), chorus_case()]
    out += [arith_case(op) for op in ("add", "sub", "mul", "div")]
    out += [special_consts_case(), placement_case()]
    return out


def coverage(case_list):
    """the (op name, kind name) pairs the cases run, kind None for ops without a kind table"""
    ops = {v: k for k, v in OP.items()}
    tables = dict(osc=OSC, filter=FILT, biquad=BIQUAD, nonlin=NONLIN, delay=DELAY)
    seen = set()
    for _, d, *_ in case_list:
        for op, kind, dst, src in d.stages:
            name = ops[op]
            if name in tables:
                seen.add((name, {v: k for k, v in tables[name].items()}[kind]))
            else:
                seen.add((name, None))
    return seen
