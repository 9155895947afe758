"""The bank matrix: every instantiation of the two bank kernels, block-constant and modulated, as consecutive blocks of banks held
to the oracle. CPU-importable, no device.

An instantiation is named by its key:
  K1  bank_kernel<OSC, FILT, ENV, OUT, MIX, MOD>              (FILT_T, OSC_T, ENV, OUT, MIX, MOD)        480 kernels
  K2  delay_bank_kernel<OSC, FILT, ENV, OUTMODE, MIX, MODK>   (FILT_T, saw|generic, ENV, OUTMODE, MIX, MODK) 240 kernels
The bank's description fixes FILT, OSC and ENV (and the delay line); OUT, MIX, the output type and the streams are chosen per call. So
the keys are grouped by description: one GPU bank and one oracle bank per group, whose blocks run the group's keys one after the other,
a different instantiation on every block and blocks of different lengths, so that each kernel starts from state another one left.

The runtime branches inside the kernels are spread over the keys by a deterministic rotation (not a product): all nine oscillators,
ADSR and AR, gates and per-sample triggers, holdtimes other than 1, the seven biquad types, every store path, the voice counts and
block lengths where the kernels change shape, K2's ring schedules, and stream values at the corners of the straight-line increment
(0 Hz, negative, 2^-70, 2^61, above the sample rate, +inf, NaN: on one voice of a K1 thread pair and on a whole warp) and of the
coefficient design (cutoffs below the lores clamp, at and above the sample rate, SVF cutoffs at and above Nyquist). `tags()` lists
what each block exercises; tests/test_bank_matrix.py checks that every branch occurs in each kernel family.

Sinewave and coswave keep finite, moderate phases (their bar is libdevice's sin / cos against glibc's, 1e-12): no 2^61, inf or NaN
frequency on them. Values that leave a voice non-finite for good (2^61, inf, NaN frequencies; a lores / hires cutoff at or above the
sample rate, where the design divides 0 by 0) come late in a group, on a few voices, and only in every other group, so that the
other blocks keep a finite bus to compare. They are not fed to the low-pass-only SVF family (K1 and K2 `svf_lp`): it returns the
SVF's `low` output where the reference adds band, high and notch times 0, which is NaN once the state is not finite.
"""
import zlib
from dataclasses import dataclass, field

import numpy as np

SR = 48000.0
K_FM_PREFETCH = 8                                         # kFmPrefetch, bank_kernels.cuh: steps of look-ahead on a stream

FILT_T = ("none", "lores", "hires", "svf", "svf_lp", "biquad")     # FILT_T_* of bank_kernels.cuh, in enum order
OSC_T = ("sine", "phasor", "saw", "generic")                         # OSC_T_*
CUTOFF_MOD = ("lores", "hires", "svf", "svf_lp")                     # the families with a per-sample coefficient design
OUT_MIX = ((True, True), (True, False), (False, True))               # K1: out + mix, out, mix only
K2_OUT = (("f64", True), ("f64", False), ("f32", True), ("f32", False), ("none", True))     # DL_OUT_* x MIX; no output: bus only
K1_GENERIC = ("coswave", "square", "pulse", "impulse", "triangle", "phasorbetween")
K2_GENERIC = ("sinewave", "coswave", "phasor", "square", "pulse", "impulse", "triangle", "phasorbetween")
TRIG_OSC = ("sinewave", "coswave")
BIQUADS = ("lowpass", "highpass", "bandpass", "notch", "peak", "lowshelf", "highshelf")
VS = (1, 31, 33, 64, 97, 300)                             # a lone voice, partial warps and pairs, more than one 128-thread CTA
BS = (1, 5, 16, 17, 40, 129)                              # shorter than the look-ahead, one K2 window, ragged windows
TAPS = 128
GATE_MODES = ("gate", "tv", "full", "empty")              # [on, off) interval, per-sample bytes, held over the block, none
FM_CORNERS = (0.0, -300.0, 2.0 ** -70, 1.5 * SR)          # leave the voice finite
FM_POISON = (2.0 ** 61, np.inf, np.nan)                   # leave it non-finite (or its phase beyond 2^40) for good
CUT_LOW = (5.0, 0.0, -100.0, 9.999)                       # below the lores / hires clamp of 10 Hz


def k1_mods(filt):
    return (0, 1, 2, 3) if filt in CUTOFF_MOD else (0, 1)


K1_KEYS = [(f, o, e, out, mix, m) for f in FILT_T for o in OSC_T for e in (0, 1) for out, mix in OUT_MIX for m in k1_mods(f)]
K2_KEYS = [(f, o, e, om, mix, mk) for f in FILT_T for o in ("saw", "generic") for e in (0, 1) for om, mix in K2_OUT for mk in (0, 1)]


def key_of(desc, call):
    """The instantiation a block runs: desc = dict(osc, filt, env, delay, svf_mix), call = dict(out, mix, f32, freq_tv, cutoff_tv)
    (booleans). Restates the dispatch of mxb_bank_process_mod (bank.cu:561-598), launch_bank_filt (bank_k.cu:11-41) and
    launch_delay_filt (delay_k.cu:12-26)."""
    filt = desc["filt"]
    if filt == "svf" and tuple(float(x) for x in desc.get("svf_mix", (1.0, 0.0, 0.0, 0.0))) == (1.0, 0.0, 0.0, 0.0):
        filt = "svf_lp"                                   # bank.cu:572-573: the SVF with mix (1, 0, 0, 0)
    env = 1 if desc.get("env") else 0                     # bank.cu:565: ADSR and AR share ENV = 1 (env_ar is a runtime flag)
    fm, cm = bool(call.get("freq_tv")), bool(call.get("cutoff_tv"))
    assert not (cm and filt not in CUTOFF_MOD), "per-sample cutoff is refused for this filter (bank.cu:500-502)"
    if desc.get("delay"):
        osc = "saw" if desc["osc"] == "saw" else "generic"                                 # bank.cu:584
        outmode = "none" if not call["out"] else ("f32" if call["f32"] else "f64")      # bank.cu:585
        mix = True if outmode == "none" else bool(call["mix"])                           # delay_k.cu:21: no output, bus only
        return "k2", (filt, osc, env, outmode, mix, int(fm or cm))                       # bank.cu:586: any stream -> MODK
    osc = {"sinewave": "sine", "phasor": "phasor", "saw": "saw"}.get(desc["osc"], "generic")    # bank.cu:561-564
    return "k1", (filt, osc, env, bool(call["out"]), bool(call["mix"]), int(fm) | 2 * int(cm))  # bank_k.cu:24-29


def kernel_key(symbol):
    """The key of a demangled kernel symbol (cu++filt), or None for other symbols."""
    import re
    m = re.search(r"(delay_bank_kernel|bank_kernel)<\(int\)(\d+), \(int\)(\d+), \(int\)(\d+), \((?:bool|int)\)(\d+), \(bool\)(\d+), "
                  r"\((?:int|bool)\)(\d+)>", symbol)
    if not m:
        return None
    name, osc, filt, env, a, mix, mod = m.group(1), *(int(x) for x in m.groups()[1:])
    if name == "bank_kernel":
        return "k1", (FILT_T[filt], OSC_T[osc], env, bool(a), bool(mix), mod)
    return "k2", (FILT_T[filt], OSC_T[osc], env, ("none", "f64", "f32")[a], bool(mix), mod)


@dataclass
class Block:
    n: int
    key: tuple
    out: bool
    mix: bool
    f32: bool = False
    fm: bool = False
    cm: bool = False
    gate: str = "none"            # GATE_MODES or "none" (no envelope)
    size_tv: bool = False
    misaligned: bool = False      # K1: `out` one element past an aligned device address
    poison: bool = False          # this block's frequency stream carries FM_POISON values
    cut_nan: bool = False         # this block's cutoff stream reaches the sample rate (lores / hires: NaN from here on)
    exact: bool = True            # bit-identical expected (no sin / cos, no per-sample design so far in the group)
    tags: set = field(default_factory=set)


@dataclass
class Group:
    name: str
    family: str                   # "k1" | "k2"
    index: int
    desc: dict                    # osc, filt, env, delay, svf_mix, biquad_type
    V: int
    sched: str = ""               # K2: uniform | ragged | literal | position | nonpos
    steady: bool = False          # K2 ADSR: envelopes that reach their steady states within a window (ESTEADY)
    blocks: list = field(default_factory=list)

    @property
    def trig(self):
        return self.desc["osc"] in TRIG_OSC

    @property
    def max_frames(self):
        return max(b.n for b in self.blocks)

    def bank_kw(self):
        d = self.desc
        kw = dict(osc=d["osc"], filt=d["filt"], env=d["env"], svf_mix=d["svf_mix"], biquad_type=d["biquad_type"])
        if d["delay"]:
            kw.update(delay=d["delay"], delay_capacity=TAPS)
        return kw


def _rng(*key):
    return np.random.default_rng([zlib.crc32(repr(k).encode()) for k in key])


def _order_k1(filt):
    """Every (OUT, MIX) with every MOD once; non-cutoff keys first (bit-identical bars as long as possible), each block a new key"""
    seq = []
    for mods in ((0, 1), (2, 3)) if filt in CUTOFF_MOD else ((0, 1),):
        for r in range(3):
            for j, m in enumerate(mods):
                seq.append((OUT_MIX[(r + j) % 3], m))
    return seq


def _order_k2():
    return [(K2_OUT[(r + j) % 5], mk) for r in range(5) for j, mk in enumerate((1, 0))]


def _groups():
    groups, gi = [], 0
    k1_generic = k2_generic = bq = adsr_k2 = 0
    for family in ("k1", "k2"):
        for fi, filt in enumerate(FILT_T):
            for osc_t in (OSC_T if family == "k1" else ("saw", "generic")):
                for env in (0, 1):
                    if osc_t == "generic":
                        if family == "k1":
                            osc = K1_GENERIC[k1_generic % len(K1_GENERIC)]; k1_generic += 1
                        else:
                            osc = K2_GENERIC[k2_generic % len(K2_GENERIC)]; k2_generic += 1
                    else:
                        osc = {"sine": "sinewave"}.get(osc_t, osc_t)
                    env_kind = False if not env else ("ar" if (gi // 2) % 2 else "adsr")
                    btype = "lowpass"
                    if filt == "biquad":
                        btype = BIQUADS[bq % len(BIQUADS)]; bq += 1
                    svf_mix = (1.0, 0.0, 0.0, 0.0) if filt != "svf" else ((0.3, 0.2, 0.4, 0.1), (0.0, 1.0, 0.0, 0.0), (0.0, 0.0, 1.0, 1.0))[gi % 3]
                    g = Group(name="", family=family, index=gi,
                              desc=dict(osc=osc, filt="svf" if filt == "svf_lp" else filt, env=env_kind, svf_mix=svf_mix, biquad_type=btype,
                                        delay=False),
                              V=VS[gi % 6] if family == "k1" else VS[(gi + 3) % 6])
                    if family == "k2":
                        g.sched = ("uniform", "ragged", "literal", "position", "uniform", "nonpos")[gi % 6]
                        g.desc["delay"] = "position" if g.sched == "position" else "dl"
                        if env_kind == "adsr":
                            g.steady = adsr_k2 % 2 == 0; adsr_k2 += 1
                    g.name = f"{family}-{filt}-{osc}-{env_kind or 'noenv'}-V{g.V}" + (f"-{g.sched}" if family == "k2" else "") + \
                             (f"-{btype}" if filt == "biquad" else "")
                    _blocks(g, filt)
                    groups.append(g)
                    gi += 1
    return groups


def _blocks(g, filt):
    k2 = g.family == "k2"
    order = _order_k2() if k2 else _order_k1(filt)
    # The low-pass-only SVF family returns `low` where maxiSVF::play returns low*1 + band*0 + high*0 + notch*0 (bank_kernels.cuh:190):
    # the same value while the state is finite, NaN in the reference once it is not. So no poison on svf_lp.
    poison_ok = not g.trig and g.index % 2 == 1 and filt != "svf_lp"
    mod_blocks = [i for i, (_, m) in enumerate(order) if m]
    fm_only = [i for i, (_, m) in enumerate(order) if (m == 1)] if not k2 else mod_blocks[:2]
    poison_at = fm_only[-1] if poison_ok else -1
    cut_blocks = [i for i, (_, m) in enumerate(order) if (m & 2)] if not k2 else \
        ([i for i in mod_blocks[2:]] if filt in CUTOFF_MOD else [])
    nan_at = cut_blocks[-1] if (filt in ("lores", "hires") and g.index % 2 == 0 and cut_blocks) else -1
    exact = not g.trig
    ph, ph_known = 0, True                                 # K2 uniform: ring index at the start of the block
    ar_fm = 0
    for i, (om, m) in enumerate(order + [(None, 0)]):
        last = om is None
        n = BS[(g.index + i) % len(BS)]
        if k2:
            if last:
                outmode, mix, mk = "f64", False, 0
            else:
                (outmode, mix), mk = om, m
            fm = cm = False
            if mk:
                j = mod_blocks.index(i)
                kind = ("freq", "freq", "cutoff", "both", "cutoff")[j] if filt in CUTOFF_MOD else "freq"
                fm, cm = kind in ("freq", "both"), kind in ("cutoff", "both")
            b = Block(n=n, key=None, out=outmode != "none", mix=mix, f32=outmode == "f32", fm=fm, cm=cm)
        else:
            if last:
                (out, mix), m = (True, True), 0
            else:
                (out, mix), m = om, m
            b = Block(n=n, key=None, out=out, mix=mix, fm=bool(m & 1), cm=bool(m & 2))
            if out:
                b.f32 = (g.index + i) % 2 == 1
                b.misaligned = (g.index + i) % 5 == 2
        b.poison = i == poison_at
        b.cut_nan = i == nan_at
        if g.desc["env"]:
            b.gate = GATE_MODES[(g.index + i) % 4]
            if g.desc["env"] == "ar" and b.fm:                 # maxiEnv::ar under FM with per-sample triggers, on every other FM block
                ar_fm += 1
                b.gate = "tv" if ar_fm % 2 else b.gate
        b.size_tv = k2 and not last and (g.index + i) % 3 == 0
        if last:
            b.gate = "gate" if g.desc["env"] else "none"
        if b.cm:
            exact = False
        b.exact = exact
        _, b.key = key_of(g.desc, dict(out=b.out, mix=b.mix, f32=b.f32, freq_tv=b.fm, cutoff_tv=b.cm))
        b.tags = _tags(g, b, ph if ph_known else None)
        if k2:
            if b.size_tv:
                ph_known = False
            elif ph_known and g.sched == "uniform":
                p0 = ph if ph < 64 else 0
                ph = (p0 + n - 1) % 64 + 1
        g.blocks.append(b)


def _tags(g, b, ph):
    """what a block exercises, for the coverage test"""
    d, k2, V = g.desc, g.family == "k2", g.V
    t = {f"osc:{d['osc']}", f"V:{V}", f"B:{b.n}"}
    if d["env"]:
        t.add(f"env:{d['env']}")
        t.add(f"trig:{b.gate}")
        if b.gate == "tv":
            t.update(f"tv:{p}" for p in ("never", "always", "alternate")[:V])
        t.add("holdtime!=1")
        if b.fm and d["env"] == "ar":
            t.add("env:ar+fm")
        if b.fm and d["env"] == "ar" and b.gate == "tv":
            t.add("env:ar+fm+tv")
    if d["filt"] == "biquad":
        t.add(f"biquad:{d['biquad_type']}")
    if b.fm or b.cm:
        t.add("stream")
        if b.n < K_FM_PREFETCH:
            t.add("stream:short")
        if not b.out:
            t.add("stream:mix-only")
    if b.fm:
        t.update(("fm:0", "fm:negative", "fm:2^-70", "fm:above-sr") if not g.trig else ("fm:0", "fm:negative"))
        if V > 1:
            t.add("fm:pair")
        if V >= 32:
            t.add("fm:warp")
        if b.poison and (V >= 5 or b.n >= 3):
            t.update(("fm:2^61", "fm:inf", "fm:nan"))
        if d["osc"] == "phasorbetween":
            t.add("fm:phasorbetween")
    if b.cm:
        t.add("cut:below-10")
        if d["filt"] == "svf":
            t.update(("cut:nyquist", "cut:above-nyquist", "cut:above-sr-svf"))
        if b.cut_nan:
            t.add("cut:sr")
            if V > 1:
                t.add("cut:above-sr")
        if d["filt"] in ("lores", "hires"):
            t.add("res<1")
    if b.mix:
        t.add("pan:outside")
    if not k2:
        if b.out:
            paired = V % 2 == 0 and not b.misaligned
            t.add(f"store:{'paired' if paired else 'scalar'}{32 if b.f32 else 64}")
            if b.misaligned:
                t.add("store:misaligned")
    else:
        t.add(f"store:{'none' if not b.out else ('f32' if b.f32 else 'f64')}")
        if b.size_tv:
            t.update(("sched:size-tv", "sched:size<=0", "sched:size==taps"))
        elif g.sched == "position":
            t.add("sched:position")
        elif g.sched == "uniform" and ph is not None and (ph if ph < 64 else 0) % 16 == 0:
            t.add("sched:uniform")
        else:
            t.add("sched:generic")
            if g.sched in ("literal", "nonpos"):
                t.add("sched:literal")
            if g.sched == "nonpos":
                t.update(("sched:size<=0", "sched:size==taps"))
        # full or empty gate, every voice of the warp in sustain or release from the first window on: the two-statement windows
        if g.steady and not (b.fm or b.cm) and b.gate in ("full", "empty") and b.n > 16:
            t.add("esteady")
    return t


GROUPS = _groups()
K1_GROUPS = [g for g in GROUPS if g.family == "k1"]
K2_GROUPS = [g for g in GROUPS if g.family == "k2"]


# ------------------------------------------------------------------------------------------------ parameters and streams

def params(g):
    """the per-voice parameters of a group's banks (the same arrays for the GPU bank and the oracle)"""
    V, d = g.V, g.desc
    r = _rng("params", g.name)
    u = lambda: r.random(V)
    p = {"freq": 55.0 * np.exp2(5.0 * u()), "phase": u(), "duty": -0.2 + 1.4 * u()}
    p["phasor_start"] = 0.4 * u()
    p["phasor_end"] = 0.5 + 0.5 * u()
    pan = u()
    pan[: min(4, V)] = (-0.5, 1.5, 1.0, 0.0)[: min(4, V)] if V > 1 else ((1.5,) if g.index % 2 else (-0.5,))
    p["pan"] = pan
    if d["filt"] in ("lores", "hires"):
        p["cutoff"] = 100.0 * np.power(80.0, u()); p["resonance"] = 1.0 + 7.0 * u()
        p["resonance"][: min(2, V)] = (0.5, 0.0)[: min(2, V)] if V > 1 else (0.5,)      # below 1: the design's clamp
    elif d["filt"] == "svf":
        p["cutoff"] = 100.0 * np.power(80.0, u()); p["resonance"] = 0.5 + 4.5 * u()
    elif d["filt"] == "biquad":
        p["gain"] = np.linspace(-12.0, 12.0, V); p["cutoff"] = 100.0 * np.power(80.0, u()); p["resonance"] = 0.5 + 3.5 * u()
    if d["env"]:
        if g.steady:
            p["env_attack"] = np.full(V, 0.5); p["env_decay"] = np.full(V, 0.5); p["env_sustain"] = np.full(V, 0.3)
            p["env_release"] = np.choose(np.arange(V) % 3, [0.999, 0.5, 0.0])
            p["env_holdtime"] = np.choose(np.arange(V) % 3, [1.0, 0.0, 3.0])
        else:
            ms = lambda lo, hi: lo + (hi - lo) * u()
            p["env_attack"] = 1 - np.power(0.01, 1.0 / (ms(0.1, 3.0) * SR * 0.001))
            p["env_decay"] = np.power(0.01, 1.0 / (ms(1.0, 20.0) * SR * 0.001))
            p["env_sustain"] = 0.2 + 0.7 * u()
            p["env_release"] = np.power(0.01, 1.0 / (ms(0.5, 10.0) * SR * 0.001))
            p["env_holdtime"] = np.resize(np.array([1.0, 0.0, 3.0, 40.0, 2.0, 1.0, 300.0]), V)
    if d["delay"]:
        if g.sched == "uniform":
            size = np.full(V, 64.0)
        elif g.sched == "ragged":
            size = r.integers(32, TAPS + 1, V).astype(np.float64)
        elif g.sched == "literal":
            size = np.where(np.arange(V) % 3 == 0, r.integers(1, 32, V), r.integers(32, TAPS + 1, V)).astype(np.float64)
        elif g.sched == "nonpos":
            size = r.integers(32, TAPS + 1, V).astype(np.float64)
            size[: min(4, V)] = (0.0, -3.0, 1.0, float(TAPS))[: min(4, V)]
            if V == 1:
                size[0] = 0.0
        else:
            size = r.integers(1, TAPS + 1, V).astype(np.float64)
        p["delay_size"] = size
        p["delay_feedback"] = 0.1 + 0.8 * u()
        if g.sched == "position":
            p["delay_position"] = r.integers(0, 2 * TAPS, V).astype(np.float64)        # positions >= size read slot 0
    return p


def _trigger_bytes(r, n, V):
    t = np.zeros((n, V), dtype=np.uint8)
    for v in range(V):
        pos = int(r.integers(0, 20))
        while pos < n:
            ln = int(r.integers(1, 30))
            t[pos:pos + ln, v] = 1
            pos += ln + int(r.integers(1, 40))
    t[:, 0] = 0                               # never
    if V > 1:
        t[:, 1] = 1                           # always
    if V > 2:
        t[:, 2] = 0; t[::2, 2] = 1            # every other sample
    return t


def streams(g, i):
    """the call of block i: dict(trig_on, trig_off, trig_tv, freq_tv, cutoff_tv, delay_size_tv) (arrays or None)"""
    b, V, n = g.blocks[i], g.V, g.blocks[i].n
    r = _rng("streams", g.name, i)
    s = dict(trig_on=None, trig_off=None, trig_tv=None, freq_tv=None, cutoff_tv=None, delay_size_tv=None)
    if b.gate == "gate":
        s["trig_on"] = r.integers(0, n // 4 + 1, V).astype(np.int32)
        s["trig_off"] = r.integers(n // 2, n + 1, V).astype(np.int32)
    elif b.gate == "full":
        s["trig_on"] = np.zeros(V, np.int32); s["trig_off"] = np.full(V, n, np.int32)
    elif b.gate == "empty":
        s["trig_on"] = np.zeros(V, np.int32); s["trig_off"] = np.zeros(V, np.int32)
    elif b.gate == "tv":
        s["trig_tv"] = _trigger_bytes(r, n, V)
    t = (sum(x.n for x in g.blocks[:i]) + np.arange(n))[:, None] / SR
    if b.fm:
        carrier = 110.0 * np.exp2(3.0 * r.random(V)); depth = 50.0 * r.random(V); rate = 0.5 + 8.0 * r.random(V)
        f = carrier[None, :] + depth[None, :] * np.sin(2 * np.pi * rate[None, :] * t)
        if g.trig:
            f[0, 0] = FM_CORNERS[i % 2]                               # 0 Hz or negative: the phase stays moderate
        else:
            f[0, 0] = FM_CORNERS[i % len(FM_CORNERS)]                 # one voice of a thread pair; its neighbour is sane
            if n > 1:
                f[1, 0] = FM_CORNERS[(i + 1) % len(FM_CORNERS)]
                f[n - 1, V - 1] = FM_CORNERS[(i + 2) % len(FM_CORNERS)]
            for c in FM_CORNERS:                                      # each corner somewhere in the block
                f[int(r.integers(0, n)), int(r.integers(0, V))] = c
        f[n // 2, : min(32, V)] = 0.0                                 # a whole warp
        if b.poison:
            for k, c in enumerate(FM_POISON):
                f[max(0, n - 1 - k), min(2 + k, V - 1)] = c
        s["freq_tv"] = f
    if b.cm:
        centre = 200.0 * np.exp2(4.0 * r.random(V)); depth = 1.5 * r.random(V); rate = 0.2 + 6.0 * r.random(V)
        c = centre[None, :] * np.exp2(depth[None, :] * np.sin(2 * np.pi * rate[None, :] * t))
        c[0, 0] = CUT_LOW[i % len(CUT_LOW)]
        c[n - 1, V - 1] = CUT_LOW[(i + 1) % len(CUT_LOW)]
        if g.desc["filt"] == "svf":                                   # no clamp: Nyquist, above it, above the sample rate
            c[n // 2, 0] = SR / 2
            c[n // 2, min(1, V - 1)] = 0.625 * SR
            c[n - 1, min(3, V - 1)] = 1.25 * SR
        if b.cut_nan:                                                 # lores / hires: clamped to sr, z == 1, 0 / 0
            c[n - 1, max(0, V - 2)] = 2 * SR
            c[n - 1, V - 1] = SR
        s["cutoff_tv"] = c
    if b.size_tv:
        sz = np.floor(1 + TAPS * r.random((n, V)))
        sz = np.minimum(sz, TAPS)
        sz[0, 0] = 0.0
        sz[n - 1, V - 1] = -2.0
        sz[n // 2, :] = TAPS
        s["delay_size_tv"] = sz
    return s


def required_tags(family):
    """the branches every family must reach somewhere in the table"""
    req = {f"osc:{o}" for o in ("sinewave", "phasor", "saw") + K1_GENERIC} | {"env:adsr", "env:ar", "trig:gate", "trig:tv", "trig:full",
                                                                               "trig:empty", "tv:never", "tv:always", "tv:alternate",
                                                                               "holdtime!=1", "env:ar+fm", "env:ar+fm+tv"}
    req |= {f"V:{v}" for v in VS} | {f"B:{n}" for n in BS}
    req |= {"stream:short", "stream:mix-only", "fm:pair", "fm:warp", "fm:0", "fm:negative", "fm:2^-70", "fm:above-sr", "fm:2^61", "fm:inf",
            "fm:nan", "fm:phasorbetween", "cut:below-10", "cut:sr", "cut:above-sr", "cut:nyquist", "cut:above-nyquist", "res<1", "pan:outside"}
    if family == "k1":
        req |= {"store:paired64", "store:scalar64", "store:paired32", "store:scalar32", "store:misaligned"}
    else:
        req |= {"store:f64", "store:f32", "store:none", "sched:uniform", "sched:generic", "sched:literal", "sched:position",
                "sched:size-tv", "sched:size<=0", "sched:size==taps", "esteady"}
    return req
