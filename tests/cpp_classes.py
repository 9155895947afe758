"""What each case of tests/cpp/patch_classes.cpp means, written from the reference's signatures (src/maximilian.h, src/maximilian.cpp; the
`ref` of every case cites the line whose signature the case's play() follows). CPU-importable, no device.

A case's per-voice arrays P[k], gates and streams are generated here and handed to the driver in in.bin (the layout the driver's header
comment gives). The expectation is one of:
  bank   the oracle_py.Bank configuration (the arguments of workloads.configure_bank's bank) and what each P[k] sets on it: the case must
         run on the fused bank, and its `_x1` copy (`w * 1.0` appended) as a voice patch, both against this bank;
  patch  a patchdef.PatchDef with the stages the play() records, in order, and which P[k] / stream feeds each parameter / input;
  error  the maxiError code and the block that raises it.
"""
import zlib

import numpy as np

from maximilian_b200.patchdef import ENVGEN_HOLD, PatchDef, R

ERR_UNSUPPORTED = -4
OSC_KINDS = ("sinewave", "coswave", "phasor", "saw", "square", "pulse", "impulse", "triangle", "phasorbetween")
OSC_REF = dict(sinewave="src/maximilian.h:186", coswave="src/maximilian.h:189", phasor="src/maximilian.h:193", saw="src/maximilian.h:191",
               square="src/maximilian.h:183", pulse="src/maximilian.h:202", impulse="src/maximilian.h:204", triangle="src/maximilian.h:200",
               phasorbetween="src/maximilian.cpp:321")
# the driver's bank state, in order: MXB_P_PHASE, MXB_S_OSC_OUTPUT, MXB_S_FILT_0..2, MXB_S_ENV_*, MXB_S_DELAY_PHASE
BANK_STATE = ("phase", "osc_output", "filt0", "filt1", "filt2", "env_amplitude", "env_output", "env_holdcount", "env_flags", "delay_phase")


def _rng(*key):
    return np.random.default_rng([zlib.crc32(str(k).encode()) for k in key])


def U(lo, hi, integral=False, change=False):
    """a per-voice array uniform in [lo, hi) (floored when integral); the same on every block, or (change) new on block 1 and kept on 2"""
    def gen(name, k, V, blk):
        x = _rng(name, k, min(blk, 1) if change else 0).uniform(lo, hi, V)
        return np.floor(x) if integral else x
    return gen


def CHOICE(*values):
    return lambda name, k, V, blk: _rng(name, k).choice(np.array(values, dtype=np.float64), V)


def BLOCKS(*per_block):
    """a per-voice trigger value that differs from block to block: per_block[blk] chooses among its values"""
    return lambda name, k, V, blk: _rng(name, k, blk).choice(np.array(per_block[blk], dtype=np.float64), V)


def note_gates(name, V, B, blk):
    rng = _rng(name, "gate", blk)
    return rng.integers(0, B // 4 + 1, V), rng.integers(B // 2, 3 * B // 4 + 1, V)


def edge_gates(name, V, B, blk):
    """on < 0, off > B, on > off, on == off (no note) and an ordinary note, by voice and block"""
    pats = [(-5, 60), (B // 2, B + 40), (120, 40), (0, 0), (10, 100), (-3, B + 10), (B, B)]
    on, off = np.zeros(V, dtype=np.int64), np.zeros(V, dtype=np.int64)
    for v in range(V):
        on[v], off[v] = pats[(v + 2 * blk) % len(pats)]
    return on, off


def trigger_stream(name, tag, V, B, blk):
    """0 / 1 per sample: notes that start and end anywhere in the block"""
    rng = _rng(name, tag, blk)
    g = np.zeros((B, V))
    for v in range(V):
        pos = int(rng.integers(0, 20))
        while pos < B:
            ln = int(rng.integers(5, 80))
            g[pos:pos + ln, v] = 1.0
            pos += ln + int(rng.integers(10, 120))
    return g


class Case:
    def __init__(self, name, kind, ref, params, cap=0, sr=48000, gates=None, streams=(), out=True, mix=True, **kw):
        self.name, self.kind, self.ref, self.params, self.cap, self.sr = name, kind, ref, list(params), cap, sr
        self.gates, self.streams, self.out, self.mix = gates, list(streams), out, mix
        self.__dict__.update(kw)

    def data(self, V, B, blk):
        P = [g(self.name, k, V, blk) for k, g in enumerate(self.params)]
        on, off = self.gates(self.name, V, B, blk) if self.gates else (np.zeros(V), np.zeros(V))
        S = [s(self.name, k, V, B, blk) for k, s in enumerate(self.streams)]
        return P, np.asarray(on, dtype=np.int32), np.asarray(off, dtype=np.int32), S

    def write(self, path, V, B, NB, tables):
        with open(path, "wb") as f:
            f.write(np.asarray(tables, dtype=np.float64).tobytes())
            for blk in range(NB):
                P, on, off, S = self.data(V, B, blk)
                for a in P + [on.astype(np.float64), off.astype(np.float64)] + [s.reshape(-1) for s in S]:
                    f.write(np.ascontiguousarray(a, dtype=np.float64).tobytes())


# ------------------------------------------------------------------------------------------------ bank-shaped

def _bank(name, ref, params, cfg, setter, **kw):
    """cfg: oracle_py.Bank keyword arguments; setter(bank, P, blk, lib): what the play() hands the bank before block blk"""
    return Case(name, "bank", ref, params, cfg=cfg, setter=setter, **kw)


def _osc_case(kind):
    def setter(b, P, blk, lib):
        b.set("freq", P[0]); b.set("pan", P[1])
        if kind == "pulse":
            b.set("duty", P[2])
        if kind == "phasorbetween":
            b.set("phasor_start", P[2]); b.set("phasor_end", P[3])
    return _bank("osc_" + kind, OSC_REF[kind], [U(30.0, 4000.0), U(0.0, 1.0), U(0.05, 0.45), U(0.55, 1.0)], dict(osc=kind), setter)


def _biquad_case(btype, gain, suffix=""):
    def setter(b, P, blk, lib):
        b.set("freq", P[0]); b.set("gain", gain); b.set("cutoff", P[1]); b.set("resonance", P[2]); b.set("pan", P[3])
    return _bank("biquad_" + btype + suffix, "src/maximilian.h:1375", [U(30.0, 2000.0), U(200.0, 8000.0), U(0.5, 4.0), U(0.0, 1.0)],
                 dict(osc="saw", filt="biquad", biquad_type=btype), setter)


def bank_cases():
    c = [_osc_case(k) for k in OSC_KINDS]

    def ar_lores(b, P, blk, lib):
        b.set("freq", P[0]); b.set("env_attack", P[1]); b.set("env_release", P[2]); b.set("env_holdtime", P[3])
        b.set("cutoff", P[4]); b.set("resonance", P[5])
    c.append(_bank("saw_ar_lores_out", "src/maximilian.cpp:1319 ar(input, attack, release, holdtime, trigger); :455 lores(input, cutoff1, resonance)",
                   [U(30.0, 2000.0), U(0.01, 0.3), U(0.9, 0.999), CHOICE(0.0, 1.0, 5.0, 40.0), U(200.0, 5000.0), U(1.0, 6.0)],
                   dict(osc="saw", filt="lores", env="ar"), ar_lores, gates=note_gates, mix=False))

    def adsr_hires(b, P, blk, lib):
        b.set("freq", P[0]); b.set("env_attack", P[1]); b.set("env_decay", P[2]); b.set("env_sustain", P[3]); b.set("env_release", P[4])
        b.set("env_holdtime", 3.0); b.set("cutoff", P[5]); b.set("resonance", P[6]); b.set("pan", P[7])
    c.append(_bank("square_adsr_hires_bus", "src/maximilian.cpp:1362 adsr(input, attack, decay, sustain, release, holdtime, trigger); :471 hires",
                   [U(30.0, 2000.0), U(0.01, 0.3), U(0.9, 0.999), U(0.2, 0.8), U(0.9, 0.999), U(200.0, 5000.0), U(1.0, 6.0), U(0.0, 1.0)],
                   dict(osc="square", filt="hires", env="adsr"), adsr_hires, gates=note_gates, out=False))
    for btype in ("lowpass", "highpass", "bandpass", "notch"):
        c.append(_biquad_case(btype, 0.0))
    for btype in ("peak", "lowshelf", "highshelf"):
        c.append(_biquad_case(btype, 6.0, "_p6"))
        c.append(_biquad_case(btype, -6.0, "_m6"))

    def tri_svf(b, P, blk, lib):
        b.set("freq", P[0])
        b.set("env_attack", [lib.mxo_env_attack_ms_coeff(x, 48000) for x in P[1]])
        b.set("env_decay", [lib.mxo_env_decay_coeff(x, 48000) for x in P[2]])
        b.set("env_sustain", P[3]); b.set("env_release", [lib.mxo_env_decay_coeff(x, 48000) for x in P[4]]); b.set("env_holdtime", 1.0)
        b.set("cutoff", P[5]); b.set("resonance", P[6])
        b.set("delay_size", P[7]); b.set("delay_feedback", P[8]); b.set("delay_position", P[9]); b.set("pan", P[10])
    c.append(_bank("tri_adsr_svf_dlpos", "src/maximilian.cpp:1485 setAttackMS, :1474 setDecay, :1469 setRelease, :1415 adsr(input, trigger); "
                   "src/maximilian.h:1305 maxiSVF::play(w, lpmix, bpmix, hpmix, notchmix); src/maximilian.cpp:431 dlFromPosition(input, size, feedback, position)",
                   [U(30.0, 2000.0), U(1.0, 20.0), U(10.0, 100.0), U(0.2, 0.8), U(20.0, 200.0), U(200.0, 5000.0), U(0.5, 5.0),
                    U(1.0, 257.0, True), U(0.1, 0.9), U(0.0, 256.0, True), U(0.0, 1.0)],
                   dict(osc="triangle", filt="svf", env="adsr", delay="position", delay_capacity=256, svf_mix=(0.3, 0.2, 0.4, 0.1)), tri_svf,
                   cap=256, gates=note_gates))

    def saw_sum(b, P, blk, lib):
        b.set("freq", P[0]); b.set("pan", 0.0)
    c.append(_bank("saw_sum", "src/maximilian.cpp:503 stereo(input, two, x) at x = 0: the left channel is the plain sum", [U(30.0, 2000.0)],
                   dict(osc="saw"), saw_sum))

    def phase_reset(b, P, blk, lib):
        b.set("freq", P[0]); b.set("pan", P[2])
        if blk != 1:
            b.set("phase", P[1])
    c.append(_bank("phasor_phase_reset", "src/maximilian.cpp:222 phaseReset(phaseIn)", [U(30.0, 2000.0), U(0.0, 1.0), U(0.0, 1.0)],
                   dict(osc="phasor"), phase_reset))

    def default_svf(b, P, blk, lib):
        b.set("freq", P[0]); b.set("cutoff", 1000.0); b.set("resonance", 1.0); b.set("pan", P[1])
    c.append(_bank("saw_default_svf", "src/maximilian.h:1284 maxiSVF() : setParams(1000, 1)", [U(30.0, 2000.0), U(0.0, 1.0)],
                   dict(osc="saw", filt="svf"), default_svf))

    def sine_44k(b, P, blk, lib):
        b.set("freq", P[0])
        b.set("env_attack", [lib.mxo_env_attack_coeff(x, 44100) for x in P[1]])
        b.set("env_decay", [lib.mxo_env_decay_coeff(x, 44100) for x in P[2]])
        b.set("env_sustain", 0.6); b.set("env_release", [lib.mxo_env_decay_coeff(x, 44100) for x in P[3]]); b.set("env_holdtime", P[4])
        b.set("cutoff", P[5]); b.set("resonance", P[6]); b.set("delay_size", P[7]); b.set("delay_feedback", P[8]); b.set("pan", P[9])
    c.append(_bank("sine_adsr_lores_dl_44k", "src/maximilian.cpp:1479 setAttack, :1492 setSustain, src/maximilian.h:915 holdtime; "
                   "src/maximilian.cpp:420 dl(input, size, feedback); maxiSettings::setup(44100, ...)",
                   [U(30.0, 2000.0), U(1.0, 30.0), U(10.0, 100.0), U(20.0, 200.0), CHOICE(1.0, 2.0, 50.0, 500.0), U(200.0, 5000.0),
                    U(1.0, 6.0), U(1.0, 129.0, True), U(0.1, 0.9), U(0.0, 1.0)],
                   dict(osc="sinewave", filt="lores", env="adsr", delay="dl", delay_capacity=128, sample_rate=44100), sine_44k,
                   cap=128, sr=44100, gates=note_gates))

    def block_params(b, P, blk, lib):
        b.set("freq", P[0]); b.set("cutoff", P[1]); b.set("resonance", P[2]); b.set("pan", P[3])
    c.append(_bank("block_params", "src/maximilian.cpp:455 lores(input, cutoff1, resonance): arguments of every call",
                   [U(30.0, 2000.0, change=True), U(200.0, 5000.0, change=True), U(1.0, 6.0), U(0.0, 1.0, change=True)],
                   dict(osc="saw", filt="lores"), block_params))

    def gate_edges(b, P, blk, lib):
        b.set("freq", P[0]); b.set("env_attack", P[1]); b.set("env_decay", P[2]); b.set("env_sustain", P[3]); b.set("env_release", P[4])
        b.set("env_holdtime", 2.0)
    c.append(_bank("gate_edges", "src/maximilian.cpp:1362 adsr(..., holdtime, trigger): trigger == 1 on on <= t < off",
                   [U(30.0, 2000.0), U(0.01, 0.3), U(0.9, 0.999), U(0.2, 0.8), U(0.9, 0.999)],
                   dict(osc="saw", env="adsr"), gate_edges, gates=edge_gates, mix=False))
    return c


def error_cases():
    return [Case("const_change", "error", "src/maximilian.h:191 saw(frequency): a scalar is compiled into the patch", [], mix=False,
                 code=ERR_UNSUPPORTED, block=1),
            Case("biquad_unset", "error", "src/maximilian.h:1482 a0 = a1 = a2 = b1 = b2 = 0 until set()", [U(30.0, 2000.0)], mix=False,
                 code=ERR_UNSUPPORTED, block=0)]


# ------------------------------------------------------------------------------------------------ patch-shaped

def _patch(name, ref, params, build, exact, **kw):
    """build() -> (PatchDef, {parameter name: P index}, {input name: stream index}); phase(blk) -> [(stage, P index)] reset before blk"""
    return Case(name, "patch", ref, params, build=build, exact=exact, **kw)


def patch_cases():
    c = []

    def table_oscs():
        d = PatchDef()
        d.stage("osc", d.P("f0"), kind="sinebuf", dst=R(0))
        d.stage("osc", d.P("f1"), kind="sinebuf4", dst=R(1))
        d.stage("osc", d.P("f2"), kind="sawn", dst=R(2))
        d.stage("add", R(0), R(1), dst=R(3))
        d.stage("add", R(3), R(2), dst=R(4))
        d.stage("out", R(4))
        return d, dict(f0=0, f1=1, f2=2), {}
    c.append(_patch("table_oscs", "src/maximilian.h:206 sinebuf, :210 sinebuf4, :212 sawn (frequency)",
                    [U(20.0, 3000.0), U(20.0, 3000.0), U(20.0, 3000.0)], table_oscs, True))

    def filters():
        d = PatchDef()
        d.stage("osc", d.P("f"), kind="saw", dst=R(0))
        d.stage("filter", R(0), d.P("c1"), kind="lopass", dst=R(1))
        d.stage("filter", R(0), d.P("c2"), kind="hipass", dst=R(2))
        d.stage("filter", R(0), d.P("c3"), d.P("q3"), kind="bandpass", dst=R(3))
        d.stage("filter", R(0), d.P("c4"), d.P("q4"), kind="hires", dst=R(4))
        d.stage("add", R(1), R(2), dst=R(5))
        d.stage("add", R(5), R(3), dst=R(6))
        d.stage("add", R(6), R(4), dst=R(7))
        d.stage("mul", R(7), d.P("g"), dst=R(8))
        d.stage("out", R(8))
        return d, dict(f=0, c1=1, c2=2, c3=3, q3=4, c4=5, q4=6, g=7), {}
    c.append(_patch("maxifilter_patch", "src/maximilian.h:331 lopass(input, cutoff), :337 hipass(input, cutoff), "
                    ":325 bandpass(input, cutoff1, resonance), :318 hires(input, cutoff1, resonance)",
                    [U(30.0, 2000.0), U(0.05, 0.5), U(0.05, 0.5), U(200.0, 5000.0), U(0.05, 0.4), U(200.0, 5000.0), U(1.0, 6.0), U(0.5, 2.0)],
                    filters, False))

    def nonlin():
        d = PatchDef()
        d.stage("osc", d.P("f"), kind="saw", dst=R(0))
        d.stage("mul", R(0), d.K(1.5), dst=R(1))
        d.stage("nonlin", R(1), d.P("shape"), kind="atandist", dst=R(2))
        d.stage("nonlin", R(1), d.P("fshape"), kind="fastatandist", dst=R(3))
        d.stage("nonlin", R(1), kind="softclip", dst=R(4))
        d.stage("nonlin", R(1), kind="hardclip", dst=R(5))
        d.stage("nonlin", R(1), d.P("a"), d.P("b"), kind="asymclip", dst=R(6))
        d.stage("nonlin", R(1), kind="fastatan", dst=R(7))
        r = 2
        for k, x in enumerate((3, 4, 5, 6, 7)):
            d.stage("add", R(r), R(x), dst=R(8 + k))
            r = 8 + k
        d.stage("out", R(r))
        return d, dict(f=0, shape=1, fshape=2, a=3, b=4), {}
    c.append(_patch("nonlinearities", "src/maximilian.h:1054 atanDist(in, shape), :1059 fastAtanDist(in, shape), :1061 softclip(x), "
                    ":1063 hardclip(x), :1071 asymclip(x, a, b), :1073 fastatan(x)",
                    [U(30.0, 2000.0), U(0.5, 8.0), U(0.5, 8.0), U(0.5, 1.0), U(2.0, 4.0)], nonlin, False))

    def fx():
        d = PatchDef()
        d.stage("osc", d.P("f"), kind="saw", dst=R(0))
        d.stage("add", R(0), d.K(0.25), dst=R(1))
        d.stage("dcblock", R(1), d.P("R"), dst=R(2))
        d.stage("flanger", R(0), d.P("fdel"), d.P("ffb"), d.P("fspeed"), d.P("fdepth"), dst=R(3))
        d.stage("chorus", R(0), d.K(120.0), d.P("cfb"), d.P("cspeed"), d.P("cdepth"), d.IN("noise"), dst=R(4))
        d.stage("add", R(2), R(3), dst=R(5))
        d.stage("add", R(5), R(4), dst=R(6))
        d.stage("out", R(6))
        return d, dict(f=0, R=1, fdel=2, ffb=3, fspeed=4, fdepth=5, cfb=6, cspeed=7, cdepth=8), dict(noise=0)

    def noise(name, k, V, B, blk):
        from oracle import oracle_py
        return oracle_py.noise_fill(7, (blk + 1) * B * V, "port")[blk * B * V:].reshape(B, V)
    c.append(_patch("dcblock_flanger_chorus", "src/maximilian.h:1261 maxiDCBlocker::play(input, R), "
                    ":1161 flange(input, delay, feedback, speed, depth), :1195 chorus(input, delay, feedback, speed, depth)",
                    [U(30.0, 2000.0), U(0.9, 0.999), U(1.0, 100.0, True), U(0.0, 0.9), U(0.1, 20.0), U(0.0, 1.0),
                     U(0.0, 0.9), U(0.1, 10.0), U(0.2, 0.8)], fx, False, cap=512, streams=[noise]))

    def envs():
        d = PatchDef()
        d.stage("osc", d.P("f"), kind="triangle", dst=R(0))
        d.stage("env_adsr", R(0), d.IN("t0"), d.P("att"), d.P("dec"), d.P("sus"), d.P("rel"), d.P("hold"), dst=R(1))
        d.stage("env_ar", R(0), d.IN("t1"), d.P("aatt"), d.P("arel"), d.P("ahold"), dst=R(2))
        d.stage("osc", d.P("tf"), kind="square", dst=R(3))
        d.stage("env_adsr", R(0), R(3), d.K(0.0), d.K(0.0), d.K(0.0), d.K(0.0), d.P("hold3"), dst=R(4))   # coefficients: see below
        d.stage("add", R(1), R(2), dst=R(5))
        d.stage("add", R(5), R(4), dst=R(6))
        d.stage("out", R(6))
        return d, dict(f=0, att=1, dec=2, sus=3, rel=4, hold=5, aatt=6, arel=7, ahold=8, tf=9, hold3=10), dict(t0=0, t1=1)

    def envs_fix(d, lib):
        """the third envelope's coefficients: setAttackMS(2), setDecay(20), setSustain(0.5), setRelease(30) at 48 kHz"""
        op, k, dst, src = d.stages[4]
        src = list(src)
        src[2:6] = [d.K(lib.mxo_env_attack_ms_coeff(2.0, 48000)), d.K(lib.mxo_env_decay_coeff(20.0, 48000)), d.K(0.5),
                    d.K(lib.mxo_env_decay_coeff(30.0, 48000))]
        d.stages[4] = (op, k, dst, src)
    c.append(_patch("env_triggers", "src/maximilian.cpp:1362 adsr(input, attack, decay, sustain, release, holdtime, trigger), "
                    ":1319 ar(input, attack, release, holdtime, trigger), :1415 adsr(input, trigger) with :1485 setAttackMS, :1474 setDecay, "
                    ":1492 setSustain, :1469 setRelease",
                    [U(30.0, 500.0), U(0.01, 0.3), U(0.9, 0.999), U(0.2, 0.8), U(0.9, 0.999), CHOICE(0.0, 1.0, 7.0),
                     U(0.01, 0.3), U(0.9, 0.999), CHOICE(0.0, 1.0, 7.0), U(50.0, 400.0), CHOICE(1.0, 3.0, 30.0)],
                    envs, True, fix=envs_fix,
                    streams=[lambda n, k, V, B, blk: trigger_stream(n, "t0", V, B, blk), lambda n, k, V, B, blk: trigger_stream(n, "t1", V, B, blk)]))

    def modf():
        d = PatchDef()
        d.stage("osc", d.P("f"), kind="saw", dst=R(0))
        d.stage("osc", d.K(3.0), kind="sinewave", dst=R(1))
        d.stage("mul", R(1), d.K(600.0), dst=R(2))
        d.stage("add", R(2), d.K(1500.0), dst=R(3))
        d.stage("svf", R(0), R(3), d.P("res"), d.K(0.5), d.K(0.25), d.K(0.125), d.K(0.0625), dst=R(4))
        d.stage("biquad", R(0), d.K(2000.0), d.P("q"), d.K(0.0), kind="bandpass", dst=R(5))
        d.stage("add", R(4), R(5), dst=R(6))
        d.stage("out", R(6))
        return d, dict(f=0, res=1, q=2), {}
    c.append(_patch("modulated_filters", "src/maximilian.h:1287 setCutoff(cutoff) on every sample, :1293 setResonance(q), "
                    ":1375 maxiBiquad::set(filtType, cutoff, Q, peakGain)", [U(30.0, 2000.0), U(0.5, 5.0), U(0.5, 4.0)], modf, False))

    def envgen():
        d = PatchDef()
        k0 = d.envgen([0.0, 1.0, 0.3, 0.0], [1.5, 2.0, 1.0], [2.0, 1.0, 0.5], loop=False, retrigger=True)    # setup(.., false); setRetrigger(true)
        d.stage("envgen", d.P("trig"), kind=k0, dst=R(0))
        d.stage("osc", d.P("tf"), kind="square", dst=R(1))
        k1 = d.envgen([0.0, 1.0, 0.5, 0.5, 0.0], [1.0, 1.0, ENVGEN_HOLD, 2.0], [1.0, 1.0, 1.0, 1.0])     # setupADSR(1, 1, 0.5, 2)
        d.stage("envgen", R(1), kind=k1, dst=R(2))
        k2 = d.envgen([0.0, 1.0, 0.0], [2.0, 3.0], [1.0, 1.0], loop=True)                                  # setupAR(2, 3); setLoop(true)
        d.stage("envgen", d.P("trig"), kind=k2, dst=R(3))
        k3 = d.envgen([0.0, 1.0, 1.0, 0.0], [0.5, ENVGEN_HOLD, 1.0], [1.0, 1.0, 1.0])                       # setupASR(0.5, 1)
        d.stage("envgen", R(1), kind=k3, dst=R(4))
        d.stage("add", R(0), R(2), dst=R(5))
        d.stage("add", R(5), R(3), dst=R(6))
        d.stage("add", R(6), R(4), dst=R(7))
        d.stage("out", R(7))
        return d, dict(trig=0, tf=1), {}
    c.append(_patch("envgen_triggers", "src/maximilian.h:2276 maxiEnvGen::play(trigger), :2371 setup(levels, times, curves, looping, allowRetrigger), "
                    "setupAR / setupASR / setupADSR, setLoop, setRetrigger", [BLOCKS((1.0, 0.0), (0.0, 1.0), (1.0,)), U(100.0, 900.0)],
                    envgen, False))

    def arith():
        d = PatchDef()
        d.stage("osc", d.P("f"), kind="saw", dst=R(0))
        d.stage("sub", d.K(1.0), R(0), dst=R(1))          # 1.0 - w
        d.stage("sub", R(0), d.P("p"), dst=R(2))          # w - p
        d.stage("div", d.P("p"), R(0), dst=R(3))          # p / w
        d.stage("div", R(0), d.P("p"), dst=R(4))          # w / p
        d.stage("mul", R(0), R(0), dst=R(5))              # w * w
        d.stage("mul", R(1), d.K(3.0), dst=R(6))
        d.stage("add", R(6), R(2), dst=R(7))
        d.stage("mul", R(7), d.K(5.0), dst=R(8))
        d.stage("add", R(8), R(3), dst=R(9))
        d.stage("mul", R(9), d.K(7.0), dst=R(10))
        d.stage("add", R(10), R(4), dst=R(11))
        d.stage("mul", R(11), d.K(11.0), dst=R(12))
        d.stage("add", R(12), R(5), dst=R(13))
        d.stage("out", R(13))
        return d, dict(f=0, p=1), {}
    c.append(_patch("operand_order", "src/maximilian.h:191 saw(frequency); the arithmetic of a play() between the calls",
                    [U(30.0, 2000.0), U(0.5, 3.0)], arith, True))

    def stereo_sum():
        d = PatchDef()
        d.stage("osc", d.P("f0"), kind="saw", dst=R(0))
        d.stage("osc", d.P("f1"), kind="triangle", dst=R(1))
        d.stage("mix_stereo", R(0), d.P("pan"))
        d.stage("mix_stereo", R(1), d.K(0.0))
        d.stage("out", R(1))
        return d, dict(f0=0, f1=1, pan=2), {}
    c.append(_patch("stereo_and_sum", "src/maximilian.cpp:503 stereo(input, two, x); maxiVoices::sum is stereo at x = 0",
                    [U(30.0, 2000.0), U(30.0, 2000.0), U(0.0, 1.0)], stereo_sum, True))

    def resets():
        d = PatchDef()
        d.stage("osc", d.P("f0"), kind="phasor", dst=R(0))
        d.stage("osc", d.P("f1"), kind="saw", dst=R(1))
        d.stage("add", R(0), R(1), dst=R(2))
        d.stage("out", R(2))
        return d, dict(f0=0, f1=1), {}
    c.append(_patch("two_phase_resets", "src/maximilian.cpp:222 phaseReset(phaseIn), per oscillator object",
                    [U(30.0, 2000.0), U(30.0, 2000.0), U(0.0, 1.0), U(0.0, 1.0)], resets, True,
                    phase=lambda blk: [(0, 2)] if blk != 1 else [(1, 3)]))
    return c


def cases():
    return bank_cases() + error_cases() + patch_cases()
