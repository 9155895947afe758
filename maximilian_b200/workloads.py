"""Synthetic voice banks and channel streams (host side, numpy only).

The recipe is SURVEY.md section 8(d): every per-voice parameter is drawn ONCE on the host
from numpy's PCG64 (seed 20260922) as fp64 and handed identically to whatever consumes it
(the GPU bank, the CPU oracle, the reference baseline) -- parameters are never regenerated
on the device. Sample rate 48 kHz throughout.
"""
import math

import numpy as np

SEED = 20260922
SAMPLE_RATE = 48000


def voice_params(voices, seed=SEED, delay_size=4096, ragged_delay=False):
    """Dict of fp64 arrays [voices] (delay_size / env_holdtime hold integral values)."""
    rng = np.random.default_rng(seed)
    u = rng.random
    p = {}
    p["freq"] = 27.5 * np.exp2(7.25 * u(voices))            # 27.5 .. 4186 Hz
    p["phase"] = u(voices)                                  # maxiOsc::phaseReset(u)
    p["duty"] = 0.1 + 0.8 * u(voices)
    p["cutoff"] = 100.0 * np.power(80.0, u(voices))         # 100 .. 8000 Hz
    p["q_lores"] = 1.0 + 7.0 * u(voices)                    # lores/hires resonance
    p["res_svf"] = 0.5 + 4.5 * u(voices)                    # maxiSVF resonance
    p["q_biquad"] = 0.5 + 3.5 * u(voices)                   # maxiBiquad Q
    p["gain"] = np.zeros(voices)
    p["pan"] = u(voices)
    p["attack_ms"] = 1.0 + 49.0 * u(voices)
    p["decay_ms"] = 10.0 + 190.0 * u(voices)
    p["env_sustain"] = 0.2 + 0.7 * u(voices)
    p["release_ms"] = 50.0 + 450.0 * u(voices)
    p["env_holdtime"] = np.ones(voices)
    if ragged_delay:
        p["delay_size"] = rng.integers(max(1, delay_size // 4), delay_size + 1, voices).astype(np.float64)
    else:
        p["delay_size"] = np.full(voices, float(delay_size))
    p["delay_feedback"] = 0.1 + 0.8 * u(voices)
    # maxiOsc::phasorBetween(f, startphase, endphase): derived from draws above, so that the seeded sequences (and the
    # golden fixtures generated from them) stay what they were
    p["phasor_start"] = 0.4 * p["duty"]
    p["phasor_end"] = 0.5 + 0.5 * p["pan"]
    return p


def env_coeffs(p, sample_rate=SAMPLE_RATE):
    """maxiEnv::setAttack / setDecay / setRelease (src/maximilian.cpp:1469-1480) through libm pow
    (math.pow is the C library's pow, the function the reference calls)."""
    sr = float(sample_rate)
    att = np.array([1 - math.pow(0.01, 1.0 / (ms * sr * 0.001)) for ms in p["attack_ms"]])
    dec = np.array([math.pow(0.01, 1.0 / (ms * sr * 0.001)) for ms in p["decay_ms"]])
    rel = np.array([math.pow(0.01, 1.0 / (ms * sr * 0.001)) for ms in p["release_ms"]])
    return att, dec, rel


def gate(voices, block, block_index, seed=SEED):
    """Per-voice note gate of one block: trigger == 1 for trig_on <= t < trig_off.
    Every 4th block carries a note (t_on in [0, B/4], t_off in [B/2, 3B/4]); the others none."""
    if block_index % 4 != 0:
        z = np.zeros(voices, dtype=np.int32)
        return z, z.copy()
    rng = np.random.default_rng(seed + 7919 * (block_index + 1))
    on = rng.integers(0, block // 4 + 1, voices).astype(np.int32)
    off = rng.integers(block // 2, 3 * block // 4 + 1, voices).astype(np.int32)
    return on, off


def channel_streams(channels, n, seed=SEED, sample_rate=SAMPLE_RATE):
    """float32 [channels][n]: 0.5*saw(f_c) + 0.25*sin(2*pi*3.1*f_c*t) + 0.05*N(0,1)."""
    rng = np.random.default_rng(seed + 1)
    f = 27.5 * np.exp2(7.25 * rng.random(channels))
    t = np.arange(n, dtype=np.float64)[None, :] / sample_rate
    ph = (f[:, None] * t) % 1.0
    x = 0.5 * (2.0 * ph - 1.0) + 0.25 * np.sin(2 * np.pi * 3.1 * f[:, None] * t)
    x += 0.05 * rng.standard_normal((channels, n))
    return x.astype(np.float32)


def configure_bank(bank, filt, p, env=False, delay=False, sample_rate=SAMPLE_RATE):
    """Hand one parameter set to anything with a .set(name, values) method
    (the GPU bank and both CPU oracles share the parameter names)."""
    bank.set("freq", p["freq"]); bank.set("phase", p["phase"]); bank.set("duty", p["duty"])
    if "phasor_start" in p:
        bank.set("phasor_start", p["phasor_start"]); bank.set("phasor_end", p["phasor_end"])
    if filt in ("lores", "hires"):
        bank.set("cutoff", p["cutoff"]); bank.set("resonance", p["q_lores"])
    elif filt == "svf":
        bank.set("cutoff", p["cutoff"]); bank.set("resonance", p["res_svf"])
    elif filt == "biquad":
        bank.set("gain", p["gain"]); bank.set("cutoff", p["cutoff"]); bank.set("resonance", p["q_biquad"])
    if env:
        att, dec, rel = env_coeffs(p, sample_rate)
        bank.set("env_attack", att); bank.set("env_decay", dec); bank.set("env_release", rel)
        bank.set("env_sustain", p["env_sustain"]); bank.set("env_holdtime", p["env_holdtime"])
    if delay:
        bank.set("delay_size", p["delay_size"]); bank.set("delay_feedback", p["delay_feedback"])
    bank.set("pan", p["pan"])


def polysynth_patch(trigger_dtype="f64"):
    """One voice of cpp/commandline/maximilian_examples/15.polysynth/main.cpp:54-70 as a PatchDef: two pulse VCOs (the second
    detuned by a sinebuf LFO) summed into a lores VCF whose cutoff follows pitch + LFO, multiplied by the ADSR AFTER the filter.
    trigger_dtype "u8" / "bits": the per-sample trigger stream arrives as bytes / as one bit per voice-sample (maxiEnv::trigger is an
    int that a patch sets to 0 or 1)."""
    from .patchdef import PatchDef, R
    d = PatchDef()
    one = d.K(1.0)
    d.stage("env_adsr", one, d.IN("trigger", trigger_dtype), d.P("attack"), d.P("decay"), d.P("sustain"), d.P("release"), d.K(1.0), dst=R(0))   # ADSRout
    d.stage("osc", d.K(0.2), kind="sinebuf", dst=R(1))                                   # LFO1out
    d.stage("osc", d.P("f1"), d.K(0.6), kind="pulse", dst=R(2))                          # VCO1out = pulse(55*pitch, 0.6)
    d.stage("add", d.P("f2"), R(1), dst=R(3))                                             # (110*pitch) + LFO1out
    d.stage("osc", R(3), d.K(0.2), kind="pulse", dst=R(3))                               # VCO2out
    d.stage("add", R(2), R(3), dst=R(4))
    d.stage("mul", R(4), d.K(0.5), dst=R(4))                                              # (VCO1out + VCO2out) * 0.5
    d.stage("add", d.P("pitch"), R(1), dst=R(5))
    d.stage("mul", R(5), d.K(1000.0), dst=R(5))
    d.stage("add", d.K(250.0), R(5), dst=R(5))                                            # 250 + ((pitch + LFO1out) * 1000)
    d.stage("filter", R(4), R(5), d.K(10.0), kind="lores", dst=R(6))                     # VCFout
    d.stage("mul", R(6), R(0), dst=R(7))
    d.stage("div", R(7), d.K(6.0), dst=R(7))                                              # VCFout * ADSRout / 6
    d.stage("out", R(7))
    d.stage("mix_stereo", R(7), d.P("pan"))
    return d


def polysynth_pitch_patch(pitch_dtype="events", trigger_dtype="events"):
    """polysynth_patch with the voice's pitch as a stream too (f1 = 55 * pitch, f2 = 110 * pitch, the cutoff from pitch + LFO): the shape
    of a host-driven synth that plays a new note on any sample. "events" (MXB_IN_EVENTS) costs per change, "f64" per voice-sample."""
    from .patchdef import PatchDef, R
    d = PatchDef()
    one = d.K(1.0)
    pitch = d.IN("pitch", pitch_dtype)
    d.stage("env_adsr", one, d.IN("trigger", trigger_dtype), d.P("attack"), d.P("decay"), d.P("sustain"), d.P("release"), d.K(1.0), dst=R(0))
    d.stage("osc", d.K(0.2), kind="sinebuf", dst=R(1))
    d.stage("mul", d.K(55.0), pitch, dst=R(8))
    d.stage("osc", R(8), d.K(0.6), kind="pulse", dst=R(2))
    d.stage("mul", d.K(110.0), pitch, dst=R(9))
    d.stage("add", R(9), R(1), dst=R(3))
    d.stage("osc", R(3), d.K(0.2), kind="pulse", dst=R(3))
    d.stage("add", R(2), R(3), dst=R(4))
    d.stage("mul", R(4), d.K(0.5), dst=R(4))
    d.stage("add", pitch, R(1), dst=R(5))
    d.stage("mul", R(5), d.K(1000.0), dst=R(5))
    d.stage("add", d.K(250.0), R(5), dst=R(5))
    d.stage("filter", R(4), R(5), d.K(10.0), kind="lores", dst=R(6))
    d.stage("mul", R(6), R(0), dst=R(7))
    d.stage("div", R(7), d.K(6.0), dst=R(7))
    d.stage("out", R(7))
    d.stage("mix_stereo", R(7), d.P("pan"))
    return d


def note_events(voices, block, block_index, seed=SEED):
    """about one note per voice per block: a new pitch (1 .. 6) at a random frame t < block - 1, and a one-sample trigger (1 at t, 0 at
    t + 1). CSR triples (first, frame, value) of the pitch and of the trigger events."""
    rng = np.random.default_rng(seed + 505 + block_index)
    t = rng.integers(0, block - 1, voices).astype(np.int32)
    pitch = 1.0 + rng.integers(0, 6, voices).astype(np.float64)
    pe = (np.arange(voices + 1, dtype=np.int32), t, pitch)
    te = ((2 * np.arange(voices + 1)).astype(np.int32), np.stack([t, t + 1], axis=1).reshape(-1), np.tile([1.0, 0.0], voices))
    return pe, te


def polysynth_params(voices, seed=SEED):
    p = voice_params(voices, seed=seed)
    att, dec, rel = env_coeffs(p)
    pitch = 1.0 + (np.arange(voices) % 6)
    return dict(attack=att, decay=dec, sustain=p["env_sustain"], release=rel, f1=55.0 * pitch, f2=110.0 * pitch, pitch=pitch, pan=p["pan"])


def note_pattern(voices, seed=SEED):
    """(period, offset, length) per voice, samples: trigger(t, v) = ((t + offset_v) mod period_v) < length_v -- every voice plays
    notes of its own length at its own rate, several per 1024-frame block for the fast ones (10.Filters/main.cpp:27-36 writes
    maxiEnv::trigger on any sample)."""
    rng = np.random.default_rng(seed + 404)
    period = rng.integers(300, 4000, voices)
    offset = rng.integers(0, 4000, voices)
    length = (period * (0.1 + 0.6 * rng.random(voices))).astype(np.int64)
    return period.astype(np.int64), offset.astype(np.int64), length


def note_triggers(pattern, block, block_index, lo=0, hi=None, dtype=np.uint8):
    """trigger[block][hi - lo] of block `block_index` from note_pattern()"""
    period, offset, length = (a[lo:hi] for a in pattern)
    t = (np.arange(block, dtype=np.int64) + block * block_index)[:, None]
    return (((t + offset[None, :]) % period[None, :]) < length[None, :]).astype(dtype)
