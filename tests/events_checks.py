"""What the events-stream tests share: the meaning of an MXB_IN_EVENTS stream restated in numpy (the dense per-sample stream a list of
events stands for), random event lists with every corner the definition covers, and the patches the tests run both ways."""
import numpy as np

from maximilian_b200.patchdef import PatchDef, R


def events_to_dense(first, frame, value, n, held):
    """The [n][V] doubles an events stream reads, and the held values after the call (include/maxib200.h, mxb_events): event i of a
    voice takes effect at max(frame_i, the frame event i-1 took effect at), negative frames at 0; those at n or later are dropped; where
    several take effect on one frame the last wins; before a voice's first event the stream reads its held value."""
    first = np.asarray(first, dtype=np.int64); frame = np.asarray(frame, dtype=np.int64); value = np.asarray(value, dtype=np.float64)
    held = np.asarray(held, dtype=np.float64)
    V = first.size - 1
    cnt = np.maximum(np.diff(first), 0)                                  # first[v+1] <= first[v]: no events
    voice = np.repeat(np.arange(V, dtype=np.int64), cnt)
    start = np.repeat(first[:-1], cnt)
    idx = start + np.arange(voice.size) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    f = np.clip(frame[idx], 0, (1 << 31) - 1)
    eff = np.maximum.accumulate(voice * (1 << 32) + f) - voice * (1 << 32) if voice.size else f       # running max within each voice
    keep = eff < n
    voice, idx, eff = voice[keep], idx[keep], eff[keep]
    flat = eff * V + voice
    _, last = np.unique(flat[::-1], return_index=True)                   # the last event of each (frame, voice)
    last = flat.size - 1 - last
    mark = np.full(n * V, -1, dtype=np.int64)
    mark[flat[last]] = idx[last]
    mark = mark.reshape(n, V)
    at = np.maximum.accumulate(np.where(mark >= 0, np.arange(n)[:, None], -1), axis=0) if n else mark
    src = np.take_along_axis(mark, np.maximum(at, 0), axis=0)
    dense = np.where(at >= 0, value[np.maximum(src, 0)] if value.size else 0.0, held[None, :])
    return dense, (dense[-1].copy() if n else held.copy())


def random_events(rng, V, n, max_per_voice=4, lo=-3, hi_extra=3, values=None):
    """per-voice lists, unsorted, with repeated frames, negative frames, frames at and past n, and voices without events"""
    lists = []
    for v in range(V):
        k = int(rng.integers(0, max_per_voice + 1))
        fr = rng.integers(lo, n + hi_extra, k)
        if k >= 2 and rng.random() < 0.3:
            fr[1] = fr[0]                                                # several events on one frame
        if k and rng.random() < 0.2:
            fr[-1] = rng.choice([0, n - 1])
        val = values(rng, k) if values else rng.uniform(-1.0, 1.0, k)
        lists.append(list(zip(fr.tolist(), val.tolist())))
    return lists


# (name, builder(dtype) -> PatchDef reading one stream "x", params(V, rng), values(rng, k), delay_taps): one case per use of a control value
def _trigger_adsr(ty):
    d = PatchDef()
    d.stage("osc", d.P("f"), kind="saw", dst=R(0))
    d.stage("env_adsr", R(0), d.IN("x", ty), d.K(0.01), d.K(0.999), d.K(0.3), d.K(0.9995), d.K(1.0), dst=R(1))
    d.stage("out", R(1)); d.stage("mix_stereo", R(1), d.P("pan"))
    return d


def _trigger_envgen(ty):
    d = PatchDef()
    d.envgen([0.0, 1.0, 0.5, 0.0], [2.0, -46692.0, 3.0], [1.0, 2.0, 0.5], loop=False, retrigger=True)
    d.stage("envgen", d.IN("x", ty), kind=0, dst=R(0))
    d.stage("osc", d.P("f"), kind="triangle", dst=R(1))
    d.stage("mul", R(0), R(1), dst=R(2)); d.stage("out", R(2)); d.stage("mix_stereo", R(2), d.P("pan"))
    return d


def _frequency(ty):
    d = PatchDef()
    d.stage("osc", d.IN("x", ty), kind="saw", dst=R(0))
    d.stage("osc", d.IN("x", ty), d.K(0.3), kind="pulse", dst=R(1))
    d.stage("add", R(0), R(1), dst=R(2)); d.stage("out", R(2)); d.stage("mix_stereo", R(2), d.P("pan"))
    return d


def _cutoff(ty):
    d = PatchDef()
    d.stage("osc", d.P("f"), kind="saw", dst=R(0))
    d.stage("filter", R(0), d.IN("x", ty), d.K(3.0), kind="lores", dst=R(1))   # a per-sample design
    d.stage("svf", R(1), d.IN("x", ty), d.K(1.0), d.K(1.0), d.K(0.0), d.K(0.0), d.K(0.0), dst=R(2))
    d.stage("out", R(2)); d.stage("mix_stereo", R(2), d.P("pan"))
    return d


def _delay_size(ty):
    d = PatchDef()
    d.stage("osc", d.P("f"), kind="sinewave", dst=R(0))
    d.stage("delay", R(0), d.IN("x", ty), d.K(0.7), kind="dl", dst=R(1))
    d.stage("out", R(1)); d.stage("mix_stereo", R(1), d.P("pan"))
    return d


def _pan(ty):
    d = PatchDef()
    d.stage("osc", d.P("f"), kind="saw", dst=R(0))
    d.stage("out", R(0)); d.stage("mix_stereo", R(0), d.IN("x", ty))
    return d


def _f(rng, V):
    return dict(f=rng.uniform(40.0, 2000.0, V), pan=rng.uniform(0.0, 1.0, V))


CASES = [
    ("trigger_adsr", _trigger_adsr, lambda rng, k: rng.choice([0.0, 1.0], k), 0),
    ("trigger_envgen", _trigger_envgen, lambda rng, k: rng.choice([0.0, 1.0, -1.0], k), 0),
    ("frequency", _frequency, lambda rng, k: rng.uniform(20.0, 4000.0, k), 0),
    ("cutoff", _cutoff, lambda rng, k: rng.uniform(50.0, 9000.0, k), 0),
    ("delay_size", _delay_size, lambda rng, k: rng.integers(1, 64, k).astype(np.float64), 64),
    ("pan", _pan, lambda rng, k: rng.uniform(-0.2, 1.2, k), 0),
]


def budget_patch(flanger, ty):
    """doubles per voice: 16 registers + 32 parameters + 3 for each of 8 events streams + the stages' state: 61 oscillators (122), an
    AR envelope (4) and either one more oscillator (2: 200 in all) or a flanger (3: 201)"""
    d = PatchDef()
    for j in range(32):
        d.P(f"p{j}")
    for j in range(8):
        d.IN(f"e{j}", ty)
    for s in range(61):
        d.stage("osc", d.P(f"p{s % 32}") if s else d.IN("e0", ty), kind="sinewave", dst=R(s % 8))
    d.stage("env_ar", R(0), d.IN("e1", ty), d.K(0.01), d.K(0.999), d.K(1.0), dst=R(8))
    if flanger:
        d.stage("flanger", R(8), d.K(4.0), d.K(0.5), d.K(1.0), d.K(0.5), dst=R(9))
    else:
        d.stage("osc", d.IN("e7", ty), kind="saw", dst=R(9))
    d.stage("out", R(9))
    return d
