"""Voice patches with several maxiEnvGen shapes (mxb_patch_create2), shared by the oracle, GPU and C++ tests.

Each case is (name, PatchDef, parameter dict builder, input builder). The triggers are per-sample gates that swing -1 / +1 (maxiEnvGen
watches zero crossings: the positive one starts the envelope, the negative one ends a HOLD segment), short enough that many gates open
and close again inside a segment, which retriggers a shape that allows it."""
import numpy as np

from maximilian_b200.patchdef import PatchDef, R, ENVGEN_HOLD, OP, STATE_SLOTS
from maximilian_b200 import workloads as W

SLOTS = STATE_SLOTS[OP["envgen"]]      # state words of an ENVGEN stage


def swing(V, n, seed, density=0.02, hold=(3, 120)):
    """[n][V] of -1 / +1: gates that open and close at any sample, several times per block for most voices"""
    rng = np.random.default_rng(seed)
    t = -np.ones((n, V))
    for v in range(V):
        pos = int(rng.integers(0, 40))
        while pos < n:
            ln = int(rng.integers(hold[0], hold[1]))
            t[pos:pos + ln, v] = 1.0
            pos += ln + int(rng.geometric(density))
    return t


def four_shapes():
    """A linear AR, an ADSR with a HOLD segment and curve 2, a looping shape that retriggers, and a shape of no segments (a maxiEnvGen
    whose setup() was never called), each on its own stage, summed with an oscillator into the output and the bus."""
    d = PatchDef()
    ar = d.envgen([0.0, 1.0, 0.0], [1.5, 2.5], [1.0, 1.0])
    adsr = d.envgen([0.0, 1.0, 0.4, 0.4, 0.0], [1.0, 0.8, ENVGEN_HOLD, 1.2], [2.0, 2.0, 1.0, 2.0])
    loop = d.envgen([0.1, 1.0, 0.3], [0.7, 0.9], [0.5, 3.0], loop=True, retrigger=True)
    empty = d.envgen([0.0], [], [])
    d.stage("envgen", d.IN("gate"), kind=ar, dst=R(0))
    d.stage("envgen", d.IN("gate"), kind=adsr, dst=R(1))
    d.stage("envgen", d.IN("gate2"), kind=loop, dst=R(2))
    d.stage("envgen", d.IN("gate2"), kind=empty, dst=R(3))
    d.stage("osc", d.P("freq"), kind="saw", dst=R(4))
    d.stage("mul", R(4), R(0), dst=R(5))
    d.stage("add", R(1), R(2), dst=R(6))
    d.stage("mul", R(5), R(6), dst=R(6))
    d.stage("add", R(6), R(3), dst=R(6))
    d.stage("out", R(6))
    d.stage("mix_stereo", R(6), d.P("pan"))

    def params(V, seed):
        p = W.voice_params(V, seed=seed)
        return dict(freq=p["freq"], pan=p["pan"])

    def inputs(V, n, seed):
        return dict(gate=swing(V, n, seed), gate2=swing(V, n, seed + 1, density=0.05, hold=(2, 60)))
    return ("four_shapes", d, params, inputs)


def shared_shape():
    """Two stages play one shape (each with its own state: different triggers), a third stage plays a second shape."""
    d = PatchDef()
    a = d.envgen([0.0, 1.0, 0.5, 0.0], [1.0, ENVGEN_HOLD, 1.5], [2.0, 1.0, 0.5], retrigger=True)
    b = d.envgen([1.0, 0.0], [2.0], [1.0], loop=True)
    d.stage("envgen", d.IN("gate"), kind=a, dst=R(0))
    d.stage("envgen", d.IN("gate2"), kind=a, dst=R(1))
    d.stage("envgen", d.IN("gate"), kind=b, dst=R(2))
    d.stage("sub", R(0), R(1), dst=R(3))
    d.stage("add", R(3), R(2), dst=R(3))
    d.stage("out", R(3))
    d.stage("mix_stereo", R(3), d.P("pan"))

    def params(V, seed):
        return dict(pan=W.voice_params(V, seed=seed)["pan"])

    def inputs(V, n, seed):
        return dict(gate=swing(V, n, seed), gate2=swing(V, n, seed + 7, density=0.04, hold=(5, 90)))
    return ("shared_shape", d, params, inputs)


def cases():
    return [four_shapes(), shared_shape()]


def envelopes2(sample_rate=44100):
    """cpp/commandline/maximilian_examples/9.Envelopes2 as tests/cpp/patch_envelopes.cpp records it through the C++ layer (maxiPolyBLEP ->
    maxiOsc::square / triangle): three maxiEnvGen shapes, the second widening the pulse that triggers the first, the third sweeping the
    biquad cutoff."""
    d = PatchDef()
    s1 = d.envgen([0.0, 1.0, 1.0, 0.1], [200.0, ENVGEN_HOLD, 200.0], [1.0, 1.0, 1.0])          # myEnv
    s2 = d.envgen([0.0, 1.0], [10000.0], [1.0])                                              # myEnv2
    s3 = d.envgen([2000.0, 100.0], [10000.0], [0.5])                                         # myEnv3
    d.stage("envgen", d.K(1.0), kind=s2, dst=R(0))                                           # myEnv2.play(1)
    d.stage("osc", d.K(1.0), R(0), kind="pulse", dst=R(1))                                   # trig.pulse(1, ...)
    d.stage("envgen", R(1), kind=s1, dst=R(2))                                               # env = myEnv.play(...)
    d.stage("envgen", d.K(1.0), kind=s3, dst=R(3))                                           # myEnv3.play(1)
    d.stage("mul", R(2), d.K(500.0), dst=R(4))
    d.stage("add", d.K(20.0), R(4), dst=R(4))                                                # frequency = 20 + (env*500)
    d.stage("osc", R(4), kind="square", dst=R(5))
    d.stage("add", R(4), d.K(25.0), dst=R(6))
    d.stage("mul", R(6), d.K(2.0), dst=R(6))
    d.stage("osc", R(6), kind="triangle", dst=R(6))
    d.stage("add", R(5), R(6), dst=R(7))
    d.stage("biquad", R(7), R(3), d.K(2.0), d.K(3.0), kind="lowpass", dst=R(8))             # filter.set(LOWPASS, env3, 2, 3); filter.play(...)
    d.stage("out", R(8))
    return d
