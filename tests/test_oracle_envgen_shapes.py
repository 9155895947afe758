"""Several maxiEnvGen shapes in one voice patch, on the CPU. The C port (oracle/maxi_oracle.c) runs the patches of tests/envgen_cases.py
through tests/envgen_oracle.py and must give, bit for bit, what the reference's own maxiEnvGen objects gave on the same inputs: outputs,
buses and every state word of every envelope stage (tests/golden/envgen_shapes.npz, made by tests/golden/make_envgen_golden.py). The
lock-step composition itself is checked against the port running a one-shape patch directly."""
import numpy as np
import pytest

import golden_checks as G
import envgen_cases as EC
import envgen_oracle as EO
import patch_cases as PC
from maximilian_b200.patchdef import STATE_SLOTS


@pytest.mark.parametrize("case", EC.cases(), ids=lambda c: c[0])
def test_envgen_shapes_port_equals_reference_golden(port, case):
    name, d, params, inputs = case
    g = G.load("envgen_shapes")
    V, B, NB = int(g["V"]), int(g["B"]), int(g["NB"])
    p = EO.ShapesPatch(port, d, V, kind="port")
    for k in params(V, 3):
        p.set(k, g[f"{name}/param/{k}"])
    ins = {k: g[f"{name}/in/{k}"] for k in d.inputs}
    for blk in range(NB):
        o, m = p.process(B, {k: a[blk * B:(blk + 1) * B] for k, a in ins.items()}, want_mix=True)
        assert np.array_equal(o, g[name + "/out"][blk]) and np.array_equal(m, g[name + "/mix"][blk]), (name, blk)
        assert np.abs(o).max() > 1e-3
    states = {}
    for si in p.eg:
        s = np.stack([p.get_state(si, sl) for sl in range(EC.SLOTS)])
        # nxcHappened is indeterminate in the reference until the first trigger, and a shape of no segments is never triggered
        check = [sl for sl in range(EC.SLOTS) if not (sl == 3 and len(d.shapes[d.stages[si][1]][1]) == 0)]
        assert np.array_equal(s[check], g[f"{name}/state/{si}"][check]), (name, si)
        states[si] = s
    assert max(s[1].max() for s in states.values()) >= 1                              # segments were played through
    if name == "four_shapes":
        assert np.all(states[3][0] == 0.0) and np.all(states[3][2] == 0.0)            # the shape of no segments never triggers, plays 0
        assert np.any(states[1][2] == 2.0) or np.any(states[1][1] >= 2)                # the ADSR reached its HOLD
    else:
        assert not np.array_equal(states[0][0], states[1][0])                         # one shape, two stages, two states


def test_lock_step_composition_equals_the_direct_run(port):
    """A one-shape patch (maxiEnvGen with HOLD and retrigger, flanger, delay lines) through tests/envgen_oracle.py and through the port
    directly: the same outputs, bus and state of every stage, bit for bit."""
    name, d, params, inputs, exact, taps = PC.envgen_flanger()
    V, B = 10, 256
    a = EO.ShapesPatch(port, d, V, delay_taps=taps, kind="port")
    b = port.Patch(d, V, delay_taps=taps, kind="port")
    for k, v in params(V, 4).items():
        a.set(k, v); b.set(k, v)
    for blk in range(3):
        x = inputs(V, B, blk, 9)
        oa, ma = a.process(B, x, want_mix=True); ob, mb = b.process(B, x, want_mix=True)
        assert np.array_equal(oa, ob) and np.array_equal(ma, mb), blk
    for si, st in enumerate(d.stages):
        for sl in range(STATE_SLOTS.get(st[0], 0)):
            assert np.array_equal(a.get_state(si, sl), b.get_state(si, sl)), (si, sl)
