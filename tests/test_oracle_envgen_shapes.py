"""Several maxiEnvGen shapes in one voice patch, on the CPU. The C port (oracle/maxi_oracle.c) runs the patches of tests/envgen_cases.py
and must give, bit for bit, what the reference's own maxiEnvGen objects gave on the same inputs: outputs, buses and every state word of
every envelope stage (tests/golden/envgen_shapes.npz, made by tests/golden/make_envgen_golden.py)."""
import numpy as np
import pytest

import golden_checks as G
import envgen_cases as EC
from patch_checks import bad_kind_patch
from maximilian_b200.patchdef import OP


@pytest.mark.parametrize("case", EC.cases(), ids=lambda c: c[0])
def test_envgen_shapes_port_equals_reference_golden(port, case):
    name, d, params, inputs = case
    g = G.load("envgen_shapes")
    V, B, NB = int(g["V"]), int(g["B"]), int(g["NB"])
    p = port.Patch(d, V, kind="port")
    eg = [si for si, st in enumerate(d.stages) if st[0] == OP["envgen"]]
    for k in params(V, 3):
        p.set(k, g[f"{name}/param/{k}"])
    ins = {k: g[f"{name}/in/{k}"] for k in d.inputs}
    for blk in range(NB):
        o, m = p.process(B, {k: a[blk * B:(blk + 1) * B] for k, a in ins.items()}, want_mix=True)
        assert np.array_equal(o, g[name + "/out"][blk]) and np.array_equal(m, g[name + "/mix"][blk]), (name, blk)
        assert np.abs(o).max() > 1e-3
    states = {}
    for si in eg:
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


@pytest.mark.parametrize("kind", [-1, 1, 4])
def test_port_refuses_an_envgen_kind_outside_the_shapes(port, kind):
    """An ENVGEN stage plays shapes[kind]: with one shape only kind 0 is accepted, as mxb_patch_create accepts it."""
    port.Patch(bad_kind_patch("envgen", 0), 4, kind="port")
    with pytest.raises(RuntimeError, match="mxo_patch_create"):
        port.Patch(bad_kind_patch("envgen", kind), 4, kind="port")
