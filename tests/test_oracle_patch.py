"""Voice patches (include/maxib200.h mxb_patch; tests/patch_cases.py) on the CPU: the plain-C interpreter of oracle/maxi_oracle.c
against the same stage lists run by the reference's own objects (oracle/ref_shim.cpp) -- bit for bit, outputs, buses and the state
of every stage, as recorded from them (oracle/replay.py) -- and against the committed fixture tests/golden/patches.npz."""
import numpy as np
import pytest

import golden_checks as G
from oracle.replay import same
import patch_cases as PC
from patch_checks import set_tables
from maximilian_b200.patchdef import STATE_SLOTS as SLOTS


def test_tables_fixture_is_the_references(port, reference):
    g = G.load("tables")
    s, t, b = reference.get_tables("reference")
    assert same(s, g["sine"], equal_nan=False) and same(t, g["transition"], equal_nan=False) and b == float(g["sine_before"])
    assert s.size == 514 and t.size == 1001


@pytest.mark.parametrize("case", PC.cases(), ids=lambda c: c[0])
def test_patch_port_equals_reference(port, reference, case):
    name, d, params, inputs, exact, taps = case
    set_tables(port, library=False)
    V, B = 24, 200
    po = port.Patch(d, V, delay_taps=taps, kind="port"); pr = reference.Patch(d, V, delay_taps=taps, kind="reference")
    for k, v in params(V, 11).items():
        po.set(k, v); pr.set(k, v)
    for blk in range(3):
        ins = inputs(V, B, blk, 7)
        oo, mo = po.process(B, ins, want_mix=True); orr, mr = pr.process(B, ins, want_mix=True)
        assert same(oo, orr), (name, blk)
        assert same(mo, mr), (name, blk)
        assert np.isfinite(oo).all() and np.abs(oo).max() > 1e-3
    for si, (op, kind, dst, src) in enumerate(d.stages):
        for sl in range(SLOTS.get(op, 0)):
            if op == 5 and kind in (5, 6) and sl == 1:
                continue                                   # lopass / hipass keep one value (outputs[0])
            if op == 4 and sl == 3:
                continue                                   # nxcHappened is indeterminate in the reference until the first trigger
            assert same(po.get_state(si, sl), pr.get_state(si, sl), equal_nan=False), (name, si, sl)
        if op in (10, 11):
            for v in range(0, V, 5):
                assert same(po.ring(si, v, taps), pr.ring(si, v, taps), equal_nan=False), (name, si, v)


@pytest.mark.parametrize("case", PC.cases(), ids=lambda c: c[0])
def test_patch_golden_exact(port, case):
    """tests/golden/patches.npz (made by the compiled reference) replayed through the C port: exact, wherever gcc runs."""
    name, d, params, inputs, exact, taps = case
    set_tables(port, library=False)
    g = G.load("patches")
    V, B, NB = int(g["V"]), int(g["B"]), int(g["NB"])
    p = port.Patch(d, V, delay_taps=taps, kind="port")
    for k, v in params(V, 2468).items():
        p.set(k, v)
    for blk in range(NB):
        ins = {k: g[f"{name}/in/{k}/{blk}"] for k in d.inputs}
        o, m = p.process(B, ins, want_mix=True)
        assert np.array_equal(o, g[name + "/out"][blk], equal_nan=True), (name, blk)
        assert np.array_equal(m, g[name + "/mix"][blk], equal_nan=True), (name, blk)


def test_chorus_port_equals_reference(port, reference):
    """maxiChorus: the reference draws its noise from libc rand(); the port is fed the sequence the same libc produces after the same
    srand (oracle_py.noise_fill), in the (frame, voice) order the reference's loop draws it. Outputs, buses, both delay lines' indices
    and contents, the lores state: bit for bit."""
    name, d, params, _, exact, taps = PC.chorus()
    V, B, NB, seed = 9, 150, 3, 777
    noise = port.noise_fill(seed, NB * B * V, "port").reshape(NB, B, V)
    assert same(noise, reference.noise_fill(seed, NB * B * V, "reference").reshape(NB, B, V), equal_nan=False)
    assert np.abs(noise).max() <= 1.0 and noise.std() > 0.5
    po = port.Patch(d, V, delay_taps=taps, kind="port"); pr = reference.Patch(d, V, delay_taps=taps, kind="reference")
    for k, v in params(V, 3).items():
        po.set(k, v); pr.set(k, v)
    reference.srand(seed, "reference")
    si = [i for i, st in enumerate(d.stages) if st[0] == 18][0]
    for blk in range(NB):
        orr, mr = pr.process(B, {"noise": noise[blk]}, want_mix=True)          # draws from rand() itself
        oo, mo = po.process(B, {"noise": noise[blk]}, want_mix=True)
        assert same(oo, orr, equal_nan=False), blk
        assert same(mo, mr, equal_nan=False), blk
        assert np.isfinite(oo).all() and np.abs(oo).max() > 1e-3
    for sl in range(4):
        assert same(po.get_state(si, sl), pr.get_state(si, sl), equal_nan=False), sl
    for v in range(V):
        assert same(po.ring(si, v, 2 * taps), pr.ring(si, v, 2 * taps), equal_nan=False), v
    assert len({int(x) for x in po.get_state(si, 0)} | {int(x) for x in po.get_state(si, 1)}) > 2      # the lines are swept: indices diverged


def test_chorus_golden_exact(port):
    g = G.load("chorus")
    name, d, params, _, exact, taps = PC.chorus()
    V, B, NB = int(g["V"]), int(g["B"]), int(g["NB"])
    assert int(g["taps"]) == taps
    p = port.Patch(d, V, delay_taps=taps, kind="port")
    for k, v in params(V, 99).items():
        p.set(k, v)
    for blk in range(NB):
        o, m = p.process(B, {"noise": g["noise"][blk]}, want_mix=True)
        assert np.array_equal(o, g["out"][blk]) and np.array_equal(m, g["mix"][blk]), blk


def test_registers_read_zero_until_written(port):
    from maximilian_b200.patchdef import PatchDef, R
    d = PatchDef()
    d.stage("add", R(3), d.K(1.5), dst=R(0))        # R3 was written by the PREVIOUS sample's last stage: must read 0 here
    d.stage("out", R(0))
    d.stage("add", R(0), d.K(1.0), dst=R(3))
    o, _ = port.Patch(d, 3, kind="port").process(4)
    assert np.all(o == 1.5)
