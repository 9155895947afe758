"""The voice-patch matrix (tests/patch_matrix.py) on the CPU: the plain-C interpreter of oracle/maxi_oracle.c against the same stage
lists run by the reference's own objects (oracle/ref_shim.cpp, as recorded by oracle/replay.py), bit for bit -- outputs, buses, every
state slot and the rings over three blocks -- and the code the library generates for each case: it compiles for sm_90a, it hoists
exactly the designs, increments and rates whose operands are parameters and constants, and it carries every constant's bits."""
import re
import struct

import numpy as np
import pytest

import patch_matrix as PM
from patch_checks import set_tables
from maximilian_b200 import capi
from maximilian_b200.patchdef import OP, FILT, KINDS, STATE_SLOTS as SLOTS
from oracle.replay import same
CASES = PM.cases()


def _ids(c):
    return c[0]


def test_matrix_covers_every_op_and_kind():
    seen = PM.coverage(CASES)
    for op, table in KINDS.items():
        for kind in table:
            assert (op, kind) in seen, (op, kind)
    for op in OP:
        assert any(o == op for o, _ in seen), op
    assert len({c[0] for c in CASES}) == len(CASES)


@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_matrix_port_equals_reference(port, reference, case):
    name, d, params, inputs, exact, taps = case
    set_tables(port, library=False)
    V, B, NB, seed = 24, 200, 3, 7
    ins = [inputs(V, B, blk, seed) for blk in range(NB)]          # before srand: the port's noise_fill re-seeds libc's rand() as well
    po = port.Patch(d, V, delay_taps=taps, kind="port"); pr = reference.Patch(d, V, delay_taps=taps, kind="reference")
    for k, v in params(V, 11).items():
        po.set(k, v); pr.set(k, v)
    if any(st[0] == OP["chorus"] for st in d.stages):
        reference.srand(seed, "reference")                        # the reference draws the chorus noise itself
    for blk in range(NB):
        oo, mo = po.process(B, ins[blk], want_mix=True); orr, mr = pr.process(B, ins[blk], want_mix=True)
        assert same(oo, orr), (name, blk)
        assert same(mo, mr), (name, blk)
    for si, (op, kind, dst, src) in enumerate(d.stages):
        for sl in range(SLOTS.get(op, 0)):
            if op == OP["filter"] and kind in (FILT["lopass"], FILT["hipass"]) and sl == 1:
                continue                                          # lopass / hipass keep one value (outputs[0])
            if op == OP["envgen"] and sl == 3:
                continue                                          # nxcHappened is indeterminate in the reference until the first trigger
            assert same(po.get_state(si, sl), pr.get_state(si, sl)), (name, si, sl)
        if op in (OP["delay"], OP["flanger"], OP["chorus"]):
            n = taps * (2 if op == OP["chorus"] else 1)
            for v in range(V):
                assert same(po.ring(si, v, n), pr.ring(si, v, n)), (name, si, v)


def test_envgen_nan_curve_plays_nan_like_the_reference(port):
    """maxiMap::linlin's std::min / std::max keep a NaN: the segment with the NaN curve plays NaN, the others do not"""
    name, d, params, inputs, exact, taps = [c for c in CASES if c[0] == "envgen_nan_curve"][0]
    V, B = 8, 200
    p = port.Patch(d, V, kind="port")
    for k, v in params(V, 3).items():
        p.set(k, v)
    o, _ = p.process(B, inputs(V, B, 0, 3))
    assert np.isnan(o).any() and np.isfinite(o).any()


def _invariant(s):
    return s < 0 or (s >> 8) in (1, 2)


def _hoisted(d):
    """(stage, marker of its design / increment / rate in the generated source, whether that belongs before the sample loop)"""
    out = []
    for i, (op, kind, dst, src) in enumerate(d.stages):
        inv = lambda *ks: all(_invariant(src[k]) for k in ks)      # noqa: E731
        if op == OP["osc"] and kind < 9:
            out.append((i, f"const double inc{i} = ", inv(0, 1, 2)))
        elif op == OP["filter"] and kind in (FILT["lores"], FILT["hires"]):
            out.append((i, f"filt_design<FILT_T_LORES>(f{i}, ", inv(1, 2)))
        elif op == OP["filter"] and kind == FILT["bandpass"]:
            out.append((i, f"double bc0_{i}, ", inv(1, 2)))
        elif op == OP["svf"]:
            out.append((i, f"filt_design<FILT_T_SVF>(f{i}, ", inv(1, 2)))
        elif op == OP["biquad"]:
            out.append((i, f"f{i}.c0 = cf[0]", inv(1, 2, 3)))
        elif op == OP["chorus"]:
            out.append((i, f"filt_design<FILT_T_LORES>(f{i}, ", inv(3)))
        elif op in (OP["env_adsr"], OP["env_ar"]):
            fields = dict(att=2, dec=3, sus=4, rel=5, holdtime=6) if op == OP["env_adsr"] else dict(att=2, rel=3, holdtime=4)
            out += [(i, f"\n e{i}.{f} = ", inv(k)) for f, k in fields.items()]       # a statement of its own (not the initialiser)
    return out


def _emits(text, marker):
    if marker.startswith("\n "):
        return re.search(r"\n\s+" + re.escape(marker[2:]), text) is not None
    return marker in text


@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_matrix_codegen(case):
    name, d, params, inputs, exact, taps = case
    src = capi.patch_codegen(d, compile=True)
    head, loop = src.split("for (int t = 0", 1)
    for i, marker, pre in _hoisted(d):
        assert _emits(head, marker) == pre and _emits(loop, marker) == (not pre), (name, i, marker, pre)
    for j, c in enumerate(d.consts):
        bits = struct.unpack("<Q", struct.pack("<d", c))[0]
        assert f"const double c{j} = __longlong_as_double(0x{bits:016x}LL);" in head, (name, j, c)
    assert len(re.findall(r"__longlong_as_double\(0x[0-9a-f]{16}LL\)", src)) == len(d.consts)


def test_matrix_uses_every_operand_class_and_every_special_constant():
    classes = set()
    for _, d, *_ in CASES:
        for op, kind, dst, src in d.stages:
            classes |= {s >> 8 for s in src if s >= 0}
    assert classes == {0, 1, 2, 3}
    bits = {struct.pack("<d", c) for _, d, *_ in CASES for c in d.consts}
    for c in (-0.0, float("inf"), float("-inf"), float("nan"), 5e-324, 2.2250738585072009e-308, 1e-300):
        assert struct.pack("<d", c) in bits, c
    # every input element type feeds a trigger
    types = {d.input_types.get(n, "f64") for _, d, *_ in CASES for n in d.inputs}
    assert types == {"f64", "u8", "bits"}


def test_state_slots_table_is_the_ports(port):
    """patchdef.STATE_SLOTS against the C port: a stage has exactly that many state words, every op of the matrix"""
    seen = set()
    for name, d, params, inputs, exact, taps in CASES:
        p = port.Patch(d, 4, delay_taps=taps, kind="port")
        for si, (op, *_) in enumerate(d.stages):
            n = SLOTS.get(op, 0)
            with pytest.raises(RuntimeError):
                p.get_state(si, n)
            if n:
                assert p.get_state(si, n - 1).shape == (4,)
            seen.add(op)
    assert seen == set(OP.values())
