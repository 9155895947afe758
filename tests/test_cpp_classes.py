"""Every recording class of the C++ layer (include/maximilian_b200.hpp) through tests/cpp/patch_classes.cpp, against the oracle running what
the reference's signatures say each play() means (tests/cpp_classes.py): the argument order of every recorded stage, the operand order of
the operators, the router (maxiVoices::matchChain / runBank) from both sides, and the per-block handling of parameters, gates and phase
resets. Bars of DESIGN.md §2: the bank route bit-identical (sine / cos 1e-9), a voice patch bit-identical when every stage is exact and 1e-9
relative otherwise, the bus 1e-9 relative, and the two patch kernels bit-identical to each other."""
import os
import re
import subprocess

import numpy as np
import pytest

import cpp_classes as CC
import golden_checks as G
import patch_checks as PK
from maximilian_b200.patchdef import OP, STATE_SLOTS
from test_cpp_dropin import ROOT, compile_patch

SRC = os.path.join(ROOT, "tests", "cpp", "patch_classes.cpp")
HEADER = os.path.join(ROOT, "include", "maximilian_b200.hpp")
V, B, NB = 37, 200, 3
MODES = ("fused", "interpret")
CASES = {c.name: c for c in CC.cases()}
BANK = [n for n, c in CASES.items() if c.kind == "bank"]
PATCH = [n for n, c in CASES.items() if c.kind == "patch"]
ERROR = [n for n, c in CASES.items() if c.kind == "error"]
MAX_STAGES = 64
RECORDING_CLASSES = ("maxiOsc", "maxiFilter", "maxiSVF", "maxiBiquad", "maxiEnv", "maxiEnvGen", "maxiDelayline", "maxiFlanger", "maxiChorus",
                     "maxiDCBlocker", "maxiNonlinearity", "maxiMix")


@pytest.fixture(scope="module")
def bindir(tmp_path_factory):
    return tmp_path_factory.mktemp("classes")


@pytest.fixture(scope="module")
def exe(bindir):
    return compile_patch(bindir, SRC)


def test_driver_compiles_and_prints_usage(exe):
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr


def test_driver_and_table_name_the_same_cases(exe):
    r = subprocess.run([exe, "--list"], capture_output=True, text=True, check=True)
    listed = dict(line.split() for line in r.stdout.splitlines())
    assert set(listed) == set(CASES)
    assert {n for n, b in listed.items() if b == "1"} == set(BANK)
    assert all(CASES[n].ref.startswith("src/maximilian.") for n in CASES)


def _public_methods(src, cls):
    body = re.search(r"\nclass %s \{\npublic:\n(.*?)\n(?:private:|\};)" % cls, src, re.S).group(1)
    return set(re.findall(r"^\s+(?:template <[^>]*>\s*)?(?:maxiSignal|void|bool)\s+(\w+)\(", body, re.M))


def test_every_recording_method_is_called():
    """every public method of maxiOsc ... maxiMix that records into a play() (the getters getLoop / getRetrigger read the shape back) and
    maxiVoices::sum / out is called by some case"""
    hdr, drv = open(HEADER).read(), open(SRC).read()
    methods = {(cls, m) for cls in RECORDING_CLASSES for m in _public_methods(hdr, cls) if not m.startswith("get")}
    assert len(methods) >= 40 and ("maxiNonlinearity", "asymclip") in methods and ("maxiEnv", "ar") in methods
    methods |= {("maxiVoices", "sum"), ("maxiVoices", "out")}
    missing = sorted(f"{c}::{m}" for c, m in methods if not re.search(r"(\.|->)%s\(" % m, drv))
    assert not missing, missing
    # both maxiEnv::adsr overloads, with every trigger kind: interval gate, stream and signal
    assert re.search(r"adsr\(w, r\.p\(1\), r\.p\(2\), r\.p\(3\), r\.p\(4\), 3, r\.gate\(\)\)", drv)
    assert "adsr(x, r.p(1), r.p(2), r.p(3), r.p(4), r.p(5), r.stream(0))" in drv and "e3.adsr(x, t)" in drv
    assert "adsr(w, r.gate())" in drv and "ar(x, r.p(6), r.p(7), r.p(8), r.stream(1))" in drv


# ------------------------------------------------------------------------------------------------ GPU

@pytest.fixture(scope="module")
def runs(port, exe, tmp_path_factory):
    """every case through the driver: one process per patch mode, many cases each. {(case, mode): (status, out.bin path)}"""
    d = tmp_path_factory.mktemp("classes_runs")
    g = G.load("tables")
    tables = np.concatenate([g["sine"], g["transition"], [float(g["sine_before"])]])
    for name, c in CASES.items():
        c.write(d / f"{name}.in", V, B, NB, tables)
    res = {}
    for mode in MODES:
        names = ([n + "_x1" for n in BANK] + PATCH) + (BANK + ERROR if mode == "fused" else [])
        lst = d / f"{mode}.list"
        lst.write_text("".join(f"{n} {d / (n.removesuffix('_x1') + '.in')} {d / f'{n}.{mode}.out'} {V} {B} {NB}\n" for n in names))
        r = subprocess.run([exe, "--batch", str(lst)], capture_output=True, text=True, env=dict(os.environ, MXB_PATCH_MODE=mode))
        assert r.returncode == 0, r.stderr
        status = dict(line.split(" ", 1) for line in r.stdout.splitlines())
        assert set(status) == set(names), r.stderr
        for n in names:
            res[(n, mode)] = (status[n], d / f"{n}.{mode}.out")
    return res


def _read(path, fused):
    raw = np.fromfile(path, dtype=np.float64)
    o, blocks = 0, []
    for _ in range(NB):
        out = raw[o:o + B * V].reshape(B, V); o += B * V
        mix = raw[o:o + 2 * B].reshape(B, 2); o += 2 * B
        blocks.append((out, mix, raw[o])); o += 1
    state = {}
    if fused:
        for name in CC.BANK_STATE:
            state[name] = raw[o:o + V]; o += V
        n = int(raw[o]); o += 1
        state["ring"] = raw[o:o + V * n].reshape(V, n); o += V * n
    else:
        for st in range(MAX_STAGES):
            k = int(raw[o]); o += 1
            state[st] = [raw[o + j * V:o + (j + 1) * V] for j in range(k)]; o += k * V
            n = int(raw[o]); o += 1
            state[(st, "ring")] = raw[o:o + V * n].reshape(V, n); o += V * n
    assert o == raw.size
    return blocks, state


def _cmp(got, ref, exact, what):
    if exact:
        assert np.array_equal(got, ref, equal_nan=True), f"{what}: not bit-identical, max abs err {np.nanmax(np.abs(got - ref))}"
    else:
        assert np.array_equal(np.isnan(got), np.isnan(ref)), what
        np.testing.assert_allclose(got, ref, rtol=1e-9, atol=1e-12, err_msg=what)


def _bus(got, ref, what):
    np.testing.assert_allclose(got, ref, rtol=1e-9, atol=1e-11, err_msg=what)


def _bank_oracle(port, c):
    lib = port.load("port")
    o = port.Bank(V, kind="port", **c.cfg)
    outs = []
    for blk in range(NB):
        P, on, off, _ = c.data(V, B, blk)
        c.setter(o, P, blk, lib)
        outs.append(o.process(B, on if c.gates else None, off if c.gates else None, want_out=True, want_mix=True))
    return o, outs


def _bank_state_names(cfg):
    filt = cfg.get("filt", "none")
    names = ["phase", "osc_output"] + (["filt0", "filt1"] if filt != "none" else []) + (["filt2"] if filt == "svf" else [])
    names += ["env_amplitude", "env_output", "env_holdcount", "env_flags"] if cfg.get("env") else []
    return names + (["delay_phase"] if cfg.get("delay") else [])


INTEGRAL = ("env_holdcount", "env_flags", "delay_phase")


@pytest.mark.gpu
@pytest.mark.parametrize("name", BANK)
def test_bank_shaped_case_runs_fused_and_matches_oracle(port, runs, name):
    c = CASES[name]
    status, path = runs[(name, "fused")]
    assert status == "ok", status
    blocks, state = _read(path, True)
    o, outs = _bank_oracle(port, c)
    exact = c.cfg["osc"] not in ("sinewave", "coswave")
    for blk, ((out, mix, fused), (oo, mo)) in enumerate(zip(blocks, outs)):
        assert fused == 1.0, f"blk{blk}: the chain did not run on the fused bank"
        if c.out:
            _cmp(out, oo, exact, f"blk{blk} out")
        if c.mix:
            _bus(mix, mo, f"blk{blk} bus")
    assert np.abs(outs[-1][0]).max() > 1e-3
    for s in _bank_state_names(c.cfg):
        _cmp(state[s], o.get(s), exact or s in INTEGRAL or s == "phase", s)
    if c.cfg.get("delay"):
        ring = np.stack([o.ring(v, c.cap) for v in range(V)])
        _cmp(state["ring"], ring, exact, "ring")


def _x1_stage_map(cfg):
    """(stage, [(slot, bank state name)]) of the chain's stages in the `_x1` voice patch, in recording order"""
    m = [[(0, "phase"), (1, "osc_output")]]
    if cfg.get("env"):
        m.append([(0, "env_amplitude"), (1, "env_output"), (2, "env_holdcount"), (3, "env_flags")])
    filt = cfg.get("filt", "none")
    if filt != "none":
        m.append([(0, "filt0"), (1, "filt1")] + ([(2, "filt2")] if filt == "svf" else []))
    if cfg.get("delay"):
        m.append([(0, "delay_phase")])
    return list(enumerate(m))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", BANK)
def test_bank_shaped_case_with_identity_runs_as_patch_and_matches_oracle(port, runs, name, mode):
    """the same play() with `w * 1.0` appended: matchChain refuses it, so the runBank mapping and the patch stages meet one oracle"""
    c = CASES[name]
    status, path = runs[(name + "_x1", mode)]
    assert status == "ok", status
    blocks, state = _read(path, False)
    o, outs = _bank_oracle(port, c)
    exact = c.cfg["osc"] not in ("sinewave", "coswave") and c.cfg.get("filt", "none") == "none"
    for blk, ((out, mix, fused), (oo, mo)) in enumerate(zip(blocks, outs)):
        assert fused == 0.0, f"blk{blk}: w * 1.0 ran on the fused bank"
        if c.out:
            _cmp(out, oo, exact, f"blk{blk} out")
        if c.mix:
            _bus(mix, mo, f"blk{blk} bus")
    smap = _x1_stage_map(c.cfg)
    for st, slots in smap:
        assert len(state[st]) == len(slots), f"stage {st}: {len(state[st])} state slots"
        for slot, s in slots:
            _cmp(state[st][slot], o.get(s), exact or s in INTEGRAL or s == "phase", f"stage {st} {s}")
    assert len(state[len(smap)]) == 0, "the stage after the chain is the identity, without state"
    if c.cfg.get("delay"):
        ring = np.stack([o.ring(v, c.cap) for v in range(V)])
        _cmp(state[(len(smap) - 1, "ring")], ring, exact, "ring")
    if mode == "interpret":
        a, b = np.fromfile(path), np.fromfile(runs[(name + "_x1", "fused")][1])
        assert np.array_equal(a, b, equal_nan=True), "the interpreting and the generated kernel differ"


def _patch_oracle(port, c):
    lib = port.load("port")
    d, pmap, imap = c.build()
    if getattr(c, "fix", None):
        c.fix(d, lib)
    PK.set_tables(port, library=False)
    o = port.Patch(d, V, sample_rate=c.sr, delay_taps=c.cap, kind="port")
    outs = []
    for blk in range(NB):
        P, _, _, S = c.data(V, B, blk)
        for pname, k in pmap.items():
            o.set(pname, P[k])
        for st, k in (c.phase(blk) if getattr(c, "phase", None) else []):
            o.set_state(st, 0, P[k])
        outs.append(o.process(B, {iname: S[k] for iname, k in imap.items()}, want_out=True, want_mix=c.mix))
    return d, o, outs


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", PATCH)
def test_patch_shaped_case_matches_oracle(port, runs, name, mode):
    c = CASES[name]
    status, path = runs[(name, mode)]
    assert status == "ok", status
    blocks, state = _read(path, False)
    d, o, outs = _patch_oracle(port, c)
    for blk, ((out, mix, fused), (oo, mo)) in enumerate(zip(blocks, outs)):
        assert fused == 0.0, f"blk{blk}: ran on the fused bank"
        _cmp(out, oo, c.exact, f"blk{blk} out")
        if c.mix:
            _bus(mix, mo, f"blk{blk} bus")
    assert np.abs(outs[-1][0]).max() > 1e-3
    for st in range(MAX_STAGES):
        op = d.stages[st][0] if st < len(d.stages) else None
        assert len(state[st]) == STATE_SLOTS.get(op, 0), f"stage {st}: {len(state[st])} state slots"
        for slot, got in enumerate(state[st]):
            _cmp(got, o.get_state(st, slot), c.exact or slot in PK.INT_SLOTS.get(op, ()), f"stage {st} slot {slot}")
    for st, lines in PK.ring_stages(d):
        ring = np.stack([o.ring(st, v, lines * c.cap) for v in range(V)])
        _cmp(state[(st, "ring")], ring, c.exact, f"ring of stage {st}")
    if mode == "interpret":
        a, b = np.fromfile(path), np.fromfile(runs[(name, "fused")][1])
        assert np.array_equal(a, b, equal_nan=True), "the interpreting and the generated kernel differ"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ERROR)
def test_unsupported_play_raises(runs, name):
    c = CASES[name]
    assert runs[(name, "fused")][0] == f"maxiError {c.code} {c.block}"
