"""Every instantiation of the bank kernels (tests/bank_matrix.py: 480 K1 and 240 K2 keys, grouped by bank description) against the
oracle: each group's blocks run one after the other on one GPU bank and on one port.Bank fed the same streams, and after every block
the output, the bus, every state array the bank exposes and (K2) the rings of voices 0, 1, 31, 32, V/2 and V-1 are compared.

Bars (DESIGN.md §2): bit-identical, NaN positions included, while the group's chain has no sin / cos and no per-sample design has run
(a swept cutoff leaves the filter state within 1e-9 of the oracle's, so every later block of the group is held to 1e-9 relative +
1e-12); sinewave / coswave 1e-12 absolute at the oscillator and the envelope, 1e-9 relative + 1e-12 behind a filter (a biquad at a
low cutoff holds states in the thousands, and its output is a difference of them: the sin difference comes out ~1e-12 relative); the
bus 1e-9 relative; integer state exact; fp32 output the oracle's rounded to float32, bit for bit, wherever the fp64 chain is
bit-identical (otherwise the fp64 bar plus the float32 rounding).
"""
import numpy as np
import pytest

import bank_matrix as M
from maximilian_b200 import capi

pytestmark = pytest.mark.gpu


def _close(got, ref, tol, what):
    if tol is None:
        assert np.array_equal(got, ref, equal_nan=True), \
            f"{what}: not bit-identical ({np.count_nonzero(~((got == ref) | (np.isnan(got) & np.isnan(ref))))} values differ)"
    else:
        assert np.array_equal(np.isnan(got), np.isnan(ref)), f"{what}: NaN positions differ"
        np.testing.assert_allclose(got, ref, rtol=tol[0], atol=tol[1], err_msg=what)


def _device_block(bank, b, s, V):
    """K1 with `out` one element past an aligned device address (the scalar stores of an even bank), every stream on the device"""
    import torch
    dev = torch.device("cuda", 0)
    n = b.n
    buf = torch.full((n * V + 2,), -7.0, dtype=torch.float32 if b.f32 else torch.float64, device=dev)
    out = buf[1:1 + n * V]
    mix = torch.empty((n, 2), dtype=torch.float64, device=dev) if b.mix else None
    d = {k: (torch.from_numpy(np.ascontiguousarray(v)).to(dev) if v is not None else None) for k, v in s.items()}
    ptr = lambda k: d[k].data_ptr() if d[k] is not None else None
    bank.process_mod_device(n, out_ptr=out.data_ptr(), mix_ptr=mix.data_ptr() if mix is not None else None, freq_tv_ptr=ptr("freq_tv"),
                            cutoff_tv_ptr=ptr("cutoff_tv"), delay_size_tv_ptr=ptr("delay_size_tv"), trig_tv_ptr=ptr("trig_tv"),
                            trig_on_ptr=ptr("trig_on"), trig_off_ptr=ptr("trig_off"), f32=b.f32)
    torch.cuda.synchronize()
    assert buf[0].item() == -7.0 and buf[-1].item() == -7.0, "the store wrote outside `out`"
    return out.cpu().numpy().reshape(n, V), (mix.cpu().numpy() if mix is not None else None)


@pytest.mark.parametrize("group", M.GROUPS, ids=lambda g: g.name)
def test_bank_matrix_group(port, group):
    g, V = group, group.V
    gb = capi.Bank(V, max_frames=g.max_frames, **g.bank_kw())
    ob = port.Bank(V, **g.bank_kw())
    for name, v in M.params(g).items():
        gb.set(name, v); ob.set(name, v)
    filt = g.desc["filt"] != "none"
    trig = (0.0, 1e-12) if g.trig else None
    trig_state = (1e-9, 1e-12) if g.trig else None
    trig_out = trig_state if filt else trig
    rings = sorted({v for v in (0, 1, 31, 32, V // 2, V - 1) if v < V})
    for i, b in enumerate(g.blocks):
        s = M.streams(g, i)
        what = f"block {i} {b.key} ({b.n} frames)"
        if b.misaligned:
            og, mg = _device_block(gb, b, s, V)
        else:
            og, mg = gb.process(b.n, s["trig_on"], s["trig_off"], want_out=b.out, want_mix=b.mix,
                                out_dtype=np.float32 if b.f32 else np.float64, freq_tv=s["freq_tv"], cutoff_tv=s["cutoff_tv"],
                                delay_size_tv=s["delay_size_tv"], trig_tv=s["trig_tv"])
        oo, mo = ob.process(b.n, s["trig_on"], s["trig_off"], want_mix=b.mix, freq_tv=s["freq_tv"], cutoff_tv=s["cutoff_tv"],
                            delay_size_tv=s["delay_size_tv"], trig_tv=s["trig_tv"])
        swept = any(x.cm for x in g.blocks[:i + 1])          # the filter state carries a per-sample design from here on
        tol = None if b.exact else ((1e-9, 1e-12) if swept else trig_out)
        tol_state = (1e-9, 1e-12) if swept else trig_state
        if b.out:
            if b.f32:
                assert og.dtype == np.float32
                if tol is None:
                    _close(og, oo.astype(np.float32), None, f"{what}: fp32 output")
                else:
                    _close(og.astype(np.float64), oo, (tol[0] + 2.0 ** -24, tol[1]), f"{what}: fp32 output")
            else:
                _close(og, oo, tol, f"{what}: output")
        if b.mix:
            _close(mg, mo, (1e-9, 1e-11), f"{what}: bus")
        assert np.array_equal(gb.get("phase"), ob.get("phase"), equal_nan=True), f"{what}: phase"
        _close(gb.get("osc_output"), ob.get("osc_output"), trig, f"{what}: osc_output")
        if filt:
            for name in ("filt0", "filt1", "filt2"):
                _close(gb.get(name), ob.get(name), tol_state, f"{what}: {name}")
        if g.desc["env"]:
            assert np.array_equal(gb.get("env_amplitude"), ob.get("env_amplitude"), equal_nan=True), f"{what}: env_amplitude"
            _close(gb.get("env_output"), ob.get("env_output"), trig, f"{what}: env_output")
            for name in ("env_holdcount", "env_flags"):
                assert np.array_equal(gb.get(name), ob.get(name)), f"{what}: {name}"
        if g.desc["delay"]:
            assert np.array_equal(gb.get("delay_phase"), ob.get("delay_phase")), f"{what}: delay_phase"
            for v in rings:
                _close(gb.ring(v, M.TAPS), ob.ring(v, M.TAPS), tol, f"{what}: ring of voice {v}")
