"""K6, the peer-memory mix exchange, with every rank on one device: 2, 3, 4 (and 8 for S1) processes share the card, each owning a voice
shard, connected through CUDA IPC exactly as ranks on separate GPUs are. Every kernel-side step of the protocol runs for real: the pushes into
peers' lanes, the stride between source ranks, both slots, the flags, the last-CTA ticket and the rank-order sum.

Each rank runs its handle next to a twin without the exchange (tests/exchange_ranks.py). The twins' buses are the lanes, so every rank's
bus must equal ((0.0 + L_0) + L_1) + ... bit for bit; worlds of 3 and more also pin the order of that sum, which two ranks cannot
(a + b == b + a). The exchange must leave every handle's output and state as the twin's, its status mask must stay 0, and the bus must
match the oracle's whole-bank or whole-patch mix to fp64 reassociation. What one device cannot check -- the ordering of NVLink traffic by
the system-scope fences, and timing across GPUs -- stays with test_gpu_exchange.py's multi-GPU tests."""
import os

import numpy as np
import pytest

import events_checks as EV
import exchange_ranks as ER
from maximilian_b200 import shard
from maximilian_b200 import workloads as W

pytestmark = pytest.mark.gpu

WORLDS = [2, 3, 4]
RTOL, ATOL = 1e-9, 1e-10


def _tables():
    t = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tables.npz"))
    return t["sine"], t["transition"], float(t["sine_before"])


_runs = {}


def _ranks(world):
    """{rank: {scenario: result}} of one spawn of `world` ranks on device 0 (every scenario; S1 alone at world 8), run once per module"""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    if world not in _runs:
        names = ["s1"] if world == 8 else list(ER.SCENARIOS)
        try:
            _runs[world] = shard.run_ranks(world, ER.run_scenarios, (names, _tables()), devices=[0] * world)
        except Exception as e:          # kept, so that the other tests of this world report it without spawning again
            _runs[world] = e
    r = _runs[world]
    if isinstance(r, shard.RankStartError):
        pytest.skip(f"a second process cannot create a context on this device (exclusive-process compute mode?): {r}")
    if isinstance(r, Exception):
        raise r
    return r


def _scenario(world, name):
    res = _ranks(world)
    out = []
    for r in range(world):
        s = res[r][name]
        assert "error" not in s, f"world {world} rank {r} {name}:\n{s['error']}"
        assert s["status"] == 0, f"world {world} rank {r} {name}: exchange status mask {s['status']:#x}"
        out.append(s)
    return out


def _rank_sum(lanes):
    s = np.zeros_like(lanes[0])
    for lane in lanes:                  # the kernel's order: s = 0.0; s += lane_r for r = 0 .. world - 1
        s = s + lane
    return s


def _same_state(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        assert np.array_equal(a[k], b[k]), f"{what}: state {k} differs from the twin's"


def _check(ranks, part, world, what, exchanged=True):
    """every rank's bus == the rank-order sum of the twins' buses (exchanged=False: == its own twin's), bit for bit; out and state as the
    twin's. Returns rank 0's buses."""
    parts = [s["parts"][part] for s in ranks]
    for k in range(len(parts[0]["bus"])):
        exp = _rank_sum([p["twin"][k] for p in parts])
        for r, p in enumerate(parts):
            want = exp if exchanged else p["twin"][k]
            got = p["bus"][k]
            assert got.shape == want.shape, f"{what}: world {world} rank {r} block {k}: bus of shape {got.shape}, expected {want.shape}"
            bad = np.flatnonzero(np.any(got != want, axis=1))
            assert bad.size == 0, (f"{what}: world {world} rank {r} block {k} ({want.shape[0]} frames): {bad.size} frames differ from the "
                                   f"rank-order sum, first at frame {bad[0]}, max |diff| {np.abs(got - want).max():.3e}")
    for r, p in enumerate(parts):
        if p["out"] is not None:
            for k, (o, t) in enumerate(zip(p["out"], p["twin_out"])):
                assert np.array_equal(o, t), f"{what}: world {world} rank {r} block {k}: out differs from the twin's"
        _same_state(*p["state"], f"{what}: world {world} rank {r}")
    return parts[0]["bus"]


def _close(buses, oracle, what):
    assert len(buses) == len(oracle)
    for k, (g, o) in enumerate(zip(buses, oracle)):
        np.testing.assert_allclose(g, o, rtol=RTOL, atol=ATOL, err_msg=f"{what}: block {k} against the oracle")


_oracle = {}


def _saw_biquad_oracle(port, V, blocks, seed=3):
    key = ("saw_biquad", V, tuple(blocks), seed)
    if key not in _oracle:
        o = port.Bank(V, osc="saw", filt="biquad")
        W.configure_bank(o, "biquad", W.voice_params(V, seed=seed))
        _oracle[key] = [o.process(n, want_out=False, want_mix=True)[1] for n in blocks]
    return _oracle[key]


def _delay_oracle(port, V, blocks, seed):
    o = port.Bank(V, osc="saw", filt="none", env=True, delay=True, delay_capacity=ER.S2_CAP)
    W.configure_bank(o, "none", W.voice_params(V, seed=seed, delay_size=ER.S2_CAP, ragged_delay=True), env=True, delay=True)
    return [o.process(n, *ER.delay_gates(V, n, k, seed), want_out=False, want_mix=True)[1] for k, n in enumerate(blocks)]


def _polysynth_oracle(port, V, blocks, seed):
    port.set_tables(*_tables(), "port")
    o = port.Patch(W.polysynth_patch("u8"), V, kind="port")
    for k, v in W.polysynth_params(V, seed=seed).items():
        o.set(k, v)
    pat = W.note_pattern(V, seed=seed)
    return [o.process(n, {"trigger": W.note_triggers(pat, n, k).astype(np.float64)}, want_out=False, want_mix=True)[1]
            for k, n in enumerate(blocks)]


@pytest.mark.parametrize("world", WORLDS + [8])
def test_s1_bank_bus(world, port):
    """saw -> biquad, 6001 voices in uneven shards; blocks of 1, 256, 7, 256, 129 and 33 frames: both slots three times each, a full bus,
    rows past one stride of the final loop, short buses whose lanes lie max_doubles apart"""
    s = _scenario(world, "s1")
    _close(_check(s, "main", world, "S1"), _saw_biquad_oracle(port, ER.S1_V, ER.S1_BLOCKS), f"S1 world {world}")


@pytest.mark.parametrize("world", WORLDS)
def test_s2_delay_bank_out_and_bus(world, port):
    """saw -> ADSR -> maxiDelayline::dl (the delay kernel, its own warp count), gates sliced from whole-bank arrays: out and bus"""
    s = _scenario(world, "s2")
    _close(_check(s, "main", world, "S2"), _delay_oracle(port, ER.S2_V, ER.S2_BLOCKS, 5), f"S2 world {world}")


@pytest.mark.parametrize("world", WORLDS)
def test_s3_tiny_shards(world, port):
    """world + 1 voices (one rank with 2, the others 1), then 33-voice shards of a delay bank (a second warp with one voice)"""
    s = _scenario(world, "s3")
    _close(_check(s, "tiny", world, "S3 tiny"), _saw_biquad_oracle(port, world + 1, ER.S3_BLOCKS, seed=13), f"S3 tiny world {world}")
    _close(_check(s, "warp33", world, "S3 33 voices"), _delay_oracle(port, 33 * world, ER.S3_BLOCKS, 17), f"S3 33 voices world {world}")


@pytest.mark.parametrize("world", WORLDS)
def test_s4_oversized_bus_refused_on_every_rank(world, port):
    """a bus of max_doubles + 2 values: MXB_ERR_INVALID on every rank before any kernel, state as the twin's; the next block exchanges"""
    s = _scenario(world, "s4")
    for r, x in enumerate(s):
        assert len(x["refusals"]) == 2
        for f in x["refusals"]:
            assert f["error"] is not None and "-> -1" in f["error"], f"rank {r}: {f['error']}"
            assert f["launches"] == 0, f"rank {r}: a refused call launched {f['launches']} kernels"
            _same_state(*f["state"], f"S4 world {world} rank {r} after a refused call")
    valid = [n for n in ER.S4_CALLS if n <= ER.B]
    _close(_check(s, "main", world, "S4"), _saw_biquad_oracle(port, ER.S1_V, valid), f"S4 world {world}")


@pytest.mark.parametrize("world", WORLDS)
def test_s5_voice_patch_mixed_modes(world, port):
    """the polysynth, even ranks fused and odd ranks interpreted, every rank switching after the second block: the same bus bits"""
    s = _scenario(world, "s5")
    _close(_check(s, "main", world, "S5"), _polysynth_oracle(port, ER.S5_V, ER.S5_BLOCKS, 9), f"S5 world {world}")


@pytest.mark.parametrize("world", WORLDS)
def test_s6_patch_with_events_streams(world, port):
    """pitch and trigger as events streams sliced per shard; the oracle reads the equivalent dense streams of the whole patch"""
    s = _scenario(world, "s6")
    bus = _check(s, "main", world, "S6")
    port.set_tables(*_tables(), "port")
    o = port.Patch(W.polysynth_pitch_patch("f64", "f64"), ER.S6_V, kind="port")
    prm = W.polysynth_params(ER.S6_V, seed=31)
    for k in ("attack", "decay", "sustain", "release", "pan"):
        o.set(k, prm[k])
    held = {"pitch": np.zeros(ER.S6_V), "trigger": np.zeros(ER.S6_V)}
    mixes = []
    for k, n in enumerate(ER.S6_BLOCKS):
        pe, te = W.note_events(ER.S6_V, n, k, seed=77)
        dp, held["pitch"] = EV.events_to_dense(*pe, n, held["pitch"])
        dt, held["trigger"] = EV.events_to_dense(*te, n, held["trigger"])
        mixes.append(o.process(n, {"pitch": dp, "trigger": dt}, want_out=False, want_mix=True)[1])
    _close(bus, mixes, f"S6 world {world}")


@pytest.mark.parametrize("world", WORLDS)
def test_s7_one_exchange_two_handles_in_turn(world, port):
    """the exchange on a bank, detached (the bank's bus is local again), then on a patch after a 0-frame call that launches nothing"""
    s = _scenario(world, "s7")
    _close(_check(s, "bank", world, "S7 bank"), _saw_biquad_oracle(port, ER.S1_V, ER.S7_BANK_BLOCKS), f"S7 bank world {world}")
    _check(s, "detached", world, "S7 detached", exchanged=False)
    for r, x in enumerate(s):
        assert x["zero"] == dict(launches=0, shape=(0, 2)), f"rank {r}: {x['zero']}"
    _close(_check(s, "patch", world, "S7 patch"), _polysynth_oracle(port, ER.S5_V, ER.S7_PATCH_BLOCKS, 9), f"S7 patch world {world}")


@pytest.mark.parametrize("world", WORLDS)
def test_s8_device_and_split_async_memory(world):
    """S1's blocks with the bus in device memory on a non-blocking stream and with MXB_MEM_SPLIT | MXB_MEM_ASYNC into page-locked host
    memory: after a synchronisation the status mask is 0 and the buses are S1's host-path buses, bit for bit"""
    s = _scenario(world, "s8")
    s1 = _scenario(world, "s1")
    for r, x in enumerate(s):
        assert x["mode_status"] == 0, f"rank {r}: exchange status mask {x['mode_status']:#x}"
    for part in ("device", "split"):
        bus = _check(s, part, world, f"S8 {part}")
        for k, (a, b) in enumerate(zip(bus, s1[0]["parts"]["main"]["bus"])):
            assert np.array_equal(a, b), f"S8 {part} world {world} block {k}: differs from S1's host path"

