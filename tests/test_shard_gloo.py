"""Host-side logic of the N > 1 path on CPU: two processes (gloo, 127.0.0.1), each owning its voice shard;
the all-reduced stereo mix must equal the single-process mix of the whole bank (fp64 reassociation only), and
the materialised per-voice output of a shard must equal the corresponding columns bit for bit.
The per-shard DSP is the plain-C oracle here (no GPU in this container) -- what is under test is the sharding,
the reduction and the max-over-ranks timing helper that bench.py uses with NCCL on the GPU box."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from maximilian_b200 import shard
from maximilian_b200 import workloads as W

V, B = 1000, 64


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle import oracle_py as O
    p = W.voice_params(V, seed=77)
    lo, hi = shard.shard_range(V, rank, world)
    ps = {k: v[lo:hi] for k, v in p.items()}
    b = O.Bank(hi - lo, osc="saw", filt="biquad", kind="port")
    W.configure_bank(b, "biquad", ps)
    out, mix = b.process(B, want_mix=True)
    m = torch.from_numpy(mix.copy())
    shard.allreduce_mix(m)
    slowest = shard.max_over_ranks(1.0 + rank, torch.device("cpu"))
    q.put((rank, lo, hi, out, m.numpy(), slowest))
    dist.barrier()
    dist.destroy_process_group()


def test_shard_range_partitions():
    for total, world in ((1000, 2), (1 << 20, 8), (7, 3), (5, 8)):
        r = [shard.shard_range(total, k, world) for k in range(world)]
        assert r[0][0] == 0 and r[-1][1] == total
        assert all(r[i][1] == r[i + 1][0] for i in range(world - 1))
        sizes = [b - a for a, b in r]
        assert max(sizes) - min(sizes) <= 1


def test_two_rank_mix_allreduce_matches_full_bank(port):
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    pnum = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, pnum, q)) for r in range(world)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=120) for _ in range(world)], key=lambda x: x[0])
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)

    p = W.voice_params(V, seed=77)
    full = port.Bank(V, osc="saw", filt="biquad")
    W.configure_bank(full, "biquad", p)
    out, mix = full.process(B, want_mix=True)
    for rank, lo, hi, o, m, slowest in res:
        assert np.array_equal(o, out[:, lo:hi])                 # voices are independent: shard == columns of the whole
        np.testing.assert_allclose(m, mix, rtol=1e-12, atol=1e-12)
        assert slowest == float(world)                          # max over ranks
    assert np.array_equal(res[0][4], res[1][4])                 # every rank holds the same reduced bus


def _patch_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle import oracle_py as O
    t = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tables.npz"))
    O.set_tables(t["sine"], t["transition"], float(t["sine_before"]), "port")
    Vp, Bp, nb = 300, 96, 3
    lo, hi = shard.shard_range(Vp, rank, world)
    o = O.Patch(W.polysynth_patch("u8"), hi - lo, kind="port")
    for k, v in W.polysynth_params(Vp, seed=21).items():
        o.set(k, np.ascontiguousarray(v[lo:hi]))
    pat = W.note_pattern(Vp, seed=21)
    outs, buses = [], []
    for blk in range(nb):
        out, mix = o.process(Bp, {"trigger": W.note_triggers(pat, Bp, blk, lo, hi).astype(np.float64)}, want_mix=True)
        m = torch.from_numpy(mix.copy())
        shard.allreduce_mix(m)
        outs.append(out.copy()); buses.append(m.numpy().copy())
    q.put((rank, lo, hi, np.stack(outs), np.stack(buses)))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_sharded_voice_patch_matches_the_whole_patch(port):
    """The polysynth voice patch sharded like maximilian_b200/shard.py's exchange ranks shard it on the GPUs (parameters and the per-sample
    trigger stream sliced per rank): shard outputs are the whole patch's columns bit for bit, the reduced bus is the whole patch's bus."""
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    pnum = _free_port()
    procs = [ctx.Process(target=_patch_worker, args=(r, world, pnum, q)) for r in range(world)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=120) for _ in range(world)], key=lambda x: x[0])
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)

    t = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tables.npz"))
    port.set_tables(t["sine"], t["transition"], float(t["sine_before"]), "port")
    Vp, Bp, nb = 300, 96, 3
    full = port.Patch(W.polysynth_patch("u8"), Vp, kind="port")
    for k, v in W.polysynth_params(Vp, seed=21).items():
        full.set(k, v)
    pat = W.note_pattern(Vp, seed=21)
    for blk in range(nb):
        out, mix = full.process(Bp, {"trigger": W.note_triggers(pat, Bp, blk).astype(np.float64)}, want_mix=True)
        for rank, lo, hi, outs, buses in res:
            assert np.array_equal(outs[blk], out[:, lo:hi])
            np.testing.assert_allclose(buses[blk], mix, rtol=1e-12, atol=1e-12)
    assert np.array_equal(res[0][4], res[1][4])


def test_events_stream_shards_are_the_voices_of_the_whole_stream():
    """tests/exchange_ranks.slice_events (each rank's part of a whole-bank events stream) against a per-voice loop over the whole stream"""
    import events_checks as EV
    from exchange_ranks import slice_events
    from maximilian_b200 import capi
    rng = np.random.default_rng(4)
    V, n = 37, 64
    whole = capi.pack_events(EV.random_events(rng, V, n))
    first, frame, value = whole
    for world in (1, 2, 3, 4, 8, 37):
        for rank in range(world):
            lo, hi = shard.shard_range(V, rank, world)
            lists = [[(int(frame[i]), float(value[i])) for i in range(first[v], first[v + 1])] for v in range(lo, hi)]
            want = capi.pack_events(lists)
            got = slice_events(whole, lo, hi)
            for g, w, what in zip(got, want, ("first", "frame", "value")):
                assert g.dtype == w.dtype and np.array_equal(g, w), (world, rank, what)
