"""Voice sharding across the GPUs of one box: the only multi-GPU structure the path has.

Voices (and STFT channels) are independent (no reference function couples two voices, SURVEY.md 8e), so rank r
of `world` owns the contiguous voice range shard_range(V, r, world) with all of its state; nothing moves
between GPUs except the stereo mix bus: one sum all-reduce of mix[n_frames][2] fp64 (16 KiB at 1024 frames)
per block, over NCCL/NVLink on the device (or gloo on the CPU for the host-logic tests).
"""
import torch
import torch.distributed as dist


def shard_range(total, rank, world):
    """Contiguous [lo, hi) of `total` items owned by `rank`; sizes differ by at most one."""
    base, rem = divmod(int(total), int(world))
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def allreduce_mix(mix, group=None):
    """In-place sum of the per-rank mix bus. `mix`: torch tensor [n_frames][channels] (cuda for nccl, cpu for gloo).
    Summation order over ranks is fixed by the backend's algorithm for a given world size: results are
    run-to-run reproducible, and differ from a sequential CPU sum only by fp64 reassociation (<= 1e-12 rel)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(mix, op=dist.ReduceOp.SUM, group=group)
    return mix


def max_over_ranks(value, device):
    """Device-side max of a python float over all ranks (timing: a multi-GPU step is as slow as its slowest rank)."""
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


# ---- one process per rank without torch.distributed: the peer-memory mix exchange driven over multiprocessing queues ----

class RankStartError(RuntimeError):
    """A rank could not create its device context (an exclusive-process device, for one): every rank was released and reaped."""


class RankLink:
    """A rank's side of the handshake with the parent (run_ranks): publish the rank's exchange handle, get every rank's back."""

    def __init__(self, rank, q_in, q_out):
        self.rank, self.q_in, self.q_out, self.reported = rank, q_in, q_out, False

    def report(self, kind, payload):
        self.reported = True
        self.q_out.put((self.rank, kind, payload))

    def handshake(self, handle):
        """handle: this rank's Exchange.local_handle(). Returns the handles of all ranks in rank order (for Exchange.connect), or None
        when the parent released the ranks because one of them could not start."""
        self.report("handle", handle)
        return self.q_in.get(timeout=180)


def _rank_main(body, rank, world, device, q_in, q_out, results, args):
    """One rank: its context on `device`, then body(rank, world, ctx, link, *args); what the body returns goes to the parent."""
    import traceback
    from maximilian_b200 import capi
    link = RankLink(rank, q_in, q_out)
    try:
        ctx = capi.Context(device, 48000)
    except capi.MxbError as e:
        link.report("no-context", f"rank {rank} on device {device}: {e}")
        return
    try:
        results.put((rank, "ok", body(rank, world, ctx, link, *args)))
    except BaseException:
        tb = traceback.format_exc()
        if not link.reported:
            link.report("error", tb)
        results.put((rank, "error", tb))


def run_ranks(world, body, args=(), devices=None):
    """Spawns `world` processes; rank r creates a context on devices[r] (default: device r) and runs
    body(rank, world, ctx, link, *args), which must call link.handshake() exactly once. Returns {rank: what the body returned}.
    Raises RankStartError (with the CUDA error text) when a rank could not create its context, RuntimeError (with the rank's
    traceback) when a body raised. Every child is joined, or killed if it is still alive, before this returns."""
    import torch.multiprocessing as mp
    devices = list(range(world)) if devices is None else list(devices)
    assert len(devices) == world
    ctx = mp.get_context("spawn")
    q_ins = [ctx.Queue() for _ in range(world)]
    q_out, results = ctx.Queue(), ctx.Queue()
    procs = [ctx.Process(target=_rank_main, args=(body, r, world, devices[r], q_ins[r], q_out, results, tuple(args))) for r in range(world)]
    [p.start() for p in procs]
    try:
        got = {}
        for _ in range(world):
            r, kind, payload = q_out.get(timeout=180)
            got[r] = (kind, payload)
        failed = {r: v for r, v in got.items() if v[0] != "handle"}
        if failed:
            for r in range(world):
                q_ins[r].put(None)             # release the ranks that started: their handshake returns None
            [p.join(timeout=60) for p in procs]
            texts = "\n".join(f"{v[1]}" for r, v in sorted(failed.items()))
            if all(v[0] == "no-context" for v in failed.values()):
                raise RankStartError(texts)
            raise RuntimeError(texts)
        handles = [got[r][1] for r in range(world)]
        for r in range(world):
            q_ins[r].put(handles)
        res = {}
        for _ in range(world):
            r, kind, payload = results.get(timeout=600)
            if kind != "ok":
                raise RuntimeError(f"rank {r}:\n{payload}")
            res[r] = payload
        [p.join(timeout=60) for p in procs]
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()                           # exactly the processes started above
                p.join(timeout=60)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    return res


def _exchange_rank(rank, world, ctx, link, V, B, nblk, seed, silent_rank, what="bank", tables=None):
    import numpy as np
    from maximilian_b200 import capi
    from maximilian_b200 import workloads as W
    p = W.voice_params(V, seed=seed)
    lo, hi = shard_range(V, rank, world)
    if what == "patch":       # the polysynth voice patch (workloads.polysynth_patch), its bus exchanged like a bank's
        capi.set_tables(*tables, ctx=ctx)
        pat = W.note_pattern(V, seed=seed)
        bank = capi.Patch(W.polysynth_patch("u8"), hi - lo, max_frames=B, ctx=ctx)
        for k, v in W.polysynth_params(V, seed=seed).items():
            bank.set(k, np.ascontiguousarray(v[lo:hi]))
    else:
        bank = capi.Bank(hi - lo, osc="saw", filt="biquad", max_frames=B, ctx=ctx)
        W.configure_bank(bank, "biquad", {k: v[lo:hi] for k, v in p.items()})
    ex = capi.Exchange(ctx, rank, world, max_doubles=2 * B)
    handles = link.handshake(ex.local_handle())
    if handles is None:
        return None
    ex.connect(handles)
    ex.attach(bank)
    if rank == silent_rank:                      # a rank that connected and then never runs its blocks
        import time
        time.sleep(3.0)
        return "silent"
    mixes, err = [], None
    try:
        for blk in range(nblk):
            if what == "patch":
                _, m = bank.process(B, {"trigger": W.note_triggers(pat, B, blk, lo, hi)}, want_out=False, want_mix=True)
            else:
                _, m = bank.process(B, want_out=False, want_mix=True)
            mixes.append(m.copy())
    except capi.MxbError as e:
        err = str(e)
    return np.stack(mixes) if mixes else None, err, ex.status()


def run_exchange_ranks(world, V, B, nblk, seed=3, silent_rank=-1, timeout_ms=None, what="bank", tables=None):
    """Spawns `world` processes, one per GPU, each owning a voice shard of a saw -> biquad bank with the peer-memory mix
    exchange attached (the IPC handles travel through multiprocessing queues; no NCCL anywhere). Returns
    {rank: (buses [nblk][B][2] | None, error text | None, exchange status mask)}. silent_rank: that rank connects and then
    never processes (the others must come back with a time-out error instead of hanging). what="patch": the polysynth voice patch instead
    of the bank (tables = (sine514, transition1001, sine_before) for its sinebuf LFO)."""
    import os
    if timeout_ms is not None:
        os.environ["MXB_EXCHANGE_TIMEOUT_MS"] = str(timeout_ms)
    try:
        return run_ranks(world, _exchange_rank, (V, B, nblk, seed, silent_rank, what, tables))
    finally:
        if timeout_ms is not None:
            os.environ.pop("MXB_EXCHANGE_TIMEOUT_MS", None)
