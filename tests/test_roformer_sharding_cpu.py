"""CPU: time-sharding of the Roformer chunk grid (b200/sharded.py `plan_start_shards`, RoformerEngine's `dist=` path).

The Roformer grid places chunks at i*step until one would run past the end of the track; every later start is clamped to N - chunk, so the
last start can repeat (mdxc_separator.py:320-341).  The planner is checked on the released grids against a brute-force restatement of its
rule, and the control flow (ShardRunner.run_units, halo isend/irecv, gather_cols) runs over gloo with the chunk outputs injected and the
ranged Hamming overlap-add with counter restated in numpy (the kernel itself is parity-tested on the GPU): the sharded result must equal the
single-process one exactly."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

SR = 44100


def roformer_starts(N, C, step):
    """RoformerEngine.chunk_starts restated."""
    return [i if i + C <= N else N - C for i in range(0, N, step)]


def ola_starts_range(chunks, starts, window, q0, q1):
    """numpy restatement of b200sep_overlap_add_starts_range: chunks (n, channels, C) at starts (global order) -> (channels, q1 - q0).
    Per output sample the contributions are added in chunk order, as the kernel does."""
    C = chunks.shape[2]
    acc = np.zeros((chunks.shape[1], q1 - q0), np.float32)
    cnt = np.zeros(q1 - q0, np.float32)
    for x, s in zip(chunks, starts):
        lo, hi = max(s, q0), min(s + C, q1)
        if hi > lo:
            acc[:, lo - q0 : hi - q0] += x[:, lo - s : hi - s] * window[lo - s : hi - s]
            cnt[lo - q0 : hi - q0] += window[lo - s : hi - s]
    return acc / np.maximum(cnt, np.float32(1e-10))


def _hamming(C):
    m = np.arange(C, dtype=np.float64)
    return (0.54 - 0.46 * np.cos(2.0 * np.pi * m / (C - 1))).astype(np.float32)


# ------------------------------------------------------------------------------------------------ planner on the released grids
GRIDS = [(n_sec * SR, hop, overlap) for n_sec in (10, 300, 600) for hop in (441, 512) for overlap in (8, 2)]


@pytest.mark.parametrize("N,hop,overlap", GRIDS)
def test_plan_start_shards_on_roformer_grids(N, hop, overlap):
    from audio_separator.separator.b200.sharded import plan_start_shards

    C = hop * (801 - 1)
    step = min(overlap * SR, C)
    starts = roformer_starts(N, C, step)
    n = len(starts)
    tail = [i for i, s in enumerate(starts) if s == N - C]
    for world in (1, 2, 4, 8):
        qs = [N * r // world for r in range(world + 1)]
        owner = [next(r for r in range(world) if qs[r] <= min(s, N - 1) < qs[r + 1]) for s in starts]
        need = [[i for i, s in enumerate(starts) if s < qs[r + 1] and s + C > qs[r]] for r in range(world)]
        too_short = any(owner[i] < r - 1 for r in range(world) for i in need[r])
        if too_short:  # a halo would need units from more than one neighbour
            with pytest.raises(ValueError, match="track too short"):
                plan_start_shards(starts, C, N, world)
            continue
        sh = plan_start_shards(starts, C, N, world)
        assert [(s.q0, s.q1) for s in sh] == list(zip(qs, qs[1:]))  # contiguous, disjoint, covering [0, N)
        assert sh[0].c0 == 0 and sh[-1].c1 == n and all(a.c1 == b.c0 for a, b in zip(sh, sh[1:]))
        for r, s in enumerate(sh):
            assert list(range(s.c0, s.c1)) == [i for i in range(n) if owner[i] == r]  # a unit belongs to the rank holding its start
            assert need[r] and s.c0 - s.halo <= need[r][0] and need[r][-1] < s.c1  # every unit covering the range is local
            assert s.halo == sum(1 for i in range(s.c0) if starts[i] + C > s.q0) if r else s.halo == 0  # the left neighbour's units that reach in
        assert all(a.send == b.halo for a, b in zip(sh, sh[1:])) and sh[-1].send == 0
        assert len({next(r for r, s in enumerate(sh) if s.c0 <= i < s.c1) for i in tail}) == 1  # repeated tail starts on one rank
    if N == 10 * SR and overlap == 2:
        assert len(tail) > 1  # the grid does exercise repeated starts


def test_plan_start_shards_rejects_short_tracks_and_bad_grids():
    from audio_separator.separator.b200.sharded import plan_start_shards

    C = 441 * 800
    starts = roformer_starts(10 * SR, C, 2 * SR)
    plan_start_shards(starts, C, 10 * SR, 1)
    with pytest.raises(ValueError, match="track too short"):
        plan_start_shards(starts, C, 10 * SR, 8)  # ranges of 55 125 samples, chunks of 352 800
    with pytest.raises(ValueError):
        plan_start_shards([], C, 10 * SR, 2)
    with pytest.raises(ValueError):
        plan_start_shards([0, 100, 50], 200, 400, 2)


# ------------------------------------------------------------------------------------------------ control flow over gloo
# (N, chunk, step): step < chunk with three starts clamped to N - chunk; step == chunk (only the tail chunk overlaps); an odd-sized grid
SMALL_GRIDS = [(1000, 64, 24), (1000, 64, 64), (1234, 100, 30)]


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from audio_separator.separator.b200.sharded import ShardRunner, plan_start_shards

    runner = ShardRunner(dist)
    diffs = []
    for gi, (N, C, step) in enumerate(SMALL_GRIDS):
        channels = 4  # two stems x stereo
        starts = roformer_starts(N, C, step)
        units = np.random.default_rng(10 + gi).standard_normal((len(starts), channels, C)).astype(np.float32)
        win = _hamming(C)
        shards = plan_start_shards(starts, C, N, world)
        sh = shards[rank]
        local = torch.zeros((sh.halo + sh.n_own, channels, C))
        order = []

        def compute(buf, slot0, unit0, n):  # stands in for the batched Roformer forward of the chunks [unit0, unit0 + n)
            order.append((unit0, n))
            buf[slot0 : slot0 + n] = torch.from_numpy(units[unit0 : unit0 + n])

        runner.wait_all(runner.run_units(sh, local, compute, max_batch=3))
        assert sorted(u for u0, n in order for u in range(u0, u0 + n)) == list(range(sh.c0, sh.c1))  # every own chunk exactly once
        if sh.send and rank + 1 < world:  # the batches holding the chunks the right neighbour needs ran first
            touches = [u0 + n > sh.c1 - sh.send for u0, n in order]
            assert touches[0] and touches == sorted(touches, reverse=True), (order, sh)
        first = sh.c0 - sh.halo
        part = ola_starts_range(local.numpy(), starts[first : sh.c1], win, sh.q0, sh.q1)
        full = runner.gather_cols(torch.from_numpy(part), [(s.q0, s.q1) for s in shards], N)
        if rank == 0:
            ref = ola_starts_range(units, starts, win, 0, N)
            diffs.append(float(np.abs(full.numpy() - ref).max()))
    if rank == 0:
        q.put(diffs)
    dist.barrier()
    dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.parametrize("world", [2, 3])
def test_roformer_sharded_overlap_add_is_exact(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(180)
    codes = [p.exitcode for p in procs]
    for p in procs:  # a rank that died leaves its peers waiting: do not leave them behind
        if p.is_alive():
            p.kill()
    assert codes == [0] * world, codes
    assert q.get(timeout=5) == [0.0] * len(SMALL_GRIDS)  # same contributions in the same order per output sample


def test_roformer_grid_halo_is_real():
    """The gloo grids exchange chunks: with step < chunk every rank past the first receives a halo."""
    from audio_separator.separator.b200.sharded import plan_start_shards

    N, C, step = SMALL_GRIDS[0]
    starts = roformer_starts(N, C, step)
    assert starts.count(N - C) == 3
    for world in (2, 3):
        sh = plan_start_shards(starts, C, N, world)
        assert all(s.halo >= 2 for s in sh[1:])
