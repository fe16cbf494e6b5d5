"""CPU (gloo, world_size 2 and 3): the time-sharding control flow of audio_separator/separator/b200/sharded.py.

The chunked engines (MdxEngine, MdxcEngine, DemucsEngine) all run `ShardRunner.run_units` (unit order, balanced batches, halo
isend/irecv), an overlap-add of their own output range, and `gather_rows` / `gather_cols`.  These tests execute exactly that code over gloo
with the per-unit compute and the range overlap-add injected as numpy restatements of the kernels (the kernels themselves are parity-tested
on the GPU): the sharded result must equal the single-process oracle sample for sample."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import mdx_oracle as O

SMALL = dict(n_fft=1536, hop_length=256, dim_f=768, dim_t=32, segment_size=32, g=8)


def ola_range(local, first_chunk, n_chunks, chunk, step, L, trim, N, q0, q1, use_window):
    """numpy restatement of b200sep_demix_overlap_add_range (gather form of mdx_separator.py:348-401)."""
    out = np.zeros((q1 - q0, 2), np.float32)
    for q in range(q0, q1):
        p = q + trim
        i_lo = 0 if p - chunk + 1 <= 0 else (p - chunk + step) // step
        i_hi = min(p // step, n_chunks - 1)
        res, div = np.zeros(2, np.float32), np.float32(0)
        for i in range(i_lo, i_hi + 1):
            s, e = i * step, min(i * step + chunk, L)
            if p >= e:
                continue
            w = np.float32(np.hanning(e - s)[p - s]) if use_window else np.float32(1)
            res += local[i - first_chunk][:, p - s] * w
            div += w
        out[q - q0] = res / div
    return out


def _mdx_worker(rank, world, port, n_samples, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from audio_separator.separator.b200.sharded import ShardRunner, plan_shards

    cfg = O.MDXConfig(**SMALL)
    mix = O.normalize(O.synth_music(n_samples, seed=5), 0.9, 0.0)
    L, step, starts = O.chunk_starts(n_samples, cfg)
    n_chunks, T = len(starts), cfg.chunk_size
    shards = plan_shards(n_samples, L, step, T, cfg.trim, n_chunks, world)
    sh = shards[rank]
    mixture = np.zeros((2, L), np.float32)
    mixture[:, cfg.trim : cfg.trim + n_samples] = mix
    order = []

    def compute(buf, slot0, unit0, n):  # stands in for b200sep_mdx_run_model on the chunks [unit0, unit0 + n)
        order.append((unit0, n))
        for j in range(n):
            c = unit0 + j
            part = np.zeros((1, 2, T), np.float32)
            e = min(c * step + T, L)
            part[0, :, : e - c * step] = mixture[:, c * step : e]
            buf[slot0 + j] = torch.from_numpy(O.run_model(part, cfg, lambda s: s * 0.5)[0])

    runner = ShardRunner(dist)
    local = torch.zeros((sh.halo + sh.n_own, 2, T))
    runner.wait_all(runner.run_units(sh, local, compute, max_batch=2))
    assert sorted(u for u0, n in order for u in range(u0, u0 + n)) == list(range(sh.c0, sh.c1))  # every own chunk exactly once
    if sh.send and rank + 1 < world:
        assert order[0][0] + order[0][1] == sh.c1  # the batch holding the trailing chunks ran first (its transfer overlaps the rest)
    full = torch.zeros((n_samples, 2))
    if sh.q1 > sh.q0:
        full[sh.q0 : sh.q1] = torch.from_numpy(ola_range(local.numpy(), sh.c0 - sh.halo, n_chunks, T, step, L, cfg.trim, n_samples, sh.q0, sh.q1, True))
    runner.gather_rows([full], shards, dim=0)
    if rank == 0:
        ref = O.demix(mix, cfg, lambda s: s * 0.5)
        q.put(float(np.abs(full.numpy().T - ref).max()))
    dist.barrier()
    dist.destroy_process_group()


def _range_worker(rank, world, port, kind, q):
    """MDX23C (rectangular, `overlap` chunks per sample) and Demucs (triangle weights, offset grid of the shift trick) on plan_range_shards."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from audio_separator.separator.b200.sharded import ShardRunner, plan_range_shards

    rng = np.random.default_rng(3)
    C = 3
    if kind == "rect":  # mdxc_separator.py:361-402 with chunk 64, overlap 4
        T, stride, N = 64, 16, 1000
        pad = stride - (N - T) % stride
        base = T - stride
        n_units = (base + N + pad + base - T) // stride + 1
        passes = [(base, 1.0)]
    else:  # apply.py:197-250: two shifted passes, segment 90, stride 67
        T, stride, N, ms = 90, 67, 1500, 40
        passes = [(ms - o, 0.5) for o in (13, 31)]
    units_of = {}
    for base, _ in passes:
        length = N + base if kind == "tri" else None
        n_units_p = len(range(0, length, stride)) if kind == "tri" else n_units
        units_of[base] = rng.standard_normal((n_units_p, C, T)).astype(np.float32)

    def weight(n):
        if kind == "rect":
            return np.float32(1)
        wmax = np.float32(max(T - T // 2, T // 2))
        return np.float32((n + 1) if n < T // 2 else (T - n)) / wmax

    def ola(units, first, n_units_p, base, q0, q1, acc):  # gather form, units[0] is global unit `first`
        for qo in range(q0, q1):
            p = qo + base
            i_lo = 0 if p - T + 1 <= 0 else (p - T + stride) // stride
            i_hi = min(p // stride, n_units_p - 1)
            a, sw = np.zeros(C, np.float32), np.float32(0)
            for i in range(i_lo, i_hi + 1):
                w = weight(p - i * stride)
                a += w * units[i - first][:, p - i * stride]
                sw += w
            acc[:, qo - q0] += a / (sw if kind == "tri" else np.float32(4))

    runner = ShardRunner(dist)
    r0, r1 = N * rank // world, N * (rank + 1) // world
    mine = np.zeros((C, r1 - r0), np.float32)
    for base, scale in passes:
        units = units_of[base]
        sh = plan_range_shards(N, world, len(units), stride, T, base)[rank]
        assert (sh.q0, sh.q1) == (r0, r1)
        local = torch.zeros((sh.halo + sh.n_own, C, T))

        def compute(buf, slot0, unit0, n):
            buf[slot0 : slot0 + n] = torch.from_numpy(units[unit0 : unit0 + n])

        runner.wait_all(runner.run_units(sh, local, compute, max_batch=3))
        part = np.zeros_like(mine)
        ola(local.numpy(), sh.c0 - sh.halo, len(units), base, sh.q0, sh.q1, part)
        mine += np.float32(scale) * part
    full = runner.gather_cols(torch.from_numpy(mine), [(N * r // world, N * (r + 1) // world) for r in range(world)], N)
    if rank == 0:
        ref = np.zeros((C, N), np.float32)
        for base, scale in passes:
            part = np.zeros((C, N), np.float32)
            ola(units_of[base], 0, len(units_of[base]), base, 0, N, part)
            ref += np.float32(scale) * part
        q.put(float(np.abs(full.numpy() - ref).max()))
    dist.barrier()
    dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _spawn(target, world, *args):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port) + args + (q,)) for r in range(world)]
    for p_ in procs:
        p_.start()
    for p_ in procs:
        p_.join(180)
        assert p_.exitcode == 0
    return q.get(timeout=5)


@pytest.mark.parametrize("world,n_samples", [(2, 30000), (3, 52345)])
def test_time_sharded_demix_matches_single_process(world, n_samples):
    assert _spawn(_mdx_worker, world, n_samples) <= 2e-6


@pytest.mark.parametrize("world,kind", [(2, "rect"), (3, "rect"), (2, "tri"), (3, "tri")])
def test_range_sharded_overlap_add_is_exact(world, kind):
    assert _spawn(_range_worker, world, kind) == 0.0  # same contributions in the same order per output sample


def test_plan_shards_properties():
    from audio_separator.separator.b200.sharded import plan_shards

    cfg = O.MDXConfig()
    N = 13_230_000
    L, step, starts = O.chunk_starts(N, cfg)
    for world in (1, 2, 4, 8):
        sh = plan_shards(N, L, step, cfg.chunk_size, cfg.trim, len(starts), world)
        assert sh[0].c0 == 0 and sh[-1].c1 == 68 and sh[0].q0 == 0 and sh[-1].q1 == N
        assert all(a.c1 == b.c0 and a.q1 == b.q0 for a, b in zip(sh, sh[1:]))  # contiguous, disjoint
        assert max(s.c1 - s.c0 for s in sh) - min(s.c1 - s.c0 for s in sh) <= 1  # balanced
        assert [s.halo for s in sh] == [0] + [1] * (world - 1)  # overlap 0.25 -> one chunk of halo
        assert [s.send for s in sh] == [1] * (world - 1) + [0]
    with pytest.raises(ValueError):
        plan_shards(1000, 3000, 100, 950, 10, 3, 3)  # 9 halo chunks needed, neighbours own 1


def test_plan_range_shards_properties():
    from audio_separator.separator.b200.sharded import balanced_batches, plan_range_shards

    # MDX23C, BASELINE config 4: 10-min track, chunk 261120, overlap 8 -> 818 chunks; every sample is covered by 8 chunks, so up to 8 chunks (7 when the boundary sits on the hop grid) of halo
    N, T, hop = 26_460_000, 261120, 32640
    front = T - hop
    pad = hop - (N - T) % hop
    n_chunks = (front + N + pad + front - T) // hop + 1
    assert n_chunks == 818
    # htdemucs_ft, config 3: segment 343980, stride 257985 on the shifted grid of one pass
    for (n_units, stride, ulen, base, halo_max) in ((n_chunks, hop, T, front, 8), (len(range(0, 13_230_000 + 22050 - 777, 257985)), 257985, 343980, 22050 - 777, 2)):
        n_out = N if stride == hop else 13_230_000
        for world in (1, 2, 4, 8):
            sh = plan_range_shards(n_out, world, n_units, stride, ulen, base)
            assert sh[0].c0 == 0 and sh[-1].c1 == n_units and sh[0].q0 == 0 and sh[-1].q1 == n_out
            assert all(a.c1 == b.c0 and a.q1 == b.q0 for a, b in zip(sh, sh[1:]))
            assert sh[0].halo == 0 and all(1 <= s.halo <= halo_max for s in sh[1:]) and all(a.send == b.halo for a, b in zip(sh, sh[1:]))
            for s in sh:  # every unit covering [q0, q1) is local
                need_lo = max(0, (s.q0 + base - ulen) // stride + 1)
                need_hi = min((s.q1 - 1 + base) // stride, n_units - 1)
                assert s.c0 - s.halo <= need_lo and need_hi < s.c1
            assert max(s.n_own for s in sh) - min(s.n_own for s in sh) <= (8 if stride == hop else 1) + 1
    with pytest.raises(ValueError):
        plan_range_shards(1000, 8, 40, 25, 400, 0)  # ranges of 125 samples, units of 400: a halo would span several ranks
    assert balanced_batches(9, 4) == [3, 3, 3] and balanced_batches(8, 4) == [4, 4] and balanced_batches(0, 4) == [] and sum(balanced_batches(52, 8)) == 52
