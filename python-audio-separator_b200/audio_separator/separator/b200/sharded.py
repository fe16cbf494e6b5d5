"""Time-sharding of ONE track across the GPUs of a box (BASELINE north_star: "chunks shard by time across the 8 GPUs
with overlap-region halo exchange via NCCL").

The reference has no multi-GPU path (SURVEY.md section 2.1); this is new.  All three chunked architectures have the same
structure (SURVEY.md section 8e): independent units (MDX chunks, mdx_separator.py:335-348; MDX23C chunks, mdxc_separator.py:361-402;
Demucs segments, demucs/apply.py:215-250) placed every `stride` samples, coupled only by the overlap-add.  The Roformer chunks
(mdxc_separator.py:320-341) are placed every `step` samples until one would run past the end, and every later start is clamped to N - chunk.
Two planning rules:

* `plan_shards`        -- MDX: contiguous chunk ranges, rank r finalises the padded positions [c0*step, c1*step).
* `plan_start_shards`  -- Roformer (explicit start list), and through `plan_range_shards` MDX23C / Demucs (regular grid): rank r finalises
                          a fixed range [q0, q1) of OUTPUT samples (the same for every pass of a Demucs bag / shift loop, so the
                          accumulation order per sample is the single-GPU order and the result is bit-identical); a unit belongs to
                          the rank its first output sample falls in.
* `plan_patch_shards`  -- VR: the patches do not overlap (the 128-frame crop of every prediction), so rank r owns a contiguous run of the single-GPU
                          loop's forwards, finalises their mask columns and needs no halo (`shard_patches`).
In the first two, a rank needs the trailing units of its LEFT neighbour that reach into its range: one `isend`/`irecv` pair between
time-neighbours (NCCL p2p over NVLink), posted as soon as those units are computed so the transfer overlaps the remaining forwards.
The finalised slices go to rank 0 with point-to-point receives straight into the full-size stem buffers, or -- end-to-end entry points --
every rank copies its own slice into a host buffer shared between the ranks (8 PCIe links in parallel, no gather at all).

This module is pure host logic: the planners and `ShardRunner` (the control flow: unit order, halo exchange, gather) import only the
standard library and torch, and run unchanged on CPU tensors with gloo (tests/test_sharding_cpu.py injects the compute).  The engines that
use them (MdxEngine, MdxcEngine in engine.py; RoformerEngine, DemucsEngine, VREngine) supply the CUDA compute and overlap-add; a single GPU
is a world of size 1 through the same code.
"""
from __future__ import annotations

from bisect import bisect_left, bisect_right
from dataclasses import dataclass

import torch


@dataclass
class Shard:
    rank: int
    c0: int  # first own unit (chunk / segment)
    c1: int  # one past the last own unit
    halo: int  # units received from the left neighbour: [c0 - halo, c0)
    q0: int  # first output sample (unpadded coordinates) this rank finalises
    q1: int  # one past the last
    send: int = 0  # own trailing units the right neighbour needs: [c1 - send, c1)

    @property
    def n_own(self):
        return self.c1 - self.c0


def plan_shards(n_samples: int, total_len: int, step: int, chunk: int, trim: int, n_chunks: int, world: int) -> list[Shard]:
    """MDX.  Contiguous, balanced chunk ranges; rank r finalises the padded positions [c0*step, c1*step) (last rank: to the end)."""
    k = -(-chunk // step) - 1  # chunks of the left neighbour that reach into a rank's range
    base, rem = divmod(n_chunks, world)
    shards, c0 = [], 0
    for r in range(world):
        c1 = c0 + base + (1 if r < rem else 0)
        p0 = c0 * step
        p1 = total_len if r == world - 1 else c1 * step
        q0 = min(max(p0 - trim, 0), n_samples)
        q1 = min(max(p1 - trim, 0), n_samples)
        halo = min(k, c0) if c1 > c0 else 0
        shards.append(Shard(r, c0, c1, halo, q0, q1))
        c0 = c1
    for s in shards[1:]:
        left = shards[s.rank - 1]
        if s.halo > left.c1 - left.c0 and s.c1 > s.c0:
            raise ValueError(f"track too short to shard over {world} ranks: rank {s.rank} needs {s.halo} halo chunks, its neighbour owns {left.c1 - left.c0}")
        left.send = s.halo
    return shards


def plan_start_shards(starts, unit_len: int, n_out: int, world: int) -> list[Shard]:
    """Units at explicit, nondecreasing output positions: unit i covers the output samples [starts[i], starts[i] + unit_len).  Rank r finalises
    the output samples [n_out*r/world, n_out*(r+1)/world) and owns the units whose start lies in that range (starts before 0 go to rank 0, starts
    at or past n_out to the last rank), so repeated starts -- the Roformer grid clamps every tail chunk to n_out - unit_len -- land on one rank.
    Its halo is the run of its left neighbour's units that reach into the range."""
    n_units = len(starts)
    if n_units < 1 or unit_len < 1 or any(b < a for a, b in zip(starts, starts[1:])):
        raise ValueError("plan_start_shards: bad grid (no units, or starts not nondecreasing)")
    qs = [n_out * r // world for r in range(world + 1)]
    u0 = [0] + [bisect_left(starts, qs[r]) for r in range(1, world)] + [n_units]
    shards = []
    for r in range(world):
        need_lo = 0 if r == 0 else bisect_right(starts, qs[r] - unit_len)  # first unit that ends past q0
        c0, c1 = u0[r], u0[r + 1]
        halo = max(0, c0 - need_lo) if qs[r + 1] > qs[r] else 0
        if r > 0 and halo > 0 and c0 - halo < u0[r - 1]:
            raise ValueError(f"track too short to shard over {world} ranks: rank {r} needs units from {c0 - halo}, its left neighbour owns [{u0[r - 1]}, {c0})")
        shards.append(Shard(r, c0, c1, halo, qs[r], qs[r + 1]))
    for s in shards[1:]:
        shards[s.rank - 1].send = s.halo
    return shards


def plan_range_shards(n_out: int, world: int, n_units: int, stride: int, unit_len: int, base: int) -> list[Shard]:
    """MDX23C / Demucs: `plan_start_shards` on the regular grid, unit i covering the output samples [i*stride - base, i*stride - base + unit_len)."""
    if n_units < 1 or stride < 1 or unit_len < 1:
        raise ValueError("plan_range_shards: bad grid")
    return plan_start_shards(range(-base, n_units * stride - base, stride), unit_len, n_out, world)


def plan_patch_shards(n_patches: int, world: int, roi: int = 1, batch: int = 1) -> list[Shard]:
    """VR: patch p reads only its own input window and writes only the mask columns [p*roi, (p+1)*roi), so there is no halo and no overlap-add.
    The patches run in forwards of `batch` (the last one holds the remainder); rank r owns the contiguous forwards [G*r/W, G*(r+1)/W) of the
    G = ceil(n_patches / batch) of the single-GPU loop, i.e. the patches [c0, c1), and finalises the mask columns [c0*roi, c1*roi).  Every patch is then
    predicted in the same forward, at the same batch slot, as on one GPU.  With batch 1 that is [P*r/W, P*(r+1)/W); ranks may be empty."""
    if n_patches < 0 or world < 1 or roi < 1 or batch < 1:
        raise ValueError("plan_patch_shards: bad arguments")
    groups = -(-n_patches // batch)
    shards = []
    for r in range(world):
        c0, c1 = (min(groups * q // world * batch, n_patches) for q in (r, r + 1))
        shards.append(Shard(r, c0, c1, 0, c0 * roi, c1 * roi))
    return shards


def shard_patches(runner: "ShardRunner", n_patches: int, roi: int, batch: int, predict):
    """The VR patch loop over the ranks: predict(p0, p1) -> this rank's mask columns (..., (p1 - p0) * roi) of the patches [p0, p1), run in
    forwards of `batch` starting at p0.  Returns the full (..., n_patches * roi) mask on rank 0 (gather_cols), None on the other ranks."""
    shards = plan_patch_shards(n_patches, runner.world, roi, batch)
    sh = shards[runner.rank]
    return runner.gather_cols(predict(sh.c0, sh.c1), [(s.q0, s.q1) for s in shards], n_patches * roi)


def balanced_batches(n: int, max_batch: int) -> list[int]:
    """n units as ceil(n / max_batch) batches of nearly equal size (9 at max 4 -> 3+3+3, not 4+4+1: a 1-unit forward costs almost as much as a full one)."""
    if n <= 0:
        return []
    k = -(-n // max_batch)
    return [n // k + (1 if i < n % k else 0) for i in range(k)]


class ShardRunner:
    """The control flow shared by the sharded engines, over torch.distributed (nccl on the GPUs, gloo in the CPU tests).

    compute(local, slot0, unit0, n): fill local[slot0 : slot0 + n] with the outputs of the global units [unit0, unit0 + n).
    """

    def __init__(self, dist, group=None):
        self.dist, self.group = dist, group
        self.rank = dist.get_rank(group) if dist is not None else 0
        self.world = dist.get_world_size(group) if dist is not None else 1

    def _peer(self, r):
        return r if self.group is None else self.dist.get_global_rank(self.group, r)

    def out_range(self, n: int, rank: int | None = None):
        """The output samples [n*r/W, n*(r+1)/W) rank r (default: this rank) finalises in the even partition of n."""
        r = self.rank if rank is None else rank
        return n * r // self.world, n * (r + 1) // self.world

    def run_units(self, sh: Shard, local: torch.Tensor, compute, max_batch: int):
        """Own units into local[halo:] in balanced batches; the batches holding the trailing `send` units run FIRST and the p2p pair is posted
        right after them, so the transfer to the right neighbour overlaps the remaining forwards.  Returns the outstanding requests
        (wait_all before the overlap-add)."""
        n_own = sh.n_own
        assert local.shape[0] == sh.halo + n_own
        spans, u = [], sh.c0
        for b in balanced_batches(n_own, max_batch):
            spans.append((u, b))
            u += b
        send = min(sh.send, n_own) if self.rank + 1 < self.world else 0
        head = [sp for sp in spans if sp[0] + sp[1] > sh.c1 - send] if send else []
        rest = [sp for sp in spans if sp not in head]
        reqs, posted = [], False
        for unit0, n in head:
            compute(local, sh.halo + unit0 - sh.c0, unit0, n)
        if head or sh.halo:
            reqs += self._post(sh, local)
            posted = True
        for unit0, n in rest:
            compute(local, sh.halo + unit0 - sh.c0, unit0, n)
        assert posted or (sh.halo == 0 and send == 0)
        return reqs

    def _post(self, sh: Shard, local: torch.Tensor):
        dist = self.dist
        if dist is None or self.world == 1:
            return []
        ops = []
        n = local.shape[0]
        if sh.send > 0 and self.rank + 1 < self.world:
            ops.append(dist.P2POp(dist.isend, local[n - sh.send : n], self._peer(self.rank + 1), self.group))
        if sh.halo > 0:
            ops.append(dist.P2POp(dist.irecv, local[: sh.halo], self._peer(self.rank - 1), self.group))
        return list(dist.batch_isend_irecv(ops)) if ops else []

    @staticmethod
    def wait_all(reqs):
        for r in reqs:
            r.wait()

    def gather_rows(self, bufs, shards, dim=0):
        """Rank 0 receives every other rank's finalised slice [q0, q1) along `dim` straight into its full-size buffers."""
        dist = self.dist
        if dist is None or self.world == 1:
            return
        ops = []
        me = shards[self.rank]
        if self.rank == 0:
            for s in shards[1:]:
                if s.q1 > s.q0:
                    for buf in bufs:
                        ops.append(dist.P2POp(dist.irecv, buf.narrow(dim, s.q0, s.q1 - s.q0), self._peer(s.rank), self.group))
        elif me.q1 > me.q0:
            for buf in bufs:
                ops.append(dist.P2POp(dist.isend, buf.narrow(dim, me.q0, me.q1 - me.q0), self._peer(0), self.group))
        if ops:
            for req in dist.batch_isend_irecv(ops):
                req.wait()


    def gather_cols(self, part: torch.Tensor, ranges, n_total: int):
        """part (..., q1 - q0) on every rank -> the full (..., n_total) tensor on rank 0 (None elsewhere).  Slices along the LAST axis are not
        contiguous in the destination, so rank 0 receives into per-rank staging tensors and copies them in place.  In a world of 1, `part` is
        returned as it is."""
        if self.world == 1:
            return part
        dist = self.dist
        part = part.contiguous()
        if self.rank != 0:
            if part.numel():
                dist.batch_isend_irecv([dist.P2POp(dist.isend, part, self._peer(0), self.group)])[0].wait()
            return None
        full = torch.empty(part.shape[:-1] + (n_total,), dtype=part.dtype, device=part.device)
        full[..., ranges[0][0] : ranges[0][1]] = part
        stage, ops = [], []
        for r in range(1, self.world):
            q0, q1 = ranges[r]
            if q1 > q0:
                t = torch.empty(part.shape[:-1] + (q1 - q0,), dtype=part.dtype, device=part.device)
                stage.append((q0, q1, t))
                ops.append(dist.P2POp(dist.irecv, t, self._peer(r), self.group))
        if ops:
            for req in dist.batch_isend_irecv(ops):
                req.wait()
        for q0, q1, t in stage:
            full[..., q0:q1] = t
        return full

    def gather(self, part: torch.Tensor, n: int):
        """gather_cols over the even partition of n (out_range): every rank's (..., q1 - q0) slice -> the full (..., n) tensor on rank 0."""
        return self.gather_cols(part, [self.out_range(n, r) for r in range(self.world)], n)
