"""CPU: splitting the VR patches of one track over ranks (b200/sharded.py `plan_patch_shards`, `shard_patches`; VREngine's `dist=` path).

A VR patch reads its own input window of `window` frames and writes only the `roi` mask columns left after the 2*offset crop, so the ranks need no
halo.  The planner is checked for ownership, contiguity, balance and empty ranks, and for running every patch in the same forward (same batch size,
same slot) as the single-GPU loop.  The protocol runs over gloo at world sizes 2 and 3 with a deterministic predict_mask injected; the injected
prediction also depends on the batch size and the slot of each patch, so a rank that batched its patches differently from one GPU would be
caught.  The gathered mask, with and without test-time augmentation, must equal the single-process mask exactly."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def single_gpu_forwards(n_patches, batch):
    """The forwards of VREngine's patch loop on one GPU: [i, i + batch) from 0, the last one holding the remainder."""
    return [(i, min(batch, n_patches - i)) for i in range(0, n_patches, batch)]


@pytest.mark.parametrize("batch", [1, 2, 3, 4])
def test_plan_patch_shards_properties(batch):
    from audio_separator.separator.b200.sharded import plan_patch_shards

    roi = 256
    for n_patches in (0, 1, 2, 3, 5, 7, 8, 17, 65, 66, 130):
        fwd = single_gpu_forwards(n_patches, batch)
        for world in (1, 2, 3, 4, 8):
            sh = plan_patch_shards(n_patches, world, roi, batch)
            assert [s.rank for s in sh] == list(range(world))
            assert sh[0].c0 == 0 and sh[-1].c1 == n_patches and all(a.c1 == b.c0 for a, b in zip(sh, sh[1:]))  # contiguous, covering
            owners = [r for r, s in enumerate(sh) for _ in range(s.c0, s.c1)]
            assert len(owners) == n_patches  # every patch owned exactly once
            assert all((s.q0, s.q1) == (s.c0 * roi, s.c1 * roi) and s.halo == 0 and s.send == 0 for s in sh)
            # a rank's forwards are forwards of the single-GPU loop, and the ranks' forward counts differ by at most one
            per_rank = [[f for f in fwd if s.c0 <= f[0] < s.c1] for s in sh]
            assert all(sum(n for _, n in fr) == s.n_own and all(f[0] + f[1] <= s.c1 for f in fr) for fr, s in zip(per_rank, sh))
            counts = [len(fr) for fr in per_rank]
            assert max(counts) - min(counts) <= 1
            if batch == 1:
                assert [(s.c0, s.c1) for s in sh] == [(n_patches * r // world, n_patches * (r + 1) // world) for r in range(world)]
            if n_patches < world:
                assert sum(1 for s in sh if s.n_own == 0) >= world - n_patches  # empty ranks exist and are legal
    with pytest.raises(ValueError):
        plan_patch_shards(5, 0)
    with pytest.raises(ValueError):
        plan_patch_shards(5, 2, roi=0)


# ------------------------------------------------------------------------------------------------ protocol over gloo
# (n_frame, window, offset, batch): roi = window - 2*offset; several patches per rank; fewer patches than ranks; the VR 5.1 offset
CASES = [(1000, 64, 16, 3), (333, 48, 8, 1), (40, 64, 16, 4), (700, 40, 8, 2)]
NB = 9


def fake_predict(windows, off):
    """Stands in for VRNet.predict_mask: (b, 2, nb, window) -> (b, 2, nb, roi).  Deterministic, depends on the whole window, and on the batch size
    and the slot of each patch (as a kernel whose tiling depends on the batch could)."""
    b, _, _, w = windows.shape
    mean = windows.mean(dim=-1, keepdim=True)
    slot = torch.arange(b, dtype=windows.dtype).view(b, 1, 1, 1)
    return torch.tanh(windows[..., off : w - off] * 1.5 + mean) + 1e-3 * (b + 7 * slot)


def patch_mask(mag, roi, window, batch, p0, p1):
    """The patch loop of VREngine._predict restated: the patches [p0, p1) in forwards of `batch` from p0 -> (2, nb, (p1 - p0) * roi)."""
    nb = mag.shape[1]
    out = torch.empty((2, nb, p1 - p0, roi))
    for i in range(p0, p1, batch):
        b = min(batch, p1 - i)
        win = torch.stack([mag[:, :, (i + j) * roi : (i + j) * roi + window] for j in range(b)])
        out[:, :, i - p0 : i - p0 + b] = fake_predict(win, (window - roi) // 2).permute(1, 2, 0, 3)
    return out.reshape(2, nb, (p1 - p0) * roi)


def padded_mag(spec_mag, pad_l, pad_r):
    m = torch.nn.functional.pad(spec_mag, (pad_l, pad_r))
    return m / m.max()


def masks(spec_mag, window, offset, batch, tta, runner=None):
    """VREngine.masks restated on CPU tensors; with `runner` the patches go through shard_patches (None on the ranks other than 0)."""
    from audio_separator.separator.b200.sharded import shard_patches

    n_frame = spec_mag.shape[2]
    roi = window - 2 * offset
    pad_l, pad_r = offset, roi - n_frame % roi + offset
    out = []
    for extra in ((0, roi // 2) if tta else (0,)):
        mag = padded_mag(spec_mag, pad_l + extra, pad_r + extra)
        patches = (mag.shape[2] - 2 * offset) // roi
        if runner is None:
            out.append(patch_mask(mag, roi, window, batch, 0, patches))
        else:
            out.append(shard_patches(runner, patches, roi, batch, lambda p0, p1: patch_mask(mag, roi, window, batch, p0, p1)))
    if out[0] is None:
        assert all(m is None for m in out)
        return None
    if tta:
        return out, out[0][..., :n_frame] * 0.5 + out[1][..., roi // 2 : roi // 2 + n_frame] * 0.5
    return out, out[0]


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from audio_separator.separator.b200.sharded import ShardRunner

    runner = ShardRunner(dist)
    res = []
    for ci, (n_frame, window, offset, batch) in enumerate(CASES):
        spec_mag = torch.from_numpy(np.abs(np.random.default_rng(40 + ci).standard_normal((2, NB, n_frame))).astype(np.float32))
        for tta in (False, True):
            got = masks(spec_mag, window, offset, batch, tta, runner)
            if rank != 0:
                assert got is None
                continue
            ref = masks(spec_mag, window, offset, batch, tta)
            (passes, avg), (ref_passes, ref_avg) = got, ref
            same = all(torch.equal(a, b) for a, b in zip(passes, ref_passes)) and torch.equal(avg, ref_avg)
            res.append((ci, tta, same, avg.shape[-1] >= n_frame))
    if rank == 0:
        q.put(res)
    dist.barrier()
    dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.parametrize("world", [2, 3])
def test_vr_sharded_masks_equal_single_process(world):
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
    res = q.get(timeout=5)
    assert len(res) == 2 * len(CASES)
    for ci, tta, same, covers in res:
        assert same and covers, (CASES[ci], tta)


def test_fake_predict_sees_the_batching():
    """The injected prediction is not batch-invariant, so the gloo test above does check that the ranks batch like one GPU."""
    mag = padded_mag(torch.rand((2, NB, 300)), 16, 40)
    roi = 32
    whole = patch_mask(mag, roi, 64, 3, 0, 9)
    shifted = torch.cat([patch_mask(mag, roi, 64, 3, 0, 4), patch_mask(mag, roi, 64, 3, 4, 9)], dim=-1)  # a split inside a forward
    assert not torch.equal(whole, shifted)
