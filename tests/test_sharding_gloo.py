"""CPU-only, world_size 2 over gloo: the host-side logic of the disparity-sharded path --
shard ranges and the packed-key exchange whose min reproduces the reference's WTA tie-break.
The key packing below emulates, in numpy, what wta_kernel<T, false> emits on the device."""
import os

import numpy as np
import pytest

from primestereomatch_b200.sharding import shard_range


def order_key(c):
    c = (c + np.float32(0.0)).astype(np.float32)  # -0 -> +0
    u = c.view(np.uint32).astype(np.uint64)
    neg = (u & np.uint64(0x80000000)) != 0
    return np.where(neg, (~u) & np.uint64(0xFFFFFFFF), u | np.uint64(0x80000000))


def local_keys(vol, d_begin):
    """strict-< scan over the owned slices, global d = 0 excluded, (+inf, 0) when nothing selected."""
    D, H, W = vol.shape
    mc = np.full((H, W), np.inf, np.float32)
    md = np.zeros((H, W), np.uint64)
    for dl in range(D):
        d = d_begin + dl
        if d == 0:
            continue
        better = vol[dl] < mc
        mc = np.where(better, vol[dl], mc)
        md = np.where(better, np.uint64(d), md)
    return (order_key(mc) << np.uint64(32)) | md


def test_shard_ranges_cover_and_partition():
    for D in (2, 7, 64, 128, 256):
        for world in (1, 2, 3, 4, 8):
            if world > D:
                with pytest.raises(ValueError):
                    shard_range(D, world, 0)
                continue
            got = []
            for r in range(world):
                b, n = shard_range(D, world, r)
                assert n >= 1
                got += list(range(b, b + n))
            assert got == list(range(D))


def _worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rng = np.random.default_rng(123)  # same volume on every rank; each uses its own shard
    D, H, W = 13, 24, 40
    vol = rng.normal(0, 1, (D, H, W)).astype(np.float32)
    vol[3, :, :8] = vol[9, :, :8]          # cross-shard exact tie -> lowest d must win
    vol[5, 2, :] = -0.0; vol[11, 2, :] = 0.0; vol[[d for d in range(D) if d not in (5, 11)], 2, :] = 1.0
    vol[:, 4, :] = np.nan                  # nothing selectable -> 0
    vol[0] = -1e30                         # d=0 never a candidate
    b, n = shard_range(D, world, rank)
    keys = local_keys(vol[b:b + n], b)
    t = torch.from_numpy(keys.view(np.int64).reshape(-1))
    gathered = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(gathered, t)
    allk = np.stack([g.numpy().view(np.uint64) for g in gathered])
    dis = (allk.min(axis=0) & np.uint64(0xFF)).astype(np.uint8).reshape(H, W)
    if rank == 0:
        from oracle import oracle as O
        want = O.wta(vol)
        q.put(bool(np.array_equal(dis, want)) and int(dis[2, 0]) == 5 and int(dis[4, 0]) == 0)
    dist.destroy_process_group()


def test_two_rank_key_exchange_matches_wta():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert q.get(timeout=5) is True


def test_band_rows_partition_the_image():
    from primestereomatch_b200.sharding import band_rows
    for H in (1, 7, 375, 1080):
        for world in (1, 2, 3, 8):
            covered = []
            for r in range(world):
                r0, r1, rows = band_rows(H, world, r)
                assert 0 <= r0 <= r1 <= H and r1 - r0 <= rows
                covered += list(range(r0, r1))
            assert covered == list(range(H))
