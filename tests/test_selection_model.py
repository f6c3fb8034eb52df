"""CPU: the packed-key model of disparity selection (selection_cases.py) against the C oracle's restatement of DispSel
(O.wta).  On volumes holding NaN of both signs with payloads, +-inf, -0 next to +0, FLT_MAX, denormals and exact ties,
the min over the keys of any partition of [0, D) into blocks or shards is the one-scan key, and the key's low bits are
the oracle's map."""
import numpy as np
import pytest

import selection_cases as S
from oracle import oracle as O

F32 = np.float32


def special_volume(D, H=12, W=17, seed=0):
    rng = np.random.default_rng([seed, D])
    vol = rng.random((D, H, W), dtype=F32) + F32(1)
    nan = np.array([0x7FC00000, 0xFFC01234, 0x7FA00001, 0xFF800001], np.uint32).view(F32)
    specials = np.concatenate([nan, np.array([np.inf, -np.inf, -0.0, 0.0, np.finfo(F32).max, -np.finfo(F32).max,
                                              1e-45, -1e-45, 1e-40, np.finfo(F32).tiny], F32)])
    mask = rng.random(vol.shape) < 0.3
    vol[mask] = rng.choice(specials, int(mask.sum()))
    # exact ties: a pair of slices equal on a row band, a constant column
    for _ in range(3):
        a, b = rng.choice(D, 2, replace=False)
        vol[b, : H // 2] = vol[a, : H // 2]
    vol[:, :, 3] = F32(0.5)
    vol[:, 4, :] = F32(1.0)
    vol[rng.integers(1, D), 4, :] = F32(-0.0)
    vol[rng.integers(1, D), 4, :] = F32(0.0)
    vol[:, 5, :] = np.array([0x7FC00000], np.uint32).view(F32)[0]     # all NaN: d = 0
    vol[:, 6, :] = np.inf                                               # all +inf: d = 0
    vol[:, 7, ::2] = np.where(np.arange(D)[:, None] % 2, np.inf, np.nan)
    vol[:, 8, :] = np.finfo(F32).max                                    # ties at FLT_MAX: d = 1
    vol[0, 9, :] = -np.inf                                              # d = 0 never a candidate
    vol[:, 10, :] = F32(1.0)
    vol[D - 1, 10, :] = -np.inf                                         # the last slice wins
    vol[1:, 11, :] = np.array([1e-45], F32)                             # denormal ties: d = 1
    return vol


VOLUMES = [(D, seed) for D in (2, 3, 7, 16, 29) for seed in (0, 1)]


@pytest.mark.parametrize("D,seed", VOLUMES)
def test_key_bits_are_the_oracle_maps(D, seed):
    vol = special_volume(D, seed=seed)
    k = S.scan_keys(vol)
    assert k.dtype == np.uint64
    np.testing.assert_array_equal(S.disparity(k, np.uint16), O.wta(vol, np.uint16))
    np.testing.assert_array_equal(S.disparity(k, np.uint8), O.wta(vol))
    assert (k[5] == S.NO_WINNER).all() and (k[6] == S.NO_WINNER).all() and (k[7, ::2] == S.NO_WINNER).all()
    assert (S.disparity(k[8], np.uint16) == 1).all() and (S.disparity(k[11], np.uint16) == 1).all()
    assert (S.disparity(k[10], np.uint16) == D - 1).all()
    assert (k[4] >> S.U64(32) == S.order_key(F32(0.0))).all()         # the -0 / +0 winner's key is +0's
    if D > 2:
        assert (S.disparity(k[9], np.uint16) != 0).any()


@pytest.mark.parametrize("D,seed", VOLUMES)
def test_every_block_partition_folds_to_one_scan(D, seed):
    vol = special_volume(D, seed=seed)
    want = S.scan_keys(vol)
    for B in range(1, D + 1):
        blocks = S.block_ranges(0, D, B)
        assert [d for b, n in blocks for d in range(b, b + n)] == list(range(D))
        np.testing.assert_array_equal(S.fold(vol, blocks), want, f"B = {B}")


@pytest.mark.parametrize("D,seed", VOLUMES)
def test_every_shard_split_folds_to_one_scan(D, seed):
    vol = special_volume(D, seed=seed)
    want = S.scan_keys(vol)
    for n in range(1, min(8, D) + 1):
        np.testing.assert_array_equal(S.fold(vol, S.shard_ranges(D, n)), want, f"{n} shards")
        for B in (1, 2, 3, 5):
            np.testing.assert_array_equal(S.fold(vol, S.multi_ranges(D, n, B)), want, f"{n} shards, blocks of {B}")
        # one shard with blocks whose first does not start at a multiple of B: the shard's keys are its scan's
        b, c = S.shard_range(D, n, n - 1)
        sub = vol[b:b + c]
        np.testing.assert_array_equal(S.fold(sub, S.block_ranges(b, c, 3), b), S.scan_keys(sub, b))


def test_order_key_orders_like_less_than():
    v = np.array([-np.inf, -np.finfo(F32).max, -1.0, -1e-45, -0.0, 0.0, 1e-45, np.finfo(F32).tiny, 1.0,
                  np.finfo(F32).max, np.inf], F32)
    k = S.order_key(v)
    assert (np.diff(k.astype(np.int64)) > 0)[[0, 1, 2, 3, 5, 6, 7, 8, 9]].all()
    assert k[4] == k[5]                                                  # -0 and +0 tie
    assert S.NO_WINNER == S.order_key(F32(np.inf)) << S.U64(32)
    assert (S.order_key(v[:-1]) << S.U64(32) | S.U64(65535) < S.NO_WINNER).all()


def test_seam_ties_counts_only_ties_across_seams():
    vol = np.full((6, 1, 3), 2.0, F32)
    vol[2, 0, :] = vol[4, 0, :] = 1.0      # winner 2, tied with 4
    vol[5, 0, 1] = 1.0
    k = S.scan_keys(vol)
    assert S.seam_ties(vol, k, [(0, 6)]) == 0
    assert S.seam_ties(vol, k, [(0, 4), (4, 2)]) == 3
    assert S.seam_ties(vol, k, [(0, 3), (3, 3)]) == 3
    assert S.seam_ties(vol, k, [(0, 5), (5, 1)]) == 1
