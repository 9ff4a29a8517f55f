"""The step kernel's placement of the environments by contact load, as host arithmetic (dm_plan_env_order, the rule dm_env_order_kernel
follows): a permutation of the padded environments; the two environments of a W = 16 warp are neighbours in the descending sort (stable: ties
by environment id); the snake dealing gives every block its share of heavy warps, give or take one, in descending load over its warp slots;
the padding environments come last."""
import numpy as np
import pytest

from deepmimic_b200.capi import plan_env_order

# (padded environments, environments per block, tile width): the spin kick / dog plans on 132 SMs and small odd shapes
SHAPES = [(4096, 16, 16), (1008, 8, 16), (2048, 8, 32), (4088, 28, 16), (64, 4, 16), (42, 14, 32)]


def _keys(n_pad, n_real, rng):
    keys = np.full(n_pad, -1, dtype=np.int32)
    k = rng.choice([0, 0, 0, 3, 6, 9, 12, 15, 18, 21, 24, 25, 26, 28], size=n_real)   # flight / single / double stance row counts
    keys[:n_real] = k
    return keys


@pytest.mark.parametrize("n_pad,tiles,w", SHAPES)
def test_plan_is_sorted_dealt_permutation(n_pad, tiles, w):
    rng = np.random.default_rng(n_pad + tiles + w)
    n_real = n_pad - (n_pad // 97)
    keys = _keys(n_pad, n_real, rng)
    order = plan_env_order(keys, tiles, w)
    assert np.array_equal(np.sort(order), np.arange(n_pad))
    per_warp = 32 // w
    blocks, warps = n_pad // tiles, tiles // per_warp
    # the sorted sequence: descending key, ties by id; padding (-1) last
    ref = sorted(range(n_pad), key=lambda e: (-keys[e], e))
    # a warp holds consecutive environments of the sorted sequence, in sorted order over its tiles
    rank = np.empty(n_pad, dtype=np.int64); rank[np.array(ref)] = np.arange(n_pad)
    r = rank[order].reshape(blocks, warps, per_warp)
    assert (r[..., 0] % per_warp == 0).all() and (np.diff(r, axis=2) == 1).all()
    # snake dealing: block b's warp slot s holds sorted warp s * B + (b or B - 1 - b)
    g = r[..., 0] // per_warp
    b = np.arange(blocks)[:, None]; s = np.arange(warps)[None, :]
    assert np.array_equal(g, s * blocks + np.where(s % 2 == 0, b, blocks - 1 - b))
    # within a block, loads descend over the warp slots
    wl = keys[order].reshape(blocks, warps, per_warp).max(axis=2)
    assert (np.diff(wl, axis=1) <= 0).all()
    # every block holds its share of heavy warps (+-1), for every threshold
    for thr in (1, 13, 22):
        heavy = (wl >= thr).sum(axis=1)
        assert heavy.max() - heavy.min() <= 1
    # padding last: after every real environment of its block
    pad = (order >= n_real).reshape(blocks, tiles)
    assert not (pad[:, :-1] & ~pad[:, 1:]).any()


def test_plan_pairs_equal_loads():
    """W = 16: with index placement 1 - (1 - p)^2 of the warps carry a heavy environment, sorted only about p"""
    rng = np.random.default_rng(3)
    n = 4096
    keys = np.where(rng.random(n) < 0.3, 26, 6).astype(np.int32)
    order = plan_env_order(keys, 16, 16)
    sorted_heavy = (keys[order].reshape(-1, 2).max(axis=1) > 22).mean()
    index_heavy = (keys.reshape(-1, 2).max(axis=1) > 22).mean()
    assert abs(sorted_heavy - (keys > 22).mean()) <= 1.0 / 2048 and index_heavy > 0.45


def test_plan_identity_for_equal_keys():
    """equal keys: ties by id, so one block of W = 32 environments keeps the index order"""
    assert np.array_equal(plan_env_order(np.zeros(14, dtype=np.int32), 14, 32), np.arange(14))


@pytest.mark.parametrize("n_pad,tiles,w", [(100, 16, 16), (64, 3, 16), (64, 4, 8), (0, 4, 16)])
def test_plan_refuses_bad_shapes(n_pad, tiles, w):
    with pytest.raises(RuntimeError, match="dm_plan_env_order"):
        plan_env_order(np.zeros(max(n_pad, 1), dtype=np.int32)[:n_pad], tiles, w)
