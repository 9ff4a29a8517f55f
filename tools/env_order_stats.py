"""How much the placement of the environments by contact load (dm_set_env_order) can save, on bench.py's workload after its pre-roll and
warm-up (48 + 4 policy steps of random actions, 20 s episodes): the key histogram (solver rows of each environment's last Bullet sub-step),
the fraction of warps per storage mode of the constraint solve (solve_rows: a warp takes its larger environment's row count), and the sum over
warps of that maximum, with index placement and with sorted placement; and how well a key predicts: the fraction of environments whose storage
mode after the first Update of the next policy step equals their key's.
  python tools/env_order_stats.py [--arg-file args/train_humanoid3d_spinkick_args.txt] [--envs 4096]"""
import argparse
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def mode(rows, w):
    """solve_rows' storage mode for a warp's maximum row count: none, W x W square, kSq2 x kSq2 square, packed triangle"""
    sq2 = 22 if w == 16 else 36
    return np.where(rows == 0, 0, np.where(rows <= w, 1, np.where(rows <= sq2, 2, 3)))


MODES = ("no rows", "square W", "square kSq2", "packed")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arg-file", default="args/train_humanoid3d_spinkick_args.txt")
    ap.add_argument("--envs", type=int, default=0, help="default: 4096 (humanoid3d) / 2048 (dog3d), as bench.py")
    ap.add_argument("--preroll", type=int, default=52)
    a = ap.parse_args()
    import torch
    from bench import scene_args
    from deepmimic_b200.assets import asset_root
    from deepmimic_b200.capi import BatchedCore, plan_env_order
    n = a.envs or (2048 if "dog" in a.arg_file else 4096)
    core = BatchedCore(scene_args(a.arg_file), n, asset_root(prefer_archive=True), seed=1000)
    stream = torch.cuda.ExternalStream(core.stream())
    with torch.cuda.stream(stream):
        off, scl, lo, hi = (torch.tensor(core.static(k), dtype=torch.float32, device="cuda") for k in (2, 3, 4, 5))
        g = torch.Generator(device="cuda"); g.manual_seed(7)
        core.reset(True, max_time=np.full(n, 20.0))
        core.set_episode_limit(20.0)
        act = lambda: torch.clamp(-off + 0.25 / scl * torch.randn(n, core.dims.action_size, device="cuda", generator=g), lo, hi).contiguous()
        for _ in range(a.preroll):
            core.set_action(act()); core.update(1 / 600., 20); core.reset(False)
        core.sync()
        keys, _, tiles, w = core.env_order()
        core.set_action(act()); core.update(1 / 600., 1)
        core.sync()
        nxt = core.env_order()[0]
    per_warp = 32 // w
    real = keys[:n]
    print("%s, %d envs, tile width %d, %d envs per block" % (a.arg_file, n, w, tiles))
    hist = np.bincount(real, minlength=real.max() + 1)
    print("key histogram (rows: envs): " + ", ".join("%d: %d" % (k, c) for k, c in enumerate(hist) if c))
    res = {}
    for name, order in (("index", np.arange(len(keys))), ("sorted", plan_env_order(keys, tiles, w))):
        wmax = np.maximum(keys[order], 0).reshape(-1, per_warp).max(axis=1)
        m = mode(wmax, w)
        res[name] = wmax.sum()
        print("%-6s placement: warps per mode %s ; sum over warps of max rows %d" % (
            name, ", ".join("%s %.1f%%" % (MODES[k], 100.0 * (m == k).mean()) for k in range(4)), wmax.sum()))
    print("sorted / index sum of max rows: %.3f" % (res["sorted"] / res["index"]))
    same = mode(real, w) == mode(nxt[:n], w)
    print("key predicts the storage mode after the next Update: %.1f%% of envs" % (100.0 * same.mean()))


if __name__ == "__main__":
    main()
