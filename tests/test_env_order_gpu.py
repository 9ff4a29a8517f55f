"""Placement of the environments in the step kernel by contact load (dm_set_env_order, dm_env_order_kernel): it only changes which
environments share a warp, a block and an SM, so every output must equal the index placement's bit for bit -- observations, rewards, flags,
the AMP task outputs and the full simulator snapshot of every environment, over policy steps with resets.  The device order is a permutation
of the padded environments with the padding last, equals the host rule (dm_plan_env_order) for the keys it was made from, and repeats."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SYN56 = ["--motion_file", "data/datasets/synthetic_locomotion_56.txt", "--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]
WORKLOADS = {
    "spinkick4096": (["--arg_file", "args/train_humanoid3d_spinkick_args.txt"], 4096),
    "walk4096": (["--arg_file", "args/train_humanoid3d_walk_args.txt"], 4096),
    "target_amp56_4096": (SYN56, 4096),
    "dog_trot2048": (["--arg_file", "args/train_dog3d_trot_args.txt"], 2048),   # W = 32: index placement either way
    "spinkick1001": (["--arg_file", "args/train_humanoid3d_spinkick_args.txt"], 1001),   # padded to 1008 on 132 SMs: one warp holds a real and a padding env
}
STEPS = 64


def _run(asset_root, args, n, order_on, steps=STEPS, keep_order=False):
    """`steps` policy steps of random actions with resets of the finished episodes; returns the outputs of every step, the final snapshots
    and (keep_order) the keys before and the placement of every step launch"""
    import torch
    from deepmimic_b200.capi import BatchedCore
    core = BatchedCore(args, n, asset_root, device=0, seed=11)
    core.set_env_order(order_on)
    d = core.dims
    task = d.goal_size > 0
    off, scl, lo, hi = (torch.tensor(core.static(k), dtype=torch.float32, device="cuda") for k in (2, 3, 4, 5))
    g = torch.Generator(device="cuda"); g.manual_seed(5)
    bank = torch.clamp(-off + 0.25 / scl * torch.randn(4, n, d.action_size, device="cuda", generator=g), lo, hi).contiguous()
    core.reset(True)
    outs, orders = [], []
    for i in range(steps):
        st = torch.zeros(n, d.state_size, device="cuda"); rw = torch.zeros(n, device="cuda"); fl = torch.zeros(n, 4, dtype=torch.int32, device="cuda")
        core.set_action(bank[i % 4])
        if keep_order:
            keys = core.env_order()[0]
        core.update(1.0 / 600.0, 20)
        if keep_order:
            orders.append((keys,) + core.env_order()[1:])
        core.observe(st, rw)
        core.flags(fl)
        step = [st, rw, fl]
        if task:
            goal = torch.zeros(n, d.goal_size, device="cuda"); amp = torch.zeros(n, d.amp_obs_size, device="cuda"); rim = torch.zeros(n, device="cuda")
            core.record_goal(goal); core.amp_obs_agent(amp); core.reward_imitate(rim)
            step += [goal, amp, rim]
        core.sync()
        outs.append([x.cpu().numpy() for x in step])
        core.reset(False)
    snaps = np.stack([core.get_snapshot(e) for e in range(n)])
    assert core.counters()[1] == 0
    core.close()
    return outs, snaps, orders


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_env_order_outputs_bit_identical(asset_root, name):
    args, n = WORKLOADS[name]
    on_out, on_snap, _ = _run(asset_root, args, n, True)
    off_out, off_snap, _ = _run(asset_root, args, n, False)
    for s, (a, b) in enumerate(zip(on_out, off_out)):
        for k, (x, y) in enumerate(zip(a, b)):
            if not np.array_equal(_bits(x), _bits(y)):
                bad = np.unique(np.nonzero((x != y).reshape(n, -1))[0])
                pytest.fail("%s: step %d output %d differs in %d environments (first %s)" % (name, s, k, len(bad), bad[:8].tolist()))
    bad = np.unique(np.nonzero((on_snap != off_snap).reshape(n, -1))[0])
    assert np.array_equal(_bits(on_snap), _bits(off_snap)), "%s: final snapshots differ in %d environments (first %s)" % (name, len(bad), bad[:8].tolist())


def test_env_order_device_matches_host_rule(asset_root):
    from deepmimic_b200.capi import plan_env_order
    args, n = WORKLOADS["spinkick1001"]
    _, _, orders = _run(asset_root, args, n, True, steps=24, keep_order=True)
    _, _, again = _run(asset_root, args, n, True, steps=24, keep_order=True)
    heavy = 0
    for (keys, order, tiles, w), (keys2, order2, _, _) in zip(orders, again):
        npad = len(order)
        assert npad >= n and npad % tiles == 0
        assert np.array_equal(np.sort(order), np.arange(npad))
        assert (keys[n:] == -1).all() and (keys[:n] >= 0).all()
        assert np.array_equal(order, plan_env_order(keys, tiles, w))
        # padding environments sit behind every real environment of their block
        per_block = order.reshape(-1, tiles)
        for blk in per_block:
            pad = blk >= n
            assert not (pad[:-1] & ~pad[1:]).any()
        assert np.array_equal(keys, keys2) and np.array_equal(order, order2)   # same run, same placement
        heavy += int((keys[:n] > 0).sum())
    assert heavy > 0   # the keys carry contact loads, not only zeros
