"""Diagnostic: free-running target_amp policy on the CUDA path; prints env 0's task block / goal / root per policy step and compares every
step's goal with a host recomputation from the snapshot."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from deepmimic_b200.assets import asset_root
from deepmimic_b200.env import DeepMimicBatchEnv
from deepmimic_b200.rollout import BatchedRollout, build_gated_policy, load_actor_weights
from tests.test_task_scenes_cpu import fixture_task_actor, TARGET
root = asset_root(True)
a = fixture_task_actor("target")
env = DeepMimicBatchEnv(TARGET, num_envs=64, asset_root=root, seed=9)
env.set_mode(1); env.reset(True)
G = env.get_goal_size()
ro = BatchedRollout(env, policy=load_actor_weights(build_gated_policy(226, G, 28), a), exp_rate=0.0)
ro.s_norm.set_mean_std(a["s_norm_mean"], a["s_norm_std"]); ro.g_norm.set_mean_std(a["g_norm_mean"], a["g_norm_std"]); ro.a_norm.set_mean_std(a["a_norm_mean"], a["a_norm_std"])
core = env._core
nl = core.dims.num_joints
inside = 0; tot = 0
for k in range(int(os.environ.get("DIAG_STEPS", "240"))):
    traj = ro.collect(1, record_stats=False)
    torch.cuda.synchronize()
    g = traj["goals"][0].cpu().numpy(); r = traj["rewards"][0].cpu().numpy(); term = traj["terminate"][0].cpu().numpy(); done = traj["dones"][0].cpu().numpy()
    inside += (g[:, 2] < 0.5).sum(); tot += len(g)
    if k % 4 == 0 or done[0]:
        tb = core.task_state(0); s = core.get_snapshot(0)
        rx, rz = s[0] / 4.0, s[2] / 4.0
        print("step %3d env0: goal(before step) %s reward %.3f done %d term %d | root (%.2f %.2f) target (%.2f %.2f) dist %.2f speed %.2f timer %.2f/%.2f draws %d | mean reward all %.3f inside frac so far %.3f"
              % (k, np.round(g[0], 3), r[0], done[0], term[0], rx, rz, tb[0], tb[1], np.hypot(tb[0] - rx, tb[1] - rz), tb[2], tb[4], tb[5], int(tb[12]), r.mean(), inside / tot), flush=True)
