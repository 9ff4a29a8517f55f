"""Tiny workload for compute-sanitizer (memcheck / racecheck / initcheck): a few policy steps of 8 humanoid environments that are on the
ground (contacts, limits, resets) with their poses, then the expert sampler for a row count above num_envs and not a multiple of its block.  usage: compute-sanitizer --tool racecheck python tools/sanitize_run.py"""
import os, sys
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import numpy as np
import torch
from deepmimic_b200.assets import asset_root
from deepmimic_b200.capi import BatchedCore

arg = sys.argv[1] if len(sys.argv) > 1 else "args/train_humanoid3d_spinkick_args.txt"
N = 8
core = BatchedCore(["--arg_file", arg], N, asset_root(True), seed=3)
S, A = core.dims.state_size, core.dims.action_size
stream = torch.cuda.ExternalStream(core.stream())
with torch.cuda.stream(stream):
    obs = torch.zeros(N, S, device="cuda"); rew = torch.zeros(N, device="cuda"); fl = torch.zeros(N, 4, dtype=torch.int32, device="cuda")
    amp = torch.zeros(N, core.dims.amp_obs_size, device="cuda")
    pose = torch.zeros(N, core.dims.pose_dim, device="cuda"); vel = torch.zeros(N, core.dims.pose_dim, device="cuda")
    g = torch.Generator(device="cuda"); g.manual_seed(1)
    off = torch.tensor(core.static(2), dtype=torch.float32, device="cuda"); scl = torch.tensor(core.static(3), dtype=torch.float32, device="cuda")
    for step in range(6):
        a = (-off + 0.5 / scl * torch.randn(N, A, device="cuda", generator=g)).contiguous()
        core.set_action(a); core.update(1 / 600., 20); core.observe(obs, rew); core.flags(fl); core.amp_obs_agent(amp); core.record_pose(pose, vel); core.reset(False)
    exp = torch.zeros(21, core.dims.amp_obs_size, device="cuda"); eclip = torch.zeros(21, dtype=torch.int32, device="cuda")
    etime = torch.zeros(21, dtype=torch.float64, device="cuda")
    core.sample_amp_obs_expert(exp, eclip, etime)
core.sync()
print("done", float(rew.mean()), int(fl[:, 1].sum()), core.counters())
