"""GPU parity of the AMP task scenes target_amp / heading_amp (BASELINE.json config 5; SURVEY.md 8(f) rank 2): goals, task rewards, target /
heading updates on the device's draw stream, per-environment clips of a --kin_ctrl clips dataset, expert observations from dataset clips, the
imitation reward against the active clip -- against the oracle through the C ABI; plus the reference's pretrained task policies (fp16 fixtures)
driving the CUDA path.  Validated on hardware (these tests were opt-in while the device code had never run).
R/DeepMimicCore/scenes/SceneTargetAMP.cpp:3-80,136-145,185-224,259-292; SceneHeadingAMP.cpp:3-48,136-205; anim/ClipsController.cpp:204-243."""
import numpy as np
import pytest

from tests import amp_states as A
from tests.oracle_binding import Oracle

pytestmark = pytest.mark.gpu

MINI = ["--motion_file", "data/datasets/test_clips_mini.txt"]                    # 4-clip dataset of the committed asset archive (--kin_ctrl clips)
TARGET = MINI + ["--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]
TARGET_FAST = ["--rand_target_time_min", "1", "--rand_target_time_max", "2"] + TARGET   # several target re-draws inside a short comparison
HEADING = MINI + ["--arg_file", "args/train_amp_heading_humanoid3d_locomotion_args.txt"]
SYN56 = ["--motion_file", "data/datasets/synthetic_locomotion_56.txt", "--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]   # config 5's shape: 56 clips
N = 32


@pytest.mark.parametrize("args", [TARGET_FAST, HEADING])
def test_task_goal_reward_and_updates_match_the_oracle(asset_root, args):
    """Free-running comparison over 3 s under one random action sequence per environment: same draw stream (seed, global env id), so the
    target timers, headings and speeds must agree exactly in count and to rounding in value; goals and rewards to the fp32 state's accuracy."""
    import torch
    from deepmimic_b200 import capi
    core = capi.BatchedCore(args, N, asset_root, seed=21, global_env_offset=100)
    P, task_seed, env_base = core.task_params()
    G = core.dims.goal_size
    assert G == 3 and env_base == 100
    kin_time = np.linspace(0.0, 0.7, N); theta = np.linspace(-3.0, 3.0, N); max_time = np.full(N, 20.0); clip = np.arange(N) % 4
    core.reset(force_all=True, kin_time=kin_time, max_time=max_time, rot_theta=theta, clip=clip)
    oracles = []
    for e in range(N):
        o = Oracle(args, asset_root)
        o.set_task_stream(task_seed, env_base + e, 0)
        o.reset(kin_time[e], theta[e], 20.0, clip=int(clip[e]))
        oracles.append(o)
    # the reset state itself (one clip per environment) and the expert observations from given clips
    st0 = torch.zeros(N, core.dims.state_size, device="cuda"); amp = torch.zeros(N, core.dims.amp_obs_size, device="cuda")
    torch.cuda.synchronize()
    core.observe(st0, None)
    eclip = (np.arange(N) + 1) % 4; etime = np.linspace(0.05, 0.75, N)
    core.amp_obs_expert(amp, kin_time=etime, clip=eclip)
    core.sync()
    for e, o in enumerate(oracles):
        np.testing.assert_allclose(st0[e].cpu().numpy(), o.record_state(), atol=2e-4)
        A.check_split(amp[e].cpu().numpy(), o.record_amp_obs_expert(etime[e], clip=int(eclip[e])), o.pose_dim, A.max_level(asset_root, "humanoid3d"), e)
    goal = torch.zeros(N, G, device="cuda"); rew = torch.zeros(N, device="cuda"); rew_im = torch.zeros(N, device="cuda"); flags = torch.zeros(N, 4, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    rng = np.random.default_rng(5)
    st = oracles[0].action_statics()
    worst_goal = worst_rew = worst_im = 0.0
    checked = 0
    for step in range(90):
        # teacher forcing: every policy step starts from the oracle's exact state (simulator snapshot + task block), so the comparison is
        # one step deep and free of the chaotic drift of contacts
        live = [e for e, o in enumerate(oracles) if not o.is_episode_end()]
        for e in live:
            o = oracles[e]
            core.set_snapshot(e, o.get_snapshot())
            tb = core.task_state(e); ts = o.task_state()
            tb[0], tb[1] = ts["target_pos"][0], ts["target_pos"][2]
            tb[2:6] = [ts["target_speed"], ts["target_heading"], ts["timer"], ts["timer_max"]]
            tb[6:9] = ts["prev_action_com"]; tb[12] = o.task_counter()
            core.set_task_state(e, tb)
        a = np.clip(-st[0] + 0.1 / st[1] * rng.standard_normal((N, oracles[0].action_size)), st[2], st[3])
        core.set_action(torch.as_tensor(a, dtype=torch.float32, device="cuda"))
        torch.cuda.synchronize()
        core.update(1.0 / 600.0, 20)
        core.record_goal(goal); core.observe(None, rew); core.reward_imitate(rew_im); core.flags(flags); core.sync()
        g, r, f, ri = goal.cpu().numpy(), rew.cpu().numpy(), flags.cpu().numpy(), rew_im.cpu().numpy()
        for e in live:
            o = oracles[e]
            o.set_action(a[e].astype(np.float32).astype(np.float64))
            for _ in range(20):
                o.update(1.0 / 600.0)
                if o.is_episode_end():
                    break
            if o.is_episode_end() or f[e, 1]:
                continue                                                                     # an episode ended inside the step: flags are checked elsewhere
            tb = core.task_state(e); ts = o.task_state()
            assert int(tb[12]) == o.task_counter(), (step, e)                               # same number of draws consumed
            np.testing.assert_allclose(tb[2:6], [ts["target_speed"], ts["target_heading"], ts["timer"], ts["timer_max"]], atol=1e-9)
            np.testing.assert_allclose([tb[0], tb[1]], ts["target_pos"][[0, 2]], atol=2e-3)  # target = root position (fp32 sim state) + draw
            np.testing.assert_allclose(tb[6:9], ts["prev_action_com"], atol=1e-4)           # COM at the action (fp32 link frames)
            np.testing.assert_allclose(tb[9:12], o.calc_com(), atol=2e-3)                    # COM after 20 free updates
            worst_goal = max(worst_goal, float(np.abs(g[e] - o.record_goal()).max()))
            if not o.has_fallen():
                worst_rew = max(worst_rew, abs(float(r[e]) - o.calc_reward()))
                worst_im = max(worst_im, abs(float(ri[e]) - o.calc_reward_imitate()))   # CalcRewardImitate against the env's clip, on the free-run state
            checked += 1
    # random actions make most characters fall within the first second: the count only guards against an empty comparison
    print("task scene %s: %d environment-steps compared, worst goal error %.2e, worst task reward error %.2e, worst imitation reward error %.2e"
          % (args[-1], checked, worst_goal, worst_rew, worst_im))
    assert checked > 250
    assert worst_goal < 5e-3 and worst_rew < 1e-2 and worst_im < 2e-2, (worst_goal, worst_rew, worst_im)
    core.close()



@pytest.mark.parametrize("task,args", [("target", TARGET), ("heading", HEADING)])
def test_fixture_task_policies_through_the_cuda_path(asset_root, task, args):
    """The reference's pretrained task policies (fp16 fixtures) driving 64 environments for 20 s through the batched env + goal-conditioned
    rollout: targets reached (the oracle under the same policy: 0.30 of the steps inside the success radius, mean reward 0.58 over 12 draw
    streams) / heading followed (oracle 0.96)."""
    import torch
    from deepmimic_b200.env import DeepMimicBatchEnv
    from deepmimic_b200.rollout import BatchedRollout, build_gated_policy, load_actor_weights
    from tests.test_task_scenes_cpu import fixture_task_actor
    a = fixture_task_actor(task)
    env = DeepMimicBatchEnv(args, num_envs=64, asset_root=asset_root, seed=9)
    assert env.get_name() == ("Target AMP" if task == "target" else "Heading AMP")
    env.set_mode(1)
    env.reset(True)
    G = env.get_goal_size()
    ro = BatchedRollout(env, policy=load_actor_weights(build_gated_policy(226, G, 28), a), exp_rate=0.0)
    ro.s_norm.set_mean_std(a["s_norm_mean"], a["s_norm_std"]); ro.g_norm.set_mean_std(a["g_norm_mean"], a["g_norm_std"]); ro.a_norm.set_mean_std(a["a_norm_mean"], a["a_norm_std"])
    traj = ro.collect(600, record_stats=False)
    torch.cuda.synchronize()
    falls = int((traj["terminate"] == 1).sum())
    mean_r = float(traj["rewards"].mean())
    if task == "target":
        inside = float((traj["goals"][:, :, 2] < 0.5).float().mean())
        print("target policy on the CUDA path: %d failed episodes in 64 x 600 steps, inside the success radius %.3f of the steps, mean reward %.3f" % (falls, inside, mean_r))
        assert falls <= 12 and inside > 0.15 and mean_r > 0.45, (falls, inside, mean_r)
    else:
        print("heading policy on the CUDA path: %d failed episodes, mean reward %.3f" % (falls, mean_r))
        assert falls <= 6 and mean_r > 0.8, (falls, mean_r)
    assert env.check_solver_capacity() == 0


def test_config5_shape_4096_envs_56_clip_dataset(asset_root):
    """BASELINE.json configs[4]: target_amp, 4096 environments, a 56-clip dataset (synthetic, over the archive's locomotion clips), AMP agent
    observations recorded next to the imitation reward.  Every environment draws its own clip; state 226, goal 3, AMP observation 226; a few
    policy steps under random actions stay finite; the clip draw follows the dataset's sampling weights."""
    import torch
    from deepmimic_b200.capi import BatchedCore
    Nn = 4096
    core = BatchedCore(SYN56, Nn, asset_root, device=0, seed=3)
    d = core.dims
    assert (d.state_size, d.goal_size, d.amp_obs_size, d.action_size) == (226, 3, 226, 28)
    dur, cdf = core.clip_table()
    assert len(dur) == 56
    st = torch.zeros(Nn, 226, device="cuda"); goal = torch.zeros(Nn, 3, device="cuda"); rew = torch.zeros(Nn, device="cuda"); rim = torch.zeros(Nn, device="cuda")
    amp = torch.zeros(Nn, 226, device="cuda"); exp = torch.zeros(Nn, 226, device="cuda"); fl = torch.zeros(Nn, 4, dtype=torch.int32, device="cuda")
    off = torch.tensor(core.static(2), dtype=torch.float32, device="cuda"); scl = torch.tensor(core.static(3), dtype=torch.float32, device="cuda")
    lo = torch.tensor(core.static(4), dtype=torch.float32, device="cuda"); hi = torch.tensor(core.static(5), dtype=torch.float32, device="cuda")
    g = torch.Generator(device="cuda"); g.manual_seed(1)
    core.reward_imitate(rim); core.sync()
    assert float(rim.min()) > 0.95 and float(rim.median()) > 0.999   # right after a reset the simulated character sits on its clip pose (lifted out of the ground where needed)
    for step in range(6):
        a = torch.clamp(-off + 0.25 / scl * torch.randn(Nn, 28, device="cuda", generator=g), lo, hi).contiguous()
        core.set_action(a); core.update(1.0 / 600.0, 20)
        core.observe(st, rew); core.record_goal(goal); core.reward_imitate(rim); core.amp_obs_agent(amp); core.amp_obs_expert(exp); core.flags(fl)
        core.reset(False)
    core.sync()
    for t in (st, goal, rew, rim, amp, exp):
        assert bool(torch.isfinite(t).all())
    assert 0.0 <= float(rim.min()) and float(rim.max()) <= 1.0 and float(rew.max()) <= 1.0
    assert abs(float(goal[:, :2].norm(dim=1).median()) - 1.0) < 1e-3       # unit direction to the target in the heading frame
    assert core.counters()[1] == 0
