"""GPU parity tests of the two AMP task scenes that are outside SURVEY.md 8 (heading_amp_getup, strike_amp; the verdict of round 1 marks them
out of scope) and whose device glue is therefore still opt-in.  target_amp / heading_amp / --sync_char_root_rot moved to the default suite in
round 2 (tests/test_task_scenes_gpu.py, tests/test_parity2_gpu.py).

OPT-IN: the device half of the task scenes (dm_task.cuh inside dm_step_kernel<.., TASK>, dm_task_reset_kernel, dm_task_observe_kernel) was
written after round 1's GPU budget was spent and has never run on hardware.  dm_create refuses the scenes unless
DM_EXPERIMENTAL_TASK_SCENES=1; these tests additionally need DM_RUN_UNVALIDATED_GPU_TESTS=1 so that the default `pytest -m gpu` run only
contains tests of code that has been validated on hardware.  To validate: run with both variables set, fix what breaks, then drop the gates."""
import os

import numpy as np
import pytest

from tests.oracle_binding import Oracle

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(os.environ.get("DM_RUN_UNVALIDATED_GPU_TESTS") != "1", reason="task-scene device code not yet validated on hardware (opt-in)")]

MINI = ["--motion_file", "data/datasets/test_clips_mini.txt"]                    # 4-clip dataset of the committed asset archive (--kin_ctrl clips)
TARGET = ["--rand_target_time_min", "1", "--rand_target_time_max", "2"] + MINI + ["--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]
HEADING = MINI + ["--arg_file", "args/train_amp_heading_humanoid3d_locomotion_args.txt"]
# heading_amp_getup / strike_amp on the same assets (clips 1, 2 of the mini dataset stand in for the get-up motions; see tests/test_task_scenes_cpu.py)
GETUP = ["--scene", "heading_amp_getup", "--getup_motion_ids", "1", "2", "--getup_height_root", "1.2", "--getup_height_head", "2.0", "--head_id", "2"] + HEADING
STRIKE = ["--scene", "strike_amp", "--target_hit_reset_time", "2", "--target_radius", "0.2", "--target_min", "-0.5", "1.2", "0.6", "--target_max", "0.5", "1.4", "1.1",
          "--tar_near_dist", "1.4", "--tar_far_prob", "0.4", "--strike_bodies", "8", "--fail_tar_contact_bodies", "0", "1", "2", "--init_hit_prob", "0.1",
          "--hit_tar_speed", "1.5", "--tar_reward_scale", "2"] + TARGET
N = 32


@pytest.mark.parametrize("args", [GETUP, STRIKE])
def test_task_goal_reward_and_updates_match_the_oracle(asset_root, args, monkeypatch):
    """Free-running comparison over 3 s under one random action sequence per environment: same draw stream (seed, global env id), so the
    target timers, headings and speeds must agree exactly in count and to rounding in value; goals and rewards to the fp32 state's accuracy."""
    import torch
    from deepmimic_b200 import capi
    monkeypatch.setenv("DM_EXPERIMENTAL_TASK_SCENES", "1")
    core = capi.BatchedCore(args, N, asset_root, seed=21, global_env_offset=100)
    P, task_seed, env_base = core.task_params()
    G = core.dims.goal_size
    assert G == (4 if args in (GETUP, STRIKE) else 3) and env_base == 100
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
        np.testing.assert_allclose(amp[e].cpu().numpy(), o.record_amp_obs_expert(etime[e], clip=int(eclip[e])), atol=2e-3)
    goal = torch.zeros(N, G, device="cuda"); rew = torch.zeros(N, device="cuda"); flags = torch.zeros(N, 4, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    if args is STRIKE:   # every 4th environment gets its target right at the (moving) hand so that hits, holds and successes occur in the run
        for e in range(0, N, 4):
            o = oracles[e]
            pos, _, lv, _ = o.body_state()
            ts = o.task_state()
            o.set_task_state(pos[8] + 0.02 * lv[8] / (np.linalg.norm(lv[8]) + 1e-9), 1.0, 0.0, ts["timer"], ts["timer_max"], ts["prev_action_com"])
            o.set_strike_state(False, -1.0)
    rng = np.random.default_rng(5)
    st = oracles[0].action_statics()
    worst_goal = worst_rew = 0.0
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
            if args is GETUP:
                tb[16 + 3] = o.getup_state()["timer"]
            if args is STRIKE:
                ss = o.strike_state()
                tb[16 + 0], tb[16 + 1], tb[16 + 2] = ss["target_height"], float(ss["hit"]), ss["hit_time"]
            core.set_task_state(e, tb)
        a = np.clip(-st[0] + 0.1 / st[1] * rng.standard_normal((N, oracles[0].action_size)), st[2], st[3])
        core.set_action(torch.as_tensor(a, dtype=torch.float32, device="cuda"))
        torch.cuda.synchronize()
        core.update(1.0 / 600.0, 20)
        core.record_goal(goal); core.observe(None, rew); core.flags(flags); core.sync()
        g, r, f = goal.cpu().numpy(), rew.cpu().numpy(), flags.cpu().numpy()
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
            if args is GETUP:
                assert tb[16 + 3] == pytest.approx(o.getup_state()["timer"], abs=1e-9)
            if args is STRIKE:
                ss = o.strike_state()
                assert bool(tb[16 + 1]) == ss["hit"] and tb[16 + 0] == pytest.approx(ss["target_height"], abs=1e-9)
                if ss["hit"]:
                    assert tb[16 + 2] == pytest.approx(ss["hit_time"], abs=1e-9)
            worst_goal = max(worst_goal, float(np.abs(g[e] - o.record_goal()).max()))
            if not o.has_fallen():
                worst_rew = max(worst_rew, abs(float(r[e]) - o.calc_reward()))
            checked += 1
    # random actions make most characters fall within the first second: the count only guards against an empty comparison
    print("task scene %s: %d environment-steps compared, worst goal error %.2e, worst reward error %.2e" % (args[0:2], checked, worst_goal, worst_rew))
    assert checked > 250
    assert worst_goal < 5e-3 and worst_rew < 1e-2, (worst_goal, worst_rew)
    core.close()


GETUP_REAL = ["--arg_file", "args/train_amp_heading_getup_humanoid3d_locomotion_getup_args.txt"]      # the reference's own 4-clip get-up dataset (in the archive)
STRIKE_REAL = MINI + ["--arg_file", "args/train_amp_strike_humanoid3d_walk_punch_args.txt"]


@pytest.mark.parametrize("task,args", [("heading_getup", GETUP_REAL), ("strike", STRIKE_REAL)])
def test_fixture_task_policies_through_the_cuda_path(asset_root, task, args, monkeypatch):
    """The reference's pretrained task policies (fp16 fixtures) driving 64 environments for 20 s through the batched env + goal-conditioned
    rollout: targets reached / heading followed / up from the ground and walking / target punched, like in the oracle (tests/test_task_scenes_cpu.py)."""
    import torch
    from deepmimic_b200.env import DeepMimicBatchEnv
    from deepmimic_b200.rollout import BatchedRollout, build_gated_policy, load_actor_weights
    from tests.test_task_scenes_cpu import fixture_task_actor
    monkeypatch.setenv("DM_EXPERIMENTAL_TASK_SCENES", "1")
    a = fixture_task_actor(task)
    env = DeepMimicBatchEnv(args, num_envs=64, asset_root=asset_root, seed=9)
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
        inside = (traj["goals"][:, :, 2] < 0.5).float().mean()
        assert falls <= 6 and float(inside) > 0.08 and mean_r > 0.4, (falls, float(inside), mean_r)
    elif task == "heading":
        assert falls <= 6 and mean_r > 0.8, (falls, mean_r)
    elif task == "heading_getup":   # test mode: a fall starts a get-up instead of ending the episode; half of the start clips lie on the ground
        assert falls == 0 and float(traj["rewards"][300:].mean()) > 0.8, (falls, float(traj["rewards"][300:].mean()))
        assert float(traj["goals"][0, :, 3].max()) > 0.7 and float(traj["goals"][-1, :, 3].max()) < 0.5       # get-up phase: some start near 1 (lying down), nobody is still getting up at the end
    else:                           # strike: episodes end with the success code 2 s after the hit and restart; most environments get there at least once
        succ = int((traj["terminate"] == 2).sum())
        assert succ >= 32 and falls <= 16, (succ, falls)
