"""GPU parity of the two task scenes of dm_task_ext.cuh, heading_amp_getup and strike_amp, against the CPU oracle.

The scene formulas themselves are checked on the host (tests/test_task_scenes_cpu.py runs dm_task_ext.cuh against the oracle through
tests/task_shim.cpp).  These tests check the device glue around them: which lane publishes which body's position and velocity to lane 0
of the step kernel, when in the update the scene timer is read, the fall-flag override while a character gets up, the recovery branch of
the reset kernel, the task reset / observe kernels, and indexing by the real environment id under placement by contact load.

Most tests are teacher-forced update by update (the protocol of tests/test_push_gpu.py): before every update(DT, 1) the oracle's simulator
snapshot and its task block are loaded into the GPU environment, so the comparison is one update deep and free of the chaotic drift of
contacts.  Tolerances come from the stated teacher-forced bounds of tests/test_parity_gpu.py: |dq| <= 1e-3; |dqd| <= 1e-3 contact-free and
<= 0.5 (max) with contacts.  Published body values are in addition compared with the oracle's evaluation of the GPU's own post-update
state (a second oracle loaded with the GPU snapshot), where only fp32 rounding of the forward kinematics separates the two."""
import numpy as np
import pytest

from tests import amp_states as A
from tests.oracle_binding import Oracle
from tests.task_states import airborne as _airborne, load as _load, lying as _lying, set_clocks as _set_clocks
from tests.parity_util import SnapLayout, random_policy_action

pytestmark = pytest.mark.gpu

DT = 1.0 / 600.0
SCALE = 4.0                                           # --world_scale of the humanoid argument files
NJ = 15
LAY = SnapLayout(NJ)
CLK = LAY.scal                                        # snapshot clocks: +0 kin time, +8 ctrl, +9 init offset, +10 prev action, +11 need action, +12 timer, +13 timer max
# task block as returned by BatchedCore.task_state: dm_task.cuh slots 0..15, then the dm_task_ext.cuh slots
K_COUNTER, K_RESET_SEEN = 12, 13
X_TAR_Y, X_HIT, X_HIT_TIME, X_GETUP, X_NEAR, X_CFAIL, X_HEAD_Y, X_RECOVER = range(16, 24)
PARENTS = [-1, 0, 1, 0, 3, 4, 1, 6, 7, 0, 9, 10, 1, 12, 13]   # humanoid3d.txt
HIT_RESET = 2.0
FAIL_DIST = 15.0

MINI = ["--motion_file", "data/datasets/test_clips_mini.txt"]                    # 4-clip dataset of the committed asset archive (--kin_ctrl clips)
TARGET = ["--rand_target_time_min", "1", "--rand_target_time_max", "2"] + MINI + ["--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]
HEADING = MINI + ["--arg_file", "args/train_amp_heading_humanoid3d_locomotion_args.txt"]


# heading_amp_getup / strike_amp on the same assets (clips 1, 2 of the mini dataset stand in for the get-up motions; see tests/test_task_scenes_cpu.py)
def getup_args(head=2, recover=0.0):
    return ["--scene", "heading_amp_getup", "--getup_motion_ids", "1", "2", "--getup_height_root", "1.2", "--getup_height_head", "2.0",
            "--head_id", str(head), "--recover_episode_prob", repr(float(recover))] + HEADING


def strike_args(strike=(8,), fail=(0, 1, 2), radius=0.2, hit_speed=1.5):
    return ["--scene", "strike_amp", "--target_hit_reset_time", repr(HIT_RESET), "--target_radius", repr(radius), "--target_min", "-0.5", "1.2", "0.6",
            "--target_max", "0.5", "1.4", "1.1", "--tar_near_dist", "1.4", "--tar_far_prob", "0.4", "--strike_bodies"] + [str(b) for b in strike] + [
            "--fail_tar_contact_bodies"] + [str(b) for b in fail] + ["--init_hit_prob", "0.1", "--hit_tar_speed", repr(float(hit_speed)),
            "--tar_reward_scale", "2"] + TARGET


GETUP = getup_args()
STRIKE = strike_args()


# ---------------------------------------------------------------------------------------------------------------- helpers
def _core(args, n, asset_root, seed=21, offset=100, placement=False, mode=0):
    from deepmimic_b200 import capi
    core = capi.BatchedCore(args, n, asset_root, seed=seed, global_env_offset=offset)
    core.set_env_order(placement)
    core.set_mode(mode)
    return core


def _oracle(args, asset_root, core=None, env=0, mode=0):
    o = Oracle(args, asset_root)
    o.set_mode(mode)
    if core is not None:
        _, seed, base = core.task_params()
        o.set_task_stream(seed, base + env, 0)
    return o


def _outputs(core):
    """goal [N, G], reward [N], flags [N, 4] (need action, done, terminate, valid) as numpy"""
    import torch
    N, G = core.num_envs, core.dims.goal_size
    goal = torch.zeros(N, G, device="cuda"); rew = torch.zeros(N, device="cuda"); fl = torch.zeros(N, 4, dtype=torch.int32, device="cuda")
    core.record_goal(goal); core.observe(None, rew); core.flags(fl); core.sync()
    return goal.cpu().numpy().astype(np.float64), rew.cpu().numpy().astype(np.float64), fl.cpu().numpy()


def _set_target(o, pos, hit=False, hit_time=-1.0):
    ts = o.task_state()
    o.set_task_state(np.asarray(pos, dtype=np.float64), ts["target_speed"], ts["target_heading"], ts["timer"], ts["timer_max"], ts["prev_action_com"])
    o.set_strike_state(hit, hit_time)


def _mirror_bodies(mirror, core, e):
    """body COM positions and velocities of the GPU's own state of environment e, evaluated by the oracle, and the root (base) position"""
    s = core.get_snapshot(e)
    mirror.set_snapshot(s)
    pos, _, lv, _ = mirror.body_state()
    return pos, lv, s[0:3] / SCALE


def _near_r(tpos, root, pos, vel, s, vhit):
    """CalcRewardTargetNear of one strike body in float64 (SceneStrikeAMP.cpp:72-112)"""
    d = np.array([tpos[0] - root[0], 0.0, tpos[2] - root[2]])
    n = np.linalg.norm(d)
    u = d / n if n > 1e-5 else np.zeros(3)
    e = np.asarray(tpos) - pos
    vr = min(max(float(u @ vel) / vhit, 0.0), 1.0)
    return 0.2 * np.exp(-s * float(e @ e)) + 0.8 * vr * vr


def _chain(b):
    out = []
    while b >= 0:
        out.append(b); b = PARENTS[b]
    return out


def _pos_bound(pos, b):
    """|dq| <= 1e-3 (root position in m, quaternion components) through the lever arms: a quaternion component error of 1e-3 turns a joint by at
    most 2 sqrt(3) 1e-3 rad; the lever from joint a to body b's COM is at most |p_b - p_a| + |p_a - p_parent(a)|"""
    lev = sum(np.linalg.norm(pos[b] - pos[a]) + (np.linalg.norm(pos[a] - pos[PARENTS[a]]) if a > 0 else 0.0) for a in _chain(b))
    return 1e-3 + 2 * np.sqrt(3) * 1e-3 * lev, lev


def _vel_bound(pos, av, b, contact):
    """the qd bound (1e-3 contact-free, 0.5 with contacts) through the same lever arms, plus the angle error times the angular velocity"""
    _, lev = _pos_bound(pos, b)
    eqd = 0.5 if contact else 1e-3
    return eqd / SCALE + eqd * lev + 2 * np.sqrt(3) * 1e-3 * lev * np.abs(av).max()


def _near_bound(tpos, root, pos, vel, s, vhit, dp, dv):
    """first-order bound of the near term under |d pos| <= dp, |d root| <= dp, |d vel| <= dv (numerical gradient)"""
    g = 0.0
    for what, d in (("p", dp), ("v", dv), ("r", dp)):
        for k in range(3):
            h = np.zeros(3); h[k] = 1e-6
            a = dict(p=pos, v=vel, r=root)
            lo = dict(a); hi = dict(a)
            lo[what] = a[what] - h; hi[what] = a[what] + h
            der = (_near_r(tpos, hi["r"], hi["p"], hi["v"], s, vhit) - _near_r(tpos, lo["r"], lo["p"], lo["v"], s, vhit)) / 2e-6
            g += abs(der) * d
    return g + 1e-9


def _flags_of(o):
    return int(o.is_episode_end()), int(o.check_terminate()), int(o.check_valid_episode())


# ---------------------------------------------------------------------------------------------------------------- free-running
@pytest.mark.parametrize("args", [GETUP, STRIKE], ids=["getup", "strike"])
def test_task_goal_reward_and_updates_match_the_oracle(asset_root, args):
    """Free-running comparison over 3 s under one random action sequence per environment: same draw stream (seed, global env id), so the
    target timers, headings and speeds must agree exactly in count and to rounding in value; goals and rewards to the fp32 state's accuracy.
    Every policy step starts from the oracle's state (teacher forcing per 20-update step); the per-update tests below check ended episodes."""
    import torch
    N = 32
    core = _core(args, N, asset_root)
    P, task_seed, env_base = core.task_params()
    G = core.dims.goal_size
    assert G == 4 and env_base == 100
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
    goal = torch.zeros(N, G, device="cuda"); rew = torch.zeros(N, device="cuda"); flags = torch.zeros(N, 4, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    if args is STRIKE:   # every 4th environment gets its target right at the (moving) hand so that hits, holds and successes occur in the run
        for e in range(0, N, 4):
            o = oracles[e]
            pos, _, lv, _ = o.body_state()
            _set_target(o, pos[8] + 0.02 * lv[8] / (np.linalg.norm(lv[8]) + 1e-9))
    rng = np.random.default_rng(5)
    st = oracles[0].action_statics()
    worst_goal = worst_rew = 0.0
    checked = 0
    for step in range(90):
        live = [e for e, o in enumerate(oracles) if not o.is_episode_end()]
        for e in live:
            _load(core, e, oracles[e])
        a = np.clip(-st[0] + 0.1 / st[1] * rng.standard_normal((N, oracles[0].action_size)), st[2], st[3])
        core.set_action(torch.as_tensor(a, dtype=torch.float32, device="cuda"))
        torch.cuda.synchronize()
        core.update(DT, 20)
        core.record_goal(goal); core.observe(None, rew); core.flags(flags); core.sync()
        g, r, f = goal.cpu().numpy(), rew.cpu().numpy(), flags.cpu().numpy()
        for e in live:
            o = oracles[e]
            o.set_action(a[e].astype(np.float32).astype(np.float64))
            for _ in range(20):
                o.update(DT)
                if o.is_episode_end():
                    break
            if o.is_episode_end() or f[e, 1]:
                continue                                                                     # ended inside the step: checked update by update below
            tb = core.task_state(e); ts = o.task_state()
            assert int(tb[K_COUNTER]) == o.task_counter(), (step, e)                        # same number of draws consumed
            np.testing.assert_allclose(tb[2:6], [ts["target_speed"], ts["target_heading"], ts["timer"], ts["timer_max"]], atol=1e-9)
            np.testing.assert_allclose([tb[0], tb[1]], ts["target_pos"][[0, 2]], atol=2e-3)  # target = root position (fp32 sim state) + draw
            np.testing.assert_allclose(tb[6:9], ts["prev_action_com"], atol=1e-4)           # COM at the action (fp32 link frames)
            np.testing.assert_allclose(tb[9:12], o.calc_com(), atol=2e-3)                    # COM after 20 free updates
            if args is GETUP:
                assert tb[X_GETUP] == pytest.approx(o.getup_state()["timer"], abs=1e-9)
            else:
                ss = o.strike_state()
                assert bool(tb[X_HIT]) == ss["hit"] and tb[X_TAR_Y] == pytest.approx(ss["target_height"], abs=1e-9)
                if ss["hit"]:
                    assert tb[X_HIT_TIME] == pytest.approx(ss["hit_time"], abs=1e-9)
            worst_goal = max(worst_goal, float(np.abs(g[e] - o.record_goal()).max()))
            if not o.has_fallen():
                worst_rew = max(worst_rew, abs(float(r[e]) - o.calc_reward()))
            checked += 1
    # random actions make most characters fall within the first second: the count only guards against an empty comparison.  The strike goal is
    # the target in the root's frame, up to 10 m away: 20 free updates of heading drift (1e-3 rad) move it by up to 1e-2 (measured 9.1e-3)
    print("task scene %s: %d environment-steps compared, worst goal error %.2e, worst reward error %.2e" % (args[0:2], checked, worst_goal, worst_rew))
    assert checked > 250
    assert worst_goal < (1.5e-2 if args is STRIKE else 5e-3) and worst_rew < 1e-2, (worst_goal, worst_rew)
    core.close()


GETUP_REAL = ["--arg_file", "args/train_amp_heading_getup_humanoid3d_locomotion_getup_args.txt"]      # the reference's own 4-clip get-up dataset (in the archive)
STRIKE_REAL = MINI + ["--arg_file", "args/train_amp_strike_humanoid3d_walk_punch_args.txt"]


@pytest.mark.parametrize("task,args", [("heading_getup", GETUP_REAL), ("strike", STRIKE_REAL)])
def test_fixture_task_policies_through_the_cuda_path(asset_root, task, args):
    """The reference's pretrained task policies (fp16 fixtures) driving 64 environments for 20 s through the batched env + goal-conditioned
    rollout: up from the ground and walking / target punched, like in the oracle (tests/test_task_scenes_cpu.py)."""
    import torch
    from deepmimic_b200.env import DeepMimicBatchEnv
    from deepmimic_b200.rollout import BatchedRollout, build_gated_policy, load_actor_weights
    from tests.test_task_scenes_cpu import fixture_task_actor
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
    if task == "heading_getup":     # test mode: a fall starts a get-up instead of ending the episode; half of the start clips lie on the ground
        assert falls == 0 and float(traj["rewards"][300:].mean()) > 0.8, (falls, float(traj["rewards"][300:].mean()))
        assert float(traj["goals"][0, :, 3].max()) > 0.7 and float(traj["goals"][-1, :, 3].max()) < 0.5       # get-up phase: some start near 1 (lying down), nobody is still getting up at the end
    else:   # strike: episodes end with the success code 2 s after the hit and restart; code 1 also counts a forbidden body at the target and
        # falls from the run / backflip starts of the mini dataset (the oracle ends 9 of 12 such test episodes with code 1, 3 with code 2)
        succ = int((traj["terminate"] == 2).sum())
        assert succ >= 32 and falls <= 4 * succ, (succ, falls)


# ---------------------------------------------------------------------------------------------------------------- a. published bodies
def _forced_start(args, asset_root, core, envs, mode, lying=()):
    """one oracle per teacher-forced environment: reset on a non-get-up clip (0 / 3) at different times, the first two lifted 2 m (airborne),
    the ones in `lying` brought to the ground"""
    orcs = {}
    for k, e in enumerate(envs):
        o = _oracle(args, asset_root, core, e, mode)
        o.reset(0.1 + 0.17 * k, 0.3 * k, 20.0, clip=3 * (k % 2))
        if e in lying:
            _lying(o, 100 + k)
        elif k < 2:
            _airborne(o)
        orcs[e] = o
    return orcs


@pytest.mark.parametrize("head", range(NJ))
def test_getup_publishes_the_head_body_height(asset_root, head):
    """kXHeadY after every update is the COM height of body --head_id, for all 15 humanoid bodies, airborne and in ground contact"""
    args = getup_args(head=head)
    n, envs = 37, (0, 17, 36, 20)
    mode = head % 2
    core = _core(args, n, asset_root, seed=3 + head, offset=1000 + 7 * head, placement=head % 3 != 0, mode=mode)
    core.reset(True, kin_time=np.full(n, 0.2), max_time=np.full(n, 20.0), rot_theta=np.zeros(n), clip=np.zeros(n, dtype=np.int32))
    orcs = _forced_start(args, asset_root, core, envs, mode, lying=(20,))
    mirror = Oracle(args, asset_root)
    rng = np.random.default_rng(head)
    off, scl, lo, hi = mirror.action_statics()
    worst_m, worst_o, worst_ratio, cnt = 0.0, 0.0, 0.0, 0
    for upd in range(24):
        for e, o in orcs.items():
            if o.need_new_action() and e != 20:
                o.set_action(random_policy_action(rng, off, scl, lo, hi))
            _load(core, e, o)
        core.update(DT, 1)
        for e, o in orcs.items():
            o.update(DT)
            tb = core.task_state(e)
            pos_o = o.body_state()[0]
            pos_g, _, _ = _mirror_bodies(mirror, core, e)
            em = abs(tb[X_HEAD_Y] - pos_g[head, 1]); eo = abs(tb[X_HEAD_Y] - pos_o[head, 1])
            bound, _ = _pos_bound(pos_o, head)
            assert em <= 1e-4, (upd, e, tb[X_HEAD_Y], pos_g[head, 1])
            assert eo <= bound, (upd, e, eo, bound)
            worst_m, worst_o, worst_ratio = max(worst_m, em), max(worst_o, eo), max(worst_ratio, eo / bound)
            cnt += 1
    print("get-up head %d: %d updates, |head y - GPU state| max %.2e, |head y - oracle| max %.2e (%.2f of the bound)" % (head, cnt, worst_m, worst_o, worst_ratio))


STRIKE_BODIES = (0, 1, 4, 5, 8)     # root, a spherical child of the root, a revolute joint, a foot in ground contact, a fixed leaf (right wrist)


@pytest.mark.parametrize("regime", ["position", "velocity"])
@pytest.mark.parametrize("body", STRIKE_BODIES)
def test_strike_publishes_the_strike_and_forbidden_bodies(asset_root, body, regime):
    """kXNearR (0.2 exp(-s d^2) + 0.8 clamp(v / v_hit, 0, 1)^2 of the strike body) and kXContactFail (forbidden body inside the target sphere)
    after every update, for each body class, airborne and in ground contact.  position: --hit_tar_speed 1e6 leaves the distance term alone;
    velocity: the target along the body's horizontal velocity and v_hit = 6 m/s above its speed keep the velocity term unclamped."""
    vhit = 1e6 if regime == "position" else 6.0
    radius = 0.05
    args = strike_args(strike=(body,), fail=(body,), radius=radius, hit_speed=vhit)
    n, envs = 37, (0, 17, 36, 20)
    mode = 1 if regime == "velocity" else 0
    core = _core(args, n, asset_root, seed=5 + body, offset=3000 + body, placement=regime == "velocity", mode=mode)
    core.reset(True, kin_time=np.full(n, 0.2), max_time=np.full(n, 20.0), rot_theta=np.zeros(n), clip=np.zeros(n, dtype=np.int32))
    orcs = _forced_start(args, asset_root, core, envs, mode)
    mirror = Oracle(args, asset_root)
    rng = np.random.default_rng(body)
    off, scl, lo, hi = mirror.action_statics()
    worst_m = worst_o = worst_ratio = 0.0
    inside = outside = unclamped = contact_upd = 0
    for upd in range(30):
        for k, (e, o) in enumerate(orcs.items()):
            if o.need_new_action():
                o.set_action(random_policy_action(rng, off, scl, lo, hi))
            pos, _, lv, _ = o.body_state()
            root = o.get_snapshot()[0:3] / SCALE
            if regime == "position":
                if (upd + k) % 3 == 0:
                    tpos = pos[body] + lv[body] * DT                                     # where the body will be: inside the sphere
                else:
                    d = rng.standard_normal(3); tpos = pos[body] + rng.uniform(0.15, 0.5) * d / np.linalg.norm(d)
            else:
                vh = np.array([lv[body][0], 0.0, lv[body][2]])
                u = vh / np.linalg.norm(vh) if np.linalg.norm(vh) > 1e-3 else np.array([1.0, 0.0, 0.0])
                tpos = root + 0.8 * u; tpos[1] = pos[body][1]
            _set_target(o, tpos)
            _load(core, e, o)
        core.update(DT, 1)
        for e, o in orcs.items():
            o.update(DT)
            tb = core.task_state(e)
            tpos = np.array([tb[0], tb[X_TAR_Y], tb[1]])
            s = o.get_snapshot()
            contact = sum(LAY.contact_counts(s)) > 0
            contact_upd += contact
            pos_o, _, lv_o, av_o = o.body_state()
            root_o = s[0:3] / SCALE
            pos_g, lv_g, root_g = _mirror_bodies(mirror, core, e)
            want_m = _near_r(tpos, root_g, pos_g[body], lv_g[body], 2.0, vhit)
            want_o = _near_r(tpos, root_o, pos_o[body], lv_o[body], 2.0, vhit)
            dp, _ = _pos_bound(pos_o, body)
            bound = _near_bound(tpos, root_o, pos_o[body], lv_o[body], 2.0, vhit, dp, _vel_bound(pos_o, av_o, body, contact))
            em, eo = abs(tb[X_NEAR] - want_m), abs(tb[X_NEAR] - want_o)
            assert em <= 1e-4, (upd, e, tb[X_NEAR], want_m)
            assert eo <= bound, (upd, e, eo, bound)
            worst_m, worst_o, worst_ratio = max(worst_m, em), max(worst_o, eo), max(worst_ratio, eo / bound)
            if regime == "velocity":
                d = np.array([tpos[0] - root_g[0], 0.0, tpos[2] - root_g[2]])
                unclamped += 0.0 < float(d @ lv_g[body]) / np.linalg.norm(d) < vhit
            # forbidden body: a decision on the GPU's own state, away from the threshold by more than its fp32 rounding
            dist = np.linalg.norm(tpos - pos_g[body])
            if abs(dist - radius) > 1e-4:
                assert tb[X_CFAIL] == float(dist < radius), (upd, e, dist)
                inside += dist < radius; outside += dist >= radius
    print("strike body %d (%s): 120 updates (%d in contact), near term |GPU - GPU state| max %.2e, |GPU - oracle| max %.2e (%.2f of the bound); "
          "forbidden body inside %d / outside %d; unclamped velocity term %d" % (body, regime, contact_upd, worst_m, worst_o, worst_ratio, inside, outside, unclamped))
    assert 5 <= contact_upd <= 115
    if regime == "position":
        assert inside >= 20 and outside >= 40
    else:
        assert unclamped >= 60


# ---------------------------------------------------------------------------------------------------------------- b. strike decisions
def _check_step(core, orcs, g, r, f, rew_tol=5e-3, goal_tol=5e-3):
    worst = [0.0, 0.0]
    for e, o in orcs.items():
        assert tuple(f[e, 1:4]) == _flags_of(o), (e, f[e], _flags_of(o))
        er = abs(r[e] - o.calc_reward()); eg = float(np.abs(g[e] - o.record_goal()).max())
        assert er <= rew_tol and eg <= goal_tol, (e, r[e], o.calc_reward(), g[e], o.record_goal())
        worst = [max(worst[0], er), max(worst[1], eg)]
    return worst


@pytest.mark.parametrize("hit_speed", [1.5, 0.0])
@pytest.mark.parametrize("mode", [0, 1], ids=["train", "test"])
def test_strike_decisions_match_the_oracle_update_by_update(asset_root, mode, hit_speed):
    """Constructed cases, each clearly on one side of its threshold: a fast strike body inside the sphere hits, a slow one does not (unless
    --hit_tar_speed 0, where one moving away hits too); a forbidden body inside the sphere and a root beyond --tar_fail_dist end the episode
    with code 1; rewards in the hit, near and far regimes, fallen characters included.  Flags, reward and goal after every update, hit and hit
    time exactly."""
    args = strike_args(hit_speed=hit_speed)
    n = 37
    core = _core(args, n, asset_root, seed=31, offset=5000, placement=mode == 0, mode=mode)
    core.reset(True, kin_time=np.full(n, 0.2), max_time=np.full(n, 20.0), rot_theta=np.zeros(n), clip=np.zeros(n, dtype=np.int32))
    cases = ["fast", "slow", "away", "forbidden", "beyond", "within", "near", "far_fallen", "near_fallen"]
    envs = [0, 4, 9, 13, 18, 22, 27, 31, 36]
    orcs, case_of = {}, {}
    for k, (e, c) in enumerate(zip(envs, cases)):
        o = _oracle(args, asset_root, core, e, mode)
        o.reset(0.15 + 0.1 * k, 0.0, 20.0, clip=0)
        if c.endswith("fallen"):
            _lying(o, 7 + k)
        else:
            pos = o.body_state()[0]
            h = np.array([pos[8][0] - pos[0][0], 0.0, pos[8][2] - pos[0][2]]); h /= np.linalg.norm(h)
            _airborne(o, vel={"fast": 3.0, "slow": 0.3, "away": -3.0}.get(c, 0.0) * h)
        _set_clocks(o, timer_max=20.0)
        orcs[e] = o; case_of[e] = c
    for e, o in orcs.items():   # targets from the oracle's state
        c = case_of[e]
        pos, _, lv, _ = o.body_state()
        root = o.get_snapshot()[0:3] / SCALE
        if c in ("fast", "slow", "away"):
            tpos = pos[8] + lv[8] * DT
        elif c == "forbidden":
            tpos = pos[1] + lv[1] * DT
            assert np.linalg.norm(tpos - pos[8]) > 0.3
        elif c in ("beyond", "within", "far_fallen"):
            tpos = root + np.array([FAIL_DIST + (0.5 if c == "beyond" else -0.5 if c == "within" else -5.0), 0.0, 0.0]); tpos[1] = 1.3
        else:
            tpos = root + np.array([0.0, 0.0, 1.0]); tpos[1] = 1.3
        _set_target(o, tpos)
    hits = {}
    fallen_upd = dict(far_fallen=0, near_fallen=0)
    worst = [0.0, 0.0]
    for upd in range(24):
        for e, o in orcs.items():
            _load(core, e, o)
        core.update(DT, 1)
        for o in orcs.values():
            o.update(DT)
        g, r, f = _outputs(core)
        w = _check_step(core, orcs, g, r, f)
        worst = [max(worst[0], w[0]), max(worst[1], w[1])]
        for e, o in orcs.items():
            tb = core.task_state(e); ss = o.strike_state()
            assert bool(tb[X_HIT]) == ss["hit"], (upd, case_of[e])
            if ss["hit"]:
                assert abs(tb[X_HIT_TIME] - ss["hit_time"]) <= 1e-12
                assert g[e, 3] == pytest.approx(ss["phase"], abs=1e-6)
                hits.setdefault(case_of[e], upd)
            assert int(tb[K_COUNTER]) == o.task_counter()
        for e, o in orcs.items():
            c = case_of[e]
            if c.endswith("fallen"):
                fallen_upd[c] += o.has_fallen()
                if c == "far_fallen" and mode == 0 and o.has_fallen():
                    assert r[e] == 0.0
            elif upd == 0:   # the constructed decisions, on the first update
                assert f[e, 2] == (1 if c in ("forbidden", "beyond") else 0), (c, f[e])
                if mode == 1:
                    assert r[e] == 0.0
                elif c == "near":
                    assert 0.3 < r[e] < 0.6
                elif c == "within":
                    assert 0.0 <= r[e] < 0.3
    # the constructed decisions hold on the first update; later the PD controller swings the arm, and further hits are compared with the oracle
    want_hits = {"fast", "slow", "away"} if hit_speed == 0.0 else {"fast"}
    assert {c for c, u in hits.items() if u == 0} == want_hits, hits
    assert fallen_upd["far_fallen"] >= 4, fallen_upd
    if mode == 0:
        assert r[envs[0]] == 1.0   # the hit holds
    print("strike decisions (mode %d, hit speed %g): 24 updates x %d cases, hits %s, fallen updates %s, worst reward error %.2e, worst goal error %.2e"
          % (mode, hit_speed, len(cases), sorted(hits), fallen_upd, worst[0], worst[1]))


@pytest.mark.parametrize("mode", [0, 1], ids=["train", "test"])
def test_strike_success_lands_on_the_oracle_update(asset_root, mode):
    """A target hit at t_hit: terminate code 2 on the first update where scene_time - t_hit >= hit_reset_time, inside a 20-update launch.
    One case meets the threshold with equality (the f64 timers are exact: t0 in [2, 4) and t_hit = T_k - 2 make the difference exactly 2.0),
    the others half an update past it.  The test-mode reward is timer_max - scene_time at the success."""
    args = strike_args()
    n = 37
    core = _core(args, n, asset_root, seed=41, offset=7000, placement=True, mode=mode)
    core.reset(True, kin_time=np.full(n, 0.2), max_time=np.full(n, 20.0), rot_theta=np.zeros(n), clip=np.zeros(n, dtype=np.int32))
    cases = {0: (7, 0.0), 11: (7, 0.5), 23: (1, 0.5), 36: (13, 0.0), 30: (19, 0.5)}   # env: (update of the success, how far before it the threshold lies in dt)
    orcs, want = {}, {}
    for k, (e, (ks, frac)) in enumerate(cases.items()):
        o = _oracle(args, asset_root, core, e, mode)
        o.reset(0.2 + 0.1 * k, 0.0, 20.0, clip=0)
        _airborne(o)
        t0 = 2.5 + 0.1 * k
        _set_clocks(o, timer=t0, timer_max=20.0)
        T = t0
        for _ in range(ks):
            T += DT
        t_hit = (T - frac * DT) - HIT_RESET
        assert frac != 0.0 or T - t_hit == HIT_RESET
        root = o.get_snapshot()[0:3] / SCALE
        _set_target(o, root + np.array([0.0, 1.3, -3.0]), True, t_hit)
        _load(core, e, o)
        n_upd = 0
        while not o.is_episode_end() and n_upd < 20:
            o.update(DT); n_upd += 1
        assert o.check_terminate() == 2 and n_upd == ks, (e, n_upd, ks)
        orcs[e] = o; want[e] = n_upd
    core.update(DT, 20)
    g, r, f = _outputs(core)
    for e, o in orcs.items():
        s = core.get_snapshot(e)
        assert tuple(f[e, 1:4]) == (1, 2, 1), (e, f[e])
        assert s[CLK + 12] == o.get_snapshot()[CLK + 12], (e, s[CLK + 12], o.get_snapshot()[CLK + 12])   # ended on the same update
        assert g[e, 3] == pytest.approx(o.strike_state()["phase"], abs=1e-6)
        assert r[e] == pytest.approx(o.calc_reward(), abs=1e-5)
        if mode == 1:
            assert r[e] == pytest.approx(20.0 - s[CLK + 12], abs=1e-5) and r[e] > 17.0
    print("strike success (mode %d): the code-2 update of %d environments matches the oracle (%s)" % (mode, len(orcs), want))


# ---------------------------------------------------------------------------------------------------------------- c. get-up
@pytest.mark.parametrize("mode", [0, 1], ids=["train", "test"])
def test_getup_reset_timer_and_phase(asset_root, mode):
    """A reset into a get-up clip at kin_time k starts the get-up timer at k (phase 1 - k / getup_time); any other clip leaves it at the end
    (phase 0).  Timer, phase, draw counter and goal against the oracle under the same task stream."""
    args = GETUP
    n = 37
    core = _core(args, n, asset_root, seed=51, offset=9000, placement=mode == 1, mode=mode)
    kt = np.linspace(0.05, 0.9, n); clip = np.arange(n) % 4
    counters = [int(core.task_state(e)[K_COUNTER]) for e in range(n)]
    core.reset(True, kin_time=kt, max_time=np.full(n, 20.0), rot_theta=np.linspace(-2, 2, n), clip=clip)
    g, _, _ = _outputs(core)
    P, seed, base = core.task_params()
    getup_time = P[16]
    o = _oracle(args, asset_root, mode=mode)
    for e in range(n):
        o.set_task_stream(seed, base + e, counters[e])
        o.reset(kt[e], np.linspace(-2, 2, n)[e], 20.0, clip=int(clip[e]))
        tb = core.task_state(e)
        if clip[e] in (1, 2):
            assert tb[X_GETUP] == kt[e] and g[e, 3] == pytest.approx(1.0 - kt[e] / getup_time, abs=1e-6)
        else:
            assert tb[X_GETUP] == getup_time and g[e, 3] == 0.0   # the end of the get-up
        assert tb[X_GETUP] == pytest.approx(o.getup_state()["timer"], abs=1e-12) and int(tb[K_COUNTER]) == o.task_counter()
        np.testing.assert_allclose(g[e], o.record_goal(), atol=1e-5)


@pytest.mark.parametrize("mode", [0, 1], ids=["train", "test"])
def test_getup_fall_override_and_test_mode_restart(asset_root, mode):
    """Characters lying on the ground with fall-contact bodies: while the get-up timer runs, the episode does not end and the reward is the
    get-up reward; on the first update where the timer reaches getup_time with contact, train mode ends the episode with code 1 and test mode
    restarts the timer at 0 -- on the same update as the oracle.  A standing character past its get-up gets the heading reward."""
    args = GETUP
    n = 37
    core = _core(args, n, asset_root, seed=61, offset=11000, placement=mode == 0, mode=mode)
    core.reset(True, kin_time=np.full(n, 0.2), max_time=np.full(n, 20.0), rot_theta=np.zeros(n), clip=np.zeros(n, dtype=np.int32))
    P, _, _ = core.task_params()
    getup_time = P[16]
    cases = {0: 10.5, 12: 3.5, 25: None, 36: -1.0}   # env: updates until the get-up ends (lying), None: standing airborne, past the get-up; -1: lying, getting up throughout
    orcs = {}
    for k, (e, c) in enumerate(cases.items()):
        o = _oracle(args, asset_root, core, e, mode)
        o.reset(0.2 + 0.1 * k, 0.0, 20.0, clip=0)
        if c is None:
            _airborne(o)
        else:
            _lying(o, 40 + k)
        _set_clocks(o, timer=0.5, timer_max=20.0)
        o.set_getup_timer(getup_time + 1.0 if c is None else getup_time - (c if c > 0 else 60.0) * DT)
        orcs[e] = o
    ends = {}
    worst = [0.0, 0.0]
    for upd in range(24):
        for e, o in orcs.items():
            _load(core, e, o)
        core.update(DT, 1)
        for o in orcs.values():
            o.update(DT)
        g, r, f = _outputs(core)
        w = _check_step(core, orcs, g, r, f)
        worst = [max(worst[0], w[0]), max(worst[1], w[1])]
        for e, o in orcs.items():
            gs = o.getup_state()
            tb = core.task_state(e)
            assert tb[X_GETUP] == gs["timer"], (upd, e, tb[X_GETUP], gs["timer"])   # f64, same additions
            if cases[e] is not None:
                assert gs["contact_fall"], (upd, e)                                   # the construction: lying in contact throughout
            if gs["getting_up"]:
                ry = core.get_snapshot(e)[1] / SCALE
                assert f[e, 1] == 0 and r[e] == pytest.approx(0.2 * np.clip(ry / 1.2, 0, 1) + 0.8 * np.clip(tb[X_HEAD_Y] / 2.0, 0, 1), abs=1e-5)
            if cases[e] is not None and cases[e] > 0 and upd + 1 >= cases[e] and e not in ends:
                ends[e] = upd
                if mode == 0:
                    assert tuple(f[e, 1:3]) == (1, 1), (upd, e, f[e])
                else:
                    assert f[e, 1] == 0 and tb[X_GETUP] == 0.0, (upd, e, tb[X_GETUP])
    assert sorted(ends) == [0, 12] and ends[0] == 10 and ends[12] == 3, ends
    print("get-up (mode %d): 24 updates x 4 cases, worst reward error %.2e, worst goal error %.2e" % (mode, worst[0], worst[1]))


# ---------------------------------------------------------------------------------------------------------------- d. recovery episodes
@pytest.mark.parametrize("prob", [1.0, 0.5, 0.0])
def test_recovery_episodes_match_the_oracle(asset_root, prob):
    """Train mode, --recover_episode_prob p, 67 environments: two thirds brought to a fall (terminate 1), the rest ending on the time limit
    (code 0).  After reset(False) the recovery coins, draw counters, reset counters and the set of recovered environments match the oracle
    exactly; a recovered environment keeps its simulated state bit for bit (contact manifold included), target, heading and speed, restarts its
    clocks, flags, get-up timer and previous-action COM; its next 40 updates match the oracle teacher-forced.  With p = 1 a reset after
    switching to test mode recovers nobody."""
    args = getup_args(recover=prob)
    n = 67
    core = _core(args, n, asset_root, seed=71, offset=13000, placement=prob == 0.5, mode=0)
    kt = np.linspace(0.1, 0.5, n); clip = np.where(np.arange(n) % 2 == 0, 0, 3).astype(np.int32)
    core.reset(True, kin_time=kt, max_time=np.full(n, 20.0), rot_theta=np.zeros(n), clip=clip)
    orcs = {}
    fall = [e for e in range(n) if e % 3 != 2]
    for e in range(n):
        o = _oracle(args, asset_root, core, e, 0)
        o.reset(kt[e], 0.0, 20.0, clip=int(clip[e]))
        if e in fall:
            _lying(o, 200 + e)
            _set_clocks(o, timer=0.3, timer_max=20.0)
        else:
            _airborne(o)
            _set_clocks(o, timer=0.3, timer_max=0.3 + 0.5 * DT)
        orcs[e] = o
    for e, o in orcs.items():
        _load(core, e, o)
    core.update(DT, 1)
    for o in orcs.values():
        o.update(DT)
    _, _, f = _outputs(core)
    for e, o in orcs.items():
        assert tuple(f[e, 1:4]) == _flags_of(o) == (1, 1 if e in fall else 0, 1), (e, f[e], _flags_of(o))
    before = {e: core.get_snapshot(e) for e in range(n)}
    tb_before = {e: core.task_state(e) for e in range(n)}
    o_before = {e: o.get_snapshot() for e, o in orcs.items()}
    kt2 = np.linspace(0.2, 0.6, n); mt2 = 5.0 + 0.01 * np.arange(n); clip2 = ((np.arange(n) + 1) % 4).astype(np.int32)
    core.reset(False, kin_time=kt2, max_time=mt2, rot_theta=np.zeros(n), clip=clip2)
    for e, o in orcs.items():
        o.reset(kt2[e], 0.0, mt2[e], clip=int(clip2[e]))
    rec_g, rec_o = [], []
    for e, o in orcs.items():
        s, so = core.get_snapshot(e), o.get_snapshot()
        tb = core.task_state(e)
        assert int(tb[K_COUNTER]) == o.task_counter(), e
        assert int(tb[K_RESET_SEEN]) == int(tb_before[e][K_RESET_SEEN]) + 1, e
        if np.array_equal(so[:CLK], o_before[e][:CLK]):
            rec_o.append(e)
        if np.array_equal(s[:CLK], before[e][:CLK]):
            rec_g.append(e)
    assert rec_g == rec_o, (rec_g, rec_o)
    assert set(rec_g) <= set(fall)
    if prob == 1.0:
        assert rec_g == fall
    elif prob == 0.0:
        assert rec_g == []
    else:
        assert 0 < len(rec_g) < len(fall)
    _, _, f = _outputs(core)
    for e in rec_g:
        s, tb = core.get_snapshot(e), core.task_state(e)
        assert np.array_equal(s[CLK + 16:], before[e][CLK + 16:])                             # PD targets kept
        assert np.array_equal(s[CLK:CLK + 8], before[e][CLK:CLK + 8])                         # kinematic time and origin kept
        assert (s[CLK + 8], s[CLK + 9], s[CLK + 10], s[CLK + 11], s[CLK + 12], s[CLK + 13]) == (0.0, 0.0, 0.0, 1.0, 0.0, mt2[e])
        assert tuple(f[e]) == (1, 0, 0, 1)
        assert tb[X_GETUP] == 0.0 and np.all(tb[6:9] == 0.0) and tb[X_RECOVER] == 0.0
        assert np.array_equal(tb[0:6], tb_before[e][0:6])                                      # target, speed, heading, target timer
    for e in range(n):
        if e not in rec_g:
            assert core.get_snapshot(e)[CLK + 8] == kt2[e]                                     # a normal reset
    # the recovered characters' next 40 updates, teacher-forced
    sub = {e: orcs[e] for e in rec_g[:6]}
    worst = [0.0, 0.0]
    for upd in range(40):
        for e, o in sub.items():
            _load(core, e, o)
        core.update(DT, 1)
        for o in sub.values():
            o.update(DT)
        g, r, f = _outputs(core)
        w = _check_step(core, sub, g, r, f)
        worst = [max(worst[0], w[0]), max(worst[1], w[1])]
        for e, o in sub.items():
            assert core.task_state(e)[X_GETUP] == o.getup_state()["timer"]
    print("recovery p=%g: %d fell, %d recovered (GPU and oracle), 40 updates of %d recovered: worst reward error %.2e, goal %.2e"
          % (prob, len(fall), len(rec_g), len(sub), worst[0], worst[1]))
    if prob == 1.0:   # a reset in test mode never recovers
        for e in fall:
            o = orcs[e]
            _lying(o, 300 + e)
            _set_clocks(o, timer=0.3, timer_max=20.0)
            o.set_getup_timer(100.0)
            _load(core, e, o)
        core.update(DT, 1)
        for e in fall:
            orcs[e].update(DT)
        _, _, f = _outputs(core)
        fell = [e for e in fall if orcs[e].check_terminate() == 1]
        assert len(fell) >= 10 and all(tuple(f[e, 1:4]) == _flags_of(orcs[e]) for e in fall)
        before = {e: core.get_snapshot(e) for e in fell}
        core.set_mode(1)
        core.reset(False, kin_time=kt2, max_time=mt2, rot_theta=np.zeros(n), clip=clip2)
        for e in fell:
            orcs[e].set_mode(1)
            orcs[e].reset(kt2[e], 0.0, mt2[e], clip=int(clip2[e]))
            assert not np.array_equal(core.get_snapshot(e)[:CLK], before[e][:CLK])
            assert int(core.task_state(e)[K_COUNTER]) == orcs[e].task_counter()


# ---------------------------------------------------------------------------------------------------------------- e. strike reset draws
@pytest.mark.parametrize("mode", [0, 1], ids=["train", "test"])
def test_strike_reset_draws_match_the_oracle(asset_root, mode):
    """259 environments at a global id above 2^31, two forced resets with given clips: target position (far and near regime), initial hit and
    its time in [-hit_reset_time, 0] (train only), draw counter, target timer and the goal after the reset, against the oracle under the same
    task stream: counters exactly, f64 values to 1e-9"""
    args = STRIKE
    n = 259
    core = _core(args, n, asset_root, seed=2024, offset=2 ** 31 + 12345, placement=mode == 0, mode=mode)
    P, seed, base = core.task_params()
    assert base == 2 ** 31 + 12345
    o = _oracle(args, asset_root, mode=mode)
    far = near = init_hits = 0
    for rnd in range(2):
        kt = np.linspace(0.05, 0.8, n)[::(1 if rnd == 0 else -1)].copy(); th = np.linspace(-3.0, 3.0, n); mt = np.full(n, 20.0)
        clip = ((np.arange(n) + rnd) % 4).astype(np.int32)
        counters = [int(core.task_state(e)[K_COUNTER]) for e in range(n)]
        core.reset(True, kin_time=kt, max_time=mt, rot_theta=th, clip=clip)
        g, _, _ = _outputs(core)
        for e in range(n):
            o.set_task_stream(seed, base + e, counters[e])
            o.reset(kt[e], th[e], mt[e], clip=int(clip[e]))
            tb = core.task_state(e); ts = o.task_state(); ss = o.strike_state()
            assert int(tb[K_COUNTER]) == o.task_counter(), (rnd, e)
            # the target hangs off the root position of the fp32 state (as in the host shim test): x, z to 1e-7; the rest is f64 draws
            assert abs(tb[0] - ts["target_pos"][0]) <= 1e-7 and abs(tb[1] - ts["target_pos"][2]) <= 1e-7
            assert abs(tb[X_TAR_Y] - ss["target_height"]) <= 1e-9
            assert bool(tb[X_HIT]) == ss["hit"] and abs(tb[X_HIT_TIME] - ss["hit_time"]) <= 1e-9
            assert tb[4] == 0.0 and abs(tb[5] - ts["timer_max"]) <= 1e-9
            np.testing.assert_allclose(g[e], o.record_goal(), atol=2e-5, rtol=1e-5)
            if ss["hit"]:
                init_hits += 1
                assert -HIT_RESET <= tb[X_HIT_TIME] <= 0.0
            else:
                assert tb[X_HIT_TIME] == -1.0
            # the regime coin is the draw after the target timer's
            is_far = o.u01(seed, base + e, counters[e] + 1) < 0.4
            far += is_far; near += not is_far
    print("strike resets (mode %d): %d far / %d near targets, %d initial hits" % (mode, far, near, init_hits))
    assert far > 100 and near > 200
    assert (init_hits > 20) if mode == 0 else (init_hits == 0)


# ---------------------------------------------------------------------------------------------------------------- f. state round trip
@pytest.mark.parametrize("scene", ["strike", "getup"])
def test_save_and_load_state_mid_hit_hold_and_mid_getup(asset_root, scene):
    """The whole batch saved in the middle of a hit hold (strike) or of a get-up, loaded into a fresh handle: the next 40 updates give
    bit-identical goals, rewards, flags and task blocks on both handles"""
    import torch
    args = STRIKE if scene == "strike" else GETUP
    n = 37
    a, b = (_core(args, n, asset_root, seed=81, offset=15000, placement=True) for _ in range(2))
    kt = np.linspace(0.1, 0.7, n); clip = (np.arange(n) % 4).astype(np.int32)
    a.reset(True, kin_time=kt, max_time=np.full(n, 20.0), rot_theta=np.zeros(n), clip=clip)
    a.update(DT, 5)
    a.sync()
    for e in range(n):
        tb = a.task_state(e)
        if scene == "strike":   # every environment holds a hit made 0.5 s ago
            tb[X_HIT], tb[X_HIT_TIME] = 1.0, a.get_snapshot(e)[CLK + 12] - 0.5
        a.set_task_state(e, tb)
    if scene == "getup":
        assert sum(a.task_state(e)[X_GETUP] < 1.0 for e in range(n)) >= 10   # half of the environments are getting up
    b.load_state(a.save_state())
    rng = np.random.default_rng(3)
    for upd in range(40):
        if upd % 20 == 0:
            act = torch.as_tensor(0.1 * rng.standard_normal((n, a.dims.action_size)), dtype=torch.float32, device="cuda")
            for c in (a, b):
                c.set_action(act)
        outs = []
        for c in (a, b):
            c.update(DT, 1)
            outs.append(_outputs(c) + (np.stack([c.task_state(e) for e in range(n)]),))
        for x, y in zip(*outs):
            assert np.array_equal(x, y), upd

