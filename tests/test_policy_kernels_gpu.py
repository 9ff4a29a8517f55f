"""The policy-rate kernels of dm_policy.cu against the CPU oracle, branch by branch: dm_observe_kernel (state observation and imitation
reward) and dm_reset_kernel, on the constructed inputs of tests/policy_states.py (checked to reach their branches by
tests/test_policy_states_cpu.py).

Observations and rewards are pure functions of one state: the oracle's simulator snapshot is loaded into the environment, then observe.
Tolerances (DESIGN.md section 4): observation <= 2e-4, reward <= 2e-5; reset q <= 2e-5, qd <= 2e-4, clocks <= 1e-12; flags and counters
exact.  Where the root's x axis is within 5 degrees of vertical the heading (atan2 of the axis' horizontal part) is ill-conditioned in fp32:
such states are held to the tolerance plus a first-order term of a heading error of 1e-6 / |horizontal part| rad, and counted."""
import numpy as np
import pytest

from tests import policy_states as P
from tests.oracle_binding import Oracle
from tests.parity_util import SnapLayout, compare_sim_state, joint_types_from_assets, quat_err

pytestmark = pytest.mark.gpu

DT = P.DT
OBS_TOL, REW_TOL, Q_TOL, QD_TOL, CLOCK_TOL = 2e-4, 2e-5, 2e-5, 2e-4, 1e-12
COND_MIN = np.sin(np.radians(5.0))
CLOCKS = (0, 8, 9, 10, 12, 13)          # snapshot clocks: kin time, ctrl, init offset, prev action, timer, timer max
HEADER_BYTES = 160                       # dm_save_state's header


@pytest.fixture(scope="module")
def assets(asset_root, tmp_path_factory):
    return P.make_assets(asset_root, str(tmp_path_factory.mktemp("policy") / "assets"))


def _core(args, n, assets, seed=5, mode=0):
    from deepmimic_b200 import capi
    core = capi.BatchedCore(args, n, assets, seed=seed, global_env_offset=0)
    core.set_mode(mode)
    return core


def _heading_cond(snap):
    """|horizontal part| of the simulated root's x axis (the snapshot holds the world->base quaternion, the root rotation's inverse)"""
    qx, qy, qz, qw = -snap[3], -snap[4], -snap[5], snap[6]
    return float(np.hypot(1.0 - 2.0 * (qy * qy + qz * qz), 2.0 * (qx * qz - qw * qy)))


def _obs_bound(snap, ref):
    c = _heading_cond(snap)
    return (OBS_TOL, False) if c >= COND_MIN else (OBS_TOL + 1e-6 / c * max(1.0, float(np.abs(ref).max())), True)


def _rew_bound(snap):
    # d reward / d heading <= 0.15 * 10 * 2 * sum |rel end effector|^2 <= 12 (four end effectors within 1 m of the root)
    c = _heading_cond(snap)
    return (REW_TOL, False) if c >= COND_MIN else (REW_TOL + 12.0 * 1e-6 / c, True)


def _np(t):
    return t.cpu().numpy().astype(np.float64)


# ---------------------------------------------------------------------------------------------------------------- observation layouts
@pytest.mark.parametrize("ctrl", P.CTRLS, ids=["%s-phase%d-rot%d%s" % (c, p, r, "-wpos" if w else "") for c, p, r, w in P.CTRLS])
def test_observation_layouts_match_the_oracle(assets, ctrl):
    """every combination of phase input and world root rotation (and world root position) on standing, walking, airborne and lying states
    at several headings; W = 16 (humanoid3d) and W = 32 (dog3d); two NaN guard rows after the last row keep their NaN"""
    import torch
    args = P.ctrl_args(*ctrl)
    o = Oracle(args, assets)
    states = P.observation_states(o)
    n = len(states)
    core = _core(args, n, assets)
    S = core.dims.state_size
    assert S == o.state_size
    for e, s in enumerate(states):
        core.set_snapshot(e, s.snap)
    obs = torch.full((n + 2, S), float("nan"), device="cuda")
    torch.cuda.synchronize()   # the buffers are written on the handle's own stream
    core.observe(obs, None)
    core.sync()
    g = _np(obs)
    assert np.isnan(g[n:]).all(), "observe wrote past row N"
    worst, ill = 0.0, 0
    for e, s in enumerate(states):
        o.set_snapshot(s.snap)
        ref = o.record_state()
        bound, is_ill = _obs_bound(s.snap, ref)
        ill += is_ill
        err = float(np.abs(g[e] - ref).max())
        assert err <= bound, (s.name, err, bound, int(np.abs(g[e] - ref).argmax()))
        if not is_ill:
            worst = max(worst, err)
    print("%s: %d states, worst observation error %.2e, %d with an ill-conditioned heading" % (ctrl, n, worst, ill))
    core.close()


# ---------------------------------------------------------------------------------------------------------------- imitation reward
REWARD_CLIPS = [P.WALK, P.SPINKICK, P.BACKFLIP, P.FACEDOWN, P.FACEUP, P.WALK_ONCE]


@pytest.mark.parametrize("motion", REWARD_CLIPS, ids=[m.split("/")[-1][:-4] for m in REWARD_CLIPS])
def test_imitation_reward_matches_the_oracle_on_constructed_states(assets, motion):
    """the imitation reward of one state in the imitate scene on one clip: inside an antipodal and a held-frame interval of eigen_slerp,
    cycles 0, 1, 5 and 9 of a looping clip, 0 / inside / exactly the end / past the end of a non-looping one; each on the clip (pose
    differences in the QuatTheta dead zone) and near it.  dm_calc_reward_imitate gives the same bits as dm_observe's reward."""
    import torch
    args = P.imitate_args(motion)
    o = Oracle(args, assets)
    states = P.reward_states(o, P.clip_times(assets, motion))
    n = len(states)
    core = _core(args, n, assets)
    for e, s in enumerate(states):
        core.set_snapshot(e, s.snap)
    rw = torch.full((n + 2,), float("nan"), device="cuda"); ri = torch.full((n + 2,), float("nan"), device="cuda")
    torch.cuda.synchronize()
    core.observe(None, rw)
    core.reward_imitate(ri)
    core.sync()
    g, gi = _np(rw), _np(ri)
    assert np.isnan(g[n:]).all() and np.isnan(gi[n:]).all()
    assert g[:n].tobytes() == gi[:n].tobytes()
    worst, ill = 0.0, 0
    for e, s in enumerate(states):
        o.set_snapshot(s.snap)
        assert not o.has_fallen(), s.name
        ref = o.calc_reward()
        bound, is_ill = _rew_bound(s.snap)
        ill += is_ill
        err = abs(g[e] - ref)
        assert err <= bound, (s.name, g[e], ref, o.reward_terms())
        if not is_ill:
            worst = max(worst, err)
    print("%s: %d states, worst reward error %.2e, %d with an ill-conditioned heading" % (motion, n, worst, ill))
    core.close()


def test_fallen_character_earns_no_imitation_reward(assets):
    """set_snapshot clears the fallen flag, so the fallen states are reached through one teacher-forced update of lying characters: the
    oracle has fallen, the device flags the fall (terminate 1, done) and both rewards are exactly 0"""
    import torch
    args = P.imitate_args(P.WALK)
    o = Oracle(args, assets)
    snaps = [P.lying(o, 300 + k, 0.1 + 0.3 * k, 1.1 * k - 1.5) for k in range(4)]
    n = len(snaps)
    core = _core(args, n, assets)
    for e, s in enumerate(snaps):
        core.set_snapshot(e, s)
    core.update(DT, 1)
    rw = torch.full((n,), float("nan"), device="cuda"); fl = torch.zeros(n, 4, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    core.observe(None, rw)
    core.flags(fl)
    core.sync()
    g, f = _np(rw), fl.cpu().numpy()
    for e, s in enumerate(snaps):
        o.set_snapshot(s)
        o.update(DT)
        assert o.has_fallen() and o.calc_reward() == 0.0
        assert f[e, 1] == 1 and f[e, 2] == o.check_terminate() == 1, (e, f[e])
        assert g[e] == 0.0, (e, g[e])
    core.close()


@pytest.mark.parametrize("scene", list(P.CLIPS_ARGS))
def test_clips_imitation_reward_matches_the_oracle(assets, scene):
    """--kin_ctrl clips (heading_amp on the two-clip dataset, heading_amp_getup on the archive's get-up dataset): the imitation reward against
    the environment's own clip for every clip of the dataset -- reset with the clip injected, then the oracle's snapshot -- at 0, inside,
    the end, past the end, and cycles 1 and 5 of the looping clips"""
    import torch
    args = P.CLIPS_ARGS[scene]
    o = Oracle(args, assets)
    dur, _, _, loop = o.clip_table()
    grid = []
    for c in range(len(dur)):
        times = [0.0, 0.47 * dur[c], dur[c], dur[c] + 0.37] + ([1.31 * dur[c], 5.23 * dur[c]] if loop[c] else [])
        grid += [(c, kt, near) for kt in times for near in (False, True)]
    n = len(grid)
    core = _core(args, n, assets)
    kin = np.array([kt for _, kt, _ in grid]); th = np.linspace(-2.9, 2.9, n); clip = np.array([c for c, _, _ in grid], dtype=np.int32)
    core.reset(True, kin_time=kin, max_time=np.full(n, 20.0), rot_theta=th, clip=clip)
    refs, snaps = [], []
    for e, (c, kt, near) in enumerate(grid):
        o.reset(kt, th[e], 20.0, clip=c)
        if near:
            o.set_action(np.zeros(o.action_size) - o.action_statics()[0])
            for _ in range(4):
                o.update(DT)
        snaps.append(o.get_snapshot())
        refs.append(None if o.has_fallen() else o.calc_reward_imitate())
        core.set_snapshot(e, snaps[-1])
    ri = torch.full((n + 1,), float("nan"), device="cuda")
    torch.cuda.synchronize()
    core.reward_imitate(ri)
    core.sync()
    g = _np(ri)
    assert np.isnan(g[n]) and all(core.task_state(e)[13] >= 1 for e in range(n))
    worst, ill, compared = 0.0, 0, 0
    for e, (c, kt, near) in enumerate(grid):
        if refs[e] is None:
            continue
        bound, is_ill = _rew_bound(snaps[e])
        ill += is_ill
        assert abs(g[e] - refs[e]) <= bound, (scene, c, kt, near, g[e], refs[e])
        worst = max(worst, 0.0 if is_ill else abs(g[e] - refs[e]))
        compared += 1
    print("%s: %d of %d states compared (the rest have fallen in the oracle), worst reward error %.2e, %d ill-conditioned" % (scene, compared, n, worst, ill))
    assert compared >= n - 4
    core.close()


# ---------------------------------------------------------------------------------------------------------------- reset
def _blob(core):
    """dm_save_state's first per-environment blocks -- sim, time, flags, contact manifold, AMP history -- as [padded_envs, bytes] views, and
    the padded environment count"""
    b = core.save_state()
    pe, nl = int(b[28:32].view(np.int32)[0]), int(b[36:40].view(np.int32)[0])
    sizes = [(16 + 12 * nl) * 4, 16 * 8, 8 * 4, nl * 48 * 4, 2 * core.dims.pose_dim * 4]
    out, off = [], HEADER_BYTES
    for s in sizes:
        out.append(b[off:off + pe * s].reshape(pe, s))
        off += pe * s
    return out, pe


def _reset_counter(blocks, e):
    return int(blocks[2][e].view(np.int32)[7])


def _check_reset(o, core, e, lay, jt, what):
    so, sg = o.get_snapshot(), core.get_snapshot(e)
    eq, eqd = compare_sim_state(lay, so, sg, jt)
    assert eq <= Q_TOL and eqd <= QD_TOL, (what, eq, eqd)
    q = lay.scal
    ck = max(abs(so[q + k] - sg[q + k]) for k in CLOCKS)
    assert ck <= CLOCK_TOL, (what, [(so[q + k], sg[q + k]) for k in CLOCKS])
    assert np.abs(so[q + 1:q + 4] - sg[q + 1:q + 4]).max() <= Q_TOL and quat_err(so[q + 4:q + 8], sg[q + 4:q + 8]) <= Q_TOL, (what, so[q:q + 8], sg[q:q + 8])
    assert sg[q + 11] == so[q + 11] == 1
    assert not sg[lay.mani:lay.scal].any(), (what, "manifold not empty")
    return eq, eqd


def _reset_and_compare(core, o, args, assets, ch, kin, th, mt, clip, mode, what):
    import torch
    n = len(kin)
    before, _ = _blob(core)
    core.reset(True, kin_time=kin, max_time=mt, rot_theta=th, clip=clip)
    after, pe = _blob(core)
    fl = torch.zeros(n, 4, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    core.flags(fl)
    core.sync()
    f = fl.cpu().numpy()
    lay, jt = SnapLayout(o.num_joints), joint_types_from_assets(assets, P.CHAR_FILE[ch])
    worst_q = worst_qd = 0.0
    for e in range(n):
        if clip is None:
            o.reset(kin[e], th[e], mt[e])
        else:
            o.reset(kin[e], th[e], mt[e], clip=int(clip[e]))
        eq, eqd = _check_reset(o, core, e, lay, jt, (what, e, kin[e], th[e], None if clip is None else clip[e]))
        worst_q, worst_qd = max(worst_q, eq), max(worst_qd, eqd)
        assert tuple(f[e]) == (1, 0, 0, 1), (what, e, f[e])
        assert _reset_counter(after, e) == _reset_counter(before, e) + 1
    for e in range(n, pe):   # the padding environments stay frozen
        assert all(b[e].tobytes() == a[e].tobytes() for b, a in zip(before, after)), (what, "padding", e)
    return worst_q, worst_qd


RESET_CASES = {"walk": ("humanoid3d", P.WALK), "walk_once": ("humanoid3d", P.WALK_ONCE), "faceup": ("humanoid3d", P.FACEUP),
               "spinkick": ("humanoid3d", P.SPINKICK), "dog": ("dog3d", None)}


def reset_times(assets, case, dur):
    """start times of the reset grid: inside the clip, at and past the end, several cycles on; the faceup times include poses the oracle
    lifts off the ground and poses it leaves; spinkick's include its antipodal interval"""
    if case == "walk":
        return [0.0, 0.31, 0.9 * dur, 1.5 * dur, 5.4 * dur]
    if case == "walk_once":
        return [0.0, 0.6, dur, dur + 0.4, 2.5]
    if case == "faceup":
        return [0.0, 0.5, 1.64, 1.97, 2.62, 3.11, dur, dur + 0.5]
    if case == "spinkick":
        a, b, _ = P.intervals(assets, P.SPINKICK, "antipodal")[0]
        return [0.5 * (a + b), 0.6, 1.9]
    return [0.0, 0.2, 0.55, 1.3 * dur]


@pytest.mark.parametrize("mode", [0, 1], ids=["train", "test"])
@pytest.mark.parametrize("rand_rot", [True, False], ids=["rand_rot", "no_rot"])
@pytest.mark.parametrize("case", list(RESET_CASES))
def test_reset_matches_the_oracle(assets, case, rand_rot, mode):
    """grids of start time x theta with --enable_rand_rot_reset on (theta used) and off (theta ignored), train mode (the injected episode
    length) and test mode (the timer maximum): simulated state, clocks, kinematic origin, flags, reset counter, empty manifold, frozen padding"""
    ch, motion = RESET_CASES[case]
    args = (P.imitate_args(motion, rand_rot) if motion else ["--enable_rand_rot_reset", "true" if rand_rot else "false", "--arg_file", P.TROT_ARGS])
    o = Oracle(args, assets)
    o.set_mode(mode)
    times = reset_times(assets, case, o.motion_duration)
    grid = [(kt, th) for kt in times for th in (0.0, 2.5, -3.0)]
    n = len(grid)
    core = _core(args, n, assets, mode=mode)
    kin, th = np.array([g[0] for g in grid]), np.array([g[1] for g in grid])
    mt = np.linspace(3.0, 9.0, n)
    q, qd = _reset_and_compare(core, o, args, assets, ch, kin, th, mt, None, mode, case)
    print("reset %s rand_rot=%s mode=%d: %d environments, |dq| %.2e |dqd| %.2e" % (case, rand_rot, mode, n, q, qd))
    core.close()


@pytest.mark.parametrize("mode", [0, 1], ids=["train", "test"])
@pytest.mark.parametrize("scene", list(P.CLIPS_ARGS))
def test_task_scene_reset_matches_the_oracle(assets, scene, mode):
    """task-scene resets with the clip injected: every clip of the dataset, start times inside, at and past the new clip's end -- past the
    end of a looping clip the cycle offset goes into the kinematic origin, past the end of a non-looping one the character starts at rest"""
    args = P.CLIPS_ARGS[scene]
    o = Oracle(args, assets)
    o.set_mode(mode)
    dur = o.clip_table()[0]
    grid = [(c, kt, th) for c in range(len(dur)) for kt in (0.0, 0.55, dur[c], 2.0, 3.5) for th in (0.4, -2.7)]
    n = len(grid)
    core = _core(args, n, assets, mode=mode)
    clip = np.array([g[0] for g in grid], dtype=np.int32); kin = np.array([g[1] for g in grid]); th = np.array([g[2] for g in grid])
    q, qd = _reset_and_compare(core, o, args, assets, "humanoid3d", kin, th, np.linspace(3.0, 9.0, n), clip, mode, scene)
    print("task reset %s mode=%d: %d environments, |dq| %.2e |dqd| %.2e" % (scene, mode, n, q, qd))
    core.close()


@pytest.mark.parametrize("scene", ["imitate", "task"])
def test_reset_past_the_end_of_a_non_looping_clip_starts_at_rest(assets, scene):
    """a non-looping clip that ends in motion (the walk with "Loop": "none"), started at and past its end: the oracle's CalcFrameVel returns
    zero velocities there, so the reset character is at rest -- root and joints, exactly"""
    args = P.imitate_args(P.WALK_ONCE) if scene == "imitate" else P.CLIPS_ARGS["heading_pair"]
    o = Oracle(args, assets)
    clip = None if scene == "imitate" else np.ones(4, dtype=np.int32)
    d = o.motion_duration if scene == "imitate" else o.clip_table()[0][1]
    kin = np.array([d, d + 1e-9, d + 0.4, 3.5])
    core = _core(args, 4, assets)
    core.reset(True, kin_time=kin, max_time=np.full(4, 20.0), rot_theta=np.array([0.0, 1.0, -2.0, 3.0]), clip=clip)
    lay = SnapLayout(o.num_joints)
    for e in range(4):
        s = core.get_snapshot(e)
        assert not s[lay.base_omega].any() and not s[lay.base_vel].any() and not s[lay.jvel:lay.mani].any(), (scene, kin[e], s[7:13])
    core.close()


# ---------------------------------------------------------------------------------------------------------------- batch edges
@pytest.mark.parametrize("ch,n", [("humanoid3d", 37), ("humanoid3d", 1001), ("dog3d", 33)])
def test_selective_reset_and_batch_edges(assets, ch, n):
    """N not a multiple of the tiles per block: every observation row, reward and imitation reward equals the same snapshot evaluated in
    environment 0, bit for bit, and NaN guard rows after row N keep their NaN; reset(force_all=False) resets exactly the done environments
    (compared with the oracle) and leaves every other environment -- the W = 16 warp partner included -- and the padding bit-identical"""
    import torch
    args = P.ctrl_args(ch, 1, 1)
    o = Oracle(args, assets)
    pool = [s.snap for s in P.observation_states(o)]
    K = len(pool)
    core = _core(args, n, assets, seed=11)
    S = core.dims.state_size
    for e in range(n):
        core.set_snapshot(e, pool[e % K])
    G = 3
    obs = torch.full((n + G, S), float("nan"), device="cuda"); rw = torch.full((n + G,), float("nan"), device="cuda")
    ri = torch.full((n + G,), float("nan"), device="cuda")
    torch.cuda.synchronize()
    core.observe(obs, rw)
    core.reward_imitate(ri)
    core.sync()
    go, gr, gi = obs.cpu().numpy(), rw.cpu().numpy(), ri.cpu().numpy()
    assert np.isnan(go[n:]).all() and np.isnan(gr[n:]).all() and np.isnan(gi[n:]).all()
    o1 = torch.zeros(n, S, device="cuda"); r1 = torch.zeros(n, device="cuda")
    torch.cuda.synchronize()
    ref = []
    for k in range(K):
        core.set_snapshot(0, pool[k])
        core.observe(o1, r1)
        core.sync()
        ref.append((o1[0].cpu().numpy().copy(), r1[0].cpu().numpy().copy()))
    for e in range(n):
        ro, rr = ref[e % K]
        assert go[e].tobytes() == ro.tobytes() and gr[e].tobytes() == rr.tobytes() == gi[e].tobytes(), e
    # selective reset: environments 0, 2 mod 5 and the last one reach their episode's time limit in the next update
    timed_out = [e for e in range(n) if e == 0 or e % 5 == 2 or e == n - 1]
    lay = SnapLayout(o.num_joints)
    for e in range(n):
        s = pool[e % K].copy()
        if e in timed_out:
            s[lay.scal + 12] = s[lay.scal + 13] = 1.0
        else:
            s[lay.scal + 12], s[lay.scal + 13] = 0.0, 100.0
        core.set_snapshot(e, s)
    core.update(DT, 1)
    fl = torch.zeros(n, 4, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    core.flags(fl)
    core.sync()
    done = np.nonzero(fl.cpu().numpy()[:, 1])[0]
    assert set(timed_out) <= set(done.tolist())
    if core.dims.num_joints <= 16:
        assert 1 not in done    # environment 0's warp partner
    before, pe = _blob(core)
    kin = (0.137 * np.arange(n)) % o.motion_duration; th = np.linspace(-3.0, 3.0, n); mt = np.linspace(2.0, 8.0, n)
    core.reset(False, kin_time=kin, max_time=mt, rot_theta=th)
    after, _ = _blob(core)
    jt = joint_types_from_assets(assets, P.CHAR_FILE[ch])
    for e in range(pe):
        same = all(b[e].tobytes() == a[e].tobytes() for b, a in zip(before, after))
        if e in done:
            assert not same and _reset_counter(after, e) == _reset_counter(before, e) + 1
        else:
            assert same, ("environment %d changed without being done" % e)
    for e in done[:: max(1, len(done) // 40)]:
        o.reset(kin[e], th[e], mt[e])
        _check_reset(o, core, int(e), lay, jt, ("selective", int(e)))
    core.close()
