"""The target_amp / heading_amp device code against the oracle on the constructed inputs of tests/task_states.py: the step kernel's TASK glue
(COM after the update and at the new action, target timer, redraw around the root, distance failure) in its plain, push and dynamics-table
instantiations, dm_task_reset_kernel and dm_task_observe_kernel.

Teacher-forced (the protocol of tests/test_task_ext_gpu.py): before every update the oracle's snapshot and task block, draw counter included,
are loaded into the environment.  Two comparisons per update:

1. the logic on the GPU's own state: a second oracle loaded with the GPU's post-update snapshot and task block evaluates goal, reward and COM.
   Only the device's fp32 COM separates the two.  It is a mass-weighted sum of the link COM positions of the fp32 forward kinematics: each
   position the end of about 32 fp32 operations per tree level, the sum 2 nl more, so |d com| <= n u S per component with n = 32 maxlevel +
   2 nl = 158 (humanoid3d: maxlevel 4, 15 links), u = 2^-24 and S = max(1, |com|) (DC below).  The reward's bound is that error of the COM
   after the update through the reward's first derivative (central differences of the float64 restatement task_states.ref_reward), plus
   the float32 rounding of the output, u |r|; the previous-action COM is the GPU's own kKPrevCom on both sides.  The goal is computed in double from the same fp32 root on both
   sides: its bound is the float32 rounding of the output, u max(1, |g|), plus the heading's error from the stored fp32 quaternion's
   departure from unit length eps = | |q|^2 - 1 | (the device's x-axis formula assumes |q| = 1: to first order the heading moves by at most
   eps / |x_xz|, counted twice) and the two sides' different double formulas for the heading (4 u / |x_xz|), times max(1, |g|); in the target
   scene the root the oracle derives from the snapshot differs from the stored one by rounding, 4 u max(1, |root|), over the target distance;
   where the root's x axis is within 5 degrees of vertical, in addition the first-order
   heading allowance of tests/amp_states.py, 1e-6 / |x_xz| max(1, |g|).
2. against the oracle's own update: the state within the tolerances of tests/test_parity_gpu.py (|dq| <= 1e-3; |dqd| <= 1e-3 contact-free,
   0.5 with contacts).  kKCom against the oracle's COM within that state error through the lever arms (1e-3 + 2 sqrt(3) 1e-3 times the
   longest joint chain to a body COM, the bound of tests/test_task_ext_gpu.py for a body position) plus DC; kKPrevCom against the oracle's
   prev_action_com exactly where the update took no new action (the loaded value is kept), within DC where it did.

Decisions are exact: the update of a redraw, the draw counter, the terminate code and its update, the zero reward of a fallen character.
Timers, heading and speed agree to 1e-9 (pure double); a target that was not redrawn to 1e-9, a redrawn one relative to its own root (the
draw) to 1e-7, since the oracle draws around its double root and the snapshot holds it in fp32."""
import math

import numpy as np
import pytest

from tests import amp_states as A
from tests import task_states as S
from tests.dynamics_ref import edited_asset_tree, lumped_leaves
from tests.oracle_binding import Oracle, PushOracle
from tests.parity_util import compare_sim_state, joint_types_from_assets
from tests.test_task_ext_gpu import _pos_bound

pytestmark = pytest.mark.gpu

DT = S.DT
U = 2.0 ** -24
N_COM = 32 * 4 + 2 * S.NJ
CHAR = "data/characters/humanoid3d.txt"
CTRL = "data/controllers/humanoid3d_ctrl.txt"
TOTALS = {}


def _core(args, n, asset_root, seed=21, offset=100, placement=False, mode=0):
    from deepmimic_b200 import capi
    core = capi.BatchedCore(args, n, asset_root, seed=seed, global_env_offset=offset)
    core.set_env_order(placement)
    core.set_mode(mode)
    return core


def _outputs(core, n_rows=None):
    import torch
    N, G = core.num_envs, core.dims.goal_size
    R = N if n_rows is None else n_rows
    goal = torch.full((R, G), -7.0, device="cuda"); rew = torch.full((R,), -7.0, device="cuda"); fl = torch.zeros(N, 4, dtype=torch.int32, device="cuda")
    core.record_goal(goal); core.observe(None, rew); core.flags(fl); core.sync()
    return goal.cpu().numpy().astype(np.float64), rew.cpu().numpy().astype(np.float64), fl.cpu().numpy()


def DC(com):
    return N_COM * U * max(1.0, float(np.abs(com).max()))


def _mirror(mirror, core, e):
    """the oracle evaluating the GPU's own post-update state and task block of environment e"""
    s, tb = core.get_snapshot(e), core.task_state(e)
    mirror.set_snapshot(s)
    mirror.set_task_state(np.array([tb[0], 0.0, tb[1]]), tb[2], tb[3], tb[4], tb[5], tb[6:9])
    return s, tb


def _reward_bound(scene, p, tb, root, sd, fallen, r):
    """|d r| under |d com| <= DC (first order, central differences of the float64 restatement); the previous-action COM is the GPU's own on
    both sides"""
    if fallen:
        return 0.0
    com, prev = tb[9:12], tb[6:9]
    f = lambda c: S.ref_reward(scene, p, tb[0:2], tb[2], tb[3], root, c, prev, sd, False)
    g = 0.0
    for k in (0, 2):
        h = np.zeros(3); h[k] = 1e-7
        g += abs(f(com + h) - f(com - h)) / 2e-7 * DC(com)
    return g + U * abs(r) + 1e-9


def _check_mirror(mirror, core, e, st_scene, p, g, r, fl):
    """comparison 1; returns (reward error, reward error / bound, goal error, goal error / bound, COM error / bound, tilted)"""
    s, tb = _mirror(mirror, core, e)
    com_m = mirror.calc_com()
    ec = float(np.abs(tb[9:12] - com_m).max())
    assert ec <= DC(com_m), (e, tb[9:12], com_m)
    fallen = mirror.has_fallen()
    root = s[[0, 2]] / S.SCALE
    sd = s[S.CLK + 8] - s[S.CLK + 10]
    rm = mirror.calc_reward()
    if fallen:
        assert r[e] == 0.0, (e, r[e])
    br = _reward_bound(st_scene, p, tb, root, sd, fallen, rm)
    er = abs(r[e] - rm)
    assert er <= br, (e, r[e], rm, br)
    gm = mirror.record_goal()
    cond = math.hypot(1.0 - 2.0 * (s[4] ** 2 + s[5] ** 2), 2.0 * (s[3] * s[5] + s[6] * s[4]))
    eps = abs(float(np.dot(s[3:7], s[3:7])) - 1.0)            # the stored fp32 quaternion's departure from unit length
    gs = max(1.0, float(np.abs(gm).max()))
    bg = U * gs + (2.0 * eps + 4.0 * U) / cond * gs + 1e-12
    if st_scene == "target":   # the oracle's root is the double position its pose derives from the snapshot: 4 u |root| over the distance
        bg += 4.0 * U * max(1.0, float(np.abs(root).max())) / max(float(gm[2]), 1e-4) * gs
    tilted = cond < A.COND_MIN
    if tilted:
        bg += 1e-6 / cond * gs
    eg = float(np.abs(g[e] - gm).max())
    assert eg <= bg, (e, g[e], gm, bg)
    return er, (er / br if br > 0 else 0.0), eg, eg / bg, ec / DC(com_m), tilted


def _com_bound(o):
    """|d com| under the parity state tolerance: the largest body-position bound of the oracle's state, plus DC"""
    pos = o.body_state()[0]
    return max(_pos_bound(pos, b)[0] for b in range(S.NJ)) + DC(o.calc_com())


def _check_oracle(core, e, o, f, jt, c_before, new_action):
    """comparison 2 and the exact decisions; returns (|dq|, |dqd|, kKCom error / its bound)"""
    so, sg = o.get_snapshot(), core.get_snapshot(e)
    contact = sum(S.LAY.contact_counts(so)) > 0
    eq, eqd = compare_sim_state(S.LAY, so, sg, jt)
    assert eq <= 1e-3 and eqd <= (0.5 if contact else 1e-3), (e, eq, eqd)
    tb, ts = core.task_state(e), o.task_state()
    assert int(tb[S.K_COUNTER]) == o.task_counter(), (e, tb[S.K_COUNTER], o.task_counter())
    assert int(f[e, 2]) == o.check_terminate() and int(f[e, 1]) == int(o.is_episode_end()), (e, f[e], o.check_terminate())
    assert np.abs(tb[2:6] - [ts["target_speed"], ts["target_heading"], ts["timer"], ts["timer_max"]]).max() <= 1e-9
    if o.task_counter() != c_before:   # redrawn around each side's own root: the draw to 1e-7 (the oracle's root is its double state)
        rg, ro = sg[[0, 2]] / S.SCALE, so[[0, 2]] / S.SCALE
        assert np.abs((tb[0:2] - rg) - (ts["target_pos"][[0, 2]] - ro)).max() <= 1e-7
    else:
        assert np.abs(tb[0:2] - ts["target_pos"][[0, 2]]).max() <= 1e-9
    epc = float(np.abs(tb[6:9] - ts["prev_action_com"]).max())
    assert epc <= (DC(ts["prev_action_com"]) if new_action else 0.0), (e, tb[6:9], ts["prev_action_com"])
    ec, bc = float(np.abs(tb[9:12] - o.calc_com()).max()), _com_bound(o)
    assert ec <= bc, (e, tb[9:12], o.calc_com(), bc)
    return eq, eqd, ec / bc


STATES = {"target": S.target_states, "heading": S.heading_states}


def _mass_vectors(asset_root, k, seed=3):
    """k non-uniform mass-factor vectors, each lumped wrist carrying its elbow's factor"""
    lp = lumped_leaves(f"{asset_root}/{CHAR}")
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(k):
        m = rng.uniform(0.7, 1.3, S.NJ).astype(np.float32)
        for l, q in enumerate(lp):
            if q >= 0:
                m[l] = m[q]
        out.append(m)
    return out


def _warp_partners(core, e):
    """the environments that shared environment e's warp in the last step launch"""
    _, order, _, W = core.env_order()
    slot = int(np.nonzero(order == e)[0][0])
    per = 32 // W
    return [int(x) for x in order[slot - slot % per: slot - slot % per + per] if x != e]


def _run_states(asset_root, scene, mode, inst, seed, offset, tmp=None):
    """every state of the scene in its own environment of a 37-environment batch (placement by contact load in train mode, by index with
    the dynamics table), 3 teacher-forced updates; inst: 'plain', 'push' (a push on every environment during the comparison) or 'dyn'
    (three distinct non-uniform mass-factor vectors over the compared environments, environment e holding vector e % 3, each against an
    oracle built from its own edited asset tree; every other environment holds a fourth vector)"""
    states = STATES[scene]()
    n = 37
    envs = [(3 * k + 1) % n for k in range(len(states))]
    assert len(set(envs)) == len(envs)
    groups = {}
    for st in states:
        groups.setdefault(tuple(st.extra), []).append(st)
    jt = joint_types_from_assets(asset_root, CHAR)
    worst = dict(er=0.0, rr=0.0, eg=0.0, rg=0.0, rc=0.0, rco=0.0, eq=0.0, eqd=0.0, tilted=0, cases=0)
    trees = {}
    if inst == "dyn":
        vecs = _mass_vectors(asset_root, 4)
        trees = {v: edited_asset_tree(asset_root, str(tmp / ("v%d" % v)), CHAR, CTRL, 1.0, 1.0, 1.0, vecs[v]) for v in range(3)}
    for extra, sts in groups.items():
        args = sts[0].args
        p = S.scene_params(asset_root, args)
        core = _core(args, n, asset_root, seed=seed, offset=offset, placement=mode == 0 and inst != "dyn", mode=mode)
        _, tseed, base = core.task_params()
        cls = PushOracle if inst == "push" else Oracle
        key_of = lambda e: e % 3 if inst == "dyn" else 0
        assets_of = lambda e: trees[e % 3] if inst == "dyn" else asset_root
        if inst == "dyn":
            tab = np.ones((n, 4 + S.NJ), dtype=np.float32)
            tab[:, 4:] = vecs[3]
            for st in sts:
                e = envs[states.index(st)]
                tab[e, 4:] = vecs[e % 3]
            core.set_dynamics(tab)
        if inst == "push":
            body = np.full(n, 3, dtype=np.int32); force = np.tile(np.array([[40.0, 10.0, -30.0]], dtype=np.float32), (n, 1))
            core.set_pushes(body, force, np.zeros(n), np.full(n, 100.0))
        orcs, mirrors = {}, {}
        for st in sts:
            e = envs[states.index(st)]
            o = cls(args, assets_of(e))
            o.set_mode(mode)
            o.set_task_stream(tseed, base + e, 7)
            st.prepare(o, p, (tseed, base + e), states.index(st))
            if inst == "push":
                o.set_push(3, np.array([40.0, 10.0, -30.0]), 0.0, 100.0)
            orcs[e] = (st, o)
            if key_of(e) not in mirrors:
                mirrors[key_of(e)] = cls(args, assets_of(e))
        for upd in range(3):
            before, acted = {}, {}
            for e, (st, o) in orcs.items():
                S.load(core, e, o)
                before[e] = o.task_counter()
                acted[e] = o.need_new_action()
            core.update(DT, 1)
            for st, o in orcs.values():
                o.update(DT)
            g, r, f = _outputs(core)
            for e, (st, o) in orcs.items():
                if inst == "dyn" and upd == 0:   # environment e's warp partners hold other factors
                    for q in _warp_partners(core, e):
                        assert not np.array_equal(tab[q, 4:], tab[e, 4:]), (e, q)
                er, rr, eg, rg, rc, tilted = _check_mirror(mirrors[key_of(e)], core, e, scene, p, g, r, f)
                eq, eqd, rco = _check_oracle(core, e, o, f, jt, before[e], acted[e])
                if o.has_fallen():
                    assert r[e] == 0.0
                worst = dict(er=max(worst["er"], er), rr=max(worst["rr"], rr), eg=max(worst["eg"], eg), rg=max(worst["rg"], rg), rc=max(worst["rc"], rc),
                             rco=max(worst["rco"], rco), eq=max(worst["eq"], eq), eqd=max(worst["eqd"], eqd), tilted=worst["tilted"] + tilted,
                             cases=worst["cases"] + 1)
        core.close()
    return worst


@pytest.mark.parametrize("mode,inst", [(0, "plain"), (1, "plain"), (0, "push"), (0, "dyn")],
                         ids=["train-plain", "test-plain", "train-push", "train-dyn"])
@pytest.mark.parametrize("scene", ["target", "heading"])
def test_states_match_the_oracle(asset_root, tmp_path, scene, mode, inst):
    w = _run_states(asset_root, scene, mode, inst, seed=31 + mode, offset=2 ** 31 + 1000 * mode, tmp=tmp_path)
    print("%s %s %s: %d state-updates, reward max %.2e (%.3f of bound), goal max %.2e (%.3f of bound, %d tilted), COM %.3f of bound on the GPU "
          "state, %.3f against the oracle, |dq| %.2e |dqd| %.2e" % (scene, ["train", "test"][mode], inst, w["cases"], w["er"], w["rr"], w["eg"],
                                                                   w["rg"], w["tilted"], w["rc"], w["rco"], w["eq"], w["eqd"]))
    assert w["cases"] >= 3 * len(STATES[scene]())


@pytest.mark.parametrize("scene", ["target", "heading"])
def test_draws_follow_the_environment_not_its_slot(asset_root, scene):
    """Train mode, placement by contact load: characters lying on the ground (many solver rows) in the middle environments and airborne ones
    (no rows) whose target timer expires on both sides of them, so that the placement, which sorts by the rows of the previous launch, moves
    expiring environments to other slots of the step launch whichever way it sorts (asserted with env_order).  Every redraw must come from the stream of the environment's own global id: counters, targets, headings and speeds
    against the oracle under that stream (comparison 2)."""
    st = next(x for x in STATES[scene]() if x.expire)
    lie = next(x for x in STATES[scene]() if x.kind == "lying")
    args = st.args
    p = S.scene_params(asset_root, args)
    n = 37
    core = _core(args, n, asset_root, seed=77, offset=2 ** 31 + 4321, placement=True)
    _, tseed, base = core.task_params()
    jt = joint_types_from_assets(asset_root, CHAR)
    expiring = list(range(0, 10)) + list(range(26, n))
    lying = list(range(10, 26))
    orcs = {}

    def prepared():
        for e in lying + expiring:
            o = Oracle(args, asset_root)
            o.set_task_stream(tseed, base + e, 5)
            (st if e in expiring else lie).prepare(o, p, (tseed, base + e), e)
            orcs[e] = o
            S.load(core, e, o)
    prepared()
    core.update(DT, 1)           # the launch that records each environment's contact load: the next placement sorts by it
    prepared()
    before = {e: o.task_counter() for e, o in orcs.items()}
    core.update(DT, 1)
    for o in orcs.values():
        o.update(DT)
    _, order, _, _ = core.env_order()
    moved = [e for e in expiring if int(np.nonzero(order == e)[0][0]) != e]
    assert len(moved) >= 4, order
    _, _, f = _outputs(core)
    for e in expiring:
        assert orcs[e].task_counter() != before[e]
        _check_oracle(core, e, orcs[e], f, jt, before[e], False)
    print("%s: %d of %d expiring environments placed in another slot, their redraws on their own streams" % (scene, len(moved), len(expiring)))


# ---------------------------------------------------------------------------------------------------------------- launches
@pytest.mark.parametrize("launch", S.launches(), ids=repr)
def test_launches_match_the_oracle(asset_root, launch):
    """A 20-update launch from set_action (60 for three policy steps, the action reused): the target timer expiring on chosen updates (two and
    more expiries, timer_max met with equality), the root moving at 2.7 m/s so that a redraw around the wrong update's root is visible.
    Draw counter and timers exactly / to 1e-9, the target to the oracle's within the free-running airborne root's drift, kKPrevCom at the
    last new action against the oracle's prev_action_com, the step duration ctrl - prev_action = 19 / 600 exactly as the oracle's, and goal,
    reward and COM on the GPU's own state (comparison 1)."""
    import torch
    n = 37
    args = launch.args
    p = S.scene_params(asset_root, args)
    jt = joint_types_from_assets(asset_root, CHAR)
    core = _core(args, n, asset_root, seed=5, offset=3000, placement=True)
    _, tseed, base = core.task_params()
    envs = [0, 17, 36]
    orcs = {}
    for k, e in enumerate(envs):
        o = Oracle(args, asset_root)
        o.set_task_stream(tseed, base + e, 11)
        launch.prepare(o, k)
        orcs[e] = o
    acts = np.zeros((n, core.dims.action_size), dtype=np.float32)
    for e, o in orcs.items():
        S.load(core, e, o)
        acts[e] = -o.action_statics()[0] + 0.05 * np.cos(np.arange(o.action_size) + envs.index(e))
        o.set_action(acts[e].astype(np.float64))
    core.set_action(torch.as_tensor(acts, device="cuda"))
    core.update(DT, launch.updates)
    for o in orcs.values():
        for _ in range(launch.updates):
            o.update(DT)
    g, r, f = _outputs(core)
    mirror = Oracle(args, asset_root)
    w_t = w_pc = 0.0
    for e, o in orcs.items():
        tb, ts = core.task_state(e), o.task_state()
        sg, so = core.get_snapshot(e), o.get_snapshot()
        assert int(tb[S.K_COUNTER]) == o.task_counter(), (e, tb[S.K_COUNTER], o.task_counter())
        assert np.abs(tb[2:6] - [ts["target_speed"], ts["target_heading"], ts["timer"], ts["timer_max"]]).max() <= 1e-9
        assert sg[S.CLK + 8] - sg[S.CLK + 10] == so[S.CLK + 8] - so[S.CLK + 10] == pytest.approx(19 * DT, abs=1e-12)
        eq, _ = compare_sim_state(S.LAY, so, sg, jt)
        drift = float(np.abs(sg[0:3] - so[0:3]).max()) / S.SCALE
        et = float(np.abs(tb[0:2] - ts["target_pos"][[0, 2]]).max())
        assert et <= 2 * drift + 1e-7, (e, et, drift)
        epc = float(np.abs(tb[6:9] - ts["prev_action_com"]).max())
        assert epc <= 2 * drift + DC(ts["prev_action_com"]) + 1e-7, (e, epc, drift)
        assert int(f[e, 2]) == o.check_terminate() == 0
        _check_mirror(mirror, core, e, launch.scene, p, g, r, f)
        w_t, w_pc = max(w_t, et), max(w_pc, epc)
    print("%s: target |GPU - oracle| max %.2e, previous-action COM max %.2e, counters exact" % (launch, w_t, w_pc))


# ---------------------------------------------------------------------------------------------------------------- reset kernel
@pytest.mark.parametrize("n", [37, 1001])
@pytest.mark.parametrize("scene", ["target", "heading"])
def test_reset_kernel_draws_and_untouched_blocks(asset_root, scene, n):
    """Forced resets at a global environment id above 2^31: target, speed, heading, timers and counters against the oracle under the same
    stream; then reset(force_all=False) with a third of the environments done leaves every other task block (warp partners and padding
    included) bit-identical.  The reward read right after a reset (step_dur = 0, both COMs 0) is the oracle's, or in the target scene 0.4
    above it where the oracle's avg_vel is -inf (recorded, DESIGN.md section 4)."""
    args = S.SCENES[scene]
    core = _core(args, n, asset_root, seed=2024, offset=2 ** 31 + 12345, placement=n == 37)
    _, tseed, base = core.task_params()
    o = Oracle(args, asset_root)
    kt = np.linspace(0.05, 0.8, n); th = np.linspace(-3.0, 3.0, n); clip = (np.arange(n) % 4).astype(np.int32)
    counters = [int(core.task_state(e)[S.K_COUNTER]) for e in range(n)]
    core.reset(True, kin_time=kt, max_time=np.full(n, 20.0), rot_theta=th, clip=clip)
    g, r, _ = _outputs(core)
    nan_dev = nan_orc = agree = 0
    for e in range(n) if n < 100 else range(0, n, 7):
        o.set_task_stream(tseed, base + e, counters[e])
        o.reset(kt[e], th[e], 20.0, clip=int(clip[e]))
        tb, ts = core.task_state(e), o.task_state()
        assert int(tb[S.K_COUNTER]) == o.task_counter(), e
        assert abs(tb[0] - ts["target_pos"][0]) <= 1e-7 and abs(tb[1] - ts["target_pos"][2]) <= 1e-7
        assert np.abs(tb[2:6] - [ts["target_speed"], ts["target_heading"], ts["timer"], ts["timer_max"]]).max() <= 1e-9
        assert np.all(tb[6:12] == 0.0)
        np.testing.assert_allclose(g[e], o.record_goal(), atol=2e-5, rtol=1e-5)
        ro = o.calc_reward()
        nan_dev += math.isnan(r[e]); nan_orc += math.isnan(ro)
        same = (math.isnan(r[e]) and math.isnan(ro)) or abs(r[e] - ro) <= 1e-5
        agree += same
        if not same:
            # DESIGN.md section 4: the device's COMs are 0 after a reset, so avg_vel = 0 / 0 and enable_min_tar_vel's fmax gives the full
            # velocity term; the oracle's live COM over step_dur = 0 is -inf where the COM lies behind the target direction: 0.4 less
            assert scene == "target" and abs(r[e] - ro - 0.4) <= 1e-5, (e, r[e], ro)
    TOTALS.setdefault("reset_reward", []).append((scene, n, nan_dev, nan_orc, agree))
    print("%s N=%d: post-reset reward NaN on the device %d, in the oracle %d, agreeing %d" % (scene, n, nan_dev, nan_orc, agree))
    # a partial reset: a third of the environments done
    for e in range(0, n, 3):
        s = core.get_snapshot(e); s[S.CLK + 12] = s[S.CLK + 13] + 1.0; core.set_snapshot(e, s)
    core.update(DT, 1)
    _, _, f = _outputs(core)
    done = [e for e in range(n) if f[e, 1]]
    assert set(range(0, n, 3)) <= set(done)
    before = {e: core.task_state(e) for e in range(n)}
    core.reset(False)
    core.sync()
    for e in range(n):
        tb = core.task_state(e)
        if e in done:
            assert tb[S.K_RESET_SEEN] == before[e][S.K_RESET_SEEN] + 1
        else:
            assert np.array_equal(tb, before[e]), e


# ---------------------------------------------------------------------------------------------------------------- batch edges
@pytest.mark.parametrize("placement", [True, False], ids=["placed", "by_index"])
@pytest.mark.parametrize("n", [37, 1001])
def test_rows_equal_environment_0_and_guard_rows(asset_root, n, placement):
    """One state of each reward regime loaded into environment 0 and into a spread of other rows: after one update every such row's goal,
    reward, flags and task block equal environment 0's bit for bit (placement and warp position do not matter); goal and reward rows past N
    of an oversized output keep their guard values."""
    for scene in ("target", "heading"):
        states = [st for st in STATES[scene]() if not st.extra][:4]
        args = S.SCENES[scene]
        p = S.scene_params(asset_root, args)
        core = _core(args, n, asset_root, seed=9, offset=0, placement=placement)
        _, tseed, _ = core.task_params()
        rows = sorted({0, 1, 15, 16, 17, n // 2, n - 2, n - 1})
        for st in states:
            o = Oracle(args, asset_root)
            o.set_task_stream(tseed, 0, 3)
            st.prepare(o, p, (tseed, 0), 0)
            for e in rows:
                S.load(core, e, o)
                tb = core.task_state(e); tb[S.K_COUNTER] = 3; core.set_task_state(e, tb)
            core.update(DT, 1)
            g, r, f = _outputs(core, n_rows=n + 5)
            t0 = core.task_state(0); t0[S.K_RESET_SEEN] = 0
            for e in rows:
                te = core.task_state(e); te[S.K_RESET_SEEN] = 0
                # the draw stream is keyed by the global id: only the counter-independent part must match when the timer runs
                assert np.array_equal(g[e], g[0]) and (r[e] == r[0] or (math.isnan(r[e]) and math.isnan(r[0]))) and np.array_equal(f[e], f[0]), (st, e)
                assert np.array_equal(te, t0), (st, e)
            assert np.all(g[n:] == -7.0) and np.all(r[n:] == -7.0)
        core.close()
