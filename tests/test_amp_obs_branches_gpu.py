"""The AMP observation kernel of dm_policy.cu (amp_obs_tile behind dm_amp_obs_kernel, both instantiations) and the history it reads
(dm_set_action_kernel, dm_reset_kernel, the handle's initial fill) against the CPU oracle, branch by branch, on the constructed inputs of
tests/amp_states.py (checked to reach their branches by tests/test_amp_states_cpu.py):

  - agent pairs: set_snapshot(S_prev), set_action (stores every real environment's history), set_snapshot(S_now), amp_obs_agent; the oracle
    runs the same sequence with update_hist;
  - imitate_amp resets (InitHist), in train and test mode, and two teacher-forced policy steps;
  - the task scenes: a fresh handle's first observation (the initial history), teacher-forced policy steps, and an episode that ends followed
    by reset(force_all=False) with the clip and time injected, whose first observation carries the old episode's history;
  - expert observations at the times of amp_states.expert_times, for the scene's clip (dm_amp_obs_kernel<.., false>) and every clip of
    three datasets (<.., true>), each row over its own environment's ground height;
  - N = 37 and 1001 (humanoid3d, W = 16, four environments per 64-thread block, a padded last block) and 33 (dog3d, W = 32): every row equals
    the same pair evaluated in environment 0, bit for bit, and NaN guard rows after row N keep their NaN.

Bounds (derivation in tests/amp_states.py and DESIGN.md section 4): per part n u max(1, |largest element of the part|) with n = 32 maxlevel
+ 64 and u = 2^-24 (humanoid3d 1.1e-5, dog3d 1.5e-5 at scale 1), capped at 2e-4 (pose) and 2e-3 (velocity); rows whose now root has its x
axis within 5 degrees of vertical add a heading error of 1e-6 / |x_xz| rad through the part's scale, and are counted.  Each test prints its
branches' maxima against their bounds."""
import math
import time

import numpy as np
import pytest

from tests import amp_states as A
from tests import policy_states as P
from tests.oracle_binding import Oracle

pytestmark = pytest.mark.gpu

DT = P.DT


@pytest.fixture(scope="module", autouse=True)
def _file_time():
    t0 = time.time()
    yield
    print("\ntest_amp_obs_branches_gpu.py: %.1f s" % (time.time() - t0))


@pytest.fixture(scope="module")
def assets(asset_root, tmp_path_factory):
    return P.make_assets(asset_root, str(tmp_path_factory.mktemp("amp") / "assets"))


def _core(args, n, assets, seed=5, mode=0):
    from deepmimic_b200 import capi
    core = capi.BatchedCore(args, n, assets, seed=seed, global_env_offset=0)
    core.set_mode(mode)
    return core


def _np(t):
    return t.cpu().numpy().astype(np.float64)


class Tally:
    """per-branch maxima: pose and velocity error, their ratio to the bound, rows, rows with the heading allowance"""
    def __init__(self, what):
        self.what, self.rows = what, {}

    def add(self, branch, r):
        ep, ev, rp, rv, ill = r
        t = self.rows.setdefault(branch, [0.0, 0.0, 0.0, 0.0, 0, 0])
        t[0], t[1], t[2], t[3] = max(t[0], ep), max(t[1], ev), max(t[2], rp), max(t[3], rv)
        t[4] += 1
        t[5] += ill

    def report(self):
        for b, t in self.rows.items():
            print("%s / %s: %d rows, pose %.2e (%.2f of bound), vel %.2e (%.2f of bound), heading allowance %d"
                  % (self.what, b, t[4], t[0], t[2], t[1], t[3], t[5]))


def _amp(core, n, guard=2):
    import torch
    return torch.full((n + guard, core.dims.amp_obs_size), float("nan"), device="cuda")


def _record_agent(core, n):
    import torch
    out = _amp(core, n)
    torch.cuda.synchronize()
    core.amp_obs_agent(out)
    core.sync()
    g = _np(out)
    assert np.isnan(g[n:]).all(), "amp_obs_agent wrote past row N"
    return g


def _set_action_all(core, n, acts=None):
    import torch
    a = torch.zeros(n, core.dims.action_size, device="cuda") if acts is None else torch.tensor(acts, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    core.set_action(a)
    core.sync()


def _load_pairs(core, pairs, n):
    """environment e := pair e % len(pairs): its history from S_prev through set_action, then S_now"""
    for e in range(n):
        core.set_snapshot(e, pairs[e % len(pairs)].prev)
    _set_action_all(core, n)
    for e in range(n):
        core.set_snapshot(e, pairs[e % len(pairs)].now)


# ---------------------------------------------------------------------------------------------------------------- agent pairs
@pytest.mark.parametrize("local_root", [True, False], ids=["local_root", "world_root"])
@pytest.mark.parametrize("ch", ["humanoid3d", "dog3d"])
def test_agent_pairs_match_the_oracle(assets, ch, local_root):
    """headings in every quadrant and at +-pi, the root's x axis near vertical, w < 0, revolute angles past +-pi, near-clip, walking,
    airborne and lying states; the dog's spherical joints with non-identity child rotations"""
    args = A.amp_args(ch, local_root)
    o = Oracle(args, assets)
    pairs = A.agent_pairs(o, assets, ch)
    n, ml = len(pairs), A.max_level(assets, ch)
    core = _core(args, n, assets)
    _load_pairs(core, pairs, n)
    g = _record_agent(core, n)
    ps = A.split(core.dims.amp_obs_size, o.pose_dim)
    tally = Tally("agent %s %s" % (ch, "local root" if local_root else "world root"))
    for e, p in enumerate(pairs):
        o.set_snapshot(p.prev); o.update_hist(); o.set_snapshot(p.now)
        tally.add(p.kind, A.check(g[e], o.record_amp_obs_agent(), ps, ml, (ch, local_root, p.name)))
    tally.report()
    assert tally.rows["tilt"][5] == 4
    core.close()


# ---------------------------------------------------------------------------------------------------------------- imitate_amp resets
RESET_CONFIGS = {"walk local": ("humanoid3d", A.amp_args("humanoid3d", True, P.WALK), P.WALK),
                 "walk world": ("humanoid3d", A.amp_args("humanoid3d", False, P.WALK), P.WALK),
                 "walk_once local": ("humanoid3d", A.amp_args("humanoid3d", True, P.WALK_ONCE), P.WALK_ONCE),
                 "walk_once world": ("humanoid3d", A.amp_args("humanoid3d", False, P.WALK_ONCE), P.WALK_ONCE),
                 "spinkick": ("humanoid3d", A.PARITY["spinkick"], P.SPINKICK),
                 "dog_local": ("dog3d", A.PARITY["dog_local"], "data/motions/dog3d_trot.txt")}


def _policy_steps(core, n, runs, steps, tally, ps, ml, what, rng):
    """teacher-forced policy steps: every (environment, oracle) in `runs` starts each step from the oracle's state with the new-action flag
    set, both apply the same action, the oracle runs 20 updates and the device observes the oracle's state after them"""
    off, scl, lo, hi = runs[0][1].action_statics()
    for step in range(steps):
        acts = np.zeros((n, core.dims.action_size))
        for e, o in runs:
            s = A.acting(o.get_snapshot(), o.num_joints)
            o.set_snapshot(s)
            core.set_snapshot(e, s)
            acts[e] = P.random_policy_action(rng, off, scl, lo, hi)
        _set_action_all(core, n, acts)
        for e, o in runs:
            o.set_action(acts[e])
            for _ in range(20):
                o.update(DT)
            core.set_snapshot(e, o.get_snapshot())
        g = _record_agent(core, n)
        for e, o in runs:
            tally.add("policy step", A.check(g[e], o.record_amp_obs_agent(), ps, ml, (what, "step", step, e)))


@pytest.mark.parametrize("mode", [0, 1], ids=["train", "test"])
@pytest.mark.parametrize("config", list(RESET_CONFIGS))
def test_imitate_amp_reset_history_matches_the_oracle(assets, config, mode):
    """InitHist: kin times in [0, 1/30) (previous cycle / clamped at frame 0), inside, dur - eps, dur and past it (the history sample past
    the end of a non-looping clip is at rest), cycles 1 and 5, rot_theta 0, +-pi and others; the spin kick and dog local-root grids of the
    former parity test; then two teacher-forced policy steps of one environment"""
    ch, args, motion = RESET_CONFIGS[config]
    o = Oracle(args, assets)
    o.set_mode(mode)
    d = o.motion_duration
    cases = A.reset_cases(motion, d)
    if config == "spinkick":
        cases += [("parity", kt, 0.0) for kt in np.linspace(0.02, 0.97 * d, 8)]
    if config == "dog_local":
        cases += [("parity", kt, th) for kt, th in zip(np.linspace(0.02, 0.97 * d, 8), np.linspace(-2.5, 2.5, 8))]
    n, ml = len(cases), A.max_level(assets, ch)
    core = _core(args, n, assets, mode=mode)
    kin = np.array([c[1] for c in cases]); th = np.array([c[2] for c in cases]); mt = np.linspace(3.0, 9.0, n)
    core.reset(True, kin_time=kin, max_time=mt, rot_theta=th)
    g = _record_agent(core, n)
    ps = A.split(core.dims.amp_obs_size, o.pose_dim)
    tally = Tally("reset %s mode %d" % (config, mode))
    for e, (lb, kt, t) in enumerate(cases):
        o.reset(kt, t, mt[e])
        tally.add("InitHist " + lb.replace(" th", ""), A.check(g[e], o.record_amp_obs_agent(), ps, ml, (config, mode, lb, kt, t)))
    e = 3
    o.reset(kin[e], th[e], mt[e])
    _policy_steps(core, n, [(e, o)], 2, tally, ps, ml, config, np.random.default_rng(3))
    tally.report()
    core.close()


# ---------------------------------------------------------------------------------------------------------------- task scenes
@pytest.mark.parametrize("scene", list(A.TASK_SCENES))
def test_task_scene_history_matches_the_oracle(assets, scene):
    """a fresh handle's first observation (the history is the identity pose at rest on both sides), three teacher-forced policy steps, then
    an episode that ends on its timer and reset(force_all=False) with the clip and time injected: the new episode's first observation
    carries the old episode's history (task scenes do not InitHist)"""
    args = A.TASK_SCENES[scene]
    n, ml = 8, A.max_level(assets, "humanoid3d")
    oracles = [Oracle(args, assets) for _ in range(n)]
    nclip = oracles[0].num_clips()
    kin = np.linspace(0.05, 0.9, n); th = np.linspace(-3.0, 3.0, n); mt = np.full(n, 20.0); clip = (np.arange(n) % nclip).astype(np.int32)
    core = _core(args, n, assets)
    core.reset(True, kin_time=kin, max_time=mt, rot_theta=th, clip=clip)
    g = _record_agent(core, n)
    ps = A.split(core.dims.amp_obs_size, oracles[0].pose_dim)
    tally = Tally("task %s" % scene)
    for e, o in enumerate(oracles):
        o.reset(kin[e], th[e], mt[e], clip=int(clip[e]))
        tally.add("fresh handle", A.check(g[e], o.record_amp_obs_agent(), ps, ml, (scene, "fresh", e)))
    runs = list(enumerate(oracles))
    _policy_steps(core, n, runs, 3, tally, ps, ml, scene, np.random.default_rng(8))
    # the episode ends on its timer in the next update; the history is the state the last action was chosen from
    scal = 13 + 55 * oracles[0].num_joints
    acts = np.zeros((n, core.dims.action_size))
    off, scl, lo, hi = oracles[0].action_statics()
    rng = np.random.default_rng(9)
    for e, o in runs:
        s = A.acting(o.get_snapshot(), o.num_joints)
        s[scal + 12] = s[scal + 13] = 1.0
        o.set_snapshot(s)
        core.set_snapshot(e, s)
        acts[e] = P.random_policy_action(rng, off, scl, lo, hi)
    _set_action_all(core, n, acts)
    core.update(DT, 1)
    for e, o in runs:
        o.set_action(acts[e])
        o.update(DT)
        assert o.is_episode_end()
    kin2 = np.linspace(0.6, 0.1, n); th2 = np.linspace(2.0, -2.9, n); clip2 = ((np.arange(n) + 1) % nclip).astype(np.int32)
    core.reset(False, kin_time=kin2, max_time=mt, rot_theta=th2, clip=clip2)
    g = _record_agent(core, n)
    for e, o in runs:
        o.reset(kin2[e], th2[e], mt[e], clip=int(clip2[e]))
        assert o.current_clip() == clip2[e]
        tally.add("kept history", A.check(g[e], o.record_amp_obs_agent(), ps, ml, (scene, "kept", e)))
    tally.report()
    core.close()


# ---------------------------------------------------------------------------------------------------------------- expert
EXPERT_CONFIGS = {"walk local": RESET_CONFIGS["walk local"], "walk_once world": RESET_CONFIGS["walk_once world"],
                  "spinkick": RESET_CONFIGS["spinkick"], "dog_local": RESET_CONFIGS["dog_local"]}


def _expert_compare(core, o, rows, tally, ml, what):
    """rows [(label, clip or None, time)], environment e over its own ground height; returns nothing, asserts every row"""
    n = len(rows)
    base = o.get_snapshot()
    hs = A.origin_heights(n)
    for e in range(n):
        core.set_snapshot(e, A.with_origin_y(base, o.num_joints, hs[e]))
    out = _amp(core, n)
    kt = np.array([r[2] for r in rows])
    clips = None if rows[0][1] is None else np.array([r[1] for r in rows], dtype=np.int32)
    import torch
    torch.cuda.synchronize()
    core.amp_obs_expert(out, kin_time=kt, clip=clips)
    core.sync()
    g = _np(out)
    assert np.isnan(g[n:]).all()
    ps = A.split(core.dims.amp_obs_size, o.pose_dim)
    for e, (lb, c, t) in enumerate(rows):
        o.set_snapshot(A.with_origin_y(base, o.num_joints, hs[e]))
        ref = o.record_amp_obs_expert(t) if c is None else o.record_amp_obs_expert(t, clip=c)
        tally.add(lb if c is None else ("clip k > 0 " + lb if c > 0 and "interval" in lb else lb), A.check(g[e], ref, ps, ml, (what, c, lb, t)))


@pytest.mark.parametrize("config", list(EXPERT_CONFIGS))
def test_expert_observation_matches_the_oracle(assets, config):
    """dm_amp_obs_kernel<.., TASKV = false>: the scene's own clip at 0, in (0, 1/30), 1/30, exact frame times, the first and last frame
    intervals, dur - eps, dur, dur + eps and 1.9 dur (and the former parity test's times), each row over a ground height of its own"""
    ch, args, motion = EXPERT_CONFIGS[config]
    o = Oracle(args, assets)
    d = o.motion_duration
    rows = [(lb, None, t) for lb, t in A.expert_times(assets, motion)]
    rows += [("parity", None, t) for t in (0.01, 0.2, 0.5 * d, d - 0.001, d + 0.1, 0.031, 0.77 * d, 1.9 * d)]
    core = _core(args, len(rows), assets)
    o.reset(0.2, 0.7, 20.0)
    tally = Tally("expert %s" % config)
    _expert_compare(core, o, rows, tally, A.max_level(assets, ch), config)
    tally.report()
    core.close()


@pytest.mark.parametrize("dataset", list(A.DATASETS))
def test_dataset_expert_observation_matches_the_oracle(assets, dataset):
    """dm_amp_obs_kernel<.., TASKV = true>: every clip of the dataset at the times of amp_states.expert_times -- clip k > 0's first and
    last frame intervals read its own frames and frame velocities (ClipInfo.frame_off) -- each row over a ground height of its own"""
    args = A.DATASETS[dataset]
    o = Oracle(args, assets)
    files = A.dataset_clips(assets, args)
    rows = [(lb, c, t) for c, m in enumerate(files) for lb, t in A.expert_times(assets, m)]
    core = _core(args, len(rows), assets)
    o.reset(0.2, 0.7, 20.0, clip=0)
    tally = Tally("dataset expert %s" % dataset)
    _expert_compare(core, o, rows, tally, A.max_level(assets, "humanoid3d"), dataset)
    tally.report()
    core.close()


# ---------------------------------------------------------------------------------------------------------------- batch edges
@pytest.mark.parametrize("ch,n", [("humanoid3d", 37), ("humanoid3d", 1001), ("dog3d", 33)])
def test_rows_do_not_depend_on_the_environment(assets, ch, n):
    """N not a multiple of the tiles per block: every row equals the same (history, now) pair evaluated in environment 0, bit for bit --
    environment 0, the middle ones, the last one beside the padding -- and the guard rows after row N keep their NaN"""
    args = A.amp_args(ch, True)
    o = Oracle(args, assets)
    pairs = A.agent_pairs(o, assets, ch)
    K = len(pairs)
    core = _core(args, n, assets, seed=11)
    _load_pairs(core, pairs, n)
    g = _record_agent(core, n)
    for k in range(K):
        core.set_snapshot(0, pairs[k].prev)
        _set_action_all(core, n)
        core.set_snapshot(0, pairs[k].now)
        r = _record_agent(core, n)[0]
        for e in range(k, n, K):
            assert g[e].tobytes() == r.tobytes(), (ch, n, e, pairs[k].name)
    print("%s N = %d: %d rows bit-identical to environment 0 (%d pairs)" % (ch, n, n, K))
    core.close()
