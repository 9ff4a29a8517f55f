"""Per-environment dynamics on the GPU: unit factors bit-identical to the plain kernels, one environment's factors leaving the others
bit-identical, the scale identity (masses, gains and torque limits doubled move the character as before), the randomised table against the
Python restatement (tests/dynamics_ref.py) from the device's own reset counters, the state blob's round trip and refusals, and the refusals of
the three entry points."""
import os

import numpy as np
import pytest

from tests import dynamics_ref as ref
from tests.parity_util import SnapLayout, compare_sim_state, joint_types_from_assets

pytestmark = pytest.mark.gpu
DT = 1.0 / 600.0
SPINKICK = ["--arg_file", "args/run_humanoid3d_spinkick_args.txt"]
HEADER = 160   # capi.cu: StateHeader


def _core(n, seed=21, args=SPINKICK):
    from deepmimic_b200.assets import asset_root
    from deepmimic_b200.capi import BatchedCore
    c = BatchedCore(args, n, asset_root(prefer_archive=True), device=0, seed=seed)
    c.set_episode_limit(1.0, 2.5)
    c.reset(True)
    return c


def _actions(core, rng):
    import torch
    return torch.as_tensor(0.3 * rng.standard_normal((core.num_envs, core.dims.action_size)), dtype=torch.float32, device="cuda")


def _observe(core):
    import torch
    st = torch.zeros(core.num_envs, core.dims.state_size, device="cuda")
    rw = torch.zeros(core.num_envs, device="cuda")
    core.observe(st, rw)
    core.sync()
    return st.cpu().numpy(), rw.cpu().numpy()


def _blocks(core, blob):
    """(SIM [n_pad, stride] float32, TIME [n_pad, 16] float64, FLAGS [n_pad, 8] int32) of a save_state() blob"""
    n_pad = int(blob[28:32].view(np.int32)[0])
    ss = 16 + 12 * core.dims.num_joints
    off = HEADER
    sim = blob[off:off + n_pad * ss * 4].view(np.float32).reshape(n_pad, ss)
    off += n_pad * ss * 4
    tm = blob[off:off + n_pad * 16 * 8].view(np.float64).reshape(n_pad, 16)
    off += n_pad * 16 * 8
    fl = blob[off:off + n_pad * 8 * 4].view(np.int32).reshape(n_pad, 8)
    return sim, tm, fl


def _dyn(core):
    """the table as numpy, after the handle's stream (dynamics() is stream-ordered on it)"""
    t = core.dynamics()
    core.sync()
    return t.cpu().numpy()


def _unit(core):
    return np.ones((core.num_envs, 4 + core.dims.num_joints), dtype=np.float32)


def _run(core, acts, resets=True):
    out = []
    for a in acts:
        core.set_action(a)
        core.update(DT, 20)
        out.append(_observe(core))
        if resets:
            core.reset(False)
    return out


def test_unit_factors_are_bit_identical_and_one_environment_leaves_the_others():
    """From a saved state of 64 spin-kick environments with placement by contact load on, 12 policy steps with resets: the dynamics kernels with
    unit factors give observations, rewards and a state blob bit-identical to the plain kernels' (the blob with the table at its end).  Factors
    on environment 5 alone leave the other 63 bit-identical and change environment 5."""
    rng = np.random.default_rng(3)
    base = _core(64)
    base.set_env_order(True)
    _run(base, [_actions(base, rng) for _ in range(6)])
    blob = base.save_state()
    acts = [_actions(base, rng) for _ in range(12)]
    plain, unit, one = _core(64), _core(64), _core(64)
    for c in (plain, unit, one):
        c.load_state(blob)
        c.set_env_order(True)
    unit.set_dynamics(_unit(unit))
    f = _unit(one)
    f[5, :4] = (0.5, 1.3, 0.8, 0.7)
    f[5, 4:] = 1.2
    one.set_dynamics(f)
    rp, ru, r1 = _run(plain, acts), _run(unit, acts), _run(one, acts)
    for (sp, wp), (su, wu), (s1, w1) in zip(rp, ru, r1):
        assert sp.tobytes() == su.tobytes() and wp.tobytes() == wu.tobytes()
        keep = np.arange(64) != 5
        assert sp[keep].tobytes() == s1[keep].tobytes() and wp[keep].tobytes() == w1[keep].tobytes()
    bp, bu, b1 = plain.save_state(), unit.save_state(), one.save_state()
    n_pad = int(bp[28:32].view(np.int32)[0])
    assert len(bu) == len(bp) + n_pad * 160
    assert bp[HEADER:].tobytes() == bu[HEADER:len(bp)].tobytes()
    sp, tp, fp = _blocks(plain, bp)
    s1, t1, f1 = _blocks(one, b1)
    keep = np.arange(n_pad) != 5
    assert sp[keep].tobytes() == s1[keep].tobytes() and tp[keep].tobytes() == t1[keep].tobytes()
    assert sp[5].tobytes() != s1[5].tobytes()


def test_scale_identity(asset_root):
    """Masses, Kp, Kd and torque limits all doubled scale the equations of motion, Stable-PD, the torque clamp and the friction cone together:
    from the same 32 snapshots of a random-action rollout, 10 updates move the character as on the nominal handle, within the parity tests'
    tolerances (pose 1e-3, velocities 5e-2), and the imitation reward (COM term included) agrees to 2e-5.  Environments where a joint-limit row
    reaches its fixed impulse cap are where the identity does not hold; none of these states reaches it in 10 updates."""
    rng = np.random.default_rng(11)
    nom, dbl = _core(32), _core(32)
    acts = [_actions(nom, rng) for _ in range(4)]
    _run(nom, acts[:3], resets=False)
    snaps = [nom.get_snapshot(e) for e in range(32)]
    for c in (nom, dbl):
        for e, s in enumerate(snaps):
            c.set_snapshot(e, s)
    f = _unit(dbl)
    f[:, 1:] = 2.0
    dbl.set_dynamics(f)
    for c in (nom, dbl):
        c.set_action(acts[3])
        c.update(DT, 10)
    lay = SnapLayout(nom.dims.num_joints)
    jt = joint_types_from_assets(asset_root, "data/characters/humanoid3d.txt")
    worst_q = worst_qd = 0.0
    for e in range(32):
        eq, eqd = compare_sim_state(lay, nom.get_snapshot(e), dbl.get_snapshot(e), jt)
        worst_q, worst_qd = max(worst_q, eq), max(worst_qd, eqd)
    _, wn = _observe(nom)
    _, wd = _observe(dbl)
    print("scale identity: worst |dq| %.3g |dqd| %.3g |dr| %.3g" % (worst_q, worst_qd, np.abs(wn - wd).max()))
    assert worst_q < 1e-3 and worst_qd < 5e-2 and np.abs(wn - wd).max() < 2e-5


BOUNDS = dict(friction=(0.4, 1.2), kp=(0.8, 1.2), kd=(0.7, 1.3), torque_limit=(0.5, 1.0), mass=(0.7, 1.3))
LOHI = [v for k in ref.KINDS for v in BOUNDS[k]]


def test_randomised_table_equals_the_restatement_and_resumes(asset_root):
    """256 spin-kick environments, 60 policy steps with resets (none after every fourth step): after every step the table equals the restatement
    from the device's reset counters, bit for bit.  A save after 40 steps, loaded into a fresh randomised handle, continues bit-identically; a
    plain handle and a handle of other bounds refuse the blob, and the randomised handle refuses the plain handle's."""
    lp = ref.lumped_leaves(os.path.join(asset_root, "data", "characters", "humanoid3d.txt"))
    rng = np.random.default_rng(7)
    a = _core(256, seed=13)
    a.set_env_order(True)
    a.set_dynamics_randomization(LOHI)
    acts = [_actions(a, rng) for _ in range(60)]
    seed = ref.dyn_seed(13)
    seen = set()
    blob40, rec_a = None, []
    for step, x in enumerate(acts):
        a.set_action(x)
        a.update(DT, 20)
        if step % 4 != 3:
            a.reset(False)
        _, _, fl = _blocks(a, a.save_state())
        tab = _dyn(a)
        for e in range(256):
            r = int(fl[e, 7])
            seen.add((e, r))
            assert tab[e].tobytes() == ref.draw_env(LOHI, seed, e, r, lp).tobytes(), (step, e, r)
        if step == 39:
            blob40 = a.save_state()
        if step >= 40:
            rec_a.append((tab, _observe(a)))
    assert len(seen) > 256 + 100   # episodes restarted
    b = _core(256, seed=13)
    b.set_env_order(True)
    b.set_dynamics_randomization(LOHI)
    b.load_state(blob40)
    for step, x in enumerate(acts[40:]):
        b.set_action(x)
        b.update(DT, 20)
        if (step + 40) % 4 != 3:
            b.reset(False)
        tab = _dyn(b)
        st, rw = _observe(b)
        assert tab.tobytes() == rec_a[step][0].tobytes()
        assert st.tobytes() == rec_a[step][1][0].tobytes() and rw.tobytes() == rec_a[step][1][1].tobytes()
    assert a.save_state().tobytes() == b.save_state().tobytes()
    plain = _core(256, seed=13)
    with pytest.raises(RuntimeError, match="another dynamics table"):
        plain.load_state(blob40)
    with pytest.raises(RuntimeError, match="another dynamics table"):
        b.load_state(plain.save_state())
    other = _core(256, seed=13)
    other.set_dynamics_randomization([v * 0.5 if i % 2 == 0 else v for i, v in enumerate(LOHI)])
    with pytest.raises(RuntimeError, match="dynamics randomisation"):
        other.load_state(blob40)


def test_refusals():
    c = _core(4)
    nl = c.dims.num_joints
    with pytest.raises(RuntimeError, match="no dynamics table"):
        _dyn(c)
    for env, col, val, match in ((2, 0, -0.5, "environment 2: friction"), (1, 1, np.inf, "environment 1: kp"), (3, 2, np.nan, "environment 3: kd"),
                                 (0, 3, -1.0, "environment 0: torque_limit"), (2, 4 + 3, 0.0, "environment 2: mass of link 3"),
                                 (1, 4 + 8, 1.5, "environment 1: mass of link 8 differs from its parent link 7")):
        f = _unit(c)
        f[env, col] = val
        with pytest.raises(RuntimeError, match=match):
            c.set_dynamics(f)
    f = _unit(c)
    f[:, 4 + 7] = f[:, 4 + 8] = 1.5   # a wrist with its elbow's factor
    c.set_dynamics(f)
    assert np.array_equal(_dyn(c), f)
    with pytest.raises(RuntimeError, match="dm_set_dynamics, which own"):
        c.set_dynamics_randomization(LOHI)
    r = _core(4)
    for k, (lo, hi), match in ((0, (1.2, 0.4), "friction: lo > hi"), (1, (-0.1, 1.0), "kp: a bound is negative"), (2, (0.5, np.inf), "kd: a bound is not finite"),
                               (3, (np.nan, 1.0), "torque_limit: a bound is not finite"), (4, (0.0, 1.3), "mass: lo must be > 0")):
        lohi = list(LOHI)
        lohi[2 * k], lohi[2 * k + 1] = lo, hi
        with pytest.raises(RuntimeError, match=match):
            r.set_dynamics_randomization(lohi)
    r.set_dynamics_randomization(LOHI)
    with pytest.raises(RuntimeError, match="randomised"):
        r.set_dynamics(_unit(r))
    assert _dyn(r).shape == (4, 4 + nl)


ORACLE_CASES = [  # name, arguments, character, controller, placement by contact load
    ("spinkick", SPINKICK, "humanoid3d", "humanoid3d_phase_rot_ctrl", True),
    ("dog_trot", ["--arg_file", "args/run_dog3d_trot_args.txt"], "dog3d", "dog3d_phase_rot_ctrl", False),
    ("target_amp", ["--motion_file", "data/datasets/test_clips_mini.txt", "--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"],
     "humanoid3d", None, True),
]


@pytest.mark.parametrize("case", ORACLE_CASES, ids=[c[0] for c in ORACLE_CASES])
def test_factors_match_the_oracle_built_from_edited_assets(asset_root, tmp_path, case):
    """Environment 0 with non-uniform mass factors (each lumped wrist with its elbow's), friction 0.6, Kp x 1.2, Kd x 0.8 and torque limits
    x 0.9, every other environment with other factors (so that whichever environment shares environment 0's W = 16 warp differs from it):
    teacher-forced over 20 updates from two clip times against the CPU oracle built from asset files with those masses, gains and limits edited
    and its contact friction set to 0.81 x 0.6.  q and q-dot within the parity tests' tolerances (1e-3, 5e-2), the imitation reward (its COM
    term weighs the edited masses) within 2e-5 for the imitate scenes.  Spin kick runs the W = 16 imitate kernel with placement on, dog trot the W = 32 one, target_amp
    the W = 16 task kernel."""
    import json
    import torch
    from deepmimic_b200.capi import BatchedCore
    from tests.oracle_binding import Oracle
    name, args, char, ctrl, placement = case
    char_file = "data/characters/%s.txt" % char
    if ctrl is None:   # the scene's own controller file, from its arg file
        words = open(os.path.join(asset_root, args[-1])).read().split()
        ctrl_file = words[words.index("--char_ctrl_files") + 1]
    else:
        ctrl_file = "data/controllers/%s.txt" % ctrl
    lp = ref.lumped_leaves(os.path.join(asset_root, char_file))
    nl = len(lp)
    rng = np.random.default_rng(1)
    mass = rng.uniform(0.7, 1.3, nl).astype(np.float32)
    for l, p in enumerate(lp):
        if p >= 0:
            mass[l] = mass[p]
    fr, kp, kd, tl = 0.6, 1.2, 0.8, 0.9
    tree = ref.edited_asset_tree(asset_root, str(tmp_path / "assets"), char_file, ctrl_file, kp, kd, tl, mass)
    assert json.load(open(os.path.join(tree, char_file)))["BodyDefs"][1]["Mass"] != json.load(open(os.path.join(asset_root, char_file)))["BodyDefs"][1]["Mass"]
    orc = Oracle(args, tree)
    orc.set_friction(fr)
    N = 64
    core = BatchedCore(args, N, asset_root, device=0, seed=1)
    core.set_env_order(placement)
    tab = np.empty((N, 4 + nl), dtype=np.float32)
    tab[:, :4] = (1.3, 0.9, 1.1, 1.0)
    tab[:, 4:] = 1.1
    tab[0, :4] = (fr, kp, kd, tl)
    tab[0, 4:] = mass
    core.set_dynamics(tab)
    lay = SnapLayout(nl)
    jt = joint_types_from_assets(asset_root, char_file)
    worst_q = worst_qd = worst_r = 0.0
    contacts = 0
    rw = torch.zeros(N, device="cuda")
    for kin_time in (0.4, 0.9):
        orc.reset(kin_time, 0.0, 20.0)
        orc.set_action(0.1 * rng.standard_normal(orc.action_size))
        for _ in range(20):
            core.set_snapshot(0, orc.get_snapshot())
            core.update(DT, 1)
            orc.update(DT)
            so, sg = orc.get_snapshot(), core.get_snapshot(0)
            eq, eqd = compare_sim_state(lay, so, sg, jt)
            worst_q, worst_qd = max(worst_q, eq), max(worst_qd, eqd)
            contacts += sum(lay.contact_counts(so))
        if name != "target_amp":   # the task scene's imitation reward also needs the environment's clip of the dataset, not in the snapshot
            core.set_snapshot(0, orc.get_snapshot())
            core.reward_imitate(rw)
            core.sync()
            worst_r = max(worst_r, abs(orc.calc_reward_imitate() - rw[0].item()))
    print("%s: worst |dq| %.3g |dqd| %.3g |dr| %.3g, %d contact points" % (name, worst_q, worst_qd, worst_r, contacts))
    assert contacts > 0
    assert worst_q < 1e-3 and worst_qd < 5e-2 and worst_r < 2e-5


def test_trainer_resumes_bit_for_bit_under_randomised_dynamics(asset_root, tmp_path):
    """--rand_mass 0.8,1.2 --rand_friction 0.5,1.5 on the training handle: 3 iterations straight against 1, a checkpoint, a fresh Trainer from
    it and 2 more, every tensor of the state, the env blobs (the table included) and the log rows but wall time bit-identical.  The evaluation
    handle has no dynamics table; a Trainer without the randomisation refuses the checkpoint."""
    from tests.test_train_gpu import AGENT, SPINKICK_TRAIN, _equal_states, _trainer
    dr = dict(mass=(0.8, 1.2), friction=(0.5, 1.5))
    v = dict(AGENT, OutputIters=2, TestEpisodes=8)
    a = _trainer(asset_root, SPINKICK_TRAIN, v, num_envs=256, dynamics_randomization=dr)
    rows_a = [a.iteration() for _ in range(3)]
    b = _trainer(asset_root, SPINKICK_TRAIN, v, num_envs=256, dynamics_randomization=dr)
    rows_b = [b.iteration()]
    b.save(str(tmp_path / "c.pt"))
    del b
    c = _trainer(asset_root, SPINKICK_TRAIN, v, num_envs=256, dynamics_randomization=dr)
    c.load(str(tmp_path / "c.pt"))
    rows_b += [c.iteration() for _ in range(2)]
    strip = lambda r: {k: x for k, x in r.items() if k != "Wall_Time"}
    assert [repr(strip(r)) for r in rows_a] == [repr(strip(r)) for r in rows_b]
    assert not _equal_states(a.state_dict(), c.state_dict())
    tab = _dyn(a.env._core)
    assert tab[:, 0].min() >= 0.5 and tab[:, 0].max() <= 1.5 and tab[:, 4:].min() >= 0.8 and tab[:, 4:].max() <= 1.2
    assert np.all(tab[:, 1:4] == 1.0) and len(np.unique(tab[:, 0])) > 200
    with pytest.raises(RuntimeError, match="no dynamics table"):
        a.test_env._core.dynamics()
    d = _trainer(asset_root, SPINKICK_TRAIN, v, num_envs=256)
    with pytest.raises(ValueError, match="dynamics randomisation"):
        d.load(str(tmp_path / "c.pt"))


def _run_cmd(asset_root, prefix, out, n, extra):
    import subprocess
    import sys
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-m", "deepmimic_b200.run", "--asset_root", asset_root] + SPINKICK + [
        "--model_files", prefix, "--output_path", str(out), "--num_envs", str(n), "--episode_time", "6"] + list(extra)
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=repo), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout


def test_dynamics_sweep_of_the_spinkick_policy(asset_root, tmp_path):
    """The committed spin-kick fp16 policy in test mode, 128 environments of 6 s, plain and with --dynamics_sweep friction=1,0.2 and
    mass=1,1.5: the environments with the nominal value run exactly the plain run's episodes (unit factors are the plain kernel bit for bit),
    the run log gets the Dyn_<KIND> column and the summary one line per value"""
    from deepmimic_b200.formats import read_table_log
    from tests.test_run_cpu import _bundle, _fixture
    prefix = _bundle(tmp_path, _fixture("policy_humanoid3d_spinkick_fp16.npz"))
    N = 128
    _run_cmd(asset_root, prefix, tmp_path / "plain", N, [])
    plain = read_table_log(str(tmp_path / "plain" / "run_log.txt"))
    surv = {}
    for kind, vals in (("friction", (1.0, 0.2)), ("mass", (1.0, 1.5))):
        out = tmp_path / kind
        stdout = _run_cmd(asset_root, prefix, out, N, ["--dynamics_sweep", "%s=%s" % (kind, ",".join("%g" % x for x in vals))])
        print(stdout)
        log = read_table_log(str(out / "run_log.txt"))
        col = log["Dyn_" + kind]
        assert list(col) == [vals[e % 2] for e in range(N)]
        nom = col == 1.0
        assert np.array_equal(log["Terminate"][nom], plain["Terminate"][nom]) and np.array_equal(log["Return"][nom], plain["Return"][nom])
        lines = [l for l in stdout.splitlines() if l.startswith(kind + " x ")]
        assert len(lines) == 2 and "64 episodes" in lines[0]
        for x in vals:
            surv[(kind, x)] = float(np.mean(log["Terminate"][col == x] != 1))
    print("survival by factor:", surv)
    assert surv[("friction", 1.0)] == surv[("mass", 1.0)]
    # measured (H100, this seed and batch): 0.969 of the nominal episodes survive 6 s, 0.031 at friction x 0.2, 0.0 with every mass x 1.5
    assert surv[("friction", 1.0)] >= 0.9
    assert surv[("friction", 0.2)] <= 0.25
    assert surv[("mass", 1.5)] <= 0.25
