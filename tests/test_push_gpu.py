"""Pushes on the GPU: the step kernel's push instantiations against the CPU oracle (teacher-forced, airborne and in ground contact, every
body class), the push window and its clearing on the device, placement by contact load, the refusals of dm_set_pushes and dm_save_state,
and the push-robustness sweep of a trained skill through the run command."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.oracle_binding import PushOracle
from tests.parity_util import SnapLayout, compare_sim_state, joint_types_from_assets, random_policy_action
from tests.test_run_cpu import _bundle, _fixture

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = 1.0 / 600.0
SPINKICK = ["--arg_file", "args/run_humanoid3d_spinkick_args.txt"]
DOG = ["--arg_file", "args/train_dog3d_trot_args.txt"]
TARGET = ["--motion_file", "data/datasets/test_clips_mini.txt", "--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]


def _body_classes(asset_root, char_file):
    """root, the first spherical, the first revolute joint's body and the first fixed leaf (lumped into its parent), where the character has one"""
    import json
    d = json.load(open(os.path.join(asset_root, char_file)))
    J = d["Skeleton"]["Joints"]
    types, parents = [j["Type"] for j in J], [j["Parent"] for j in J]
    kids = [sum(1 for p in parents if p == i) for i in range(len(J))]
    out = [0]
    for want in ("spherical", "revolute"):
        out += [i for i in range(1, len(J)) if types[i] == want][:1]
    out += [i for i in range(1, len(J)) if types[i] == "fixed" and kids[i] == 0 and types[parents[i]] != "fixed"][:1]
    return out


def _pushes(n, env, body, force, start=0.0, duration=100.0):
    b = np.full(n, -1, dtype=np.int32); f = np.zeros((n, 3), dtype=np.float32)
    b[env] = body; f[env] = force
    return b, f, np.full(n, start), np.full(n, duration)


CASES = [("spinkick", SPINKICK, "data/characters/humanoid3d.txt", 64, True),
         ("dog trot", DOG, "data/characters/dog3d.txt", 4, False),
         ("target_amp", TARGET, "data/characters/humanoid3d.txt", 4, False)]


@pytest.mark.parametrize("name,args,char,n,placement", CASES, ids=[c[0] for c in CASES])
def test_teacher_forced_push_matches_the_oracle(asset_root, name, args, char, n, placement):
    """Every Update(1/600) starts from the oracle's exact state; a push of 200-1000 N acts on one body of environment 0 in both.  Tolerances
    of test_parity_gpu.py: |dq| <= 1e-3; |dqd| contact-free <= 1e-3 (dog3d 6e-3), with contacts median <= 2e-3, p99 <= 5e-2, max <= 0.5;
    at most 2 % of the updates on a contact branch the oracle takes under ulp-level noise (not checked further here)."""
    from deepmimic_b200.capi import BatchedCore
    core = BatchedCore(args, n, asset_root, device=0, seed=1234)
    core.set_env_order(placement)
    orc = PushOracle(args, asset_root)
    jt = joint_types_from_assets(asset_root, char)
    lay = SnapLayout(orc.num_joints)
    off, scl, lo, hi = orc.action_statics()
    rng = np.random.default_rng(7)
    bodies = _body_classes(asset_root, char)
    eqs, eqds, ncs, odd, total = [], [], [], 0, 0
    for k, body in enumerate(bodies):
        for airborne in (False, True):
            F = rng.uniform(200.0, 1000.0) * np.array([np.cos(k + 0.5), 0.3 * (-1) ** k, np.sin(k + 0.5)])
            orc.reset(0.1 + 0.2 * k, 0.0, 20.0)
            if airborne:
                p, v = orc.get_pose()
                p = p.copy(); p[1] += 2.0
                orc.set_pose_vel(p, v)
            orc.set_push(body, F, 0.0, 100.0)
            core.set_pushes(*_pushes(n, 0, body, F.astype(np.float32)))
            for upd in range(40):
                if orc.need_new_action():
                    orc.set_action(random_policy_action(rng, off, scl, lo, hi))
                if orc.is_episode_end():
                    break
                core.set_snapshot(0, orc.get_snapshot())
                core.update(DT, 1)
                orc.update(DT)
                so, sg = orc.get_snapshot(), core.get_snapshot(0)
                eq, eqd = compare_sim_state(lay, so, sg, jt)
                total += 1
                if eq > 1e-3 or eqd > 0.5 or lay.contact_counts(so) != lay.contact_counts(sg):
                    odd += 1
                    continue
                eqs.append(eq); eqds.append(eqd); ncs.append(sum(lay.contact_counts(so)))
    eqs, eqds, ncs = np.array(eqs), np.array(eqds), np.array(ncs)
    print("push parity %s bodies %s: %d updates (%d with contacts, %d off-branch) |dq| max %.2e |dqd| median %.2e p99 %.2e max %.2e contact-free max %.2e"
          % (name, bodies, total, int((ncs > 0).sum()), odd, eqs.max(), np.median(eqds), np.percentile(eqds, 99), eqds.max(), eqds[ncs == 0].max()))
    assert odd <= max(1, total // 50)
    assert (ncs > 0).sum() > 20 and (ncs == 0).sum() > 20
    assert eqds[ncs == 0].max() <= (6e-3 if "dog" in name else 1e-3)
    assert eqs.max() <= 1e-3 and np.median(eqds) <= 2e-3 and np.percentile(eqds, 99) <= 5e-2 and eqds.max() <= 0.5


def test_push_window_and_clearing_on_the_device(asset_root):
    """From a reset, GPU and oracle apply the push in the same updates (start and duration off the update boundaries); the entry reads
    cleared after the window and after a reset"""
    from deepmimic_b200.capi import BatchedCore
    n = 4
    core = BatchedCore(SPINKICK, n, asset_root, device=0, seed=3)
    orc = PushOracle(SPINKICK, asset_root)
    jt = joint_types_from_assets(asset_root, "data/characters/humanoid3d.txt")
    lay = SnapLayout(orc.num_joints)
    orc.reset(0.4, 0.0, 20.0)
    core.set_snapshot(0, orc.get_snapshot())
    start, dur, F = 5.5 * DT, 3.2 * DT, np.array([600.0, 0.0, -300.0])
    orc.set_push(0, F, start, dur)
    core.set_pushes(*_pushes(n, 0, 0, F.astype(np.float32), start, dur))
    worst = 0.0
    for upd in range(14):
        core.set_snapshot(0, orc.get_snapshot())
        core.update(DT, 1)
        orc.update(DT)
        eq, eqd = compare_sim_state(lay, orc.get_snapshot(), core.get_snapshot(0), jt)
        worst = max(worst, eqd)
        t_next = (upd + 1) * DT          # the timer after this update: cleared once it reaches start + duration
        assert core.pushes()[0] == (-1 if t_next >= start + dur - 1e-12 else 0), upd
    assert worst < 5e-2
    core.set_pushes(*_pushes(n, 1, 4, np.array([500.0, 0.0, 0.0], dtype=np.float32)))
    assert list(core.pushes()) == [-1, 4, -1, -1]
    core.reset(False)                    # env 1 is not done: kept
    assert list(core.pushes()) == [-1, 4, -1, -1]
    core.reset(True)
    assert list(core.pushes()) == [-1, -1, -1, -1]


def test_placement_moves_a_push_with_its_environment(asset_root):
    """A batch of 64 with placement by contact load: two handles continue from the same saved state for one update, the second with a push on
    environment k.  The push moves only k; every other environment matches the plain handle within the teacher-forced tolerance (|dq| <= 1e-3,
    |dqd| <= 0.5; reported: bit-identical or not -- the push kernel is compiled separately)"""
    import torch
    from deepmimic_b200.capi import BatchedCore
    n, k = 64, 37
    cores = [BatchedCore(SPINKICK, n, asset_root, device=0, seed=11) for _ in range(2)]
    a, b = cores
    for c in cores:
        c.set_env_order(True)
    a.reset(True, kin_time=np.linspace(0.0, 1.2, n), max_time=np.full(n, 20.0), rot_theta=np.zeros(n))
    rng = np.random.default_rng(2)
    for step in range(6):   # a spread of contact loads, so that placement reorders the tiles
        a.set_action(torch.as_tensor(0.05 * rng.standard_normal((n, a.dims.action_size)), dtype=torch.float32, device="cuda"))
        a.update(DT, 20)
    b.load_state(a.save_state())
    b.set_pushes(*_pushes(n, k, 0, np.array([0.0, 0.0, 800.0], dtype=np.float32)))
    for c in cores:
        c.update(DT, 1)
        c.sync()
    runs = [np.stack([c.get_snapshot(e) for e in range(n)]) for c in cores]
    keys, order, _, _ = b.env_order()
    assert not np.array_equal(order, np.arange(len(order)))   # placement did reorder
    lay = SnapLayout(15)
    jt = joint_types_from_assets(asset_root, "data/characters/humanoid3d.txt")
    others = [e for e in range(n) if e != k]
    same = bool(np.array_equal(runs[0][others], runs[1][others]))
    errs = np.array([compare_sim_state(lay, runs[0][e], runs[1][e], jt) for e in others])
    eq_k, eqd_k = compare_sim_state(lay, runs[0][k], runs[1][k], jt)
    print("placement: other environments bit-identical %s (worst |dq| %.2e |dqd| %.2e); pushed environment |dqd| %.3f" % (same, errs[:, 0].max(), errs[:, 1].max(), eqd_k))
    assert errs[:, 0].max() <= 1e-3 and errs[:, 1].max() <= 0.5
    assert eqd_k > 0.05


def test_set_pushes_refusals_and_save_state(asset_root):
    from deepmimic_b200.capi import BatchedCore
    n = 4
    core = BatchedCore(SPINKICK, n, asset_root, device=0, seed=5)
    blob = core.save_state()             # no push table yet
    ok = _pushes(n, 2, 1, np.array([100.0, 0.0, 0.0], dtype=np.float32), 1.0, 0.2)
    for i, bad, match in ((0, np.full(n, 15, dtype=np.int32), "body out of"), (0, np.full(n, -2, dtype=np.int32), "body out of"),
                          (1, np.full((n, 3), np.nan, dtype=np.float32), "force"), (2, np.full(n, np.inf), "start"),
                          (3, np.full(n, -0.1), "duration"), (3, np.full(n, np.nan), "duration")):
        a = list(ok); a[i] = bad
        with pytest.raises(RuntimeError, match=match):
            core.set_pushes(*a)
    with pytest.raises(ValueError, match="force must be float32"):
        core.set_pushes(ok[0], ok[1].astype(np.float64), ok[2], ok[3])
    with pytest.raises(ValueError, match="body must be int32"):
        core.set_pushes(ok[0][:2], ok[1], ok[2], ok[3])
    core.set_pushes(*ok)
    with pytest.raises(RuntimeError, match="pending push"):
        core.save_state()
    core.update(DT, 20 * 45)             # 1.5 s: past the window (1.0 s + 0.2 s), or the episode ended before it (then frozen until its reset)
    core.reset(False)
    core.sync()
    assert (core.pushes() == -1).all()
    b2 = core.save_state()
    core.load_state(blob)
    core.load_state(b2)
    assert len(b2) == len(blob)


def _run_push(asset_root, prefix, out, n, forces, extra=()):
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-m", "deepmimic_b200.run", "--asset_root", asset_root] + SPINKICK + [
        "--model_files", prefix, "--output_path", str(out), "--num_envs", str(n), "--push_forces", forces] + list(extra)
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=REPO), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout


def test_push_sweep_of_the_spinkick_policy(asset_root, tmp_path):
    """The committed spin-kick fp16 policy in test mode through the CUDA path, 160 environments of 6 s: root pushes at 2 s for 0.2 s make falls
    more frequent with the force (pinned with margin around the measured fractions), and the run command writes the sweep's columns and its
    per-force summary"""
    from deepmimic_b200.formats import read_table_log
    prefix = _bundle(tmp_path, _fixture("policy_humanoid3d_spinkick_fp16.npz"))
    forces = [0.0, 150.0, 300.0, 600.0, 1200.0]
    out = tmp_path / "out"
    stdout = _run_push(asset_root, prefix, out, 160, ",".join("%g" % f for f in forces), ["--episode_time", "6"])
    print(stdout)
    log = read_table_log(str(out / "run_log.txt"))
    assert list(log["Push_Force"]) == [forces[e % len(forces)] for e in range(160)]
    assert ((log["Push_Dir"] >= 0) & (log["Push_Dir"] < 2 * np.pi)).all()
    fell = {f: float(np.mean(log["Terminate"][log["Push_Force"] == f] == 1)) for f in forces}
    print("fall fraction by push force:", fell)
    lines = [l for l in stdout.splitlines() if l.startswith("push ")]
    assert len(lines) == len(forces) and "32 episodes" in lines[0]
    # measured (H100, this seed and batch): 0.031 / 0.031 / 0.44 / 1.0 / 1.0 of the episodes fall at 0 / 150 / 300 / 600 / 1200 N
    assert fell[0.0] <= 1 / 16 and fell[150.0] <= 0.15
    assert 0.2 <= fell[300.0] <= 0.7
    assert fell[600.0] >= 0.85 and fell[1200.0] >= 0.85 and fell[1200.0] > fell[0.0]
