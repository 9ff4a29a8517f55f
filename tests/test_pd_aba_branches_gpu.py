"""The step kernel's Stable-PD stage, articulated-body solve and position integration against the CPU oracle on the constructed states of
tests/char_shapes.py, on the constructed characters (16, 17, 32 links, 96 dofs; one and three Bullet sub-steps) and the shipped ones.

  1. every state, one teacher-forced update per environment (dt 1/600; the integ_clamp states 1/60, 1/40 with three sub-steps): q within
     max(Q_FLOOR, 8 x the update's own oracle envelope over 16 fp32-rounding replicas), q-dot within max(QD_FLOOR[character], 8 x its
     envelope) (tools/qd_envelope.py's protocol, char_shapes.bounds), the valid and terminate flags equal.  Every state is airborne, so the
     envelope is fp32 rounding alone.  Measured on an H100 80GB HBM3 at 700 W (the floors are chosen from this, char_shapes.py):
       largest q-dot error among the updates whose 8 x envelope is below 3e-4, per character: c16 2.7e-5, c17 1.1e-5, c32 2.9e-5,
       c96 7.6e-5, humanoid3d 9.5e-5, dog3d 1.5e-4 (its free states, the only updates of any character where a floor is the bound);
       floors QD_FLOOR: c16 6e-5, c17 3e-5, c32 6e-5, c96 2e-4, humanoid3d 2e-4, dog3d 3e-4; Q_FLOOR 1e-5 over |dq| at most 5.1e-7;
       largest error / bound outside integ_clamp, q-dot: c16 0.44, c17 0.17, c32 0.27, c96 0.38, humanoid3d 0.48, dog3d 0.63 (a clamp
       state, bounded by its envelope; 0.48 where the floor binds); q at most 0.05; the integ_clamp updates (q-dot errors up to 6e-2)
       at most 0.48 (q) and 0.15 (q-dot) of their envelope bounds; the push and dynamics updates of 4 at most 0.25.
     A kernel that clamps the torque per component instead of by its norm fails on the clamp, sph_err (past pi) and integ_clamp states
     of every character, by 33 to 3 x 10^5 times the bound.  One that replaces the root's Stable-PD bias quirk by w x v passes, with
     errors of the same size: an equivalent change (tests/test_char_shapes_cpu.py states and checks the identity);
  2. 20 updates in one launch and 20 single launches give bit-identical snapshots on every constructed character;
  3. partners do not matter on c16 (W = 16, index placement: environments (2k, 2k+1) share a warp);
  4. the push kernel (aba_solve_push) on c32 with a push on a leaf lumped into a spherical parent, a fixed leaf under a fixed link and one under
     the root (not lumped), a fixed link with children and the root; the dynamics kernel (aba_solve_dyn) with non-unit mass factors, gains
     and torque limits against the oracle built from edited assets, on c16 and c32; one teacher-forced update each, bounds as in 1;
  5. observation and imitation reward of the constructed states within 2e-4 / 2e-5 (tests/test_policy_kernels_gpu.py): dm_policy.cu's
     per-link loops at 16, 17, 31 and 32 links."""
import numpy as np
import pytest

from tests import char_shapes as C
from tests.oracle_binding import Oracle
from tests.parity_util import SnapLayout, compare_sim_state

pytestmark = pytest.mark.gpu
ALL = list(C.CHARS) + list(C.SHIPPED)


@pytest.fixture(scope="module")
def roots(asset_root, tmp_path_factory):
    return C.write_root(asset_root, str(tmp_path_factory.mktemp("char_shapes") / "assets")), asset_root


def _root(roots, name):
    return roots[1] if name in C.SHIPPED else roots[0]


def _core(args, root, n, seed=3):
    from deepmimic_b200.capi import BatchedCore
    core = BatchedCore(args, n, root, device=0, seed=seed)
    core.set_env_order(False)
    return core


def _one_update(args, root, snaps, dt):
    """device snapshots and flags after one update of every snapshot (one launch)"""
    import torch
    n = len(snaps)
    core = _core(args, root, n)
    for e, s in enumerate(snaps):
        core.set_snapshot(e, s)
    core.update(dt, 1)
    fl = torch.zeros(n, 4, dtype=torch.int32, device="cuda")
    core.flags(fl)
    core.sync()
    out = [core.get_snapshot(e) for e in range(n)], fl.cpu().numpy()
    core.close()
    return out


def _check(name, lay, jt, so, sg, env):
    eq, eqd = compare_sim_state(lay, so, sg, jt)
    bq, bqd = C.bounds(name, env)
    return eq, eqd, eq / bq, eqd / bqd


@pytest.mark.parametrize("name", ALL)
def test_updates_match_the_oracle_branch_by_branch(roots, name):
    root = _root(roots, name)
    args = C.args_of(name)
    orc, orc2 = Oracle(args, root), Oracle(args, root)
    J = C.load_joints(root, name)
    lay = SnapLayout(len(J)); jt = [j["Type"] for j in J]
    lib = C.library(orc, root, name)
    rng = np.random.default_rng(11)
    per = {}
    bad = []
    for dt in sorted({st.dt for st in lib}):
        group = [st for st in lib if st.dt == dt]
        dev, fl = _one_update(args, root, [st.snap for st in group], dt)
        for e, st in enumerate(group):
            orc.set_snapshot(st.snap)
            orc.update(dt)
            so = orc.get_snapshot()
            flags = (int(orc.check_terminate() != 0), int(orc.check_valid_episode()))
            env = C.envelope(orc2, lay, jt, st.snap, so, dt, rng)
            eq, eqd, rq, rqd = _check(name, lay, jt, so, dev[e], env)
            c = per.setdefault(st.cls, dict(n=0, q=0.0, qd=0.0, rq=0.0, rqd=0.0))
            c["n"] += 1; c["q"] = max(c["q"], eq); c["qd"] = max(c["qd"], eqd); c["rq"] = max(c["rq"], rq); c["rqd"] = max(c["rqd"], rqd)
            if rq > 1.0 or rqd > 1.0 or not np.isfinite(dev[e]).all():
                bad.append("%s: |dq| %.2e (%.2f of the bound) |dqd| %.2e (%.2f of the bound)" % (st, eq, rq, eqd, rqd))
            if (fl[e, 2], fl[e, 3]) != flags:
                bad.append("%s: terminate / valid flags %d %d, oracle %d %d" % (st, fl[e, 2], fl[e, 3], *flags))
    print("%s: %d updates compared" % (name, sum(c["n"] for c in per.values())))
    for k in C.CLASSES:
        if k in per:
            c = per[k]
            print("  %-12s %2d states  max |dq| %.2e |dqd| %.2e  max / bound: q %.3f qd %.3f" % (k, c["n"], c["q"], c["qd"], c["rq"], c["rqd"]))
    for b in bad:
        print("  MISMATCH " + b)
    assert not bad


@pytest.mark.parametrize("name", list(C.CHARS))
def test_fused_launch_equals_single_launches(roots, name):
    """20 updates in one launch (one table build) and 20 launches of one update give the same bits"""
    args = C.args_of(name)
    orc = Oracle(args, roots[0])
    snaps = [st.snap for st in C.library(orc, roots[0], name) if st.dt == C.DT]
    n = len(snaps)
    out = []
    for fused in (True, False):
        core = _core(args, roots[0], n)
        for e, s in enumerate(snaps):
            core.set_snapshot(e, s)
        if fused:
            core.update(C.DT, 20)
        else:
            for _ in range(20):
                core.update(C.DT, 1)
        core.sync()
        out.append([core.get_snapshot(e) for e in range(n)])
        core.close()
    for e in range(n):
        assert np.array_equal(out[0][e], out[1][e]), (name, e)
    print("%s: %d environments x 20 updates, fused == single launches" % (name, n))


def test_partners_do_not_change_an_environments_result(roots):
    name = "c16"
    args = C.args_of(name)
    lib = [st for st in C.library(Oracle(args, roots[0]), roots[0], name) if st.dt == C.DT]
    partners = [st for st in lib if st.cls in ("free", "clamp", "rev_wrap")][::2]
    snaps, where = [], {}
    for si, st in enumerate(lib):
        for p in partners:
            for first in (True, False):
                where.setdefault(si, []).append(len(snaps) + (0 if first else 1))
                snaps += [st.snap, p.snap] if first else [p.snap, st.snap]
    core = _core(args, roots[0], len(snaps))
    for e, s in enumerate(snaps):
        core.set_snapshot(e, s)
    core.update(C.DT, 5)
    core.sync()
    res = [core.get_snapshot(e) for e in range(len(snaps))]
    core.close()
    for si, envs in where.items():
        assert np.isfinite(res[envs[0]]).all()
        for e in envs[1:]:
            assert np.array_equal(res[e], res[envs[0]]), "%s depends on its partner (environment %d)" % (lib[si], e)
    print("partners: %d states x %d partners x 2 sides, equal" % (len(lib), len(partners)))


def test_push_kernel_on_each_body_class(roots):
    """c32: 10 is a leaf lumped into spherical 7, 4 a fixed leaf under fixed 1, 5 a fixed leaf under the root, 1 a fixed link with children"""
    from tests.push_oracle import PushOracle
    name = "c32"
    args = C.args_of(name)
    root = roots[0]
    J = C.load_joints(root, name)
    T = C.dyn_tree(J)
    assert T[10]["lumped"] and J[7]["Type"] == "spherical" and not T[4]["lumped"] and J[1]["Type"] == "fixed" and not T[5]["lumped"] and T[1]["children"]
    lay = SnapLayout(len(J)); jt = [j["Type"] for j in J]
    orc, orc2 = PushOracle(args, root), PushOracle(args, root)
    free = [st for st in C.library(Oracle(args, root), root, name) if st.cls == "free"]
    rng = np.random.default_rng(5)
    n = len(free)
    worst = (0.0, 0.0)
    for k, body in enumerate((10, 4, 5, 1, 0)):
        F = np.array([300.0 * np.cos(k), 150.0, 300.0 * np.sin(k)])
        core = _core(args, root, n)
        b = np.full(n, body, dtype=np.int32); f = np.tile(F.astype(np.float32), (n, 1))
        core.set_pushes(b, f, np.zeros(n), np.full(n, 100.0))
        for e, st in enumerate(free):
            core.set_snapshot(e, st.snap)
        core.update(C.DT, 1)
        core.sync()
        for e, st in enumerate(free):
            for o in (orc, orc2):
                o.set_push(body, F, 0.0, 100.0)
            orc.set_snapshot(st.snap)
            orc.update(C.DT)
            so = orc.get_snapshot()
            nopush = Oracle(args, root); nopush.set_snapshot(st.snap); nopush.update(C.DT)
            assert compare_sim_state(lay, so, nopush.get_snapshot(), jt)[1] > 10 * C.QD_FLOOR[name]   # the push moves the update
            env = C.envelope(orc2, lay, jt, st.snap, so, C.DT, rng)
            eq, eqd, rq, rqd = _check(name, lay, jt, so, core.get_snapshot(e), env)
            worst = (max(worst[0], rq), max(worst[1], rqd))
            assert rq <= 1.0 and rqd <= 1.0, (body, st, eq, eqd, rq, rqd)
        core.close()
    print("push on c32 bodies 10, 4, 5, 1, 0: %d updates, max / bound q %.3f qd %.3f" % (5 * n, *worst))


@pytest.mark.parametrize("name", ["c16", "c32"])
def test_dynamics_kernel_matches_the_oracle_built_from_edited_assets(roots, tmp_path, name):
    from tests.dynamics_oracle import DynamicsOracle, edited_asset_tree
    from tests.dynamics_ref import lumped_leaves
    import os
    root = roots[0]
    args = C.args_of(name)
    lp = lumped_leaves(os.path.join(root, C.char_file(name)))
    nl = len(lp)
    rng = np.random.default_rng(2)
    mass = rng.uniform(0.7, 1.3, nl).astype(np.float32)
    for l, p in enumerate(lp):
        if p >= 0:
            mass[l] = mass[p]
    kp, kd, tl = 1.2, 0.8, 0.9
    tree = edited_asset_tree(root, str(tmp_path / "edited"), C.char_file(name), "data/controllers/%s_ctrl.txt" % name, kp, kd, tl, mass)
    orc, orc2 = DynamicsOracle(args, tree), DynamicsOracle(args, tree)
    J = C.load_joints(root, name)
    lay = SnapLayout(nl); jt = [j["Type"] for j in J]
    states = [st for st in C.library(Oracle(args, root), root, name) if st.cls in ("free", "clamp", "rev_wrap", "integ")]
    n = len(states)
    core = _core(args, root, n)
    tab = np.empty((n, 4 + nl), dtype=np.float32)
    tab[:, :4] = (1.0, kp, kd, tl)
    tab[:, 4:] = mass
    core.set_dynamics(tab)
    for e, st in enumerate(states):
        core.set_snapshot(e, st.snap)
    core.update(C.DT, 1)
    core.sync()
    worst = (0.0, 0.0)
    for e, st in enumerate(states):
        orc.set_snapshot(st.snap)
        orc.update(C.DT)
        so = orc.get_snapshot()
        env = C.envelope(orc2, lay, jt, st.snap, so, C.DT, rng)
        eq, eqd, rq, rqd = _check(name, lay, jt, so, core.get_snapshot(e), env)
        worst = (max(worst[0], rq), max(worst[1], rqd))
        assert rq <= 1.0 and rqd <= 1.0, (st, eq, eqd, rq, rqd)
    core.close()
    print("dynamics factors on %s: %d updates, max / bound q %.3f qd %.3f" % (name, n, *worst))


@pytest.mark.parametrize("name", list(C.CHARS))
def test_observation_and_reward_match_the_oracle(roots, name):
    import torch
    args = C.args_of(name)
    orc = Oracle(args, roots[0])
    lib = [st for st in C.library(orc, roots[0], name) if st.cls in ("free", "clamp", "sph_err", "rev_wrap", "integ", "substeps")]
    n = len(lib)
    core = _core(args, roots[0], n)
    for e, st in enumerate(lib):
        core.set_snapshot(e, st.snap)
    S = core.dims.state_size
    assert S == orc.state_size
    obs = torch.full((n, S), float("nan"), device="cuda"); rw = torch.full((n,), float("nan"), device="cuda")
    torch.cuda.synchronize()
    core.observe(obs, rw)
    core.sync()
    g, r = obs.cpu().numpy(), rw.cpu().numpy()
    wo = wr = 0.0
    for e, st in enumerate(lib):
        orc.set_snapshot(st.snap)
        wo = max(wo, float(np.abs(g[e] - orc.record_state()).max()))
        wr = max(wr, abs(float(r[e]) - orc.calc_reward()))
    core.close()
    print("%s: %d states, worst observation error %.2e, reward error %.2e" % (name, n, wo, wr))
    assert wo <= 2e-4 and wr <= 2e-5
