"""GPU parity: the CUDA path called through the C ABI against the CPU oracle on identical inputs.
Tolerances (BASELINE.md / SURVEY.md 8(d)): teacher-forced single Update(1/600): |dq|, |dqd| <= 1e-3;
reward / observation as pure functions of identical state <= 2e-5 (fp32 vs the reference's f64)."""
import numpy as np
import pytest

from tests.oracle_binding import Oracle
from tests.parity_util import SnapLayout, compare_sim_state, joint_types_from_assets, random_policy_action

pytestmark = pytest.mark.gpu

CASES = [
    ("args/run_humanoid3d_spinkick_args.txt", "data/characters/humanoid3d.txt"),
    ("args/train_humanoid3d_walk_args.txt", "data/characters/humanoid3d.txt"),
    ("args/train_dog3d_trot_args.txt", "data/characters/dog3d.txt"),
]


def _mk(asset_root, arg_file, num_envs):
    import torch
    from deepmimic_b200.capi import BatchedCore
    assert torch.cuda.is_available()
    core = BatchedCore(["--arg_file", arg_file], num_envs, asset_root, device=0, seed=1234)
    orc = Oracle(["--arg_file", arg_file], asset_root)
    return core, orc


@pytest.mark.parametrize("arg_file,char_file", CASES)
def test_reset_obs_reward_match_oracle(asset_root, arg_file, char_file):
    import torch
    core, orc = _mk(asset_root, arg_file, 8)
    jt = joint_types_from_assets(asset_root, char_file)
    lay = SnapLayout(orc.num_joints)
    times = np.linspace(0.0, 0.95 * orc.motion_duration, 8)
    core.reset(True, kin_time=times, max_time=np.full(8, 20.0), rot_theta=np.zeros(8))
    st = torch.zeros(8, core.dims.state_size, device="cuda"); rw = torch.zeros(8, device="cuda")
    core.observe(st, rw); core.sync()
    for e, t0 in enumerate(times):
        orc.reset(float(t0), 0.0, 20.0)
        so, sg = orc.get_snapshot(), core.get_snapshot(e)
        eq, eqd = compare_sim_state(lay, so, sg, jt)
        assert eq < 2e-5 and eqd < 2e-4, (e, eq, eqd)
        assert np.abs(so[lay.scal:lay.scal + 14] - sg[lay.scal:lay.scal + 14]).max() < 1e-5
        assert abs(orc.calc_reward() - rw[e].item()) < 2e-5, (orc.reward_terms(), rw[e].item())
        assert np.abs(orc.record_state() - st[e].cpu().numpy().astype(np.float64)).max() < 1e-4


def _explained_by_branch_flip(orc2, lay, jt, before, sg, rng, tries=64):
    """Contact handling has discrete branches (a cached manifold point kept or dropped at the breaking threshold, the support
    vertex of a flat box).  At a state that sits on such a threshold the ORACLE ITSELF flips under ulp-level input noise.
    Returns True when the oracle, restarted from `before` with 1e-6 relative noise on the velocities, reproduces the GPU
    result -- i.e. the GPU took a branch the reference arithmetic also takes, rather than computing something different."""
    nl = lay.nl
    for _ in range(tries):
        p = before.copy()
        p[lay.jvel: lay.jvel + 3 * nl] *= 1.0 + 1e-6 * rng.standard_normal(3 * nl)
        p[7:13] *= 1.0 + 1e-6 * rng.standard_normal(6)
        orc2.set_snapshot(p)
        orc2.update(1.0 / 600.0)
        s2 = orc2.get_snapshot()
        eq, eqd = compare_sim_state(lay, s2, sg, jt)
        if eq <= 1e-4 and eqd <= 5e-2 and lay.contact_counts(s2) == lay.contact_counts(sg):
            return True
    return False


@pytest.mark.parametrize("arg_file,char_file", CASES)
def test_teacher_forced_update_matches_oracle(asset_root, arg_file, char_file):
    """Each Update(1/600) starts from the oracle's exact state (q, qd, PD targets, contact cache, clocks).

    Stated fp32 tolerances (DESIGN.md "Parity"):
      q   (quaternion components, angles, root position in m): <= 1e-3 always            (measured <= 6e-5)
      qd  contact-free updates: <= 1e-3 humanoid3d / 6e-3 dog3d                           (measured 4e-4 / 4.4e-3)
      qd  updates with active contact rows: median <= 2e-3, p99 <= 5e-2, max <= 0.5 rad/s -- Bullet's Baumgarte term
          (erp / h = 240 1/s) amplifies ulp-level (1e-6) differences of two correct fp32 forward-kinematics evaluations into
          ~1e-3 relative impulse differences on the light foot links; the oracle itself is only defined to that level.
      contact cache: identical point counts per link after every update; need_new_action flag identical."""
    import torch
    core, orc = _mk(asset_root, arg_file, 4)
    orc2 = Oracle(["--arg_file", arg_file], asset_root)
    jt = joint_types_from_assets(asset_root, char_file)
    lay = SnapLayout(orc.num_joints)
    off, scl, lo, hi = orc.action_statics()
    rng = np.random.default_rng(1234)
    rng2 = np.random.default_rng(99)
    dog = "dog" in arg_file
    eqs, eqds, ncs = [], [], []
    flips, total = 0, 0
    worst_r = worst_s = 0.0
    rw = torch.zeros(4, device="cuda"); st = torch.zeros(4, core.dims.state_size, device="cuda")
    for t0 in (0.0, 0.3, 0.6, 0.9):
        orc.reset(t0 * orc.motion_duration / 1.283282, 0.0, 20.0)
        for upd in range(200):
            if orc.need_new_action():
                orc.set_action(random_policy_action(rng, off, scl, lo, hi))
            if orc.is_episode_end():
                break
            before = orc.get_snapshot()
            core.set_snapshot(0, before)
            core.update(1.0 / 600.0, 1)
            orc.update(1.0 / 600.0)
            so, sg = orc.get_snapshot(), core.get_snapshot(0)
            eq, eqd = compare_sim_state(lay, so, sg, jt)
            total += 1
            assert bool(sg[lay.scal + 11]) == orc.need_new_action()
            if eq > 1e-3 or eqd > 0.5 or lay.contact_counts(so) != lay.contact_counts(sg):
                assert _explained_by_branch_flip(orc2, lay, jt, before, sg, rng2), (t0, upd, eq, eqd, lay.contact_counts(so), lay.contact_counts(sg))
                flips += 1
                continue
            eqs.append(eq); eqds.append(eqd); ncs.append(sum(lay.contact_counts(so)))
            if upd % 5 == 0 and not orc.has_fallen():   # reward / observation as pure functions of the oracle's post-state
                core.set_snapshot(1, so)
                core.observe(st, rw); core.sync()
                worst_r = max(worst_r, abs(orc.calc_reward() - rw[1].item()))
                worst_s = max(worst_s, np.abs(orc.record_state() - st[1].cpu().numpy().astype(np.float64)).max())
    eqs, eqds, ncs = np.array(eqs), np.array(eqds), np.array(ncs)
    print("teacher-forced %s: %d branch flips in %d updates" % (arg_file, flips, total))
    assert flips <= max(1, total // 100)
    print("teacher-forced %s: %d updates (%d with contacts) |dq| max %.2e ; |dqd| median %.2e p99 %.2e max %.2e (contact-free max %.2e) ; reward %.1e obs %.1e"
          % (arg_file, len(eqs), int((ncs > 0).sum()), eqs.max(), np.median(eqds), np.percentile(eqds, 99), eqds.max(), eqds[ncs == 0].max(), worst_r, worst_s))
    assert (ncs > 0).sum() > 50
    assert eqds[ncs == 0].max() <= (6e-3 if dog else 1e-3)
    assert np.median(eqds) <= 2e-3 and np.percentile(eqds, 99) <= 5e-2 and eqds.max() <= 0.5
    assert worst_r < 2e-5 and worst_s < 2e-4
    assert core.counters()[1] == 0   # solver row capacity never exceeded


def test_free_running_statistics_match_oracle(asset_root):
    """Chaotic divergence makes free-running trajectories incomparable; compare distributions instead (SURVEY 7, hard part 2)."""
    import torch
    arg_file = "args/train_humanoid3d_walk_args.txt"
    core, orc = _mk(asset_root, arg_file, 64)
    off, scl, lo, hi = orc.action_statics()
    rng = np.random.default_rng(7)
    N, A = 64, core.dims.action_size
    times = rng.uniform(0, orc.motion_duration, N)
    core.reset(True, kin_time=times, max_time=np.full(N, 20.0), rot_theta=np.zeros(N))
    acts = np.stack([np.stack([random_policy_action(rng, off, scl, lo, hi) for _ in range(N)]) for _ in range(12)])
    rw = torch.zeros(N, device="cuda"); fl = torch.zeros(N, 4, dtype=torch.int32, device="cuda")
    g_rewards, g_done = [], np.zeros(N, bool)
    for s in range(12):
        core.observe(None, rw); core.flags(fl); core.sync()
        g_done |= fl[:, 1].cpu().numpy().astype(bool)
        g_rewards.append(np.where(g_done, np.nan, rw.cpu().numpy()))
        core.set_action(torch.tensor(acts[s], dtype=torch.float32, device="cuda"))
        core.update(1.0 / 600.0, 20)
    o_rewards, o_done = [], np.zeros(N, bool)
    for e in range(N):
        orc.reset(float(times[e]), 0.0, 20.0)
        rs = []
        for s in range(12):
            rs.append(np.nan if o_done[e] else orc.calc_reward())
            orc.set_action(acts[s][e])
            for _ in range(20):
                if not o_done[e]:
                    orc.update(1.0 / 600.0)
                    o_done[e] |= orc.is_episode_end()
        o_rewards.append(rs)
    core.flags(fl); core.sync()
    g_done |= fl[:, 1].cpu().numpy().astype(bool)
    g = np.array(g_rewards).T; o = np.array(o_rewards)
    # first steps are still tightly coupled
    assert np.nanmax(np.abs(g[:, :2] - o[:, :2])) < 5e-3
    assert abs(np.nanmean(g) - np.nanmean(o)) < 0.03
    assert abs(g_done.mean() - o_done.mean()) < 0.15


def test_many_contacts_general_solver_path(asset_root):
    """With fall termination switched off the character ends up lying on the ground with up to ~10 contact points (30+ solver rows):
    more rows than lanes, so the packed-triangle / multi-slot path of the constraint solver is exercised (the common path handles
    <= W rows).  Same teacher-forced comparison and tolerances as above."""
    args = ["--enable_char_contact_fall", "false", "--arg_file", "args/run_humanoid3d_spinkick_args.txt"]
    import torch
    from deepmimic_b200.capi import BatchedCore
    core = BatchedCore(args, 4, asset_root, device=0, seed=3)
    orc = Oracle(args, asset_root); orc2 = Oracle(args, asset_root)
    jt = joint_types_from_assets(asset_root, "data/characters/humanoid3d.txt")
    lay = SnapLayout(orc.num_joints)
    rng2 = np.random.default_rng(5)
    orc.reset(0.3, 0.0, 20.0)
    zero = np.zeros(orc.action_size)
    eqs, eqds, ncs, flips = [], [], [], 0
    for upd in range(900):
        if orc.need_new_action():
            orc.set_action(zero)
        assert not orc.is_episode_end()
        before = orc.get_snapshot()
        if upd < 600:          # let it fall on the oracle alone; compare the contact-rich part
            orc.update(1.0 / 600.0)
            continue
        core.set_snapshot(0, before)
        core.update(1.0 / 600.0, 1)
        orc.update(1.0 / 600.0)
        so, sg = orc.get_snapshot(), core.get_snapshot(0)
        eq, eqd = compare_sim_state(lay, so, sg, jt)
        if eq > 1e-3 or eqd > 0.5 or lay.contact_counts(so) != lay.contact_counts(sg):
            assert _explained_by_branch_flip(orc2, lay, jt, before, sg, rng2), (upd, eq, eqd, lay.contact_counts(so), lay.contact_counts(sg))
            flips += 1
            continue
        eqs.append(eq); eqds.append(eqd); ncs.append(sum(lay.contact_counts(so)))
    eqs, eqds, ncs = np.array(eqs), np.array(eqds), np.array(ncs)
    print("many contacts: %d updates, contact points max %d mean %.1f, branch flips %d ; |dq| max %.2e ; |dqd| median %.2e p99 %.2e max %.2e"
          % (len(eqs), ncs.max(), ncs.mean(), flips, eqs.max(), np.median(eqds), np.percentile(eqds, 99), eqds.max()))
    assert ncs.max() >= 6            # more than 16 rows at some point
    assert flips <= max(2, len(eqs) // 50)
    assert np.median(eqds) <= 2e-3 and np.percentile(eqds, 99) <= 5e-2 and eqds.max() <= 0.5
    assert core.counters()[1] == 0   # row capacity (36 rows) not exceeded
