"""The step kernel's constraint solve against the CPU oracle on constructed states (tests/solver_states.py) that drive each of its branches
on purpose: the storage modes of solve_rows (W x W square, kSq2 square, packed triangle), shallow and deep joint-limit rows, the limit
impulse cap, the coordinate clamp at 100 and vel_pass, friction rows skipped for a point whose normal impulse is 0, HasVelExploded and
the row overflow.

  1. every state, one teacher-forced Update(1/600) per environment: q within 1e-3, q-dot within max(1e-3 / 6e-3 dog, 8 x that update's own
     oracle envelope over 16 fp32-rounding replicas) (tests/test_qd_envelope_gpu.py's protocol), the cached points' impulses within
     max(1e-3 (1 + |lambda|), 8 x their envelope), the valid and terminate flags equal -- or a contact branch flip the oracle reproduces
     under the same noise, at most 1 % of the updates (two of the ~200 per character);
  2. the device's solver row count of the last sub-step (the contact-load key, W = 16) equals the oracle's NL + 3P, truncated for an
     environment that overflowed; every storage mode is entered by at least one warp;
  3. partners do not matter (W = 16, index placement: warps hold environments (2k, 2k+1)): light and heavy states next to partners of every
     bucket, on both sides, and a partner whose episode ends 3 updates into a fused 20-update launch -- each state's snapshot,
     observation and reward are float-equal whatever its partner, and equal again with placement by contact load;
  4. overflow: counters()[1] counts exactly the environments that overflowed; their state stays finite."""
import numpy as np
import pytest

from tests import solver_states as S
from tests.oracle_binding import Oracle
from tests.parity_util import SnapLayout, compare_sim_state, joint_types_from_assets
from tools.env_order_stats import MODES, mode
from tools.qd_envelope import envelope, impulse_err, perturb

pytestmark = pytest.mark.gpu

ENVS = {"humanoid3d": 256, "dog3d": 192}   # every state of the library at least once, several blocks (humanoid 32, dog 16 environments per block)


def _load(core, snaps):
    for e, s in enumerate(snaps):
        core.set_snapshot(e, s)


def _truncated(nl, p, maxrows):
    return nl + 3 * p if nl + 3 * p <= maxrows else nl + 3 * ((maxrows - nl) // 3)


@pytest.mark.parametrize("ch", list(S.CHARS))
def test_constraint_solve_branches_match_the_oracle(asset_root, ch):
    import torch
    from deepmimic_b200.capi import BatchedCore
    c = S.CHARS[ch]
    n, W, maxrows = ENVS[ch], c["W"], c["maxrows"]
    orc, orc2 = Oracle(c["args"], asset_root), Oracle(c["args"], asset_root)
    lay = SnapLayout(orc.num_joints); jt = joint_types_from_assets(asset_root, c["char"])
    lib = S.build(orc, asset_root, ch)
    floor = 6e-3 if ch == "dog3d" else 1e-3
    rng = np.random.default_rng(7)
    # oracle side, once per state: result, branches, flags, envelope over 16 replicas
    ref = []
    for st in lib:
        rows, after = S.last_rows(orc, st.snap)
        veq, veqd, _, vimp = envelope(orc, orc2, lay, jt, st.snap, after, rng, 16, impulses=True)
        ref.append(dict(after=after, rows=rows, valid=orc.check_valid_episode(), term=orc.check_terminate() != 0, env=(veq, veqd, vimp),
                        over=bool(((rows[:, S.LIMITS] + 3 * rows[:, S.POINTS]) > maxrows).any())))
    # device side: environment e holds state e mod len(lib); a fresh handle (the overflow flag is sticky until the handle goes)
    core = BatchedCore(c["args"], n, asset_root, device=0, seed=3)
    core.set_env_order(False)
    idx = [e % len(lib) for e in range(n)]
    _load(core, [lib[i].snap for i in idx])
    core.update(S.DT, 1)
    fl = torch.zeros(n, 4, dtype=torch.int32, device="cuda"); core.flags(fl); core.sync()
    fl = fl.cpu().numpy()
    keys = core.env_order()[0][:n]
    over_envs = sum(ref[i]["over"] for i in idx)
    assert core.counters()[1] == over_envs, (core.counters()[1], over_envs)
    stats = dict(total=0, flips=0, unexplained=[], clamp=0, deep=0, sat=0, overflow=0, skip=0)
    errs = []   # gpu |dqd| / envelope bound, gpu impulse error / bound
    bad = []    # flag, row-count and finiteness mismatches
    rows_dev = np.zeros(n, dtype=np.int64)
    for e, i in enumerate(idx):
        st, r = lib[i], ref[i]
        sg = core.get_snapshot(e)
        rr = r["rows"]
        stats["clamp"] += int(rr[:, S.CLAMP_ABA].any() or rr[:, S.CLAMP_PGS].any())
        stats["deep"] += int(rr[:, S.LIMIT_DEEP].any()); stats["sat"] += int(rr[:, S.LIMIT_SAT].any()); stats["skip"] += int(rr[:, S.FRICTION_SKIP].any())
        nr_oracle = _truncated(int(rr[-1, S.LIMITS]), int(rr[-1, S.POINTS]), maxrows)
        rows_dev[e] = keys[e] if W == 16 else nr_oracle
        if r["over"]:   # the kernel truncates the contact points, the oracle does not: finite state and the truncated row count only
            stats["overflow"] += 1
            if not np.isfinite(sg).all():
                bad.append("%s env %d: overflowing environment is not finite" % (st, e))
            if W == 16 and rr[-1, S.LIMITS] + 3 * rr[-1, S.POINTS] > maxrows and keys[e] != nr_oracle:   # overflowed in the last sub-step
                bad.append("%s env %d: device rows %d, truncated oracle rows %d" % (st, e, keys[e], nr_oracle))
            continue
        stats["total"] += 1
        so = r["after"]
        veq, veqd, vimp = r["env"]
        eq, eqd = compare_sim_state(lay, so, sg, jt)
        same = lay.contact_counts(so) == lay.contact_counts(sg)
        ei = impulse_err(lay, so, sg)
        imp_bound = max(8.0 * vimp, 1e-3 * (1.0 + max(abs(so[lay.mani + 12 * k + 7]) for k in range(4 * lay.nl))))
        ok = same and eq <= 1e-3 and eqd <= max(floor, 8.0 * veqd) and ei <= imp_bound
        if ok:
            if fl[e, 3] != int(r["valid"]) or fl[e, 2] != int(r["term"]):
                bad.append("%s env %d: valid / terminate flags %d %d, oracle %d %d" % (st, e, fl[e, 3], fl[e, 2], r["valid"], r["term"]))
            if W == 16 and keys[e] != nr_oracle:
                bad.append("%s env %d: device rows %d, oracle NL + 3P %d" % (st, e, keys[e], nr_oracle))
            errs.append((eqd / max(floor, 8.0 * veqd), ei / imp_bound))
            continue
        # outlier: a contact branch flip the oracle reproduces under fp32 rounding noise, or a finding
        stats["flips"] += 1
        print("  branch flip: %s env %d, contacts %s vs %s" % (st, e, lay.contact_counts(so), lay.contact_counts(sg)))
        hit = False
        for _ in range(64):
            orc2.set_snapshot(perturb(lay, st.snap, rng, rel=4 * 2.0 ** -24))
            orc2.update(S.DT)
            s2 = orc2.get_snapshot()
            e2, e2d = compare_sim_state(lay, s2, sg, jt)
            if lay.contact_counts(s2) == lay.contact_counts(sg) and e2 <= 1e-3 and e2d <= max(floor, 8.0 * veqd, 0.1 * eqd):
                hit = True
                break
        if not hit:
            stats["unexplained"].append("%s env %d: |dq| %.2e |dqd| %.2e (bound %.2e) impulses %.2e (bound %.2e) contacts %s vs %s" % (
                st, e, eq, eqd, max(floor, 8.0 * veqd), ei, imp_bound, lay.contact_counts(so), lay.contact_counts(sg)))
    # storage modes entered per warp: W = 16 from the device keys of the pairs (2k, 2k+1), W = 32 from the oracle's row counts
    wmax = rows_dev.reshape(-1, 32 // W).max(axis=1)
    wm = mode(wmax, W)
    er = np.array(errs)
    pct = lambda a, p: float(np.percentile(a, p))
    print("%s: %d environments (%d states), %d warps per mode: %s" % (ch, n, len(lib), len(wm), ", ".join("%s %d" % (MODES[k], (wm == k).sum()) for k in range(4))))
    print("  compared %d updates; |dqd| / bound p50 %.3f p90 %.3f p99 %.3f max %.3f; impulses / bound p50 %.3f p90 %.3f max %.3f" % (
        stats["total"], pct(er[:, 0], 50), pct(er[:, 0], 90), pct(er[:, 0], 99), er[:, 0].max(), pct(er[:, 1], 50), pct(er[:, 1], 90), er[:, 1].max()))
    print("  branch flips %d (%d unexplained); updates with clamp %d, deep limit %d, limit impulse at the cap %d, friction skipped %d, overflow %d" % (
        stats["flips"], len(stats["unexplained"]), stats["clamp"], stats["deep"], stats["sat"], stats["skip"], stats["overflow"]))
    for u in stats["unexplained"]:
        print("  UNEXPLAINED " + u)
    for u in bad:
        print("  MISMATCH " + u)
    assert not bad and not stats["unexplained"]
    # 1 % of the ~200 compared updates per character is two flips; each must be one the oracle reproduces (unexplained above)
    assert stats["flips"] <= max(2, stats["total"] // 100)
    assert all((wm == k).any() for k in range(4)), "a storage mode of solve_rows was entered by no warp"
    assert stats["clamp"] > 0 and stats["deep"] > 0 and stats["skip"] > 0 and stats["overflow"] > 0
    assert stats["sat"] > 0 or ch == "dog3d"   # the dog's limited joints cannot reach the cap (tests/test_solver_states_cpu.py)


def test_partners_do_not_change_an_environments_result(asset_root):
    import torch
    from deepmimic_b200.capi import BatchedCore
    ch = "humanoid3d"
    c = S.CHARS[ch]
    args = ["--enable_char_contact_fall", "false"] + c["args"]   # laid-flat states must not end their episodes
    orc = Oracle(args, asset_root)
    lay = SnapLayout(orc.num_joints)
    lib = S.build(orc, asset_root, ch)
    buckets = {}
    for st in lib:
        rows, _ = S.last_rows(orc, st.snap)
        b = S.bucket(int(rows[-1, S.LIMITS] + 3 * rows[-1, S.POINTS]), ch)
        buckets.setdefault(b, []).append(st)
    assert all(b in buckets for b in range(5)), sorted(buckets)
    light = [buckets[0][0], buckets[1][0], buckets[1][len(buckets[1]) // 2]]
    heavy = [buckets[2][0], buckets[3][0], buckets[4][0]]
    ender = buckets[1][1].snap.copy()
    ender[lay.scal + 13] = ender[lay.scal + 12] + 3.0 * S.DT - 1e-9   # timer max: the episode ends after 3 of the 20 updates
    partners = [b[-1].snap for b in (buckets[k] for k in range(5))] + [ender]
    snaps, where = [], {}
    for si, s in enumerate(light + heavy):
        for p in partners:
            for first in (True, False):
                where.setdefault(si, []).append(len(snaps) + (0 if first else 1))
                snaps += [s.snap, p] if first else [p, s.snap]
    n = 256
    assert len(snaps) <= n
    while len(snaps) < n:
        snaps.append(buckets[0][0].snap)
    results = {}
    for order_on in (False, True):
        core = BatchedCore(args, n, asset_root, device=0, seed=5)
        core.set_env_order(order_on)
        _load(core, snaps)
        core.update(S.DT, 20)
        st = torch.zeros(n, core.dims.state_size, device="cuda"); rw = torch.zeros(n, device="cuda")
        core.observe(st, rw); core.sync()
        st, rw = st.cpu().numpy(), rw.cpu().numpy()
        results[order_on] = [(core.get_snapshot(e), st[e], rw[e]) for e in range(n)]
        core.close()
    checked = 0
    for si, envs in where.items():
        s0, o0, r0 = results[False][envs[0]]
        assert np.isfinite(s0).all()
        for e in envs:
            for order_on in (False, True):
                s, o, r = results[order_on][e]
                name = "%s (%s), env %d, placement by load %s" % ((light + heavy)[si], "light" if si < len(light) else "heavy", e, order_on)
                assert np.array_equal(s, s0), "snapshot of %s depends on its partner" % name
                assert np.array_equal(o, o0), "observation of %s depends on its partner" % name
                assert r == r0, "reward of %s depends on its partner" % name
                checked += 1
    print("partners: %d subjects x %d partners x 2 sides x 2 placements = %d environment results equal" % (len(where), len(partners), checked))
