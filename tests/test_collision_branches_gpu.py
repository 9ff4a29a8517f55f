"""The step kernel's collision pass (dm_step.cu: collide) against the CPU oracle on constructed states (tests/contact_states.py) that
drive each of its branches on purpose: the support vertex of every box corner, capsule end and sphere, a new point added to a cache of
0-3 points, the nearest cached point replaced, sortCachedPoints' 16 (deepest, replaced) combinations on a box, a capsule and a sphere,
the refresh's removals by distance and by lateral drift in every subset of a full cache, the contact-fall tolerance, and the point
count a link carries from one sub-step to the next within a launch.

  1. every state, one teacher-forced Update(1/600) per environment: the manifolds slot by slot -- valid flags and point counts equal,
     lifetimes equal exactly (they say which cached point went to which slot), local point A, anchor B (x, z) and distance within
     max(1e-5, 8 x that field's envelope over 16 fp32-rounding replicas of the oracle) in scaled units; impulses, q and q-dot under
     tests/test_solver_branches_gpu.py's protocol.  Only valid slots are compared: after a removal the kernel leaves stale floats behind
     a cleared flag where the oracle's snapshot has zeros.  No branch flip is allowed: the states are built with margins (the CPU test
     checks them), so a flip is a finding.  The episode-end, terminate and valid flags and the imitation reward (0 for a fallen
     character) equal the oracle's.
  2. the release / re-contact states, one 40-update launch against 40 single-update launches: bit-identical snapshots, manifolds
     included, and the test link's point count and lifetimes equal to the oracle's after the 40 updates."""
import numpy as np
import pytest

from tests import contact_states as CS
from tests.oracle_binding import Oracle
from tests.parity_util import SnapLayout, compare_sim_state, joint_types_from_assets
from tools.qd_envelope import impulse_err, perturb

pytestmark = pytest.mark.gpu

ENVS = {"humanoid3d": 256, "dog3d": 192}   # every state at least once, several blocks (humanoid 32, dog 16 environments per block)
FIELDS = (("A", [1, 2, 3]), ("B", [4, 6]), ("distance", [10]))


def _valid(lay, s):
    return np.array([[lay.manifold(s, j, c)[0] != 0 for c in range(4)] for j in range(lay.nl)])


def _field_err(lay, a, b, cols):
    """max |difference| of manifold columns cols over the slots valid in both snapshots"""
    worst = 0.0
    for j in range(lay.nl):
        for c in range(4):
            ma, mb = lay.manifold(a, j, c), lay.manifold(b, j, c)
            if ma[0] != 0 and mb[0] != 0:
                worst = max(worst, float(np.abs(ma[cols] - mb[cols]).max()))
    return worst


def _oracle_side(orc, orc2, lay, jt, st, rng):
    """the oracle's result of one update from st, its flags and reward, and its envelope over 16 replicas"""
    taps, after = CS.contacts(orc, st.snap)
    r = dict(after=after, taps=taps, end=orc.is_episode_end(), term=orc.check_terminate() != 0, valid=orc.check_valid_episode(),
             reward=orc.calc_reward())
    env = dict(q=0.0, qd=0.0, imp=0.0, **{f: 0.0 for f, _ in FIELDS})
    for _ in range(16):
        orc2.set_snapshot(perturb(lay, st.snap, rng))
        orc2.update(CS.DT)
        s2 = orc2.get_snapshot()
        assert np.array_equal(_valid(lay, s2), _valid(lay, after)), "%s: the oracle's own manifold moves under rounding noise" % st
        eq, eqd = compare_sim_state(lay, after, s2, jt)
        env["q"], env["qd"] = max(env["q"], eq), max(env["qd"], eqd)
        env["imp"] = max(env["imp"], impulse_err(lay, after, s2))
        for f, cols in FIELDS:
            env[f] = max(env[f], _field_err(lay, after, s2, cols))
    r["env"] = env
    return r


@pytest.mark.parametrize("ch", list(CS.CHARS))
def test_collision_branches_match_the_oracle(asset_root, ch):
    import torch
    from deepmimic_b200.capi import BatchedCore
    c = CS.CHARS[ch]
    n = ENVS[ch]
    orc, orc2 = Oracle(c["args"], asset_root), Oracle(c["args"], asset_root)
    lay = SnapLayout(orc.num_joints); jt = joint_types_from_assets(asset_root, c["char"])
    lib = [st for st in CS.build(orc, asset_root, ch) if st.cls != "release"]
    assert len(lib) <= n
    floor = 6e-3 if ch == "dog3d" else 1e-3
    rng = np.random.default_rng(9)
    ref = [_oracle_side(orc, orc2, lay, jt, st, rng) for st in lib]
    core = BatchedCore(c["args"], n, asset_root, device=0, seed=3)
    core.set_env_order(False)
    idx = [e % len(lib) for e in range(n)]
    for e, i in enumerate(idx):
        core.set_snapshot(e, lib[i].snap)
    core.update(CS.DT, 1)
    fl = torch.zeros(n, 4, dtype=torch.int32, device="cuda"); core.flags(fl)
    obs = torch.zeros(n, core.dims.state_size, device="cuda"); rw = torch.zeros(n, device="cuda")
    core.observe(obs, rw); core.sync()
    fl, rw = fl.cpu().numpy(), rw.cpu().numpy()
    bad = []
    worst = dict(q=0.0, qd=0.0, imp=0.0, **{f: 0.0 for f, _ in FIELDS})   # measured maxima
    ratio = dict(qd=0.0, imp=0.0, **{f: 0.0 for f, _ in FIELDS})          # measured / bound
    fallen = 0
    for e, i in enumerate(idx):
        st, r = lib[i], ref[i]
        so, sg = r["after"], core.get_snapshot(e)
        vo, vg = _valid(lay, so), _valid(lay, sg)
        if not np.array_equal(vo, vg):
            bad.append("%s env %d: valid slots %s, oracle %s" % (st, e, vg.sum(1).tolist(), vo.sum(1).tolist()))
            continue
        life_o = np.array([lay.manifold(so, j, k)[11] for j in range(lay.nl) for k in range(4)]).reshape(lay.nl, 4)
        life_g = np.array([lay.manifold(sg, j, k)[11] for j in range(lay.nl) for k in range(4)]).reshape(lay.nl, 4)
        if not np.array_equal(life_o[vo], life_g[vg]):
            bad.append("%s env %d: lifetimes %s, oracle %s" % (st, e, life_g[vg].tolist(), life_o[vo].tolist()))
        env = r["env"]
        for f, cols in FIELDS:
            err = _field_err(lay, so, sg, cols)
            bound = max(1e-5, 8.0 * env[f])
            worst[f] = max(worst[f], err); ratio[f] = max(ratio[f], err / bound)
            if err > bound:
                bad.append("%s env %d: %s off by %.2e (bound %.2e)" % (st, e, f, err, bound))
        eq, eqd = compare_sim_state(lay, so, sg, jt)
        ei = impulse_err(lay, so, sg)
        imp_bound = max(8.0 * env["imp"], 1e-3 * (1.0 + max(abs(so[lay.mani + 12 * k + 7]) for k in range(4 * lay.nl))))
        qd_bound = max(floor, 8.0 * env["qd"])
        worst["q"], worst["qd"], worst["imp"] = max(worst["q"], eq), max(worst["qd"], eqd), max(worst["imp"], ei)
        ratio["qd"], ratio["imp"] = max(ratio["qd"], eqd / qd_bound), max(ratio["imp"], ei / imp_bound)
        if eq > 1e-3 or eqd > qd_bound or ei > imp_bound:
            bad.append("%s env %d: |dq| %.2e |dqd| %.2e (bound %.2e) impulses %.2e (bound %.2e)" % (st, e, eq, eqd, qd_bound, ei, imp_bound))
        flags, oflags = (int(fl[e, 1]), int(fl[e, 2]), int(fl[e, 3])), (int(r["end"]), int(r["term"]), int(r["valid"]))
        if flags != oflags:
            bad.append("%s env %d: episode end / terminate / valid %s, oracle %s" % (st, e, flags, oflags))
        if (rw[e] == 0.0) != (r["reward"] == 0.0):
            bad.append("%s env %d: reward %.6g, oracle %.6g" % (st, e, rw[e], r["reward"]))
        fallen += int(r["reward"] == 0.0 and r["term"])
    print("%s: %d environments (%d states), %d fallen; measured maxima: |dq| %.2e |dqd| %.2e impulses %.2e A %.2e B %.2e distance %.2e" % (
        ch, n, len(lib), fallen, worst["q"], worst["qd"], worst["imp"], worst["A"], worst["B"], worst["distance"]))
    print("  largest measured / bound: |dqd| %.3f impulses %.3f A %.3f B %.3f distance %.3f" % (
        ratio["qd"], ratio["imp"], ratio["A"], ratio["B"], ratio["distance"]))
    for b in bad[:40]:
        print("  MISMATCH " + b)
    assert not bad, "%d mismatches" % len(bad)
    fall = [i for i, st in enumerate(lib) if st.cls == "fall"]
    assert any(ref[i]["term"] for i in fall) and not all(ref[i]["term"] for i in fall)


@pytest.mark.parametrize("ch", list(CS.CHARS))
def test_fused_and_single_launches_agree_through_release_and_recontact(asset_root, ch):
    from deepmimic_b200.capi import BatchedCore
    c = CS.CHARS[ch]
    args = ["--enable_char_contact_fall", "false"] + c["args"]   # a dog's head touching down must not end the episode mid-sequence
    orc = Oracle(args, asset_root)
    lay = SnapLayout(orc.num_joints)
    lib = CS.build(orc, asset_root, ch)
    rel = [st for st in lib if st.cls == "release"]
    snaps = [st.snap for st in rel] + [st.snap for st in lib if st.cls in ("refresh", "removal")]
    n = 64
    snaps = [snaps[e % len(snaps)] for e in range(n)]
    out = []
    for fused in (True, False):
        core = BatchedCore(args, n, asset_root, device=0, seed=3)
        core.set_env_order(False)
        for e, s in enumerate(snaps):
            core.set_snapshot(e, s)
        if fused:
            core.update(CS.DT, CS.RELEASE_UPDATES)
        else:
            for _ in range(CS.RELEASE_UPDATES):
                core.update(CS.DT, 1)
        core.sync()
        out.append([core.get_snapshot(e) for e in range(n)])
        core.close()
    diff = [e for e in range(n) if not np.array_equal(out[0][e], out[1][e])]
    assert not diff, "environments %s differ between one 40-update launch and 40 single launches" % diff
    for k, st in enumerate(rel):
        orc.set_snapshot(st.snap)
        seq = []
        for _ in range(CS.RELEASE_UPDATES):
            orc.update(CS.DT)
            seq += [int(t[st.link, CS.EVENT]) for t in orc.last_contacts()]
        so, sg = orc.get_snapshot(), out[0][k]
        j = st.link
        mo = np.array([lay.manifold(so, j, c) for c in range(4)]); mg = np.array([lay.manifold(sg, j, c) for c in range(4)])
        first = seq.index(CS.ADD)
        print("%s %s: removed in sub-step 1, re-added in sub-step %d of %d; points after %d (oracle %d), lifetimes %s (oracle %s)" % (
            ch, st, first + 1, len(seq), int((mg[:, 0] != 0).sum()), int((mo[:, 0] != 0).sum()), mg[mg[:, 0] != 0, 11].tolist(), mo[mo[:, 0] != 0, 11].tolist()))
        assert 10 <= first <= len(seq) - 20
        assert np.array_equal(mo[:, 0] != 0, mg[:, 0] != 0) and np.array_equal(mo[mo[:, 0] != 0, 11], mg[mg[:, 0] != 0, 11])
