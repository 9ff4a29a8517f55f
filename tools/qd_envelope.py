#!/usr/bin/env python
"""Sensitivity envelope of the ORACLE's own Update(1/600): how far does its post-update q / qd move when the pre-update state is
perturbed by fp32 rounding noise (relative 2^-24 ~ 6e-8 per component, i.e. what storing the state in fp32 -- as Bullet does -- already
costs)?  The CUDA path evaluates the same formulas in fp32 in a different (equally valid) order, so its distance from the oracle cannot be
expected to be smaller than this envelope.  CPU only.  Prints percentiles per contact class; tests/test_qd_envelope_gpu.py uses the same
protocol next to the GPU-vs-oracle comparison.
  python tools/qd_envelope.py [arg_file] [replicas]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests.oracle_binding import Oracle   # noqa: E402
from tests.parity_util import SnapLayout, compare_sim_state, joint_types_from_assets, random_policy_action   # noqa: E402

ULP = 2.0 ** -24


def perturb(lay, snap, rng, rel=ULP):
    """fp32-rounding-sized relative noise on the dynamic state (base position / rotation / velocities, joint positions / velocities)"""
    p = snap.copy()
    n = lay.mani            # everything before the manifold block: base 13 + joint pos 4 nl + joint vel 3 nl
    p[:n] *= 1.0 + rel * rng.uniform(-1.0, 1.0, n)
    q = p[lay.base_quat]; p[lay.base_quat] = q / np.linalg.norm(q)
    for j in range(lay.nl):
        jp = p[lay.jpos + 4 * j: lay.jpos + 4 * j + 4]
        nn = np.linalg.norm(jp)
        if abs(nn - 1.0) < 1e-3:
            p[lay.jpos + 4 * j: lay.jpos + 4 * j + 4] = jp / nn
    return p


def impulse_err(lay, a, b):
    """max |difference| of the cached points' impulses (normal, lateral 1, lateral 2) over the manifold slots both snapshots hold"""
    worst = 0.0
    for j in range(lay.nl):
        for c in range(4):
            ma, mb = lay.manifold(a, j, c), lay.manifold(b, j, c)
            if ma[0] != 0 and mb[0] != 0:
                worst = max(worst, float(np.abs(ma[7:10] - mb[7:10]).max()))
    return worst


def envelope(orc, orc2, lay, jt, before, after, rng, replicas, impulses=False):
    """worst |dq|, |dqd| (and, with impulses, worst cached-point impulse difference) of the replicas that keep the contact counts of
    `after`, and the number of replicas that changed them"""
    worst_q = worst_qd = worst_imp = 0.0
    flips = 0
    for _ in range(replicas):
        orc2.set_snapshot(perturb(lay, before, rng))
        orc2.update(1.0 / 600.0)
        s2 = orc2.get_snapshot()
        if lay.contact_counts(s2) != lay.contact_counts(after):
            flips += 1
            continue
        eq, eqd = compare_sim_state(lay, after, s2, jt)
        worst_q, worst_qd = max(worst_q, eq), max(worst_qd, eqd)
        worst_imp = max(worst_imp, impulse_err(lay, after, s2))
    if impulses:
        return worst_q, worst_qd, flips, worst_imp
    return worst_q, worst_qd, flips


def main():
    from deepmimic_b200.assets import asset_root
    root = asset_root(prefer_archive=True)
    arg_file = sys.argv[1] if len(sys.argv) > 1 else "args/run_humanoid3d_spinkick_args.txt"
    replicas = int(sys.argv[2]) if len(sys.argv) > 2 else 4
    char = "data/characters/dog3d.txt" if "dog" in arg_file else "data/characters/humanoid3d.txt"
    orc, orc2 = Oracle(["--arg_file", arg_file], root), Oracle(["--arg_file", arg_file], root)
    lay = SnapLayout(orc.num_joints); jt = joint_types_from_assets(root, char)
    off, scl, lo, hi = orc.action_statics()
    rng = np.random.default_rng(1234); rng2 = np.random.default_rng(7)
    rows = []
    for t0 in (0.0, 0.3, 0.6, 0.9):
        orc.reset(t0 * orc.motion_duration / 1.283282, 0.0, 20.0)
        for upd in range(200):
            if orc.need_new_action():
                orc.set_action(random_policy_action(rng, off, scl, lo, hi))
            if orc.is_episode_end():
                break
            before = orc.get_snapshot()
            orc.update(1.0 / 600.0)
            after = orc.get_snapshot()
            eq, eqd, fl = envelope(orc, orc2, lay, jt, before, after, rng2, replicas)
            rows.append((sum(lay.contact_counts(after)), eq, eqd, fl))
    rows = np.array(rows)
    for name, m in (("contact-free", rows[:, 0] == 0), ("with contacts", rows[:, 0] > 0)):
        r = rows[m]
        if len(r) == 0:
            continue
        print("%s %-13s %4d updates: envelope |dq| median %.2e p99 %.2e max %.2e ; |dqd| median %.2e p90 %.2e p99 %.2e max %.2e ; branch flips in %d replicas"
              % (os.path.basename(arg_file), name, len(r), np.median(r[:, 1]), np.percentile(r[:, 1], 99), r[:, 1].max(), np.median(r[:, 2]), np.percentile(r[:, 2], 90),
                 np.percentile(r[:, 2], 99), r[:, 2].max(), int(r[:, 3].sum())))


if __name__ == "__main__":
    main()
