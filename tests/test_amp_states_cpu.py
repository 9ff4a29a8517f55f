"""The constructed inputs of tests/amp_states.py reach, in the oracle and on the clip tables, the branches of the AMP observation kernel they
were built for (tests/test_amp_obs_branches_gpu.py compares the kernels with the oracle on them): headings in every quadrant and at +-pi, the
root's x axis near vertical, w < 0, revolute angles past +-pi, the dog's non-identity child rotations, the history's and the expert's
previous sample before 0 (previous cycle or clamped), past the end of a non-looping clip, at exact frame times, in the first and last frame
interval of clip k > 0, distinct ground heights, and the history a reset keeps or re-initialises.  Every decision an input does not target
is at least 10 % of its threshold away from it."""
import json
import math
import os

import numpy as np
import pytest

from tests import amp_states as A
from tests import policy_states as P
from tests.oracle_binding import Oracle


@pytest.fixture(scope="module")
def assets(asset_root, tmp_path_factory):
    return P.make_assets(asset_root, str(tmp_path_factory.mktemp("amp") / "assets"))


def _snap_quats(snap, layout):
    """w of the stored root (world -> base) quaternion and of every spherical joint's"""
    w = [snap[6]] + [snap[13 + 4 * j + 3] for j, (_, t, _) in enumerate(layout) if t == "spherical"]
    return np.array(w)


@pytest.mark.parametrize("ch", ["humanoid3d", "dog3d"])
def test_agent_pairs_reach_their_branches(assets, ch):
    o = Oracle(A.amp_args(ch, False), assets)
    lay = P.joint_layout(assets, ch)
    pairs = A.agent_pairs(o, assets, ch)
    quadrants, at_pi, tilt, neg, wrap = set(), 0, 0, 0, 0
    for p in pairs:
        o.set_snapshot(p.prev)
        o.update_hist()
        o.set_snapshot(p.now)
        ref = o.record_amp_obs_agent()
        c = A.heading_cond(ref)
        h = math.atan2(-ref[6], ref[4])          # local root off: the pose block's tangent is the root's x axis in the world
        if p.kind == "tilt":
            assert c <= A.COND_MIN / 1.1, (p.name, c)
            tilt += 1
        else:
            assert c >= 1.1 * A.COND_MIN, (p.name, c)
        if p.kind == "heading":
            if abs(abs(h) - math.pi) < 1e-6:
                at_pi += 1
            else:
                assert min(abs(h), abs(abs(h) - math.pi / 2), abs(abs(h) - math.pi)) >= 0.1, (p.name, h)   # off the quadrant edges
                quadrants.add((h > 0, abs(h) > math.pi / 2))
        if p.kind == "negated":
            assert (_snap_quats(p.prev, lay) < 0).sum() >= 0.5 * len(_snap_quats(p.prev, lay))
            neg += 1
        if p.kind == "wrapped":
            rev = [13 + 4 * j for j, (_, t, _) in enumerate(lay) if t == "revolute"]
            assert rev and all(abs(p.prev[i]) > 1.1 * math.pi or abs(p.prev[i]) > math.pi + 0.1 for i in rev), p.name
            wrap += 1
    print("%s: %d pairs, quadrants %d, at +-pi %d, tilted %d, w < 0 %d, revolute wrap %d" % (ch, len(pairs), len(quadrants), at_pi, tilt, neg, wrap))
    assert len(quadrants) == 4 and at_pi >= 2 and tilt >= 4 and neg >= 4 and wrap >= 3
    if ch == "dog3d":   # spherical joints with a non-identity child rotation (AttachTheta of the body): neck and the two tail links
        with open(os.path.join(assets, P.CHAR_FILE[ch])) as f:
            bodies = json.load(f)["BodyDefs"]
        rotated = [n for j, (n, t, _) in enumerate(lay) if t == "spherical" and any(bodies[j]["AttachTheta" + a] != 0 for a in "XYZ")]
        assert len(rotated) >= 3, rotated


@pytest.mark.parametrize("motion", [P.WALK, P.WALK_ONCE])
def test_reset_cases_reach_their_branches(assets, motion):
    loop, t, _ = P.read_clip(assets, motion)
    dur = t[-1]
    cases = A.reset_cases(motion, dur)
    before0 = clamped = over = 0
    cycles = set()
    for lb, kt, th in cases:
        tp = kt - A.QDT
        if tp < 0:
            assert kt < A.QDT and (loop and tp < 0 or not loop)
            before0 += loop
            clamped += not loop
        else:
            assert tp >= 0.1 * A.QDT, (lb, tp)
        if not loop:
            if tp >= dur:
                over += 1
                assert tp - dur >= 0.1 * A.QDT, lb
            else:
                assert dur - tp >= 0.1 * A.QDT, lb
        else:
            cycles.add(int(math.floor(kt / dur)))
    thetas = {th for _, _, th in cases}
    print("%s: %d resets, history before 0 in the previous cycle %d, clamped at frame 0 %d, past the end %d, cycles %s" % (
        motion, len(cases), before0, clamped, over, sorted(cycles)))
    assert {0.0, math.pi, -math.pi} <= thetas and len(thetas) >= 5
    if loop:
        assert before0 >= 4 and {0, 1, 5} <= cycles
    else:
        assert clamped >= 4 and over >= 2 and any(lb == "dur-eps" for lb, _, _ in cases) and any(kt == dur for _, kt, _ in cases)


@pytest.mark.parametrize("dataset", list(A.DATASETS))
def test_expert_times_reach_their_branches(assets, dataset):
    args = A.DATASETS[dataset]
    o = Oracle(args, assets)
    dur_t, _, _, loop_t = o.clip_table()
    files = A.dataset_clips(assets, args)
    assert len(files) == len(dur_t)
    counts = dict(before0=0, clamped=0, over=0, exact=0, first_k=0, last_k=0)
    for c, m in enumerate(files):
        loop, ft, _ = P.read_clip(assets, m)
        assert loop == bool(loop_t[c]) and ft[-1] == dur_t[c]     # the clip table's duration is the running sum read_clip restates
        dur = ft[-1]
        for lb, t in A.expert_times(assets, m):
            tp = t - A.QDT
            if tp < 0:
                counts["before0" if loop else "clamped"] += 1
            if not loop and t >= dur:
                counts["over"] += 1
            if lb.startswith("frame"):
                assert t in ft
                counts["exact"] += 1
            if c > 0 and lb == "first interval":
                assert ft[0] < t < ft[1]
                counts["first_k"] += 1
            if c > 0 and lb == "last interval":
                assert ft[-2] < t < ft[-1]
                counts["last_k"] += 1
    print("%s: %d clips (%d looping): %s" % (dataset, len(files), int(loop_t.sum()), counts))
    assert counts["exact"] == 3 * len(files) and counts["first_k"] == counts["last_k"] == len(files) - 1
    assert counts["before0" if loop_t.any() else "clamped"] >= 3
    if not loop_t.all():
        assert counts["clamped"] >= 3 and counts["over"] >= 4
    h = A.origin_heights(64)
    assert len(set(h.tolist())) == 64 and np.diff(h).min() > 1e-2


def test_task_scene_reset_keeps_the_history_and_imitate_amp_reinitialises_it(assets):
    """in the oracle: after an episode that ends, a task scene's first observation carries the last action's pose (the kept history); an
    imitate_amp reset's carries InitHist, the kinematic character one query period before the controller time"""
    o = Oracle(A.TASK_SCENES["heading"], assets)
    b = Oracle(A.TASK_SCENES["heading"], assets)
    o.reset(0.3, 1.2, 20.0, clip=1)
    s_a = P.walking(o, 0.3, 1.2, 5, 17)
    s_a = A.acting(s_a, o.num_joints)
    assert not (o.set_snapshot(P.walking(o, 0.3, 1.2, 5, 17)) or o.need_new_action())   # the flag is what makes the next update UpdateHist
    o.set_snapshot(s_a)
    off, _, _, _ = o.action_statics()
    o.set_action(-off)
    o.update(P.DT)                          # UpdateHist: the history is s_a's pose
    o.reset(0.9, -2.0, 20.0, clip=2)
    o.set_snapshot(o.get_snapshot())        # the state rounded to fp32 as the snapshot holds it, on both sides
    got = o.record_amp_obs_agent()
    b.set_snapshot(s_a); b.update_hist(); b.set_snapshot(o.get_snapshot())
    assert np.array_equal(got, b.record_amp_obs_agent())
    o2 = Oracle(A.amp_args("humanoid3d", True, P.WALK), assets)
    o2.reset(0.6, 0.8, 20.0)
    kept = np.abs(got - o2.record_amp_obs_agent()).max()
    assert kept > 1e-2
    # imitate_amp: InitHist at kin time - 1/30
    for kt in (0.011, 0.6):
        o2.reset(kt, 0.8, 20.0)
        s = o2.get_snapshot()
        o2.set_snapshot(s)
        got = o2.record_amp_obs_agent()
        p, v = o2.kin_frame(kt - A.QDT)
        o2.set_pose_vel(p, v); o2.update_hist(); o2.set_snapshot(s)
        assert np.abs(got - o2.record_amp_obs_agent()).max() < 1e-12, kt
