"""The constructed inputs of tests/task_states.py take, in the oracle, the branches of the target_amp / heading_amp logic they were built for
(tests/test_task_branches_gpu.py compares the device with the oracle on them), with every decision at least 10 % of its threshold away from
it, and together they reach every branch: the reward regimes, the goal's quadrants and fallback, the distance failure and the redraw that
prevents it, the heading scene's turns, speed changes, clamp and fixed speed, and timers expiring on a chosen update of a launch."""
import math

import numpy as np
import pytest

from tests import amp_states as A
from tests import task_states as S
from tests.oracle_binding import Oracle

SEED, ENV = 12345, 2 ** 31 + 77
PI = math.pi

TARGET_BRANCHES = {"slow", "fast", "away", "success", "td0", "goal_fallback", "fallen", "fail", "expire_no_fail", "min_vel_on", "min_vel_off",
                   "quadrant", "at_pi", "tilt"}
HEADING_BRANCHES = {"slow", "fast", "away", "fallen", "wound", "sharp", "normal", "speed_change", "speed_clamp", "speed_fixed", "min_vel_on",
                    "min_vel_off", "expire"}


def far(x, thr, what, rel=0.1, scale=None):
    """x is at least rel * (scale or |thr|) away from thr"""
    assert abs(x - thr) >= rel * (abs(thr) if scale is None else scale), (what, x, thr)


def evaluate(o, st, p):
    """one update of the prepared oracle; returns the branches it took (asserting the margins)"""
    ts0, c0 = o.task_state(), o.task_counter()
    o.update(S.DT)
    s = o.get_snapshot()
    ts = o.task_state()
    root = S.root_xz(o)
    com = o.calc_com()
    sd = s[S.CLK + 8] - s[S.CLK + 10]
    assert sd == pytest.approx(S.STEP_UPDATES * S.DT, abs=1e-12)
    fallen = o.has_fallen()
    br = set()
    tar = ts["target_pos"][[0, 2]]
    terms = {}
    want = S.ref_reward(st.scene, p, tar, ts["target_speed"], ts["target_heading"], root, com, ts["prev_action_com"], sd, fallen, terms)
    got = o.calc_reward()
    assert got == pytest.approx(want, abs=1e-7), (st, got, want)   # the restatement reads the root and COM rounded to the snapshot
    if st.kind == "lying":
        assert fallen
    else:
        assert not fallen and sum(S.LAY.contact_counts(s)) == 0, st
    expired = o.task_counter() != c0
    assert expired == bool(st.expire), st
    t0 = ts0["timer"] + S.DT
    if expired:
        br.add("expire")
        far(t0, ts0["timer_max"], "timer", scale=S.DT)
    else:
        far(t0, ts0["timer_max"], "timer")
    br.add(terms.get("branch"))
    speed = ts["target_speed"]
    if "avg" in terms and not fallen:
        if terms.get("td", 1.0) > 1e-4:
            far(terms["avg"], 0.0, "avg vs 0", scale=speed)
        else:
            assert terms["avg"] == 0.0                           # unit vector 0: exactly 0 on both sides
        if terms["avg"] > 0:
            far(terms["avg"], speed, "avg vs speed")
            if terms["avg"] > speed:
                br.add("min_vel_on" if p["enable_min_tar_vel"] else "min_vel_off")
            elif not p["enable_min_tar_vel"]:
                br.add("min_vel_off")
    g = o.record_goal()
    rh = S.heading_of_snapshot(s)
    cond = math.hypot(1.0 - 2.0 * (s[4] ** 2 + s[5] ** 2), 2.0 * (s[3] * s[5] + s[6] * s[4]))   # |x_xz| of the root's x axis
    if st.tilt is not None:
        assert cond <= A.COND_MIN / 1.1, cond
        br.add("tilt")
    else:
        assert cond >= 1.1 * A.COND_MIN, cond
        np.testing.assert_allclose(g, S.ref_goal(st.scene, tar, speed, ts["target_heading"], root, rh), atol=1e-6)   # the oracle keeps its state in double
    if st.scene == "target":
        d = math.hypot(*(tar - root))
        if d <= 1e-4:
            assert d <= 1e-4 / 1.1 and g[0] == 1.0 and g[1] == 0.0
            br.add("goal_fallback")
        else:
            far(d, 1e-4, "goal distance")
        dsq = d * d
        fail = dsq > p["tar_fail_dist"] ** 2
        assert (o.check_terminate() == 1) == (fail or fallen)
        if fail:
            br.add("fail")
        far(dsq, p["tar_fail_dist"] ** 2, "fail distance")
        if p["target_succ_dist"] > 0:
            far(dsq, p["target_succ_dist"] ** 2, "success distance")
        if "td" in terms:
            far(terms["td"], 1e-4, "td")
        if expired:
            d0 = S.root_xz(o)
            assert math.hypot(*(ts0["target_pos"][[0, 2]] - d0)) > p["tar_fail_dist"] and not fail
            br.add("expire_no_fail")
        if st.name.startswith("heading"):
            if abs(abs(rh) - PI) < 1e-2:                        # at the cut of atan2 (the update turns the root by ~1e-3 rad)
                br.add("at_pi")
            else:
                assert min(abs(rh), abs(abs(rh) - PI / 2), abs(abs(rh) - PI)) >= 0.1, rh
                br.add("quadrant")
    else:
        assert o.check_terminate() == int(fallen)
        if abs(ts["target_heading"]) > 10 * PI:
            br.add("wound")
        if expired:
            k, h, sp, hb = S.heading_redraw(o, p, (SEED, ENV), c0, ts0["target_heading"], ts0["target_speed"])
            if "speed_clamp" in hb:   # the draw lies in (max, min]: the clamp returns max
                assert sp == p["tar_speed_max"] < p["tar_speed_min"]
            assert o.task_counter() == k and ts["target_heading"] == h and ts["target_speed"] == sp, (st, o.task_counter(), k)
            br |= hb
    return br


@pytest.mark.parametrize("scene", ["target", "heading"])
def test_states_reach_their_branches(asset_root, scene):
    states = S.target_states() if scene == "target" else S.heading_states()
    seen = set()
    for k, st in enumerate(states):
        o = Oracle(st.args, asset_root)
        o.set_task_stream(SEED, ENV, 5)
        p = S.scene_params(asset_root, st.args)
        st.prepare(o, p, (SEED, ENV), k)
        br = evaluate(o, st, p)
        assert st.branches <= br, (st, st.branches, br)
        seen |= br
        print("%-32s %s" % (st, sorted(br)))
    want = TARGET_BRANCHES if scene == "target" else HEADING_BRANCHES
    assert want <= seen, want - seen


@pytest.mark.parametrize("launch", S.launches(), ids=repr)
def test_launches_expire_on_their_updates(asset_root, launch):
    """in a 20-update launch the target timer expires on the chosen updates (an exact timer_max with equality); the previous-action COM is
    taken on the first update and the step duration after it is (n - 1) / 600"""
    o = Oracle(launch.args, asset_root)
    o.set_task_stream(SEED, ENV, 0)
    launch.prepare(o)
    com0 = o.calc_com()
    want = [launch.first]
    if launch.period is not None:
        while want[-1] + launch.period <= launch.updates:
            want.append(want[-1] + launch.period)
    got = []
    for u in range(1, launch.updates + 1):
        c = o.task_counter(); ts = o.task_state()
        o.update(S.DT)
        if u == 1:
            np.testing.assert_allclose(o.task_state()["prev_action_com"], com0, atol=1e-12)
        if o.task_counter() != c:
            got.append(u)
            if launch.exact and u == launch.first:
                assert ts["timer"] + S.DT == ts["timer_max"]
        else:
            assert ts["timer"] + S.DT < o.task_state()["timer_max"]
    s = o.get_snapshot()
    steps = launch.updates // 20
    assert o.task_state()["prev_action_com"][0] != com0[0] or steps == 1
    assert s[S.CLK + 8] - s[S.CLK + 10] == pytest.approx(19 * S.DT, abs=1e-12)
    assert got == want and sum(S.LAY.contact_counts(s)) == 0, (got, want)
    print("%s: expiries on updates %s" % (launch, got))
