"""Goal courses on the CPU: the shared host / device course rule of dm_course.cuh through a g++ shim against the numpy restatement
(tests/course_ref.py) -- heading goals before, at, between and after keyframes, waypoint advance and the record; the run options and their
refusals; run_episodes' aggregation of course records; and ptxas's figures for the course kernel and the marked render kernel."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from tests import course_ref as ref
from tests.native import nvcc, ptxas_report, shared_library

HERE = os.path.dirname(os.path.abspath(__file__))
HEADING, TARGET = 2, 1   # dm_task.cuh: kTaskHeading, kTaskTarget
dp = C.POINTER(C.c_double)
fp = C.POINTER(C.c_float)


@pytest.fixture(scope="module")
def shim():
    L = shared_library(os.path.join(HERE, "course_shim.cpp"), ["-O2"])
    L.shim_course_set.argtypes = [C.c_int, dp, C.c_double]
    L.shim_heading_goal.argtypes = [C.c_double, dp]
    L.shim_course_start.argtypes = [C.c_int, C.c_double, C.c_double, C.c_double, fp]
    L.shim_course_step.argtypes = [C.c_int, C.c_double, C.c_double, C.c_double, fp]
    L.shim_course_state.argtypes = [dp, C.POINTER(C.c_int)]
    return L


def _set(shim, rows, succ=0.5):
    r = np.zeros((len(rows), 3))
    r[:, :np.asarray(rows).shape[1]] = rows
    shim.shim_course_set(len(rows), r.ctypes.data_as(dp), succ)


def _call(shim, fn, kind, rx, rz, tau):
    rec = np.zeros(4, dtype=np.float32)
    fn(kind, rx, rz, tau, rec.ctypes.data_as(fp))
    tk, pr = np.zeros(6), np.zeros(2, dtype=np.int32)
    shim.shim_course_state(tk.ctypes.data_as(dp), pr.ctypes.data_as(C.POINTER(C.c_int)))
    return rec, tk, pr


def test_layout(shim):
    from deepmimic_b200.capi import MAX_COURSE_POINTS
    assert shim.shim_course_bytes() == 440 and shim.shim_course_max_points() == MAX_COURSE_POINTS == 16


HEADING_ROWS = [[0.5, 0.0, 1.0], [2.0, 1.5707963267948966, 1.5], [2.5, 6.283185307179586, 0.0], [4.0, -1.0, 2.0]]


@pytest.mark.parametrize("tau", [0.0, 0.25, 0.5, 0.5 + 1e-12, 1.0, 1.9999999, 2.0, 2.1, 2.5, 3.7, 4.0, 4.0 + 1e-9, 50.0,
                                 1.0 / 30.0 * 17, 1.0 / 30.0 * 61])
def test_heading_goal_matches_the_restatement_bit_for_bit(shim, tau):
    """before the first keyframe, at each keyframe, between them and after the last: h and v equal the restatement's bits (no fused
    multiply-add); at a keyframe the row itself"""
    _set(shim, HEADING_ROWS)
    hv = np.zeros(2)
    shim.shim_heading_goal(tau, hv.ctypes.data_as(dp))
    assert tuple(hv) == ref.heading_goal(HEADING_ROWS, tau)
    for t, h, v in HEADING_ROWS:
        if tau == t:
            assert tuple(hv) == (h, v)


def test_heading_goal_of_one_row_and_an_unwrapped_turn(shim):
    _set(shim, [[3.0, 0.7, 1.2]])
    hv = np.zeros(2)
    for tau in (0.0, 3.0, 9.0):
        shim.shim_heading_goal(tau, hv.ctypes.data_as(dp))
        assert tuple(hv) == (0.7, 1.2)
    _set(shim, [[0.0, 0.0, 1.0], [4.0, 2 * math.pi, 1.0]])
    shim.shim_heading_goal(2.0, hv.ctypes.data_as(dp))
    assert hv[0] == math.pi   # half of one full turn, not 0


def test_heading_record_and_goal_over_a_run(shim):
    """start, then steps of 1/30 s with a drifting root: the task block's heading, speed and parked timer, and the record (goal point, along-
    and cross-track speed against the goal in force during the step), against the restatement"""
    _set(shim, HEADING_ROWS)
    c = ref.Course("heading", HEADING_ROWS)
    rng = np.random.default_rng(3)
    rx, rz, tau = 0.3, -1.2, 0.0
    rec, tk, pr = _call(shim, shim.shim_course_start, HEADING, rx, rz, tau)
    want = c.start(rx, rz, tau)
    assert np.allclose(rec, want, rtol=1e-6, atol=1e-6) and rec[2] == 0 and rec[3] == 0 and pr[0] == 0 and pr[1] == 7
    for k in range(150):
        rx, rz, tau = rx + rng.normal(0.04, 0.02), rz + rng.normal(-0.01, 0.02), (k + 1) / 30.0
        in_force = c.goal
        rec, tk, pr = _call(shim, shim.shim_course_step, HEADING, rx, rz, tau)
        want = c.step(rx, rz, tau)
        assert np.allclose(rec, want.astype(np.float32), rtol=1e-6, atol=1e-6), (k, rec, want)
        assert (tk[3], tk[2]) == c.goal and tk[4] == 0.0 and tk[5] == np.inf
        # the goal point: 1.5 m ahead of the root along the heading in force during the step
        h = in_force[0]
        assert abs(rec[0] - (rx + 1.5 * math.cos(h))) < 1e-5 and abs(rec[1] - (rz - 1.5 * math.sin(h))) < 1e-5


def test_heading_record_of_an_interval_of_no_time(shim):
    _set(shim, HEADING_ROWS)
    _call(shim, shim.shim_course_start, HEADING, 1.0, 2.0, 0.7)
    rec, _, _ = _call(shim, shim.shim_course_step, HEADING, 1.5, 2.5, 0.7)
    assert rec[2] == 0 and rec[3] == 0


def test_heading_speeds_of_a_straight_walk():
    """the restatement's definitions on a constructed walk: 1.2 m/s along heading pi/2 (-z) with 0.3 m/s towards heading pi (-x)"""
    c = ref.Course("heading", [[0.0, math.pi / 2, 1.5]])
    c.start(0.0, 0.0, 0.0)
    rec = c.step(-0.3 * 0.5, -1.2 * 0.5, 0.5)
    assert abs(rec[2] - (1.2 - 1.5)) < 1e-12 and abs(rec[3] - 0.3) < 1e-12


TARGET_ROWS = [[2.0, 0.0], [2.3, 0.1], [2.0, 3.0], [-1.0, 3.0]]


def test_target_advance_and_record(shim):
    """waypoints relative to the start root; the advance at the success radius (strict), two waypoints inside one radius in one call, the
    last one kept once reached; the record after the advance"""
    _set(shim, TARGET_ROWS, succ=0.5)
    c = ref.Course("target", TARGET_ROWS, succ_dist=0.5)
    org = (1.0, -1.0)
    rec, tk, pr = _call(shim, shim.shim_course_start, TARGET, org[0], org[1], 0.0)
    assert np.allclose(rec, c.start(org[0], org[1], 0.0)) and (tk[0], tk[1]) == (3.0, -1.0) and tk[5] == np.inf
    path = [(2.0, -1.0, 0, 0), (org[0] + 2.0 - 0.5, -1.0, 0, 0),   # exactly on the radius: not reached
            (org[0] + 2.2, -1.0 + 0.05, 2, 2),                      # inside both the first and the second waypoint's radius
            (org[0] + 2.0, -1.0 + 2.6, 3, 3),                       # third reached: the last is the goal
            (org[0] - 1.0, -1.0 + 3.4, 4, 3),                       # last reached: active stays on it, reached 4
            (5.0, 5.0, 4, 3)]
    for k, (x, z, reached, goal_idx) in enumerate(path):
        rec, tk, pr = _call(shim, shim.shim_course_step, TARGET, x, z, (k + 1) / 30.0)
        want = c.step(x, z, (k + 1) / 30.0)
        assert np.allclose(rec, want.astype(np.float32), rtol=1e-6, atol=1e-6), (k, rec, want)
        wx, wz = org[0] + TARGET_ROWS[goal_idx][0], org[1] + TARGET_ROWS[goal_idx][1]
        assert pr[0] == reached and rec[2] == reached and (tk[0], tk[1]) == (wx, wz), (k, pr, tk)
        assert abs(rec[3] - math.hypot(x - wx, z - wz)) < 1e-5


# ---- run options and aggregation

def test_run_course_options_parse_and_refuse():
    from deepmimic_b200.run import build_parser
    ap = build_parser()
    o = ap.parse_known_args([])[0]
    assert o.heading_course is None and o.target_course is None
    assert ap.parse_known_args(["--heading_course", "0:0:1.5,4:0:1.5,6:1.5708:1.5"])[0].heading_course == [[0, 0, 1.5], [4, 0, 1.5],
                                                                                                         [6, 1.5708, 1.5]]
    assert ap.parse_known_args(["--target_course", "2:0,2:-2.5"])[0].target_course == [[2, 0], [2, -2.5]]
    for bad in ("", "1:2", "0:0:1:4", "a:0:1", "1:0:1,0.5:0:1", "2:0:1,2:0:1", "-1:0:1", "0:0:-1", "0:nan:1", "0:inf:1",
                ",".join(["%d:0:1" % k for k in range(17)])):
        with pytest.raises(SystemExit):
            ap.parse_known_args(["--heading_course", bad])
    for bad in ("", "1", "1:2:3", "x:1", "1:nan", ",".join(["1:%d" % k for k in range(17)])):
        with pytest.raises(SystemExit):
            ap.parse_known_args(["--target_course", bad])
    with pytest.raises(SystemExit):
        ap.parse_known_args(["--heading_course", "0:0:1", "--target_course", "1:1"])


def test_course_markers_follow_the_records():
    from deepmimic_b200.run import MARKER_HEIGHT, MARKER_RADIUS, course_markers
    rec = np.arange(20, dtype=np.float32).reshape(5, 4)
    m = course_markers(rec, 3)
    assert m.shape == (4, 4)
    assert np.array_equal(m[:, 0], rec[[0, 0, 1, 2], 0]) and np.array_equal(m[:, 2], rec[[0, 0, 1, 2], 1])
    assert np.all(m[:, 1] == np.float32(MARKER_HEIGHT)) and np.all(m[:, 3] == np.float32(MARKER_RADIUS))


def test_run_episodes_aggregates_the_first_episode():
    """a synthetic record of 3 environments over 6 steps: the means over each first episode only, the waypoints at its last step and the
    time of the step that reached the last waypoint"""
    import torch
    from deepmimic_b200.rollout import course_stats
    T, N = 6, 3
    dones = torch.zeros(T, N, dtype=torch.bool)
    dones[2, 0] = True    # env 0: steps 0..2
    dones[5, 1] = True    # env 1: steps 0..5
    dones[0, 2] = True    # env 2: step 0 only
    rec = torch.zeros(T, N, 4)
    rec[..., 2] = torch.tensor([[0.1, -0.2, 5.0], [-0.3, 0.2, 9.0], [0.2, 0.2, 9.0], [7.0, 0.2, 9.0], [7.0, -0.2, 9.0], [7.0, 0.2, 9.0]])
    rec[..., 3] = -2 * rec[..., 2]
    h = course_stats("heading", rec, dones, [3, 3, 3], 1 / 30)
    assert torch.allclose(h["speed_err"], torch.tensor([0.2, 0.2, 5.0])) and torch.allclose(h["cross_speed"], torch.tensor([0.4, 0.4, 10.0]))
    rec[..., 2] = torch.tensor([[0, 0, 1], [1, 0, 1], [2, 1, 1], [3, 1, 1], [3, 2, 1], [3, 2, 1]], dtype=torch.float32)
    t = course_stats("target", rec, dones, [2, 2, 2], 1 / 30)
    assert t["waypoints"].tolist() == [2.0, 2.0, 1.0]
    ct = t["course_time"]
    assert abs(ct[0].item() - 3 / 30) < 1e-6 and abs(ct[1].item() - 5 / 30) < 1e-6 and math.isnan(ct[2].item())


def test_marker_restatement_without_a_marker_is_the_renderer_restatement(asset_root):
    """render_marker_ref with radius <= 0 is render_ref.render exactly; with a marker in front of the camera its pixels carry id -3"""
    from tests import render_marker_ref as MR
    from tests import render_ref as RR
    from deepmimic_b200.formats import read_motion
    ch = RR.Character(asset_root, "data/characters/humanoid3d.txt")
    pose = read_motion(os.path.join(asset_root, "data/motions/humanoid3d_walk.txt"))["frames"][0]
    R, c = ch.frames(pose)
    cam = dict(yaw=0.6, pitch=0.25, distance=4.0, target_height=0.9, fov_y=0.78)
    a, b = RR.render(ch, R, c, (pose[0], pose[2]), cam, 48, 32), MR.render_marked(ch, R, c, (pose[0], pose[2]), cam, 48, 32, (0, 0, 0, 0.0))
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    m = MR.render_marked(ch, R, c, (pose[0], pose[2]), cam, 48, 32, (pose[0], 0.9, pose[2], 2.0))   # a sphere around the whole character
    assert (m["ids"] == MR.MARKER).sum() > 100 and not (m["ids"] >= 0).any()


# ---- resources

@pytest.mark.skipif(nvcc() is None, reason="needs nvcc")
def test_course_and_marked_render_kernels_do_not_spill(tmp_path):
    """ptxas: no spills in the course kernel (its stack frame is the double-precision sine / cosine's argument reduction), none and no stack
    in the marked render kernel"""
    rep = ptxas_report(os.path.join("kernels", "dm_course.cu"), str(tmp_path))
    (entry,) = [e for e in rep if "dm_course_kernel" in e]
    for name, stack, stores, loads in rep[entry][1]:
        assert stores == 0 and loads == 0, (name, stack, stores, loads)
    rep = ptxas_report(os.path.join("kernels", "dm_render.cu"), str(tmp_path))
    (entry,) = [e for e in rep if "dm_render_marked_kernel" in e]
    for name, stack, stores, loads in rep[entry][1]:
        assert stack == 0 and stores == 0 and loads == 0, (name, stack, stores, loads)
