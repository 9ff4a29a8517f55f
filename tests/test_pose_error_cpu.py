"""The tracking error's float64 restatement (tests/pose_error_ref.py) on known answers, the new kernels' ptxas resources and the argument
handling of run --pose_error; no GPU needed."""
import os
import re

import numpy as np
import pytest

from tests import pose_error_ref as R
from tests.native import nvcc, ptxas_report
from tests.render_ref import Character


@pytest.fixture(scope="module")
def humanoid(asset_root):
    return Character(asset_root, "data/characters/humanoid3d.txt")


def _random_poses(ch, rng, L):
    p = np.zeros((L, ch.pose_dim))
    p[:, 0:3] = rng.normal(size=(L, 3))
    for k in range(ch.n):
        o = 3 if ch.type[k] == "root" else ch.pose_off[k]
        if ch.type[k] in ("root", "spherical"):
            q = rng.normal(size=(L, 4))
            p[:, o:o + 4] = q / np.linalg.norm(q, axis=1, keepdims=True)
        elif ch.type[k] == "revolute":
            p[:, o] = rng.uniform(-2.0, 2.0, L)
    return p


def test_identical_sequences_score_zero(humanoid):
    a = _random_poses(humanoid, np.random.default_rng(0), 7)
    assert R.errors(humanoid, a, a.copy()) == (0.0, 0.0)


def test_hand_worked_three_by_three():
    d = np.array([[1.0, 2.0, 6.0], [0.5, 3.0, 1.0], [4.0, 0.25, 2.0]])
    # D row by row: [2, 4, 10], [2.5, 5.5, 6], [6.5, 3, 5]; D(2, 2) = min(5.5 + 2 * 2, 6 + 2, 3 + 2) = 5
    lock, warped = R.errors_of_distances(d)
    assert lock == 2.0 and warped == 5.0 / 6.0


def test_one_frame_and_symmetry_and_the_bound(humanoid):
    rng = np.random.default_rng(1)
    a, r = _random_poses(humanoid, rng, 1), _random_poses(humanoid, rng, 1)
    lock, warped = R.errors(humanoid, a, r)
    assert lock == pytest.approx(warped, rel=1e-15)
    for L in (2, 5, 13):
        a, r = _random_poses(humanoid, rng, L), _random_poses(humanoid, rng, L)
        ab, ba = R.errors(humanoid, a, r), R.errors(humanoid, r, a)
        assert ab == pytest.approx(ba, rel=1e-13)
        assert ab[1] <= ab[0] + 1e-15 and ab[1] > 0.0


def test_features_ignore_the_root_offset_and_heading(humanoid):
    rng = np.random.default_rng(2)
    for p in _random_poses(humanoid, rng, 6):
        f = R.features(humanoid, p)
        q = p.copy()
        q[0] += 3.7; q[2] -= 1.2
        th = rng.uniform(-np.pi, np.pi)
        yq = np.array([np.cos(0.5 * th), 0.0, np.sin(0.5 * th), 0.0])   # rotation about y, w first
        w1, v1 = yq[0], yq[1:]
        w2, v2 = p[3], p[4:7]
        q[3] = w1 * w2 - v1 @ v2
        q[4:7] = w1 * v2 + w2 * v1 + np.cross(v1, v2)
        np.testing.assert_allclose(R.features(humanoid, q), f, atol=1e-12)


def test_a_lagging_motion_warps_to_near_zero(humanoid):
    """a smooth motion against itself three frames late: the phase-locked error sees the lag, the warped one almost not"""
    L, k = 60, 3
    t = np.arange(L + k) / 30.0
    p = np.zeros((L + k, humanoid.pose_dim))
    p[:, 1] = 0.9; p[:, 3] = 1.0
    for j in range(1, humanoid.n):
        o = humanoid.pose_off[j]
        if humanoid.type[j] == "spherical":
            ang = 0.6 * np.sin(2.0 * t + j)
            p[:, o] = np.cos(0.5 * ang); p[:, o + 3] = np.sin(0.5 * ang)
        elif humanoid.type[j] == "revolute":
            p[:, o] = -0.8 + 0.6 * np.sin(2.0 * t + j)
    lock, warped = R.errors(humanoid, p[k:], p[:L])
    assert lock > 0.02 and warped < 0.1 * lock, (lock, warped)


@pytest.mark.skipif(nvcc() is None, reason="needs nvcc")
def test_pose_error_kernels_spill_nothing(tmp_path):
    rep = ptxas_report(os.path.join("kernels", "dm_pose_error.cu"), str(tmp_path))
    entries = [e for e in rep if re.search(r"dm_pose_(feature|dtw)_kernel", e)]
    assert len(entries) == 3, list(rep)
    for e in entries:
        for name, _, stores, loads in rep[e][1]:
            assert stores == 0 and loads == 0, "%s: %d B spill stores, %d B spill loads" % (name, stores, loads)
    pol = ptxas_report(os.path.join("kernels", "dm_policy.cu"), str(tmp_path))
    kin = [e for e in pol if "dm_kin_pose_kernel" in e]
    assert len(kin) == 2
    for e in kin:
        for name, _, stores, loads in pol[e][1]:
            assert stores == 0 and loads == 0, "%s: %d B spill stores, %d B spill loads" % (name, stores, loads)


def test_run_pose_error_option():
    from deepmimic_b200.run import build_parser
    opts, rest = build_parser().parse_known_args(["--pose_error", "--arg_file", "x.txt"])
    assert opts.pose_error and rest == ["--arg_file", "x.txt"]
    opts, _ = build_parser().parse_known_args([])
    assert opts.pose_error is False
    with pytest.raises(SystemExit):
        build_parser().parse_known_args(["--pose_error=1"])
