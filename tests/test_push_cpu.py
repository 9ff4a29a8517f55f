"""Pushes on the CPU: the oracle's timed external force (known answers from the total linear momentum) and the push-robustness options of
`python -m deepmimic_b200.run`.  CPU only."""
import numpy as np
import pytest

from tests.push_oracle import PushOracle

SPINKICK = ["--arg_file", "args/run_humanoid3d_spinkick_args.txt"]
# The semi-implicit Bullet step conserves the linear momentum only up to terms of second order in the step (the second sub-step's velocities
# are mapped to momentum at the configuration the first one moved to): 1e-3 of F dt at the reference's 1/600 s, 1e-5 at 1/6000 s and 4e-6
# at 1/60000 s with these pushes.  The known answers use the short update.
DT = 1.0 / 60000.0
# root, chest (spherical), right knee (revolute), right wrist (a fixed leaf)
BODIES = (0, 1, 4, 8)


def _airborne(o, kin_time=0.3):
    """reset, then lift the character 2 m clear of the ground and stop it: no contact, Stable-PD torques only"""
    o.reset(kin_time, 0.0, 20.0)
    p, _ = o.get_pose()
    p = p.copy()
    p[1] += 2.0
    o.set_pose_vel(p, np.zeros_like(p))


def _momentum(o, masses):
    _, _, lv, _ = o.body_state()
    return (masses[:, None] * lv).sum(axis=0)


@pytest.fixture(scope="module")
def spinkick(asset_root):
    o = PushOracle(SPINKICK, asset_root)
    return o, o.link_table()[:, 0].copy()


@pytest.mark.parametrize("body", BODIES)
def test_push_adds_f_dt_to_the_linear_momentum(spinkick, body):
    o, m = spinkick
    F = np.array([310.0, -120.0, 455.0])
    snap = None
    p_free = p_push = None
    for push in (False, True):
        _airborne(o)
        if snap is None:
            snap = o.get_snapshot()
        else:
            o.set_snapshot(snap)
        if push:
            o.set_push(body, F, 0.0, 0.5)
        o.update(DT)
        if push:
            p_push = _momentum(o, m)
        else:
            p_free = _momentum(o, m)
    dp = p_push - p_free
    assert np.abs(dp - F * DT).max() <= 1e-4 * np.abs(F * DT).max(), (body, dp, F * DT)


def test_push_window_counts_whole_updates(spinkick):
    o, m = spinkick
    F = np.array([0.0, 250.0, -400.0])
    start, dur = 3.5 * DT, 4.2 * DT          # off the update boundaries: t = 4, 5, 6, 7 DT lie in [3.5, 7.7) DT
    n_upd = 10
    runs = []
    for push in (False, True):
        _airborne(o)
        if push:
            o.set_push(0, F, start, dur)
        for _ in range(n_upd):
            o.update(DT)
        runs.append(_momentum(o, m))
    t = np.arange(n_upd) * DT
    inside = int(np.sum((start <= t) & (t < start + dur)))
    assert inside == 4
    dp = runs[1] - runs[0]
    assert np.abs(dp - F * DT * inside).max() <= 2e-4 * np.abs(F * DT * inside).max(), (dp, F * DT * inside)


def test_reset_clears_the_push(spinkick):
    o, m = spinkick
    _airborne(o)
    o.set_push(1, [500.0, 0.0, 0.0], 0.0, 10.0)
    assert o.push_body() == 1
    o.reset(0.3, 0.0, 20.0)
    assert o.push_body() == -1
    runs = []
    for push in (False, True):
        _airborne(o)
        if push:
            o.set_push(1, [500.0, 0.0, 0.0], 0.0, 10.0)
            o.reset(0.3, 0.0, 20.0)
            p, _ = o.get_pose()
            p = p.copy(); p[1] += 2.0
            o.set_pose_vel(p, np.zeros_like(p))
        o.update(DT)
        runs.append(_momentum(o, m))
    assert np.array_equal(runs[0], runs[1])


# ---- python -m deepmimic_b200.run --push_forces


def test_run_push_options_parse_and_refuse(capsys):
    from deepmimic_b200.run import build_parser, main
    o, rest = build_parser().parse_known_args(["--push_forces", "0,250.5,1000", "--push_body", "1", "--arg_file", "x.txt"])
    assert o.push_forces == [0.0, 250.5, 1000.0] and o.push_body == 1 and o.push_time == 2.0 and o.push_duration == 0.2
    assert rest == ["--arg_file", "x.txt"]
    o, _ = build_parser().parse_known_args([])
    assert o.push_forces is None
    for bad in ("-5", "100,-1", "a,b", "inf", "nan"):
        with pytest.raises(SystemExit):
            build_parser().parse_known_args(["--push_forces", bad])
        err = capsys.readouterr().err
        assert "push forces must be" in err or "comma-separated" in err, err
    with pytest.raises(SystemExit, match="push_duration"):
        main(["--push_forces", "100", "--push_duration", "-1", "--arg_file", "args/run_humanoid3d_spinkick_args.txt"])


def test_run_push_forces_without_a_model_are_refused(asset_root):
    from deepmimic_b200.run import main
    with pytest.raises(SystemExit, match="no --model_files"):
        main(["--asset_root", asset_root, "--push_forces", "100,200", "--arg_file", "args/train_humanoid3d_spinkick_args.txt"])


def test_run_push_plan_deals_environments_over_forces():
    from deepmimic_b200.run import push_plan
    forces = [0.0, 100.0, 400.0]
    mag, ang, force = push_plan(forces, 10, seed=7)
    assert list(mag) == [forces[e % 3] for e in range(10)]
    assert force.dtype == np.float32 and force.shape == (10, 3) and (force[:, 1] == 0).all()
    assert np.allclose(np.hypot(force[:, 0], force[:, 2]), mag, rtol=1e-6)
    assert ((ang >= 0) & (ang < 2 * np.pi)).all()
    mag2, ang2, force2 = push_plan(forces, 10, seed=7)
    assert np.array_equal(ang, ang2) and np.array_equal(force, force2)
    assert not np.array_equal(ang, push_plan(forces, 10, seed=8)[1])
