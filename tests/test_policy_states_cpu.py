"""The constructed inputs of tests/policy_states.py reach, in the oracle and on the clip files, the branches of dm_policy.cu they were built
for (tests/test_policy_kernels_gpu.py compares the kernels with the oracle on them): eigen_slerp's antipodal sign flip and near-parallel blend,
QuatTheta's dead zone, loop cycles 0, 1 and >= 5, a non-looping clip at 0, inside, at and past its end, the ground lift of the reset (by a
capsule among others) and fallen characters.  Without this check the inputs could decay into states that exercise nothing."""
import numpy as np
import pytest

from tests import policy_states as P
from tests.oracle_binding import Oracle


@pytest.fixture(scope="module")
def assets(asset_root, tmp_path_factory):
    return P.make_assets(asset_root, str(tmp_path_factory.mktemp("policy") / "assets"))


def test_constructed_assets_load_in_the_oracle(assets):
    for ch, p, r, w in P.CTRLS:
        o = Oracle(P.ctrl_args(ch, p, r, w), assets)
        assert o.state_size == p + 1 + 15 * o.num_joints
    o = Oracle(P.imitate_args(P.WALK_ONCE), assets)
    loop, t, _ = P.read_clip(assets, P.WALK_ONCE)
    assert not loop and o.motion_duration == pytest.approx(1.266616, abs=1e-9)
    d = o.motion_duration
    _, v_in = o.kin_frame(d - 1e-3)
    _, v_end = o.kin_frame(d)
    assert np.abs(v_in).max() > 1.0 and not v_end.any()          # ends in motion; at rest from the end on
    dur, _, _, lp = Oracle(P.CLIPS_ARGS["heading_pair"], assets).clip_table()
    assert dur == pytest.approx([3.7665, 1.2666], abs=1e-4) and not lp.any()
    dur, _, _, lp = Oracle(P.CLIPS_ARGS["getup_real"], assets).clip_table()
    assert list(lp) == [1, 1, 0, 0]


@pytest.mark.parametrize("motion", [P.SPINKICK, P.BACKFLIP, P.FACEDOWN])
def test_antipodal_frame_pairs_are_sampled(assets, motion):
    """each of these clips has one frame pair whose quaternions of one joint have a negative dot product; the reward states sample it"""
    iv = P.intervals(assets, motion, "antipodal")
    assert len(iv) == 1
    loop, t, _ = P.read_clip(assets, motion)
    times = dict(P.clip_times(assets, motion))
    label = "antipodal %s" % iv[0][2]
    assert P.in_intervals(times[label], iv, t[-1], loop) == [iv[0][2]]


@pytest.mark.parametrize("motion", [P.WALK, P.SPINKICK, P.BACKFLIP, P.FACEDOWN, P.FACEUP, P.WALK_ONCE])
def test_reward_times_reach_their_branches(assets, motion):
    loop, t, _ = P.read_clip(assets, motion)
    dur = t[-1]
    times = P.clip_times(assets, motion)
    held = P.intervals(assets, motion, "held")
    if held:
        kt = [kt for lb, kt in times if lb.startswith("held")]
        assert len(kt) == 1 and P.in_intervals(kt[0], held, dur, loop)
    if loop:
        cycles = sorted(int(np.floor(kt / dur)) for lb, kt in times if lb.startswith("cycle"))
        assert cycles[:2] == [0, 1] and max(cycles) >= 5
    else:
        kts = dict(times)
        assert kts["start"] == 0.0 and 0 < kts["inside"] < dur and kts["end"] == dur and kts["past end"] > dur
    # QuatTheta's dead zone: on the clip every joint's rotation difference is inside it; near the clip some are outside
    o = Oracle(P.imitate_args(motion), assets)
    states = P.reward_states(o, times)
    for s in states:
        o.set_snapshot(s.snap)
        assert P.snapshot_kin_time(s.snap, o.num_joints) == pytest.approx(dict(times)[s.name.rsplit(" ", 1)[0]], abs=1e-12)
        hs = P.quat_half_sines(o, assets)
        if s.kind == "on clip":
            assert max(hs.values()) <= P.DEAD_ZONE, (s.name, hs)
        else:
            assert max(hs.values()) > 10 * P.DEAD_ZONE, (s.name, hs)
        assert not o.has_fallen(), s.name


def test_reset_lifts_some_states_off_the_ground_and_not_others(assets):
    """the face-up get-up clip lying on the ground: at some start times a body reaches within 1 mm of the ground and the oracle lifts the
    character (the lowest body ends 1 mm above it), among them states whose lowest body is a tilted capsule; at others it does not"""
    o = Oracle(P.imitate_args(P.FACEUP), assets)
    lifted, kept, capsule = [], [], []
    for kt in (0.0, 0.5, 1.64, 1.97, 2.62, 3.11, o.motion_duration, o.motion_duration + 0.5):
        o.reset(kt, 0.0, 20.0)
        lift = o.get_snapshot()[1] / P.SCALE - P.clip_root_y(assets, P.FACEUP, kt)
        low = min(P.link_bottoms(o, assets))
        if lift > 1e-6:
            lifted.append(kt)
            assert low[0] == pytest.approx(0.001, abs=1e-5)
            if low[1] == "capsule" and low[2] > 0.05:
                capsule.append(kt)
        else:
            kept.append(kt)
            assert low[0] > 0.001 - 1e-5
    print("lifted at", lifted, "of which capsule-lowest", capsule, "; kept at", kept)
    assert len(lifted) >= 3 and len(kept) >= 3 and len(capsule) >= 2


def test_fallen_states_have_fallen(assets):
    o = Oracle(P.imitate_args(P.WALK), assets)
    for k in range(4):
        s = P.lying(o, 300 + k, 0.1 + 0.3 * k, 1.1 * k - 1.5)
        o.set_snapshot(s)
        o.update(P.DT)
        assert o.has_fallen() and o.check_terminate() == 1 and o.calc_reward() == 0.0


@pytest.mark.parametrize("ch", ["humanoid3d", "dog3d"])
def test_observation_states_cover_standing_airborne_and_lying(assets, ch):
    o = Oracle(P.ctrl_args(ch, 1, 1), assets)
    states = P.observation_states(o)
    kinds = {}
    for s in states:
        o.set_snapshot(s.snap)
        low = min(b[0] for b in P.link_bottoms(o, assets, ch))
        kinds.setdefault(s.kind, []).append(low)
        if s.kind == "airborne":
            assert low > 1.0
    assert set(kinds) == {"stand", "walk", "airborne", "lying"}
    # a lying character is low: its root within 0.5 m of the ground
    for s in states:
        if s.kind == "lying":
            assert s.snap[1] / P.SCALE < 0.5, (ch, s.name, s.snap[1] / P.SCALE)
