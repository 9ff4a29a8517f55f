"""Control latency on the GPU: zero delay bit-identical to the plain kernels (and to the dynamics kernel on a randomised handle), delays against
the plain kernel given each action the same number of updates late (one update per launch, and across launch boundaries), the hold of the reset
pose, the isolation of the environments, the randomised table against the Python restatement (tests/latency_ref.py) from the device's reset
counters and across shards, the state blob's round trip in the middle of a policy step and its refusals, the refusals of the entry points,
training and the latency sweep of a trained skill; the first episode's hold when the table comes after the handle's own reset; and the held
and delayed updates teacher-forced against the CPU oracle."""
import os

import numpy as np
import pytest

from tests import latency_ref as ref

pytestmark = pytest.mark.gpu
DT = 1.0 / 600.0
U = 20
SPINKICK = ["--arg_file", "args/run_humanoid3d_spinkick_args.txt"]
DOG = ["--arg_file", "args/train_dog3d_trot_args.txt"]
TARGET = ["--motion_file", "data/datasets/test_clips_mini.txt", "--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]
HEADER = 160   # capi.cu: StateHeader
LAT_HEADER = 8   # capi.cu: LatencyHeader, after the header of a blob with a latency table


def _core(n, seed=21, args=SPINKICK, offset=0):
    from deepmimic_b200.assets import asset_root
    from deepmimic_b200.capi import BatchedCore
    c = BatchedCore(args, n, asset_root(prefer_archive=True), device=0, seed=seed, global_env_offset=offset)
    c.set_episode_limit(1.0, 2.5)
    c.reset(True)
    return c


def _actions(core, rng):
    import torch
    return torch.as_tensor(0.3 * rng.standard_normal((core.num_envs, core.dims.action_size)), dtype=torch.float32, device="cuda")


def _observe(core):
    import torch
    st = torch.zeros(core.num_envs, core.dims.state_size, device="cuda")
    rw = torch.zeros(core.num_envs, device="cuda")
    core.observe(st, rw)
    core.sync()
    return st.cpu().numpy(), rw.cpu().numpy()


def _state(core, blob=None):
    """the blob's device blocks without the header (and the latency header and table of a latency handle)"""
    b = core.save_state() if blob is None else blob
    n_pad = int(b[28:32].view(np.int32)[0])
    lat = int(b[62:64].view(np.int16)[0])
    return b[HEADER + LAT_HEADER:len(b) - n_pad * 528] if lat else b[HEADER:]


def _physics(core):
    """the SIM, TIME, FLAGS and manifold blocks of the handle's blob: its simulation state without the placement key (DevState::load)"""
    b = core.save_state()
    n_pad, nl = int(b[28:32].view(np.int32)[0]), int(b[36:40].view(np.int32)[0])
    off = HEADER + (LAT_HEADER if int(b[62:64].view(np.int16)[0]) else 0)
    return b[off:off + n_pad * ((16 + 12 * nl) * 4 + 16 * 8 + 8 * 4 + nl * 48 * 4)]


def _flags(blob):
    """FLAGS [n_pad, 8] int32 of a blob (after SIM and TIME)"""
    n_pad = int(blob[28:32].view(np.int32)[0])
    nl = int(blob[36:40].view(np.int32)[0])
    lat = int(blob[62:64].view(np.int16)[0])
    off = HEADER + (LAT_HEADER if lat else 0) + n_pad * (16 + 12 * nl) * 4 + n_pad * 16 * 8
    return blob[off:off + n_pad * 32].view(np.int32).reshape(n_pad, 8)


def _delays(core):
    t = core.action_latency()
    core.sync()
    return np.rint(t.cpu().numpy() / DT).astype(int)


def _run(core, acts, resets=True):
    out = []
    for a in acts:
        core.set_action(a)
        core.update(DT, U)
        out.append(_observe(core) + (_state(core),))
        if resets:
            core.reset(False)
    return out


ZERO_CASES = [("spinkick", SPINKICK, 64, True), ("dog_trot", DOG, 8, False), ("target_amp", TARGET, 16, True)]


@pytest.mark.parametrize("name,args,n,placement", ZERO_CASES, ids=[c[0] for c in ZERO_CASES])
def test_zero_delay_is_bit_identical(name, args, n, placement):
    """From a saved state, 12 policy steps with resets and placement by contact load (W = 16): a handle whose delays are all 0 gives
    observations, rewards, flags and simulation state bit-identical to a plain handle's"""
    rng = np.random.default_rng(3)
    base = _core(n, args=args)
    base.set_env_order(placement)
    _run(base, [_actions(base, rng) for _ in range(6)])
    blob = base.save_state()
    acts = [_actions(base, rng) for _ in range(12)]
    plain, zero = _core(n, args=args), _core(n, args=args)
    for c in (plain, zero):
        c.load_state(blob)
        c.set_env_order(placement)
    zero.set_action_latency(np.zeros(n))
    assert np.all(_delays(zero) == 0)
    rp, rz = _run(plain, acts), _run(zero, acts)
    for (sp, wp, bp), (sz, wz, bz) in zip(rp, rz):
        assert sp.tobytes() == sz.tobytes() and wp.tobytes() == wz.tobytes()
        assert bp.tobytes() == bz.tobytes()


def test_zero_delay_on_a_randomised_dynamics_handle():
    """Zero delay on a handle with randomised dynamics is bit-identical to that handle without a latency table"""
    rng = np.random.default_rng(4)
    lohi = [0.4, 1.2, 0.8, 1.2, 0.7, 1.3, 0.5, 1.0, 0.7, 1.3]
    a, b = _core(32), _core(32)
    for c in (a, b):
        c.set_env_order(True)
        c.set_dynamics_randomization(lohi)
    b.set_action_latency(np.zeros(32))
    acts = [_actions(a, rng) for _ in range(12)]
    for (sa, wa, ba), (sb, wb, bb) in zip(_run(a, acts), _run(b, acts)):
        assert sa.tobytes() == sb.tobytes() and wa.tobytes() == wb.tobytes() and ba.tobytes() == bb.tobytes()


def _late_plain(plain, prev, new, delays):
    """one policy step on the plain handle with environment e's action set delays[e] updates late: one-update launches, and before update k
    every environment gets its new action if k >= delay else its previous one (the same targets again).  The action rows are complete and
    kept alive before the handle's stream reads them."""
    import torch
    d = torch.as_tensor(delays, device="cuda")
    rows = [torch.where((k >= d)[:, None], new, prev).contiguous() for k in range(U)]
    torch.cuda.synchronize()
    for k in range(U):
        plain.set_action(rows[k])
        plain.update(DT, 1)
    plain.sync()


@pytest.mark.parametrize("chunk", [U, 5, 1], ids=["one launch", "launches of 5", "launches of 1"])
def test_delays_equal_the_action_set_late(chunk):
    """16 spin-kick environments from a mid-episode state, placement by contact load (two environments per W = 16 warp with different
    delays), delays 0, 1, 7, 12 and 19 over three policy steps: the latency handle's simulation state, observations and rewards equal, bit
    for bit, a plain handle's that gets each environment's action that many updates late.  The latency handle runs its policy steps in one
    launch, in launches of 5 updates (d = 7 and 12 take effect in a later launch than the action's) or of 1.  Environments 8-15 have no delay."""
    rng = np.random.default_rng(5)
    n = 16
    base = _core(n)
    base.set_env_order(True)
    _run(base, [_actions(base, rng) for _ in range(4)], resets=False)
    blob = base.save_state()
    delays = np.array([1, 7, 19, 12, 0, 7, 1, 19] + [0] * 8)
    plain, lat = _core(n), _core(n)
    prev = _actions(plain, rng)
    for c in (plain, lat):   # the targets the first delayed actions replace
        c.load_state(blob)
        c.set_env_order(True)
        c.set_action(prev)
        c.update(DT, U)
    lat.set_action_latency(delays * DT)
    assert np.array_equal(_delays(lat), delays)
    for step in range(3):
        new = _actions(plain, rng)
        _late_plain(plain, prev, new, delays)
        lat.set_action(new)
        for _ in range(U // chunk):
            lat.update(DT, chunk)
        sp, wp = _observe(plain)
        sl, wl = _observe(lat)
        assert sp.tobytes() == sl.tobytes() and wp.tobytes() == wl.tobytes(), step
        assert _physics(plain).tobytes() == _physics(lat).tobytes(), step
        prev = new


def test_a_pending_action_is_replaced_and_a_reset_holds_the_start_pose():
    """A second action set while the first is pending replaces it; after a reset the PD targets are the reset pose (snapshot targets equal the
    joint rotations and angles) until the delayed first action takes effect, and the update counter restarts its clock"""
    rng = np.random.default_rng(6)
    n = 4
    lat = _core(n)
    from deepmimic_b200.assets import asset_root
    from tests.parity_util import joint_types_from_assets
    lat.set_action_latency(np.full(n, 7 * DT))
    lat.reset(True)
    nl = lat.dims.num_joints
    b = lat.save_state()
    n_pad = int(b[28:32].view(np.int32)[0])
    sim = b[HEADER + LAT_HEADER:HEADER + LAT_HEADER + n_pad * (16 + 12 * nl) * 4].view(np.float32).reshape(n_pad, 16 + 12 * nl)
    jt = joint_types_from_assets(asset_root(prefer_archive=True), "data/characters/humanoid3d.txt")
    moving = [l for l in range(1, nl) if jt[l].lower() in ("spherical", "revolute")]
    assert len(moving) >= 10
    for e in range(n):
        jp, tg = sim[e, 16:16 + 4 * nl].reshape(nl, 4), sim[e, 16 + 8 * nl:16 + 12 * nl].reshape(nl, 4)
        assert np.array_equal(jp[moving], tg[moving]), e
    # replaced: a then b within one pending window equals b alone
    a, b = _actions(lat, rng), _actions(lat, rng)
    blob = lat.save_state()
    lat.set_action(a)
    lat.set_action(b)
    lat.update(DT, U)
    two = _state(lat)
    lat.load_state(blob)
    lat.set_action(b)
    lat.update(DT, U)
    assert two.tobytes() == _state(lat).tobytes()


def test_isolation():
    """Delays on environments 3 and 5 leave the other environments bit-identical to a plain handle's"""
    rng = np.random.default_rng(8)
    n = 32
    plain, lat = _core(n), _core(n)
    for c in (plain, lat):
        c.set_env_order(True)
    d = np.zeros(n)
    d[3], d[5] = 4 * DT, 19 * DT
    lat.set_action_latency(d)
    acts = [_actions(plain, rng) for _ in range(8)]
    keep = np.ones(n, dtype=bool)
    keep[[3, 5]] = False
    changed = False
    for (sp, wp, _), (sl, wl, _) in zip(_run(plain, acts), _run(lat, acts)):
        assert sp[keep].tobytes() == sl[keep].tobytes() and wp[keep].tobytes() == wl[keep].tobytes()
        changed |= sp[3].tobytes() != sl[3].tobytes()
    assert changed


def test_randomised_delays_follow_the_restatement_and_shards():
    """256 environments, 40 policy steps with resets: after every step each environment's delay is the restatement's for its reset counter
    (so the ones a reset did not restart keep theirs); the same seed repeats the draws; a shard at global_env_offset 128 draws its
    environments' delays as the whole batch does"""
    rng = np.random.default_rng(9)
    lo, hi = 2, 17
    a = _core(256, seed=13)
    a.set_env_order(True)
    a.set_action_latency_randomization(lo * DT, hi * DT)
    seed = ref.lat_seed(13)
    seen = set()
    for step in range(40):
        a.set_action(_actions(a, rng))
        a.update(DT, U)
        a.reset(False)
        fl = _flags(a.save_state())
        d = _delays(a)
        for e in range(256):
            r = int(fl[e, 7])
            seen.add((e, r))
            assert d[e] == ref.draw(lo, hi, seed, e, r), (step, e, r)
    assert len(seen) > 256 + 100 and len(set(d)) == hi - lo + 1
    shard = _core(128, seed=13, offset=128)
    shard.set_action_latency_randomization(lo * DT, hi * DT)
    fl, d = _flags(shard.save_state()), _delays(shard)
    assert all(d[e] == ref.draw(lo, hi, seed, 128 + e, int(fl[e, 7])) for e in range(128))
    again = _core(128, seed=13, offset=128)
    again.set_action_latency_randomization(lo * DT, hi * DT)
    assert np.array_equal(_delays(again), d)


def test_blob_mid_step_resumes_and_refusals():
    """A save 5 updates into a policy step with actions pending (delays 12 and 19), a load into a fresh randomised handle and the rest of the
    step and two more continue bit-identically to not saving.  Blobs with and without a table, and of other bounds, are refused across."""
    rng = np.random.default_rng(10)
    a = _core(64, seed=13)
    a.set_action_latency_randomization(12 * DT, 19 * DT)
    acts = [_actions(a, rng) for _ in range(4)]
    a.set_action(acts[0])
    a.update(DT, U)
    a.reset(False)
    a.set_action(acts[1])
    a.update(DT, 5)
    blob = a.save_state()
    b = _core(64, seed=13)
    b.set_action_latency_randomization(12 * DT, 19 * DT)
    b.load_state(blob)
    for c in (a, b):
        c.update(DT, U - 5)
        c.reset(False)
        for x in acts[2:]:
            c.set_action(x)
            c.update(DT, U)
            c.reset(False)
    assert a.save_state().tobytes() == b.save_state().tobytes()
    assert _observe(a)[0].tobytes() == _observe(b)[0].tobytes()
    plain = _core(64, seed=13)
    with pytest.raises(RuntimeError, match="another action latency table"):
        plain.load_state(blob)
    with pytest.raises(RuntimeError, match="another action latency table"):
        b.load_state(plain.save_state())
    other = _core(64, seed=13)
    other.set_action_latency_randomization(0.0, 19 * DT)
    with pytest.raises(RuntimeError, match="action latency randomisation"):
        other.load_state(blob)
    explicit = _core(64, seed=13)
    explicit.set_action_latency(np.zeros(64))
    with pytest.raises(RuntimeError, match="action latency randomisation"):
        explicit.load_state(blob)


def test_refusals():
    from deepmimic_b200 import capi
    c = _core(4)
    with pytest.raises(RuntimeError, match="no latency table"):
        c.action_latency()
    with pytest.raises(ValueError, match="environment 2"):
        c.set_action_latency([0.0, 0.0, 0.04, 0.0])
    d = np.zeros(4, dtype=np.int32)
    d[1] = 20
    import ctypes as C
    assert capi.lib().dm_set_action_latency(c.h, d.ctypes.data_as(C.POINTER(C.c_int32))) != 0
    assert "environment 1: delay 20" in capi.lib().dm_last_error().decode()
    assert capi.lib().dm_set_action_latency_randomization(c.h, 5, 3) != 0
    assert "lo 5 > hi 3" in capi.lib().dm_last_error().decode()
    c.set_action_latency([0.0, DT, 2 * DT, 19 * DT])
    assert list(_delays(c)) == [0, 1, 2, 19]
    with pytest.raises(RuntimeError, match="dm_set_action_latency, which own"):
        c.set_action_latency_randomization(0.0, 0.01)
    r = _core(4)
    r.set_action_latency_randomization(0.0, 0.01)
    with pytest.raises(RuntimeError, match="randomised"):
        r.set_action_latency(np.zeros(4))


def test_trainer_resumes_bit_for_bit_under_latency(asset_root, tmp_path):
    """--rand_latency 0,0.03 on 512 training environments: 3 iterations straight against 1, a checkpoint, a fresh Trainer from it and 2 more,
    the log rows but wall time bit-identical and finite.  The evaluation handle has no latency table; a Trainer without the option refuses the
    checkpoint."""
    from tests.test_train_gpu import AGENT, SPINKICK_TRAIN, _trainer
    lr = (0.0, 0.03)
    v = dict(AGENT, OutputIters=2, TestEpisodes=8)
    a = _trainer(asset_root, SPINKICK_TRAIN, v, num_envs=512, latency_randomization=lr)
    rows_a = [a.iteration() for _ in range(3)]
    b = _trainer(asset_root, SPINKICK_TRAIN, v, num_envs=512, latency_randomization=lr)
    rows_b = [b.iteration()]
    b.save(str(tmp_path / "c.pt"))
    del b
    c = _trainer(asset_root, SPINKICK_TRAIN, v, num_envs=512, latency_randomization=lr)
    c.load(str(tmp_path / "c.pt"))
    rows_b += [c.iteration() for _ in range(2)]
    strip = lambda r: {k: x for k, x in r.items() if k != "Wall_Time"}
    assert [repr(strip(r)) for r in rows_a] == [repr(strip(r)) for r in rows_b]
    assert all(np.isfinite(float(x)) for r in rows_a for k, x in strip(r).items() if isinstance(x, (int, float)))
    d = _delays(a.env._core)
    assert d.min() == 0 and d.max() == 18 and len(set(d)) == 19
    with pytest.raises(RuntimeError, match="no latency table"):
        a.test_env._core.action_latency()
    e = _trainer(asset_root, SPINKICK_TRAIN, v, num_envs=512)
    with pytest.raises(ValueError, match="latency randomisation"):
        e.load(str(tmp_path / "c.pt"))


def test_latency_sweep_of_the_spinkick_policy(asset_root, tmp_path):
    """The committed spin-kick fp16 policy in test mode, 96 environments of 6 s, plain and with --latency_sweep 0,0.0167,0.0317: the
    zero-delay environments run exactly the plain run's episodes, the log gets the Latency column and the summary one line per value"""
    from deepmimic_b200.formats import read_table_log
    from tests.test_dynamics_gpu import _run_cmd
    from tests.test_run_cpu import _bundle, _fixture
    prefix = _bundle(tmp_path, _fixture("policy_humanoid3d_spinkick_fp16.npz"))
    N = 96
    _run_cmd(asset_root, prefix, tmp_path / "plain", N, [])
    plain = read_table_log(str(tmp_path / "plain" / "run_log.txt"))
    stdout = _run_cmd(asset_root, prefix, tmp_path / "lat", N, ["--latency_sweep", "0,0.0167,0.0317"])
    print(stdout)
    log = read_table_log(str(tmp_path / "lat" / "run_log.txt"))
    want = [0.0, 10 * DT, 19 * DT]
    assert np.allclose(log["Latency"], [want[e % 3] for e in range(N)], rtol=0, atol=1e-12)
    z = log["Latency"] == 0.0
    assert np.array_equal(log["Terminate"][z], plain["Terminate"][z]) and np.array_equal(log["Return"][z], plain["Return"][z])
    lines = [l for l in stdout.splitlines() if l.startswith("latency ")]
    assert len(lines) == 3 and all("32 episodes" in l for l in lines)


def _blob_targets(core):
    """(jp, tg) [n_pad, links, 4] of the handle's blob: the joint state and the PD target slot of every environment"""
    b = core.save_state()
    n_pad, nl = int(b[28:32].view(np.int32)[0]), int(b[36:40].view(np.int32)[0])
    off = HEADER + (LAT_HEADER if int(b[62:64].view(np.int16)[0]) else 0)
    sim = b[off:off + n_pad * (16 + 12 * nl) * 4].view(np.float32).reshape(n_pad, 16 + 12 * nl)
    return sim[:, 16:16 + 4 * nl].reshape(n_pad, nl, 4), sim[:, 16 + 8 * nl:].reshape(n_pad, nl, 4)


def test_first_episode_holds_its_start_pose(asset_root):
    """A table set after the handle's own first reset (the constructor's, as DeepMimicBatchEnv and run do) holds that episode's start pose
    exactly as a table set before the reset: the same injected reset, then two policy steps with delays 3 and 19, give bit-identical blobs.
    A table set in the middle of an episode keeps the targets it finds."""
    from tests.parity_util import joint_types_from_assets
    rng = np.random.default_rng(12)
    n = 8
    d = np.array([3, 19] * 4) * DT
    K, M, Z = np.linspace(0.1, 1.2, n), np.full(n, 20.0), np.zeros(n)
    after, before = _core(n), _core(n)
    after.reset(True, kin_time=K, max_time=M, rot_theta=Z)
    after.set_action_latency(d)
    before.set_action_latency(d)
    before.reset(True, kin_time=K, max_time=M, rot_theta=Z)
    jt = joint_types_from_assets(asset_root, "data/characters/humanoid3d.txt")
    moving = [l for l in range(1, len(jt)) if jt[l].lower() in ("spherical", "revolute")]
    jp, tg = _blob_targets(after)
    assert np.array_equal(jp[:n, moving], tg[:n, moving])
    assert after.save_state().tobytes() == before.save_state().tobytes()
    for _ in range(2):
        a = _actions(after, rng)
        for c in (after, before):
            c.set_action(a)
            c.update(DT, U)
        assert after.save_state().tobytes() == before.save_state().tobytes()
    mid = _core(n)
    mid.set_action(_actions(mid, rng))
    mid.update(DT, 5)
    _, tg0 = _blob_targets(mid)
    mid.set_action_latency(d)
    assert np.array_equal(_blob_targets(mid)[1], tg0)


@pytest.mark.parametrize("kin_time", [0.35, 1.1])
def test_held_and_delayed_updates_match_the_oracle(asset_root, kin_time):
    """Teacher-forced against the CPU oracle, update by update: from a reset with a latency table, environments with delays 0, 1, 7 and 19 run
    two policy steps in one-update launches; before every update the oracle takes the environment's state (PD targets included), and it gets
    the action (dmo_set_action) d updates late.  The held updates after the reset and the update at which the delayed targets take effect
    are compared with test_parity_gpu.py's tolerances (|dq| <= 1e-3; |dqd| contact-free <= 1e-3, with contacts median <= 2e-3, p99 <= 5e-2,
    max <= 0.5; at most 2 % of the updates on a contact branch the oracle takes under ulp-level noise)."""
    import torch
    from deepmimic_b200.capi import BatchedCore
    from tests.oracle_binding import Oracle
    from tests.parity_util import SnapLayout, compare_sim_state, joint_types_from_assets, random_policy_action
    delays = [0, 1, 7, 19]
    n = len(delays)
    core = BatchedCore(SPINKICK, n, asset_root, device=0, seed=1234)
    core.set_env_order(False)
    core.set_action_latency(np.array(delays) * DT)
    core.reset(True, kin_time=np.full(n, kin_time), max_time=np.full(n, 20.0), rot_theta=np.zeros(n))
    orcs = [Oracle(SPINKICK, asset_root) for _ in range(n)]
    jt = joint_types_from_assets(asset_root, "data/characters/humanoid3d.txt")
    lay = SnapLayout(orcs[0].num_joints)
    off, scl, lo, hi = orcs[0].action_statics()
    rng = np.random.default_rng(int(kin_time * 100))
    eqs, eqds, ncs, odd, total = [], [], [], 0, 0
    live = [True] * n
    for step in range(2):
        a = np.stack([random_policy_action(rng, off, scl, lo, hi) for _ in range(n)]).astype(np.float32)
        core.set_action(torch.as_tensor(a, device="cuda"))
        for k in range(U):
            for e in range(n):
                if live[e]:
                    orcs[e].set_snapshot(core.get_snapshot(e))
                    if k == delays[e]:
                        orcs[e].set_action(a[e].astype(np.float64))
            core.update(DT, 1)
            for e in range(n):
                if not live[e]:
                    continue
                orcs[e].update(DT)
                so, sg = orcs[e].get_snapshot(), core.get_snapshot(e)
                eq, eqd = compare_sim_state(lay, so, sg, jt)
                total += 1
                if eq > 1e-3 or eqd > 0.5 or lay.contact_counts(so) != lay.contact_counts(sg):
                    odd += 1
                else:
                    eqs.append(eq); eqds.append(eqd); ncs.append(sum(lay.contact_counts(so)))
                if orcs[e].is_episode_end():
                    live[e] = False
    eqs, eqds, ncs = np.array(eqs), np.array(eqds), np.array(ncs)
    print("latency parity kin_time %g: %d updates (%d with contacts, %d off-branch) |dq| max %.2e |dqd| median %.2e p99 %.2e max %.2e"
          % (kin_time, total, int((ncs > 0).sum()), odd, eqs.max(), np.median(eqds), np.percentile(eqds, 99), eqds.max()))
    assert total >= 100 and odd <= max(1, total // 50)
    if (ncs == 0).any():
        assert eqds[ncs == 0].max() <= 1e-3
    assert eqs.max() <= 1e-3 and np.median(eqds) <= 2e-3 and np.percentile(eqds, 99) <= 5e-2 and eqds.max() <= 0.5
