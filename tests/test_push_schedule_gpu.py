"""The push schedule on the GPU: the drawn entries against the Python restatement (tests/push_schedule_ref.py) from the device's own timers
and reset counters, teacher-forced physics of the scheduled pushes against the CPU oracle, independence of the global_env_offset split,
the state blob's round trip and its refusals, the refusals of the entry point, and bit-exact resumption of a Trainer under pushes."""
import numpy as np
import pytest

from tests import push_schedule_ref as ref
from tests.oracle_binding import PushOracle
from tests.parity_util import SnapLayout, compare_sim_state, joint_types_from_assets, random_policy_action
from tests.test_train_gpu import AGENT, SPINKICK_TRAIN, _equal_states, _trainer

pytestmark = pytest.mark.gpu
DT = 1.0 / 600.0
SPINKICK = ["--arg_file", "args/run_humanoid3d_spinkick_args.txt"]
SCHED = dict(bodies=[0, 1, 2, 7], force=(100.0, 600.0), duration=(0.1, 0.3), gap=(0.0, 0.4))   # gaps shorter than a policy step start late


def _blob_fields(core, blob):
    """(timers [N], reset counters [N], done flags [N]) of the real environments from a save_state() blob: header, SIM, TIME, FLAGS blocks"""
    n_pad = int(blob[28:32].view(np.int32)[0])
    nl = core.dims.num_joints
    off = 160 + n_pad * (16 + 12 * nl) * 4   # the 160-byte header (capi.cu: StateHeader), then the SIM block
    tm = blob[off:off + n_pad * 16 * 8].view(np.float64).reshape(n_pad, 16)
    off += n_pad * 16 * 8
    fl = blob[off:off + n_pad * 8 * 4].view(np.int32).reshape(n_pad, 8)
    N = core.num_envs
    return tm[:N, 4].copy(), fl[:N, 7].copy(), fl[:N, 1].copy()


def _actions(core, rng):
    import torch
    return torch.as_tensor(0.3 * rng.standard_normal((core.num_envs, core.dims.action_size)), dtype=torch.float32, device="cuda")


def _core(n, seed=21, offset=0, sched=SCHED):
    from deepmimic_b200.assets import asset_root
    from deepmimic_b200.capi import BatchedCore
    c = BatchedCore(SPINKICK, n, asset_root(prefer_archive=True), device=0, seed=seed, global_env_offset=offset)
    c.set_episode_limit(1.0, 2.5)
    c.reset(True)
    if sched is not None:
        c.set_push_schedule(**sched)
    return c


def test_drawn_entries_equal_the_restatement():
    """256 environments, placement by contact load on, 60 policy steps of random actions with resets (none after every fourth step, so that
    finished environments stay frozen through an update).  Before each dm_update the restatement runs on the device's timers, reset counters and
    done flags and on its entries; after it, the schedule blocks equal the restatement's bit for bit, and so do the entries (body, start,
    duration; the force to one float32 ulp: the device's cos / sin and glibc's may round the last double bit differently), an entry whose window
    the update's 20 steps passed reading empty, as pushes() does."""
    core = _core(256)
    core.set_env_order(True)
    rng = np.random.default_rng(4)
    N, seed = core.num_envs, ref.push_seed(21)
    blocks = [[0.0, 0.0, 0.0] for _ in range(N)]
    stats = dict(drawn=0, late=0, frozen=0, resets=0, cleared=0, force_exact=0)
    for step in range(60):
        timer, resets, done = _blob_fields(core, core.save_state())
        tab = core.push_table()
        want = []
        for e in range(N):
            ent = ref.Entry(tab["body"][e], tab["force"][e], tab["start"][e], tab["duration"][e])
            if done[e]:
                stats["frozen"] += 1
            else:
                was = ent.body
                stats["resets"] += float(resets[e]) != blocks[e][0]
                ref.schedule_env(SCHED["bodies"], SCHED["force"], SCHED["duration"], SCHED["gap"], seed, e, int(resets[e]), timer[e], blocks[e], ent)
                if was == -1:
                    stats["drawn"] += 1
                    stats["late"] += ent.start == timer[e] and timer[e] > 0.0
            want.append(ent)
        core.set_action(_actions(core, rng))
        core.update(DT, 20)
        after = core.push_table(schedule=True)
        t_after, _, _ = _blob_fields(core, core.save_state())
        assert np.array_equal(after["sched"], np.array(blocks)), step
        for e, w in enumerate(want):
            if w.body >= 0 and t_after[e] >= w.start + w.duration:
                w.body = -1
                stats["cleared"] += 1
            assert after["body"][e] == w.body, (step, e)
            if w.body >= 0:
                assert after["start"][e] == w.start and after["duration"][e] == w.duration, (step, e)
                np.testing.assert_array_max_ulp(after["force"][e], w.force, maxulp=1)
                stats["force_exact"] += bool(np.array_equal(after["force"][e], w.force))
        assert np.array_equal(core.pushes(), after["body"])
        if step % 4 != 3:
            core.reset(False)
    print("schedule over 60 steps of 256 environments:", stats)
    assert stats["drawn"] > 500 and stats["late"] > 0 and stats["frozen"] > 0 and stats["resets"] > 256 and stats["cleared"] > 100


def test_scheduled_pushes_teacher_forced_against_the_oracle(asset_root):
    """Environment 0 of a scheduled handle, every Update(1/600) from the oracle's exact state; PushOracle gets the entry the schedule drew for
    that update.  Tolerances of tests/test_push_gpu.py; the entry clears on the device at the end of the update after which the timer reaches
    its end, and pushes act in both runs."""
    core = _core(64, sched=dict(SCHED, gap=(0.02, 0.1)))
    orc = PushOracle(SPINKICK, asset_root)
    jt = joint_types_from_assets(asset_root, "data/characters/humanoid3d.txt")
    lay = SnapLayout(orc.num_joints)
    off, scl, lo, hi = orc.action_statics()
    rng = np.random.default_rng(5)
    eqs, eqds, ncs, odd, total, pushed, bodies_seen = [], [], [], 0, 0, 0, set()
    prev = None
    for ep in range(3):
        orc.reset(0.1 + 0.3 * ep, 0.0, 20.0)
        for upd in range(300):
            if orc.need_new_action():
                orc.set_action(random_policy_action(rng, off, scl, lo, hi))
            if orc.is_episode_end():
                break
            snap = orc.get_snapshot()
            t = snap[13 + 55 * orc.num_joints + 12]   # the episode timer at the update's start (include/deepmimic_b200.h: the snapshot layout)
            core.set_snapshot(0, snap)
            core.update(DT, 1)
            tab = core.push_table()
            cur = (int(tab["body"][0]), tab["force"][0].astype(np.float64), float(tab["start"][0]), float(tab["duration"][0]))
            entry = cur if cur[0] >= 0 else prev     # empty after the update: the entry of this update cleared at its end
            prev = cur if cur[0] >= 0 else None
            if entry is not None:
                orc.set_push(*entry)
                if entry[2] <= t < entry[2] + entry[3]:
                    pushed += 1; bodies_seen.add(entry[0])
                assert (cur[0] < 0) == (t + DT >= entry[2] + entry[3]), upd
            else:
                orc.set_push(-1, np.zeros(3), 0.0, 0.0)
            orc.update(DT)
            so, sg = orc.get_snapshot(), core.get_snapshot(0)
            eq, eqd = compare_sim_state(lay, so, sg, jt)
            total += 1
            if eq > 1e-3 or eqd > 0.5 or lay.contact_counts(so) != lay.contact_counts(sg):
                odd += 1
                continue
            eqs.append(eq); eqds.append(eqd); ncs.append(sum(lay.contact_counts(so)))
        prev = None
        core.reset(True)   # the next episode: a new reset counter, the schedule starts over
    eqs, eqds, ncs = np.array(eqs), np.array(eqds), np.array(ncs)
    print("scheduled pushes teacher-forced: %d updates (%d pushed, bodies %s, %d off-branch) |dq| max %.2e |dqd| median %.2e p99 %.2e max %.2e"
          % (total, pushed, sorted(bodies_seen), odd, eqs.max(), np.median(eqds), np.percentile(eqds, 99), eqds.max()))
    assert pushed > 60 and len(bodies_seen) >= 2
    assert odd <= max(1, total // 50)
    assert eqs.max() <= 1e-3 and np.median(eqds) <= 2e-3 and np.percentile(eqds, 99) <= 5e-2 and eqds.max() <= 0.5


def test_schedule_is_independent_of_the_split():
    """one handle of 64 environments against two of 32 with global_env_offset 0 and 32, the same seed, schedule and actions: the same push
    tables and schedule blocks after every policy step"""
    import torch
    one = _core(64, seed=8)
    two = [_core(32, seed=8, offset=0), _core(32, seed=8, offset=32)]
    for c in [one] + two:
        c.set_env_order(False)
    rng = np.random.default_rng(6)
    for step in range(30):
        a = _actions(one, rng)
        one.set_action(a); one.update(DT, 20)
        for k, c in enumerate(two):
            c.set_action(a[32 * k:32 * (k + 1)].contiguous()); c.update(DT, 20)
        t1 = one.push_table(schedule=True)
        t2 = [c.push_table(schedule=True) for c in two]
        for key in t1:
            assert np.array_equal(t1[key], np.concatenate([t[key] for t in t2])), (step, key)
        for c in [one] + two:
            c.reset(False)
    torch.cuda.synchronize()
    assert (t1["sched"][:, 1] > 0).all()


def test_save_and_load_continue_bit_for_bit():
    """20 steps, save; 12 more on the saved handle and on a fresh scheduled handle that loads the blob: every push table and the final blobs
    bit-identical.  A handle without a schedule refuses the blob, a scheduled handle refuses a blob saved without one or under another schedule"""
    rng = np.random.default_rng(9)
    a = _core(256, seed=13)
    acts = [_actions(a, rng) for _ in range(32)]

    def run(c, steps):
        rec = []
        for x in steps:
            c.set_action(x); c.update(DT, 20)
            rec.append(c.push_table(schedule=True))
            c.reset(False)
        return rec
    run(a, acts[:20])
    blob = a.save_state()                                 # pending pushes are part of a scheduled handle's blob
    assert (a.push_table()["body"] >= 0).any()
    rec_a = run(a, acts[20:])
    b = _core(256, seed=13)
    b.load_state(blob)
    rec_b = run(b, acts[20:])
    assert all(np.array_equal(x[k], y[k]) for x, y in zip(rec_a, rec_b) for k in x)
    assert np.array_equal(a.save_state(), b.save_state())
    plain = _core(256, seed=13, sched=None)
    with pytest.raises(RuntimeError, match="another push schedule"):
        plain.load_state(blob)
    with pytest.raises(RuntimeError, match="another push schedule"):
        b.load_state(plain.save_state())
    other = _core(256, seed=13, sched=dict(SCHED, gap=(0.05, 0.5)))
    with pytest.raises(RuntimeError, match="another push schedule"):
        other.load_state(blob)
    n_pad = int(blob[28:32].view(np.int32)[0])
    assert len(plain.save_state()) + n_pad * (32 + 24) == len(blob)   # the push table and the schedule block on top of the plain blob


def test_refusals():
    c = _core(4, sched=None)
    for kw, match in ((dict(bodies=[15]), "h_bodies\\[0\\] = 15"), (dict(bodies=[0, -1]), "h_bodies\\[1\\]"), (dict(bodies=[0] * 33), "n_bodies 33"),
                      (dict(force=(600.0, 100.0)), "force2: lo > hi"), (dict(force=(-1.0, 100.0)), "force2: a bound is negative"),
                      (dict(duration=(0.1, np.inf)), "duration2: a bound is not finite"), (dict(gap=(np.nan, 1.0)), "gap2: a bound is not finite")):
        with pytest.raises(RuntimeError, match=match):
            c.set_push_schedule(**dict(SCHED, **kw))
    with pytest.raises(ValueError, match="bodies must be integers"):
        c.set_push_schedule(**dict(SCHED, bodies=[0.5]))
    with pytest.raises(RuntimeError, match="no push schedule"):
        c.push_table(schedule=True)
    c.set_push_schedule(**SCHED)
    c.set_push_schedule(**dict(SCHED, bodies=[3]))          # later calls replace the parameters
    with pytest.raises(RuntimeError, match="push schedule"):
        c.set_pushes(np.full(4, -1, dtype=np.int32), np.zeros((4, 3), dtype=np.float32), np.zeros(4), np.zeros(4))
    m = _core(4, sched=None)
    m.set_pushes(np.full(4, -1, dtype=np.int32), np.zeros((4, 3), dtype=np.float32), np.zeros(4), np.zeros(4))
    with pytest.raises(RuntimeError, match="dm_set_pushes"):
        m.set_push_schedule(**SCHED)


def test_trainer_resumes_bit_for_bit_under_pushes(asset_root, tmp_path):
    """3 iterations straight against 1, a checkpoint, a fresh Trainer from it and 2 more, with a push schedule on the training handle: every
    tensor of the state, the env blobs (push table and schedule block included) and the log rows but wall time bit-identical"""
    ps = dict(bodies=[0, 2], force=[100.0, 600.0], duration=[0.1, 0.3], gap=[0.2, 1.0])
    v = dict(AGENT, OutputIters=2, TestEpisodes=8)
    a = _trainer(asset_root, SPINKICK_TRAIN, v, num_envs=256, push_schedule=ps)
    rows_a = [a.iteration() for _ in range(3)]
    b = _trainer(asset_root, SPINKICK_TRAIN, v, num_envs=256, push_schedule=ps)
    rows_b = [b.iteration()]
    b.save(str(tmp_path / "c.pt"))
    del b
    c = _trainer(asset_root, SPINKICK_TRAIN, v, num_envs=256, push_schedule=ps)
    c.load(str(tmp_path / "c.pt"))
    rows_b += [c.iteration() for _ in range(2)]
    strip = lambda r: {k: x for k, x in r.items() if k != "Wall_Time"}
    assert [repr(strip(r)) for r in rows_a] == [repr(strip(r)) for r in rows_b]
    assert not _equal_states(a.state_dict(), c.state_dict())
    assert (a.env._core.push_table()["body"] >= 0).any() and (a.test_env._core.pushes() == -1).all()
    d = _trainer(asset_root, SPINKICK_TRAIN, v, num_envs=256)
    with pytest.raises(ValueError, match="push schedule"):
        d.load(str(tmp_path / "c.pt"))
