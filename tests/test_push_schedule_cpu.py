"""The push schedule on the CPU: the shared host / device code of dm_push.cuh through a g++ shim against the Python restatement
(tests/push_schedule_ref.py), bit for bit, across resets, empty and pending entries and late starts; the train command's push options; the
Trainer's run record with and without a schedule, and the refusal of a checkpoint from another schedule."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import push_schedule_ref as ref

HERE = os.path.dirname(os.path.abspath(__file__))
DT = 1.0 / 600.0


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    """dm_push.cuh compiled with g++ (no contraction of a product into an add, as on the device with its explicit roundings)"""
    so = str(tmp_path_factory.mktemp("push_shim") / "libpush_schedule_shim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-x", "c++", os.path.join(HERE, "push_schedule_shim.cpp"),
                           "-o", so])
    L = C.CDLL(so)
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int)
    L.shim_push_schedule.argtypes = [ip, C.c_int, dp, C.c_uint64, C.c_uint64, C.c_int, C.c_double, dp, ip, C.POINTER(C.c_float), dp]
    L.shim_push_seed_key.restype = C.c_uint64
    return L


def _shim_step(L, bodies, bounds, seed, env, resets, timer, block, entry):
    b = np.ascontiguousarray(bodies, dtype=np.int32)
    bd = np.ascontiguousarray(bounds, dtype=np.float64)
    body = C.c_int(entry[0])
    force = np.ascontiguousarray(entry[1], dtype=np.float32)
    window = np.array([entry[2], entry[3]], dtype=np.float64)
    dp = C.POINTER(C.c_double)
    L.shim_push_schedule(b.ctypes.data_as(C.POINTER(C.c_int)), len(b), bd.ctypes.data_as(dp), seed, env, resets, timer, block.ctypes.data_as(dp),
                         C.byref(body), force.ctypes.data_as(C.POINTER(C.c_float)), window.ctypes.data_as(dp))
    return [body.value, force, window[0], window[1]]


SCHEDULES = [([0], (100.0, 600.0), (0.1, 0.3), (1.0, 3.0)),                 # the root only
             ([0, 1, 2, 7, 14], (0.0, 1000.0), (0.0, 0.5), (0.0, 0.2)),      # short gaps: most starts are late
             ([3] * 32, (250.0, 250.0), (0.2, 0.2), (0.5, 0.5)),             # 32 bodies, degenerate ranges
             ([5, 9], (0.0, 0.0), (1e-3, 2.0), (0.0, 0.0))]                  # zero force, zero gap


@pytest.mark.parametrize("k", range(len(SCHEDULES)))
def test_shim_matches_the_restatement_bit_for_bit(shim, k):
    """Six environments of a scripted rollout: 20-update policy steps, each environment's entry cleared as the step kernel clears it (timer
    past the window), episodes ending at random (the reset clears the entry and moves the counter), frozen environments skipped.  The shim and
    the restatement keep their own blocks and entries; after every step both equal, bit for bit.  The script meets every branch: new episodes,
    empty and pending entries, starts after the previous push and late starts moved to the timer."""
    bodies, force, duration, gap = SCHEDULES[k]
    bounds = list(force) + list(duration) + list(gap)
    seed = ref.push_seed(1234 + k)
    assert shim.shim_push_seed_key() == ref.PUSH_SEED_KEY and shim.shim_push_sched_doubles() == 3
    rng = np.random.default_rng(k)
    envs = [0, 1, 2, 77, 4095, 123456789]
    state = []
    for e in envs:
        state.append(dict(resets=1, timer=0.0, done=False, blk_s=np.zeros(3), blk_r=[0.0, 0.0, 0.0], ent_s=[-1, np.zeros(3, np.float32), 0.0, 0.0],
                          ent_r=ref.Entry()))
    seen = dict(new_episode=0, pending=0, drawn=0, late=0, after_gap=0)
    for step in range(300):
        for e, st in zip(envs, state):
            if st["done"]:   # the reset between two steps: counter moves, entry cleared, timer 0
                st["resets"] += 1; st["timer"] = 0.0; st["done"] = False
                st["ent_s"][0] = -1; st["ent_r"].body = -1
            else:
                if float(st["resets"]) != st["blk_r"][0]:
                    seen["new_episode"] += 1
                pending = st["ent_r"].body != -1
                seen["pending"] += pending
                last_end = st["blk_r"][2] if float(st["resets"]) == st["blk_r"][0] else 0.0
                st["ent_s"] = _shim_step(shim, bodies, bounds, seed, e, st["resets"], st["timer"], st["blk_s"], st["ent_s"])
                ref.schedule_env(bodies, force, duration, gap, seed, e, st["resets"], st["timer"], st["blk_r"], st["ent_r"])
                assert st["ent_s"][0] == st["ent_r"].body and st["ent_r"].body in bodies
                assert st["ent_s"][1].tobytes() == st["ent_r"].force.tobytes() and st["ent_r"].force[1] == 0.0
                assert st["ent_s"][2] == st["ent_r"].start and st["ent_s"][3] == st["ent_r"].duration
                assert list(st["blk_s"]) == st["blk_r"]
                if not pending:   # a push drawn now: in its ranges, after the previous one, never before the timer
                    r = st["ent_r"]
                    seen["drawn"] += 1
                    seen["late"] += r.start == st["timer"] and st["timer"] > last_end + gap[0]
                    seen["after_gap"] += r.start > st["timer"]
                    assert force[0] * (1 - 1e-6) - 1e-6 <= float(np.hypot(r.force[0], r.force[2])) <= force[1] * (1 + 1e-6) + 1e-6
                    assert duration[0] <= r.duration <= duration[1] and r.start >= st["timer"] and r.start >= last_end + gap[0]
                # the 20 updates of the step: the entry clears at the end of the update after which the timer reaches its end
                for _ in range(20):
                    st["timer"] += DT
                    if st["ent_r"].body >= 0 and st["timer"] >= st["ent_r"].start + st["ent_r"].duration:
                        st["ent_r"].body = -1; st["ent_s"][0] = -1
                st["done"] = rng.random() < 0.02
    print("branches:", seen)
    assert seen["new_episode"] >= 6 and seen["pending"] > 0 and seen["drawn"] > 6
    if k == 1:
        assert seen["late"] > 0
    if k in (0, 2):
        assert seen["after_gap"] > 0


def test_a_new_episode_restarts_the_draws():
    """the draw counter restarts at a new episode: an environment's first push of an episode is the same in every episode (start moved to
    the timer when the schedule first meets it late), and the global environment id keys the stream"""
    bodies, force, duration, gap = SCHEDULES[0]
    seed = ref.push_seed(7)
    firsts = []
    for resets, timer in ((1, 0.0), (2, 0.0), (5, 0.0), (9, 4.0)):
        blk, ent = [0.0, 0.0, 0.0], ref.Entry()
        ref.schedule_env(bodies, force, duration, gap, seed, 3, resets, timer, blk, ent)
        firsts.append((ent.body, ent.force.tobytes(), ent.start, ent.duration))
        assert blk[1] == 5.0 and blk[2] == ent.start + ent.duration
    assert firsts[0] == firsts[1] == firsts[2]
    assert firsts[3][2] == 4.0 and firsts[3][3] == firsts[0][3]     # late start moved to the timer, same draws
    blk, ent = [0.0, 0.0, 0.0], ref.Entry()
    ref.schedule_env(bodies, force, duration, gap, seed, 4, 1, 0.0, blk, ent)
    assert (ent.start, ent.duration) != firsts[0][2:]


# ---- the train command's options
def _parse(argv):
    from deepmimic_b200.train import build_parser, push_schedule
    opts, rest = build_parser().parse_known_args(argv)
    return push_schedule(opts), rest


FULL = ["--push_force", "100,600", "--push_bodies", "0,1", "--push_duration", "0.1,0.3", "--push_interval", "1,3"]


def test_push_options_parse():
    ps, rest = _parse(["--arg_file", "a.txt"] + FULL + ["--scene", "imitate"])
    assert ps == dict(bodies=[0, 1], force=[100.0, 600.0], duration=[0.1, 0.3], gap=[1.0, 3.0])
    assert rest == ["--arg_file", "a.txt", "--scene", "imitate"]      # not passed on to the scene
    assert _parse(["--arg_file", "a.txt"]) == (None, ["--arg_file", "a.txt"])


@pytest.mark.parametrize("opt,bad", [("--push_force", "600,100"), ("--push_force", "-1,5"), ("--push_force", "1"), ("--push_force", "1,2,3"),
                                     ("--push_force", "nan,5"), ("--push_duration", "0,inf"), ("--push_interval", "a,b"),
                                     ("--push_bodies", "-1"), ("--push_bodies", "0.5"), ("--push_bodies", ",".join(["0"] * 33)), ("--push_bodies", "")])
def test_push_options_refuse_bad_values(opt, bad):
    argv = list(FULL)
    argv[argv.index(opt) + 1] = bad
    with pytest.raises(SystemExit):
        _parse(argv)


@pytest.mark.parametrize("drop", ["--push_force", "--push_bodies", "--push_duration", "--push_interval"])
def test_push_options_come_together(drop, capsys):
    argv = list(FULL)
    i = argv.index(drop)
    del argv[i:i + 2]
    with pytest.raises(SystemExit, match=drop):
        _parse(argv)


# ---- the Trainer's run record
class _PushStandIn:
    """tests/test_train_cpu.py's stand-in env with set_push_schedule recorded"""

    def __new__(cls, n, amp):
        from tests.test_train_cpu import _StandInEnv

        class Env(_StandInEnv):
            def set_push_schedule(self, bodies, force, duration, gap):
                self.push_schedule = dict(bodies=bodies, force=force, duration=duration, gap=gap)
        return Env(n, amp)


def _trainer(ps, n=8):
    import torch
    from deepmimic_b200 import trainer as tr
    from tests.test_train_cpu import PPO, _edit
    torch.manual_seed(0)
    cfg = tr.AgentConfig(_edit(PPO, InitSamples=16, TestEpisodes=4, MiniBatchSize=16))
    env, test_env = _PushStandIn(n, False), _PushStandIn(4, False)
    t = tr.Trainer(["--scene", "stand-in"], cfg, "", n, window_steps=4, backend="torch", seed=3, env=env, test_env=test_env, push_schedule=ps)
    return t, env, test_env


PS = dict(bodies=(0, 1), force=(100, 600), duration=(0.1, 0.3), gap=(1.0, 3.0))


def test_run_record_and_checkpoints_with_and_without_a_schedule(tmp_path):
    a, env, test_env = _trainer(None)
    assert "push_schedule" not in a.run and not hasattr(env, "push_schedule") and not hasattr(test_env, "push_schedule")
    b, env, test_env = _trainer(PS)
    want = dict(bodies=[0, 1], force=[100.0, 600.0], duration=[0.1, 0.3], gap=[1.0, 3.0])
    assert b.run["push_schedule"] == want and env.push_schedule == want
    assert not hasattr(test_env, "push_schedule")                     # the evaluation handle runs without pushes
    for t in (a, b):
        t.iteration()
    a.save(str(tmp_path / "none.pt"))
    b.save(str(tmp_path / "push.pt"))
    _trainer(None)[0].load(str(tmp_path / "none.pt"))
    _trainer(dict(PS))[0].load(str(tmp_path / "push.pt"))
    for ps, path in ((None, "push.pt"), (PS, "none.pt"), (dict(PS, force=(100, 601)), "push.pt"), (dict(PS, bodies=[0]), "push.pt")):
        with pytest.raises(ValueError, match="push schedule"):
            _trainer(ps)[0].load(str(tmp_path / path))


@pytest.mark.parametrize("bad", [dict(bodies=[0], force=(1, 2), duration=(1, 2)), dict(PS, gap=(1, 2, 3)), [1, 2]])
def test_trainer_refuses_a_malformed_schedule(bad):
    with pytest.raises(ValueError, match="push_schedule"):
        _trainer(bad)
