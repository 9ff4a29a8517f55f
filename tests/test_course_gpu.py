"""Goal courses and goal markers on the GPU: a course handle against the task-state hook bit for bit, isolation of the environments without a
course, no redraws, the record against tests/course_ref.py, the setter's restart and every refusal, the marked renderer against
dm_render_poses and a float64 restatement, and the reference's pretrained heading policy steered along a course through `run`."""
import ctypes as C
import math

import numpy as np
import pytest

from tests import course_ref as ref
from tests import render_marker_ref as MR
from tests import render_ref as RR
from tests.test_run_cpu import _bundle, _fixture

pytestmark = pytest.mark.gpu
MINI = ["--motion_file", "data/datasets/test_clips_mini.txt"]
HEADING = MINI + ["--arg_file", "args/train_amp_heading_humanoid3d_locomotion_args.txt"]
TARGET = MINI + ["--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]
HEADING_ROWS = [[0.0, 0.3, 1.0], [0.4, 1.2, 1.6], [0.9, -0.5, 0.4], [2.0, 6.0, 1.2]]
TARGET_ROWS = [[0.3, 0.0], [0.45, 0.1], [1.5, -1.0], [-2.0, 2.0]]
SCENES = {"heading": (HEADING, HEADING_ROWS), "target": (TARGET, TARGET_ROWS)}
GOAL_SLOTS = [0, 1, 2, 3, 4, 5]   # dm_task.cuh: kKTarX, kKTarZ, kKSpeed, kKHeading, kKTimer, kKTimerMax
COUNTER = 12                       # kKCounter


def _env(asset_root, args, n, seed=3):
    from deepmimic_b200.env import DeepMimicBatchEnv
    return DeepMimicBatchEnv(args, n, asset_root, device=0, seed=seed)


def _tau(env, e):
    nl = env._core.dims.num_joints
    return float(env._core.get_snapshot(e)[13 + 55 * nl + 12])   # the snapshot's clocks: episode time (kTTimer)


def _hook(course_env, plain_env):
    """the existing hook: the plain handle's task blocks get the course handle's goal and the parked timer through dm_set_task_state"""
    for e in range(plain_env.num_envs):
        a, b = course_env._core.task_state(e), plain_env._core.task_state(e)
        b[GOAL_SLOTS] = a[GOAL_SLOTS]
        plain_env._core.set_task_state(e, b)


def _observe(env):
    pose, _ = env.record_pose()
    return [t.clone() for t in (env.record_state(), env.calc_reward(), env.record_goal(), pose)] + [env._refresh_flags().clone()]


def _roots(env):
    pose, _ = env.record_pose()
    p = pose.double().cpu().numpy()
    return p[:, 0], p[:, 2]


@pytest.mark.parametrize("scene", ["heading", "target"])
def test_course_equals_the_task_state_hook(asset_root, scene):
    """a handle with a course against an identical handle without one whose task blocks get the same goal and a parked timer through
    dm_get_task_state / dm_set_task_state after every update and reset: observations, rewards, goals, poses, flags and whole task blocks
    identical over 200 policy steps with resets.  Along the way: the course handle's draw counters never move inside an episode, its heading
    goals are course_ref's bits at the episode time, and its record matches course_ref on dm_record_pose's roots within 1e-5."""
    import torch
    args, rows = SCENES[scene]
    N = 8
    course, plain = _env(asset_root, args, N), _env(asset_root, args, N)
    course.set_goal_course(np.asarray(rows))
    _hook(course, plain)
    succ = course._core.task_params()[0][4]
    refs = [ref.Course(scene, rows, succ) for _ in range(N)]
    rx, rz = _roots(course)
    for e in range(N):
        refs[e].start(rx[e], rz[e], _tau(course, e))
    counters = [course._core.task_state(e)[COUNTER] for e in range(N)]
    g = torch.Generator(device="cuda").manual_seed(11)
    resets = 0
    for step in range(200):
        a = 0.4 * torch.randn(N, course.get_action_size(), device="cuda", generator=g)
        for env in (course, plain):
            env.set_action(a)
            env.update(env.UPDATE_DT, env.get_updates_per_action())
        _hook(course, plain)
        rec = course.course_record().double().cpu().numpy()
        rx, rz = _roots(course)
        for e in range(N):
            want = refs[e].step(rx[e], rz[e], _tau(course, e))
            assert np.allclose(rec[e], want, rtol=1e-5, atol=1e-5), (step, e, rec[e], want)
            tk = course._core.task_state(e)
            if scene == "heading":
                assert (tk[3], tk[2]) == ref.heading_goal(rows, _tau(course, e)), (step, e)
            assert tk[COUNTER] == counters[e] and tk[4] == 0.0 and tk[5] == np.inf, (step, e, tk)
            assert np.array_equal(tk, plain._core.task_state(e)), (step, e)
        for x, y in zip(_observe(course), _observe(plain)):
            assert torch.equal(x, y), step
        done = course.is_episode_end().cpu().numpy()
        resets += int(done.sum())
        for env in (course, plain):
            env.reset()
        _hook(course, plain)
        rx, rz = _roots(course)
        for e in np.nonzero(done)[0]:
            want = refs[e].start(rx[e], rz[e], _tau(course, e))
            assert np.allclose(course.course_record()[e].double().cpu().numpy(), want, rtol=1e-5, atol=1e-5)
            counters[e] = course._core.task_state(e)[COUNTER]
        for x, y in zip(_observe(course), _observe(plain)):
            assert torch.equal(x, y), step
    print("%s: %d resets in 200 policy steps of 8 environments" % (scene, resets))
    assert resets > 0


@pytest.mark.parametrize("scene", ["heading", "target"])
def test_environments_without_a_course_are_untouched(asset_root, scene):
    """every other environment of a course handle has count 0 (courses and no-course environments share warps): those are bit-identical
    to the same environments of a handle without a course, task blocks included, over 100 policy steps with resets"""
    import torch
    args, rows = SCENES[scene]
    N = 32
    course, plain = _env(asset_root, args, N, seed=5), _env(asset_root, args, N, seed=5)
    r = np.broadcast_to(np.asarray(rows, dtype=np.float64), (N,) + np.asarray(rows).shape)
    counts = np.where(np.arange(N) % 2 == 0, len(rows), 0)
    course.set_goal_course(r, counts)
    free = np.nonzero(counts == 0)[0]
    g = torch.Generator(device="cuda").manual_seed(2)
    for step in range(100):
        a = 0.4 * torch.randn(N, course.get_action_size(), device="cuda", generator=g)
        for env in (course, plain):
            env.step(a)
        for x, y in zip(_observe(course), _observe(plain)):
            assert torch.equal(x[free], y[free]), step
        for env in (course, plain):
            env.reset()
        if step % 10 == 0:
            for e in free:
                assert np.array_equal(course._core.task_state(int(e)), plain._core.task_state(int(e))), (step, e)


@pytest.mark.parametrize("scene", ["heading", "target"])
def test_setter_restarts_mid_episode(asset_root, scene):
    """a second dm_set_goal_course 12 policy steps into the episode: origin at the current root, goal for the current episode time, a
    record of no interval; a count dropped to 0 keeps its goal until the environment's reset"""
    import torch
    args, rows = SCENES[scene]
    N = 4
    env = _env(asset_root, args, N)
    env.set_mode(1)   # test mode: 20 s episodes, so that no reset falls inside the test
    env.reset(True)
    env.set_goal_course(np.asarray(rows))
    for _ in range(12):
        env.step(torch.zeros(N, env.get_action_size(), device="cuda"))
    new = np.asarray(rows)[::-1].copy()
    if scene == "heading":
        new[:, 0] = np.asarray(rows)[:, 0]
    r = np.broadcast_to(new, (N,) + new.shape)
    counts = np.array([len(new)] * (N - 1) + [0])
    before = env._core.task_state(N - 1)
    env.set_goal_course(r, counts)
    rx, rz = _roots(env)
    rec = env.course_record().double().cpu().numpy()
    succ = env._core.task_params()[0][4]
    for e in range(N - 1):
        want = ref.Course(scene, new, succ).start(rx[e], rz[e], _tau(env, e))
        tk = env._core.task_state(e)
        assert np.allclose(rec[e], want, rtol=1e-5, atol=1e-5)
        if scene == "heading":
            assert (tk[3], tk[2]) == ref.heading_goal(new, _tau(env, e)) and rec[e, 2] == 0 and rec[e, 3] == 0
        else:
            assert (tk[0], tk[1]) == (rx[e] + new[0, 0], rz[e] + new[0, 1]) and rec[e, 2] == 0
    assert np.array_equal(env._core.task_state(N - 1), before)
    env.step(torch.zeros(N, env.get_action_size(), device="cuda"))
    after = env._core.task_state(N - 1)
    assert np.array_equal(after[GOAL_SLOTS[:4]], before[GOAL_SLOTS[:4]]) and after[5] == np.inf


def test_refusals_name_their_argument(asset_root):
    from deepmimic_b200.capi import MAX_COURSE_POINTS, BatchedCore, HostModel, lib
    L = lib()

    def call(core, counts, rows):
        n = np.ascontiguousarray(counts, dtype=np.int32)
        r = np.ascontiguousarray(rows, dtype=np.float64)
        rc = L.dm_set_goal_course(core.h, n.ctypes.data_as(C.POINTER(C.c_int32)), r.ctypes.data_as(C.POINTER(C.c_double)))
        return rc, L.dm_last_error().decode()

    def rows_of(pts, N=2):
        r = np.zeros((N, MAX_COURSE_POINTS, 3))
        r[:, :len(pts), :] = pts
        return r

    core = BatchedCore(HEADING, 2, asset_root, device=0)
    ok = [[0.0, 0.0, 1.0], [1.0, 0.5, 1.0]]
    assert call(core, [2, 2], rows_of(ok))[0] == 0
    for counts, pts, name in (([17, 2], ok, "count 17"), ([-1, 2], ok, "count -1"), ([2, 2], [[0, float("nan"), 1], [1, 0, 1]], "heading"),
                              ([2, 2], [[0, 0, float("inf")], [1, 0, 1]], "speed"), ([2, 2], [[0, 0, 1], [float("nan"), 0, 1]], "time"),
                              ([2, 2], [[1.0, 0, 1], [1.0, 0, 1]], "not after"), ([2, 2], [[1.0, 0, 1], [0.5, 0, 1]], "not after"),
                              ([2, 2], [[-0.1, 0, 1], [1.0, 0, 1]], "negative"), ([2, 2], [[0, 0, 1], [1, 0, -0.5]], "speed")):
        rc, err = call(core, counts, rows_of(pts))
        assert rc != 0 and "dm_set_goal_course" in err and name in err, (counts, pts, err)
    with pytest.raises(RuntimeError, match="goal course"):
        core.save_state()
    tcore = BatchedCore(TARGET, 2, asset_root, device=0)
    rc, err = call(tcore, [2, 2], rows_of([[1.0, float("inf"), 0.0], [0, 0, 0]]))
    assert rc != 0 and "dz" in err
    assert call(tcore, [2, 2], rows_of([[1.0, 0.0, float("nan")], [0, 0, 0]]))[0] == 0   # the unused value is not read
    blob = BatchedCore(TARGET, 2, asset_root, device=0).save_state()
    with pytest.raises(RuntimeError, match="goal course"):
        tcore.load_state(blob)
    for args, scene in ((["--arg_file", "args/run_humanoid3d_spinkick_args.txt"], "imitate"),
                        (MINI + ["--arg_file", "args/train_amp_strike_humanoid3d_walk_punch_args.txt"], "strike_amp")):
        rc, err = call(BatchedCore(args, 2, asset_root, device=0), [1, 1], rows_of([[0, 0, 1]]))
        assert rc != 0 and "no courses" in err and scene in err, err
    host = HostModel(HEADING, asset_root)
    rc, err = call(host, [1, 1], rows_of([[0, 0, 1]]))
    assert rc != 0 and "host-only" in err
    with pytest.raises(RuntimeError, match="no course"):
        import torch
        BatchedCore(HEADING, 2, asset_root, device=0).course_record(torch.zeros(2, 4, device="cuda"))


def test_markers_render_like_the_restatement(asset_root):
    """24 poses of random-action steps: with every radius <= 0 the marked kernel gives dm_render_poses's bytes; with markers around the
    character it matches render_marker_ref under test_render_gpu's rule (ids on >= 99.9 % of pixels and only at id boundaries, RGB within 3
    away from edges, silhouettes within 8 and at most 1 % over 3), and marker pixels carry id -3"""
    import torch
    from deepmimic_b200.capi import BatchedCore
    W, H = 240, 136
    cam = dict(yaw=0.6, pitch=0.35, distance=4.0, target_height=0.6, fov_y=0.9)
    env = _env(asset_root, HEADING, 24, seed=4)
    g = torch.Generator(device="cuda").manual_seed(1)
    for _ in range(6):
        env.step(0.3 * torch.randn(24, env.get_action_size(), device="cuda", generator=g))
    pose = env.record_pose()[0].clone()
    core = BatchedCore(HEADING, 1, asset_root, device=0)
    rng = np.random.default_rng(0)
    p = pose.double().cpu().numpy()
    mk = np.stack([p[:, 0] + rng.uniform(-1.2, 1.2, 24), rng.uniform(0.05, 1.0, 24), p[:, 2] + rng.uniform(-1.2, 1.2, 24),
                   rng.uniform(0.08, 0.4, 24)], axis=1).astype(np.float32)
    mk[::6, 3] = 0.0
    none = mk.copy()
    none[:, 3] = -np.abs(none[:, 3])
    marks, no_marks = torch.as_tensor(mk, device="cuda"), torch.as_tensor(none, device="cuda")
    torch.cuda.synchronize()   # the inputs are made on torch's stream, the renders run on the handle's
    plain = core.render_poses(pose, cam, W, H)
    off = core.render_poses(pose, cam, W, H, markers=no_marks)
    marked = core.render_poses(pose, cam, W, H, markers=marks)
    core.sync()
    assert torch.equal(off[0], plain[0]) and torch.equal(off[1], plain[1])
    rgb, ids = marked[0].cpu().numpy(), marked[1].cpu().numpy()
    char = RR.Character(asset_root, "data/characters/humanoid3d.txt")
    bad_ids = off_edge = bad_rgb = sil = sil_over3 = sil_worst = marker_px = 0
    for i in range(24):
        R, c = char.frames(p[i])
        want = MR.render_marked(char, R, c, (p[i, 0], p[i, 2]), cam, W, H, mk[i])
        diff = ids[i] != want["ids"]
        bad_ids += int(diff.sum())
        off_edge += int((diff & ~RR.near_boundary(want["ids"])).sum())
        ok = ~diff
        for k in ("shadow", "checker", "face"):
            ok &= ~RR.near_boundary(want[k])
        silhouette = ok & RR.near_boundary(want["ids"])
        err = np.abs(rgb[i].astype(np.int16) - want["rgb"].astype(np.int16)).max(axis=-1)
        bad_rgb += int((err[ok & ~silhouette] > 3).sum())
        sil += int(silhouette.sum())
        sil_over3 += int((err[silhouette] > 3).sum())
        sil_worst = max(sil_worst, int(err[silhouette].max(initial=0)))
        marker_px += int((ids[i] == MR.MARKER).sum())
        if mk[i, 3] <= 0:
            assert not (ids[i] == MR.MARKER).any()
    total = 24 * W * H
    print("markers: %d marker pixels; %d of %d pixels with another id (%d off an id boundary), %d more than 3 levels off; %d silhouette "
          "pixels, %d more than 3 levels off, worst %d" % (marker_px, bad_ids, total, off_edge, bad_rgb, sil, sil_over3, sil_worst))
    assert marker_px > 1000
    assert bad_ids <= 1e-3 * total and off_edge == 0 and bad_rgb == 0
    assert sil_worst <= 8 and sil_over3 <= 0.01 * sil


# The bounds below are twice the values measured on an H100 80GB HBM3 at 700 W (DESIGN.md section 8, "Steering task skills").
def test_pretrained_heading_policy_follows_a_course(asset_root, tmp_path):
    """run --heading_course 0:0:1.5,4:0:1.5,6:1.5708:1.5 on the reference's pretrained heading policy, 64 environments, 20 s episodes: the
    columns and the summary are written, and the policy walks the course -- mean speed error, cross-track speed and fall fraction below
    bounds of twice the measured values, and more than half the --render frames draw the goal marker (measured: every one)"""
    from deepmimic_b200 import run
    from deepmimic_b200.formats import read_table_log
    out = tmp_path / "out"
    prefix = _bundle(tmp_path, _fixture("policy_humanoid3d_amp_heading_locomotion_fp16.npz"))
    res = run.main(["--asset_root", asset_root, "--motion_file", "data/datasets/synthetic_locomotion_56.txt", "--arg_file",
                    "args/train_amp_heading_humanoid3d_locomotion_args.txt", "--model_files", prefix, "--output_path", str(out),
                    "--num_envs", "64", "--heading_course", "0:0:1.5,4:0:1.5,6:1.5708:1.5", "--render", "1", "--render_size", "160x96"])
    log = read_table_log(str(out / "run_log.txt"))
    assert np.allclose(log["Speed_Err"], res["speed_err"]) and np.allclose(log["Cross_Speed"], res["cross_speed"])
    speed, cross, fell = float(np.mean(res["speed_err"])), float(np.mean(res["cross_speed"])), float(np.mean(res["terminate"] == 1))
    print("pretrained heading policy on the course: speed error %.4f m/s, cross-track speed %.4f m/s, fall fraction %.4f, mean length %.1f" % (
        speed, cross, fell, float(np.mean(res["lengths"]))))
    assert math.isfinite(speed) and math.isfinite(cross)
    assert speed < SPEED_ERR_BOUND and cross < CROSS_SPEED_BOUND and fell <= FALL_BOUND
    from tests.test_render_cpu import read_apng
    frames, _, _ = read_apng(str(out / "render_0.png"))
    f = frames.astype(int)
    green = (f[..., 1] - f[..., 0] > 30) & (f[..., 1] - f[..., 2] > 30)   # only the marker's colour is this green
    print("frames with the marker: %d of %d" % (int(green.reshape(frames.shape[0], -1).any(axis=1).sum()), frames.shape[0]))
    assert green.reshape(frames.shape[0], -1).any(axis=1).mean() > 0.5


# measured: speed error 0.4441 m/s, cross-track speed 0.2995 m/s, 2 of 64 episodes ended by a fall (0.0312), mean length 584.0 policy steps
SPEED_ERR_BOUND, CROSS_SPEED_BOUND, FALL_BOUND = 0.89, 0.60, 0.0625
