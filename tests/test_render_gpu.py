"""The device renderer (dm_render_poses) on the GPU: against the float64 reference (tests/render_ref.py) on the oracle's collision frames,
batch and repeat invariance, no effect on the simulation, `run --render` and the render command, and the C ABI's refusals."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import contact_states as CS
from tests import render_ref as RR
from tests.oracle_binding import Oracle
from tests.parity_util import random_policy_action
from tests.test_render_cpu import read_apng
from tests.test_run_cpu import _bundle, _fixture

pytestmark = pytest.mark.gpu
CAMERAS = [dict(yaw=0.6, pitch=0.25, distance=4.0, target_height=0.9, fov_y=0.7853981633974483),
           dict(yaw=2.4, pitch=0.7, distance=2.5, target_height=0.3, fov_y=1.0)]


def _states(orc, asset_root, ch):
    """every 8th state of the contact library (links on and in the ground) and 8 random-action policy steps from a reset"""
    snaps = [s.snap for s in CS.build(orc, asset_root, ch)[::8]]
    off, scale, lo, hi = orc.action_statics()
    rng = np.random.default_rng(5)
    orc.reset(0.2, 0.5, 20.0)
    for _ in range(8):
        orc.set_action(random_policy_action(rng, off, scale, lo, hi))
        for _ in range(20):
            orc.update(CS.DT)
        snaps.append(orc.get_snapshot())
    return snaps


@pytest.mark.parametrize("ch", ["humanoid3d", "dog3d"])
def test_device_render_matches_the_reference(asset_root, ch):
    """the same states in the oracle and the device (set_snapshot, then record_pose and render_poses); the reference draws the oracle's
    collision frames.  Hit ids agree on >= 99.9 % of the pixels and every disagreeing pixel lies within one pixel of an id boundary of the
    reference.  Where the ids agree, RGB is within 3 levels except within one pixel of a shadow edge, a checker-cell edge or an edge between
    two faces of a box of the reference, where the shading jumps and the float32 ray may fall on the other side.  Silhouette pixels (within
    one pixel of an id boundary, away from those edges), where the normal turns to grazing, stay in the check with a bound of their own: none
    more than 8 levels off and at most 1 % of them more than 3.  Measured on an H100 80GB HBM3 at 700 W, 23 views of 320 x 180 per character
    and camera: humanoid3d 7 and 4, dog3d 6 and 1 pixels with another id, none away from an id boundary; no pixel away from the edges more
    than 3 levels off; of 1582 / 1974 (humanoid3d) and 937 / 1393 (dog3d) silhouette pixels, one (humanoid3d, first camera) 4 levels and one
    3 levels off, every other within 1."""
    import torch
    from deepmimic_b200.capi import BatchedCore
    W, H = 320, 180
    orc = Oracle(CS.CHARS[ch]["args"], asset_root)
    char = RR.Character(asset_root, CS.CHARS[ch]["char"])
    snaps = _states(orc, asset_root, ch)
    core = BatchedCore(CS.CHARS[ch]["args"], len(snaps), asset_root, device=0, seed=1)
    for i, s in enumerate(snaps):
        core.set_snapshot(i, s)
    pose = torch.empty(len(snaps), core.dims.pose_dim, device="cuda")
    core.record_pose(pose, None)
    for cam in CAMERAS:
        rgb, ids = core.render_poses(pose, cam, W, H)
        core.sync()
        rgb, ids = rgb.cpu().numpy(), ids.cpu().numpy()
        bad_ids = bad_rgb = off_edge = total = sil = sil_over3 = sil_worst = 0
        for i, s in enumerate(snaps):
            orc.set_snapshot(s)
            B, P = orc.collider_frames()
            root = orc.get_pose()[0]
            ref = RR.render(char, B, P / CS.SCALE, (root[0], root[2]), cam, W, H)
            diff = ids[i] != ref["ids"]
            bad_ids += int(diff.sum())
            off_edge += int((diff & ~RR.near_boundary(ref["ids"])).sum())
            ok = ~diff
            for k in ("shadow", "checker", "face"):
                ok &= ~RR.near_boundary(ref[k])
            silhouette = ok & RR.near_boundary(ref["ids"])
            err = np.abs(rgb[i].astype(np.int16) - ref["rgb"].astype(np.int16)).max(axis=-1)
            bad_rgb += int((err[ok & ~silhouette] > 3).sum())
            sil += int(silhouette.sum())
            sil_over3 += int((err[silhouette] > 3).sum())
            sil_worst = max(sil_worst, int(err[silhouette].max(initial=0)))
            total += W * H
        print("%s camera %s: %d of %d pixels with another id (%d off an id boundary), %d agreeing pixels more than 3 levels off; "
              "%d silhouette pixels, %d more than 3 levels off, worst %d" % (ch, cam, bad_ids, total, off_edge, bad_rgb, sil, sil_over3, sil_worst))
        assert bad_ids <= 1e-3 * total and off_edge == 0 and bad_rgb == 0
        assert sil_worst <= 8 and sil_over3 <= 0.01 * sil


def test_views_render_the_same_alone_in_a_batch_and_again(asset_root):
    import torch
    from deepmimic_b200.capi import BatchedCore
    args = CS.CHARS["humanoid3d"]["args"]
    core = BatchedCore(args, 64, asset_root, device=0, seed=2)
    core.reset(True)
    pose = torch.empty(64, core.dims.pose_dim, device="cuda")
    core.record_pose(pose, None)
    pose[:, 0] += torch.linspace(-3, 3, 64, device="cuda")   # 64 different views
    batch = core.render_poses(pose, None, 200, 120)
    again = core.render_poses(pose, None, 200, 120)
    one = BatchedCore(args, 1, asset_root, device=0, seed=2)
    for v in (0, 17, 63):
        alone = one.render_poses(pose[v:v + 1].contiguous(), None, 200, 120)
        one.sync(); core.sync()
        for a, b, c in zip(alone, batch, again):
            assert torch.equal(a[0], b[v]) and torch.equal(b[v], c[v])
    assert torch.equal(batch[0], again[0]) and torch.equal(batch[1], again[1])
    ids_only = core.render_poses(pose, None, 200, 120, rgb=False)
    core.sync()
    assert ids_only[0] is None and torch.equal(ids_only[1], batch[1])


def test_render_leaves_the_simulation_alone(asset_root):
    """a rollout that renders every policy step, without a host synchronisation, gives bit-identical observations, rewards, flags and
    state_dict() to one that never renders"""
    import torch
    from deepmimic_b200.env import DeepMimicBatchEnv
    args = ["--arg_file", "args/train_humanoid3d_spinkick_args.txt"]
    runs = []
    for render in (False, True):
        env = DeepMimicBatchEnv(args, 48, asset_root, device=0, seed=7)
        g = torch.Generator(device="cuda").manual_seed(3)
        rec = []
        for step in range(12):
            a = 0.3 * torch.randn(env.num_envs, env.get_action_size(), device="cuda", generator=g)
            env.set_action(a)
            env.update(env.UPDATE_DT, env.get_updates_per_action())
            if render:   # any host synchronisation inside render() raises
                torch.cuda.set_sync_debug_mode("error")
                try:
                    rgb, ids = env.render(env_ids=[0, 5, 47] if step % 2 else None, width=64, height=48)
                finally:
                    torch.cuda.set_sync_debug_mode("default")
                assert rgb.shape[0] == (3 if step % 2 else 48)
            rec += [env.record_state().clone(), env.calc_reward().clone(), env._refresh_flags().clone()]
            env.reset()
        torch.cuda.synchronize()
        runs.append((rec, env.state_dict()["blob"]))
    for a, b in zip(runs[0][0], runs[1][0]):
        assert torch.equal(a, b)
    assert torch.equal(runs[0][1], runs[1][1])


def test_run_render_writes_the_episodes(asset_root, tmp_path, monkeypatch):
    """run --render 2: two animated PNGs of length + 1 frames at the policy step duration, frame 0 = render_poses of the first recorded pose"""
    import torch
    from deepmimic_b200 import render as rd
    from deepmimic_b200 import run
    from deepmimic_b200.capi import BatchedCore
    from deepmimic_b200.formats import read_table_log
    seen = {}
    real = rd.write_pose_apng

    def spy(core, path, poses, durations, camera=None, size=(640, 360), chunk=32):
        seen[path] = np.array(poses)
        return real(core, path, poses, durations, camera, size, chunk)

    monkeypatch.setattr(rd, "write_pose_apng", spy)
    args = ["--arg_file", "args/run_humanoid3d_spinkick_args.txt"]
    out = tmp_path / "out"
    run.main(["--asset_root", asset_root] + args + ["--model_files", _bundle(tmp_path, _fixture("policy_humanoid3d_spinkick_fp16.npz")),
                                                    "--output_path", str(out), "--num_envs", "8", "--render", "2", "--episode_time", "2",
                                                    "--render_size", "160x96"])
    log = read_table_log(str(out / "run_log.txt"))
    assert not (out / "motion_0.txt").exists() and not (out / "render_2.png").exists()
    core = BatchedCore(args, 1, asset_root, device=0)
    for e in range(2):
        path = str(out / ("render_%d.png" % e))
        frames, delays, _ = read_apng(path)
        assert frames.shape == (int(log["Length"][e]) + 1, 96, 160, 3)
        assert all(abs(n / d - 1 / 30) < 1e-9 for n, d in delays)
        rgb, _ = core.render_poses(torch.as_tensor(seen[path][:1], dtype=torch.float32, device="cuda"), None, 160, 96, ids=False)
        core.sync()
        assert np.array_equal(frames[0], rgb[0].cpu().numpy())


def test_render_command_plays_a_motion_file(asset_root, tmp_path):
    from deepmimic_b200 import render as rd
    from deepmimic_b200.formats import read_motion
    out = str(tmp_path / "spinkick.png")
    rd.main(["--asset_root", asset_root, "--arg_file", "args/run_humanoid3d_spinkick_args.txt", "--motion_file",
             "data/motions/humanoid3d_spinkick.txt", "--output", out, "--render_size", "128x80"])
    m = read_motion(os.path.join(asset_root, "data/motions/humanoid3d_spinkick.txt"))
    frames, delays, _ = read_apng(out)
    assert frames.shape == (m["frames"].shape[0], 80, 128, 3)
    for (n, d), want in zip(delays, m["durations"]):
        assert abs(n / d - want) < 1e-6
    assert (frames[0] != frames[-1]).any()


def test_render_command_reads_motion_files_relative_to_the_working_directory(asset_root, tmp_path, monkeypatch):
    """a motion file written where `run` writes them (output/motion_<env>.txt under the working directory) plays by its relative path, and a
    motion of another character is refused by the command, naming the frame size"""
    from deepmimic_b200 import render as rd
    from deepmimic_b200.formats import read_motion, write_motion
    monkeypatch.chdir(tmp_path)
    os.makedirs("output")
    clip = read_motion(os.path.join(asset_root, "data/motions/humanoid3d_spinkick.txt"))["frames"][:12]
    write_motion("output/motion_0.txt", clip, [1 / 30] * 12, loop="none")
    args = ["--asset_root", asset_root, "--arg_file", "args/run_humanoid3d_spinkick_args.txt", "--render_size", "64x48"]
    rd.main(args + ["--motion_file", "output/motion_0.txt", "--output", "output/motion_0.png"])
    frames, delays, _ = read_apng("output/motion_0.png")
    assert frames.shape == (12, 48, 64, 3) and delays[0] == (1, 30)
    dog = read_motion(os.path.join(asset_root, "data/motions/dog3d_trot.txt"))
    write_motion("output/dog.txt", dog["frames"], dog["durations"], loop="none")
    with pytest.raises(SystemExit, match="values per frame"):
        rd.main(args + ["--motion_file", "output/dog.txt", "--output", "output/dog.png"])


def test_c_abi_refuses_bad_arguments_by_name(asset_root):
    import torch
    from deepmimic_b200.capi import BatchedCore, HostModel, camera_struct, lib
    L = lib()
    args = CS.CHARS["humanoid3d"]["args"]
    core = BatchedCore(args, 1, asset_root, device=0)
    pose = torch.zeros(2, core.dims.pose_dim, device="cuda")
    pose[:, 3] = 1.0
    rgb = torch.empty(2, 64, 64, 3, dtype=torch.uint8, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())

    def call(h=core.h, n=2, pose_=p(pose), cam=None, w=64, hh=64, out=p(rgb), ids=None):
        c = camera_struct(cam)
        rc = L.dm_render_poses(h, n, pose_, C.byref(c), w, hh, out, ids)
        return rc, L.dm_last_error().decode()

    assert call()[0] == 0
    host = HostModel(args, asset_root)
    for kw, name in ((dict(h=host.h), "host-only"), (dict(n=0), "n_views"), (dict(n=65536), "n_views"), (dict(w=15), "width"),
                     (dict(w=4097), "width"), (dict(hh=8), "height"), (dict(pose_=None), "d_pose"), (dict(out=None), "d_rgb and d_ids"),
                     (dict(cam=dict(yaw=float("nan"))), "yaw"), (dict(cam=dict(pitch=float("inf"))), "pitch"),
                     (dict(cam=dict(target_height=float("nan"))), "target_height"), (dict(cam=dict(distance=0.0)), "distance"),
                     (dict(cam=dict(fov_y=0.0)), "fov_y"), (dict(cam=dict(fov_y=3.2)), "fov_y")):
        rc, err = call(**kw)
        assert rc != 0 and name in err, (kw, err)
    core.sync()
