"""The renderer without a device: the float64 reference (tests/render_ref.py) against the oracle's collider frames and known answers, the
animated PNG writer read back by a standard-library reader, the options of `run --render` and of the render command, and the render kernel's
resources as ptxas reports them."""
import os
import struct
import types
import zlib

import numpy as np
import pytest

from deepmimic_b200 import render as rd
from deepmimic_b200 import run
from deepmimic_b200.formats import write_apng
from tests import contact_states as CS
from tests import render_ref as RR
from tests.oracle_binding import Oracle
from tests.parity_util import random_policy_action

PNG_SIG = b"\x89PNG\r\n\x1a\n"


def read_apng(path):
    """(frames uint8 [T, H, W, 3], delays [(num, den)] * T, chunk types in file order) of an RGB8 animated PNG written without filters other
    than type 0; asserts every CRC, the chunk order, contiguous sequence numbers and the acTL frame count"""
    import binascii
    data = open(path, "rb").read()
    assert data[:8] == PNG_SIG
    pos, chunks = 8, []
    while pos < len(data):
        n, = struct.unpack(">I", data[pos:pos + 4])
        kind, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        crc, = struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])
        assert crc == binascii.crc32(kind + body) & 0xFFFFFFFF, kind
        chunks.append((kind, body))
        pos += 12 + n
    kinds = [k for k, _ in chunks]
    assert kinds[0] == b"IHDR" and kinds[1] == b"acTL" and kinds[2] == b"fcTL" and kinds[3] == b"IDAT" and kinds[-1] == b"IEND"
    W, H, depth, ctype, comp, filt, inter = struct.unpack(">IIBBBBB", chunks[0][1])
    assert (depth, ctype, comp, filt, inter) == (8, 2, 0, 0, 0)
    nframes, plays = struct.unpack(">II", chunks[1][1])
    frames, delays, seq, cur = [], [], 0, None

    def decode(buf):
        raw = np.frombuffer(zlib.decompress(buf), dtype=np.uint8).reshape(H, 1 + 3 * W)
        assert (raw[:, 0] == 0).all()
        return raw[:, 1:].reshape(H, W, 3)

    for kind, body in chunks[2:-1]:
        if kind == b"fcTL":
            s, w, h, x, y, dn, dd, dispose, blend = struct.unpack(">IIIIIHHBB", body)
            assert s == seq and (w, h, x, y) == (W, H, 0, 0)
            seq += 1
            delays.append((dn, dd))
            cur = kind
        elif kind == b"IDAT":
            assert len(frames) == 0 and cur == b"fcTL"
            frames.append(decode(body))
            cur = kind
        elif kind == b"fdAT":
            s, = struct.unpack(">I", body[:4])
            assert s == seq and cur == b"fcTL"
            seq += 1
            frames.append(decode(body[4:]))
            cur = kind
        else:
            raise AssertionError("unexpected chunk %r" % kind)
    assert nframes == len(frames) == len(delays)
    return np.stack(frames), delays, kinds


# ---- forward kinematics of pose rows against the oracle's collision frames

@pytest.mark.parametrize("ch", ["humanoid3d", "dog3d"])
def test_pose_row_frames_match_the_oracles_collider_frames(asset_root, ch):
    """every state of the contact library and 24 random-action policy steps from three reset times: the reference's frames of the oracle's
    pose row (BuildPose) equal the collision pass's frames (divided by the world scale) to 1e-5 m and 1e-5 in every rotation entry"""
    orc = Oracle(CS.CHARS[ch]["args"], asset_root)
    char = RR.Character(asset_root, CS.CHARS[ch]["char"])
    assert char.pose_dim == orc.pose_dim
    snaps = [s.snap for s in CS.build(orc, asset_root, ch)]
    off, scale, lo, hi = orc.action_statics()
    rng = np.random.default_rng(3)
    for t0 in (0.0, 0.4, 0.9):
        orc.reset(t0, 0.3, 20.0)
        for _ in range(8):
            orc.set_action(random_policy_action(rng, off, scale, lo, hi))
            for _ in range(20):
                orc.update(CS.DT)
            snaps.append(orc.get_snapshot())
    worst_p = worst_r = 0.0
    for s in snaps:
        orc.set_snapshot(s)
        B, P = orc.collider_frames()
        R, c = char.frames(orc.get_pose()[0])
        worst_p, worst_r = max(worst_p, np.abs(c - P / CS.SCALE).max()), max(worst_r, np.abs(R - B).max())
    print("%s: %d states, worst |dc| %.3g m, |dR| %.3g" % (ch, len(snaps), worst_p, worst_r))
    assert worst_p < 1e-5 and worst_r < 1e-5
    if ch == "dog3d":   # the dog's quarter-turn body frames (neck, tail) are among the links checked
        assert sum(abs(abs(z) - 1.5708) < 1e-6 for z in (np.arctan2(R[1, 0], R[0, 0]) for R in char.body_rot)) == 3


# ---- known answers of the reference renderer

def _one_shape(shape, he):
    return types.SimpleNamespace(n=1, shape=[shape], he=[np.asarray(he, dtype=np.float64)])


NO_SHAPES = types.SimpleNamespace(n=0, shape=[], he=[])


def test_sphere_at_the_look_at_point_covers_the_centre_pixel():
    cam = dict(yaw=0.7, pitch=0.3, distance=4.0, target_height=1.1, fov_y=0.8)
    out = RR.render(_one_shape(RR.SPHERE, [0.05, 0, 0]), np.eye(3)[None], np.array([[0.4, 1.1, -0.2]]), (0.4, -0.2), cam, 65, 49)
    assert out["ids"][24, 32] == 0
    assert (out["ids"] == 0).sum() < 20   # a small disc, not the frame


def test_box_silhouette_columns_match_the_projection():
    """seen head-on (yaw 0, pitch 0) a box's centre row covers the columns whose ray slope is within its front face: |sx| <= a / (D - c)"""
    W, H, D, a, b, c = 101, 41, 5.0, 0.3, 0.2, 0.25
    cam = dict(yaw=0.0, pitch=0.0, distance=D, target_height=1.0, fov_y=0.6)
    out = RR.render(_one_shape(RR.BOX, [a, b, c]), np.eye(3)[None], np.array([[0.0, 1.0, 0.0]]), (0.0, 0.0), cam, W, H)
    tx = np.tan(0.3) * W / H
    sx = (2.0 * (np.arange(W) + 0.5) / W - 1.0) * tx
    want = np.where(np.abs(sx) <= a / (D - c), 0, -1)
    assert np.min(np.abs(np.abs(sx) - a / (D - c))) > 1e-3   # no column on the edge
    assert (out["ids"][H // 2] == want).all()


def test_checker_colour_of_a_ground_pixel():
    """the centre ray hits the look-at point on the ground: cell (0, 0) is the light grey, cell (1, 0) the dark one, each lit by the ambient
    term and the sun at n . light = 2 / sqrt(6): 0.62 * (0.35 + 0.65 * 0.81650) = 0.54605 -> 139, 0.50 * 0.88072 = 0.44036 -> 112"""
    for x, want in ((0.3, 139), (1.3, 112)):
        cam = dict(yaw=0.2, pitch=0.9, distance=3.0, target_height=0.0, fov_y=0.8)
        out = RR.render(NO_SHAPES, np.zeros((0, 3, 3)), np.zeros((0, 3)), (x, 0.2), cam, 33, 33)
        assert out["ids"][16, 16] == RR.GROUND
        assert (out["rgb"][16, 16] == want).all(), out["rgb"][16, 16]


def test_shadow_darkens_by_the_ambient_share():
    """a sphere on the light's ray above the look-at point shadows it: the pixel drops from base * (0.35 + 0.65 * L.y) to base * 0.35"""
    q = np.array([0.3, 0.0, 0.2])
    cam = dict(yaw=np.pi + np.pi / 4, pitch=0.7, distance=3.0, target_height=0.0, fov_y=0.8)
    lit = RR.render(NO_SHAPES, np.zeros((0, 3, 3)), np.zeros((0, 3)), (q[0], q[2]), cam, 33, 33)
    dark = RR.render(_one_shape(RR.SPHERE, [0.2, 0, 0]), np.eye(3)[None], (q + 1.0 * RR.LIGHT)[None], (q[0], q[2]), cam, 33, 33)
    assert dark["ids"][16, 16] == RR.GROUND and dark["shadow"][16, 16] and not lit["shadow"][16, 16]
    assert (lit["rgb"][16, 16] == round(255 * 0.62 * (0.35 + 0.65 * 2 / np.sqrt(6)))).all()
    assert (dark["rgb"][16, 16] == round(255 * 0.62 * 0.35)).all()


# ---- the animated PNG writer

def test_apng_round_trip(tmp_path):
    rng = np.random.default_rng(0)
    frames = rng.integers(0, 256, (5, 17, 23, 3), dtype=np.uint8)
    durations = [1 / 30, 0.05, 0.0333333, 0.1, 0.0]
    path = str(tmp_path / "a.png")
    write_apng(path, frames, durations)
    got, delays, kinds = read_apng(path)
    assert np.array_equal(got, frames)
    assert kinds == [b"IHDR", b"acTL", b"fcTL", b"IDAT"] + [b"fcTL", b"fdAT"] * 4 + [b"IEND"]
    assert delays[0] == (1, 30) and delays[1] == (1, 20) and delays[4][0] == 0
    for (n, d), want in zip(delays, durations):
        assert abs(n / d - want) < 1e-6
    write_apng(path, iter(list(frames)), durations)   # frames consumed one at a time give the same file
    assert np.array_equal(read_apng(path)[0], frames)


def test_apng_refusals(tmp_path):
    p = str(tmp_path / "a.png")
    f = np.zeros((2, 16, 16, 3), dtype=np.uint8)
    with pytest.raises(ValueError):
        write_apng(p, f, [0.1])
    with pytest.raises(ValueError):
        write_apng(p, f, [0.1, 0.1, 0.1])
    with pytest.raises(ValueError):
        write_apng(p, f.astype(np.float32), [0.1, 0.1])
    with pytest.raises(ValueError):
        write_apng(p, f, [0.1, float("nan")])
    with pytest.raises(ValueError):
        write_apng(p, f, [0.1, 1e6])


# ---- options

def test_run_render_options():
    opts, rest = run.build_parser().parse_known_args(["--arg_file", "x", "--render", "2", "--render_size", "320x200", "--camera", "0.5,0.2,3,1,60"])
    assert opts.render == 2 and opts.render_size == (320, 200) and rest == ["--arg_file", "x"]
    assert opts.camera == dict(yaw=0.5, pitch=0.2, distance=3.0, target_height=1.0, fov_y=np.radians(60.0))
    opts, _ = run.build_parser().parse_known_args([])
    assert opts.render == 0 and opts.render_size == (640, 360) and opts.camera is None
    for bad in (["--render_size", "8x8"], ["--render_size", "640"], ["--render_size", "5000x100"], ["--camera", "0,0,0,1,60"],
                ["--camera", "0,0,3,1,180"], ["--camera", "0,0,3,1"], ["--camera", "0,nan,3,1,60"]):
        with pytest.raises(SystemExit):
            run.build_parser().parse_known_args(bad)


def test_run_refuses_more_renders_than_environments(asset_root):
    with pytest.raises(SystemExit, match="--render"):
        run.main(["--asset_root", asset_root, "--arg_file", "args/run_humanoid3d_spinkick_args.txt", "--num_envs", "2", "--render", "3"])


def test_render_command_options_and_refusals(asset_root, tmp_path):
    opts, rest = rd.build_parser().parse_known_args(["--arg_file", "a", "--output", "o.png", "--motion_file", "m.txt", "--camera", "1,0.1,2,0.5,40"])
    assert opts.output == "o.png" and rest == ["--arg_file", "a", "--motion_file", "m.txt"] and opts.camera["fov_y"] == np.radians(40.0)
    with pytest.raises(SystemExit):   # --output is required
        rd.build_parser().parse_known_args(["--arg_file", "a"])
    with pytest.raises(SystemExit, match="render: "):
        rd.main(["--asset_root", asset_root, "--arg_file", "args/run_humanoid3d_spinkick_args.txt", "--output", str(tmp_path / "o.png"),
                 "--motion_file", str(tmp_path / "missing.txt")])
    bad = tmp_path / "bad.txt"
    bad.write_text('{"Loop": "none", "Frames": []}')
    with pytest.raises(SystemExit, match="render: "):
        rd.main(["--asset_root", asset_root, "--arg_file", "args/run_humanoid3d_spinkick_args.txt", "--output", str(tmp_path / "o.png"),
                 "--motion_file", str(bad)])


def test_render_handle_arguments_leave_the_motion_file_to_the_command(asset_root, tmp_path, monkeypatch):
    """the handle that draws a motion file loads the arg file's own clip, since the simulation's loader resolves a relative --motion_file under
    the asset root only; the command line's --motion_file is dropped (with its values), and an absolute path stands in where the arg file
    names no clip.  The arguments load through the host loaders from any working directory."""
    from deepmimic_b200.capi import HostModel
    from deepmimic_b200.formats import read_motion, write_motion
    monkeypatch.chdir(tmp_path)
    os.makedirs("output")
    m = read_motion(os.path.join(asset_root, "data/motions/humanoid3d_spinkick.txt"))
    write_motion("output/motion_0.txt", m["frames"][:5], [1 / 30] * 5, loop="none")
    args = ["--motion_file", "output/motion_0.txt", "--arg_file", "args/run_humanoid3d_spinkick_args.txt", "--num_sim_substeps", "2"]
    with pytest.raises(RuntimeError, match="cannot open JSON file"):   # what the handle would get with the command line as it stands
        HostModel(args, asset_root)
    got = rd.core_args(args, asset_root, "output/motion_0.txt")
    assert got == ["--arg_file", "args/run_humanoid3d_spinkick_args.txt", "--num_sim_substeps", "2"]
    assert HostModel(got, asset_root).dims.pose_dim == 43
    assert rd.core_args(["--motion_file", "output/motion_0.txt", "--scene", "imitate"], asset_root, "output/motion_0.txt") == [
        "--motion_file", str(tmp_path / "output" / "motion_0.txt"), "--scene", "imitate"]


# ---- resources

def test_render_kernel_keeps_out_of_local_memory(tmp_path):
    from tests.test_step_resources_cpu import nvcc, ptxas_report
    if nvcc() is None:
        pytest.skip("needs nvcc")
    rep = ptxas_report(os.path.join("kernels", "dm_render.cu"), str(tmp_path))
    (entry,) = [e for e in rep if "dm_render_kernel" in e]
    for name, stack, stores, loads in rep[entry]:
        assert stack == 0 and stores == 0 and loads == 0, (name, stack, stores, loads)
