"""Watch a motion: play one motion file once through as an animated PNG, drawn by the device ray caster (dm_render_poses) with the character
of an arg file.  The counterpart of the reference's kin_char playback in its viewer, for the reference clips, BVH imports
(deepmimic_b200/bvh.py) and the motion files `deepmimic_b200.run --record_motion` writes.

    python -m deepmimic_b200.render --arg_file args/run_humanoid3d_spinkick_args.txt [--motion_file PATH] --output OUT.png
        [--render_size 640x360] [--camera yaw,pitch,distance,height,fov_deg] [--device 0] [--asset_root DIR]

--motion_file is read from the argument list, the command line before the arg file, as deepmimic_b200.train reads its paths.  One frame per
motion frame, each shown for the file's frame duration.  The camera follows the root: it looks at (root x, height, root z) from `distance`
metres away, at `yaw` about the vertical axis (0: from +z) and `pitch` above the horizon (radians), with a vertical field of view of
`fov_deg` degrees.  write_pose_apng is the function `deepmimic_b200.run --render` writes its episodes with."""
import argparse
import math
import os
import sys

from .capi import DEFAULT_CAMERA


def parse_size(text):
    """WxH: two integers in [16, 4096]"""
    try:
        w, h = (int(x) for x in text.lower().split("x"))
    except ValueError:
        raise argparse.ArgumentTypeError("need WxH, got %r" % text)
    if not (16 <= w <= 4096 and 16 <= h <= 4096):
        raise argparse.ArgumentTypeError("width and height must be in [16, 4096], got %r" % text)
    return w, h


def parse_camera(text):
    """yaw,pitch,distance,height,fov_deg: yaw and pitch in radians, distance > 0 and height in metres, 0 < fov_deg < 180"""
    try:
        v = [float(x) for x in text.split(",")]
    except ValueError:
        v = []
    if len(v) != 5 or not all(math.isfinite(x) for x in v):
        raise argparse.ArgumentTypeError("need five finite numbers yaw,pitch,distance,height,fov_deg, got %r" % text)
    if not v[2] > 0.0 or not 0.0 < v[4] < 180.0:
        raise argparse.ArgumentTypeError("need distance > 0 and 0 < fov_deg < 180, got %r" % text)
    return dict(yaw=v[0], pitch=v[1], distance=v[2], target_height=v[3], fov_y=math.radians(v[4]))


def add_view_options(ap):
    """--render_size and --camera, shared with deepmimic_b200.run"""
    ap.add_argument("--render_size", type=parse_size, default=(640, 360), metavar="WxH", help="frame size in pixels (default 640x360)")
    ap.add_argument("--camera", type=parse_camera, default=None, metavar="YAW,PITCH,DIST,HEIGHT,FOV_DEG",
                    help="camera tracking the root (default %s)" % ",".join("%g" % x for x in (
                        DEFAULT_CAMERA["yaw"], DEFAULT_CAMERA["pitch"], DEFAULT_CAMERA["distance"], DEFAULT_CAMERA["target_height"],
                        math.degrees(DEFAULT_CAMERA["fov_y"]))))


def write_pose_apng(core, path, poses, durations, camera=None, size=(640, 360), chunk=32, markers=None):
    """pose rows [F, pose_dim] (numpy or tensor, the dm_record_pose layout) drawn as core's character (a BatchedCore) into the animated PNG
    `path`, frame f shown for durations[f] seconds; markers [F, 4] (x, y, z, radius) adds a sphere to each frame (BatchedCore.render_poses).
    The rows are rendered and copied to the host `chunk` at a time on the handle's stream, so device memory does not grow with F; the frames
    go to the file as they arrive."""
    import torch
    width, height = size
    dev = torch.device("cuda", core.device)

    def frames():
        with torch.cuda.device(dev), torch.cuda.stream(torch.cuda.ExternalStream(core.stream(), device=dev)):
            for a in range(0, len(poses), chunk):
                rows = torch.as_tensor(poses[a:a + chunk], dtype=torch.float32).to(dev).contiguous()
                mk = None if markers is None else torch.as_tensor(markers[a:a + chunk], dtype=torch.float32).to(dev).contiguous()
                rgb, _ = core.render_poses(rows, camera, width, height, ids=False, markers=mk)
                yield from rgb.cpu().numpy()   # a copy to pageable memory: waits for the handle's stream

    from .formats import write_apng
    write_apng(path, frames(), durations)


def core_args(scene_args, asset_root, motion_file):
    """the arguments of the handle that draws `motion_file` (a resolved path): the scene arguments without the command line's --motion_file,
    so that the handle loads the arg file's own clip (only its character is used, and the simulation's loader resolves a relative path under
    the asset root only); the absolute motion file path when the arg file names no clip"""
    from .train import arg_table, first_arg
    out, skip = [], False
    for tok in scene_args:
        if tok.startswith("--"):
            skip = tok == "--motion_file"
        if not skip:
            out.append(tok)
    if not first_arg(arg_table(out, asset_root, "render"), "motion_file"):
        out = ["--motion_file", os.path.abspath(motion_file)] + out
    return out


def build_parser():
    ap = argparse.ArgumentParser(prog="python -m deepmimic_b200.render", description=__doc__.split("\n\n")[0], allow_abbrev=False)
    ap.add_argument("--output", required=True, help="the animated PNG to write")
    ap.add_argument("--asset_root", default=None, help="the reference's data / args tree (default: the bundled asset archive)")
    ap.add_argument("--device", type=int, default=0)
    add_view_options(ap)
    return ap


def main(argv=None):
    from .assets import asset_root as default_asset_root
    from .formats import read_motion
    from .train import _resolve, arg_table, first_arg
    opts, scene_args = build_parser().parse_known_args(sys.argv[1:] if argv is None else argv)
    root = opts.asset_root or default_asset_root()
    table = arg_table(scene_args, root, "render")
    motion_file = first_arg(table, "motion_file")
    if not motion_file:
        raise SystemExit("render: no --motion_file in the arguments or the arg file")
    motion_file = _resolve(root, motion_file)
    try:
        m = read_motion(motion_file)
    except (OSError, ValueError) as e:
        raise SystemExit("render: %s" % e)
    from .capi import BatchedCore
    try:
        core = BatchedCore(core_args(scene_args, root, motion_file), 1, root, device=opts.device)
    except RuntimeError as e:
        raise SystemExit("render: %s" % e)
    if m["frames"].shape[1] != core.dims.pose_dim:
        raise SystemExit("render: %s has %d values per frame, the character's pose has %d" % (motion_file, m["frames"].shape[1], core.dims.pose_dim))
    write_pose_apng(core, opts.output, m["frames"], m["durations"], opts.camera, opts.render_size)
    print("%s: %d frames of %s" % (opts.output, m["frames"].shape[0], motion_file))
    return dict(frames=m["frames"].shape[0], durations=m["durations"])


if __name__ == "__main__":
    main()
