"""Cost of the device renderer: dm_render_poses timed with CUDA events after warm-up (64 views at 640 x 360 and 4 views at 1280 x 720,
humanoid3d and dog3d), and the host cost of `run --render` for one 20 s episode (601 frames at 640 x 360), split into rendering with the copy
to the host and the animated PNG encoding, against write_pose_apng end to end, in alternating rounds.  Prints the card's name and power
limit with the results.

  python tools/render_time.py [--launches 200] [--rounds 3] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

CHARS = {"humanoid3d": ["--arg_file", "args/run_humanoid3d_spinkick_args.txt"], "dog3d": ["--arg_file", "args/run_dog3d_trot_args.txt"]}
CONFIGS = [(64, 640, 360), (4, 1280, 720)]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3, help="rounds of the host-cost measurement")
    ap.add_argument("--out", default=None, help="also write the results as render_time.json here")
    opts = ap.parse_args()
    import numpy as np
    import torch
    from deepmimic_b200.assets import asset_root
    from deepmimic_b200.capi import BatchedCore
    from deepmimic_b200.formats import write_apng
    from deepmimic_b200.render import write_pose_apng
    root = asset_root()
    res = dict(card=card(), kernel=[], run_render={})
    print("card: %s" % res["card"])
    for ch, args in CHARS.items():
        core = BatchedCore(args, 64, root, device=0, seed=1)
        pose = torch.empty(64, core.dims.pose_dim, device="cuda")
        core.record_pose(pose, None)
        stream = torch.cuda.ExternalStream(core.stream())
        for V, W, H in CONFIGS:
            rows = pose[:V].contiguous()
            rgb = torch.empty(V, H, W, 3, dtype=torch.uint8, device="cuda")
            ids = torch.empty(V, H, W, dtype=torch.int16, device="cuda")
            for _ in range(10):
                core.render_poses(rows, None, W, H, rgb=rgb, ids=ids)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(opts.launches):
                core.render_poses(rows, None, W, H, rgb=rgb, ids=ids)
            e1.record(stream)
            e1.synchronize()
            ms = e0.elapsed_time(e1) / opts.launches
            r = dict(character=ch, views=V, width=W, height=H, ms_per_launch=ms, mpix_per_s=V * W * H / ms / 1e3)
            res["kernel"].append(r)
            print("%-10s %2d views %4d x %3d: %.3f ms per launch, %.0f Mpixel/s" % (ch, V, W, H, ms, r["mpix_per_s"]))
    # run --render's host side for one 20 s episode: the clip's poses replayed at the policy step (601 frames)
    core = BatchedCore(CHARS["humanoid3d"], 601, root, device=0, seed=1)
    core.reset(True, kin_time=np.arange(601) / 30.0, max_time=np.full(601, 30.0), rot_theta=np.zeros(601))
    pose = torch.empty(601, core.dims.pose_dim, device="cuda")
    core.record_pose(pose, None)
    core.sync()
    frames_host = pose.double().cpu().numpy()
    dev = torch.device("cuda", 0)

    def render_chunks():
        with torch.cuda.stream(torch.cuda.ExternalStream(core.stream(), device=dev)):
            return [core.render_poses(torch.as_tensor(frames_host[a:a + 32], dtype=torch.float32).to(dev).contiguous(), None, 640, 360,
                                      ids=False)[0].cpu().numpy() for a in range(0, 601, 32)]

    rounds = []
    with tempfile.TemporaryDirectory() as tmp:
        write_pose_apng(core, os.path.join(tmp, "warm.png"), frames_host[:32], [1 / 30] * 32)
        for _ in range(opts.rounds):   # the three parts alternate within a round; the encoder reads the 32-frame chunks, as write_pose_apng does
            t0 = time.perf_counter()
            chunks = render_chunks()
            t1 = time.perf_counter()
            write_apng(os.path.join(tmp, "enc.png"), (f for c in chunks for f in c), [1 / 30] * 601)
            t2 = time.perf_counter()
            write_pose_apng(core, os.path.join(tmp, "all.png"), frames_host, [1 / 30] * 601)
            t3 = time.perf_counter()
            rounds.append(dict(render_and_copy_s=t1 - t0, encode_s=t2 - t1, write_pose_apng_s=t3 - t2))
            print("run --render, one 601-frame 640 x 360 episode: render + copy %.3f s, APNG encoding %.3f s, write_pose_apng end to end %.3f s"
                  % (t1 - t0, t2 - t1, t3 - t2))
        size = os.path.getsize(os.path.join(tmp, "all.png"))
    res["run_render"] = dict(frames=601, width=640, height=360, rounds=rounds, file_bytes=size)
    print("APNG file %.1f MB" % (size / 1e6))
    if opts.out:
        os.makedirs(opts.out, exist_ok=True)
        json.dump(res, open(os.path.join(opts.out, "render_time.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
