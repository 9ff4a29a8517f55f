"""Device time of dm_pose_error (CUDA events, median of repeated calls) for 4096 humanoid3d and 2048 dog3d episodes of 600 frames, and the
wall time of `run` against `run --pose_error` at 4096 environments on the golden spin-kick policy.  Prints the card's name and power limit.

  python tools/pose_error_time.py [--reps 20] [--skip_run]
"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def time_kernel(args, n, T, reps):
    import torch
    from deepmimic_b200.assets import asset_root
    from deepmimic_b200.capi import BatchedCore
    core = BatchedCore(args, 1, asset_root(), device=0, seed=0)
    P = core.dims.pose_dim
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randn(T, n, P, device="cuda", generator=g)
    r = torch.randn(T, n, P, device="cuda", generator=g)
    L = torch.full((n,), T, dtype=torch.int32, device="cuda")
    lock, dtw = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
    core.pose_error(a, r, L, lock, dtw)
    core.sync()
    ms = []
    s = torch.cuda.ExternalStream(core.stream())
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        core.pose_error(a, r, L, lock, dtw)
        e1.record(s)
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    ms.sort()
    core.close()
    return ms[len(ms) // 2], ms[0], ms[-1]


def time_run(n, extra):
    from deepmimic_b200.assets import asset_root
    from tests.test_run_cpu import _bundle, _fixture
    tmp = tempfile.mkdtemp()
    prefix = _bundle(tmp, _fixture("policy_humanoid3d_spinkick_fp16.npz"))
    cmd = [sys.executable, "-m", "deepmimic_b200.run", "--asset_root", asset_root(), "--arg_file", "args/run_humanoid3d_spinkick_args.txt",
           "--model_files", prefix, "--output_path", os.path.join(tmp, "out"), "--num_envs", str(n)] + extra
    t0 = time.time()
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=REPO), capture_output=True, text=True)
    dt = time.time() - t0
    assert r.returncode == 0, r.stderr[-2000:]
    return dt, r.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--skip_run", action="store_true")
    opts = ap.parse_args()
    print("card: %s" % card())
    for name, args, n in (("humanoid3d", ["--arg_file", "args/run_humanoid3d_spinkick_args.txt"], 4096),
                          ("dog3d", ["--arg_file", "args/run_dog3d_trot_args.txt"], 2048)):
        med, lo, hi = time_kernel(args, n, 600, opts.reps)
        print("dm_pose_error %s: %d episodes x 600 frames: median %.2f ms (min %.2f, max %.2f) over %d calls" % (name, n, med, lo, hi, opts.reps))
    if not opts.skip_run:
        for rnd in range(2):
            for extra in ([], ["--pose_error"]):
                dt, out = time_run(4096, extra)
                print("run%s, 4096 environments, round %d: %.1f s wall\n  %s" % (" --pose_error" if extra else "", rnd, dt, out.replace("\n", "\n  ")))


if __name__ == "__main__":
    main()
