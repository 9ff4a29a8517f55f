"""Cost of a goal course: device-timed policy steps (dm_set_action, then dm_update of 20 updates) on 4096 heading_amp environments (test
mode), a handle without a course against one whose every environment follows a four-point heading course, in alternating rounds.  Both
step the same seeded random actions from the same reset.  A separate profiled round gives dm_course_kernel's own time per launch from
torch.profiler.

    python tools/course_time.py [--num_envs 4096] [--steps 30] [--rounds 5] [--out course_time.json]

Prints the card's name, power limit and SM clocks, then per handle the median milliseconds per policy step of each round, and the course
kernel's mean time."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

ARGS = ["--motion_file", "data/datasets/test_clips_mini.txt", "--arg_file", "args/train_amp_heading_humanoid3d_locomotion_args.txt"]
COURSE = [[0.0, 0.0, 1.5], [4.0, 0.0, 1.5], [6.0, 1.5708, 1.5], [12.0, 3.1416, 1.0]]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi unavailable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num_envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from deepmimic_b200.assets import asset_root
    from deepmimic_b200.capi import MAX_COURSE_POINTS, BatchedCore
    assert torch.cuda.is_available(), "course_time needs a CUDA device"
    root, N = asset_root(), a.num_envs
    handles = {}
    for name in ("plain", "course"):
        c = BatchedCore(ARGS, N, root, device=0, seed=1)
        c.set_mode(1)
        handles[name] = c
    rows = np.zeros((N, MAX_COURSE_POINTS, 3))
    rows[:, :len(COURSE)] = COURSE
    rng = np.random.default_rng(3)
    A = handles["plain"].dims.action_size
    actions = [torch.as_tensor(0.05 * rng.standard_normal((N, A)), dtype=torch.float32, device="cuda") for _ in range(a.steps)]
    print("card: name, power limit, max SM clock, SM clock:", card(), flush=True)

    def run(c, timed):
        c.reset(True, kin_time=np.linspace(0.0, 1.2, N), max_time=np.full(N, 1e9), rot_theta=np.zeros(N))
        if c is handles["course"]:
            c.set_goal_course(np.full(N, len(COURSE), dtype=np.int32), rows)
        c.sync()
        ms = []
        st = torch.cuda.ExternalStream(c.stream())   # events on the handle's own stream bracket the policy step alone
        for i in range(a.steps):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(st); c.set_action(actions[i]); c.update(1.0 / 600.0, 20); e.record(st)
            if timed:
                torch.cuda.synchronize()
                ms.append(s.elapsed_time(e))
        c.sync()
        return ms

    res = {k: [] for k in handles}
    for rnd in range(a.rounds + 1):   # round 0 warms up both handles
        for name, c in handles.items():
            ms = run(c, True)
            if rnd > 0:
                res[name].append(float(np.median(ms)))
        if rnd > 0:
            print("round %d: %s" % (rnd, "  ".join("%s %.4f ms" % (k, v[-1]) for k, v in res.items())), flush=True)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(handles["course"], False)
        torch.cuda.synchronize()
    kern = [ev for ev in prof.key_averages() if "dm_course_kernel" in ev.key]
    course_us = (kern[0].device_time_total / kern[0].count) if kern else float("nan")
    print("dm_course_kernel: %d launches, %.2f us per launch" % (kern[0].count if kern else 0, course_us))
    out = dict(card=card(), num_envs=N, updates_per_step=20, rounds=res, median={k: float(np.median(v)) for k, v in res.items()},
               spread={k: [min(v), max(v)] for k, v in res.items()}, course_kernel_us=course_us)
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump(out, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
