"""Cost of the push schedule on 4096 spin-kick environments (train mode, placement by contact load on, random actions, episode limits of
1-2.5 s so that episodes end and restart):
  * the scheduler kernel alone: its device time per launch from torch.profiler (CUDA activities), over the dm_update calls of a scheduled
    handle, in a run of its own;
  * the policy-step rate with the schedule off and on: two handles in alternating rounds, each round `--steps` policy steps of set_action,
    dm_update (20 updates), observe and reset of the finished episodes, timed by events on the handle's stream.

    python tools/push_schedule_time.py [--num_envs 4096] [--steps 60] [--rounds 5] [--out push_schedule_time.json]

Prints the card's name, power limit and SM clocks, the kernel's mean / median time per launch and per round the rates of both handles."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.push_time import card  # noqa: E402

SCHED = dict(bodies=[0, 2], force=(100.0, 600.0), duration=(0.1, 0.3), gap=(1.0, 3.0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num_envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from deepmimic_b200.assets import asset_root
    from deepmimic_b200.capi import BatchedCore
    assert torch.cuda.is_available(), "push_schedule_time needs a CUDA device"
    root, N = asset_root(), a.num_envs
    args = ["--arg_file", "args/train_humanoid3d_spinkick_args.txt"]
    handles = {}
    for name in ("off", "on"):
        c = BatchedCore(args, N, root, device=0, seed=1)
        c.set_episode_limit(1.0, 2.5)
        if name == "on":
            c.set_push_schedule(**SCHED)
        handles[name] = c
    A = handles["off"].dims.action_size
    rng = np.random.default_rng(3)
    actions = [torch.as_tensor(0.2 * rng.standard_normal((N, A)), dtype=torch.float32, device="cuda") for _ in range(a.steps)]
    obs = torch.empty(N, handles["off"].dims.state_size, device="cuda")
    rew = torch.empty(N, device="cuda")
    print("card: name, power limit, max SM clock, SM clock:", card(), flush=True)

    def steps(c):
        for x in actions:
            c.set_action(x); c.update(1.0 / 600.0, 20); c.observe(obs, rew); c.reset(False)

    rates = {k: [] for k in handles}
    for rnd in range(a.rounds + 1):   # round 0 warms up both handles
        for name, c in handles.items():
            c.reset(True)
            c.sync()
            st = torch.cuda.ExternalStream(c.stream())
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(st); steps(c); e.record(st)
            torch.cuda.synchronize()
            if rnd > 0:
                rates[name].append(N * a.steps / (s.elapsed_time(e) * 1e-3))
        if rnd > 0:
            print("round %d: policy steps/s off %.4g M, on %.4g M" % (rnd, rates["off"][-1] * 1e-6, rates["on"][-1] * 1e-6), flush=True)
    # the kernel alone, profiled in a run of its own after the timed rounds
    c = handles["on"]
    c.reset(True); c.sync()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        steps(c)
        c.sync()
    us = [ev.device_time_total for ev in prof.events() if "dm_push_schedule_kernel" in ev.name]
    print(prof.key_averages().table(sort_by="device_time_total", row_limit=12))
    assert len(us) == a.steps, "expected one scheduler launch per dm_update, found %d" % len(us)
    out = dict(card=card(), num_envs=N, steps_per_round=a.steps, schedule=SCHED, kernel_us=dict(mean=float(np.mean(us)), median=float(np.median(us)),
               min=float(np.min(us)), max=float(np.max(us)), launches=len(us)),
               rates=rates, median_rate={k: float(np.median(v)) for k, v in rates.items()}, spread={k: [min(v), max(v)] for k, v in rates.items()})
    print("dm_push_schedule_kernel: mean %.2f us, median %.2f us per launch (%d launches)" % (out["kernel_us"]["mean"], out["kernel_us"]["median"], len(us)))
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump(out, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
