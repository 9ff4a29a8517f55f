"""Cost of the step kernel's latency instantiation: device-timed dm_update launches of 20 updates on 4096 spin-kick environments (test mode,
placement by contact load on), for four handles in alternating rounds -- a plain handle, a dynamics handle with unit factors, a latency
handle with every delay 0, and a latency handle with delays drawn over [0, 19] updates.  Every handle steps the same seeded random actions
from the same reset.

    python tools/latency_time.py [--num_envs 4096] [--launches 30] [--rounds 5] [--out latency_time.json]

Prints the card's name, power limit and SM clocks, then per handle the median milliseconds per launch of each round."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi unavailable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num_envs", type=int, default=4096)
    ap.add_argument("--launches", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from deepmimic_b200.assets import asset_root
    from deepmimic_b200.capi import BatchedCore
    assert torch.cuda.is_available(), "latency_time needs a CUDA device"
    root, N = asset_root(), a.num_envs
    args = ["--arg_file", "args/run_humanoid3d_spinkick_args.txt"]
    handles = {}
    for name in ("plain", "dyn_unit", "lat_zero", "lat_random"):
        c = BatchedCore(args, N, root, device=0, seed=1)
        c.set_mode(1)
        if name == "dyn_unit":
            c.set_dynamics(np.ones((N, 4 + c.dims.num_joints), dtype=np.float32))
        elif name == "lat_zero":
            c.set_action_latency(np.zeros(N))
        elif name == "lat_random":
            c.set_action_latency_randomization(0.0, 19 / 600.0)
        handles[name] = c
    rng = np.random.default_rng(3)
    A = handles["plain"].dims.action_size
    actions = [torch.as_tensor(0.05 * rng.standard_normal((N, A)), dtype=torch.float32, device="cuda") for _ in range(a.launches)]
    print("card: name, power limit, max SM clock, SM clock:", card(), flush=True)
    res = {k: [] for k in handles}
    for rnd in range(a.rounds + 1):   # round 0 warms up every handle
        for name, c in handles.items():
            c.reset(True, kin_time=np.linspace(0.0, 1.2, N), max_time=np.full(N, 1e9), rot_theta=np.zeros(N))
            c.sync()
            ms = []
            for i in range(a.launches):
                c.set_action(actions[i])
                c.sync()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                st = torch.cuda.ExternalStream(c.stream())   # events on the handle's own stream bracket the launch alone
                s.record(st); c.update(1.0 / 600.0, 20); e.record(st)
                torch.cuda.synchronize()
                ms.append(s.elapsed_time(e))
            if rnd > 0:
                res[name].append(float(np.median(ms)))
        if rnd > 0:
            print("round %d: %s" % (rnd, "  ".join("%s %.4f ms" % (k, v[-1]) for k, v in res.items())), flush=True)
    out = dict(card=card(), num_envs=N, updates_per_launch=20, rounds=res,
               median={k: float(np.median(v)) for k, v in res.items()}, spread={k: [min(v), max(v)] for k, v in res.items()})
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump(out, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
