"""Time of the expert AMP observations of one window of T policy steps x N environments: one dm_sample_amp_obs_expert call of T N rows
(draws on the device, no host synchronisation) against T calls of dm_record_amp_obs_expert (host draws, each staged with a stream
synchronisation).  Workloads: spin kick and target_amp with the 56-clip dataset, 4096 environments.  Both paths are timed between two events
on the handle's stream around --repeat windows (10 x --repeat for the sampler, whose window is short); for the host-draw path that elapsed time includes the host's staging stalls between the
kernels, so it is an end-to-end figure, not kernel time.  --rounds alternate the two paths and the spread over the rounds is printed.  Prints
the card and its power limit.

    python tools/expert_sample_time.py [--envs 4096] [--steps 32] [--repeat 200] [--rounds 5]"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

WORKLOADS = [("spinkick", ["--arg_file", "args/run_humanoid3d_spinkick_args.txt"]),
             ("target_amp 56 clips", ["--motion_file", "data/datasets/synthetic_locomotion_56.txt", "--arg_file",
                                      "args/train_amp_target_humanoid3d_locomotion_args.txt"])]


def main():
    import torch
    from deepmimic_b200.assets import asset_root
    from deepmimic_b200.capi import BatchedCore
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--repeat", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("expert_sample_time.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("device: %s; nvidia-smi: %s" % (torch.cuda.get_device_name(0), q.stdout.strip() or "n/a"))
    for name, args in WORKLOADS:
        core = BatchedCore(args, a.envs, asset_root(), device=0, seed=1)
        stream = torch.cuda.ExternalStream(core.stream())
        T, N, M = a.steps, a.envs, core.dims.amp_obs_size
        out = torch.zeros(T * N, M, device="cuda")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def window_sampled():
            core.sample_amp_obs_expert(out)

        def window_host_draws():
            for t in range(T):
                core.amp_obs_expert(out[t * N:(t + 1) * N])

        paths = (("sampler, 1 call of %d rows" % (T * N), window_sampled), ("host draws, %d calls of %d rows" % (T, N), window_host_draws))
        times = {label: [] for label, _ in paths}
        for label, fn in paths:   # warm-up
            fn(); fn()
        for _ in range(a.rounds):
            for label, fn in paths:
                core.sync()
                e0.record(stream)
                reps = a.repeat * (10 if fn is window_sampled else 1)
                for _ in range(reps):
                    fn()
                e1.record(stream)
                core.sync()
                times[label].append(e0.elapsed_time(e1) / reps)
        for label, _ in paths:
            t = sorted(times[label])
            print("%-20s %-34s %8.3f ms per window (min %.3f, median %.3f, max %.3f over %d alternating rounds; elapsed between stream events)"
                  % (name, label, t[len(t) // 2], t[0], t[len(t) // 2], t[-1], a.rounds))
        core.close()


if __name__ == "__main__":
    main()
