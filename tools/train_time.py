"""Per-phase device time of steady-state training iterations (Trainer.iteration), and the host synchronisations per iteration.  Workloads: spin
kick (PPO agent, plain networks) and target_amp with the 56-clip dataset (AMP agent, gated networks and the discriminator), 4096 environments,
T = 32, with the agent values of tests/test_train_gpu.py.  Phases: collect (the window, with the episode statistics), store (the disc buffers
and the expert draws), disc_update, ppo_update, normalizers (the update and the refresh of the rollout's handles), each between two CUDA events
on the current stream around --iters iterations after --warmup; evaluation (TestEpisodes episodes on the evaluation handle) and checkpoint
(Trainer.state_dict(), which synchronises: host wall clock) are timed on their own.  Host synchronisations are counted with torch's sync debug
mode (every synchronising torch call) plus the library's one in set_sample_count.  The run is one rank; a Trainer with a process group of
more than one rank adds one synchronisation per PPO update (PPOLearner's check that every rank's window has the same size and an explored
sample), and its evaluation's sum over the ranks stays within the evaluation's last synchronisation.  Prints the card and its power limit.

    python tools/train_time.py [--envs 4096] [--steps 32] [--warmup 2] [--iters 5]"""
import argparse
import contextlib
import os
import subprocess
import sys
import time
import warnings

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch
    from deepmimic_b200.assets import asset_root
    from deepmimic_b200.trainer import AgentConfig, Trainer
    from tests.test_train_gpu import AGENT, AMP_AGENT, SPINKICK_TRAIN, TARGET56
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_time.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("device: %s; nvidia-smi: %s" % (torch.cuda.get_device_name(0), q.stdout.strip() or "n/a"))
    for name, args, values in (("spinkick PPO", SPINKICK_TRAIN, AGENT), ("target_amp 56 clips AMP", TARGET56, AMP_AGENT)):
        tr = Trainer(args, AgentConfig(dict(values, OutputIters=10 ** 6)), asset_root(), a.envs, window_steps=a.steps, backend="tensor_core", seed=1)
        events = {}

        @contextlib.contextmanager
        def hook(phase):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            yield
            e1.record()
            events.setdefault(phase, []).append((e0, e1))
        for _ in range(a.warmup):
            tr.iteration()
        torch.cuda.synchronize()
        tr.phase_hook = hook
        total0, total1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        total0.record()
        torch.cuda.set_sync_debug_mode("warn")
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            for _ in range(a.iters):
                tr.iteration()
        torch.cuda.set_sync_debug_mode("default")
        total1.record()
        torch.cuda.synchronize()
        syncs = sum("synchroniz" in str(w.message) for w in caught)
        tr.phase_hook = None
        ms = {p: sorted(e0.elapsed_time(e1) for e0, e1 in ev) for p, ev in events.items()}
        print("%s, %d envs, T = %d (%d samples per iteration), %d iterations after %d warm-up:" % (name, a.envs, a.steps, a.envs * a.steps, a.iters, a.warmup))
        for p, v in ms.items():
            print("  %-12s median %8.2f ms (min %.2f, max %.2f over %d)" % (p, v[len(v) // 2], v[0], v[-1], len(v)))
        print("  %-12s %8.2f ms per iteration (events around the iterations)" % ("iteration", total0.elapsed_time(total1) / a.iters))
        print("  host synchronisations per iteration: %.1f torch + 1 set_sample_count" % (syncs / a.iters))
        ev = []
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); tr.evaluate(); e1.record(); torch.cuda.synchronize()
            ev.append(e0.elapsed_time(e1))
        ck = []
        for _ in range(3):
            t0 = time.perf_counter(); tr.state_dict(); ck.append(1e3 * (time.perf_counter() - t0))
        print("  %-12s median %8.2f ms over 3 (%d episodes)" % ("evaluation", sorted(ev)[1], tr.test_env.num_envs))
        print("  %-12s median %8.2f ms over 3 (state_dict, host wall clock)" % ("checkpoint", sorted(ck)[1]))
        tr.close()
        del tr
        torch.cuda.synchronize()


if __name__ == "__main__":
    main()
