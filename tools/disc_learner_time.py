"""Device-clock time of the AMP discriminator's update (deepmimic_b200/learner.py: AMPDiscLearner): imitate_amp humanoid3d (226 AMP inputs,
1024-512 discriminator), 4096 agent + 4096 expert rows per step, one update() of --steps steps and one minibatch step alone, on both backends.
Prints the card and its power limit.

    python tools/disc_learner_time.py [--envs 4096] [--batch 4096] [--steps 8] [--repeat 5]"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch
    from deepmimic_b200.assets import asset_root
    from deepmimic_b200.env import DeepMimicBatchEnv
    from deepmimic_b200.learner import AMPDiscLearner
    from deepmimic_b200.rollout import BatchedRollout, build_discriminator
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--repeat", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("disc_learner_time.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("device: %s; nvidia-smi: %s" % (torch.cuda.get_device_name(0), q.stdout.strip() or "n/a"))
    env = DeepMimicBatchEnv(["--scene", "imitate_amp", "--arg_file", "args/train_humanoid3d_walk_args.txt"], num_envs=a.envs, asset_root=asset_root(),
                            seed=1)
    env.reset(True)
    torch.manual_seed(0)
    ro = BatchedRollout(env, exp_rate=0.8, backend="tensor_core", disc=build_discriminator(env.get_amp_obs_size()))
    traj = ro.collect(8)
    M = env.get_amp_obs_size()
    agent = traj["amp_obs"].reshape(-1, M).contiguous()
    expert = torch.cat([env.record_amp_obs_expert().clone() for _ in range(8)])
    hp = dict(stepsize=1e-5, momentum=0.9, weight_decay=5e-4, logit_reg_weight=0.05, grad_penalty=10.0, batch_size=a.batch, steps=a.steps)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn, n):
        for _ in range(2):
            fn()
        torch.cuda.synchronize(); e0.record()
        for _ in range(n):
            fn()
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n
    for backend in ("torch", "tensor_core"):
        ln = AMPDiscLearner(ro, **hp, backend=backend)
        t_up = timed(lambda: ln.update(agent, expert), a.repeat)
        ai = torch.arange(a.batch, device="cuda") % agent.shape[0]
        ei = torch.arange(a.batch, device="cuda") % expert.shape[0]
        stats = [torch.zeros((), device="cuda") for _ in range(6)]
        tc = None
        if backend == "tensor_core":
            ln._tc.set_weights(stream=torch.cuda.current_stream().cuda_stream)
            tc = ln._tc_batch(agent, expert)
        t_mb = timed(lambda: ln.minibatch_step(agent, expert, ai, ei, stats, tc), 10 * a.repeat)
        print("%-11s update of %d steps x (%d agent + %d expert rows, %d inputs): %8.2f ms; one minibatch step: %7.3f ms"
              % (backend, a.steps, a.batch, a.batch, M, t_up, t_mb))


if __name__ == "__main__":
    main()
