"""Device-clock time of the PPO learner (deepmimic_b200/learner.py): one update() of a 32 x 4096 spin-kick window (227 inputs, 28 actions,
1024-512 actor and critic), minibatch 4096, on both backends, and one minibatch step (critic + actor) alone.  Prints the card and its power limit.
--scene target_amp: the same over a target_amp window (226 state and 3 goal inputs, 28 actions) with the pretrained gated actor and a random
gated critic, the reference's fc_2layers_gated_1024units.

    python tools/learner_time.py [--scene spinkick|target_amp] [--steps 32] [--envs 4096] [--minibatch 4096] [--repeat 5]"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import numpy as np
    import torch
    from deepmimic_b200.assets import asset_root
    from deepmimic_b200.env import DeepMimicBatchEnv
    from deepmimic_b200.learner import PPOLearner
    from deepmimic_b200.rollout import BatchedRollout, build_critic, build_gated_policy, load_actor_weights
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene", choices=("spinkick", "target_amp"), default="spinkick")
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--minibatch", type=int, default=4096)
    ap.add_argument("--repeat", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("learner_time.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("device: %s; nvidia-smi: %s" % (torch.cuda.get_device_name(0), q.stdout.strip() or "n/a"))
    gold = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
    if a.scene == "spinkick":
        env = DeepMimicBatchEnv(["--arg_file", "args/train_humanoid3d_spinkick_args.txt"], num_envs=a.envs, asset_root=asset_root(), seed=1)
        env.reset(True)
        torch.manual_seed(0)
        ro = BatchedRollout(env, exp_rate=0.8, backend="tensor_core", critic=build_critic(env.get_state_size()), discount=0.95, td_lambda=0.95)
        f = np.load(os.path.join(gold, "policy_humanoid3d_spinkick_fp16.npz"))
        load_actor_weights(ro.policy, {k: f[k].astype(np.float32) for k in f.files})
    else:
        args = ["--motion_file", "data/datasets/test_clips_mini.txt", "--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]
        env = DeepMimicBatchEnv(args, num_envs=a.envs, asset_root=asset_root(), seed=1)
        env.reset(True)
        S, G, A = env.get_state_size(), env.get_goal_size(), env.get_action_size()
        f = np.load(os.path.join(gold, "policy_humanoid3d_amp_target_locomotion_fp16.npz"))
        g = lambda k: f[k].astype(np.float32)
        actor = dict(hidden=[(g("w0"), g("b0")), (g("w1"), g("b1"))], mean=(g("wm"), g("bm")), logstd=g("logstd"), gate_common=(g("gcw"), g("gcb")),
                     gates=[dict(hidden=(g("g%d_hidden_w" % i), g("g%d_hidden_b" % i)), bias=(g("g%d_bias_w" % i), g("g%d_bias_b" % i)),
                                 scale=(g("g%d_scale_w" % i), g("g%d_scale_b" % i))) for i in range(2)])
        torch.manual_seed(0)
        ro = BatchedRollout(env, policy=load_actor_weights(build_gated_policy(S, G, A), actor), exp_rate=0.8, backend="tensor_core",
                            critic=build_critic(S, G), discount=0.95, td_lambda=0.95)
        ro.s_norm.set_mean_std(g("s_mean"), g("s_std")); ro.g_norm.set_mean_std(g("g_mean"), g("g_std")); ro.a_norm.set_mean_std(g("a_mean"), g("a_std"))
    traj = ro.collect(a.steps)
    hp = dict(actor_stepsize=2.5e-6, actor_momentum=0.9, actor_weight_decay=5e-4, critic_stepsize=1e-2, critic_momentum=0.9, critic_weight_decay=1e-3,
              ratio_clip=0.2, norm_adv_clip=4.0, minibatch_size=a.minibatch, epochs=1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn, n):
        for _ in range(2):
            fn()
        torch.cuda.synchronize(); e0.record()
        for _ in range(n):
            fn()
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n
    mbs = -(-a.steps * a.envs // a.minibatch)
    for backend in ("torch", "tensor_core"):
        ln = PPOLearner(ro, **hp, backend=backend)
        t_up = timed(lambda: ln.update(traj), a.repeat)
        w = ln.window(traj)
        c = torch.arange(a.minibatch, device="cuda") % w["R"]
        x = w["exp_idx"][torch.arange(a.minibatch, device="cuda") % w["exp_idx"].numel()]
        stats = [torch.zeros((), device="cuda") for _ in range(3)]
        tc = None
        if backend == "tensor_core":
            st = torch.cuda.current_stream().cuda_stream
            ln._tc_critic.set_weights(stream=st); ln._tc_actor.set_weights(stream=st)
            tc = ln._tc_batch(w)
        t_mb = timed(lambda: ln.minibatch_step(w, c, x, stats, tc), 10 * a.repeat)
        print("%s, %-11s update of %d x %d (%d minibatches of %d): %8.2f ms; one minibatch step (critic + actor): %7.3f ms"
              % (a.scene, backend, a.steps, a.envs, mbs, a.minibatch, t_up, t_mb))


if __name__ == "__main__":
    main()
