"""Where does a device-resident rollout step spend its time?  CUDA events around the actor and around the environment step, host time per step,
for both actor backends (diagnosis tool for the rollout rates of tests/test_mlp_gpu.py and tests/test_mlp_gated_gpu.py): the spin-kick imitation
scene with the plain actor, then the target_amp task scene with the gated actor; then the target_amp rollout rate without and with the AMP
discriminator (agent AMP observations and amp_rewards recorded every step, tests/test_amp_reward_gpu.py) on both backends; then the spin-kick and
target_amp rollout rates without and with the PPO critic (values of [s_k; s'_k] every step, the return scan at the end, tests/test_value_targets_gpu.py)
on both backends."""
import os, sys, time
import numpy as np
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch
from deepmimic_b200.assets import asset_root
from deepmimic_b200.env import DeepMimicBatchEnv
from deepmimic_b200.rollout import BatchedRollout, build_critic, build_discriminator, build_gated_policy, build_policy, load_actor_weights
sys.path.insert(0, os.path.join(REPO, "tests"))
from test_task_scenes_cpu import fixture_task_actor
f = np.load(os.path.join(REPO, "tests", "golden", "policy_humanoid3d_spinkick_fp16.npz"))
a = {k: f[k].astype(np.float64) for k in f.files}
root = asset_root(True)
at = fixture_task_actor("target")
TARGET = ["--motion_file", "data/datasets/test_clips_mini.txt", "--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]


def make_rollout(scene, backend, **extra):
    """4096 environments of spin kick (pretrained actor, 20 s episodes) or target_amp (pretrained gated target actor), exploration noise on"""
    if scene == "spinkick":
        env = DeepMimicBatchEnv(["--arg_file", "args/train_humanoid3d_spinkick_args.txt"], num_envs=4096, asset_root=root, seed=4)
        env._core.set_episode_limit(20.0); env.reset(True)
        ro = BatchedRollout(env, policy=load_actor_weights(build_policy(227, 28), a), exp_rate=1.0, backend=backend, **extra)
        ro.s_norm.set_mean_std(a["s_mean"], a["s_std"]); ro.a_norm.set_mean_std(a["a_mean"], a["a_std"])
    else:
        env = DeepMimicBatchEnv(TARGET, num_envs=4096, asset_root=root, seed=4)
        env.reset(True)
        ro = BatchedRollout(env, policy=load_actor_weights(build_gated_policy(226, 3, 28), at), exp_rate=1.0, backend=backend, **extra)
        ro.s_norm.set_mean_std(at["s_norm_mean"], at["s_norm_std"]); ro.g_norm.set_mean_std(at["g_norm_mean"], at["g_norm_std"]); ro.a_norm.set_mean_std(at["a_norm_mean"], at["a_norm_std"])
    return env, ro


for scene, backend in [("spinkick", "tensor_core"), ("spinkick", "torch"), ("spinkick", "tensor_core"), ("target", "tensor_core"), ("target", "torch"), ("target", "tensor_core")]:
    env, ro = make_rollout(scene, backend)
    ro.collect(8, record_stats=False); torch.cuda.synchronize()
    t0 = time.perf_counter(); ro.collect(48, record_stats=False); torch.cuda.synchronize(); dt = time.perf_counter() - t0
    # manual loop with events
    s = env.record_state(); ev = []
    th = time.perf_counter()
    for k in range(32):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        explore = torch.rand(4096, device="cuda") < 1.0
        g = env.record_goal() if scene == "target" else None
        e[0].record()
        if backend == "tensor_core":
            act, logp = ro._act_tensor_core(s, explore, g)
        elif g is not None:
            na, logp = ro.policy.sample(ro.s_norm.normalize(s), ro.g_norm.normalize(g), explore, ro.gen); act = ro.a_norm.unnormalize(na).contiguous()
        else:
            na, logp = ro.policy.sample(ro.s_norm.normalize(s), explore, ro.gen); act = ro.a_norm.unnormalize(na).contiguous()
        e[1].record()
        s, r, done, term = env.step(act)
        e[2].record()
        env.reset(); s = env.record_state()
        e[3].record()
        ev.append(e)
    host = time.perf_counter() - th
    torch.cuda.synchronize()
    wall = time.perf_counter() - th
    g = lambda i, j: np.median([x[i].elapsed_time(x[j]) for x in ev])
    print("%-8s %-11s collect(48): %.0f steps/s | manual loop: actor %.3f ms, env.step %.3f ms, reset+observe %.3f ms (GPU, median) ; host enqueue %.3f ms/step, wall %.3f ms/step"
          % (scene, backend, 4096 * 48 / dt, g(0, 1), g(1, 2), g(2, 3), 1e3 * host / 32, 1e3 * wall / 32))

# target_amp collect() rate with and without the discriminator, alternating; best of two 48-step windows each
for backend in ("tensor_core", "torch"):
    rates = {}
    for with_disc in (False, True, False, True):
        env = DeepMimicBatchEnv(TARGET, num_envs=4096, asset_root=root, seed=4)
        env.reset(True)
        torch.manual_seed(0)
        extra = dict(disc=build_discriminator(env.get_amp_obs_size()), task_reward_lerp=0.5) if with_disc else {}
        ro = BatchedRollout(env, policy=load_actor_weights(build_gated_policy(226, 3, 28), at), exp_rate=1.0, backend=backend, **extra)
        ro.s_norm.set_mean_std(at["s_norm_mean"], at["s_norm_std"]); ro.g_norm.set_mean_std(at["g_norm_mean"], at["g_norm_std"]); ro.a_norm.set_mean_std(at["a_norm_mean"], at["a_norm_std"])
        ro.collect(8, record_stats=False); torch.cuda.synchronize()
        for _ in range(2):
            t0 = time.perf_counter(); ro.collect(48, record_stats=False); torch.cuda.synchronize()
            rates[with_disc] = max(rates.get(with_disc, 0.0), 4096 * 48 / (time.perf_counter() - t0))
        assert env.counters()[1] == 0
        del ro, env
    print("target_amp %-11s collect(48): %.0f steps/s without the discriminator, %.0f with it" % (backend, rates[False], rates[True]))

# collect() rate with and without the PPO critic (discount 0.95, lambda 0.95), alternating; best of two 48-step windows each
for scene in ("spinkick", "target"):
    for backend in ("tensor_core", "torch"):
        rates = {}
        for with_critic in (False, True, False, True):
            torch.manual_seed(0)
            extra = dict(critic=build_critic(226 if scene == "target" else 227, 3 if scene == "target" else 0), discount=0.95, td_lambda=0.95) if with_critic else {}
            env, ro = make_rollout(scene, backend, **extra)
            ro.collect(8, record_stats=False); torch.cuda.synchronize()
            for _ in range(2):
                t0 = time.perf_counter(); ro.collect(48, record_stats=False); torch.cuda.synchronize()
                rates[with_critic] = max(rates.get(with_critic, 0.0), 4096 * 48 / (time.perf_counter() - t0))
            assert env.counters()[1] == 0
            del ro, env
        print("%-8s %-11s collect(48): %.0f steps/s without the critic, %.0f with it (%.3f ms more per policy step)"
              % (scene, backend, rates[False], rates[True], 1e3 * 4096 * (1.0 / rates[True] - 1.0 / rates[False])))
