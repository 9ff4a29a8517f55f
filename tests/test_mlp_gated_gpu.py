"""The gated (goal-conditioned) actor of the AMP task scenes on the tensor cores (dm_mlp_create_gated / dm_mlp_forward_gated, kernels/dm_mlp.cu)
against the fp32 torch actor it replaces in the rollout shim: R/learning/nets/fc_2layers_gated_1024units.py:6-58, rollout.build_gated_policy.
Tolerance as for the plain actor (tests/test_mlp_gpu.py): activations are rounded to fp16 between the layers -- here also the normalised goal,
the gate trunk and the gate hidden layers -- and the weights are carried as fp16 hi + lo pairs: normalised action error <= 1e-3, un-normalised
<= 2e-3 on the pretrained policies."""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
MINI = ["--motion_file", "data/datasets/test_clips_mini.txt"]
TARGET = MINI + ["--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]
HEADING = MINI + ["--arg_file", "args/train_amp_heading_humanoid3d_locomotion_args.txt"]


def _torch_gated_actor(actor, s, g, s_clip=math.inf, g_clip=math.inf):
    """fp32 torch restatement (TF32 off): normalised and un-normalised actions"""
    import torch
    t = lambda a: torch.tensor(np.asarray(a, dtype=np.float32), device="cuda")
    lin = lambda x, wb: x @ t(wb[0]) + t(wb[1])
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ns = ((s - t(actor["s_norm_mean"])) / t(actor["s_norm_std"])).clamp(-s_clip, s_clip)
        ng = ((g - t(actor["g_norm_mean"])) / t(actor["g_norm_std"])).clamp(-g_clip, g_clip)
        gc = torch.relu(lin(ng, actor["gate_common"]))
        h = torch.cat([ns, ng], dim=-1)
        for wb, gt in zip(actor["hidden"], actor["gates"]):
            gh = torch.relu(lin(gc, gt["hidden"]))
            h = torch.relu(2.0 * torch.sigmoid(lin(gh, gt["scale"])) * lin(h, wb) + lin(gh, gt["bias"]))
        a = lin(h, actor["mean"])
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    return a, a * t(actor["a_norm_std"]) + t(actor["a_norm_mean"])


def _gated_mlp(actor, rows, s_clip=math.inf, g_clip=math.inf):
    from deepmimic_b200.capi import TensorCoreGatedMLP
    return TensorCoreGatedMLP(actor, s_mean=actor["s_norm_mean"], s_std=actor["s_norm_std"], s_clip=s_clip, g_mean=actor["g_norm_mean"],
                              g_std=actor["g_norm_std"], g_clip=g_clip, a_mean=actor["a_norm_mean"], a_std=actor["a_norm_std"], max_rows=rows)


@pytest.mark.parametrize("task,args", [("target", TARGET), ("heading", HEADING)])
def test_pretrained_task_actor_on_tensor_cores_matches_fp32(asset_root, task, args):
    """the reference's pretrained target / heading actors (fp16 fixtures) on states and goals of a random-action rollout of the CUDA simulation"""
    import torch
    from deepmimic_b200.capi import BatchedCore
    from tests.test_task_scenes_cpu import fixture_task_actor
    actor = fixture_task_actor(task)
    N = 4096
    core = BatchedCore(args, N, asset_root, device=0, seed=5)
    S, G, A = core.dims.state_size, core.dims.goal_size, core.dims.action_size
    assert (S, G, A) == (226, 3, 28)
    stream = torch.cuda.ExternalStream(core.stream())
    with torch.cuda.stream(stream):
        off = torch.tensor(core.static(2), dtype=torch.float32, device="cuda"); scl = torch.tensor(core.static(3), dtype=torch.float32, device="cuda")
        lo = torch.tensor(core.static(4), dtype=torch.float32, device="cuda"); hi = torch.tensor(core.static(5), dtype=torch.float32, device="cuda")
        gen = torch.Generator(device="cuda"); gen.manual_seed(1)
        obs = torch.zeros(N, S, device="cuda"); goal = torch.zeros(N, G, device="cuda")
        for _ in range(6):
            a = torch.clamp(-off + 0.25 / scl * torch.randn(N, A, device="cuda", generator=gen), lo, hi).contiguous()
            core.set_action(a); core.update(1.0 / 600.0, 20); core.reset(False)
        core.observe(obs, None); core.record_goal(goal)
        mlp = _gated_mlp(actor, N)
        out = torch.zeros(N, A, device="cuda")
        mlp.forward(obs, goal, out, stream=stream.cuda_stream)
        ref_n, ref = _torch_gated_actor(actor, obs, goal)
        stream.synchronize()
        a_mean, a_std = (torch.tensor(actor[k], dtype=torch.float32, device="cuda") for k in ("a_norm_mean", "a_norm_std"))
        err = (out - ref).abs().max().item()
        err_n = ((out - a_mean) / a_std - ref_n).abs().max().item()
        print("%s: tensor-core gated actor vs fp32 torch gated actor on %d simulated (state, goal) rows: max |action error| %.2e (normalised %.2e), "
              "action rms %.3f, goal rms %.3f; %d launches" % (task, N, err, err_n, ref.pow(2).mean().sqrt().item(), goal.pow(2).mean().sqrt().item(), mlp.launches()))
        assert torch.isfinite(out).all() and mlp.launches() == 6
        assert err_n <= 1e-3 and err <= 2e-3
        # exploration noise is added in normalised action space; a partial batch (1000 rows: not a multiple of 128) leaves the other rows alone
        noise = 0.05 * torch.randn(N, A, device="cuda", generator=gen)
        out2 = torch.full((N, A), 7.0, device="cuda")
        mlp.forward(obs[:1000].contiguous(), goal[:1000].contiguous(), out2, noise=noise[:1000].contiguous(), stream=stream.cuda_stream)
        stream.synchronize()
        want = out[:1000] + noise[:1000] * a_std
        assert (out2[:1000] - want).abs().max().item() < 1e-5 and bool((out2[1000:] == 7.0).all())
    core.close()


def _random_gated_actor(rng, in_dim, goal_dim, h0, h1, out_dim, gate_common, gate_hidden):
    """xavier-scale fp32 weights (NOT fp16-representable, so the hi + lo split is exercised), nonzero biases, random normalisers"""
    xav = lambda a, b: rng.uniform(-1, 1, (a, b)).astype(np.float32) * np.sqrt(6.0 / (a + b))
    wb = lambda a, b: (xav(a, b), 0.1 * rng.standard_normal(b).astype(np.float32))
    return dict(hidden=[wb(in_dim + goal_dim, h0), wb(h0, h1)], mean=wb(h1, out_dim), gate_common=wb(goal_dim, gate_common),
                gates=[dict(hidden=wb(gate_common, gate_hidden), scale=wb(gate_hidden, h), bias=wb(gate_hidden, h)) for h in (h0, h1)],
                s_norm_mean=rng.standard_normal(in_dim).astype(np.float32), s_norm_std=rng.uniform(0.5, 2.0, in_dim).astype(np.float32),
                g_norm_mean=rng.standard_normal(goal_dim).astype(np.float32), g_norm_std=rng.uniform(0.5, 2.0, goal_dim).astype(np.float32),
                a_norm_mean=rng.standard_normal(out_dim).astype(np.float32), a_norm_std=rng.uniform(0.5, 2.0, out_dim).astype(np.float32))


@pytest.mark.parametrize("in_dim,goal_dim,h0,h1,out_dim,gate_common,gate_hidden,rows", [
    (226, 3, 1024, 512, 28, 128, 64, 300),     # target / heading
    (226, 4, 1024, 512, 28, 128, 64, 300),     # get-up / strike: 230-wide trunk
    (64, 2, 256, 256, 5, 48, 20, 128),         # small network, gate sizes below the tile widths
])
def test_random_gated_networks(in_dim, goal_dim, h0, h1, out_dim, gate_common, gate_hidden, rows):
    """random gated networks, inputs of unit scale through clipped normalisers (clip 3)"""
    import torch
    rng = np.random.default_rng(in_dim + goal_dim)
    actor = _random_gated_actor(rng, in_dim, goal_dim, h0, h1, out_dim, gate_common, gate_hidden)
    x = torch.tensor((actor["s_norm_mean"] + actor["s_norm_std"] * 2.0 * rng.standard_normal((rows, in_dim))).astype(np.float32), device="cuda")
    g = torch.tensor((actor["g_norm_mean"] + actor["g_norm_std"] * 2.0 * rng.standard_normal((rows, goal_dim))).astype(np.float32), device="cuda")
    mlp = _gated_mlp(actor, rows, s_clip=3.0, g_clip=3.0)
    out = torch.zeros(rows, out_dim, device="cuda")
    torch.cuda.synchronize()
    mlp.forward(x, g, out, stream=torch.cuda.current_stream().cuda_stream)
    ref_n, ref = _torch_gated_actor(actor, x, g, 3.0, 3.0)
    torch.cuda.synchronize()
    a_mean, a_std = (torch.tensor(actor[k], device="cuda") for k in ("a_norm_mean", "a_norm_std"))
    err_n = ((out - a_mean) / a_std - ref_n).abs().max().item()
    print("random gated %d+%d-%d-%d-%d network (gates %d / %d), %d rows: normalised action error %.2e (output rms %.3f)"
          % (in_dim, goal_dim, h0, h1, out_dim, gate_common, gate_hidden, rows, err_n, ref_n.pow(2).mean().sqrt().item()))
    assert torch.isfinite(out).all() and err_n <= 2e-3 * max(1.0, ref_n.abs().max().item())


def test_gated_actor_refusals():
    """errors through dm_last_error: wrong handle kind for the forward call, null goal, rows out of range, unsupported gate sizes and layer
    counts, out_dim > 64"""
    import ctypes as C
    import torch
    from deepmimic_b200 import capi
    from deepmimic_b200.capi import TensorCoreGatedMLP, TensorCoreMLP
    rng = np.random.default_rng(0)
    actor = _random_gated_actor(rng, 64, 2, 128, 128, 5, 32, 16)
    gated = _gated_mlp(actor, 128)
    plain = TensorCoreMLP(*actor["hidden"][0], *actor["hidden"][1], *actor["mean"], max_rows=128)   # 66 -> 128 -> 128 -> 5
    obs, goal, act = torch.zeros(128, 64, device="cuda"), torch.zeros(128, 2, device="cuda"), torch.zeros(128, 5, device="cuda")
    L, ptr = capi.lib(), lambda t: C.c_void_p(t.data_ptr())
    assert L.dm_mlp_forward(gated.h, ptr(obs), None, ptr(act), 128, None) != 0 and b"gated actor" in L.dm_last_error()
    assert L.dm_mlp_forward_gated(plain.h, ptr(obs), ptr(goal), None, ptr(act), 128, None) != 0 and b"plain actor" in L.dm_last_error()
    with pytest.raises(RuntimeError, match="null observation, goal"):
        gated.forward(obs, None, act)
    big = torch.zeros(129, 64, device="cuda")
    with pytest.raises(RuntimeError, match="rows out of range"):
        gated.forward(big, torch.zeros(129, 2, device="cuda"), torch.zeros(129, 5, device="cuda"))
    assert L.dm_mlp_forward_gated(gated.h, ptr(obs), ptr(goal), None, ptr(act), 0, None) != 0 and b"rows out of range" in L.dm_last_error()
    for sizes, msg in [((64, 2, 128, 128, 5, 129, 16), "gate sizes"), ((64, 2, 128, 128, 5, 32, 65), "gate sizes"), ((64, 2, 128, 128, 65, 32, 16), "bad sizes"),
                       ((64, 65, 128, 128, 5, 32, 16), "bad sizes")]:
        with pytest.raises(RuntimeError, match=msg):
            _gated_mlp(_random_gated_actor(rng, *sizes), 128)
    three = dict(actor, hidden=actor["hidden"] + [actor["hidden"][1]], gates=actor["gates"] + [actor["gates"][1]])
    with pytest.raises(ValueError, match="exactly two hidden layers"):
        TensorCoreGatedMLP(three)
    torch.cuda.synchronize()
    # the handles still work after the refused calls
    gated.forward(obs, goal, act); plain.forward(torch.zeros(128, 66, device="cuda"), act)
    torch.cuda.synchronize()
    assert gated.launches() == 6 and plain.launches() == 4


def _task_rollout(asset_root, task, args, backend, num_envs, steps, exp_rate, seed=9):
    import torch
    from deepmimic_b200.env import DeepMimicBatchEnv
    from deepmimic_b200.rollout import BatchedRollout, build_gated_policy, load_actor_weights
    from tests.test_task_scenes_cpu import fixture_task_actor
    a = fixture_task_actor(task)
    env = DeepMimicBatchEnv(args, num_envs=num_envs, asset_root=asset_root, seed=seed)
    env.set_mode(1)
    env.reset(True)
    ro = BatchedRollout(env, policy=load_actor_weights(build_gated_policy(226, env.get_goal_size(), 28), a), exp_rate=exp_rate, backend=backend)
    ro.s_norm.set_mean_std(a["s_norm_mean"], a["s_norm_std"]); ro.g_norm.set_mean_std(a["g_norm_mean"], a["g_norm_std"]); ro.a_norm.set_mean_std(a["a_norm_mean"], a["a_norm_std"])
    traj = ro.collect(steps, record_stats=False) if steps else None
    torch.cuda.synchronize()
    return env, ro, traj


@pytest.mark.parametrize("task,args", [("target", TARGET), ("heading", HEADING)])
def test_rollout_with_the_tensor_core_gated_actor_keeps_the_pretrained_behaviour(asset_root, task, args):
    """the pretrained task policies through BatchedRollout(backend="tensor_core"), 64 environments x 600 steps, with the thresholds of
    tests/test_task_scenes_gpu.py::test_fixture_task_policies_through_the_cuda_path; the torch backend's statistics beside them.
    Free-running contacts are chaotic, so the two backends' trajectories part after a few steps and are compared by statistics: the mean
    reward of 64 x 600 steps, within 0.05.  The per-environment mean rewards spread by 0.067 (standard deviation, both scenes, either backend,
    measured on an H100), so the difference of two such 64-environment means has a standard deviation of 0.067 * sqrt(2 / 64) = 0.012:
    0.05 is four of them."""
    res = {}
    for backend in ("tensor_core", "torch"):
        env, ro, traj = _task_rollout(asset_root, task, args, backend, 64, 600, 0.0)
        falls, mean_r = int((traj["terminate"] == 1).sum()), float(traj["rewards"].mean())
        inside = float((traj["goals"][:, :, 2] < 0.5).float().mean()) if task == "target" else float("nan")
        res[backend] = (falls, mean_r, inside, float(traj["rewards"].mean(0).std()))
        assert env.check_solver_capacity() == 0
    print("%s policy, 64 x 600 steps: tensor-core actor %d failed episodes, mean reward %.3f, inside radius %.3f, spread of the per-environment mean "
          "reward %.3f | torch actor %d, %.3f, %.3f, %.3f" % ((task,) + res["tensor_core"] + res["torch"]))
    falls, mean_r, inside, _ = res["tensor_core"]
    if task == "target":
        assert falls <= 12 and inside > 0.15 and mean_r > 0.45, res
    else:
        assert falls <= 6 and mean_r > 0.8, res
    assert abs(mean_r - res["torch"][1]) < 0.05, res


def test_gated_actor_step_time_and_task_rollout_rate(asset_root):
    """device clock: one 4096-row gated actor step (normalise, network, noise, un-normalise, log-probability) on the tensor cores against the
    torch gated actor; wall clock: the rollout rate of 4096 target_amp environments with either actor (printed)"""
    import time
    import torch
    ros, rates = {}, {}
    for backend in ("tensor_core", "torch"):
        env, ro, _ = _task_rollout(asset_root, "target", TARGET, backend, 4096, 0, 1.0, seed=4)
        ro.collect(8, record_stats=False); torch.cuda.synchronize()
        best = 0.0
        for _ in range(2):
            t0 = time.perf_counter(); ro.collect(48, record_stats=False); torch.cuda.synchronize()
            best = max(best, 4096 * 48 / (time.perf_counter() - t0))
        rates[backend], ros[backend] = best, ro
    print("target_amp rollout, 4096 envs: %.0f policy steps/s with the tensor-core gated actor, %.0f with the torch gated actor" % (rates["tensor_core"], rates["torch"]))
    gen = torch.Generator(device="cuda"); gen.manual_seed(2)
    x = torch.randn(4096, 226, device="cuda", generator=gen); g = torch.randn(4096, 3, device="cuda", generator=gen)
    explore = torch.ones(4096, dtype=torch.bool, device="cuda")

    def gpu_us(f, n=20):
        for _ in range(3): f()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record()
        for _ in range(n): f()
        e1.record(); torch.cuda.synchronize()
        return 1e3 * e0.elapsed_time(e1) / n
    tc, th = ros["tensor_core"], ros["torch"]
    t_tc = gpu_us(lambda: tc._act_tensor_core(x, explore, g))
    with torch.no_grad():
        t_th = gpu_us(lambda: th.a_norm.unnormalize(th.policy.sample(th.s_norm.normalize(x), th.g_norm.normalize(g), explore, th.gen)[0]))
    print("gated actor step (normalise, network, noise, un-normalise, log-probability) on 4096 (state, goal) rows: %.0f us on the wgmma kernels, "
          "%.0f us with the torch modules" % (t_tc, t_th))
    assert t_tc < t_th
