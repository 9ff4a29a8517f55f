"""The AMP discriminator's style reward on the tensor cores (dm_mlp_forward_style_reward, kernels/dm_mlp.cu: dm_mlp_style_reward_kernel) against
the fp32 torch discriminator of the rollout shim (rollout.build_discriminator, rollout.amp_rewards), and its recording in BatchedRollout.collect.
Tolerance as for the actors (tests/test_mlp_gpu.py): activations are rounded to fp16 between the layers, weights are fp16 hi + lo pairs, so the
logit is within 2e-3 max(1, max |d|) of fp32 and so is the style reward (its slope |(1 - d) / 2| is at most 1 where it is not clamped)."""
import contextlib
import ctypes as C
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
MINI = ["--motion_file", "data/datasets/test_clips_mini.txt"]
TARGET = MINI + ["--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]
IMITATE_AMP = ["--scene", "imitate_amp", "--arg_file", "args/train_humanoid3d_walk_args.txt"]
DOG_AMP = ["--scene", "imitate_amp", "--arg_file", "args/train_dog3d_trot_args.txt"]


@contextlib.contextmanager
def _no_tf32():
    import torch
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def _amp_rows(asset_root, args, n, seed=5):
    """agent AMP observations and env rewards of n environments after six random-action policy steps of the CUDA simulation"""
    import torch
    from deepmimic_b200.capi import BatchedCore
    core = BatchedCore(args, n, asset_root, device=0, seed=seed)
    stream = torch.cuda.ExternalStream(core.stream())
    with torch.cuda.stream(stream):
        st = lambda k: torch.tensor(core.static(k), dtype=torch.float32, device="cuda")
        off, scl, lo, hi = st(2), st(3), st(4), st(5)
        gen = torch.Generator(device="cuda"); gen.manual_seed(1)
        amp, rew = torch.zeros(n, core.dims.amp_obs_size, device="cuda"), torch.zeros(n, device="cuda")
        for _ in range(6):
            a = torch.clamp(-off + 0.25 / scl * torch.randn(n, core.dims.action_size, device="cuda", generator=gen), lo, hi).contiguous()
            core.set_action(a); core.update(1.0 / 600.0, 20); core.observe(None, rew); core.reset(False)
        core.amp_obs_agent(amp)
    stream.synchronize()
    over = core.counters()[1]
    core.close()
    assert over == 0
    return amp, rew


def _spread_disc(rng, amp, clip=3.0):
    """random xavier discriminator weights (not fp16-representable: the hi + lo split is exercised) and a clipped normaliser from the data; the
    logit head is rescaled so that the logits have mean 1 and standard deviation 3, i.e. fall on both sides of the reward's clamp (d < -1, d > 3)"""
    import torch
    m = amp.shape[1]
    xav = lambda a, b: rng.uniform(-1, 1, (a, b)).astype(np.float32) * np.sqrt(6.0 / (a + b))
    d = dict(hidden=[(xav(m, 1024), 0.1 * rng.standard_normal(1024).astype(np.float32)), (xav(1024, 512), 0.1 * rng.standard_normal(512).astype(np.float32))],
             logit=(xav(512, 1), np.zeros(1, np.float32)),
             mean=amp.mean(0).cpu().numpy(), std=amp.std(0).clamp_min(0.05).cpu().numpy(), clip=clip)
    d0 = _torch_logits(d, amp)
    c = 3.0 / d0.std().item()
    d["logit"] = (d["logit"][0] * c, np.array([1.0 - c * d0.mean().item()], np.float32))
    return d


def _torch_logits(d, x):
    import torch
    t = lambda a: torch.tensor(np.asarray(a, dtype=np.float32), device="cuda")
    with _no_tf32():
        h = ((x - t(d["mean"])) / t(d["std"])).clamp(-d["clip"], d["clip"])
        for w, b in d["hidden"]:
            h = torch.relu(h @ t(w) + t(b))
        return (h @ t(d["logit"][0]) + t(d["logit"][1]))[:, 0]


def _tc_disc(d, rows):
    from deepmimic_b200.capi import TensorCoreMLP
    return TensorCoreMLP(*d["hidden"][0], *d["hidden"][1], *d["logit"], in_mean=d["mean"], in_std=d["std"], in_clip=d["clip"], max_rows=rows)


@pytest.mark.parametrize("scene,args,width", [("imitate_amp humanoid3d", IMITATE_AMP, 226), ("imitate_amp dog3d", DOG_AMP, 426), ("target_amp", TARGET, 226)])
def test_style_reward_on_real_amp_observations_matches_fp32(asset_root, scene, args, width):
    import torch
    from deepmimic_b200.rollout import amp_rewards
    N = 4096
    amp, task = _amp_rows(asset_root, args, N)
    assert amp.shape == (N, width)
    d = _spread_disc(np.random.default_rng(width), amp)
    ref = _torch_logits(d, amp)
    ref_style, _ = amp_rewards(ref)
    frac = lambda m: float(m.float().mean())
    assert frac(ref < -1.0) > 0.05 and frac(ref > 3.0) > 0.05 and frac((ref > -1.0) & (ref < 3.0)) > 0.2
    mlp = _tc_disc(d, N)
    logit, style, reward = (torch.full((N,), 7.0, device="cuda") for _ in range(3))
    st = torch.cuda.current_stream().cuda_stream
    mlp.style_reward(amp, reward, logit=logit, style=style, stream=st)
    torch.cuda.synchronize()
    bound = 2e-3 * max(1.0, ref.abs().max().item())
    err_d, err_s = (logit - ref).abs().max().item(), (style - ref_style).abs().max().item()
    print("%s, %d AMP observations of width %d: logit error %.2e, style-reward error %.2e (bound %.2e; logits in [%.1f, %.1f])"
          % (scene, N, width, err_d, err_s, bound, ref.min().item(), ref.max().item()))
    assert err_d <= bound and err_s <= bound
    assert torch.equal(reward, style)                                   # no task reward: the style reward itself
    torch.testing.assert_close(style, amp_rewards(logit)[0], rtol=0, atol=1e-6)
    # blended with the env's reward (the task reward in target_amp)
    reward2 = torch.zeros(N, device="cuda")
    mlp.style_reward(amp, reward2, task_reward=task, task_lerp=0.3, stream=st)
    torch.cuda.synchronize()
    assert (reward2 - (0.7 * style + 0.3 * task)).abs().max().item() <= 1e-6
    assert mlp.launches() == 8


def test_partial_batch_and_edge_cases():
    """a 1000-row batch leaves the other rows alone; NULL task reward, task_lerp 0 (the style reward) and 1 (the task reward, exactly)"""
    import torch
    N, rows = 4096, 1000
    gen = torch.Generator(device="cuda"); gen.manual_seed(3)
    x = torch.randn(N, 226, device="cuda", generator=gen)
    d = _spread_disc(np.random.default_rng(7), x)
    mlp = _tc_disc(d, N)
    task = torch.rand(N, device="cuda", generator=gen)
    full_l, full_s, full_r = (torch.zeros(N, device="cuda") for _ in range(3))
    mlp.style_reward(x, full_r, logit=full_l, style=full_s)
    outs = [torch.full((N,), 7.0, device="cuda") for _ in range(3)]
    mlp.style_reward(x[:rows].contiguous(), outs[2], task_reward=task[:rows].contiguous(), task_lerp=0.0, logit=outs[0], style=outs[1])
    torch.cuda.synchronize()
    for o, want in zip(outs, (full_l, full_s, full_s)):
        assert torch.equal(o[:rows], want[:rows]) and bool((o[rows:] == 7.0).all())
    r1 = torch.zeros(N, device="cuda")
    mlp.style_reward(x, r1, task_reward=task, task_lerp=1.0)
    torch.cuda.synchronize()
    assert torch.equal(r1, task)


def test_style_reward_refusals_and_launch_count():
    """errors through dm_last_error: a gated handle, out_dim != 1, task_lerp outside [0, 1] or NaN, rows out of range, NULL AMP observations or
    rewards; the refused calls launch nothing and the handle keeps working (4 launches per call)"""
    import torch
    from deepmimic_b200 import capi
    from deepmimic_b200.capi import TensorCoreMLP
    from tests.test_mlp_gated_gpu import _gated_mlp, _random_gated_actor
    rng = np.random.default_rng(0)
    gated = _gated_mlp(_random_gated_actor(rng, 64, 2, 128, 128, 5, 32, 16), 128)
    wb = lambda a, b: (rng.standard_normal((a, b)).astype(np.float32) / np.sqrt(a), np.zeros(b, np.float32))
    actor = TensorCoreMLP(*wb(64, 128), *wb(128, 128), *wb(128, 5), max_rows=128)
    disc = TensorCoreMLP(*wb(64, 128), *wb(128, 128), *wb(128, 1), max_rows=128)
    x, r, task = torch.zeros(128, 64, device="cuda"), torch.zeros(128, device="cuda"), torch.zeros(128, device="cuda")
    L, ptr = capi.lib(), lambda t: C.c_void_p(t.data_ptr())
    call = lambda h, obs=x, rew=r, lerp=0.0, rows=128: L.dm_mlp_forward_style_reward(h, obs if obs is None else ptr(obs), ptr(task), lerp, None, None,
                                                                                      rew if rew is None else ptr(rew), rows, None)
    assert call(gated.h) != 0 and b"gated actor" in L.dm_last_error()
    assert call(actor.h) != 0 and b"one output" in L.dm_last_error()
    for lerp in (-0.1, 1.1, math.nan):
        assert call(disc.h, lerp=lerp) != 0 and b"task_lerp" in L.dm_last_error()
    for rows in (0, 129):
        assert call(disc.h, rows=rows) != 0 and b"rows out of range" in L.dm_last_error()
    assert call(disc.h, obs=None) != 0 and b"null AMP observation" in L.dm_last_error()
    assert call(disc.h, rew=None) != 0 and b"null AMP observation or reward" in L.dm_last_error()
    with pytest.raises(RuntimeError, match="task_lerp"):
        disc.style_reward(x, r, task_reward=task, task_lerp=2.0)
    assert disc.launches() == 0 and gated.launches() == 0 and actor.launches() == 0
    assert call(disc.h, lerp=0.5) == 0 and disc.launches() == 4
    disc.style_reward(x, r)
    torch.cuda.synchronize()
    assert disc.launches() == 8


def _amp_env(asset_root, args, n, seed):
    from deepmimic_b200.env import DeepMimicBatchEnv
    env = DeepMimicBatchEnv(args, num_envs=n, asset_root=asset_root, seed=seed)
    env.reset(True)
    return env


@pytest.mark.parametrize("args,lerp", [(IMITATE_AMP, None), (TARGET, 0.5)])
@pytest.mark.parametrize("backend", ["torch", "tensor_core"])
def test_rollout_records_amp_obs_and_rewards(asset_root, args, lerp, backend):
    """BatchedRollout(disc=...), 64 environments x 600 steps: the agent AMP observations are those of a hand-written step / record / reset loop
    given the same actions, the torch discriminator reproduces the recorded logits, amp_rewards is the style reward (imitate_amp) or its blend
    with the task reward (target_amp)"""
    import torch
    from deepmimic_b200.rollout import BatchedRollout, amp_rewards, build_discriminator
    N, T = 64, 600
    torch.manual_seed(0)
    env = _amp_env(asset_root, args, N, seed=11)
    disc = build_discriminator(env.get_amp_obs_size())
    ro = BatchedRollout(env, exp_rate=0.0, backend=backend, disc=disc, task_reward_lerp=lerp)
    traj = ro.collect(T, record_stats=False)
    torch.cuda.synchronize()
    assert env.counters()[1] == 0 and int(traj["dones"].sum()) > 0
    # the same actions through a hand-written loop on a second handle with the same seed
    env2 = _amp_env(asset_root, args, N, seed=11)
    amp2 = torch.empty_like(traj["amp_obs"])
    for k in range(T):
        env2.step(traj["actions"][k].contiguous())
        amp2[k] = env2.record_amp_obs_agent()
        env2.reset()
    torch.cuda.synchronize()
    assert torch.equal(traj["amp_obs"], amp2) and env2.counters()[1] == 0
    with torch.no_grad(), _no_tf32():
        d = disc(ro.amp_norm.normalize(traj["amp_obs"]))[..., 0]
    bound = 2e-3 * max(1.0, d.abs().max().item())
    err = (traj["disc_logits"] - d).abs().max().item()
    print("%s, %s backend, %d x %d steps: %d episode ends, logit error %.2e (bound %.2e), mean style reward %.3f, mean amp reward %.3f"
          % (env.get_name(), backend, N, T, int(traj["dones"].sum()), err, bound, traj["style_rewards"].mean().item(), traj["amp_rewards"].mean().item()))
    assert err <= bound
    assert (traj["style_rewards"] - amp_rewards(d)[0]).abs().max().item() <= bound
    if lerp is None:
        assert torch.equal(traj["amp_rewards"], traj["style_rewards"])
    else:
        assert (traj["amp_rewards"] - ((1 - lerp) * traj["style_rewards"] + lerp * traj["rewards"])).abs().max().item() <= 1e-6


def test_style_reward_step_time():
    """device clock, 4096 rows: the tensor-core discriminator reward (four launches) against the fp32 torch discriminator and its reward ops"""
    import torch
    from deepmimic_b200.capi import TensorCoreMLP
    from deepmimic_b200.rollout import DeviceNormalizer, amp_rewards, build_discriminator
    N, M, lerp = 4096, 226, 0.5
    torch.manual_seed(0)
    disc = build_discriminator(M).cuda()
    norm = DeviceNormalizer(M, device="cuda")
    gen = torch.Generator(device="cuda"); gen.manual_seed(2)
    norm.set_mean_std(np.zeros(M), np.full(M, 2.0))
    x, task = torch.randn(N, M, device="cuda", generator=gen), torch.rand(N, device="cuda", generator=gen)
    g = lambda t: t.detach().float().cpu().numpy()
    tc = TensorCoreMLP(g(disc.hidden[0].weight).T, g(disc.hidden[0].bias), g(disc.hidden[1].weight).T, g(disc.hidden[1].bias), g(disc.logit.weight).T,
                       g(disc.logit.bias), in_mean=g(norm.mean), in_std=g(norm.std), max_rows=N)
    logit, style, reward = (torch.zeros(N, device="cuda") for _ in range(3))

    def gpu_us(f, n=50):
        for _ in range(5): f()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record()
        for _ in range(n): f()
        e1.record(); torch.cuda.synchronize()
        return 1e3 * e0.elapsed_time(e1) / n
    st = torch.cuda.current_stream().cuda_stream
    t_tc = gpu_us(lambda: tc.style_reward(x, reward, task_reward=task, task_lerp=lerp, logit=logit, style=style, stream=st))
    with torch.no_grad():
        t_th = gpu_us(lambda: amp_rewards(disc(norm.normalize(x))[:, 0], task, lerp))
    print("discriminator reward on %d AMP observations (normalise, network, style reward, blend): %.0f us on the wgmma kernels, %.0f us with the fp32 "
          "torch discriminator" % (N, t_tc, t_th))
    assert t_tc < t_th
