"""PPO value targets on the GPU: the TD(lambda) return scan (dm_td_lambda_returns, kernels/dm_returns.cu) against the path-by-path numpy restatement
of the reference's compute_return (tests/test_value_targets_cpu.py), the critic on the tensor cores (plain and gated dm_mlp handles with one output
and the value normaliser) against the fp32 torch critic, and both through BatchedRollout(critic=...).collect on both backends."""
import contextlib
import ctypes as C
import math

import numpy as np
import pytest

from tests.test_value_targets_cpu import path_returns, synthetic_window

pytestmark = pytest.mark.gpu
SPINKICK = ["--arg_file", "args/train_humanoid3d_spinkick_args.txt"]
DOG = ["--arg_file", "args/train_dog3d_trot_args.txt"]
TARGET = ["--motion_file", "data/datasets/test_clips_mini.txt", "--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]


@contextlib.contextmanager
def _no_tf32():
    import torch
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def _cuda(*arrays):
    import torch
    return [torch.as_tensor(a).cuda().contiguous() for a in arrays]


@pytest.mark.parametrize("gamma", [0.0, 0.95])
def test_return_kernel_matches_the_restatement(gamma):
    """[600, 4096] synthetic window with Null, Fail and Succ ends and paths cut by the window, lambda 0, 0.95 and 1"""
    import torch
    from deepmimic_b200.capi import td_lambda_returns
    T, N = 600, 4096
    r, v, ev, done, term = synthetic_window(np.random.default_rng(int(gamma * 100)), T, N, p_done=0.02)
    assert all((done & (term == c)).sum() > 1000 for c in (0, 1, 2))
    vf, vs = (0.0, 0.0) if gamma == 0 else (0.0, 1.0 / (1.0 - gamma))
    tr, tv, tev, tdone, tterm = _cuda(r, v, ev, done, term)
    for lam in (0.0, 0.95, 1.0):
        ret, adv = torch.full((T, N), 7.0, device="cuda"), torch.full((T, N), 7.0, device="cuda")
        td_lambda_returns(tr, tv, tev, tdone, tterm, gamma, lam, vf, vs, ret, adv)
        torch.cuda.synchronize()
        want = path_returns(r, v, ev, done, term, gamma, lam, vf, vs)
        bound = 1e-5 * max(1.0, 1.0 / (1.0 - gamma))
        err, err_a = np.abs(ret.cpu().numpy() - want).max(), np.abs(adv.cpu().numpy() - (want - v)).max()
        print("gamma %.2f lambda %.2f: max return error %.2e, advantage error %.2e (bound %.1e)" % (gamma, lam, err, err_a, bound))
        assert err <= bound and err_a <= bound


def test_return_kernel_refusals():
    """errors through dm_last_error: T or N <= 0, discount outside [0, 1), lambda outside [0, 1] (NaN included), NULL pointers"""
    import torch
    from deepmimic_b200 import capi
    T, N = 4, 8
    f = torch.zeros(T, N, device="cuda")
    d, tm = torch.zeros(T, N, dtype=torch.bool, device="cuda"), torch.zeros(T, N, dtype=torch.int32, device="cuda")
    L, p = capi.lib(), lambda t: None if t is None else C.c_void_p(t.data_ptr())
    call = lambda T=T, N=N, g=0.9, lam=0.9, rew=f, out=f: L.dm_td_lambda_returns(p(rew), p(f), p(f), p(d), p(tm), T, N, g, lam, 0.0, 1.0, p(out), p(f), None)
    for kw, msg in ((dict(T=0), b"T and N"), (dict(N=-1), b"T and N"), (dict(g=1.0), b"discount"), (dict(g=-0.1), b"discount"), (dict(g=math.nan), b"discount"),
                    (dict(lam=1.5), b"td_lambda"), (dict(lam=-0.1), b"td_lambda"), (dict(lam=math.nan), b"td_lambda"), (dict(rew=None), b"null pointer"),
                    (dict(out=None), b"null pointer")):
        assert call(**kw) != 0 and msg in L.dm_last_error(), kw
    assert call() == 0 and call(g=0.0, lam=1.0) == 0
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="discount"):
        capi.td_lambda_returns(f, f, f, d, tm, 1.0, 0.9, 0.0, 1.0, f, f)
    with pytest.raises(ValueError, match="terminate"):
        capi.td_lambda_returns(f, f, f, d, tm.long(), 0.9, 0.9, 0.0, 1.0, f, f)


def _rollout(asset_root, args, n, backend, seed=11, critic_seed=0, limits=(0.5, 3.0), with_disc=False):
    """BatchedRollout with a random critic (and the env's random-initialised actor, noise 0.5: the characters fall) over n environments whose
    episodes end by time limit after limits[0] .. limits[1] seconds; with_disc: a random AMP discriminator, task_reward_lerp 0.5"""
    import torch
    from deepmimic_b200.env import DeepMimicBatchEnv
    from deepmimic_b200.rollout import BatchedRollout, build_critic, build_discriminator
    env = DeepMimicBatchEnv(args, num_envs=n, asset_root=asset_root, seed=seed)
    env._core.set_episode_limit(*limits)
    env.reset(True)
    torch.manual_seed(critic_seed)
    critic = build_critic(env.get_state_size(), env.get_goal_size())
    kw = dict(disc=build_discriminator(env.get_amp_obs_size()), task_reward_lerp=0.5) if with_disc else {}
    return env, BatchedRollout(env, noise=0.5, backend=backend, critic=critic, discount=0.95, td_lambda=0.95, **kw)


def _torch_values(ro, s, g=None):
    import torch
    with torch.no_grad(), _no_tf32():
        ns = ro.s_norm.normalize(s)
        out = ro.critic(ns) if g is None else ro.critic(ns, ro.g_norm.normalize(g))
        return ro.val_norm.unnormalize(out)[..., 0]


@pytest.mark.parametrize("scene,args,width,goal", [("spinkick", SPINKICK, 227, 0), ("dog3d trot", DOG, 347, 0), ("target_amp", TARGET, 226, 3)])
def test_tensor_core_critic_matches_fp32(asset_root, scene, args, width, goal):
    """4096 simulated states (two steps of 2048 environments under random actions), the critic on the wgmma kernels against the fp32 torch
    critic, both behind the rollout's state normaliser: normalised value error <= 1e-3 max(1, max |normalised value|), the actors' bound
    (tests/test_mlp_gpu.py) for outputs of magnitude up to 1, and relative to the output beyond (the fp16 activations carry a relative error)"""
    import torch
    env, ro = _rollout(asset_root, args, 2048, "tensor_core", limits=(20.0, 20.0))
    traj = ro.collect(6, record_stats=False)
    s = traj["states"][-2:].reshape(4096, width).contiguous()
    g = traj["goals"][-2:].reshape(4096, goal).contiguous() if goal else None
    assert s.shape == (4096, width)
    v = torch.full((4096,), 7.0, device="cuda")
    ro._critic_values(s, g, v)
    torch.cuda.synchronize()
    ref = _torch_values(ro, s, g)
    err = ((v - ref).abs() / ro.val_norm.std).max().item()
    bound = 1e-3 * max(1.0, ((ref - ro.val_norm.mean) / ro.val_norm.std).abs().max().item())
    print("%s critic, 4096 states of width %d (+ %d goal): normalised value error %.2e (bound %.2e); values in [%.2f, %.2f]"
          % (scene, width, goal, err, bound, ref.min().item(), ref.max().item()))
    assert err <= bound and ref.std().item() > 1e-2
    assert env.counters()[1] == 0


@pytest.mark.parametrize("scene,args", [("spinkick", SPINKICK), ("target_amp", TARGET)])
@pytest.mark.parametrize("backend", ["torch", "tensor_core"])
def test_rollout_value_targets(asset_root, scene, args, backend):
    """BatchedRollout(critic=...), 64 environments x 600 steps with Null (time limit) and Fail (fall) ends: end_values continues values where a path
    goes on, is the critic of the pre-reset state where it ends, and the returns are the restatement's; with a discriminator they run over
    amp_rewards"""
    import torch
    N, T = 64, 600
    amp = scene == "target_amp"
    env, ro = _rollout(asset_root, args, N, backend, with_disc=amp)
    traj = ro.collect(T, record_stats=False)
    torch.cuda.synchronize()
    done, term = traj["dones"], traj["terminate"]
    n_null, n_fail = int((done & (term == 0)).sum()), int((done & (term == 1)).sum())
    assert env.counters()[1] == 0 and n_null > 0 and n_fail > 0
    v, ev = traj["values"], traj["end_values"]
    cont = ~done[:-1]
    if backend == "tensor_core":
        assert torch.equal(ev[:-1][cont], v[1:][cont])          # a row's value does not depend on the other rows of the forward
    else:
        assert (ev[:-1][cont] - v[1:][cont]).abs().max().item() <= 1e-5 * max(1.0, v.abs().max().item())
    # the pre-reset states (and goals) of the same actions through a hand-written step / record / reset loop on a second handle with the same seed
    env2 = _rollout(asset_root, args, N, backend)[0]
    ends_s, ends_g = [], []
    for k in range(T):
        s2, _, d2, _ = env2.step(traj["actions"][k].contiguous())
        assert torch.equal(d2, done[k])
        ends_s.append(s2[d2].clone())
        if env2.get_goal_size():
            ends_g.append(env2.record_goal()[d2].clone())
        env2.reset()
    torch.cuda.synchronize()
    assert env2.counters()[1] == 0
    want = _torch_values(ro, torch.cat(ends_s), torch.cat(ends_g) if ends_g else None)
    got = ev[done]                                              # row-major order of (k, n) = the loop's order
    # tensor cores: the critic test's bound, 1e-3 of the value normaliser's std per unit of the largest normalised value
    tol = (1e-3 * ro.val_norm.std.item() * max(1.0, ((want - ro.val_norm.mean) / ro.val_norm.std).abs().max().item()) if backend == "tensor_core"
           else 1e-5 * max(1.0, want.abs().max().item()))
    err = (got - want).abs().max().item()
    rewards = traj["amp_rewards"] if amp else traj["rewards"]
    ret = path_returns(rewards.cpu().numpy(), v.cpu().numpy(), ev.cpu().numpy(), done.cpu().numpy(), term.cpu().numpy(), 0.95, 0.95, ro.val_fail, ro.val_succ)
    err_r = np.abs(traj["returns"].cpu().numpy() - ret).max()
    print("%s, %s backend, %d x %d steps: %d null and %d fail ends; end-value error %.2e (bound %.1e; values in [%.1f, %.1f]), return error %.2e, mean return %.2f"
          % (scene, backend, N, T, n_null, n_fail, err, tol, v.min().item(), v.max().item(), err_r, traj["returns"].mean().item()))
    assert err <= tol and err_r <= 1e-5 * 20
    torch.testing.assert_close(traj["advantages"], traj["returns"] - v, rtol=0, atol=1e-5)
    if amp:
        other = path_returns(traj["rewards"].cpu().numpy(), v.cpu().numpy(), ev.cpu().numpy(), done.cpu().numpy(), term.cpu().numpy(), 0.95, 0.95, 0.0, 20.0)
        assert np.abs(other - ret).max() > 1e-2


def _gpu_us(f, n=30):
    import torch
    for _ in range(3):
        f()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(n):
        f()
    e1.record(); torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / n


def test_value_targets_time():
    """device clock: the tensor-core critic step (8192 rows, [s_k; s'_k] of 4096 environments) against the torch critic, and the return kernel
    against a torch loop over T, at T x N = 600 x 4096"""
    import torch
    from deepmimic_b200.capi import TensorCoreMLP, td_lambda_returns
    from deepmimic_b200.rollout import DeviceNormalizer, build_critic, td_lambda_returns_host
    N, S = 4096, 227
    torch.manual_seed(0)
    critic = build_critic(S).cuda()
    norm, vnorm = DeviceNormalizer(S, device="cuda"), DeviceNormalizer(1, device="cuda")
    norm.set_mean_std(np.zeros(S), np.full(S, 2.0)); vnorm.set_mean_std([10.0], [10.0])
    g = lambda t: t.detach().float().cpu().numpy()
    wb = lambda l: (g(l.weight).T, g(l.bias))
    tc = TensorCoreMLP(*wb(critic.hidden[0]), *wb(critic.hidden[1]), *wb(critic.out), in_mean=g(norm.mean), in_std=g(norm.std), out_mean=[10.0], out_std=[10.0], max_rows=2 * N)
    x, v = torch.randn(2 * N, S, device="cuda"), torch.zeros(2 * N, 1, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    t_tc = _gpu_us(lambda: tc.forward(x, v, stream=st))
    with torch.no_grad():
        t_th = _gpu_us(lambda: vnorm.unnormalize(critic(norm.normalize(x))))
    T = 600
    r, vv, ev, done, term = _cuda(*synthetic_window(np.random.default_rng(0), T, N))
    ret, adv = torch.empty(T, N, device="cuda"), torch.empty(T, N, device="cuda")
    t_k = _gpu_us(lambda: td_lambda_returns(r, vv, ev, done, term, 0.95, 0.95, 0.0, 20.0, ret, adv, stream=st))
    ret2, adv2 = torch.empty_like(ret), torch.empty_like(adv)
    t_loop = _gpu_us(lambda: td_lambda_returns_host(r, vv, ev, done, term, 0.95, 0.95, 0.0, 20.0, ret2, adv2), n=3)
    torch.cuda.synchronize()
    assert (ret - ret2).abs().max().item() <= 1e-4
    print("critic on %d rows: %.0f us on the wgmma kernels, %.0f us with the fp32 torch critic; returns of %d x %d: %.0f us kernel, %.0f us torch loop over T"
          % (2 * N, t_tc, t_th, T, N, t_k, t_loop))
    assert t_tc < t_th and t_k < t_loop
