"""The PPO learner on the GPU: the tensor-core minibatch step (dm_learn_step: kernels/dm_learn.cu and the backward GEMMs of kernels/dm_mlp.cu)
against fp32 torch autograd (TF32 off), whole updates on both backends, determinism, the re-tiling of the rollout's handles, the direction of
the steps and the update time."""
import contextlib
import copy
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
SPINKICK = ["--arg_file", "args/train_humanoid3d_spinkick_args.txt"]
DOG = ["--arg_file", "args/train_dog3d_trot_args.txt"]
HP = dict(actor_stepsize=2.5e-6, actor_momentum=0.9, actor_weight_decay=5e-4, critic_stepsize=1e-2, critic_momentum=0.9, critic_weight_decay=1e-3,
          ratio_clip=0.2, norm_adv_clip=4.0, epochs=1)


@contextlib.contextmanager
def _no_tf32():
    import torch
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def _rollout(asset_root, args, n, backend, pretrained=False, seed=11):
    """BatchedRollout with a random critic; the actor is the pretrained spin-kick fixture or the env's random one (noise 0.2)"""
    import torch
    from deepmimic_b200.env import DeepMimicBatchEnv
    from deepmimic_b200.rollout import BatchedRollout, build_critic, load_actor_weights
    env = DeepMimicBatchEnv(args, num_envs=n, asset_root=asset_root, seed=seed)
    env._core.set_episode_limit(0.5, 3.0)
    env.reset(True)
    torch.manual_seed(0)
    critic = build_critic(env.get_state_size())
    ro = BatchedRollout(env, noise=0.2, exp_rate=0.8, backend=backend, critic=critic, discount=0.95, td_lambda=0.95, seed=seed)
    if pretrained:
        f = np.load(os.path.join(GOLD, "policy_humanoid3d_spinkick_fp16.npz"))
        load_actor_weights(ro.policy, {k: f[k].astype(np.float32) for k in f.files})
        ro.s_norm.set_mean_std(f["s_mean"].astype(np.float32), f["s_std"].astype(np.float32))
    return env, ro


class _ShapeEnv:
    """a stand-in env on the GPU with arbitrary sizes: enough surface for BatchedRollout's and PPOLearner's constructors"""

    def __init__(self, n, S, A):
        import torch
        self.num_envs, self.device, self.S, self.A = n, torch.device("cuda", 0), S, A

    def get_state_size(self, agent_id=0): return self.S
    def get_action_size(self, agent_id=0): return self.A
    def get_goal_size(self, agent_id=0): return 0
    def build_state_norm_groups(self, agent_id=0): return np.zeros(self.S, dtype=np.int32)
    def build_state_offset(self, agent_id=0): return np.full(self.S, 0.1)
    def build_state_scale(self, agent_id=0): return np.full(self.S, 0.5)
    def build_action_offset(self, agent_id=0): return np.zeros(self.A)
    def build_action_scale(self, agent_id=0): return np.ones(self.A)
    def build_action_bound_min(self, agent_id=0): return np.full(self.A, -0.5)
    def build_action_bound_max(self, agent_id=0): return np.full(self.A, 0.5)
    def get_reward_min(self, agent_id=0): return 0.0
    def get_reward_max(self, agent_id=0): return 1.0
    def get_reward_fail(self, agent_id=0): return 0.0
    def get_reward_succ(self, agent_id=0): return 1.0


def _random_shapes(S=100, A=5, hidden=(200, 96), T=4, N=150):
    import torch
    from deepmimic_b200.learner import gaussian_log_prob
    from deepmimic_b200.rollout import BatchedRollout, build_critic, build_policy
    torch.manual_seed(1)
    env = _ShapeEnv(N, S, A)
    ro = BatchedRollout(env, policy=build_policy(S, A, noise=0.3, init_output_scale=0.3, hidden=hidden), critic=build_critic(S, hidden=hidden),
                        discount=0.95, td_lambda=0.95, seed=2)
    g = torch.Generator(device="cuda").manual_seed(3)
    traj = dict(states=torch.randn(T, N, S, device="cuda", generator=g), actions=0.4 * torch.randn(T, N, A, device="cuda", generator=g),
                returns=25.0 * torch.rand(T, N, device="cuda", generator=g) - 2.0, values=20.0 * torch.rand(T, N, device="cuda", generator=g),
                explore=torch.rand(T, N, device="cuda", generator=g) < 0.7)
    with torch.no_grad():
        traj["logps"] = gaussian_log_prob(ro.a_norm.normalize(traj["actions"]), ro.policy(ro.s_norm.normalize(traj["states"])), ro.policy.logstd)
        traj["logps"] += 0.5 * (torch.rand(T, N, device="cuda", generator=g) - 0.5)
    return ro, traj


def _window(asset_root, case):
    if case == "random shapes":
        return _random_shapes()
    env, ro = _rollout(asset_root, SPINKICK if case == "spinkick" else DOG, 512, "torch", pretrained=case == "spinkick")
    return ro, ro.collect(16)


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _fp16_activation_grads(ln, w, c, a):
    """fp32 torch autograd of the same losses through a forward whose normalised input and hidden activations are rounded to fp16, as the
    tensor-core forward stores them (the weights stay fp32: the kernels carry them as hi + lo)"""
    import torch
    from deepmimic_b200.learner import bound_loss, clipped_surrogate, critic_loss, gaussian_log_prob, weight_decay_loss
    ro = ln.ro
    r16 = lambda x: x.half().float()

    def fwd(net, out, idx):
        h = r16(ro.s_norm.normalize(w["states"][idx]))
        for l in net.hidden:
            h = r16(torch.relu(l(h)))
        return out(h)
    lc = critic_loss(fwd(ro.critic, ro.critic.out, c)[:, 0], w["norm_tar"][c]) + ln.critic_weight_decay * weight_decay_loss(ro.critic)
    mu = fwd(ro.policy, ro.policy.mean, a)
    ratio = (gaussian_log_prob(w["norm_a"][a], mu, ro.policy.logstd.detach()) - w["old_logp"][a]).exp()
    la = (-clipped_surrogate(w["adv"][a], ratio, ln.ratio_clip).mean() + bound_loss(mu, ln.bound_min, ln.bound_max)
          + ln.actor_weight_decay * weight_decay_loss(ro.policy))
    return torch.autograd.grad(lc, ln.critic_params) + torch.autograd.grad(la, ln.actor_params)


@pytest.mark.parametrize("case,B", [("spinkick", 4096), ("dog3d trot", 2048), ("random shapes", 200)])
def test_minibatch_gradients_match_fp32(asset_root, case, B):
    """one critic step and one actor step at stepsize 1 and momentum 0 (w -= g) from zero accumulators: g = w_before - w_after against fp32 torch
    autograd of the same minibatch.  Against the same arithmetic with fp16-rounded activations (what the kernels compute), relative Frobenius
    error per parameter tensor <= 1e-2.  Against the plain fp32 network the fp16 activations themselves show: the actor's gradient carries the
    forward's error in mu amplified by (a - mu) / sigma^2 (2e-2 on the pretrained spin-kick actor, 7e-2 on a random network), and a random
    network on random targets has a first-layer gradient that is mostly cancellation (2.8e-2 for its critic); bound 1e-1"""
    import torch
    from deepmimic_b200.learner import PPOLearner
    ro, traj = _window(asset_root, case)
    hp = dict(HP, actor_stepsize=1.0, actor_momentum=0.0, critic_stepsize=1.0, critic_momentum=0.0, minibatch_size=B)
    ln = PPOLearner(ro, **hp, backend="tensor_core")
    w = ln.window(traj)
    g = torch.Generator(device="cuda").manual_seed(5)
    c = torch.randint(0, w["R"], (B,), device="cuda", generator=g)
    a = w["exp_idx"][torch.randint(0, w["exp_idx"].numel(), (B,), device="cuda", generator=g)]
    with _no_tf32():
        ref = torch.autograd.grad(ln.critic_loss(w, c)[0], ln.critic_params) + torch.autograd.grad(ln.actor_loss(w, a)[0], ln.actor_params)
        ref16 = _fp16_activation_grads(ln, w, c, a)
    params = ln.critic_params + ln.actor_params
    before = [p.detach().clone() for p in params]
    st = torch.cuda.current_stream().cuda_stream
    ln._tc_critic.set_weights(stream=st); ln._tc_actor.set_weights(stream=st)
    ln.minibatch_step(w, c, a, None, ln._tc_batch(w))
    torch.cuda.synchronize()
    errs = [_rel(b - p.detach(), r) for b, p, r in zip(before, params, ref)]
    errs16 = [_rel(b - p.detach(), r) for b, p, r in zip(before, params, ref16)]
    names = ["critic." + n for n, _ in ro.critic.named_parameters()] + ["actor." + n for n, p in ro.policy.named_parameters() if n != "logstd"]
    print("%s, B = %d: relative gradient error per tensor vs fp16-activation / plain fp32 torch: %s"
          % (case, B, ", ".join("%s %.1e / %.1e" % (n, e16, e) for n, e16, e in zip(names, errs16, errs))))
    assert max(errs16) <= 1e-2 and max(errs) <= 1e-1


@pytest.mark.parametrize("rows", [2176, 3000, 200])
def test_minibatch_smaller_than_the_workspace(asset_root, rows):
    """a workspace built for 4096 rows steps a smaller minibatch (the dW split count of such a row count can exceed that of 4096 rows: 17 against
    16 splits for the first layer at 2176 rows): gradients against the fp16-activation reference <= 1e-2"""
    import torch
    from deepmimic_b200.learner import PPOLearner
    ro, traj = _window(asset_root, "spinkick")
    hp = dict(HP, actor_stepsize=1.0, actor_momentum=0.0, critic_stepsize=1.0, critic_momentum=0.0, minibatch_size=4096)
    ln = PPOLearner(ro, **hp, backend="tensor_core")
    w = ln.window(traj)
    g = torch.Generator(device="cuda").manual_seed(rows)
    c = torch.randint(0, w["R"], (rows,), device="cuda", generator=g)
    a = w["exp_idx"][torch.randint(0, w["exp_idx"].numel(), (rows,), device="cuda", generator=g)]
    with _no_tf32():
        ref16 = _fp16_activation_grads(ln, w, c, a)
    params = ln.critic_params + ln.actor_params
    before = [p.detach().clone() for p in params]
    st = torch.cuda.current_stream().cuda_stream
    ln._tc_critic.set_weights(stream=st); ln._tc_actor.set_weights(stream=st)
    keep, actor, critic = ln._tc_batch(w)
    actor.rows = critic.rows = rows
    ln.minibatch_step(w, c, a, None, (keep, actor, critic))
    torch.cuda.synchronize()
    errs16 = [_rel(b - p.detach(), r) for b, p, r in zip(before, params, ref16)]
    print("%d rows in a 4096-row workspace: worst relative gradient error vs the fp16-activation reference %.1e" % (rows, max(errs16)))
    assert max(errs16) <= 1e-2


def test_update_on_both_backends_agrees(asset_root):
    """a whole update() of a 16-step window of 4096 environments, minibatch 4096, same seed, from the same weights on both backends: per tensor
    |w_tc - w_torch| <= 5e-2 |w_torch - w_0| (the actor's fp16-forward deviation of test_minibatch_gradients_match_fp32; measured 2.8e-2 on the
    first layer), statistics within 2e-2"""
    import torch
    from deepmimic_b200.learner import PPOLearner, clip_fraction
    env, ro = _rollout(asset_root, SPINKICK, 4096, "torch", pretrained=True)
    traj = ro.collect(16)
    w0 = {k: v.detach().clone() for k, v in list(ro.policy.state_dict().items()) + [("critic." + k, v) for k, v in ro.critic.state_dict().items()]}
    ln = PPOLearner(ro, **HP, minibatch_size=4096, seed=3)
    # the rollout and the learner see the same actor: the first minibatch's ratio is 1 and nothing is clipped
    with _no_tf32():
        wnd = ln.window(traj)
        _, _, ratio = ln.actor_loss(wnd, wnd["exp_idx"][:4096])
    r_err = (ratio - 1).abs().max().item()
    assert clip_fraction(ratio, ln.ratio_clip).item() == 0.0
    with _no_tf32():
        s_th = ln.update(traj)
    w_th = {k: v.detach().clone() for k, v in list(ro.policy.state_dict().items()) + [("critic." + k, v) for k, v in ro.critic.state_dict().items()]}
    ro.policy.load_state_dict({k: v for k, v in w0.items() if not k.startswith("critic.")})
    ro.critic.load_state_dict({k[7:]: v for k, v in w0.items() if k.startswith("critic.")})
    s_tc = PPOLearner(ro, **HP, minibatch_size=4096, seed=3, backend="tensor_core").update(traj)
    torch.cuda.synchronize()
    w_tc = {k: v.detach().clone() for k, v in list(ro.policy.state_dict().items()) + [("critic." + k, v) for k, v in ro.critic.state_dict().items()]}
    worst = 0.0
    for k in w0:
        moved = (w_th[k] - w0[k]).norm().item()
        if k.endswith("logstd"):
            assert moved == 0.0 and torch.equal(w_tc[k], w0[k])
            continue
        e = (w_tc[k] - w_th[k]).norm().item() / moved
        worst = max(worst, e)
        assert e <= 5e-2, (k, e)
    print("update of 16 x 4096: first-minibatch |ratio - 1| %.1e; weights: worst |w_tc - w_torch| / |w_torch - w_0| %.1e; torch %s; tensor cores %s"
          % (r_err, worst, {k: round(v.item(), 5) for k, v in s_th.items()}, {k: round(v.item(), 5) for k, v in s_tc.items()}))
    assert r_err <= 1e-5
    for k in s_th:
        assert abs(s_tc[k].item() - s_th[k].item()) <= 2e-2 * max(abs(s_th[k].item()), 1e-2), k


def test_first_minibatch_ratio_on_a_tensor_core_rollout(asset_root):
    """a tensor-core rollout and a tensor-core learner see the same actor: the first minibatch's probability ratios (dm_learn_batch.ratio) are 1
    to 1e-5 and nothing is clipped"""
    import torch
    from deepmimic_b200.learner import PPOLearner
    env, ro = _rollout(asset_root, SPINKICK, 2048, "tensor_core", pretrained=True)
    traj = ro.collect(8, record_stats=False)
    ln = PPOLearner(ro, **HP, minibatch_size=2048, backend="tensor_core")
    w = ln.window(traj)
    ratio = torch.full((2048,), 7.0, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    ln._tc_critic.set_weights(stream=st); ln._tc_actor.set_weights(stream=st)
    tc = ln._tc_batch(w, ratio=ratio)
    ln.minibatch_step(w, torch.arange(2048, device="cuda"), w["exp_idx"][:2048].contiguous(), None, tc)
    torch.cuda.synchronize()
    r_err = (ratio - 1).abs().max().item()
    print("tensor-core rollout and learner: first-minibatch |ratio - 1| %.1e, clip fraction %g" % (r_err, tc[0]["stats_a"][1].item()))
    assert r_err <= 1e-5 and tc[0]["stats_a"][1].item() == 0.0


def test_tensor_core_update_is_deterministic_and_refreshes_the_rollout(asset_root):
    """two tensor-core updates from the same weights and seed: bit-identical parameters and statistics; after update() the rollout's
    tensor-core actor and critic give bit-identical outputs to handles built afresh from the updated torch modules and the state normaliser
    that the caller updated before update()"""
    import torch
    from deepmimic_b200.learner import PPOLearner
    env, ro = _rollout(asset_root, SPINKICK, 2048, "tensor_core", pretrained=True)
    traj = ro.collect(8)
    mean0 = ro.s_norm.mean.clone()
    ro.s_norm.update()                       # the statistics the rollout's handles were built with are now stale
    assert not torch.equal(mean0, ro.s_norm.mean)
    p0, c0 = copy.deepcopy(ro.policy.state_dict()), copy.deepcopy(ro.critic.state_dict())
    runs = []
    for _ in range(2):
        ro.policy.load_state_dict(p0); ro.critic.load_state_dict(c0)
        s = PPOLearner(ro, **HP, minibatch_size=2048, seed=9, backend="tensor_core").update(traj)
        torch.cuda.synchronize()
        runs.append(([p.detach().clone() for p in list(ro.policy.parameters()) + list(ro.critic.parameters())], {k: v.clone() for k, v in s.items()}))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0]))
    assert all(torch.equal(runs[0][1][k], runs[1][1][k]) for k in runs[0][1])
    assert any(not torch.equal(a, p0[k]) for k, a in zip(p0, runs[0][0]))
    # the handles re-tiled by update() against fresh ones
    s = traj["states"][-1].contiguous()
    st = torch.cuda.current_stream().cuda_stream
    a1, v1 = torch.empty(2048, env.get_action_size(), device="cuda"), torch.empty(2048, 1, device="cuda")
    ro._tc.forward(s, a1, stream=st); ro._tc_critic.forward(s, v1, stream=st)
    ro.refresh_tensor_core_policy()
    a2, v2 = torch.empty_like(a1), torch.empty_like(v1)
    ro._tc.forward(s, a2, stream=st); ro._tc_critic.forward(s, v2, stream=st)
    torch.cuda.synchronize()
    assert torch.equal(a1, a2) and torch.equal(v1, v2)


@pytest.mark.parametrize("backend", ["torch", "tensor_core"])
def test_steps_go_downhill(asset_root, backend):
    """one actor step on a minibatch raises its clipped surrogate; 50 critic steps on a fixed minibatch lower the critic loss"""
    import torch
    from deepmimic_b200.learner import PPOLearner, clipped_surrogate, gaussian_log_prob
    env, ro = _rollout(asset_root, SPINKICK, 2048, "torch", pretrained=True)
    traj = ro.collect(4)
    ln = PPOLearner(ro, **dict(HP, actor_stepsize=1e-4, actor_weight_decay=0.0, critic_weight_decay=0.0), minibatch_size=2048, backend=backend)
    w = ln.window(traj)
    a = w["exp_idx"][:2048]
    c = torch.arange(2048, device="cuda")

    def surrogate():
        with torch.no_grad(), _no_tf32():
            mu = ro.policy(ro.s_norm.normalize(w["states"][a]))
            ratio = (gaussian_log_prob(w["norm_a"][a], mu, ro.policy.logstd) - w["old_logp"][a]).exp()
            return clipped_surrogate(w["adv"][a], ratio, ln.ratio_clip).mean().item()

    def closs():
        with torch.no_grad(), _no_tf32():
            return ln.critic_loss(w, c)[1].item()
    st = torch.cuda.current_stream().cuda_stream
    tc = None
    if backend == "tensor_core":
        ln._tc_critic.set_weights(stream=st); ln._tc_actor.set_weights(stream=st)
        tc = ln._tc_batch(w)
    stats = [torch.zeros((), device="cuda") for _ in range(3)]
    s0, l0 = surrogate(), closs()
    with _no_tf32():
        ln.minibatch_step(w, c, a, stats, tc)
    s1 = surrogate()
    for _ in range(49):
        with _no_tf32():
            ln.minibatch_step(w, c, a, stats, tc)
    l1 = closs()
    print("%s: surrogate %.6f -> %.6f after one step; critic loss %.4f -> %.4f after 50 steps" % (backend, s0, s1, l0, l1))
    assert s1 > s0 and l1 < l0


def _gpu_ms(f, n=5):
    import torch
    for _ in range(2):
        f()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(n):
        f()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def test_update_time():
    """device clock: one update() of a 32 x 4096 window (227 inputs, 28 actions), minibatch 4096, on both backends"""
    import torch
    from deepmimic_b200.learner import PPOLearner
    from deepmimic_b200.rollout import BatchedRollout, build_critic, build_policy
    from deepmimic_b200.learner import gaussian_log_prob
    T, N, S, A = 32, 4096, 227, 28
    torch.manual_seed(0)
    env = _ShapeEnv(N, S, A)
    ro = BatchedRollout(env, policy=build_policy(S, A), critic=build_critic(S), discount=0.95, td_lambda=0.95)
    g = torch.Generator(device="cuda").manual_seed(0)
    traj = dict(states=torch.randn(T, N, S, device="cuda", generator=g), actions=0.05 * torch.randn(T, N, A, device="cuda", generator=g),
                returns=20.0 * torch.rand(T, N, device="cuda", generator=g), values=20.0 * torch.rand(T, N, device="cuda", generator=g),
                explore=torch.rand(T, N, device="cuda", generator=g) < 0.8)
    with torch.no_grad():
        traj["logps"] = gaussian_log_prob(traj["actions"], ro.policy(ro.s_norm.normalize(traj["states"])), ro.policy.logstd)
    times = {}
    for backend in ("torch", "tensor_core"):
        ln = PPOLearner(ro, **HP, minibatch_size=4096, backend=backend)
        with _no_tf32():
            times[backend] = _gpu_ms(lambda: ln.update(traj), n=3)
    print("update of a %d x %d window, minibatch 4096: %.1f ms fp32 torch, %.1f ms tensor cores" % (T, N, times["torch"], times["tensor_core"]))
    assert times["tensor_core"] < times["torch"]
