"""CPU tests of the PPO learner (deepmimic_b200/learner.py) on the torch backend: one minibatch's actor and critic gradients against a numpy
restatement of PPOAgent's losses, the advantage and target rules, the minibatch schedule, the momentum optimiser, the exploration flag that
collect() records, and the refusals."""
import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from deepmimic_b200.learner import PPOLearner, minibatch_schedule, momentum_step
from deepmimic_b200.rollout import BatchedRollout, build_critic, build_gated_policy, build_policy
from tests.test_rollout_cpu import _FakeEnv
from tests.test_value_targets_cpu import _RewardEnv

HP = dict(actor_stepsize=1e-3, actor_momentum=0.9, actor_weight_decay=5e-3, critic_stepsize=1e-2, critic_momentum=0.9, critic_weight_decay=1e-3,
          ratio_clip=0.2, norm_adv_clip=4.0, minibatch_size=16, epochs=1)


class _FakeLearnEnv(_FakeEnv):
    """_FakeEnv with reward bounds and action bounds (normalised: [-0.2, 0.2] in both dimensions)"""
    get_reward_min, get_reward_max, get_reward_fail, get_reward_succ = (_RewardEnv.get_reward_min, _RewardEnv.get_reward_max,
                                                                          _RewardEnv.get_reward_fail, _RewardEnv.get_reward_succ)

    def build_action_bound_min(self, agent_id=0): return -0.2 / self.build_action_scale() - self.build_action_offset()
    def build_action_bound_max(self, agent_id=0): return 0.2 / self.build_action_scale() - self.build_action_offset()


def _setup(N=8, T=4, goal=0, seed=0, **hp):
    torch.manual_seed(seed)
    env = _FakeLearnEnv(N, goal)
    # sigma 0.5: log-probabilities of order 1, so the fp32 ratio is exact to ~1e-7
    policy = (build_gated_policy(5, goal, 2, noise=0.5, hidden=(32, 16), gate_common=8, gate_hidden=4) if goal
              else build_policy(5, 2, noise=0.5, hidden=(32, 16)))
    with torch.no_grad():
        policy.mean.weight.normal_(0.0, 0.3)
        policy.mean.bias.copy_(torch.tensor([0.3, -0.3]))     # the means fall on both sides of the bounds
    critic = build_critic(5, goal, hidden=(32, 16), gate_common=8, gate_hidden=4)
    ro = BatchedRollout(env, policy=policy, exp_rate=0.5, seed=1, critic=critic, discount=0.95, td_lambda=0.95)
    return ro, PPOLearner(ro, **dict(HP, **hp))


def _window(ro, T, N, seed=0):
    """a synthetic window: random states and actions, returns beyond the value bounds [0, 20], old log-probabilities that put the ratio on both
    sides of the clip range"""
    g = torch.Generator().manual_seed(seed)
    S, A = 5, 2
    traj = dict(states=torch.randn(T, N, S, generator=g), actions=ro.a_norm.unnormalize(0.3 * torch.randn(T, N, A, generator=g)),
                returns=30.0 * torch.rand(T, N, generator=g) - 5.0, values=20.0 * torch.rand(T, N, generator=g),
                explore=torch.rand(T, N, generator=g) < 0.6)
    with torch.no_grad():
        mu = ro.policy(ro.s_norm.normalize(traj["states"]))
        from deepmimic_b200.learner import gaussian_log_prob
        lp = gaussian_log_prob(ro.a_norm.normalize(traj["actions"]), mu, ro.policy.logstd)
    traj["logps"] = lp + 1.2 * (torch.rand(T, N, generator=g) - 0.5)
    return traj


def _np_forward(layers, x):
    hs = [x]
    for W, b in layers[:-1]:
        hs.append(np.maximum(hs[-1] @ W.T + b, 0.0))
    W, b = layers[-1]
    return hs, hs[-1] @ W.T + b


def _np_backward(layers, hs, dy, wd):
    """gradients (dW, db) per layer of sum-over-rows dy at the output, + wd W on the weights"""
    grads = [None] * len(layers)
    for i in range(len(layers) - 1, -1, -1):
        W, _ = layers[i]
        grads[i] = (dy.T @ hs[i] + wd * W, dy.sum(0))
        if i:
            dy = (dy @ W) * (hs[i] > 0)
    return grads


def _np_layers(net, out):
    g = lambda t: t.detach().double().numpy()
    return [(g(l.weight), g(l.bias)) for l in list(net.hidden) + [out]]


def test_one_minibatch_gradients_match_the_numpy_restatement():
    T, N = 8, 16
    ro, ln = _setup(N, T)
    traj = _window(ro, T, N)
    w = ln.window(traj)
    idx = torch.arange(0, 96, 2)
    eidx = w["exp_idx"][:48]
    # actor: numpy restatement of the clipped surrogate + bound loss + weight decay
    x = ro.s_norm.normalize(w["states"][eidx]).double().numpy()
    layers = _np_layers(ro.policy, ro.policy.mean)
    hs, mu = _np_forward(layers, x)
    sig = ro.policy.logstd.detach().exp().double().numpy()
    a = w["norm_a"][eidx].double().numpy()
    logp = (-0.5 * ((a - mu) / sig) ** 2 - np.log(sig) - 0.5 * np.log(2 * np.pi)).sum(1)
    ratio = np.exp(logp - w["old_logp"][eidx].double().numpy())
    adv = w["adv"][eidx].double().numpy()
    eps = HP["ratio_clip"]
    l0, l1 = adv * ratio, adv * np.clip(ratio, 1 - eps, 1 + eps)
    active = (l0 <= l1) | ((ratio >= 1 - eps) & (ratio <= 1 + eps))
    lo, hi = ln.bound_min.double().numpy(), ln.bound_max.double().numpy()
    vmin, vmax = np.minimum(mu - lo, 0), np.maximum(mu - hi, 0)
    # the cases the rule distinguishes are all present
    assert (active & (adv > 0)).any() and (active & (adv < 0)).any() and (~active & (adv > 0)).any() and (~active & (adv < 0)).any()
    assert (vmin < 0).any() and (vmax > 0).any()
    B = len(eidx)
    dmu = (np.where(active, -adv * ratio, 0.0)[:, None] * (a - mu) / sig ** 2 + vmin + vmax) / B
    want = _np_backward(layers, hs, dmu, HP["actor_weight_decay"])
    total, loss, r = ln.actor_loss(w, eidx)
    np.testing.assert_allclose(r.detach().double().numpy(), ratio, rtol=1e-5)
    np.testing.assert_allclose(loss.item(), -np.minimum(l0, l1).mean() + 0.5 * (vmin ** 2 + vmax ** 2).sum(1).mean(), rtol=1e-5)
    got = torch.autograd.grad(total, ln.actor_params)
    names = [n for n, _ in ro.policy.named_parameters() if n != "logstd"]
    assert "logstd" not in names and len(got) == 6
    flat = [g for pair in want for g in pair]
    order = {n: i for i, n in enumerate(["hidden.0.weight", "hidden.0.bias", "hidden.1.weight", "hidden.1.bias", "mean.weight", "mean.bias"])}
    for n, g in zip(names, got):
        ref = flat[order[n]]
        err = np.linalg.norm(g.double().numpy() - ref) / np.linalg.norm(ref)
        assert err <= 1e-5, (n, err)
    # critic: 0.5 mean (norm target - norm V)^2 + weight decay on the weights only
    x = ro.s_norm.normalize(w["states"][idx]).double().numpy()
    layers = _np_layers(ro.critic, ro.critic.out)
    hs, out = _np_forward(layers, x)
    tar = (np.clip(traj["returns"].reshape(-1)[idx].double().numpy(), 0.0, 20.0) - 10.0) / 10.0
    want = _np_backward(layers, hs, (out - tar[:, None]) / len(idx), HP["critic_weight_decay"])
    total, loss = ln.critic_loss(w, idx)
    np.testing.assert_allclose(loss.item(), 0.5 * ((out[:, 0] - tar) ** 2).mean(), rtol=1e-5)
    got = torch.autograd.grad(total, ln.critic_params)
    for g, ref in zip(got, [g for pair in want for g in pair]):
        assert np.linalg.norm(g.double().numpy() - ref) / np.linalg.norm(ref) <= 1e-5
    # a whole update moves every trained parameter and leaves log-std alone
    before = {n: p.detach().clone() for n, p in ro.policy.named_parameters()}
    stats = ln.update(traj)
    assert set(stats) == {"actor_loss", "critic_loss", "clip_frac", "adv_mean", "adv_std", "exp_samples"}
    assert all(s.dim() == 0 for s in stats.values())
    for n, p in ro.policy.named_parameters():
        assert torch.equal(p, before[n]) == (n == "logstd"), n


def test_advantages_use_explored_samples_and_are_clipped():
    T, N = 4, 8
    ro, ln = _setup(N, T, norm_adv_clip=0.5)
    traj = _window(ro, T, N)
    traj["returns"][~traj["explore"]] = 1e4          # unexplored samples must not enter the statistics
    w = ln.window(traj)
    e = traj["explore"].reshape(-1)
    raw = (traj["returns"] - traj["values"]).reshape(-1)[e].double().numpy()
    assert w["adv_mean"].item() == pytest.approx(raw.mean(), rel=1e-5) and w["adv_std"].item() == pytest.approx(raw.std(), rel=1e-5)
    want = np.clip((raw - raw.mean()) / (raw.std() + 1e-5), -0.5, 0.5)
    np.testing.assert_allclose(w["adv"][w["exp_idx"]].numpy(), want, rtol=1e-5, atol=1e-6)
    assert (np.abs(want) == 0.5).any() and torch.equal(w["exp_idx"], e.nonzero()[:, 0])
    # critic targets: the returns clipped to [0, 1] / (1 - 0.95) = [0, 20], in the value normaliser's space (mean 10, std 10)
    ret = traj["returns"].reshape(-1)
    np.testing.assert_allclose(w["norm_tar"].numpy(), ((ret.clamp(0, 20) - 10) / 10).numpy(), rtol=1e-6)
    assert (ret < 0).any() and (ret > 20).any()
    assert w["norm_tar"].min().item() == pytest.approx(-1.0) and w["norm_tar"].max().item() == pytest.approx(1.0)


def test_minibatch_schedule_count_size_wrap_and_reshuffle():
    g = torch.Generator().manual_seed(3)
    mbs = list(minibatch_schedule(10, 5, 4, 2, g))
    assert len(mbs) == 2 * 3 and all(c.shape == (4,) and a.shape == (4,) for c, a in mbs)
    # replay the draws: per epoch a critic and an actor order; the actor's is redrawn after minibatches whose positions wrap
    r = torch.Generator().manual_seed(3)
    cperm, aperm0 = torch.randperm(10, generator=r), torch.randperm(5, generator=r)
    assert torch.equal(mbs[0][0], cperm[[0, 1, 2, 3]]) and torch.equal(mbs[2][0], cperm[[8, 9, 0, 1]])
    assert torch.equal(mbs[0][1], aperm0[[0, 1, 2, 3]])
    assert torch.equal(mbs[1][1], aperm0[[4, 0, 1, 2]])            # wraps: reshuffled afterwards
    aperm1 = torch.randperm(5, generator=r)
    assert torch.equal(mbs[2][1], aperm1[[3, 4, 0, 1]])
    torch.randperm(5, generator=r)                                 # minibatch 2 wrapped too
    cperm_e1, aperm_e1 = torch.randperm(10, generator=r), torch.randperm(5, generator=r)
    assert torch.equal(mbs[3][0], cperm_e1[[0, 1, 2, 3]]) and torch.equal(mbs[3][1], aperm_e1[[0, 1, 2, 3]])
    # fewer samples than rows: one minibatch, positions taken modulo the set sizes
    (c, a), = list(minibatch_schedule(3, 2, 8, 1, torch.Generator().manual_seed(0)))
    assert sorted(np.bincount(c.numpy()).tolist()) == [2, 3, 3] and np.bincount(a.numpy()).tolist() == [4, 4]


def test_two_momentum_steps():
    p, acc = torch.tensor([1.0, -2.0]), torch.zeros(2)
    g1, g2 = torch.tensor([0.5, 1.0]), torch.tensor([-1.0, 2.0])
    momentum_step([p], [acc], [g1], 0.1, 0.9)
    torch.testing.assert_close(acc, g1)
    torch.testing.assert_close(p, torch.tensor([1.0 - 0.05, -2.0 - 0.1]))
    momentum_step([p], [acc], [g2], 0.1, 0.9)
    a2 = 0.9 * g1 + g2
    torch.testing.assert_close(acc, a2)
    torch.testing.assert_close(p, torch.tensor([1.0 - 0.05, -2.0 - 0.1]) - 0.1 * a2)


@pytest.mark.parametrize("rate", [0.0, 1.0, 0.5])
def test_collect_records_the_exploration_draw(rate):
    N, T = 6, 5
    env = _FakeLearnEnv(N, 0)
    torch.manual_seed(0)
    ro = BatchedRollout(env, exp_rate=rate, seed=7)
    traj = ro.collect(T, record_stats=False)
    ex = traj["explore"]
    assert ex.dtype == torch.bool and ex.shape == (T, N)
    if rate == 0.0:
        assert not ex.any()
    elif rate == 1.0:
        assert ex.all()
    else:
        # the rollout draws per step: the exploration uniforms, then the actor's Gaussian noise
        g = torch.Generator().manual_seed(7)
        want = []
        for _ in range(T):
            want.append(torch.rand(N, generator=g) < rate)
            torch.randn(N, 2, generator=g)
        assert torch.equal(ex, torch.stack(want)) and ex.any() and not ex.all()


def test_refusals():
    ro, _ = _setup()
    for key in HP:
        with pytest.raises(ValueError, match=key):
            PPOLearner(ro, **dict(HP, **{key: None}))
    for key, v in (("actor_stepsize", 0.0), ("critic_stepsize", -1.0), ("actor_momentum", 1.0), ("critic_momentum", -0.1),
                   ("actor_weight_decay", -1e-3), ("critic_weight_decay", math.nan), ("ratio_clip", 0.0), ("ratio_clip", 1.0),
                   ("norm_adv_clip", 0.0), ("minibatch_size", 0), ("minibatch_size", 4.0), ("epochs", 0)):
        with pytest.raises(ValueError, match=key):
            PPOLearner(ro, **dict(HP, **{key: v}))
    with pytest.raises(ValueError, match="backend"):
        PPOLearner(ro, **HP, backend="cublas")
    with pytest.raises(ValueError, match="critic"):
        PPOLearner(BatchedRollout(_FakeLearnEnv(4, 0)), **HP)
    ro, ln = _setup()
    traj = _window(ro, 4, 8)
    for key in ("returns", "explore"):
        with pytest.raises(ValueError, match=key):
            ln.update({k: v for k, v in traj.items() if k != key})
    traj["explore"][:] = False
    with pytest.raises(ValueError, match="explored"):
        ln.update(traj)
    gro, _ = _setup(goal=3)
    with pytest.raises(ValueError, match="plain"):
        PPOLearner(gro, **HP, backend="tensor_core")


def test_gated_update_on_the_torch_backend():
    """the goal-conditioned networks train on the torch backend: every trained parameter moves, the losses are finite"""
    ro, ln = _setup(goal=3)
    traj = ro.collect(4)
    before = [p.detach().clone() for p in ln.actor_params + ln.critic_params]
    stats = ln.update(traj)
    assert all(math.isfinite(v.item()) for v in stats.values())
    moved = [not torch.equal(p, b) for p, b in zip(ln.actor_params + ln.critic_params, before)]
    assert sum(moved) >= len(moved) - 2     # gate layers whose relu is closed on every row may not move


def test_replaced_parameters_and_non_device_tensors_are_refused():
    """a network whose parameters were replaced after the learner was built is refused at update(); the C ABI's device pointers need
    contiguous float32 CUDA tensors"""
    from deepmimic_b200.capi import _check_device_f32
    ro, ln = _setup()
    traj = _window(ro, 4, 8)
    ro.critic.out.weight = torch.nn.Parameter(ro.critic.out.weight.detach().clone())
    with pytest.raises(ValueError, match="replaced"):
        ln.update(traj)
    for t in (torch.zeros(3), [0.0] * 3):
        with pytest.raises(ValueError, match="float32 CUDA"):
            _check_device_f32(t, "test")
