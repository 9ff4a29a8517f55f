"""CPU tests of the AMP discriminator's update (deepmimic_b200/learner.py: AMPDiscLearner and its rules) on the torch backend: the rules against
numpy restatements, the closed-form gradient-penalty decomposition that the tensor-core step implements against torch's double backward, the
refusals, reproducibility and the direction of the steps."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
from deepmimic_b200.learner import (AMPDiscLearner, disc_accuracies, disc_grad_penalty, disc_input_grad, disc_logit_reg_loss, disc_loss,
                                    disc_weight_decay_loss)
from deepmimic_b200.rollout import BatchedRollout, build_discriminator
from tests.test_amp_reward_cpu import _FakeAMPEnv

HP = dict(stepsize=1e-2, momentum=0.9, weight_decay=1e-3, logit_reg_weight=0.05, grad_penalty=10.0, batch_size=32, steps=4)


def _setup(seed=0, **hp):
    torch.manual_seed(seed)
    env = _FakeAMPEnv(4, 0, "Imitate AMP")
    ro = BatchedRollout(env, exp_rate=0.0, seed=1, disc=build_discriminator(_FakeAMPEnv.M, hidden=(32, 16)))
    return ro, AMPDiscLearner(ro, **dict(HP, **hp))


def _pools(seed=0, Ra=200, Re=150):
    """agent and expert AMP observations that a discriminator can tell apart (the expert's are shifted)"""
    g = torch.Generator().manual_seed(seed)
    M = _FakeAMPEnv.M
    return torch.randn(Ra, M, generator=g) * 0.4 + 0.3, torch.randn(Re, M, generator=g) * 0.4 + 0.8


def test_rules_match_numpy_at_known_values():
    d_e = torch.tensor([1.5, -0.25, 0.0, 2.0], dtype=torch.float64)
    d_a = torch.tensor([-1.0, 0.5, -3.0], dtype=torch.float64)
    ne, na = d_e.numpy(), d_a.numpy()
    assert disc_loss(d_e, d_a).item() == pytest.approx(0.5 * (0.5 * np.mean((ne - 1) ** 2) + 0.5 * np.mean((na + 1) ** 2)), rel=1e-15)
    acc_e, acc_a = disc_accuracies(d_e, d_a)
    assert acc_e.item() == 0.5 and acc_a.item() == pytest.approx(2 / 3)   # d = 0 counts as neither side's success
    g = torch.tensor([[1.0, 2.0, -2.0], [0.0, 0.5, 0.0]], dtype=torch.float64)
    assert disc_grad_penalty(g).item() == pytest.approx(0.5 * (9.0 + 0.25) / 2, rel=1e-15)
    disc = build_discriminator(5, hidden=(4, 3)).double()
    ws = [l.weight.detach().numpy() for l in list(disc.hidden) + [disc.logit]]
    assert disc_weight_decay_loss(disc).item() == pytest.approx(sum(0.5 * (w ** 2).sum() for w in ws), rel=1e-14)   # the logit layer included
    assert disc_logit_reg_loss(disc).item() == pytest.approx(0.5 * (ws[2] ** 2).sum(), rel=1e-14)


def test_gradient_penalty_closed_forms_match_double_backward():
    """a small ReLU net in float64: g = dd/dx = W0^T (m0 (W1^T (m1 w2))) and the weight gradients of P = 0.5 mean ||g||^2 with the masks held
    constant (u1 = m1 w2, u0 = m0 (W1^T u1), e = g, q0 = m0 (W0 e), q1 = m1 (W1 q0): dP/dW0 = mean u0 e^T, dP/dW1 = mean u1 q0^T,
    dP/dw2 = mean q1) against torch's double backward to 1e-12; the biases get exactly nothing"""
    torch.manual_seed(3)
    disc = build_discriminator(7, hidden=(13, 11)).double()
    with torch.no_grad():
        for l in disc.hidden:
            l.bias.uniform_(-0.5, 0.5)
    x = torch.randn(40, 7, dtype=torch.float64)
    d, g = disc_input_grad(disc, x)
    P = disc_grad_penalty(g)
    params = list(disc.parameters())
    grads = torch.autograd.grad(P, params, allow_unused=True)
    grads = [torch.zeros_like(p) if gr is None else gr for p, gr in zip(params, grads)]
    (W0, b0), (W1, b1), (w2, b2) = [(l.weight.detach().numpy(), l.bias.detach().numpy()) for l in list(disc.hidden) + [disc.logit]]
    X = x.numpy()
    a0 = X @ W0.T + b0
    m0 = (a0 > 0).astype(np.float64)
    a1 = np.maximum(a0, 0) @ W1.T + b1
    m1 = (a1 > 0).astype(np.float64)
    B = X.shape[0]
    u1 = m1 * w2[0]
    u0 = m0 * (u1 @ W1)
    e = u0 @ W0
    q0 = m0 * (e @ W0.T)
    q1 = m1 * (q0 @ W1.T)
    np.testing.assert_allclose(d.detach().numpy(), np.maximum(a1, 0) @ w2[0] + b2[0], rtol=0, atol=1e-12)
    np.testing.assert_allclose(g.detach().numpy(), e, rtol=0, atol=1e-12)
    closed = {"hidden.0.weight": u0.T @ e / B, "hidden.1.weight": u1.T @ q0 / B, "logit.weight": q1.sum(0, keepdims=True) / B}
    for (name, _), gr in zip(disc.named_parameters(), grads):
        if name.endswith("bias"):
            assert torch.count_nonzero(gr).item() == 0, name
        else:
            np.testing.assert_allclose(gr.numpy(), closed[name], rtol=0, atol=1e-12 * max(1.0, np.abs(closed[name]).max()))


def test_one_torch_step_matches_the_numpy_restatement():
    """one step at stepsize 1, momentum 0 from zero accumulators: w_before - w_after is the gradient of disc_loss + w_gp P + wd sum ||W||^2 / 2 +
    logit_reg ||w_logit||^2 / 2 restated in numpy (forward, backward, the closed-form penalty gradients)"""
    ro, ln = _setup(stepsize=1.0, momentum=0.0)
    agent, expert = _pools()
    ai, ei = torch.arange(0, 64, 2), torch.arange(10, 42)
    layers = list(ln.disc.hidden) + [ln.disc.logit]
    before = [(l.weight.detach().double().numpy().copy(), l.bias.detach().double().numpy().copy()) for l in layers]
    stats = [torch.zeros(()) for _ in range(6)]
    ln.minibatch_step(agent, expert, ai, ei, stats)
    norm = lambda x: ro.amp_norm.normalize(x).double().numpy()
    xa, xe = norm(agent[ai]), norm(expert[ei])
    B = 32
    (W0, b0), (W1, b1), (w2, b2) = before

    def fwd(x):
        h0 = np.maximum(x @ W0.T + b0, 0)
        h1 = np.maximum(h0 @ W1.T + b1, 0)
        return [x, h0, h1], h1 @ w2[0] + b2[0]
    ha, da = fwd(xa)
    he, de = fwd(xe)
    # least-squares loss, backward over both sides (sum convention, 1 / B)
    hs = [np.concatenate([p, q]) for p, q in zip(ha, he)]
    dy = np.concatenate([0.5 * (da + 1), 0.5 * (de - 1)])[:, None] / B
    grads = {}
    for i, (W, _) in reversed(list(enumerate(before))):
        grads[i] = [dy.T @ hs[i], dy.sum(0)]
        dy = (dy @ W) * (hs[i] > 0)
    # the penalty's closed forms on the expert rows
    m0, m1 = (he[1] > 0).astype(float), (he[2] > 0).astype(float)
    u1 = m1 * w2[0]
    u0 = m0 * (u1 @ W1)
    e = u0 @ W0
    q0 = m0 * (e @ W0.T)
    q1 = m1 * (q0 @ W1.T)
    for i, pg in enumerate([u0.T @ e, u1.T @ q0, q1.sum(0, keepdims=True)]):
        grads[i][0] = grads[i][0] + HP["grad_penalty"] * pg / B + HP["weight_decay"] * before[i][0]
    grads[2][0] += HP["logit_reg_weight"] * w2
    for i, l in enumerate(layers):
        np.testing.assert_allclose(before[i][0] - l.weight.detach().double().numpy(), grads[i][0], rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(before[i][1] - l.bias.detach().double().numpy(), grads[i][1], rtol=1e-4, atol=1e-6)
    assert stats[0].item() == pytest.approx(0.5 * (0.5 * np.mean((de - 1) ** 2) + 0.5 * np.mean((da + 1) ** 2)), rel=1e-5)
    assert stats[1].item() == pytest.approx(0.5 * (e ** 2).sum(1).mean(), rel=1e-5)
    assert stats[2].item() == pytest.approx(np.mean(de > 0)) and stats[3].item() == pytest.approx(np.mean(da < 0))
    assert stats[4].item() == pytest.approx(de.mean(), rel=1e-5, abs=1e-6) and stats[5].item() == pytest.approx(da.mean(), rel=1e-5, abs=1e-6)


def test_hyperparameters_are_required_and_validated():
    ro, _ = _setup()
    for name, bad in (("stepsize", 0.0), ("stepsize", None), ("momentum", 1.0), ("momentum", -0.1), ("weight_decay", -1e-3),
                      ("logit_reg_weight", float("nan")), ("grad_penalty", -1.0), ("grad_penalty", None), ("batch_size", 0), ("batch_size", 2.0),
                      ("steps", 0), ("steps", True)):
        with pytest.raises(ValueError, match=name):
            AMPDiscLearner(ro, **dict(HP, **{name: bad}))
    with pytest.raises(ValueError, match="backend"):
        AMPDiscLearner(ro, **HP, backend="cuda")
    with pytest.raises(ValueError, match="tensor_core learner needs a CUDA device"):
        AMPDiscLearner(ro, **HP, backend="tensor_core")
    plain = BatchedRollout(_FakeAMPEnv(4, 0, "Imitate AMP"), exp_rate=0.0)
    with pytest.raises(ValueError, match="discriminator"):
        AMPDiscLearner(plain, **HP)
    ln = AMPDiscLearner(ro, **HP)
    agent, expert = _pools()
    with pytest.raises(ValueError, match="expert_amp_obs"):
        ln.update(agent, expert[:, :3])
    ro.disc.logit.weight = torch.nn.Parameter(ro.disc.logit.weight.detach().clone())
    with pytest.raises(ValueError, match="replaced"):
        ln.update(agent, expert)


def test_seeded_update_is_reproducible():
    runs = []
    for _ in range(2):
        ro, ln = _setup(seed=4)
        s = ln.update(*_pools())
        runs.append(([p.detach().clone() for p in ro.disc.parameters()], s))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0]))
    assert all(torch.equal(runs[0][1][k], runs[1][1][k]) for k in runs[0][1])
    assert sorted(runs[0][1]) == sorted(["disc_loss", "grad_penalty", "acc_expert", "acc_agent", "logit_expert", "logit_agent"])
    assert all(v.dim() == 0 for v in runs[0][1].values())


def test_fifty_steps_lower_the_loss_and_raise_both_accuracies():
    ro, ln = _setup(seed=2, steps=50, batch_size=64, momentum=0.5)
    agent, expert = _pools()
    full = lambda: ln.loss(ro.amp_norm.normalize(agent), ro.amp_norm.normalize(expert))
    _, l0, _, de0, da0 = full()
    ln.update(agent, expert)
    _, l1, _, de1, da1 = full()
    acc0, acc1 = disc_accuracies(de0, da0), disc_accuracies(de1, da1)
    print("disc_loss %.4f -> %.4f, acc_expert %.3f -> %.3f, acc_agent %.3f -> %.3f"
          % (l0.item(), l1.item(), acc0[0].item(), acc1[0].item(), acc0[1].item(), acc1[1].item()))
    assert l1.item() < l0.item() and acc1[0].item() > acc0[0].item() and acc1[1].item() > acc0[1].item()
