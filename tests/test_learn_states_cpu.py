"""The float64 restatement of tests/learn_states.py against deepmimic_b200/learner.py (torch autograd in float64) at known values, and the
constructed minibatches of learn_states: every row reaches the branch it is built for, each decision at least 10 % of its threshold away,
and together they reach all of them."""
import math

import numpy as np
import pytest

from tests import learn_states as L


def _torch():
    return pytest.importorskip("torch")


def test_actor_restatement_matches_the_torch_backend():
    """gaussian_logp, the surrogate's and the bound loss's per-row gradients, the clip fraction: restatement against learner.py's functions
    under float64 autograd, on a construction with every kind and every bound regime"""
    torch = _torch()
    from deepmimic_b200 import learner as ln
    c = L.actor_case(7, 48, 40, seed=3)
    mu = torch.tensor(c["mu"], dtype=torch.float64, requires_grad=True)
    a, ls = torch.tensor(c["norm_a"], dtype=torch.float64), torch.tensor(c["logstd"], dtype=torch.float64)
    old, adv = torch.tensor(c["old_logp"], dtype=torch.float64), torch.tensor(c["adv"], dtype=torch.float64)
    lo, hi = torch.tensor(c["bound_min"], dtype=torch.float64), torch.tensor(c["bound_max"], dtype=torch.float64)
    lp = ln.gaussian_log_prob(a, mu, ls)
    ratio = (lp - old).exp()
    rows = mu.shape[0]
    loss = rows * (-ln.clipped_surrogate(adv, ratio, L.EPS).mean() + ln.bound_loss(mu, lo, hi))
    dy, = torch.autograd.grad(loss, mu)
    ref = L.actor_rows(c["norm_a"], c["mu"], c["logstd"], c["old_logp"], c["adv"], L.EPS, c["bound_min"], c["bound_max"])
    np.testing.assert_allclose(lp.detach().numpy(), L.gaussian_logp(c["norm_a"], c["mu"], c["logstd"]), rtol=1e-14)
    np.testing.assert_allclose(ratio.detach().numpy(), ref["ratio"], rtol=1e-12)
    np.testing.assert_allclose(dy.numpy(), ref["dy"], rtol=1e-9, atol=1e-12)
    assert ln.clip_fraction(ratio.detach(), L.EPS).item() == pytest.approx(ref["clipped"].mean(), abs=1e-7)
    surr = ln.clipped_surrogate(adv, ratio.detach(), L.EPS).numpy()
    np.testing.assert_allclose(surr, ref["surr"], rtol=1e-12)
    np.testing.assert_allclose(ln.bound_loss(mu.detach(), lo, hi).item() * rows, ref["bound"].sum(), rtol=1e-12)


def test_tie_and_inclusive_bounds_match_the_torch_backend():
    """a tie outside the range (adv ratio == adv clip(ratio) in fp32 arithmetic, here at adv = 0) passes the gradient to the unclipped term;
    a ratio exactly on 1 + eps is inside; in both the restatement and learner.clipped_surrogate"""
    torch = _torch()
    from deepmimic_b200 import learner as ln
    eps = 0.25    # exact in fp32, so that 1 + eps is too (with eps = 0.2 in fp32, |1.2f - 1| > 0.2f while 1.2f <= 1 + 0.2f)
    r = torch.tensor([1.0 + eps, 1.5, 0.5], dtype=torch.float64, requires_grad=True)
    adv = torch.tensor([2.0, 0.0, -1.0], dtype=torch.float64)
    g, = torch.autograd.grad(ln.clipped_surrogate(adv, r, eps).sum(), r)
    active, clipped = L.ratio_clip_rule(adv.numpy(), r.detach().numpy(), eps)
    assert list(active) == [True, True, False] and list(clipped) == [False, True, True]
    assert g[0].item() == 2.0 and g[2].item() == 0.0


def test_critic_and_disc_restatement_match_the_torch_backend():
    torch = _torch()
    from deepmimic_b200 import learner as ln
    c = L.critic_case(30, 24, seed=1)
    v = torch.tensor(c["out"], dtype=torch.float64, requires_grad=True)
    dv, = torch.autograd.grad(30 * ln.critic_loss(v, torch.tensor(c["target"], dtype=torch.float64)), v)
    np.testing.assert_allclose(dv.numpy(), L.critic_dy(c["out"], c["target"]), rtol=1e-12)
    d = L.disc_case(13)
    da = torch.tensor(d["d_a"], dtype=torch.float64, requires_grad=True)
    de = torch.tensor(d["d_e"], dtype=torch.float64, requires_grad=True)
    loss = ln.disc_loss(de, da)
    ga, ge = torch.autograd.grad(13 * loss, (da, de))
    ref = L.disc_rows(d["d_a"], d["d_e"])
    np.testing.assert_allclose(ga.numpy(), ref["dy_agent"], rtol=1e-12)
    np.testing.assert_allclose(ge.numpy(), ref["dy_expert"], rtol=1e-12)
    assert loss.item() == pytest.approx(ref["loss"], rel=1e-12)
    acc_e, acc_a = ln.disc_accuracies(de.detach(), da.detach())
    assert (acc_e.item(), acc_a.item()) == pytest.approx((ref["acc_expert"], ref["acc_agent"]), abs=1e-7)


def test_momentum_restatement_matches_the_torch_backend():
    torch = _torch()
    from deepmimic_b200 import learner as ln
    g = np.random.default_rng(0)
    w, acc, grad = g.standard_normal(9), g.standard_normal(9), g.standard_normal(9)
    pw, pa = torch.tensor(w), torch.tensor(acc)
    ln.momentum_step([pw], [pa], [torch.tensor(grad) + 1e-3 * torch.tensor(w)], 1e-2, 0.9)
    w2, a2 = L.momentum_update(w, acc, grad, 1e-2, 0.9, 1e-3)
    np.testing.assert_allclose(pw.numpy(), w2, rtol=1e-14)
    np.testing.assert_allclose(pa.numpy(), a2, rtol=1e-14)


@pytest.mark.parametrize("A,rows,tags", [(28, 129, 129), (58, 128, 128), (64, 127, 127), (1, 1, 1), (28, 4096, 509)])
def test_actor_constructions_reach_their_branches(A, rows, tags):
    """each tagged row takes the (active, clipped) of its kind, its ratio at least 10 % of eps from both thresholds (ratio 1 rows: exactly
    at 1 in float64); mu components are below, above, inside or exactly on the bounds, 0.1 away when not on them; adv 0 rows have adv 0 and
    the others |adv| >= 0.5"""
    c = L.actor_case(A, rows, tags, seed=rows + A)
    ref = L.actor_rows(c["norm_a"], c["mu"], c["logstd"], c["old_logp"], c["adv"], L.EPS, c["bound_min"], c["bound_max"])
    tagged = np.nonzero(c["tag"] >= 0)[0]
    assert len(tagged) == tags and len(set(c["tag"][tagged])) == tags and c["tag"][tagged].min() >= 1
    for r in range(rows):
        k = c["kind"][r]
        sign, target, active, clipped = L._ACTOR_KIND[k]
        assert (bool(ref["active"][r]), bool(ref["clipped"][r])) == (active, clipped), (r, k, ref["ratio"][r])
        for edge in (1.0 - L.EPS, 1.0 + L.EPS):
            assert abs(ref["ratio"][r] - edge) >= 0.1 * L.EPS
        assert abs(ref["ratio"][r] / target - 1.0) <= 1e-5        # the fp32 old_logp
        assert (c["adv"][r] == 0) if sign == 0 else (np.sign(c["adv"][r]) == sign and abs(c["adv"][r]) >= 0.5)
    d = np.stack([c["mu"] - L.LO, c["mu"] - L.HI])
    assert np.all((d == 0) | (np.abs(d) >= 0.1))
    if tags >= 8:
        assert set(c["kind"][tagged]) == set(L.ACTOR_KINDS)
    if tags * A >= 5:
        m = c["mu"][tagged]
        for name, v in L.MU_KINDS:
            assert np.any(m == np.float32(v)), name
        assert np.any(m < L.LO) and np.any(m > L.HI) and np.any((m > L.LO) & (m < L.HI))
        assert np.any(ref["dy"][tagged] != 0) and np.any(~ref["active"][tagged])


def test_edge_constructions_sit_on_the_clip_edge():
    c = L.actor_case(28, 64, 64, seed=17, edge=True)
    ref = L.actor_rows(c["norm_a"], c["mu"], c["logstd"], c["old_logp"], c["adv"], L.EPS, c["bound_min"], c["bound_max"])
    np.testing.assert_allclose(ref["ratio"], c["target"], rtol=2e-8, atol=0)
    assert set(c["target"].round(6)) == {0.8, 1.2} and len(set(c["target"])) == 10


def test_tagged_trunk_is_one_hot_in_fp16():
    """every hidden value of the tagged trunk is an fp16-exact integer and the last hidden layer is exactly one-hot at the tag (tag 0 for the
    zero input of a padding row, nothing for BLANK), for every tag the shipped 1024-512 trunk carries"""
    S, h0, h1 = 10, 1024, 512
    w0, b0, w1, b1 = L.tagged_trunk(S, h0, h1)
    n = L.tag_count(h0, h1)
    t = np.arange(-1, n).astype(np.float64)
    x = np.zeros((len(t) + 1, S)); x[:-1, 0] = t; x[-1, 0] = L.BLANK
    h0v = np.maximum(x @ w0.T.astype(np.float64) + b0, 0.0)
    assert np.all(h0v == h0v.astype(np.float16).astype(np.float64)) and h0v.max() <= 2048
    h = L.trunk_hidden(w0, b0, w1, b1, x)
    want = np.zeros_like(h)
    for i, tag in enumerate(t):
        if tag >= 0:
            want[i, int(tag)] = 1.0
    assert np.array_equal(h, want)
    assert n == 512


def test_critic_and_disc_constructions():
    c = L.critic_case(129, 129, seed=129)
    err = c["out"].astype(np.float64) - c["target"]
    assert np.any(err > 0) and np.any(err < 0) and np.any(err == 0)
    assert np.array_equal(err, c["err"])                   # the targets are exact in fp32
    for rows in (1, 127, 128, 129, 254):
        d = L.disc_case(rows)
        assert len(set(d["tag_a"]) | set(d["tag_e"])) == 2 * rows and 2 * rows < L.tag_count(1024, 512)
        if rows >= len(L.D_VALUES):
            for v in L.D_VALUES:
                assert v in d["d_a"] and v in d["d_e"]
    w2, _ = L.output_layer(np.arange(1, 9), np.array(L.D_VALUES, np.float32), 16, padding_value=5.0)
    assert w2[0, 0] == 5.0 and list(w2[0, 1:9]) == list(L.D_VALUES)


def test_prep_restatement():
    """clip on and off, and the float64 values of fp16 operands within prep_bound"""
    s = np.array([1.0, 3.0, -9.0, 0.25], np.float32)
    mean, istd = np.array([0, 1, 0, 0.5], np.float32), np.array([1, 2, 1, 4], np.float32)
    np.testing.assert_array_equal(L.prep_operand(s, mean, istd, 2.0), [1.0, 2.0, -2.0, -1.0])
    np.testing.assert_array_equal(L.prep_operand(s, mean, istd, 0.0), [1.0, 4.0, -9.0, -1.0])
    x = np.random.default_rng(0).standard_normal(1000) * 100
    assert np.all(np.abs(x.astype(np.float16).astype(np.float64) - x) <= L.prep_bound(x))
    with np.errstate(over="ignore"):
        assert math.isinf(np.float16(1e5))                   # why the preparation saturates at HALF_MAX
