"""The gated networks' backward (DESIGN.md section 8, dm_learn_gated_step) restated in float64 numpy against torch autograd of the gated actor
and critic, and the size refusals of the gated tensor-core learner's wrapper.  No GPU."""
import numpy as np
import pytest
import torch


def _gated_backward(net, head, ns, ng, dy):
    """the gated layer's forward and backward as the tensor-core step computes them: for l in {0, 1}, x_0 = [ns | ng], x_1 = h_0,
      gc = relu(Wgc ng + bgc), g_l = relu(Wgh_l gc + bgh_l),
      z_l = W_l x_l + b_l, s_l = Ws_l g_l + bs_l, t_l = Wt_l g_l + bt_l, h_l = relu(2 sigma(s_l) z_l + t_l);
    given dh_l: p = dh_l 1[h_l > 0], dz_l = 2 sigma(s_l) p, ds_l = 2 sigma(s_l) (1 - sigma(s_l)) z_l p, dt_l = p, dh_0 = W_1^T dz_1,
      dg_l = (Ws_l^T ds_l + Wt_l^T dt_l) 1[g_l > 0], dgc = (sum_l Wgh_l^T dg_l) 1[gc > 0].
    Returns {parameter name: gradient of sum(dy * output)} and the gates g_l."""
    P = {n: p.detach().double().numpy() for n, p in net.named_parameters()}
    P.update({"head.weight": head.weight.detach().double().numpy(), "head.bias": head.bias.detach().double().numpy()})
    relu = lambda v: np.maximum(v, 0.0)
    gc = relu(ng @ P["gate_common.weight"].T + P["gate_common.bias"])
    x, saved = [np.concatenate([ns, ng], axis=1)], []
    for l in range(2):
        g = relu(gc @ P["gate_hidden.%d.weight" % l].T + P["gate_hidden.%d.bias" % l])
        z = x[l] @ P["hidden.%d.weight" % l].T + P["hidden.%d.bias" % l]
        sig = 1.0 / (1.0 + np.exp(-(g @ P["gate_scale.%d.weight" % l].T + P["gate_scale.%d.bias" % l])))
        h = relu(2.0 * sig * z + g @ P["gate_bias.%d.weight" % l].T + P["gate_bias.%d.bias" % l])
        saved.append((g, z, sig, h))
        x.append(h)
    grads = {"head.weight": dy.T @ x[2], "head.bias": dy.sum(0)}
    dh = dy @ P["head.weight"]
    dgc_in = 0.0
    for l in (1, 0):
        g, z, sig, h = saved[l]
        p = dh * (h > 0)
        dz, ds, dt = 2.0 * sig * p, 2.0 * sig * (1.0 - sig) * z * p, p
        grads["hidden.%d.weight" % l], grads["hidden.%d.bias" % l] = dz.T @ x[l], dz.sum(0)
        grads["gate_scale.%d.weight" % l], grads["gate_scale.%d.bias" % l] = ds.T @ g, ds.sum(0)
        grads["gate_bias.%d.weight" % l], grads["gate_bias.%d.bias" % l] = dt.T @ g, dt.sum(0)
        dg = (ds @ P["gate_scale.%d.weight" % l] + dt @ P["gate_bias.%d.weight" % l]) * (g > 0)
        grads["gate_hidden.%d.weight" % l], grads["gate_hidden.%d.bias" % l] = dg.T @ gc, dg.sum(0)
        dgc_in = dgc_in + dg @ P["gate_hidden.%d.weight" % l]
        dh = dz @ P["hidden.1.weight"] if l == 1 else None
    dgc = dgc_in * (gc > 0)
    grads["gate_common.weight"], grads["gate_common.bias"] = dgc.T @ ng, dgc.sum(0)
    return grads, [s[0] for s in saved]


@pytest.mark.parametrize("kind", ["actor", "critic"])
def test_gated_backward_restatement_matches_autograd(kind):
    """the restated backward of every one of the ten parameter pairs against float64 torch autograd of build_gated_policy / build_critic(S, G),
    to 1e-12 relative, with gate units closed on some rows and open on others"""
    from deepmimic_b200.rollout import build_critic, build_gated_policy
    S, G, A, hidden, gc, gh, B = 11, 3, 4, (12, 9), 7, 5, 64
    torch.manual_seed(3)
    if kind == "actor":
        net = build_gated_policy(S, G, A, init_output_scale=0.5, hidden=hidden, gate_common=gc, gate_hidden=gh).double()
        head = net.mean
    else:
        net = build_critic(S, G, hidden=hidden, gate_common=gc, gate_hidden=gh).double()
        head = net.out
    with torch.no_grad():   # shifted gate biases: some gate units close on some rows
        for l in net.gate_hidden:
            l.bias.copy_(torch.linspace(-0.8, 0.8, l.bias.numel(), dtype=torch.float64))
        for l in list(net.gate_scale) + list(net.gate_bias) + list(net.hidden):
            l.bias.normal_(0.0, 0.3)
    rng = np.random.default_rng(4)
    ns, ng = rng.normal(size=(B, S)), rng.normal(size=(B, G))
    dy = rng.normal(size=(B, head.weight.shape[0]))
    out = net(torch.from_numpy(ns), torch.from_numpy(ng))
    params = [(n, p) for n, p in net.named_parameters() if n != "logstd"]
    ref = torch.autograd.grad((out * torch.from_numpy(dy)).sum(), [p for _, p in params])
    got, gates = _gated_backward(net, head, ns, ng, dy)
    for g in gates:
        assert (g == 0).any() and (g > 0).any()
    assert len(params) == 20
    for (n, _), r in zip(params, ref):
        key = "head." + n.split(".", 1)[1] if n.startswith(("mean.", "out.")) else n
        r = r.numpy()
        assert np.linalg.norm(got[key] - r) <= 1e-12 * max(np.linalg.norm(r), 1e-300), n


def test_gated_learner_wrapper_refuses_unsupported_sizes():
    """TensorCoreGatedLearner checks the network before it calls the library: the kind, a plain network, the limits of dm_mlp_create_gated
    (goal size <= 64, gate_common <= 128, gate_hidden <= 64, at most 64 outputs); TensorCoreLearner refuses a gated network"""
    from deepmimic_b200.capi import TensorCoreGatedLearner, TensorCoreLearner
    from deepmimic_b200.rollout import build_critic, build_gated_policy, build_policy
    small = dict(hidden=(16, 8))
    ok = build_gated_policy(10, 3, 4, **small, gate_common=8, gate_hidden=4)
    for kind in ("disc", "value"):
        with pytest.raises(ValueError, match="kind"):
            TensorCoreGatedLearner(ok, {}, kind, 128)
    with pytest.raises(ValueError, match="gated network"):
        TensorCoreGatedLearner(build_policy(10, 4, **small), {}, "actor", 128)
    with pytest.raises(ValueError, match="gated network"):
        TensorCoreGatedLearner(build_gated_policy(10, 3, 4, hidden=(16, 8, 8), gate_common=8, gate_hidden=4), {}, "actor", 128)
    for net, what in ((build_gated_policy(10, 65, 4, **small, gate_common=8, gate_hidden=4), "goal size"),
                      (build_gated_policy(10, 3, 4, **small, gate_common=129, gate_hidden=4), "gate_common"),
                      (build_gated_policy(10, 3, 4, **small, gate_common=8, gate_hidden=65), "gate_hidden"),
                      (build_gated_policy(10, 3, 65, **small, gate_common=8, gate_hidden=4), "outputs")):
        with pytest.raises(ValueError, match=what):
            TensorCoreGatedLearner(net, {}, "actor", 128)
    with pytest.raises(ValueError, match="TensorCoreGatedLearner"):
        TensorCoreLearner(build_critic(10, 3, **small, gate_common=8, gate_hidden=4), {}, "critic", 128)
