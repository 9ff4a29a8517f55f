"""The tensor-core learners' per-row rules on the GPU (kernels/dm_learn.cu), row by row against the float64 restatement of tests/learn_states.py.

The observable: the output layer's weight gradient of a step (TensorCoreLearner.grad, which leaves the parameters alone) over the tagged trunk
of learn_states.  Column `tag` of that gradient is (1 / rows) dY of the one row with that tag: the dW GEMM adds the row's fp16 hi and lo
parts times an exact 1 and zeros from every other row, so the only errors are the hi + lo split (2^-22 |dY| + 2^-25) and two roundings of the
1 / rows scaling.  Column 0 collects the rows past the minibatch, which must carry dY = 0.  The outputs are exact (fp16-exact W2 entries times
a one-hot fp16 row, plus b2 = 0), so each row's mu, value or logit is chosen, and the actor's decisions are taken on the kernel's own ratio
(dm_learn_batch.ratio) with TF's rule in fp32; that ratio is checked against float64 separately.  The input preparation is checked through
the first layer's gradient of a one-row step, dW0 = dZ0 x^T: column k over the column of an input that is exactly 1.0 recovers the kernel's
fp16 operand x_k to 3 u.  Every bound is stated where it is used; -s prints each check's worst error / bound."""
import numpy as np
import pytest

from tests import learn_states as L

pytestmark = pytest.mark.gpu
U = L.U32
WORST = {}


def _t(a, dtype=None):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a), device="cuda", dtype=dtype)


def _report(name, err, bound):
    """asserts err <= bound elementwise and prints the worst ratio"""
    err, bound = np.asarray(err, np.float64), np.asarray(bound, np.float64)
    ratio = float(np.max(err / bound)) if err.size else 0.0
    WORST[name] = max(WORST.get(name, 0.0), ratio)
    print("%-52s worst error / bound %.3f" % (name, ratio))
    assert np.all(err <= bound), (name, float(np.max(err - bound)))


def _load(layer, w, b):
    import torch
    with torch.no_grad():
        layer.weight.copy_(_t(w)); layer.bias.copy_(_t(b))


def _learner(net, kind, max_rows, gated=False):
    import torch
    from deepmimic_b200.capi import TensorCoreGatedLearner, TensorCoreLearner, tc_layers
    acc = {p: torch.zeros_like(p) for l in tc_layers(net, kind) for p in (l.weight, l.bias)}
    tc = (TensorCoreGatedLearner if gated else TensorCoreLearner)(net, acc, kind, max_rows)
    tc.set_weights()
    return tc, acc


class _Batch:
    """a dm_learn_batch (or dm_learn_gated_batch) and the device tensors it points into"""

    def __init__(self, states, idx, rows, mean, istd, clip, actor=None, targets=None, eps=L.EPS, lr=0.0, mom=0.0, wd=0.0, goal=None):
        import torch
        from deepmimic_b200.capi import DmLearnBatch, DmLearnGatedBatch
        k = self.keep = dict(states=_t(states, torch.float32), idx=_t(idx, torch.int64), mean=_t(mean, torch.float32), istd=_t(istd, torch.float32),
                             stats=torch.zeros(2, device="cuda"), ratio=torch.full((rows,), float("nan"), device="cuda"))
        p = lambda name: k[name].data_ptr()
        f = dict(states=p("states"), idx=p("idx"), rows=rows, in_mean=p("mean"), in_istd=p("istd"), in_clip=clip, stepsize=lr, momentum=mom,
                 weight_decay=wd, stats=p("stats"))
        if actor is not None:
            for name in ("norm_a", "old_logp", "adv", "logstd", "bound_min", "bound_max"):
                k[name] = _t(actor[name], torch.float32)
            f.update(norm_actions=p("norm_a"), old_logp=p("old_logp"), adv=p("adv"), logstd=p("logstd"), bound_min=p("bound_min"),
                     bound_max=p("bound_max"), ratio_clip=eps, ratio=p("ratio"))
        else:
            k["targets"] = _t(targets, torch.float32)
            f.update(norm_targets=p("targets"))
        self.b = DmLearnBatch(**f)
        if goal is not None:
            for name in ("goals", "g_mean", "g_istd"):
                k[name] = _t(goal[name], torch.float32)
            self.b = DmLearnGatedBatch(batch=self.b, goals=p("goals"), g_mean=p("g_mean"), g_istd=p("g_istd"), g_clip=goal["g_clip"])


def _grad(tc, batch):
    """(flat gradient, {parameter: view}) of one TensorCoreLearner.grad"""
    import torch
    g = torch.empty(tc.grad_size(), device="cuda")
    tc.grad(batch.b, g)
    torch.cuda.synchronize()
    return g, tc.grad_views(g)


def _row_dy(view, tags, rows):
    """the rows' dY from the output layer's weight gradient [out, h1]: column tag times rows (float64)"""
    return view.double().cpu().numpy()[:, tags].T * rows


# ---- the PPO actor
ACTOR_SHAPES = [  # (name, in_dim, hidden, actions, rows, workspace rows, gated goal size)
    ("spinkick actor, 129 rows", 227, (1024, 512), 28, 129, 4096, 0),
    ("spinkick actor, workspace maximum", 227, (1024, 512), 28, 4096, 4096, 0),
    ("dog trot actor, 128 rows", 347, (1024, 512), 58, 128, 2048, 0),
    ("out 64, in 127, 127 rows", 127, (256, 192), 64, 127, 512, 0),
    ("out 1, in 128, 1 row", 128, (128, 128), 1, 1, 256, 0),
    ("out 28, in 129, 200 rows", 129, (256, 128), 28, 200, 256, 0),
    ("target_amp gated actor 226 + 3, 129 rows", 226, (1024, 512), 28, 129, 4096, 3),
]


def _actor_net(S, hidden, A, G, tags, mu):
    """the actor (plain or gated) over the tagged trunk with output columns mu; gated: the gates neutral (scale 2 sigmoid(0) = 1, bias 0)"""
    import torch
    from deepmimic_b200.rollout import build_gated_policy, build_policy
    torch.manual_seed(0)
    net = (build_gated_policy(S, G, A, hidden=hidden) if G else build_policy(S, A, hidden=hidden)).cuda()
    w0, b0, w1, b1 = L.tagged_trunk(S + G, *hidden)
    _load(net.hidden[0], w0, b0); _load(net.hidden[1], w1, b1)
    _load(net.mean, *L.output_layer(tags, mu, hidden[1], padding_value=0.375))
    if G:
        for l in list(net.gate_scale) + list(net.gate_bias):
            _load(l, np.zeros(tuple(l.weight.shape), np.float32), np.zeros(l.bias.shape[0], np.float32))
    return net


def _actor_setup(S, hidden, A, rows, max_rows, G, case):
    net = _actor_net(S, hidden, A, G, case["tag"], case["mu"])
    tc, _ = _learner(net, "actor", max_rows, gated=bool(G))
    states = L.state_rows(case["tag"], S, 1)
    goal = None
    if G:
        goal = dict(goals=np.random.default_rng(2).standard_normal((rows, G)).astype(np.float32), g_mean=np.zeros(G, np.float32),
                    g_istd=np.ones(G, np.float32), g_clip=0.0)
    return net, tc, states, goal


def _check_actor(name, net, tc, batch, case, rows, eps=L.EPS):
    """per-row dY, ratio and statistics of one grad() of an actor batch; returns the kernel's ratio"""
    import torch
    _, views = _grad(tc, batch)
    ratio = batch.keep["ratio"].cpu().numpy()
    adv = batch.keep["adv"].cpu().numpy()
    ref = L.actor_rows(case["norm_a"], case["mu"], case["logstd"], case["old_logp"], adv, eps, case["bound_min"], case["bound_max"], ratio=ratio)
    r64 = L.actor_rows(case["norm_a"], case["mu"], case["logstd"], case["old_logp"], adv, eps, case["bound_min"], case["bound_max"])["ratio"]
    _report(name + ": ratio", np.abs(ratio - r64), L.ratio_bound(case["norm_a"], case["mu"], case["logstd"], case["old_logp"], r64))
    tagged = np.nonzero(case["tag"] >= 0)[0]
    dy = _row_dy(views[net.mean.weight], case["tag"][tagged], rows)
    bound = L.actor_dy_bound(case["norm_a"][tagged], case["mu"][tagged], case["logstd"], adv[tagged], ratio[tagged]) + 4 * U * np.abs(ref["dy"][tagged])
    _report(name + ": dY per tagged row", np.abs(dy - ref["dy"][tagged]), bound)
    if rows % 128:
        pad = views[net.mean.weight][:, 0].abs().max().item()
        assert pad == 0.0, "rows past the minibatch carry dY %g" % pad
    # the bias gradient: every row's dY summed by the dW GEMM (fp32, K = rows terms)
    db = views[net.mean.bias].double().cpu().numpy() * rows
    full = L.actor_dy_bound(case["norm_a"], case["mu"], case["logstd"], adv, ratio) + 4 * U * np.abs(ref["dy"])
    _report(name + ": output bias gradient (all rows)", np.abs(db - ref["dy"].sum(0)), full.sum(0) + (rows + 2) * U * np.abs(ref["dy"]).sum(0))
    # statistics: the clip fraction is an exact count; |surrogate + bound loss| sums in a fixed fp32 tree
    st = batch.keep["stats"].cpu().numpy()
    inv = np.float32(1.0) / np.float32(rows)
    assert st[1] == np.float32(np.float32(ref["clipped"].sum()) * inv), (st[1], ref["clipped"].sum())
    loss = abs((-ref["surr"] + ref["bound"]).sum() / rows)
    terms = (np.abs(ref["surr"]) + ref["bound"]).sum() / rows
    _report(name + ": |surrogate + bound loss|", abs(st[0] - loss), (rows + 160) * 4 * U * terms + 1e-30)
    return ratio, ref


@pytest.mark.parametrize("name,S,hidden,A,rows,max_rows,G", ACTOR_SHAPES, ids=[s[0] for s in ACTOR_SHAPES])
def test_actor_head_rows(name, S, hidden, A, rows, max_rows, G):
    """every clip quadrant, advantage 0, ratio 1 and every bound regime, row by row; the kernel's decisions agree with the construction's
    intent (each at least 10 % of eps from its threshold, tests/test_learn_states_cpu.py)"""
    tags = min(rows, L.tag_count(*hidden) - 1)
    case = L.actor_case(A, rows, tags, seed=rows + A)
    net, tc, states, goal = _actor_setup(S, hidden, A, rows, max_rows, G, case)
    batch = _Batch(states, np.arange(rows), rows, np.zeros(S), np.ones(S), 0.0, actor=case, goal=goal)
    ratio, ref = _check_actor(name, net, tc, batch, case, rows)
    for r in np.nonzero(case["tag"] >= 0)[0]:
        want = L._ACTOR_KIND[case["kind"][r]]
        assert (bool(ref["active"][r]), bool(ref["clipped"][r])) == (want[2], want[3]), (r, case["kind"][r], ratio[r])


def test_actor_statistics_accumulate():
    """three grad() calls on one batch: the clip fraction is three times the count exactly, the loss three times within its bound"""
    rows, A, hidden = 129, 28, (256, 192)
    case = L.actor_case(A, rows, rows, seed=5)
    net, tc, states, _ = _actor_setup(227, hidden, A, rows, 256, 0, case)
    batch = _Batch(states, np.arange(rows), rows, np.zeros(227), np.ones(227), 0.0, actor=case)
    one = None
    for i in range(3):
        _grad(tc, batch)
        st = batch.keep["stats"].cpu().numpy().copy()
        one = st if one is None else one
        inv = np.float32(1) / np.float32(rows)
        c = np.float32(np.float32(L.ratio_clip_rule(case["adv"], batch.keep["ratio"].cpu().numpy(), L.EPS)[1].sum()) * inv)
        assert st[1] == np.float32(c * (i + 1)) or (i == 2 and st[1] == np.float32(np.float32(c + c) + c)), (i, st[1], c)
        assert abs(st[0] - (i + 1) * one[0]) <= 4 * U * (i + 1) * abs(one[0])
    print("statistics after three steps: %s (one step %s)" % (st, one))


def test_actor_rows_at_the_clip_edge():
    """rows whose ratio lands within ulps of 1 +- eps.  Pass 1 reads the kernel's ratios; pass 2 gives every row outside the range an
    advantage for which adv ratio and adv clip(ratio) round to the same fp32 value (a tie: TF passes the gradient to the unclipped term,
    so such a row is active); pass 3 sets ratio_clip to |ratio - 1| of one row, which then lies on the range's bound (inside, not clipped)"""
    rows, A, hidden = 64, 28, (256, 128)
    case = L.actor_case(A, rows, rows, seed=17, edge=True)
    net, tc, states, _ = _actor_setup(227, hidden, A, rows, 128, 0, case)
    batch = _Batch(states, np.arange(rows), rows, np.zeros(227), np.ones(227), 0.0, actor=case)
    ratio, ref = _check_actor("clip edge, pass 1", net, tc, batch, case, rows)
    assert np.all(np.abs(ratio.astype(np.float64) - case["target"]) <= 4e-7), "the edge rows must land within ulps of 1 +- eps"
    # pass 2: ties outside the range
    e = np.float32(L.EPS)
    lo, hi = np.float32(1) - e, np.float32(1) + e
    adv = case["adv"].copy()
    ties = 0
    cand = np.float32(1.0) + np.arange(1, 1 << 16, dtype=np.float32) * np.float32(2.0 ** -13)
    for r in range(rows):
        if lo <= ratio[r] <= hi:
            continue
        rc = np.clip(ratio[r], lo, hi)
        same = np.nonzero(cand * ratio[r] == cand * rc)[0]       # none once the ratio is more than about an ulp outside
        if same.size:
            adv[r] = cand[same[0]] * (1 if ratio[r] > hi else -1)   # the side where the tie decides: adv > 0 above the range, < 0 below
            ties += 1
    assert ties >= 4
    tied = dict(case, adv=adv.astype(np.float32))
    batch = _Batch(states, np.arange(rows), rows, np.zeros(227), np.ones(227), 0.0, actor=tied)
    _, ref = _check_actor("clip edge, pass 2 (ties)", net, tc, batch, tied, rows)
    tie = adv != case["adv"]
    assert np.all(ref["active"][tie]) and np.all(ref["clipped"][tie])
    # pass 3: ratio_clip = |ratio - 1| of the first row above the range
    r = int(np.nonzero(ratio > hi)[0][0])
    eps = float(np.abs(ratio[r] - np.float32(1)))
    batch = _Batch(states, np.arange(rows), rows, np.zeros(227), np.ones(227), 0.0, actor=case, eps=eps)
    _, ref = _check_actor("clip edge, pass 3 (ratio on the bound)", net, tc, batch, case, rows, eps=eps)
    assert ref["active"][r] and not ref["clipped"][r]
    print("clip edge: %d tied rows; ratio_clip %.9g puts row %d on the bound" % (ties, eps, r))


def test_actor_head_past_fp16_range():
    """pessimistic rows (advantage -4, the advantage clip; sigma 0.05; |a - mu| 0.2) whose dY = -adv ratio (a - mu) / sigma^2 passes fp16's
    largest finite 65504: hi saturates at +-65504 and lo carries the rest, so |dY| up to 131008 keeps 2^-11 |dY - hi| relative accuracy
    and larger |dY| saturate at +-131008 instead of reaching the GEMMs as inf and NaN.  Rows inside fp16's range keep their bits (the other
    tests)"""
    import torch
    rows, A, hidden = 6, 1, (128, 128)
    case = L.actor_case(A, rows, rows, seed=3, kinds=("hi pessimistic",))
    case["mu"][:] = 0.125
    case["norm_a"][:] = np.float32(0.125 + 0.2)
    target = np.array([1.5, 150.0, 250.0, 320.0, 1000.0, 1e5])
    case["adv"][:] = -4.0
    case["old_logp"] = (L.gaussian_logp(case["norm_a"], case["mu"], case["logstd"]) - np.log(target)).astype(np.float32)
    net, tc, states, _ = _actor_setup(16, hidden, A, rows, 128, 0, case)
    batch = _Batch(states, np.arange(rows), rows, np.zeros(16), np.ones(16), 0.0, actor=case)
    g, views = _grad(tc, batch)
    assert torch.isfinite(g).all(), "a row past fp16's range makes the step's gradient non-finite"
    ratio = batch.keep["ratio"].cpu().numpy()
    ref = L.actor_rows(case["norm_a"], case["mu"], case["logstd"], case["old_logp"], case["adv"], L.EPS, case["bound_min"], case["bound_max"], ratio=ratio)
    dy = _row_dy(views[net.mean.weight], case["tag"], rows)[:, 0]
    want = np.clip(ref["dy"][:, 0], -2 * L.HALF_MAX, 2 * L.HALF_MAX)
    bound = L.actor_dy_bound(case["norm_a"], case["mu"], case["logstd"], case["adv"], ratio)[:, 0] + 4 * U * np.abs(want)
    bound += np.where(np.abs(want) > L.HALF_MAX, 2.0 ** -11 * (np.abs(want) - L.HALF_MAX), 0.0)
    print("dY past fp16's range: reference %s, kernel %s" % (ref["dy"][:, 0], dy))
    _report("actor dY past fp16's range", np.abs(dy - want), bound)


# ---- the critic
@pytest.mark.parametrize("rows,hidden,S,max_rows", [(129, (1024, 512), 227, 4096), (1, (128, 128), 63, 128), (128, (256, 256), 64, 128),
                                                   (4096, (1024, 512), 227, 4096)])
def test_critic_head_rows(rows, hidden, S, max_rows):
    """value errors positive, negative and exactly zero, row by row: dY = V - target (one fp32 subtraction, u |dY|, and the split)"""
    import torch
    from deepmimic_b200.rollout import build_critic
    tags = min(rows, L.tag_count(*hidden) - 1)
    case = L.critic_case(rows, tags, seed=rows)
    torch.manual_seed(0)
    net = build_critic(S, hidden=hidden).cuda()
    w0, b0, w1, b1 = L.tagged_trunk(S, *hidden)
    _load(net.hidden[0], w0, b0); _load(net.hidden[1], w1, b1)
    _load(net.out, *L.output_layer(case["tag"], case["out"], hidden[1], padding_value=2.0))
    tc, _ = _learner(net, "critic", max_rows)
    batch = _Batch(L.state_rows(case["tag"], S, 4), np.arange(rows), rows, np.zeros(S), np.ones(S), 0.0, targets=case["target"])
    _, views = _grad(tc, batch)
    want = L.critic_dy(case["out"], case["target"])
    tagged = np.nonzero(case["tag"] >= 0)[0]
    dy = _row_dy(views[net.out.weight], case["tag"][tagged], rows)[:, 0]
    _report("critic dY per tagged row, %d rows" % rows, np.abs(dy - want[tagged]), 6 * U * np.abs(want[tagged]) + 2.0 ** -25)
    assert np.all(dy[want[tagged] == 0] == 0)
    if rows % 128:
        assert views[net.out.weight][0, 0].item() == 0.0
    loss = 0.5 * (want ** 2).sum() / rows
    _report("critic loss statistic, %d rows" % rows, abs(batch.keep["stats"][0].item() - loss), (rows + 160) * 4 * U * loss + 1e-30)


# ---- the discriminator
def _disc(in_dim, hidden, max_side):
    import torch
    from deepmimic_b200.rollout import build_discriminator
    torch.manual_seed(0)
    net = build_discriminator(in_dim, hidden=hidden).cuda()
    tc, acc = _learner(net, "disc", 2 * max_side)
    return net, tc, acc


class _DiscBatch:
    def __init__(self, agent, expert, rows, mean, istd, clip, lr=0.0, mom=0.0, wd=0.0, reg=0.0, gp=0.0, a_idx=None, e_idx=None):
        import torch
        from deepmimic_b200.capi import DmLearnDiscBatch
        k = self.keep = dict(agent=_t(agent, torch.float32), expert=_t(expert, torch.float32), mean=_t(mean, torch.float32), istd=_t(istd, torch.float32),
                             a_idx=_t(np.arange(rows) if a_idx is None else a_idx, torch.int64), e_idx=_t(np.arange(rows) if e_idx is None else e_idx, torch.int64),
                             stats=torch.zeros(6, device="cuda"))
        p = lambda name: k[name].data_ptr()
        self.b = DmLearnDiscBatch(agent=p("agent"), expert=p("expert"), agent_idx=p("a_idx"), expert_idx=p("e_idx"), rows=rows, in_mean=p("mean"),
                                  in_istd=p("istd"), in_clip=clip, stepsize=lr, momentum=mom, weight_decay=wd, logit_reg_weight=reg,
                                  grad_penalty_weight=gp, stats=p("stats"))


@pytest.mark.parametrize("rows,max_side", [(1, 256), (127, 256), (128, 256), (129, 256), (254, 254)])
def test_disc_head_rows(rows, max_side):
    """agent rows at [0, rows), expert rows at [E, E + rows), E = pad128(rows) (rows = 128: E = rows), logits 0, +-1 and beyond on both
    sides, row by row; padding rows of both sides (logit 5) carry dY = 0 and stay out of the statistics.  Accuracies and mean logits are
    exact (multiples of 0.5 summed in fp32), the loss within two roundings"""
    S, hidden = 226, (1024, 512)
    case = L.disc_case(rows)
    net, tc, _ = _disc(S, hidden, max_side)
    w0, b0, w1, b1 = L.tagged_trunk(S, *hidden)
    _load(net.hidden[0], w0, b0); _load(net.hidden[1], w1, b1)
    tags = np.concatenate([case["tag_a"], case["tag_e"]])
    _load(net.logit, *L.output_layer(tags, np.concatenate([case["d_a"], case["d_e"]]), hidden[1], padding_value=5.0))
    tc.set_weights()
    batch = _DiscBatch(L.state_rows(case["tag_a"], S, 5), L.state_rows(case["tag_e"], S, 6), rows, np.zeros(S), np.ones(S), 0.0)
    _, views = _grad(tc, batch)
    ref = L.disc_rows(case["d_a"], case["d_e"])
    dy = _row_dy(views[net.logit.weight], tags, rows)[:, 0]
    want = np.concatenate([ref["dy_agent"], ref["dy_expert"]])
    _report("disc dY per row, %d rows per side" % rows, np.abs(dy - want), 4 * U * np.abs(want) + 2.0 ** -25)
    if rows % 128:
        assert views[net.logit.weight][0, 0].item() == 0.0, "padding rows carry dY"
    st = batch.keep["stats"].cpu().numpy()
    inv = np.float32(1) / np.float32(rows)
    exact = lambda x: np.float32(np.float32(x) * inv)
    assert st[2] == exact((case["d_e"] > 0).sum()) and st[3] == exact((case["d_a"] < 0).sum()), st
    assert st[4] == exact(case["d_e"].astype(np.float64).sum()) and st[5] == exact(case["d_a"].astype(np.float64).sum()), st
    _report("disc loss statistic, %d rows per side" % rows, abs(st[0] - ref["loss"]), 3 * U * ref["loss"])


def _penalty_ref(net, x_e):
    """float64 d(0.5 sum_r ||dd/dx_r||^2)/dW over the real expert rows x_e (normalised, fp16-rounded), ReLU masks of the fp16-rounded forward
    (constant under the double backward); and the same with every weight replaced by its magnitude (the sum of |terms| of each entry)"""
    import torch
    out = []
    for absolute in (False, True):
        Ws = [(l.weight.detach().double(), l.bias.detach().double()) for l in list(net.hidden) + [net.logit]]
        x = x_e.double().clone().requires_grad_(True)
        h, masks = x, []
        r16 = lambda v: v.half().double()
        for W, b in Ws[:2]:
            z = h @ W.T + b
            masks.append((z > 0).double())
            h = r16(torch.relu(z))
        params = [W.abs().clone().requires_grad_(True) if absolute else W.clone().requires_grad_(True) for W, _ in Ws]
        h = x
        for (W, b), m in zip(zip(params[:2], [b for _, b in Ws[:2]]), masks):
            h = m * (h @ W.T + b)
        d = h @ params[2].T
        g, = torch.autograd.grad(d.sum(), x, create_graph=True)
        pen = 0.5 * (g ** 2).sum()
        out.append([v.detach() for v in torch.autograd.grad(pen, params)])
    return out


@pytest.mark.parametrize("rows", [5, 128])
def test_disc_penalty_weight_gradients(rows):
    """the penalty's contribution, grad(gp_w = 1) - grad(gp_w = 0) times rows, against the float64 double backward over the real expert rows
    only (rows = 5: 123 padding rows per side, whose activations relu(b) > 0 would add if they were seeded).  Bound per entry: the e, q0, q1
    operands of the penalty's dW GEMMs are fp16 (hi only, 2^-11 each, two of them on a path), the chain's fp32 sums (K u over
    K = Ng + N0 + N1), applied to the sum of |terms|; plus the fp32 cancellation of the two grads (2 u (|s| + |q|))"""
    import torch
    S, hidden = 226, (1024, 512)
    net, tc, _ = _disc(S, hidden, 256)
    with torch.no_grad():
        for l in net.hidden:
            l.bias.uniform_(0.05, 0.2)
    tc.set_weights()
    g = np.random.default_rng(rows)
    agent, expert = g.standard_normal((rows, S)).astype(np.float32), g.standard_normal((rows, S)).astype(np.float32)
    grads = []
    for gp in (0.0, 1.0):
        batch = _DiscBatch(agent, expert, rows, np.zeros(S), np.ones(S), 0.0, gp=gp)
        flat, views = _grad(tc, batch)
        grads.append({p: v.double() * rows for p, v in views.items()})
    ref, mag = _penalty_ref(net, _t(expert).half().float())
    K = 256 + 1024 + 512
    c = 2 * 2.0 ** -11 + 3 * K * U
    for i, l in enumerate(list(net.hidden) + [net.logit]):
        pen = grads[1][l.weight] - grads[0][l.weight]
        err = (pen - ref[i]).abs()
        bound = c * mag[i] + 2 * U * (grads[0][l.weight].abs() + pen.abs()) + 1e-30
        _report("disc penalty dW, layer %d, %d rows" % (i, rows), err.cpu().numpy(), bound.cpu().numpy())
        assert (grads[1][l.bias] == grads[0][l.bias]).all(), "the penalty has no bias gradient"


# ---- the input preparation
def _prep_net(S, hidden, G=0, seed=0):
    """a critic whose first-layer units all have positive pre-activations (b0 = 8, small weights), so dW0 = dZ0 x^T with dZ0 != 0 (the
    critic's dY = V - target is never 0 at target -100)"""
    import torch
    from deepmimic_b200.rollout import build_critic
    torch.manual_seed(seed)
    net = build_critic(S, G, hidden=hidden).cuda()
    with torch.no_grad():
        net.hidden[0].weight.mul_(1e-3); net.hidden[0].bias.fill_(8.0); net.hidden[1].bias.fill_(1.0)
        if G:
            net.gate_common.weight.mul_(1e-3); net.gate_common.bias.fill_(4.0)
            for l in net.gate_hidden:
                l.bias.fill_(1.0)
    return net


def _recover(dw, ref_col):
    """the fp16 operand row from a one-row first-layer gradient [units, inputs]: column k over the column of the exact 1.0 input, at the unit
    with the largest |dZ0| (both columns are dZ0 (hi + lo) times an fp16 input, one fp32 rounding each: 3 u relative)"""
    dw = dw.double().cpu().numpy()
    k = int(np.argmax(np.abs(dw[:, ref_col])))
    assert dw[k, ref_col] != 0.0
    return dw[k] / dw[k, ref_col]


def _prep_case(S, clip, seed, window=300000):
    """one sample far into a window of `window` rows: column 0 is exactly 1.0 (mean 0, istd 1); the others normalised to +-1.5 clip (past
    the clip either way, and inside), std at the 0.02 floor on every fourth column.  The mean and 1 / std arrays are followed by NaN in memory
    (the in_dim tail must not be read)"""
    g = np.random.default_rng(seed)
    mean = np.concatenate([[0.0], g.uniform(-1, 1, S - 1)]).astype(np.float32)
    std = np.concatenate([[1.0], np.where(np.arange(1, S) % 4 == 0, 0.02, g.uniform(0.2, 2.0, S - 1))]).astype(np.float32)
    istd = (np.float32(1) / std).astype(np.float32)
    lim = 1.5 * (clip if clip > 0 else 10.0)
    s = (mean + g.uniform(-lim, lim, S).astype(np.float32) * std).astype(np.float32)
    s[0] = 1.0
    nan = np.full(64, np.nan, np.float32)
    return s, np.concatenate([mean, nan]), np.concatenate([istd, nan]), window - 7


def _window_states(s, window, idx, S):
    import torch
    states = torch.randn(window, S, device="cuda")
    states[idx] = _t(s)
    return states


@pytest.mark.parametrize("S,clip", [(63, 5.0), (64, 5.0), (65, 2.0), (227, 5.0), (128, 0.0)])
def test_prep_operands(S, clip):
    """the PPO networks' and the discriminator's prepared fp16 operand of one row gathered from far into the window, element by element against the
    float64 normalised input: clipped at +-clip, or (clip off, in_clip <= 0) as is; the in_dim tail (NaN past the normaliser arrays) unread"""
    import torch
    from deepmimic_b200.capi import DmLearnBatch
    s, mean, istd, idx = _prep_case(S, clip, S)
    want = L.prep_operand(s, mean[:S], istd[:S], clip)
    states = _window_states(s, 300000, idx, S)
    net = _prep_net(S, (256, 128))
    tc, _ = _learner(net, "critic", 128)
    batch = _Batch(np.zeros((1, S)), [idx], 1, mean, istd, clip, targets=np.full(300000, -100.0))   # targets are read by sample index
    batch.keep["states"] = states
    batch.b.states = states.data_ptr()
    g, views = _grad(tc, batch)
    assert torch.isfinite(g).all()
    x = _recover(views[net.hidden[0].weight], 0)
    _report("PPO prep operand, in %d, clip %g" % (S, clip), np.abs(x - want), L.prep_bound(want) + 3 * U * np.abs(want))
    # the discriminator's agent and expert sides
    dnet, dtc, _ = _disc(S, (256, 128), 128)
    with torch.no_grad():
        dnet.hidden[0].weight.mul_(1e-3); dnet.hidden[0].bias.fill_(8.0); dnet.hidden[1].bias.fill_(1.0)
    dtc.set_weights()
    for side in ("agent", "expert"):
        other = _t(mean[:S]).reshape(1, S)   # normalised exactly to 0
        db = _DiscBatch(np.zeros((1, S)), np.zeros((1, S)), 1, mean, istd, clip, a_idx=[idx if side == "agent" else 0], e_idx=[idx if side == "expert" else 0])
        db.keep.update(agent=states if side == "agent" else other, expert=states if side == "expert" else other)
        db.b.agent, db.b.expert = db.keep["agent"].data_ptr(), db.keep["expert"].data_ptr()
        _, dv = _grad(dtc, db)
        # one row of each side: dW0 = dZ0_a x_a^T + dZ0_e x_e^T with the other side's input all zero
        x = _recover(dv[dnet.hidden[0].weight], 0)
        _report("disc prep operand (%s side), in %d, clip %g" % (side, S, clip), np.abs(x - want), L.prep_bound(want) + 3 * U * np.abs(want))


def test_prep_past_fp16_range():
    """clip off and a deviation of 2000 standard deviations at the 0.02 floor: the normalised input 1e5 is past fp16's range; the operand
    saturates at +-65504 (the clip the preparation applies when none is set) instead of reaching the GEMMs as inf"""
    import torch
    S = 64
    s, mean, istd, idx = _prep_case(S, 0.0, 9)
    istd[1], mean[1], s[1], istd[2], mean[2], s[2] = 50.0, 0.0, 2000.0, 50.0, 0.0, -2000.0
    want = np.clip(L.prep_operand(s, mean[:S], istd[:S], 0.0), -L.HALF_MAX, L.HALF_MAX)
    states = _window_states(s, 1000, 3, S)
    net = _prep_net(S, (128, 128))
    with torch.no_grad():
        net.hidden[0].weight[:, 1:3] = 0.0     # the forward stays as it was; dW0 still carries the operand
    tc, _ = _learner(net, "critic", 128)
    batch = _Batch(np.zeros((1, S)), [3], 1, mean, istd, 0.0, targets=np.full(1000, -100.0))
    batch.keep["states"] = states
    batch.b.states = states.data_ptr()
    g, views = _grad(tc, batch)
    assert torch.isfinite(g).all(), "an input past fp16's range makes the step's gradient non-finite"
    x = _recover(views[net.hidden[0].weight], 0)
    _report("prep operand past fp16's range", np.abs(x - want), L.prep_bound(want) + 3 * U * np.abs(want))


@pytest.mark.parametrize("S,G", [(62, 3), (226, 3), (100, 40)])
def test_gated_prep_operands(S, G):
    """the gated critic's trunk operand [state | goal] (goal columns across a 64-column chunk boundary at S = 62) and the gate's own goal tile,
    with the goal's clip (2) distinct from the state's (5): goal values normalised to +-3.5 must clip at 2, state values at 5"""
    import torch
    s, mean, istd, idx = _prep_case(S, 5.0, S + G)
    gg = np.random.default_rng(G)
    g_mean = gg.uniform(-1, 1, G).astype(np.float32); g_mean[0] = 0.0
    g_std = gg.uniform(0.5, 2, G).astype(np.float32); g_std[0] = 1.0
    g_istd = (np.float32(1) / g_std).astype(np.float32)
    goal = (g_mean + np.array([3.5, -3.5, 1.25] * G, np.float32)[:G] * g_std).astype(np.float32)
    goal[0] = 1.0
    want_s = L.prep_operand(s, mean[:S], istd[:S], 5.0)
    want_g = L.prep_operand(goal, g_mean, g_istd, 2.0)
    states = _window_states(s, 300000, idx, S)
    goals = torch.randn(300000, G, device="cuda")
    goals[idx] = _t(goal)
    net = _prep_net(S, (256, 128), G=G)
    tc, _ = _learner(net, "critic", 128, gated=True)
    batch = _Batch(np.zeros((1, S)), [idx], 1, mean, istd, 5.0, targets=np.full(300000, -100.0),
                   goal=dict(goals=np.zeros((1, G)), g_mean=g_mean, g_istd=g_istd, g_clip=2.0))
    batch.keep.update(states=states, goals=goals)
    batch.b.states, batch.b.goals = states.data_ptr(), goals.data_ptr()
    g, views = _grad(tc, batch)
    assert torch.isfinite(g).all()
    x = _recover(views[net.hidden[0].weight], 0)
    want = np.concatenate([want_s, want_g])
    _report("gated trunk operand, %d + %d" % (S, G), np.abs(x - want), L.prep_bound(want) + 3 * U * np.abs(want))
    xg = _recover(views[net.gate_common.weight], 0)
    _report("gated gate-tile operand, %d + %d" % (S, G), np.abs(xg - want_g), L.prep_bound(want_g) + 3 * U * np.abs(want_g))


# ---- the optimiser
def _opt_bound(w, acc, lr, mom, wd, steps):
    """float64 trajectory of momentum_update with zero gradients and its error bound: per step the kernel rounds wd w (u), the FMA
    m acc + g (u) and the FMA w - lr acc (u); the accumulator's error reaches w through lr"""
    w, a = w.astype(np.float64), acc.astype(np.float64)
    ew, ea = np.zeros_like(w), np.zeros_like(w)
    for _ in range(steps):
        w2, a2 = L.momentum_update(w, a, 0.0, lr, mom, wd)
        ea = mom * ea + wd * ew + 2 * U * (np.abs(a2) + wd * np.abs(w))
        ew = ew + lr * ea + U * (np.abs(w2) + lr * np.abs(a2))
        w, a = w2, a2
    return w, a, ew, ea


def test_optimiser_arithmetic_ppo():
    """a critic batch whose values equal their targets has dY = 0 on every row, so every gradient is exactly 0 and three steps are pure
    optimiser arithmetic: accumulators preloaded with nonzero values, momentum 0.9, acc = m acc + wd w on the weights and m acc on the
    biases (no decay), w -= lr acc"""
    import torch
    from deepmimic_b200.rollout import build_critic
    rows, S, hidden = 129, 100, (256, 128)
    torch.manual_seed(0)
    net = build_critic(S, hidden=hidden).cuda()
    with torch.no_grad():
        net.out.weight.zero_(); net.out.bias.fill_(0.75)
        for l in net.hidden:
            l.bias.uniform_(-0.5, 0.5)
    tc, acc = _learner(net, "critic", 256)
    with torch.no_grad():   # the output layer's accumulators stay 0, so its parameters, and every row's dY = 0, stay as they are
        for p, a in acc.items():
            if p is not net.out.weight and p is not net.out.bias:
                a.uniform_(-1.0, 1.0)
    before = {p: (p.detach().double().cpu().numpy(), acc[p].double().cpu().numpy()) for p in acc}
    lr, mom, wd = 1e-2, 0.9, 1e-3
    batch = _Batch(np.random.default_rng(0).standard_normal((rows, S)), np.arange(rows), rows, np.zeros(S), np.ones(S), 0.0,
                   targets=np.full(rows, 0.75, np.float32), lr=lr, mom=mom, wd=wd)
    for _ in range(3):
        tc.step(batch.b)
    torch.cuda.synchronize()
    for name, p in [("w%d" % i, l.weight) for i, l in enumerate(list(net.hidden) + [net.out])] + [("b%d" % i, l.bias) for i, l in enumerate(list(net.hidden) + [net.out])]:
        w0, a0 = before[p]
        w, a, ew, ea = _opt_bound(w0, a0, lr, mom, 0.0 if name[0] == "b" else wd, 3)
        _report("optimiser, critic %s weights" % name if name[0] == "w" else "optimiser, critic %s bias" % name,
                np.abs(p.detach().double().cpu().numpy() - w), ew + 1e-45)
        _report("optimiser, critic %s accumulator" % name, np.abs(acc[p].double().cpu().numpy() - a), ea + 1e-45)


def test_optimiser_arithmetic_disc():
    """a discriminator with zero logit weights: the hidden layers' loss and penalty gradients are exactly 0, so one step updates them by
    acc = m acc + wd w (no logit regulariser: it acts on the logit layer's weights only) and acc = m acc on their biases"""
    import torch
    rows, S, hidden = 129, 100, (256, 128)
    net, tc, acc = _disc(S, hidden, 256)
    with torch.no_grad():
        net.logit.weight.zero_(); net.logit.bias.fill_(0.25)
        for l in net.hidden:
            l.bias.uniform_(-0.5, 0.5)
        for a in acc.values():
            a.uniform_(-1.0, 1.0)
    tc.set_weights()
    before = {p: (p.detach().double().cpu().numpy(), acc[p].double().cpu().numpy()) for p in acc}
    lr, mom, wd = 1e-2, 0.9, 1e-3
    g = np.random.default_rng(1)
    batch = _DiscBatch(g.standard_normal((rows, S)), g.standard_normal((rows, S)), rows, np.zeros(S), np.ones(S), 0.0, lr=lr, mom=mom, wd=wd,
                       reg=0.5, gp=10.0)
    tc.step(batch.b)
    torch.cuda.synchronize()
    for i, l in enumerate(net.hidden):
        for p, decay in ((l.weight, wd), (l.bias, 0.0)):
            w0, a0 = before[p]
            w, a, ew, ea = _opt_bound(w0, a0, lr, mom, decay, 1)
            _report("optimiser, disc layer %d %s" % (i, "weights" if decay else "bias"), np.abs(p.detach().double().cpu().numpy() - w), ew + 1e-45)
            _report("optimiser, disc layer %d %s accumulator" % (i, "weights" if decay else "bias"), np.abs(acc[p].double().cpu().numpy() - a), ea + 1e-45)


def test_zz_print_worst():
    """the worst error / bound of every check this module ran"""
    for k, v in sorted(WORST.items()):
        print("  %-60s %.3f" % (k, v))
