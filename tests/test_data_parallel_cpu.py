"""CPU tests of data-parallel training (deepmimic_b200/learner.py: DataParallel, process_group=) on the torch backend: two ranks in a gloo
group, each a spawned process that is joined before the test returns.  The PPO and discriminator updates leave both ranks with bit-identical
parameters and accumulators, equal to a float64 restatement that averages the two ranks' minibatch gradients by hand; the normalisers' sum
over ranks equals one update over the concatenated samples; unequal windows are refused; and the Trainer's bookkeeping on two ranks over the
CPU stand-in env (global sample count, one log, refusals, a world-2 checkpoint that resumes bit for bit, another world size refused)."""
import os

import pytest

torch = pytest.importorskip("torch")
import torch.distributed as dist
import torch.multiprocessing as mp

from deepmimic_b200.learner import (AMPDiscLearner, PPOLearner, bound_loss, clipped_surrogate, critic_loss, disc_grad_penalty, disc_input_grad,
                                    disc_loss, gaussian_log_prob, minibatch_schedule)
from deepmimic_b200.rollout import DeviceNormalizer

pytestmark = pytest.mark.skipif(not dist.is_available() or not dist.is_gloo_available(), reason="torch.distributed with gloo")

WORLD = 2


def _worker(rank, scenario, init_file, out_dir):
    os.environ.setdefault("GLOO_SOCKET_IFNAME", "lo")
    dist.init_process_group("gloo", init_method="file://" + init_file, rank=rank, world_size=WORLD)
    try:
        torch.save(SCENARIOS[scenario](rank, dist.group.WORLD), os.path.join(out_dir, "rank%d.pt" % rank))
    finally:
        dist.destroy_process_group()


def _run(tmp_path, scenario):
    """the scenario's result of every rank"""
    os.environ["DP_TEST_DIR"] = str(tmp_path)
    mp.spawn(_worker, args=(scenario, str(tmp_path / "init"), str(tmp_path)), nprocs=WORLD, join=True)
    return [torch.load(tmp_path / ("rank%d.pt" % r), weights_only=False) for r in range(WORLD)]


# ---- the scenarios (run in each rank)
def _ppo(rank, group):
    from tests.test_learner_cpu import HP, _setup, _window
    T, N = 4, 8
    ro, _ = _setup(N, T, seed=rank)                      # different initial weights: the learner broadcasts rank 0's
    ln = PPOLearner(ro, **dict(HP, minibatch_size=16, epochs=2), seed=5 + rank, process_group=group)
    traj = _window(ro, T, N, seed=10 + rank)
    start = {k: v.detach().clone() for k, v in list(ro.policy.state_dict().items()) + [("critic." + k, v) for k, v in ro.critic.state_dict().items()]}
    w = ln.window(traj)
    g = torch.Generator()
    g.set_state(ln.gen.get_state())
    sched = list(minibatch_schedule(w["R"], w["exp_idx"].numel(), ln.minibatch_size, ln.epochs, g))
    stats = ln.update(traj)
    return dict(start=start, w={k: v for k, v in w.items() if torch.is_tensor(v)}, sched=sched, minibatch=ln.minibatch_size,
                params=[p.detach().clone() for p in ln.actor_params + ln.critic_params],
                accs=[ln.acc[p].clone() for p in ln.actor_params + ln.critic_params],
                stats={k: v.clone() for k, v in stats.items()}, s_norm=(ro.s_norm.mean, ro.s_norm.std), bounds=(ln.bound_min, ln.bound_max))


def _disc(rank, group):
    from tests.test_disc_learner_cpu import HP, _pools, _setup
    ro, _ = _setup(seed=rank)
    ln = AMPDiscLearner(ro, **dict(HP, batch_size=32, steps=3), seed=7 + rank, process_group=group)
    agent, expert = _pools(seed=20 + rank, Ra=100 + 20 * rank, Re=90)
    start = [p.detach().clone() for p in ln.params]
    g = torch.Generator()
    g.set_state(ln.gen.get_state())
    draws = []
    for _ in range(ln.steps):
        a = torch.randint(0, agent.shape[0], (ln.batch_size,), generator=g)
        draws.append((a, torch.randint(0, expert.shape[0], (ln.batch_size,), generator=g)))
    stats = ln.update(agent, expert)
    n = ro.amp_norm
    return dict(start=start, agent=agent, expert=expert, draws=draws, params=[p.detach().clone() for p in ln.params],
                accs=[ln.acc[p].clone() for p in ln.params], stats={k: v.clone() for k, v in stats.items()}, norm=(n.mean, n.std))


def _normalizer(rank, group):
    g = torch.Generator().manual_seed(30 + rank)
    n = DeviceNormalizer(6, group_ids=[0, 0, 1, 1, -1, 0])
    x = torch.randn(50 + 30 * rank, 6, generator=g) * 2.0 + rank
    n.record(x)
    n.update(all_reduce=lambda t: dist.all_reduce(t, group=group))
    return dict(x=x, mean=n.mean, std=n.std, count=n.count)


def _unequal(rank, group):
    from tests.test_learner_cpu import HP, _setup, _window
    T, N = 4 + rank, 8
    ro, _ = _setup(N, T)
    ln = PPOLearner(ro, **HP, process_group=group)
    try:
        ln.update(_window(ro, T, N))
    except ValueError as e:
        return str(e)
    return None


def _agent():
    from tests.test_train_cpu import AMP, _edit
    return _edit(AMP, InitSamples=40, NormalizerSamples=150, TarClipFrac=0.2, DiscBatchSize=12, DiscBufferSize=50, MiniBatchSize=16, OutputIters=2,
                 TestEpisodes=4)


def _trainer(n, group=None, log_path=None, n_env=None):
    """a Trainer of n environments in all (n_env per rank) over the CPU stand-in env of tests/test_train_cpu.py"""
    from deepmimic_b200 import trainer as tr
    from tests.test_train_cpu import _StandInEnv

    class Env(_StandInEnv):
        def expert_sample_count(self, set_to=None):
            before = getattr(self, "count", 0)
            if set_to is not None:
                self.count = set_to
            return before

    world = dist.get_world_size(group) if group is not None else 1
    torch.manual_seed(0)
    cfg = tr.AgentConfig(_agent())
    return tr.Trainer(["--scene", "stand-in"], cfg, "", n, window_steps=4, backend="torch", seed=3, env=Env(n_env or n // world, cfg.amp),
                      test_env=Env(-(-4 // world), cfg.amp), log_path=log_path, process_group=group)


def _trainer_state(t):
    s = t.state_dict()
    return dict(nets=s["nets"], accs=s["accs"], norms={k: v["mean"] for k, v in s["norms"].items()}, buffers=s["buffers"]["agent"]["rows"])


def _trainer_run(rank, group):
    from deepmimic_b200.train import rank_path
    out = os.environ["DP_TEST_DIR"]
    refused = []
    for kw in (dict(n=15), dict(n=16, n_env=7)):   # a total the world does not divide; an env of another size than the rank's share
        try:
            _trainer(kw["n"], group, n_env=kw.get("n_env"))
        except ValueError as e:
            refused.append(str(e))
    a = _trainer(16, group, log_path=os.path.join(out, "log.txt"))
    rows_a = [a.iteration() for _ in range(5)]
    counts = dict(samples=list(a.env.sample_counts), expert_start=a.env.expert_sample_count(), has_log=a.log is not None)
    a.close()
    b = _trainer(16, group)
    rows_b = [b.iteration() for _ in range(3)]
    ckpt = rank_path(os.path.join(out, "agent0_checkpoint.pt"), rank)
    b.save(ckpt)
    c = _trainer(16, group)
    c.load(ckpt)
    rows_b += [c.iteration() for _ in range(2)]
    strip = lambda r: {k: x for k, x in r.items() if k != "Wall_Time"}
    return dict(refused=refused, rows_a=[strip(r) for r in rows_a], rows_b=[strip(r) for r in rows_b], counts=counts, ckpt=ckpt,
                state_a=_trainer_state(a), state_c=_trainer_state(c))


SCENARIOS = dict(ppo=_ppo, disc=_disc, normalizer=_normalizer, unequal=_unequal, trainer=_trainer_run)


def _same_on_every_rank(res, key):
    for a, b in zip(res[0][key], res[1][key]):
        assert torch.equal(a, b), key


def _rel(got, want):
    return ((got.double() - want).norm() / want.norm()).item()


def test_ppo_update_is_the_ranks_mean_gradient_step(tmp_path):
    from tests.test_learner_cpu import HP, _setup
    res = _run(tmp_path, "ppo")
    _same_on_every_rank(res, "params")
    _same_on_every_rank(res, "accs")
    assert res[0]["minibatch"] == 8
    for k in res[0]["stats"]:   # the statistics are the ranks' means, the same on both
        assert torch.equal(res[0]["stats"][k], res[1]["stats"][k]), k
    # float64 restatement: rank 0's initial networks, each step on the mean of both ranks' gradients, then the weight decay and the momentum
    ro, _ = _setup(8, 4, seed=0)
    policy, critic = ro.policy.double(), ro.critic.double()
    with torch.no_grad():
        for name, p in list(policy.named_parameters()) + [("critic." + n, p) for n, p in critic.named_parameters()]:
            p.copy_(res[0]["start"][name])
    a_params = [p for n, p in policy.named_parameters() if n != "logstd"]
    c_params = list(critic.parameters())
    acc = {p: torch.zeros_like(p) for p in a_params + c_params}
    mean, std = (x.double() for x in res[0]["s_norm"])
    lo, hi = (x.double() for x in res[0]["bounds"])
    W = [{k: v.double() if v.is_floating_point() else v for k, v in r["w"].items()} for r in res]

    def step(params, loss_fn, stepsize, momentum, wd, net):
        gs = [torch.autograd.grad(loss_fn(r), params) for r in range(WORLD)]
        names = {p: n for n, p in net.named_parameters()}
        with torch.no_grad():
            for i, p in enumerate(params):
                g = (gs[0][i] + gs[1][i]) / WORLD + (wd * p if names[p].endswith("weight") else 0.0)
                acc[p].mul_(momentum).add_(g)
                p.sub_(stepsize * acc[p])

    for k in range(len(res[0]["sched"])):
        def c_loss(r):
            idx = res[r]["sched"][k][0]
            return critic_loss(critic((W[r]["states"][idx] - mean) / std)[:, 0], W[r]["norm_tar"][idx])

        def a_loss(r):
            idx = W[r]["exp_idx"][res[r]["sched"][k][1]]
            mu = policy((W[r]["states"][idx] - mean) / std)
            ratio = (gaussian_log_prob(W[r]["norm_a"][idx], mu, policy.logstd.detach()) - W[r]["old_logp"][idx]).exp()
            return -clipped_surrogate(W[r]["adv"][idx], ratio, HP["ratio_clip"]).mean() + bound_loss(mu, lo, hi)

        step(c_params, c_loss, HP["critic_stepsize"], HP["critic_momentum"], HP["critic_weight_decay"], critic)
        step(a_params, a_loss, HP["actor_stepsize"], HP["actor_momentum"], HP["actor_weight_decay"], policy)
    start = [res[0]["start"][n] for n, _ in policy.named_parameters() if n != "logstd"] + [res[0]["start"]["critic." + n] for n, _ in critic.named_parameters()]
    # weights to a few fp32 roundings of their values (a delta of 1e-3 on weights of 0.3 keeps ~4 digits in fp32)
    for got, want, p0, a_got, p in zip(res[0]["params"], [p.detach() for p in a_params + c_params], start, res[0]["accs"], a_params + c_params):
        assert _rel(a_got, acc[p]) <= 1e-5                # the accumulators: the steps' gradient sums
        assert (got.double() - want).abs().max().item() <= 1e-6 and not torch.equal(got, p0)


def test_disc_update_is_the_ranks_mean_gradient_step(tmp_path):
    from tests.test_disc_learner_cpu import HP, _setup
    res = _run(tmp_path, "disc")
    _same_on_every_rank(res, "params")
    _same_on_every_rank(res, "accs")
    ro, _ = _setup(seed=0)
    disc = ro.disc.double()
    params = list(disc.parameters())
    with torch.no_grad():
        for p, s in zip(params, res[0]["start"]):
            p.copy_(s)
    acc = {p: torch.zeros_like(p) for p in params}
    mean, std = (x.double() for x in res[0]["norm"])
    names = {p: n for n, p in disc.named_parameters()}
    for k in range(len(res[0]["draws"])):
        gs = []
        for r in res:
            a, e = r["draws"][k]
            d_a = disc((r["agent"].double()[a] - mean) / std)[:, 0]
            d_e, g = disc_input_grad(disc, (r["expert"].double()[e] - mean) / std)
            gs.append(torch.autograd.grad(disc_loss(d_e, d_a) + HP["grad_penalty"] * disc_grad_penalty(g), params))
        with torch.no_grad():
            for i, p in enumerate(params):
                g = (gs[0][i] + gs[1][i]) / WORLD
                if names[p].endswith("weight"):
                    g = g + HP["weight_decay"] * p + (HP["logit_reg_weight"] * p if names[p] == "logit.weight" else 0.0)
                acc[p].mul_(HP["momentum"]).add_(g)
                p.sub_(HP["stepsize"] * acc[p])
    for got, p0, a_got, p in zip(res[0]["params"], res[0]["start"], res[0]["accs"], params):
        assert _rel(a_got, acc[p]) <= 1e-5
        assert (got.double() - p.detach()).abs().max().item() <= 1e-6 and not torch.equal(got, p0)


def test_normalizer_sum_over_ranks_equals_one_update_over_all_samples(tmp_path):
    res = _run(tmp_path, "normalizer")
    one = DeviceNormalizer(6, group_ids=[0, 0, 1, 1, -1, 0])
    one.record(torch.cat([r["x"] for r in res]))
    one.update()
    for r in res:
        assert r["count"] == one.count == 130
        torch.testing.assert_close(r["mean"], one.mean, rtol=1e-6, atol=1e-6)
        torch.testing.assert_close(r["std"], one.std, rtol=1e-6, atol=1e-6)


def test_unequal_windows_are_refused(tmp_path):
    res = _run(tmp_path, "unequal")
    assert all(r is not None and "window sizes differ" in r for r in res)


def _equal(a, b):
    if torch.is_tensor(a):
        return torch.equal(a, b)
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_equal(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))
    return a == b or (a != a and b != b)   # NaN rows (no finished episode yet) compare equal


def test_trainer_on_two_ranks(tmp_path):
    """global sample count, one log, refusals, identical networks on both ranks, a world-2 checkpoint that resumes bit for bit, and a
    checkpoint refused at another world size"""
    res = _run(tmp_path, "trainer")
    for r in res:
        assert len(r["refused"]) == 2 and "divisible by the world size" in r["refused"][0] and "share" in r["refused"][1]
        assert r["counts"]["samples"] == [4 * 16 * (k + 1) for k in range(5)]           # both ranks' samples
        assert [row["Samples"] for row in r["rows_a"]] == [4 * 16 * (k + 1) for k in range(5)]
        assert _equal(r["rows_a"], r["rows_b"])                                          # 3 + 2 iterations around a checkpoint
        assert _equal(r["state_a"], r["state_c"])
    assert [r["counts"]["has_log"] for r in res] == [True, False]
    assert res[0]["counts"]["expert_start"] != res[1]["counts"]["expert_start"]          # disjoint expert draws
    assert _equal(res[0]["rows_a"], res[1]["rows_a"])                                    # every rank logs the same row
    assert _equal(res[0]["state_a"]["nets"], res[1]["state_a"]["nets"]) and _equal(res[0]["state_a"]["accs"], res[1]["state_a"]["accs"])
    assert not _equal(res[0]["state_a"]["buffers"], res[1]["state_a"]["buffers"])        # per-rank disc buffers
    log = (tmp_path / "log.txt").read_text().splitlines()
    assert len(log) == 1 + 5                                                             # a header and one row per iteration, once
    assert res[1]["ckpt"].endswith("agent0_checkpoint.rank1.pt")
    one = _trainer(16)
    with pytest.raises(ValueError, match="world size"):
        one.load(res[0]["ckpt"])
