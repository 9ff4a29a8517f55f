"""Data-parallel training on the GPU: the tensor-core step split around its gradient (dm_learn_*grad / dm_learn_*apply) against the fused step,
bit for bit, for the plain and gated actor and critic and the discriminator; the flat gradient against torch autograd; and two ranks on one
GPU (a gloo group over CUDA tensors, spawned processes joined before the test returns) whose updates equal, bit for bit, one process that
adds the two ranks' gradients and applies half their sum; and a world-2 Trainer on one GPU."""
import os

import pytest

pytestmark = pytest.mark.gpu
WORLD = 2
HP = dict(actor_stepsize=2.5e-6, actor_momentum=0.9, actor_weight_decay=5e-4, critic_stepsize=1e-2, critic_momentum=0.9, critic_weight_decay=1e-3,
          ratio_clip=0.2, norm_adv_clip=4.0, epochs=1)
DISC_HP = dict(stepsize=1e-2, momentum=0.9, weight_decay=1e-3, logit_reg_weight=0.05, grad_penalty=5.0)


def _ppo_case(kind, rank=0):
    """a random-shapes PPO rollout and window (the learner GPU tests' stand-ins); rank > 0 permutes the window's environments"""
    import torch
    if kind == "plain":
        from tests.test_learner_gpu import _random_shapes
    else:
        from tests.test_gated_learner_gpu import _random_shapes
    ro, traj = _random_shapes()
    if rank:
        perm = torch.randperm(traj["returns"].shape[1], generator=torch.Generator().manual_seed(rank)).cuda()
        traj = {k: v[:, perm] for k, v in traj.items()}
    return ro, traj


def _disc_case(rank=0):
    """a random-shapes discriminator rollout and pools (the disc learner GPU tests' stand-ins); rank > 0 draws from other pools, with the same
    AMP normaliser (the ranks' normalisers are summed over the ranks, so they are equal)"""
    from tests.test_disc_learner_gpu import _pools, _rollout
    agent, expert = _pools(None, "random shapes", 3000)
    ro = _rollout(agent, expert, hidden=(200, 96))
    if rank:
        agent, expert = agent[500 * rank:] + 0.1, expert.flip(0)
    return ro, agent.contiguous(), expert.contiguous()


def _params_and_accs(ln, params):
    return [p.detach().clone() for p in params] + [ln.acc[p].clone() for p in params]


def _restore(ln, params, saved):
    import torch
    with torch.no_grad():
        for p, s in zip(params, saved[:len(params)]):
            p.copy_(s)
        for p, s in zip(params, saved[len(params):]):
            ln.acc[p].copy_(s)


def _bit_equal(a, b):
    import torch
    return all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("kind", ["plain", "gated"])
def test_grad_then_apply_is_the_fused_step_bit_for_bit(kind):
    import torch
    from deepmimic_b200.learner import PPOLearner
    ro, traj = _ppo_case(kind)
    ln = PPOLearner(ro, **HP, minibatch_size=200, backend="tensor_core")
    params = ln.critic_params + ln.actor_params
    w = ln.window(traj)
    g = torch.Generator(device="cuda").manual_seed(9)
    steps = [(torch.randint(0, w["R"], (200,), device="cuda", generator=g),
              w["exp_idx"][torch.randint(0, w["exp_idx"].numel(), (200,), device="cuda", generator=g)]) for _ in range(4)]
    start = _params_and_accs(ln, params)
    st = torch.cuda.current_stream().cuda_stream
    runs = []
    for split in (False, True):
        _restore(ln, params, start)
        ln._tc_critic.set_weights(stream=st)
        ln._tc_actor.set_weights(stream=st)
        keep, actor, critic = ln._tc_batch(w)
        grads = {tc: torch.full((tc.grad_size(),), float("nan"), device="cuda") for tc in (ln._tc_actor, ln._tc_critic)}
        for c, a in steps:
            for tc, batch, idx in ((ln._tc_critic, critic, c), (ln._tc_actor, actor, a)):
                batch.idx = idx.data_ptr()
                if split:
                    tc.grad(batch, grads[tc], stream=st)
                    tc.apply(batch, grads[tc], 1.0, stream=st)
                else:
                    tc.step(batch, stream=st)
        torch.cuda.synchronize()
        runs.append(_params_and_accs(ln, params) + [keep["stats_a"].clone(), keep["stats_c"].clone()])
    assert _bit_equal(runs[0], runs[1])
    assert not _bit_equal(runs[0][:len(params)], start[:len(params)])


@pytest.mark.parametrize("kind", ["plain", "gated"])
def test_flat_gradient_is_the_mean_gradient_without_weight_decay(kind):
    """the flat buffer against fp32 autograd through fp16-rounded activations (the learner GPU tests' reference), the weight decay's
    gradient taken out; the same tolerance as those tests"""
    import torch
    from deepmimic_b200.learner import PPOLearner
    if kind == "plain":
        from tests.test_learner_gpu import _fp16_activation_grads, _no_tf32
    else:
        from tests.test_gated_learner_gpu import _fp16_activation_grads, _no_tf32
    ro, traj = _ppo_case(kind)
    ln = PPOLearner(ro, **HP, minibatch_size=200, backend="tensor_core")
    w = ln.window(traj)
    c = torch.arange(0, 400, 2, device="cuda")
    a = w["exp_idx"][:200].contiguous()
    st = torch.cuda.current_stream().cuda_stream
    ln._tc_critic.set_weights(stream=st)
    ln._tc_actor.set_weights(stream=st)
    keep, actor, critic = ln._tc_batch(w)
    flat = {}
    for tc, batch, idx in ((ln._tc_critic, critic, c), (ln._tc_actor, actor, a)):
        batch.idx = idx.data_ptr()
        flat[tc] = torch.empty(tc.grad_size(), device="cuda")
        tc.grad(batch, flat[tc], stream=st)
    views = {**ln._tc_critic.grad_views(flat[ln._tc_critic]), **ln._tc_actor.grad_views(flat[ln._tc_actor])}
    assert len(views) == len(ln.critic_params) + len(ln.actor_params)
    with _no_tf32():
        ref = _fp16_activation_grads(ln, w, c, a)
    names = {p: n for net in (ro.critic, ro.policy) for n, p in net.named_parameters()}
    for p, r in zip(ln.critic_params + ln.actor_params, ref):
        wd = ln.critic_weight_decay if any(p is q for q in ln.critic_params) else ln.actor_weight_decay
        want = r - wd * p.detach() if names[p].endswith("weight") else r
        err = ((views[p] - want).norm() / want.norm().clamp_min(1e-30)).item()
        assert err <= 1e-2, (names[p], err)


def test_disc_grad_then_apply_is_the_fused_step_bit_for_bit():
    import torch
    from deepmimic_b200.learner import AMPDiscLearner
    ro, agent, expert = _disc_case()
    ln = AMPDiscLearner(ro, **DISC_HP, batch_size=700, steps=1, backend="tensor_core")
    g = torch.Generator(device="cuda").manual_seed(4)
    steps = [(torch.randint(0, agent.shape[0], (700,), device="cuda", generator=g),
              torch.randint(0, expert.shape[0], (700,), device="cuda", generator=g)) for _ in range(4)]
    start = _params_and_accs(ln, ln.params)
    st = torch.cuda.current_stream().cuda_stream
    runs = []
    for split in (False, True):
        _restore(ln, ln.params, start)
        ln._tc.set_weights(stream=st)
        keep, batch = ln._tc_batch(agent, expert)
        grad = torch.full((ln._tc.grad_size(),), float("nan"), device="cuda")
        for a, e in steps:
            batch.agent_idx, batch.expert_idx = a.data_ptr(), e.data_ptr()
            if split:
                ln._tc.grad(batch, grad, stream=st)
                ln._tc.apply(batch, grad, 1.0, stream=st)
            else:
                ln._tc.step(batch, stream=st)
        torch.cuda.synchronize()
        runs.append(_params_and_accs(ln, ln.params) + [keep["stats"].clone()])
    assert _bit_equal(runs[0], runs[1])
    assert not _bit_equal(runs[0][:len(ln.params)], start[:len(ln.params)])


def test_disc_flat_gradient_is_the_mean_gradient_without_the_regularisers():
    """the discriminator's flat buffer (least-squares loss plus the weighted penalty) against fp32 autograd with a double backward through
    fp16-rounded activations (the disc learner GPU tests' reference), weight decay and logit regulariser taken out; their tolerance"""
    import torch
    from deepmimic_b200.learner import AMPDiscLearner
    from tests.test_disc_learner_gpu import _fp16_activation_ref, _no_tf32
    ro, agent, expert = _disc_case()
    ln = AMPDiscLearner(ro, **DISC_HP, batch_size=700, steps=1, backend="tensor_core")
    g = torch.Generator(device="cuda").manual_seed(5)
    a = torch.randint(0, agent.shape[0], (700,), device="cuda", generator=g)
    e = torch.randint(0, expert.shape[0], (700,), device="cuda", generator=g)
    st = torch.cuda.current_stream().cuda_stream
    ln._tc.set_weights(stream=st)
    keep, batch = ln._tc_batch(agent, expert)
    batch.agent_idx, batch.expert_idx = a.data_ptr(), e.data_ptr()
    flat = torch.empty(ln._tc.grad_size(), device="cuda")
    ln._tc.grad(batch, flat, stream=st)
    views = ln._tc.grad_views(flat)
    with _no_tf32():
        ref, _ = _fp16_activation_ref(ln, agent, expert, a, e)
    names = {p: n for n, p in ln.disc.named_parameters()}
    for p, r in zip(ln.params, ref):
        want = r
        if names[p].endswith("weight"):
            want = want - ln.weight_decay * p.detach() - (ln.logit_reg_weight * p.detach() if names[p] == "logit.weight" else 0.0)
        err = ((views[p] - want).norm() / want.norm().clamp_min(1e-30)).item()
        assert err <= 1e-2, (names[p], err)


def test_split_entries_refuse_bad_input():
    import torch
    from deepmimic_b200.learner import PPOLearner
    ro, traj = _ppo_case("plain")
    ln = PPOLearner(ro, **HP, minibatch_size=200, backend="tensor_core")
    keep, actor, critic = ln._tc_batch(ln.window(traj))
    with pytest.raises(ValueError, match="grad"):
        ln._tc_actor.grad(actor, torch.empty(ln._tc_actor.grad_size() - 1, device="cuda"))
    actor.stepsize = -1.0
    with pytest.raises(RuntimeError, match="stepsize"):
        ln._tc_actor.apply(actor, torch.zeros(ln._tc_actor.grad_size(), device="cuda"))
    with pytest.raises(RuntimeError, match="finite"):
        ln._tc_critic.apply(critic, torch.zeros(ln._tc_critic.grad_size(), device="cuda"), float("inf"))


# ---- two ranks on one GPU
def _worker(rank, scenario, init_file, out_dir):
    import torch
    import torch.distributed as dist
    os.environ.setdefault("GLOO_SOCKET_IFNAME", "lo")
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method="file://" + init_file, rank=rank, world_size=WORLD)
    try:
        torch.save(SCENARIOS[scenario](rank, dist.group.WORLD), os.path.join(out_dir, "rank%d.pt" % rank))
    finally:
        dist.destroy_process_group()


def _run(tmp_path, scenario):
    import torch
    import torch.multiprocessing as mp
    os.environ["DP_TEST_DIR"] = str(tmp_path)
    mp.spawn(_worker, args=(scenario, str(tmp_path / "init"), str(tmp_path)), nprocs=WORLD, join=True)
    return [torch.load(tmp_path / ("rank%d.pt" % r), map_location="cuda:0", weights_only=False) for r in range(WORLD)]


def _ppo_rank(rank, group):
    from deepmimic_b200.learner import PPOLearner
    ro, traj = _ppo_case("plain", rank)
    ln = PPOLearner(ro, **dict(HP, epochs=2), minibatch_size=400, backend="tensor_core", seed=5 + rank, process_group=group)
    ln.update(traj)
    return _params_and_accs(ln, ln.critic_params + ln.actor_params)


def _disc_rank(rank, group):
    from deepmimic_b200.learner import AMPDiscLearner
    ro, agent, expert = _disc_case(rank)
    ln = AMPDiscLearner(ro, **DISC_HP, batch_size=1400, steps=3, backend="tensor_core", seed=7 + rank, process_group=group)
    ln.update(agent, expert)
    return _params_and_accs(ln, ln.params)


TRAIN_PPO = dict(
    AgentType="PPO", ActorNet="fc_2layers_1024units", ActorStepsize=1e-5, ActorMomentum=0.9, ActorWeightDecay=5e-4, ActorInitOutputScale=0.01,
    CriticNet="fc_2layers_1024units", CriticStepsize=0.01, CriticMomentum=0.9, CriticWeightDecay=0, Discount=0.95, TDLambda=0.95,
    MiniBatchSize=1024, Epochs=1, RatioClip=0.2, NormAdvClip=4, TarClipFrac=0.2, ActorStepsizeDecay=0.5, InitSamples=1, NormalizerSamples=1000000,
    ExpAnnealSamples=64000000, ExpParamsBeg={"Rate": 1, "Noise": 0.05}, ExpParamsEnd={"Rate": 0.2, "Noise": 0.05}, OutputIters=10,
    IntOutputIters=0, TestEpisodes=4)
TRAIN_AGENTS = dict(spinkick=TRAIN_PPO,
                    target_amp=dict(TRAIN_PPO, AgentType="AMP", ActorNet="fc_2layers_gated_1024units", CriticNet="fc_2layers_gated_1024units",
                                    ActorStepsize=2e-6, DiscNet="fc_2layers_1024units", DiscStepSize=1e-5, DiscMomentum=0.9, DiscWeightDecay=5e-4,
                                    DiscLogitRegWeight=0.05, DiscGradPenalty=10, DiscBatchSize=1024, DiscStepsPerBatch=1, DiscBufferSize=20000,
                                    DiscInitOutputScale=1, TaskRewardLerp=0.5))
TRAIN_ARGS = dict(spinkick=["--arg_file", "args/train_humanoid3d_spinkick_args.txt"],
                  target_amp=["--motion_file", "data/datasets/synthetic_locomotion_56.txt", "--arg_file",
                              "args/train_amp_target_humanoid3d_locomotion_args.txt"])


def _trainer_rank(scene, rank, group):
    import torch
    from deepmimic_b200.assets import asset_root
    from deepmimic_b200.trainer import AgentConfig, Trainer
    tr = Trainer(TRAIN_ARGS[scene], AgentConfig(TRAIN_AGENTS[scene]), asset_root(), 2 * 384, window_steps=16, backend="tensor_core", seed=0,
                 device=0, log_path=os.path.join(os.environ["DP_TEST_DIR"], "log.txt"), process_group=group)
    rows = [tr.iteration() for _ in range(3)]
    s = tr.state_dict()
    out = dict(rows=rows, nets=s["nets"], has_log=tr.log is not None)
    if tr.amp:
        out["expert"] = tr.expert_buf.filled()[:256].clone()
    tr.close()
    torch.cuda.synchronize()
    return out


SCENARIOS = dict(ppo=_ppo_rank, disc=_disc_rank, train_spinkick=lambda r, g: _trainer_rank("spinkick", r, g),
                 train_target_amp=lambda r, g: _trainer_rank("target_amp", r, g))


def test_two_ranks_ppo_update_is_half_the_sum_of_their_gradients(tmp_path):
    import torch
    from deepmimic_b200.learner import PPOLearner, minibatch_schedule
    res = _run(tmp_path, "ppo")
    assert _bit_equal(res[0], res[1])
    # one process: each rank's window and minibatch draws, grad on each, the two buffers added, apply(scale 0.5)
    cases = [_ppo_case("plain", r) for r in range(WORLD)]
    ro = cases[0][0]
    ln = PPOLearner(ro, **dict(HP, epochs=2), minibatch_size=200, backend="tensor_core")
    params = ln.critic_params + ln.actor_params
    st = torch.cuda.current_stream().cuda_stream
    ln._tc_critic.set_weights(stream=st)
    ln._tc_actor.set_weights(stream=st)
    ws = [ln.window(traj) for _, traj in cases]
    tcs = [ln._tc_batch(w) for w in ws]
    scheds = [list(minibatch_schedule(w["R"], w["exp_idx"].numel(), 200, 2, torch.Generator(device="cuda").manual_seed(5 + r), "cuda"))
              for r, w in enumerate(ws)]
    assert len(scheds[0]) == len(scheds[1])
    for k in range(len(scheds[0])):
        for tc, which in ((ln._tc_critic, 2), (ln._tc_actor, 1)):
            g = [torch.empty(tc.grad_size(), device="cuda") for _ in range(WORLD)]
            for r in range(WORLD):
                c, a = scheds[r][k]
                batch = tcs[r][which]
                idx = c if which == 2 else ws[r]["exp_idx"][a].contiguous()
                batch.idx = idx.data_ptr()
                tc.grad(batch, g[r], stream=st)
                torch.cuda.synchronize()
            tc.apply(tcs[0][which], g[0] + g[1], 0.5, stream=st)
    torch.cuda.synchronize()
    assert _bit_equal(res[0], _params_and_accs(ln, params))


def test_two_ranks_disc_update_is_half_the_sum_of_their_gradients(tmp_path):
    import torch
    from deepmimic_b200.learner import AMPDiscLearner
    res = _run(tmp_path, "disc")
    assert _bit_equal(res[0], res[1])
    cases = [_disc_case(r) for r in range(WORLD)]
    ln = AMPDiscLearner(cases[0][0], **DISC_HP, batch_size=700, steps=3, backend="tensor_core")
    st = torch.cuda.current_stream().cuda_stream
    ln._tc.set_weights(stream=st)
    batches = [ln._tc_batch(agent, expert) for _, agent, expert in cases]
    gens = [torch.Generator(device="cuda").manual_seed(7 + r) for r in range(WORLD)]
    for _ in range(3):
        g = [torch.empty(ln._tc.grad_size(), device="cuda") for _ in range(WORLD)]
        for r, (_, agent, expert) in enumerate(cases):
            a = torch.randint(0, agent.shape[0], (700,), generator=gens[r], device="cuda")
            e = torch.randint(0, expert.shape[0], (700,), generator=gens[r], device="cuda")
            batch = batches[r][1]
            batch.agent_idx, batch.expert_idx = a.data_ptr(), e.data_ptr()
            ln._tc.grad(batch, g[r], stream=st)
            torch.cuda.synchronize()
        ln._tc.apply(batches[0][1], g[0] + g[1], 0.5, stream=st)
    torch.cuda.synchronize()
    assert _bit_equal(res[0], _params_and_accs(ln, ln.params))


@pytest.mark.parametrize("scene", ["spinkick", "target_amp"])
def test_trainer_on_two_ranks_of_one_gpu(tmp_path, scene):
    """three world-2 Trainer iterations, 384 environments per rank: identical networks on both ranks, finite losses, the same rows, one log,
    and (target_amp) different expert rows on each rank"""
    import math
    import torch
    res = _run(tmp_path, "train_" + scene)
    for name in res[0]["nets"]:
        assert all(torch.equal(res[0]["nets"][name][k], res[1]["nets"][name][k]) for k in res[0]["nets"][name]), name
    for r in res:
        for row in r["rows"]:
            assert all(math.isfinite(row[k]) for k in row if k.endswith("_Loss")), row
            assert row["Samples"] == 16 * 768 * (row["Iteration"] + 1)
    strip = lambda rows: [{k: v for k, v in row.items() if k != "Wall_Time"} for row in rows]
    assert str(strip(res[0]["rows"])) == str(strip(res[1]["rows"]))
    assert [r["has_log"] for r in res] == [True, False]
    assert len((tmp_path / "log.txt").read_text().splitlines()) == 1 + 3
    if scene == "target_amp":
        assert not torch.equal(res[0]["expert"], res[1]["expert"])
