"""The AMP discriminator's update on the GPU: the tensor-core step (dm_learn_disc_step: kernels/dm_learn.cu and the backward GEMMs of
kernels/dm_mlp.cu) against fp32 torch double-backward autograd (TF32 off), minibatches smaller than the workspace, determinism, whole updates on
both backends, the direction of the steps, the re-tiling of the rollout's discriminator and a short imitate_amp training loop."""
import contextlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
IMITATE_AMP = ["--scene", "imitate_amp", "--arg_file", "args/train_humanoid3d_walk_args.txt"]
DOG_AMP = ["--scene", "imitate_amp", "--arg_file", "args/train_dog3d_trot_args.txt"]
HP = dict(stepsize=1e-3, momentum=0.9, weight_decay=5e-4, logit_reg_weight=0.05, grad_penalty=10.0)


@contextlib.contextmanager
def _no_tf32():
    import torch
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


class _AMPShapeEnv:
    """a stand-in AMP env on the GPU with an arbitrary AMP observation width: enough surface for BatchedRollout(disc=...) and AMPDiscLearner"""

    def __init__(self, M):
        import torch
        self.num_envs, self.device, self.M = 128, torch.device("cuda", 0), M

    def get_name(self): return "Imitate AMP"
    def enable_amp_task_reward(self): return False
    def get_state_size(self, agent_id=0): return 4
    def get_action_size(self, agent_id=0): return 2
    def get_goal_size(self, agent_id=0): return 0
    def build_state_norm_groups(self, agent_id=0): return np.zeros(4, dtype=np.int32)
    def build_state_offset(self, agent_id=0): return np.zeros(4)
    def build_state_scale(self, agent_id=0): return np.ones(4)
    def build_action_offset(self, agent_id=0): return np.zeros(2)
    def build_action_scale(self, agent_id=0): return np.ones(2)
    def get_amp_obs_size(self): return self.M
    def get_amp_obs_offset(self): return np.zeros(self.M)
    def get_amp_obs_scale(self): return np.ones(self.M)
    def get_amp_obs_norm_group(self): return np.zeros(self.M, dtype=np.int32)


def _sim_pools(asset_root, args, n):
    """agent AMP observations of n environments after a few random-action steps, and expert AMP observations of the reference motion"""
    import torch
    from deepmimic_b200.env import DeepMimicBatchEnv
    env = DeepMimicBatchEnv(args, num_envs=n, asset_root=asset_root, seed=3)
    env.reset(True)
    g = torch.Generator(device="cuda").manual_seed(1)
    lo = torch.as_tensor(env.build_action_bound_min(), dtype=torch.float32, device="cuda")
    hi = torch.as_tensor(env.build_action_bound_max(), dtype=torch.float32, device="cuda")
    off = torch.as_tensor(env.build_action_offset(), dtype=torch.float32, device="cuda")
    scl = torch.as_tensor(env.build_action_scale(), dtype=torch.float32, device="cuda")
    for _ in range(4):
        a = torch.clamp(-off + 0.25 / scl * torch.randn(n, env.get_action_size(), device="cuda", generator=g), lo, hi)
        env.set_action(a.contiguous())
        env.update(1.0 / 600.0, 20)
        env.reset()
    agent = env.record_amp_obs_agent().clone()
    expert = env.record_amp_obs_expert().clone()
    torch.cuda.synchronize()
    return agent, expert


def _pools(asset_root, case, n):
    import torch
    if case == "random shapes":
        g = torch.Generator(device="cuda").manual_seed(7)
        return torch.randn(n, 100, device="cuda", generator=g) * 0.5 + 0.2, torch.randn(n, 100, device="cuda", generator=g) * 0.7 - 0.1
    return _sim_pools(asset_root, IMITATE_AMP if case == "imitate_amp humanoid3d" else DOG_AMP, n)


def _rollout(agent, expert, hidden=(1024, 512), seed=0):
    """BatchedRollout with a random discriminator on an AMP stand-in of the pools' width; amp_norm from the pools, clipped at 3 (the clip is
    exercised)"""
    import torch
    from deepmimic_b200.rollout import BatchedRollout, build_discriminator
    torch.manual_seed(seed)
    M = agent.shape[1]
    ro = BatchedRollout(_AMPShapeEnv(M), exp_rate=0.0, disc=build_discriminator(M, hidden=hidden))
    both = torch.cat([agent, expert])
    ro.amp_norm.set_mean_std(both.mean(0).cpu().numpy(), both.std(0).clamp_min(0.05).cpu().numpy())
    ro.amp_norm.clip = 3.0
    return ro


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _fp16_activation_ref(ln, agent, expert, ai, ei):
    """fp32 autograd (double backward for the penalty) of the total loss through a forward whose normalised input and hidden activations are
    rounded to fp16, as the tensor-core forward stores them (the weights stay fp32: the kernels carry them as hi + lo).  Returns the gradients
    and the statistics [disc_loss, grad_penalty, acc_expert, acc_agent, logit_expert, logit_agent]"""
    import torch
    from deepmimic_b200.learner import disc_accuracies, disc_grad_penalty, disc_logit_reg_loss, disc_loss, disc_weight_decay_loss
    disc, norm = ln.disc, ln.ro.amp_norm
    r16 = lambda x: x.half().float()

    def fwd(x):
        h = r16(x)
        for l in disc.hidden:
            h = r16(torch.relu(l(h)))
        return disc.logit(h)[:, 0]
    d_a = fwd(norm.normalize(agent[ai]))
    xe = norm.normalize(expert[ei]).detach().requires_grad_(True)
    d_e = fwd(xe)
    g, = torch.autograd.grad(d_e.sum(), xe, create_graph=True)
    loss, gp = disc_loss(d_e, d_a), disc_grad_penalty(g)
    total = loss + ln.grad_penalty * gp + ln.weight_decay * disc_weight_decay_loss(disc) + ln.logit_reg_weight * disc_logit_reg_loss(disc)
    grads = torch.autograd.grad(total, ln.params)
    acc_e, acc_a = disc_accuracies(d_e, d_a)
    return grads, [v.item() for v in (loss, gp, acc_e, acc_a, d_e.mean(), d_a.mean())]


def _tc_step(ln, agent, expert, ai, ei, rows=None):
    """one tensor-core step on the rows ai, ei (rows: a smaller minibatch in the workspace); returns the statistics it wrote"""
    import torch
    st = torch.cuda.current_stream().cuda_stream
    ln._tc.set_weights(stream=st)
    keep, batch = ln._tc_batch(agent.contiguous(), expert.contiguous())
    if rows is not None:
        batch.rows = rows
    ln.minibatch_step(agent, expert, ai, ei, None, (keep, batch))
    torch.cuda.synchronize()
    return keep["stats"].tolist()


STAT_NAMES = ("disc_loss", "grad_penalty", "acc_expert", "acc_agent", "logit_expert", "logit_agent")


def _check_step(ln, agent, expert, ai, ei, label, rows=None):
    import torch
    with _no_tf32():
        ref, ref_stats = _fp16_activation_ref(ln, agent, expert, ai, ei)
    before = [p.detach().clone() for p in ln.params]
    stats = _tc_step(ln, agent, expert, ai, ei, rows)
    errs = [_rel(b - p.detach(), r) for b, p, r in zip(before, ln.params, ref)]
    serr = [abs(s - r) / max(abs(r), 1.0) for s, r in zip(stats, ref_stats)]
    names = [n for n, _ in ln.disc.named_parameters()]
    print("%s: relative gradient error per tensor vs fp16-activation fp32 autograd: %s; statistics %s (worst error %.1e)"
          % (label, ", ".join("%s %.1e" % (n, e) for n, e in zip(names, errs)), {k: round(v, 5) for k, v in zip(STAT_NAMES, stats)}, max(serr)))
    assert all(np.isfinite(stats))
    return max(errs), max(serr)


@pytest.mark.parametrize("gp,reg", [(0.0, 0.0), (10.0, 0.0), (0.0, 0.05), (10.0, 0.05)])
@pytest.mark.parametrize("case,B", [("imitate_amp humanoid3d", 4096), ("dog3d", 2048), ("random shapes", 200)])
def test_step_gradients_and_statistics_match_fp32(asset_root, case, B, gp, reg):
    """one step at stepsize 1, momentum 0 from zero accumulators: w_before - w_after against fp32 double-backward autograd of the same minibatch
    through fp16-rounded activations, relative Frobenius error per parameter tensor <= 2e-3; the statistics within 1e-3 (relative, or absolute
    below 1)"""
    import torch
    from deepmimic_b200.learner import AMPDiscLearner
    agent, expert = _pools(asset_root, case, max(B, 512))
    ro = _rollout(agent, expert, hidden=(200, 96) if case == "random shapes" else (1024, 512))
    ln = AMPDiscLearner(ro, **dict(HP, stepsize=1.0, momentum=0.0, grad_penalty=gp, logit_reg_weight=reg), batch_size=B, steps=1, backend="tensor_core")
    g = torch.Generator(device="cuda").manual_seed(B)
    ai = torch.randint(0, agent.shape[0], (B,), device="cuda", generator=g)
    ei = torch.randint(0, expert.shape[0], (B,), device="cuda", generator=g)
    e_grad, e_stat = _check_step(ln, agent, expert, ai, ei, "%s (%d inputs), B = %d, grad_penalty %g, logit_reg %g" % (case, agent.shape[1], B, gp, reg))
    assert e_grad <= 2e-3 and e_stat <= 1e-3


@pytest.mark.parametrize("rows", [200, 3000])
def test_minibatch_smaller_than_the_workspace(asset_root, rows):
    """a workspace sized for 4096 rows per side steps 200- and 3000-row minibatches: the same bounds against the same reference"""
    import torch
    from deepmimic_b200.learner import AMPDiscLearner
    agent, expert = _pools(asset_root, "imitate_amp humanoid3d", 4096)
    ro = _rollout(agent, expert)
    ln = AMPDiscLearner(ro, **dict(HP, stepsize=1.0, momentum=0.0), batch_size=4096, steps=1, backend="tensor_core")
    g = torch.Generator(device="cuda").manual_seed(rows)
    ai = torch.randint(0, agent.shape[0], (rows,), device="cuda", generator=g)
    ei = torch.randint(0, expert.shape[0], (rows,), device="cuda", generator=g)
    e_grad, e_stat = _check_step(ln, agent, expert, ai, ei, "%d rows per side in a 4096-row workspace" % rows, rows=rows)
    assert e_grad <= 2e-3 and e_stat <= 1e-3


def _state(ro):
    return [p.detach().clone() for p in ro.disc.parameters()]


def test_updates_deterministic_and_backends_agree(asset_root):
    """two tensor-core updates from the same weights and seed: bit-identical weights and statistics.  A whole update (20 steps of 4096 + 4096
    rows) on both backends: per tensor |w_tc - w_torch| <= 2e-2 |w_torch - w_0|"""
    import torch
    from deepmimic_b200.learner import AMPDiscLearner
    agent, expert = _pools(asset_root, "imitate_amp humanoid3d", 4096)
    ro = _rollout(agent, expert)
    w0 = _state(ro)
    runs = []
    for backend in ("tensor_core", "tensor_core", "torch"):
        with torch.no_grad():
            for p, w in zip(ro.disc.parameters(), w0):
                p.copy_(w)
        with _no_tf32():
            s = AMPDiscLearner(ro, **HP, batch_size=4096, steps=20, seed=5, backend=backend).update(agent, expert)
        torch.cuda.synchronize()
        runs.append((_state(ro), {k: v.item() for k, v in s.items()}))
    (w_a, s_a), (w_b, s_b), (w_th, s_th) = runs
    assert all(torch.equal(a, b) for a, b in zip(w_a, w_b)) and s_a == s_b
    worst = 0.0
    for n, a, t, z in zip([n for n, _ in ro.disc.named_parameters()], w_a, w_th, w0):
        e = (a - t).norm().item() / (t - z).norm().item()
        worst = max(worst, e)
        assert e <= 2e-2, (n, e)
    print("update of 20 steps x (4096 + 4096) rows: worst |w_tc - w_torch| / |w_torch - w_0| %.1e; torch %s; tensor cores %s"
          % (worst, {k: round(v, 5) for k, v in s_th.items()}, {k: round(v, 5) for k, v in s_a.items()}))
    for k in s_th:
        assert abs(s_a[k] - s_th[k]) <= 1e-2 * max(abs(s_th[k]), 1.0), k


@pytest.mark.parametrize("backend", ["torch", "tensor_core"])
def test_fifty_steps_lower_the_loss_and_raise_both_accuracies(asset_root, backend):
    import torch
    from deepmimic_b200.learner import AMPDiscLearner, disc_accuracies
    agent, expert = _pools(asset_root, "imitate_amp humanoid3d", 4096)
    ro = _rollout(agent, expert)
    with torch.no_grad():   # logits centred on 0 over both pools: both accuracies start below 1
        ro.disc.logit.bias -= ro.disc(ro.amp_norm.normalize(torch.cat([agent, expert])))[:, 0].mean()
    ln = AMPDiscLearner(ro, **dict(HP, stepsize=1e-3), batch_size=1024, steps=50, seed=2, backend=backend)

    def full():
        with torch.no_grad(), _no_tf32():
            d_a, d_e = ro.disc(ro.amp_norm.normalize(agent))[:, 0], ro.disc(ro.amp_norm.normalize(expert))[:, 0]
            from deepmimic_b200.learner import disc_loss
            return disc_loss(d_e, d_a).item(), [v.item() for v in disc_accuracies(d_e, d_a)]
    l0, a0 = full()
    with _no_tf32():
        ln.update(agent, expert)
    l1, a1 = full()
    print("%s: disc_loss %.4f -> %.4f, acc_expert %.3f -> %.3f, acc_agent %.3f -> %.3f" % (backend, l0, l1, a0[0], a1[0], a0[1], a1[1]))
    assert l1 < l0 and a1[0] > a0[0] and a1[1] > a0[1]


def _amp_rollout(asset_root, n, critic=False):
    import torch
    from deepmimic_b200.env import DeepMimicBatchEnv
    from deepmimic_b200.rollout import BatchedRollout, build_critic, build_discriminator
    env = DeepMimicBatchEnv(IMITATE_AMP, num_envs=n, asset_root=asset_root, seed=4)
    env.reset(True)
    torch.manual_seed(0)
    kw = dict(critic=build_critic(env.get_state_size()), discount=0.95, td_lambda=0.95) if critic else {}
    return env, BatchedRollout(env, noise=0.2, exp_rate=0.8, backend="tensor_core", disc=build_discriminator(env.get_amp_obs_size()), seed=4, **kw)


def test_update_refreshes_the_rollouts_discriminator(asset_root):
    """after update() the rollout's re-tiled discriminator (new weights, amp_norm's statistics updated by the caller before update()) gives
    bit-identical logits and style rewards to a handle built afresh"""
    import torch
    from deepmimic_b200.learner import AMPDiscLearner
    env, ro = _amp_rollout(asset_root, 1024)
    traj = ro.collect(4)
    ro.amp_norm.update()
    M = env.get_amp_obs_size()
    agent = traj["amp_obs"].reshape(-1, M)
    expert = env.record_amp_obs_expert().clone()
    AMPDiscLearner(ro, **HP, batch_size=1024, steps=5, backend="tensor_core").update(agent, expert)
    x = agent[:1024].contiguous()
    st = torch.cuda.current_stream().cuda_stream
    r1, l1 = torch.empty(1024, device="cuda"), torch.empty(1024, device="cuda")
    ro._tc_disc.style_reward(x, r1, logit=l1, stream=st)
    ro.refresh_tensor_core_policy()
    r2, l2 = torch.empty_like(r1), torch.empty_like(l1)
    ro._tc_disc.style_reward(x, r2, logit=l2, stream=st)
    torch.cuda.synchronize()
    assert torch.equal(l1, l2) and torch.equal(r1, r2)


def test_imitate_amp_training_loop(asset_root):
    """512 environments: collect(32) with the discriminator and the critic, then the PPO update and the discriminator update on the tensor
    cores, three times: every output finite, the style rewards change from one iteration to the next"""
    import torch
    from deepmimic_b200.learner import AMPDiscLearner, PPOLearner
    env, ro = _amp_rollout(asset_root, 512, critic=True)
    ppo = PPOLearner(ro, actor_stepsize=2.5e-6, actor_momentum=0.9, actor_weight_decay=5e-4, critic_stepsize=1e-2, critic_momentum=0.9,
                     critic_weight_decay=1e-3, ratio_clip=0.2, norm_adv_clip=4.0, minibatch_size=4096, epochs=1, backend="tensor_core")
    dl = AMPDiscLearner(ro, **HP, batch_size=2048, steps=8, backend="tensor_core")
    M, styles = env.get_amp_obs_size(), []
    for it in range(3):
        traj = ro.collect(32)
        ro.amp_norm.update()
        s_ppo = ppo.update(traj)
        expert = torch.cat([env.record_amp_obs_expert().clone() for _ in range(4)])
        s_disc = dl.update(traj["amp_obs"].reshape(-1, M), expert)
        vals = [v.item() for v in list(s_ppo.values()) + list(s_disc.values())]
        styles.append(traj["style_rewards"].clone())
        print("iteration %d: mean style reward %.4f; PPO %s; discriminator %s" % (it, styles[-1].mean().item(), {k: round(v.item(), 4) for k, v in s_ppo.items()},
                                                                                  {k: round(v.item(), 4) for k, v in s_disc.items()}))
        assert all(np.isfinite(vals)) and all(torch.isfinite(traj[k]).all() for k in ("amp_obs", "disc_logits", "style_rewards", "returns"))
    assert not torch.equal(styles[0], styles[1]) and not torch.equal(styles[1], styles[2])
