"""The PPO learner of the gated task-scene networks on the GPU: the tensor-core minibatch step (dm_learn_gated_step: kernels/dm_learn.cu and
the backward GEMMs of kernels/dm_mlp.cu) against fp32 torch autograd (TF32 off), minibatches smaller than the workspace, whole updates on both
backends, determinism, the device re-tiling of the rollout's gated handles, the direction of the steps, a short target_amp training loop and
the update time."""
import contextlib
import copy
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
MINI = ["--motion_file", "data/datasets/test_clips_mini.txt"]
TARGET = MINI + ["--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]
HEADING = MINI + ["--arg_file", "args/train_amp_heading_humanoid3d_locomotion_args.txt"]
HP = dict(actor_stepsize=2.5e-6, actor_momentum=0.9, actor_weight_decay=5e-4, critic_stepsize=1e-2, critic_momentum=0.9, critic_weight_decay=1e-3,
          ratio_clip=0.2, norm_adv_clip=4.0, epochs=1)
DISC_HP = dict(stepsize=1e-3, momentum=0.9, weight_decay=5e-4, logit_reg_weight=0.05, grad_penalty=10.0)


@contextlib.contextmanager
def _no_tf32():
    import torch
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def _task_rollout(asset_root, task, n, backend, disc=False, seed=11):
    """BatchedRollout of a task scene with the pretrained gated actor fixture (noise 0.2, exploration 0.8) and a random gated critic"""
    import torch
    from deepmimic_b200.env import DeepMimicBatchEnv
    from deepmimic_b200.rollout import BatchedRollout, build_critic, build_discriminator, build_gated_policy, load_actor_weights
    from tests.test_task_scenes_cpu import fixture_task_actor
    a = fixture_task_actor(task)
    env = DeepMimicBatchEnv(TARGET if task == "target" else HEADING, num_envs=n, asset_root=asset_root, seed=seed)
    env._core.set_episode_limit(0.5, 3.0)
    env.reset(True)
    S, G = env.get_state_size(), env.get_goal_size()
    torch.manual_seed(0)
    kw = dict(disc=build_discriminator(env.get_amp_obs_size()), task_reward_lerp=0.5) if disc else {}
    ro = BatchedRollout(env, policy=load_actor_weights(build_gated_policy(S, G, env.get_action_size(), noise=0.2), a), noise=0.2, exp_rate=0.8,
                        backend=backend, critic=build_critic(S, G), discount=0.95, td_lambda=0.95, seed=seed, **kw)
    ro.s_norm.set_mean_std(a["s_norm_mean"], a["s_norm_std"]); ro.g_norm.set_mean_std(a["g_norm_mean"], a["g_norm_std"])
    ro.a_norm.set_mean_std(a["a_norm_mean"], a["a_norm_std"])
    return env, ro


class _GoalShapeEnv:
    """a stand-in goal-conditioned env on the GPU with arbitrary sizes: enough surface for BatchedRollout's and PPOLearner's constructors"""

    def __init__(self, n, S, G, A):
        import torch
        self.num_envs, self.device, self.S, self.G, self.A = n, torch.device("cuda", 0), S, G, A

    def get_state_size(self, agent_id=0): return self.S
    def get_goal_size(self, agent_id=0): return self.G
    def get_action_size(self, agent_id=0): return self.A
    def build_state_norm_groups(self, agent_id=0): return np.zeros(self.S, dtype=np.int32)
    def build_state_offset(self, agent_id=0): return np.full(self.S, 0.1)
    def build_state_scale(self, agent_id=0): return np.full(self.S, 0.5)
    def build_goal_norm_groups(self, agent_id=0): return np.zeros(self.G, dtype=np.int32)
    def build_goal_offset(self, agent_id=0): return np.full(self.G, -0.2)
    def build_goal_scale(self, agent_id=0): return np.full(self.G, 2.0)
    def build_action_offset(self, agent_id=0): return np.zeros(self.A)
    def build_action_scale(self, agent_id=0): return np.ones(self.A)
    def build_action_bound_min(self, agent_id=0): return np.full(self.A, -0.5)
    def build_action_bound_max(self, agent_id=0): return np.full(self.A, 0.5)
    def get_reward_min(self, agent_id=0): return 0.0
    def get_reward_max(self, agent_id=0): return 1.0
    def get_reward_fail(self, agent_id=0): return 0.0
    def get_reward_succ(self, agent_id=0): return 1.0


def _random_shapes(S=100, G=5, A=5, hidden=(180, 72), gc=40, gh=24, T=4, N=150):
    """trunk widths that pad differently to 64 (the rollout's handles) and to 128 (the learner's)"""
    import torch
    from deepmimic_b200.learner import gaussian_log_prob
    from deepmimic_b200.rollout import BatchedRollout, build_critic, build_gated_policy
    torch.manual_seed(1)
    env = _GoalShapeEnv(N, S, G, A)
    ro = BatchedRollout(env, policy=build_gated_policy(S, G, A, noise=0.3, init_output_scale=0.3, hidden=hidden, gate_common=gc, gate_hidden=gh),
                        critic=build_critic(S, G, hidden=hidden, gate_common=gc, gate_hidden=gh), discount=0.95, td_lambda=0.95, seed=2)
    g = torch.Generator(device="cuda").manual_seed(3)
    traj = dict(states=torch.randn(T, N, S, device="cuda", generator=g), goals=torch.randn(T, N, G, device="cuda", generator=g),
                actions=0.4 * torch.randn(T, N, A, device="cuda", generator=g), returns=25.0 * torch.rand(T, N, device="cuda", generator=g) - 2.0,
                values=20.0 * torch.rand(T, N, device="cuda", generator=g), explore=torch.rand(T, N, device="cuda", generator=g) < 0.7)
    with torch.no_grad():
        mu = ro.policy(ro.s_norm.normalize(traj["states"]), ro.g_norm.normalize(traj["goals"]))
        traj["logps"] = gaussian_log_prob(ro.a_norm.normalize(traj["actions"]), mu, ro.policy.logstd)
        traj["logps"] += 0.5 * (torch.rand(T, N, device="cuda", generator=g) - 0.5)
    return ro, traj


def _window(asset_root, case):
    if case == "random shapes":
        return _random_shapes()
    env, ro = _task_rollout(asset_root, case.split("_")[0], 512, "torch")
    return ro, ro.collect(16)


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _fp16_activation_grads(ln, w, c, a):
    """fp32 torch autograd of the same losses through a gated forward whose stored activations are rounded to fp16 as the tensor-core forward
    stores them: [ns | ng], ng, gc, g_l and h_l (the weights stay fp32: the kernels carry them as hi + lo)"""
    import torch
    from deepmimic_b200.learner import bound_loss, clipped_surrogate, critic_loss, gaussian_log_prob, weight_decay_loss
    ro = ln.ro
    r16 = lambda x: x.half().float()

    def fwd(net, head, idx):
        ns, ng = r16(ro.s_norm.normalize(w["states"][idx])), r16(ro.g_norm.normalize(w["goals"][idx]))
        gc = r16(torch.relu(net.gate_common(ng)))
        h = torch.cat([ns, ng], dim=-1)
        for l, gh, gb, gs in zip(net.hidden, net.gate_hidden, net.gate_bias, net.gate_scale):
            g = r16(torch.relu(gh(gc)))
            h = r16(torch.relu(2.0 * torch.sigmoid(gs(g)) * l(h) + gb(g)))
        return head(h)
    lc = critic_loss(fwd(ro.critic, ro.critic.out, c)[:, 0], w["norm_tar"][c]) + ln.critic_weight_decay * weight_decay_loss(ro.critic)
    mu = fwd(ro.policy, ro.policy.mean, a)
    ratio = (gaussian_log_prob(w["norm_a"][a], mu, ro.policy.logstd.detach()) - w["old_logp"][a]).exp()
    la = (-clipped_surrogate(w["adv"][a], ratio, ln.ratio_clip).mean() + bound_loss(mu, ln.bound_min, ln.bound_max)
          + ln.actor_weight_decay * weight_decay_loss(ro.policy))
    return torch.autograd.grad(lc, ln.critic_params) + torch.autograd.grad(la, ln.actor_params)


def _names(ro):
    return ["critic." + n for n, _ in ro.critic.named_parameters()] + ["actor." + n for n, p in ro.policy.named_parameters() if n != "logstd"]


def _one_step(ln, w, c, a, rows=None):
    """one tensor-core critic step and one actor step at the learner's settings; returns the parameters' change"""
    import torch
    params = ln.critic_params + ln.actor_params
    before = [p.detach().clone() for p in params]
    st = torch.cuda.current_stream().cuda_stream
    ln._tc_critic.set_weights(stream=st); ln._tc_actor.set_weights(stream=st)
    keep, actor, critic = ln._tc_batch(w)
    if rows is not None:
        actor.rows = critic.rows = rows
    ln.minibatch_step(w, c, a, None, (keep, actor, critic))
    torch.cuda.synchronize()
    return [b - p.detach() for b, p in zip(before, params)]


@pytest.mark.parametrize("case,B", [("target_amp", 4096), ("heading_amp", 4096), ("random shapes", 200)])
def test_gated_minibatch_gradients_match_fp32(asset_root, case, B):
    """one critic step and one actor step at stepsize 1 and momentum 0 (w -= g) from zero accumulators: g = w_before - w_after of all ten
    parameter pairs of both networks against fp32 torch autograd of the same minibatch through a forward with the same fp16-rounded
    activations, relative Frobenius error per tensor <= 1e-2 (the numbers are printed; the plain fp32 network's are printed beside them)"""
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
    got = _one_step(ln, w, c, a)
    errs = [_rel(d, r) for d, r in zip(got, ref)]
    errs16 = [_rel(d, r) for d, r in zip(got, ref16)]
    print("%s, B = %d: relative gradient error per tensor vs fp16-activation / plain fp32 torch: %s"
          % (case, B, ", ".join("%s %.1e / %.1e" % (n, e16, e) for n, e16, e in zip(_names(ro), errs16, errs))))
    assert len(errs16) == 40 and max(errs16) <= 1e-2


@pytest.mark.parametrize("rows", [200, 3000])
def test_gated_minibatch_smaller_than_the_workspace(asset_root, rows):
    """a workspace built for 4096 rows steps a smaller minibatch: gradients against the fp16-activation reference <= 1e-2"""
    import torch
    from deepmimic_b200.learner import PPOLearner
    ro, traj = _window(asset_root, "target_amp")
    hp = dict(HP, actor_stepsize=1.0, actor_momentum=0.0, critic_stepsize=1.0, critic_momentum=0.0, minibatch_size=4096)
    ln = PPOLearner(ro, **hp, backend="tensor_core")
    w = ln.window(traj)
    g = torch.Generator(device="cuda").manual_seed(rows)
    c = torch.randint(0, w["R"], (rows,), device="cuda", generator=g)
    a = w["exp_idx"][torch.randint(0, w["exp_idx"].numel(), (rows,), device="cuda", generator=g)]
    with _no_tf32():
        ref16 = _fp16_activation_grads(ln, w, c, a)
    errs16 = [_rel(d, r) for d, r in zip(_one_step(ln, w, c, a, rows=rows), ref16)]
    print("%d rows in a 4096-row workspace: worst relative gradient error vs the fp16-activation reference %.1e" % (rows, max(errs16)))
    assert max(errs16) <= 1e-2


def _weights(ro):
    return {k: v.detach().clone() for k, v in list(ro.policy.state_dict().items()) + [("critic." + k, v) for k, v in ro.critic.state_dict().items()]}


def _load(ro, w0):
    ro.policy.load_state_dict({k: v for k, v in w0.items() if not k.startswith("critic.")})
    ro.critic.load_state_dict({k[7:]: v for k, v in w0.items() if k.startswith("critic.")})


def test_gated_update_on_both_backends_agrees(asset_root):
    """a whole update() of a 16-step target_amp window of 4096 environments, minibatch 4096, same seed, from the same weights on both
    backends: per tensor r = |w_tc - w_torch| / |w_torch - w_0|, median <= 2e-2 and worst <= 1e-1; statistics within 2e-2.
    Measured on an H100: median 1.1e-2, worst 7.9e-2 on the actor's gate_scale.1.weight (the plain networks' worst is 2.8e-2).  That is the
    fp16 forward's deviation from the fp32 network, not the backward's: one step of that tensor matches the fp16-activation reference to 6e-4
    (test_gated_minibatch_gradients_match_fp32) and already differs from plain fp32 autograd by 6.8e-3 on the first minibatch; the update
    carries that deviation through 16 momentum steps."""
    import torch
    from deepmimic_b200.learner import PPOLearner
    env, ro = _task_rollout(asset_root, "target", 4096, "torch")
    traj = ro.collect(16)
    w0 = _weights(ro)
    with _no_tf32():
        s_th = PPOLearner(ro, **HP, minibatch_size=4096, seed=3).update(traj)
    w_th = _weights(ro)
    _load(ro, w0)
    s_tc = PPOLearner(ro, **HP, minibatch_size=4096, seed=3, backend="tensor_core").update(traj)
    torch.cuda.synchronize()
    w_tc = _weights(ro)
    errs = {}
    for k in w0:
        moved = (w_th[k] - w0[k]).norm().item()
        if k.endswith("logstd"):
            assert moved == 0.0 and torch.equal(w_tc[k], w0[k])
            continue
        errs[k] = (w_tc[k] - w_th[k]).norm().item() / max(moved, 1e-30)
    e = np.array(list(errs.values()))
    top = sorted(errs, key=errs.get, reverse=True)[:4]
    print("gated update of 16 x 4096: |w_tc - w_torch| / |w_torch - w_0| median %.1e, largest %s; torch %s; tensor cores %s"
          % (np.median(e), ", ".join("%s %.1e" % (k, errs[k]) for k in top), {k: round(v.item(), 5) for k, v in s_th.items()},
             {k: round(v.item(), 5) for k, v in s_tc.items()}))
    assert np.median(e) <= 2e-2 and e.max() <= 1e-1
    for k in s_th:
        assert abs(s_tc[k].item() - s_th[k].item()) <= 2e-2 * max(abs(s_th[k].item()), 1e-2), k


def test_first_minibatch_ratio_on_a_tensor_core_gated_rollout(asset_root):
    """a tensor-core gated rollout and a tensor-core gated learner see the same actor: the first minibatch's probability ratios are 1 to 1e-5
    and nothing is clipped"""
    import torch
    from deepmimic_b200.learner import PPOLearner
    env, ro = _task_rollout(asset_root, "target", 2048, "tensor_core")
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
    print("tensor-core gated rollout and learner: first-minibatch |ratio - 1| %.1e, clip fraction %g" % (r_err, tc[0]["stats_a"][1].item()))
    assert r_err <= 1e-5 and tc[0]["stats_a"][1].item() == 0.0


def test_gated_update_is_deterministic_and_refreshes_the_rollout(asset_root):
    """two tensor-core updates from the same weights and seed: bit-identical parameters and statistics; after update() the rollout's gated
    actor and critic, re-tiled on the device, give bit-identical outputs to handles rebuilt by refresh_tensor_core_policy() after the caller
    updated s_norm and g_norm"""
    import torch
    from deepmimic_b200.learner import PPOLearner
    env, ro = _task_rollout(asset_root, "target", 2048, "tensor_core")
    traj = ro.collect(8)
    s0, g0 = ro.s_norm.mean.clone(), ro.g_norm.mean.clone()
    ro.s_norm.update(); ro.g_norm.update()
    assert not torch.equal(s0, ro.s_norm.mean) and not torch.equal(g0, ro.g_norm.mean)
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
    s, g = traj["states"][-1].contiguous(), traj["goals"][-1].contiguous()
    st = torch.cuda.current_stream().cuda_stream
    a1, v1 = torch.empty(2048, env.get_action_size(), device="cuda"), torch.empty(2048, 1, device="cuda")
    ro._tc.forward(s, g, a1, stream=st); ro._tc_critic.forward(s, g, v1, stream=st)
    ro.refresh_tensor_core_policy()
    a2, v2 = torch.empty_like(a1), torch.empty_like(v1)
    ro._tc.forward(s, g, a2, stream=st); ro._tc_critic.forward(s, g, v2, stream=st)
    torch.cuda.synchronize()
    assert torch.equal(a1, a2) and torch.equal(v1, v2)


def test_gated_steps_go_downhill(asset_root):
    """tensor cores: one actor step on a minibatch raises its clipped surrogate; 50 critic steps on a fixed minibatch lower the critic loss"""
    import torch
    from deepmimic_b200.learner import PPOLearner, clipped_surrogate, gaussian_log_prob
    env, ro = _task_rollout(asset_root, "target", 2048, "torch")
    traj = ro.collect(4)
    ln = PPOLearner(ro, **dict(HP, actor_stepsize=1e-4, actor_weight_decay=0.0, critic_weight_decay=0.0), minibatch_size=2048, backend="tensor_core")
    w = ln.window(traj)
    a = w["exp_idx"][:2048]
    c = torch.arange(2048, device="cuda")

    def surrogate():
        with torch.no_grad(), _no_tf32():
            mu = ro.policy(*ln._inputs(w, a))
            ratio = (gaussian_log_prob(w["norm_a"][a], mu, ro.policy.logstd) - w["old_logp"][a]).exp()
            return clipped_surrogate(w["adv"][a], ratio, ln.ratio_clip).mean().item()

    def closs():
        with torch.no_grad(), _no_tf32():
            return ln.critic_loss(w, c)[1].item()
    st = torch.cuda.current_stream().cuda_stream
    ln._tc_critic.set_weights(stream=st); ln._tc_actor.set_weights(stream=st)
    tc = ln._tc_batch(w)
    stats = [torch.zeros((), device="cuda") for _ in range(3)]
    s0, l0 = surrogate(), closs()
    ln.minibatch_step(w, c, a, stats, tc)
    s1 = surrogate()
    for _ in range(49):
        ln.minibatch_step(w, c, a, stats, tc)
    l1 = closs()
    print("gated, tensor cores: surrogate %.6f -> %.6f after one step; critic loss %.4f -> %.4f after 50 steps" % (s0, s1, l0, l1))
    assert s1 > s0 and l1 < l0


def test_target_amp_training_loop_on_the_tensor_cores(asset_root):
    """512 target_amp environments: collect(32) with the discriminator and the critic, then the PPO update and the discriminator update, all
    on the tensor cores, three times: every output finite"""
    import torch
    from deepmimic_b200.learner import AMPDiscLearner, PPOLearner
    env, ro = _task_rollout(asset_root, "target", 512, "tensor_core", disc=True)
    ppo = PPOLearner(ro, **HP, minibatch_size=4096, backend="tensor_core")
    dl = AMPDiscLearner(ro, **DISC_HP, batch_size=2048, steps=8, backend="tensor_core")
    M = env.get_amp_obs_size()
    for it in range(3):
        traj = ro.collect(32)
        ro.amp_norm.update()
        s_ppo = ppo.update(traj)
        expert = torch.cat([env.record_amp_obs_expert().clone() for _ in range(4)])
        s_disc = dl.update(traj["amp_obs"].reshape(-1, M), expert)
        vals = [v.item() for v in list(s_ppo.values()) + list(s_disc.values())]
        print("iteration %d: mean reward %.4f; PPO %s; discriminator %s" % (it, traj["amp_rewards"].mean().item(), {k: round(v.item(), 4) for k, v in s_ppo.items()},
                                                                           {k: round(v.item(), 4) for k, v in s_disc.items()}))
        assert all(np.isfinite(vals)) and all(torch.isfinite(traj[k]).all() for k in ("amp_obs", "disc_logits", "amp_rewards", "returns", "actions"))
        assert all(torch.isfinite(p).all() for p in list(ro.policy.parameters()) + list(ro.critic.parameters()))
    assert env.counters()[1] == 0


def test_the_two_families_refuse_each_other():
    """the plain entry points refuse a gated workspace or handle and the gated ones a plain one, each with a message naming the other"""
    import ctypes as C
    import torch
    from deepmimic_b200.capi import DmLearnBatch, DmLearnGatedBatch, DmLearnGatedNet, DmLearnNet, lib
    L = lib()
    gl = C.c_void_p(L.dm_learn_create_gated(0, 0, 20, 3, 64, 64, 4, 32, 16, 128))
    pl = C.c_void_p(L.dm_learn_create(0, 0, 20, 64, 64, 4, 128))
    assert gl.value and pl.value
    try:
        assert L.dm_learn_step(gl, C.byref(DmLearnNet()), C.byref(DmLearnBatch()), None) != 0 and b"gated" in L.dm_last_error()
        assert L.dm_learn_set_weights(gl, C.byref(DmLearnNet()), None) != 0 and b"gated" in L.dm_last_error()
        assert L.dm_learn_gated_step(pl, C.byref(DmLearnGatedNet()), C.byref(DmLearnGatedBatch()), None) != 0 and b"plain" in L.dm_last_error()
        assert L.dm_learn_set_gated_weights(pl, C.byref(DmLearnGatedNet()), None) != 0 and b"plain" in L.dm_last_error()
        assert not L.dm_learn_create_gated(0, 0, 20, 65, 64, 64, 4, 32, 16, 128) and b"goal_dim" in L.dm_last_error()
        assert not L.dm_learn_create_gated(0, 1, 20, 3, 64, 64, 2, 32, 16, 128) and b"critic" in L.dm_last_error()
    finally:
        L.dm_learn_destroy(gl); L.dm_learn_destroy(pl)
    torch.cuda.synchronize()


def _gpu_ms(f, n=3):
    import torch
    for _ in range(2):
        f()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(n):
        f()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def test_gated_update_time():
    """device clock: one update() of a 32 x 4096 window of target_amp's sizes (226 state and 3 goal inputs, 28 actions, the reference's gated
    1024-512 networks), minibatch 4096, on both backends"""
    import torch
    from deepmimic_b200.learner import PPOLearner, gaussian_log_prob
    from deepmimic_b200.rollout import BatchedRollout, build_critic, build_gated_policy
    T, N, S, G, A = 32, 4096, 226, 3, 28
    torch.manual_seed(0)
    env = _GoalShapeEnv(N, S, G, A)
    ro = BatchedRollout(env, policy=build_gated_policy(S, G, A), critic=build_critic(S, G), discount=0.95, td_lambda=0.95)
    g = torch.Generator(device="cuda").manual_seed(0)
    traj = dict(states=torch.randn(T, N, S, device="cuda", generator=g), goals=torch.randn(T, N, G, device="cuda", generator=g),
                actions=0.05 * torch.randn(T, N, A, device="cuda", generator=g), returns=20.0 * torch.rand(T, N, device="cuda", generator=g),
                values=20.0 * torch.rand(T, N, device="cuda", generator=g), explore=torch.rand(T, N, device="cuda", generator=g) < 0.8)
    with torch.no_grad():
        traj["logps"] = gaussian_log_prob(traj["actions"], ro.policy(ro.s_norm.normalize(traj["states"]), ro.g_norm.normalize(traj["goals"])), ro.policy.logstd)
    times = {}
    for backend in ("torch", "tensor_core"):
        ln = PPOLearner(ro, **HP, minibatch_size=4096, backend=backend)
        with _no_tf32():
            times[backend] = _gpu_ms(lambda: ln.update(traj))
    print("gated update of a %d x %d window, minibatch 4096: %.1f ms fp32 torch, %.1f ms tensor cores" % (T, N, times["torch"], times["tensor_core"]))
    assert times["tensor_core"] < times["torch"]
