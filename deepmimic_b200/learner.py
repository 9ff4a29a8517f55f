"""The learners: one PPOAgent._update over a window collected by BatchedRollout(critic=...) (R/learning/ppo_agent.py: _update,
_update_actor, _update_critic, _build_losses; pg_agent.py; tf_util.py: calc_bound_loss; solvers/mpi_solver.py wrapping TF's MomentumOptimizer),
and the AMP discriminator's update (R/learning/amp_agent.py: _build_losses, _disc_grad_penalty_loss, _disc_weight_decay_loss,
_disc_logit_reg_loss, _update_disc / _step_disc).

The reference tree is not vendored here; its rules are restated below, one function per rule, and the CPU tests pin them there
(tests/test_learner_cpu.py, tests/test_disc_learner_cpu.py).  Where a restatement and the reference disagree, the reference is right.

  PPOLearner(rollout, ...).update(traj)   one epoch loop over the window: per minibatch one critic step, then one actor step
    backend "torch"        autograd over the rollout's torch modules (plain or gated networks, CPU or CUDA tensors): the reference the
                           tensor-core backend is tested against
    backend "tensor_core"  the minibatch steps on the library's own sm_90a kernels (kernels/dm_learn.cu and the backward GEMMs of
                           kernels/dm_mlp.cu): dm_learn_step for the plain networks, dm_learn_gated_step for the gated networks of the task
                           scenes (CUDA only)
  AMPDiscLearner(rollout, ...).update(agent_amp_obs, expert_amp_obs)   `steps` discriminator steps on minibatches drawn from the two pools
    backend "torch"        autograd with a double backward for the gradient penalty (CPU or CUDA tensors)
    backend "tensor_core"  dm_learn_disc_step: the penalty's weight gradients as first-order GEMMs (the ReLU masks are constant), every AMP scene

Documented deviations: minibatches are shuffled / drawn by a seeded torch.Generator on the data's device, not the reference's numpy stream; the
statistics leave out the weight-decay (and logit-regulariser) terms of the losses (the reference's logged losses include them); the normalisers
are not updated here (DeviceNormalizer.update stays the caller's call, as the reference's normaliser schedule is), nor are the AMP replay
buffers kept (deepmimic_b200/trainer.py: DeviceReplayBuffer, with the TarClipFrac, exploration and normaliser schedules).  The loop that
drives both learners, with checkpoints, is deepmimic_b200/trainer.py: Trainer.

Data parallelism (mpi_run.py --num_workers N, solvers/mpi_solver.py: MPISolver): both learners take process_group=; with a group of more than
one rank, the networks are broadcast from the group's first rank at construction (MPISolver.sync), and every minibatch step averages the
ranks' flat gradients (one torch.distributed.all_reduce per network and step) before the weight decay and the momentum step, so every rank
applies the same update and keeps the same weights.  The tensor-core backend splits its step around that sum (TensorCoreLearner.grad /
apply).  The weight-decay terms are added once after the average: they depend on the weights alone, which are equal on every rank, so the
result is MPISolver's average of the whole gradient.  Without a group, or with a group of one rank, the learners run exactly as without one."""
import math

ADV_EPS = 1e-5   # PPOAgent.ADV_EPS


def clipped_value_targets(returns, val_min, val_max):
    """The critic's targets: the TD(lambda) returns clipped to the value bounds [r_min, r_max] / (1 - discount) (PPOAgent._update clips new_vals
    to val_min / val_max after the advantages are taken from the unclipped returns)."""
    return returns.clamp(val_min, val_max)


def normalized_advantages(returns, values, exp_idx, norm_adv_clip):
    """PPOAgent._update: adv = new_vals - vals over the explored samples only (exp_idx), normalised with their mean and their (population,
    np.std) std plus ADV_EPS, then clipped to +-norm_adv_clip.  Returns (adv of the explored samples in exp_idx's order, mean, std)."""
    adv = (returns - values)[exp_idx]
    mean, std = adv.mean(), adv.std(unbiased=False)
    return ((adv - mean) / (std + ADV_EPS)).clamp(-norm_adv_clip, norm_adv_clip), mean, std


def critic_loss(norm_out, norm_targets):
    """PPOAgent._build_losses: 0.5 mean((norm(target) - norm(V))^2) in the value normaliser's space"""
    return 0.5 * (norm_targets - norm_out).square().mean()


def gaussian_log_prob(norm_a, mu, logstd):
    """log N(norm_a; mu, exp(logstd)) summed over the action (PGAgent's logp of the normalised action; sigma is the constant norm_a_std_tf)"""
    return (-0.5 * ((norm_a - mu) / logstd.exp()).square() - logstd - 0.5 * math.log(2.0 * math.pi)).sum(dim=-1)


def clipped_surrogate(adv, ratio, ratio_clip):
    """PPOAgent._build_losses: min(adv ratio, adv clip(ratio, 1 - eps, 1 + eps)) per row, with the gradient TF gives it: tf.minimum passes the
    gradient to its first argument on ties, tf.clip_by_value passes it inside the clip range, bounds included.  A row therefore contributes
    adv ratio dlogp when the unclipped term is the minimum or the ratio lies inside the range, and nothing otherwise."""
    l0 = adv * ratio
    l1 = adv * ratio.clamp(1.0 - ratio_clip, 1.0 + ratio_clip)
    return l0.where(l0 <= l1, l1)


def clip_fraction(ratio, ratio_clip):
    """PPOAgent.clip_frac_tf: the fraction of rows with |ratio - 1| > eps"""
    return ((ratio - 1.0).abs() > ratio_clip).float().mean()


def bound_loss(mu, bound_min, bound_max):
    """TFUtil.calc_bound_loss on the normalised action mean: 0.5 mean_rows sum_j (min(mu - lo, 0)^2 + max(mu - hi, 0)^2), lo / hi the normalised
    action bounds"""
    vmin, vmax = (mu - bound_min).clamp(max=0.0), (mu - bound_max).clamp(min=0.0)
    return 0.5 * (vmin.square().sum(dim=-1) + vmax.square().sum(dim=-1)).mean()


def weight_decay_loss(net):
    """PPOAgent._weight_decay_loss: sum ||W||^2 / 2 (tf.nn.l2_loss) over the network's weight matrices; variables named bias are skipped, and the
    actor's log-std is a constant, not a variable"""
    return sum(0.5 * p.square().sum() for n, p in net.named_parameters() if n.endswith("weight"))


def trained_parameters(net):
    """the optimiser's variables: every parameter but the actor's log-std (norm_a_std_tf is a constant in the reference)"""
    return [p for n, p in net.named_parameters() if n != "logstd"]


def minibatch_schedule(num_critic, num_actor, minibatch_size, epochs, generator, device="cpu"):
    """PPOAgent._update's loop: ceil(num_critic / B) minibatches per epoch, each of exactly B rows; minibatch b takes the positions b B .. b B + B - 1
    modulo each set's size from that set's shuffled order (critic: every sample, actor: the explored ones).  Both orders are reshuffled at every
    epoch, and the actor's also right after a minibatch whose positions wrapped or reached its last entry (shuffle_actor).  Yields
    (critic positions, actor positions), int64 tensors of B entries on `device`.  The shuffles draw from `generator` (a documented deviation
    from the reference's numpy stream); no host synchronisation."""
    import torch
    B = minibatch_size
    for _ in range(epochs):
        cperm = torch.randperm(num_critic, generator=generator, device=device)
        aperm = torch.randperm(num_actor, generator=generator, device=device)
        for b in range(-(-num_critic // B)):
            pos = torch.arange(b * B, (b + 1) * B, device=device)
            yield cperm[pos % num_critic], aperm[pos % num_actor]
            first, last = (b * B) % num_actor, ((b + 1) * B - 1) % num_actor
            if last < first or last == num_actor - 1:
                aperm = torch.randperm(num_actor, generator=generator, device=device)


def momentum_step(params, accs, grads, stepsize, momentum):
    """TF MomentumOptimizer (what MPISolver wraps): acc = momentum acc + g; w -= stepsize acc"""
    for p, a, g in zip(params, accs, grads):
        a.mul_(momentum).add_(g)
        p.sub_(stepsize * a)


class DataParallel:
    """A learner's ranks: the torch.distributed process group `group` of world > 1 ranks (NCCL on the GPUs; gloo also takes CPU and CUDA
    tensors).  Collectives are stream-ordered on NCCL and add no host synchronisation there."""

    def __init__(self, group):
        import torch.distributed as dist
        self.dist, self.group = dist, group
        self.world = dist.get_world_size(group)
        self.src = dist.get_global_rank(group, 0)

    @staticmethod
    def of(group):
        """a DataParallel for `group`, or None without a group or with a group of one rank"""
        if group is None:
            return None
        import torch.distributed as dist
        return DataParallel(group) if dist.get_world_size(group) > 1 else None

    def broadcast(self, tensors):
        """the group's first rank's values into `tensors` on every rank (MPISolver.sync)"""
        for x in tensors:
            self.dist.broadcast(x.data, self.src, group=self.group)

    def sum(self, x):
        """x summed over the ranks, in place; returns x"""
        self.dist.all_reduce(x, group=self.group)
        return x

    def mean_grads(self, grads):
        """the ranks' mean of each gradient in `grads`: one all-reduce of their flat concatenation"""
        import torch
        flat = self.sum(torch.cat([g.reshape(-1) for g in grads])) / self.world
        return [v.view_as(g) for v, g in zip(flat.split([g.numel() for g in grads]), grads)]

    def mean_stats(self, values):
        """the ranks' means of the 0-d tensors `values` (one all-reduce of their stack)"""
        import torch
        return list(self.sum(torch.stack([v.float().reshape(()) for v in values])) / self.world)

    def check_window(self, n, explored):
        """refuses, on every rank at once, a window size `n` (a host int) that differs between the ranks, or a window without an explored
        sample on any rank (`explored`: a 0-d bool device tensor): a rank that ran more minibatch steps than another, or none, would leave the
        others waiting for ever in a collective.  One all-reduce and one host synchronisation."""
        import torch
        x = torch.stack([torch.tensor(n, device=explored.device), torch.tensor(-n, device=explored.device), (~explored).long()])
        self.dist.all_reduce(x, op=self.dist.ReduceOp.MAX, group=self.group)
        hi, lo, empty = x.tolist()
        if hi != n or -lo != n:
            raise ValueError("data-parallel learner: the ranks' window sizes differ (%d to %d); every rank must run the same number of "
                             "minibatch steps" % (-lo, hi))
        if empty:
            raise ValueError("data-parallel learner: a rank's window has no explored sample (the actor trains on explored actions only)")


def _check_indices(device, *indices):
    """refuses a minibatch index tensor the tensor-core step cannot read.  indices: (name, index tensor, rows of its batch) triples; each tensor
    must be contiguous int64 with the batch's rows entries on `device`"""
    import torch
    for name, idx, rows in indices:
        if idx.dtype != torch.int64 or not idx.is_contiguous() or idx.device != device or idx.numel() != rows:
            raise ValueError("%s must be a contiguous int64 tensor of %d entries on %s" % (name, rows, device))


def _tc_step(tc, batch, dp, grad, stream):
    """one tensor-core minibatch step of the workspace tc: fused without a group (dp None), or the flat gradient into `grad`, its sum over the
    ranks and the step on the ranks' mean"""
    if dp is None:
        tc.step(batch, stream=stream)
        return
    tc.grad(batch, grad, stream=stream)
    dp.sum(grad)
    tc.apply(batch, grad, 1.0 / dp.world, stream=stream)


def _weight_decay_grads(net, params, grads, weight_decay):
    """grads plus the gradient of weight_decay * weight_decay_loss(net): weight_decay w on the weights, nothing on the biases"""
    names = {p: n for n, p in net.named_parameters()}
    return [g + weight_decay * p.detach() if names[p].endswith("weight") else g for p, g in zip(params, grads)]


def _check(name, v, lo, hi, lo_open=False, hi_open=False):
    bad = v is None or not (isinstance(v, (int, float)) and math.isfinite(float(v)))
    if not bad:
        v = float(v)
        bad = v < lo or v > hi or (lo_open and v == lo) or (hi_open and v == hi)
    if bad:
        raise ValueError("%s must be in %s%s, %s%s (got %r)" % (name, "(" if lo_open else "[", lo, hi, ")" if hi_open else "]", v))
    return float(v)


class PPOLearner:
    """One PPOAgent._update per update(traj) over a window of BatchedRollout(critic=...).collect(): the rollout's policy, critic and normalisers
    (s_norm, g_norm, a_norm, val_norm).  Every hyperparameter is required (the reference reads them from an agent file; the asset archive has none).
    The momentum accumulators are the learner's; after update() the torch modules hold the new weights and the rollout's tensor-core actor and
    critic, where they exist, hold those weights and the normalisers' statistics that the update trained with.  A normaliser updated after
    update() reaches those handles with the next update() or with rollout.refresh_tensor_core_policy().

    process_group (data parallelism, see the module docstring): minibatch_size is the job's total (MiniBatchSize); each rank's minibatches have
    ceil(minibatch_size / world) rows (the maintainer's reading of the reference's _local_mini_batch_size, not checked against its source).
    The advantages are normalised over the rank's own explored samples (the reading of PPOAgent._update, which takes their mean and std over
    the worker's samples; not checked against its source either).  Every rank's window must have the same size, so that all ranks run the
    same number of minibatch steps, and at least one explored sample: update() refuses, on every rank, a window that breaks either (one more
    host synchronisation).  update()'s statistics are the ranks' means (exp_samples: the ranks' total, an integer)."""

    def __init__(self, rollout, *, actor_stepsize=None, actor_momentum=None, actor_weight_decay=None, critic_stepsize=None, critic_momentum=None,
                 critic_weight_decay=None, ratio_clip=None, norm_adv_clip=None, minibatch_size=None, epochs=None, backend="torch", seed=0,
                 process_group=None):
        import torch
        self.torch, self.ro = torch, rollout
        if rollout.critic is None:
            raise ValueError("the PPO learner needs a rollout with a critic (BatchedRollout(critic=..., discount=..., td_lambda=...))")
        inf = float("inf")
        self.actor_stepsize = _check("actor_stepsize", actor_stepsize, 0.0, inf, lo_open=True, hi_open=True)
        self.actor_momentum = _check("actor_momentum", actor_momentum, 0.0, 1.0, hi_open=True)
        self.actor_weight_decay = _check("actor_weight_decay", actor_weight_decay, 0.0, inf, hi_open=True)
        self.critic_stepsize = _check("critic_stepsize", critic_stepsize, 0.0, inf, lo_open=True, hi_open=True)
        self.critic_momentum = _check("critic_momentum", critic_momentum, 0.0, 1.0, hi_open=True)
        self.critic_weight_decay = _check("critic_weight_decay", critic_weight_decay, 0.0, inf, hi_open=True)
        self.ratio_clip = _check("ratio_clip", ratio_clip, 0.0, 1.0, lo_open=True, hi_open=True)
        self.norm_adv_clip = _check("norm_adv_clip", norm_adv_clip, 0.0, inf, lo_open=True, hi_open=True)
        for name, v in (("minibatch_size", minibatch_size), ("epochs", epochs)):
            if not isinstance(v, int) or isinstance(v, bool) or v < 1:
                raise ValueError("%s must be a positive int (got %r)" % (name, v))
        self.dp = DataParallel.of(process_group)
        self.world = self.dp.world if self.dp else 1
        self.minibatch_size, self.epochs = -(-minibatch_size // self.world), epochs
        if backend not in ("torch", "tensor_core"):
            raise ValueError("backend must be 'torch' or 'tensor_core'")
        self.backend = backend
        env, dev = rollout.env, rollout.env.device
        self.device = dev
        self.policy, self.critic = rollout.policy, rollout.critic
        self.val_min = env.get_reward_min() / (1.0 - rollout.discount)
        self.val_max = env.get_reward_max() / (1.0 - rollout.discount)
        f = lambda a: torch.as_tensor(a, dtype=torch.float32, device=dev)
        self.bound_min = rollout.a_norm.normalize(f(env.build_action_bound_min()))
        self.bound_max = rollout.a_norm.normalize(f(env.build_action_bound_max()))
        self.actor_params, self.critic_params = trained_parameters(self.policy), trained_parameters(self.critic)
        self.acc = {p: torch.zeros_like(p, memory_format=torch.contiguous_format) for p in self.actor_params + self.critic_params}
        self.gen = torch.Generator(device=dev)
        self.gen.manual_seed(seed)
        if self.dp:
            with torch.no_grad():
                self.dp.broadcast(list(self.policy.parameters()) + list(self.critic.parameters()))
        if backend == "tensor_core":
            if dev.type != "cuda":
                raise ValueError("the tensor_core learner needs a CUDA device; on the CPU, plain and gated networks train with backend='torch'")
            from .capi import TensorCoreGatedLearner, TensorCoreLearner
            di = dev.index or 0
            cls = TensorCoreGatedLearner if rollout.goal_size > 0 else TensorCoreLearner
            self._tc_actor = cls(self.policy, self.acc, "actor", self.minibatch_size, device=di)
            self._tc_critic = cls(self.critic, self.acc, "critic", self.minibatch_size, device=di)
            # the flat gradients the ranks sum
            self._grad_actor = torch.empty(self._tc_actor.grad_size(), device=dev) if self.dp else None
            self._grad_critic = torch.empty(self._tc_critic.grad_size(), device=dev) if self.dp else None
        if self.dp:   # the rollout's tensor-core actor and critic collect with the broadcast weights
            rollout.retile_tensor_core("actor", "critic")

    # ---- the window: everything a minibatch step reads, computed once per update
    def window(self, traj):
        """flattened [T N] views of the window and the per-sample tensors of the rules above; the one host synchronisation of update() sizes the
        explored set"""
        t, ro = self.torch, self.ro
        for key in ("states", "actions", "logps", "returns", "values", "explore") + (("goals",) if ro.goal_size else ()):
            if key not in traj:
                raise ValueError("traj has no %r: collect() with a critic returns it" % key)
        R = traj["returns"].numel()
        w = dict(R=R, states=traj["states"].reshape(R, -1), norm_a=ro.a_norm.normalize(traj["actions"].reshape(R, -1)),
                 old_logp=traj["logps"].reshape(R))
        if ro.goal_size:
            w["goals"] = traj["goals"].reshape(R, -1)
        ret, val = traj["returns"].reshape(R), traj["values"].reshape(R)
        exp_idx = traj["explore"].reshape(R).nonzero()[:, 0]
        if exp_idx.numel() == 0:
            raise ValueError("the window has no explored sample: the actor trains on explored actions only (exp_rate > 0)")
        adv, w["adv_mean"], w["adv_std"] = normalized_advantages(ret, val, exp_idx, self.norm_adv_clip)
        w["adv"] = t.zeros(R, device=ret.device)
        w["adv"][exp_idx] = adv
        w["exp_idx"] = exp_idx
        w["norm_tar"] = ro.val_norm.normalize(clipped_value_targets(ret, self.val_min, self.val_max))
        return w

    def _inputs(self, w, idx):
        ro = self.ro
        ns = ro.s_norm.normalize(w["states"][idx])
        return (ns,) if not ro.goal_size else (ns, ro.g_norm.normalize(w["goals"][idx]))

    def critic_loss(self, w, idx):
        """(loss with weight decay, loss) of the critic on the window samples idx (torch autograd)"""
        loss = critic_loss(self.critic(*self._inputs(w, idx))[:, 0], w["norm_tar"][idx])
        return loss + self.critic_weight_decay * weight_decay_loss(self.critic), loss

    def actor_loss(self, w, idx):
        """(loss with weight decay, surrogate + bound loss, ratio) of the actor on the explored window samples idx (torch autograd)"""
        mu = self.policy(*self._inputs(w, idx))
        ratio = (gaussian_log_prob(w["norm_a"][idx], mu, self.policy.logstd.detach()) - w["old_logp"][idx]).exp()
        loss = -clipped_surrogate(w["adv"][idx], ratio, self.ratio_clip).mean() + bound_loss(mu, self.bound_min, self.bound_max)
        return loss + self.actor_weight_decay * weight_decay_loss(self.policy), loss, ratio

    # ---- one minibatch: a critic step, then an actor step
    def _tc_batch(self, w, ratio=None):
        """the dm_learn_batch (gated networks: dm_learn_gated_batch) of the actor and of the critic over the window w (and the tensors they
        point into); ratio: an optional float32 CUDA tensor [minibatch_size] that receives the actor's per-row probability ratios of the last
        step"""
        from .capi import DmLearnBatch, DmLearnGatedBatch
        t, ro = self.torch, self.ro
        keep = dict(istd=(1.0 / ro.s_norm.std).contiguous(), mean=ro.s_norm.mean.contiguous(), old=w["old_logp"].contiguous(),
                    logstd=self.policy.logstd.detach().contiguous(), states=w["states"].contiguous(), norm_a=w["norm_a"].contiguous(),
                    lo=self.bound_min.contiguous(), hi=self.bound_max.contiguous(), adv=w["adv"].contiguous(), tar=w["norm_tar"].contiguous(),
                    stats_a=t.zeros(2, device=self.device), stats_c=t.zeros(1, device=self.device))
        p = lambda x: x.data_ptr()
        clip = 0.0 if math.isinf(ro.s_norm.clip) else float(ro.s_norm.clip)
        common = dict(states=p(keep["states"]), rows=self.minibatch_size, in_mean=p(keep["mean"]), in_istd=p(keep["istd"]), in_clip=clip)
        actor = DmLearnBatch(**common, norm_actions=p(keep["norm_a"]), old_logp=p(keep["old"]), adv=p(keep["adv"]), logstd=p(keep["logstd"]),
                             bound_min=p(keep["lo"]), bound_max=p(keep["hi"]), ratio_clip=self.ratio_clip, ratio=None if ratio is None else p(ratio),
                             stepsize=self.actor_stepsize,
                             momentum=self.actor_momentum, weight_decay=self.actor_weight_decay, stats=p(keep["stats_a"]))
        critic = DmLearnBatch(**common, norm_targets=p(keep["tar"]), stepsize=self.critic_stepsize, momentum=self.critic_momentum,
                              weight_decay=self.critic_weight_decay, stats=p(keep["stats_c"]))
        if ro.goal_size:
            keep.update(goals=w["goals"].contiguous(), g_mean=ro.g_norm.mean.contiguous(), g_istd=(1.0 / ro.g_norm.std).contiguous())
            g_clip = 0.0 if math.isinf(ro.g_norm.clip) else float(ro.g_norm.clip)
            goal = dict(goals=p(keep["goals"]), g_mean=p(keep["g_mean"]), g_istd=p(keep["g_istd"]), g_clip=g_clip)
            actor, critic = DmLearnGatedBatch(batch=actor, **goal), DmLearnGatedBatch(batch=critic, **goal)
        return keep, actor, critic

    def minibatch_step(self, w, critic_idx, actor_idx, stats, tc=None):
        """one critic step on the window samples critic_idx, then one actor step on the samples actor_idx; stats (3 zero-d tensors: actor loss,
        critic loss, clip fraction) accumulate"""
        if self.backend == "tensor_core":
            keep, actor, critic = tc
            _check_indices(self.device, ("critic_idx", critic_idx, critic.rows), ("actor_idx", actor_idx, actor.rows))
            st = self.torch.cuda.current_stream(self.device).cuda_stream
            critic.idx = critic_idx.data_ptr()
            _tc_step(self._tc_critic, critic, self.dp, self._grad_critic, st)
            actor.idx = actor_idx.data_ptr()
            _tc_step(self._tc_actor, actor, self.dp, self._grad_actor, st)
            return
        t = self.torch
        total, loss = self.critic_loss(w, critic_idx)
        grads = self._grads(total, loss, self.critic, self.critic_params, self.critic_weight_decay)
        with t.no_grad():
            momentum_step(self.critic_params, [self.acc[p] for p in self.critic_params], grads, self.critic_stepsize, self.critic_momentum)
            stats[1] += loss.detach()
        total, loss, ratio = self.actor_loss(w, actor_idx)
        grads = self._grads(total, loss, self.policy, self.actor_params, self.actor_weight_decay)
        with t.no_grad():
            momentum_step(self.actor_params, [self.acc[p] for p in self.actor_params], grads, self.actor_stepsize, self.actor_momentum)
            stats[0] += loss.detach().abs()      # PPOAgent._update logs the mean of |actor loss| over the minibatches
            stats[2] += clip_fraction(ratio.detach(), self.ratio_clip)

    def _grads(self, total, loss, net, params, weight_decay):
        """the step's gradient: of `total` (the loss with its weight decay), or (data parallel) the ranks' mean gradient of `loss` plus the
        weight decay's"""
        t = self.torch
        if not self.dp:
            return t.autograd.grad(total, params)
        return _weight_decay_grads(net, params, self.dp.mean_grads(t.autograd.grad(loss, params)), weight_decay)

    def update(self, traj):
        """one PPOAgent._update over the window traj (collect() with a critic); returns 0-d device tensors: actor_loss, critic_loss, clip_frac
        (means over the minibatch steps), adv_mean, adv_std, exp_samples"""
        t = self.torch
        same = lambda now, then: len(now) == len(then) and all(x is y for x, y in zip(now, then))
        if not same(trained_parameters(self.policy), self.actor_params) or not same(trained_parameters(self.critic), self.critic_params):
            raise ValueError("the policy's or the critic's parameters were replaced after the learner was built: build a new PPOLearner")
        if self.dp:
            if "explore" not in traj:
                raise ValueError("traj has no 'explore': collect() with a critic returns it")
            self.dp.check_window(traj["returns"].numel(), traj["explore"].any())
        w = self.window(traj)
        n_exp = w["exp_idx"].numel()
        stats = [t.zeros((), device=self.device) for _ in range(3)]
        tc = None
        if self.backend == "tensor_core":
            st = t.cuda.current_stream(self.device).cuda_stream
            self._tc_critic.set_weights(stream=st)
            self._tc_actor.set_weights(stream=st)
            tc = self._tc_batch(w)
        steps = 0
        for c, a in minibatch_schedule(w["R"], n_exp, self.minibatch_size, self.epochs, self.gen, self.device):
            self.minibatch_step(w, c, w["exp_idx"][a], stats, tc)
            steps += 1
        if tc is not None:
            keep = tc[0]
            stats = [keep["stats_a"][0], keep["stats_c"][0], keep["stats_a"][1]]
        self.ro.retile_tensor_core("actor", "critic")
        out = dict(actor_loss=stats[0] / steps, critic_loss=stats[1] / steps, clip_frac=stats[2] / steps, adv_mean=w["adv_mean"],
                   adv_std=w["adv_std"], exp_samples=t.tensor(n_exp, device=self.device))
        if self.dp:
            keys = ("actor_loss", "critic_loss", "clip_frac", "adv_mean", "adv_std")
            x = self.dp.sum(t.stack([out[k].double() for k in keys] + [out["exp_samples"].double()]))
            out = dict(zip(keys, (x[:-1] / self.world).float()), exp_samples=x[-1].round().long())   # the explored samples of all ranks
        return out


# ---- the AMP discriminator (R/learning/amp_agent.py)
def disc_loss(d_expert, d_agent):
    """AMPAgent._build_losses, the least-squares loss (Peng et al. 2021, eq. 8): 0.5 (0.5 mean (d_e - 1)^2 + 0.5 mean (d_a + 1)^2) over the
    expert logits d_e and the agent logits d_a"""
    return 0.5 * (0.5 * (d_expert - 1.0).square().mean() + 0.5 * (d_agent + 1.0).square().mean())


def disc_grad_penalty(grad):
    """AMPAgent._disc_grad_penalty_loss: 0.5 mean_rows ||dd_e / dx_e||^2, grad = dd_e / dx_e [rows, inputs] taken w.r.t. the normalised, clipped
    expert input (so no clip mask applies).  The factor 0.5 is eq. 8's w_gp / 2 with w_gp the penalty's weight; that the reference carries it
    in this term rather than in the weight could not be checked against its source here."""
    return 0.5 * grad.square().sum(dim=-1).mean()


def disc_input_grad(disc, norm_x, create_graph=True):
    """(logits d [rows], dd / dx [rows, inputs]) of the discriminator at the normalised inputs norm_x; with create_graph the gradient is itself
    differentiable (the penalty's double backward)"""
    import torch
    x = norm_x.detach().requires_grad_(True)
    d = disc(x)[:, 0]
    g, = torch.autograd.grad(d.sum(), x, create_graph=create_graph)
    return d, g


def disc_weight_decay_loss(disc):
    """AMPAgent._disc_weight_decay_loss: sum ||W||^2 / 2 over the discriminator's weight matrices, biases skipped.  The logit layer's weights are
    included; whether the reference's variable scope covers the logit layer could not be checked against its source here."""
    return weight_decay_loss(disc)


def disc_logit_reg_loss(disc):
    """AMPAgent._disc_logit_reg_loss: ||w_logit||^2 / 2 on the logit layer's weights only"""
    return 0.5 * disc.logit.weight.square().sum()


def disc_accuracies(d_expert, d_agent):
    """AMPAgent's logged accuracies: (mean(d_e > 0), mean(d_a < 0))"""
    return (d_expert > 0).float().mean(), (d_agent < 0).float().mean()


class AMPDiscLearner:
    """The AMP discriminator's update (AMPAgent._update_disc): `steps` minibatch steps, each on batch_size agent and batch_size expert rows
    drawn uniformly with replacement from the two pools by a seeded device torch.Generator (the draws are a documented deviation from the
    reference's numpy stream, the sampling rule is not), with TF's momentum rule (momentum_step) on
      disc_loss + grad_penalty grad_penalty + weight_decay sum ||W||^2 / 2 + logit_reg_weight ||w_logit||^2 / 2.
    The inputs are normalised by the rollout's amp_norm as collect() normalises them.  Every hyperparameter is required (the reference reads
    DiscStepSize, DiscMomentum, ... from the agent file; the asset archive has none).  The momentum accumulators are the learner's; keeping a
    replay buffer of agent observations and refreshing amp_norm stay the caller's.  After update() the torch discriminator holds the new
    weights and the rollout's tensor-core discriminator, where it exists, those weights and amp_norm's current statistics.

    process_group (data parallelism, see the module docstring): batch_size is the job's total (DiscBatchSize); each rank draws
    ceil(batch_size / world) agent and as many expert rows per step from its own pools (the maintainer's reading of the reference's
    _local_mini_batch_size, not checked against its source).  Every rank must run the same `steps`.  update()'s statistics are the ranks'
    means."""

    def __init__(self, rollout, *, stepsize=None, momentum=None, weight_decay=None, logit_reg_weight=None, grad_penalty=None, batch_size=None,
                 steps=None, backend="torch", seed=0, process_group=None):
        import torch
        self.torch, self.ro = torch, rollout
        if getattr(rollout, "disc", None) is None:
            raise ValueError("the discriminator learner needs a rollout with a discriminator (BatchedRollout(disc=...) in an AMP scene)")
        inf = float("inf")
        self.stepsize = _check("stepsize", stepsize, 0.0, inf, lo_open=True, hi_open=True)
        self.momentum = _check("momentum", momentum, 0.0, 1.0, hi_open=True)
        self.weight_decay = _check("weight_decay", weight_decay, 0.0, inf, hi_open=True)
        self.logit_reg_weight = _check("logit_reg_weight", logit_reg_weight, 0.0, inf, hi_open=True)
        self.grad_penalty = _check("grad_penalty", grad_penalty, 0.0, inf, hi_open=True)
        for name, v in (("batch_size", batch_size), ("steps", steps)):
            if not isinstance(v, int) or isinstance(v, bool) or v < 1:
                raise ValueError("%s must be a positive int (got %r)" % (name, v))
        self.dp = DataParallel.of(process_group)
        self.world = self.dp.world if self.dp else 1
        self.batch_size, self.steps = -(-batch_size // self.world), steps
        if backend not in ("torch", "tensor_core"):
            raise ValueError("backend must be 'torch' or 'tensor_core'")
        self.backend = backend
        self.disc, self.device = rollout.disc, rollout.env.device
        self.params = list(self.disc.parameters())
        self.acc = {p: torch.zeros_like(p, memory_format=torch.contiguous_format) for p in self.params}
        self.gen = torch.Generator(device=self.device)
        self.gen.manual_seed(seed)
        if self.dp:
            with torch.no_grad():
                self.dp.broadcast(self.params)
        if backend == "tensor_core":
            if self.device.type != "cuda":
                raise ValueError("the tensor_core learner needs a CUDA device")
            from .capi import TensorCoreLearner
            self._tc = TensorCoreLearner(self.disc, self.acc, "disc", 2 * self.batch_size, device=self.device.index or 0)
            self._grad = torch.empty(self._tc.grad_size(), device=self.device) if self.dp else None   # the flat gradient the ranks sum
        if self.dp:   # the rollout's tensor-core discriminator scores with the broadcast weights
            rollout.retile_tensor_core("disc")

    def loss(self, norm_agent, norm_expert):
        """(total loss with the regularisers, disc_loss, grad_penalty, d_e, d_a) on normalised agent and expert rows (torch autograd)"""
        d_a = self.disc(norm_agent)[:, 0]
        d_e, g = disc_input_grad(self.disc, norm_expert)
        loss, gp = disc_loss(d_e, d_a), disc_grad_penalty(g)
        total = (loss + self.grad_penalty * gp + self.weight_decay * disc_weight_decay_loss(self.disc)
                 + self.logit_reg_weight * disc_logit_reg_loss(self.disc))
        return total, loss, gp, d_e, d_a

    def _tc_batch(self, agent, expert):
        """the dm_learn_disc_batch over the two pools (and the tensors it points into); the index pointers are set per step"""
        from .capi import DmLearnDiscBatch
        t, norm = self.torch, self.ro.amp_norm
        keep = dict(agent=agent, expert=expert, mean=norm.mean.contiguous(), istd=(1.0 / norm.std).contiguous(), stats=t.zeros(6, device=self.device))
        p = lambda x: x.data_ptr()
        clip = 0.0 if math.isinf(norm.clip) else float(norm.clip)
        batch = DmLearnDiscBatch(agent=p(agent), expert=p(expert), rows=self.batch_size, in_mean=p(keep["mean"]), in_istd=p(keep["istd"]), in_clip=clip,
                                 stepsize=self.stepsize, momentum=self.momentum, weight_decay=self.weight_decay,
                                 logit_reg_weight=self.logit_reg_weight, grad_penalty_weight=self.grad_penalty, stats=p(keep["stats"]))
        return keep, batch

    def minibatch_step(self, agent, expert, agent_idx, expert_idx, stats, tc=None):
        """one step on the pool rows agent_idx, expert_idx; stats (6 zero-d tensors: disc_loss, grad_penalty, acc_expert, acc_agent, logit_expert,
        logit_agent) accumulate (tensor_core: into the batch's statistics)"""
        t = self.torch
        if self.backend == "tensor_core":
            keep, batch = tc
            _check_indices(self.device, ("agent_idx", agent_idx, batch.rows), ("expert_idx", expert_idx, batch.rows))
            batch.agent_idx, batch.expert_idx = agent_idx.data_ptr(), expert_idx.data_ptr()
            _tc_step(self._tc, batch, self.dp, self._grad, t.cuda.current_stream(self.device).cuda_stream)
            return
        norm = self.ro.amp_norm
        total, loss, gp, d_e, d_a = self.loss(norm.normalize(agent[agent_idx]), norm.normalize(expert[expert_idx]))
        if not self.dp:
            grads = t.autograd.grad(total, self.params)
        else:
            # the ranks' mean gradient of the loss and the penalty, then the weight decay and the logit regulariser of the (common) weights
            grads = _weight_decay_grads(self.disc, self.params, self.dp.mean_grads(t.autograd.grad(loss + self.grad_penalty * gp, self.params)),
                                        self.weight_decay)
            grads = [g + self.logit_reg_weight * p.detach() if p is self.disc.logit.weight else g for p, g in zip(self.params, grads)]
        with t.no_grad():
            momentum_step(self.params, [self.acc[p] for p in self.params], grads, self.stepsize, self.momentum)
            acc_e, acc_a = disc_accuracies(d_e, d_a)
            for s, v in zip(stats, (loss, gp, acc_e, acc_a, d_e.mean(), d_a.mean())):
                s += v.detach()

    def update(self, agent_amp_obs, expert_amp_obs):
        """`steps` discriminator steps on minibatches drawn from the pools agent_amp_obs [Ra, M] and expert_amp_obs [Re, M] (device tensors, e.g.
        traj["amp_obs"].reshape(-1, M) and clones of env.record_amp_obs_expert()).  No host synchronisation.  Returns 0-d device tensors, means
        over the steps: disc_loss (without the regularisers), grad_penalty (unweighted), acc_expert, acc_agent, logit_expert, logit_agent."""
        t = self.torch
        now = list(self.disc.parameters())
        if len(now) != len(self.params) or any(a is not b for a, b in zip(now, self.params)):
            raise ValueError("the discriminator's parameters were replaced after the learner was built: build a new AMPDiscLearner")
        M = self.ro.amp_norm.mean.numel()
        for name, x in (("agent_amp_obs", agent_amp_obs), ("expert_amp_obs", expert_amp_obs)):
            if x.dim() != 2 or x.shape[1] != M or x.shape[0] < 1 or x.device != self.device or x.dtype != t.float32:
                raise ValueError("%s must be a float32 [rows, %d] tensor on %s (got %s %s on %s)" % (name, M, self.device, x.dtype, tuple(x.shape), x.device))
        agent, expert = agent_amp_obs.contiguous(), expert_amp_obs.contiguous()
        stats = [t.zeros((), device=self.device) for _ in range(6)]
        tc = None
        if self.backend == "tensor_core":
            st = t.cuda.current_stream(self.device).cuda_stream
            self._tc.set_weights(stream=st)
            tc = self._tc_batch(agent, expert)
        B = self.batch_size
        for _ in range(self.steps):
            a = t.randint(0, agent.shape[0], (B,), generator=self.gen, device=self.device)
            e = t.randint(0, expert.shape[0], (B,), generator=self.gen, device=self.device)
            self.minibatch_step(agent, expert, a, e, stats, tc)
        if tc is not None:
            stats = list(tc[0]["stats"])
        self.ro.retile_tensor_core("disc")
        keys = ("disc_loss", "grad_penalty", "acc_expert", "acc_agent", "logit_expert", "logit_agent")
        stats = [s / self.steps for s in stats]
        return dict(zip(keys, self.dp.mean_stats(stats) if self.dp else stats))
