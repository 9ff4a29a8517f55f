"""Batched policy rollout over the batched environment (SURVEY.md 8(f) rank 1): what the reference does per env and per MPI worker
in RLWorld.update_agents -> RLAgent._update_new_action (R/learning/rl_world.py:94-132, R/learning/rl_agent.py:319-343), done for all
N environments of a rank at once with observations, actions and rewards staying on the device.

  DeviceNormalizer   R/learning/normalizer.py (mean / std / clip, group-wise running statistics), torch tensors
  GaussianMLPPolicy  actor of PPOAgent: fc_2layers_1024units -> Gaussian mean (+ state-independent log-std bias = log(noise))
                     (R/learning/ppo_agent.py:52-90, pg_agent.py:140-160, nets/fc_2layers_1024units.py, tf_util.py:27-39)
  Discriminator      the AMP agent's discriminator (R/learning/amp_agent.py): fc_2layers_1024units over the normalised AMP observation, one-unit
                     logit; its style reward max(0, 1 - 0.25 (1 - d)^2) is the AMP paper's least-squares reward (Peng et al. 2021, eq. 7)
  Critic             the PPO critic (R/learning/ppo_agent.py: _build_net_critic): the actor's trunk over the actor's normalised inputs, a
                     one-unit output un-normalised by the value normaliser (val_norm_from_rewards; terminal_values gives val_fail / val_succ)
  BatchedRollout     record_state -> normalise -> actor -> un-normalise -> set_action -> 20 x update -> reward / flags -> masked reset,
                     collecting [T, N, .] trajectory tensors for a learner; with a discriminator also the agent's AMP observation of every
                     transition and the style reward (blended with the task reward in the AMP task scenes) that an AMP learner trains on;
                     with a critic also the values of every state and of every step's pre-reset end state, and the TD(lambda) returns and
                     advantages of the window (R/learning/rl_util.py: compute_return), scanned on the device (kernels/dm_returns.cu)

With backend "torch" the MLPs run as plain torch matmuls (cuBLAS); with backend "tensor_core" the actor's inference (plain or gated), the
discriminator's reward and the critic's values run on the library's own wgmma kernels (kernels/dm_mlp.cu).  The reference's TF1 checkpoints
are read by deepmimic_b200/tf_checkpoint.py (TensorBundle reader, no TensorFlow) and loaded with load_actor_weights; without a
checkpoint the weights are random-initialised the way the reference initialises them."""
import math

import numpy as np


class DeviceNormalizer:
    NORM_GROUP_SINGLE = 0
    NORM_GROUP_NONE = -1

    def __init__(self, size, group_ids=None, eps=0.02, clip=float("inf"), device="cpu"):
        import torch
        self.torch = torch
        self.eps, self.clip = eps, clip
        self.mean = torch.zeros(size, device=device)
        self.mean_sq = torch.zeros(size, device=device)
        self.std = torch.ones(size, device=device)
        self.count = 0
        g = np.zeros(size, dtype=np.int64) if group_ids is None else np.asarray(group_ids, dtype=np.int64)
        self.group_ids = g
        self.new_count = 0
        self.new_sum = torch.zeros(size, device=device)
        self.new_sum_sq = torch.zeros(size, device=device)

    def set_mean_std(self, mean, std):
        t = self.torch
        self.mean = t.as_tensor(np.asarray(mean), dtype=t.float32, device=self.mean.device).clone()
        self.std = t.as_tensor(np.asarray(std), dtype=t.float32, device=self.mean.device).clone()
        self.mean_sq = self.std * self.std + self.mean * self.mean

    def normalize(self, x):
        y = (x - self.mean) / self.std
        return y if math.isinf(self.clip) else y.clamp(-self.clip, self.clip)

    def unnormalize(self, y):
        return y * self.std + self.mean

    def record(self, x):
        x = x.reshape(-1, self.mean.numel())
        self.new_count += x.shape[0]
        self.new_sum += x.sum(dim=0)
        self.new_sum_sq += (x * x).sum(dim=0)

    def _process_group_data(self, new, old):
        out = new.clone()
        for gid in np.unique(self.group_ids):
            idx = self.torch.as_tensor(np.nonzero(self.group_ids == gid)[0], device=new.device)
            if gid == self.NORM_GROUP_NONE:
                out[idx] = old[idx]
            elif gid != self.NORM_GROUP_SINGLE:
                out[idx] = new[idx].mean()
        return out

    def update(self, all_reduce=None):
        """Fold the recorded samples into the running statistics; `all_reduce(tensor)` sums over ranks (torch.distributed) if given."""
        t = self.torch
        cnt = t.tensor([float(self.new_count)], device=self.mean.device)
        s, sq = self.new_sum.clone(), self.new_sum_sq.clone()
        if all_reduce is not None:
            for x in (cnt, s, sq):
                all_reduce(x)
        n = int(cnt.item())
        if n > 0:
            total = self.count + n
            new_mean = self._process_group_data(s / n, self.mean)
            new_mean_sq = self._process_group_data(sq / n, self.mean_sq)
            w_old, w_new = self.count / total, n / total
            self.mean = w_old * self.mean + w_new * new_mean
            self.mean_sq = w_old * self.mean_sq + w_new * new_mean_sq
            self.count = total
            self.std = t.sqrt((self.mean_sq - self.mean * self.mean).clamp_min(0)).clamp_min(self.eps)
        self.new_count = 0
        self.new_sum.zero_(); self.new_sum_sq.zero_()


def build_policy(state_size, action_size, init_output_scale=0.01, noise=0.05, hidden=(1024, 512)):
    import torch

    class GaussianMLPPolicy(torch.nn.Module):
        def __init__(self):
            super().__init__()
            dims = [state_size] + list(hidden)
            self.hidden = torch.nn.ModuleList([torch.nn.Linear(a, b) for a, b in zip(dims[:-1], dims[1:])])
            for l in self.hidden:
                torch.nn.init.xavier_uniform_(l.weight); torch.nn.init.zeros_(l.bias)
            self.mean = torch.nn.Linear(dims[-1], action_size)
            torch.nn.init.uniform_(self.mean.weight, -init_output_scale, init_output_scale); torch.nn.init.zeros_(self.mean.bias)
            self.logstd = torch.nn.Parameter(torch.full((action_size,), math.log(noise)))

        def forward(self, norm_s):
            h = norm_s
            for l in self.hidden:
                h = torch.relu(l(h))      # fc_net leaves the last layer linear, build_net applies the activation afterwards
            return self.mean(h)

        def sample(self, norm_s, explore_mask=None, generator=None):
            """Normalised action and its log-probability; rows with explore_mask False take the mode."""
            mu = self.forward(norm_s)
            std = self.logstd.exp()
            eps = torch.randn(mu.shape, device=mu.device, generator=generator)
            if explore_mask is not None:
                eps = eps * explore_mask[:, None].to(eps.dtype)
            a = mu + std * eps
            logp = (-0.5 * eps * eps - self.logstd - 0.5 * math.log(2 * math.pi)).sum(dim=-1)
            return a, logp

    return GaussianMLPPolicy()


def build_gated_policy(state_size, goal_size, action_size, init_output_scale=0.01, noise=0.05, hidden=(1024, 512), gate_common=128, gate_hidden=64):
    """The goal-conditioned actor of the reference's AMP task agents, `fc_2layers_gated_1024units`
    (R/learning/nets/fc_2layers_gated_1024units.py:6-58): the trunk sees [norm_s, norm_g]; every hidden layer's pre-activation is scaled by
    2*sigmoid(.) and shifted by a bias, both computed from the normalised goal through gate_common (128, relu) and a 64-unit relu layer."""
    import torch

    class GatedGaussianMLPPolicy(torch.nn.Module):
        def __init__(self):
            super().__init__()
            dims = [state_size + goal_size] + list(hidden)
            lin = torch.nn.Linear
            self.goal_size = goal_size
            self.hidden = torch.nn.ModuleList([lin(a, b) for a, b in zip(dims[:-1], dims[1:])])
            self.gate_common = lin(goal_size, gate_common)
            self.gate_hidden = torch.nn.ModuleList([lin(gate_common, gate_hidden) for _ in hidden])
            self.gate_bias = torch.nn.ModuleList([lin(gate_hidden, h) for h in hidden])
            self.gate_scale = torch.nn.ModuleList([lin(gate_hidden, h) for h in hidden])
            for l in list(self.hidden) + [self.gate_common] + list(self.gate_hidden) + list(self.gate_bias) + list(self.gate_scale):
                torch.nn.init.xavier_uniform_(l.weight); torch.nn.init.zeros_(l.bias)
            self.mean = lin(dims[-1], action_size)
            torch.nn.init.uniform_(self.mean.weight, -init_output_scale, init_output_scale); torch.nn.init.zeros_(self.mean.bias)
            self.logstd = torch.nn.Parameter(torch.full((action_size,), math.log(noise)))

        def forward(self, norm_s, norm_g):
            return self.mean(_gated_trunk(self, norm_s, norm_g))

        def sample(self, norm_s, norm_g, explore_mask=None, generator=None):
            mu = self.forward(norm_s, norm_g)
            std = self.logstd.exp()
            eps = torch.randn(mu.shape, device=mu.device, generator=generator)
            if explore_mask is not None:
                eps = eps * explore_mask[:, None].to(eps.dtype)
            a = mu + std * eps
            logp = (-0.5 * eps * eps - self.logstd - 0.5 * math.log(2 * math.pi)).sum(dim=-1)
            return a, logp

    return GatedGaussianMLPPolicy()


def _gated_trunk(net, norm_s, norm_g):
    """the hidden layers of fc_2layers_gated_1024units (net: hidden, gate_common, gate_hidden, gate_bias, gate_scale)"""
    import torch
    gc = torch.relu(net.gate_common(norm_g))
    h = torch.cat([norm_s, norm_g], dim=-1)
    for l, gh, gb, gs in zip(net.hidden, net.gate_hidden, net.gate_bias, net.gate_scale):
        gate = torch.relu(gh(gc))
        h = torch.relu(2.0 * torch.sigmoid(gs(gate)) * l(h) + gb(gate))
    return h


def build_critic(state_size, goal_size=0, hidden=(1024, 512), gate_common=128, gate_hidden=64):
    """The PPO critic (PPOAgent._build_net_critic, R/learning/ppo_agent.py): a trunk over the actor's own normalised inputs, then a one-unit
    linear output, the normalised value; V = val_norm.unnormalize(output).  The trunk is the one this rollout builds for the actor: the plain
    fc_2layers_1024units over norm_s when goal_size is 0, the gated fc_2layers_gated_1024units over (norm_s, norm_g) otherwise.  The reference
    names the critic's network in an agent file, and the asset archive has no agent files.  Xavier-uniform weights and zero biases everywhere,
    the output layer included (tf.contrib.layers.xavier_initializer).  forward(norm_s[, norm_g]) returns [rows, 1]."""
    import torch

    class Critic(torch.nn.Module):
        def __init__(self):
            super().__init__()
            lin = torch.nn.Linear
            dims = [state_size + goal_size] + list(hidden)
            self.goal_size = goal_size
            self.hidden = torch.nn.ModuleList([lin(a, b) for a, b in zip(dims[:-1], dims[1:])])
            layers = list(self.hidden)
            if goal_size > 0:
                self.gate_common = lin(goal_size, gate_common)
                self.gate_hidden = torch.nn.ModuleList([lin(gate_common, gate_hidden) for _ in hidden])
                self.gate_bias = torch.nn.ModuleList([lin(gate_hidden, h) for h in hidden])
                self.gate_scale = torch.nn.ModuleList([lin(gate_hidden, h) for h in hidden])
                layers += [self.gate_common] + list(self.gate_hidden) + list(self.gate_bias) + list(self.gate_scale)
            self.out = lin(dims[-1], 1)
            for l in layers + [self.out]:
                torch.nn.init.xavier_uniform_(l.weight); torch.nn.init.zeros_(l.bias)

        def forward(self, norm_s, norm_g=None):
            if self.goal_size > 0:
                return self.out(_gated_trunk(self, norm_s, norm_g))
            h = norm_s
            for l in self.hidden:
                h = torch.relu(l(h))
            return self.out(h)

    return Critic()


def val_norm_from_rewards(env, discount, device="cpu"):
    """The value normaliser of PGAgent (_calc_val_bounds, _calc_val_offset_scale): values lie in [r_min, r_max] / (1 - discount), so
    mean = (val_max + val_min) / 2 and std = (val_max - val_min) / 2 (mean 10, std 10 for rewards in [0, 1] at discount 0.95)."""
    val_min, val_max = env.get_reward_min() / (1.0 - discount), env.get_reward_max() / (1.0 - discount)
    n = DeviceNormalizer(1, device=device)
    n.set_mean_std([0.5 * (val_max + val_min)], [0.5 * (val_max - val_min)])
    return n


def terminal_values(env, discount):
    """(val_fail, val_succ) of RLAgent._calc_term_vals: the value of a failed / succeeded episode's terminal state, r / (1 - discount), 0 at
    discount 0"""
    if discount == 0:
        return 0.0, 0.0
    return env.get_reward_fail() / (1.0 - discount), env.get_reward_succ() / (1.0 - discount)


def build_discriminator(amp_obs_size, hidden=(1024, 512), init_output_scale=1.0):
    """The AMP agent's discriminator (R/learning/amp_agent.py): the fc_2layers_1024units ReLU trunk (xavier-uniform weights, zero biases) over
    the normalised AMP observation and a one-unit linear logit whose weights are uniform in [-init_output_scale, init_output_scale].
    forward(norm_amp_obs) returns the logits [rows, 1]."""
    import torch

    class Discriminator(torch.nn.Module):
        def __init__(self):
            super().__init__()
            dims = [amp_obs_size] + list(hidden)
            self.hidden = torch.nn.ModuleList([torch.nn.Linear(a, b) for a, b in zip(dims[:-1], dims[1:])])
            for l in self.hidden:
                torch.nn.init.xavier_uniform_(l.weight); torch.nn.init.zeros_(l.bias)
            self.logit = torch.nn.Linear(dims[-1], 1)
            torch.nn.init.uniform_(self.logit.weight, -init_output_scale, init_output_scale); torch.nn.init.zeros_(self.logit.bias)

        def forward(self, norm_amp_obs):
            h = norm_amp_obs
            for l in self.hidden:
                h = torch.relu(l(h))
            return self.logit(h)

    return Discriminator()


def amp_rewards(logits, task_reward=None, task_lerp=0.0):
    """(style, reward) from discriminator logits d: style = max(0, 1 - 0.25 (1 - d)^2) (Peng et al. 2021, eq. 7) and the reward an AMP
    learner trains on, (1 - task_lerp) style + task_lerp task_reward, or style without a task reward."""
    style = (1.0 - 0.25 * (1.0 - logits) ** 2).clamp_min(0.0)
    return style, (style if task_reward is None else (1.0 - task_lerp) * style + task_lerp * task_reward)


def load_disc_weights(disc, d):
    """Copies discriminator weights {"hidden": [(w, b), ...], "logit": (w, b)} into a Discriminator (build_discriminator).  TF dense kernels are
    [in, out]; torch Linear weights are [out, in]."""
    import torch
    if len(d["hidden"]) != len(disc.hidden):
        raise ValueError("the discriminator has %d hidden layers, the weights %d" % (len(disc.hidden), len(d["hidden"])))
    f = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float32))
    with torch.no_grad():
        for layer, (w, b) in zip(list(disc.hidden) + [disc.logit], list(d["hidden"]) + [d["logit"]]):
            layer.weight.copy_(f(w).reshape(layer.weight.shape[::-1]).t()); layer.bias.copy_(f(b).reshape(layer.bias.shape))
    return disc


def load_critic_weights(critic, d):
    """Copies critic weights (deepmimic_b200.tf_checkpoint.load_critic: {"hidden": [(w, b), ...], "out": (w, b)}, and "gate_common" / "gates"
    for the gated trunk) into a Critic (build_critic).  TF dense kernels are [in, out]; torch Linear weights are [out, in]."""
    import torch
    if len(d["hidden"]) != len(critic.hidden):
        raise ValueError("the critic has %d hidden layers, the weights %d" % (len(critic.hidden), len(d["hidden"])))
    if ("gate_common" in d) != (critic.goal_size > 0):
        raise ValueError("gated weights need a goal-conditioned critic and plain weights a plain one")
    f = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float32))
    pairs = list(zip(critic.hidden, d["hidden"])) + [(critic.out, d["out"])]
    if critic.goal_size > 0:
        pairs.append((critic.gate_common, d["gate_common"]))
        for i, g in enumerate(d["gates"]):
            pairs += [(critic.gate_hidden[i], g["hidden"]), (critic.gate_bias[i], g["bias"]), (critic.gate_scale[i], g["scale"])]
    with torch.no_grad():
        for layer, (w, b) in pairs:
            layer.weight.copy_(f(w).reshape(layer.weight.shape[::-1]).t()); layer.bias.copy_(f(b).reshape(layer.bias.shape))
    return critic


def load_actor_weights(policy, actor):
    """Copies a reference actor (deepmimic_b200.tf_checkpoint.load_actor, or the tests/golden fixture keys w0 b0 w1 b1 wm bm logstd) into a
    GaussianMLPPolicy.  TF dense kernels are [in, out]; torch Linear weights are [out, in]."""
    import torch
    if "hidden" in actor:
        hidden, mean, logstd = actor["hidden"], actor["mean"], actor["logstd"]
    else:
        hidden, mean, logstd = [(actor["w0"], actor["b0"]), (actor["w1"], actor["b1"])], (actor["wm"], actor["bm"]), actor["logstd"]
    with torch.no_grad():
        for layer, (w, b) in zip(policy.hidden, hidden):
            layer.weight.copy_(torch.as_tensor(np.asarray(w, dtype=np.float32)).t()); layer.bias.copy_(torch.as_tensor(np.asarray(b, dtype=np.float32)))
        policy.mean.weight.copy_(torch.as_tensor(np.asarray(mean[0], dtype=np.float32)).t()); policy.mean.bias.copy_(torch.as_tensor(np.asarray(mean[1], dtype=np.float32)))
        policy.logstd.copy_(torch.as_tensor(np.asarray(logstd, dtype=np.float32)))
        if "gate_common" in actor:
            put = lambda layer, wb: (layer.weight.copy_(torch.as_tensor(np.asarray(wb[0], dtype=np.float32)).t()), layer.bias.copy_(torch.as_tensor(np.asarray(wb[1], dtype=np.float32))))
            put(policy.gate_common, actor["gate_common"])
            for i, g in enumerate(actor["gates"]):
                put(policy.gate_hidden[i], g["hidden"]); put(policy.gate_bias[i], g["bias"]); put(policy.gate_scale[i], g["scale"])
    return policy


def td_lambda_returns_host(rewards, values, end_values, done, terminate, discount, td_lambda, val_fail, val_succ, returns, advantages):
    """dm_td_lambda_returns's rule as torch ops on CPU tensors [T, N] (a CPU device has no kernel; on a CUDA device collect() always runs the
    kernel, capi.td_lambda_returns): returns and advantages are written."""
    import torch as t
    v_next = t.where(done & (terminate == 1), t.full_like(end_values, val_fail), end_values)
    v_next = t.where(done & (terminate == 2), t.full_like(end_values, val_succ), v_next)
    T = rewards.shape[0]
    for k in range(T - 1, -1, -1):
        g_next = v_next[k] if k == T - 1 else t.where(done[k], v_next[k], returns[k + 1])
        returns[k] = rewards[k] + discount * ((1.0 - td_lambda) * v_next[k] + td_lambda * g_next)
    advantages.copy_(returns - values)
    return returns, advantages


class _nullcontext:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


class BatchedRollout:
    """backend "torch": the policy is a torch module (cuBLAS GEMMs, eager normalisers) -- needed for training.
    backend "tensor_core": inference of the actor on the library's own tensor-core kernels (dm_mlp_*, kernels/dm_mlp.cu) on the environment's
    stream.  The plain 2-layer actor: normaliser, three GEMMs, bias / ReLU and the action un-normalisation in four launches (operand preparation
    + one per layer).  The gated actor of the goal-conditioned task scenes: six launches (operand preparation of [state | goal], gate trunk, both
    gate hidden layers, the two gated trunk layers, output layer).  The weights and the normaliser statistics are snapshotted by
    refresh_tensor_core_policy() (call it again after a learner update).

    disc (AMP scenes only): a Discriminator (build_discriminator) over the normalised agent AMP observation (normaliser amp_norm).  collect()
    then also returns the agent's AMP observation of every transition and the discriminator's logits, style rewards and amp_rewards, the reward
    an AMP learner trains on: the style reward in imitate_amp (the scene's own reward is not used there), (1 - task_reward_lerp) style +
    task_reward_lerp task reward in the task scenes, which need task_reward_lerp.  On the tensor_core backend the discriminator's reward runs in
    four launches (operand preparation, two hidden layers, the logit head with the reward epilogue).  learner.AMPDiscLearner trains the
    discriminator and refreshes its tensor-core handle (weights and amp_norm) on the device after every update().

    critic: a Critic (build_critic) with discount and td_lambda, which the reference reads from the agent file (Discount, TDLambda; there is no
    default).  val_norm is built from the env's reward bounds (val_norm_from_rewards).  collect() then also evaluates the critic on every
    state s_k and on the state s'_k each step ends in, before the reset (the terminal state of a finished episode, which RLAgent._end_path
    keeps), and runs the TD(lambda) return scan of rl_util.compute_return on the device (dm_td_lambda_returns, on either backend).  On the
    tensor_core backend the critic runs as one forward over the 2N rows [s_k; s'_k] on the plain or gated dm_mlp kernels."""

    def __init__(self, env, policy=None, exp_rate=1.0, noise=0.05, seed=0, backend="torch", disc=None, task_reward_lerp=None, critic=None,
                 discount=None, td_lambda=None):
        import torch
        self.torch, self.env = torch, env
        dev = env.device
        S, A, G = env.get_state_size(), env.get_action_size(), env.get_goal_size()
        self.goal_size = G
        # goal-conditioned scenes (AMP tasks) use the reference's gated actor; everything else the plain 1024-512 MLP
        self.policy = (policy or (build_gated_policy(S, G, A, noise=noise) if G > 0 else build_policy(S, A, noise=noise))).to(dev)
        if G > 0:
            self.g_norm = DeviceNormalizer(G, env.build_goal_norm_groups(), device=dev)
            self.g_norm.set_mean_std(-env.build_goal_offset(), 1.0 / env.build_goal_scale())
        self.s_norm = DeviceNormalizer(S, env.build_state_norm_groups(), device=dev)
        self.s_norm.set_mean_std(-env.build_state_offset(), 1.0 / env.build_state_scale())
        self.a_norm = DeviceNormalizer(A, device=dev)
        self.a_norm.set_mean_std(-env.build_action_offset(), 1.0 / env.build_action_scale())
        self.exp_rate = exp_rate
        self.gen = torch.Generator(device=dev); self.gen.manual_seed(seed)
        self.backend, self._tc = backend, None
        if backend not in ("torch", "tensor_core"):
            raise ValueError("backend must be 'torch' or 'tensor_core'")
        self.disc, self._tc_disc = None, None
        if disc is not None:
            if "AMP" not in env.get_name():
                raise ValueError("a discriminator needs an AMP scene (this one is %r)" % env.get_name())
            self._amp_task_reward = env.enable_amp_task_reward()
            if self._amp_task_reward:
                # the reference reads TaskRewardLerp from the agent file; there is no default to fall back on
                if task_reward_lerp is None or not 0.0 <= float(task_reward_lerp) <= 1.0:
                    raise ValueError("scene %r blends style and task rewards: task_reward_lerp in [0, 1] is required" % env.get_name())
                self.task_reward_lerp = float(task_reward_lerp)
            elif task_reward_lerp:
                raise ValueError("scene %r has no AMP task reward: task_reward_lerp must be 0 or None" % env.get_name())
            else:
                self.task_reward_lerp = 0.0
            self.disc = disc.to(dev)
            M = env.get_amp_obs_size()
            self.amp_norm = DeviceNormalizer(M, env.get_amp_obs_norm_group(), device=dev)
            self.amp_norm.set_mean_std(-env.get_amp_obs_offset(), 1.0 / env.get_amp_obs_scale())
        self.critic, self._tc_critic = None, None
        if critic is None:
            if discount is not None or td_lambda is not None:
                raise ValueError("discount and td_lambda are the critic's: they need a critic")
        else:
            # the reference reads Discount and TDLambda from the agent file; there is no default to fall back on
            if discount is None or not 0.0 <= float(discount) < 1.0:
                raise ValueError("a critic needs a discount in [0, 1)")
            if td_lambda is None or not 0.0 <= float(td_lambda) <= 1.0:
                raise ValueError("a critic needs a td_lambda in [0, 1]")
            if getattr(critic, "goal_size", 0) != G:
                raise ValueError("the critic sees %d goal values, the scene has %d" % (getattr(critic, "goal_size", 0), G))
            self.critic = critic.to(dev)
            self.discount, self.td_lambda = float(discount), float(td_lambda)
            self.val_norm = val_norm_from_rewards(env, self.discount, device=dev)
            self.val_fail, self.val_succ = terminal_values(env, self.discount)

    def refresh_tensor_core_policy(self):
        """(re)builds the dm_mlp handles from the current torch policy, discriminator, critic and normalisers"""
        from .capi import TensorCoreGatedMLP, TensorCoreMLP
        pol, env = self.policy, self.env
        if len(pol.hidden) != 2:
            raise ValueError("the tensor_core backend implements exactly two hidden layers")
        g = lambda t: t.detach().float().cpu().numpy()
        if self._tc is not None:
            self._tc.close()
        wb = lambda l: (g(l.weight).T, g(l.bias))
        gated = lambda net, head: dict(hidden=[wb(l) for l in net.hidden], mean=wb(head), gate_common=wb(net.gate_common),
                                       gates=[dict(hidden=wb(h), scale=wb(sc), bias=wb(b)) for h, sc, b in zip(net.gate_hidden, net.gate_scale, net.gate_bias)])
        if self.goal_size > 0:
            self._tc = TensorCoreGatedMLP(gated(pol, pol.mean), s_mean=g(self.s_norm.mean), s_std=g(self.s_norm.std), s_clip=self.s_norm.clip, g_mean=g(self.g_norm.mean),
                                          g_std=g(self.g_norm.std), g_clip=self.g_norm.clip, a_mean=g(self.a_norm.mean), a_std=g(self.a_norm.std),
                                          max_rows=env.num_envs, device=env.device.index or 0)
        else:
            self._tc = TensorCoreMLP(g(pol.hidden[0].weight).T, g(pol.hidden[0].bias), g(pol.hidden[1].weight).T, g(pol.hidden[1].bias), g(pol.mean.weight).T, g(pol.mean.bias),
                                     in_mean=g(self.s_norm.mean), in_std=g(self.s_norm.std), in_clip=self.s_norm.clip, out_mean=g(self.a_norm.mean), out_std=g(self.a_norm.std),
                                     max_rows=env.num_envs, device=env.device.index or 0)
        self._tc_act = self.torch.empty(env.num_envs, env.get_action_size(), device=env.device)
        if self.disc is not None:
            d = self.disc
            if len(d.hidden) != 2:
                raise ValueError("the tensor_core backend implements exactly two hidden layers")
            if self._tc_disc is not None:
                self._tc_disc.close()
            self._tc_disc = TensorCoreMLP(g(d.hidden[0].weight).T, g(d.hidden[0].bias), g(d.hidden[1].weight).T, g(d.hidden[1].bias), g(d.logit.weight).T, g(d.logit.bias),
                                          in_mean=g(self.amp_norm.mean), in_std=g(self.amp_norm.std), in_clip=self.amp_norm.clip, max_rows=env.num_envs,
                                          device=env.device.index or 0)
        if self.critic is not None:
            c = self.critic
            if len(c.hidden) != 2:
                raise ValueError("the tensor_core backend implements exactly two hidden layers")
            if self._tc_critic is not None:
                self._tc_critic.close()
            # one output unit un-normalised by val_norm; 2N rows: [s_k; s'_k] in one forward
            vm, vs = g(self.val_norm.mean), g(self.val_norm.std)
            if self.goal_size > 0:
                self._tc_critic = TensorCoreGatedMLP(gated(c, c.out), s_mean=g(self.s_norm.mean), s_std=g(self.s_norm.std), s_clip=self.s_norm.clip,
                                                     g_mean=g(self.g_norm.mean), g_std=g(self.g_norm.std), g_clip=self.g_norm.clip, a_mean=vm, a_std=vs,
                                                     max_rows=2 * env.num_envs, device=env.device.index or 0)
            else:
                self._tc_critic = TensorCoreMLP(*wb(c.hidden[0]), *wb(c.hidden[1]), *wb(c.out), in_mean=g(self.s_norm.mean), in_std=g(self.s_norm.std),
                                                in_clip=self.s_norm.clip, out_mean=vm, out_std=vs, max_rows=2 * env.num_envs, device=env.device.index or 0)
        return self._tc

    def retile_tensor_core(self, *roles):
        """the existing tensor-core handles of `roles` ("actor", "critic", "disc") take the torch modules' current weights and the normalisers'
        current statistics, re-tiled and copied on the device (the discriminator: amp_norm and the identity output normaliser)"""
        from .capi import tc_layers
        t, dev = self.torch, self.env.device
        c = lambda n: (n.mean.contiguous(), n.std.contiguous())
        for role in roles:
            tc, net = dict(actor=(self._tc, self.policy), critic=(self._tc_critic, self.critic), disc=(self._tc_disc, self.disc))[role]
            if tc is None:
                continue
            st = t.cuda.current_stream(dev).cuda_stream
            tc.set_weights_device(tc_layers(net, role), stream=st)
            if role == "disc":
                tc.set_normalizers_device(*c(self.amp_norm), t.zeros(1, device=dev), t.ones(1, device=dev), stream=st)
            else:
                goal = c(self.g_norm) if self.goal_size > 0 else ()
                tc.set_normalizers_device(*c(self.s_norm), *goal, *c(self.a_norm if role == "actor" else self.val_norm), stream=st)

    def _act_tensor_core(self, s, explore, g=None):
        """un-normalised actions and log-probabilities from the tensor-core actor (exploration noise is drawn in torch, added in the kernel's epilogue);
        g: the goals, for the gated actor of the goal-conditioned scenes"""
        t = self.torch
        if self._tc is None:
            self.refresh_tensor_core_policy()
        std = self.policy.logstd.detach().exp()
        eps = t.randn(s.shape[0], std.shape[0], device=s.device, generator=self.gen) * explore[:, None].to(s.dtype)
        noise = (std * eps).contiguous()
        cur = t.cuda.current_stream(s.device)
        if g is None:
            self._tc.forward(s.contiguous(), self._tc_act, noise=noise, stream=cur.cuda_stream)
        else:
            self._tc.forward(s.contiguous(), g.contiguous(), self._tc_act, noise=noise, stream=cur.cuda_stream)
        logp = (-0.5 * eps * eps - self.policy.logstd.detach() - 0.5 * math.log(2 * math.pi)).sum(dim=-1)
        return self._tc_act, logp

    def _disc_rewards(self, amp, r, out, k):
        """the discriminator's logits, style rewards and amp_rewards of step k from the agent AMP observations amp and the env rewards r"""
        task = r if self._amp_task_reward else None
        logit, style, reward = out["disc_logits"][k], out["style_rewards"][k], out["amp_rewards"][k]
        if self.backend == "tensor_core":
            self._tc_disc.style_reward(amp, reward, task_reward=task, task_lerp=self.task_reward_lerp, logit=logit, style=style,
                                       stream=self.torch.cuda.current_stream(amp.device).cuda_stream)
        else:
            d = self.disc(self.amp_norm.normalize(amp))[:, 0]
            st, rw = amp_rewards(d, task, self.task_reward_lerp)
            logit.copy_(d); style.copy_(st); reward.copy_(rw)

    def _critic_values(self, x, g, v):
        """V (un-normalised) of the rows x [2N, S] (and goals g [2N, G] in the goal-conditioned scenes) into v [2N]"""
        if self.backend == "tensor_core":
            st = self.torch.cuda.current_stream(x.device).cuda_stream
            if g is None:
                self._tc_critic.forward(x, v[:, None], stream=st)
            else:
                self._tc_critic.forward(x, g, v[:, None], stream=st)
        else:
            ns = self.s_norm.normalize(x)
            out = self.critic(ns) if g is None else self.critic(ns, self.g_norm.normalize(g))
            v.copy_(self.val_norm.unnormalize(out)[:, 0])

    def _returns(self, out):
        """TD(lambda) returns and advantages of the window over amp_rewards (with a discriminator: AMPAgent trains on them) or rewards"""
        t = self.torch
        r = out["amp_rewards"] if self.disc is not None else out["rewards"]
        args = (r, out["values"], out["end_values"], out["dones"], out["terminate"], self.discount, self.td_lambda, self.val_fail, self.val_succ,
                out["returns"], out["advantages"])
        if r.is_cuda:
            from .capi import td_lambda_returns
            td_lambda_returns(*args, stream=t.cuda.current_stream(r.device).cuda_stream)
        else:
            td_lambda_returns_host(*args)

    @property
    def stream(self):
        return self.env.stream

    def collect(self, num_steps, record_stats=True, record_pose=False, record_kin_pose=False, record_course=False):
        """num_steps policy steps of all environments; returns dict of [T, N, .] tensors (states, actions, logps, rewards, dones, terminate,
        explore = the exploration draw of each step (True: the action was sampled, False: the mode was taken); goals
        in the goal-conditioned scenes; with a discriminator amp_obs, disc_logits, style_rewards, amp_rewards; with a critic values = V(s_k),
        end_values = V(s'_k) of the state step k ended in (before the reset), returns and advantages = returns - values).  rewards is the env's
        reward.  A path still running at the last step is bootstrapped with its end value, as the reference bootstraps a path that ends by time
        limit (a deviation: the reference stores only complete paths).  record_pose adds the simulated characters' poses (env.record_pose),
        [T, N, pose_dim] each: poses / vels at s_k, end_poses / end_vels at s'_k, before the reset, like values / end_values.  record_kin_pose
        adds kin_poses [T, N, pose_dim], the kinematic characters' poses (env.record_kin_pose) at s_k, recorded next to poses.  record_course
        (an env with a goal course, env.set_goal_course) adds course [T, N, 4], env.course_record() after step k and before its reset."""
        t, env = self.torch, self.env
        N, S, A = env.num_envs, env.get_state_size(), env.get_action_size()
        out = dict(states=t.empty(num_steps, N, S, device=env.device), actions=t.empty(num_steps, N, A, device=env.device),
                   logps=t.empty(num_steps, N, device=env.device), rewards=t.empty(num_steps, N, device=env.device),
                   dones=t.empty(num_steps, N, dtype=t.bool, device=env.device), terminate=t.empty(num_steps, N, dtype=t.int32, device=env.device),
                   explore=t.empty(num_steps, N, dtype=t.bool, device=env.device))
        G = self.goal_size
        if G > 0:
            out["goals"] = t.empty(num_steps, N, G, device=env.device)
        if self.disc is not None:
            out["amp_obs"] = t.empty(num_steps, N, env.get_amp_obs_size(), device=env.device)
            for key in ("disc_logits", "style_rewards", "amp_rewards"):
                out[key] = t.empty(num_steps, N, device=env.device)
        if record_pose:
            P = env.get_pose_dim()
            for key in ("poses", "vels", "end_poses", "end_vels"):
                out[key] = t.empty(num_steps, N, P, device=env.device)
        if record_kin_pose:
            out["kin_poses"] = t.empty(num_steps, N, env.get_pose_dim(), device=env.device)
        if record_course:
            out["course"] = t.empty(num_steps, N, 4, device=env.device)
        crit = self.critic is not None
        if crit:
            for key in ("values", "end_values", "returns", "advantages"):
                out[key] = t.empty(num_steps, N, device=env.device)
            # critic inputs [s_k; s'_k] (and goals) and its outputs [V(s_k) | V(s'_k)] per step
            x2, v2 = t.empty(2 * N, S, device=env.device), t.empty(num_steps, 2 * N, device=env.device)
            g2 = t.empty(2 * N, G, device=env.device) if G > 0 else None
        # the whole loop runs on the environment's stream: with the actor and the bookkeeping on another stream every env call is a pair of
        # cross-stream event waits (measured: 0.4 ms of bubbles per policy step); the caller's stream waits for the trajectory at the end
        caller = t.cuda.current_stream(env.device) if env.device.type == "cuda" else None
        if caller is not None:
            env.stream.wait_stream(caller)
        with t.no_grad(), (t.cuda.stream(env.stream) if caller is not None else _nullcontext()):
            s = env.record_state()
            for k in range(num_steps):
                out["states"][k] = s
                if record_pose:
                    p, v = env.record_pose()
                    out["poses"][k] = p; out["vels"][k] = v
                if record_kin_pose:
                    out["kin_poses"][k] = env.record_kin_pose()
                if crit:
                    x2[:N] = s
                if record_stats:
                    self.s_norm.record(s)
                explore = t.rand(N, device=env.device, generator=self.gen) < self.exp_rate
                out["explore"][k] = explore   # RLAgent's EXP_ACTION_FLAG: PPOAgent._update trains the actor on these samples only
                if G > 0:   # RLAgent._update_new_action records the goal next to the state (R/learning/rl_agent.py:319-343)
                    g = env.record_goal()
                    out["goals"][k] = g
                    if crit:
                        g2[:N] = g
                    if record_stats:
                        self.g_norm.record(g)
                if self.backend == "tensor_core":
                    a, logp = self._act_tensor_core(s, explore, g if G > 0 else None)
                elif G > 0:
                    na, logp = self.policy.sample(self.s_norm.normalize(s), self.g_norm.normalize(g), explore, self.gen)
                else:
                    na, logp = self.policy.sample(self.s_norm.normalize(s), explore, self.gen)
                if self.backend != "tensor_core":
                    a = self.a_norm.unnormalize(na).contiguous()
                s, r, done, term = env.step(a)
                out["actions"][k] = a; out["logps"][k] = logp; out["rewards"][k] = r; out["dones"][k] = done; out["terminate"][k] = term
                if record_pose:   # before the reset: the end pose of a finished episode is its terminal pose
                    p, v = env.record_pose()
                    out["end_poses"][k] = p; out["end_vels"][k] = v
                if record_course:
                    out["course"][k] = env.course_record()
                if self.disc is not None:
                    # before the reset: the last transition of a finished episode is the agent's own motion, not the restarted state
                    amp = env.record_amp_obs_agent()
                    out["amp_obs"][k] = amp
                    if record_stats:
                        self.amp_norm.record(amp)
                    self._disc_rewards(out["amp_obs"][k], out["rewards"][k], out, k)
                if crit:
                    # before the reset: s'_k of a finished episode is its terminal state (and goal), not the restarted one
                    x2[N:] = s
                    if G > 0:
                        g2[N:] = env.record_goal()
                    self._critic_values(x2, g2, v2[k])
                env.reset()                # restarts exactly the finished episodes
                # the restarted environments need the observation of their new state.  Unconditional (one more ~10 us observation kernel) instead of
                # `if done.any()`: that test is a host synchronisation per policy step, which leaves the GPU idle while the host launches the
                # next step's small kernels (measured: 1.52 M -> see tests/test_mlp_gpu.py for the current rates)
                s = env.record_state()
            if crit:
                out["values"].copy_(v2[:, :N]); out["end_values"].copy_(v2[:, N:])
                self._returns(out)
        if caller is not None:
            caller.wait_stream(env.stream)
        return out


def course_stats(kind, course, dones, counts, step_dt):
    """aggregates of every environment's first episode from collect's course records [T, N, 4] and dones [T, N] (T covering it): kind
    "heading" -> dict(speed_err [N], the mean |along-track speed - commanded speed|, and cross_speed [N], the mean |cross-track speed|, over the
    episode's steps, m/s); "target" -> dict(waypoints [N], the waypoints reached, and course_time [N], the episode time in s at the end of the
    step that reached the last of counts[e] waypoints, NaN if none did; step_dt: the policy step in s)"""
    import torch as t
    d = dones.to(t.int32)
    first = (t.cumsum(d, 0) - d) == 0   # the steps of the first episode: no episode end before them
    steps = first.sum(0)
    if kind == "heading":
        f = first.to(course.dtype)
        return dict(speed_err=(course[..., 2].abs() * f).sum(0) / steps, cross_speed=(course[..., 3].abs() * f).sum(0) / steps)
    last = (steps - 1).clamp(min=0).long()
    reached = course[last, t.arange(course.shape[1], device=course.device), 2]
    done_all = first & (course[..., 2] >= t.as_tensor(counts, device=course.device).to(course.dtype))
    k = t.argmax(done_all.to(t.int32), 0)
    ctime = t.where(done_all.any(0), (k + 1).to(course.dtype) * step_dt, t.full_like(reached, float("nan")))
    return dict(waypoints=reached, course_time=ctime)


def run_episodes(ro, pose_envs=0, limit=1 << 16, pose_error=False, course=False):
    """One complete episode of every environment of ro's env from its current state, in chunks of 32 policy steps of ro.collect (the
    environments that finish first keep running into their next episode, which is not counted).  Set the env's mode and ro's exploration
    before the call (test mode, exp_rate 0 for an evaluation).  One host synchronisation per chunk.  Returns dict(returns [N] float32, lengths
    [N] int32 = policy steps, terminate [N] int32 = the terminate code of the episode's last step: 0 time limit, 1 fail, 2 success); with
    pose_envs > 0 also poses and end_poses of the first pose_envs environments, lists of the chunks' [32, pose_envs, pose_dim] tensors
    (episode_motion assembles an environment's frames); the other environments' poses are not kept.  pose_error=True keeps every environment's
    poses and kin poses (the simulated and the kinematic character at the step's start, collect's poses and kin_poses) and adds pose_err and
    pose_err_dtw [N] float32, the phase-locked and the time-warped tracking error in metres of each episode (one BatchedCore.pose_error call;
    the terminal pose is not scored).  That keeps 2 x T x N x pose_dim floats: 2 x 428 MB at N = 4096, T = 608 and pose_dim 43 (humanoid3d),
    plus the call's scratch of about as much again.  course=True (an env with a goal course) adds course [T, N, 4] (collect's records of
    every step run) and course_stats' aggregates of each first episode: speed_err and cross_speed in the heading scenes, waypoints and
    course_time in the target scene.
    RuntimeError when an episode runs longer than `limit` policy steps."""
    import torch as t
    env = ro.env
    n = env.num_envs
    ret, ended = t.zeros(n, device=env.device), t.zeros(n, dtype=t.bool, device=env.device)
    length, term = t.zeros(n, dtype=t.int32, device=env.device), t.zeros(n, dtype=t.int32, device=env.device)
    poses, end_poses, all_poses, kin_poses, courses, dones = [], [], [], [], [], []
    for _ in range(0, limit, 32):
        traj = ro.collect(32, record_stats=False, record_pose=bool(pose_envs or pose_error), record_kin_pose=pose_error, record_course=course)
        if course:
            courses.append(traj["course"]); dones.append(traj["dones"])
        if pose_envs:
            poses.append(traj["poses"][:, :pose_envs].clone()); end_poses.append(traj["end_poses"][:, :pose_envs].clone())
        if pose_error:
            all_poses.append(traj["poses"]); kin_poses.append(traj["kin_poses"])
        for r, d, c in zip(traj["rewards"], traj["dones"], traj["terminate"]):
            ret += t.where(ended, t.zeros_like(r), r)
            length += (~ended).int()
            term = t.where(ended, term, c)
            ended |= d
        if bool(ended.all()):
            out = dict(returns=ret, lengths=length, terminate=term)
            if pose_envs:
                out.update(poses=poses, end_poses=end_poses)
            if pose_error:
                a, r = t.cat(all_poses), t.cat(kin_poses)
                del all_poses[:], kin_poses[:]
                env._pre()   # the call runs on the handle's stream
                lock, dtw = env._core.pose_error(a, r, length)
                env._post()
                out.update(pose_err=lock, pose_err_dtw=dtw)
            if course:
                rec = t.cat(courses)
                out.update(course=rec, **course_stats(env.course_kind, rec, t.cat(dones), env.course_counts,
                                                      env.get_updates_per_action() * env.UPDATE_DT))
            return out
    raise RuntimeError("an episode ran longer than %d policy steps" % limit)


def episode_motion(poses, end_poses, env_index, length):
    """the frames of environment env_index's first episode of `length` policy steps: the poses it took its actions in (steps 0 .. length - 1)
    and the terminal pose its last step ended in, [length + 1, pose_dim] float64 on the host.  poses / end_poses: [T, N, pose_dim] tensors or
    run_episodes' lists of chunks."""
    import torch as t
    cat = lambda x: t.cat(list(x)) if isinstance(x, (list, tuple)) else x
    p, e = cat(poses), cat(end_poses)
    if not 1 <= length <= p.shape[0]:
        raise ValueError("an episode of %d steps does not fit %d recorded steps" % (length, p.shape[0]))
    return t.cat([p[:length, env_index], e[length - 1:length, env_index]]).double().cpu().numpy()

