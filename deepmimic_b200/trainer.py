"""The reference agent's training iteration (R/learning/rl_agent.py: RLAgent._train, _update_exp_params; ppo_agent.py: PPOAgent._update,
update_actor_stepsize; amp_agent.py: AMPAgent._update_disc and its replay buffers, replay_buffer_rand_storage.py) over BatchedRollout.collect,
PPOLearner.update and AMPDiscLearner.update, its agent files and its checkpoints.

The reference tree is not vendored here; each rule is restated below as one function with the reading it follows, and tests/test_trainer_cpu.py
and tests/test_train_cpu.py pin them.  These are readings of the reference that could not be checked against its source here; where they and
the reference disagree, the reference is right.

  DeviceReplayBuffer   ReplayBufferRandStorage on a torch device tensor: the AMP agent's two disc buffers (agent and expert observations)
  update_actor_stepsize, disc_steps_per_iter, exploration_params, train_schedule   the iteration's schedules
  AgentConfig          an agent file (--agent_files) of PPOAgent / AMPAgent, validated
  Trainer              the loop: one iteration() = collect a window, store the AMP observations, train, update the normalisers; evaluation,
                       a tabular log and bit-exact checkpoints (state_dict / load_state_dict)

Agent-file keys (AgentConfig.from_json).  Every key of the first two groups is required; any key not in this table is refused by name:
  used by the loop
    AgentType              "PPO" or "AMP" (an AMP agent adds the discriminator, its learner and its replay buffers)
    ActorNet, CriticNet    fc_2layers_1024units (scenes without a goal) or fc_2layers_gated_1024units (the goal-conditioned task scenes)
    ActorStepsize, ActorMomentum, ActorWeightDecay, ActorInitOutputScale      PPOLearner and build_policy / build_gated_policy
    CriticStepsize, CriticMomentum, CriticWeightDecay                          PPOLearner
    Discount, TDLambda                          BatchedRollout's critic and return scan
    MiniBatchSize, Epochs, RatioClip, NormAdvClip                              PPOLearner
    TarClipFrac, ActorStepsizeDecay             update_actor_stepsize after every PPO update (TarClipFrac < 0 turns it off)
    InitSamples, NormalizerSamples              train_schedule
    ExpAnnealSamples, ExpParamsBeg, ExpParamsEnd   exploration_params: Rate is the exploration rate of each window; Noise of ExpParamsBeg is
                                                the actor's fixed standard deviation; the other fields are accepted and do not act
    OutputIters            an evaluation (Test_Return) and a checkpoint every OutputIters iterations
    IntOutputIters         an intermediate checkpoint every IntOutputIters iterations (0: none)
    TestEpisodes           the episodes of an evaluation, one per environment of the evaluation handle
  used by AMP agents only (refused in a PPO agent file)
    DiscNet                fc_2layers_1024units
    DiscStepSize, DiscMomentum, DiscWeightDecay, DiscLogitRegWeight, DiscGradPenalty, DiscBatchSize   AMPDiscLearner
    DiscStepsPerBatch      disc_steps_per_iter
    DiscBufferSize         the capacity of both disc buffers, agent and expert observations
    DiscInitOutputScale    build_discriminator
    TaskRewardLerp         BatchedRollout: the blend of style and task rewards (must be 0 in imitate_amp, which has no task reward)
  replaced by the batched loop (accepted, do not act)
    BatchSize, ReplayBufferSize   the window of window_steps x num_envs samples that each iteration collects and trains on
    UpdatePeriod, ItersPerUpdate  one update per window
  refused
    any other key; net names other than the two above; an AgentType other than PPO and AMP"""
import math

EXP_PARAM_KEYS = ("Rate", "InitActionRate", "Noise", "NoiseInternal", "Temp")   # ExpParams of the reference's agent files


class DeviceReplayBuffer:
    """ReplayBufferRandStorage (R/learning/replay_buffer_rand_storage.py) on a [capacity, width] device tensor.

    store(rows): n rows fill the free slots in order; once the buffer is full, the rest of a store overwrites slots drawn uniformly, distinct
    within that draw (np.random.choice(capacity, k, replace=False)), over the whole buffer -- including the slots the same store has just
    filled, so a store that crosses the end can keep fewer than n of its rows.  A store must be smaller than the buffer (the reference
    asserts it: a path longer than the buffer).  sample(n): n rows uniformly with replacement from the filled part.  The maintainer's reading
    of the reference, in particular the draw over the whole buffer for a store that crosses the end; not checked against its source.

    The draws come from a seeded torch.Generator on the buffer's device, not the reference's numpy stream; the fill level is host arithmetic,
    so neither call synchronises the host."""

    def __init__(self, capacity, width, device, seed=0, dtype=None):
        import torch
        if capacity < 2:
            raise ValueError("DeviceReplayBuffer: capacity must be at least 2 (got %d)" % capacity)
        self.capacity, self.width = int(capacity), int(width)
        self.rows = torch.zeros(self.capacity, self.width, device=device, dtype=dtype or torch.float32)
        self.generator = torch.Generator(device=self.rows.device)
        self.generator.manual_seed(int(seed))
        self.size = 0          # filled slots
        self.total_count = 0   # rows ever stored

    def store(self, data):
        import torch
        n = data.shape[0]
        if n == 0:
            return
        if n >= self.capacity:
            raise ValueError("DeviceReplayBuffer.store: a store of %d rows must be smaller than the buffer (%d)" % (n, self.capacity))
        if tuple(data.shape[1:]) != (self.width,):
            raise ValueError("DeviceReplayBuffer.store: rows of width %d expected (got %s)" % (self.width, tuple(data.shape[1:])))
        fill = min(n, self.capacity - self.size)
        if fill:
            self.rows[self.size:self.size + fill] = data[:fill]
        if fill < n:
            slots = torch.randperm(self.capacity, generator=self.generator, device=self.rows.device)[:n - fill]
            self.rows.index_copy_(0, slots, data[fill:].to(self.rows.dtype))
        self.size = min(self.size + n, self.capacity)
        self.total_count += n

    def filled(self):
        """the filled part, [size, width] (a view): what AMPDiscLearner.update draws its minibatches from"""
        return self.rows[:self.size]

    def sample(self, n):
        import torch
        if self.size == 0:
            raise ValueError("DeviceReplayBuffer.sample: the buffer is empty")
        idx = torch.randint(0, self.size, (int(n),), generator=self.generator, device=self.rows.device)
        return self.rows[idx]

    def state_dict(self):
        return dict(rows=self.rows.clone(), size=self.size, total_count=self.total_count, generator=self.generator.get_state())

    def load_state_dict(self, s):
        if tuple(s["rows"].shape) != (self.capacity, self.width):
            raise ValueError("DeviceReplayBuffer.load_state_dict: a [%d, %d] buffer expected (got %s)" % (self.capacity, self.width, tuple(s["rows"].shape)))
        self.rows.copy_(s["rows"])
        self.size, self.total_count = int(s["size"]), int(s["total_count"])
        self.generator.set_state(s["generator"])


def update_actor_stepsize(stepsize, clip_frac, tar_clip_frac, decay, iteration):
    """PPOAgent.update_actor_stepsize: TarClipFrac control of the actor's stepsize after an update.  Acts only when tar_clip_frac >= 0 and
    iteration > 5 (the warm-up); the tolerance band is [tar / 1.5, tar * 1.5]; a clip fraction above the band multiplies the stepsize by decay
    (ActorStepsizeDecay), one below it divides it by decay; the result is clipped to [1e-8, 1e-2].  The stepsize is returned unchanged
    otherwise.  The maintainer's reading of the reference, not checked against its source."""
    if tar_clip_frac < 0 or iteration <= 5:
        return stepsize
    if clip_frac > tar_clip_frac * 1.5:
        stepsize *= decay
    elif clip_frac < tar_clip_frac / 1.5:
        stepsize /= decay
    return min(max(stepsize, 1e-8), 1e-2)


def disc_steps_per_iter(samples, steps_per_batch, batch_size):
    """AMPAgent._update_disc: ceil(DiscStepsPerBatch * samples / DiscBatchSize) discriminator steps for an iteration that stored `samples`
    agent observations.  The maintainer's reading of the reference, not checked against its source."""
    return int(math.ceil(steps_per_batch * samples / batch_size))


def exploration_params(beg, end, samples, anneal_samples):
    """RLAgent._update_exp_params: every ExpParams field lerped from ExpParamsBeg to ExpParamsEnd by clip(samples / ExpAnnealSamples, 0, 1).
    Only Rate acts in the batched loop; the actor's sigma stays ExpParamsBeg.Noise (the reference builds the actor's std once), and Temp,
    InitActionRate and NoiseInternal are logged and unused by PPO.  Missing fields read as 0."""
    t = min(max(samples / anneal_samples, 0.0), 1.0) if anneal_samples > 0 else 0.0
    return {k: (1.0 - t) * float(beg.get(k, 0.0)) + t * float(end.get(k, 0.0)) for k in EXP_PARAM_KEYS}


def train_schedule(total_samples, initialized, need_normalizer_update, init_samples, normalizer_samples):
    """RLAgent._train after a window, with total_samples counting it: returns (train, initialized, update_normalizers, need_normalizer_update).

    1. An initialised agent trains (one iteration: discriminator, then PPO update); an uninitialised one only becomes initialised once
       total_samples >= InitSamples, without training in that call.
    2. Then, while the normaliser still needs updates, the window's records are folded in (update_normalizers), and the need continues while
       NormalizerSamples > total_samples -- so the window that crosses NormalizerSamples is still recorded.
    A window is recorded into the normalisers only while need_normalizer_update held when it was stored (RLAgent._store_path).  The
    maintainer's reading of the reference, not checked against its source."""
    train = bool(initialized)
    if not initialized and total_samples >= init_samples:
        initialized = True
    update = bool(need_normalizer_update)
    if update:
        need_normalizer_update = normalizer_samples > total_samples
    return train, initialized, update, need_normalizer_update


# ---- agent files
NETS = ("fc_2layers_1024units", "fc_2layers_gated_1024units")
_INF = float("inf")
# key -> (kind, lo, hi, lo_open, hi_open): kind "int" / "num" / "net" / "exp" / "type"
_PPO_KEYS = {
    "AgentType": ("type",), "ActorNet": ("net",), "CriticNet": ("net",),
    "ActorStepsize": ("num", 0.0, _INF, True, True), "ActorMomentum": ("num", 0.0, 1.0, False, True),
    "ActorWeightDecay": ("num", 0.0, _INF, False, True), "ActorInitOutputScale": ("num", 0.0, _INF, True, True),
    "CriticStepsize": ("num", 0.0, _INF, True, True), "CriticMomentum": ("num", 0.0, 1.0, False, True),
    "CriticWeightDecay": ("num", 0.0, _INF, False, True),
    "Discount": ("num", 0.0, 1.0, False, True), "TDLambda": ("num", 0.0, 1.0, False, False),
    "MiniBatchSize": ("int", 1), "Epochs": ("int", 1), "RatioClip": ("num", 0.0, 1.0, True, True), "NormAdvClip": ("num", 0.0, _INF, True, True),
    "TarClipFrac": ("num", -_INF, 1.0, True, False), "ActorStepsizeDecay": ("num", 0.0, _INF, True, True),
    "InitSamples": ("int", 0), "NormalizerSamples": ("int", 0), "ExpAnnealSamples": ("num", 0.0, _INF, False, True),
    "ExpParamsBeg": ("exp",), "ExpParamsEnd": ("exp",), "OutputIters": ("int", 1), "IntOutputIters": ("int", 0), "TestEpisodes": ("int", 1),
}
_AMP_KEYS = {
    "DiscNet": ("net",), "DiscStepSize": ("num", 0.0, _INF, True, True), "DiscMomentum": ("num", 0.0, 1.0, False, True),
    "DiscWeightDecay": ("num", 0.0, _INF, False, True), "DiscLogitRegWeight": ("num", 0.0, _INF, False, True),
    "DiscGradPenalty": ("num", 0.0, _INF, False, True), "DiscBatchSize": ("int", 1), "DiscStepsPerBatch": ("num", 0.0, _INF, True, True),
    "DiscBufferSize": ("int", 2), "DiscInitOutputScale": ("num", 0.0, _INF, True, True), "TaskRewardLerp": ("num", 0.0, 1.0, False, False),
}
_REPLACED_KEYS = ("BatchSize", "ReplayBufferSize", "UpdatePeriod", "ItersPerUpdate")


def _check_value(key, spec, v):
    kind = spec[0]
    if kind == "type":
        if v not in ("PPO", "AMP"):
            raise ValueError("agent file: %s must be \"PPO\" or \"AMP\" (got %r)" % (key, v))
    elif kind == "net":
        if v not in NETS:
            raise ValueError("agent file: %s %r is not supported (supported: %s)" % (key, v, ", ".join(NETS)))
    elif kind == "exp":
        if not isinstance(v, dict):
            raise ValueError("agent file: %s must be an object" % key)
        for k, x in v.items():
            if k not in EXP_PARAM_KEYS:
                raise ValueError("agent file: unknown key %s.%s (known: %s)" % (key, k, ", ".join(EXP_PARAM_KEYS)))
            _check_value("%s.%s" % (key, k), ("num", 0.0, 1.0, False, False) if k == "Rate" else ("num", -_INF, _INF, True, True), x)
        if "Rate" not in v:
            raise ValueError("agent file: %s.Rate is missing" % key)
    elif kind == "int":
        if isinstance(v, bool) or not isinstance(v, (int, float)) or v != int(v) or v < spec[1]:
            raise ValueError("agent file: %s must be an integer >= %d (got %r)" % (key, spec[1], v))
    else:
        _, lo, hi, lo_open, hi_open = spec
        bad = isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(float(v))
        if not bad:
            bad = v < lo or v > hi or (lo_open and v == lo) or (hi_open and v == hi)
        if bad:
            raise ValueError("agent file: %s must be in %s%s, %s%s (got %r)" % (key, "(" if lo_open else "[", lo, hi, ")" if hi_open else "]", v))


class AgentConfig:
    """A validated agent file of the reference (PPOAgent / AMPAgent; the key table is in this module's docstring).  cfg[key] reads a value;
    integer keys read as int.  values is the file's content as parsed (what a checkpoint compares)."""

    def __init__(self, values):
        if not isinstance(values, dict):
            raise ValueError("agent file: a JSON object expected")
        agent_type = values.get("AgentType")
        _check_value("AgentType", _PPO_KEYS["AgentType"], agent_type)
        known = dict(_PPO_KEYS, **_AMP_KEYS) if agent_type == "AMP" else _PPO_KEYS
        for k in values:
            if k in _AMP_KEYS and agent_type != "AMP":
                raise ValueError("agent file: %s is an AMP agent key (AgentType is %s)" % (k, agent_type))
            if k not in known and k not in _REPLACED_KEYS:
                raise ValueError("agent file: unknown key %s" % k)
        for k, spec in known.items():
            if k not in values:
                raise ValueError("agent file: %s is missing" % k)
            _check_value(k, spec, values[k])
        if agent_type == "AMP" and values["DiscNet"] != NETS[0]:
            raise ValueError("agent file: DiscNet %r is not supported (supported: %s)" % (values["DiscNet"], NETS[0]))
        self.values = values
        self.amp = agent_type == "AMP"

    @classmethod
    def from_json(cls, path):
        import json
        with open(path) as f:
            return cls(json.load(f))

    def __getitem__(self, key):
        v = self.values[key]
        spec = dict(_PPO_KEYS, **_AMP_KEYS)[key]
        return int(v) if spec[0] == "int" else v


# ---- the loop
def _store_rows(buf, rows):
    """rows into a DeviceReplayBuffer in order, in stores smaller than its capacity"""
    step = buf.capacity - 1
    for i in range(0, rows.shape[0], step):
        buf.store(rows[i:i + step])


_NORM_FIELDS = ("mean", "mean_sq", "std", "new_sum", "new_sum_sq")
PUSH_SCHEDULE_KEYS = ("bodies", "force", "duration", "gap")


def push_schedule_record(ps):
    """a push schedule dict(bodies, force, duration, gap) in the run record's form: bodies a list of ints, the other three [lo, hi] lists of
    floats.  Only the form is checked here; the library refuses out-of-range values by name (DeepMimicBatchEnv.set_push_schedule)."""
    if ps is None:
        return None
    if not isinstance(ps, dict) or set(ps) != set(PUSH_SCHEDULE_KEYS):
        raise ValueError("push_schedule: a dict with exactly the keys %s expected" % ", ".join(PUSH_SCHEDULE_KEYS))
    out = dict(bodies=[int(b) for b in ps["bodies"]])
    for k in PUSH_SCHEDULE_KEYS[1:]:
        v = [float(x) for x in ps[k]]
        if len(v) != 2:
            raise ValueError("push_schedule: %s must be a (lo, hi) pair" % k)
        out[k] = v
    return out


DYNAMICS_KINDS = ("friction", "kp", "kd", "torque_limit", "mass")


def dynamics_record(dr):
    """a dynamics randomisation dict(friction=(lo, hi), kp=..., kd=..., torque_limit=..., mass=...) in the run record's form: every kind a
    [lo, hi] list of floats, an omitted kind [1, 1].  Only the form is checked here; the library refuses out-of-range bounds by name
    (DeepMimicBatchEnv.set_dynamics_randomization)."""
    if dr is None:
        return None
    if not isinstance(dr, dict) or not set(dr) <= set(DYNAMICS_KINDS):
        raise ValueError("dynamics_randomization: a dict with keys among %s expected" % ", ".join(DYNAMICS_KINDS))
    out = {}
    for k in DYNAMICS_KINDS:
        v = [float(x) for x in dr.get(k, (1.0, 1.0))]
        if len(v) != 2:
            raise ValueError("dynamics_randomization: %s must be a (lo, hi) pair" % k)
        out[k] = v
    return out


def latency_record(lr):
    """a latency randomisation (lo_s, hi_s) in the run record's form: [lo, hi] in seconds, each rounded to a whole update
    (DeepMimicBatchEnv.set_action_latency_randomization).  Refused unless both lie in [0, (updates_per_action - 1) UPDATE_DT] after rounding and
    lo <= hi."""
    from .capi import UPDATE_DT, UPDATES_PER_ACTION, latency_updates
    if lr is None:
        return None
    v = list(lr)
    if len(v) != 2:
        raise ValueError("latency_randomization: a (lo, hi) pair in seconds expected")
    d = [latency_updates(x, UPDATES_PER_ACTION, "latency_randomization") for x in v]
    if d[0] > d[1]:
        raise ValueError("latency_randomization: lo %r s > hi %r s" % (v[0], v[1]))
    return [x * UPDATE_DT for x in d]


class Trainer:
    """RLAgent's training loop over one batched environment (a reading of the reference, not checked against its source).

    Trainer(args, config, asset_root, num_envs, ...) builds the env (seed), the rollout on `backend` with the actor, the critic and, for an AMP
    agent, the discriminator (random initialisation under torch.manual_seed(seed)), PPOLearner and AMPDiscLearner, the two disc buffers, and the
    evaluation handle: TestEpisodes environments in test mode whose start state is saved once and restored before every evaluation, so that
    Test_Return depends on the weights alone.  iteration() runs one iteration and returns its log row; log_path (optional) receives the rows
    as a formats.TableLog (append=True continues an existing log).  state_dict() / load_state_dict() hold everything the following iterations
    read, so a run resumed from a checkpoint continues bit for bit.  env and test_env replace the two handles (tests drive the loop's
    bookkeeping with stand-ins on the CPU).

    model_files (--model_files): a reference TensorBundle prefix or a Trainer checkpoint (deepmimic_b200/model_files.py) whose actor, critic,
    discriminator (a Trainer checkpoint's, for an AMP agent) and normalisers replace the random initialisation.  The run still starts at
    iteration 0 with zero momentum and freshly seeded generators; the loaded normalisers keep their statistics and count (NormalizerSamples
    when the file has no count).  What the file lacks stays as initialised and is listed in model_notes.  The path joins the run record that
    load_state_dict compares: a run started from model files resumes with the same model_files (and arguments).

    Host synchronisations: none per policy step; per iteration a fixed number, independent of window_steps, of the minibatch and discriminator
    step counts (tools/train_time.py counts them).  With a process group of more than one rank, each PPO update adds one (the learners' check
    that every rank's window has the same size).

    push_schedule (train --push_force etc.): dict(bodies, force, duration, gap) of DeepMimicBatchEnv.set_push_schedule, applied to the training
    handle only (Test_Return stays an evaluation without pushes).  It joins the run record, so a checkpoint resumes only with the same schedule;
    the training handle's state blob carries the pushes drawn so far.

    dynamics_randomization (train --rand_friction etc.): dict of (lo, hi) per kind of DeepMimicBatchEnv.set_dynamics_randomization, applied to
    the training handle only (Test_Return stays an evaluation on the nominal model).  It joins the run record, so a checkpoint resumes only with
    the same bounds; the training handle's state blob carries the factors.

    latency_randomization (train --rand_latency): (lo, hi) seconds of DeepMimicBatchEnv.set_action_latency_randomization, applied to the
    training handle only (Test_Return stays an evaluation without delay).  It joins the run record, rounded to whole updates, so a checkpoint
    resumes only with the same bounds; the training handle's state blob carries the delays and pending actions.

    Several GPUs (mpi_run.py --num_workers N): process_group, a torch.distributed group of one rank per GPU.  num_envs is the job's total, which
    must be divisible by the world size; each rank steps its contiguous share (global_env_offset = rank * num_envs / world, so every
    environment's reset stream is the one it has on one GPU), and evaluates ceil(TestEpisodes / world) episodes.  The learners average the
    ranks' gradients (PPOLearner, AMPDiscLearner with the same group); the rollout, learner and disc-buffer generators are seeded with
    seed + 1000 rank, and the expert sampler of rank r starts at call count r 2^40, so the ranks' exploration, minibatches and expert rows
    differ.  The normalisers' statistics, the sample count, the finished episodes' returns and the evaluation's returns and episode counts are
    summed over the ranks, so every rank logs the same row; only the first rank writes the log.  The disc buffers stay per rank (the
    reference's per-worker buffers).  Each rank's state_dict() is its own (simulation state, generators, buffers); its run record holds the
    world size and the state its rank, both of which load_state_dict() requires to match."""

    def __init__(self, args, config, asset_root, num_envs, window_steps=32, backend="tensor_core", seed=0, device=0, log_path=None, append_log=False,
                 env=None, test_env=None, process_group=None, model_files=None, push_schedule=None,
                 dynamics_randomization=None, latency_randomization=None):
        import torch
        from .env import DeepMimicBatchEnv
        from .learner import AMPDiscLearner, DataParallel, PPOLearner
        from .rollout import BatchedRollout, build_critic, build_discriminator, build_gated_policy, build_policy
        self.torch = torch
        if not isinstance(config, AgentConfig):
            raise ValueError("config must be an AgentConfig")
        if window_steps < 1 or num_envs < 1:
            raise ValueError("num_envs and window_steps must be positive")
        self.dp = DataParallel.of(process_group)
        self.world = self.dp.world if self.dp else 1
        self.rank = self.dp.dist.get_rank(process_group) if self.dp else 0
        if num_envs % self.world:
            raise ValueError("num_envs (%d, the job's total) must be divisible by the world size (%d)" % (num_envs, self.world))
        local = num_envs // self.world
        self.args, self.config, self.backend, self.seed = list(args), config, backend, int(seed)
        self.window_steps = int(window_steps)
        # what a checkpoint must match
        self.run = dict(args=self.args, agent=config.values, num_envs=int(num_envs), window_steps=self.window_steps, backend=backend, seed=self.seed,
                        world=self.world, model_files=model_files)
        push_schedule = push_schedule_record(push_schedule)
        if push_schedule is not None:   # runs without a schedule keep the record they had
            self.run["push_schedule"] = push_schedule
        dynamics_randomization = dynamics_record(dynamics_randomization)
        if dynamics_randomization is not None:   # runs without randomised dynamics keep the record they had
            self.run["dynamics_randomization"] = dynamics_randomization
        latency_randomization = latency_record(latency_randomization)
        if latency_randomization is not None:   # runs without latency keep the record they had
            self.run["latency_randomization"] = latency_randomization
        rs = self.seed + 1000 * self.rank   # the rank's generators
        cfg = config
        self.env = env = env or DeepMimicBatchEnv(self.args, local, asset_root, device=device, seed=self.seed, global_env_offset=self.rank * local)
        if env.num_envs != local:
            raise ValueError("env has %d environments; this rank's share of num_envs is %d" % (env.num_envs, local))
        if push_schedule is not None:
            env.set_push_schedule(**push_schedule)
        if dynamics_randomization is not None:
            env.set_dynamics_randomization(**dynamics_randomization)
        if latency_randomization is not None:
            env.set_action_latency_randomization(*latency_randomization)
        S, A, G = env.get_state_size(), env.get_action_size(), env.get_goal_size()
        net = NETS[1] if G > 0 else NETS[0]
        for key in ("ActorNet", "CriticNet"):
            if cfg[key] != net:
                raise ValueError("agent file: %s %s does not fit scene %r, which needs %s" % (key, cfg[key], env.get_name(), net))
        self.amp = cfg.amp
        noise = float(cfg["ExpParamsBeg"].get("Noise", 0.0))
        if not noise > 0.0:
            raise ValueError("agent file: ExpParamsBeg.Noise, the actor's standard deviation, must be positive")
        torch.manual_seed(self.seed)
        scale = cfg["ActorInitOutputScale"]
        policy = build_gated_policy(S, G, A, init_output_scale=scale, noise=noise) if G > 0 else build_policy(S, A, init_output_scale=scale, noise=noise)
        critic = build_critic(S, G)
        disc = build_discriminator(env.get_amp_obs_size(), init_output_scale=cfg["DiscInitOutputScale"]) if self.amp else None
        self.ro = BatchedRollout(env, policy, exp_rate=cfg["ExpParamsBeg"]["Rate"], noise=noise, seed=rs, backend=backend, disc=disc,
                                 task_reward_lerp=cfg["TaskRewardLerp"] if self.amp else None, critic=critic, discount=cfg["Discount"],
                                 td_lambda=cfg["TDLambda"])
        self.model_notes = []
        if model_files is not None:
            # before the learners take the parameters; a normaliser without a count in the file counts NormalizerSamples samples, so the
            # first windows' statistics are weighed against it rather than replacing it (a reading of RLAgent.load_model that has not been
            # checked against the reference's source)
            from .model_files import load_model_files
            loaded = load_model_files(model_files, policy, self._all_norms(), critic=self.ro.critic, disc=self.ro.disc)
            for name, count in loaded["counts"].items():
                self._all_norms()[name].count = cfg["NormalizerSamples"] if count is None else count
            self.model_notes = loaded["notes"]
        self.ppo = PPOLearner(self.ro, actor_stepsize=cfg["ActorStepsize"], actor_momentum=cfg["ActorMomentum"], actor_weight_decay=cfg["ActorWeightDecay"],
                              critic_stepsize=cfg["CriticStepsize"], critic_momentum=cfg["CriticMomentum"], critic_weight_decay=cfg["CriticWeightDecay"],
                              ratio_clip=cfg["RatioClip"], norm_adv_clip=cfg["NormAdvClip"], minibatch_size=cfg["MiniBatchSize"], epochs=cfg["Epochs"],
                              backend=backend, seed=rs + 1, process_group=process_group)
        self.disc = self.agent_buf = self.expert_buf = None
        if self.amp:
            self.disc = AMPDiscLearner(self.ro, stepsize=cfg["DiscStepSize"], momentum=cfg["DiscMomentum"], weight_decay=cfg["DiscWeightDecay"],
                                       logit_reg_weight=cfg["DiscLogitRegWeight"], grad_penalty=cfg["DiscGradPenalty"], batch_size=cfg["DiscBatchSize"],
                                       steps=1, backend=backend, seed=rs + 2, process_group=process_group)
            M = env.get_amp_obs_size()
            self.agent_buf = DeviceReplayBuffer(cfg["DiscBufferSize"], M, env.device, seed=rs + 3)
            self.expert_buf = DeviceReplayBuffer(cfg["DiscBufferSize"], M, env.device, seed=rs + 4)
            if self.dp:
                env.expert_sample_count(self.rank << 40)
        # evaluation: a small handle in test mode, restored to its start state before every evaluation
        te = -(-cfg["TestEpisodes"] // self.world)
        self.test_env = test_env or DeepMimicBatchEnv(self.args, te, asset_root, device=device, seed=self.seed, global_env_offset=self.rank * te)
        self.test_env.set_mode(1)
        self.test_env.reset(True)
        self._test_start = self.test_env.state_dict()
        self.test_ro = BatchedRollout(self.test_env, policy, exp_rate=0.0, noise=noise, seed=rs, backend=backend)
        self.test_ro.s_norm, self.test_ro.a_norm = self.ro.s_norm, self.ro.a_norm
        if G > 0:
            self.test_ro.g_norm = self.ro.g_norm
        # the loop's own state
        self.iter, self.total_samples = 0, 0
        self.initialized, self.need_normalizer_update = False, True
        self.test_return = float("nan")
        self.ep_ret = torch.zeros(env.num_envs, device=env.device)
        self.ep_len = torch.zeros(env.num_envs, device=env.device)
        self.phase_hook = None   # tools/train_time.py: phase_hook(name) -> context manager around each phase
        self.log = None
        if log_path is not None and self.rank == 0:
            from .formats import TableLog
            self.log = TableLog(log_path, append=append_log)

    # ---- normalisers: the ones the normaliser phase updates, and every one a checkpoint holds
    def _updated_norms(self):
        ro = self.ro
        return [ro.s_norm] + ([ro.g_norm] if ro.goal_size > 0 else []) + ([ro.amp_norm] if self.amp else [])

    def _all_norms(self):
        ro = self.ro
        n = dict(s_norm=ro.s_norm, a_norm=ro.a_norm, val_norm=ro.val_norm)
        if ro.goal_size > 0:
            n["g_norm"] = ro.g_norm
        if self.amp:
            n["amp_norm"] = ro.amp_norm
        return n

    def _phase(self, name):
        from .rollout import _nullcontext
        return self.phase_hook(name) if self.phase_hook is not None else _nullcontext()

    def _episode_sums(self, traj):
        """[returns of the episodes that ended in the window, their lengths in policy steps, their count] as a device tensor; the per-env
        accumulators carry the running episodes into the next window"""
        t = self.torch
        sums = t.zeros(3, device=self.env.device)
        for r, d in zip(traj["rewards"], traj["dones"]):
            self.ep_ret += r
            self.ep_len += 1.0
            df = d.float()
            sums += t.stack([(self.ep_ret * df).sum(), (self.ep_len * df).sum(), df.sum()])
            keep = 1.0 - df
            self.ep_ret *= keep
            self.ep_len *= keep
        return self.dp.sum(sums) if self.dp else sums

    def iteration(self):
        """one iteration of the loop; returns its log row (a dict)"""
        import time
        t, cfg, ro, env = self.torch, self.config, self.ro, self.env
        T, N = self.window_steps, env.num_envs
        t0 = time.time()
        ro.exp_rate = exploration_params(cfg["ExpParamsBeg"], cfg["ExpParamsEnd"], self.total_samples, cfg["ExpAnnealSamples"])["Rate"]
        with self._phase("collect"):
            traj = ro.collect(T, record_stats=self.need_normalizer_update)
            ep = self._episode_sums(traj)
        self.total_samples += T * N * self.world
        env.set_sample_count(self.total_samples)
        train, self.initialized, update_norms, self.need_normalizer_update = train_schedule(
            self.total_samples, self.initialized, self.need_normalizer_update, cfg["InitSamples"], cfg["NormalizerSamples"])
        zero = t.zeros((), device=env.device)
        s_ppo = dict(actor_loss=zero, critic_loss=zero, clip_frac=zero, adv_mean=zero, adv_std=zero)
        s_disc = dict(disc_loss=zero, grad_penalty=zero, acc_expert=zero, acc_agent=zero, logit_expert=zero, logit_agent=zero)
        if self.amp:
            with self._phase("store"):
                for k in range(T):
                    _store_rows(self.agent_buf, traj["amp_obs"][k])
                _store_rows(self.expert_buf, env.sample_amp_obs_expert(T * N))
        if train:
            if self.amp:
                with self._phase("disc_update"):
                    self.disc.steps = disc_steps_per_iter(T * N * self.world, cfg["DiscStepsPerBatch"], cfg["DiscBatchSize"])
                    s_disc = self.disc.update(self.agent_buf.filled(), self.expert_buf.filled())
            with self._phase("ppo_update"):
                s_ppo = self.ppo.update(traj)
                clip_frac = s_ppo["clip_frac"].item()
                self.ppo.actor_stepsize = update_actor_stepsize(self.ppo.actor_stepsize, clip_frac, cfg["TarClipFrac"], cfg["ActorStepsizeDecay"], self.iter)
        if update_norms:
            with self._phase("normalizers"):
                for n in self._updated_norms():
                    n.update(all_reduce=self.dp.sum if self.dp else None)
                # the rollout's tensor-core handles act on the new statistics from the next collect() on, as the torch backend does
                ro.retile_tensor_core("actor", "critic", "disc")
        it = self.iter
        self.iter += 1
        if it % cfg["OutputIters"] == 0:
            with self._phase("evaluation"):
                self.test_return = self.evaluate()
        # the row: one host read of every device statistic
        names = ["Actor_Loss", "Critic_Loss", "Clip_Frac", "Adv_Mean", "Adv_Std"]
        vals = [s_ppo[k] for k in ("actor_loss", "critic_loss", "clip_frac", "adv_mean", "adv_std")]
        if self.amp:
            names += ["Disc_Loss", "Disc_Grad_Penalty", "Disc_Acc_Expert", "Disc_Acc_Agent", "Disc_Logit_Expert", "Disc_Logit_Agent"]
            vals += [s_disc[k] for k in ("disc_loss", "grad_penalty", "acc_expert", "acc_agent", "logit_expert", "logit_agent")]
        for label, n in (("State", ro.s_norm), ("Goal", getattr(ro, "g_norm", None) if ro.goal_size else None), ("AMP_Obs", ro.amp_norm if self.amp else None)):
            if n is not None:
                names += [label + "_Mean", label + "_Std"]
                vals += [n.mean.mean(), n.std.mean()]
        host = t.stack([v.float().reshape(()) for v in vals] + list(ep)).tolist()
        ended = host[-1]
        row = dict(Iteration=it, Wall_Time=time.time() - t0, Samples=self.total_samples,
                   Train_Return=host[-3] / ended if ended else float("nan"), Train_Path_Len=host[-2] / ended if ended else float("nan"),
                   Test_Return=self.test_return, Exp_Rate=ro.exp_rate, Actor_Stepsize=self.ppo.actor_stepsize)
        row.update(zip(names, host[:len(names)]))
        if self.log is not None:
            for k, v in row.items():
                self.log.log_tabular(k, v)
            self.log.dump_tabular()
        return row

    def evaluate(self):
        """Test_Return: the mean return of one complete episode of each evaluation environment (test mode, exploration off), from the start
        state the evaluation handle had when it was created; with several ranks, the sum of every rank's returns over their number of episodes.
        One host synchronisation per 32 policy steps."""
        from .rollout import run_episodes
        t, env, ro = self.torch, self.test_env, self.test_ro
        env.load_state_dict(self._test_start)
        ro.gen.manual_seed(self.seed + 1000 * self.rank)
        if self.backend == "tensor_core":
            ro.refresh_tensor_core_policy()
        try:
            ret = run_episodes(ro)["returns"]
        except RuntimeError as e:
            raise RuntimeError("evaluation: %s" % e) from None
        if not self.dp:
            return ret.mean().item()
        s = self.dp.sum(t.stack([ret.sum(), t.tensor(float(env.num_envs), device=env.device)])).tolist()
        return s[0] / s[1]

    # ---- checkpoints
    def state_dict(self):
        """everything the following iterations read: the run's settings, the counters and schedule flags, the actor stepsize, the networks and
        both learners' momentum accumulators, every normaliser, every generator, both disc buffers, the episode accumulators and the training
        handle's simulation state.  Tensors and Python values only (torch.load(weights_only=True) reads it)."""
        t, ro = self.torch, self.ro
        c = lambda x: x.detach().clone()
        nets = dict(actor={k: c(v) for k, v in ro.policy.state_dict().items()}, critic={k: c(v) for k, v in ro.critic.state_dict().items()})
        accs = dict(ppo=[c(self.ppo.acc[p]) for p in self.ppo.actor_params + self.ppo.critic_params])
        gens = dict(rollout=ro.gen.get_state(), ppo=self.ppo.gen.get_state())
        bufs = {}
        if self.amp:
            nets["disc"] = {k: c(v) for k, v in ro.disc.state_dict().items()}
            accs["disc"] = [c(self.disc.acc[p]) for p in self.disc.params]
            gens["disc"] = self.disc.gen.get_state()
            bufs = dict(agent=self.agent_buf.state_dict(), expert=self.expert_buf.state_dict())
        norms = {name: dict({f: c(getattr(n, f)) for f in _NORM_FIELDS}, count=n.count, new_count=n.new_count) for name, n in self._all_norms().items()}
        return dict(run=self.run, rank=self.rank, iteration=self.iter, samples=self.total_samples, initialized=self.initialized,
                    need_normalizer_update=self.need_normalizer_update, actor_stepsize=self.ppo.actor_stepsize, test_return=self.test_return,
                    nets=nets, accs=accs, norms=norms, generators=gens, buffers=bufs, episodes=dict(ret=c(self.ep_ret), len=c(self.ep_len)),
                    env=self.env.state_dict())

    def load_state_dict(self, s):
        """restores state_dict() of a run with the same settings (arguments, agent file, num_envs, window_steps, backend, seed; a difference
        is refused).  Parameters and accumulators are loaded in place (the tensor-core learners hold their addresses); the rollout's
        tensor-core handles are rebuilt from the loaded weights and normalisers."""
        t, ro = self.torch, self.ro
        if s["run"].get("model_files") != self.run["model_files"]:   # a checkpoint without the key is a run from random initialisation
            raise ValueError("checkpoint: its run started from model files %s, this one from %s: resume with the arguments the run started with, "
                             "--model_files included" % (s["run"].get("model_files"), self.run["model_files"]))
        if s["run"].get("push_schedule") != self.run.get("push_schedule"):   # a checkpoint without the key is a run without pushes
            raise ValueError("checkpoint: its run trained under the push schedule %s, this one under %s: resume with the push options the run "
                             "started with" % (s["run"].get("push_schedule"), self.run.get("push_schedule")))
        if s["run"].get("dynamics_randomization") != self.run.get("dynamics_randomization"):   # a checkpoint without the key is a nominal run
            raise ValueError("checkpoint: its run trained under the dynamics randomisation %s, this one under %s: resume with the --rand_* "
                             "options the run started with" % (s["run"].get("dynamics_randomization"), self.run.get("dynamics_randomization")))
        if s["run"].get("latency_randomization") != self.run.get("latency_randomization"):   # a checkpoint without the key is a run without delay
            raise ValueError("checkpoint: its run trained under the latency randomisation %s, this one under %s: resume with the --rand_latency "
                             "option the run started with" % (s["run"].get("latency_randomization"), self.run.get("latency_randomization")))
        for k in self.run:
            if s["run"].get(k, 1 if k == "world" else None) != self.run[k]:   # a checkpoint without a world size is a one-rank run's
                raise ValueError("checkpoint: its %s differs from this run's" % ("agent file" if k == "agent" else "world size" if k == "world" else k))
        if s.get("rank", 0) != self.rank:
            raise ValueError("checkpoint: it is rank %d's, not this rank's (%d)" % (s.get("rank", 0), self.rank))
        with t.no_grad():
            for name, net in (("actor", ro.policy), ("critic", ro.critic)) + ((("disc", ro.disc),) if self.amp else ()):
                for k, v in net.state_dict().items():
                    v.copy_(s["nets"][name][k])
            for p, a in zip(self.ppo.actor_params + self.ppo.critic_params, s["accs"]["ppo"]):
                self.ppo.acc[p].copy_(a)
            if self.amp:
                for p, a in zip(self.disc.params, s["accs"]["disc"]):
                    self.disc.acc[p].copy_(a)
        for name, n in self._all_norms().items():
            d = s["norms"][name]
            for f in _NORM_FIELDS:
                setattr(n, f, d[f].to(n.mean.device).clone())
            n.count, n.new_count = int(d["count"]), int(d["new_count"])
        ro.gen.set_state(s["generators"]["rollout"])
        self.ppo.gen.set_state(s["generators"]["ppo"])
        if self.amp:
            self.disc.gen.set_state(s["generators"]["disc"])
            self.agent_buf.load_state_dict(s["buffers"]["agent"])
            self.expert_buf.load_state_dict(s["buffers"]["expert"])
        self.ep_ret.copy_(s["episodes"]["ret"])
        self.ep_len.copy_(s["episodes"]["len"])
        self.env.load_state_dict(s["env"])
        self.iter, self.total_samples = int(s["iteration"]), int(s["samples"])
        self.initialized, self.need_normalizer_update = bool(s["initialized"]), bool(s["need_normalizer_update"])
        self.ppo.actor_stepsize, self.test_return = float(s["actor_stepsize"]), float(s["test_return"])
        if self.backend == "tensor_core":
            ro.refresh_tensor_core_policy()

    def save(self, path):
        """state_dict() to path (torch.save), through a temporary file so that an interrupted write leaves the previous checkpoint"""
        import os
        tmp = path + ".tmp"
        self.torch.save(self.state_dict(), tmp)
        os.replace(tmp, path)

    def load(self, path):
        self.load_state_dict(self.torch.load(path, map_location="cpu", weights_only=True))

    def close(self):
        if self.log is not None:
            self.log.close()
            self.log = None
