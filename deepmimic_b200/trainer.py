"""Pieces of the reference agent's training iteration (R/learning/rl_agent.py: RLAgent._train, _update_exp_params; ppo_agent.py:
PPOAgent.update_actor_stepsize; amp_agent.py: AMPAgent._update_disc and its replay buffers, replay_buffer_rand_storage.py) that sit between
BatchedRollout.collect, PPOLearner.update and AMPDiscLearner.update.

The reference tree is not vendored here; each rule is restated below as one function with the reading it follows, and tests/test_trainer_cpu.py
pins it against a numpy restatement.  These are readings of the reference that could not be checked against its source here; where they and the
reference disagree, the reference is right.

  DeviceReplayBuffer   ReplayBufferRandStorage on a torch device tensor: the AMP agent's two disc buffers (agent and expert observations)
  update_actor_stepsize, disc_steps_per_iter, exploration_params, train_schedule   the iteration's schedules"""
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
