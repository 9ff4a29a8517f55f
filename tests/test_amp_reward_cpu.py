"""CPU tests of the AMP discriminator's reward in the rollout shim: the torch discriminator against a numpy restatement of the reference's
network (R/learning/amp_agent.py: fc_2layers_1024units trunk, one-unit logit), the least-squares style reward of Peng et al. 2021 (eq. 7) at known
answers, its blend with the task reward, and BatchedRollout.collect's recording of the agent's AMP observations on a CPU stand-in env."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
from deepmimic_b200.rollout import BatchedRollout, amp_rewards, build_discriminator, load_disc_weights
from tests.test_rollout_cpu import _FakeEnv


def _random_disc(rng, m, hidden):
    dims = [m] + list(hidden)
    wb = lambda a, b: (rng.standard_normal((a, b)) / np.sqrt(a), 0.1 * rng.standard_normal(b))
    return dict(hidden=[wb(a, b) for a, b in zip(dims[:-1], dims[1:])], logit=wb(dims[-1], 1))


def test_discriminator_matches_numpy_restatement():
    rng = np.random.default_rng(3)
    d = _random_disc(rng, 20, (32, 16))
    disc = load_disc_weights(build_discriminator(20, hidden=(32, 16)), d).double()
    x = rng.standard_normal((7, 20))
    h = x
    for w, b in d["hidden"]:
        h = np.maximum(h @ w + b, 0.0)
    want = h @ d["logit"][0] + d["logit"][1]
    with torch.no_grad():
        got = disc(torch.as_tensor(x)).numpy()
    assert got.shape == (7, 1)
    np.testing.assert_allclose(got, want, atol=1e-12)
    # default shape: the actor's 1024-512 trunk; the logit weights are uniform in [-init_output_scale, init_output_scale], biases zero
    torch.manual_seed(0)
    full = build_discriminator(226, init_output_scale=0.5)
    assert [l.weight.shape for l in full.hidden] == [(1024, 226), (512, 1024)] and full.logit.weight.shape == (1, 512)
    assert float(full.logit.weight.detach().abs().max()) <= 0.5 and float(full.logit.bias.detach().abs().max()) == 0.0
    with pytest.raises(ValueError, match="hidden layers"):
        load_disc_weights(full, d | dict(hidden=d["hidden"][:1]))


def test_style_reward_known_answers_and_blend():
    d = torch.tensor([1.0, 0.0, 2.0, -1.0, 3.0, 5.0, -7.0])
    style, reward = amp_rewards(d)
    assert style.tolist() == [1.0, 0.75, 0.75, 0.0, 0.0, 0.0, 0.0] and torch.equal(reward, style)   # clamped at 0 beyond |1 - d| = 2
    task = torch.tensor([0.2, 0.9, 0.0, 1.0, 0.5, 0.3, 0.7])
    for lerp in (0.0, 0.5, 1.0):
        s, r = amp_rewards(d, task, lerp)
        assert torch.equal(s, style)
        torch.testing.assert_close(r, (1.0 - lerp) * style + lerp * task, rtol=0, atol=1e-7)
    assert torch.equal(amp_rewards(d, task, 0.0)[1], style) and torch.equal(amp_rewards(d, task, 1.0)[1], task)


class _FakeAMPEnv(_FakeEnv):
    """_FakeEnv with the AMP surface: the agent's AMP observation encodes the episode clock, so an observation taken after the reset (clock 0)
    is told apart from the finished episode's last one"""
    M = 6

    def __init__(self, n, goal_size, name):
        super().__init__(n, goal_size)
        self.name = name

    def get_name(self): return self.name
    def enable_amp_task_reward(self): return self.G > 0
    def get_amp_obs_size(self): return self.M
    def get_amp_obs_offset(self): return np.full(self.M, -0.5)
    def get_amp_obs_scale(self): return np.full(self.M, 2.0)
    def get_amp_obs_norm_group(self): return np.zeros(self.M, dtype=np.int32)

    def record_amp_obs_agent(self, agent_id=0):
        return self.t[:, None] * self.torch.linspace(1.0, 2.0, self.M)[None, :] - 1.0


@pytest.mark.parametrize("goal_size,name,lerp", [(0, "Imitate AMP", None), (3, "Target AMP", 0.5)])
def test_collect_records_the_agent_amp_obs_before_the_reset(goal_size, name, lerp):
    torch.manual_seed(0)
    env = _FakeAMPEnv(4, goal_size, name)
    disc = build_discriminator(_FakeAMPEnv.M, hidden=(16, 8))
    ro = BatchedRollout(env, exp_rate=0.0, seed=1, disc=disc, task_reward_lerp=lerp)
    traj = ro.collect(9, record_stats=True)
    assert traj["amp_obs"].shape == (9, 4, 6) and all(traj[k].shape == (9, 4) for k in ("disc_logits", "style_rewards", "amp_rewards"))
    # env 0's episodes last 3 steps (done at k = 2, 5, 8), env 1's 4 (k = 3, 7): the last transition carries the finished episode's clock
    clock = traj["amp_obs"][:, :, 0] + 1.0
    assert clock[:, 0].tolist() == [1, 2, 3] * 3 and clock[:, 1].tolist() == [1, 2, 3, 4, 1, 2, 3, 4, 1]
    assert ro.amp_norm.new_count == 9 * 4                                  # record_stats folds the AMP observations into amp_norm
    torch.testing.assert_close(ro.amp_norm.mean, torch.full((6,), 0.5))   # mean = -offset, std = 1 / scale
    with torch.no_grad():
        d = disc(ro.amp_norm.normalize(traj["amp_obs"]))[..., 0]
    torch.testing.assert_close(traj["disc_logits"], d)
    style, reward = amp_rewards(d, traj["rewards"] if goal_size else None, lerp or 0.0)
    torch.testing.assert_close(traj["style_rewards"], style)
    torch.testing.assert_close(traj["amp_rewards"], reward)
    if goal_size:
        assert not torch.equal(traj["amp_rewards"], traj["style_rewards"])
    else:
        assert torch.equal(traj["amp_rewards"], traj["style_rewards"])     # imitate_amp trains on the style reward alone


def test_collect_without_disc_and_refusals():
    env = _FakeAMPEnv(4, 0, "Imitate AMP")
    traj = BatchedRollout(env, exp_rate=0.0).collect(3, record_stats=False)
    assert not {"amp_obs", "disc_logits", "style_rewards", "amp_rewards"} & set(traj)
    disc = build_discriminator(_FakeAMPEnv.M, hidden=(16, 8))
    with pytest.raises(ValueError, match="AMP scene"):
        BatchedRollout(_FakeAMPEnv(4, 0, "Imitate"), disc=disc)
    for bad in (None, 1.5, -0.1):
        with pytest.raises(ValueError, match="task_reward_lerp"):
            BatchedRollout(_FakeAMPEnv(4, 3, "Target AMP"), disc=disc, task_reward_lerp=bad)
    with pytest.raises(ValueError, match="no AMP task reward"):
        BatchedRollout(_FakeAMPEnv(4, 0, "Imitate AMP"), disc=disc, task_reward_lerp=0.3)
