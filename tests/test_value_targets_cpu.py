"""CPU tests of the PPO value targets of the rollout shim: a numpy restatement of the reference's return computation (R/learning/rl_util.py:
compute_return, applied path by path with PPOAgent._compute_batch_vals's terminal values) at hand-computed answers, the value normaliser and
terminal values (PGAgent._calc_val_offset_scale, RLAgent._calc_term_vals), the critic (PPOAgent._build_net_critic) against numpy, the
checkpoint reader's critic, and BatchedRollout.collect's critic values on a CPU stand-in env."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
from deepmimic_b200.rollout import (BatchedRollout, build_critic, load_critic_weights, td_lambda_returns_host, terminal_values,
                                    val_norm_from_rewards)
from tests.test_rollout_cpu import _FakeEnv

FAIL, SUCC = 1, 2


def compute_return(rewards, gamma, td_lambda, val_t):
    """rl_util.compute_return: the TD(lambda) return of one path; val_t has one more entry than rewards (the value of the path's end)"""
    ret = [0.0] * len(rewards)
    ret[-1] = rewards[-1] + gamma * val_t[-1]
    for i in reversed(range(len(rewards) - 1)):
        ret[i] = rewards[i] + gamma * ((1.0 - td_lambda) * val_t[i + 1] + td_lambda * ret[i + 1])
    return ret


def path_returns(r, v, ev, done, term, gamma, td_lambda, val_fail, val_succ):
    """[T, N] returns, path by path: each environment's column is split after every done step; a path's end value is val_fail / val_succ at a
    Fail / Succ end and the critic's value of the state it ended in (end_values) at a Null end or where the window cuts it at step T - 1; the
    values inside a path are the critic's values of its states"""
    r, v, ev, done, term = (np.asarray(x).tolist() for x in (r, v, ev, done, term))
    T, N = len(r), len(r[0])
    out = np.zeros((T, N))
    for n in range(N):
        a = 0
        while a < T:
            b = a
            while b < T - 1 and not done[b][n]:
                b += 1
            end = ev[b][n]
            if done[b][n] and term[b][n] == FAIL:
                end = val_fail
            elif done[b][n] and term[b][n] == SUCC:
                end = val_succ
            out[a:b + 1, n] = compute_return([r[k][n] for k in range(a, b + 1)], gamma, td_lambda, [v[k][n] for k in range(a, b + 1)] + [end])
            a = b + 1
    return out


def synthetic_window(rng, T, N, p_done=0.05):
    """random rewards / values / flags with all three terminate codes; end_values[k] = values[k + 1] where the path goes on, as collect() records"""
    r = rng.random((T, N)).astype(np.float32)
    v = (20.0 * rng.random((T, N))).astype(np.float32)
    done = rng.random((T, N)) < p_done
    term = np.where(done, rng.integers(0, 3, (T, N)), 0).astype(np.int32)
    ev = (20.0 * rng.random((T, N))).astype(np.float32)
    ev[:-1] = np.where(done[:-1], ev[:-1], v[1:])
    return r, v, ev, done, term


def _one(T, r, v, ev, done, term, gamma, lam, vf=0.0, vs=2.0):
    col = lambda x, dt=np.float32: np.asarray(x, dtype=dt).reshape(T, 1)
    return path_returns(col(r), col(v), col(ev), col(done, bool), col(term, np.int32), gamma, lam, vf, vs)[:, 0].tolist()


def test_restatement_at_hand_computed_answers():
    # constant reward 1 and V = 2 = 1 / (1 - 0.5) everywhere, no end: the fixed point, for every lambda
    for lam in (0.0, 0.5, 1.0):
        assert _one(3, [1, 1, 1], [2, 2, 2], [2, 2, 2], [0, 0, 0], [0, 0, 0], 0.5, lam) == [2.0, 2.0, 2.0]
    # a two-step path ending at step 1, lambda 1: Fail (val_fail 0), Succ (val_succ 2), Null (end value 4)
    assert _one(2, [1, 1], [9, 9], [9, 4], [0, 1], [0, FAIL], 0.5, 1.0) == [1.5, 1.0]
    assert _one(2, [1, 1], [9, 9], [9, 4], [0, 1], [0, SUCC], 0.5, 1.0) == [2.0, 2.0]
    assert _one(2, [1, 1], [9, 9], [9, 4], [0, 1], [0, 0], 0.5, 1.0) == [2.5, 3.0]
    # lambda 0: one-step targets r + gamma V(s'); lambda 0.5 mixes them with the next return
    assert _one(2, [1, 1], [9, 3], [3, 4], [0, 0], [0, 0], 0.5, 0.0) == [2.5, 3.0]
    assert _one(2, [1, 1], [9, 3], [3, 4], [0, 0], [0, 0], 0.5, 0.5) == [1 + 0.5 * (0.5 * 3 + 0.5 * 3.0), 3.0]
    # gamma 0: the reward itself
    assert _one(3, [0.25, 0.5, 0.75], [9, 9, 9], [9, 9, 9], [1, 0, 0], [FAIL, 0, 0], 0.0, 0.95, 0.0, 0.0) == [0.25, 0.5, 0.75]
    # an episode ends at step 0 (Fail), the next one is cut by the window at step 2 and bootstrapped with end_values[2] = 6
    assert _one(3, [1, 1, 1], [9, 2, 2], [9, 2, 6], [1, 0, 0], [FAIL, 0, 0], 0.5, 1.0) == [1.0, 1 + 0.5 * 4.0, 4.0]


@pytest.mark.parametrize("gamma,lam", [(0.0, 0.95), (0.95, 0.0), (0.95, 0.95), (0.95, 1.0)])
def test_host_scan_matches_the_restatement(gamma, lam):
    """td_lambda_returns_host (the kernel's rule, one step at a time for all environments) against the path-by-path restatement"""
    rng = np.random.default_rng(int(100 * gamma + 10 * lam))
    r, v, ev, done, term = synthetic_window(rng, 50, 40, p_done=0.1)
    vf, vs = terminal_values(_RewardEnv(), gamma)
    want = path_returns(r, v, ev, done, term, gamma, lam, vf, vs)
    tt = lambda x: torch.as_tensor(x)
    ret, adv = torch.empty(50, 40), torch.empty(50, 40)
    td_lambda_returns_host(tt(r), tt(v), tt(ev), tt(done), tt(term), gamma, lam, vf, vs, ret, adv)
    bound = 1e-5 * max(1.0, 1.0 / (1.0 - gamma))
    assert np.abs(ret.numpy() - want).max() <= bound and np.abs(adv.numpy() - (want - v)).max() <= bound


class _RewardEnv:
    def get_reward_min(self, agent_id=0): return 0.0
    def get_reward_max(self, agent_id=0): return 1.0
    def get_reward_fail(self, agent_id=0): return 0.0
    def get_reward_succ(self, agent_id=0): return 1.0


def test_value_normaliser_and_terminal_values():
    n = val_norm_from_rewards(_RewardEnv(), 0.95)
    assert n.mean.tolist() == pytest.approx([10.0]) and n.std.tolist() == pytest.approx([10.0])
    assert terminal_values(_RewardEnv(), 0.95) == pytest.approx((0.0, 20.0))
    assert terminal_values(_RewardEnv(), 0.0) == (0.0, 0.0)
    torch.testing.assert_close(n.unnormalize(torch.tensor([-1.0, 0.0, 1.0])), torch.tensor([0.0, 10.0, 20.0]))


def _random_critic(rng, s, g, hidden=(32, 16), gc=8, gh=4):
    # float32-representable weights: the torch critic holds float32 parameters
    wb = lambda a, b: ((rng.standard_normal((a, b)) / np.sqrt(a)).astype(np.float32).astype(np.float64), (0.1 * rng.standard_normal(b)).astype(np.float32).astype(np.float64))
    dims = [s + g] + list(hidden)
    d = dict(hidden=[wb(a, b) for a, b in zip(dims[:-1], dims[1:])], out=wb(dims[-1], 1))
    if g:
        d["gate_common"] = wb(g, gc)
        d["gates"] = [dict(hidden=wb(gc, gh), bias=wb(gh, h), scale=wb(gh, h)) for h in hidden]
    return d


def _np_critic(d, s, g=None):
    relu = lambda x: np.maximum(x, 0.0)
    if g is None:
        h = s
        for w, b in d["hidden"]:
            h = relu(h @ w + b)
    else:
        gc = relu(g @ d["gate_common"][0] + d["gate_common"][1])
        h = np.concatenate([s, g], axis=1)
        for (w, b), gt in zip(d["hidden"], d["gates"]):
            gate = relu(gc @ gt["hidden"][0] + gt["hidden"][1])
            scale = 2.0 / (1.0 + np.exp(-(gate @ gt["scale"][0] + gt["scale"][1])))
            h = relu(scale * (h @ w + b) + gate @ gt["bias"][0] + gt["bias"][1])
    return h @ d["out"][0] + d["out"][1]


@pytest.mark.parametrize("goal_size", [0, 3])
def test_critic_matches_numpy_restatement(goal_size):
    rng = np.random.default_rng(goal_size)
    d = _random_critic(rng, 20, goal_size)
    c = load_critic_weights(build_critic(20, goal_size, hidden=(32, 16), gate_common=8, gate_hidden=4), d).double()
    s, g = rng.standard_normal((7, 20)), rng.standard_normal((7, goal_size))
    with torch.no_grad():
        got = (c(torch.as_tensor(s), torch.as_tensor(g)) if goal_size else c(torch.as_tensor(s))).numpy()
    assert got.shape == (7, 1)
    np.testing.assert_allclose(got, _np_critic(d, s, g if goal_size else None), atol=1e-12)
    # default shape: the actor's 1024-512 trunk (gated with a 128-unit gate trunk and 64-unit gate layers) and a one-unit output, xavier-uniform
    # weights and zero biases
    torch.manual_seed(0)
    full = build_critic(226, goal_size)
    assert [l.weight.shape for l in full.hidden] == [(1024, 226 + goal_size), (512, 1024)] and full.out.weight.shape == (1, 512)
    assert float(full.out.weight.detach().abs().max()) <= np.sqrt(6.0 / 513) and float(full.out.bias.detach().abs().max()) == 0.0
    assert hasattr(full, "gate_common") == (goal_size > 0)
    with pytest.raises(ValueError, match="hidden layers"):
        load_critic_weights(full, d | dict(hidden=d["hidden"][:1]))
    with pytest.raises(ValueError, match="goal-conditioned critic"):
        load_critic_weights(build_critic(20, 3 - goal_size, hidden=(32, 16)), d)


def test_checkpoint_reader_returns_the_critic(tmp_path):
    from deepmimic_b200.tf_checkpoint import load_critic
    from tests.test_tf_checkpoint_cpu import write_bundle
    rng = np.random.default_rng(1)
    d = _random_critic(rng, 6, 3, hidden=(5, 4), gc=8, gh=4)
    c, a = "agent/main/critic/", "agent/main/actor/"
    t = {}
    put = lambda name, wb: t.update({c + name + "/kernel": wb[0], c + name + "/bias": wb[1]})
    for i, wb in enumerate(d["hidden"]):
        put("%d/dense" % i, wb)
    put("dense", d["out"]); put("gate_common/0/dense", d["gate_common"])
    for i, gt in enumerate(d["gates"]):
        put("gate%d/0/dense" % i, gt["hidden"]); put("gate%d/dense" % i, gt["bias"]); put("gate%d/dense_1" % i, gt["scale"])
    t.update({a + "0/dense/kernel": rng.standard_normal((9, 5)), "agent/resource/val_norm/mean": np.array([10.0]), "agent/resource/val_norm/std": np.array([10.0]),
              "agent/resource/s_norm/mean": rng.standard_normal(6), "agent/resource/s_norm/std": rng.random(6) + 0.5})
    t = {k: np.asarray(v, dtype=np.float32) for k, v in t.items()}
    prefix = str(tmp_path / "ppo.ckpt")
    write_bundle(prefix, t)
    got = load_critic(prefix)
    assert [w.shape for w, _ in got["hidden"]] == [(9, 5), (5, 4)] and got["out"][0].shape == (4, 1) and got["gate_common"][0].shape == (3, 8)
    assert np.array_equal(got["gates"][1]["scale"][0], t[c + "gate1/dense_1/kernel"]) and np.array_equal(got["gates"][0]["bias"][1], t[c + "gate0/dense/bias"])
    assert got["val_norm_mean"].tolist() == [10.0] and got["val_norm_std"].tolist() == [10.0] and "g_norm_mean" not in got
    critic = load_critic_weights(build_critic(6, 3, hidden=(5, 4), gate_common=8, gate_hidden=4), got).double()
    s, g = rng.standard_normal((4, 6)), rng.standard_normal((4, 3))
    with torch.no_grad():
        np.testing.assert_allclose(critic(torch.as_tensor(s), torch.as_tensor(g)).numpy(), _np_critic(d, s, g), atol=1e-5)


class _FakeCriticEnv(_FakeEnv):
    """_FakeEnv with reward bounds and all terminate codes: env 0's episodes (3 steps) end in Fail, env 1's (4 steps) by time limit (Null),
    env 2's (3 steps) in Succ.  The state and goal encode the episode clock, so a restarted state (clock 0) is told apart from a terminal one."""
    get_reward_min, get_reward_max, get_reward_fail, get_reward_succ = (_RewardEnv.get_reward_min, _RewardEnv.get_reward_max,
                                                                          _RewardEnv.get_reward_fail, _RewardEnv.get_reward_succ)

    def step(self, a):
        s, r, done, _ = super().step(a)
        code = self.torch.tensor([FAIL, 0, SUCC, 0] * self.num_envs, dtype=self.torch.int32)[:self.num_envs]
        return s, r, done, self.torch.where(done, code, self.torch.zeros_like(code))


@pytest.mark.parametrize("goal_size", [0, 3])
def test_collect_records_values_of_the_terminal_states(goal_size):
    torch.manual_seed(0)
    env = _FakeCriticEnv(4, goal_size)
    critic = build_critic(5, goal_size, hidden=(16, 8), gate_common=8, gate_hidden=4)
    ro = BatchedRollout(env, exp_rate=0.0, seed=1, critic=critic, discount=0.95, td_lambda=0.9)
    assert ro.val_norm.mean.tolist() == pytest.approx([10.0]) and (ro.val_fail, ro.val_succ) == pytest.approx((0.0, 20.0))
    T = 9
    traj = ro.collect(T, record_stats=False)
    assert all(traj[k].shape == (T, 4) for k in ("values", "end_values", "returns", "advantages"))
    done = traj["dones"]
    assert done[:, 0].nonzero().flatten().tolist() == [2, 5, 8] and traj["terminate"][2].tolist() == [FAIL, 0, SUCC, 0]

    def V(s, g):
        with torch.no_grad():
            out = critic(ro.s_norm.normalize(s), ro.g_norm.normalize(g)) if goal_size else critic(ro.s_norm.normalize(s))
        return ro.val_norm.unnormalize(out)[..., 0]
    goals = traj["goals"] if goal_size else None
    torch.testing.assert_close(traj["values"], V(traj["states"], goals))
    # where the path goes on, the end value is the next state's value
    torch.testing.assert_close(traj["end_values"][:-1][~done[:-1]], traj["values"][1:][~done[:-1]])
    # at a done step it is the critic of the pre-reset state (clock 3 or 4) and goal, not of the restarted one (clock 0)
    clock = torch.tensor([3.0, 4.0, 3.0, 4.0])
    term_s = clock[:, None] + torch.arange(5.0)[None, :]
    term_g = torch.stack([clock, -clock, torch.ones(4)], dim=1)[:, :goal_size]
    for k, n in done.nonzero().tolist():
        torch.testing.assert_close(traj["end_values"][k, n], V(term_s[n:n + 1], term_g[n:n + 1])[0])
        assert not torch.allclose(traj["end_values"][k, n], V(torch.arange(5.0)[None], torch.tensor([[0.0, 0.0, 1.0]])[:, :goal_size])[0])
    want = path_returns(traj["rewards"], traj["values"], traj["end_values"], done, traj["terminate"], 0.95, 0.9, 0.0, 20.0)
    assert np.abs(traj["returns"].numpy() - want).max() <= 1e-5 * 20
    torch.testing.assert_close(traj["advantages"], traj["returns"] - traj["values"])


def test_collect_without_critic_and_refusals():
    env = _FakeCriticEnv(4, 0)
    traj = BatchedRollout(env, exp_rate=0.0).collect(3, record_stats=False)
    assert not {"values", "end_values", "returns", "advantages"} & set(traj)
    critic = build_critic(5, 0, hidden=(16, 8))
    for kw, msg in ((dict(discount=0.95), "need a critic"), (dict(td_lambda=0.95), "need a critic")):
        with pytest.raises(ValueError, match=msg):
            BatchedRollout(_FakeCriticEnv(4, 0), **kw)
    for d, lam in ((None, 0.95), (1.0, 0.95), (-0.1, 0.95), (float("nan"), 0.95)):
        with pytest.raises(ValueError, match="discount"):
            BatchedRollout(_FakeCriticEnv(4, 0), critic=critic, discount=d, td_lambda=lam)
    for lam in (None, 1.5, -0.1, float("nan")):
        with pytest.raises(ValueError, match="td_lambda"):
            BatchedRollout(_FakeCriticEnv(4, 0), critic=critic, discount=0.95, td_lambda=lam)
    with pytest.raises(ValueError, match="goal values"):
        BatchedRollout(_FakeCriticEnv(4, 3), critic=critic, discount=0.95, td_lambda=0.95)
