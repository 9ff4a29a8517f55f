"""The training loop without a device: agent files (AgentConfig), the command line's argument resolution, and the bookkeeping of
Trainer.iteration() -- exploration rate, normaliser recording, sample counts, the InitSamples / NormalizerSamples phases, the discriminator's
step count and the actor stepsize control -- over a stand-in environment on the CPU."""
import copy
import json
import math

import numpy as np
import pytest

from deepmimic_b200 import trainer as tr
from deepmimic_b200.train import build_parser, resolve_args

PPO = {
    "AgentType": "PPO", "ActorNet": "fc_2layers_1024units", "ActorStepsize": 2.5e-6, "ActorMomentum": 0.9, "ActorWeightDecay": 5e-4,
    "ActorInitOutputScale": 0.01, "CriticNet": "fc_2layers_1024units", "CriticStepsize": 0.01, "CriticMomentum": 0.9, "CriticWeightDecay": 0,
    "Discount": 0.95, "TDLambda": 0.95, "BatchSize": 4096, "MiniBatchSize": 256, "Epochs": 1, "RatioClip": 0.2, "NormAdvClip": 4,
    "TarClipFrac": -1, "ActorStepsizeDecay": 0.5, "InitSamples": 1, "NormalizerSamples": 1000000, "ExpAnnealSamples": 64000000,
    "ExpParamsBeg": {"Rate": 1, "InitActionRate": 1, "Noise": 0.05, "NoiseInternal": 0, "Temp": 0.1},
    "ExpParamsEnd": {"Rate": 0.2, "InitActionRate": 0.01, "Noise": 0.05, "NoiseInternal": 0, "Temp": 0.001},
    "OutputIters": 10, "IntOutputIters": 400, "TestEpisodes": 32,
}
AMP = dict(PPO, AgentType="AMP", DiscNet="fc_2layers_1024units", DiscStepSize=1e-5, DiscMomentum=0.9, DiscWeightDecay=5e-4, DiscLogitRegWeight=0.05,
           DiscGradPenalty=10, DiscBatchSize=256, DiscStepsPerBatch=1, DiscBufferSize=100000, DiscInitOutputScale=1, TaskRewardLerp=0.0)


def _write(tmp_path, values, name="agent.txt"):
    p = tmp_path / name
    p.write_text(json.dumps(values, indent=1))
    return str(p)


@pytest.mark.parametrize("values", [PPO, AMP], ids=["ppo", "amp"])
def test_agent_files_parse(tmp_path, values):
    cfg = tr.AgentConfig.from_json(_write(tmp_path, values))
    assert cfg.amp == (values["AgentType"] == "AMP")
    assert cfg["MiniBatchSize"] == 256 and isinstance(cfg["MiniBatchSize"], int) and cfg["ActorStepsize"] == 2.5e-6
    assert cfg["ExpParamsEnd"]["Rate"] == 0.2 and cfg.values == values
    if cfg.amp:
        assert cfg["DiscBufferSize"] == 100000 and cfg["DiscNet"] == "fc_2layers_1024units"


def _edit(base, **kw):
    v = copy.deepcopy(base)
    for k, x in kw.items():
        if x is None:
            del v[k]
        else:
            v[k] = x
    return v


@pytest.mark.parametrize("base,edit,match", [
    (PPO, dict(Discount=None), "Discount is missing"),
    (AMP, dict(DiscGradPenalty=None), "DiscGradPenalty is missing"),
    (PPO, dict(ActorLearningRate=1e-3), "unknown key ActorLearningRate"),
    (PPO, dict(DiscStepSize=1e-5), "DiscStepSize is an AMP agent key"),
    (PPO, dict(ExpParamsBeg={"Rate": 1, "Noise": 0.05, "Sigma": 1}), "unknown key ExpParamsBeg.Sigma"),
    (PPO, dict(RatioClip=1.5), "RatioClip must be in"),
    (PPO, dict(Discount=1.0), "Discount must be in"),
    (PPO, dict(MiniBatchSize=0), "MiniBatchSize must be an integer"),
    (PPO, dict(Epochs=1.5), "Epochs must be an integer"),
    (AMP, dict(TaskRewardLerp=2), "TaskRewardLerp must be in"),
    (PPO, dict(ExpParamsEnd={"Rate": 1.2}), "ExpParamsEnd.Rate must be in"),
    (PPO, dict(ActorNet="fc_3layers_1024units"), "ActorNet 'fc_3layers_1024units' is not supported"),
    (AMP, dict(DiscNet="fc_2layers_gated_1024units"), "DiscNet 'fc_2layers_gated_1024units' is not supported"),
    (PPO, dict(AgentType="SAC"), "AgentType must be"),
])
def test_agent_file_errors_name_the_key(tmp_path, base, edit, match):
    with pytest.raises(ValueError, match=match):
        tr.AgentConfig.from_json(_write(tmp_path, _edit(base, **edit)))


def test_cli_argument_resolution(tmp_path):
    root = tmp_path / "assets"
    (root / "args").mkdir(parents=True)
    (root / "data" / "agents").mkdir(parents=True)
    (root / "data" / "agents" / "a.txt").write_text("{}")
    (root / "args" / "train_x_args.txt").write_text("--scene imitate\n\n--agent_files data/agents/a.txt\n--output_path out_file\n"
                                                   "#--int_output_path output/intermediate\n")
    opts, rest = build_parser().parse_known_args(["--arg_file", "args/train_x_args.txt", "--num_envs", "64", "--scene", "imitate",
                                                  "--max_iters", "3", "--time_lim_min", "-1"])
    assert opts.num_envs == 64 and opts.max_iters == 3 and opts.window_steps == 32 and opts.backend == "tensor_core"
    assert rest == ["--arg_file", "args/train_x_args.txt", "--scene", "imitate", "--time_lim_min", "-1"]
    agent, out, intp = resolve_args(rest, str(root))
    assert agent == str(root / "data" / "agents" / "a.txt") and out == "out_file" and intp == ""   # commented out in the file
    agent, out, intp = resolve_args(rest + ["--output_path", "mine", "--int_output_path", "mine/int", "--agent_files", "/abs/b.txt"], str(root))
    assert (agent, out, intp) == ("/abs/b.txt", "mine", "mine/int")   # the command line wins over the arg file


# ---- the loop over a stand-in env
class _StandInEnv:
    """N environments on the CPU: episode of env i ends every 3 + i % 4 policy steps, reward from the action; AMP observations of width 6"""

    def __init__(self, n, amp=True):
        import torch
        self.torch, self.num_envs, self.device, self.amp = torch, n, torch.device("cpu"), amp
        self.S, self.A, self.M = 5, 3, 6
        self.t = torch.zeros(n)
        self.period = torch.tensor([3 + i % 4 for i in range(n)], dtype=torch.float32)
        self.sample_counts, self.mode, self.expert_rows = [], 0, []
        self.stream = None

    def get_name(self): return "Imitate AMP" if self.amp else "Imitate"
    def enable_amp_task_reward(self): return False
    def get_state_size(self, agent_id=0): return self.S
    def get_action_size(self, agent_id=0): return self.A
    def get_goal_size(self, agent_id=0): return 0
    def build_state_norm_groups(self, agent_id=0): return np.zeros(self.S, dtype=np.int32)
    def build_state_offset(self, agent_id=0): return np.zeros(self.S)
    def build_state_scale(self, agent_id=0): return np.ones(self.S)
    def build_action_offset(self, agent_id=0): return np.zeros(self.A)
    def build_action_scale(self, agent_id=0): return np.ones(self.A)
    def build_action_bound_min(self, agent_id=0): return -np.ones(self.A)
    def build_action_bound_max(self, agent_id=0): return np.ones(self.A)
    def get_reward_min(self, agent_id=0): return 0.0
    def get_reward_max(self, agent_id=0): return 1.0
    def get_reward_fail(self, agent_id=0): return 0.0
    def get_reward_succ(self, agent_id=0): return 1.0
    def get_amp_obs_size(self): return self.M
    def get_amp_obs_offset(self): return np.zeros(self.M)
    def get_amp_obs_scale(self): return np.ones(self.M)
    def get_amp_obs_norm_group(self): return np.zeros(self.M, dtype=np.int32)
    def set_mode(self, m): self.mode = m
    def set_sample_count(self, c): self.sample_counts.append(c)
    def state_dict(self): return dict(t=self.t.clone())
    def load_state_dict(self, s): self.t = s["t"].clone()

    def record_state(self):
        t = self.torch
        return t.stack([self.t, self.t / self.period, t.ones_like(self.t), self.period, t.zeros_like(self.t)], dim=1)

    def step(self, a):
        t = self.torch
        self.t += 1
        self._done = self.t >= self.period
        self._a = a
        return self.record_state(), (1.0 - 0.1 * a.square().mean(dim=1)).clamp(0, 1), self._done, t.where(self._done, 1, 0).int()

    def reset(self, force_all=False):
        self.t = self.torch.where(self._done if not force_all else self.torch.ones_like(self.t, dtype=self.torch.bool), 0.0, self.t)

    def record_amp_obs_agent(self):
        return self.torch.cat([self.record_state(), self._a[:, :1]], dim=1)

    def sample_amp_obs_expert(self, rows):
        self.expert_rows.append(rows)
        return self.torch.ones(rows, self.M) * 0.5


def _trainer(values, n=8, T=4):
    import torch
    torch.manual_seed(0)
    cfg = tr.AgentConfig(values)
    t = tr.Trainer(["--scene", "stand-in"], cfg, "", n, window_steps=T, backend="torch", seed=3, env=_StandInEnv(n, cfg.amp),
                   test_env=_StandInEnv(4, cfg.amp))
    flags = []
    collect = t.ro.collect

    def spy(num_steps, record_stats=True):
        flags.append(record_stats)
        return collect(num_steps, record_stats=record_stats)
    t.ro.collect = spy
    return t, flags


def test_iteration_bookkeeping():
    """32 samples per window; InitSamples 70 (windows 1-2 initialise at 64 -> 96: the third window crosses it), NormalizerSamples 120; exploration
    annealed over 256 samples; TarClipFrac control on; DiscStepsPerBatch 2 at DiscBatchSize 12"""
    T, N = 4, 8
    v = _edit(AMP, InitSamples=70, NormalizerSamples=120, ExpAnnealSamples=256, TarClipFrac=0.2, ActorStepsizeDecay=0.5, DiscStepsPerBatch=2,
              DiscBatchSize=12, DiscBufferSize=20, MiniBatchSize=16, OutputIters=3, TestEpisodes=4)
    t, flags = _trainer(v, N, T)
    disc_steps = []
    upd = t.disc.update

    def disc_spy(a, e):
        disc_steps.append((t.disc.steps, a.shape[0], e.shape[0]))
        return upd(a, e)
    t.disc.update = disc_spy
    rows, stepsize = [], PPO["ActorStepsize"]
    for k in range(9):
        row = t.iteration()
        rows.append(row)
        samples = T * N * (k + 1)
        assert row["Iteration"] == k and row["Samples"] == samples and t.env.sample_counts[-1] == samples
        assert row["Exp_Rate"] == pytest.approx(1.0 + (0.2 - 1.0) * min(T * N * k / 256, 1.0))
        # recorded while the normaliser still needed updates when the window was stored: windows 1-4 (the fourth crosses 120)
        assert flags[k] == (T * N * k < 120)
        assert t.initialized == (samples >= 70)
        if k >= 3:   # initialised at the window that crossed InitSamples (96), training from the next one
            stepsize = tr.update_actor_stepsize(stepsize, row["Clip_Frac"], 0.2, 0.5, k)
        assert row["Actor_Stepsize"] == stepsize
        assert t.env.expert_rows[-1] == T * N
        assert math.isfinite(row["Train_Return"]) and math.isfinite(row["Test_Return"])
    # trained from the fourth window on: ceil(2 * 32 / 12) = 6 steps on the full buffers (4 windows of 32 rows stored in a 20-row buffer)
    assert disc_steps == [(6, 20, 20)] * 6
    assert t.agent_buf.size == 20 and t.expert_buf.size == 20
    assert not t.need_normalizer_update and t.ro.s_norm.count == 4 * T * N


def test_iteration_phases_without_training():
    """before InitSamples no update runs: the weights, the stepsize and the learners' statistics stay as they were"""
    import torch
    t, _ = _trainer(_edit(PPO, InitSamples=10 ** 6, TarClipFrac=0.2, OutputIters=5, TestEpisodes=4))
    w0 = [p.detach().clone() for p in t.ro.policy.parameters()]
    for _ in range(7):
        row = t.iteration()
        assert row["Actor_Loss"] == 0.0 and row["Actor_Stepsize"] == PPO["ActorStepsize"]
    assert all(torch.equal(a, b) for a, b in zip(w0, t.ro.policy.parameters()))
    assert t.ro.s_norm.count == 7 * 32 and not t.initialized


def test_checkpoint_round_trip_on_the_stand_in(tmp_path):
    """4 + 4 iterations with a checkpoint in between equal 8 straight ones (weights, accumulators, normalisers, buffers, rows); a checkpoint of
    another run is refused"""
    import torch
    v = _edit(AMP, InitSamples=40, NormalizerSamples=150, TarClipFrac=0.2, DiscBatchSize=12, DiscBufferSize=50, MiniBatchSize=16, OutputIters=2,
              TestEpisodes=4)
    a, _ = _trainer(v)
    rows_a = [a.iteration() for _ in range(8)]
    b, _ = _trainer(v)
    rows_b = [b.iteration() for _ in range(4)]
    b.save(str(tmp_path / "c.pt"))
    c, _ = _trainer(v)
    c.load(str(tmp_path / "c.pt"))
    rows_b += [c.iteration() for _ in range(4)]
    strip = lambda r: {k: x for k, x in r.items() if k != "Wall_Time"}
    assert [str(strip(r)) for r in rows_a] == [str(strip(r)) for r in rows_b]
    sa, sc = a.state_dict(), c.state_dict()
    for name in ("actor", "critic", "disc"):
        assert all(torch.equal(sa["nets"][name][k], sc["nets"][name][k]) for k in sa["nets"][name])
    assert all(torch.equal(x, y) for x, y in zip(sa["accs"]["ppo"] + sa["accs"]["disc"], sc["accs"]["ppo"] + sc["accs"]["disc"]))
    assert torch.equal(sa["buffers"]["agent"]["rows"], sc["buffers"]["agent"]["rows"])
    assert all(torch.equal(sa["norms"]["s_norm"][f], sc["norms"]["s_norm"][f]) for f in ("mean", "std", "new_sum"))
    d, _ = _trainer(_edit(v, DiscBatchSize=13))
    with pytest.raises(ValueError, match="agent file"):
        d.load(str(tmp_path / "c.pt"))
