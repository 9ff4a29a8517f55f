"""Running a trained skill without a device: the run command's argument resolution, the model-file loader (deepmimic_b200/model_files.py) on
reference TensorBundles written from the golden policy fixtures and on a Trainer checkpoint of a stand-in run, the resumption of a run started
from model files, and the assembly of an episode's motion file."""
import os

import numpy as np
import pytest

from deepmimic_b200 import trainer as tr
from deepmimic_b200.model_files import load_model_files
from deepmimic_b200.rollout import DeviceNormalizer, build_critic, build_gated_policy, build_policy, load_actor_weights
from deepmimic_b200.train import arg_table, first_arg, resolve_model_files
from tests.test_tf_checkpoint_cpu import write_bundle
from tests.test_train_cpu import PPO, _StandInEnv

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
A = "agent/main/actor/"


def _fixture(name):
    f = np.load(os.path.join(GOLD, name))
    return {k: f[k].astype(np.float32) for k in f.files}


def _bundle(tmp_path, fx, counts=None, critic=None):
    """a reference TensorBundle with the fixture's actor and normalisers (and int32 counts / a critic when given); returns its prefix"""
    t = {A + "0/dense/kernel": fx["w0"], A + "0/dense/bias": fx["b0"], A + "1/dense/kernel": fx["w1"], A + "1/dense/bias": fx["b1"],
         A + "dist_gauss_diag/mean/kernel": fx["wm"], A + "dist_gauss_diag/mean/bias": fx["bm"], A + "dist_gauss_diag/logstd/bias": fx["logstd"]}
    if "gcw" in fx:
        t[A + "gate_common/0/dense/kernel"], t[A + "gate_common/0/dense/bias"] = fx["gcw"], fx["gcb"]
        for i in range(2):
            for part, scope in (("hidden", "gate%d/0/dense"), ("bias", "gate%d/dense"), ("scale", "gate%d/dense_1")):
                t[A + scope % i + "/kernel"], t[A + scope % i + "/bias"] = fx["g%d_%s_w" % (i, part)], fx["g%d_%s_b" % (i, part)]
    for nm, key in (("s_norm", "s"), ("g_norm", "g"), ("a_norm", "a")):
        if key + "_mean" in fx:
            t["agent/resource/%s/mean" % nm], t["agent/resource/%s/std" % nm] = fx[key + "_mean"], fx[key + "_std"]
    for nm, c in (counts or {}).items():
        t["agent/resource/%s/count" % nm] = np.array(c, dtype=np.int32)
    t.update(critic or {})
    prefix = str(tmp_path / "policy.ckpt")
    write_bundle(prefix, t)
    return prefix


def _fixture_actor(fx):
    a = dict(hidden=[(fx["w0"], fx["b0"]), (fx["w1"], fx["b1"])], mean=(fx["wm"], fx["bm"]), logstd=fx["logstd"])
    if "gcw" in fx:
        a["gate_common"] = (fx["gcw"], fx["gcb"])
        a["gates"] = [dict(hidden=(fx["g%d_hidden_w" % i], fx["g%d_hidden_b" % i]), bias=(fx["g%d_bias_w" % i], fx["g%d_bias_b" % i]),
                           scale=(fx["g%d_scale_w" % i], fx["g%d_scale_b" % i])) for i in range(2)]
    return a


def _equal_modules(a, b):
    sa, sb = a.state_dict(), b.state_dict()
    return set(sa) == set(sb) and all(np.array_equal(sa[k].numpy(), sb[k].numpy()) for k in sa)


def _norms(S, A, G=0):
    n = dict(s_norm=DeviceNormalizer(S), a_norm=DeviceNormalizer(A))
    if G:
        n["g_norm"] = DeviceNormalizer(G)
    return n


def test_model_files_and_output_path_resolution(tmp_path):
    root = tmp_path / "assets"
    (root / "args").mkdir(parents=True)
    (root / "data" / "policies").mkdir(parents=True)
    (root / "data" / "policies" / "p.ckpt.index").write_bytes(b"")
    (root / "args" / "run_x_args.txt").write_text("--scene imitate\n--agent_files data/agents/a.txt\n--train_agents false\n\n"
                                                   "--model_files data/policies/p.ckpt\n#--output_path commented\n")
    args = ["--arg_file", "args/run_x_args.txt"]
    assert resolve_model_files(args, str(root), "run") == str(root / "data" / "policies" / "p.ckpt")   # a prefix: its .index exists
    assert first_arg(arg_table(args, str(root), "run"), "output_path") == ""
    mine = ["--model_files", "/abs/agent0_checkpoint.pt", "--output_path", "mine"] + args
    assert resolve_model_files(mine, str(root), "run") == "/abs/agent0_checkpoint.pt"                  # the command line wins
    assert first_arg(arg_table(mine, str(root), "run"), "output_path") == "mine"
    assert resolve_model_files(["--scene", "imitate"], str(root)) is None
    with pytest.raises(SystemExit, match="run: arg file args/missing.txt not found"):
        arg_table(["--arg_file", "args/missing.txt"], str(root), "run")


@pytest.mark.parametrize("fixture,S,G,A", [("policy_humanoid3d_spinkick_fp16.npz", 227, 0, 28), ("policy_humanoid3d_amp_target_locomotion_fp16.npz", 226, 3, 28)],
                         ids=["spinkick", "target_amp gated"])
def test_bundle_loads_the_modules_load_actor_weights_builds(tmp_path, fixture, S, G, A):
    fx = _fixture(fixture)
    prefix = _bundle(tmp_path, fx, counts=dict(s_norm=[123456]))
    build = (lambda: build_gated_policy(S, G, A)) if G else (lambda: build_policy(S, A))
    got, want = build(), load_actor_weights(build(), _fixture_actor(fx))
    norms = _norms(S, A, G)
    with pytest.warns(UserWarning, match="has no critic"):
        res = load_model_files(prefix, got, norms, critic=build_critic(S, G))
    assert res["kind"] == "bundle" and _equal_modules(got, want)
    assert res["counts"] == dict(s_norm=123456, a_norm=None, **(dict(g_norm=None) if G else {}))   # the int32 count is read
    assert np.array_equal(norms["s_norm"].mean.numpy(), fx["s_mean"]) and np.array_equal(norms["s_norm"].std.numpy(), fx["s_std"])
    assert np.array_equal(norms["a_norm"].std.numpy(), fx["a_std"])
    if G:
        assert np.array_equal(norms["g_norm"].mean.numpy(), fx["g_mean"])


def test_bundle_with_a_critic_and_value_normaliser(tmp_path):
    rng = np.random.default_rng(0)
    c = "agent/main/critic/"
    crit = {c + "0/dense/kernel": rng.standard_normal((227, 1024)), c + "0/dense/bias": rng.standard_normal(1024), c + "1/dense/kernel": rng.standard_normal((1024, 512)),
            c + "1/dense/bias": rng.standard_normal(512), c + "dense/kernel": rng.standard_normal((512, 1)), c + "dense/bias": rng.standard_normal(1),
            "agent/resource/val_norm/mean": np.array([10.0]), "agent/resource/val_norm/std": np.array([5.0]), "agent/resource/val_norm/count": np.array([7], dtype=np.int32)}
    crit = {k: (v if v.dtype == np.int32 else v.astype(np.float32)) for k, v in crit.items()}
    prefix = _bundle(tmp_path, _fixture("policy_humanoid3d_spinkick_fp16.npz"), critic=crit)
    critic, norms = build_critic(227), dict(_norms(227, 28), val_norm=DeviceNormalizer(1))
    res = load_model_files(prefix, build_policy(227, 28), norms, critic=critic)
    assert np.array_equal(critic.out.weight.detach().numpy(), crit[c + "dense/kernel"].T) and np.array_equal(critic.hidden[1].bias.detach().numpy(), crit[c + "1/dense/bias"])
    assert res["counts"]["val_norm"] == 7 and float(norms["val_norm"].std[0]) == 5.0 and not res["notes"]


@pytest.mark.parametrize("rows,cols,match", [(220, 1, "its critic's state size is 220, this scene's critic needs 227"),
                                              (227, 2, "its critic's output size is 2, this scene's critic needs 1")])
def test_bundle_critic_refusals_name_the_field_before_anything_is_written(tmp_path, rows, cols, match):
    rng = np.random.default_rng(0)
    c = "agent/main/critic/"
    crit = {c + "0/dense/kernel": rng.standard_normal((rows, 1024)), c + "0/dense/bias": np.zeros(1024), c + "1/dense/kernel": rng.standard_normal((1024, 512)),
            c + "1/dense/bias": np.zeros(512), c + "dense/kernel": rng.standard_normal((512, cols)), c + "dense/bias": np.zeros(cols)}
    prefix = _bundle(tmp_path, _fixture("policy_humanoid3d_spinkick_fp16.npz"), critic={k: v.astype(np.float32) for k, v in crit.items()})
    policy, critic, norms = build_policy(227, 28), build_critic(227), _norms(227, 28)
    before = [{k: v.clone() for k, v in m.state_dict().items()} for m in (policy, critic)]
    with pytest.raises(ValueError, match=match):
        load_model_files(prefix, policy, norms, critic=critic)
    for b, m in zip(before, (policy, critic)):
        assert all(np.array_equal(b[k].numpy(), v.numpy()) for k, v in m.state_dict().items())
    assert float(norms["s_norm"].mean.abs().sum()) == 0.0


@pytest.mark.parametrize("build,match", [
    (lambda: build_policy(226, 28), "state size is 227, this scene's actor needs 226"),
    (lambda: build_policy(227, 29), "action size is 28, this scene's actor needs 29"),
    (lambda: build_policy(227, 28, hidden=(1024, 256)), r"hidden widths is \(1024, 512\), this scene's actor needs \(1024, 256\)"),
    (lambda: build_gated_policy(224, 3, 28), "network is plain, this scene's actor needs gated"),
])
def test_bundle_refusals_name_the_field(tmp_path, build, match):
    prefix = _bundle(tmp_path, _fixture("policy_humanoid3d_spinkick_fp16.npz"))
    policy = build()
    before = {k: v.clone() for k, v in policy.state_dict().items()}
    with pytest.raises(ValueError, match=match):
        load_model_files(prefix, policy, {})
    assert all(np.array_equal(before[k].numpy(), v.numpy()) for k, v in policy.state_dict().items())   # nothing written


def test_gated_bundle_refused_by_a_plain_scene_and_missing_files(tmp_path):
    prefix = _bundle(tmp_path, _fixture("policy_humanoid3d_amp_target_locomotion_fp16.npz"))
    with pytest.raises(ValueError, match="network is gated, this scene's actor needs plain"):
        load_model_files(prefix, build_policy(226, 28), {})
    with pytest.raises(ValueError, match="goal size is 3, this scene's actor needs 4"):
        load_model_files(prefix, build_gated_policy(225, 4, 28), {})
    with pytest.raises(FileNotFoundError, match="model file %s not found" % str(tmp_path / "nope.ckpt")):
        load_model_files(str(tmp_path / "nope.ckpt"), build_policy(226, 28), {})


def _stand_in_trainer(values, model_files=None, seed=3):
    import torch
    torch.manual_seed(0)
    cfg = tr.AgentConfig(values)
    return tr.Trainer(["--scene", "stand-in"], cfg, "", 8, window_steps=4, backend="torch", seed=seed, env=_StandInEnv(8, cfg.amp),
                      test_env=_StandInEnv(4, cfg.amp), model_files=model_files)


@pytest.mark.parametrize("amp", [False, True], ids=["ppo", "amp"])
def test_trainer_checkpoint_loads(tmp_path, amp):
    values = dict(PPO, InitSamples=1, NormalizerSamples=1000, OutputIters=100)
    if amp:
        from tests.test_train_cpu import AMP
        values = dict(AMP, InitSamples=1, NormalizerSamples=1000, OutputIters=100, DiscBufferSize=1000, DiscBatchSize=16)
    src = _stand_in_trainer(values)
    for _ in range(3):
        src.iteration()
    path = str(tmp_path / "agent0_checkpoint.pt")
    src.save(path)
    dst = _stand_in_trainer(values, model_files=path, seed=11)
    assert dst.iter == 0 and dst.total_samples == 0 and dst.run["model_files"] == path and not dst.model_notes
    for a, b in ((src.ro.policy, dst.ro.policy), (src.ro.critic, dst.ro.critic)) + (((src.ro.disc, dst.ro.disc),) if amp else ()):
        assert _equal_modules(a, b)
    for name, n in src._all_norms().items():
        m = dst._all_norms()[name]
        assert m.count == n.count and np.array_equal(m.mean.numpy(), n.mean.numpy()) and np.array_equal(m.std.numpy(), n.std.numpy()), name
        assert m.new_count == 0 and float(m.new_sum.abs().sum()) == 0.0
    assert all(float(a.abs().sum()) == 0.0 for a in dst.ppo.acc.values())   # zero momentum
    dst.iteration()                                                       # trains from there
    # a run record without model_files (an older checkpoint) counts as None: a plain run resumes it, a run from model files does not
    import torch
    s = torch.load(path, weights_only=True)
    del s["run"]["model_files"]
    torch.save(s, str(tmp_path / "old.pt"))
    _stand_in_trainer(values).load(str(tmp_path / "old.pt"))
    with pytest.raises(ValueError, match="its run started from model files None, this one from"):
        _stand_in_trainer(values, model_files=path).load(str(tmp_path / "old.pt"))


def test_loaded_normalisers_without_a_count_count_normalizer_samples(tmp_path):
    """a bundle without counts: the normalisers the loop updates start at NormalizerSamples, so the first window is weighed against the
    loaded statistics instead of replacing them"""
    S = 5
    rng = np.random.default_rng(1)
    fx = dict(w0=rng.standard_normal((S, 1024)), b0=np.zeros(1024), w1=rng.standard_normal((1024, 512)), b1=np.zeros(512), wm=rng.standard_normal((512, 3)),
              bm=np.zeros(3), logstd=np.full(3, -3.0), s_mean=np.full(S, 0.25), s_std=np.full(S, 2.0), a_mean=np.zeros(3), a_std=np.ones(3))
    prefix = _bundle(tmp_path, {k: v.astype(np.float32) for k, v in fx.items()})
    values = dict(PPO, InitSamples=1, NormalizerSamples=1000, OutputIters=100)
    with pytest.warns(UserWarning):
        t = _stand_in_trainer(values, model_files=prefix)
    assert any("has no critic" in n for n in t.model_notes)
    assert t.ro.s_norm.count == 1000 and np.array_equal(t.ro.s_norm.mean.numpy(), np.full(S, 0.25, dtype=np.float32))
    t.iteration()   # one window of 32 samples folded into 1000: the stand-in's third state entry is always 1
    assert t.ro.s_norm.count == 1032
    assert abs(float(t.ro.s_norm.mean[2]) - (0.25 * 1000 / 1032 + 32 / 1032)) < 1e-6


def test_a_run_from_model_files_resumes_with_its_model_files(tmp_path):
    """a run started from model files: 2 iterations, a checkpoint, a new Trainer with the same model files loads it and its next 2 iterations
    equal a straight run's bit for bit; a Trainer without the model files, or with other ones, is refused with both named"""
    values = dict(PPO, InitSamples=1, NormalizerSamples=1000, OutputIters=1)
    src = _stand_in_trainer(values)
    src.iteration()
    model = str(tmp_path / "model.pt")
    src.save(model)
    straight = _stand_in_trainer(values, model_files=model)
    rows_a = [straight.iteration() for _ in range(4)]
    first = _stand_in_trainer(values, model_files=model)
    rows_b = [first.iteration() for _ in range(2)]
    ckpt = str(tmp_path / "agent0_checkpoint.pt")
    first.save(ckpt)
    resumed = _stand_in_trainer(values, model_files=model)
    resumed.load(ckpt)
    rows_b += [resumed.iteration() for _ in range(2)]
    strip = lambda r: {k: x for k, x in r.items() if k != "Wall_Time"}
    assert [repr(strip(r)) for r in rows_a] == [repr(strip(r)) for r in rows_b]
    assert _equal_modules(straight.ro.policy, resumed.ro.policy) and _equal_modules(straight.ro.critic, resumed.ro.critic)
    with pytest.raises(ValueError, match="started from model files %s, this one from None: resume with the arguments the run started with" % model):
        _stand_in_trainer(values).load(ckpt)
    with pytest.raises(ValueError, match="started from model files %s, this one from %s" % (model, ckpt)):
        _stand_in_trainer(values, model_files=ckpt).load(ckpt)


def test_episode_motion_file_round_trip(tmp_path):
    """run_episodes' chunks -> episode_motion -> formats.write_motion: the frames are the episode's poses and its terminal end pose, and
    read_motion returns exactly what was written (the reference's %.10f numbers)"""
    import torch
    from deepmimic_b200.formats import read_motion
    from deepmimic_b200.rollout import episode_motion
    from deepmimic_b200.run import write_episode_motions
    g = torch.Generator().manual_seed(0)
    T, N, P = 32, 3, 43
    poses = [torch.randn(T, N, P, generator=g) for _ in range(2)]
    end_poses = [torch.randn(T, N, P, generator=g) for _ in range(2)]
    lengths = torch.tensor([40, 1, 64], dtype=torch.int32)
    paths = write_episode_motions(str(tmp_path / "motion_%d.txt"), dict(poses=poses, end_poses=end_poses, lengths=lengths), 3, 1.0 / 30.0)
    allp, alle = torch.cat(poses), torch.cat(end_poses)
    for e, path in enumerate(paths):
        L = int(lengths[e])
        frames = episode_motion(poses, end_poses, e, L)
        assert frames.shape == (L + 1, P)
        assert np.array_equal(frames[:L], allp[:L, e].double().numpy()) and np.array_equal(frames[L], alle[L - 1, e].double().numpy())
        m = read_motion(path)
        assert m["loop"] == "none" and m["frames"].shape == (L + 1, P)
        assert np.array_equal(m["frames"], np.vectorize(lambda v: float("%.10f" % v))(frames))
        assert np.array_equal(m["durations"], np.array([float("%.10f" % (1.0 / 30.0))] * L + [0.0]))
    with pytest.raises(ValueError, match="does not fit"):
        episode_motion(poses, end_poses, 0, 65)
