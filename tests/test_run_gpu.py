"""Running a trained skill on the GPU: dm_record_pose against the CPU oracle's BuildPose / BuildVel and a restatement from dm_get_snapshot,
collect(record_pose=True), the run command on the golden policies (as reference TensorBundles) with its motion files, the Trainer's
--model_files round trip, and the resumption of a command-line run started from model files."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.oracle_binding import Oracle
from tests.parity_util import SnapLayout, joint_types_from_assets
from tests.test_run_cpu import _bundle, _fixture

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPINKICK = ["--arg_file", "args/run_humanoid3d_spinkick_args.txt"]
SPINKICK_TRAIN = ["--arg_file", "args/train_humanoid3d_spinkick_args.txt"]
DOG = ["--arg_file", "args/run_dog3d_trot_args.txt"]
TARGET = ["--motion_file", "data/datasets/synthetic_locomotion_56.txt", "--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]
CASES = [("spinkick", SPINKICK, "data/characters/humanoid3d.txt"), ("dog trot", DOG, "data/characters/dog3d.txt"),
         ("target_amp", TARGET, "data/characters/humanoid3d.txt")]


def _restated(snap, lay, jtypes, pose_off, P, scale):
    """what dm_pose_kernel writes for the root and the revolute joints, restated in float32 from a snapshot; NaN where it is not restated
    (the spherical joints, which go through the joint frame's rotation: the oracle checks those)"""
    f = np.float32
    inv = f(1.0) / f(scale)
    p, v = np.full(P, np.nan, dtype=np.float32), np.full(P, np.nan, dtype=np.float32)
    s = snap.astype(np.float32)
    p[0:3] = inv * s[0:3]
    q = np.array([s[6], -s[3], -s[4], -s[5]], dtype=np.float32)     # w, x, y, z of the conjugated world->base quaternion
    p[3:7] = -q if q[0] < 0 else q
    v[0:3] = inv * s[10:13]; v[3:6] = s[7:10]; v[6] = 0.0
    two_pi, pi = f(6.283185307179586), f(3.14159265358979)
    for j, t in enumerate(jtypes):
        if j > 0 and t == "revolute":
            a = np.fmod(s[lay.jpos + 4 * j], two_pi)
            a = a - two_pi if a > pi else (a + two_pi if a < -pi else a)
            p[pose_off[j]] = a
            v[pose_off[j]] = s[lay.jvel + 3 * j]
    return p, v


def _canon(x, pose_off, jtypes):
    """quaternion blocks (root and spherical joints) with w >= 0"""
    x = x.copy()
    for j, t in enumerate(jtypes):
        o = 3 if j == 0 else pose_off[j]
        if j == 0 or t == "spherical":
            if x[o] < 0:
                x[o:o + 4] = -x[o:o + 4]
    return x


@pytest.mark.parametrize("name,args,char", CASES, ids=[c[0] for c in CASES])
def test_record_pose_matches_the_oracle_and_the_snapshot(asset_root, name, args, char):
    """1001 environments (a padded batch), placement by contact load on, 40 policy steps of random actions with resets, then dm_record_pose
    of every environment.  Teacher-forced: the oracle is set to an environment's simulated state and its BuildPose / BuildVel is compared
    within fp32 rounding; the root and revolute entries equal a float32 restatement from dm_get_snapshot bit for bit; rows past the real
    environments are not written"""
    import torch
    from deepmimic_b200.capi import BatchedCore, HostModel, lib
    N = 1001
    core = BatchedCore(args, N, asset_root, device=0, seed=11)
    core.set_env_order(True)
    host = HostModel(args, asset_root)
    P, nl = core.dims.pose_dim, core.dims.num_joints
    pose_off, jtypes = host.info("pose_offsets"), joint_types_from_assets(asset_root, char)
    lay = SnapLayout(nl)
    orc = Oracle(args, asset_root)
    g = torch.Generator(device="cuda").manual_seed(3)
    off = torch.as_tensor(-host.static(2), dtype=torch.float32, device="cuda")
    scl = torch.as_tensor(1.0 / host.static(3), dtype=torch.float32, device="cuda")
    core.reset(True)
    for _ in range(40):
        core.set_action((off + 0.25 * scl * torch.randn(N, core.dims.action_size, device="cuda", generator=g)).contiguous())
        core.update(1.0 / 600.0, core.dims.updates_per_action)
        core.reset(False)
    big_p = torch.full((N + 7, P), float("nan"), device="cuda")
    big_v = torch.full((N + 7, P), float("nan"), device="cuda")
    assert lib().dm_record_pose(core.h, big_p.data_ptr(), big_v.data_ptr()) == 0
    pose, vel = torch.empty(N, P, device="cuda"), torch.empty(N, P, device="cuda")
    core.record_pose(pose, vel)
    only_vel = torch.empty(N, P, device="cuda")
    core.record_pose(None, only_vel)
    core.sync()
    assert torch.isnan(big_p[N:]).all() and torch.isnan(big_v[N:]).all()
    assert torch.equal(big_p[:N], pose) and torch.equal(big_v[:N], vel) and torch.equal(only_vel, vel)
    pose, vel = pose.cpu().numpy(), vel.cpu().numpy()
    worst_p = worst_v = 0.0
    for e in list(range(0, N, 37)) + [N - 1]:
        snap = core.get_snapshot(e)
        orc.set_snapshot(snap)
        po, vo = orc.get_pose()
        assert pose[e, 3] >= 0 and all(pose[e, pose_off[j]] >= 0 for j, t in enumerate(jtypes) if j > 0 and t == "spherical")
        worst_p = max(worst_p, np.abs(_canon(po, pose_off, jtypes) - pose[e]).max())
        worst_v = max(worst_v, np.abs(vo - vel[e]).max())
        rp, rv = _restated(snap, lay, jtypes, pose_off, P, 4.0)
        m = ~np.isnan(rp)
        assert np.array_equal(rp[m].view(np.uint32), pose[e][m].view(np.uint32)), (e, np.nonzero(rp[m] != pose[e][m]))
        m = ~np.isnan(rv)
        assert np.array_equal(rv[m].view(np.uint32), vel[e][m].view(np.uint32)), (e, np.nonzero(rv[m] != vel[e][m]))
    print("%s: record_pose against the oracle, max |pose| error %.2e, max |vel| error %.2e" % (name, worst_p, worst_v))
    assert worst_p < 2e-5 and worst_v < 2e-4


def test_collect_with_poses(asset_root):
    """random-initialised actor on the training arg file (short episodes): record_pose=True leaves every other key bit-identical, end_poses
    continues poses at the steps that did not end an episode, and a restarted episode's first pose is the reset's (root x, z = 0)"""
    import torch
    from deepmimic_b200.env import DeepMimicBatchEnv
    from deepmimic_b200.rollout import BatchedRollout, build_policy
    outs = []
    for record in (False, True):
        torch.manual_seed(0)
        env = DeepMimicBatchEnv(SPINKICK_TRAIN, 512, asset_root, seed=2)
        ro = BatchedRollout(env, policy=build_policy(env.get_state_size(), env.get_action_size()), exp_rate=1.0, seed=1, backend="tensor_core")
        outs.append(ro.collect(48, record_pose=record))
    a, b = outs
    assert set(b) == set(a) | {"poses", "vels", "end_poses", "end_vels"}
    for k in a:
        assert torch.equal(a[k], b[k]), k
    done = b["dones"][:-1]
    assert int(done.sum()) > 0 and int((~done).sum()) > 0
    keep = ~done
    assert torch.equal(b["end_poses"][:-1][keep], b["poses"][1:][keep]) and torch.equal(b["end_vels"][:-1][keep], b["vels"][1:][keep])
    restart = b["poses"][1:][done]
    assert (restart[:, 0] == 0).all() and (restart[:, 2] == 0).all()
    assert (b["end_poses"][:-1][done][:, [0, 2]] != 0).any(dim=1).all()


def _run_cmd(asset_root, args, prefix, out, n, k):
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-m", "deepmimic_b200.run", "--asset_root", asset_root] + args + [
        "--model_files", prefix, "--output_path", str(out), "--num_envs", str(n), "--record_motion", str(k)]
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=REPO), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout


@pytest.mark.parametrize("name,args,fixture,n,full", [
    ("spinkick", SPINKICK, "policy_humanoid3d_spinkick_fp16.npz", 32, True),
    ("dog trot", DOG, "policy_dog3d_trot_fp16.npz", 16, True),
    ("target_amp", TARGET, "policy_humanoid3d_amp_target_locomotion_fp16.npz", 8, False),
])
def test_run_command(asset_root, tmp_path, name, args, fixture, n, full):
    """python -m deepmimic_b200.run on a golden policy written as a reference TensorBundle: one episode per environment; spin kick and dog
    trot run their full test-mode episodes without a Fail; the motion files load through the simulation's loaders as --motion_file with one
    frame per policy step and the terminal one, and a handle reset at a frame's time puts the character in that frame's pose"""
    import torch
    from deepmimic_b200.capi import BatchedCore, HostModel
    from deepmimic_b200.formats import read_motion, read_table_log
    prefix = _bundle(tmp_path, _fixture(fixture))
    out = tmp_path / "out"
    stdout = _run_cmd(asset_root, args, prefix, out, n, 2)
    print(name, stdout.strip())
    log = read_table_log(str(out / "run_log.txt"))
    assert list(log["Env"]) == list(range(n))
    if full:   # the run arg files set no limit: --episode_time's 20 s, 600 policy steps at 30 Hz, end every episode at the same step
        assert (log["Terminate"] == 0).all() and (log["Length"] == log["Length"][0]).all() and log["Length"][0] >= 600, (log["Terminate"], log["Length"])
    for e in range(2):
        path = str(out / ("motion_%d.txt" % e))
        m = read_motion(path)
        assert m["frames"].shape[0] == log["Length"][e] + 1 and m["loop"] == "none"
        margs = ["--motion_file", path] + (DOG if "dog" in name else SPINKICK)
        lay = HostModel(margs, asset_root).layout()
        assert lay["frames"] == m["frames"].shape[0] and lay["loop"] == 0
        # the loaded frames: a reset at frame k's time (durations summed as the loader sums them) starts the simulated character in frame k
        # (root x, z moved to 0, the root raised off the ground if needed; quaternions normalised by the loader, fp32 on the device)
        F = m["frames"].shape[0]
        ks = np.unique(np.linspace(0, F - 1, 24).astype(int))
        times = np.concatenate([[0.0], np.cumsum(m["durations"][:-1])])[ks]
        core = BatchedCore(margs, len(ks), asset_root, device=0, seed=1)
        core.reset(True, kin_time=times, max_time=np.full(len(ks), 20.0), rot_theta=np.zeros(len(ks)))
        pose = torch.empty(len(ks), core.dims.pose_dim, device="cuda")
        core.record_pose(pose, None)
        core.sync()
        got, want = pose.cpu().numpy().astype(np.float64), m["frames"][ks]
        assert (got[:, 0] == 0).all() and (got[:, 2] == 0).all() and (got[:, 1] >= want[:, 1] - 1e-5).all()
        err = np.abs(got[:, 3:] - want[:, 3:]).max()
        assert err < 2e-5, (e, err, int(np.abs(got[:, 3:] - want[:, 3:]).argmax()))


def test_trainer_model_files_round_trip(asset_root, tmp_path):
    """a short run, saved; a new Trainer from that checkpoint (same TestEpisodes and seed) evaluates bit for bit as the source before any
    iteration; a Trainer started from the spin-kick policy's bundle evaluates far above random initialisation at iteration 0"""
    from deepmimic_b200.trainer import AgentConfig, Trainer
    from tests.test_train_gpu import AGENT
    v = AgentConfig(dict(AGENT, InitSamples=1, OutputIters=100, TestEpisodes=16))
    src = Trainer(SPINKICK_TRAIN, v, asset_root, 512, window_steps=8, backend="tensor_core", seed=7)
    for _ in range(3):
        src.iteration()
    path = str(tmp_path / "agent0_checkpoint.pt")
    src.save(path)
    want = src.evaluate()
    dst = Trainer(SPINKICK_TRAIN, v, asset_root, 512, window_steps=8, backend="tensor_core", seed=7, model_files=path)
    got = dst.evaluate()
    print("model files round trip: Test_Return %r (source) %r (loaded)" % (want, got))
    assert got == want
    pre = Trainer(SPINKICK_TRAIN, v, asset_root, 512, window_steps=8, backend="tensor_core", seed=7,
                  model_files=_bundle(tmp_path, _fixture("policy_humanoid3d_spinkick_fp16.npz")))
    row = pre.iteration()
    print("Trainer from the spin-kick policy: iteration 0 Test_Return %.3f" % row["Test_Return"])
    assert row["Test_Return"] > 100.0


def test_cli_resumes_a_run_started_from_model_files(asset_root, tmp_path):
    """python -m deepmimic_b200.train from a reference TensorBundle (--model_files on the command line): 2 iterations, then --resume with
    the same arguments to 4 gives the log a straight 4-iteration run writes (but wall time); --resume without --model_files is refused with
    an error that names the checkpoint's model files"""
    import json
    from deepmimic_b200.formats import read_table_log
    from tests.test_train_gpu import AGENT
    agent = tmp_path / "agent.txt"
    agent.write_text(json.dumps(dict(AGENT, OutputIters=1, TestEpisodes=4, InitSamples=1)))
    prefix = _bundle(tmp_path, _fixture("policy_humanoid3d_spinkick_fp16.npz"))
    base = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-m", "deepmimic_b200.train", "--asset_root", asset_root] + SPINKICK_TRAIN + [
        "--agent_files", str(agent), "--num_envs", "256", "--window_steps", "8"]
    env = dict(os.environ, PYTHONPATH=REPO)
    run = lambda out, extra: subprocess.run(base + ["--output_path", str(tmp_path / out)] + extra, cwd=str(tmp_path), env=env, capture_output=True, text=True)
    for out, extra in (("straight", ["--model_files", prefix, "--max_iters", "4"]), ("split", ["--model_files", prefix, "--max_iters", "2"]),
                       ("split", ["--model_files", prefix, "--max_iters", "4", "--resume", str(tmp_path / "split" / "agent0_checkpoint.pt")])):
        r = run(out, extra)
        assert r.returncode == 0, r.stderr[-3000:]
    a, b = read_table_log(str(tmp_path / "straight" / "agent0_log.txt")), read_table_log(str(tmp_path / "split" / "agent0_log.txt"))
    assert list(b["Iteration"]) == [0, 1, 2, 3]
    for k in a:
        if k != "Wall_Time":
            assert np.array_equal(a[k], b[k], equal_nan=True), k
    print("train from model files: Test_Return %s" % list(a["Test_Return"]))
    r = run("split", ["--max_iters", "5", "--resume", str(tmp_path / "split" / "agent0_checkpoint.pt")])
    assert r.returncode != 0 and "started from model files %s, this one from None" % prefix in r.stderr, r.stderr[-3000:]

