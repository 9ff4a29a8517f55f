"""The kinematic character's pose (dm_record_kin_pose) against the CPU oracle, the tracking-error kernels (dm_pose_error) against the float64
restatement of tests/pose_error_ref.py, and run --pose_error on the golden spin-kick policy."""
import numpy as np
import pytest

from tests import pose_error_ref as R
from tests.oracle_binding import Oracle
from tests.render_ref import Character
from tests.test_run_gpu import CASES, SPINKICK, _canon, _run_cmd
from tests.test_run_cpu import _bundle, _fixture

pytestmark = pytest.mark.gpu


def _random_run(core, host, N, steps, seed, resets=True):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    off = torch.as_tensor(-host.static(2), dtype=torch.float32, device="cuda")
    scl = torch.as_tensor(1.0 / host.static(3), dtype=torch.float32, device="cuda")
    for _ in range(steps):
        core.set_action((off + 0.25 * scl * torch.randn(N, core.dims.action_size, device="cuda", generator=g)).contiguous())
        core.update(1.0 / 600.0, core.dims.updates_per_action)
        if resets:
            core.reset(False)


@pytest.mark.parametrize("name,args,char", CASES, ids=[c[0] for c in CASES])
def test_kin_pose_matches_the_oracle(asset_root, name, args, char):
    """a padded batch of 1001 environments after 40 policy steps of random actions with resets: teacher-forced, every sampled environment's
    kinematic pose equals the oracle's get_kin_pose within fp32 rounding (w >= 0; the dataset scene with the oracle on the environment's clip);
    rows past N are not written; right after a reset the simulated and the kinematic character coincide (phase-locked distance < 1e-5 m)"""
    import torch
    from deepmimic_b200.capi import BatchedCore, HostModel, lib
    from tests.parity_util import joint_types_from_assets
    N = 1001
    core = BatchedCore(args, N, asset_root, device=0, seed=11)
    host = HostModel(args, asset_root)
    P = core.dims.pose_dim
    pose_off, jtypes = host.info("pose_offsets"), joint_types_from_assets(asset_root, char)
    orc = Oracle(args, asset_root)
    clips = name == "target_amp"
    if clips:   # every environment on a known clip of the dataset: injected at the reset, no resets after it
        nclip = len(core.clip_table()[0])
        clip = np.arange(N, dtype=np.int32) % nclip
        core.reset(True, kin_time=np.linspace(0.0, 3.0, N), max_time=np.full(N, 100.0), rot_theta=np.linspace(-3.0, 3.0, N), clip=clip)
    else:
        core.reset(True)
    _random_run(core, host, N, 40, 3, resets=not clips)
    big = torch.full((N + 7, P), float("nan"), device="cuda")
    assert lib().dm_record_kin_pose(core.h, big.data_ptr()) == 0
    kin = torch.empty(N, P, device="cuda")
    core.record_kin_pose(kin)
    core.sync()
    assert torch.isnan(big[N:]).all() and torch.equal(big[:N], kin)
    kin = kin.cpu().numpy()
    worst = 0.0
    for e in list(range(0, N, 37)) + [N - 1]:
        snap = core.get_snapshot(e)
        if clips:
            orc.reset(0.0, 0.0, 100.0, clip=int(clip[e]))
        orc.set_snapshot(snap)
        ko = orc.get_kin_pose()[0]
        assert kin[e, 3] >= 0 and all(kin[e, pose_off[j]] >= 0 for j, t in enumerate(jtypes) if j > 0 and t == "spherical")
        worst = max(worst, np.abs(_canon(ko, pose_off, jtypes) - kin[e]).max())
    print("%s: record_kin_pose against the oracle, max error %.2e" % (name, worst))
    assert worst < 2e-5
    # right after a forced reset the two characters coincide
    core.reset(True)
    sim, kin = torch.empty(N, P, device="cuda"), torch.empty(N, P, device="cuda")
    core.record_pose(sim, None)
    core.record_kin_pose(kin)
    lock, dtw = core.pose_error(sim[None].contiguous(), kin[None].contiguous(), torch.ones(N, dtype=torch.int32, device="cuda"))
    core.sync()
    print("%s: after a reset, worst phase-locked distance %.2e m" % (name, float(lock.max())))
    assert float(lock.max()) < 1e-5 and torch.equal(lock, dtw)
    core.close()


# ---------------------------------------------------------------------------------------------------------------- the error kernels
CHARS = [("humanoid3d", ["--arg_file", "args/run_humanoid3d_spinkick_args.txt"], "data/characters/humanoid3d.txt"),
         ("dog3d", ["--arg_file", "args/run_dog3d_trot_args.txt"], "data/characters/dog3d.txt")]


def _sequences(core, host, n, T, seed):
    """[T, n, P] simulated and kinematic poses of n environments under random actions with resets"""
    import torch
    P = core.dims.pose_dim
    a, r = torch.empty(T, n, P, device="cuda"), torch.empty(T, n, P, device="cuda")
    core.reset(True)
    for t in range(T):
        core.record_pose(a[t], None)
        core.record_kin_pose(r[t])
        _random_run(core, host, n, 1, seed + t)
    core.sync()
    return a, r


@pytest.mark.parametrize("name,args,char", CHARS, ids=[c[0] for c in CHARS])
def test_pose_error_matches_the_restatement(asset_root, name, args, char):
    """lengths 1, 2, 33, 600 and 1500 (over the block's 128 rows: strip boundaries) against the float64 restatement within 1e-4 relative +
    1e-6 m; NaN for lengths 0, -3 and T + 1; bit-identical on a repeat, alone against in the batch, and with a and r swapped; refusals"""
    import torch
    from deepmimic_b200.capi import BatchedCore, HostModel, lib
    T, lens = 1500, [1, 2, 33, 600, 1500, 0, -3, 1501]
    n = len(lens)
    core = BatchedCore(args, n, asset_root, device=0, seed=5)
    host = HostModel(args, asset_root)
    a, r = _sequences(core, host, n, T, 7)
    L = torch.tensor(lens, dtype=torch.int32, device="cuda")
    lock, dtw = core.pose_error(a, r, L)
    lock2, dtw2 = core.pose_error(a, r, L)
    slock, sdtw = core.pose_error(r, a, L)
    core.sync()
    same = lambda x, y: torch.equal(x.view(torch.int32), y.view(torch.int32))   # bit for bit, NaN included
    assert same(lock, lock2) and same(dtw, dtw2)
    assert same(lock, slock) and same(dtw, sdtw)
    for e in range(n):
        one_l, one_d = core.pose_error(a[:, e:e + 1].contiguous(), r[:, e:e + 1].contiguous(), L[e:e + 1].contiguous())
        core.sync()
        assert same(one_l, lock[e:e + 1]) and same(one_d, dtw[e:e + 1]), e
    ch = Character(asset_root, char)
    an, rn = a.cpu().double().numpy(), r.cpu().double().numpy()
    gl, gd = lock.cpu().numpy(), dtw.cpu().numpy()
    worst = 0.0
    for e, l in enumerate(lens):
        if not 1 <= l <= T:
            assert np.isnan(gl[e]) and np.isnan(gd[e]), (e, l)
            continue
        fa = np.stack([R.features(ch, p) for p in an[:l, e]]); fr = np.stack([R.features(ch, p) for p in rn[:l, e]])
        d = R.distance_matrix(fa, fr)
        want_l = float(np.mean(np.diag(d)))
        want_d = R.dtw(d) if l <= 600 else None
        assert abs(gl[e] - want_l) <= 1e-4 * want_l + 1e-6, (l, gl[e], want_l)
        worst = max(worst, abs(gl[e] - want_l) / max(want_l, 1e-6))
        if want_d is not None:
            assert abs(gd[e] - want_d) <= 1e-4 * want_d + 1e-6, (l, gd[e], want_d)
            worst = max(worst, abs(gd[e] - want_d) / max(want_d, 1e-6))
        assert gd[e] <= gl[e], (l, gd[e], gl[e])
    print("%s: pose error against the restatement, worst relative error %.2e" % (name, worst))
    # refusals by name
    for T_, n_, pa, pr, pl, what in ((0, n, a, r, L, "T 0"), (T, 0, a, r, L, "n 0"), (T, n, None, r, L, "d_a is NULL"), (T, n, a, None, L, "d_r is NULL"),
                                     (T, n, a, r, None, "d_len is NULL")):
        ptr = lambda t: t.data_ptr() if t is not None else None
        assert lib().dm_pose_error(core.h, T_, n_, ptr(pa), ptr(pr), ptr(pl), lock.data_ptr(), None) != 0
        assert what in lib().dm_last_error().decode(), lib().dm_last_error()
    core.close()


def test_dtw_forgives_a_lag(asset_root):
    """the kinematic sequence of a run of L + 3 steps against itself 3 frames late: the warped error is a small part of the phase-locked one"""
    import torch
    from deepmimic_b200.capi import BatchedCore, HostModel
    args = CHARS[0][1]
    n, L, k = 16, 200, 3
    core = BatchedCore(args, n, asset_root, device=0, seed=5)
    host = HostModel(args, asset_root)
    _, r = _sequences(core, host, n, L + k, 9)
    lock, dtw = core.pose_error(r[k:].contiguous(), r[:L].contiguous(), torch.full((n,), L, dtype=torch.int32, device="cuda"))
    core.sync()
    print("lag of %d frames: phase-locked %s, warped %s" % (k, lock.cpu().numpy().round(4), dtw.cpu().numpy().round(4)))
    assert (dtw < 0.25 * lock).all() and (lock > 0.0).all()
    core.close()


def test_run_pose_error_on_the_spinkick_policy(asset_root, tmp_path):
    """run --pose_error on the golden spin-kick policy: both columns, e_dtw <= e_lock per episode, a mean e_lock below a randomly
    initialised actor's on the same arguments"""
    import torch
    from deepmimic_b200.env import DeepMimicBatchEnv
    from deepmimic_b200.formats import read_table_log
    from deepmimic_b200.rollout import BatchedRollout, run_episodes
    n = 32
    prefix = _bundle(tmp_path, _fixture("policy_humanoid3d_spinkick_fp16.npz"))
    out = tmp_path / "out"
    stdout = _run_cmd(asset_root, SPINKICK + ["--pose_error"], prefix, out, n, 0)
    print(stdout.strip())
    log = read_table_log(str(out / "run_log.txt"))
    lock, dtw = np.asarray(log["Pose_Err"]), np.asarray(log["Pose_Err_DTW"])
    assert len(lock) == n and np.isfinite(lock).all() and (dtw <= lock).all() and (lock > 0).all()
    assert "pose error" in stdout and "time-warped" in stdout
    torch.manual_seed(0)
    env = DeepMimicBatchEnv(SPINKICK + ["--time_end_lim_min", "20.0", "--time_end_lim_max", "20.0"], n, asset_root, seed=0)
    env.set_mode(1)
    env.reset(True)
    ro = BatchedRollout(env, exp_rate=0.0, seed=0, backend="tensor_core")
    ep = run_episodes(ro, pose_error=True)
    rand_lock = float(ep["pose_err"].mean())
    print("spin kick: policy pose error %.4f m (DTW %.4f m), random actor %.4f m" % (lock.mean(), dtw.mean(), rand_lock))
    assert (ep["pose_err_dtw"] <= ep["pose_err"]).all() and lock.mean() < rand_lock
