"""Expert AMP observations drawn on the device (dm_sample_amp_obs_expert, kernels/dm_policy.cu: dm_amp_expert_sample_kernel): every row is the
expert branch of dm_amp_obs_kernel at a clip and time drawn in the kernel, so with the draws returned it must equal dm_record_amp_obs_expert(_clips)
fed those draws bit for bit, and the oracle's RecordAMPObsExpert to the pose / velocity bounds of tests/amp_states.py.  The draws follow the dataset's sampling
weights and U(0, clip duration), move on with every call, repeat under the same seed, and the call enqueues without a host synchronisation (it
can be captured in a CUDA graph)."""
import numpy as np
import pytest

from tests import amp_states as A
from tests.oracle_binding import Oracle

pytestmark = pytest.mark.gpu

MINI = ["--motion_file", "data/datasets/test_clips_mini.txt"]
TARGET = MINI + ["--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]
IMITATE_AMP = ["--scene", "imitate_amp", "--arg_file", "args/train_humanoid3d_walk_args.txt"]
DOG_AMP = ["--scene", "imitate_amp", "--arg_file", "args/train_dog3d_trot_args.txt"]
SYN56 = ["--motion_file", "data/datasets/synthetic_locomotion_56.txt", "--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]
N = 40


def _core(asset_root, args, n=N, seed=7):
    """a handle whose environments were reset to known clip times, clips and ground heights (so the oracle can be put in the same state)"""
    from deepmimic_b200.capi import BatchedCore
    core = BatchedCore(args, n, asset_root, device=0, seed=seed)
    task = core.dims.goal_size > 0
    kin = np.linspace(0.05, 0.6, n)
    clip = (np.arange(n) % len(core.clip_table()[0])) if task else None
    core.reset(True, kin_time=kin, max_time=np.full(n, 20.0), rot_theta=np.zeros(n), clip=clip)
    return core, task, kin, clip


def _sample(core, rows):
    import torch
    out = torch.full((rows, core.dims.amp_obs_size), float("nan"), device="cuda")
    clip = torch.full((rows,), -1, dtype=torch.int32, device="cuda")
    time = torch.full((rows,), float("nan"), dtype=torch.float64, device="cuda")
    core.sample_amp_obs_expert(out, clip, time)
    core.sync()
    return out, clip, time


@pytest.mark.parametrize("scene,args", [("imitate_amp humanoid3d", IMITATE_AMP), ("imitate_amp dog3d", DOG_AMP), ("target_amp", TARGET)])
@pytest.mark.parametrize("rows", [17, N, 101])
def test_sampled_rows_replay_through_the_host_draw_entry(asset_root, scene, args, rows):
    """rows below, equal to and above num_envs, none a multiple of the block's tiles: row r is bit-identical to row r % N of
    dm_record_amp_obs_expert(_clips) given row r's clip and time, and matches the oracle's record_amp_obs_expert(time, clip) to the bounds of tests/amp_states.py"""
    import torch
    core, task, kin, rclip = _core(asset_root, args)
    out, clip, time = _sample(core, rows)
    clip, time = clip.cpu().numpy(), time.cpu().numpy()
    assert bool(torch.isfinite(out).all())
    dur, _ = core.clip_table() if task else (np.array([core.dims.motion_duration]), None)
    assert (clip >= 0).all() and (clip < len(dur)).all() and (task or (clip == 0).all())
    assert (time >= 0).all() and (time < dur[clip]).all()
    ref = torch.zeros(N, core.dims.amp_obs_size, device="cuda")
    for k in range(0, rows, N):
        n = min(N, rows - k)
        kt = np.full(N, 0.1); kt[:n] = time[k:k + n]
        kc = np.zeros(N, np.int32); kc[:n] = clip[k:k + n]
        core.amp_obs_expert(ref, kin_time=kt, clip=kc if task else None)
        core.sync()
        assert torch.equal(out[k:k + n], ref[:n]), (scene, rows, k)
    o = Oracle(args, asset_root)
    g = out.cpu().numpy().astype(np.float64)
    for r in list(range(min(rows, 12))) + [rows - 1]:
        e = r % N
        o.reset(float(kin[e]), 0.0, 20.0, **(dict(clip=int(rclip[e])) if task else {}))   # the expert's ground height is environment e's
        want = o.record_amp_obs_expert(float(time[r]), **(dict(clip=int(clip[r])) if task else {}))
        A.check_split(g[r], want, o.pose_dim, A.max_level(asset_root, "dog3d" if "dog" in scene else "humanoid3d"), (scene, r))
    core.close()


def test_clip_and_time_draws_follow_the_dataset(asset_root):
    """target_amp with the 56-clip dataset, 2^17 rows: the clip counts pass a chi-square test against the dataset's sampling weights and the
    times, as fractions of their clip's duration, a Kolmogorov-Smirnov test against U(0, 1)"""
    from scipy import stats
    core, _, _, _ = _core(asset_root, SYN56, n=256, seed=11)
    dur, cdf = core.clip_table()
    _, clip, time = _sample(core, 1 << 17)
    clip, time = clip.cpu().numpy(), time.cpu().numpy()
    w = np.diff(np.concatenate([[0.0], cdf]))
    counts = np.bincount(clip, minlength=len(dur))
    p_clip = stats.chisquare(counts, w / w.sum() * len(clip)).pvalue
    frac = time / dur[clip]
    assert frac.min() >= 0.0 and frac.max() < 1.0
    p_time = stats.kstest(frac, "uniform").pvalue
    print("chi-square p %.3g over %d clips, KS p %.3g" % (p_clip, len(dur), p_time))
    assert p_clip > 1e-3 and p_time > 1e-3
    core.close()


def test_draws_move_on_and_repeat_under_the_seed(asset_root):
    """two calls give different draws; a new handle with the same seed repeats both calls' rows; the call counter can be read and set back"""
    import torch
    core, _, _, _ = _core(asset_root, TARGET, seed=3)
    a, ca, ta = _sample(core, 70)
    b, cb, tb = _sample(core, 70)
    assert not torch.equal(ta, tb) and not torch.equal(a, b)
    assert core.expert_sample_count() == 2
    again, _, _, _ = _core(asset_root, TARGET, seed=3)
    a2, ca2, ta2 = _sample(again, 70)
    b2, cb2, tb2 = _sample(again, 70)
    assert torch.equal(a, a2) and torch.equal(ca, ca2) and torch.equal(ta, ta2)
    assert torch.equal(b, b2) and torch.equal(cb, cb2) and torch.equal(tb, tb2)
    assert again.expert_sample_count(set_to=1) == 2
    b3, _, tb3 = _sample(again, 70)
    assert torch.equal(b, b3) and torch.equal(tb, tb3)
    other, _, _, _ = _core(asset_root, TARGET, seed=4)
    assert not torch.equal(_sample(other, 70)[2], ta)
    for c in (core, again, other):
        c.close()


def test_sampler_is_captured_by_a_cuda_graph(asset_root):
    """the call only enqueues work on the handle's stream: it can be captured, and each replay writes the captured call's rows"""
    import torch
    core, _, _, _ = _core(asset_root, TARGET, seed=5)
    rows = 300
    out = torch.zeros(rows, core.dims.amp_obs_size, device="cuda")
    time = torch.zeros(rows, dtype=torch.float64, device="cuda")
    stream = torch.cuda.ExternalStream(core.stream())
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    c0 = core.expert_sample_count()
    with torch.cuda.graph(graph, stream=stream):
        core.sample_amp_obs_expert(out, None, time)
    out.zero_(); time.zero_()
    graph.replay()
    torch.cuda.synchronize()
    got, got_t = out.clone(), time.clone()
    core.expert_sample_count(set_to=c0)
    want, _, want_t = _sample(core, rows)
    assert torch.equal(got, want) and torch.equal(got_t, want_t) and bool(torch.isfinite(got).all())
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    core.close()


def test_env_sample_amp_obs_expert(asset_root):
    """DeepMimicBatchEnv.sample_amp_obs_expert(rows): a fresh [rows, amp_obs_size] tensor per call, ordered before the caller's stream, equal to
    the handle's call with the same counter"""
    import torch
    from deepmimic_b200.env import DeepMimicBatchEnv
    env = DeepMimicBatchEnv(IMITATE_AMP, 16, asset_root, seed=2)
    x = env.sample_amp_obs_expert(37)
    y = env.sample_amp_obs_expert(37)
    assert tuple(x.shape) == (37, env.get_amp_obs_size()) and x.data_ptr() != y.data_ptr()
    assert bool(torch.isfinite(x).all()) and not torch.equal(x, y)
    env._core.expert_sample_count(set_to=0)
    out = torch.zeros_like(x)
    env._core.sample_amp_obs_expert(out)
    env.sync()
    assert torch.equal(out, x)


@pytest.mark.parametrize("scene,args", [("imitate_amp dog3d", DOG_AMP), ("target_amp", TARGET)])
def test_sampler_writes_stay_inside_their_rows(asset_root, scene, args):
    """rows above num_envs and not a multiple of the block (W = 32 and W = 16 tiles): guard rows after the output and guard entries after the
    clip / time arrays keep their values, so the tail tiles write nothing past row rows - 1"""
    import torch
    core, _, _, _ = _core(asset_root, args)
    rows, pad, M = 53, 7, core.dims.amp_obs_size
    big = torch.full((rows + pad, M), 1234.5, device="cuda")
    bclip = torch.full((rows + pad,), -77, dtype=torch.int32, device="cuda")
    btime = torch.full((rows + pad,), -3.25, dtype=torch.float64, device="cuda")
    core.sample_amp_obs_expert(big[:rows], bclip[:rows], btime[:rows])
    core.sync()
    assert bool((big[rows:] == 1234.5).all()) and bool((bclip[rows:] == -77).all()) and bool((btime[rows:] == -3.25).all())
    assert bool(torch.isfinite(big[:rows]).all()) and bool((bclip[:rows] >= 0).all()) and bool((btime[:rows] >= 0).all())
    core.close()
