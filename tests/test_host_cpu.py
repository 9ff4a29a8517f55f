"""CPU-side tests (no GPU): the C-ABI library loads and exports what include/deepmimic_b200.h declares, the host loaders
agree with the oracle's independent loaders, compute entry points fail loudly without a device, the cDeepMimicCore facade
exposes the reference's SWIG surface, and the N>1 sharding / exchange logic works under gloo with world_size 2."""
import ctypes as C
import os
import re
import socket

import numpy as np
import pytest

from deepmimic_b200 import capi
from deepmimic_b200.sharding import StepExchange, pack_rows, shard_range
from tests.oracle_binding import Oracle

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARG_FILES = ["args/train_humanoid3d_spinkick_args.txt", "args/train_humanoid3d_walk_args.txt", "args/train_humanoid3d_backflip_args.txt",
             "args/train_dog3d_trot_args.txt"]


def header_functions():
    src = open(os.path.join(REPO, "include", "deepmimic_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dm_[a-z_0-9]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    L = capi.lib()
    names = header_functions()
    assert len(names) >= 20
    for n in names:
        assert hasattr(L, n), "libdeepmimic_b200.so does not export %s" % n
    assert sorted(capi.EXPORTS) == names, "capi.EXPORTS and the header disagree: %s" % (set(capi.EXPORTS) ^ set(names))


def test_header_cites_reference_for_each_entry_point():
    src = open(os.path.join(REPO, "include", "deepmimic_b200.h")).read()
    assert src.count("DeepMimicCore.") >= 10 and "extern \"C\"" in src
    assert "torch" not in src.lower().replace("torch tensors", "")   # plain pointers and sizes only


@pytest.mark.parametrize("arg_file", ARG_FILES)
def test_host_loader_matches_oracle_loader(asset_root, arg_file):
    m = capi.HostModel(["--arg_file", arg_file], asset_root)
    o = Oracle(["--arg_file", arg_file], asset_root)
    assert m.dims.num_joints == o.num_joints and m.dims.pose_dim == o.pose_dim
    assert m.dims.state_size == o.state_size and m.dims.action_size == o.action_size
    assert m.dims.snapshot_size == o.snapshot_size and m.layout()["frames"] == o.num_frames
    assert abs(m.dims.motion_duration - o.motion_duration) < 1e-12
    st = o.action_statics()
    for kind, ref in zip((capi.DM_ACTION_OFFSET, capi.DM_ACTION_SCALE, capi.DM_ACTION_BOUND_MIN, capi.DM_ACTION_BOUND_MAX), st):
        np.testing.assert_allclose(m.static(kind), ref, rtol=0, atol=1e-12)
    par = m.info("parents")
    assert par[0] == -1 and all(0 <= par[j] < j for j in range(1, len(par)))
    lay = m.layout()
    assert lay["links"] == m.dims.num_joints and lay["dofs"] == m.dims.num_dofs and lay["loop"] == 1
    # state normalisation statics: phase slot only (CtController.cpp:54-69)
    off, scl, grp = m.static(capi.DM_STATE_OFFSET), m.static(capi.DM_STATE_SCALE), m.static(capi.DM_STATE_NORM_GROUPS)
    assert off[0] == -0.5 and scl[0] == 2.0 and grp[0] == -1 and not off[1:].any() and (scl[1:] == 1).all() and not grp[1:].any()


def test_humanoid_layout_constants(asset_root):
    m = capi.HostModel(["--arg_file", ARG_FILES[0]], asset_root)
    assert (m.dims.num_joints, m.dims.pose_dim, m.dims.num_dofs, m.dims.state_size, m.dims.action_size) == (15, 43, 34, 197 + 30, 36 - 8)
    assert m.dims.updates_per_action == 20 and m.dims.num_update_substeps == 10   # --num_update_substeps of the arg file (DeepMimicCore.cpp:236)
    assert list(m.info("end_effectors").nonzero()[0]) == [5, 8, 11, 14]
    fall = m.info("fall_bodies")
    assert fall[0] == 1 and fall[5] == 0 and fall[11] == 0       # feet may touch the ground (--fall_contact_bodies)


def test_loader_errors_are_reported(asset_root):
    L = capi.lib()
    with pytest.raises(RuntimeError, match="Failed to load args"):
        capi.HostModel(["--arg_file", "args/does_not_exist.txt"], asset_root)
    with pytest.raises(RuntimeError):
        capi.HostModel(["--scene", "imitate", "--character_files", "data/characters/nope.txt"], asset_root)
    with pytest.raises(RuntimeError, match="Unsupported scene"):
        capi.HostModel(["--scene", "dribble_amp", "--arg_file", ARG_FILES[0]], asset_root)     # first key wins: the scene is overridden
    for extra, msg in ((["--char_ctrls", "ct_vel"], "Unsupported character controller"), (["--enable_char_soft_contact", "true"], "enable_char_soft_contact"),
                       (["--enable_root_rot_fail", "true"], "enable_root_rot_fail"), (["--char_types", "biped3d"], "Unsupported character type"),
                       (["--character_files", "data/characters/humanoid3d.txt", "data/characters/dog3d.txt"], "more than one character"),
                       (["--sync_char_root_rot", "true", "--motion_file", "data/datasets/test_clips_mini.txt", "--arg_file",
                         "args/train_amp_target_humanoid3d_locomotion_args.txt"], "sync_char_root_rot true in an AMP task scene")):
        with pytest.raises(RuntimeError, match=msg):
            capi.HostModel(extra + ["--arg_file", ARG_FILES[0]], asset_root)
    with pytest.raises(RuntimeError, match="Unsupported timer type"):
        capi.HostModel(["--timer_type", "exp", "--arg_file", ARG_FILES[0]], asset_root)
    m = capi.HostModel(["--scene", "imitate_amp", "--arg_file", ARG_FILES[0]], asset_root)       # the AMP variant of the imitate scene loads
    assert m.dims.amp_obs_size == 226
    assert L.dm_last_error()


def test_sample_count_anneals_episode_time_limits(asset_root):
    """cRLSceneSimChar::UpdateTimerParams (RLSceneSimChar.cpp:330-347): Blend(params, params_end, clamp(count / anneal, 0, 1)^4)."""
    m = capi.HostModel(["--arg_file", ARG_FILES[0]], asset_root)     # time_lim 0.5 -> 20 over --anneal_samples 32000000
    np.testing.assert_allclose(m.time_limits(), [0.5, 0.5, 20.0])
    for count, t in [(0, 0.0), (8000000, 0.25), (16000000, 0.5), (32000000, 1.0), (10 ** 9, 1.0), (-5, 0.0)]:
        m.set_sample_count(count)
        want = 0.5 + (20.0 - 0.5) * t ** 4
        np.testing.assert_allclose(m.time_limits(), [want, want, 20.0], rtol=1e-14)
    # different min / max; and no --anneal_samples: the count is ignored
    m = capi.HostModel(["--time_lim_min", "1", "--time_lim_max", "3", "--time_end_lim_min", "5", "--time_end_lim_max", "11", "--anneal_samples", "100",
                        "--arg_file", ARG_FILES[0]], asset_root)
    m.set_sample_count(50)
    np.testing.assert_allclose(m.time_limits(), [1 + 4 / 16.0, 3 + 8 / 16.0, 11.0], rtol=1e-14)
    m = capi.HostModel(["--anneal_samples", "-1", "--arg_file", ARG_FILES[0]], asset_root)
    m.set_sample_count(10 ** 8)
    np.testing.assert_allclose(m.time_limits(), [0.5, 0.5, 20.0])


def test_compute_entry_points_fail_loudly_without_device(asset_root):
    """No CPU fallback: a host-only handle refuses every compute call; dm_create refuses when no CUDA device exists."""
    L = capi.lib()
    m = capi.HostModel(["--arg_file", ARG_FILES[0]], asset_root)
    assert L.dm_update(m.h, 1.0 / 600.0, 1) != 0 and b"no CPU fallback" in L.dm_last_error()
    assert L.dm_reset(m.h, 1, None, None, None) != 0
    assert L.dm_observe(m.h, None, None) != 0
    assert L.dm_step_host(m.h, None, 0.0, 0, None, None, None) != 0
    assert L.dm_sync(m.h) != 0
    import torch
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CUDA device|CUDA|cuda"):
            capi.BatchedCore(["--arg_file", ARG_FILES[0]], 4, asset_root)


REFERENCE_CORE_METHODS = """SeedRand ParseArgs Init Update Reset GetTime GetName EnableDraw Draw Keyboard MouseClick MouseMove Reshape Shutdown IsDone
SetPlaybackSpeed SetUpdatesPerSec GetWinWidth GetWinHeight GetNumUpdateSubsteps IsRLScene GetNumAgents NeedNewAction RecordState RecordGoal
SetAction LogVal GetActionSpace GetStateSize GetGoalSize GetActionSize GetNumActions BuildStateOffset BuildStateScale BuildGoalOffset
BuildGoalScale BuildActionOffset BuildActionScale BuildActionBoundMin BuildActionBoundMax BuildStateNormGroups BuildGoalNormGroups CalcReward
GetRewardMin GetRewardMax GetRewardFail GetRewardSucc EnableAMPTaskReward GetAMPObsSize GetAMPObsOffset GetAMPObsScale GetAMPObsNormGroup
RecordAMPObsExpert RecordAMPObsAgent IsEpisodeEnd CheckValidEpisode CheckTerminate SetMode SetSampleCount""".split()


def test_facade_module_mirrors_reference_surface():
    """The names are the public methods of cDeepMimicCore (R/DeepMimicCore/DeepMimicCore.h:12-88)."""
    import sys
    sys.path.insert(0, os.path.join(REPO, "deepmimic_b200"))
    try:
        from DeepMimicCore import DeepMimicCore
    finally:
        sys.path.pop(0)
    core = DeepMimicCore.cDeepMimicCore(False)
    for n in REFERENCE_CORE_METHODS:
        assert callable(getattr(core, n)), n
    assert core.GetNumAgents() == 1 and core.IsRLScene() and core.GetName() == "Imitate" and not core.EnableDraw()
    import torch
    if not torch.cuda.is_available():
        core.ParseArgs(["--arg_file", ARG_FILES[0], "--asset_root", "/nonexistent"])
        with pytest.raises(RuntimeError):
            core.Init()


# ---- sharding
def test_shard_range_partitions_exactly():
    for total in (0, 1, 7, 4096, 4097, 32768):
        for world in (1, 2, 3, 4, 8):
            spans = [shard_range(total, r, world) for r in range(world)]
            assert spans[0][0] == 0 and sum(c for _, c in spans) == total
            for (o0, c0), (o1, _) in zip(spans, spans[1:]):
                assert o0 + c0 == o1
            cs = [c for _, c in spans]
            assert max(cs) - min(cs) <= 1
    with pytest.raises(ValueError):
        shard_range(8, 2, 2)


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _exchange_worker(rank, world, port, total, width, q):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        off, cnt = shard_range(total, rank, world)
        x = StepExchange(total, width, rank, world, "cpu")
        S = width - 2
        ids = torch.arange(off, off + cnt, dtype=torch.float32)
        obs = ids[:, None] * 10 + torch.arange(S, dtype=torch.float32)[None, :]          # row content is a function of the GLOBAL env id
        rows = pack_rows(torch.zeros(cnt, width), obs, ids * 0.5, (ids.long() % 3 == 0))
        for _ in range(3):
            g = x.gather(rows).clone()
        # timing rule of bench.py: max over ranks
        t = torch.tensor([float(rank + 1)], dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        q.put((rank, g.numpy(), float(t.item())))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("total", [8, 7])   # even shards and ragged shards
def test_step_exchange_gloo_world2(total):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port, world, width = _free_port(), 2, 6
    procs = [ctx.Process(target=_exchange_worker, args=(r, world, port, total, width, q)) for r in range(world)]
    [p.start() for p in procs]
    got = [q.get(timeout=120) for _ in range(world)]
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    ids = np.arange(total, dtype=np.float32)
    expect = np.concatenate([ids[:, None] * 10 + np.arange(width - 2)[None, :], (ids * 0.5)[:, None], (ids.astype(int) % 3 == 0)[:, None]], axis=1)
    for rank, g, tmax in got:
        np.testing.assert_array_equal(g[:total], expect)      # every rank sees the whole job, in global env order
        assert tmax == 2.0


class _MockCore:
    """stands in for BatchedCore in the CPU tests of the exchange classes: observe / flags fill rows that are functions of the GLOBAL env id"""

    def __init__(self, off, cnt, S):
        self.off, self.cnt, self.S, self.step = off, cnt, S, 0

    def observe(self, obs, rew):
        import torch
        ids = torch.arange(self.off, self.off + self.cnt, dtype=torch.float32)
        obs.copy_(ids[:, None] * 10 + torch.arange(self.S, dtype=torch.float32)[None, :] + 1000.0 * self.step)
        rew.copy_(ids * 0.5 + self.step)

    def flags(self, out):
        import torch
        ids = torch.arange(self.off, self.off + self.cnt)
        out.zero_()
        out[:, 1] = ((ids + self.step) % 3 == 0).to(out.dtype)


def _rows_worker(rank, world, port, N, S, q):
    import torch
    import torch.distributed as dist
    from deepmimic_b200.sharding import make_exchange
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        core = _MockCore(rank * N, N, S)
        x = make_exchange("nccl", core, N, S, rank, world, "cpu")      # NcclRows; the backend of the process group decides the transport
        out = []
        for step in range(3):
            core.step = step
            x.publish(step)
            if step > 0:
                x.consume(step - 1)
            o, r, d = x.rows(step)
            out.append((o.clone().numpy(), r.clone().numpy(), d.clone().numpy()))
        q.put((rank, out))
    finally:
        dist.destroy_process_group()


def test_rows_exchange_in_place_all_gather_gloo_world2():
    """NcclRows (the collective variant of the policy-step exchange, bench.py --exchange nccl): planes layout, the local observe output is
    this rank's slice of the gathered buffer, one in-place all-gather per step.  Every rank must see every rank's rows of the step."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port, world, N, S = _free_port(), 2, 5, 4
    procs = [ctx.Process(target=_rows_worker, args=(r, world, port, N, S, q)) for r in range(world)]
    [p.start() for p in procs]
    got = [q.get(timeout=120) for _ in range(world)]
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    ids = np.arange(world * N, dtype=np.float32)
    for rank, out in got:
        for step, (o, r, d) in enumerate(out):
            assert o.shape == (world, N, S) and r.shape == (world, N) and d.shape == (world, N)
            np.testing.assert_array_equal(o.reshape(world * N, S), ids[:, None] * 10 + np.arange(S)[None, :] + 1000.0 * step)
            np.testing.assert_array_equal(r.reshape(-1), ids * 0.5 + step)
            np.testing.assert_array_equal(d.reshape(-1), ((ids.astype(int) + step) % 3 == 0).astype(np.float32))


def test_malformed_assets_are_rejected_with_messages(asset_root, tmp_path):
    """Ragged / empty / mismatching inputs: the loaders of the C-ABI library and of the oracle refuse them with the reference's messages
    (cMotion::LoadJson Motion.cpp:104-141,303-360; cKinTree::Load KinTree.cpp:204-258; cClipsController::LoadMotions ClipsController.cpp:145-188)."""
    import json
    walk = json.load(open(os.path.join(asset_root, "data/motions/humanoid3d_walk.txt")))
    char = json.load(open(os.path.join(asset_root, "data/characters/humanoid3d.txt")))

    def write(name, obj):
        p = os.path.join(str(tmp_path), name)
        json.dump(obj, open(p, "w"))
        return p

    base = ["--arg_file", ARG_FILES[1]]
    ragged = dict(walk); ragged["Frames"] = [f[:] for f in walk["Frames"][:5]]; ragged["Frames"][3] = ragged["Frames"][3][:-2]
    cases = [
        (["--motion_file", write("ragged.txt", ragged)], "ragged frame"),
        (["--motion_file", write("empty.txt", {"Loop": "wrap", "Frames": []})], "Failed to load motion"),
        (["--motion_file", write("noframes.txt", {"Loop": "wrap"})], "Failed to load motion"),
        (["--motion_file", write("badloop.txt", {"Loop": "sometimes", "Frames": walk["Frames"][:4]})], "Unsupported loop mode"),
        (["--motion_file", os.path.join(asset_root, "data/motions/dog3d_trot.txt")], "DOF mismatch"),
    ]
    bad_char = json.loads(json.dumps(char)); bad_char["Skeleton"]["Joints"][3]["Type"] = "ball_and_socket"
    cases.append((["--character_files", write("badjoint.txt", bad_char)], "Unsupported joint type"))
    bad_char = json.loads(json.dumps(char)); bad_char["BodyDefs"] = bad_char["BodyDefs"][:-1]
    cases.append((["--character_files", write("fewbodies.txt", bad_char)], "joint / body count mismatch"))
    bad_char = json.loads(json.dumps(char)); bad_char["Skeleton"]["Joints"][2]["Parent"] = 7
    cases.append((["--character_files", write("badparent.txt", bad_char)], "Parent id must be"))
    open(os.path.join(str(tmp_path), "notjson.txt"), "w").write("{ this is not json")
    cases.append((["--character_files", os.path.join(str(tmp_path), "notjson.txt")], None))
    for extra, msg in cases:
        with pytest.raises(RuntimeError, match=msg):
            capi.HostModel(extra + base, asset_root)
        with pytest.raises(RuntimeError, match=msg):
            Oracle(extra + base, asset_root)
    # clip datasets (oracle; the C-ABI loader takes them in the task scenes only)
    ds_missing = write("ds_missing.txt", {"Motions": [{"File": "data/motions/humanoid3d_walk.txt"}, {"File": "data/motions/nope.txt"}]})
    ds_empty = write("ds_empty.txt", {"Motions": []})
    for ds in (ds_missing, ds_empty, write("ds_nokey.txt", {"Clips": []})):
        with pytest.raises(RuntimeError):
            Oracle(["--kin_ctrl", "clips", "--motion_file", ds] + base, asset_root)


@pytest.mark.parametrize("arg_file,envs,width,per_block,h100_per_block,rows", [("args/train_humanoid3d_spinkick_args.txt", 4096, 16, 28, 16, 32),
                                                                                ("args/train_dog3d_trot_args.txt", 2048, 32, 14, 8, 52),
                                                                                ("args/train_amp_target_humanoid3d_locomotion_args.txt", 4096, 16, 28, 16, 32)])
def test_launch_plan_of_the_baseline_configurations_spreads_evenly_over_the_fewest_waves(asset_root, arg_file, envs, width, per_block, h100_per_block, rows):
    """dm_plan_launch (host arithmetic of dm_create): with 227 KB of shared memory per block, per_block environments fill a block.  On a device
    with 148 SMs the BASELINE.json configurations are ONE wave of full blocks -- dog3d only since its row capacity went from 60 to 52 (171
    blocks in two waves before); on the 132 SMs of an H100 they need two waves, and the environments are spread evenly over both
    (h100_per_block each: a wave takes as long as its fullest block).  The 16-byte alignment the kernels' 128-bit accesses rely on holds, and a device with
    too little shared memory is refused with an error."""
    from deepmimic_b200.capi import HostModel
    extra = ["--motion_file", "data/datasets/synthetic_locomotion_56.txt"] if "_amp_" in arg_file else []
    hm = HostModel(extra + ["--arg_file", arg_file], asset_root)
    p = hm.plan_launch(envs, num_sms=148)
    assert p["tile_width"] == width and p["envs_per_block"] == per_block and p["max_rows"] == rows
    assert p["blocks"] <= 148 and p["blocks"] * p["envs_per_block"] == p["padded_envs"] >= envs
    h = hm.plan_launch(envs)                             # H100 SXM: 132 SMs
    assert h["tile_width"] == width and h["envs_per_block"] == h100_per_block and h["max_rows"] == rows
    assert 132 < h["blocks"] <= 2 * 132 and h["blocks"] * h["envs_per_block"] == h["padded_envs"] >= envs
    assert p["smem_bytes"] <= 232448
    assert p["env_floats"] % 16 == 0 and p["hot_floats"] % 4 == 0 and p["y_offset"] % 4 == 0
    assert p["smem_bytes"] == 4 * (p["hot_floats"] + p["envs_per_block"] * p["env_floats"]) + 1024
    half = hm.plan_launch(envs // 8)                     # fewer environments: fewer per block, still whole warps for the 16-lane tiles
    assert half["envs_per_block"] <= per_block and (width == 32 or half["envs_per_block"] % 2 == 0)
    with pytest.raises(RuntimeError):
        hm.plan_launch(envs, smem_bytes_per_block=8 * 1024)
