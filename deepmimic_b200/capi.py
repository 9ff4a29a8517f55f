"""ctypes binding of the C ABI (include/deepmimic_b200.h).  Device buffers are torch CUDA tensors; torch is only
the allocator / stream plumbing here.  Raises if the CUDA library is missing -- there is no CPU fallback."""
import ctypes as C
import os

import numpy as np

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB_PATH = os.environ.get("DM_LIB", os.path.join(_REPO, "deepmimic_b200", "libdeepmimic_b200.so"))   # DM_LIB: profile build (tools/section_profile.py)
_lib = None


class DmDims(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("num_envs", "num_joints", "pose_dim", "num_dofs", "state_size", "goal_size", "action_size", "snapshot_size",
                                        "updates_per_action", "num_update_substeps")] + [("motion_duration", C.c_double), ("amp_obs_size", C.c_int)]


_fp = C.POINTER(C.c_float)


class DmMlpGatedWeights(C.Structure):
    """dm_mlp_gated_weights of include/deepmimic_b200.h"""
    _fields_ = ([(n, C.c_int) for n in ("in_dim", "goal_dim", "h0", "h1", "out_dim", "gate_common", "gate_hidden")]
                + [(n, _fp) for n in ("w0", "b0", "w1", "b1", "w2", "b2", "gc_w", "gc_b")]
                + [(n, _fp * 2) for n in ("gh_w", "gh_b", "gs_w", "gs_b", "gb_w", "gb_b")]
                + [(n, _fp) for n in ("s_mean", "s_std", "g_mean", "g_std", "a_mean", "a_std")] + [("s_clip", C.c_float), ("g_clip", C.c_float)])


class DmLearnNet(C.Structure):
    """dm_learn_net of include/deepmimic_b200.h"""
    _fields_ = [(n, C.c_void_p * 3) for n in ("w", "b", "acc_w", "acc_b")]


class DmLearnBatch(C.Structure):
    """dm_learn_batch of include/deepmimic_b200.h"""
    _fields_ = ([("states", C.c_void_p), ("idx", C.c_void_p), ("rows", C.c_int), ("in_mean", C.c_void_p), ("in_istd", C.c_void_p), ("in_clip", C.c_float)]
                + [(n, C.c_void_p) for n in ("norm_actions", "old_logp", "adv", "logstd", "bound_min", "bound_max")]
                + [("ratio_clip", C.c_float), ("ratio", C.c_void_p), ("norm_targets", C.c_void_p)]
                + [(n, C.c_float) for n in ("stepsize", "momentum", "weight_decay")] + [("stats", C.c_void_p)])


class DmLearnDiscBatch(C.Structure):
    """dm_learn_disc_batch of include/deepmimic_b200.h"""
    _fields_ = ([(n, C.c_void_p) for n in ("agent", "expert", "agent_idx", "expert_idx")] + [("rows", C.c_int), ("in_mean", C.c_void_p),
                ("in_istd", C.c_void_p), ("in_clip", C.c_float)]
                + [(n, C.c_float) for n in ("stepsize", "momentum", "weight_decay", "logit_reg_weight", "grad_penalty_weight")] + [("stats", C.c_void_p)])


class DmLearnGatedNet(C.Structure):
    """dm_learn_gated_net of include/deepmimic_b200.h"""
    _fields_ = [(n, C.c_void_p * 10) for n in ("w", "b", "acc_w", "acc_b")]


class DmLearnGatedBatch(C.Structure):
    """dm_learn_gated_batch of include/deepmimic_b200.h; the dm_learn_batch fields read and write through it"""
    _anonymous_ = ("batch",)
    _fields_ = [("batch", DmLearnBatch), ("goals", C.c_void_p), ("g_mean", C.c_void_p), ("g_istd", C.c_void_p), ("g_clip", C.c_float)]


DM_STATE_OFFSET, DM_STATE_SCALE, DM_ACTION_OFFSET, DM_ACTION_SCALE, DM_ACTION_BOUND_MIN, DM_ACTION_BOUND_MAX, DM_STATE_NORM_GROUPS = range(7)

class DmCamera(C.Structure):
    _fields_ = [("yaw", C.c_float), ("pitch", C.c_float), ("distance", C.c_float), ("target_height", C.c_float), ("fov_y", C.c_float)]


EXPORTS = ["dm_create", "dm_load_host", "dm_plan_launch", "dm_get_model_info", "dm_get_link_table", "dm_destroy", "dm_last_error", "dm_get_dims", "dm_get_static", "dm_get_scene_name", "dm_stream", "dm_sync", "dm_set_mode", "dm_set_sample_count", "dm_get_time_limits", "dm_reset", "dm_set_action",
           "dm_update", "dm_set_pushes", "dm_get_pushes", "dm_set_push_schedule", "dm_get_push_table", "dm_set_dynamics", "dm_get_dynamics", "dm_set_dynamics_randomization", "dm_set_action_latency", "dm_set_action_latency_randomization", "dm_get_action_latency", "dm_set_goal_course", "dm_get_course_record", "dm_set_env_order", "dm_plan_env_order", "dm_get_env_order", "dm_record_state", "dm_record_goal", "dm_record_pose", "dm_render_poses", "dm_render_poses_marked", "dm_record_kin_pose", "dm_pose_error", "dm_goal_host", "dm_reset_clips", "dm_record_amp_obs_expert_clips", "dm_get_clip_table", "dm_get_task_state", "dm_set_task_state", "dm_get_task_params", "dm_calc_reward", "dm_calc_reward_imitate", "dm_record_amp_obs_agent", "dm_record_amp_obs_expert", "dm_amp_obs_host", "dm_sample_amp_obs_expert", "dm_expert_sample_count", "dm_observe", "dm_get_flags", "dm_step_host", "dm_step_host_reset", "dm_set_time_limits", "dm_exchange_create", "dm_exchange_connect", "dm_exchange_publish", "dm_exchange_acquire", "dm_exchange_release", "dm_exchange_status", "dm_exchange_destroy", "dm_set_timing", "dm_step_host_timing", "dm_get_snapshot",
           "dm_set_snapshot", "dm_state_size", "dm_save_state", "dm_load_state", "dm_get_counters", "dm_get_section_profile", "dm_mlp_create", "dm_mlp_forward", "dm_mlp_create_gated", "dm_mlp_forward_gated",
           "dm_mlp_forward_style_reward", "dm_mlp_launches", "dm_mlp_destroy", "dm_td_lambda_returns", "dm_mlp_set_weights_device", "dm_learn_create",
           "dm_mlp_set_normalizers_device", "dm_learn_set_weights", "dm_learn_step", "dm_learn_disc_step", "dm_learn_destroy",
           "dm_learn_create_gated", "dm_learn_set_gated_weights", "dm_learn_gated_step", "dm_mlp_set_gated_weights_device", "dm_mlp_set_gated_normalizers_device",
           "dm_learn_grad_size", "dm_learn_grad", "dm_learn_apply", "dm_learn_gated_grad", "dm_learn_gated_apply", "dm_learn_disc_grad", "dm_learn_disc_apply"]


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise RuntimeError("deepmimic_b200: %s is missing -- run `python -c 'import __graft_entry__ as g; g.build()'`. "
                               "There is no CPU fallback." % _LIB_PATH)
        L = C.CDLL(_LIB_PATH)
        vp, dp, fp, ip = C.c_void_p, C.POINTER(C.c_double), C.c_void_p, C.c_void_p
        L.dm_create.restype = vp
        L.dm_create.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_char_p), C.c_int, C.c_int, C.c_uint64, C.c_uint64]
        L.dm_destroy.argtypes = [vp]
        L.dm_load_host.restype = vp
        L.dm_load_host.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_char_p)]
        L.dm_get_model_info.argtypes = [vp, C.c_int, C.POINTER(C.c_int)]
        L.dm_plan_launch.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
        L.dm_get_link_table.argtypes = [vp, dp]
        L.dm_last_error.restype = C.c_char_p
        L.dm_get_dims.argtypes = [vp, C.POINTER(DmDims)]
        L.dm_get_static.argtypes = [vp, C.c_int, dp]
        L.dm_get_scene_name.argtypes = [vp, C.c_char_p, C.c_int]
        L.dm_stream.restype = vp
        L.dm_stream.argtypes = [vp]
        L.dm_sync.argtypes = [vp]
        L.dm_set_mode.argtypes = [vp, C.c_int]
        L.dm_set_sample_count.argtypes = [vp, C.c_longlong]
        L.dm_get_time_limits.argtypes = [vp, dp]
        L.dm_reset.argtypes = [vp, C.c_int, dp, dp, dp]
        L.dm_set_action.argtypes = [vp, fp]
        L.dm_update.argtypes = [vp, C.c_double, C.c_int]
        L.dm_set_env_order.argtypes = [vp, C.c_int]
        if hasattr(L, "dm_set_pushes"):   # a library built before pushes (the base build of tools/ab_step.py) still loads; calling them fails
            L.dm_set_pushes.argtypes = [vp, C.POINTER(C.c_int32), fp, dp, dp]
            L.dm_get_pushes.argtypes = [vp, C.POINTER(C.c_int32)]
        if hasattr(L, "dm_set_push_schedule"):   # likewise a library built before push schedules
            L.dm_set_push_schedule.argtypes = [vp, C.POINTER(C.c_int32), C.c_int, dp, dp, dp]
            L.dm_get_push_table.argtypes = [vp, C.POINTER(C.c_int32), fp, dp, dp]
        if hasattr(L, "dm_set_dynamics"):   # likewise a library built before dynamics tables
            L.dm_set_dynamics.argtypes = [vp, fp]
            L.dm_get_dynamics.argtypes = [vp, C.c_void_p]
            L.dm_set_dynamics_randomization.argtypes = [vp, dp]
        if hasattr(L, "dm_set_action_latency"):   # likewise a library built before latency tables
            L.dm_set_action_latency.argtypes = [vp, C.POINTER(C.c_int32)]
            L.dm_set_action_latency_randomization.argtypes = [vp, C.c_int, C.c_int]
            L.dm_get_action_latency.argtypes = [vp, C.c_void_p]
        if hasattr(L, "dm_render_poses"):   # likewise a library built before the renderer
            L.dm_render_poses.argtypes = [vp, C.c_int, C.c_void_p, C.POINTER(DmCamera), C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        if hasattr(L, "dm_set_goal_course"):   # and before goal courses and the marked renderer
            L.dm_set_goal_course.argtypes = [vp, C.POINTER(C.c_int32), dp]
            L.dm_get_course_record.argtypes = [vp, C.c_void_p]
            L.dm_render_poses_marked.argtypes = [vp, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(DmCamera), C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        if hasattr(L, "dm_pose_error"):   # and before the tracking error
            L.dm_record_kin_pose.argtypes = [vp, fp]
            L.dm_pose_error.argtypes = [vp, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.dm_plan_env_order.argtypes = [C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
        L.dm_get_env_order.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.dm_record_state.argtypes = [vp, fp]
        L.dm_record_goal.argtypes = [vp, fp]
        L.dm_record_pose.argtypes = [vp, fp, fp]
        L.dm_calc_reward.argtypes = [vp, fp]
        L.dm_calc_reward_imitate.argtypes = [vp, fp]
        L.dm_goal_host.argtypes = [vp, fp]
        L.dm_reset_clips.argtypes = [vp, C.c_int, C.POINTER(C.c_int), dp, dp, dp]
        L.dm_record_amp_obs_expert_clips.argtypes = [vp, C.POINTER(C.c_int), dp, fp]
        L.dm_get_clip_table.argtypes = [vp, C.POINTER(C.c_int), dp, dp]
        L.dm_get_task_state.argtypes = [vp, C.c_int, dp]
        L.dm_set_task_state.argtypes = [vp, C.c_int, dp]
        L.dm_get_task_params.argtypes = [vp, dp, C.POINTER(C.c_uint64)]
        L.dm_record_amp_obs_agent.argtypes = [vp, fp]
        L.dm_record_amp_obs_expert.argtypes = [vp, dp, fp]
        L.dm_amp_obs_host.argtypes = [vp, C.c_int, dp, fp]
        L.dm_sample_amp_obs_expert.argtypes = [vp, C.c_int, vp, vp, vp]
        L.dm_expert_sample_count.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.dm_observe.argtypes = [vp, fp, fp]
        L.dm_get_flags.argtypes = [vp, ip]
        L.dm_step_host.argtypes = [vp, fp, C.c_double, C.c_int, fp, fp, ip]
        L.dm_step_host_reset.argtypes = [vp, fp, C.c_double, C.c_int, fp, fp, ip, C.c_int]
        L.dm_set_time_limits.argtypes = [vp, C.c_double, C.c_double]
        L.dm_exchange_create.argtypes = [vp, C.c_int, C.c_int, C.c_void_p]
        L.dm_exchange_connect.argtypes = [vp, C.c_void_p]
        L.dm_exchange_publish.argtypes = [vp, C.c_longlong]
        L.dm_exchange_acquire.argtypes = [vp, C.c_longlong, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
        L.dm_exchange_release.argtypes = [vp, C.c_longlong]
        L.dm_exchange_status.argtypes = [vp, C.POINTER(C.c_int)]
        L.dm_exchange_destroy.argtypes = [vp]
        L.dm_set_timing.argtypes = [vp, C.c_int]
        L.dm_step_host_timing.argtypes = [vp, dp]
        L.dm_get_snapshot.argtypes = [vp, C.c_int, dp]
        L.dm_set_snapshot.argtypes = [vp, C.c_int, dp]
        L.dm_state_size.argtypes = [vp, C.POINTER(C.c_size_t)]
        L.dm_save_state.argtypes = [vp, C.c_void_p]
        L.dm_load_state.argtypes = [vp, C.c_void_p]
        L.dm_get_counters.argtypes = [vp, C.POINTER(C.c_int64)]
        L.dm_get_section_profile.argtypes = [vp, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        fpp = C.POINTER(C.c_float)
        L.dm_mlp_create.restype = vp
        L.dm_mlp_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, fpp, fpp, fpp, fpp, fpp, fpp, fpp, fpp, C.c_float, fpp, fpp, C.c_int]
        L.dm_mlp_forward.argtypes = [vp, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.dm_mlp_create_gated.restype = vp
        L.dm_mlp_create_gated.argtypes = [C.c_int, C.POINTER(DmMlpGatedWeights), C.c_int]
        L.dm_mlp_forward_gated.argtypes = [vp, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.dm_mlp_forward_style_reward.argtypes = [vp, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.dm_mlp_launches.restype = C.c_longlong
        L.dm_mlp_launches.argtypes = [vp]
        L.dm_mlp_destroy.argtypes = [vp]
        L.dm_td_lambda_returns.argtypes = [vp] * 5 + [C.c_int, C.c_int] + [C.c_float] * 4 + [vp, vp, vp]
        L.dm_mlp_set_weights_device.argtypes = [vp] * 8
        L.dm_mlp_set_normalizers_device.argtypes = [vp] * 6
        L.dm_learn_create.restype = vp
        L.dm_learn_create.argtypes = [C.c_int] * 7
        L.dm_learn_set_weights.argtypes = [vp, C.POINTER(DmLearnNet), vp]
        L.dm_learn_step.argtypes = [vp, C.POINTER(DmLearnNet), C.POINTER(DmLearnBatch), vp]
        L.dm_learn_disc_step.argtypes = [vp, C.POINTER(DmLearnNet), C.POINTER(DmLearnDiscBatch), vp]
        L.dm_learn_destroy.argtypes = [vp]
        L.dm_learn_create_gated.restype = vp
        L.dm_learn_create_gated.argtypes = [C.c_int] * 10
        L.dm_learn_set_gated_weights.argtypes = [vp, C.POINTER(DmLearnGatedNet), vp]
        L.dm_learn_gated_step.argtypes = [vp, C.POINTER(DmLearnGatedNet), C.POINTER(DmLearnGatedBatch), vp]
        L.dm_mlp_set_gated_weights_device.argtypes = [vp, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), vp]
        L.dm_mlp_set_gated_normalizers_device.argtypes = [vp] * 8
        L.dm_learn_grad_size.restype = C.c_longlong
        L.dm_learn_grad_size.argtypes = [vp]
        for kind, net, batch in (("", DmLearnNet, DmLearnBatch), ("gated_", DmLearnGatedNet, DmLearnGatedBatch), ("disc_", DmLearnNet, DmLearnDiscBatch)):
            getattr(L, "dm_learn_%sgrad" % kind).argtypes = [vp, C.POINTER(net), C.POINTER(batch), vp, vp]
            getattr(L, "dm_learn_%sapply" % kind).argtypes = [vp, C.POINTER(net), C.POINTER(batch), vp, C.c_float, vp]
        _lib = L
    return _lib


def _check_device_f32(t, what, shape=None, device=None):
    """a contiguous float32 CUDA tensor (of the given shape, on the given device): what the C ABI's raw device pointers require"""
    import torch
    if (not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous()
            or (shape is not None and tuple(t.shape) != tuple(shape)) or (device is not None and t.device != device)):
        raise ValueError("%s: need a contiguous float32 CUDA tensor%s%s (got %s)" % (what, "" if shape is None else " of shape %s" % (tuple(shape),),
                         "" if device is None else " on %s" % device, "a %s" % type(t).__name__ if not isinstance(t, torch.Tensor)
                         else "%s %s on %s%s" % (t.dtype, tuple(t.shape), t.device, "" if t.is_contiguous() else ", not contiguous")))


# the renderer's default view: from the front-right, a little above the pelvis, 45 degrees vertical field of view
DEFAULT_CAMERA = dict(yaw=0.6, pitch=0.25, distance=4.0, target_height=0.9, fov_y=0.7853981633974483)


def camera_struct(camera=None):
    """dm_camera of a dict with the keys of DEFAULT_CAMERA (missing keys take its values), or of DEFAULT_CAMERA for None"""
    c = dict(DEFAULT_CAMERA, **(camera or {}))
    unknown = set(c) - set(DEFAULT_CAMERA)
    if unknown:
        raise ValueError("camera: unknown keys %s" % sorted(unknown))
    return DmCamera(*(float(c[k]) for k in ("yaw", "pitch", "distance", "target_height", "fov_y")))


UPDATE_DT = 1.0 / 600.0   # the library's update timestep; a control latency is a whole number of these
UPDATES_PER_ACTION = 20   # dm_dims::updates_per_action of every shipped controller (capi.cu: kUpdatesPerAction); a delay is below it


def latency_updates(seconds, updates_per_action=UPDATES_PER_ACTION, what="latency"):
    """a control latency in seconds -> whole updates (nearest), refused unless finite and within [0, (updates_per_action - 1) UPDATE_DT] after
    rounding"""
    s = float(seconds)
    if not np.isfinite(s):
        raise ValueError("%s: %r s is not a finite number" % (what, seconds))
    d = int(round(s / UPDATE_DT))
    if d < 0 or d > updates_per_action - 1:
        raise ValueError("%s: %r s rounds to %d updates, outside [0, %d] (0 to %.4f s)" % (what, seconds, d, updates_per_action - 1,
                                                                                             (updates_per_action - 1) * UPDATE_DT))
    return d


MAX_COURSE_POINTS = 16   # rows of a goal course per environment (dm_course.cuh: kMaxCoursePoints)


def _dptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_double)) if a is not None else None


def _call(fn, *args, stream=None):
    """calls the C function `fn` with args and then the cudaStream_t handle `stream` (int or None); a nonzero return raises
    RuntimeError("fn: <dm_last_error>")"""
    if getattr(lib(), fn)(*args, C.c_void_p(stream) if stream else None) != 0:
        raise RuntimeError("%s: %s" % (fn, lib().dm_last_error().decode()))


def td_lambda_returns(rewards, values, end_values, done, terminate, discount, td_lambda, val_fail, val_succ, returns, advantages, stream=None):
    """dm_td_lambda_returns: TD(lambda) returns and advantages of a [T, N] rollout window on the device.  rewards, values, end_values, returns,
    advantages: contiguous float32 CUDA tensors [T, N]; done: bool (or uint8) [T, N]; terminate: int32 [T, N]; stream: cudaStream_t handle (int)
    or None.  returns and advantages are written."""
    T, N = rewards.shape
    for name, x, dt in (("rewards", rewards, "float32"), ("values", values, "float32"), ("end_values", end_values, "float32"), ("returns", returns, "float32"),
                        ("advantages", advantages, "float32"), ("done", done, ("bool", "uint8")), ("terminate", terminate, "int32")):
        if tuple(x.shape) != (T, N) or not x.is_contiguous() or not x.is_cuda or str(x.dtype).replace("torch.", "") not in (dt if isinstance(dt, tuple) else (dt,)):
            raise ValueError("td_lambda_returns: %s must be a contiguous %s CUDA tensor [%d, %d]" % (name, dt, T, N))
    ptr = lambda t: C.c_void_p(t.data_ptr())
    _call("dm_td_lambda_returns", ptr(rewards), ptr(values), ptr(end_values), ptr(done), ptr(terminate), T, N, float(discount), float(td_lambda),
          float(val_fail), float(val_succ), ptr(returns), ptr(advantages), stream=stream)
    return returns, advantages


def plan_env_order(keys, tiles, tile_width):
    """dm_plan_env_order: the step kernel's placement of len(keys) (padded) environments by contact load, as host arithmetic; returns order
    [len(keys)] int32 (order[slot] = environment)"""
    k = np.ascontiguousarray(keys, dtype=np.int32)
    out = np.zeros(len(k), dtype=np.int32)
    ip = C.POINTER(C.c_int)
    if lib().dm_plan_env_order(k.ctypes.data_as(ip), len(k), int(tiles), int(tile_width), out.ctypes.data_as(ip)) != 0:
        raise RuntimeError(lib().dm_last_error().decode())
    return out


class BatchedCore:
    """Thin object wrapper over a dm_handle."""

    def __init__(self, args, num_envs, asset_root, device=0, seed=0, global_env_offset=0):
        L = lib()
        enc = [a.encode() for a in args]
        arr = (C.c_char_p * len(enc))(*enc)
        self.h = L.dm_create(asset_root.encode(), len(enc), arr, num_envs, device, seed, global_env_offset)
        if not self.h:
            raise RuntimeError("dm_create failed: %s" % L.dm_last_error().decode())
        self.h = C.c_void_p(self.h)
        d = DmDims()
        L.dm_get_dims(self.h, C.byref(d))
        self.dims = d
        self.num_envs = d.num_envs
        self.device = device

    def _chk(self, rc):
        if rc != 0:
            raise RuntimeError("deepmimic_b200: %s" % lib().dm_last_error().decode())

    def close(self):
        if self.h:
            lib().dm_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def static(self, kind):
        n = self.dims.state_size if kind in (DM_STATE_OFFSET, DM_STATE_SCALE, DM_STATE_NORM_GROUPS) else self.dims.action_size
        out = np.zeros(n, dtype=np.float64)
        self._chk(lib().dm_get_static(self.h, kind, _dptr(out)))
        return out

    def scene_name(self):
        buf = C.create_string_buffer(64)
        self._chk(lib().dm_get_scene_name(self.h, buf, 64))
        return buf.value.decode()

    def reset(self, force_all=True, kin_time=None, max_time=None, rot_theta=None, clip=None):
        f = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)
        kt, mt, th = f(kin_time), f(max_time), f(rot_theta)
        if clip is None:
            self._chk(lib().dm_reset(self.h, 1 if force_all else 0, _dptr(kt), _dptr(mt), _dptr(th)))
        else:   # task scenes with a clip dataset: the controller's clip draw injected
            c = np.ascontiguousarray(clip, dtype=np.int32)
            self._chk(lib().dm_reset_clips(self.h, 1 if force_all else 0, c.ctypes.data_as(C.POINTER(C.c_int)), _dptr(kt), _dptr(mt), _dptr(th)))

    def clip_table(self):
        n = C.c_int(0)
        lib().dm_get_clip_table(self.h, C.byref(n), None, None)
        dur, cdf = np.zeros(n.value), np.zeros(n.value)
        lib().dm_get_clip_table(self.h, C.byref(n), _dptr(dur), _dptr(cdf))
        return dur, cdf

    def set_action(self, actions):  # torch float32 cuda tensor [N, A]
        self._chk(lib().dm_set_action(self.h, C.c_void_p(actions.data_ptr())))

    def update(self, dt, n_updates=1):
        self._chk(lib().dm_update(self.h, dt, n_updates))

    def set_pushes(self, body, force, start, duration):
        """dm_set_pushes: a timed external force per environment -- body [N] int32 (-1: none), force [N, 3] float32 (world axes, unscaled N,
        at the body's COM), start and duration [N] float64 (seconds on the episode timer).  numpy arrays or tensors (copied to the host) of
        exactly these shapes and dtypes; the library refuses out-of-range values by name.  Synchronises the handle's stream."""
        N = self.num_envs
        arrs = []
        for name, a, dt, shape in (("body", body, np.int32, (N,)), ("force", force, np.float32, (N, 3)), ("start", start, np.float64, (N,)),
                                   ("duration", duration, np.float64, (N,))):
            if hasattr(a, "detach"):
                a = a.detach().cpu().numpy()
            a = np.asarray(a)
            if a.dtype != dt or a.shape != shape:
                raise ValueError("set_pushes: %s must be %s of shape %s, got %s of shape %s" % (name, np.dtype(dt).name, shape, a.dtype, a.shape))
            arrs.append(np.ascontiguousarray(a))
        b, f, s, d = arrs
        self._chk(lib().dm_set_pushes(self.h, b.ctypes.data_as(C.POINTER(C.c_int32)), f.ctypes.data_as(C.POINTER(C.c_float)), _dptr(s), _dptr(d)))

    def pushes(self):
        """dm_get_pushes: every environment's pending push body, int32 [N] (-1: none).  Synchronises the handle's stream."""
        out = np.zeros(self.num_envs, dtype=np.int32)
        self._chk(lib().dm_get_pushes(self.h, out.ctypes.data_as(C.POINTER(C.c_int32))))
        return out

    def set_push_schedule(self, bodies, force, duration, gap):
        """dm_set_push_schedule: random pushes drawn on the device at every update() -- bodies (1 to 32 body ids drawn from), force, duration and
        gap (lo, hi) of the magnitude in N, the push length in s and the time after the previous push in s.  The library refuses out-of-range
        values by name.  Synchronises the handle's stream on the first call (allocation)."""
        b = np.ascontiguousarray(np.asarray(bodies).reshape(-1))
        if b.dtype.kind not in "iu":
            raise ValueError("set_push_schedule: bodies must be integers, got %s" % b.dtype)
        b = b.astype(np.int32)
        pairs = []
        for name, a in (("force", force), ("duration", duration), ("gap", gap)):
            a = np.ascontiguousarray(a, dtype=np.float64)
            if a.shape != (2,):
                raise ValueError("set_push_schedule: %s must be a (lo, hi) pair, got shape %s" % (name, a.shape))
            pairs.append(a)
        f, d, g = pairs
        self._chk(lib().dm_set_push_schedule(self.h, b.ctypes.data_as(C.POINTER(C.c_int32)), int(b.size), _dptr(f), _dptr(d), _dptr(g)))

    def push_table(self, schedule=False):
        """dm_get_push_table: every environment's push-table entry as dict(body [N] int32 (-1: none), force [N, 3] float32, start [N], duration
        [N] float64) and, with schedule=True (handles with a push schedule only), sched [N, 3] float64: the schedule block (reset counter seen,
        draw counter, last_end).  Synchronises the handle's stream."""
        N = self.num_envs
        body, force, window = np.zeros(N, dtype=np.int32), np.zeros((N, 3), dtype=np.float32), np.zeros((N, 2))
        sched = np.zeros((N, 3)) if schedule else None
        self._chk(lib().dm_get_push_table(self.h, body.ctypes.data_as(C.POINTER(C.c_int32)), C.c_void_p(force.ctypes.data), _dptr(window), _dptr(sched)))
        out = dict(body=body, force=force, start=window[:, 0].copy(), duration=window[:, 1].copy())
        if schedule:
            out["sched"] = sched
        return out

    DYNAMICS_KINDS = ("friction", "kp", "kd", "torque_limit", "mass")

    def set_dynamics(self, factors):
        """dm_set_dynamics: explicit per-environment factors, float32 [N, 4 + links] (friction, kp, kd, torque_limit, one mass factor per link),
        kept across resets.  A numpy array or tensor (copied to the host); the library refuses out-of-range values by name.  Synchronises the
        handle's stream."""
        if hasattr(factors, "detach"):
            factors = factors.detach().cpu().numpy()
        a = np.asarray(factors)
        shape = (self.num_envs, 4 + self.dims.num_joints)
        if a.dtype != np.float32 or a.shape != shape:
            raise ValueError("set_dynamics: factors must be float32 of shape %s, got %s of shape %s" % (shape, a.dtype, a.shape))
        a = np.ascontiguousarray(a)
        self._chk(lib().dm_set_dynamics(self.h, a.ctypes.data_as(C.POINTER(C.c_float))))

    def dynamics(self, out=None):
        """dm_get_dynamics: every environment's factors as a float32 tensor [N, 4 + links] on the handle's device (stream-ordered, no host
        synchronisation).  Refused on a handle without a dynamics table."""
        import torch
        shape = (self.num_envs, 4 + self.dims.num_joints)
        if out is None:
            out = torch.empty(shape, dtype=torch.float32, device=torch.device("cuda", self.device))
        elif out.dtype != torch.float32 or tuple(out.shape) != shape or not out.is_contiguous() or out.device != torch.device("cuda", self.device):
            raise ValueError("dynamics: out must be a contiguous float32 tensor of shape %s on cuda:%d" % (shape, self.device))
        self._chk(lib().dm_get_dynamics(self.h, C.c_void_p(out.data_ptr())))
        return out

    def set_dynamics_randomization(self, lohi):
        """dm_set_dynamics_randomization: draw every environment's factors on the device now and at every reset; lohi: 10 floats, (lo, hi) of
        friction, kp, kd, torque_limit and mass in that order.  The library refuses out-of-range bounds by name."""
        a = np.ascontiguousarray(lohi, dtype=np.float64).reshape(-1)
        if a.shape != (10,):
            raise ValueError("set_dynamics_randomization: lohi must hold 10 bounds, got %d" % a.size)
        self._chk(lib().dm_set_dynamics_randomization(self.h, _dptr(a)))

    def set_action_latency(self, seconds):
        """dm_set_action_latency: every environment's control latency, [N] seconds (a sequence, numpy array or tensor), each rounded to the
        nearest whole update and refused outside [0, (updates_per_action - 1) dt]; kept across resets.  Synchronises the handle's stream."""
        if hasattr(seconds, "detach"):
            seconds = seconds.detach().cpu().numpy()
        a = np.asarray(seconds, dtype=np.float64).reshape(-1)
        if a.shape != (self.num_envs,):
            raise ValueError("set_action_latency: need %d delays, got %d" % (self.num_envs, a.size))
        U = self.dims.updates_per_action
        d = np.array([latency_updates(x, U, "set_action_latency: environment %d" % e) for e, x in enumerate(a)], dtype=np.int32)
        self._chk(lib().dm_set_action_latency(self.h, d.ctypes.data_as(C.POINTER(C.c_int32))))

    def set_action_latency_randomization(self, lo, hi):
        """dm_set_action_latency_randomization: draw every environment's control latency uniformly among the whole updates of [lo, hi] seconds
        (each bound rounded to the nearest update), on the device, now and at every reset"""
        U = self.dims.updates_per_action
        dlo, dhi = latency_updates(lo, U, "set_action_latency_randomization: lo"), latency_updates(hi, U, "set_action_latency_randomization: hi")
        self._chk(lib().dm_set_action_latency_randomization(self.h, dlo, dhi))

    def action_latency(self):
        """dm_get_action_latency: every environment's current control latency in seconds, a float64 tensor [N] on the handle's device
        (stream-ordered, no host synchronisation).  Refused on a handle without a latency table."""
        import torch
        # the scratch tensor belongs to the handle's stream, which writes and reads it: the caching allocator reuses it only after that work
        with torch.cuda.stream(torch.cuda.ExternalStream(self.stream(), device=self.device)):
            out = torch.empty(self.num_envs, dtype=torch.int32, device=torch.device("cuda", self.device))
            self._chk(lib().dm_get_action_latency(self.h, C.c_void_p(out.data_ptr())))
            return out.to(torch.float64) * UPDATE_DT

    def set_goal_course(self, counts, rows):
        """dm_set_goal_course: every environment's goal course, counts [N] int (0 to MAX_COURSE_POINTS; 0 keeps the scene's own goals) and rows
        [N, MAX_COURSE_POINTS, 3] float64 (heading scenes: episode time s, heading rad, speed m/s; target scene: waypoint dx, dz in m and an
        unused value).  Numpy arrays or tensors (copied to the host); the library refuses bad values by name.  Every course restarts now, from
        the current root and episode time.  Synchronises the handle's stream."""
        if hasattr(counts, "detach"):
            counts = counts.detach().cpu().numpy()
        if hasattr(rows, "detach"):
            rows = rows.detach().cpu().numpy()
        n = np.ascontiguousarray(counts, dtype=np.int32).reshape(-1)
        r = np.ascontiguousarray(rows, dtype=np.float64)
        if n.shape != (self.num_envs,):
            raise ValueError("set_goal_course: counts must hold %d values, got %d" % (self.num_envs, n.size))
        if r.shape != (self.num_envs, MAX_COURSE_POINTS, 3):
            raise ValueError("set_goal_course: rows must be [%d, %d, 3], got %s" % (self.num_envs, MAX_COURSE_POINTS, r.shape))
        self._chk(lib().dm_set_goal_course(self.h, n.ctypes.data_as(C.POINTER(C.c_int32)), _dptr(r)))

    def course_record(self, out):
        """dm_get_course_record: every environment's record of its last course call into out, a contiguous float32 tensor [N, 4] on the
        handle's device (heading: goal point x, z, along-track speed error, cross-track speed; target: goal waypoint x, z, waypoints reached,
        distance to the goal waypoint).  Stream-ordered, no host synchronisation.  Refused on a handle without a course."""
        _check_device_f32(out, "course_record: out", (self.num_envs, 4))
        self._chk(lib().dm_get_course_record(self.h, C.c_void_p(out.data_ptr())))
        return out

    def set_env_order(self, on):
        """dm_set_env_order: place the environments in the step kernel by contact load (the default; tile width 16 only) or by index"""
        self._chk(lib().dm_set_env_order(self.h, 1 if on else 0))

    def env_order(self):
        """dm_get_env_order: (keys now, placement of the last step launch: padded_envs int32 each, environments per block, tile width)"""
        ip = C.POINTER(C.c_int)
        plan = np.zeros(3, dtype=np.int32)
        self._chk(lib().dm_get_env_order(self.h, plan.ctypes.data_as(ip), None, None))
        keys, order = np.zeros(plan[0], dtype=np.int32), np.zeros(plan[0], dtype=np.int32)
        self._chk(lib().dm_get_env_order(self.h, plan.ctypes.data_as(ip), keys.ctypes.data_as(ip), order.ctypes.data_as(ip)))
        return keys, order, int(plan[1]), int(plan[2])

    def observe(self, state=None, reward=None):
        self._chk(lib().dm_observe(self.h, C.c_void_p(state.data_ptr()) if state is not None else None,
                                   C.c_void_p(reward.data_ptr()) if reward is not None else None))

    def record_pose(self, pose=None, vel=None):
        """dm_record_pose: the simulated characters' pose and velocity rows in the reference's layout (cSimCharacter::BuildPose / BuildVel) into
        contiguous float32 CUDA tensors [N, pose_dim]; either may be None.  Stream-ordered on the handle's stream."""
        P = self.dims.pose_dim
        for name, t in (("pose", pose), ("vel", vel)):
            if t is not None:
                _check_device_f32(t, "record_pose: " + name, (self.num_envs, P))
        self._chk(lib().dm_record_pose(self.h, C.c_void_p(pose.data_ptr()) if pose is not None else None,
                                       C.c_void_p(vel.data_ptr()) if vel is not None else None))

    def record_kin_pose(self, pose):
        """dm_record_kin_pose: the kinematic characters' poses (the clip at every environment's kin time, in the world; what the imitation reward
        compares against) in record_pose's layout into a contiguous float32 CUDA tensor [N, pose_dim].  Stream-ordered on the handle's stream."""
        _check_device_f32(pose, "record_kin_pose: pose", (self.num_envs, self.dims.pose_dim))
        self._chk(lib().dm_record_kin_pose(self.h, C.c_void_p(pose.data_ptr())))

    def pose_error(self, a, r, lengths, lock=None, dtw=None):
        """dm_pose_error: the phase-locked and the time-warped tracking error in metres of n episodes, a and r [T, n, pose_dim] pose rows (contiguous
        float32 tensors on the handle's device, record_pose's layout), lengths [n] int32 frames.  Returns (lock [n], dtw [n]) float32; pass tensors
        to fill them in place, or False to skip that output.  A length outside [1, T] gives NaN.  Stream-ordered on the handle's stream."""
        import torch
        dev = torch.device("cuda", self.device)
        P = self.dims.pose_dim
        if a.dim() != 3 or a.shape[2] != P:
            raise ValueError("pose_error: a must be [T, n, %d], got %s" % (P, tuple(a.shape)))
        T, n = a.shape[0], a.shape[1]
        _check_device_f32(a, "pose_error: a", device=dev)
        _check_device_f32(r, "pose_error: r", (T, n, P), device=dev)
        if (not isinstance(lengths, torch.Tensor) or lengths.dtype != torch.int32 or tuple(lengths.shape) != (n,) or lengths.device != dev
                or not lengths.is_contiguous()):
            raise ValueError("pose_error: lengths must be a contiguous int32 tensor of shape (%d,) on %s" % (n, dev))
        outs = []
        for name, t in (("lock", lock), ("dtw", dtw)):
            if t is False:
                outs.append(None)
                continue
            if t is None:
                t = torch.empty(n, dtype=torch.float32, device=dev)
            _check_device_f32(t, "pose_error: " + name, (n,), device=dev)
            outs.append(t)
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        self._chk(lib().dm_pose_error(self.h, T, n, ptr(a), ptr(r), ptr(lengths), ptr(outs[0]), ptr(outs[1])))
        return outs[0], outs[1]

    def render_poses(self, pose, camera=None, width=640, height=360, rgb=None, ids=None, markers=None):
        """dm_render_poses: pose rows [V, pose_dim] (a contiguous float32 tensor on the handle's device, dm_record_pose's layout) drawn as this handle's
        character by the device ray caster, seen from `camera` (a dict of yaw, pitch, distance, target_height, fov_y in radians and metres;
        missing keys and None: DEFAULT_CAMERA).  Returns (rgb uint8 [V, height, width, 3], ids int16 [V, height, width]: -1 sky, -2 ground, k link
        k, -3 marker); pass rgb / ids tensors to fill them in place, or False to skip that output.  markers: [V, 4] float32 (x, y, z, radius in
        metres; radius <= 0 draws none) on the handle's device draws one sphere per view (dm_render_poses_marked).  Stream-ordered on the
        handle's stream."""
        import torch
        P = self.dims.pose_dim
        if pose.dim() != 2 or pose.shape[1] != P:
            raise ValueError("render_poses: pose must be [V, %d], got %s" % (P, tuple(pose.shape)))
        dev = torch.device("cuda", self.device)
        _check_device_f32(pose, "render_poses: pose", device=dev)
        V = pose.shape[0]
        outs = []
        for name, t, dt, shape in (("rgb", rgb, torch.uint8, (V, height, width, 3)), ("ids", ids, torch.int16, (V, height, width))):
            if t is False:
                outs.append(None)
                continue
            if t is None:
                t = torch.empty(shape, dtype=dt, device=dev)
            elif (not isinstance(t, torch.Tensor) or t.dtype != dt or tuple(t.shape) != shape or t.device != dev or not t.is_contiguous()):
                raise ValueError("render_poses: %s must be a contiguous %s tensor of shape %s on %s" % (name, dt, shape, dev))
            outs.append(t)
        cam = camera_struct(camera)
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        if markers is None:
            self._chk(lib().dm_render_poses(self.h, V, ptr(pose), C.byref(cam), int(width), int(height), ptr(outs[0]), ptr(outs[1])))
        else:
            _check_device_f32(markers, "render_poses: markers", (V, 4), device=dev)
            self._chk(lib().dm_render_poses_marked(self.h, V, ptr(pose), ptr(markers), C.byref(cam), int(width), int(height), ptr(outs[0]),
                                                   ptr(outs[1])))
        return outs[0], outs[1]

    def reward_imitate(self, out):  # torch float32 cuda tensor [N]: CalcRewardImitate also in the task scenes (active clip of the dataset)
        self._chk(lib().dm_calc_reward_imitate(self.h, C.c_void_p(out.data_ptr())))

    def record_goal(self, out):  # torch float32 cuda tensor [N, goal_size]; task scenes only
        self._chk(lib().dm_record_goal(self.h, C.c_void_p(out.data_ptr())))

    def goal_host(self):
        out = np.zeros((self.num_envs, self.dims.goal_size), dtype=np.float32)
        self._chk(lib().dm_goal_host(self.h, C.c_void_p(out.ctypes.data)))
        return out

    def task_state(self, env):
        out = np.zeros(24, dtype=np.float64)     # dm_task.cuh block (16) | dm_task_ext.cuh block (8)
        self._chk(lib().dm_get_task_state(self.h, env, _dptr(out)))
        return out

    def set_task_state(self, env, block):
        b = np.ascontiguousarray(block, dtype=np.float64)
        self._chk(lib().dm_set_task_state(self.h, env, _dptr(b)))

    def plan_launch(self, num_envs, smem_bytes_per_block=232448, num_sms=132):
        """dm_plan_launch: launch plan of the step kernel on a device with that much opt-in shared memory per block and that many SMs (H100 SXM defaults)"""
        out = (C.c_int * 9)()
        if lib().dm_plan_launch(self.h, int(num_envs), int(smem_bytes_per_block), int(num_sms), out) != 0:
            raise RuntimeError(lib().dm_last_error().decode())
        keys = ("tile_width", "envs_per_block", "blocks", "smem_bytes", "max_rows", "env_floats", "hot_floats", "y_offset", "padded_envs")
        return dict(zip(keys, [int(v) for v in out]))

    def task_params(self):
        out = np.zeros(48, dtype=np.float64)     # [0:16] dm_task.cuh constants, [16:48] dm_task_ext.cuh constants
        key = (C.c_uint64 * 2)()
        self._chk(lib().dm_get_task_params(self.h, _dptr(out), key))
        return out, int(key[0]), int(key[1])

    def amp_obs_agent(self, out):  # torch float32 cuda tensor [N, amp_obs_size]
        self._chk(lib().dm_record_amp_obs_agent(self.h, C.c_void_p(out.data_ptr())))

    def amp_obs_expert(self, out, kin_time=None, clip=None):
        kt = None if kin_time is None else np.ascontiguousarray(kin_time, dtype=np.float64)
        if clip is None:
            self._chk(lib().dm_record_amp_obs_expert(self.h, _dptr(kt), C.c_void_p(out.data_ptr())))
        else:
            c = np.ascontiguousarray(clip, dtype=np.int32)
            self._chk(lib().dm_record_amp_obs_expert_clips(self.h, c.ctypes.data_as(C.POINTER(C.c_int)), _dptr(kt), C.c_void_p(out.data_ptr())))

    def sample_amp_obs_expert(self, out, clip=None, time=None):
        """dm_sample_amp_obs_expert: out.shape[0] expert AMP observations into out [rows, amp_obs_size] (contiguous float32 CUDA tensor), clip
        and time drawn on the device, enqueued on the handle's stream without a host synchronisation.  clip [rows] int32 and time [rows]
        float64 contiguous CUDA tensors receive the draws when given."""
        import torch
        rows = out.shape[0] if out.dim() == 2 else 0
        _check_device_f32(out, "sample_amp_obs_expert: out", (rows, self.dims.amp_obs_size))
        for name, t, dt in (("clip", clip, torch.int32), ("time", time, torch.float64)):
            if t is not None and (not t.is_cuda or t.dtype != dt or tuple(t.shape) != (rows,) or not t.is_contiguous()):
                raise ValueError("sample_amp_obs_expert: %s must be a contiguous %s CUDA tensor [%d]" % (name, dt, rows))
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        self._chk(lib().dm_sample_amp_obs_expert(self.h, rows, ptr(out), ptr(clip), ptr(time)))

    def expert_sample_count(self, set_to=None):
        """the expert sampler's call counter (the key of its next draws); set_to replaces it.  Returns the value before the call."""
        got = C.c_uint64(0)
        new = None if set_to is None else C.byref(C.c_uint64(int(set_to)))
        self._chk(lib().dm_expert_sample_count(self.h, new, C.byref(got)))
        return int(got.value)

    def flags(self, out):  # torch int32 cuda tensor [N, 4]
        self._chk(lib().dm_get_flags(self.h, C.c_void_p(out.data_ptr())))

    def sync(self):
        self._chk(lib().dm_sync(self.h))

    def set_mode(self, mode):
        self._chk(lib().dm_set_mode(self.h, mode))

    def set_sample_count(self, count):
        self._chk(lib().dm_set_sample_count(self.h, int(count)))

    def time_limits(self):
        out = np.zeros(3, dtype=np.float64)
        self._chk(lib().dm_get_time_limits(self.h, _dptr(out)))
        return out

    def step_host(self, actions, dt, n_updates, state, reward, flags, reset_done=False):  # numpy host arrays
        p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)
        self._chk(lib().dm_step_host_reset(self.h, p(actions), dt, n_updates, p(state), p(reward), p(flags), 1 if reset_done else 0))

    def set_episode_limit(self, seconds_min, seconds_max=None):
        self._chk(lib().dm_set_time_limits(self.h, float(seconds_min), float(seconds_min if seconds_max is None else seconds_max)))

    # ---- multi-GPU exchange over NVLink peer memory (dm_exchange_*)
    def exchange_create(self, rank, world):
        buf = C.create_string_buffer(64)
        self._chk(lib().dm_exchange_create(self.h, rank, world, buf))
        return bytes(buf.raw)

    def exchange_connect(self, handles):   # world x 64 bytes, rank order
        blob = b"".join(handles)
        self._chk(lib().dm_exchange_connect(self.h, C.c_char_p(blob)))

    def exchange_publish(self, step):
        self._chk(lib().dm_exchange_publish(self.h, int(step)))

    def exchange_acquire(self, step):
        o, r, d = C.c_void_p(), C.c_void_p(), C.c_void_p()
        self._chk(lib().dm_exchange_acquire(self.h, int(step), C.byref(o), C.byref(r), C.byref(d)))
        return o.value, r.value, d.value

    def exchange_release(self, step):
        self._chk(lib().dm_exchange_release(self.h, int(step)))

    def exchange_status(self):
        s = C.c_int(0)
        self._chk(lib().dm_exchange_status(self.h, C.byref(s)))
        return s.value

    def set_timing(self, on=True):
        self._chk(lib().dm_set_timing(self.h, 1 if on else 0))

    def step_host_timing(self):
        """last dm_step_host: dict of device ms per phase and host wall ms (enqueue / wait / staging copies)"""
        o = np.zeros(8, dtype=np.float64)
        self._chk(lib().dm_step_host_timing(self.h, _dptr(o)))
        return dict(h2d_set_action_ms=o[0], update_ms=o[1], observe_flags_ms=o[2], d2h_ms=o[3], host_enqueue_ms=o[4], host_wait_ms=o[5], host_copy_ms=o[6])

    def get_snapshot(self, env):
        out = np.zeros(self.dims.snapshot_size, dtype=np.float64)
        self._chk(lib().dm_get_snapshot(self.h, env, _dptr(out)))
        return out

    def set_snapshot(self, env, snap):
        s = np.ascontiguousarray(snap, dtype=np.float64)
        self._chk(lib().dm_set_snapshot(self.h, env, _dptr(s)))

    def save_state(self):
        """dm_save_state: the whole batch's simulation state as a uint8 array (synchronises the handle's stream)"""
        n = C.c_size_t(0)
        self._chk(lib().dm_state_size(self.h, C.byref(n)))
        out = np.zeros(n.value, dtype=np.uint8)
        self._chk(lib().dm_save_state(self.h, C.c_void_p(out.ctypes.data)))
        return out

    def load_state(self, buf):
        """dm_load_state: restores a save_state() blob of a handle made with the same arguments, environment count and seed (synchronises the
        handle's stream); a mismatch raises, naming the field"""
        b = np.ascontiguousarray(buf, dtype=np.uint8)
        # the header's byte count (bytes 16..23) must match the blob: dm_load_state then compares the header with this handle field by field
        if b.ndim != 1 or b.size < 24 or int(b[16:24].view(np.uint64)[0]) != b.size:
            raise ValueError("load_state: not a complete save_state() blob (%s bytes)" % (b.shape,))
        self._chk(lib().dm_load_state(self.h, C.c_void_p(b.ctypes.data)))

    def counters(self):
        out = (C.c_int64 * 2)()
        self._chk(lib().dm_get_counters(self.h, out))
        return int(out[0]), int(out[1])

    def section_profile(self):
        """profile build only: [blocks, warps per block, 18] uint32 section cycle counters of the last update launch"""
        nb, nw = C.c_int(0), C.c_int(0)
        self._chk(lib().dm_get_section_profile(self.h, None, C.byref(nb), C.byref(nw)))
        out = np.zeros((nb.value, nw.value, 18), dtype=np.uint32)
        self._chk(lib().dm_get_section_profile(self.h, C.c_void_p(out.ctypes.data), None, None))
        return out

    def stream(self):
        return lib().dm_stream(self.h)


class HostModel:
    """dm_load_host handle: the host loaders and the flat model, no device (used by the CPU tests and by tools)."""
    INFO = dict(parents=0, joint_types=1, dof_offsets=2, pose_offsets=3, fall_bodies=4, end_effectors=5)

    def __init__(self, args, asset_root):
        L = lib()
        enc = [a.encode() for a in args]
        arr = (C.c_char_p * len(enc))(*enc)
        h = L.dm_load_host(asset_root.encode(), len(enc), arr)
        if not h:
            raise RuntimeError("dm_load_host failed: %s" % L.dm_last_error().decode())
        self.h = C.c_void_p(h)
        self.dims = DmDims()
        L.dm_get_dims(self.h, C.byref(self.dims))

    def static(self, kind):
        n = self.dims.state_size if kind in (DM_STATE_OFFSET, DM_STATE_SCALE, DM_STATE_NORM_GROUPS) else self.dims.action_size
        out = np.zeros(n, dtype=np.float64)
        if lib().dm_get_static(self.h, kind, _dptr(out)) != 0:
            raise RuntimeError(lib().dm_last_error().decode())
        return out

    def plan_launch(self, num_envs, smem_bytes_per_block=232448, num_sms=132):
        """dm_plan_launch: launch plan of the step kernel on a device with that much opt-in shared memory per block and that many SMs (H100 SXM defaults)"""
        out = (C.c_int * 9)()
        if lib().dm_plan_launch(self.h, int(num_envs), int(smem_bytes_per_block), int(num_sms), out) != 0:
            raise RuntimeError(lib().dm_last_error().decode())
        keys = ("tile_width", "envs_per_block", "blocks", "smem_bytes", "max_rows", "env_floats", "hot_floats", "y_offset", "padded_envs")
        return dict(zip(keys, [int(v) for v in out]))

    def task_params(self):
        out = np.zeros(48, dtype=np.float64)     # [0:16] dm_task.cuh constants, [16:48] dm_task_ext.cuh constants
        key = (C.c_uint64 * 2)()
        lib().dm_get_task_params(self.h, _dptr(out), key)
        return out, int(key[0]), int(key[1])

    def clip_table(self):
        n = C.c_int(0)
        lib().dm_get_clip_table(self.h, C.byref(n), None, None)
        dur, cdf = np.zeros(n.value), np.zeros(n.value)
        lib().dm_get_clip_table(self.h, C.byref(n), _dptr(dur), _dptr(cdf))
        return dur, cdf

    def set_sample_count(self, count):
        if lib().dm_set_sample_count(self.h, int(count)) != 0:
            raise RuntimeError(lib().dm_last_error().decode())

    def time_limits(self):
        out = np.zeros(3, dtype=np.float64)
        lib().dm_get_time_limits(self.h, _dptr(out))
        return out

    def info(self, name):
        out = (C.c_int * self.dims.num_joints)()
        if lib().dm_get_model_info(self.h, self.INFO[name], out) != 0:
            raise RuntimeError(lib().dm_last_error().decode())
        return np.array(out[:], dtype=np.int64)

    def link_table(self):
        """[num_joints, 24]: mass, inertiaB[3], inertiaD[3], dvec[3], evec[3], zrot xyzw, axis[3], half extents[3], breaking threshold"""
        out = np.zeros((self.dims.num_joints, 24), dtype=np.float64)
        lib().dm_get_link_table(self.h, _dptr(out))
        return out

    def layout(self):
        out = (C.c_int * 6)()
        lib().dm_get_model_info(self.h, 6, out)
        return dict(zip(("links", "dofs", "chain_stride", "tree_depth", "frames", "loop"), out[:]))

    def close(self):
        if self.h:
            lib().dm_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _MlpHandle:
    """a dm_mlp_* handle self.h (plain or gated): its launch count and its release"""

    def launches(self):
        return int(lib().dm_mlp_launches(self.h))

    def close(self):
        if self.h:
            lib().dm_mlp_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class TensorCoreMLP(_MlpHandle):
    """dm_mlp_* handle: the actor network (normalise -> 2 hidden ReLU layers -> linear -> un-normalise) on the tensor cores (wgmma).
    weights: the reference's dense kernels, [inputs x units] float arrays (deepmimic_b200.tf_checkpoint.load_actor / the fixture files).
    With one output unit and no output normaliser the handle is an AMP discriminator: style_reward() runs it with the reward epilogue."""

    def __init__(self, w0, b0, w1, b1, w2, b2, in_mean=None, in_std=None, in_clip=float("inf"), out_mean=None, out_std=None, max_rows=4096, device=0):
        L = lib()
        f = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float32)
        w0, b0, w1, b1, w2, b2, in_mean, in_std, out_mean, out_std = (f(x) for x in (w0, b0, w1, b1, w2, b2, in_mean, in_std, out_mean, out_std))
        self.in_dim, self.h0 = w0.shape
        self.h1, self.out_dim = w2.shape
        assert w1.shape == (self.h0, self.h1) and b0.shape == (self.h0,) and b1.shape == (self.h1,) and b2.shape == (self.out_dim,)
        p = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_float))
        clip = 0.0 if not np.isfinite(in_clip) else float(in_clip)
        self.h = L.dm_mlp_create(device, self.in_dim, self.h0, self.h1, self.out_dim, p(w0), p(b0), p(w1), p(b1), p(w2), p(b2), p(in_mean), p(in_std), clip, p(out_mean), p(out_std), max_rows)
        if not self.h:
            raise RuntimeError("dm_mlp_create failed: %s" % L.dm_last_error().decode())
        self.h = C.c_void_p(self.h)
        self.max_rows = max_rows

    def forward(self, obs, actions, noise=None, stream=None):
        """obs [rows, in_dim], actions [rows, out_dim] (written), noise [rows, out_dim] or None: contiguous float32 CUDA tensors; stream: cudaStream_t handle (int) or None"""
        rows = obs.shape[0]
        _call("dm_mlp_forward", self.h, C.c_void_p(obs.data_ptr()), C.c_void_p(noise.data_ptr()) if noise is not None else None, C.c_void_p(actions.data_ptr()),
              rows, stream=stream)
        return actions

    def set_weights_device(self, layers, stream=None):
        """dm_mlp_set_weights_device: re-tiles the handle on the device from three torch Linear layers with fp32 CUDA parameters (the two hidden
        layers and the output layer; [out, in] weights); the normalisers are kept"""
        shapes = [(self.h0, self.in_dim), (self.h0,), (self.h1, self.h0), (self.h1,), (self.out_dim, self.h1), (self.out_dim,)]
        tensors = [t for l in layers for t in (l.weight, l.bias)]
        for t, shape in zip(tensors, shapes):
            _check_device_f32(t, "set_weights_device", shape)
        ptrs = [C.c_void_p(t.data_ptr()) for t in tensors]
        _call("dm_mlp_set_weights_device", self.h, *ptrs, stream=stream)

    def set_normalizers_device(self, in_mean, in_std, out_mean, out_std, stream=None):
        """dm_mlp_set_normalizers_device: the input and output normalisers from contiguous float32 CUDA tensors ([in_dim], [out_dim]) on the
        device, the values dm_mlp_create would store"""
        for name, t, n in (("in_mean", in_mean, self.in_dim), ("in_std", in_std, self.in_dim), ("out_mean", out_mean, self.out_dim), ("out_std", out_std, self.out_dim)):
            _check_device_f32(t, "set_normalizers_device: " + name, (n,))
        _call("dm_mlp_set_normalizers_device", self.h, *[C.c_void_p(t.data_ptr()) for t in (in_mean, in_std, out_mean, out_std)], stream=stream)

    def style_reward(self, amp_obs, reward, task_reward=None, task_lerp=0.0, logit=None, style=None, stream=None):
        """dm_mlp_forward_style_reward: the discriminator's logit d on amp_obs [rows, in_dim], style = max(0, 1 - 0.25 (1 - d)^2) and
        reward [rows] (written) = (1 - task_lerp) style + task_lerp task_reward, or style without task_reward.  logit / style [rows] are
        written when given.  Contiguous float32 CUDA tensors; stream: cudaStream_t handle (int) or None"""
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        _call("dm_mlp_forward_style_reward", self.h, ptr(amp_obs), ptr(task_reward), float(task_lerp), ptr(logit), ptr(style), ptr(reward), amp_obs.shape[0],
              stream=stream)
        return reward

class TensorCoreGatedMLP(_MlpHandle):
    """dm_mlp_* handle of the gated (goal-conditioned) actor of the AMP task scenes, fc_2layers_gated_1024units, on the tensor cores (wgmma).
    actor: the reference's layout (deepmimic_b200.tf_checkpoint.load_actor, tests.test_task_scenes_cpu.fixture_task_actor): hidden [(w, b)] x 2,
    mean (w, b), gate_common (w, b), gates [dict(hidden=(w, b), scale=(w, b), bias=(w, b))] x 2; dense kernels are [inputs x units] arrays."""

    def __init__(self, actor, s_mean=None, s_std=None, s_clip=float("inf"), g_mean=None, g_std=None, g_clip=float("inf"), a_mean=None, a_std=None,
                 max_rows=4096, device=0):
        L = lib()
        f = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float32)
        hidden, gates = actor["hidden"], actor["gates"]
        if len(hidden) != 2 or len(gates) != 2:
            raise ValueError("the tensor-core gated actor implements exactly two hidden layers (got %d, %d gates)" % (len(hidden), len(gates)))
        (w0, b0), (w1, b1), (w2, b2), (gcw, gcb) = [(f(w), f(b)) for w, b in list(hidden) + [actor["mean"], actor["gate_common"]]]
        gh, gs, gb = ([(f(g[k][0]), f(g[k][1])) for g in gates] for k in ("hidden", "scale", "bias"))
        norms = [f(x) for x in (s_mean, s_std, g_mean, g_std, a_mean, a_std)]
        self.goal_dim, gate_common = gcw.shape
        self.in_dim, self.out_dim = w0.shape[0] - self.goal_dim, w2.shape[1]
        gate_hidden = gh[0][0].shape[1]
        self.h0, self.h1, self.gate_common, self.gate_hidden = w0.shape[1], w1.shape[1], gate_common, gate_hidden
        p = lambda a: None if a is None else a.ctypes.data_as(_fp)
        pair = lambda ab, i: (_fp * 2)(p(ab[0][i]), p(ab[1][i]))
        W = DmMlpGatedWeights(self.in_dim, self.goal_dim, w0.shape[1], w1.shape[1], self.out_dim, gate_common, gate_hidden,
                              p(w0), p(b0), p(w1), p(b1), p(w2), p(b2), p(gcw), p(gcb),
                              pair(gh, 0), pair(gh, 1), pair(gs, 0), pair(gs, 1), pair(gb, 0), pair(gb, 1),
                              *[p(a) for a in norms], 0.0 if not np.isfinite(s_clip) else float(s_clip), 0.0 if not np.isfinite(g_clip) else float(g_clip))
        self.h = L.dm_mlp_create_gated(device, C.byref(W), max_rows)
        if not self.h:
            raise RuntimeError("dm_mlp_create_gated failed: %s" % L.dm_last_error().decode())
        self.h = C.c_void_p(self.h)
        self.max_rows = max_rows

    def forward(self, obs, goal, actions, noise=None, stream=None):
        """obs [rows, in_dim], goal [rows, goal_dim], actions [rows, out_dim] (written), noise [rows, out_dim] or None: contiguous float32 CUDA
        tensors; stream: cudaStream_t handle (int) or None"""
        rows = obs.shape[0]
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        _call("dm_mlp_forward_gated", self.h, ptr(obs), ptr(goal), ptr(noise), ptr(actions), rows, stream=stream)
        return actions

    def set_weights_device(self, layers, stream=None):
        """dm_mlp_set_gated_weights_device: re-tiles the handle on the device from the ten torch Linear layers of gated_layers(net, head)
        with fp32 CUDA parameters ([out, in] weights); the normalisers are kept"""
        S, G, h0, h1, A, GC, GH = self.in_dim, self.goal_dim, self.h0, self.h1, self.out_dim, self.gate_common, self.gate_hidden
        shapes = _gated_shapes(S, G, h0, h1, A, GC, GH)
        if len(layers) != 10:
            raise ValueError("set_weights_device: need the ten layers of gated_layers() (got %d)" % len(layers))
        for l, shape in zip(layers, shapes):
            _check_device_f32(l.weight, "set_weights_device", shape)
            _check_device_f32(l.bias, "set_weights_device", shape[:1])
        w = (C.c_void_p * 10)(*[l.weight.data_ptr() for l in layers])
        b = (C.c_void_p * 10)(*[l.bias.data_ptr() for l in layers])
        _call("dm_mlp_set_gated_weights_device", self.h, w, b, stream=stream)

    def set_normalizers_device(self, s_mean, s_std, g_mean, g_std, out_mean, out_std, stream=None):
        """dm_mlp_set_gated_normalizers_device: the state, goal and output normalisers from contiguous float32 CUDA tensors ([in_dim],
        [goal_dim], [out_dim]) on the device, the values dm_mlp_create_gated would store"""
        ts = (("s_mean", s_mean, self.in_dim), ("s_std", s_std, self.in_dim), ("g_mean", g_mean, self.goal_dim), ("g_std", g_std, self.goal_dim),
              ("out_mean", out_mean, self.out_dim), ("out_std", out_std, self.out_dim))
        for name, t, n in ts:
            _check_device_f32(t, "set_normalizers_device: " + name, (n,))
        _call("dm_mlp_set_gated_normalizers_device", self.h, *[C.c_void_p(t.data_ptr()) for _, t, _ in ts], stream=stream)

class TensorCoreLearner:
    """dm_learn_* workspace: minibatch steps of a plain 2-layer torch network on the tensor cores: PPO steps of build_policy (kind "actor") and
    build_critic (kind "critic"), AMP discriminator steps of build_discriminator (kind "disc", max_rows = agent + expert rows of a step).  The
    network's parameters and the momentum accumulators `acc` ({parameter: tensor}) are updated in place; both must be contiguous float32 CUDA
    tensors on the workspace's device.  Their device pointers are read again (and checked) by every set_weights(), so a network moved after
    construction is picked up there, or refused."""
    KINDS = dict(actor=0, critic=1, disc=2)
    _NET, _SET = DmLearnNet, "dm_learn_set_weights"

    def __init__(self, net, acc, kind, max_rows, device=0):
        if kind not in self.KINDS:
            raise ValueError("kind must be 'actor', 'critic' or 'disc' (got %r)" % (kind,))
        if getattr(net, "goal_size", 0) or hasattr(net, "gate_common") or len(net.hidden) != 2:
            raise ValueError("the tensor-core learner implements the plain network with exactly two hidden layers (gated networks: "
                             "TensorCoreGatedLearner)")
        self.layers = tc_layers(net, kind)
        self._step_fn, self._grad_fn, self._apply_fn = (("dm_learn_disc_step", "dm_learn_disc_grad", "dm_learn_disc_apply") if kind == "disc" else
                                                        ("dm_learn_step", "dm_learn_grad", "dm_learn_apply"))
        self.acc, self.device = acc, device
        ins, outs = [l.weight.shape[1] for l in self.layers], [l.weight.shape[0] for l in self.layers]
        L = lib()
        self.h = L.dm_learn_create(device, self.KINDS[kind], ins[0], outs[0], outs[1], outs[2], max_rows)
        if not self.h:
            raise RuntimeError("dm_learn_create failed: %s" % L.dm_last_error().decode())
        self.h = C.c_void_p(self.h)
        self.net = None
        self._bind()

    def _bind(self):
        import torch
        dev = torch.device("cuda", self.device)
        for l in self.layers:
            for p in (l.weight, l.bias):
                if p not in self.acc:
                    raise ValueError("TensorCoreLearner: a parameter has no momentum accumulator (the network's parameters were replaced)")
                _check_device_f32(p, "TensorCoreLearner parameter", None, dev)
                _check_device_f32(self.acc[p], "TensorCoreLearner accumulator", tuple(p.shape), dev)
        p = lambda t: C.c_void_p(t.data_ptr())
        arr = lambda ts: (C.c_void_p * len(ts))(*[p(t) for t in ts])
        self.net = self._NET(arr([l.weight for l in self.layers]), arr([l.bias for l in self.layers]),
                             arr([self.acc[l.weight] for l in self.layers]), arr([self.acc[l.bias] for l in self.layers]))

    def set_weights(self, stream=None):
        """binds the parameters' current storage (checked) and loads their values into the workspace's tiles"""
        self._bind()
        _call(self._SET, self.h, C.byref(self.net), stream=stream)

    def step(self, batch, stream=None):
        """batch: a DmLearnBatch (kinds "actor", "critic"), a DmLearnDiscBatch (kind "disc") or a DmLearnGatedBatch (TensorCoreGatedLearner)"""
        _call(self._step_fn, self.h, C.byref(self.net), C.byref(batch), stream=stream)

    # ---- the step split around its gradient (data-parallel training): step(b) == grad(b, g); apply(b, g, 1.0), bit for bit
    def grad_size(self):
        """dm_learn_grad_size: the floats of the flat gradient, the parameter pairs of self.layers as [weight, bias] each"""
        return int(lib().dm_learn_grad_size(self.h))

    def grad_views(self, grad):
        """{parameter: view of the flat gradient `grad` (a tensor of grad_size() floats) with the parameter's shape}"""
        views, off = {}, 0
        for l in self.layers:
            for p in (l.weight, l.bias):
                views[p] = grad[off:off + p.numel()].view(p.shape)
                off += p.numel()
        return views

    def _check_grad(self, grad, what):
        import torch
        _check_device_f32(grad, what, (self.grad_size(),), torch.device("cuda", self.device))

    def grad(self, batch, grad, stream=None):
        """dm_learn_(gated_|disc_)grad: the step's forward, head (its statistics accumulate) and backward, then the mean gradient over the
        batch's rows without the weight decay (and logit regulariser) into `grad`, a contiguous float32 CUDA tensor of grad_size() floats;
        the parameters are not changed"""
        self._check_grad(grad, "grad")
        _call(self._grad_fn, self.h, C.byref(self.net), C.byref(batch), C.c_void_p(grad.data_ptr()), stream=stream)

    def apply(self, batch, grad, scale=1.0, stream=None):
        """dm_learn_(gated_|disc_)apply: the optimiser step on scale * grad plus the weight decay (and logit regulariser) with the batch's
        stepsize and momentum, and the re-tiling"""
        self._check_grad(grad, "apply")
        _call(self._apply_fn, self.h, C.byref(self.net), C.byref(batch), C.c_void_p(grad.data_ptr()), C.c_float(scale), stream=stream)

    def close(self):
        if self.h:
            lib().dm_learn_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def gated_layers(net, head):
    """the ten Linear layers of a gated network (build_gated_policy, or build_critic with a goal) in dm_learn_gated_net's order: hidden[0],
    hidden[1], the output layer `head`, gate_common, gate_hidden[0], gate_hidden[1], gate_scale[0], gate_scale[1], gate_bias[0], gate_bias[1]"""
    return (list(net.hidden) + [head, net.gate_common] + list(net.gate_hidden) + list(net.gate_scale) + list(net.gate_bias))


def tc_layers(net, role):
    """the layers the tensor-core entries take for `net` in `role`: the hidden layers and the head (actor: mean, critic: out, disc: logit), or gated_layers()"""
    head = getattr(net, dict(actor="mean", critic="out", disc="logit")[role])
    return gated_layers(net, head) if hasattr(net, "gate_common") else list(net.hidden) + [head]


def _gated_shapes(S, G, h0, h1, A, GC, GH):
    """the [out, in] weight shapes of gated_layers() for state size S, goal size G, hidden (h0, h1), A outputs and gate sizes GC, GH"""
    return [(h0, S + G), (h1, h0), (A, h1), (GC, G), (GH, GC), (GH, GC), (h0, GH), (h1, GH), (h0, GH), (h1, GH)]


class TensorCoreGatedLearner(TensorCoreLearner):
    """dm_learn_*_gated workspace: PPO minibatch steps of the gated actor (build_gated_policy, kind "actor") or the gated critic (build_critic
    with a goal, kind "critic") of the AMP task scenes, as TensorCoreLearner does for the plain networks (same contract for the parameters and
    accumulators; the ten parameter pairs of gated_layers()).  The sizes dm_mlp_create_gated accepts: two hidden layers, goal size <= 64,
    gate_common <= 128, gate_hidden <= 64, at most 64 outputs."""
    KINDS = dict(actor=0, critic=1)
    _NET, _SET, _step_fn, _grad_fn, _apply_fn = DmLearnGatedNet, "dm_learn_set_gated_weights", "dm_learn_gated_step", "dm_learn_gated_grad", "dm_learn_gated_apply"

    def __init__(self, net, acc, kind, max_rows, device=0):
        if kind not in self.KINDS:
            raise ValueError("kind must be 'actor' or 'critic' (got %r)" % (kind,))
        G = getattr(net, "goal_size", 0)
        if not G or not hasattr(net, "gate_common") or len(net.hidden) != 2 or len(net.gate_hidden) != 2:
            raise ValueError("the gated tensor-core learner implements the gated network with exactly two hidden layers (plain networks: "
                             "TensorCoreLearner)")
        self.layers = tc_layers(net, kind)
        h0, h1, A = (l.weight.shape[0] for l in self.layers[:3])
        S = self.layers[0].weight.shape[1] - G
        GC, GH = net.gate_common.weight.shape[0], net.gate_hidden[0].weight.shape[0]
        for name, v, hi in (("goal size", G, 64), ("gate_common", GC, 128), ("gate_hidden", GH, 64), ("outputs", A, 64)):
            if v > hi:
                raise ValueError("the gated tensor-core learner supports %s <= %d (got %d)" % (name, hi, v))
        for l, shape in zip(self.layers, _gated_shapes(S, G, h0, h1, A, GC, GH)):
            if tuple(l.weight.shape) != shape or tuple(l.bias.shape) != shape[:1]:
                raise ValueError("the gated network's layers do not have the shapes of one gated network: %s against %s" % (tuple(l.weight.shape), shape))
        self.acc, self.device = acc, device
        L = lib()
        self.h = L.dm_learn_create_gated(device, self.KINDS[kind], S, G, h0, h1, A, GC, GH, max_rows)
        if not self.h:
            raise RuntimeError("dm_learn_create_gated failed: %s" % L.dm_last_error().decode())
        self.h = C.c_void_p(self.h)
        self.net = None
        self._bind()
