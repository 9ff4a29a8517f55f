"""Batched mirror of the reference's Python env surface (R/env/deepmimic_env.py:6-187, R/env/env.py:6-230) over the
C ABI.  Method names and meanings follow DeepMimicEnv; what was a per-agent vector there is an [N, .] CUDA tensor here
(N environments of this rank), and `agent_id` is accepted and ignored (the imitation scene has one agent).
For the unmodified single-env reference wrapper use the `DeepMimicCore` package next to this file instead."""
import numpy as np

from .capi import (BatchedCore, DM_ACTION_BOUND_MAX, DM_ACTION_BOUND_MIN, DM_ACTION_OFFSET, DM_ACTION_SCALE, DM_STATE_NORM_GROUPS,
                   DM_STATE_OFFSET, DM_STATE_SCALE)
from .sharding import StepExchange, pack_rows, rank_world, shard_range


class DeepMimicBatchEnv:
    class Terminate:
        Null, Fail, Succ = 0, 1, 2

    UPDATE_DT = 1.0 / 600.0   # the reference's update timestep (600 Hz), step()'s default

    def __init__(self, args, num_envs, asset_root, device=0, seed=0, global_env_offset=0):
        import torch
        self.torch = torch
        self._core = BatchedCore(list(args), num_envs, asset_root, device=device, seed=seed, global_env_offset=global_env_offset)
        d = self._core.dims
        self.num_envs, self.device = d.num_envs, torch.device("cuda", device)
        self.stream = torch.cuda.ExternalStream(self._core.stream(), device=device)
        with torch.cuda.stream(self.stream):
            self._obs = torch.zeros(d.num_envs, d.state_size, device=self.device)
            self._rew = torch.zeros(d.num_envs, device=self.device)
            self._flags = torch.zeros(d.num_envs, 4, dtype=torch.int32, device=self.device)
        self._time = 0.0
        self._core.reset(True)

    # ---- stream ordering: the library works on its own stream; these two event waits make every method safe to call
    # from torch's current stream (inputs produced there are complete before the kernels read them, returned tensors are
    # complete before the caller's next op on that stream reads them).  No host synchronisation.
    def _pre(self):
        self.stream.wait_stream(self.torch.cuda.current_stream(self.device))

    def _post(self):
        self.torch.cuda.current_stream(self.device).wait_stream(self.stream)

    # ---- scene control (cDeepMimicCore::Update / Reset / GetTime, DeepMimicCore.cpp:88-139)
    def update(self, timestep, n_updates=1):
        self._core.update(timestep, n_updates)
        self._time += timestep * n_updates

    def reset(self, force_all=False):
        """Restarts finished episodes (every environment with force_all)."""
        self._pre()
        self._core.reset(force_all)

    def get_time(self):
        return self._time

    def set_pushes(self, body, force, start, duration):
        """Push the characters: environment e's body body[e] (-1: none) gets force[e] (world axes, unscaled N, at the body's COM) in every
        update whose episode time at its start t satisfies start[e] <= t < start[e] + duration[e].  Shapes [N], [N, 3], [N], [N]; dtypes int32,
        float32, float64, float64 (numpy arrays or tensors).  An entry clears once its window has passed and at the environment's reset."""
        self._pre()
        self._core.set_pushes(body, force, start, duration)

    def set_push_schedule(self, bodies, force, duration, gap):
        """Push the characters at random, for training under pushes: at every update() each running environment whose push has ended gets the
        next one, on a body drawn from `bodies`, horizontal, of magnitude in force = (lo, hi) N, for duration = (lo, hi) s, starting gap = (lo,
        hi) s after the end of the previous push of its episode.  The draws are made on the device from the env's seed and each environment's
        global id (include/deepmimic_b200.h: dm_set_push_schedule); state_dict() carries them."""
        self._pre()
        self._core.set_push_schedule(bodies, force, duration, gap)

    def set_dynamics(self, friction=None, kp=None, kd=None, torque_limit=None, mass=None):
        """Vary the dynamics per environment: friction, kp, kd and torque_limit [N] multiply the contact friction coefficient, every PD
        controller's Kp and Kd and every joint's torque limit; mass [N, links] multiplies every body's mass (and with it both inertias).  An
        omitted kind is 1.  Kept across resets; state_dict() carries them.  The policy's observations do not see them."""
        N, nl = self._core.num_envs, self._core.dims.num_joints
        f = np.ones((N, 4 + nl), dtype=np.float32)
        for j, (name, a) in enumerate((("friction", friction), ("kp", kp), ("kd", kd), ("torque_limit", torque_limit))):
            if a is not None:
                a = np.asarray(a.detach().cpu().numpy() if hasattr(a, "detach") else a, dtype=np.float32)
                if a.shape != (N,):
                    raise ValueError("set_dynamics: %s must have shape (%d,), got %s" % (name, N, a.shape))
                f[:, j] = a
        if mass is not None:
            m = np.asarray(mass.detach().cpu().numpy() if hasattr(mass, "detach") else mass, dtype=np.float32)
            if m.shape != (N, nl):
                raise ValueError("set_dynamics: mass must have shape (%d, %d), got %s" % (N, nl, m.shape))
            f[:, 4:] = m
        self._pre()
        self._core.set_dynamics(f)

    def dynamics(self):
        """every environment's factors as device tensors: dict(friction, kp, kd, torque_limit [N], mass [N, links]).  No host synchronisation."""
        self._pre()
        t = self._core.dynamics()
        self._post()
        return dict(friction=t[:, 0], kp=t[:, 1], kd=t[:, 2], torque_limit=t[:, 3], mass=t[:, 4:])

    def set_dynamics_randomization(self, friction=(1.0, 1.0), kp=(1.0, 1.0), kd=(1.0, 1.0), torque_limit=(1.0, 1.0), mass=(1.0, 1.0)):
        """Randomise the dynamics for training: every environment draws its factors (as in set_dynamics; one mass factor per body) uniformly in
        each kind's (lo, hi) on the device, now and at every reset, from the env's seed and its global id
        (include/deepmimic_b200.h: dm_set_dynamics_randomization).  An omitted kind stays 1.  state_dict() carries the table."""
        lohi = []
        for name, p in (("friction", friction), ("kp", kp), ("kd", kd), ("torque_limit", torque_limit), ("mass", mass)):
            p = tuple(float(v) for v in p)
            if len(p) != 2:
                raise ValueError("set_dynamics_randomization: %s must be a (lo, hi) pair" % name)
            lohi += p
        self._pre()
        self._core.set_dynamics_randomization(lohi)

    def set_action_latency(self, seconds):
        """Delay every environment's actions: the PD targets of an action take effect seconds[e] after set_action (a whole number of updates,
        rounded to the nearest, in [0, (updates_per_action - 1) UPDATE_DT]); until then the previous targets act, and a reset holds the start
        pose.  [N] seconds; kept across resets; state_dict() carries them and any pending action.  The policy's observations do not see it."""
        self._pre()
        self._core.set_action_latency(seconds)

    def set_action_latency_randomization(self, lo, hi):
        """Randomise the control latency for training: every environment draws its delay uniformly among the whole updates of [lo, hi] seconds on
        the device, now and at every reset, from the env's seed and its global id (include/deepmimic_b200.h: dm_set_action_latency_randomization)"""
        self._pre()
        self._core.set_action_latency_randomization(lo, hi)

    def action_latency(self):
        """every environment's current control latency in seconds, a float64 device tensor [N].  No host synchronisation."""
        self._pre()
        t = self._core.action_latency()
        self._post()
        return t

    def set_goal_course(self, rows, counts=None):
        """Steer the heading and target scenes: commanded goals instead of the scene's random ones (include/deepmimic_b200.h:
        dm_set_goal_course).  heading_amp / heading_amp_getup: rows of (episode time s, heading rad, speed m/s), times increasing from >= 0, the
        goal linear in time between them; target_amp: rows of (dx, dz) m, waypoints relative to the root where the course starts, each
        reached within the scene's success radius.  rows [K, 3 or 2] gives every environment the same course; [N, K, 3 or 2] with counts [N]
        (default K each; 0 keeps the scene's own goals) gives each its own.  K <= 16.  Every course restarts now and at each reset;
        course_record() reports how it is followed.  Synchronises the stream."""
        from .capi import MAX_COURSE_POINTS
        kind = int(self._core.task_params()[0][0])
        width = 2 if kind == 1 else 3   # target_amp: (dx, dz); the heading scenes (t, h, v); the library refuses the other scenes
        r = np.asarray(rows.detach().cpu().numpy() if hasattr(rows, "detach") else rows, dtype=np.float64)
        N = self.num_envs
        if r.ndim == 2:
            if counts is not None:
                raise ValueError("set_goal_course: counts go with per-environment rows [N, K, %d]" % width)
            r = np.broadcast_to(r, (N,) + r.shape)
        if r.ndim != 3 or r.shape[0] != N or r.shape[2] != width or not 1 <= r.shape[1] <= MAX_COURSE_POINTS:
            raise ValueError("set_goal_course: rows must be [K, %d] or [%d, K, %d] with 1 <= K <= %d in this scene, got %s" % (
                width, N, width, MAX_COURSE_POINTS, r.shape))
        K = r.shape[1]
        n = np.full(N, K, dtype=np.int32) if counts is None else np.asarray(counts, dtype=np.int64).reshape(-1)
        if n.shape != (N,) or n.min() < 0 or n.max() > K:
            raise ValueError("set_goal_course: counts must be %d values in [0, %d]" % (N, K))
        full = np.zeros((N, MAX_COURSE_POINTS, 3))
        full[:, :K, :width] = r
        self._pre()
        self._core.set_goal_course(n.astype(np.int32), full)
        self.course_counts = n.astype(np.int32)
        self.course_kind = "target" if kind == 1 else "heading"

    def course_record(self):
        """[N, 4] float32: every environment's record of its last step (or course start): heading scenes (goal point 1.5 m ahead of the root
        along the commanded heading x, z; along-track speed minus the commanded speed; cross-track speed towards heading + pi / 2, m/s); the
        target scene (the goal waypoint's x, z; waypoints reached; distance to the goal waypoint, m).  A view of a buffer rewritten by the next
        call, like record_state; no host synchronisation."""
        if getattr(self, "_course_rec", None) is None:
            with self.torch.cuda.stream(self.stream):
                self._course_rec = self.torch.zeros(self.num_envs, 4, device=self.device)
        self._pre()
        self._core.course_record(self._course_rec)
        self._post()
        return self._course_rec

    def get_name(self):
        """cScene::GetName of the configured scene (SceneImitate.cpp:209, SceneImitateAMP.cpp:211, SceneTargetAMP.cpp:233, ...)"""
        return self._core.scene_name()

    def is_rl_scene(self):
        return True

    def get_num_agents(self):
        return 1

    def get_updates_per_action(self):
        """updates per policy step (20 for the shipped arg files: 30 Hz queries at 600 Hz updates)"""
        return self._core.dims.updates_per_action

    def get_num_update_substeps(self):
        return self._core.dims.num_update_substeps

    def set_mode(self, mode):
        self._core.set_mode(int(mode))

    def set_sample_count(self, count):
        """RLWorld feeds the learner's sample count back every iteration (R/learning/rl_agent.py -> env.set_sample_count):
        anneals the episode time limits of the following resets."""
        self._pre()
        self._core.set_sample_count(int(count))
        self._post()

    # ---- per-step queries; tensors are views of buffers rewritten by the next call
    def _refresh_flags(self):
        self._pre()
        self._core.flags(self._flags)
        self._post()
        return self._flags

    def need_new_action(self, agent_id=0):
        return self._refresh_flags()[:, 0].bool()

    def record_state(self, agent_id=0):
        self._pre()
        self._core.observe(self._obs, None)
        self._post()
        return self._obs

    def record_goal(self, agent_id=0):
        """[N, goal_size] float32 (goal_size 0 outside the AMP task scenes, 3 in target_amp / heading_amp)."""
        g = self._core.dims.goal_size
        if g == 0:
            return self.torch.zeros(self.num_envs, 0, device=self.device)
        if getattr(self, "_goal", None) is None:
            with self.torch.cuda.stream(self.stream):
                self._goal = self.torch.zeros(self.num_envs, g, device=self.device)
        self._pre()
        self._core.record_goal(self._goal)
        self._post()
        return self._goal

    def record_pose(self, agent_id=0):
        """(pose, vel): [N, pose_dim] float32 each, every simulated character's pose and velocity in the reference's layout
        (cSimCharacter::BuildPose / BuildVel: root position, root quaternion w x y z, joint quaternions or angles; root linear and angular
        velocity, joint velocities), what cMotion files hold per frame.  Views of buffers rewritten by the next call, like record_state."""
        if getattr(self, "_pose", None) is None:
            P = self._core.dims.pose_dim
            with self.torch.cuda.stream(self.stream):
                self._pose = self.torch.zeros(self.num_envs, P, device=self.device)
                self._vel = self.torch.zeros(self.num_envs, P, device=self.device)
        self._pre()
        self._core.record_pose(self._pose, self._vel)
        self._post()
        return self._pose, self._vel

    def record_kin_pose(self, agent_id=0):
        """[N, pose_dim] float32: every kinematic character's pose (the clip at the environment's kin time, placed in the world as the imitation
        reward compares it) in record_pose's layout.  A view of a buffer rewritten by the next call, like record_pose."""
        if getattr(self, "_kin_pose", None) is None:
            with self.torch.cuda.stream(self.stream):
                self._kin_pose = self.torch.zeros(self.num_envs, self._core.dims.pose_dim, device=self.device)
        self._pre()
        self._core.record_kin_pose(self._kin_pose)
        self._post()
        return self._kin_pose

    def render(self, env_ids=None, **kw):
        """(rgb uint8 [V, H, W, 3], ids int16 [V, H, W]) device tensors: the current simulated characters of env_ids (default all; a sequence
        or tensor of environment indices) drawn by the device ray caster from their record_pose rows; keyword arguments are
        BatchedCore.render_poses' (camera, width, height, rgb, ids).  Ordered on the caller's stream like record_state, no host
        synchronisation (host indices go to the device through pinned memory); the simulation state is not touched."""
        pose, _ = self.record_pose()
        if env_ids is not None:
            idx = self.torch.as_tensor(env_ids, dtype=self.torch.long)
            if not idx.is_cuda:
                idx = idx.pin_memory()
            pose = pose[idx.to(self.device, non_blocking=True)].contiguous()
        self._pre()
        out = self._core.render_poses(pose, **kw)
        self._post()
        return out

    def set_action(self, agent_id_or_actions, actions=None):
        a = agent_id_or_actions if actions is None else actions
        if tuple(a.shape) != (self.num_envs, self.get_action_size()) or a.dtype != self.torch.float32 or not a.is_cuda:
            raise ValueError("actions must be a float32 CUDA tensor [%d, %d]" % (self.num_envs, self.get_action_size()))
        self._pre()
        self._core.set_action(a.contiguous())

    def calc_reward(self, agent_id=0):
        self._pre()
        self._core.observe(None, self._rew)
        self._post()
        return self._rew

    # ---- AMP observations (R/env/deepmimic_env.py:147-166)
    def get_amp_obs_size(self):
        return self._core.dims.amp_obs_size

    def enable_amp_task_reward(self):
        return self._core.dims.goal_size > 0                # cSceneTargetAMP::EnableAMPTaskReward (SceneTargetAMP.cpp:222-225); false in imitate_amp

    def get_amp_obs_offset(self):
        return np.zeros(self.get_amp_obs_size())

    def get_amp_obs_scale(self):
        return np.ones(self.get_amp_obs_size())

    def get_amp_obs_norm_group(self):
        return np.zeros(self.get_amp_obs_size(), dtype=np.int32)

    def _amp_buf(self, which):
        # two buffers: the AMP agent fetches the agent's and the expert's observations of a step and stores both (R/learning/amp_agent.py:244-285)
        name = "_amp_" + which
        if not hasattr(self, name):
            with self.torch.cuda.stream(self.stream):
                setattr(self, name, self.torch.zeros(self.num_envs, self.get_amp_obs_size(), device=self.device))
        return getattr(self, name)

    def record_amp_obs_agent(self, agent_id=0):
        buf = self._amp_buf("agent")
        self._pre(); self._core.amp_obs_agent(buf); self._post()
        return buf

    def record_amp_obs_expert(self, agent_id=0, kin_time=None):
        buf = self._amp_buf("expert")
        self._pre(); self._core.amp_obs_expert(buf, kin_time); self._post()
        return buf

    def expert_sample_count(self, set_to=None):
        """the expert sampler's call counter, the key of sample_amp_obs_expert's next draws (dm_expert_sample_count); set_to replaces it.
        Returns the value before the call.  Handles of one seed draw the same rows at the same count: data-parallel ranks start from
        disjoint counts."""
        return self._core.expert_sample_count(set_to)

    def sample_amp_obs_expert(self, rows):
        """[rows, amp_obs_size] float32: `rows` expert AMP observations (any count), clip and time drawn on the device per row
        (dm_sample_amp_obs_expert).  A new tensor each call, allocated on the caller's current stream and complete before that stream's next
        op, like any tensor torch makes there (a consumer on another stream needs the usual record_stream); no host synchronisation."""
        out = self.torch.empty(int(rows), self.get_amp_obs_size(), device=self.device)
        self._pre(); self._core.sample_amp_obs_expert(out); self._post()
        return out

    def is_episode_end(self):
        return self._refresh_flags()[:, 1].bool()

    def check_terminate(self, agent_id=0):
        return self._refresh_flags()[:, 2]

    def check_valid_episode(self):
        return self._refresh_flags()[:, 3].bool()

    def step(self, actions, timestep=UPDATE_DT):
        """One policy step: SetAction, the controller's query period worth of Update(timestep) calls (20 at the
        reference's 600 Hz / 30 Hz), then state, reward and flags.  Returns (obs, reward, done, terminate)."""
        self.set_action(actions)
        self.update(timestep, self._core.dims.updates_per_action)
        self._core.observe(self._obs, self._rew)
        f = self._refresh_flags()          # ends with _post(): obs / reward / flags are ordered before the caller's stream
        return self._obs, self._rew, f[:, 1].bool(), f[:, 2]

    # ---- sizes and normalisation statics (DeepMimicCore.cpp:246-330)
    def get_action_space(self, agent_id=0):
        return 0  # ActionSpace.Continuous

    def get_state_size(self, agent_id=0):
        return self._core.dims.state_size

    def get_pose_dim(self, agent_id=0):
        """length of a pose or velocity row of record_pose (43 humanoid3d, 83 dog3d)"""
        return self._core.dims.pose_dim

    def get_goal_size(self, agent_id=0):
        return self._core.dims.goal_size

    def get_action_size(self, agent_id=0):
        return self._core.dims.action_size

    def get_num_actions(self, agent_id=0):
        return 0

    def build_state_offset(self, agent_id=0):
        return np.array(self._core.static(DM_STATE_OFFSET))

    def build_state_scale(self, agent_id=0):
        return np.array(self._core.static(DM_STATE_SCALE))

    def _task_kind(self):
        """0 none, 1 target_amp, 2 heading_amp, 3 heading_amp_getup, 4 strike_amp (dm_task.cuh: TaskKind)"""
        return int(self._core.task_params()[0][0]) if self._core.dims.goal_size > 0 else 0

    def build_goal_offset(self, agent_id=0):
        off = np.zeros(self._core.dims.goal_size)           # cRLSceneSimChar::BuildGoalOffsetScale (RLSceneSimChar.cpp:111-116)
        if self._task_kind() == 3:
            off[3] = -0.5                                   # the get-up phase (SceneHeadingAMPGetup.cpp:142-149)
        return off

    def build_goal_scale(self, agent_id=0):
        scl = np.ones(self._core.dims.goal_size)
        if self._task_kind() == 3:
            scl[3] = 2.0
        return scl

    def build_action_offset(self, agent_id=0):
        return np.array(self._core.static(DM_ACTION_OFFSET))

    def build_action_scale(self, agent_id=0):
        return np.array(self._core.static(DM_ACTION_SCALE))

    def build_action_bound_min(self, agent_id=0):
        return np.array(self._core.static(DM_ACTION_BOUND_MIN))

    def build_action_bound_max(self, agent_id=0):
        return np.array(self._core.static(DM_ACTION_BOUND_MAX))

    def build_state_norm_groups(self, agent_id=0):
        return np.array(self._core.static(DM_STATE_NORM_GROUPS), dtype=np.int32)

    def build_goal_norm_groups(self, agent_id=0):
        g = np.zeros(self._core.dims.goal_size, dtype=np.int32)      # gNormGroupSingle (RLSceneSimChar.cpp:136-140)
        kind = self._task_kind()
        if kind == 3:
            g[3] = -1                                                # gNormGroupNone for the get-up phase (SceneHeadingAMPGetup.cpp:151-157)
        elif kind == 4:
            g[:] = -1                                                # no normalisation of the strike goal (SceneStrikeAMP.cpp:401-405)
        return g

    def get_reward_min(self, agent_id=0):
        return 0.0

    def get_reward_max(self, agent_id=0):
        return 1.0

    def get_reward_fail(self, agent_id=0):
        return 0.0

    def get_reward_succ(self, agent_id=0):
        return 1.0

    def state_dict(self):
        """the whole batch's simulation state (BatchedCore.save_state: every environment's device blocks, the draw counters, mode and time
        limits) and get_time()'s clock; ordered after the caller's stream's work, and synchronising.  blob is a CPU uint8 tensor."""
        import torch
        self._pre()
        return dict(blob=torch.from_numpy(self._core.save_state()), time=self._time)

    def load_state_dict(self, s):
        """restores state_dict() of an env made with the same arguments, num_envs and seed; the caller's stream then waits for the copies"""
        self._pre()
        self._core.load_state(np.asarray(s["blob"]))
        self._time = float(s["time"])
        self._post()

    def sync(self):
        self._core.sync()

    def counters(self):
        """(kernel launches so far, environments whose constraint solver ran out of row capacity).  The second number must stay 0: a
        truncated contact set is a silent deviation from the reference physics (DESIGN.md 5.5)."""
        return self._core.counters()

    def check_solver_capacity(self, raise_on_overflow=True):
        """Call at reset / collect boundaries (host synchronisation).  Raises (or warns) when any environment exceeded the solver's row
        capacity since the handle was created.  The capacity is fixed per character (32 rows humanoid3d, 52 dog3d; DESIGN.md 5.5), so the
        affected episodes are invalid: their contact sets were truncated."""
        over = self._core.counters()[1]
        if over:
            msg = ("deepmimic_b200: %d environment(s) exceeded the contact-solver row capacity of this character; contacts were truncated, "
                   "treat the affected episodes as invalid" % over)
            if raise_on_overflow:
                raise RuntimeError(msg)
            import warnings
            warnings.warn(msg)
        return over


class ShardedDeepMimicEnv(DeepMimicBatchEnv):
    """One process per GPU: this rank owns shard_range(total_envs, rank, world) of the job's environments.  `step` keeps the base
    class's contract (the LOCAL rows: obs, reward, done, terminate -- what a replicated policy acts on); `step_gathered` additionally
    all-gathers every rank's [obs | reward | done] rows so that each rank (the learner) sees the whole job's transitions."""

    def __init__(self, args, total_envs, asset_root, seed=0):
        rank, world, local_rank = rank_world()
        off, cnt = shard_range(total_envs, rank, world)
        super().__init__(args, cnt, asset_root, device=local_rank, seed=seed, global_env_offset=off)
        self.rank, self.world, self.total_envs, self.env_offset = rank, world, total_envs, off
        S = self.get_state_size()
        with self.torch.cuda.stream(self.stream):
            self._rows = self.torch.zeros(cnt, S + 2, device=self.device)
            self._xchg = StepExchange(total_envs, S + 2, rank, world, self.device)

    def gather_rows(self, obs, rew, done):
        """local [cnt, .] rows -> the job's [total_envs, .] rows in global environment order (same on every rank)"""
        allrows = self._xchg.gather(pack_rows(self._rows, obs, rew, done))    # on the caller's stream, after _post()
        S = self.get_state_size()
        return allrows[:, :S], allrows[:, S], allrows[:, S + 1] > 0.5

    def step_gathered(self, actions, timestep=1.0 / 600.0):
        """step() for this rank's environments, then the all-gather: returns (local 4-tuple, (all_obs, all_reward, all_done))."""
        local = self.step(actions, timestep)
        return local, self.gather_rows(local[0], local[1], local[2])
