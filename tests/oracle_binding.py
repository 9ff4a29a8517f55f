"""ctypes binding of the CPU oracle (oracle/libdm_oracle.so).  TEST INFRASTRUCTURE: only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this."""
import ctypes as C

import numpy as np

from deepmimic_b200.build import build_oracle
from tests.dynamics_ref import FRICTION

_LIB = None


def load_oracle():
    """the oracle library, loaded once per process after `make` in oracle/: a change to the oracle or to a header it includes rebuilds it,
    and a current library is loaded as it is"""
    global _LIB
    if _LIB is not None:
        return _LIB
    L = C.CDLL(build_oracle())
    L.dmo_create.restype = C.c_void_p
    L.dmo_create.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_char_p)]
    L.dmo_last_error.restype = C.c_char_p
    for f in ("dmo_calc_reward", "dmo_calc_reward_imitate", "dmo_motion_duration", "dmo_get_time", "dmo_calc_reward_terms", "dmo_u01"):
        getattr(L, f).restype = C.c_double
    L.dmo_u01.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64]
    L.dmo_set_task_stream.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64]
    L.dmo_task_counter.restype = C.c_uint64
    L.dmo_task_counter.argtypes = [C.c_void_p]
    L.dmo_update_pushed.argtypes = [C.c_void_p, C.c_double, C.c_int, C.POINTER(C.c_double), C.c_double, C.c_double]
    L.dmo_set_contact_friction.argtypes = [C.c_void_p, C.c_double]
    _LIB = L
    return L


def dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


class Oracle:
    def __init__(self, args, asset_root):
        L = load_oracle()
        enc = [a.encode() for a in args]
        arr = (C.c_char_p * len(enc))(*enc)
        h = L.dmo_create(asset_root.encode(), len(enc), arr)
        if not h:
            raise RuntimeError("oracle create failed: %s" % L.dmo_last_error().decode())
        self.L, self.h = L, C.c_void_p(h)
        d = (C.c_int * 8)()
        L.dmo_get_dims(self.h, d)
        (self.num_joints, self.pose_dim, self.num_dofs, self.state_size, self.action_size, self.goal_size, self.snapshot_size, self.num_frames) = list(d)
        self.motion_duration = L.dmo_motion_duration(self.h)

    def close(self):
        if self.h:
            self.L.dmo_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self, kin_time=0.0, rot_theta=0.0, max_time=20.0, clip=None):
        if clip is None:
            self.L.dmo_reset(self.h, C.c_double(kin_time), C.c_double(rot_theta), C.c_double(max_time))
        else:
            self.L.dmo_reset_clip(self.h, int(clip), C.c_double(kin_time), C.c_double(rot_theta), C.c_double(max_time))
        self.motion_duration = self.L.dmo_motion_duration(self.h)

    # ---- clip dataset (--kin_ctrl clips)
    def num_clips(self):
        return int(self.L.dmo_num_clips(self.h))

    def clip_table(self):
        n = self.num_clips()
        dur, w, cdf = np.zeros(n), np.zeros(n), np.zeros(n)
        loop = np.zeros(n, dtype=np.int32)
        self.L.dmo_clip_table(self.h, dp(dur), dp(w), dp(cdf), loop.ctypes.data_as(C.POINTER(C.c_int)))
        return dur, w, cdf, loop

    def current_clip(self):
        return int(self.L.dmo_current_clip(self.h))

    def select_clip(self, u01):
        return int(self.L.dmo_select_clip(self.h, C.c_double(u01)))

    # ---- AMP task scenes (target_amp / heading_amp)
    def set_task_stream(self, seed, env, counter=0):
        self.L.dmo_set_task_stream(self.h, seed, env, counter)

    def task_counter(self):
        return int(self.L.dmo_task_counter(self.h))

    def u01(self, seed, a, b):
        return float(self.L.dmo_u01(seed, a, b))

    def record_goal(self):
        out = np.zeros(self.goal_size)
        self.L.dmo_record_goal(self.h, dp(out))
        return out

    def task_state(self):
        """dict(target_pos, target_speed, target_heading, timer, timer_max, prev_action_com)"""
        o = np.zeros(10)
        self.L.dmo_get_task_state(self.h, dp(o))
        return dict(target_pos=o[0:3].copy(), target_speed=o[3], target_heading=o[4], timer=o[5], timer_max=o[6], prev_action_com=o[7:10].copy())

    def set_task_state(self, target_pos, target_speed, target_heading, timer, timer_max, prev_action_com):
        o = np.concatenate([np.asarray(target_pos, dtype=np.float64), [target_speed, target_heading, timer, timer_max], np.asarray(prev_action_com, dtype=np.float64)])
        self.L.dmo_set_task_state(self.h, dp(o))

    def getup_state(self):
        """heading_amp_getup: dict(timer, getup_time, getting_up, contact_fall)"""
        o = np.zeros(4)
        self.L.dmo_get_getup_state(self.h, dp(o))
        return dict(timer=o[0], getup_time=o[1], getting_up=bool(o[2]), contact_fall=bool(o[3]))

    def set_getup_timer(self, t):
        self.L.dmo_set_getup_timer(self.h, C.c_double(t))

    def strike_state(self):
        """strike_amp: dict(hit, hit_time, phase, target_height)"""
        o = np.zeros(4)
        self.L.dmo_get_strike_state(self.h, dp(o))
        return dict(hit=bool(o[0]), hit_time=o[1], phase=o[2], target_height=o[3])

    def set_strike_state(self, hit, hit_time):
        self.L.dmo_set_strike_state(self.h, int(bool(hit)), C.c_double(hit_time))

    def check_target_succ(self):
        return bool(self.L.dmo_check_target_succ(self.h))

    def enable_amp_task_reward(self):
        return bool(self.L.dmo_enable_amp_task_reward(self.h))

    def calc_com(self):
        o = np.zeros(3)
        self.L.dmo_calc_com(self.h, dp(o))
        return o

    def set_mode(self, mode):
        """0 train, 1 test (cRLScene::SetMode): test-mode timer limits, no recovery episodes or initial hits, test-mode get-ups and rewards"""
        self.L.dmo_set_mode(self.h, int(mode))

    def update(self, dt):
        self.L.dmo_update(self.h, C.c_double(dt))

    def set_friction(self, factor):
        """the contact friction coefficient becomes 0.81 x factor"""
        self.L.dmo_set_contact_friction(self.h, C.c_double(FRICTION * float(factor)))

    def set_action(self, a):
        a = np.ascontiguousarray(a, dtype=np.float64)
        self.L.dmo_set_action(self.h, dp(a))

    def record_state(self):
        out = np.zeros(self.state_size)
        self.L.dmo_record_state(self.h, dp(out))
        return out

    def calc_reward(self):
        return self.L.dmo_calc_reward(self.h)

    def calc_reward_imitate(self):
        return self.L.dmo_calc_reward_imitate(self.h)

    def amp_obs_size(self):
        return int(self.L.dmo_amp_obs_size(self.h))

    def record_amp_obs_agent(self):
        out = np.zeros(self.amp_obs_size())
        self.L.dmo_record_amp_obs_agent(self.h, dp(out))
        return out

    def update_hist(self):
        """the AMP history := the current pose / vel (UpdateHist, what the first update after set_action does)"""
        self.L.dmo_update_hist(self.h)

    def record_amp_obs_expert(self, kin_time, clip=None):
        out = np.zeros(self.amp_obs_size())
        if clip is None:
            self.L.dmo_record_amp_obs_expert(self.h, C.c_double(kin_time), dp(out))
        else:
            self.L.dmo_record_amp_obs_expert_clip(self.h, int(clip), C.c_double(kin_time), dp(out))
        return out

    def reward_terms(self):
        e = np.zeros(5)
        r = self.L.dmo_calc_reward_terms(self.h, dp(e))
        return r, e

    def need_new_action(self):
        return bool(self.L.dmo_need_new_action(self.h))

    def is_episode_end(self):
        return bool(self.L.dmo_is_episode_end(self.h))

    def check_terminate(self):
        return int(self.L.dmo_check_terminate(self.h))

    def check_valid_episode(self):
        return bool(self.L.dmo_check_valid_episode(self.h))

    def has_fallen(self):
        return bool(self.L.dmo_has_fallen(self.h))

    def get_time(self):
        return self.L.dmo_get_time(self.h)

    def get_pose(self):
        p, v = np.zeros(self.pose_dim), np.zeros(self.pose_dim)
        self.L.dmo_get_pose(self.h, dp(p), dp(v))
        return p, v

    def get_kin_pose(self):
        p, v = np.zeros(self.pose_dim), np.zeros(self.pose_dim)
        self.L.dmo_get_kin_pose(self.h, dp(p), dp(v))
        return p, v

    def kin_frame(self, t):
        p, v = np.zeros(self.pose_dim), np.zeros(self.pose_dim)
        self.L.dmo_kin_frame(self.h, C.c_double(t), dp(p), dp(v))
        return p, v

    def set_pose_vel(self, p, v):
        p = np.ascontiguousarray(p, dtype=np.float64); v = np.ascontiguousarray(v, dtype=np.float64)
        self.L.dmo_set_pose_vel(self.h, dp(p), dp(v))

    def body_state(self):
        """World position, rotation (w,x,y,z), linear and angular velocity of every body."""
        n = self.num_joints
        pos, rot, lv, av = np.zeros((n, 3)), np.zeros((n, 4)), np.zeros((n, 3)), np.zeros((n, 3))
        self.L.dmo_body_state(self.h, dp(pos), dp(rot), dp(lv), dp(av))
        return pos, rot, lv, av

    def link_table(self):
        out = np.zeros((self.num_joints, 24))
        self.L.dmo_link_table(self.h, dp(out))
        return out

    def get_snapshot(self):
        s = np.zeros(self.snapshot_size)
        self.L.dmo_get_snapshot(self.h, dp(s))
        return s

    def set_snapshot(self, s):
        s = np.ascontiguousarray(s, dtype=np.float64)
        self.L.dmo_set_snapshot(self.h, dp(s))

    def action_statics(self):
        o, s, lo, hi = (np.zeros(self.action_size) for _ in range(4))
        self.L.dmo_action_statics(self.h, dp(o), dp(s), dp(lo), dp(hi))
        return o, s, lo, hi

    def rbd_mass_bias(self):
        M = np.zeros((self.pose_dim, self.pose_dim)); Cb = np.zeros(self.pose_dim)
        self.L.dmo_rbd_mass_bias(self.h, dp(M), dp(Cb))
        return M, Cb

    def inv_dyna(self, acc):
        acc = np.ascontiguousarray(acc, dtype=np.float64); tau = np.zeros(self.pose_dim)
        self.L.dmo_inv_dyna(self.h, dp(acc), dp(tau))
        return tau

    def spd_tau(self, dt):
        tau = np.zeros(self.pose_dim)
        self.L.dmo_spd_tau(self.h, C.c_double(dt), dp(tau))
        return tau

    def debug_taps(self, sub=0):
        out = np.zeros(2 * self.num_dofs + 64, dtype=np.float32)
        (self.L.dmo_debug_taps if sub == 0 else self.L.dmo_debug_taps1)(self.h, fp(out))
        n = self.num_dofs
        return out[:n], out[n:2 * n], out[2 * n:]

    def last_rows(self, max_substeps=8):
        """branches of the constraint solve per Bullet sub-step of the last update: int array [sub-steps, 7] of (limit rows, contact points,
        clamp in the unconstrained update, clamp after PGS, limit rows at the impulse cap, friction rows skipped in the last sweep,
        limit rows past the split-impulse threshold); solver rows = limit rows + 3 contact points"""
        out = np.zeros((max_substeps, 7), dtype=np.int32)
        n = self.L.dmo_last_rows(self.h, out.ctypes.data_as(C.POINTER(C.c_int)), max_substeps)
        return out[:n].copy()

    def last_contacts(self, max_substeps=8):
        """branches of the link-plane collision per Bullet sub-step of the last update: int array [sub-steps, links, 6] of (event, slot written,
        deepest slot kept out of a full cache or -1, mask of slots removed by distance, mask removed by lateral drift, points after the
        refresh); events 0 none, 1 added to a free slot, 2 replaced the nearest cached point, 3 inserted into a full cache (sortCachedPoints);
        removal masks number the slots as they were when the refresh started"""
        out = np.zeros((max_substeps, self.num_joints, 6), dtype=np.int32)
        n = self.L.dmo_last_contacts(self.h, out.ctypes.data_as(C.POINTER(C.c_int)), max_substeps)
        return out[:n].copy()

    def collider_frames(self):
        """each link's collider frame as of the last set_snapshot: (worldBasis [links, 3, 3], worldPos [links, 3]), scaled units"""
        out = np.zeros((self.num_joints, 12))
        self.L.dmo_collider_frames(self.h, dp(out))
        return out[:, :9].reshape(-1, 3, 3).copy(), out[:, 9:].copy()

    def bullet_aba(self, joint_tau, with_gravity=True):
        jt = np.ascontiguousarray(joint_tau, dtype=np.float32); out = np.zeros(self.num_dofs, dtype=np.float32)
        self.L.dmo_bullet_aba(self.h, fp(jt), 1 if with_gravity else 0, fp(out))
        return out


class PushOracle(Oracle):
    """Oracle with set_push: like the device's push table, a push acts in every update whose timer value at its start t satisfies
    start <= t < start + duration, and a reset clears it (cWorld::Reset clears its perturbations)"""
    _push = None

    def set_push(self, body, force, start, duration):
        """push body `body` (-1: none) with `force` (world axes, unscaled N) at its COM in every update whose timer value at its start t
        satisfies start <= t < start + duration"""
        self._push = None if body < 0 else (int(body), np.ascontiguousarray(force, dtype=np.float64), float(start), float(duration))

    def push_body(self):
        return -1 if self._push is None else self._push[0]

    def reset(self, *a, **k):
        super().reset(*a, **k)
        self._push = None

    def update(self, dt):
        if self._push is None:
            return super().update(dt)
        b, f, s, d = self._push
        self.L.dmo_update_pushed(self.h, C.c_double(dt), b, dp(f), C.c_double(s), C.c_double(d))
