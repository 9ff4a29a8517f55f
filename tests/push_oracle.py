"""The CPU oracle with a timed push (tests/push_oracle.cpp: oracle/dm_oracle.cpp plus dmo_push_update), built with g++ into a temporary
directory on first use.  PushOracle is tests.oracle_binding.Oracle with set_push: like the device's push table, a push acts in every update
whose timer value at its start t satisfies start <= t < start + duration, and a reset clears it (cWorld::Reset clears its perturbations)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tests.oracle_binding import Oracle, dp

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
_LIB = None


def load_push_oracle():
    global _LIB
    if _LIB is not None:
        return _LIB
    src = os.path.join(HERE, "push_oracle.cpp")
    deps = [src] + [os.path.join(REPO, "oracle", f) for f in ("dm_oracle.cpp", "bullet_mb.hpp", "rbd.hpp", "omath.hpp")]
    key = hashlib.sha1(b"".join(open(f, "rb").read() for f in deps)).hexdigest()[:16]
    so = os.path.join(tempfile.gettempdir(), "dm_push_oracle_%d_%s.so" % (os.getuid(), key))
    if not os.path.exists(so):
        tmp = "%s.%d.tmp" % (so, os.getpid())
        subprocess.check_call(["g++", "-O3", "-std=c++17", "-fPIC", "-shared", src, "-o", tmp])
        os.replace(tmp, so)
    L = C.CDLL(so)
    L.dmo_create.restype = C.c_void_p
    L.dmo_create.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_char_p)]
    L.dmo_last_error.restype = C.c_char_p
    for f in ("dmo_calc_reward", "dmo_calc_reward_imitate", "dmo_motion_duration", "dmo_get_time", "dmo_calc_reward_terms", "dmo_u01"):
        getattr(L, f).restype = C.c_double
    L.dmo_u01.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64]
    L.dmo_set_task_stream.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64]
    L.dmo_task_counter.restype = C.c_uint64
    L.dmo_task_counter.argtypes = [C.c_void_p]
    L.dmo_push_update.argtypes = [C.c_void_p, C.c_double, C.c_int, C.POINTER(C.c_double), C.c_double, C.c_double]
    _LIB = L
    return L


class PushOracle(Oracle):
    def __init__(self, args, asset_root):
        L = load_push_oracle()
        enc = [a.encode() for a in args]
        h = L.dmo_create(asset_root.encode(), len(enc), (C.c_char_p * len(enc))(*enc))
        if not h:
            raise RuntimeError("oracle create failed: %s" % L.dmo_last_error().decode())
        self.L, self.h = L, C.c_void_p(h)
        d = (C.c_int * 8)()
        L.dmo_get_dims(self.h, d)
        (self.num_joints, self.pose_dim, self.num_dofs, self.state_size, self.action_size, self.goal_size, self.snapshot_size, self.num_frames) = list(d)
        self.motion_duration = L.dmo_motion_duration(self.h)
        self._push = None

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
        self.L.dmo_push_update(self.h, C.c_double(dt), b, dp(f), C.c_double(s), C.c_double(d))
