"""The CPU oracle with a settable contact friction coefficient (tests/dynamics_oracle.cpp: oracle/dm_oracle.cpp plus dmo_set_friction), built
with g++ into a temporary directory on first use, and the edited asset tree that restates a dynamics factor set in the reference's own files."""
import ctypes as C
import hashlib
import json
import os
import shutil
import subprocess
import tempfile

from tests.oracle_binding import Oracle

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
FRICTION = 0.9 * 0.9   # link x ground (oracle/dm_oracle.cpp)
_LIB = None


def load_dynamics_oracle():
    global _LIB
    if _LIB is not None:
        return _LIB
    src = os.path.join(HERE, "dynamics_oracle.cpp")
    deps = [src] + [os.path.join(REPO, "oracle", f) for f in ("dm_oracle.cpp", "bullet_mb.hpp", "rbd.hpp", "omath.hpp")]
    key = hashlib.sha1(b"".join(open(f, "rb").read() for f in deps)).hexdigest()[:16]
    so = os.path.join(tempfile.gettempdir(), "dm_dynamics_oracle_%d_%s.so" % (os.getuid(), key))
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
    L.dmo_set_friction.argtypes = [C.c_void_p, C.c_double]
    _LIB = L
    return L


class DynamicsOracle(Oracle):
    """tests.oracle_binding.Oracle on this library, with set_friction(factor): the coefficient becomes 0.81 x factor"""

    def __init__(self, args, asset_root):
        L = load_dynamics_oracle()
        enc = [a.encode() for a in args]
        h = L.dmo_create(asset_root.encode(), len(enc), (C.c_char_p * len(enc))(*enc))
        if not h:
            raise RuntimeError("oracle create failed: %s" % L.dmo_last_error().decode())
        self.L, self.h = L, C.c_void_p(h)
        d = (C.c_int * 8)()
        L.dmo_get_dims(self.h, d)
        (self.num_joints, self.pose_dim, self.num_dofs, self.state_size, self.action_size, self.goal_size, self.snapshot_size, self.num_frames) = list(d)
        self.motion_duration = L.dmo_motion_duration(self.h)

    def set_friction(self, factor):
        self.L.dmo_set_friction(self.h, C.c_double(FRICTION * float(factor)))


def edited_asset_tree(src_root, dst, char_file, ctrl_file, kp, kd, torque_limit, mass):
    """a copy of the asset tree at dst with the character's Mass (times mass[link]) and TorqueLim (times torque_limit) and the controller's
    Kp and Kd (times kp, kd) edited: the reference built from these files is the model the factors stand for"""
    shutil.copytree(src_root, dst, copy_function=shutil.copyfile)   # the files without their modes: the tree may be read-only
    cp = os.path.join(dst, char_file)
    c = json.load(open(cp))
    for b in c["BodyDefs"]:
        b["Mass"] = float(b["Mass"]) * float(mass[b["ID"]])
    for j in c["Skeleton"]["Joints"]:
        if "TorqueLim" in j:
            j["TorqueLim"] = float(j["TorqueLim"]) * float(torque_limit)
    json.dump(c, open(cp, "w"), indent=1)
    kp_ = os.path.join(dst, ctrl_file)
    k = json.load(open(kp_))
    for p in k["PDControllers"]:
        p["Kp"] = float(p["Kp"]) * float(kp)
        p["Kd"] = float(p["Kd"]) * float(kd)
    json.dump(k, open(kp_, "w"), indent=1)
    return dst
