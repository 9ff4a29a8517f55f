"""A Python restatement of the dynamics draw (deepmimic_b200/csrc/kernels/dm_dynamics.cuh: dyn_draw_env) and of the character's part of its
rule, for the CPU shim test and the GPU tests.  Plain IEEE double arithmetic with one rounding per operation, float32 rounding of the stored
factors.  Also the edited asset tree that restates a dynamics factor set in the reference's own files."""
import json
import os
import shutil

import numpy as np

from tests.push_schedule_ref import u01

DYN_SEED_KEY = 0x64796e616d696373   # "dynamics"
KINDS = ("friction", "kp", "kd", "torque_limit", "mass")
FRICTION = 0.9 * 0.9   # link x ground: the oracle's default contact friction


def dyn_seed(handle_seed):
    return handle_seed ^ DYN_SEED_KEY


def lumped_leaves(char_path):
    """[parent or -1 per link]: a fixed joint without children whose parent has degrees of freedom is lumped into the parent's body"""
    joints = json.load(open(char_path))["Skeleton"]["Joints"]
    dof = lambda j: j["Type"].lower() not in ("fixed", "none")
    children = {}
    for j in joints:
        children.setdefault(j["Parent"], []).append(j["ID"])
    out = []
    for j in joints:
        p = j["Parent"]
        out.append(p if j["Type"].lower() == "fixed" and not children.get(j["ID"]) and p >= 0 and dof(joints[p]) else -1)
    return out


def link_masses(char_path):
    return [float(b["Mass"]) if b.get("Shape", "null") != "null" else 0.0 for b in json.load(open(char_path))["BodyDefs"]]


def draw_env(lohi, seed, env, resets, leaf_parent):
    """float32 [4 + links]: friction, kp, kd, torque_limit, mass per link of the episode with reset counter `resets`; seed is the stream's"""
    nl = len(leaf_parent)
    k0 = 64 * resets
    f = np.ones(4 + nl, dtype=np.float32)
    lerp = lambda k, u: lohi[2 * k] + u * (lohi[2 * k + 1] - lohi[2 * k])
    for j in range(4):
        f[j] = np.float32(lerp(j, u01(seed, env, k0 + j)))
    for l in range(nl):
        if leaf_parent[l] < 0:
            f[4 + l] = np.float32(lerp(4, u01(seed, env, k0 + 4 + l)))
    for l in range(nl):
        if leaf_parent[l] >= 0:
            f[4 + l] = f[4 + leaf_parent[l]]
    return f


def total_mass(masses, f):
    """sum of mass * factor in double, link order, stored as float32"""
    m = 0.0
    for l, ml in enumerate(masses):
        m += float(np.float32(ml)) * float(f[4 + l])
    return np.float32(m)


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
