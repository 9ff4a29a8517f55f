"""Constructed inputs of the policy-rate kernels of dm_policy.cu (dm_observe_kernel: state observation and imitation reward;
dm_reset_kernel), built to reach the branches the shipped argument files never reach.  tests/test_policy_states_cpu.py checks in the oracle
and on the clip files that each input reaches its branch; tests/test_policy_kernels_gpu.py compares the kernels with the oracle on them.

make_assets() copies the committed asset archive and adds:
  - controllers for every combination of phase input and world root rotation, for humanoid3d and dog3d, and a humanoid3d controller with
    RecordWorldRootPos (no shipped argument file uses these layouts);
  - humanoid3d_walk with "Loop": "none": a non-looping clip that ends in motion (the shipped non-looping get-up clips end at rest);
  - a two-clip dataset: get-up face-up (3.77 s, non-looping) and that clip (1.27 s).
Every state is a simulator snapshot of the oracle, deterministic for a given archive."""
import json
import os
import shutil

import numpy as np

from tests.oracle_binding import Oracle
from tests.parity_util import random_policy_action

DT = 1.0 / 600.0
SCALE = 4.0
WALK_ARGS = "args/train_humanoid3d_walk_args.txt"
TROT_ARGS = "args/train_dog3d_trot_args.txt"
HEADING_ARGS = "args/train_amp_heading_humanoid3d_locomotion_args.txt"
GETUP_ARGS = "args/train_amp_heading_getup_humanoid3d_locomotion_getup_args.txt"
WALK = "data/motions/humanoid3d_walk.txt"
WALK_ONCE = "data/motions/humanoid3d_walk_once.txt"
FACEUP = "data/motions/humanoid3d_getup_faceup.txt"
SPINKICK = "data/motions/humanoid3d_spinkick.txt"
BACKFLIP = "data/motions/humanoid3d_backflip.txt"
FACEDOWN = "data/motions/humanoid3d_getup_facedown.txt"
PAIR = "data/datasets/getup_faceup_walk_once.txt"
CHAR_FILE = {"humanoid3d": "data/characters/humanoid3d.txt", "dog3d": "data/characters/dog3d.txt"}
CHAR_ARGS = {"humanoid3d": WALK_ARGS, "dog3d": TROT_ARGS}
SQ_EPS = 1.0 - 1.1920929e-7          # eigen_slerp's near-parallel threshold on |q0 . q1|
DEAD_ZONE = 1e-4                     # cMathUtil::QuatTheta: sin(theta / 2) <= 1e-4 counts as 0


# ---------------------------------------------------------------------------------------------------------------- assets
def ctrl_file(ch, phase, rot, pos=False):
    return "data/controllers/%s_p%d_r%d%s_ctrl.txt" % (ch, phase, rot, "_wpos" if pos else "")


# (character, phase input, world root rotation, world root position)
CTRLS = [(ch, p, r, False) for ch in ("humanoid3d", "dog3d") for p in (0, 1) for r in (0, 1)] + [("humanoid3d", 1, 1, True), ("humanoid3d", 0, 0, True)]


def make_assets(src, dst):
    """a copy of the asset tree src at dst with the constructed controllers, the non-looping walk and the two-clip dataset"""
    shutil.copytree(src, dst)
    for ch, p, r, w in CTRLS:
        with open(os.path.join(src, "data/controllers/%s_ctrl.txt" % ch)) as f:
            d = json.load(f)
        d["EnablePhaseInput"], d["RecordWorldRootRot"], d["RecordWorldRootPos"] = bool(p), bool(r), bool(w)
        with open(os.path.join(dst, ctrl_file(ch, p, r, w)), "w") as f:
            json.dump(d, f, indent=1)
    with open(os.path.join(src, WALK)) as f:
        m = json.load(f)
    m["Loop"] = "none"
    with open(os.path.join(dst, WALK_ONCE), "w") as f:
        json.dump(m, f)
    with open(os.path.join(dst, PAIR), "w") as f:
        json.dump({"Motions": [{"Weight": 1, "File": FACEUP}, {"Weight": 1, "File": WALK_ONCE}]}, f, indent=1)
    return dst


def ctrl_args(ch, phase, rot, pos=False):
    return ["--char_ctrl_files", ctrl_file(ch, phase, rot, pos), "--enable_rand_rot_reset", "true", "--arg_file", CHAR_ARGS[ch]]


def imitate_args(motion, rand_rot=True):
    """the humanoid imitate scene on one clip"""
    return ["--motion_file", motion, "--enable_rand_rot_reset", "true" if rand_rot else "false", "--arg_file", WALK_ARGS]


# the CLIPS scenes (--kin_ctrl clips): heading_amp on the two-clip dataset, heading_amp_getup on the archive's four-clip get-up dataset
# (run and walk loop, the two get-up clips do not); no recovery episodes, so that every reset is a full one
CLIPS_ARGS = {"heading_pair": ["--motion_file", PAIR, "--arg_file", HEADING_ARGS],
              "getup_real": ["--recover_episode_prob", "0", "--arg_file", GETUP_ARGS]}


# ---------------------------------------------------------------------------------------------------------------- clips with numpy
def joint_layout(asset_root, ch="humanoid3d"):
    """[(name, type, pose offset)] of the character, root first"""
    with open(os.path.join(asset_root, CHAR_FILE[ch])) as f:
        joints = json.load(f)["Skeleton"]["Joints"]
    out, off = [("root", "none", 0)], 7
    for j in joints[1:]:
        out.append((j["Name"], j["Type"], off))
        off += {"spherical": 4, "revolute": 1}.get(j["Type"], 0)
    return out


def read_clip(asset_root, motion):
    """(loop, frame times, frames [F, pose_dim] with unit quaternions) of a clip file"""
    with open(os.path.join(asset_root, motion)) as f:
        d = json.load(f)
    fr = np.array(d["Frames"], dtype=np.float64)
    t = np.concatenate([[0.0], np.cumsum(fr[:-1, 0])])
    return d.get("Loop", "wrap") == "wrap", t, fr[:, 1:]


def quat_dots(asset_root, motion, ch="humanoid3d"):
    """{joint name: q_f . q_{f+1} for every frame pair} of the root and the spherical joints (what eigen_slerp branches on)"""
    _, _, fr = read_clip(asset_root, motion)
    out = {}
    for name, typ, off in joint_layout(asset_root, ch):
        o = 3 if name == "root" else off
        if name == "root" or typ == "spherical":
            q = fr[:, o:o + 4] / np.linalg.norm(fr[:, o:o + 4], axis=1, keepdims=True)
            out[name] = (q[:-1] * q[1:]).sum(1)
    return out


def intervals(asset_root, motion, kind):
    """[(t0, t1, joint)]: the frame intervals whose interpolation takes eigen_slerp's antipodal sign flip (kind "antipodal": d < 0) or its
    near-parallel linear blend (kind "held": |d| >= 1 - eps)"""
    _, t, _ = read_clip(asset_root, motion)
    out = []
    for name, d in quat_dots(asset_root, motion).items():
        hit = d < 0 if kind == "antipodal" else np.abs(d) >= SQ_EPS
        out += [(t[i], t[i + 1], name) for i in np.nonzero(hit)[0]]
    return out


def clip_root_y(asset_root, motion, time):
    """the clip's own root height at `time` (frames interpolated linearly, clamped at the ends; a cycle does not move the root up)"""
    loop, t, fr = read_clip(asset_root, motion)
    tt = time - np.floor(time / t[-1]) * t[-1] if loop else min(max(time, 0.0), t[-1])
    return float(np.interp(tt, t, fr[:, 1]))


def _qmat(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def link_bottoms(o, asset_root, ch="humanoid3d"):
    """[(lowest point of the body's world AABB in m, shape, |world y . body y|)] of every body of the oracle's simulated character, from the
    character file's shapes (capsule: radius Param0 / 2 around a segment of length Param1 along the body's y axis)"""
    with open(os.path.join(asset_root, CHAR_FILE[ch])) as f:
        bodies = json.load(f)["BodyDefs"]
    pos, rot, _, _ = o.body_state()
    out = []
    for b, bd in enumerate(bodies):
        ry = np.abs(_qmat(rot[b])[1])
        if bd["Shape"] == "sphere":
            e = bd["Param0"] / 2
        elif bd["Shape"] == "capsule":
            r = bd["Param0"] / 2
            e = ry @ np.array([r, r + bd["Param1"] / 2, r])
        else:
            e = ry @ (np.array([bd["Param0"], bd["Param1"], bd["Param2"]]) / 2)
        out.append((pos[b][1] - e, bd["Shape"], ry[1]))
    return out


def in_intervals(time, iv, dur, loop):
    tt = time - np.floor(time / dur) * dur if loop else time
    return [name for (a, b, name) in iv if a < tt < b]


# ---------------------------------------------------------------------------------------------------------------- states
class State:
    def __init__(self, name, snap, kind):
        self.name, self.snap, self.kind = name, snap, kind


def snapshot_kin_time(s, nl):
    return s[13 + 55 * nl]


def _act(o, rng, sigma=0.25):
    off, scl, lo, hi = o.action_statics()
    o.set_action(random_policy_action(rng, off, scl, lo, hi, sigma=sigma))


def near_kin(o, kt, theta, seed, n=4):
    """the simulated character a few updates after a reset at kt - n DT under one random action, the kinematic clock set back to exactly kt:
    close to the clip at kt with joint errors above the QuatTheta dead zone"""
    o.reset(kt - n * DT, theta, 20.0)
    _act(o, np.random.default_rng(seed))
    for _ in range(n):
        o.update(DT)
    s = o.get_snapshot()
    s[13 + 55 * o.num_joints] = kt
    o.set_snapshot(s)
    return o.get_snapshot()


def airborne(o, kt, theta, seed, lift=2.0):
    """a reset state lifted by `lift` m with random root and joint velocities"""
    o.reset(kt, theta, 20.0)
    p, v = o.get_pose()
    rng = np.random.default_rng(seed)
    p = p.copy(); p[1] += lift
    v = v + rng.standard_normal(v.shape[0])
    o.set_pose_vel(p, v)
    return o.get_snapshot()


def lying(o, seed, kt=0.2, theta=0.0):
    """the character on the ground: 1.5 s of wild random actions, then 0.5 s under the zero action"""
    o.reset(kt, theta, 100.0)
    off, scl, lo, hi = o.action_statics()
    rng = np.random.default_rng(seed)
    for _ in range(900):
        if o.need_new_action():
            o.set_action(random_policy_action(rng, off, scl, lo, hi, sigma=1.0))
        o.update(DT)
    o.set_action(-off)
    for _ in range(300):
        o.update(DT)
    return o.get_snapshot()


def walking(o, kt, theta, seed, updates):
    """`updates` updates under random policy actions after a reset"""
    o.reset(kt, theta, 100.0)
    rng = np.random.default_rng(seed)
    for _ in range(updates):
        if o.need_new_action():
            _act(o, rng)
        o.update(DT)
    return o.get_snapshot()


def observation_states(o):
    """standing (reset), walking, airborne and lying states at several headings"""
    d = o.motion_duration
    st = [State("reset t=%.2f th=%.1f" % (kt, th), None, "stand") for kt, th in ((0.0, 0.0), (0.37 * d, 1.2), (0.81 * d, -2.6))]
    for s, (kt, th) in zip(st, ((0.0, 0.0), (0.37 * d, 1.2), (0.81 * d, -2.6))):
        o.reset(kt, th, 20.0)
        s.snap = o.get_snapshot()
    st += [State("walking %d" % k, walking(o, 0.2 * k * d, 0.9 * k - 2.0, 40 + k, 12 + 17 * k), "walk") for k in range(4)]
    st += [State("airborne %d" % k, airborne(o, 0.3 * k * d, 1.7 * k - 2.5, 60 + k), "airborne") for k in range(3)]
    st += [State("lying %d" % k, lying(o, 80 + k, 0.1 + 0.2 * k, 2.1 * k - 2.0), "lying") for k in range(3)]
    return st


def reward_states(o, times):
    """for every kinematic time: the reset state there (the simulated character on the clip: pose differences in the QuatTheta dead zone)
    and a near-kin state (errors above it).  times: [(label, kin time)]"""
    out = []
    for k, (label, kt) in enumerate(times):
        th = 0.7 * k - 2.0
        o.reset(kt, th, 20.0)
        out.append(State("%s reset" % label, o.get_snapshot(), "on clip"))
        out.append(State("%s near" % label, near_kin(o, kt, th, 200 + k), "near clip"))
    return out


def clip_times(asset_root, motion):
    """the kinematic times of the imitation-reward states of one clip: an antipodal and a held-frame interval where the clip has one;
    cycles 0, 1 and >= 5 of a looping clip; 0, inside, exactly the end and past the end of a non-looping clip"""
    loop, t, _ = read_clip(asset_root, motion)
    dur = t[-1]
    out = []
    for kind in ("antipodal", "held"):
        iv = intervals(asset_root, motion, kind)
        if iv:
            a, b, name = iv[len(iv) // 2]
            out.append(("%s %s" % (kind, name), 0.5 * (a + b)))
    if loop:
        out += [("cycle 0", 0.43 * dur), ("cycle 1", 1.27 * dur), ("cycle 5", 5.61 * dur), ("cycle 9", 9.08 * dur)]
    else:
        out += [("start", 0.0), ("inside", 0.52 * dur), ("end", dur), ("past end", dur + 0.41)]
    return out


def quat_half_sines(o, asset_root, ch="humanoid3d"):
    """{joint: sin(theta / 2)} of the rotation between the oracle's simulated and kinematic pose, for the root and every spherical joint
    (the quantity QuatTheta's dead zone tests)"""
    p, _ = o.get_pose()
    k, _ = o.get_kin_pose()
    out = {}
    for name, typ, off in joint_layout(asset_root, ch):
        if name != "root" and typ != "spherical":
            continue
        o4 = 3 if name == "root" else off
        a, b = p[o4:o4 + 4] / np.linalg.norm(p[o4:o4 + 4]), k[o4:o4 + 4] / np.linalg.norm(k[o4:o4 + 4])
        w = a[0] * b[0] + a[1:] @ b[1:]
        out[name] = float(np.sqrt(max(0.0, 1.0 - w * w)))
    return out
