"""Constructed inputs of the AMP observation kernel (dm_policy.cu: amp_obs_tile behind dm_amp_obs_kernel and dm_amp_expert_sample_kernel) and
of the history it reads (dm_set_action_kernel: UpdateHist; dm_reset_kernel: InitHist), built from the states of tests/policy_states.py to
reach the branches the shipped argument files never reach.  tests/test_amp_states_cpu.py checks in the oracle and on the clip tables that
each input reaches its branch; tests/test_amp_obs_branches_gpu.py compares the kernels with the oracle on them.

  - agent pairs (history = S_prev, now = S_now) for both characters: the now root's heading in every quadrant and at +-pi, its x axis within
    5 degrees of vertical, root and joint quaternions with w < 0, revolute angles stored past +-pi;
  - imitate_amp resets (InitHist): a kin time in [0, 1/30) on a looping clip (history in the previous cycle) and on the non-looping walk
    (history clamped at frame 0), interior times, dur - eps and >= dur, cycles 1 and 5, rot_theta in {0, +-pi, others};
  - expert times per clip: 0, inside (0, 1/30), exactly 1/30, exact frame times (the clip table's own doubles), the first and last frame
    intervals, dur - eps, exactly dur, dur + eps and 1.9 dur;
  - a kinematic origin height per environment, so that the expert's ground height differs between rows.

Tolerances (DESIGN.md section 4).  The kernel's inputs are fp32 (the simulator state, the clip tables) and every output element is the end of
a chain of fp32 operations, each rounding with relative error u = 2^-24: the longest chain is an end effector's, the forward kinematics
(a quaternion product and a rotation, about 32 operations per tree level) after the heading (atan2, sincos) and the clip sample (slerp,
about 64 operations with the heading).  To first order the error of an element is then at most n u S, with n = 32 maxlevel + 64 and S the
magnitude scale of its part: max(1, |largest element of the oracle's pose part|) for the pose part, likewise for the velocity part (the
local-root velocity takes the heading's error times |v|).  humanoid3d (maxlevel 4): n u = 1.1e-5; dog3d (maxlevel 6): 1.5e-5.  The bound of
a part is that, capped at the former fixed bounds (2e-4 pose, 2e-3 velocity).  Where the now root's x axis is within 5 degrees of vertical,
the heading atan2(-x_z, x_x) is ill-conditioned in fp32: such rows get the first-order term of tests/test_policy_kernels_gpu.py, a heading
error of 1e-6 / |x_xz| rad times the part's scale, and are counted."""
import json
import math
import os

import numpy as np

from tests import policy_states as P

U = 2.0 ** -24
QDT = 1.0 / 30.0                         # the controller's query period: the history / expert previous sample lies this far back
COND_MIN = math.sin(math.radians(5.0))
POSE_CAP, VEL_CAP = 2e-4, 2e-3
MINI = ["--motion_file", "data/datasets/test_clips_mini.txt"]   # 4 looping clips of the committed archive
TARGET_ARGS = MINI + ["--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]
HEADING_ARGS = MINI + ["--arg_file", P.HEADING_ARGS]
GETUP_ARGS = P.CLIPS_ARGS["getup_real"]                         # 2 looping clips, 2 non-looping get-ups
TASK_SCENES = {"target": TARGET_ARGS, "heading": HEADING_ARGS, "getup": GETUP_ARGS}
DATASETS = {"mini": TARGET_ARGS, "getup": GETUP_ARGS, "pair": P.CLIPS_ARGS["heading_pair"]}


def amp_args(ch, local_root, motion=None):
    """the imitate_amp scene of one character, --enable_amp_obs_local_root on or off"""
    m = ["--motion_file", motion] if motion else []
    return ["--scene", "imitate_amp", "--enable_amp_obs_local_root", "true" if local_root else "false", "--enable_rand_rot_reset", "true"] + m + [
        "--arg_file", P.CHAR_ARGS[ch]]


# the two configurations the former parity test covered: the humanoid spin kick without local root and the dog trot with it
PARITY = {"spinkick": ["--arg_file", "args/run_humanoid3d_spinkick_args.txt"],
          "dog_local": ["--enable_amp_obs_local_root", "true", "--arg_file", P.TROT_ARGS]}


# ---------------------------------------------------------------------------------------------------------------- tolerances
def max_level(asset_root, ch):
    with open(os.path.join(asset_root, P.CHAR_FILE[ch])) as f:
        joints = json.load(f)["Skeleton"]["Joints"]
    lv = {}
    for j in joints:
        lv[j["ID"]] = 0 if j["Parent"] < 0 else lv[j["Parent"]] + 1
    return max(lv.values())


def split(amp_size, pose_dim):
    """size of one pose block of an AMP observation [pose now | pose prev | vel now | vel prev]"""
    return amp_size // 2 - (6 + pose_dim - 7)


def heading_cond(ref):
    """|horizontal part| of the now root's x axis, from the oracle's own observation (the root tangent; a rotation about y keeps it)"""
    return float(math.hypot(ref[4], ref[6]))


def bound(ref, pose_size, maxlevel):
    """per-element bound of one AMP observation row against the oracle's `ref`, and whether the heading allowance applies"""
    g = (32 * maxlevel + 64) * U
    sp, sv = max(1.0, float(np.abs(ref[:2 * pose_size]).max())), max(1.0, float(np.abs(ref[2 * pose_size:]).max()))
    bp, bv = min(POSE_CAP, g * sp), min(VEL_CAP, g * sv)
    c = heading_cond(ref)
    ill = c < COND_MIN
    if ill:
        bp, bv = bp + 1e-6 / c * sp, bv + 1e-6 / c * sv
    out = np.full(ref.shape[0], bv)
    out[:2 * pose_size] = bp
    return out, ill


def check(g, ref, pose_size, maxlevel, what):
    """asserts one row; returns (pose error, velocity error, pose error / bound, velocity error / bound, ill-conditioned)"""
    b, ill = bound(ref, pose_size, maxlevel)
    err = np.abs(np.asarray(g, dtype=np.float64) - ref)
    assert np.isfinite(g).all(), what
    k = int(np.argmax(err / b))
    assert (err <= b).all(), (what, "element %d of pose size %d" % (k, pose_size), float(err[k]), float(b[k]), float(g[k]), float(ref[k]))
    ep, ev = float(err[:2 * pose_size].max()), float(err[2 * pose_size:].max())
    return ep, ev, ep / b[0], ev / b[-1], ill


def check_split(g, ref, pose_dim, maxlevel, what):
    """check() for callers that hold only the pose dimension"""
    return check(g, ref, split(ref.shape[0], pose_dim), maxlevel, what)


# ---------------------------------------------------------------------------------------------------------------- snapshot edits
def _qmul(a, b):   # w-first
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                     w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def _roty(a):
    return np.array([math.cos(a / 2), 0.0, math.sin(a / 2), 0.0])


def _rotz(a):
    return np.array([math.cos(a / 2), 0.0, 0.0, math.sin(a / 2)])


def heading_of(q):
    """cKinTree::CalcHeading of a w-first root quaternion: atan2(-x_z, x_x) of its x axis"""
    xx = P._qmat(q) @ np.array([1.0, 0.0, 0.0])
    return math.atan2(-xx[2], xx[0])


def with_heading(o, snap, h):
    """the state turned about the world y axis through the origin so that the root's heading is h: root position, rotation and velocities"""
    o.set_snapshot(snap)
    p, v = o.get_pose()
    d = h - heading_of(p[3:7])
    c, s = math.cos(d), math.sin(d)
    rot = lambda x: np.array([c * x[0] + s * x[2], x[1], -s * x[0] + c * x[2]])
    p, v = p.copy(), v.copy()
    p[0:3] = rot(p[0:3])
    p[3:7] = _qmul(_roty(d), p[3:7])
    v[0:3], v[3:6] = rot(v[0:3]), rot(v[3:6])
    o.set_pose_vel(p, v)
    return o.get_snapshot()


def tilted(o, snap, h, elev):
    """the root's rotation replaced by R_y(h) R_z(elev): its x axis at `elev` rad above the horizontal (|x_xz| = cos elev)"""
    o.set_snapshot(snap)
    p, v = o.get_pose()
    p = p.copy()
    p[3:7] = _qmul(_roty(h), _rotz(elev))
    o.set_pose_vel(p, v)
    return o.get_snapshot()


def negated(snap, layout):
    """the same rotations stored as -q: the root (world -> base) and every spherical joint"""
    s = snap.copy()
    s[3:7] = -s[3:7]
    for j, (_, typ, _) in enumerate(layout):
        if typ == "spherical":
            s[13 + 4 * j:17 + 4 * j] = -s[13 + 4 * j:17 + 4 * j]
    return s


def wrapped(snap, layout, k):
    """every revolute angle stored past +-pi: + 2 pi, - 2 pi, or (k = 2) replaced by +-(pi + 0.3) alternately"""
    s = snap.copy()
    rev = [j for j, (_, typ, _) in enumerate(layout) if typ == "revolute"]
    for i, j in enumerate(rev):
        a = s[13 + 4 * j]
        s[13 + 4 * j] = a + 2 * math.pi if k == 0 else (a - 2 * math.pi if k == 1 else (1 if i % 2 == 0 else -1) * (math.pi + 0.3))
    return s


# ---------------------------------------------------------------------------------------------------------------- agent pairs
class Pair:
    def __init__(self, name, prev, now, kind):
        self.name, self.prev, self.now, self.kind = name, prev, now, kind


QUADRANT_HEADINGS = [0.7, 2.3, -2.2, -0.8, math.pi, -math.pi]


def agent_pairs(o, asset_root, ch):
    """(history, now) pairs of one character: a pool of near-clip, walking, airborne and lying states paired with their neighbours, then
    the pool turned to headings in every quadrant and at +-pi, tilted to within 5 degrees of vertical, stored with w < 0 and with revolute
    angles past +-pi"""
    d = o.motion_duration
    lay = P.joint_layout(asset_root, ch)
    pool = [P.near_kin(o, 0.31 * d, 0.4, 11), P.near_kin(o, 0.77 * d, -1.9, 12), P.walking(o, 0.1 * d, 1.3, 13, 40), P.walking(o, 0.6 * d, -2.8, 14, 75),
            P.airborne(o, 0.2 * d, 2.6, 15), P.airborne(o, 0.5 * d, -0.6, 16), P.lying(o, 17, 0.2, 1.0), P.lying(o, 18, 0.4, -2.0)]
    K = len(pool)
    out = [Pair("pool %d" % k, pool[k], pool[(k + 1) % K], "plain") for k in range(K)]
    for i, h in enumerate(QUADRANT_HEADINGS):
        k = i % K
        out.append(Pair("heading %.4f" % h, pool[(k + 3) % K], with_heading(o, pool[k], h), "heading"))
    for i, (h, deg) in enumerate([(0.5, 87.0), (-2.0, 88.5), (2.9, -86.5), (-0.3, -89.0)]):
        out.append(Pair("tilt %.1f deg" % deg, pool[(i + 2) % K], tilted(o, pool[i % K], h, math.radians(deg)), "tilt"))
    for k in range(0, K, 2):
        out.append(Pair("w < 0 %d" % k, negated(pool[k], lay), negated(pool[(k + 1) % K], lay), "negated"))
    for k in range(3):
        out.append(Pair("revolute wrap %d" % k, wrapped(pool[k], lay, k), wrapped(pool[k + 4], lay, (k + 1) % 3), "wrapped"))
    return out


# ---------------------------------------------------------------------------------------------------------------- InitHist resets
def reset_cases(motion, dur):
    """(label, kin time, rot_theta) of the imitate_amp resets: looping clips at [0, 1/30), inside and cycles 1 and 5; the non-looping walk
    at [0, 1/30), inside, dur - eps, dur and past dur so that the history sample itself lies past the end"""
    if motion == P.WALK_ONCE:
        times = [("t=0", 0.0), ("t<1/30 a", 0.011), ("t<1/30 b", 0.029), ("inside", 0.52 * dur), ("dur-eps", dur - 1e-6), ("dur", dur),
                 ("history inside, kin past end", dur + 0.02), ("history past end", dur + 0.2)]
    else:
        times = [("t=0", 0.0), ("t<1/30 a", 0.011), ("t<1/30 b", 0.029), ("inside", 0.43 * dur), ("cycle 1", 1.31 * dur), ("cycle 5", 5.42 * dur)]
    thetas = [0.0, math.pi, -math.pi, 1.1, -2.4]
    return [(lb, kt, thetas[i % len(thetas)]) for i, (lb, kt) in enumerate(times)] + [(lb + " th", kt, thetas[(i + 2) % len(thetas)])
                                                                                       for i, (lb, kt) in enumerate(times)]


# ---------------------------------------------------------------------------------------------------------------- expert times
def motion_file(asset_root, args):
    """the --motion_file of an argument list (or of its --arg_file)"""
    if "--motion_file" in args:
        return args[args.index("--motion_file") + 1]
    with open(os.path.join(asset_root, args[args.index("--arg_file") + 1])) as f:
        tok = f.read().split()
    return tok[tok.index("--motion_file") + 1]


def dataset_clips(asset_root, args):
    """the clip files of a --kin_ctrl clips scene's dataset, in the dataset's order"""
    with open(os.path.join(asset_root, motion_file(asset_root, args))) as f:
        return [m["File"] for m in json.load(f)["Motions"]]


def expert_times(asset_root, motion):
    """(label, time) of the expert samples of one clip; the frame times are the clip table's own doubles (the loader's running sum)"""
    _, t, _ = P.read_clip(asset_root, motion)
    dur, F = t[-1], len(t)
    return [("0", 0.0), ("in (0, 1/30)", 0.37 * QDT), ("1/30", QDT), ("frame 1", t[1]), ("frame mid", t[F // 2]), ("frame F-2", t[F - 2]),
            ("first interval", 0.5 * (t[0] + t[1])), ("last interval", 0.5 * (t[F - 2] + t[F - 1])), ("dur-eps", dur - 1e-6), ("dur", dur),
            ("dur+eps", dur + 1e-6), ("1.9 dur", 1.9 * dur)]


def origin_heights(n):
    """a distinct kinematic-origin height per environment (the expert's ground height)"""
    return 0.037 * np.arange(n) - 0.4


def acting(snap, nl):
    """the state with the controller's need-new-action flag set: the oracle's next update stores the history (UpdateHist), as the device's
    set_action does"""
    s = snap.copy()
    s[13 + 55 * nl + 11] = 1.0
    return s


def with_origin_y(snap, nl, y):
    s = snap.copy()
    s[13 + 55 * nl + 2] = y
    return s
