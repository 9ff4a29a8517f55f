"""Constructed simulator states that drive each branch of the step kernel's constraint solve (dm_step.cu: solve_rows, pgs_sweeps and the
velocity clamp around them), built with the CPU oracle from poses and velocities set on purpose plus a few deterministic updates -- no random
rollouts.  Every state carries the class it was built for; Oracle.last_rows() tells which branches one Update(1/600) from it actually takes
(tests/test_solver_states_cpu.py keeps the library honest, tests/test_solver_branches_gpu.py compares the kernel with the oracle on it).

Classes (both characters):
  free        no contact point (lifted off the plane)
  stance      standing / stepping states, binned by the solver rows of the update's second sub-step into the storage buckets of solve_rows:
              none, <= W, <= kSq2, packed (<= maxrows), overflow (> maxrows: the character laid flat and pressed slightly into the plane)
  limit       knees and elbows (dog: forearms and legs) past each side of their limits, shallow (-0.04 < pen <= 0) and deep (pen < -0.04),
              and a limit hit at a high joint rate whose impulse saturates at maxAppliedImpulse = 100
  clamp       joint and base velocities beyond Bullet's maxCoordinateVelocity (100): clamped in the unconstrained update and after PGS
  release     cached contact points whose normal impulse goes to 0 (the link pulled off the plane): friction rows skipped
  explode     link velocities above HasVelExploded's bound"""
import numpy as np

DT = 1.0 / 600.0
CHARS = {
    "humanoid3d": dict(args=["--arg_file", "args/run_humanoid3d_spinkick_args.txt"], char="data/characters/humanoid3d.txt", W=16, sq2=22, maxrows=32),
    "dog3d": dict(args=["--arg_file", "args/train_dog3d_trot_args.txt"], char="data/characters/dog3d.txt", W=32, sq2=36, maxrows=52),
}
BUCKETS = ("none", "square W", "square kSq2", "packed", "overflow")
# Oracle.last_rows() columns
LIMITS, POINTS, CLAMP_ABA, CLAMP_PGS, LIMIT_SAT, FRICTION_SKIP, LIMIT_DEEP = range(7)


def bucket(rows, ch):
    """storage bucket of solve_rows for one environment's solver row count (tools/env_order_stats.py:mode, plus overflow)"""
    c = CHARS[ch]
    if rows == 0:
        return 0
    return 1 if rows <= c["W"] else 2 if rows <= c["sq2"] else 3 if rows <= c["maxrows"] else 4


def joint_layout(asset_root, char_file):
    """per joint: (type, limit low, limit high, pose offset); the root takes pose[0:7] (position, quaternion w x y z)"""
    import json
    import os
    d = json.load(open(os.path.join(asset_root, char_file)))
    out, off = [], 7
    for j in d["Skeleton"]["Joints"][1:]:
        n = {"spherical": 4, "revolute": 1}.get(j["Type"], 0)
        out.append((j["Type"], j.get("LimLow0", 0.0), j.get("LimHigh0", 0.0), off))
        off += n
    return [("none", 0.0, 0.0, 0)] + out


def qmul(a, b):
    aw, ax, ay, az = a; bw, bx, by, bz = b
    return np.array([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw])


def axis_angle(axis, ang):
    axis = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    return np.concatenate([[np.cos(0.5 * ang)], np.sin(0.5 * ang) * axis])


class State:
    def __init__(self, cls, name, snap):
        self.cls, self.name, self.snap = cls, name, snap

    def __repr__(self):
        return "%s/%s" % (self.cls, self.name)


def last_rows(orc, snap):
    """one Update(1/600) of the oracle from snap; returns (Oracle.last_rows() [sub-steps, 7], snapshot after)"""
    orc.set_snapshot(snap)
    orc.update(DT)
    return orc.last_rows(), orc.get_snapshot()


def _start(orc, t, pose=None, vel=None):
    """the clip's pose at time t (reset: standing on the plane, manifolds cleared, zero action), optionally replaced by pose / vel"""
    orc.reset(t, 0.0, 20.0)
    orc.set_action(np.zeros(orc.action_size))
    p, v = orc.get_pose()
    if pose is not None or vel is not None:
        orc.set_pose_vel(p if pose is None else pose, v if vel is None else vel)
    return orc.get_pose()


def _run(orc, n):
    for _ in range(n):
        orc.update(DT)
    return orc.get_snapshot()


def build(orc, asset_root, ch):
    """the state library of character ch (a list of State); deterministic"""
    c = CHARS[ch]
    jl = joint_layout(asset_root, c["char"])
    lim = [j for j, (t, lo, hi, _) in enumerate(jl) if t == "revolute"]   # humanoid: knees and elbows; dog: forearms and legs
    dur = orc.motion_duration
    out = []
    # ---- free: lifted 0.5 m above its standing pose, with the clip's velocities
    for t in (0.0, 0.37, 0.71):
        p, v = _start(orc, t * dur)
        p = p.copy(); p[1] += 0.5
        _start(orc, t * dur, p, v)
        out.append(State("free", "lifted t%.2f" % t, orc.get_snapshot()))
    # ---- stance: the clip's poses on the plane, a few updates so the manifolds fill and warm-start
    for t in np.linspace(0.0, 0.95, 12):
        _start(orc, t * dur)
        done = 0
        for k in (1, 3, 6, 10):
            out.append(State("stance", "clip t%.2f +%d" % (t, k), _run(orc, k - done)))
            done = k
    # ---- stance, heavy: the character in its rest pose (every joint at zero rotation) laid flat on either side, tilted a little so that only
    # part of it touches, pressed slightly into the plane; then a few updates so that the manifolds fill
    for roll in (0.5 * np.pi, -0.5 * np.pi):
        for tilt in (0.0, 0.15, 0.3):
            for press in (0.02, 0.04, 0.06, 0.08, 0.1):
                p, v = _start(orc, 0.0)
                p = p.copy()
                for t, lo, hi, o in jl[1:]:
                    if t == "spherical":
                        p[o:o + 4] = [1.0, 0.0, 0.0, 0.0]
                    elif t == "revolute":
                        p[o] = 0.5 * (lo + hi)
                p[3:7] = qmul(axis_angle([0.0, 0.0, 1.0], tilt), axis_angle([1.0, 0.0, 0.0], roll))
                p[1] = _lying_height(orc, p, v) - press
                _start(orc, 0.0, p, np.zeros_like(v))
                done = 0
                for k in (1, 2, 4):
                    out.append(State("stance", "flat roll %+.2f tilt %.2f press %.2f +%d" % (roll, tilt, press, k), _run(orc, k - done)))
                    done = k
    # ---- limit: each revolute joint past each side, shallow and deep, lifted (no contact) and standing
    for j in lim:
        _, lo, hi, o = jl[j]
        for side, edge, sgn in (("low", lo, -1.0), ("high", hi, 1.0)):
            for depth, pen in (("shallow", 0.02), ("deep", 0.1)):
                for lifted in (True, False):
                    p, v = _start(orc, 0.2 * dur)
                    p = p.copy(); v = v.copy()
                    p[o] = edge + sgn * pen; v[o] = 0.0
                    if lifted:
                        p[1] += 0.5
                    _start(orc, 0.2 * dur, p, v)
                    out.append(State("limit", "joint %d %s %s %s" % (j, side, depth, "lifted" if lifted else "standing"), orc.get_snapshot()))
            # a hit at a high joint rate: at the limit, moving into it at 60 rad/s -- the limit row's impulse saturates at 100
            p, v = _start(orc, 0.2 * dur)
            p = p.copy(); v = v.copy()
            p[o] = edge; v[o] = sgn * 60.0; p[1] += 0.5
            _start(orc, 0.2 * dur, p, v)
            out.append(State("limit", "joint %d %s fast hit" % (j, side), orc.get_snapshot()))
    # ---- clamp: joint rates above 100 rad/s, a base beyond the clamp, in the air and in contact
    for name, lifted in (("lifted", True), ("standing", False)):
        for what in ("joints", "base"):
            p, v = _start(orc, 0.5 * dur)
            p = p.copy(); v = v.copy()
            if lifted:
                p[1] += 0.5
            if what == "joints":
                for j, (t, lo, hi, o) in enumerate(jl):
                    if t == "spherical":
                        v[o:o + 3] = [120.0, -110.0, 105.0]
            else:
                v[0:3] = [30.0, -5.0, 0.0]          # 120 scaled units along x
                v[3:6] = [0.0, 105.0, 0.0]
            _start(orc, 0.5 * dur, p, v)
            out.append(State("clamp", "%s %s" % (what, name), orc.get_snapshot()))
    # clamp after PGS: a fast stance where contacts and limits push clamped coordinates further out
    p, v = _start(orc, 0.0)
    p = p.copy(); v = v.copy()
    for j, (t, lo, hi, o) in enumerate(jl):
        if t == "spherical":
            v[o:o + 3] = [99.9, 99.9, 99.9]
        elif t == "revolute":
            v[o] = 99.9
    v[0:3] = [0.0, -24.9, 0.0]
    _start(orc, 0.0, p, v)
    out.append(State("clamp", "fast stance", orc.get_snapshot()))
    # ---- release: standing with filled manifolds, then the character pulled upward off the plane (points still cached)
    for t in (0.0, 0.5):
        _start(orc, t * dur)
        s = _run(orc, 6)
        s = s.copy(); s[11] += 8.0   # base velocity y: +2 m/s (scaled units)
        out.append(State("release", "pulled up t%.2f" % t, s))
    # ---- explode: base spin and joint rates adding up beyond 100 rad/s in world axes
    p, v = _start(orc, 0.3 * dur)
    p = p.copy(); v = v.copy(); p[1] += 0.5
    v[3:6] = [0.0, 80.0, 0.0]
    for j, (t, lo, hi, o) in enumerate(jl):
        if t == "spherical":
            v[o:o + 3] = [0.0, 80.0, 0.0]
    _start(orc, 0.3 * dur, p, v)
    out.append(State("explode", "spin", orc.get_snapshot()))
    return out


def _lying_height(orc, p, v):
    """root height at which the lowest link of pose p just touches the plane (bisection on the oracle's contact counts)"""
    from tests.parity_util import SnapLayout
    lay = SnapLayout(orc.num_joints)
    lo, hi = -0.5, 1.5
    for _ in range(30):
        mid = 0.5 * (lo + hi)
        q = p.copy(); q[1] = mid
        orc.reset(0.0, 0.0, 20.0)
        orc.set_pose_vel(q, np.zeros_like(v))
        orc.update(DT)   # the collision pass of its first sub-step sees the pose as set
        touching = any(x > 0 for x in lay.contact_counts(orc.get_snapshot()))
        lo, hi = (mid, hi) if touching else (lo, mid)
    return hi
