"""Constructed characters of the shapes the loader accepts but neither shipped character has (capi.cu: build_device_model, plan_launch), each
written into an asset root of its own, and a library of constructed states per character that drive the step kernel's Stable-PD stage,
articulated-body solve and position integration (dm_step.cu: the PD block of the main loop, aba_solve_body and its dynamics-tree table,
quat_rotvec3, normalize_angle3, quat_integrate3) into each of their branches.  Every state is built with the CPU oracle from poses, velocities
and PD targets set on purpose; tests/test_char_shapes_cpu.py keeps the library honest, tests/test_pd_aba_branches_gpu.py compares the kernel
with the oracle on it.

Characters (every body shape on every joint kind somewhere):
  c16   16 links, W = 16 with every lane of both halves live: a revolute child of the root, an unlimited revolute joint and one whose limits take
        the reference's has_limit rule the other way, joints without TorqueLim, fixed leaves lumped into a revolute and a spherical parent
  c17   17 links (W = 32, 15 idle lanes), boxes and spheres only, one Bullet sub-step per update
  c32   32 links (no idle lane): fixed links with children, fixed leaves under the root and under a fixed link (not lumped), a non-root link with
        4 children, revolute and fixed children of the root, leaves lumped into spherical parents; three Bullet sub-steps per update
  c96   31 links, 96 dofs, a spherical chain of last depth 23

State classes (every character; the shipped ones have no unlimited revolute joint, so no rev_wrap):
  free         airborne clip poses with the clip's velocities and the pose as PD target: no contact point, no limit row
  clamp        PD errors of 2.5 rad (spherical) and 3 rad (revolute) that put torque norms above the TorqueLim, and of 0.05 rad below it
  sph_err      spherical PD targets equal to the pose advanced by dt (the dead zone of quat_rotvec3), and errors of 3.8 rad (w < 0: past pi)
  rev_wrap     unlimited revolute joints at +-3.6 and +-7.0 rad, their PD error through normalize_angle3
  root_quirk   a tilted root spinning at 16 rad/s and translating: the Stable-PD stage's root bias term (aba_solve_body, bullet == 0).  The
               term is a linear acceleration of the base origin, which every link inherits unchanged, like gravity: the joint accelerations and
               so the Stable-PD torques do not depend on it, and these states can only show that the stage runs on them
  integ        every rate below 1e-3 rad/s (the small-angle series of quat_integrate3), and every rate above it
  integ_clamp  a dt = 1/60 update (1/40 with three sub-steps) with base and joint rates of 171 rad/s: |w| h past pi / 4 (the fAngle clamp)
  substeps     c17 and c32: airborne clip poses, one and three Bullet sub-steps per update"""
import json
import os

import numpy as np

from tests.solver_states import State, axis_angle, qmul

DT = 1.0 / 600.0


CLASSES = ("free", "clamp", "sph_err", "rev_wrap", "root_quirk", "integ", "integ_clamp", "substeps")
# floors of the GPU comparison's bounds on these airborne states: q-dot (rad/s, m/s) per character, and q.  Each q-dot floor is twice the
# largest error measured on an H100 among the character's updates whose 8 x envelope is below 3e-4, rounded up (the measurement is recorded
# in tests/test_pd_aba_branches_gpu.py)
QD_FLOOR = {"c16": 6e-5, "c17": 3e-5, "c32": 6e-5, "c96": 2e-4, "humanoid3d": 2e-4, "dog3d": 3e-4}
Q_FLOOR = 1e-5


def dt_clamp(substeps):
    """the update of the integ_clamp states: 1/60, 1/40 with three sub-steps (h = 1/120: rates of 171 rad/s reach 1.1 x pi / 4 after the update)"""
    return 1.0 / 40.0 if substeps == 3 else 1.0 / 60.0


def envelope(orc2, lay, jt, before, after, dt, rng, replicas=16):
    """worst |dq|, |dqd| of the oracle's own update from `before` under fp32-rounding noise (tools/qd_envelope.py's protocol, any dt)"""
    from tests.parity_util import compare_sim_state
    from tools.qd_envelope import perturb
    wq = wqd = 0.0
    for _ in range(replicas):
        orc2.set_snapshot(perturb(lay, before, rng))
        orc2.update(dt)
        eq, eqd = compare_sim_state(lay, after, orc2.get_snapshot(), jt)
        wq, wqd = max(wq, eq), max(wqd, eqd)
    return wq, wqd


def bounds(name, env):
    """(q, q-dot) bound of the GPU comparison of an update of character `name` whose oracle envelope is env = (|dq|, |dqd|)"""
    return max(Q_FLOOR, 8.0 * env[0]), max(QD_FLOOR[name], 8.0 * env[1])
SHAPES = ("box", "capsule", "sphere")
SHIPPED = {"humanoid3d": (["--arg_file", "args/run_humanoid3d_spinkick_args.txt"], "data/characters/humanoid3d.txt"),
           "dog3d": (["--arg_file", "args/train_dog3d_trot_args.txt"], "data/characters/dog3d.txt")}


# ---- character specs: per joint (type, parent, shape, options); the root is joint 0 (type none, a sphere)
def _c16():
    return [("none", -1, "sphere", {}),
            ("revolute", 0, "box", {}), ("spherical", 1, "capsule", {}), ("spherical", 2, "sphere", {"tlim": None}),
            ("spherical", 0, "box", {}), ("revolute", 4, "capsule", {"lim": (0.2, 2.0), "tlim": None}), ("revolute", 4, "sphere", {"lim": (-1.0, -0.5)}),
            ("fixed", 6, "box", {}),
            ("spherical", 0, "capsule", {}), ("spherical", 8, "box", {}), ("revolute", 9, "sphere", {}), ("fixed", 9, "capsule", {}),
            ("spherical", 0, "sphere", {}), ("revolute", 12, "box", {}), ("spherical", 13, "capsule", {}), ("revolute", 14, "sphere", {})]


def _c17():
    bs = lambda i: ("box", "sphere")[i % 2]
    return [("none", -1, "sphere", {}),
            ("spherical", 0, bs(0), {}), ("revolute", 1, bs(1), {}), ("spherical", 2, bs(2), {}), ("revolute", 3, bs(3), {}),
            ("spherical", 0, bs(1), {}), ("spherical", 5, bs(2), {}), ("revolute", 6, bs(3), {}), ("fixed", 7, bs(4), {}),
            ("spherical", 0, bs(2), {}), ("revolute", 9, bs(3), {"lim": (0.3, 1.5), "tlim": None}), ("spherical", 10, bs(4), {}), ("revolute", 11, bs(5), {}),
            ("spherical", 0, bs(3), {}), ("spherical", 13, bs(4), {}), ("revolute", 14, bs(5), {}), ("spherical", 15, bs(6), {})]


def _c32():
    return [("none", -1, "sphere", {}),
            ("fixed", 0, "box", {}), ("spherical", 1, "capsule", {}), ("revolute", 2, "sphere", {}), ("fixed", 1, "sphere", {}),   # 1..4
            ("fixed", 0, "capsule", {}),                                                                                          # 5
            ("revolute", 0, "capsule", {}), ("spherical", 6, "box", {}),                                                          # 6, 7
            ("spherical", 7, "sphere", {}), ("revolute", 7, "box", {}), ("fixed", 7, "capsule", {}), ("spherical", 7, "capsule", {}),   # 8..11
            ("revolute", 8, "box", {}), ("spherical", 11, "sphere", {}), ("fixed", 13, "box", {}),                               # 12..14
            ("spherical", 0, "sphere", {}), ("spherical", 15, "box", {}), ("revolute", 16, "capsule", {}), ("spherical", 16, "sphere", {}),   # 15..18
            ("fixed", 16, "box", {}), ("spherical", 19, "capsule", {}), ("revolute", 20, "sphere", {"lim": (0.5, 2.5), "tlim": None}),   # 19..21
            ("spherical", 18, "box", {}), ("revolute", 22, "capsule", {}), ("spherical", 22, "sphere", {}), ("revolute", 24, "box", {}),   # 22..25
            ("fixed", 24, "sphere", {}), ("spherical", 17, "capsule", {}), ("revolute", 27, "box", {}), ("fixed", 28, "capsule", {}),   # 26..29
            ("spherical", 21, "box", {}), ("revolute", 30, "sphere", {})]                                                        # 30, 31


def _c96():
    out = [("none", -1, "sphere", {})]
    for k in range(6):   # the deepest chain: 6 spherical joints, last depth 5 + 18 = 23
        out.append(("spherical", len(out) - 1 if k else 0, SHAPES[k % 3], {}))
    for s in range(3):   # three subtrees of 8 spherical joints: a - b; b - c, d, e, f; c - g; d - h
        a = len(out)
        par = [0, a, a + 1, a + 1, a + 1, a + 1, a + 2, a + 3]
        for k, p in enumerate(par):
            out.append(("spherical", p, SHAPES[(s + k) % 3], {}))
    return out


CHARS = {"c16": (_c16, 2), "c17": (_c17, 1), "c32": (_c32, 3), "c96": (_c96, 2)}


def _offsets(spec, j):
    """joint attach point in the parent's joint frame: children of one parent spread around it"""
    p = spec[j][1]
    k = [i for i in range(len(spec)) if spec[i][1] == p].index(j)
    if p == 0:
        return [(0.0, 0.2, 0.0), (0.15, -0.1, 0.05), (-0.15, -0.1, -0.05), (0.0, -0.12, 0.15)][k % 4]
    return [(0.0, -0.22, 0.0), (0.1, -0.18, 0.06), (-0.1, -0.18, -0.06), (0.02, -0.16, 0.12)][k % 4]


def char_json(spec):
    joints, bodies = [], []
    for j, (t, p, shape, o) in enumerate(spec):
        a = _offsets(spec, j) if p >= 0 else (0.0, 0.0, 0.0)
        jd = {"ID": j, "Name": "j%d" % j, "Type": t, "Parent": p, "AttachX": a[0], "AttachY": a[1], "AttachZ": a[2],
              "AttachThetaX": 0.0 if p < 0 else 0.07 * ((j % 5) - 2), "AttachThetaY": 0.0 if p < 0 else 0.05 * ((j % 3) - 1), "AttachThetaZ": 0.0,
              "IsEndEffector": int(p >= 0 and not any(q[1] == j for q in spec)), "DiffWeight": 1.0 if p >= 0 else 0.0}
        if t == "revolute":
            lo, hi = o.get("lim", (-2.5, 0.5))
            jd.update(LimLow0=lo, LimHigh0=hi)
        elif t == "spherical":
            jd.update(LimLow0=-1.5, LimHigh0=1.5, LimLow1=-1.5, LimHigh1=1.5, LimLow2=-1.5, LimHigh2=1.5)
        if p >= 0 and o.get("tlim", 0) is not None and t != "fixed":
            jd["TorqueLim"] = 150.0 if t == "spherical" else 100.0
        joints.append(jd)
        size = {"box": (0.1, 0.16, 0.08), "capsule": (0.08, 0.1, 0.0), "sphere": (0.12, 0.12, 0.12)}[shape]
        mass = {"box": 3.0, "capsule": 2.0, "sphere": 2.5}[shape] if p >= 0 else 6.0
        bodies.append({"ID": j, "Name": "j%d" % j, "Shape": shape, "Mass": mass, "ColGroup": 1, "EnableFallContact": 1,
                       "AttachX": 0.0, "AttachY": 0.0 if p < 0 else -0.08, "AttachZ": 0.0, "AttachThetaX": 0.0, "AttachThetaY": 0.0, "AttachThetaZ": 0.0,
                       "Param0": size[0], "Param1": size[1], "Param2": size[2], "ColorR": 0.5, "ColorG": 0.5, "ColorB": 0.5, "ColorA": 1})
    return {"Skeleton": {"Joints": joints}, "BodyDefs": bodies}


def ctrl_json(spec):
    pd = []
    for j, (t, p, _, o) in enumerate(spec):
        soft = p >= 0 and o.get("tlim", 0) is None   # joints without a torque limit get small gains: their torques stay moderate
        kp, kd = (0.0, 0.0) if p < 0 or t == "fixed" else (60.0, 6.0) if soft else (400.0, 40.0) if t == "spherical" else (300.0, 30.0)
        pd.append({"ID": j, "Name": "j%d" % j, "Kp": kp, "Kd": kd, "TargetTheta0": 0, "UseWorldCoord": 0})
    return {"UpdateRate": 30, "EnablePhaseInput": True, "RecordWorldRootPos": False, "RecordWorldRootRot": True, "PDControllers": pd}


def motion_json(spec, frames=4):
    out = []
    for f in range(frames):
        row = [0.2, 0.1 * f, 1.2, 0.05 * f] + list(axis_angle([0.0, 1.0, 0.0], 0.1 * f))
        for j, (t, p, _, o) in enumerate(spec[1:], 1):
            if t == "spherical":
                row += list(axis_angle([np.sin(j), np.cos(j), 0.5], 0.15 + 0.1 * np.sin(j + f)))
            elif t == "revolute":
                lo, hi = o.get("lim", (-2.5, 0.5))
                mid = 0.5 * (lo + hi) if lo <= 0.0 else 0.0   # joints with a limit sit inside it; unlimited ones anywhere
                row.append(mid + 0.1 * np.sin(j + f))
            elif t == "planar":
                row += [0.0, 0.0, 0.0]
        out.append([float(x) for x in row])
    return {"Loop": "wrap", "Frames": out}


ARGS = """--scene imitate
--num_update_substeps 10
--num_sim_substeps %d
--world_scale 4
--terrain_file data/terrain/plane.txt
--char_types general
--character_files data/characters/%s.txt
--enable_char_soft_contact false
--fall_contact_bodies 0
--char_ctrls ct_pd
--char_ctrl_files data/controllers/%s_ctrl.txt
--kin_ctrl motion
--motion_file data/motions/%s.txt
--sync_char_root_pos true
--sync_char_root_rot false
"""


def specs(names=None):
    """{name: (spec, sub-steps)} of the constructed characters (all, or those named)"""
    return {n: (CHARS[n][0](), CHARS[n][1]) for n in (names or CHARS)}


def write_root(asset_root, dst, chars=None, edit=None):
    """an asset root at dst holding the characters of chars, a {name: (spec, sub-steps)} mapping (default: every constructed character):
    character, controller, motion and arg files, the shipped terrain linked in.  edit(name, char_json, ctrl_json) may change the JSON before
    it is written.  Returns dst."""
    for sub in ("characters", "controllers", "motions"):
        os.makedirs(os.path.join(dst, "data", sub), exist_ok=True)
    os.makedirs(os.path.join(dst, "args"), exist_ok=True)
    if not os.path.exists(os.path.join(dst, "data", "terrain")):
        os.symlink(os.path.join(asset_root, "data", "terrain"), os.path.join(dst, "data", "terrain"))
    for name, (spec, sub) in (specs() if chars is None else chars).items():
        c, k = char_json(spec), ctrl_json(spec)
        if edit is not None:
            edit(name, c, k)
        for path, text in ((("data", "characters", name + ".txt"), json.dumps(c, indent=1)), (("data", "controllers", name + "_ctrl.txt"), json.dumps(k, indent=1)),
                           (("data", "motions", name + ".txt"), json.dumps(motion_json(spec))), (("args", name + "_args.txt"), ARGS % (sub, name, name, name))):
            with open(os.path.join(dst, *path), "w") as f:
                f.write(text)
    return dst


def args_of(name):
    return SHIPPED[name][0] if name in SHIPPED else ["--arg_file", "args/%s_args.txt" % name]


def char_file(name):
    return SHIPPED[name][1] if name in SHIPPED else "data/characters/%s.txt" % name


# ---- the dynamics tree of the articulated-body passes, restated from the table build (dm_step.cu, dm_step_body)
def dyn_tree(joints):
    """joints: the character file's Skeleton.Joints.  Per link: dict(lumped, level, parent, byp, children) with level -1 for the root, 100 for
    a lumped leaf and the kinematic level - 1 otherwise; byp the root when the link hangs off it, else None; children the non-lumped ones"""
    n = len(joints)
    par = [j["Parent"] for j in joints]
    ndof = [0 if i == 0 else {"spherical": 3, "revolute": 1}.get(j["Type"], 0) for i, j in enumerate(joints)]
    kids = [[c for c in range(n) if par[c] == i] for i in range(n)]
    lumped = [ndof[i] == 0 and not kids[i] and par[i] >= 0 and ndof[par[i]] > 0 for i in range(n)]
    level = [0] * n
    for i in range(1, n):
        level[i] = level[par[i]] + 1
    out = []
    for i in range(n):
        out.append(dict(lumped=lumped[i], level=-1 if i == 0 else 100 if lumped[i] else level[i] - 1, parent=max(par[i], 0),
                        byp=par[i] if i > 0 and par[i] == 0 else None, children=[c for c in kids[i] if not lumped[c]], ndof=ndof[i],
                        kin_level=level[i]))
    return out


def last_depths(joints):
    """the deepest dof depth on the chain base -> link (capi.cu: last_depth; the base's six dofs take depths 0..5)"""
    d = []
    for i, j in enumerate(joints):
        nd = 0 if i == 0 else {"spherical": 3, "revolute": 1}.get(j["Type"], 0)
        d.append((5 if i == 0 else d[j["Parent"]]) + nd)
    return d


def has_limit(j):
    """capi.cu's rule, taken from the reference (SimCharacter.cpp:958): revolute and LimLow0 <= LimHigh1 (LimHigh1 defaults to 0)"""
    return j["Type"] == "revolute" and j.get("LimLow0", 1.0) <= j.get("LimHigh1", 0.0)


# ---- state library
def joint_layout(joints):
    """per joint: (type, pose offset, dof offset in the velocity vector, has_limit, torque limit or inf)"""
    out, off = [], 7
    for i, j in enumerate(joints):
        t = j["Type"] if i else "none"
        out.append((t, 0 if i == 0 else off, has_limit(j), float(j.get("TorqueLim", np.inf))))
        if i:
            off += {"spherical": 4, "revolute": 1}.get(t, 0)
    return out


def _tgt(orc):
    return 29 + 55 * orc.num_joints


def _set_targets(orc, snap, jl, p):
    """PD targets of the snapshot = the pose p (spherical (w, x, y, z), revolute angle)"""
    s = snap.copy()
    for j, (t, o, _, _) in enumerate(jl):
        if t == "spherical":
            s[_tgt(orc) + 4 * j: _tgt(orc) + 4 * j + 4] = p[o:o + 4]
        elif t == "revolute":
            s[_tgt(orc) + 4 * j] = p[o]
    return s


def _lifted(orc, t, vel=None, base_rot=None, base_w=None, base_v=None):
    """the clip's pose at time t lifted 2 m off the plane; vel replaces the clip's velocities; returns (snapshot with the pose as PD target, p, v)"""
    orc.reset(t, 0.0, 20.0)
    orc.set_action(np.zeros(orc.action_size))
    p, v = orc.get_pose()
    p = p.copy(); p[1] += 2.0
    v = v.copy() if vel is None else vel.copy()
    if base_rot is not None:
        p[3:7] = qmul(base_rot, p[3:7])
    if base_w is not None:
        v[3:6] = base_w
    if base_v is not None:
        v[0:3] = base_v
    orc.set_pose_vel(p, v)
    p, v = orc.get_pose()
    return orc.get_snapshot(), p, v


def _pose_inc(q, w, dt):
    """cKinTree::VelToPoseDiff: normalize(q + dt 0.5 q (x) (0, w)), (w, x, y, z)"""
    qi = q + 0.5 * dt * qmul(q, np.concatenate([[0.0], w]))
    return qi / np.linalg.norm(qi)


def build(orc, joints, name, substeps):
    """the state library of one character (a list of State, each with .dt); deterministic"""
    jl = joint_layout(joints)
    dur = orc.motion_duration
    sph = [j for j, x in enumerate(jl) if x[0] == "spherical"]
    rev = [j for j, x in enumerate(jl) if x[0] == "revolute"]
    out = []

    def add(cls, nm, snap, dt=DT):
        st = State(cls, nm, snap)
        st.dt = dt
        out.append(st)

    zero = np.zeros(orc.pose_dim)
    # ---- free
    for t in (0.0, 0.37, 0.71):
        s, p, _ = _lifted(orc, t * dur)
        add("free", "lifted t%.2f" % t, _set_targets(orc, s, jl, p))
    # ---- clamp: every joint with a torque limit driven far from (above) or close to (below) its target, at rest
    for side, ang_s, ang_r in (("above", 2.5, 3.0), ("below", 0.05, 0.05)):
        s, p, _ = _lifted(orc, 0.2 * dur, vel=zero)
        tg = p.copy()
        ax = np.array([1.0, 0.8, 0.6]) / np.linalg.norm([1.0, 0.8, 0.6])
        for j in sph:
            tg[jl[j][1]:jl[j][1] + 4] = qmul(p[jl[j][1]:jl[j][1] + 4], axis_angle(ax, ang_s))
        for j in rev:
            tg[jl[j][1]] = p[jl[j][1]] + ang_r
        add("clamp", "torque %s the limit" % side, _set_targets(orc, s, jl, tg))
    # ---- sph_err: targets in the dead zone of quat_rotvec3 (the pose advanced by dt), and 3.8 rad away (error quaternion w < 0)
    s, p, v = _lifted(orc, 0.45 * dur)
    tg = p.copy()
    for j in sph:
        o = jl[j][1]
        tg[o:o + 4] = _pose_inc(p[o:o + 4], v[o:o + 3], DT)
    add("sph_err", "dead zone", _set_targets(orc, s, jl, tg))
    s, p, _ = _lifted(orc, 0.45 * dur, vel=zero)
    tg = p.copy()
    for k, j in enumerate(sph):
        o = jl[j][1]
        tg[o:o + 4] = qmul(p[o:o + 4], axis_angle([np.cos(k), 0.5, np.sin(k)], 3.8))
    add("sph_err", "past pi", _set_targets(orc, s, jl, tg))
    # ---- rev_wrap: unlimited revolute joints past +-pi and +-2 pi
    free_rev = [j for j in rev if not jl[j][2]]
    if free_rev:
        for ang in (3.6, -3.6, 7.0, -7.0):
            s, p, v = _lifted(orc, 0.3 * dur, vel=zero)
            p = p.copy()
            for j in free_rev:
                p[jl[j][1]] = ang
            orc.set_pose_vel(p, v)
            s = orc.get_snapshot()
            tg = p.copy()
            for j in free_rev:
                tg[jl[j][1]] = 0.5
            add("rev_wrap", "angle %+.1f" % ang, _set_targets(orc, s, jl, tg))
    # ---- root_quirk: a tilted, spinning, translating root
    for k, (w, vb) in enumerate(((np.array([4.0, 14.0, -6.0]), np.array([2.5, 0.8, -1.5])), (np.array([-9.0, 5.0, 11.0]), np.array([-1.0, 0.3, 3.0])))):
        s, p, _ = _lifted(orc, (0.1 + 0.4 * k) * dur, base_rot=axis_angle([1.0, 0.0, 1.0], 0.8 + 0.5 * k), base_w=w, base_v=vb)
        add("root_quirk", "spin %.0f rad/s" % np.linalg.norm(w), _set_targets(orc, s, jl, p))
    # ---- integ: every rate below 1e-3 rad/s (targets at the pose: no PD torque to speak of), and every rate well above it
    v = zero.copy(); v[3:6] = [2e-4, -3e-4, 1e-4]
    for j in sph:
        v[jl[j][1]:jl[j][1] + 3] = [1e-4, 2e-4, -1e-4]
    s, p, _ = _lifted(orc, 0.6 * dur, vel=v)
    add("integ", "rates below 1e-3", _set_targets(orc, s, jl, p))
    v = zero.copy(); v[3:6] = [0.05, 0.02, -0.03]
    for j in sph:
        v[jl[j][1]:jl[j][1] + 3] = [0.5, -0.3, 0.2]
    for j in rev:
        v[jl[j][1]] = 0.5
    s, p, _ = _lifted(orc, 0.6 * dur, vel=v)
    add("integ", "rates above 1e-3", _set_targets(orc, s, jl, p))
    # ---- integ_clamp: a dt = 1/60 update, base and spherical rates of 171 rad/s (every component at 99)
    for sgn in (1.0, -1.0):
        v = zero.copy(); v[3:6] = [99.0 * sgn, 99.0, -99.0 * sgn]
        for j in sph:
            v[jl[j][1]:jl[j][1] + 3] = [99.0, -99.0 * sgn, 99.0]
        s, p, _ = _lifted(orc, 0.8 * dur, vel=v)
        add("integ_clamp", "dt 1/%d spin %+d" % (round(1 / dt_clamp(substeps)), sgn), _set_targets(orc, s, jl, p), dt_clamp(substeps))
    # ---- substeps
    if substeps != 2:
        s, p, _ = _lifted(orc, 0.5 * dur)
        add("substeps", "%d sub-steps" % substeps, _set_targets(orc, s, jl, p))
    return out


def load_joints(root, name):
    return load_char(root, name)["Skeleton"]["Joints"]


def load_char(root, name):
    with open(os.path.join(root, char_file(name))) as f:
        return json.load(f)


def library(orc, root, name):
    joints = load_joints(root, name)
    sub = CHARS[name][1] if name in CHARS else 2
    return build(orc, joints, name, sub)
