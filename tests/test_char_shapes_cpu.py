"""The constructed characters and state library of tests/char_shapes.py, without a device: every character loads in the host model and the
oracle and gets a launch plan; the dynamics-tree rule of the step kernel's table build, restated from the character files, sees the host
model's tree and reaches every shape of the coverage table; the loader refuses each limit by name; every state takes its branch in the oracle
with a margin of at least 10 % of the threshold; removing a branch's effect moves the oracle's one-update result by at least 10 x the bound
of the GPU comparison; the library is deterministic.

Coverage only (no effect size: the branch changes the result by less than fp32 resolves):
  * the dead zone of quat_rotvec3 (s <= 1e-6): the error it drops is below 1e-6 rad, times Kp about 4e-4 Nm;
  * the small-angle series of quat_integrate3 (|w| < 1e-3): it differs from sin(|w| h / 2) / |w| by |w|^4 h^5 / 3840, below 1e-30;
  * the root's Stable-PD bias term (the reference's BuildCjRoot quirk, dm_step.cu aba_solve_body with bullet == 0): it enters the root's
    bias acceleration in the same pure-linear slot as gravity, and a shift leaves a pure-linear spatial acceleration unchanged, so it reaches
    every link as the same linear acceleration d.  Its change of the bias force is then M [d; 0], and since Kd is zero on the base rows,
    (M + dt Kd)^-1 M [d; 0] = [d; 0]: the joint accelerations, and so the Stable-PD torques, are exactly unchanged.  A kernel with w x v
    in its place is an equivalent mutant.  test_root_quirk_cannot_change_the_stable_pd_torques asserts the identity."""
import json
import os

import numpy as np
import pytest

from tests import char_shapes as C
from tests.oracle_binding import Oracle
from tests.parity_util import SnapLayout, compare_sim_state, quat_err
from tests.solver_states import LIMITS, POINTS, axis_angle, qmul

ALL = list(C.CHARS) + list(C.SHIPPED)


@pytest.fixture(scope="module")
def roots(asset_root, tmp_path_factory):
    """(asset root of the constructed characters, the shipped asset root)"""
    return C.write_root(asset_root, str(tmp_path_factory.mktemp("char_shapes") / "assets")), asset_root


def _root(roots, name):
    return roots[1] if name in C.SHIPPED else roots[0]


def _post(orc, snap, dt):
    orc.set_snapshot(snap)
    orc.update(dt)
    return orc.last_rows(), orc.get_snapshot()


def test_characters_load_and_get_a_launch_plan(roots):
    from deepmimic_b200.capi import HostModel
    for name, (make, sub) in C.CHARS.items():
        spec = make()
        h = HostModel(C.args_of(name), roots[0])
        o = Oracle(C.args_of(name), roots[0])
        assert h.dims.num_joints == o.num_joints == len(spec)
        plan = h.plan_launch(256)
        assert plan["tile_width"] == (16 if len(spec) <= 16 else 32)
        assert plan["envs_per_block"] >= (2 if plan["tile_width"] == 16 else 1)
        print("%s: %d links, %d dofs, %d sub-steps, W = %d, %d environments per block" % (name, len(spec), o.num_dofs, sub, plan["tile_width"], plan["envs_per_block"]))
        h.close()


def _coverage(roots):
    """every row of the coverage table -> the characters that reach it, from the restated dynamics tree and the character files"""
    rows = {k: set() for k in ("fixed link with children", "fixed leaf not lumped, under the root", "fixed leaf not lumped, under a fixed link",
                               "leaf lumped into a spherical parent", "revolute child of the root", "fixed child of the root", "non-root link with 4 children",
                               "nl 16", "nl 17", "nl 32", "last depth 23", "96 dofs", "unlimited revolute joint", "has_limit with LimLow0 > 0",
                               "has_limit with LimHigh0 < 0", "joint without TorqueLim", "1 sub-step", "3 sub-steps")}
    for name, (make, sub) in C.CHARS.items():
        J = C.load_joints(roots[0], name)
        T = C.dyn_tree(J)
        typ = [j["Type"] for j in J]
        for i, t in enumerate(T):
            kids = [c for c in range(len(J)) if J[c]["Parent"] == i]
            if i and typ[i] == "fixed" and kids:
                rows["fixed link with children"].add(name)
            if i and typ[i] == "fixed" and not kids and not t["lumped"]:
                rows["fixed leaf not lumped, under the root" if J[i]["Parent"] == 0 else "fixed leaf not lumped, under a fixed link"].add(name)
            if t["lumped"] and typ[J[i]["Parent"]] == "spherical":
                rows["leaf lumped into a spherical parent"].add(name)
            if t["byp"] == 0 and typ[i] in ("revolute", "fixed"):
                rows["%s child of the root" % typ[i]].add(name)
            if i and len(kids) == 4:
                rows["non-root link with 4 children"].add(name)
            if typ[i] == "revolute":
                if not C.has_limit(J[i]):
                    rows["unlimited revolute joint"].add(name)
                elif J[i]["LimHigh0"] < 0:
                    rows["has_limit with LimHigh0 < 0"].add(name)
                if J[i]["LimLow0"] > 0 and J[i]["LimHigh0"] > J[i]["LimLow0"] and not C.has_limit(J[i]):
                    rows["has_limit with LimLow0 > 0"].add(name)
            if i and typ[i] != "fixed" and "TorqueLim" not in J[i]:
                rows["joint without TorqueLim"].add(name)
        if "nl %d" % len(J) in rows:
            rows["nl %d" % len(J)].add(name)
        if max(C.last_depths(J)) == 23:
            rows["last depth 23"].add(name)
        if 6 + sum(t["ndof"] for t in T) == 96:
            rows["96 dofs"].add(name)
        if sub != 2:
            rows["%d sub-step%s" % (sub, "s" if sub > 1 else "")].add(name)
    return rows


def test_dynamics_tree_restatement_sees_the_host_model_and_covers_every_shape(roots):
    from deepmimic_b200.capi import HostModel
    kinds = {"revolute": 0, "spherical": 1, "fixed": 2, "none": 2}
    shapes = set()
    for name in C.CHARS:
        J = C.load_joints(roots[0], name)
        T = C.dyn_tree(J)
        h = HostModel(C.args_of(name), roots[0])
        # the restatement's inputs are the host model's tree: parents, joint kinds, dof offsets, and the link table's masses
        assert list(h.info("parents")) == [j["Parent"] for j in J]
        assert list(h.info("joint_types")) == [kinds[j["Type"]] for j in J]
        off = np.concatenate([[6], 6 + np.cumsum([t["ndof"] for t in T])[:-1]])
        assert list(h.info("dof_offsets")) == list(off)
        bodies = C.load_char(roots[0], name)["BodyDefs"]
        np.testing.assert_allclose(h.link_table()[:, 0], [b["Mass"] for b in bodies], rtol=1e-7)
        assert h.layout()["dofs"] == 6 + sum(t["ndof"] for t in T)
        for i, t in enumerate(T):   # a tree the kernel's passes can walk: levels below the parent's, children listed once
            if i and not t["lumped"]:
                assert T[t["parent"]]["level"] == t["level"] - 1 and i in T[t["parent"]]["children"]
            shapes.add((J[i]["Type"], bodies[i]["Shape"]))
        h.close()
    assert {(t, s) for t in ("revolute", "spherical", "fixed") for s in C.SHAPES} <= shapes
    rows = _coverage(roots)
    for k, v in rows.items():
        print("  %-45s %s" % (k, ", ".join(sorted(v))))
    assert all(rows.values()), [k for k, v in rows.items() if not v]


def test_lumped_leaf_rules_agree(roots):
    """tests/dynamics_ref.py's lumped leaves (the draw copies their parent's mass factor) are the table build's"""
    from tests.dynamics_ref import lumped_leaves
    for name in ALL:
        J = C.load_joints(_root(roots, name), name)
        T = C.dyn_tree(J)
        lp = lumped_leaves(os.path.join(_root(roots, name), C.char_file(name)))
        assert [p >= 0 for p in lp] == [t["lumped"] for t in T], name
        assert all(p == J[i]["Parent"] for i, p in enumerate(lp) if p >= 0)


def _refusal_specs():
    sph = lambda p: ("spherical", p, "box", {})
    out = {}
    out["33 links"] = ("more links than lanes", [("none", -1, "sphere", {})] + [sph(0 if n == 1 else (n - 2) // 4 + 1) for n in range(1, 33)])
    out["5 children"] = ("more than 4 children", [("none", -1, "sphere", {}), sph(0)] + [("revolute", 1, "box", {})] * 5)
    out["chain of depth 24"] = ("dof chain too long", [("none", -1, "sphere", {})] + [sph(i) for i in range(6)] + [("revolute", 6, "box", {})])
    out["97 dofs"] = ("too many dofs", [("none", -1, "sphere", {})] + [sph(0 if i < 4 else (i - 4) // 4 + 1) for i in range(30)] + [("revolute", 8, "box", {})])
    out["non-floating root"] = ("floating-base", [("spherical", -1, "sphere", {}), sph(0)])
    out["planar joint"] = ("unsupported joint type", [("none", -1, "sphere", {}), sph(0), ("planar", 1, "box", {})])
    return out


@pytest.mark.parametrize("case", list(_refusal_specs()))
def test_loader_refuses_each_limit_by_name(asset_root, tmp_path, case):
    from deepmimic_b200.capi import HostModel
    msg, spec = _refusal_specs()[case]
    root = C.write_root(asset_root, str(tmp_path / "assets"), {"refused": (spec, 2)})
    if case == "97 dofs":
        assert 6 + sum({"spherical": 3, "revolute": 1}.get(s[0], 0) for s in spec[1:]) == 97 and len(spec) <= 32
        assert max(C.last_depths(C.load_joints(root, "refused"))) < 24
    with pytest.raises(RuntimeError, match=msg):
        HostModel(C.args_of("refused"), root)


def _sph_err(p, v, tg, dt):
    """(sin, angle) of the Stable-PD error quaternion conj(pose advanced by dt) (x) target, (w, x, y, z)"""
    qi = C._pose_inc(p, v, dt)
    e = qmul(qi * np.array([1.0, -1.0, -1.0, -1.0]), tg)
    s = np.linalg.norm(e[1:])
    return s, 2.0 * np.arctan2(s, e[0])


@pytest.mark.parametrize("name", ALL)
def test_states_reach_their_branches_with_a_margin(roots, name):
    root = _root(roots, name)
    orc = Oracle(C.args_of(name), root)
    J = C.load_joints(root, name)
    jl = C.joint_layout(J)
    nl = len(J)
    lay = SnapLayout(nl)
    sub = C.CHARS[name][1] if name in C.CHARS else 2
    lib = C.library(orc, root, name)
    count = {}
    for st in lib:
        count[st.cls] = count.get(st.cls, 0) + 1
        rows, after = _post(orc, st.snap, st.dt)
        assert len(rows) == sub
        if st.cls != "integ_clamp":   # airborne, inside every limit: no constraint row (the 1/60 update whips the links around)
            assert not rows[:, LIMITS].any() and not rows[:, POINTS].any(), (st, rows)
        assert sum(lay.contact_counts(after)) == 0, st
        orc.set_snapshot(st.snap)
        p, v = orc.get_pose()
        tgt = lambda j: st.snap[lay.tgt + 4 * j: lay.tgt + 4 * j + 4]
        if st.cls == "clamp":
            # above: some spherical and some revolute joint at >= 1.1 x its limit; below: every joint at <= 0.9 x
            tau = orc.spd_tau(st.dt)
            over = {"spherical": 0, "revolute": 0}
            for j, (t, o, _, lim) in enumerate(jl):
                if t in over and np.isfinite(lim):
                    m = np.linalg.norm(tau[o:o + (3 if t == "spherical" else 1)])
                    over[t] += m >= 1.1 * lim
                    assert "above" in st.name or m <= 0.9 * lim, (st, j, m, lim)
            assert "below" in st.name or all(over[t] > 0 for t in over if any(x[0] == t and np.isfinite(x[3]) for x in jl)), (st, over)
        elif st.cls == "sph_err":
            for j, (t, o, _, _) in enumerate(jl):
                if t == "spherical":
                    s, ang = _sph_err(p[o:o + 4], v[o:o + 3], tgt(j), st.dt)
                    assert (s <= 1e-6 / 1.1) if "dead" in st.name else (ang >= 1.1 * np.pi), (st, j, s, ang)
        elif st.cls == "rev_wrap":
            jp = st.snap[lay.jpos:lay.jpos + 4 * nl].reshape(nl, 4)[:, 0]
            free = [j for j, x in enumerate(jl) if x[0] == "revolute" and not x[2]]
            thr = np.pi if abs(jp[free[0]]) < 5 else 2 * np.pi
            assert all(abs(jp[j]) >= 1.1 * thr for j in free), (st, jp[free])
        elif st.cls == "root_quirk":
            assert 10.0 <= np.linalg.norm(st.snap[lay.base_omega]) <= 20.0
        if st.cls in ("integ", "integ_clamp"):
            rates = [np.linalg.norm(after[lay.base_omega])] + [np.linalg.norm(after[lay.jvel + 3 * j: lay.jvel + 3 * j + 3]) for j, x in enumerate(jl) if x[0] == "spherical"]
            if "below" in st.name:
                assert max(rates) <= 0.9e-3, (st, rates)
            elif "above" in st.name:
                assert min(rates) >= 1.1e-3, (st, rates)
            else:
                h = st.dt / sub
                assert rates[0] * h >= 1.1 * np.pi / 4 and max(rates[1:]) * h >= 1.1 * np.pi / 4, (st, rates, h)
    want = set(C.CLASSES) - ({"rev_wrap"} if not any(x[0] == "revolute" and not x[2] for x in jl) else set()) - ({"substeps"} if sub == 2 else set())
    assert set(count) == want, (sorted(count), sorted(want))
    print("%s: %s" % (name, ", ".join("%s %d" % (k, count[k]) for k in C.CLASSES if k in count)))


def test_has_limit_rule_in_the_oracle(roots):
    """c16: joint 5 (LimLow0 0.2, LimHigh0 2) far below LimLow0 makes no limit row; joint 6 (LimLow0 -1, LimHigh0 -0.5) above LimHigh0 makes one"""
    orc = Oracle(C.args_of("c16"), roots[0])
    J = C.load_joints(roots[0], "c16")
    jl = C.joint_layout(J)
    assert not C.has_limit(J[5]) and C.has_limit(J[6]) and J[5]["LimLow0"] > 0 and J[6]["LimHigh0"] < 0
    for j, ang, rows in ((5, -1.0, 0), (6, 0.0, 1)):
        s, p, v = C._lifted(orc, 0.0, vel=np.zeros(orc.pose_dim))
        p = p.copy(); p[jl[j][1]] = ang
        orc.set_pose_vel(p, v)
        r, _ = _post(orc, C._set_targets(orc, orc.get_snapshot(), jl, p), C.DT)
        assert r[0, LIMITS] == rows, (j, r)


# ---- effect sizes
def _gains(orc, root, name, jl):
    """Kp and Kd per row of the pose layout, from the controller file the character's arg file names"""
    with open(os.path.join(root, C.args_of(name)[1])) as f:
        words = f.read().split()
    with open(os.path.join(root, words[words.index("--char_ctrl_files") + 1])) as f:
        ctrl = json.load(f)["PDControllers"]
    Kp, Kd = np.zeros(orc.pose_dim), np.zeros(orc.pose_dim)
    for j, (t, o, _, _) in enumerate(jl):
        n = {"spherical": 4, "revolute": 1}.get(t, 0)
        Kp[o:o + n], Kd[o:o + n] = ctrl[j]["Kp"], ctrl[j]["Kd"]
    return Kp, Kd


def _clamped(tau, jl):
    t = tau.copy()
    for j, (k, o, _, lim) in enumerate(jl):
        n = 3 if k == "spherical" else 1 if k == "revolute" else 0
        m = np.linalg.norm(t[o:o + n]) if n else 0.0
        if n and m > lim:
            t[o:o + n] *= lim / m
    return t


def _aba_dqd(orc, jl, tau_a, tau_b, dt):
    """first-order change of one update's generalised velocities when the applied (clamped) joint torques change from tau_a to tau_b:
    dt x the difference of Bullet's articulated-body accelerations (the oracle's restatement), base rows in m/s"""
    def jt(tau):
        out = []
        for t, o, _, _ in jl:
            out += list(16.0 * tau[o:o + 3]) if t == "spherical" else [16.0 * tau[o]] if t == "revolute" else []
        return np.array(out)
    d = orc.bullet_aba(jt(tau_b), True).astype(np.float64) - orc.bullet_aba(jt(tau_a), True).astype(np.float64)
    d[3:6] /= 4.0
    return dt * np.abs(d).max()


def _spd_dtau(orc, root, name, jl, dt, de):
    """change of the Stable-PD torque (pose layout) for a change de of the PD error:
    tau = Kp e + Kd (-v - dt a), a = (M + dt Kd)^-1 (Kp e - Kd v - C)"""
    Kp, Kd = _gains(orc, root, name, jl)
    M, _ = orc.rbd_mass_bias()
    live = [i for i in range(orc.pose_dim) if M[i, i] != 0]
    A = M[np.ix_(live, live)] + np.diag(dt * Kd[live])
    da = np.zeros(orc.pose_dim)
    da[live] = np.linalg.solve(A, (Kp * de)[live])
    return Kp * de - Kd * dt * da


@pytest.mark.parametrize("name", list(C.CHARS))
def test_each_branch_moves_the_update_by_ten_times_the_bound(roots, tmp_path, name):
    """the oracle's one-update result without each branch's effect, against the real one, in units of the bound the GPU comparison applies
    to that update (char_shapes.bounds: the character's q-dot floor, Q_FLOOR, or 8 x the update's envelope where that is larger):
      clamp        the oracle built from the character with every TorqueLim x 1e6
      rev_wrap     the same state with the PD target moved by the 2 pi k the wrap takes off
      sph_err      (past pi) the unwrapped error's Stable-PD torque, clamped, through Bullet's articulated-body accelerations (first order)
      integ_clamp  the quaternion step at |w| h against the clamped pi / 4 (q)"""
    root = roots[0]
    J = C.load_joints(root, name)
    jl = C.joint_layout(J)
    nl = len(J)
    lay = SnapLayout(nl)
    jt = [j["Type"] for j in J]
    orc, orc2 = Oracle(C.args_of(name), root), Oracle(C.args_of(name), root)
    lib = C.library(orc, root, name)
    big = C.write_root(root, str(tmp_path / "big"), C.specs([name]), edit=lambda n, c, k: [j.update(TorqueLim=1e6 * j["TorqueLim"]) for j in c["Skeleton"]["Joints"] if "TorqueLim" in j])
    orc_big = Oracle(C.args_of(name), big)
    rng = np.random.default_rng(3)
    eff = {}
    for st in lib:
        _, real = _post(orc, st.snap, st.dt)
        bq, bqd = C.bounds(name, C.envelope(orc2, lay, jt, st.snap, real, st.dt, rng))
        if st.cls == "clamp" and "above" in st.name:
            _, alt = _post(orc_big, st.snap, st.dt)
            eff["clamp"] = compare_sim_state(lay, real, alt, jt)[1] / bqd
        elif st.cls == "rev_wrap":
            s = st.snap.copy()
            for j, (t, o, lim, _) in enumerate(jl):
                if t == "revolute" and not lim:
                    a = st.snap[lay.jpos + 4 * j]
                    s[lay.tgt + 4 * j] -= a - (np.fmod(a + np.pi * np.sign(a), 2 * np.pi) - np.pi * np.sign(a))
            _, alt = _post(orc, s, st.dt)
            eff["rev_wrap"] = min(eff.get("rev_wrap", np.inf), compare_sim_state(lay, real, alt, jt)[1] / bqd)
        elif st.cls == "sph_err" and "past" in st.name:
            orc.set_snapshot(st.snap)
            p, v = orc.get_pose()
            de = np.zeros(orc.pose_dim)
            for j, (t, o, _, _) in enumerate(jl):
                if t == "spherical":
                    tg = st.snap[lay.tgt + 4 * j: lay.tgt + 4 * j + 4]
                    s_, ang = _sph_err(p[o:o + 4], v[o:o + 3], tg, st.dt)
                    e = qmul(C._pose_inc(p[o:o + 4], v[o:o + 3], st.dt) * np.array([1.0, -1.0, -1.0, -1.0]), tg)
                    de[o:o + 3] = e[1:] / s_ * 2 * np.pi   # unwrapped minus wrapped rotation vector: ang - (ang - 2 pi) along the axis
            tau = orc.spd_tau(st.dt)
            eff["sph_err"] = _aba_dqd(orc, jl, _clamped(tau, jl), _clamped(tau + _spd_dtau(orc, root, name, jl, st.dt, de), jl), st.dt) / bqd
        elif st.cls == "integ_clamp":
            h = st.dt / C.CHARS[name][1]
            worst = 0.0
            for w in [real[lay.base_omega]] + [real[lay.jvel + 3 * j: lay.jvel + 3 * j + 3] for j, x in enumerate(jl) if x[0] == "spherical"]:
                n = np.linalg.norm(w)
                if n * h > np.pi / 4:
                    worst = max(worst, quat_err(axis_angle(w, n * h), axis_angle(w, np.pi / 4)))
            eff["integ_clamp"] = min(eff.get("integ_clamp", np.inf), worst / bq)
    print("%s: effect / bound %s" % (name, ", ".join("%s %.3g" % kv for kv in sorted(eff.items()))))
    want = {"clamp", "sph_err", "integ_clamp"} | ({"rev_wrap"} if any(x[0] == "revolute" and not x[2] for x in jl) else set())
    assert set(eff) == want, sorted(eff)
    assert all(v >= 10.0 for v in eff.values()), eff


@pytest.mark.parametrize("name", ALL)
def test_root_quirk_cannot_change_the_stable_pd_torques(roots, name):
    """the identity of the module docstring on every root_quirk state: the quirk's linear acceleration d (the kernel's R^T (w x R v) against
    w x v) is large, Kd is zero on the base rows, and (M + dt Kd)^-1 M [d; 0] = [d; 0] with the oracle's M to rounding"""
    root = _root(roots, name)
    orc = Oracle(C.args_of(name), root)
    J = C.load_joints(root, name)
    jl = C.joint_layout(J)
    lay = SnapLayout(len(J))
    _, kd = _gains(orc, root, name, jl)
    assert not kd[:7].any()
    for st in [s for s in C.library(orc, root, name) if s.cls == "root_quirk"]:
        x, y, z, w = st.snap[lay.base_quat]
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                      [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
        om, v = st.snap[lay.base_omega], st.snap[lay.base_vel] / 4.0
        d = R.T @ np.cross(om, R @ v) - np.cross(om, v)
        assert np.linalg.norm(d) > 1.0, (st, d)   # m/s^2: the quirk is not negligible on these states
        orc.set_snapshot(st.snap)
        M, _ = orc.rbd_mass_bias()
        live = [i for i in range(orc.pose_dim) if M[i, i] != 0]
        e = np.zeros(orc.pose_dim); e[0:3] = d
        A = M[np.ix_(live, live)] + np.diag(C.DT * kd[live])
        xs = np.linalg.solve(A, (M @ e)[live])
        assert np.abs(xs - e[live]).max() <= 1e-9 * np.linalg.norm(d), (st, np.abs(xs - e[live]).max())


@pytest.mark.parametrize("name", ["c32", "humanoid3d"])
def test_library_is_deterministic(roots, name):
    root = _root(roots, name)
    a = C.library(Oracle(C.args_of(name), root), root, name)
    b = C.library(Oracle(C.args_of(name), root), root, name)
    assert [(s.cls, s.name, s.dt) for s in a] == [(s.cls, s.name, s.dt) for s in b]
    assert all(np.array_equal(x.snap, y.snap) for x, y in zip(a, b))
