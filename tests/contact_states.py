"""Constructed simulator states that drive each branch of the step kernel's link-plane collision pass (dm_step.cu: collide) on one test
link, built from poses and hand-written manifolds -- no rollouts.  Every state names its test link and the branch it was built for, with
the collision tap (Oracle.last_contacts()) that the first Bullet sub-step of one Update(1/600) must produce on that link
(tests/test_contact_states_cpu.py keeps the library honest, tests/test_collision_branches_gpu.py compares the kernel with the oracle on it).

A state is built in four steps.  The character is held in its rest pose, rotated so that the test link's support vertex is the lowest of
all links by at least twice every other link's contact threshold (and, for a box or a capsule, so that the link's down direction picks the
wanted corner or end), then lowered so that the vertex sits at a chosen signed distance from the plane.  Every other manifold is empty.
The test link's cached points are written by hand: local point A (link frame), anchor B on the plane, impulses, distance and lifetime.
Velocities are zero and the PD targets equal the pose, so one update moves the link by far less than a threshold.

Cached points are placed relative to the support vertex v and the link-frame down direction d: A = v + u - h d with u perpendicular to d
puts A at height (vertex height + h) and |u| away from the vertex horizontally; B is A's projection onto the plane, plus a lateral drift.
The distance stored with a cached point is only read by sortCachedPoints' keep-deepest search (the refresh recomputes it), so it is
chosen freely to pick the deepest point.

Classes (both characters; thresholds from Oracle.link_table()):
  support    an empty manifold, the vertex penetrating and above the plane inside the threshold: each corner of a box, each end of a
             capsule, a sphere, and the humanoid's wrist (a sphere on a fixed leaf)
  add        a new point into a cache of 1, 2 or 3 points, all 2-3 thresholds away from it
  replace    the nearest cached point within the threshold is replaced and keeps its impulses and lifetime: one point within the
             threshold, two with the nearer one in the first or in the second slot, and one of four
  full       sortCachedPoints: deepest (the new point or slot 0-3) x replaced slot, all 16 combinations on a box, a capsule and a sphere
  refresh    the vertex above the threshold, points still cached and kept
  removal    every non-empty subset of a full cache removed, by distance and by lateral drift of B in both alternations (box), and one
             removal of each kind on a capsule and a sphere
  fall       the contact-fall tolerance distance <= 0.001 x scale: a fall-contact link inside it, the same link between it and the
             threshold, and a non-fall link inside it
  release    four cached points removed in the first sub-step (two by distance, two by drift) while the link falls from three thresholds
             up; it is back inside its threshold about 17 updates later, within a 40-update launch"""
import itertools

import numpy as np

from tests import solver_states as S
from tests.parity_util import SnapLayout

DT = S.DT
CHARS = S.CHARS
NONE, ADD, REPLACE, FULL = range(4)
EVENTS = ("none", "add", "replace", "full")
EVENT, SLOT, DEEPEST, RM_DIST, RM_DRIFT, COUNT = range(6)   # Oracle.last_contacts() columns
SCALE = 4.0
TOL = 0.001 * SCALE   # cContactManager: a point touches the ground at distance <= 0.001 x world scale
# test links: box, capsule and sphere for the branch classes, a fall-contact and a non-fall link for the tolerance
LINKS = {
    "humanoid3d": dict(box=5, capsule=6, sphere=2, wrist=8, fall=2, nonfall=5),      # right ankle, right shoulder, neck (head), right wrist
    "dog3d": dict(box=4, capsule=22, sphere=2, fall=4, nonfall=8),                 # head, tail tip, spine1 (chest), head, left finger
}
RELEASE_UPDATES = 40


class State:
    def __init__(self, cls, name, snap, link, expect, expect2=None):
        self.cls, self.name, self.snap, self.link = cls, name, snap, link
        self.expect = expect     # sub-step 1 tap of the test link: (event, slot, deepest, removed by distance, removed by drift, count)
        self.expect2 = expect2   # sub-step 2: (event, count), or None where the state makes no claim

    def __repr__(self):
        return "%s/%s" % (self.cls, self.name)


def link_shapes(orc):
    """per link: (shape name, half extents, contact threshold) from Oracle.link_table()"""
    lt = orc.link_table()
    out = []
    for j in range(orc.num_joints):
        he = lt[j, 20:23]
        out.append(("box" if he[2] > 0 else "capsule" if he[1] > 0 else "sphere", he.copy(), float(lt[j, 23])))
    return out


def support(shape, he, dl):
    """float64 convex->localGetSupportingVertex(dl) for a box, a capsule (radius he[0], half height he[1]) or a sphere (radius he[0])"""
    dl = np.asarray(dl, dtype=np.float64)
    if shape == "box":
        return np.where(dl >= 0, he, -he)
    sup = np.zeros(3)
    if shape == "capsule":
        sup[1] = he[1] if dl[1] >= 0 else -he[1]
    return sup + he[0] * dl / np.linalg.norm(dl)


def collide64(B, P, shape, he, thr, mani):
    """float64 restatement of one link's collision pass (btConvexPlaneCollisionAlgorithm + btPersistentManifold) from its collider frame
    (basis B, position P) and its manifold rows [4, 12] as stored in a snapshot.  Returns (tap, manifold after, decisions): tap as in
    Oracle.last_contacts(); decisions lists every comparison the pass made as (kind, value, threshold), for the margins."""
    m = [r.copy() for r in mani]
    cnt = 0
    while cnt < 4 and m[cnt][0] != 0:
        cnt += 1
    dec = []
    dl = B.T @ np.array([0.0, -1.0, 0.0])
    if shape == "box":
        dec += [("box down component", abs(x), 0.0) for x in dl]
    elif shape == "capsule":
        dec.append(("capsule end", abs(dl[1]) / np.linalg.norm(dl), 0.0))
    vtx = support(shape, he, dl)
    vw = B @ vtx + P
    dist = vw[1]
    dec.append(("vertex distance", dist, thr))
    event, slot, deepest, rd, rf = NONE, -1, -1, 0, 0
    if dist < thr:
        dd = [float(np.sum((m[k][1:4] - vtx) ** 2)) for k in range(cnt)]
        dec += [("cache match", np.sqrt(x), thr) for x in dd]
        near = [k for k in range(cnt) if dd[k] < thr * thr]
        new = np.zeros(12)
        new[0], new[1:4], new[4:7], new[10] = 1.0, vtx, (vw[0], 0.0, vw[2]), dist
        if near:
            slot = min(near, key=lambda k: dd[k])
            if len(near) > 1:
                s = sorted(np.sqrt(dd[k]) for k in near)
                dec.append(("nearest lead", s[1] - s[0], 0.1 * thr))
            new[7:10], new[11] = m[slot][7:10], m[slot][11]
            event = REPLACE
        elif cnt < 4:
            slot, event = cnt, ADD
            cnt += 1
        else:
            event = FULL
            pen = [dist] + [m[k][10] for k in range(4)]
            deepest = int(np.argmin(pen)) - 1
            s = sorted(pen)
            dec.append(("deepest lead", s[1] - s[0], 0.1 * thr))
            res = areas(vtx, [m[k][1:4] for k in range(4)])
            if deepest >= 0:
                res[deepest] = 0.0
            slot = int(np.argmax(res))
            s = sorted(res)
            dec.append(("area lead", s[3] / s[2] - 1.0 if s[2] > 0 else np.inf, 0.1))
        m[slot] = new
    # refreshContactPoints
    for k in range(cnt - 1, -1, -1):
        pa = B @ m[k][1:4] + P
        m[k][10] = pa[1] - m[k][5]
        m[k][11] += 1
    for k in range(cnt - 1, -1, -1):
        pa = B @ m[k][1:4] + P
        dec.append(("refresh distance", m[k][10], thr))
        rm = not m[k][10] <= thr
        if rm:
            rd |= 1 << k
        else:
            drift = np.sqrt((m[k][4] - pa[0]) ** 2 + (m[k][5] - (pa[1] - m[k][10])) ** 2 + (m[k][6] - pa[2]) ** 2)
            dec.append(("lateral drift", drift, thr))
            if drift > thr:
                rf |= 1 << k
                rm = True
        if rm:
            m[k] = m[cnt - 1].copy()
            m[cnt - 1] = np.zeros(12)
            cnt -= 1
    return (event, slot, deepest, rd, rf, cnt), np.array(m), dec


def areas(v, pts):
    """sortCachedPoints' four area terms (gContactCalcArea3Points): res[k] is the squared area spanned without cached point k"""
    def area(a, b):
        c = np.cross(a, b)
        return float(c @ c)
    p0, p1, p2, p3 = pts
    return [area(v - p1, p3 - p2), area(v - p0, p3 - p2), area(v - p0, p3 - p1), area(v - p0, p2 - p1)]


def _arc(a, b):
    """quaternion (w, x, y, z) of the shortest rotation taking unit vector a to unit vector b"""
    a = a / np.linalg.norm(a); b = b / np.linalg.norm(b)
    c = np.cross(a, b); w = 1.0 + a @ b
    if w < 1e-9:   # antiparallel: any perpendicular axis
        p = np.cross(a, [1.0, 0.0, 0.0] if abs(a[0]) < 0.9 else [0.0, 1.0, 0.0])
        q = np.concatenate([[0.0], p / np.linalg.norm(p)])
    else:
        q = np.concatenate([[w], c])
    return q / np.linalg.norm(q)


def _qmat(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _sphere(n=4000):
    i = np.arange(n) + 0.5
    phi = np.arccos(1.0 - 2.0 * i / n); th = np.pi * (1.0 + 5.0 ** 0.5) * i
    return np.stack([np.cos(th) * np.sin(phi), np.cos(phi), np.sin(th) * np.sin(phi)], 1)


class Builder:
    """places the character for one test link and writes its manifold; every result is checked against the oracle's collider frames"""

    def __init__(self, orc, asset_root, ch):
        self.orc, self.ch = orc, ch
        self.lay = SnapLayout(orc.num_joints)
        self.shapes = link_shapes(orc)
        self.thr = np.array([s[2] for s in self.shapes])
        self.jl = jl = S.joint_layout(asset_root, CHARS[ch]["char"])
        import json
        import os
        self.parent = [jd["Parent"] for jd in json.load(open(os.path.join(asset_root, CHARS[ch]["char"])))["Skeleton"]["Joints"]]
        orc.reset(0.0, 0.0, 20.0)
        orc.set_action(np.zeros(orc.action_size))
        p, v = orc.get_pose()
        p = p.copy()
        for t, lo, hi, o in jl[1:]:
            if t == "spherical":
                p[o:o + 4] = [1.0, 0.0, 0.0, 0.0]
            elif t == "revolute":
                p[o] = 0.0
        p[0:3] = 0.0; p[3:7] = [1.0, 0.0, 0.0, 0.0]
        orc.set_pose_vel(p, np.zeros_like(v))
        s = orc.get_snapshot()
        s[self.lay.mani:self.lay.scal] = 0.0
        s[0:3] = 0.0; s[3:7] = [0.0, 0.0, 0.0, 1.0]
        self.rest = s
        orc.set_snapshot(s)
        self.G = _sphere()

    def _heights(self, G, C, P):
        """[directions, links]: height of each link's support vertex above the base origin when G (base frame) points down"""
        H = np.zeros((len(G), len(self.shapes)))
        for j, (shape, he, _) in enumerate(self.shapes):
            dl = G @ C[j]   # rows: C_j^T g
            if shape == "box":
                vt = np.where(dl >= 0, he, -he)
            else:
                vt = he[0] * dl / np.linalg.norm(dl, axis=1, keepdims=True)
                if shape == "capsule":
                    vt[:, 1] += np.where(dl[:, 1] >= 0, he[1], -he[1])
            H[:, j] = -np.einsum("nk,nk->n", G, P[j] + vt @ C[j].T)
        return H

    def down(self, j, pred=None):
        """(joint positions, base-frame down direction) that make link j's support vertex the lowest by the widest margin (in units of j's
        threshold, after the 2 x threshold every other link keeps), among the orientations whose link-frame down directions (rows of an
        array) satisfy pred.  A spherical joint of link j, and of its child, is tried in the 24 rotations of a cube, a revolute child at
        its limits and their middle; every other joint stays at rest."""
        if pred is None and self.shapes[j][0] == "box":   # no flat face down: the corner would be decided by rounding
            pred = lambda dl: np.min(np.abs(dl), axis=1) >= 0.05
        def options(k):
            t, lo, hi, _ = self.jl[k]
            if t == "spherical":
                return [(k, q) for q in _CUBE]
            if t == "revolute":
                return [(k, np.array([a, 0.0, 0.0, 0.0])) for a in (0.0, lo + 0.05, hi - 0.05, 0.5 * (lo + hi))]
            return [None]
        kids = [k for k in range(len(self.jl)) if self.parent[k] == j]
        child = options(kids[0]) if len(kids) == 1 else [None]
        best = (-np.inf, None, None)
        for own in options(j) if self.jl[j][0] == "spherical" else [None]:
            for ch in child:
                jp = [x for x in (own, ch) if x is not None]
                C, P = self._frames(self._rest(jp))
                H = self._heights(self.G, C, P)
                gap = np.min(np.delete(H - H[:, [j]] - 2.0 * self.thr[None, :], j, axis=1), axis=1) / self.thr[j]
                if pred is not None:
                    gap = np.where(pred(self.G @ C[j]), gap, -np.inf)
                n = int(np.argmax(gap))
                if gap[n] > best[0] + 1e-9:
                    best = (gap[n], jp, self.G[n])
        assert best[0] >= 1.0, "%s link %d: no orientation leaves it lowest (gap %.2f thresholds)" % (self.ch, j, best[0])
        return best[1], best[2]

    def _rest(self, jp):
        s = self.rest.copy()
        for k, q in jp:
            s[self.lay.jpos + 4 * k: self.lay.jpos + 4 * k + 4] = q
        return s

    def place(self, j, orient, dist):
        """snapshot with link j's joint and the base rotated as orient = down(j, ...) says and lowered so that link j's support vertex is
        at signed distance dist; returns (snapshot, B_j, P_j, vertex (link frame), link-frame down direction)"""
        jp, g = orient
        s = self._rest(jp)
        qb = _arc(g, np.array([0.0, -1.0, 0.0]))          # base frame -> world
        s[3:7] = [-qb[1], -qb[2], -qb[3], qb[0]]           # Bullet's baseQuat (x, y, z, w) is world -> base
        B, P = self._frames(s)
        shape, he, _ = self.shapes[j]
        dl = B[j].T @ np.array([0.0, -1.0, 0.0])
        vtx = support(shape, he, dl)
        s[1] += dist - (B[j] @ vtx + P[j])[1]
        B, P = self._frames(s)
        # PD targets = the pose (the oracle's pose of this snapshot), so that one update moves nothing but what gravity and contacts do
        self.orc.set_snapshot(s)
        pose, _ = self.orc.get_pose()
        for jj, (t, lo, hi, o) in enumerate(self.jl):
            n = {"spherical": 4, "revolute": 1}.get(t, 0)
            s[self.lay.tgt + 4 * jj: self.lay.tgt + 4 * jj + n] = pose[o:o + n]
        dl = B[j].T @ np.array([0.0, -1.0, 0.0])
        return s, B[j], P[j], support(shape, he, dl), dl / np.linalg.norm(dl)

    def _frames(self, s):
        self.orc.set_snapshot(s)
        return self.orc.collider_frames()

    def point(self, B, P, v, d, u, h, drift=(0.0, 0.0), dist=0.0, imp=(0.0, 0.0, 0.0), life=1):
        """one manifold row: A = v + u - h d (u is first made perpendicular to d), B = A's projection + lateral drift (world x, z)"""
        u = np.asarray(u, dtype=np.float64)
        u = u - (u @ d) * d
        A = v + u - h * d
        aw = B @ A + P
        return np.array([1.0, *A, aw[0] + drift[0], 0.0, aw[2] + drift[1], *imp, dist, life])

    def write(self, s, j, rows):
        s = s.copy()
        o = self.lay.mani + 4 * j * 12
        s[o:o + 48] = 0.0
        for c, r in enumerate(rows):
            s[o + 12 * c: o + 12 * c + 12] = r
        return s


def _perp(d, rng, rmin, rmax):
    """a vector perpendicular to d with length in [rmin, rmax]"""
    a = np.cross(d, [1.0, 0.0, 0.0] if abs(d[0]) < 0.9 else [0.0, 1.0, 0.0]); a /= np.linalg.norm(a)
    b = np.cross(d, a)
    t = rng.uniform(0.0, 2.0 * np.pi); r = rng.uniform(rmin, rmax)
    return r * (np.cos(t) * a + np.sin(t) * b)


def _cube_rotations():
    """the 24 rotations of a cube as Bullet joint quaternions (x, y, z, w), identity first"""
    out = []
    for perm in itertools.permutations(range(3)):
        for signs in itertools.product((1.0, -1.0), repeat=3):
            R = np.zeros((3, 3))
            for r, c in enumerate(perm):
                R[r, c] = signs[r]
            if np.linalg.det(R) < 0:
                continue
            w = 0.5 * np.sqrt(max(0.0, 1.0 + np.trace(R)))
            if w > 1e-6:
                q = np.array([(R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w), w])
            else:
                k = int(np.argmax(np.diag(R)))
                x = np.sqrt(max(0.0, (R[k, k] + 1.0) / 2.0))
                q = np.zeros(4); q[k] = x
                for i in range(3):
                    if i != k:
                        q[i] = R[k, i] / (2.0 * x)
            out.append(q / np.linalg.norm(q))
    return out


_CUBE = _cube_rotations()
LIFE = (11, 23, 37, 41)


def _imp(k):
    return (0.2 + 0.1 * k, 0.03 * (k + 1), -0.02 * (k + 1))


def _full_cache(b, j, s, B, P, v, d, deepest, replaced, rng, d0):
    """four cached points for which sortCachedPoints keeps `deepest` (-1: the new point) and replaces `replaced`, both decisions with a
    10 % lead; among 4096 candidate layouts, one where dropping keep-deepest, and building res[1] from Pt(3) - Pt(1), would change the
    slot, where there is one"""
    thr = b.thr[j]
    n = 4096
    e1 = np.cross(d, [1.0, 0.0, 0.0] if abs(d[0]) < 0.9 else [0.0, 1.0, 0.0]); e1 /= np.linalg.norm(e1)
    e2 = np.cross(d, e1)
    ang = rng.uniform(0.0, 2.0 * np.pi, (n, 4)); rad = rng.uniform(1.5, 4.0, (n, 4)) * thr
    us = rad[..., None] * (np.cos(ang)[..., None] * e1 + np.sin(ang)[..., None] * e2)
    hs = rng.uniform(0.1, 0.5, (n, 4)) * thr
    pts = v + us - hs[..., None] * d
    ar = lambda a, c: np.sum(np.cross(a, c) ** 2, axis=-1)
    p0, p1, p2, p3 = (pts[:, k] for k in range(4))
    res = np.stack([ar(v - p1, p3 - p2), ar(v - p0, p3 - p2), ar(v - p0, p3 - p1), ar(v - p0, p2 - p1)], 1)
    elig = res.copy()
    if deepest >= 0:
        elig[:, deepest] = 0.0
    srt = np.sort(elig, axis=1)
    sep = np.min([np.linalg.norm(pts[:, a] - pts[:, c], axis=1) for a, c in itertools.combinations(range(4), 2)], axis=0)
    ok = (np.argmax(elig, axis=1) == replaced) & (srt[:, 3] >= 1.1 * srt[:, 2]) & (sep >= 0.5 * thr)
    alt = elig.copy()
    if deepest != 1:
        alt[:, 1] = ar(v - p0, p3 - p1)
    score = (np.argmax(alt, axis=1) != replaced).astype(int)
    if deepest >= 0:
        score += 2 * (res[:, deepest] > 1.1 * res[:, replaced])
    score = np.where(ok, score, -1)
    i = int(np.argmax(score))
    assert score[i] >= 0, "no layout for deepest %d replaced %d" % (deepest, replaced)
    dists = [d0 + 0.2 * thr + 0.1 * thr * k for k in range(4)]
    if deepest >= 0:
        dists[deepest] = d0 - 0.15 * thr   # still positive: seeding the search with 0 would find no deepest point
    rows = [b.point(B, P, v, d, us[i, k], hs[i, k], dist=dists[k], imp=_imp(k), life=LIFE[k]) for k in range(4)]
    return b.write(s, j, rows)


def build(orc, asset_root, ch):
    """the state library of character ch (a list of State); deterministic"""
    b = Builder(orc, asset_root, ch)
    L = LINKS[ch]
    rng = np.random.default_rng(11)
    out = []

    def add(cls, name, s, j, expect, expect2=None):
        out.append(State(cls, name, s, j, expect, expect2))

    # ---- support vertex on an empty manifold
    jb = L["box"]
    corner_g = {}
    for sx, sy, sz in itertools.product((-1, 1), repeat=3):
        sg = np.array([sx, sy, sz])
        g = b.down(jb, lambda dl, sg=sg: np.all(np.sign(dl) == sg, axis=1) & (np.min(np.abs(dl), axis=1) >= 0.05))
        corner_g[(sx, sy, sz)] = g
        for tag, f in (("penetrating", -0.3), ("above", 0.5)):
            s, *_ = b.place(jb, g, f * b.thr[jb])
            add("support", "box corner %+d%+d%+d %s" % (sx, sy, sz, tag), s, jb, (ADD, 0, -1, 0, 0, 1), (REPLACE, 1))
    jc = L["capsule"]
    cap_g = {}
    for end in (1, -1):
        g = b.down(jc, lambda dl, end=end: end * dl[:, 1] >= 0.2)
        cap_g[end] = g
        for tag, f in (("penetrating", -0.3), ("above", 0.5)):
            s, *_ = b.place(jc, g, f * b.thr[jc])
            add("support", "capsule end %+d %s" % (end, tag), s, jc, (ADD, 0, -1, 0, 0, 1), (REPLACE, 1))
    spheres = [("sphere", L["sphere"])] + ([("wrist", L["wrist"])] if "wrist" in L else [])
    sph_g = {}
    for what, js in spheres:
        g = b.down(js)
        sph_g[js] = g
        for tag, f in (("penetrating", -0.3), ("above", 0.5)):
            s, *_ = b.place(js, g, f * b.thr[js])
            add("support", "%s %s" % (what, tag), s, js, (ADD, 0, -1, 0, 0, 1), (REPLACE, 1))

    # the box in one corner orientation for the cache classes: its vertex 0.3 thresholds above the plane
    g_box = corner_g[(1, -1, 1)]
    thr = b.thr[jb]
    s0, B, P, v, d = b.place(jb, g_box, 0.3 * thr)
    # ---- add: 1, 2, 3 cached points, 2-3 thresholds from the new vertex (well inside sqrt(thr): a match against thr would take them)
    for n in (1, 2, 3):
        rows = [b.point(B, P, v, d, _perp(d, rng, 2.0 * thr, 3.0 * thr), rng.uniform(0.1, 0.4) * thr, dist=0.3 * thr, imp=_imp(k), life=LIFE[k]) for k in range(n)]
        add("add", "box cache of %d" % n, b.write(s0, jb, rows), jb, (ADD, n, -1, 0, 0, n + 1), (REPLACE, n + 1))
    # ---- replace the nearest
    u1 = _perp(d, rng, 0.4 * thr, 0.4 * thr); u2 = _perp(d, rng, 0.7 * thr, 0.7 * thr)
    if np.linalg.norm(u1 - u2) < 1.1 * thr:
        u2 = -u2
    far = _perp(d, rng, 2.5 * thr, 2.5 * thr)
    rows = [b.point(B, P, v, d, u1, 0.1 * thr, dist=0.2 * thr, imp=_imp(0), life=LIFE[0])]
    add("replace", "box one within the threshold", b.write(s0, jb, rows), jb, (REPLACE, 0, -1, 0, 0, 1), (REPLACE, 1))
    near, other = b.point(B, P, v, d, u1, 0.0, dist=0.2 * thr, imp=_imp(0), life=LIFE[0]), b.point(B, P, v, d, u2, 0.0, dist=0.2 * thr, imp=_imp(1), life=LIFE[1])
    add("replace", "box two within, nearer first", b.write(s0, jb, [near, other]), jb, (REPLACE, 0, -1, 0, 0, 2), (REPLACE, 2))
    add("replace", "box two within, nearer second", b.write(s0, jb, [other, near]), jb, (REPLACE, 1, -1, 0, 0, 2), (REPLACE, 2))
    rows = [b.point(B, P, v, d, _perp(d, rng, 2.0 * thr, 3.0 * thr), 0.2 * thr, dist=0.2 * thr, imp=_imp(k), life=LIFE[k]) for k in range(4)]
    rows[2] = b.point(B, P, v, d, u1, 0.1 * thr, dist=0.2 * thr, imp=_imp(2), life=LIFE[2])
    add("replace", "box one of four within", b.write(s0, jb, rows), jb, (REPLACE, 2, -1, 0, 0, 4), (REPLACE, 4))

    # ---- full cache: every (deepest, replaced) pair on a box, a capsule and a sphere
    for what, j, g in (("box", jb, g_box), ("capsule", jc, cap_g[-1]), ("sphere", L["sphere"], sph_g[L["sphere"]])):
        t = b.thr[j]
        s, Bj, Pj, vj, dj = b.place(j, g, 0.3 * t)
        for deepest in (-1, 0, 1, 2, 3):
            for rep in range(4):
                if rep == deepest:
                    continue
                sf = _full_cache(b, j, s, Bj, Pj, vj, dj, deepest, rep, rng, 0.3 * t)
                add("full", "%s deepest %s replaced %d" % (what, "new" if deepest < 0 else "slot %d" % deepest, rep), sf, j,
                    (FULL, rep, deepest, 0, 0, 4), (REPLACE, 4))

    # ---- refresh without a new point, and removals: the vertex 1.4 thresholds up; kept points at 0.5 thresholds, removed ones 1.3
    # thresholds up (distance) or 1.4 thresholds off their anchor (drift)
    def refresh_rows(Bj, Pj, vj, dj, t, kinds):
        rows = []
        for k, kind in enumerate(kinds):
            u = _perp(dj, rng, 1.5 * t, 3.0 * t)
            h = (1.3 - 1.4) * t if kind == "dist" else (0.5 - 1.4) * t
            drift = (1.4 * t * np.cos(k), 1.4 * t * np.sin(k)) if kind == "drift" else (0.1 * t, 0.0)
            rows.append(b.point(Bj, Pj, vj, dj, u, h, drift=drift, dist=0.5 * t, imp=_imp(k), life=LIFE[k]))
        return rows

    s1, B, P, v, d = b.place(jb, g_box, 1.4 * thr)
    add("refresh", "box two kept", b.write(s1, jb, refresh_rows(B, P, v, d, thr, ["keep", "keep"])), jb, (NONE, -1, -1, 0, 0, 2), (NONE, 2))
    for r in range(1, 5):
        for sub in itertools.combinations(range(4), r):
            for first in ("dist", "drift"):
                kinds = ["keep"] * 4
                alt = (first, "drift" if first == "dist" else "dist")
                for i, k in enumerate(sub):
                    kinds[k] = alt[i % 2]
                rd = sum(1 << k for k in range(4) if kinds[k] == "dist")
                rf = sum(1 << k for k in range(4) if kinds[k] == "drift")
                add("removal", "box %s" % "".join({"keep": ".", "dist": "d", "drift": "f"}[x] for x in kinds),
                    b.write(s1, jb, refresh_rows(B, P, v, d, thr, kinds)), jb, (NONE, -1, -1, rd, rf, 4 - r), (NONE, 4 - r))
    for what, j, g in (("capsule", jc, cap_g[1]), ("sphere", L["sphere"], sph_g[L["sphere"]])):
        t = b.thr[j]
        s, Bj, Pj, vj, dj = b.place(j, g, 1.4 * t)
        for kind in ("dist", "drift"):
            kinds = ["keep", kind, "keep"]
            add("removal", "%s one by %s" % (what, kind), b.write(s, j, refresh_rows(Bj, Pj, vj, dj, t, kinds)), j,
                (NONE, -1, -1, 2 if kind == "dist" else 0, 2 if kind == "drift" else 0, 2), (NONE, 2))

    # ---- contact-fall tolerance: the vertex's new point is the link's only point
    jf, jn = L["fall"], L["nonfall"]
    gf = g_box if jf == jb else b.down(jf)
    gn = g_box if jn == jb else b.down(jn)
    for name, j, g, dist in (("fall link inside the tolerance", jf, gf, 0.6 * TOL), ("fall link between tolerance and threshold", jf, gf, 0.5 * (TOL + b.thr[jf])),
                             ("non-fall link inside the tolerance", jn, gn, 0.6 * TOL)):
        s, *_ = b.place(j, g, dist)
        add("fall", name, s, j, (ADD, 0, -1, 0, 0, 1), (REPLACE, 1))

    # ---- release and re-contact within one launch
    s, B, P, v, d = b.place(jb, g_box, 3.0 * thr)
    rows = []
    for k, kind in enumerate(("dist", "drift", "dist", "drift")):
        u = _perp(d, rng, 1.5 * thr, 3.0 * thr)
        h, drift = (0.2 * thr, (0.0, 0.0)) if kind == "dist" else (-2.5 * thr, (1.5 * thr * np.cos(k), 1.5 * thr * np.sin(k)))
        rows.append(b.point(B, P, v, d, u, h, drift=drift, dist=0.3 * thr, imp=_imp(k), life=LIFE[k]))
    add("release", "box falling from 3 thresholds", b.write(s, jb, rows), jb, (NONE, -1, -1, 0b0101, 0b1010, 0), (NONE, 0))
    return out


def contacts(orc, snap):
    """one Update(1/600) of the oracle from snap: (Oracle.last_contacts() [sub-steps, links, 6], snapshot after)"""
    orc.set_snapshot(snap)
    orc.update(DT)
    return orc.last_contacts(), orc.get_snapshot()
