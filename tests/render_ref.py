"""float64 restatement of the device renderer (deepmimic_b200/csrc/kernels/dm_render.cu, C ABI dm_render_poses) for the tests: the character's
collision shapes from its file, forward kinematics of pose rows, the camera, the ray casts and the shading, with the kernel's constants
restated here.  Everything in unscaled metres."""
import json
import os

import numpy as np

LIGHT = np.array([1.0, 2.0, 1.0]) / np.sqrt(6.0)
AMBIENT, DIFFUSE = 0.35, 0.65
CHAR_RGB = np.array([0.80, 0.45, 0.25])
GROUND_LIGHT, GROUND_DARK = 0.62, 0.50
SKY_HORIZON, SKY_ZENITH = np.array([0.80, 0.87, 0.95]), np.array([0.40, 0.60, 0.90])
T_MIN, SHADOW_BIAS = 1e-4, 1e-3
BOX, CAPSULE, SPHERE = 1, 2, 3
SKY, GROUND = -1, -2


def euler_mat(tx, ty, tz):
    """rotation of the character file's AttachTheta (x, y, z): Rz Ry Rx"""
    cx, sx, cy, sy, cz, sz = np.cos(tx), np.sin(tx), np.cos(ty), np.sin(ty), np.cos(tz), np.sin(tz)
    return np.array([[cy * cz, sx * sy * cz - cx * sz, cx * sy * cz + sx * sz],
                     [cy * sz, sx * sy * sz + cx * cz, cx * sy * sz - sx * cz],
                     [-sy, sx * cy, cx * cy]])


def quat_mat(w, x, y, z):
    """rotation matrix of a quaternion, normalised first"""
    n = np.sqrt(w * w + x * x + y * y + z * z)
    w, x, y, z = w / n, x / n, y / n, z / n
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


class Character:
    """joints and collision shapes of a character file (Skeleton / BodyDefs): per link parent, joint type, pose offset, attach point and
    rotation of the joint, body attach point and rotation, shape and its extents (box half extents, capsule radius and half height, sphere
    radius)"""

    def __init__(self, asset_root, char_file):
        d = json.load(open(os.path.join(asset_root, char_file)))
        joints, bodies = d["Skeleton"]["Joints"], d["BodyDefs"]
        self.n = len(joints)
        self.parent, self.type, self.pose_off, self.shape = [], [], [], []
        self.att_pt, self.att_rot, self.body_pt, self.body_rot, self.he = [], [], [], [], []
        off = 7
        for j, b in zip(joints, bodies):
            self.parent.append(int(j["Parent"]))
            self.type.append("root" if int(j["Parent"]) < 0 else j["Type"])
            self.pose_off.append(0 if self.type[-1] == "root" else off)
            off += {"root": 0, "spherical": 4, "revolute": 1, "fixed": 0}[self.type[-1]]
            self.att_pt.append(np.array([j["AttachX"], j["AttachY"], j["AttachZ"]], dtype=np.float64))
            self.att_rot.append(euler_mat(j["AttachThetaX"], j["AttachThetaY"], j["AttachThetaZ"]))
            self.body_pt.append(np.array([b["AttachX"], b["AttachY"], b["AttachZ"]], dtype=np.float64))
            self.body_rot.append(euler_mat(b["AttachThetaX"], b["AttachThetaY"], b["AttachThetaZ"]))
            s = {"box": BOX, "capsule": CAPSULE, "sphere": SPHERE}[b["Shape"]]
            p = [float(b["Param0"]), float(b["Param1"]), float(b["Param2"])]
            self.shape.append(s)
            self.he.append(0.5 * np.array(p if s == BOX else ([p[0], p[1], 0.0] if s == CAPSULE else [p[0], 0.0, 0.0])))
        self.pose_dim = off

    def frames(self, pose):
        """link world frames of a pose row (cKinTree::JointWorldTrans, then each body's attach frame): R [links, 3, 3] body -> world, c
        [links, 3] the body origin"""
        pose = np.asarray(pose, dtype=np.float64)
        JR, Jp = [None] * self.n, [None] * self.n
        R, c = np.zeros((self.n, 3, 3)), np.zeros((self.n, 3))
        for k in range(self.n):   # parents come first in a character file
            t, o = self.type[k], self.pose_off[k]
            if t == "root":
                JR[k], Jp[k] = quat_mat(*pose[3:7]), pose[0:3].copy()
            else:
                q = (quat_mat(*pose[o:o + 4]) if t == "spherical" else
                     euler_mat(0.0, 0.0, pose[o]) if t == "revolute" else np.eye(3))
                p = self.parent[k]
                JR[k] = JR[p] @ self.att_rot[k] @ q
                Jp[k] = Jp[p] + JR[p] @ self.att_pt[k]
            R[k] = JR[k] @ self.body_rot[k]
            c[k] = Jp[k] + JR[k] @ self.body_pt[k]
        return R, c


def camera_rays(root_xz, camera, width, height):
    """eye [3] and unit ray directions [height, width, 3] through the pixel centres, row 0 at the top"""
    yaw, pitch, dist, th, fov = (camera[k] for k in ("yaw", "pitch", "distance", "target_height", "fov_y"))
    back = np.array([np.cos(pitch) * np.sin(yaw), np.sin(pitch), np.cos(pitch) * np.cos(yaw)])
    right, fwd = np.array([np.cos(yaw), 0.0, -np.sin(yaw)]), -back
    up = np.cross(right, fwd)
    ty = np.tan(0.5 * fov)
    tx = ty * width / height
    eye = np.array([root_xz[0], th, root_xz[1]]) + dist * back
    sx = (2.0 * (np.arange(width) + 0.5) / width - 1.0) * tx
    sy = (1.0 - 2.0 * (np.arange(height) + 0.5) / height) * ty
    d = fwd[None, None] + sx[None, :, None] * right[None, None] + sy[:, None, None] * up[None, None]
    return eye, d / np.linalg.norm(d, axis=-1, keepdims=True)


def hit_link(R, c, shape, he, O, D):
    """nearest t > T_MIN of rays O + t D ([N, 3] each, or O [3]) with one shape in the frame (R, c): t [N] (inf: none), world normals [N, 3]
    and the face hit [N] (a box's 1 + 2 axis + (normal > 0), 0 on the curved shapes)"""
    D = np.atleast_2d(D)
    lo = np.broadcast_to((np.asarray(O) - c) @ R, D.shape)
    ld = D @ R
    N = D.shape[0]
    t = np.full(N, np.inf)
    nl = np.zeros((N, 3))
    face = np.zeros(N, dtype=np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        if shape == BOX:
            inv = 1.0 / ld
            ta, tb = (-he - lo) * inv, (he - lo) * inv
            tn, tf = np.fmin(ta, tb), np.fmax(ta, tb)
            ax = np.argmax(tn, axis=1)
            t0, t1 = tn[np.arange(N), ax], tf.min(axis=1)
            ok = (t0 <= t1) & (t0 > T_MIN)
            t[ok] = t0[ok]
            nl[np.arange(N), ax] = np.where(ld[np.arange(N), ax] > 0, -1.0, 1.0)
            face = 1 + 2 * ax + (ld[np.arange(N), ax] <= 0)
        else:
            r, h = he[0], (he[1] if shape == CAPSULE else 0.0)
            if shape == CAPSULE:
                a = ld[:, 0] ** 2 + ld[:, 2] ** 2
                b = lo[:, 0] * ld[:, 0] + lo[:, 2] * ld[:, 2]
                cc = lo[:, 0] ** 2 + lo[:, 2] ** 2 - r * r
                disc = b * b - a * cc
                tc = (-b - np.sqrt(np.maximum(disc, 0.0))) / a
                y = lo[:, 1] + tc * ld[:, 1]
                ok = (a > 0) & (disc >= 0) & (tc > T_MIN) & (np.abs(y) <= h)
                t[ok] = tc[ok]
                nl[ok] = np.stack([lo[ok, 0] + tc[ok] * ld[ok, 0], np.zeros(ok.sum()), lo[ok, 2] + tc[ok] * ld[ok, 2]], axis=1)
            for yc in (h, -h):
                oc = lo - np.array([0.0, yc, 0.0])
                b = np.einsum("ij,ij->i", oc, ld)
                disc = b * b - (np.einsum("ij,ij->i", oc, oc) - r * r)
                ts = -b - np.sqrt(np.maximum(disc, 0.0))
                ok = (disc >= 0) & (ts > T_MIN) & (ts < t)
                t[ok] = ts[ok]
                nl[ok] = oc[ok] + ts[ok, None] * ld[ok]
            nl = nl / r
    return t, nl @ R.T, face


def render(ch, R, c, root_xz, camera, width, height):
    """one view of the shapes in frames (R, c) (Character.frames, or a collision pass's frames divided by the world scale): dict(rgb uint8
    [H, W, 3], ids int16 [H, W] (-1 sky, -2 ground, k link k), shadow bool [H, W] (a lit-facing hit whose shadow ray is blocked), checker
    int [H, W] (the ground cell's parity, -1 off the ground), face int [H, W] (hit_link's face of the link hit, 0 elsewhere))"""
    eye, D = camera_rays(root_xz, camera, width, height)
    D = D.reshape(-1, 3)
    N = D.shape[0]
    tbest, ids, n = np.full(N, np.inf), np.full(N, SKY, dtype=np.int16), np.tile([0.0, 1.0, 0.0], (N, 1))
    face = np.zeros(N, dtype=np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        tg = -eye[1] / D[:, 1]
    g = (D[:, 1] < 0) & (tg > T_MIN)
    tbest[g], ids[g] = tg[g], GROUND
    for k in range(ch.n):
        t, nk, fk = hit_link(R[k], c[k], ch.shape[k], ch.he[k], eye, D)
        better = t < tbest
        tbest[better], ids[better], n[better], face[better] = t[better], k, nk[better], fk[better]
    hit = ids != SKY
    P = eye + np.where(hit, tbest, 0.0)[:, None] * D
    checker = np.where(ids == GROUND, (np.floor(P[:, 0]).astype(np.int64) + np.floor(P[:, 2]).astype(np.int64)) & 1, -1)
    base = np.where((ids == GROUND)[:, None], np.where(checker == 1, GROUND_DARK, GROUND_LIGHT)[:, None] * np.ones(3), CHAR_RGB)
    ndl = n @ LIGHT
    shadow = np.zeros(N, dtype=bool)
    cand = hit & (ndl > 0)
    so = P[cand] + SHADOW_BIAS * n[cand]
    blocked = np.zeros(so.shape[0], dtype=bool)
    for k in range(ch.n):
        t, _, _ = hit_link(R[k], c[k], ch.shape[k], ch.he[k], so, np.tile(LIGHT, (so.shape[0], 1)))
        blocked |= np.isfinite(t)
    shadow[cand] = blocked
    k = AMBIENT + np.where(cand & ~shadow, DIFFUSE * ndl, 0.0)
    s = np.maximum(D[:, 1], 0.0)[:, None]
    col = np.where(hit[:, None], base * k[:, None], SKY_HORIZON + s * (SKY_ZENITH - SKY_HORIZON))
    rgb = np.rint(255.0 * np.clip(col, 0.0, 1.0)).astype(np.uint8)
    return dict(rgb=rgb.reshape(height, width, 3), ids=ids.reshape(height, width), shadow=shadow.reshape(height, width),
                checker=checker.reshape(height, width), face=face.reshape(height, width))


def near_boundary(a):
    """True where a pixel or one of its 8 neighbours differs from another pixel of the 3 x 3 block: within one pixel of a boundary of a"""
    H, W = a.shape
    pad = np.pad(a, 1, mode="edge")
    out = np.zeros((H, W), dtype=bool)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            out |= pad[1 + dy:1 + dy + H, 1 + dx:1 + dx + W] != a
    return out
