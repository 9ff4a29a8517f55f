"""float64 restatement of the marked renderer (dm_render_marked_kernel, C ABI dm_render_poses_marked) on top of tests/render_ref.py: the same
rays, shapes and shading, plus one sphere in its own colour that is hit after the links, shaded like them, and casts and receives shadows."""
import numpy as np

from tests import render_ref as RR

MARK_RGB = np.array([0.15, 0.75, 0.30])
MARKER = -3


def render_marked(ch, R, c, root_xz, camera, width, height, marker):
    """RR.render with marker (x, y, z, radius; radius <= 0: none): dict(rgb, ids (-3 the marker), shadow, checker, face) as RR.render's"""
    x, y, z, r = (float(v) for v in marker)
    shapes = [(R[k], c[k], ch.shape[k], ch.he[k], k) for k in range(ch.n)]
    if r > 0:
        shapes.append((np.eye(3), np.array([x, y, z]), RR.SPHERE, np.array([r, 0.0, 0.0]), MARKER))
    eye, D = RR.camera_rays(root_xz, camera, width, height)
    D = D.reshape(-1, 3)
    N = D.shape[0]
    tbest, ids, n = np.full(N, np.inf), np.full(N, RR.SKY, dtype=np.int16), np.tile([0.0, 1.0, 0.0], (N, 1))
    face = np.zeros(N, dtype=np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        tg = -eye[1] / D[:, 1]
    g = (D[:, 1] < 0) & (tg > RR.T_MIN)
    tbest[g], ids[g] = tg[g], RR.GROUND
    for Rk, ck, sk, hk, idk in shapes:
        t, nk, fk = RR.hit_link(Rk, ck, sk, hk, eye, D)
        better = t < tbest
        tbest[better], ids[better], n[better], face[better] = t[better], idk, nk[better], fk[better]
    hit = ids != RR.SKY
    P = eye + np.where(hit, tbest, 0.0)[:, None] * D
    checker = np.where(ids == RR.GROUND, (np.floor(P[:, 0]).astype(np.int64) + np.floor(P[:, 2]).astype(np.int64)) & 1, -1)
    base = np.where((ids == RR.GROUND)[:, None], np.where(checker == 1, RR.GROUND_DARK, RR.GROUND_LIGHT)[:, None] * np.ones(3),
                    np.where((ids == MARKER)[:, None], MARK_RGB, RR.CHAR_RGB))
    ndl = n @ RR.LIGHT
    shadow = np.zeros(N, dtype=bool)
    cand = hit & (ndl > 0)
    so = P[cand] + RR.SHADOW_BIAS * n[cand]
    blocked = np.zeros(so.shape[0], dtype=bool)
    for Rk, ck, sk, hk, _ in shapes:
        t, _, _ = RR.hit_link(Rk, ck, sk, hk, so, np.tile(RR.LIGHT, (so.shape[0], 1)))
        blocked |= np.isfinite(t)
    shadow[cand] = blocked
    k = RR.AMBIENT + np.where(cand & ~shadow, RR.DIFFUSE * ndl, 0.0)
    s = np.maximum(D[:, 1], 0.0)[:, None]
    col = np.where(hit[:, None], base * k[:, None], RR.SKY_HORIZON + s * (RR.SKY_ZENITH - RR.SKY_HORIZON))
    rgb = np.rint(255.0 * np.clip(col, 0.0, 1.0)).astype(np.uint8)
    return dict(rgb=rgb.reshape(height, width, 3), ids=ids.reshape(height, width), shadow=shadow.reshape(height, width),
                checker=checker.reshape(height, width), face=face.reshape(height, width))
