"""float64 restatement of the tracking error (deepmimic_b200/csrc/kernels/dm_pose_error.cu, C ABI dm_pose_error) for the tests: pose features
on tests/render_ref.Character's forward kinematics, the frame distance, the phase-locked error and the full DTW recursion."""
import numpy as np

from tests.render_ref import quat_mat


def heading(root_quat):
    """atan2(-x.z, x.x) of the root rotation's image x of (1, 0, 0); root_quat (w, x, y, z)"""
    x = quat_mat(*root_quat)[:, 0]
    return np.arctan2(-x[2], x[0])


def features(ch, pose):
    """[J - 1, 3]: joint k's world origin minus the root's, rotated about y by minus the root's heading, k = 1 .. J - 1"""
    pose = np.asarray(pose, dtype=np.float64)
    Jp = joint_origins(ch, pose)
    h = heading(pose[3:7])
    c, s = np.cos(-h), np.sin(-h)
    d = Jp[1:] - Jp[0]
    return np.stack([c * d[:, 0] + s * d[:, 2], d[:, 1], -s * d[:, 0] + c * d[:, 2]], axis=1)


def joint_origins(ch, pose):
    """[J, 3] joint world origins of a pose row (cKinTree::JointWorldTrans), recovered from render_ref.Character.frames' body frames: a body's
    frame is its joint's frame moved by the body attach point and rotation"""
    R, c = ch.frames(pose)
    JR = R @ np.transpose(np.asarray(ch.body_rot), (0, 2, 1))
    return c - np.einsum("kij,kj->ki", JR, np.asarray(ch.body_pt))


def distance_matrix(fa, fr):
    """d_ij = mean_k |fa[i, k] - fr[j, k]| of feature sequences [L, J - 1, 3]"""
    return np.linalg.norm(fa[:, None] - fr[None, :], axis=3).mean(axis=2)


def dtw(d):
    """D(L-1, L-1) / 2L of D(0, 0) = 2 d_00, D(i, j) = min(D(i-1, j-1) + 2 d_ij, D(i-1, j) + d_ij, D(i, j-1) + d_ij) over a square d"""
    L = d.shape[0]
    D = np.full((L + 1, L + 1), np.inf)
    D[0, 0] = 0.0
    for i in range(L):
        for j in range(L):
            D[i + 1, j + 1] = min(D[i, j] + 2.0 * d[i, j], D[i, j + 1] + d[i, j], D[i + 1, j] + d[i, j])
    return D[L, L] / (2.0 * L)


def errors_of_distances(d):
    """(e_lock, e_dtw) of a square distance matrix"""
    return float(np.mean(np.diag(d))), float(dtw(d))


def errors(ch, a, r):
    """(e_lock, e_dtw) of pose sequences a, r [L, pose_dim]"""
    fa = np.stack([features(ch, p) for p in a])
    fr = np.stack([features(ch, p) for p in r])
    return errors_of_distances(distance_matrix(fa, fr))
