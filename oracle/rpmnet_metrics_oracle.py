"""CPU restatement (numpy / scipy) of the ModelNet raw shapes and RPMNet's metrics of geotransformer_b200
(``geob200_modelnet_raw_points_batched``, ``geob200_rpmnet_metrics_batched``; the contract is in DESIGN.md section 8a).

TEST INFRASTRUCTURE ONLY.  tests/test_rpmnet_metrics_oracle.py pins it to tests/golden/modelnet_rpmnet.npz, which
oracle/rpmnet_metrics_vectors.py writes from the reference itself.
  * raw_points: normalize_points in fp32 (numpy's own fp32 mean, norms and division).
  * Chamfer distance: the transforms composed (est gt^-1) and applied in fp64, each coordinate rounded to fp32 once; exact nearest
    neighbours (cKDTree) with fp64 distances; numpy means.
  * Anisotropic errors: scipy's from_matrix written out (det check, Gram test with isclose(atol=1e-12), polar factor U V^T of the
    SVD, Shepperd's quaternion), as_euler('xyz') by the quaternion method with its gimbal rule, unwrapped differences in degrees;
    translations in fp32.
"""
import numpy as np
from scipy.spatial import cKDTree


def raw_points(shape):
    p = np.asarray(shape, np.float32)
    p = p - p.mean(axis=0)
    return p / np.max(np.linalg.norm(p, axis=1))


def _apply64(points, T):
    p = np.asarray(points, np.float32).astype(np.float64)
    return (p @ T[:3, :3].T + T[:3, 3]).astype(np.float32)


def chamfer(raw, ref, src, gt, est):
    """(cd, cd_pq, cd_qp)"""
    gt64, est64 = np.asarray(gt, np.float64), np.asarray(est, np.float64)
    raw = np.asarray(raw, np.float32)
    pq = cKDTree(raw.astype(np.float64)).query(_apply64(src, est64).astype(np.float64), k=1)[0].mean()
    aligned = _apply64(raw, est64 @ np.linalg.inv(gt64))
    qp = cKDTree(aligned.astype(np.float64)).query(np.asarray(ref, np.float32).astype(np.float64), k=1)[0].mean()
    return pq + qp, pq, qp


def from_matrix_quat(M):
    """scipy's Rotation.from_matrix(M).as_quat() (x, y, z, w) for one matrix; ValueError for det <= 0"""
    M = np.asarray(M, np.float64)
    if np.linalg.det(M) <= 0:
        raise ValueError('Non-positive determinant (left-handed or null coordinate frame) in rotation matrix')
    if not np.all(np.isclose(M @ M.T, np.eye(3), atol=1e-12)):
        U, _, Vt = np.linalg.svd(M)
        M = U @ Vt
    tr = M[0, 0] + M[1, 1] + M[2, 2]
    c = int(np.argmax([M[0, 0], M[1, 1], M[2, 2], tr]))
    q = np.empty(4)
    if c == 3:
        q[:] = M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1], 1 + tr
    else:
        i, j, k = c, (c + 1) % 3, (c + 2) % 3
        q[i] = 1 - tr + 2 * M[i, i]
        q[j] = M[j, i] + M[i, j]
        q[k] = M[k, i] + M[i, k]
        q[3] = M[k, j] - M[j, k]
    return q / np.linalg.norm(q)


def euler_xyz(q):
    """as_euler('xyz') in radians of a unit quaternion (x, y, z, w), with scipy's gimbal rule (no warning)"""
    a, b, c, d = q[3] - q[1], q[0] + q[2], q[1] + q[3], q[2] - q[0]
    second = 2 * np.arctan2(np.hypot(c, d), np.hypot(a, b))
    half_sum, half_diff = np.arctan2(b, a), np.arctan2(d, c)
    if abs(second) <= 1e-7:
        e = [2 * half_sum, second, 0.0]
    elif abs(second - np.pi) <= 1e-7:
        e = [-2 * half_diff, second, 0.0]
    else:
        e = [half_sum - half_diff, second, half_sum + half_diff]
    e[1] -= np.pi / 2
    return np.asarray([x + 2 * np.pi if x < -np.pi else (x - 2 * np.pi if x > np.pi else x) for x in e])


def anisotropic(gt, est):
    """(r_mse, r_mae, t_mse, t_mae) of two (4, 4) fp32 transforms"""
    gt, est = np.asarray(gt, np.float32), np.asarray(est, np.float32)
    d = np.rad2deg(euler_xyz(from_matrix_quat(gt[:3, :3]))) - np.rad2deg(euler_xyz(from_matrix_quat(est[:3, :3])))
    t = gt[:3, 3] - est[:3, 3]
    return np.mean(d ** 2), np.mean(np.abs(d)), np.mean(t ** 2), np.mean(np.abs(t))


def metrics(raw, ref, src, gt, est):
    """[cd, cd_pq, cd_qp, r_mse, r_mae, t_mse, t_mae] in float64"""
    return np.asarray(list(chamfer(raw, ref, src, gt, est)) + [float(v) for v in anisotropic(gt, est)], np.float64)
