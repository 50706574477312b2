"""TEST INFRASTRUCTURE ONLY -- a numpy restatement of the rotated 3DMatch / 3DLoMatch benchmark pairs
(``geob200_rotated_pairs_batched``, the reference's ``ThreeDMatchPairDataset(rotated=True)`` with ``np.random.seed(index)`` before
the rotations).

Every rounding is spelled out, so the restatement does not depend on the BLAS numpy links: the norm of ``random_sample_rotation_v2``
is sqrt(fma(a2, a2, fma(a1, a1, a0 a0))), the 3 x 3 products are fma(a2, b2, fma(a1, b1, a0 b0)) per element, the matrix-vector
product is fma(a2, v2, fma(a0, v0, a1 v1)) (OpenBLAS's orders, as numpy 2.3 calls it on x86-64), and the points are
fp32(fma(z, r2, fma(y, r1, x r0))), the (N, 3) x (3, 3) product's order, which equals numpy's fp64 product itself, not only its
rounding to fp32.  tests/test_rotated_oracle.py pins it to the fixture written from the reference itself.  The fused multiply-adds
are exact: the product and sum are formed in rationals and rounded once.

Two forms of the rotation: ``rotations(index)`` calls scipy's ``Rotation.from_euler`` as the reference does, so its half-angle sin
and cos are the host libm's; ``rotations(index, correctly_rounded=True)`` restates scipy's quaternion arithmetic (``euler_zyx``)
with correctly rounded sin and cos (``sincos_cr``), which is what the device computes.  The two differ only where the libm's sin or
cos of a half-angle is not correctly rounded (glibc's are off by just over half an ulp in rare near-tie cases).
"""
import math
from fractions import Fraction

import numpy as np
from scipy.spatial.transform import Rotation

_SCALE_BITS = 1200                       # fixed point below every double's last bit (2^-1074)


def fma(a, b, c):
    return float(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def sincos_cr(x):
    """(sin x, cos x) correctly rounded: Taylor series in integer fixed point at 2^-1200, then one rounding each"""
    one = 1 << _SCALE_BITS
    X = int(Fraction(float(x)) * one)                  # exact: x is a multiple of 2^-1074
    X2 = X * X >> _SCALE_BITS
    s, t, k = X, X, 1
    while t:                                           # each term is off by at most one unit of 2^-1200
        t = -((t * X2 >> _SCALE_BITS) // ((2 * k) * (2 * k + 1)))
        s += t
        k += 1
    c, t, k = one, one, 1
    while t:
        t = -((t * X2 >> _SCALE_BITS) // ((2 * k - 1) * (2 * k)))
        c += t
        k += 1
    return float(Fraction(s, one)), float(Fraction(c, one))


def _compose(p, q):
    """scipy's quaternion product (x, y, z, w), in its order of operations"""
    c0 = p[1] * q[2] - p[2] * q[1]
    c1 = p[2] * q[0] - p[0] * q[2]
    c2 = p[0] * q[1] - p[1] * q[0]
    return [(p[3] * q[0] + q[3] * p[0]) + c0, (p[3] * q[1] + q[3] * p[1]) + c1, (p[3] * q[2] + q[3] * p[2]) + c2,
            p[3] * q[3] - ((p[0] * q[0] + p[1] * q[1]) + p[2] * q[2])]


def euler_zyx(a, b, c, sincos):
    """scipy's Rotation.from_euler('zyx', (a, b, c)).as_matrix() in its own arithmetic, with the given sincos of the half-angles"""
    (sz, cz), (sy, cy), (sx, cx) = sincos(float(a) * 0.5), sincos(float(b) * 0.5), sincos(float(c) * 0.5)
    q = _compose([sx, 0.0, 0.0, cx], _compose([0.0, sy, 0.0, cy], [0.0, 0.0, sz, cz]))
    x2, y2, z2, w2 = q[0] * q[0], q[1] * q[1], q[2] * q[2], q[3] * q[3]
    xy, zw, xz, yw, yz, xw = q[0] * q[1], q[2] * q[3], q[0] * q[2], q[1] * q[3], q[1] * q[2], q[0] * q[3]
    return np.array([[((x2 - y2) - z2) + w2, 2.0 * (xy - zw), 2.0 * (xz + yw)],
                     [2.0 * (xy + zw), ((-x2 + y2) - z2) + w2, 2.0 * (yz - xw)],
                     [2.0 * (xz - yw), 2.0 * (yz + xw), ((-x2 - y2) + z2) + w2]])


def libm_sincos(x):
    """the host C library's sin and cos, which scipy's Rotation calls"""
    return math.sin(x), math.cos(x)


def euler_angles(rs):
    """random_sample_rotation_v2's Euler angles on the RandomState ``rs``: 4 doubles (8 words)"""
    a = rs.random_sample(3) - 0.5
    norm = np.sqrt(fma(a[2], a[2], fma(a[1], a[1], a[0] * a[0])))
    axis = a / norm + 1e-8
    theta = np.pi * rs.random_sample()
    return axis * theta


def rotation_v2(rs, correctly_rounded=False):
    """random_sample_rotation_v2 on the RandomState ``rs``: through scipy (host libm), or the restatement with correctly rounded
    sin / cos"""
    e = euler_angles(rs)
    if correctly_rounded:
        return euler_zyx(e[0], e[1], e[2], sincos_cr)
    return Rotation.from_euler('zyx', e).as_matrix()


def rotations(index, correctly_rounded=False):
    """(R_ref, R_src) of dataset index ``index``: np.random.seed(index), then two rotations"""
    rs = np.random.RandomState(index)
    r = rotation_v2(rs, correctly_rounded)
    return r, rotation_v2(rs, correctly_rounded)


def matmul3(A, B):
    return np.array([[fma(A[i, 2], B[2, j], fma(A[i, 1], B[1, j], A[i, 0] * B[0, j])) for j in range(3)] for i in range(3)])


def matvec3(A, v):
    return np.array([fma(A[i, 2], v[2], fma(A[i, 0], v[0], A[i, 1] * v[1])) for i in range(3)])


def rotate(points, R):
    """fp32(points R^T): fma(z, R[i,2], fma(y, R[i,1], x R[i,0])) in fp64"""
    p = np.asarray(points, dtype=np.float64)
    out = np.array([[fma(z, R[i, 2], fma(y, R[i, 1], x * R[i, 0])) for i in range(3)] for x, y, z in p]).reshape(-1, 3)
    return out.astype(np.float32)


def rotated_pair(ref_points, src_points, transform, index, correctly_rounded=False, given_rotations=None):
    """{'ref_points', 'src_points', 'transform' (fp32), 'rotations' (2, 3, 3) fp64} of the pair of dataset index ``index``.
    ``given_rotations``: (R_ref, R_src) to use instead of the draws (e.g. the device's own record, which pins every product order
    independently of sin and cos)."""
    R_ref, R_src = rotations(index, correctly_rounded) if given_rotations is None else (np.asarray(given_rotations[0]), np.asarray(given_rotations[1]))
    T = np.asarray(transform, dtype=np.float64)
    rotation = matmul3(matmul3(R_ref, T[:3, :3]), R_src.T)
    out = np.eye(4)
    out[:3, :3], out[:3, 3] = rotation, matvec3(R_ref, T[:3, 3])
    return {'ref_points': rotate(ref_points, R_ref), 'src_points': rotate(src_points, R_src), 'transform': out.astype(np.float32),
            'rotations': np.stack([R_ref, R_src])}
