"""TEST INFRASTRUCTURE ONLY -- ctypes view of ``oracle/liboracle_normals.so``, the C++ restatement of Open3D's normal estimation
(``oracle/normals_oracle.cpp`` states the contract).  ``__graft_entry__.build()`` compiles it with ``build()``."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(_HERE, 'normals_oracle.cpp')
LIB_PATH = os.path.join(_HERE, 'liboracle_normals.so')
_LIB = None

OK, NONFINITE, BAD_ARG = 0, 1, 2


def build():
    """compile liboracle_normals.so: no -ffast-math, no -march=native, no FMA contraction"""
    cxx = os.environ.get('CXX', 'g++')
    if os.path.exists(LIB_PATH) and os.path.getmtime(LIB_PATH) >= os.path.getmtime(SRC):
        return LIB_PATH
    subprocess.check_call([cxx, '-O2', '-std=c++17', '-fPIC', '-shared', '-ffp-contract=off', '-o', LIB_PATH, SRC])
    return LIB_PATH


def _lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            build()
        lib = ctypes.CDLL(LIB_PATH)
        lib.normals_oracle.restype = ctypes.c_int
        lib.normals_oracle.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_double, ctypes.c_void_p,
                                       ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        lib.normals_oracle_eigen.restype = None
        lib.normals_oracle_eigen.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        _LIB = lib
    return _LIB


def estimate_normals(points, knn=30, radius=None, rows=None):
    """one cloud (N, 3) -> (normals (Q, 3) float64, neighbours (Q, knn) int32 with -1 past the count, covariances (Q, 6) float64
    as c00 c01 c02 c11 c12 c22) for the queries ``rows`` (default: every point, Q = N; the brute-force search costs O(N log N) per
    query, so large clouds are checked on a sample); raises ValueError with the error code on an error"""
    p = np.ascontiguousarray(np.asarray(points, dtype=np.float64).reshape(-1, 3))
    n = p.shape[0]
    r = None if rows is None else np.ascontiguousarray(np.asarray(rows, dtype=np.int64).reshape(-1))
    q = n if r is None else r.shape[0]
    out = np.zeros((q, 3), dtype=np.float64)
    nbr = np.zeros((q, knn), dtype=np.int32)
    cov = np.zeros((q, 6), dtype=np.float64)
    rc = _lib().normals_oracle(p.ctypes.data, n, int(knn), 0.0 if radius is None else float(radius),
                               None if r is None else r.ctypes.data, q, out.ctypes.data, nbr.ctypes.data, cov.ctypes.data)
    if rc != OK:
        raise ValueError(f'normals_oracle: error {rc}', rc)
    return out, nbr, cov


def fast_eigen3x3(cov6):
    """FastEigen3x3 of one covariance given as c00 c01 c02 c11 c12 c22"""
    c = np.ascontiguousarray(np.asarray(cov6, dtype=np.float64).reshape(6))
    out = np.zeros(3, dtype=np.float64)
    _lib().normals_oracle_eigen(c.ctypes.data, out.ctypes.data)
    return out


def regularize_normals(points, normals, positive=True):
    """The orientation contract of DESIGN.md section 8a restated column by column in numpy:
    s = (x nx + y ny) + z nz in the type T of points * normals; a row with s < 0 is "towards"; with m = 1 for towards rows and 0
    otherwise, the kept part k = n * T(m) is taken in normals' type and the flipped part f = float64(n) * float64(1 - m) in
    float64; the result is k - f (positive) or f - k, in float64.  Every product of a component with 0 or 1 is exact, so this
    fixes the signs of zeros too: a -0.0 component comes out as +0.0 on either path."""
    p = np.asarray(points)
    n = np.asarray(normals)
    t = np.result_type(p.dtype, n.dtype)
    pc, nc = p.astype(t), n.astype(t)
    s = (pc[:, 0] * nc[:, 0] + pc[:, 1] * nc[:, 1]) + pc[:, 2] * nc[:, 2]
    towards = (s < 0)[:, None]
    kept = n * towards.astype(n.dtype)
    flipped = n.astype(np.float64) * (~towards).astype(np.float64)
    return (kept - flipped) if positive else (flipped - kept)


# ---- the test clouds shared by tests/test_normals_oracle.py (CPU) and tests/test_gpu_normals.py (device) ----

def cases(seed=0):
    """name -> (points (N, 3), knn, radius or None)"""
    rng = np.random.default_rng(seed)
    out = {}
    out['random'] = (rng.uniform(-1, 1, (600, 3)), 30, None)
    out['random_k7'] = (rng.standard_normal((400, 3)), 7, None)
    uv = rng.uniform(-1, 1, (500, 2))
    out['plane_z'] = (np.concatenate([uv, np.full((500, 1), 0.25)], 1), 30, None)           # exact normal (0, 0, +-1)
    out['plane_x'] = (np.concatenate([np.full((300, 1), -2.0), uv[:300]], 1), 16, None)
    t = rng.uniform(0, 1, (200, 1))
    out['collinear'] = (t * np.array([[1.0, 2.0, -0.5]]) + 0.125, 30, None)
    out['three'] = (np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]), 30, None)
    out['two'] = (np.array([[0.0, 0.0, 0.0], [1.0, 0.5, 0.25]]), 30, None)
    out['one'] = (np.array([[3.0, -1.0, 2.0]]), 30, None)
    base = rng.uniform(0, 1, (60, 3))
    out['duplicated'] = (np.concatenate([base, base, base[:20]]), 30, None)
    out['all_same'] = (np.tile([[0.5, 0.25, -1.0]], (40, 1)), 30, None)
    g = np.stack(np.meshgrid(np.arange(6), np.arange(6), np.arange(6), indexing='ij'), -1).reshape(-1, 3).astype(np.float64)
    out['lattice_ties'] = (g * 0.5, 30, None)
    out['lattice_ties_k64'] = (g[rng.permutation(len(g))] * 0.5, 64, None)
    out['diagonal'] = (rng.standard_normal((300, 3)) * np.array([3.0, 1.0, 0.2]), 64, None)   # near-diagonal covariances
    out['axis_cross'] = (np.concatenate([np.stack([np.linspace(-1, 1, 21), np.zeros(21), np.zeros(21)], 1),
                                         np.stack([np.zeros(21), np.linspace(-2, 2, 21), np.zeros(21)], 1),
                                         np.stack([np.zeros(21), np.zeros(21), np.linspace(-3, 3, 21)], 1)]), 5, None)
    out['offset_1e5'] = (rng.uniform(-1, 1, (500, 3)) * np.array([1.0, 1.0, 0.05]) + 1e5, 30, None)
    # the hybrid radius: lattice spacing 0.5, so radius 0.5 excludes the 6 face neighbours (d2 == r2) and 0.5 + 1e-12 takes them
    out['hybrid_at'] = (g * 0.5, 30, 0.5)
    out['hybrid_past'] = (g * 0.5, 30, 0.5 + 1e-12)
    out['hybrid_random'] = (rng.uniform(-1, 1, (800, 3)), 30, 0.3)
    out['float32'] = (rng.uniform(-3, 3, (500, 3)).astype(np.float32), 30, None)
    return out


def ring_scan(rng, n=120000):
    """a KITTI-like scan: 64 elevation rings, ranges 3..80 m, float32"""
    az = rng.uniform(0, 2 * np.pi, n)
    elev = np.deg2rad(rng.integers(0, 64, n) * (28.0 / 64) - 25.0)
    r = rng.uniform(3.0, 80.0, n)
    xyz = np.stack([r * np.cos(az) * np.cos(elev), r * np.sin(az) * np.cos(elev), r * np.sin(elev) + 1.73], 1)
    return xyz.astype(np.float32)


def fragment(rng, n=300000):
    """a 3DMatch-like fragment: three walls and a sphere with 3 mm noise, float64"""
    k = n // 4
    a = np.stack([rng.uniform(0, 3, k), rng.uniform(0, 3, k), np.zeros(k)], 1)
    b = np.stack([np.zeros(k), rng.uniform(0, 3, k), rng.uniform(0, 3, k)], 1)
    c = np.stack([rng.uniform(0, 3, k), np.full(k, 3.0), rng.uniform(0, 3, k)], 1)
    d = rng.standard_normal((n - 3 * k, 3))
    d = d / np.linalg.norm(d, axis=1, keepdims=True) * 0.7 + 1.5
    return np.concatenate([a, b, c, d]) + rng.normal(0, 0.003, (n, 3))
