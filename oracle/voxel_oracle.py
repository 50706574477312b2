"""TEST INFRASTRUCTURE ONLY -- ctypes view of ``oracle/liboracle_voxel.so``, the C++ restatement of Open3D's voxel downsampling
(``oracle/voxel_oracle.cpp`` states the contract).  ``__graft_entry__.build()`` compiles it with ``build()``."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(_HERE, 'voxel_oracle.cpp')
LIB_PATH = os.path.join(_HERE, 'liboracle_voxel.so')
_LIB = None

# error codes of voxel_oracle(), the same values as the device's GEOB200_VOXEL_* status codes
OK, NONFINITE, TOO_SMALL, AXIS_LIMIT, BAD_SIZE = 0, 1, 2, 3, 4


def build():
    """compile liboracle_voxel.so: no -ffast-math, no -march=native, no FMA contraction"""
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
        lib.voxel_oracle.restype = ctypes.c_int
        lib.voxel_oracle.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_double, ctypes.c_void_p,
                                     ctypes.c_void_p, ctypes.c_void_p]
        lib.voxel_oracle_hash.restype = ctypes.c_uint64
        lib.voxel_oracle_hash.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int]
        lib.voxel_oracle_bucket_growth.restype = ctypes.c_int64
        lib.voxel_oracle_bucket_growth.argtypes = [ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64]
        _LIB = lib
    return _LIB


def voxel_down_sample(points, voxel_size, normals=None):
    """one cloud (N, 3) -> (points (M, 3) float64[, normals (M, 3) float64]); raises ValueError with the error code on an error"""
    p = np.ascontiguousarray(np.asarray(points, dtype=np.float64).reshape(-1, 3))
    nrm = None if normals is None else np.ascontiguousarray(np.asarray(normals, dtype=np.float64).reshape(-1, 3))
    n = p.shape[0]
    out = np.zeros((n, 3), dtype=np.float64)
    out_n = np.zeros((n, 3), dtype=np.float64) if nrm is not None else None
    m = ctypes.c_int64(0)
    rc = _lib().voxel_oracle(p.ctypes.data, None if nrm is None else nrm.ctypes.data, n, float(voxel_size), out.ctypes.data,
                             None if out_n is None else out_n.ctypes.data, ctypes.byref(m))
    if rc != OK:
        raise ValueError(f'voxel_oracle: error {rc}', rc)
    if nrm is None:
        return out[:m.value].copy()
    return out[:m.value].copy(), out_n[:m.value].copy()


def hash_eigen(x, y, z):
    return int(_lib().voxel_oracle_hash(int(x), int(y), int(z)))


def bucket_growth(n_keys):
    """the successive bucket counts of the oracle's map while n_keys distinct voxels are inserted"""
    out = np.zeros(64, dtype=np.uint64)
    w = _lib().voxel_oracle_bucket_growth(int(n_keys), out.ctypes.data, 64)
    return [int(v) for v in out[:min(w, 64)]]
