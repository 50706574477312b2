"""TEST INFRASTRUCTURE ONLY -- ctypes view of ``oracle/_ref/libref_ext.so``.

Presents the two functions of the reference's pybind module ``geotransformer.ext``
(reference ``geotransformer/extensions/pybind.cpp:6-18``) on CPU torch tensors, backed by the
UNMODIFIED reference C++ cores compiled by ``oracle/Makefile``.  Used to (a) pin the C restatement
``oracle/collate_oracle.c``, (b) serve as ``geotransformer.ext`` when the real reference Python is
imported by ``oracle/ref_harness.py``, and (c) time the reference CPU collate in bench.py.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def available():
    return os.path.exists(os.path.join(_HERE, '_ref', 'libref_ext.so'))


def _lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, '_ref', 'libref_ext.so')
        lib = ctypes.CDLL(path)
        lib.ref_grid_subsampling.restype = ctypes.c_int64
        lib.ref_grid_subsampling.argtypes = [
            ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_float,
            ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
        lib.ref_radius_neighbors.restype = ctypes.c_int64
        lib.ref_radius_neighbors.argtypes = [
            ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p,
            ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p, ctypes.c_int64]
        lib.ref_radius_neighbors_search.restype = ctypes.c_int64
        lib.ref_radius_neighbors_search.argtypes = [
            ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p,
            ctypes.c_void_p, ctypes.c_int64, ctypes.c_float]
        lib.ref_radius_neighbors_fetch.restype = ctypes.c_int64
        lib.ref_radius_neighbors_fetch.argtypes = [ctypes.c_void_p, ctypes.c_int64]
        _LIB = lib
    return _LIB


def _check(points, lengths):
    assert points.device.type == 'cpu' and points.dtype == torch.float32 and points.is_contiguous()
    assert lengths.device.type == 'cpu' and lengths.dtype == torch.int64 and lengths.is_contiguous()


def grid_subsampling(points, lengths, voxel_size):
    _check(points, lengths)
    n, b = points.shape[0], lengths.shape[0]
    s_points = torch.zeros((n, 3), dtype=torch.float32)
    s_lengths = torch.zeros((b,), dtype=torch.int64)
    total = _lib().ref_grid_subsampling(points.data_ptr(), n, lengths.data_ptr(), b, float(voxel_size),
                                        s_points.data_ptr(), n, s_lengths.data_ptr())
    return [s_points[:total].clone(), s_lengths]


def radius_neighbors(q_points, s_points, q_lengths, s_lengths, radius):
    _check(q_points, q_lengths)
    _check(s_points, s_lengths)
    nq, ns, b = q_points.shape[0], s_points.shape[0], q_lengths.shape[0]
    # ONE reference search; the table is allocated afterwards and filled from the kept result, as the reference's ATen
    # wrapper does (radius_neighbors.cpp:47-66)
    width = _lib().ref_radius_neighbors_search(q_points.data_ptr(), nq, s_points.data_ptr(), ns, q_lengths.data_ptr(),
                                               s_lengths.data_ptr(), b, float(radius))
    out = torch.empty((nq, width), dtype=torch.int64)
    rc = _lib().ref_radius_neighbors_fetch(out.data_ptr(), nq * width)
    assert rc == 0, 'ref_radius_neighbors_fetch: size mismatch'
    return out


def radius_neighbors_width_only(q_points, s_points, q_lengths, s_lengths, radius):
    """One search, returns only the row width (used for timing a single reference search)."""
    nq, ns, b = q_points.shape[0], s_points.shape[0], q_lengths.shape[0]
    return _lib().ref_radius_neighbors(q_points.data_ptr(), nq, s_points.data_ptr(), ns, q_lengths.data_ptr(),
                                       s_lengths.data_ptr(), b, float(radius), None, 0)
