"""The voxel downsampling oracle (oracle/voxel_oracle.cpp) against numpy and a step-by-step model of libstdc++'s unordered_map, and
the argument checks of geob200_voxel_down_sample (no GPU needed)."""
import ctypes

import numpy as np
import pytest

from geotransformer_b200 import _lib as L
from oracle import voxel_oracle as VO

MASK = (1 << 64) - 1
GROWTH = [13, 29, 59, 127, 257, 541, 1109, 2357, 5087, 10273, 20753, 42043, 85229, 172933]


def hash_eigen_py(k):
    seed = 0
    for v in k:
        seed ^= ((v & MASK) + 0x9e3779b9 + ((seed << 6) & MASK) + (seed >> 2)) & MASK
    return seed


def voxel_indices(p, v):
    lo = p.min(0) - 0.5 * v
    return np.floor((p - lo) / v).astype(np.int64)


def numpy_restatement(p, v, normals=None):
    """group by exact triple (first-occurrence order), sequential double sums in input order, division by the count"""
    k = voxel_indices(p, v)
    groups = {}
    for i, t in enumerate(tuple(int(x) for x in row) for row in k):
        groups.setdefault(t, []).append(i)
    keys = list(groups)
    pts = np.zeros((len(keys), 3))
    nrm = np.zeros((len(keys), 3))
    for g, t in enumerate(keys):
        s, sn = np.zeros(3), np.zeros(3)
        for i in groups[t]:
            s = s + p[i]
            if normals is not None:
                sn = sn + normals[i]
        pts[g] = s / float(len(groups[t]))
        nrm[g] = sn / float(len(groups[t]))
    return keys, pts, nrm


def libstdcxx_order(hashes):
    """node list of a default-constructed std::unordered_map after inserting keys 0..m-1 (bucket hashes ``hashes``) by operator[]:
    a node goes to the front of its bucket's group, or to the list front when its bucket is empty; a rehash (before insertion
    number GROWTH[p] + 1) re-inserts the nodes in list order by the same rule"""
    def insert(lst, e, nb):
        b = hashes[e] % nb
        for pos, x in enumerate(lst):
            if hashes[x] % nb == b:
                lst.insert(pos, e)
                return
        lst.insert(0, e)

    lst, phase = [], 0
    for e in range(len(hashes)):
        if e == GROWTH[phase]:
            phase += 1
            old, lst = lst, []
            for x in old:
                insert(lst, x, GROWTH[phase])
        insert(lst, e, GROWTH[phase])
    return lst


@pytest.mark.parametrize('case', ['uniform', 'negative', 'far', 'float32'])
def test_oracle_equals_numpy_restatement_and_libstdcxx_order(case):
    rng = np.random.default_rng(11)
    p = rng.random((3000, 3)) * 2.0
    v = 0.25
    if case == 'negative':
        p = p - 5.0
    elif case == 'far':
        p = p + 1e5
    elif case == 'float32':
        p = p.astype(np.float32).astype(np.float64)
    normals = rng.standard_normal((p.shape[0], 3))
    got_p, got_n = VO.voxel_down_sample(p, v, normals)
    keys, want_p, want_n = numpy_restatement(p, v, normals)
    assert got_p.shape == want_p.shape and len(keys) > 541       # past six bucket growths
    order = libstdcxx_order([hash_eigen_py(t) for t in keys])
    assert np.array_equal(got_p, want_p[order])                  # bitwise: array_equal on float64 compares values exactly
    assert np.array_equal(got_n, want_n[order])
    assert np.array_equal(VO.voxel_down_sample(p, v), got_p)


def test_hash_eigen_hand_values():
    """seed = 0; seed ^= size_t(k) + 0x9e3779b9 + (seed << 6) + (seed >> 2) for x, y, z, in uint64 (values worked out by hand)"""
    c = 0x9e3779b9
    s1 = c                                    # x = 0: 0 ^ (0 + c + 0 + 0)
    s2 = s1 ^ (c + (s1 << 6) + (s1 >> 2))     # y = 0
    s3 = s2 ^ (c + (s2 << 6) + (s2 >> 2))     # z = 0
    assert s3 == 0xa16fb581eee
    assert VO.hash_eigen(0, 0, 0) == 0xa16fb581eee
    assert VO.hash_eigen(1, 2, 3) == 0xa16fb58d153
    assert VO.hash_eigen(2097151, 2097151, 2097151) == 0xa14f3722e81
    assert VO.hash_eigen(-1, 7, 9) == 0xa16fb5830b1          # size_t(-1) wraps
    for k in [(0, 0, 0), (1, 2, 3), (5, 0, 1 << 20)]:
        assert VO.hash_eigen(*k) == hash_eigen_py(k)


def test_oracle_map_grows_like_libstdcxx_prime_policy():
    assert VO.bucket_growth(172934) == GROWTH + [351061]
    assert VO.bucket_growth(13) == [13]
    assert VO.bucket_growth(14) == [13, 29]


def test_oracle_errors_and_empty_cloud():
    assert VO.voxel_down_sample(np.zeros((0, 3)), 0.3).shape == (0, 3)
    for p, v, code in [(np.zeros((2, 3)), 0.0, VO.BAD_SIZE), (np.array([[0, 0, np.nan]]), 0.3, VO.NONFINITE),
                       (np.array([[0, 0, 0], [0, 0, np.inf]]), 0.3, VO.NONFINITE),
                       (np.array([[0.0, 0, 0], [1e9, 0, 0]]), 1e-9, VO.TOO_SMALL),
                       (np.array([[0.0, 0, 0], [3e6, 0, 0]]), 1.0, VO.AXIS_LIMIT)]:
        with pytest.raises(ValueError) as e:
            VO.voxel_down_sample(p, v)
        assert e.value.args[1] == code


def test_voxel_abi_rejects_bad_arguments_before_any_launch():
    lib = L.lib()
    lens = np.array([3, 2], dtype=np.int64)
    big = np.ones(65, dtype=np.int64)
    ws_bytes = lib.geob200_voxel_down_sample_workspace_bytes(5, 2)
    assert ws_bytes > 5 * 100
    buf = ctypes.create_string_buffer(ws_bytes)
    p = ctypes.addressof(buf)
    launches = lib.geob200_launch_count()

    def call(points=p, normals=None, n=5, lengths=lens.ctypes.data, batch=2, voxel=0.3, out=p, out_n=None, out_len=p, ws=p,
             nbytes=ws_bytes):
        return lib.geob200_voxel_down_sample(points, normals, n, lengths, batch, voxel, out, out_n, out_len, ws, nbytes, None)

    def err():
        return lib.geob200_last_error().decode()

    assert call(batch=65, lengths=big.ctypes.data, n=65) < 0 and 'batch must be in 1..64' in err()
    assert call(batch=0) < 0 and 'batch' in err()
    assert call(voxel=0.0) < 0 and 'voxel size' in err()
    assert call(voxel=-1.0) < 0 and 'voxel size' in err()
    assert call(voxel=float('nan')) < 0 and 'voxel size' in err()
    assert call(lengths=None) < 0 and 'null lengths' in err()
    assert call(out_len=None) < 0 and 'null lengths' in err()
    assert call(points=None) < 0 and 'null point' in err()
    assert call(out=None) < 0 and 'null point' in err()
    assert call(normals=p) < 0 and 'both' in err()
    assert call(n=6) < 0 and 'sum(lengths)' in err()
    assert call(nbytes=ws_bytes - 1) < 0 and 'workspace too small' in err()
    assert call(ws=None) < 0 and 'workspace too small' in err()
    neg = np.array([6, -1], dtype=np.int64)
    assert call(lengths=neg.ctypes.data) < 0 and 'negative length' in err()
    assert lib.geob200_launch_count() == launches
