"""The normal-estimation oracle (oracle/normals_oracle.cpp) against an independent numpy / scipy restatement of the contract in
DESIGN.md section 8a: neighbour sets against cKDTree with ties broken by index, covariances bit for bit against numpy cumulants,
normals against np.linalg.eigh up to sign wherever the two smallest eigenvalues are separated, and the degenerate cases; the
restatement of regularize_normals bit for bit against the reference's own function (when its checkout is present)."""
import os
import sys

import numpy as np
import pytest
from scipy.spatial import cKDTree

from oracle import normals_oracle as NO
from oracle import ref_harness

CASES = NO.cases()


def _numpy_neighbors(p, knn, radius):
    """ascending (d2, index) with d2 = ((dx dx) + dy dy) + dz dz in numpy (no FMA); -1 past the count"""
    n = p.shape[0]
    out = np.full((n, knn), -1, dtype=np.int32)
    for i in range(n):
        d = p[i] - p
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        order = np.lexsort((np.arange(n), d2))[:min(knn, n)]
        if radius is not None:
            order = order[d2[order] < radius * radius]
        out[i, :len(order)] = order
    return out


def _numpy_covariances(p, nbr):
    """nine cumulants added neighbour by neighbour from 0, divided by the count, E[ab] - E[a] E[b]"""
    n, k = nbr.shape
    c = np.zeros((n, 9))
    cnt = (nbr >= 0).sum(1)
    for t in range(k):
        ok = nbr[:, t] >= 0
        q = p[np.where(ok, nbr[:, t], 0)]
        x, y, z = q[:, 0], q[:, 1], q[:, 2]
        for j, v in enumerate((x, y, z, x * x, x * y, x * z, y * y, y * z, z * z)):
            c[ok, j] = c[ok, j] + v[ok]
    has = cnt > 0
    c[has] = c[has] / cnt[has, None].astype(np.float64)
    cov = np.stack([c[:, 3] - c[:, 0] * c[:, 0], c[:, 4] - c[:, 0] * c[:, 1], c[:, 5] - c[:, 0] * c[:, 2],
                    c[:, 6] - c[:, 1] * c[:, 1], c[:, 7] - c[:, 1] * c[:, 2], c[:, 8] - c[:, 2] * c[:, 2]], 1)
    cov[~has] = 0.0
    return cov


def _full(c):
    return np.array([[c[0], c[1], c[2]], [c[1], c[3], c[4]], [c[2], c[4], c[5]]])


def separated(cov6):
    """the two smallest eigenvalues differ by at least 1e-6 of the largest magnitude"""
    w = np.linalg.eigvalsh(_full(cov6))
    return w[1] - w[0] >= 1e-6 * max(abs(w).max(), 1e-300)


@pytest.mark.parametrize('name', sorted(CASES))
def test_oracle_matches_numpy_restatement(name):
    pts, knn, radius = CASES[name]
    p = np.asarray(pts, dtype=np.float64)
    normals, nbr, cov = NO.estimate_normals(pts, knn, radius)
    want = _numpy_neighbors(p, knn, radius)
    assert np.array_equal(nbr, want)
    # the neighbour sets against cKDTree: the distances of the first min(knn, N) neighbours
    if radius is None:
        kk = min(knn, p.shape[0])
        dist, _ = cKDTree(p).query(p, k=kk)
        dist = dist.reshape(p.shape[0], kk)
        mine = np.sqrt(((p[:, None, :] - p[nbr[:, :kk]]) ** 2).sum(-1))
        assert np.allclose(np.sort(mine, 1), dist, rtol=0, atol=1e-9 * max(1.0, np.abs(p).max()))
    else:
        tree = cKDTree(p)
        for i in range(0, p.shape[0], 37):
            inside = set(tree.query_ball_point(p[i], radius * (1 - 1e-9)))
            got = set(int(v) for v in nbr[i] if v >= 0)
            if len(inside) <= knn:
                assert inside <= got, i
    assert np.array_equal(cov, _numpy_covariances(p, nbr))
    # normals: unit, and eigh's smallest eigenvector up to sign where the eigen-gap condition holds
    cnt = (nbr >= 0).sum(1)
    for i in range(p.shape[0]):
        if cnt[i] < 3:
            assert normals[i].tolist() == [0.0, 0.0, 1.0], i
            continue
        if np.all(_full(cov[i]) == 0):
            assert normals[i].tolist() == [0.0, 0.0, 1.0], i
            continue
        assert abs(np.linalg.norm(normals[i]) - 1) < 1e-12, (i, normals[i])
        if separated(cov[i]):
            w, v = np.linalg.eigh(_full(cov[i]))
            e = v[:, 0]
            assert min(np.abs(normals[i] - e).max(), np.abs(normals[i] + e).max()) < 1e-9, (i, normals[i], e)


def test_exact_planes():
    """on an axis-aligned plane the off-axis components are exactly 0 and the axis component is +-1 up to the rounding of the
    final division by sqrt(d)"""
    for name, ax in (('plane_z', 2), ('plane_x', 0)):
        p, knn, _ = CASES[name]
        normals, _, _ = NO.estimate_normals(p, knn)
        others = [a for a in range(3) if a != ax]
        assert np.all(normals[:, others] == 0.0), name
        assert np.abs(np.abs(normals[:, ax]) - 1.0).max() <= 4.5e-16, name


def test_degenerate_cases():
    # fewer than 3 neighbours
    for name in ('two', 'one'):
        normals, _, _ = NO.estimate_normals(CASES[name][0])
        assert np.all(normals == np.array([0.0, 0.0, 1.0]))
    # a zero covariance: FastEigen3x3 returns 0, so the normal is (0, 0, 1)
    normals, _, cov = NO.estimate_normals(CASES['all_same'][0])
    assert np.all(cov == 0) and np.all(normals == np.array([0.0, 0.0, 1.0]))
    # a 3-point cloud: the plane's normal
    normals, _, _ = NO.estimate_normals(CASES['three'][0])
    assert np.all(normals[:, :2] == 0.0) and np.abs(np.abs(normals[:, 2]) - 1.0).max() <= 4.5e-16
    # the empty cloud
    normals, nbr, cov = NO.estimate_normals(np.zeros((0, 3)))
    assert normals.shape == (0, 3) and nbr.shape == (0, 30)
    # a non-finite coordinate is an error
    for bad in (np.nan, np.inf, -np.inf):
        p = np.zeros((5, 3))
        p[3, 1] = bad
        with pytest.raises(ValueError):
            NO.estimate_normals(p)


def test_eigensolver_branches():
    """the diagonal branch (norm == 0) picks the smallest diagonal entry, (0, 0, 1) on ties; the trigonometric branch returns a
    unit vector of the smallest eigenvalue"""
    assert NO.fast_eigen3x3([3, 0, 0, 1, 0, 2]).tolist() == [0.0, 1.0, 0.0]
    assert NO.fast_eigen3x3([1, 0, 0, 3, 0, 2]).tolist() == [1.0, 0.0, 0.0]
    assert NO.fast_eigen3x3([2, 0, 0, 2, 0, 2]).tolist() == [0.0, 0.0, 1.0]
    assert NO.fast_eigen3x3([1, 0, 0, 1, 0, 3]).tolist() == [0.0, 0.0, 1.0]
    assert NO.fast_eigen3x3([0, 0, 0, 0, 0, 0]).tolist() == [0.0, 0.0, 0.0]
    rng = np.random.default_rng(3)
    for _ in range(200):
        m = rng.standard_normal((3, 3))
        a = m @ m.T
        c = [a[0, 0], a[0, 1], a[0, 2], a[1, 1], a[1, 2], a[2, 2]]
        e = NO.fast_eigen3x3(c)
        w, v = np.linalg.eigh(a)
        assert abs(np.linalg.norm(e) - 1) < 1e-12
        if w[1] - w[0] >= 1e-6 * abs(w).max():
            assert min(np.abs(e - v[:, 0]).max(), np.abs(e + v[:, 0]).max()) < 1e-9


def test_hybrid_radius_boundary():
    """d2 < radius^2 is strict: on a 0.5 lattice radius 0.5 leaves only the point itself, 0.5 + 1e-12 adds the face neighbours"""
    p = CASES['hybrid_at'][0]
    _, nbr_at, _ = NO.estimate_normals(p, 30, 0.5)
    _, nbr_past, _ = NO.estimate_normals(p, 30, 0.5 + 1e-12)
    assert np.all((nbr_at >= 0).sum(1) == 1)
    inner = np.all((p > 0) & (p < 2.5), 1)
    assert np.all((nbr_past >= 0).sum(1)[inner] == 7)


# ---- regularize_normals: the restatement against the reference's own function (when its checkout is present) ----

REF = ref_harness.REF_ROOT
HAVE_REF = os.path.isfile(os.path.join(REF, 'geotransformer', 'utils', 'pointcloud.py'))
needs_ref = pytest.mark.skipif(not HAVE_REF, reason='reference checkout not present')


def _ref_pointcloud():
    if REF not in sys.path:
        sys.path.insert(0, REF)
    import importlib
    return importlib.import_module('geotransformer.utils.pointcloud')


def _orientation_inputs(p_dtype, n_dtype, seed=11):
    """random rows plus signed zeros, zero dot products and orthogonal point / normal pairs"""
    rng = np.random.default_rng(seed)
    p = rng.standard_normal((5000, 3))
    n = rng.standard_normal((5000, 3))
    n[:50] = [0.0, -0.0, 0.0]
    n[50:100] = [-0.0, -0.0, -0.0]
    p[100:150] = 0.0
    n[150:200, 2] = -0.0
    p[200:250] = [1.0, 0.0, 0.0]
    n[200:250] = [0.0, 1.0, -0.0]
    p[250:300] = -0.0
    return p.astype(p_dtype), n.astype(n_dtype)


TYPES = [(np.float32, np.float32), (np.float64, np.float64), (np.float32, np.float64), (np.float64, np.float32)]


@needs_ref
@pytest.mark.parametrize('p_dtype,n_dtype', TYPES)
@pytest.mark.parametrize('positive', [True, False])
def test_regularize_restatement_matches_the_reference(p_dtype, n_dtype, positive):
    ref = _ref_pointcloud()
    p, n = _orientation_inputs(p_dtype, n_dtype)
    want = ref.regularize_normals(p, n, positive=positive)
    got = NO.regularize_normals(p, n, positive)
    assert got.dtype == want.dtype == np.float64
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))   # signed zeros included


@pytest.mark.parametrize('p_dtype,n_dtype', TYPES)
def test_regularize_drop_in_types(p_dtype, n_dtype):
    """the drop-in takes the dot products in numpy's type of points * normals and returns float64"""
    from geotransformer_b200.utils.pointcloud import regularize_type
    assert regularize_type(p_dtype, n_dtype) == np.result_type(p_dtype, n_dtype)
    p, n = _orientation_inputs(p_dtype, n_dtype)
    assert NO.regularize_normals(p, n).dtype == np.float64


def test_regularize_restatement_orients():
    """positive: every normal with a nonzero dot product ends up facing the origin (p . n < 0); negative: facing away"""
    p, n = _orientation_inputs(np.float64, np.float64)
    s = np.einsum('ij,ij->i', p, n)
    pos, neg = NO.regularize_normals(p, n, True), NO.regularize_normals(p, n, False)
    nz = s != 0
    assert np.all(np.einsum('ij,ij->i', p, pos)[nz] < 0) and np.all(np.einsum('ij,ij->i', p, neg)[nz] > 0)
    assert np.array_equal(np.abs(pos), np.abs(n)) and np.array_equal(pos, -neg)
