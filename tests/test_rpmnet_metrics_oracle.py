"""The numpy restatement of the ModelNet raw shapes and RPMNet's metrics (oracle/rpmnet_metrics_oracle.py) against the fixture
written from the reference (tests/golden/modelnet_rpmnet.npz, oracle/rpmnet_metrics_vectors.py).  CPU only.

Bounds (DESIGN.md section 8a): raw_points bit for bit; Chamfer distance within 2e-6 (the reference's aligned coordinates are fp32
BLAS products, the contract's are fp64 rounded once); r_mse / r_mae within 1e-9 relative (LAPACK's SVD against another polar
factor, libm's atan2); t_mse / t_mae bit for bit."""
import os

import numpy as np
import pytest

from oracle import rpmnet_metrics_oracle as O

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'modelnet_rpmnet.npz')
CD_TOL = 2e-6
R_TOL = 1e-9


def _gold():
    g = np.load(GOLD)
    st = np.concatenate([[0], np.cumsum(g['length'])])
    return g, st


def test_raw_points_are_the_references():
    g, st = _gold()
    assert 600 <= g['length'].min() and g['length'].max() == 2048
    for i in range(len(g['length'])):
        assert np.array_equal(O.raw_points(g['shape'][st[i]:st[i + 1]]), g['raw_points'][st[i]:st[i + 1]]), i


def test_metrics_match_the_reference_within_the_bounds():
    g, st = _gold()
    n = 0
    for p, est, want, raises in zip(g['case_pair'], g['case_est'], g['case_metrics'], g['case_raises']):
        args = (g['raw_points'][st[p]:st[p + 1]], g['ref_points'][p], g['src_points'][p], g['transform'][p], est)
        if raises:
            with pytest.raises(ValueError):
                O.metrics(*args)
            continue
        got = O.metrics(*args)
        assert abs(got[0] - want[0]) <= CD_TOL, (p, got[0], want[0])
        assert abs(got[1] + got[2] - got[0]) <= 1e-15
        np.testing.assert_allclose(got[3:5], want[1:3], rtol=R_TOL, atol=1e-12)
        assert got[5] == want[3] and got[6] == want[4]
        n += 1
    assert n >= 100 and g['case_raises'].sum() == 1


def test_cases_cover_the_gimbal_and_non_orthogonal_inputs():
    g, _ = _gold()
    R = g['case_est'][:, :3, :3].astype(np.float64)
    gram = np.abs(R @ R.transpose(0, 2, 1) - np.eye(3)).max(axis=(1, 2))
    assert (gram > 1e-12).sum() > 50                  # fp32 rotations: the polar-factor branch
    pitch = np.arcsin(np.clip(-R[:, 2, 0], -1, 1))
    assert (np.abs(np.abs(pitch) - np.pi / 2) <= 1e-7).sum() >= 12
    assert (np.linalg.det(R) < 0).sum() == 1


def test_gimbal_rule_sets_the_third_angle_to_zero():
    from scipy.spatial.transform import Rotation
    import warnings
    for e in ([0.3, np.pi / 2, 0.2], [-1.0, -np.pi / 2, 0.5], [0.1, 0.2, 0.3], [2.0, -0.4, -3.0]):
        M = Rotation.from_euler('xyz', e).as_matrix()
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            want = Rotation.from_matrix(M).as_euler('xyz')
        np.testing.assert_allclose(O.euler_xyz(O.from_matrix_quat(M)), want, atol=1e-12)
