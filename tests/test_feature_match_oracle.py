"""CPU checks of the feature-matching restatement (oracle/feature_ransac_oracle.py) the GPU tests compare against, of the
reference fixture tests/golden/feature_match.npz, and of the argument checks of the feature-matching entry points (rejected before
any launch, so no GPU is needed)."""
import ctypes

import numpy as np
import pytest

from oracle import feature_match_vectors as V
from oracle import feature_ransac_oracle as FO
from oracle import ref_harness

GOLD = np.load(V.GOLD_PATH)


@pytest.mark.parametrize('name', list(V.CASES))
def test_restatement_nearest_neighbor_equals_the_fixture(name):
    q, s = V.inputs(name)
    d, i = FO.nearest_neighbor(q, s)
    assert np.array_equal(i, GOLD[f'{name}/nn_index'])
    assert np.abs(d - GOLD[f'{name}/nn_dist']).max() <= 1e-12 * max(1.0, np.abs(d).max())


@pytest.mark.skipif(not ref_harness.available(), reason='needs the reference checkout')
def test_generator_reproduces_the_fixture():
    fresh = V.make()
    assert set(fresh) == set(GOLD.files)
    for k, v in fresh.items():
        assert v.dtype == GOLD[k].dtype and np.array_equal(v, GOLD[k]), k


def test_edge_check_boundary():
    """exactly 0.9 passes (the checker rejects only d < 0.9 d'), just below fails, in either direction"""
    s = np.array([[0, 0, 0], [9, 0, 0], [0, 0, 0]], np.float32)
    t = np.array([[0, 0, 0], [10, 0, 0], [0, 0, 0]], np.float32)       # 9 = 0.9 * 10 exactly in double
    assert FO.edge_check(s, t) and FO.edge_check(t, s)
    s2 = s.copy()
    s2[1, 0] = np.float32(8.99)
    assert not FO.edge_check(s2, t) and not FO.edge_check(t, s2)


def test_distance_check_boundary():
    """a residual of exactly tau passes, a larger one fails"""
    s = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    t = s.copy()
    t[0, 2] = 0.5                                                        # residual 0.5 under the identity
    R, tr = np.eye(3), np.zeros(3)
    assert FO.distance_check(R, tr, s, t, 0.5)
    assert not FO.distance_check(R, tr, s, t, 0.4999)


def test_validated_prefix():
    flags = np.zeros(50, bool)
    flags[[3, 7, 8, 20, 41]] = True
    assert list(FO.validated(flags, 3)) == [3, 7, 8]
    assert list(FO.validated(flags, 1000)) == [3, 7, 8, 20, 41]       # fewer than V pass: all of them
    assert len(FO.validated(np.zeros(10, bool), 5)) == 0


def _pair(n, rng, C=16):
    src = rng.uniform(-1, 1, size=(n, 3)).astype(np.float32)
    feats = rng.normal(size=(n, C)).astype(np.float32)
    return src, src.copy(), feats, feats.copy()


def test_default_results():
    rng = np.random.default_rng(4)
    src, ref, sf, rf = _pair(40, rng)
    for kw in (dict(ransac_n=2), dict(tau=0.0), dict(tau=-1.0), dict(num_iterations=0), dict(val_iterations=0)):
        args = dict(tau=0.05, ransac_n=3, num_iterations=50, val_iterations=10)
        args.update(kw)
        out = FO.ransac_features(src, ref, sf, rf, args['tau'], args['ransac_n'], args['num_iterations'], args['val_iterations'])
        assert out['iteration'] == -1 and np.array_equal(out['transform'], np.eye(4)) and out['fitness'] == 0.0, kw
        assert out['inlier_rmse'] == 0.0 and out['num_validated'] == 0
    # nothing validates: every sample edge is 3x longer in ref than in src
    out = FO.ransac_features(src, ref * 3, sf, rf, 0.05, 3, 30, 10)
    assert out['num_validated'] == 0 and out['iteration'] == -1 and np.array_equal(out['transform'], np.eye(4))


def test_restatement_recovers_identity_pairing():
    """descriptors equal on both sides: every match is right, so the first passing sample already fits all points"""
    rng = np.random.default_rng(9)
    src, ref, sf, rf = _pair(200, rng)
    out = FO.ransac_features(src, ref, sf, rf, 0.02, 3, 40, 5)
    assert out['num_validated'] == 5 and out['inliers'] == 200 and out['iteration'] == out['val_ids'][0]
    assert np.allclose(out['transform'], np.eye(4), atol=1e-5)


def test_entry_points_reject_bad_arguments_before_any_launch():
    from geotransformer_b200 import _lib as L
    lib = L.lib()
    buf = ctypes.create_string_buffer(1 << 20)
    p = ctypes.addressof(buf)

    def err():
        return lib.geob200_last_error().decode()

    def nn(C=32, q=p, out=p, cap=16, pairs=2, ws=1 << 20, sd=None):
        return lib.geob200_feature_nn_batched(q, p, pairs, cap, 16, C, None, None, out, p, None, sd, p, ws, None)

    def ransac(rn=3, iters=100, val=10, C=32, pts=p, out=p, cap=16, ws=1 << 20):
        return lib.geob200_ransac_features_batched(pts, p, p, p, 2, cap, 16, C, None, None, 0.05, rn, iters, val, 0, 0, out, p, p, p, p, p,
                                                   None, None, None, None, None, None, None, p, ws, None)

    before = lib.geob200_launch_count()
    assert nn(C=0) < 0 and 'channels' in err()
    assert nn(C=1025) < 0 and 'channels' in err()
    assert nn(q=None) < 0 and 'null' in err()
    assert nn(out=None) < 0 and 'null' in err()
    assert nn(sd=p) < 0 and 'null' in err()
    assert nn(cap=-1) < 0 and 'capacities' in err()
    assert nn(pairs=0) < 0 and 'pairs' in err()
    assert nn(ws=16) < 0 and 'workspace' in err()
    assert ransac(rn=9) < 0 and 'ransac_n' in err()
    assert ransac(rn=-1) < 0 and 'ransac_n' in err()
    assert ransac(iters=-1) < 0 and 'num_iterations' in err()
    assert ransac(val=-1) < 0 and 'val_iterations' in err()
    assert ransac(C=0) < 0 and 'channels' in err()
    assert ransac(C=1025) < 0 and 'channels' in err()
    assert ransac(cap=-5) < 0 and 'capacities' in err()
    assert ransac(pts=None) < 0 and 'null' in err()
    assert ransac(out=None) < 0 and 'null' in err()
    assert ransac(ws=16) < 0 and 'workspace' in err()
    assert lib.geob200_feature_corr_indices(p, p, p, p, 4, 4, 3, p, p, None, p, None) < 0 and 'mode' in err()
    assert lib.geob200_feature_corr_indices(p, p, None, None, 4, 4, 1, p, p, None, p, None) < 0 and 'null' in err()
    assert lib.geob200_feature_corr_indices(p, p, p, p, -1, 4, 0, p, p, None, p, None) < 0 and 'counts' in err()
    assert lib.geob200_launch_count() == before
    assert lib.geob200_feature_nn_batched_workspace_bytes(8, 20000, 20000) > 8 * 20000 * 4
    assert lib.geob200_ransac_features_batched_workspace_bytes(8, 5000, 5000, 50000, 1000) > 8 * 50000 * 48
