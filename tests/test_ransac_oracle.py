"""CPU checks of the RANSAC restatement (oracle/ransac_oracle.py) the GPU tests compare against, and of the argument checks of the
RANSAC / correspondence-metric entry points (rejected before any launch, so no GPU is needed)."""
import ctypes

import numpy as np
import pytest
from scipy import stats
from scipy.spatial.transform import Rotation

from oracle import ransac_oracle as RO


def test_philox_known_answers():
    """Random123's known-answer vectors for philox4x32_10"""
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
              (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in cases:
        got = RO.philox4x32_10(np.array([ctr], dtype=np.uint64), key)[0]
        assert tuple(int(v) for v in got) == want, [hex(int(v)) for v in got]


@pytest.mark.parametrize('n', [3, 7, 100, 1000, 4097])
def test_sampler_is_uniform_with_replacement(n):
    draws = RO.sample_indices(seed=12345, pair=3, n=n, ransac_n=5, num_iterations=max(4000, 20 * n))
    assert draws.min() >= 0 and draws.max() < n
    counts = np.bincount(draws.ravel(), minlength=n)
    p = stats.chisquare(counts).pvalue
    assert p > 1e-4, (n, p)
    # with replacement: repeated indices inside one hypothesis occur at the birthday rate
    rep = np.mean([len(set(r)) < len(r) for r in draws])
    expect = 1.0 - np.prod([(n - j) / n for j in range(5)])
    assert abs(rep - expect) < 0.05 + 0.1 * expect, (rep, expect)


def test_sampler_depends_on_seed_pair_and_iteration_only():
    a = RO.sample_indices(7, 0, 1000, 8, 64)
    assert np.array_equal(a[:10], RO.sample_indices(7, 0, 1000, 8, 10))       # a prefix does not depend on the iteration count
    assert not np.array_equal(a, RO.sample_indices(8, 0, 1000, 8, 64))
    assert not np.array_equal(a, RO.sample_indices(7, 1, 1000, 8, 64))
    assert np.array_equal(a[:, :3], RO.sample_indices(7, 0, 1000, 3, 64))    # the first draws do not depend on ransac_n


def _synthetic(n, inlier_ratio, rng, noise=0.0, scale=1.0):
    R = Rotation.random(random_state=rng).as_matrix()
    t = rng.normal(size=3) * scale
    src = (rng.uniform(-1, 1, size=(n, 3)) * scale).astype(np.float32)
    ref = (src.astype(np.float64) @ R.T + t + rng.normal(size=(n, 3)) * noise).astype(np.float32)
    out = rng.random(n) >= inlier_ratio
    ref[out] = (rng.uniform(-1, 1, size=(int(out.sum()), 3)) * scale).astype(np.float32)
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return src, ref, T, ~out


def test_oracle_recovers_noise_free_transform():
    rng = np.random.default_rng(5)
    src, ref, T, inl = _synthetic(400, 0.10, rng)
    res = RO.ransac(src, ref, 0.05, 3, 3000, seed=1)
    assert res['inliers'] == int(inl.sum())
    assert np.allclose(res['transform'], T, atol=1e-4)
    assert res['fitness'] == pytest.approx(inl.mean(), abs=1e-6)


def test_winner_rule_and_degenerate_cases():
    assert RO.winner([3, 5, 5, 5], [0.1, 0.3, 0.2, 0.2]) == 2
    assert RO.winner([0, 0], [0.0, 0.0]) == -1
    src = np.zeros((2, 3), np.float32)
    res = RO.ransac(src, src, 0.05, 3, 10)
    assert res['iteration'] == -1 and np.array_equal(res['transform'], np.eye(4)) and res['fitness'] == 0.0


def test_entry_points_reject_bad_arguments_before_any_launch():
    from geotransformer_b200 import _lib as L
    lib = L.lib()
    buf = ctypes.create_string_buffer(1 << 20)
    p = ctypes.addressof(buf)

    def ransac(rn=3, iters=100, tau=0.05, pts=p, out=p, ws=1 << 20):
        return lib.geob200_ransac_correspondences_batched(pts, pts, 2, 16, None, tau, rn, iters, 0, 0, out, p, p, p, p, None, None, None, None,
                                                          p, ws, None)

    def err():
        return lib.geob200_last_error().decode()

    before = lib.geob200_launch_count()
    assert ransac(rn=2) < 0 and 'ransac_n' in err()
    assert ransac(rn=9) < 0 and 'ransac_n' in err()
    assert ransac(iters=0) < 0 and 'num_iterations' in err()
    assert ransac(tau=0.0) < 0 and 'distance_threshold' in err()
    assert ransac(tau=-1.0) < 0 and 'distance_threshold' in err()
    assert ransac(pts=None) < 0 and 'null' in err()
    assert ransac(out=None) < 0 and 'null' in err()
    assert ransac(ws=16) < 0 and 'workspace' in err()
    assert lib.geob200_correspondence_metrics_batched(p, p, 2, 16, None, p, 16, 0.0, p, 4, p, 1 << 20, None) < 0 and 'radius' in err()
    assert lib.geob200_correspondence_metrics_batched(p, p, 2, 16, None, None, 16, 0.1, p, 4, p, 1 << 20, None) < 0 and 'output' in err()
    assert lib.geob200_launch_count() == before
