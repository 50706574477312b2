"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/feature_match.npz from the REAL reference's get_nearest_neighbor
(geotransformer/utils/pointcloud.py:11-22) and extract_corr_indices_from_feats (geotransformer/utils/registration.py:179-212) on
seeded inputs.  Run where the reference checkout exists:   python -m oracle.feature_match_vectors

The reference calls cKDTree.query(q, k=1, n_jobs=-1); scipy >= 1.9 removed ``n_jobs`` (it is ``workers`` now), so the reference's
get_nearest_neighbor raises TypeError on the installed scipy.  The generator therefore restates that one call with workers=-1
(``_get_nearest_neighbor``) and puts it in place of the reference's function inside the reference's registration module; the
correspondence extraction itself is the reference's unmodified code.

Inputs are regenerated from their seeds by ``inputs(name)`` (float32; descriptors L2-normalised like the fine features); stored per
case: nn_dist / nn_index (query -> support), and the (ref, src) index arrays of the plain, mutual and bilateral extraction with
ref = query and src = support.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD_PATH = os.path.join(ROOT, 'tests', 'golden', 'feature_match.npz')

# name -> (rows of the query side, rows of the support side, channels, seed)
CASES = {'points3': (1500, 1300, 3, 101), 'c32': (700, 650, 32, 102), 'c256': (300, 280, 256, 103)}
MODES = ('plain', 'mutual', 'bilateral')


def inputs(name):
    nq, ns, c, seed = CASES[name]
    rng = np.random.default_rng(seed)
    if c == 3:
        q = rng.uniform(-1.5, 1.5, size=(nq, 3)).astype(np.float32)
        s = rng.uniform(-1.5, 1.5, size=(ns, 3)).astype(np.float32)
        return q, s
    base = rng.normal(size=(ns, c))
    s = base / np.linalg.norm(base, axis=1, keepdims=True)
    pick = rng.integers(0, ns, size=nq)
    q = s[pick] + 0.3 * rng.normal(size=(nq, c)) / np.sqrt(c)       # a true partner in the support plus noise
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    return q.astype(np.float32), s.astype(np.float32)


def _get_nearest_neighbor(q_points, s_points, return_index=False):
    from scipy.spatial import cKDTree
    distances, indices = cKDTree(s_points).query(q_points, k=1, workers=-1)
    return (distances, indices) if return_index else distances


def _reference_registration():
    from oracle import ref_harness
    if not ref_harness.available():
        raise RuntimeError('the reference checkout is not available')
    if ref_harness.REF_ROOT not in sys.path:
        sys.path.insert(0, ref_harness.REF_ROOT)
    import geotransformer.utils.registration as reg
    reg.get_nearest_neighbor = _get_nearest_neighbor
    return reg


def make():
    reg = _reference_registration()
    out = {}
    for name in CASES:
        q, s = inputs(name)
        q64, s64 = q.astype(np.float64), s.astype(np.float64)
        d, i = _get_nearest_neighbor(q64, s64, return_index=True)
        out[f'{name}/nn_dist'], out[f'{name}/nn_index'] = np.asarray(d, np.float64), np.asarray(i, np.int64)
        for mode in MODES:
            r, c = reg.extract_corr_indices_from_feats(q64, s64, mutual=mode == 'mutual', bilateral=mode == 'bilateral')
            out[f'{name}/{mode}/ref'], out[f'{name}/{mode}/src'] = np.asarray(r, np.int64), np.asarray(c, np.int64)
    return out


def write(path=GOLD_PATH):
    np.savez_compressed(path, **make())


if __name__ == '__main__':
    write()
    print('wrote', GOLD_PATH)
