"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/modelnet_rpmnet.npz from the REAL reference: the items of
``ModelNetPairDataset(deterministic=True)`` built as oracle/modelnet_benchmark_vectors.py builds them (same synthetic pkl, same
stubs), with their ``raw_points``, and the reference's numpy metrics (utils/registration.py: compute_modified_chamfer_distance,
compute_transform_mse_and_mae) of every pair under a list of estimates.  Run where the reference checkout exists:
    python -m oracle.rpmnet_metrics_vectors

Two names the reference calls are gone from the installed scipy (1.18) and are restored for the run:
``Rotation.from_dcm = Rotation.from_matrix`` (renamed in scipy 1.4, removed in 1.6) and ``cKDTree.query(n_jobs=...)`` (renamed
``workers`` in 1.6, removed in 1.9), which get_nearest_neighbor passes.  Neither changes a value.
Estimates per pair: identity; the ground truth; small perturbations of it; random rotations; 180-degree rotations; pitches at
and within 1e-7 rad of +-90 degrees (gimbal lock); fp32 products of an SVD (orthogonal to ~1e-7, not 1e-12); and, on pair 0, one
rotation with det < 0 (the reference raises; stored with NaN metrics and flagged).
"""
import os
import pickle
import tempfile

import numpy as np
from scipy.spatial import cKDTree
from scipy.spatial.transform import Rotation

from oracle import modelnet_benchmark_vectors as MV

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD_PATH = os.path.join(ROOT, 'tests', 'golden', 'modelnet_rpmnet.npz')


class _Tree(cKDTree):
    def query(self, x, k=1, n_jobs=None, **kw):
        if n_jobs is not None:
            kw['workers'] = n_jobs
        return super().query(x, k=k, **kw)


def _rt(R, t):
    T = np.eye(4, dtype=np.float32)
    T[:3, :3] = R
    T[:3, 3] = t
    return T


def estimates(gt, rng, with_det_neg):
    """(4, 4) fp32 estimates of one pair"""
    out = [np.eye(4, dtype=np.float32), gt.copy()]
    for s in (1e-4, 1e-2, 0.2):
        dR = Rotation.from_rotvec(rng.standard_normal(3) * s).as_matrix()
        out.append(_rt(dR @ gt[:3, :3].astype(np.float64), gt[:3, 3] + rng.standard_normal(3) * s))
    for _ in range(2):
        out.append(_rt(Rotation.random(random_state=rng).as_matrix(), rng.uniform(-0.5, 0.5, 3)))
    for axis in ([1, 0, 0], [0, 0, 1], [1, 1, 0]):
        out.append(_rt(Rotation.from_rotvec(np.pi * np.asarray(axis) / np.linalg.norm(axis)).as_matrix(), rng.uniform(-0.5, 0.5, 3)))
    for pitch in (np.pi / 2, -np.pi / 2, np.pi / 2 - 5e-8, -np.pi / 2 + 5e-8, np.pi / 2 - 3e-7):
        out.append(_rt(Rotation.from_euler('xyz', [rng.uniform(-3, 3), pitch, rng.uniform(-3, 3)]).as_matrix(), rng.uniform(-0.5, 0.5, 3)))
    for _ in range(2):
        U, _, Vt = np.linalg.svd(rng.standard_normal((3, 3)).astype(np.float32))
        R = (U @ Vt).astype(np.float32)
        if np.linalg.det(R) < 0:
            R = (U @ np.diag(np.float32([1, 1, -1])) @ Vt).astype(np.float32)
        out.append(_rt(R, rng.uniform(-0.5, 0.5, 3)))
    if with_det_neg:
        out.append(_rt(np.diag([1.0, 1.0, -1.0]), np.zeros(3)))
    return [x.astype(np.float32) for x in out]


def main():
    import geotransformer.utils.pointcloud as ref_pc
    import geotransformer.utils.registration as ref_reg
    Rotation.from_dcm = Rotation.from_matrix
    ref_pc.cKDTree = _Tree
    rng = np.random.default_rng(20261018)
    with tempfile.TemporaryDirectory() as root:
        with open(os.path.join(root, 'test.pkl'), 'wb') as f:
            pickle.dump(MV.shapes(), f)
        ds = MV._reference_dataset(root)
        rows = list(ds.data_list)
        out = {k: [] for k in ('shape', 'length', 'raw_points', 'ref_points', 'src_points', 'transform')}
        cases = {k: [] for k in ('pair', 'est', 'metrics', 'raises')}
        for i in range(len(rows)):
            d = ds[i]
            shape = rows[i]['points']
            assert d['raw_points'].dtype == np.float32 and d['raw_points'].shape == shape.shape
            for k in ('raw_points', 'ref_points', 'src_points', 'transform'):
                out[k].append(d[k])
            out['shape'].append(shape)
            out['length'].append(len(shape))
            for est in estimates(d['transform'], rng, i == 0):
                try:
                    cd = ref_reg.compute_modified_chamfer_distance(d['raw_points'], d['ref_points'], d['src_points'], d['transform'], est)
                    m = [cd] + list(ref_reg.compute_transform_mse_and_mae(d['transform'], est))
                    raises = False
                except ValueError:
                    m, raises = [np.nan] * 5, True
                cases['pair'].append(i)
                cases['est'].append(est)
                cases['metrics'].append(np.asarray([float(v) for v in m], np.float64))
                cases['raises'].append(raises)
            print(f'pair {i}: {len(shape)} points, {len(cases["pair"])} cases so far')
    arrays = {k: (np.concatenate(v) if k in ('shape', 'raw_points') else np.stack(v)) for k, v in out.items()}
    arrays['length'] = arrays['length'].astype(np.int64)
    arrays.update({f'case_{k}': np.stack(v) for k, v in cases.items()})
    np.savez_compressed(GOLD_PATH, **arrays)
    print('wrote', GOLD_PATH)


if __name__ == '__main__':
    MV.reference_class()                                  # puts the reference checkout on sys.path
    main()
