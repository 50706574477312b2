"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/modelnet_benchmark.npz from the REAL reference's
``ModelNetPairDataset(deterministic=True)`` (geotransformer/datasets/registration/modelnet/dataset.py) with the options of its val
and test loaders (EXPMN/dataset.py, config.py: num_points 717, keep_ratio 0.7, rotation 45, translation 0.5, noise 0.05, plane
crop, twice_sample, asymmetric classes 'all').  Run where the reference checkout exists:   python -m oracle.modelnet_benchmark_vectors

The dataset reads a seeded synthetic ``test.pkl`` (oracle.modelnet_benchmark_oracle.synthetic_shapes) written to a temporary
directory.  Its debug-only imports that are not installed (open3d, IPython, matplotlib, sklearn) are stubbed; none of them is called
on this path.  Cases:
  * 2 048-point shapes; a 1 024-point shape (crop of exactly 717 points); shapes of 600 .. 1 000 points (crop < 717: padding);
  * a symmetric class (label 5) in the pkl, which the asymmetric filter drops, so later indices differ from their pkl rows;
  * dataset indices 0 .. n-1 of the filtered list, and 2^31 and 2^32 - 1 (served by a list that maps those indices to a shape).
Stored per pair: the raw shape (stacked), the index, the reference's ref_points / src_points / transform, and from the numpy
restatement (checked equal to the reference here) the shape row of every output point and the smallest crop-distance gap.
"""
import os
import pickle
import sys
import tempfile
import types

import numpy as np

from oracle import modelnet_benchmark_oracle as MB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD_PATH = os.path.join(ROOT, 'tests', 'golden', 'modelnet_benchmark.npz')
REF_ROOT = '/root/reference'
OPTIONS = dict(num_points=717, rotation_magnitude=45.0, translation_magnitude=0.5, noise_magnitude=0.05, keep_ratio=0.7)
LARGE_INDICES = ((1 << 31, 0), ((1 << 32) - 1, 3))        # (dataset index, position in the filtered list of the shape it reads)


def shapes():
    """the pkl rows: sizes 2048, 2048 (label 5, dropped), 1024, 800, 2048, 1000, 2048"""
    rows = MB.synthetic_shapes(7, seed=20261017, small_every=0, labels=(0, 5, 1, 2, 3, 4, 7))
    rng = np.random.default_rng(7)
    for i, n in ((2, 1024), (3, 800), (5, 1000)):
        p = (rng.standard_normal((n, 3)) * [0.4, 0.3, 0.25] + rng.uniform(-1, 1, 3)).astype(np.float32)
        rows[i] = {'points': p, 'normals': np.zeros_like(p), 'label': rows[i]['label']}
    return rows


def reference_class():
    """the reference's ModelNetPairDataset; its uninstalled debug-only imports are stubbed for the import and removed afterwards, so
    nothing else in the process sees the stubs"""
    added = []
    for m in ('open3d', 'IPython', 'matplotlib', 'matplotlib.colors', 'matplotlib.pyplot', 'sklearn', 'sklearn.neighbors'):
        if m not in sys.modules:
            mod = types.ModuleType(m)
            mod.embed = lambda *a, **k: None
            mod.NearestNeighbors = object
            sys.modules[m] = mod
            added.append(m)
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    try:
        from geotransformer.datasets.registration.modelnet.dataset import ModelNetPairDataset
    finally:
        for m in added:
            del sys.modules[m]
    return ModelNetPairDataset


def _reference_dataset(root):
    return reference_class()(root, 'test', crop_method='plane', asymmetric=True, class_indices='all', deterministic=True,
                             twice_sample=True, twice_transform=False, return_normals=False, return_occupancy=True, **OPTIONS)


class _Rows:
    """a data_list that also answers the large indices"""

    def __init__(self, rows, extra):
        self.rows, self.extra = rows, extra

    def __getitem__(self, i):
        return self.rows[self.extra.get(i, i)]

    def __len__(self):
        return len(self.rows)


def main():
    with tempfile.TemporaryDirectory() as root:
        with open(os.path.join(root, 'test.pkl'), 'wb') as f:
            pickle.dump(shapes(), f)
        ds = _reference_dataset(root)
        rows = list(ds.data_list)
        ds.data_list = _Rows(rows, dict(LARGE_INDICES))
        cases = [(i, i) for i in range(len(rows))] + list(LARGE_INDICES)
        out = {k: [] for k in ('shape', 'length', 'index', 'ref_points', 'src_points', 'transform', 'ref_origin', 'src_origin', 'gap')}
        for index, pos in cases:
            d = ds[index]
            shape = rows[pos]['points']
            r = MB.benchmark_pair(shape, index, **OPTIONS)
            for k in ('ref_points', 'src_points', 'transform'):
                assert d[k].dtype == np.float32 and np.array_equal(d[k], r[k]), (index, k)
                out[k].append(d[k])
            out['shape'].append(shape)
            out['length'].append(len(shape))
            out['index'].append(index)
            out['ref_origin'].append(r['ref_origin'].astype(np.int32))
            out['src_origin'].append(r['src_origin'].astype(np.int32))
            out['gap'].append(r['gap'])
            print(f'index {index}: {len(shape)} points, crop {MB.crop_count(len(shape), 0.7)}, smallest distance gap {r["gap"]:.3g}')
    arrays = {k: (np.concatenate(v) if k == 'shape' else np.stack(v)) for k, v in out.items()}
    arrays['length'] = arrays['length'].astype(np.int64)
    arrays['index'] = arrays['index'].astype(np.int64)
    arrays['labels'] = np.asarray([r['label'] for r in shapes()], np.int64)
    np.savez_compressed(GOLD_PATH, **arrays)
    print('wrote', GOLD_PATH)


if __name__ == '__main__':
    main()
