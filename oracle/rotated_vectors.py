"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/rotated_3dmatch.npz from the REAL reference: the rotated 3DMatch / 3DLoMatch
benchmark (``ThreeDMatchPairDataset(..., rotated=True)``, datasets/registration/threedmatch/dataset.py) and its evaluation
``experiments/geotransformer.3dmatch.*/eval_dgr.py``.  Run where the reference checkout exists:   python -m oracle.rotated_vectors

The reference never seeds the stream of its rotations; here pair i draws from np.random.seed(i), so the generator seeds the global
generator with the index just before each item, which puts the seed right before the rotated block (no other draw happens in a test
item: point_limit is None and there is no augmentation).

Stored:
  rot/index, rot/R            the reference's random_sample_rotation_v2 for ref then src after np.random.seed(i): (n, 2, 3, 3) fp64
                              for i = 0 .. 255, 2^31-1, 2^31, 2^32-1
  tree/<subset>/metadata      the pickled metadata list of the synthetic tree (uint8), taken from tests/golden/dataset_metadata.pkl
  tree/<subset>/points        every cloud of the subset, stacked in metadata order [pcd0, pcd1 of pair 0, ...]; 3DMatch float64,
                              3DLoMatch float32 (the file dtype: numpy rotates either in fp64), a 1-point cloud included
  tree/<subset>/lengths       their sizes
  item/<subset>/ref_points, src_points (stacked), transform (n, 4, 4): the reference's items after np.random.seed(i)
  dgr/<run>/lines, sparse, corr, reg, est   eval_dgr's eval_one_epoch (verbose, test_epoch None) over oracle.eval_vectors.make_tree's
                              features, in eval_vectors' record layout; reg is every pair's (rre, rte) against the npz transform
"""
import functools
import importlib
import io
import os
import pickle
import sys
import tempfile
import types

import numpy as np

from oracle import eval_vectors as EVV
from oracle import rotated_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD_PATH = os.path.join(ROOT, 'tests', 'golden', 'rotated_3dmatch.npz')
REF_ROOT = '/root/reference'
SEEDS = tuple(range(256)) + ((1 << 31) - 1, 1 << 31, (1 << 32) - 1)
# (subset, cloud dtype, [(ref size, src size), ...])
TREE = (('3DMatch', np.float64, ((300, 250), (1, 120), (80, 400))),
        ('3DLoMatch', np.float32, ((200, 150), (90, 1), (333, 64))))
DGR_RUNS = (('3DMatch', 'lgr', None), ('3DLoMatch', 'lgr', None), ('3DMatch', 'svd', None), ('3DLoMatch', 'svd', None),
            ('3DMatch', 'svd', 1000))
TREE_SEED = 20261018


def dgr_run_name(benchmark, method, num_corr):
    return f'{benchmark}_{method}' + ('' if num_corr is None else f'_k{num_corr}')


def tree_metadata(subset):
    """the first pairs of the committed metadata slice, as many as TREE lists, renamed to fragments 2j, 2j + 1 (one cloud file
    per fragment)"""
    with open(os.path.join(ROOT, 'tests', 'golden', 'dataset_metadata.pkl'), 'rb') as f:
        entries = pickle.load(f)[f'3DMatch/{subset}']
    sizes = dict((s, z) for s, _, z in TREE)[subset]
    out = []
    for j, e in enumerate(entries[:len(sizes)]):
        e = dict(e, frag_id0=2 * j, frag_id1=2 * j + 1)
        e['pcd0'], e['pcd1'] = (f"{subset}/{e['scene_name']}/cloud_bin_{k}.pth" for k in (2 * j, 2 * j + 1))
        out.append(e)
    return out


def tree_clouds():
    """{subset: [cloud, ...]} in metadata order, from TREE_SEED"""
    rng = np.random.default_rng(TREE_SEED)
    out = {}
    for subset, dtype, sizes in TREE:
        out[subset] = [(rng.normal(size=(n, 3)) * [1.2, 0.9, 0.7] + rng.uniform(-2, 2, 3)).astype(dtype) for pair in sizes for n in pair]
    return out


def write_tree(root, metadata, clouds):
    """a 3DMatch tree in the reference's layout: {root}/metadata/{subset}.pkl and the torch.save'd clouds under {root}/data"""
    import torch
    os.makedirs(os.path.join(root, 'metadata'), exist_ok=True)
    for subset, entries in metadata.items():
        with open(os.path.join(root, 'metadata', f'{subset}.pkl'), 'wb') as f:
            pickle.dump(entries, f)
        for e, (c0, c1) in zip(entries, zip(clouds[subset][0::2], clouds[subset][1::2])):
            for name, pts in ((e['pcd0'], c0), (e['pcd1'], c1)):
                path = os.path.join(root, 'data', name)
                os.makedirs(os.path.dirname(path), exist_ok=True)
                torch.save(pts, path)
    return root


def _reference_dataset_class():
    import torch
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    mod = importlib.import_module('geotransformer.datasets.registration.threedmatch.dataset')
    # the reference calls torch.load(path) from before weights_only became the default; its clouds are pickled numpy arrays
    mod.torch.load = functools.partial(torch.load, weights_only=False)
    return mod, mod.ThreeDMatchPairDataset


def run_dgr(tree, benchmark, method, num_corr, out_dir):
    """eval_dgr's eval_one_epoch on the tree's features; returns the stored record of the run"""
    from oracle import ref_harness
    ref_harness.install()
    sys.modules['nibabel'] = nb = types.ModuleType('nibabel')
    nb.quaternions = types.ModuleType('nibabel.quaternions')
    nb.quaternions.mat2quat = EVV.mat2quat
    sys.modules['nibabel.quaternions'] = nb.quaternions
    sys.modules['matplotlib.colors'] = sys.modules['matplotlib'].colors = types.ModuleType('matplotlib.colors')
    import geotransformer.utils.pointcloud as pc
    from scipy.spatial import cKDTree

    class _Tree(cKDTree):
        def query(self, x, k=1, n_jobs=1, **kw):
            return super().query(x, k=k, workers=n_jobs, **kw)
    pc.cKDTree = _Tree
    rcfg, _ = ref_harness.load_experiment('3dmatch')
    exp_dir = os.path.join(ref_harness.REF_ROOT, 'experiments', ref_harness.EXP['3dmatch'])
    sys.modules.pop('eval_dgr', None)
    sys.path.insert(0, exp_dir)
    try:
        ev = importlib.import_module('eval_dgr')
    finally:
        sys.path.remove(exp_dir)
    rec = {k: [] for k in ('sparse', 'corr', 'reg', 'est')}
    ev.evaluate_sparse_correspondences = EVV._recorder(ev.evaluate_sparse_correspondences, rec['sparse'])
    ev.evaluate_correspondences = EVV._recorder(ev.evaluate_correspondences, rec['corr'])
    ev.compute_registration_error = EVV._recorder(ev.compute_registration_error, rec['reg'])
    ev.weighted_procrustes = EVV._recorder(ev.weighted_procrustes, rec['est'])
    # eval_dgr reads <feature_dir>/<benchmark>/epoch-<test_epoch>
    rcfg.feature_dir = os.path.join(out_dir, 'features')
    os.makedirs(os.path.join(rcfg.feature_dir, benchmark), exist_ok=True)
    os.symlink(os.path.join(tree['features'], benchmark), os.path.join(rcfg.feature_dir, benchmark, 'epoch-None'))
    args = types.SimpleNamespace(test_epoch=None, benchmark=benchmark, method=method, num_corr=num_corr, verbose=True)
    logger = EVV._Capture()
    ev.eval_one_epoch(args, rcfg, logger)
    n = len(rec['sparse'])
    assert len(rec['reg']) == n == len([ln for ln in logger.lines if ln.startswith('INFO\t') and ', id0: ' in ln])
    out = {'lines': np.array(logger.lines)}
    out['sparse'] = np.array([[d['precision'], d['recall'], d['hit_ratio']] for d in rec['sparse']], dtype=np.float64)
    out['corr'] = np.array([[d['overlap'], d['inlier_ratio'], d['residual'], d['num_corr']] for d in rec['corr']], dtype=np.float64)
    out['reg'] = np.array(rec['reg'], dtype=np.float64).reshape(n, 2)
    if method == 'svd':
        out['est'] = np.stack([np.asarray(t.detach().cpu().numpy() if hasattr(t, 'detach') else t) for t in rec['est']])
    return out


def build():
    """the golden arrays (needs the reference checkout)"""
    _, Dataset = _reference_dataset_class()
    from geotransformer.utils.pointcloud import random_sample_rotation_v2
    g = {}
    Rs = []
    for s in SEEDS:
        np.random.seed(s)
        Rs.append(np.stack([random_sample_rotation_v2(), random_sample_rotation_v2()]))
    g['rot/index'] = np.array(SEEDS, dtype=np.int64)
    g['rot/R'] = np.stack(Rs)
    metadata = {subset: tree_metadata(subset) for subset, _, _ in TREE}
    clouds = tree_clouds()
    with tempfile.TemporaryDirectory() as tmp:
        root = write_tree(os.path.join(tmp, 'threedmatch'), metadata, clouds)
        for subset, _, _ in TREE:
            buf = io.BytesIO()
            pickle.dump(metadata[subset], buf)
            g[f'tree/{subset}/metadata'] = np.frombuffer(buf.getvalue(), dtype=np.uint8)
            g[f'tree/{subset}/points'] = np.concatenate(clouds[subset])
            g[f'tree/{subset}/lengths'] = np.array([len(c) for c in clouds[subset]], dtype=np.int64)
            ds = Dataset(root, subset, rotated=True)
            items = []
            for i in range(len(ds)):
                np.random.seed(i)
                d = ds[i]
                mine = RO.rotated_pair(clouds[subset][2 * i], clouds[subset][2 * i + 1], np.vstack([
                    np.hstack([metadata[subset][i]['rotation'], metadata[subset][i]['translation'][:, None]]), [0, 0, 0, 1]]), i)
                for k in ('ref_points', 'src_points', 'transform'):
                    assert d[k].dtype == np.float32 and np.array_equal(d[k], mine[k]), (subset, i, k)
                items.append(d)
            for k in ('ref_points', 'src_points'):
                g[f'item/{subset}/{k}'] = np.concatenate([d[k] for d in items])
            g[f'item/{subset}/transform'] = np.stack([d['transform'] for d in items])
        tree = EVV.make_tree(os.path.join(tmp, 'eval_tree'))
        for bench, method, k in DGR_RUNS:
            name = dgr_run_name(bench, method, k)
            res = run_dgr(tree, bench, method, k, os.path.join(tmp, name))
            for key, v in res.items():
                g[f'dgr/{name}/{key}'] = v
    return g


def main():
    from oracle import ref_harness
    assert ref_harness.available(), 'needs the reference checkout'
    g = build()
    for s, R in zip(g['rot/index'], g['rot/R']):
        assert all(np.array_equal(a, b) for a, b in zip(R, RO.rotations(int(s)))), s
    for name in (dgr_run_name(*r) for r in DGR_RUNS):
        print(name, 'lines', len(g[f'dgr/{name}/lines']))
        for ln in g[f'dgr/{name}/lines']:
            if ln.startswith('CRITICAL'):
                print('   ', ln.split('\t', 1)[1])
    np.savez_compressed(GOLD_PATH, **g)
    print(f'wrote {GOLD_PATH} ({os.path.getsize(GOLD_PATH) / 1e3:.1f} kB)')


if __name__ == '__main__':
    sys.path.insert(0, ROOT)
    main()
