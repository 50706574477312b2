"""Dataset readers and the prefetching loader without a GPU: a synthetic dataset tree in the reference's layout, read by
``ThreeDMatchPairs`` / ``KittiPairs`` and by the reference's own dataset classes, item by item; the committed slice of the
reference's metadata; the loader's keyed order; and the argument checks of the batched histogram entry point."""
import ctypes
import functools
import os
import pickle
import sys

import numpy as np
import pytest
import torch

from geotransformer_b200 import _lib as L
from geotransformer_b200.datasets.kitti import KittiPairs
from geotransformer_b200.datasets.loader import PrefetchLoader, epoch_order
from geotransformer_b200.datasets.threedmatch import ThreeDMatchPairs, transform_from_rotation_translation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = '/root/reference'
needs_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(REF, 'geotransformer', 'datasets')), reason='reference checkout not present')


def _metadata():
    with open(os.path.join(ROOT, 'tests', 'golden', 'dataset_metadata.pkl'), 'rb') as f:
        return pickle.load(f)


def _tree(tmp_path, n=6):
    """3DMatch and KITTI trees holding the first n pairs of every split of the metadata slice, with small random clouds"""
    meta = _metadata()
    rng = np.random.default_rng(0)
    roots = {}
    for dataset in ('3DMatch', 'Kitti'):
        root = tmp_path / dataset
        (root / 'metadata').mkdir(parents=True)
        for key, entries in meta.items():
            if not key.startswith(dataset + '/'):
                continue
            entries = entries[:n]
            with open(root / 'metadata' / (key.split('/')[1] + '.pkl'), 'wb') as f:
                pickle.dump(entries, f)
            for e in entries:
                for k in ('pcd0', 'pcd1'):
                    pts = rng.normal(size=(int(rng.integers(50, 200)), 3))
                    path = (root / 'data' / e[k]) if dataset == '3DMatch' else (root / e[k])
                    path.parent.mkdir(parents=True, exist_ok=True)
                    if dataset == '3DMatch':
                        torch.save(pts, path)
                    else:
                        np.save(path, pts)
        roots[dataset] = str(root)
    return roots


def _ref_module(name, monkeypatch):
    if REF not in sys.path:
        monkeypatch.syspath_prepend(REF)
    import importlib
    return importlib.import_module(name)


def _equal(got, want):
    assert set(got) == set(want), (set(got) ^ set(want))
    for k, v in want.items():
        if isinstance(v, np.ndarray):
            assert got[k].dtype == v.dtype and np.array_equal(got[k], v), k
        else:
            assert type(got[k]) is type(v) and got[k] == v, k


def test_metadata_fixture_keys_and_transforms():
    meta = _metadata()
    assert sorted(meta) == ['3DMatch/3DLoMatch', '3DMatch/3DMatch', '3DMatch/train', '3DMatch/val', 'Kitti/test', 'Kitti/train',
                            'Kitti/val']
    for key, entries in meta.items():
        assert len(entries) == 32
        for e in entries:
            if key.startswith('3DMatch'):
                assert set(e) == {'pcd0', 'pcd1', 'rotation', 'translation', 'overlap', 'scene_name', 'frag_id0', 'frag_id1'}
                assert e['pcd0'].endswith('.pth') and e['pcd0'].split('/')[1] == e['scene_name']
                T = transform_from_rotation_translation(e['rotation'], e['translation'])
                assert abs(np.linalg.det(T[:3, :3]) - 1) < 1e-2 and np.array_equal(T[3], [0, 0, 0, 1])
            else:
                assert set(e) == {'seq_id', 'frame0', 'frame1', 'pcd0', 'pcd1', 'transform'}
                assert e['pcd0'] == f"downsampled/{e['seq_id']:02d}/{int(e['frame0']):06d}.npy"
                assert e['transform'].shape == (4, 4)


@needs_ref
def test_transform_equals_reference_function(monkeypatch):
    ref = _ref_module('geotransformer.utils.pointcloud', monkeypatch)
    for e in _metadata()['3DMatch/3DLoMatch']:
        want = ref.get_transform_from_rotation_translation(e['rotation'], e['translation'])
        assert np.array_equal(transform_from_rotation_translation(e['rotation'], e['translation']), want)


@needs_ref
@pytest.mark.parametrize('subset', ['train', 'val', '3DMatch', '3DLoMatch'])
@pytest.mark.parametrize('overlap_threshold', [None, 0.2])
def test_threedmatch_reader_equals_reference(tmp_path, monkeypatch, subset, overlap_threshold):
    roots = _tree(tmp_path)
    mod = _ref_module('geotransformer.datasets.registration.threedmatch.dataset', monkeypatch)
    # the reference calls torch.load(path) from before weights_only became the default; its clouds are pickled numpy arrays
    monkeypatch.setattr(mod.torch, 'load', functools.partial(torch.load, weights_only=False))
    want = mod.ThreeDMatchPairDataset(roots['3DMatch'], subset, overlap_threshold=overlap_threshold)
    got = ThreeDMatchPairs(roots['3DMatch'], subset, overlap_threshold=overlap_threshold)
    assert len(got) == len(want) and (len(got) > 0 or overlap_threshold is not None)
    for i in range(len(want)):
        _equal(got[i], want[i])


@needs_ref
@pytest.mark.parametrize('subset', ['train', 'val', 'test'])
def test_kitti_reader_equals_reference(tmp_path, monkeypatch, subset):
    roots = _tree(tmp_path)
    mod = _ref_module('geotransformer.datasets.registration.kitti.dataset', monkeypatch)
    want = mod.OdometryKittiPairDataset(roots['Kitti'], subset)
    got = KittiPairs(roots['Kitti'], subset)
    assert len(got) == len(want) > 0
    for i in range(len(want)):
        _equal(got[i], want[i])


def test_readers_reject_host_side_sampling(tmp_path):
    roots = _tree(tmp_path, n=1)
    with pytest.raises(NotImplementedError):
        ThreeDMatchPairs(roots['3DMatch'], 'train', rotated=True)
    with pytest.raises(NotImplementedError):
        ThreeDMatchPairs(roots['3DMatch'], '3DMatch', point_limit=5000)
    with pytest.raises(NotImplementedError):
        KittiPairs(roots['Kitti'], 'train', point_limit=5000)
    with pytest.raises(ValueError):
        KittiPairs(roots['Kitti'], '3DMatch')


class _Counting:
    def __init__(self, n):
        self.n, self.loads = n, []

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        self.loads.append(i)
        return {'index': i, 'ref_points': np.full((4, 3), i, dtype=np.float32)}


def test_loader_order_is_keyed_by_seed_and_epoch():
    n = 23
    a = PrefetchLoader(_Counting(n), 4, seed=9, pin=False)
    for e in (1, 2):
        order = epoch_order(n, 9, e)
        assert sorted(order.tolist()) == list(range(n))
        steps = list(a.epoch(e))
        assert [len(s) for s in steps] == [4] * 5 + [3] and len(a) == 6
        assert [d['index'] for s in steps for d in s] == order.tolist()
        assert all(isinstance(d['ref_points'], torch.Tensor) and float(d['ref_points'][0, 0]) == d['index'] for s in steps for d in s)
    assert not np.array_equal(epoch_order(n, 9, 1), epoch_order(n, 9, 2))
    assert not np.array_equal(epoch_order(n, 9, 1), epoch_order(n, 10, 1))
    # a resumed run (a new loader, as after a restart) visits epoch 2 exactly as the uninterrupted one, also from a later step
    b = PrefetchLoader(_Counting(n), 4, seed=9, pin=False)
    assert [d['index'] for s in b.epoch(2) for d in s] == epoch_order(n, 9, 2).tolist()
    assert [d['index'] for s in b.epoch(2, start_step=3) for d in s] == epoch_order(n, 9, 2)[12:].tolist()


def test_loader_holds_a_bounded_number_of_steps():
    ds = _Counting(40)
    loader = PrefetchLoader(ds, 2, seed=1, num_threads=2, prefetch_steps=3, pin=False)
    it = loader.epoch(0)
    next(it)
    import time
    time.sleep(0.2)
    assert len(ds.loads) <= 2 * 3      # the step handed out and the ones read ahead
    rest = list(it)
    assert len(rest) == 19 and len(ds.loads) == 40


def test_histogram_batched_rejects_bad_arguments_before_any_launch():
    lib = L.lib()
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf)
    ptrs = (ctypes.c_void_p * 2)(p, p)
    widths = np.array([8, 8], dtype=np.int64)
    rows = np.array([5, 5, 4, 4], dtype=np.int64)

    def call(stages=2, batch=1, hist_n=16, w=widths, r=rows, hists=p):
        return lib.geob200_neighbor_histogram_batched(ptrs, w.ctypes.data, r.ctypes.data, stages, batch, hist_n, 100, hists, p, p, None)
    err = lambda: lib.geob200_last_error().decode()  # noqa: E731
    assert call(stages=0) < 0 and 'num_stages' in err()
    assert call(stages=7) < 0 and 'num_stages' in err()
    assert call(batch=33) < 0 and 'batch' in err()
    assert call(hist_n=0) < 0 and 'hist_n' in err()
    assert call(hists=None) < 0 and 'null' in err()
    assert call(w=np.array([8, 0], dtype=np.int64)) < 0 and 'stage 1' in err()
    assert call(r=np.array([5, 0, 4, 4], dtype=np.int64)) < 0 and 'cloud 1 is empty' in err()
    assert lib.geob200_launch_count() == 0
