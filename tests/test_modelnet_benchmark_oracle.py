"""ModelNet validation / test pairs without a GPU: the numpy restatement (oracle/modelnet_benchmark_oracle.py) against the fixture
written from the reference's own deterministic dataset, the class filter and config values against the reference, the
Python-side option checks, and the argument checks of the C entry point (rejected before any launch)."""
import ctypes
import math
import os

import numpy as np
import pytest

from geotransformer_b200 import _lib as L
from geotransformer_b200.config import make_cfg
from geotransformer_b200.datasets import modelnet as DM
from oracle import modelnet_benchmark_oracle as MB

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'modelnet_benchmark.npz')
REF = '/root/reference'
HAVE_REF = os.path.isdir(os.path.join(REF, 'geotransformer', 'datasets'))
needs_ref = pytest.mark.skipif(not HAVE_REF, reason='reference checkout not present')


def test_restatement_reproduces_the_reference_fixture():
    g = np.load(GOLD)
    starts = np.concatenate([[0], np.cumsum(g['length'])])
    assert {0, (1 << 32) - 1} <= set(g['index'].tolist())
    crops = [MB.crop_count(int(n), 0.7) for n in g['length']]
    assert 2048 in g['length'].tolist() and min(crops) < 717 and 717 in crops
    assert 5 in g['labels'].tolist()                        # a symmetric class: dropped, so indices differ from pkl rows
    for p in range(len(g['length'])):
        r = MB.benchmark_pair(g['shape'][starts[p]:starts[p + 1]], int(g['index'][p]))
        for k in ('ref_points', 'src_points', 'transform', 'ref_origin', 'src_origin'):
            assert np.array_equal(r[k], g[k][p]), (p, k)
        assert r['gap'] == g['gap'][p] and r['gap'] > 1e-9   # every crop in the fixture is decided


def test_restatement_draws_from_the_legacy_stream():
    # a pair is a function of its index alone
    shape = MB.synthetic_shapes(1, seed=5)[0]['points']
    a = MB.benchmark_pair(shape, 11)
    b = MB.benchmark_pair(shape, 11)
    c = MB.benchmark_pair(shape, 12)
    assert all(np.array_equal(a[k], b[k]) for k in a if k != 'gap')
    assert not np.array_equal(a['ref_points'], c['ref_points'])
    # 3 x 716 is even: no Gaussian carries from ref to src, and the pair still has 716 rows per cloud
    d = MB.benchmark_pair(shape, 11, num_points=716)
    assert d['ref_points'].shape == (716, 3) and d['src_points'].shape == (716, 3)


def test_class_filter_and_config():
    assert DM.get_class_indices('all', False) == list(range(40))
    assert DM.get_class_indices('seen', False) == list(range(20))
    assert DM.get_class_indices('unseen', False) == list(range(20, 40))
    assert DM.get_class_indices([5, 0, 39], True) == [0, 39]
    assert len(DM.get_class_indices('all', True)) == 32
    with pytest.raises(ValueError):
        DM.get_class_indices('some', True)
    cfg = make_cfg('modelnet')
    assert cfg.test.noise_magnitude == 0.05 and cfg.test.class_indices == 'all'
    DM.check_options(cfg)
    for group, key, value in (('data', 'twice_sample', False), ('data', 'twice_transform', True), ('data', 'crop_method', 'point'),
                              ('data', 'voxel_size', 0.05), ('data', 'min_overlap', 0.5), ('data', 'max_overlap', 0.9),
                              ('data', 'estimate_normal', True), ('data', 'return_normals', True), ('data', 'overfitting_index', 3),
                              ('test', 'noise_magnitude', None)):
        c = make_cfg('modelnet')
        c[group][key] = value
        with pytest.raises(NotImplementedError):
            DM.check_options(c)


@needs_ref
def test_class_filter_and_config_equal_the_reference():
    from oracle.modelnet_benchmark_vectors import reference_class
    ModelNetPairDataset = reference_class()
    assert tuple(ModelNetPairDataset.ASYMMETRIC_INDICES) == DM.ASYMMETRIC_INDICES
    for ci in ('all', 'seen', 'unseen', [0, 5, 6, 38]):
        for asym in (True, False):
            assert ModelNetPairDataset.get_class_indices(ModelNetPairDataset, ci, asym) == DM.get_class_indices(ci, asym)
    path = os.path.join(REF, 'experiments', 'geotransformer.modelnet.rpmnet.stage4.gse.k3.max.oacl.stage2.sinkhorn', 'config.py')
    src = open(path).read()
    assert '_C.test.noise_magnitude = 0.05' in src and '_C.test.class_indices = "all"' in src


def test_bad_arguments_are_rejected_before_any_launch():
    lib = L.lib()
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.addressof(buf)
    n0 = lib.geob200_launch_count()

    def i64(*v):
        return (ctypes.c_int64 * len(v))(*v)

    def err():
        return lib.geob200_last_error().decode()

    def mnb(B=1, lengths=None, indices=None, m=717, keep=0.7, rot=45.0, tr=0.5, nm=0.05, ws=1 << 16, ptr=p, wsp=p):
        lengths = lengths if lengths is not None else i64(*([2048] * max(B, 1)))
        indices = indices if indices is not None else i64(*range(max(B, 1)))
        return lib.geob200_modelnet_benchmark_pairs_batched(ptr, lengths, indices, B, m, keep, rot, tr, nm, p, p, p, wsp, ws, None)

    assert mnb(B=0) < 0 and 'n_pairs' in err()
    assert mnb(lengths=i64(8193)) < 0 and '8192' in err()
    assert mnb(lengths=i64(0)) < 0 and '8192' in err()
    assert mnb(lengths=i64(1), keep=0.3) < 0 and 'keeps no point' in err()
    assert mnb(indices=i64(-1)) < 0 and 'index' in err()
    assert mnb(indices=i64(1 << 32)) < 0 and 'index' in err()
    assert mnb(m=4097) < 0 and 'num_points' in err()
    assert mnb(m=0) < 0 and 'num_points' in err()
    for bad in (math.nan, math.inf):
        assert mnb(rot=bad) < 0 and 'magnitudes' in err()
        assert mnb(tr=bad) < 0 and 'magnitudes' in err()
        assert mnb(nm=bad) < 0 and 'magnitudes' in err()
        assert mnb(keep=bad) < 0 and 'keep_ratio' in err()
    assert mnb(keep=0.0) < 0 and 'keep_ratio' in err()
    assert mnb(nm=-0.1) < 0 and 'magnitudes' in err()
    assert mnb(ptr=None) < 0 and 'null' in err()
    need = lib.geob200_modelnet_benchmark_pairs_batched_workspace_bytes(1, 717)
    assert mnb(ws=need - 1) < 0 and 'workspace' in err()
    assert mnb(wsp=None) < 0 and 'workspace' in err()
    # the workspace covers one launch: it stops growing at the per-launch pair count
    assert lib.geob200_modelnet_benchmark_pairs_batched_workspace_bytes(5000, 717) == \
        lib.geob200_modelnet_benchmark_pairs_batched_workspace_bytes(1024, 717)
    assert lib.geob200_launch_count() == n0
