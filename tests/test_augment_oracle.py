"""Training-data augmentation without a GPU: the numpy restatement (oracle/augment_oracle.py) against the reference's own
augmentation code with its random calls patched to return the restatement's draws, the rotation against scipy, the documented
Philox streams, the config values against the reference's experiment configs, and the argument checks of both entry points
(rejected before any launch)."""
import ast
import ctypes
import math
import os
import random
import sys

import numpy as np
import pytest

from geotransformer_b200 import _lib as L
from geotransformer_b200.config import make_cfg
from oracle import augment_oracle as AO
from oracle import ransac_oracle as RO
from oracle import ref_harness

REF = ref_harness.REF_ROOT
HAVE_REF = os.path.isdir(os.path.join(REF, 'geotransformer', 'datasets'))
needs_ref = pytest.mark.skipif(not HAVE_REF, reason='reference checkout not present')
EXPERIMENTS = {'3dmatch': 'geotransformer.3dmatch.stage4.gse.k3.max.oacl.stage2.sinkhorn',
               'kitti': 'geotransformer.kitti.stage5.gse.k3.max.oacl.stage2.sinkhorn',
               'modelnet': 'geotransformer.modelnet.rpmnet.stage4.gse.k3.max.oacl.stage2.sinkhorn'}


def _ref_import(name):
    if REF not in sys.path:
        sys.path.insert(0, REF)
    import importlib
    return importlib.import_module(name)


class _Draws:
    """stands in for np.random.rand / np.random.uniform / np.random.normal / random.random: returns queued values in call order"""

    def __init__(self, monkeypatch, queue):
        self.queue = list(queue)
        monkeypatch.setattr(np.random, 'rand', self.rand)
        monkeypatch.setattr(np.random, 'uniform', self.uniform)
        monkeypatch.setattr(random, 'random', self.scalar)

    def _pop(self, kind):
        k, v = self.queue.pop(0)
        assert k == kind, (k, kind)
        return v

    def rand(self, *shape):
        v = np.asarray(self._pop('rand'), dtype=np.float64)
        assert v.shape == tuple(shape), (v.shape, shape)
        return v.copy()

    def uniform(self, low=0.0, high=1.0, size=None):
        u = np.asarray(self._pop('uniform'), dtype=np.float64)
        return low + (high - low) * u

    def scalar(self):
        return float(self._pop('random'))


def _cloud(n, seed):
    return np.random.default_rng(seed).normal(size=(n, 3)).astype(np.float32).astype(np.float64)


def _gt(seed):
    rng = np.random.default_rng(seed)
    R = AO.euler_zyx(*rng.uniform(0, 2 * np.pi, 3))
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, rng.normal(size=3)
    return T.astype(np.float32).astype(np.float64)


@needs_ref
@pytest.mark.parametrize('it', [1, 2, 3, 7])
def test_3dmatch_restatement_matches_the_reference(monkeypatch, it):
    mod = _ref_import('geotransformer.datasets.registration.threedmatch.dataset')
    ref, src, T = _cloud(50, it), _cloud(60, it + 100), _gt(it)
    u, R, rot_ref, _, _, _ = AO.pair_draws(AO.THREEDMATCH, 1.0, 1, 1, 0, 7351, it, 0)
    nr, ns = AO.noise_uniforms(np.arange(50), 7351, it, 0, 0), AO.noise_uniforms(np.arange(60), 7351, it, 0, 1)
    _Draws(monkeypatch, [('rand', u[:3]), ('random', u[3]), ('rand', nr), ('rand', ns)])
    ds = mod.ThreeDMatchPairDataset.__new__(mod.ThreeDMatchPairDataset)
    ds.aug_rotation, ds.aug_noise = 1.0, 0.005
    r, s, rot, tr = ds._augment_point_cloud(ref.copy(), src.copy(), T[:3, :3].copy(), T[:3, 3].copy())
    rows_r, rows_s = np.arange(50), np.arange(60)
    want_r = AO.augment_cloud64(ref, rows_r, R, rot_ref, 1.0, np.zeros(3), 0.005, AO.THREEDMATCH, 7351, it, 0, 0)
    want_s = AO.augment_cloud64(src, rows_s, R, not rot_ref, 1.0, np.zeros(3), 0.005, AO.THREEDMATCH, 7351, it, 0, 1)
    np.testing.assert_allclose(r, want_r, rtol=0, atol=1e-12)
    np.testing.assert_allclose(s, want_s, rtol=0, atol=1e-12)
    Tw = AO.compose_transform(T, R, rot_ref, AO.THREEDMATCH, 1.0, np.zeros(3), np.zeros(3))
    np.testing.assert_allclose(rot, Tw[:3, :3], rtol=0, atol=1e-12)
    np.testing.assert_allclose(tr, Tw[:3, 3], rtol=0, atol=1e-12)


@needs_ref
@pytest.mark.parametrize('it', [1, 2, 3, 7])
def test_kitti_restatement_matches_the_reference(monkeypatch, it):
    mod = _ref_import('geotransformer.datasets.registration.kitti.dataset')
    ref, src, T = _cloud(40, it) * 10, _cloud(45, it + 100) * 10, _gt(it)
    u, R, rot_ref, scale, rs, ss = AO.pair_draws(AO.KITTI, 1.0, 0.8, 1.2, 2.0, 11, it, 3)
    nr, ns = AO.noise_uniforms(np.arange(40), 11, it, 3, 0), AO.noise_uniforms(np.arange(45), 11, it, 3, 1)
    _Draws(monkeypatch, [('rand', nr), ('rand', ns), ('rand', u[:3]), ('random', u[3]), ('random', u[4]), ('uniform', u[5:8]),
                         ('uniform', u[8:11])])
    ds = mod.OdometryKittiPairDataset.__new__(mod.OdometryKittiPairDataset)
    ds.augmentation_noise, ds.augmentation_rotation = 0.01, 1.0
    ds.augmentation_min_scale, ds.augmentation_max_scale, ds.augmentation_shift = 0.8, 1.2, 2.0
    r, s, Tr = ds._augment_point_cloud(ref.copy(), src.copy(), T.copy())
    want_r = AO.augment_cloud64(ref, np.arange(40), R, rot_ref, scale, rs, 0.01, AO.KITTI, 11, it, 3, 0)
    want_s = AO.augment_cloud64(src, np.arange(45), R, not rot_ref, scale, ss, 0.01, AO.KITTI, 11, it, 3, 1)
    np.testing.assert_allclose(r, want_r, rtol=0, atol=1e-12)
    np.testing.assert_allclose(s, want_s, rtol=0, atol=1e-12)
    np.testing.assert_allclose(Tr, AO.compose_transform(T, R, rot_ref, AO.KITTI, scale, rs, ss), rtol=0, atol=1e-12)


def _shape(n, seed):
    rng = np.random.default_rng(seed)
    p = rng.normal(size=(n, 3)) * np.array([1.0, 0.6, 0.3])
    return (p + 0.1 * np.sin(3 * p[:, [1, 2, 0]])).astype(np.float32)


@needs_ref
@pytest.mark.parametrize('it', [1, 4])
def test_modelnet_steps_match_the_reference(monkeypatch, it):
    F = _ref_import('geotransformer.transforms.functional')
    PC = _ref_import('geotransformer.utils.pointcloud')
    shape = _shape(2048, it)
    u, R, t, n_ref, n_src = AO.modelnet_draws(45.0, 0.5, 5, it, 0)
    # normalize_points
    norm = AO.normalize(shape)
    np.testing.assert_allclose(F.normalize_points(shape.astype(np.float64)), norm, rtol=0, atol=1e-12)
    # random_sample_transform
    _Draws(monkeypatch, [('rand', u[:3]), ('uniform', u[3:6])])
    Tr = PC.random_sample_transform(45.0, 0.5)
    np.testing.assert_allclose(Tr[:3, :3], R, rtol=0, atol=1e-12)
    np.testing.assert_allclose(Tr[:3, 3], t, rtol=0, atol=1e-12)
    # inverse_transform + apply_transform
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    src = PC.apply_transform(norm, PC.inverse_transform(T))
    want = AO.modelnet_pair(shape, 717, 0.7, 45.0, 0.5, 0.0, seed=5, iteration=it)
    np.testing.assert_allclose(src, want['src_points64'], rtol=0, atol=1e-12)
    # random_sample_plane + random_crop_point_cloud_with_plane (given the restatement's normals)
    _Draws(monkeypatch, [('uniform', u[6]), ('uniform', u[7])])
    np.testing.assert_allclose(F.random_sample_plane(), n_ref, rtol=0, atol=1e-12)
    for pts, nrm in ((norm, n_ref), (src, n_src)):
        got = F.random_crop_point_cloud_with_plane(pts, p_normal=nrm, keep_ratio=0.7)
        rows, _ = AO.crop_rows(pts, nrm, 0.7)
        a, b = got[np.lexsort(got.T)], pts[rows][np.lexsort(pts[rows].T)]
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-12)
    # random_jitter_points with the restatement's normals
    rows = want['ref_origin']
    jit = AO.jitter(rows, 0.05, 5, it, 0, 0)
    z = jit / 0.01
    monkeypatch.setattr(np.random, 'normal', lambda scale=1.0, size=None: scale * z)
    np.testing.assert_allclose(F.random_jitter_points(norm[rows], scale=0.01, noise_magnitude=0.05), norm[rows] + jit, rtol=0,
                               atol=1e-12)


def test_rotation_equals_scipy_from_euler_zyx():
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(0)
    for ang in rng.uniform(0, 2 * np.pi, (200, 3)):
        np.testing.assert_allclose(AO.euler_zyx(*ang), Rotation.from_euler('zyx', ang).as_matrix(), rtol=0, atol=1e-14)


def test_words_use_the_documented_key_and_counter():
    seed, it = (5 << 32) | 77, (3 << 32) | 9
    tags = {AO.tag(s, c) for s in range(1, 6) for c in (0, 1)}
    assert len(tags) == 10 and 0 not in tags                 # the target sampler and RANSAC key with tag 0
    for stream in range(1, 6):
        for cloud in (0, 1):
            w = AO.words(np.arange(4), seed, it, 2, stream, cloud)
            ctr = np.array([[j, 9, 3, 2] for j in range(4)], dtype=np.uint64)
            assert np.array_equal(w, RO.philox4x32_10(ctr, (77, 5 ^ (0xA6000000 | stream << 4 | cloud))))
    u = AO.pair_uniforms(11, seed, it, 2)
    w = AO.words(np.arange(6), seed, it, 2, AO.PAIR, 0).astype(np.int64)
    for i in range(11):
        a, b = w[i // 2, 2 * (i % 2)], w[i // 2, 2 * (i % 2) + 1]
        assert u[i] == ((a >> 5) * 2.0 ** 26 + (b >> 6)) * 2.0 ** -53 and 0.0 <= u[i] < 1.0
    assert np.all(AO.pair_uniforms(4, seed, it, 2)[4:] == 0.0)


def test_point_limit_keeps_distinct_sorted_rows():
    rows = AO.limit_rows(100, 30, 1, 2, 3, 0)
    assert len(rows) == 30 and np.all(np.diff(rows) > 0)
    assert np.array_equal(AO.limit_rows(20, 30, 1, 2, 3, 0), np.arange(20))
    assert not np.array_equal(rows, AO.limit_rows(100, 30, 1, 3, 3, 0))


def _ref_config(name):
    """{'train.point_limit': 30000, ...}: the literal assignments _C.<group>.<key> = <value> of the reference's config.py"""
    src = open(os.path.join(REF, 'experiments', EXPERIMENTS[name], 'config.py')).read()
    out = {}
    for node in ast.walk(ast.parse(src)):
        if isinstance(node, ast.Assign) and len(node.targets) == 1 and isinstance(node.targets[0], ast.Attribute):
            t = node.targets[0]
            if isinstance(t.value, ast.Attribute) and isinstance(t.value.value, ast.Name) and t.value.value.id == '_C':
                try:
                    out[f'{t.value.attr}.{t.attr}'] = ast.literal_eval(node.value)
                except ValueError:
                    pass
    return out


@needs_ref
@pytest.mark.parametrize('name', ['3dmatch', 'kitti', 'modelnet'])
def test_config_values_equal_the_reference(name):
    ref, cfg = _ref_config(name), make_cfg(name)
    keys = [k for k in ref if k.split('.')[0] in ('train', 'data') and k.split('.')[1] in
            ('point_limit', 'use_augmentation', 'augmentation_noise', 'augmentation_rotation', 'augmentation_min_scale',
             'augmentation_max_scale', 'augmentation_shift', 'num_points', 'voxel_size', 'rotation_magnitude', 'translation_magnitude',
             'keep_ratio', 'crop_method', 'asymmetric', 'twice_sample', 'twice_transform', 'noise_magnitude', 'class_indices')]
    assert len(keys) >= 4
    for k in keys:
        group, key = k.split('.')
        assert cfg[group][key] == ref[k], (k, cfg[group][key], ref[k])


def test_bad_arguments_are_rejected_before_any_launch():
    lib = L.lib()
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.addressof(buf)
    n0 = lib.geob200_launch_count()

    def lens(*v):
        return (ctypes.c_int64 * len(v))(*v)

    def err():
        return lib.geob200_last_error().decode()

    def aug(B=1, lengths=None, mode=0, limit=100, noise=0.005, rf=1.0, smin=0.8, smax=1.2, shift=2.0, ws=1 << 16, ptr=p, wsp=p):
        lengths = lengths if lengths is not None else lens(*([50] * (2 * max(B, 1))))
        return lib.geob200_augment_pairs_batched(ptr, lengths, B, p, mode, limit, noise, rf, smin, smax, shift, 1, 1, 0, p, p, p, p, wsp,
                                                 ws, None)

    assert aug(B=0) < 0 and 'pairs' in err()
    assert aug(B=33, lengths=lens(*([50] * 66))) < 0 and 'pairs' in err()
    assert aug(limit=0) < 0 and 'point_limit' in err()
    assert aug(limit=-5) < 0 and 'point_limit' in err()
    assert aug(mode=2) < 0 and 'mode' in err()
    for bad in (math.nan, math.inf):
        assert aug(noise=bad) < 0 and 'noise' in err()
        assert aug(rf=bad) < 0 and 'rotation_factor' in err()
        assert aug(smax=bad) < 0 and 'scale' in err()
        assert aug(shift=bad) < 0 and 'shift' in err()
    assert aug(smin=1.3, smax=1.2) < 0 and 'min_scale' in err()
    assert aug(ptr=None) < 0 and 'null' in err()
    assert aug(lengths=lens(50, 0)) < 0 and 'empty' in err()
    need = lib.geob200_augment_pairs_batched_workspace_bytes(100)
    assert aug(ws=need - 1) < 0 and 'workspace' in err()
    assert aug(wsp=None) < 0 and 'workspace' in err()

    def mn(B=1, lengths=None, m=717, keep=0.7, rot=45.0, tr=0.5, nm=0.05, ws=1 << 16, ptr=p, wsp=p):
        lengths = lengths if lengths is not None else lens(*([2048] * max(B, 1)))
        return lib.geob200_modelnet_pairs_batched(ptr, lengths, B, m, keep, rot, tr, nm, 1, 1, 0, p, p, p, p, wsp, ws, None)

    assert mn(B=0) < 0 and 'pairs' in err()
    assert mn(B=33, lengths=lens(*([2048] * 33))) < 0 and 'pairs' in err()
    assert mn(lengths=lens(8193)) < 0 and '8192' in err()
    assert mn(lengths=lens(1023)) < 0 and 'num_points' in err()          # round(0.7 * 1023) = 716
    assert mn(m=4097, lengths=lens(8192), keep=1.0) < 0 and 'num_points' in err()
    assert mn(m=0) < 0 and 'num_points' in err()
    for bad in (math.nan, math.inf):
        assert mn(rot=bad) < 0 and 'magnitudes' in err()
        assert mn(tr=bad) < 0 and 'magnitudes' in err()
        assert mn(nm=bad) < 0 and 'magnitudes' in err()
        assert mn(keep=bad) < 0 and 'keep_ratio' in err()
    assert mn(ptr=None) < 0 and 'null' in err()
    need = lib.geob200_modelnet_pairs_batched_workspace_bytes(2048)
    assert mn(ws=need - 1) < 0 and 'workspace' in err()
    assert lib.geob200_launch_count() == n0
