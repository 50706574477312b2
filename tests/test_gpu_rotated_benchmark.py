"""The rotated 3DMatch / 3DLoMatch benchmark on the device (``functional.rotated_pairs_batched``, ``ThreeDMatchPairs(rotated=True)``,
``test --rotated``) and the eval_dgr evaluation (``evaluate(protocol='dgr')``) against the reference's rotations, items and
eval_dgr runs (tests/golden/rotated_3dmatch.npz, written by oracle/rotated_vectors.py) and the numpy restatement
(oracle/rotated_oracle.py).

Every device result is compared bit for bit.  The device evaluates the half-angles' sin and cos correctly rounded; the reference
takes them from the host libm, which is correctly rounded except in rare near-tie cases.  So the device's rotation record equals
the restatement with correctly rounded sin / cos on every seed, and the reference's record on every seed where the two restatements
agree (tests/test_rotated_oracle.py pins which seeds of the fixture those are, and why)."""
import io
import os
import pickle
import re

import numpy as np
import pytest
import torch

from geotransformer_b200 import functional as GF
from geotransformer_b200 import test as test_driver
from geotransformer_b200 import trainval
from geotransformer_b200.datasets.threedmatch import ThreeDMatchPairs, transform_from_rotation_translation
from geotransformer_b200.evaluate import evaluate
from geotransformer_b200.synth import make_pair
from oracle import eval_vectors as EVV
from oracle import rotated_oracle as RO
from oracle import rotated_vectors as RV

pytestmark = pytest.mark.gpu

GOLD = np.load(RV.GOLD_PATH)
DEV = 'cuda'


def _call(clouds, indices, transforms):
    """clouds: [ref_0, src_0, ref_1, ...] host arrays of one dtype; returns host (ref list, src list, T, rotations)"""
    B = len(indices)
    stacked = clouds[0::2] + clouds[1::2]
    lengths = [len(c) for c in stacked]
    pts = torch.from_numpy(np.concatenate(stacked)).to(DEV)
    out, T, rot = GF.rotated_pairs_batched(pts, lengths, indices, np.asarray(transforms, dtype=np.float64))
    rows = np.split(out.cpu().numpy(), np.cumsum(lengths)[:-1])
    return rows[:B], rows[B:], T.cpu().numpy(), rot.cpu().numpy()


def _golden_tree(subset):
    meta = pickle.load(io.BytesIO(GOLD[f'tree/{subset}/metadata'].tobytes()))
    lengths = GOLD[f'tree/{subset}/lengths']
    return meta, np.split(GOLD[f'tree/{subset}/points'], np.cumsum(lengths)[:-1])


def _golden_items(subset):
    lengths = GOLD[f'tree/{subset}/lengths']
    ref = np.split(GOLD[f'item/{subset}/ref_points'], np.cumsum(lengths[0::2])[:-1])
    src = np.split(GOLD[f'item/{subset}/src_points'], np.cumsum(lengths[1::2])[:-1])
    return ref, src, GOLD[f'item/{subset}/transform']


def _transforms(meta):
    return [transform_from_rotation_translation(e['rotation'], e['translation']) for e in meta]


def _rotations_of(index, count, seed=0):
    rng = np.random.default_rng(seed)
    clouds = [rng.normal(size=(1, 3)).astype(np.float32) for _ in range(2 * count)]
    return _call(clouds, index, np.tile(np.eye(4), (count, 1, 1)))[3].reshape(count, 2, 3, 3)


def test_rotations_are_bit_identical_for_every_seed():
    index = [int(i) for i in GOLD['rot/index']]
    rot = _rotations_of(index, len(index))                                         # 259 pairs: five launches
    libm_rounded = 0
    for p, i in enumerate(index):
        cr = np.stack(RO.rotations(i, correctly_rounded=True))
        assert np.array_equal(rot[p], cr), i
        if np.array_equal(cr, GOLD['rot/R'][p]):
            assert np.array_equal(rot[p], GOLD['rot/R'][p]), i
        else:
            libm_rounded += 1                       # the host libm's sin / cos of a half-angle is not correctly rounded here
    assert libm_rounded <= 6, libm_rounded


def test_rotations_are_correctly_rounded_on_random_seeds():
    """2 048 random indices over 0 .. 2^32-1: the device's draws, norm and correctly rounded sin / cos, bit for bit"""
    index = [int(i) for i in np.random.default_rng(11).integers(0, 1 << 32, 2048)]
    rot = _rotations_of(index, len(index))
    for p, i in enumerate(index):
        assert np.array_equal(rot[p], np.stack(RO.rotations(i, correctly_rounded=True))), i


@pytest.mark.parametrize('subset', ['3DMatch', '3DLoMatch'])
def test_items_are_bit_identical_to_the_reference(subset):
    meta, clouds = _golden_tree(subset)
    ref, src, T, rot = _call(clouds, list(range(len(meta))), _transforms(meta))
    want_ref, want_src, want_T = _golden_items(subset)
    assert any(len(c) == 1 for c in clouds)                                       # the ragged batch holds a 1-point cloud
    for i in range(len(meta)):
        assert ref[i].dtype == np.float32 and np.array_equal(ref[i], want_ref[i]), (subset, i)
        assert np.array_equal(src[i], want_src[i]), (subset, i)
        assert np.array_equal(T[i], want_T[i]), (subset, i)
        # the product orders alone: the restatement from the device's own rotations
        mine = RO.rotated_pair(clouds[2 * i], clouds[2 * i + 1], _transforms(meta)[i], i, given_rotations=rot[i])
        assert np.array_equal(mine['ref_points'], ref[i]) and np.array_equal(mine['src_points'], src[i])
        assert np.array_equal(mine['transform'], T[i])


def test_one_call_equals_per_pair_calls_above_the_launch_limit():
    """150 ragged pairs (three launches) in one call equal 150 one-pair calls and the numpy restatement, bit for bit"""
    rng = np.random.default_rng(3)
    B = 150
    clouds = [(rng.normal(size=(int(rng.integers(1, 9)), 3)) * 3).astype(np.float32) for _ in range(2 * B)]
    indices = [int(i) for i in rng.integers(0, 1 << 32, B)]
    Ts = [transform_from_rotation_translation(RO.rotations(1000 + p)[0], rng.uniform(-2, 2, 3)) for p in range(B)]
    ref, src, T, rot = _call(clouds, indices, Ts)
    for p in range(B):
        r1, s1, T1, rot1 = _call(clouds[2 * p:2 * p + 2], [indices[p]], Ts[p:p + 1])
        assert np.array_equal(r1[0], ref[p]) and np.array_equal(s1[0], src[p]) and np.array_equal(T1[0], T[p])
        assert np.array_equal(rot1[0], rot[p])
        want = RO.rotated_pair(clouds[2 * p], clouds[2 * p + 1], Ts[p], indices[p], correctly_rounded=True)
        assert np.array_equal(want['ref_points'], ref[p]) and np.array_equal(want['src_points'], src[p]), p
        assert np.array_equal(want['transform'], T[p]) and np.array_equal(want['rotations'], rot[p].reshape(2, 3, 3)), p


def test_dataset_items_equal_the_reference_items(tmp_path):
    metadata, clouds = {}, {}
    for subset, _, _ in RV.TREE:
        metadata[subset], clouds[subset] = _golden_tree(subset)
    root = RV.write_tree(str(tmp_path / '3dm'), metadata, clouds)
    for subset, _, _ in RV.TREE:
        ds = ThreeDMatchPairs(root, subset, rotated=True)
        want_ref, want_src, want_T = _golden_items(subset)
        batch = ds.rotated_batch(range(len(ds)))
        for i in range(len(ds)):
            d = ds[i]
            assert d['ref_points'].dtype == np.float32 and np.array_equal(d['ref_points'], want_ref[i]), (subset, i)
            assert np.array_equal(d['src_points'], want_src[i]) and np.array_equal(d['transform'], want_T[i]), (subset, i)
            assert d['ref_feats'].shape == (len(want_ref[i]), 1) and d['scene_name'] == metadata[subset][i]['scene_name']
            assert batch[i]['ref_points'].is_cuda and np.array_equal(batch[i]['ref_points'].cpu().numpy(), want_ref[i])
            assert np.array_equal(batch[i]['transform'].cpu().numpy(), want_T[i])


def _threedmatch_tree(root, splits):
    """demo-size pairs in one real scene, float64 clouds"""
    os.makedirs(os.path.join(root, 'metadata'), exist_ok=True)
    for split, indices in splits.items():
        meta = []
        for j, i in enumerate(indices):
            pair = make_pair('demo2k', i)
            names = []
            for k, key in enumerate(('ref_points', 'src_points')):
                name = f'{split}/7-scenes-redkitchen/cloud_bin_{2 * j + k}.pth'
                os.makedirs(os.path.join(root, 'data', os.path.dirname(name)), exist_ok=True)
                torch.save(pair[key].astype(np.float64), os.path.join(root, 'data', name))
                names.append(name)
            T = pair['transform'].astype(np.float64)
            meta.append({'pcd0': names[0], 'pcd1': names[1], 'rotation': T[:3, :3], 'translation': T[:3, 3], 'overlap': 0.5,
                         'scene_name': '7-scenes-redkitchen', 'frag_id0': 2 * j, 'frag_id1': 2 * j + 1})
        with open(os.path.join(root, 'metadata', f'{split}.pkl'), 'wb') as f:
            pickle.dump(meta, f)
    return root


def test_rotated_test_driver_writes_rotated_npz_that_dgr_scores(tmp_path):
    model = trainval.build_model(trainval.make_cfg('3dmatch'), 5, torch.device('cuda', torch.cuda.current_device()))
    snap = str(tmp_path / '3dmatch.pth.tar')
    torch.save({'model': model.state_dict()}, snap)
    root = _threedmatch_tree(str(tmp_path / '3dm'), {'3DMatch': range(3)})
    out = str(tmp_path / 'out')
    test_driver.main(['--config', '3dmatch', '--benchmark', '3DMatch', '--snapshot', snap, '--dataset-root', root, '--output-dir', out,
                      '--neighbor-limits', 'config', '--rotated'])
    scene = os.path.join(out, 'features', '3DMatch', '7-scenes-redkitchen')
    assert sorted(os.listdir(scene)) == ['0_1.npz', '2_3.npz', '4_5.npz']
    ds = ThreeDMatchPairs(root, '3DMatch')
    for i in range(3):
        d = np.load(os.path.join(scene, f'{2 * i}_{2 * i + 1}.npz'))
        plain = ds[i]
        want = RO.rotated_pair(*(np.asarray(torch.load(p, weights_only=False)) for p in ds.files(i)), _transforms(ds.metadata_list)[i], i,
                               correctly_rounded=True)
        assert np.array_equal(d['transform'], want['transform']) and not np.array_equal(d['transform'], plain['transform'])
        assert np.array_equal(d['ref_points'], want['ref_points']) and np.array_equal(d['src_points'], want['src_points'])
    res = evaluate('3dmatch', 'lgr', os.path.join(out, 'features'), benchmark='3DMatch', protocol='dgr', test_epoch=7)[None]
    assert len(res['pairs']) == 3 and ('CRITICAL', 'Epoch 7') in [('CRITICAL' if lv == 50 else 'INFO', m) for lv, m in res['lines']]


def _same_lines(got, want):
    """equal line for line; RRE / RTE fields may differ by one unit of the last printed digit (the reference computes them in
    float32, the driver in double), as tests/test_gpu_benchmark.py allows for eval.py"""
    got = [f'{"INFO" if lv == 20 else "CRITICAL"}\t{m}' for lv, m in got]
    assert len(got) == len(want)
    for a, b in zip(got, want):
        if a == b:
            continue
        fa, fb = re.split(r'(RRE: |RTE: )(-?[0-9.]+|nan)', a), re.split(r'(RRE: |RTE: )(-?[0-9.]+|nan)', str(b))
        assert len(fa) == len(fb), (a, b)
        for i, (x, y) in enumerate(zip(fa, fb)):
            if i % 3 == 2:
                assert abs(float(x) - float(y)) <= 1.0001e-3, (a, b)
            else:
                assert x == y, (a, b)


@pytest.mark.parametrize('benchmark,method,num_corr', RV.DGR_RUNS)
def test_dgr_evaluation_reproduces_the_reference_lines(tmp_path, benchmark, method, num_corr):
    tree = EVV.make_tree(str(tmp_path / 'tree'))
    name = RV.dgr_run_name(benchmark, method, num_corr)
    out = evaluate('3dmatch', method, tree['features'], benchmark=benchmark, num_corr=None if num_corr is None else str(num_corr),
                   verbose=True, protocol='dgr', chunk=5)
    _same_lines(next(iter(out.values()))['lines'], list(GOLD[f'dgr/{name}/lines']))
    reg = GOLD[f'dgr/{name}/reg']
    for i, v in enumerate(next(iter(out.values()))['pairs']):
        assert abs(v['rre'] - reg[i, 0]) <= 1e-3 and abs(v['rte'] - reg[i, 1]) <= 1e-4, (name, i)
