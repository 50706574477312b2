"""The trainval and test drivers on synthetic dataset trees in the reference's layout, written from ``synth.make_pair``: training
for two epochs at B = 1 and B = 4, a run stopped after epoch 1 and resumed against uninterrupted runs, and the test's ``.npz``
tree read end to end by ``evaluate``."""
import os
import pickle

import numpy as np
import pytest
import torch

from geotransformer_b200 import test as test_driver
from geotransformer_b200 import trainval
from geotransformer_b200.evaluate import evaluate
from geotransformer_b200.synth import make_pair
from geotransformer_b200.tester import NPZ_OUTPUT_KEYS

pytestmark = pytest.mark.gpu


def _threedmatch_tree(root, splits):
    """{split: [pair index, ...]}: demo-size pairs in scene 'synthetic-scene', fragments numbered per split"""
    os.makedirs(os.path.join(root, 'metadata'), exist_ok=True)
    for split, indices in splits.items():
        meta = []
        for j, i in enumerate(indices):
            pair = make_pair('demo2k', i)
            names = []
            for k, key in enumerate(('ref_points', 'src_points')):
                name = f'{split}/synthetic-scene/cloud_bin_{2 * j + k}.pth'
                os.makedirs(os.path.join(root, 'data', os.path.dirname(name)), exist_ok=True)
                torch.save(pair[key].astype(np.float64), os.path.join(root, 'data', name))
                names.append(name)
            T = pair['transform'].astype(np.float64)
            meta.append({'pcd0': names[0], 'pcd1': names[1], 'rotation': T[:3, :3], 'translation': T[:3, 3], 'overlap': 0.5,
                         'scene_name': 'synthetic-scene', 'frag_id0': 2 * j, 'frag_id1': 2 * j + 1})
        with open(os.path.join(root, 'metadata', f'{split}.pkl'), 'wb') as f:
            pickle.dump(meta, f)
    return root


def _kitti_tree(root, splits):
    os.makedirs(os.path.join(root, 'metadata'), exist_ok=True)
    for split, (seq, indices) in splits.items():
        meta = []
        for j, i in enumerate(indices):
            pair = make_pair('kitti4k', i)
            names = [f'downsampled/{seq:02d}/{2 * j + 1:06d}.npy', f'downsampled/{seq:02d}/{2 * j:06d}.npy']
            for name, key in zip(names, ('ref_points', 'src_points')):
                os.makedirs(os.path.join(root, os.path.dirname(name)), exist_ok=True)
                np.save(os.path.join(root, name), pair[key].astype(np.float64))
            meta.append({'seq_id': seq, 'frame0': np.int64(2 * j + 1), 'frame1': 2 * j, 'pcd0': names[0], 'pcd1': names[1],
                         'transform': pair['transform'].astype(np.float64)})
        with open(os.path.join(root, 'metadata', f'{split}.pkl'), 'wb') as f:
            pickle.dump(meta, f)
    return root


def _params(output_dir, name='snapshot.pth.tar'):
    return torch.load(os.path.join(output_dir, 'snapshots', name), map_location='cpu', weights_only=False)


def _max_diff(a, b):
    return max(float((a[k].double() - b[k].double()).abs().max()) for k in a if a[k].dtype.is_floating_point)


@pytest.mark.parametrize('batch_size', [1, 4])
def test_trainval_two_epochs(tmp_path, batch_size):
    root = _threedmatch_tree(str(tmp_path / 'data'), {'train': range(6), 'val': range(6, 8)})
    out = str(tmp_path / 'out')
    engine = trainval.run('3dmatch', root, out, batch_size=batch_size, seed=3, max_epoch=2)
    steps = (6 + batch_size - 1) // batch_size
    assert (engine.epoch, engine.iteration) == (2, 2 * steps)
    for e in (1, 2):
        s = _params(out, f'epoch-{e}.pth.tar')
        assert set(s) == {'epoch', 'iteration', 'model'} and (s['epoch'], s['iteration']) == (e, e * steps)
    snap = _params(out)
    assert set(snap) == {'epoch', 'iteration', 'model', 'optimizer', 'scheduler'}
    assert _max_diff(snap['model'], _params(out, 'epoch-1.pth.tar')['model']) > 0       # the second epoch moved the weights
    log = open(os.path.join(out, 'train.log')).read()
    assert 'Calibrate neighbors: [' in log and f'Epoch: 2/2, iter: {steps}/{steps}, loss: ' in log and '[Val] Epoch: 2, loss: ' in log


def test_trainval_resume_matches_an_uninterrupted_run(tmp_path):
    """two uninterrupted runs give the run-to-run spread; a run stopped after epoch 1 and resumed must land within it"""
    root = _threedmatch_tree(str(tmp_path / 'data'), {'train': range(8), 'val': range(8, 9)})
    runs = {}
    for name in ('a', 'b'):
        trainval.run('3dmatch', root, str(tmp_path / name), batch_size=4, seed=11, max_epoch=2)
        runs[name] = _params(str(tmp_path / name))['model']
    resumed = str(tmp_path / 'resumed')
    trainval.run('3dmatch', root, resumed, batch_size=4, seed=11, max_epoch=1)
    first = _params(resumed)
    assert (first['epoch'], first['iteration']) == (1, 2)
    trainval.run('3dmatch', root, resumed, batch_size=4, seed=11, max_epoch=2, resume=True)
    snap = _params(resumed)
    assert (snap['epoch'], snap['iteration']) == (2, 4)
    spread = _max_diff(runs['a'], runs['b'])
    diff = _max_diff(runs['a'], snap['model'])
    print(f'run-to-run spread of the parameters after 2 epochs: {spread:.3e}; resumed vs uninterrupted: {diff:.3e}')
    assert diff <= max(2 * spread, 1e-6), (diff, spread)


def test_test_driver_writes_the_npz_trees_and_evaluate_reads_them(tmp_path):
    model = trainval.build_model(trainval.make_cfg('kitti'), 5, torch.device('cuda', torch.cuda.current_device()))
    snap = str(tmp_path / 'kitti.pth.tar')
    torch.save({'model': model.state_dict()}, snap)
    root = _kitti_tree(str(tmp_path / 'kitti'), {'train': (0, range(4)), 'test': (8, range(4, 7))})
    out = str(tmp_path / 'kitti_out')
    summary, per_pair = test_driver.run('kitti', snap, root, out)
    assert len(per_pair) == 3 and set(summary) >= {'RRE', 'RTE', 'RR'}
    files = sorted(os.listdir(os.path.join(out, 'features')))
    assert files == ['8_0_1.npz', '8_2_3.npz', '8_4_5.npz']
    d = np.load(os.path.join(out, 'features', files[0]))
    assert set(NPZ_OUTPUT_KEYS) | {'transform'} == set(d.files)
    res = evaluate('kitti', 'lgr', os.path.join(out, 'features'))
    assert len(res[None]['pairs']) == 3

    model = trainval.build_model(trainval.make_cfg('3dmatch'), 5, torch.device('cuda', torch.cuda.current_device()))
    snap = str(tmp_path / '3dmatch.pth.tar')
    torch.save({'model': model.state_dict()}, snap)
    root = _threedmatch_tree(str(tmp_path / '3dm'), {'train': range(3), '3DMatch': range(3, 5)})
    out = str(tmp_path / '3dm_out')
    for limits in ('calibrate', 'config'):
        summary, per_pair = test_driver.run('3dmatch', snap, root, out, benchmark='3DMatch', neighbor_limits=limits)
        assert len(per_pair) == 2
    scene = os.path.join(out, 'features', '3DMatch', 'synthetic-scene')
    assert sorted(os.listdir(scene)) == ['0_1.npz', '2_3.npz']
    assert set(np.load(os.path.join(scene, '0_1.npz')).files) == set(NPZ_OUTPUT_KEYS) | {'transform', 'overlap'}
