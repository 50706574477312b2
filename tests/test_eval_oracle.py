"""Host side of the benchmark evaluation (no GPU): nibabel's mat2quat restatement, the gt.log / gt.info readers and the est.log
writer, the meters and log lines replayed from the reference's per-pair values, argument parsing and layout discovery.
Golden data: tests/golden/eval_benchmark.npz (oracle/eval_vectors.py, from the reference's eval_one_epoch on the tree that
oracle.eval_vectors.make_tree regenerates)."""
import glob
import os

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from geotransformer_b200 import evaluate as EV
from geotransformer_b200.config import make_cfg
from geotransformer_b200.datasets import threedmatch_utils as TU
from oracle import eval_vectors as V

GOLD = np.load(V.GOLD_PATH)


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    return V.make_tree(str(tmp_path_factory.mktemp('bench')))


def test_mat2quat_restatement_matches_scipy():
    R = Rotation.random(1000, random_state=np.random.default_rng(7)).as_matrix()
    for m in R:
        q = V.mat2quat(m)
        x, y, z, w = Rotation.from_matrix(m).as_quat()
        want = np.array([w, x, y, z]) * (1 if w >= 0 else -1)
        assert np.abs(q - want).max() <= 1e-12


def test_log_writer_is_byte_identical_to_the_reference(tree, tmp_path):
    for scene in V.SCENES:
        files = EV.discover('3dmatch', tree['features'], '3DMatch')
        files = dict(files)[scene]
        pairs = [{'test_pair': EV._ids(f), 'num_fragments': TU.get_num_fragments(scene),
                  'transform': np.load(f)['estimated_transform']} for f in files]
        out = os.path.join(tmp_path, scene, 'est.log')
        TU.write_log_file(out, pairs)
        assert open(out, 'rb').read() == GOLD[f'3DMatch_lgr/estlog/{scene}'].tobytes()
        back = TU.read_log_file(out)
        assert [r['test_pair'] for r in back] == [p['test_pair'] for p in pairs]
        for r, p in zip(back, pairs):
            assert r['transform'].dtype == np.float32 and np.array_equal(r['transform'], p['transform'])


def test_gt_readers(tree):
    root = os.path.join(tree['gt_root'], '3DMatch', V.SCENES[0])
    logs, infos = TU.read_log_file(os.path.join(root, 'gt.log')), TU.read_info_file(os.path.join(root, 'gt.info'))
    assert len(logs) == len(infos) == 7 and all(r['num_fragments'] == 37 for r in logs)
    assert logs[0]['transform'].shape == (4, 4) and infos[0]['covariance'].shape == (6, 6)
    assert infos[0]['covariance'].dtype == np.float32
    text = open(os.path.join(root, 'gt.log')).read().split('\n')
    assert np.array_equal(logs[1]['transform'][0], np.array(text[6].split(), dtype=np.float32))
    gt_indices, _, _ = TU.get_gt_logs_and_infos(root, 37)
    assert gt_indices[0, 1] == -1 and gt_indices[2, 3] == -1          # adjacent: not scored
    assert gt_indices[0, 5] == 1 and gt_indices[5, 9] == -1           # (5, 9) is not in gt.log
    with pytest.raises(ValueError, match='Unsupported test scene'):
        TU.get_num_fragments('not-a-scene')
    assert TU.get_scene_abbr('sun3d-hotel_uc-scan3') == 'Hotel_1' and TU.get_scene_abbr('x') == 'x'


def _replay(config, name, tree, benchmark=None):
    """The driver's host pass (meters, lines) over the reference's own per-pair values."""
    cfg = make_cfg(config)
    sparse, corr, reg, terr = (GOLD[f'{name}/{k}'] for k in ('sparse', 'corr', 'reg', 'terr'))
    run = EV._Run(None, None)
    i = 0
    scenes = EV.discover(config, tree['features'] if config == '3dmatch' else tree['kitti'], benchmark)
    n_total = sum(len(f) for _, f in scenes)
    for scene, files in scenes:
        if config == '3dmatch':
            gt = TU.get_gt_logs_and_infos(os.path.join(tree['gt_root'], benchmark, scene), 37)
            run.scene_meters = EV._meters(['precision', 'PMR>0', 'PMR>=0.1', 'PMR>=0.3', 'PMR>=0.5', 'fmr', 'inlier_ratio', 'overlap',
                                           'rr', 'rre', 'rte'])
        for f in files:
            item = EV._load(f, config, gt if config == '3dmatch' else None)
            v = dict(precision=sparse[i, 0], recall=sparse[i, 1], hit_ratio=sparse[i, 2], overlap=corr[i, 0], inlier_ratio=corr[i, 1],
                     residual=corr[i, 2], num_corr=int(corr[i, 3]), rre=reg[i, 0], rte=reg[i, 1], error=terr[i])
            if config == '3dmatch':
                v['accepted'] = bool(terr[i] < cfg.eval.rmse_threshold ** 2)
                msg = EV._pair_3dmatch(run, cfg, TU.get_scene_abbr(scene), item, v)
            else:
                v['accepted'] = bool(reg[i, 0] < cfg.eval.rre_threshold and reg[i, 1] < cfg.eval.rte_threshold)
                msg = EV._pair_kitti(run, cfg, item, v, i, n_total)
            run.emit(EV.INFO, msg)
            i += 1
        if config == '3dmatch':
            EV._scene_end_3dmatch(run, scene, TU.get_scene_abbr(scene))
    EV._final(run, config)
    return [f'{"INFO" if lv == EV.INFO else "CRITICAL"}\t{m}' for lv, m in run.lines]


@pytest.mark.parametrize('config,benchmark,name', [('3dmatch', '3DMatch', '3DMatch_lgr'), ('3dmatch', '3DLoMatch', '3DLoMatch_lgr'),
                                                   ('kitti', None, 'kitti_lgr'), ('kitti', None, 'kitti_svd_k1000')])
def test_meters_and_lines_replay_the_reference(tree, config, benchmark, name):
    assert _replay(config, name, tree, benchmark) == list(GOLD[f'{name}/lines'])


def test_argument_parsing_and_discovery(tree):
    assert EV.parse_num_corr(None) == [None] and EV.parse_num_corr('250,1000') == [250, 1000]
    for bad in ('0', '9000', ','):
        with pytest.raises(ValueError):
            EV.parse_num_corr(bad)
    a = EV.make_parser().parse_args(['--config', 'kitti', '--method', 'svd', '--features', 'x', '--num_corr', '5000'])
    assert a.method == 'svd' and a.num_corr == '5000' and a.benchmark is None
    with pytest.raises(SystemExit):
        EV.make_parser().parse_args(['--config', 'kitti', '--method', 'icp', '--features', 'x'])
    with pytest.raises(SystemExit):
        EV.main(['--config', '3dmatch', '--method', 'lgr', '--features', 'x'])           # 3dmatch needs --benchmark / --gt-root
    scenes = EV.discover('3dmatch', tree['features'], '3DMatch')
    assert [s for s, _ in scenes] == sorted(V.SCENES)
    ids = [EV._ids(f) for f in scenes[0][1]]
    assert ids == sorted(ids) and ids[0] == [0, 1] and [10, 30] in ids
    (none, kitti), = EV.discover('kitti', tree['kitti'])
    assert none is None and [EV._ids(f) for f in kitti] == sorted(EV._ids(f) for f in glob.glob(os.path.join(tree['kitti'], '*.npz')))
    assert 'overlap' not in np.load(kitti[0]).files
