"""The rotated 3DMatch / 3DLoMatch benchmark and the eval_dgr evaluation without a GPU: the numpy restatement of the rotations and
items (oracle/rotated_oracle.py) against the fixture written from the reference (tests/golden/rotated_3dmatch.npz, written by
oracle/rotated_vectors.py), the dgr host pass replayed from the reference's per-pair values, the argument checks of
``geob200_rotated_pairs_batched``, and the drivers' options."""
import ctypes
import io
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

from geotransformer_b200 import _lib as L
from geotransformer_b200 import evaluate as EV
from geotransformer_b200 import test as test_driver
from geotransformer_b200.config import make_cfg
from geotransformer_b200.datasets import threedmatch_utils as TU
from geotransformer_b200.datasets.threedmatch import ThreeDMatchPairs
from oracle import eval_vectors as EVV
from oracle import ref_harness
from oracle import rotated_oracle as RO
from oracle import rotated_vectors as RV

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(RV.GOLD_PATH)


@pytest.fixture(scope='module')
def eval_tree(tmp_path_factory):
    return EVV.make_tree(str(tmp_path_factory.mktemp('bench')))


@pytest.mark.skipif(not ref_harness.available(), reason='reference checkout not present')
def test_golden_regenerates_from_the_reference(tmp_path):
    out = str(tmp_path / 'regen.npz')
    code = f'import numpy as np; from oracle import rotated_vectors as RV; np.savez({out!r}, **RV.build())'
    subprocess.run([sys.executable, '-c', code], cwd=ROOT, check=True, capture_output=True)
    regen = np.load(out)
    assert sorted(regen.files) == sorted(GOLD.files)
    for k in GOLD.files:
        assert regen[k].dtype == GOLD[k].dtype and np.array_equal(regen[k], GOLD[k], equal_nan=GOLD[k].dtype.kind == 'f'), k


def test_restated_draws_equal_the_reference_rotations():
    index = GOLD['rot/index']
    assert index[-1] == (1 << 32) - 1 and len(index) == 259
    for i, want in zip(index, GOLD['rot/R']):
        got = RO.rotations(int(i))
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), i


def _half_angles(index):
    rs = np.random.RandomState(index)
    return [float(x) * 0.5 for _ in range(2) for x in RO.euler_angles(rs)]


def test_correctly_rounded_rotations_differ_from_the_reference_only_where_libm_misrounds():
    """The scipy restatement with the host libm's sin / cos equals the reference on every seed; with correctly rounded sin / cos
    (what the device computes) it differs exactly on the seeds where the libm's sin or cos of a half-angle is not correctly
    rounded, which are few"""
    differs, misrounds = [], []
    for i, want in zip(GOLD['rot/index'], GOLD['rot/R']):
        i = int(i)
        rs = np.random.RandomState(i)
        libm = [RO.euler_zyx(*RO.euler_angles(rs), RO.libm_sincos) for _ in range(2)]
        assert np.array_equal(libm[0], want[0]) and np.array_equal(libm[1], want[1]), i
        if not np.array_equal(np.stack(RO.rotations(i, correctly_rounded=True)), want):
            differs.append(i)
        if any(RO.libm_sincos(x) != RO.sincos_cr(x) for x in _half_angles(i)):
            misrounds.append(i)
    assert differs == misrounds and len(differs) <= 6, (differs, misrounds)


def test_correctly_rounded_sincos():
    """sincos_cr against exact rational bounds: the Taylor partial sums bracket sin and cos, and the result is the double nearest
    to both brackets"""
    from fractions import Fraction
    for x in [0.0, 5e-324, -1e-300, 0.20991572889377652, -0.8789015320503755, 1.5707963267948966, -1.6] + \
            list(np.random.default_rng(2).uniform(-1.6, 1.6, 50)):
        s, c = RO.sincos_cr(x)
        X = Fraction(float(x))
        terms_s, terms_c, t = [], [], Fraction(1)
        for n in range(1, 60):
            t = t * X / n
            (terms_s if n % 2 else terms_c).append(t * (-1) ** ((n - 1) // 2 if n % 2 else n // 2))
        lo_s, hi_s = sum(terms_s[:-1]), sum(terms_s)
        lo_c, hi_c = 1 + sum(terms_c[:-1]), 1 + sum(terms_c)
        assert float(lo_s) == float(hi_s) == s and float(lo_c) == float(hi_c) == c, x


def test_restated_items_equal_the_reference_items():
    for subset, dtype, sizes in RV.TREE:
        meta = pickle.load(io.BytesIO(GOLD[f'tree/{subset}/metadata'].tobytes()))
        pts, lengths = GOLD[f'tree/{subset}/points'], GOLD[f'tree/{subset}/lengths']
        assert pts.dtype == dtype and list(lengths) == [n for pair in sizes for n in pair]
        clouds = np.split(pts, np.cumsum(lengths)[:-1])
        rows = {k: np.split(GOLD[f'item/{subset}/{k}'], np.cumsum(lengths[j::2])[:-1]) for j, k in enumerate(('ref_points', 'src_points'))}
        for i, e in enumerate(meta):
            T = np.eye(4)
            T[:3, :3], T[:3, 3] = e['rotation'], e['translation']
            got = RO.rotated_pair(clouds[2 * i], clouds[2 * i + 1], T, i)
            assert np.array_equal(got['ref_points'], rows['ref_points'][i]) and np.array_equal(got['src_points'], rows['src_points'][i])
            assert np.array_equal(got['transform'], GOLD[f'item/{subset}/transform'][i])


def _replay_dgr(name, tree, benchmark):
    """the dgr host pass (meters, lines) over the reference's own per-pair values"""
    cfg = make_cfg('3dmatch')
    sparse, corr, reg = (GOLD[f'dgr/{name}/{k}'] for k in ('sparse', 'corr', 'reg'))
    run = EV._Run(None, None)
    i = 0
    for scene, files in EV.discover('3dmatch', tree['features'], benchmark):
        run.scene_meters = EV._meters(['precision', 'PMR>0', 'PMR>=0.1', 'PMR>=0.3', 'PMR>=0.5', 'fmr', 'inlier_ratio', 'overlap',
                                       'rr', 'rre', 'rte'])
        for f in files:
            item = EV._load(f, '3dmatch', None, dgr=True)
            v = dict(precision=sparse[i, 0], recall=sparse[i, 1], hit_ratio=sparse[i, 2], overlap=corr[i, 0], inlier_ratio=corr[i, 1],
                     residual=corr[i, 2], num_corr=int(corr[i, 3]), rre=reg[i, 0], rte=reg[i, 1],
                     accepted=bool(reg[i, 0] < cfg.eval.rre_threshold and reg[i, 1] < cfg.eval.rte_threshold))
            run.emit(EV.INFO, EV._pair_dgr(run, cfg, TU.get_scene_abbr(scene), item, v))
            i += 1
        EV._scene_end_dgr(run, scene, TU.get_scene_abbr(scene))
    EV._final_dgr(run, None)
    return [f'{"INFO" if lv == EV.INFO else "CRITICAL"}\t{m}' for lv, m in run.lines]


@pytest.mark.parametrize('benchmark,method,num_corr', RV.DGR_RUNS)
def test_dgr_meters_and_lines_replay_the_reference(eval_tree, benchmark, method, num_corr):
    name = RV.dgr_run_name(benchmark, method, num_corr)
    lines = list(GOLD[f'dgr/{name}/lines'])
    assert _replay_dgr(name, eval_tree, benchmark) == lines
    summary = [ln for ln in lines if ln.startswith('CRITICAL\t  Registration, ')]
    assert len(summary) == 1 and summary[0].endswith(', ')                   # eval_dgr's trailing separator


def test_rotated_pairs_reject_bad_arguments_before_any_launch():
    lib = L.lib()
    buf = ctypes.create_string_buffer(1 << 12)
    p = ctypes.addressof(buf)
    n0 = lib.geob200_launch_count()

    def i64(*v):
        return (ctypes.c_int64 * len(v))(*v)

    def err():
        return lib.geob200_last_error().decode()

    def rot(B=1, lengths=None, indices=None, fp64=0, ptr=p, out=p):
        lengths = lengths if lengths is not None else i64(*([100] * max(2 * B, 2)))
        indices = indices if indices is not None else i64(*range(max(B, 1)))
        return lib.geob200_rotated_pairs_batched(ptr, fp64, lengths, indices, B, p, out, p, p, None)

    assert rot(B=0) < 0 and 'n_pairs' in err()
    assert rot(B=(1 << 30) + 1, lengths=i64(100, 100), indices=i64(0)) < 0 and 'n_pairs' in err()
    assert rot(lengths=i64(100, 0)) < 0 and 'cloud 1 has 0 points' in err()
    assert rot(lengths=i64(-3, 10)) < 0 and 'cloud 0' in err()
    assert rot(lengths=i64(1 << 31, 1)) < 0 and 'cloud 0' in err()
    assert rot(B=2, lengths=i64((1 << 31) - 1, 1, 1, 1)) < 0 and '2^31-1 rows' in err()
    assert rot(indices=i64(-1)) < 0 and 'index -1 of pair 0' in err()
    assert rot(indices=i64(1 << 32)) < 0 and 'index' in err()
    assert rot(fp64=2) < 0 and 'points_fp64' in err()
    assert rot(ptr=None) < 0 and 'null' in err()
    assert rot(out=None) < 0 and 'null' in err()
    assert lib.geob200_rotated_pairs_batched(p, 0, None, i64(0), 1, p, p, p, p, None) < 0 and 'null' in err()
    assert lib.geob200_launch_count() == n0


def test_dgr_protocol_options(eval_tree):
    a = EV.make_parser().parse_args(['--config', '3dmatch', '--benchmark', '3DMatch', '--method', 'lgr', '--features', 'x',
                                     '--protocol', 'dgr', '--test-epoch', '40'])
    assert a.protocol == 'dgr' and a.test_epoch == 40 and a.gt_root is None
    d = EV.make_parser().parse_args(['--config', '3dmatch', '--benchmark', '3DMatch', '--method', 'lgr', '--features', 'x'])
    assert d.protocol == 'gtlog' and d.test_epoch is None
    with pytest.raises(SystemExit):
        EV.main(['--config', 'kitti', '--method', 'lgr', '--features', 'x', '--protocol', 'dgr'])
    with pytest.raises(SystemExit):
        EV.main(['--config', '3dmatch', '--benchmark', '3DMatch', '--method', 'lgr', '--features', 'x', '--protocol', 'dgr',
                 '--registration-dir', 'y'])
    with pytest.raises(ValueError, match='3dmatch evaluation'):
        EV.evaluate('kitti', 'lgr', eval_tree['kitti'], protocol='dgr')
    with pytest.raises(ValueError, match='protocol'):
        EV.evaluate('3dmatch', 'lgr', eval_tree['features'], benchmark='3DMatch', protocol='eval')
    with pytest.raises(ValueError, match='gt-root'):
        EV.evaluate('3dmatch', 'lgr', eval_tree['features'], benchmark='3DMatch')
    # without --gt-root the dgr load scores against the npz transform
    f = EV.discover('3dmatch', eval_tree['features'], '3DMatch')[0][1][0]
    item = EV._load(f, '3dmatch', None, dgr=True)
    assert not item['has_cov'] and np.array_equal(item['reg_gt'], np.load(f)['transform'])


def test_rotated_reader_and_driver_options(tmp_path):
    metadata = {subset: RV.tree_metadata(subset) for subset, _, _ in RV.TREE}
    root = RV.write_tree(str(tmp_path / '3dm'), metadata, RV.tree_clouds())
    for subset, _, sizes in RV.TREE:
        ds = ThreeDMatchPairs(root, subset, rotated=True)
        assert ds.rotated and len(ds) == len(sizes)
    assert not ThreeDMatchPairs(root, '3DMatch').rotated
    with pytest.raises(ValueError, match='rotated=True'):
        ThreeDMatchPairs(root, '3DMatch').rotated_batch([0])
    a = test_driver.make_parser().parse_args(['--config', '3dmatch', '--benchmark', '3DMatch', '--snapshot', 's', '--dataset-root', 'd',
                                              '--output-dir', 'o', '--rotated'])
    assert a.rotated
    with pytest.raises(SystemExit):
        test_driver.main(['--config', 'kitti', '--snapshot', 's', '--dataset-root', 'd', '--output-dir', 'o', '--rotated'])
    with pytest.raises(ValueError, match='3dmatch'):
        test_driver.benchmark_set(make_cfg('kitti'), root, None, rotated=True)
