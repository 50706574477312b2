"""ModelNet raw shapes and RPMNet's metrics on the device (``functional.modelnet_raw_points_batched``,
``functional.rpmnet_metrics_batched``, the surface functions and ``RegistrationTester(rpmnet_metrics=True)``) against the fixture
written from the reference (tests/golden/modelnet_rpmnet.npz) within the bounds of DESIGN.md section 8a."""
import copy
import os
import pickle

import numpy as np
import pytest
import torch

from geotransformer_b200 import functional as GF
from geotransformer_b200.config import make_cfg
from geotransformer_b200.datasets.modelnet import ModelNetPairs
from geotransformer_b200.modules import registration as MR
from geotransformer_b200.utils import registration as UR
from oracle import rpmnet_metrics_oracle as O

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'modelnet_rpmnet.npz')
BENCH_GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'modelnet_benchmark.npz')
CD_TOL = 2e-6
R_TOL = 1e-9


def _gold():
    g = np.load(GOLD)
    st = np.concatenate([[0], np.cumsum(g['length'])])
    return g, st


def _cases(g, st, ok_only=True):
    sel = [i for i in range(len(g['case_pair'])) if not (ok_only and g['case_raises'][i])]
    p = g['case_pair'][sel]
    raw = [g['raw_points'][st[i]:st[i + 1]] for i in p]
    return sel, p, raw, g['ref_points'][p], g['src_points'][p], g['transform'][p], g['case_est'][sel]


def _call(raw, ref, src, gt, est, check=True):
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(np.concatenate(x), np.float32)).cuda()
    return GF.rpmnet_metrics_batched(dev(raw), [len(x) for x in raw], dev(ref), [len(x) for x in ref], dev(src), [len(x) for x in src],
                                     torch.from_numpy(np.stack(gt)).cuda(), torch.from_numpy(np.stack(est)).cuda(), check=check)


def _all(raw, ref, src, gt, est):
    rows = [_call(raw[b:b + 32], ref[b:b + 32], src[b:b + 32], gt[b:b + 32], est[b:b + 32]) for b in range(0, len(raw), 32)]
    return torch.cat(rows).cpu().numpy()


def test_raw_points_are_the_references_bit_for_bit():
    g, st = _gold()
    shapes = torch.from_numpy(g['shape']).cuda()
    got = GF.modelnet_raw_points_batched(shapes, g['length'].tolist()).cpu().numpy()
    assert np.array_equal(got, g['raw_points'])
    for i in range(len(g['length'])):                  # alone
        one = GF.modelnet_raw_points_batched(shapes[st[i]:st[i + 1]].contiguous(), [int(g['length'][i])]).cpu().numpy()
        assert np.array_equal(one, g['raw_points'][st[i]:st[i + 1]])


def test_metrics_match_the_reference_within_the_bounds():
    g, st = _gold()
    sel, p, raw, ref, src, gt, est = _cases(g, st)
    got = _all(raw, ref, src, gt, est)
    want = g['case_metrics'][sel]
    assert np.all(got[:, 7] == 0)
    cd_err = np.abs(got[:, 0] - want[:, 0])
    assert cd_err.max() <= CD_TOL, cd_err.max()
    np.testing.assert_allclose(got[:, 3:5], want[:, 1:3], rtol=R_TOL, atol=1e-12)
    assert np.array_equal(got[:, 5:7], want[:, 3:5])
    assert np.array_equal(got[:, 0], got[:, 1] + got[:, 2])
    # the restatement's Chamfer distance uses the contract's arithmetic: only the order of the mean differs
    for i in range(0, len(sel), 7):
        r = O.metrics(raw[i], ref[i], src[i], gt[i], est[i])
        np.testing.assert_allclose(got[i, :3], r[:3], rtol=1e-13)
    print(f'{len(sel)} cases: Chamfer distance within {cd_err.max():.2e} of the reference; r_mse / r_mae within '
          f'{np.max(np.abs(got[:, 3:5] - want[:, 1:3]) / np.maximum(1, np.abs(want[:, 1:3]))):.2e}')


def test_one_batch_equals_one_pair_calls_and_runs_repeat():
    g, st = _gold()
    sel, p, raw, ref, src, gt, est = _cases(g, st)
    n = 32
    batch = _call(raw[:n], ref[:n], src[:n], gt[:n], est[:n]).cpu().numpy()
    again = _call(raw[:n], ref[:n], src[:n], gt[:n], est[:n]).cpu().numpy()
    assert np.array_equal(batch.view(np.int64), again.view(np.int64))
    for i in range(n):
        one = _call(raw[i:i + 1], ref[i:i + 1], src[i:i + 1], gt[i:i + 1], est[i:i + 1]).cpu().numpy()
        assert np.array_equal(one.view(np.int64), batch[i:i + 1].view(np.int64)), i


def test_non_positive_determinant_names_the_pair():
    g, st = _gold()
    k = int(np.nonzero(g['case_raises'])[0][0])
    sel, p, raw, ref, src, gt, est = _cases(g, st)
    est = np.concatenate([est[:2], g['case_est'][k:k + 1]])
    with pytest.raises(ValueError, match='pair 2'):
        _call(raw[:3], ref[:3], src[:3], gt[:3], est)
    rows = _call(raw[:3], ref[:3], src[:3], gt[:3], est, check=False).cpu().numpy()
    assert rows[2, 7] == 2 and np.isnan(rows[2, 3]) and np.all(rows[:2, 7] == 0)
    with pytest.raises(ValueError):
        UR.compute_transform_mse_and_mae(gt[0], g['case_est'][k])
    with pytest.raises(ValueError):
        UR.compute_transform_mse_and_mae(g['case_est'][k], gt[0])


def test_surface_functions_numpy_and_cuda():
    g, st = _gold()
    sel, p, raw, ref, src, gt, est = _cases(g, st)
    want = g['case_metrics'][sel]
    for i in (0, 3, 9, 14):
        cd = UR.compute_modified_chamfer_distance(raw[i], ref[i], src[i], gt[i], est[i])
        assert isinstance(cd, np.float64) and abs(cd - want[i, 0]) <= CD_TOL
        r_mse, r_mae, t_mse, t_mae = UR.compute_transform_mse_and_mae(gt[i], est[i])
        assert isinstance(t_mse, np.float32) and t_mse == want[i, 3] and t_mae == want[i, 4]
        np.testing.assert_allclose([r_mse, r_mae], want[i, 1:3], rtol=R_TOL, atol=1e-12)
        np.testing.assert_allclose(UR.compute_rotation_mse_and_mae(gt[i][:3, :3], est[i][:3, :3]), want[i, 1:3], rtol=R_TOL, atol=1e-12)
        assert UR.compute_translation_mse_and_mae(gt[i][:3, 3], est[i][:3, 3]) == (want[i, 3], want[i, 4])
        c = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (raw[i], ref[i], src[i], gt[i], est[i])]
        cd_t = UR.compute_modified_chamfer_distance(*c)
        assert cd_t.is_cuda and float(cd_t) == cd
        t = UR.compute_transform_mse_and_mae(c[3], c[4])
        assert all(x.is_cuda for x in t) and float(t[2]) == t_mse
        rre, rte = UR.compute_registration_error(gt[i], est[i])
        assert abs(UR.compute_relative_rotation_error(gt[i][:3, :3], est[i][:3, :3]) - rre) <= 1e-9
        assert abs(UR.compute_relative_translation_error(gt[i][:3, 3], est[i][:3, 3]) - rte) <= 1e-9
        pts = src[i].astype(np.float64)
        rmse = np.linalg.norm(pts @ gt[i][:3, :3].T.astype(np.float64) + gt[i][:3, 3] - (pts @ est[i][:3, :3].T.astype(np.float64)
                                                                                           + est[i][:3, 3]), axis=1).mean()
        assert abs(UR.compute_registration_rmse(src[i], gt[i], est[i]) - rmse) <= 1e-5
    # the batched torch forms over (B, N, 3): 34 pairs, two calls
    B = 34
    idx = [i for i in range(len(sel)) if len(raw[i]) == 2048][:B]
    assert len(idx) == B
    T = lambda x: torch.from_numpy(np.stack([x[i] for i in idx])).cuda()
    cd = MR.modified_chamfer_distance(T(raw), T(ref), T(src), T(gt), T(est), reduction='none')
    assert cd.dtype == torch.float32 and cd.shape == (B,)
    np.testing.assert_allclose(cd.cpu().numpy(), want[idx, 0], atol=CD_TOL)
    assert torch.allclose(MR.modified_chamfer_distance(T(raw), T(ref), T(src), T(gt), T(est)), cd.mean())
    a = MR.anisotropic_transform_error(T(gt), T(est), reduction='none')
    np.testing.assert_allclose(torch.stack(a, 1).cpu().numpy(), want[idx, 1:5].astype(np.float32), rtol=1e-6, atol=1e-12)
    rre, rte = MR.isotropic_transform_error(T(gt), T(est), reduction='none')
    assert torch.allclose(MR.relative_rotation_error(T(gt)[:, :3, :3], T(est)[:, :3, :3]), rre)
    assert torch.allclose(MR.relative_translation_error(T(gt)[:, :3, 3], T(est)[:, :3, 3]), rte)
    assert rre.dtype == torch.float32 and float(MR.isotropic_transform_error(T(gt), T(est), reduction='sum')[0]) == pytest.approx(float(rre.sum()), rel=1e-6)


def _write_pkl(tmp_path):
    g = np.load(BENCH_GOLD)
    st = np.concatenate([[0], np.cumsum(g['length'])])
    shapes = [g['shape'][st[i]:st[i + 1]] for i in range(len(g['length']))]
    labels = g['labels'].tolist()
    n = len(labels) - 1
    rows = [shapes[0], shapes[0][::2].copy()] + shapes[1:n]
    with open(tmp_path / 'test.pkl', 'wb') as f:
        pickle.dump([{'points': r, 'normals': np.zeros_like(r), 'label': l} for r, l in zip(rows, labels)], f)
    return g


def test_modelnet_items_gain_raw_points_and_keep_their_keys(tmp_path):
    g = _write_pkl(tmp_path)
    cfg = make_cfg('modelnet')
    items = [d for c in ModelNetPairs(str(tmp_path), 'test', cfg, chunk_size=4).chunks() for d in c]
    n = len(items)
    shapes = torch.from_numpy(g['shape']).cuda()
    pts, _, T, _ = GF.modelnet_benchmark_pairs_batched(shapes[:int(g['length'][:n].sum())].contiguous(), g['length'][:n].tolist(),
                                                       list(range(n)), 717, 0.7, 45.0, 0.5, 0.05)
    st = np.concatenate([[0], np.cumsum(g['length'])])
    for p, d in enumerate(items):
        assert torch.equal(d['ref_points'], pts[p * 717:(p + 1) * 717]) and torch.equal(d['src_points'], pts[(n + p) * 717:(n + p + 1) * 717])
        assert torch.equal(d['transform'], T[p])
        assert d['raw_points'].is_cuda and d['raw_points'].dtype == torch.float32
        assert np.array_equal(d['raw_points'].cpu().numpy(), O.raw_points(g['shape'][st[p]:st[p + 1]]))


def test_tester_with_and_without_rpmnet_metrics(tmp_path, models):
    from geotransformer_b200.model import create_model
    from geotransformer_b200.tester import RPMNET, RegistrationTester
    from oracle import backbone_grad_oracle as BV
    _write_pkl(tmp_path)
    cfg, sd, _ = models('modelnet')
    cfg = copy.deepcopy(cfg)
    model = create_model(cfg)
    model.load_state_dict(sd, strict=True)
    model = model.cuda().eval()
    logs = {True: [], False: []}
    res = {}
    for flag in (False, True):
        tester = RegistrationTester(cfg, model, BV.limits('modelnet717'), chunk=4, rpmnet_metrics=flag)
        try:
            res[flag] = tester.run(ModelNetPairs(str(tmp_path), 'test', cfg, chunk_size=4), log=logs[flag].append)
        finally:
            tester.close()
    (s0, p0), (s1, p1) = res[False], res[True]
    assert not any(k.startswith('rpmnet_') for k in s0) and all('rpmnet' not in p for p in p0)
    np.testing.assert_equal({k: v for k, v in s1.items() if not k.startswith('rpmnet_')}, s0)
    np.testing.assert_equal([p['metrics'] for p in p1], [p['metrics'] for p in p0])
    assert all(l1.startswith(l0) for l0, l1 in zip(logs[False], logs[True])) and len(logs[True]) == len(logs[False])
    pairs = [d for c in ModelNetPairs(str(tmp_path), 'test', cfg).chunks() for d in c]
    for d, p in zip(pairs, p1):
        want = O.metrics(d['raw_points'].cpu().numpy(), d['ref_points'].cpu().numpy(), d['src_points'].cpu().numpy(),
                         d['transform'].cpu().numpy(), p['estimated_transform'].numpy())
        assert abs(p['rpmnet']['CD'] - want[0]) <= 1e-12 * max(1.0, want[0]) + 1e-15
        np.testing.assert_allclose([p['rpmnet'][k] for k in ('r_mse', 'r_mae')], want[3:5], rtol=R_TOL, atol=1e-12)
        assert [p['rpmnet'][k] for k in ('t_mse', 't_mae')] == list(want[5:7])
    for k in RPMNET:
        assert s1[f'rpmnet_{k}'] == pytest.approx(np.mean([p['rpmnet'][k] for p in p1]))
    with pytest.raises(ValueError):
        RegistrationTester(make_cfg('3dmatch'), model, BV.limits('modelnet717'), rpmnet_metrics=True)
    print('rpmnet summary', {k: round(v, 6) for k, v in s1.items() if k.startswith('rpmnet_')})
