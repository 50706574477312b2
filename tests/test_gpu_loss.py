"""Validation losses on the device (CoarseMatchingLoss / FineMatchingLoss / OverallLoss, reference experiments/<exp>/loss.py:10-92):
the kernels against the real reference's outputs on seeded inputs (tests/golden/losses.npz), against the torch restatement on the
forward's own outputs, teacher-forced end to end against the reference's scalars, and the batched forward / engine / tester paths
against the per-pair modules, bit for bit."""
import os

import numpy as np
import pytest
import torch

from geotransformer_b200 import functional as GF
from geotransformer_b200.loss import OverallLoss
from geotransformer_b200.model import enable_native
from geotransformer_b200.synth import make_pair
from geotransformer_b200.utils.data import registration_collate_fn_stack_mode
from oracle import loss_oracle as LO

pytestmark = pytest.mark.gpu
KEYS = ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')
LIMITS = {'3dmatch': [38, 36, 36, 38], 'modelnet': [13, 21, 27], 'kitti': [27, 75, 147, 157, 119]}
NAMES = ('loss', 'c_loss', 'f_loss')


@pytest.fixture(scope='module')
def losses():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'losses.npz'))


def _rel(a, b):
    a, b = float(a), float(b)
    if np.isnan(a) or np.isnan(b):
        return 0.0 if (np.isnan(a) and np.isnan(b)) else float('inf')
    return abs(a - b) / max(abs(b), 1e-30)


def _collate(dicts, cfg, limits):
    b = cfg.backbone
    return registration_collate_fn_stack_mode(dicts, b.num_stages, b.init_voxel_size, b.init_radius, limits)


def _bits(t):
    return t.contiguous().view(torch.int32)


def test_kernels_match_reference_loss_vectors(losses):
    worst = 0.0
    for kind, seed, shape, ls, want in zip(losses['coarse_kind'], losses['coarse_seed'], losses['coarse_shape'], losses['coarse_log_scale'],
                                           losses['coarse_value']):
        rf, sf, gi, go = LO.coarse_case(str(kind), int(seed), tuple(int(v) for v in shape))
        p = LO.coarse_params(float(ls))
        got = GF.coarse_matching_loss(rf.cuda(), sf.cuda(), gi.cuda(), go.cuda(), p.positive_margin, p.negative_margin,
                                      p.positive_optimal, p.negative_optimal, p.log_scale, p.positive_overlap)[1].item()
        e = _rel(got, want)
        assert e <= 1e-5, ('coarse', str(kind), int(seed), got, float(want))
        worst = max(worst, e)
    for kind, seed, shape, want in zip(losses['fine_kind'], losses['fine_seed'], losses['fine_shape'], losses['fine_value']):
        shape = (int(shape[0]), int(shape[1]), float(shape[2]))
        rp, sp, rm, sm, sc, T = (t.cuda() for t in LO.fine_case(str(kind), int(seed), shape))
        got = GF.fine_matching_loss(rp, sp, rm, sm, sc, T, shape[2])[2].item()
        e = _rel(got, want)
        assert e <= 1e-5, ('fine', str(kind), int(seed), got, float(want))
        worst = max(worst, e)
    assert np.isnan(losses['coarse_value']).any() and np.isnan(losses['fine_value']).any()
    print(f'loss vectors: max rel deviation from the reference {worst:.2e}')


@pytest.mark.parametrize('workload,cfg_name,index', [('demo2k', '3dmatch', 0), ('modelnet717', 'modelnet', 0), ('kitti4k', 'kitti', 0),
                                                     ('3dmatch20k', '3dmatch', 0)])
def test_modules_match_restatement_on_forward_outputs(workload, cfg_name, index, models):
    cfg, _, model = models(cfg_name)
    model = model.cuda().eval()
    pair = make_pair(workload, index)
    data = _collate([{k: pair[k] for k in KEYS}], cfg, LIMITS[cfg_name])
    out = model(data)
    got = OverallLoss(cfg)(out, data)
    cpu = {k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in out.items()}
    want = LO.overall_loss(cfg, cpu, data['transform'].cpu())
    errs = {k: _rel(got[k].item(), want[k].item()) for k in NAMES}
    print(f'{workload}: kernels {[round(got[k].item(), 6) for k in NAMES]} vs restatement rel {errs}')
    assert max(errs.values()) <= 1e-5, errs


@pytest.mark.parametrize('workload,cfg_name', [('demo2k', '3dmatch'), ('modelnet717', 'modelnet'), ('kitti4k', 'kitti')])
def test_teacher_forced_losses_match_reference(workload, cfg_name, golden, losses, models):
    """the reference's coarse correspondences forced and its ground-truth pairs substituted: what remains between the kernels'
    losses and the reference's are the features (<= 1e-4 abs) and the Sinkhorn scores (<= 2e-4 abs) of the forward; both enter the
    losses only through means over hundreds of terms, and the measured deviation is <= 1.1e-6 relative (H100), hence 1e-5"""
    cfg, _, model = models(cfg_name)
    model = model.cuda().eval()
    gold = golden(workload)
    pair = make_pair(workload, 0)
    data = _collate([{k: pair[k] for k in KEYS}], cfg, gold['neighbor_limits'].tolist())
    data['forced_node_corr'] = tuple(torch.from_numpy(gold[k]).cuda() for k in ('ref_node_corr_indices', 'src_node_corr_indices',
                                                                                 'node_corr_scores'))
    out = model(data)
    out['gt_node_corr_indices'] = torch.from_numpy(gold['gt_node_corr_indices'].astype(np.int64)).cuda()
    out['gt_node_corr_overlaps'] = torch.from_numpy(gold['gt_node_corr_overlaps'].astype(np.float32)).cuda()
    got = OverallLoss(cfg)(out, data)
    row = list(losses['pairs']).index(f'{workload}:0')
    want = losses['scalars'][row]
    errs = {k: _rel(got[k].item(), want[i]) for i, k in enumerate(NAMES)}
    print(f'{workload} teacher-forced: kernels {[got[k].item() for k in NAMES]} reference {want.tolist()} rel {errs}')
    assert max(errs.values()) <= 1e-5, errs


def _ragged_pairs():
    """demo2k pairs 0 and 1; pair 1 under a transform 100 m off (no ground-truth superpoint pair: c_loss NaN); a small pair whose
    valid superpoint pairs are fewer than num_correspondences (padding patches)"""
    a = {k: make_pair('demo2k', 0)[k] for k in KEYS}
    b = {k: make_pair('demo2k', 1)[k] for k in KEYS}
    b['transform'] = b['transform'].copy()
    b['transform'][:3, 3] += 100.0
    rng = np.random.default_rng(5)
    small = {'ref_points': (rng.random((300, 3)) * 0.25).astype(np.float32), 'src_points': (rng.random((280, 3)) * 0.25).astype(np.float32),
             'ref_feats': np.ones((300, 1), np.float32), 'src_feats': np.ones((280, 1), np.float32), 'transform': np.eye(4, dtype=np.float32)}
    return [a, small, b]


def test_forward_batch_loss_rows_equal_module_losses(models):
    cfg, _, model = models('3dmatch')
    model = model.cuda().eval()
    enable_native(model)
    loss = OverallLoss(cfg)
    dicts = _ragged_pairs()
    B = len(dicts)
    sides = [torch.cuda.Stream() for _ in range(3)]
    outs = model.forward_batch(_collate(dicts, cfg, LIMITS['3dmatch']), side_streams=sides)
    data = _collate(dicts, cfg, LIMITS['3dmatch'])
    res0, res1 = torch.zeros(B, 24, device='cuda'), torch.zeros(B, 24, device='cuda')
    rows, rows2 = torch.zeros(B, 3, device='cuda'), torch.zeros(B, 3, device='cuda')
    from geotransformer_b200.loss import Evaluator
    ev = Evaluator(cfg)
    model.forward_batch(data, evaluator=ev, results=res0, side_streams=sides, keep_outputs=False)
    model.forward_batch(data, evaluator=ev, results=res1, side_streams=sides, keep_outputs=False, loss_func=loss, loss_out=rows)
    model.forward_batch(data, evaluator=ev, results=torch.zeros(B, 24, device='cuda'), side_streams=sides, keep_outputs=False,
                        loss_func=loss, loss_out=rows2)
    torch.cuda.synchronize()
    assert torch.equal(_bits(res0), _bits(res1)), 'the (B, 24) results change with loss_out'
    assert torch.equal(_bits(rows), _bits(rows2)), 'two runs differ'
    assert int(outs[1]['ref_node_corr_indices'].shape[0]) < cfg.coarse_matching.num_correspondences
    assert outs[2]['gt_node_corr_indices'].shape[0] == 0
    for p, o in enumerate(outs):
        t = torch.stack([v for v in loss(o, {'transform': data['transform'][p]}).values()])
        assert torch.equal(_bits(t), _bits(rows[p])), (p, t.tolist(), rows[p].tolist())
    assert torch.isnan(rows[2, 1]).item() and torch.isnan(rows[2, 0]).item()
    assert not torch.isnan(rows[0]).any().item()


def _same(a, b):
    return all((np.isnan(a[k]) and np.isnan(b[k])) or a[k] == b[k] for k in NAMES)


def test_engine_and_tester_report_module_losses(models):
    from geotransformer_b200.engine import RegistrationEngine
    from geotransformer_b200.tester import METRICS, RegistrationTester
    cfg, _, model = models('3dmatch')
    model = model.cuda().eval()
    enable_native(model)
    pairs = [{k: make_pair('demo2k', i)[k] for k in KEYS} for i in range(8)]
    loss = OverallLoss(cfg)
    # module path on the forwards the engine runs
    want1 = []
    for d in pairs:
        data = _collate([d], cfg, cfg.neighbor_limits)
        want1.append(dict(zip(NAMES, loss.loss_tensor(model(data), data).tolist())))
    outs = model.forward_batch(_collate(pairs, cfg, cfg.neighbor_limits), side_streams=[torch.cuda.Stream() for _ in range(4)])
    data8 = _collate(pairs, cfg, cfg.neighbor_limits)
    want8 = [dict(zip(NAMES, loss.loss_tensor(o, {'transform': data8['transform'][p]}).tolist())) for p, o in enumerate(outs)]
    for bs, want in ((1, want1), (8, want8)):
        eng = RegistrationEngine(model, cfg, cfg.neighbor_limits, num_streams=2, loss_func=loss, batch_size=bs)
        got = eng.register(pairs)
        eng.close()
        for p, (g, w) in enumerate(zip(got, want)):
            assert _same(g['loss'], w), (bs, p, g['loss'], w)
    eng = RegistrationEngine(model, cfg, cfg.neighbor_limits, num_streams=2, batch_size=8)
    assert all('loss' not in r for r in eng.register(pairs))
    eng.close()
    tester = RegistrationTester(cfg, model, cfg.neighbor_limits, num_streams=2, with_loss=True)
    summary, per_pair = tester.run(pairs)
    tester.close()
    for e, w in zip(per_pair, want1):
        assert _same(e, w)
    for k in NAMES:
        assert summary[k] == float(np.mean([w[k] for w in want1]))
    tester = RegistrationTester(cfg, model, cfg.neighbor_limits, num_streams=2)
    summary, per_pair = tester.run(pairs[:2])
    tester.close()
    assert set(summary) == set(METRICS) and set(per_pair[0]) == {'metrics', 'num_corr', 'estimated_transform'}
