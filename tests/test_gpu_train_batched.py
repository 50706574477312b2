"""Batched training on the device: ``forward_train_batch`` against the native ``forward_batch`` (bit for bit), the per-pair stages run
alone, the per-pair target draws, the gradient of the mean over pairs against the mean of the single-pair gradients, the loss-weight
kernel against its restatement, masked and skipped steps, no host synchronisation, determinism, resumption and convergence.
The batched gradients are also checked against fp64 autograd of the restatement (oracle/backbone_grad_oracle.py,
oracle/transformer_grad_oracle.py) run on each pair alone and averaged."""
import copy

import numpy as np
import pytest
import torch

from geotransformer_b200 import functional as GF
from geotransformer_b200.model import enable_native
from geotransformer_b200.synth import make_pair
from geotransformer_b200.train import TrainingEngine, optimizer_step
from geotransformer_b200.utils.data import registration_collate_fn_stack_mode
from oracle import backbone_grad_oracle as BV
from oracle import train_oracle as TO
from oracle import transformer_grad_oracle as TG
from test_train_batched_oracle import loss_weights_restated

pytestmark = pytest.mark.gpu

CASES = [('demo2k', '3dmatch', 2), ('demo2k', '3dmatch', 3), ('modelnet717', 'modelnet', 3), ('kitti4k', 'kitti', 4),
         ('3dmatch20k', '3dmatch', 2)]


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def _fresh(cfg, sd):
    from geotransformer_b200.model import create_model
    model = create_model(cfg)
    model.load_state_dict(sd, strict=True)
    return model.cuda()


def _pair(workload, i=0):
    p = make_pair(workload, i)
    return {k: p[k] for k in ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')}


def _collate(cfg, pairs, workload):
    b = cfg.backbone
    return registration_collate_fn_stack_mode(pairs, b.num_stages, b.init_voxel_size, b.init_radius, BV.limits(workload))


def _opt_state(opt):
    return [(_bits(p), _bits(opt.state[p]['exp_avg']), _bits(opt.state[p]['exp_avg_sq']), _bits(opt.state[p]['step']))
            for g in opt.param_groups for p in g['params'] if p in opt.state]


@pytest.mark.parametrize('workload,cfg_name,B', CASES)
def test_forward_bits_equal_the_native_forward_batch(workload, cfg_name, B, models):
    cfg, sd, _ = models(cfg_name)
    model = _fresh(cfg, sd)
    pairs = [_pair(workload, i) for i in range(B)]
    data = _collate(cfg, pairs, workload)
    assert len(set(data['lengths_host'][-1])) > 1                           # ragged pairs
    out = model.forward_train_batch(dict(data), 7351, 5)
    feats_c, feats_f, y_n = out['_features']
    enable_native(model)
    with torch.no_grad():
        want_c = model._native.backbone_forward(data['features'], data)[-1]
        outs = model.forward_batch(dict(data))
    fl = cfg.model.fine_level
    want_f = torch.cat([o['ref_feats_f'] for o in outs] + [o['src_feats_f'] for o in outs])
    want_y = torch.cat([o['ref_feats_c'] for o in outs] + [o['src_feats_c'] for o in outs])
    assert want_f.shape[0] == data['points'][fl].shape[0]
    assert torch.equal(_bits(feats_c), _bits(want_c))
    assert torch.equal(_bits(feats_f), _bits(want_f))
    assert torch.equal(_bits(y_n), _bits(want_y))
    # pair p's targets are the restatement's draw (seed, iteration, pair p) from its own gt rows
    cn = [int(v) for v in data['lengths_host'][-1]]
    gi, go, gc = (t.cpu().numpy() for t in out['_stacked']['gt'])
    counts = out['_counts']['node_corr'].cpu().numpy()
    corr = out['target_corr'].cpu().numpy()
    g0 = 0
    for p in range(B):
        wr, ws, wo = TO.select_targets(gi[g0:g0 + gc[p]], go[g0:g0 + gc[p]], cfg.coarse_matching.overlap_threshold,
                                       cfg.coarse_matching.num_targets, 7351, 5, pair=p)
        g0 += cn[p] * cn[B + p]
        assert counts[p] == len(wr)
        assert np.array_equal(corr[p, :len(wr)], wr) and np.array_equal(corr[B + p, :len(wr)], ws)


@pytest.mark.parametrize('workload,cfg_name,B', CASES)
def test_each_pair_scores_equal_its_stages_run_alone(workload, cfg_name, B, models):
    """pair p's matching scores in the batch = patch scores + Sinkhorn of pair p alone, on the batch's features and targets"""
    cfg, sd, _ = models(cfg_name)
    model = _fresh(cfg, sd)
    data = _collate(cfg, [_pair(workload, i) for i in range(B)], workload)
    with torch.no_grad():
        out = model.forward_train_batch(dict(data), 7351, 2)
    fl, K = cfg.model.fine_level, model.num_points_in_patch
    cn, cf = [int(v) for v in data['lengths_host'][-1]], [int(v) for v in data['lengths_host'][fl]]
    pc, pf = data['points'][-1], data['points'][fl]
    _, feats_f, _ = out['_features']
    corr = out['target_corr']
    kc = corr.shape[1]
    oc, of = np.cumsum([0] + cn), np.cumsum([0] + cf)
    for p in range(B):
        rows_c = lambda t, o: torch.cat([t[o[p]:o[p + 1]], t[o[B + p]:o[B + p + 1]]])
        pts_c, pts_f, ff = rows_c(pc, oc), rows_c(pf, of), rows_c(feats_f, of)
        ncn, ncf = [cn[p], cn[B + p]], [cf[p], cf[B + p]]
        _, _, knn_idx, knn_masks = GF.point_to_node_partition_batched(pts_f, pts_c, ncf, ncn, K)
        c1 = torch.stack([corr[p], corr[B + p]])
        k_idx, k_masks, _ = GF.gather_patches_batched(c1, kc, ncn, ncf, knn_idx, knn_masks, pts_f)
        with torch.no_grad():
            s = model.optimal_transport(GF.patch_scores_batched(ff, ncf, k_idx[:kc], k_idx[kc:]), k_masks[:kc], k_masks[kc:])
        assert torch.equal(_bits(s), _bits(out['matching_scores'][p * kc:(p + 1) * kc])), p


# Bars, restated from the single-pair tests: every gradient's deviation relative to its own largest value, at least 1e-2 of the
# largest gradient (_whole_err).  Whole backbone against fp64 autograd of the restatement: WHOLE_TOL of test_gpu_backbone_grads.py
# (the restatement runs its own forward, so a LeakyReLU pre-activation within the two forwards' rounding difference takes the other
# slope); whole transformer: WHOLE_TOL of test_gpu_transformer_grads.py; the whole chain through OverallLoss: OVERALL_TOL and
# OVERALL_TRANSFORMER_TOL of test_gpu_train.py.
BACKBONE_TOL = 5e-2
TRANSFORMER_TOL = 2e-3
OVERALL_TOL = 0.25
OVERALL_TRANSFORMER_TOL = 5e-3
# the fp64 restatement of the backbone runs on the host: the fixture workloads only
ORACLE_CASES = [('demo2k', '3dmatch', 3), ('modelnet717', 'modelnet', 3), ('kitti4k', 'kitti', 2)]


def _whole_err(got, want, scale):
    return float((got.detach().double() - want.to(got.device).double()).abs().max()) / max(float(want.abs().max()), scale)


def _worst(got, want):
    gmax = max(float(g.abs().max()) for g in want.values())
    return max((_whole_err(got[k], want[k], 1e-2 * gmax), k) for k in want)


def _cpu(data):
    return {k: ([x.cpu() if isinstance(x, torch.Tensor) else x for x in v] if isinstance(v, list) else
                (v.cpu() if isinstance(v, torch.Tensor) else v)) for k, v in data.items()}


def _pair_rows(lens, B, p):
    """(ref rows, src rows) slices of pair p in a stacked level with 2B cloud row counts ``lens``"""
    o = np.cumsum([0] + [int(v) for v in lens])
    return slice(int(o[p]), int(o[p + 1])), slice(int(o[B + p]), int(o[B + p + 1]))


def _stacked_upstream(shapes_of_pair, lens_of_output, B, channels):
    """the upstream gradients of a batch's stacked outputs for the loss (1/B) sum_p sum_i <out_i of pair p, G_{p,i}>, where G_{p,i} =
    backbone_grad_oracle.upstream of pair p's own outputs (the gradient the restatement of pair p alone receives)"""
    ups = []
    for i, (lens, c) in enumerate(zip(lens_of_output, channels)):
        u = torch.zeros((sum(int(v) for v in lens), c), dtype=torch.float32)
        for p in range(B):
            g = BV.upstream(shapes_of_pair[p])[i] / B
            r, s = _pair_rows(lens, B, p)
            nr = r.stop - r.start
            u[r], u[s] = g[:nr], g[nr:]
        ups.append(u.cuda())
    return ups


@pytest.mark.parametrize('workload,cfg_name,B', ORACLE_CASES)
def test_batched_backbone_gradient_matches_fp64_autograd_of_the_mean(workload, cfg_name, B, models):
    """the batched backbone's parameter gradients of the mean over pairs of <outputs of pair p, G_p> against the mean over pairs of
    fp64 autograd of the restatement run on each pair alone"""
    cfg, sd, _ = models(cfg_name)
    model = _fresh(cfg, sd)
    pairs = [_pair(workload, i) for i in range(B)]
    data = _collate(cfg, pairs, workload)
    singles = [_cpu(_collate(cfg, [p], workload)) for p in pairs]
    feats = model.backbone(data['features'], data)
    lvl0 = model.backbone.finest_decoder - 1
    lens = [data['lengths_host'][lvl0 + j] for j in range(len(feats))]
    shapes = [[(int(ln[p]) + int(ln[B + p]), f.shape[1]) for ln, f in zip(lens, feats)] for p in range(B)]
    ups = _stacked_upstream(shapes, lens, B, [f.shape[1] for f in feats])
    sum((f * u).sum() for f, u in zip(feats, ups)).backward()
    keys = [k for k, _ in model.backbone.named_parameters()]
    got = {k: q.grad for k, q in model.backbone.named_parameters()}
    want = {k: torch.zeros_like(g, dtype=torch.float64, device='cpu') for k, g in got.items()}
    for single in singles:
        for k, g in BV.restatement_grads(sd, cfg, single, keys, torch.float64).items():
            want[k] += g / B
    worst = _worst(got, want)
    print(f'{workload} B={B}: batched backbone vs fp64 autograd of the mean over pairs {worst[0]:.2e} ({worst[1]})')
    assert worst[0] <= BACKBONE_TOL, worst


@pytest.mark.parametrize('workload,cfg_name,B', ORACLE_CASES + [('3dmatch20k', '3dmatch', 2)])
def test_stacked_transformer_gradient_matches_fp64_autograd_of_the_mean(workload, cfg_name, B, models):
    """the batched transformer (per-cloud self items, per-pair cross items, one structure-embedding launch) on the batch's own coarse
    features: every transformer parameter's gradient and the coarse-feature gradient of the mean over pairs of <y of pair p, G_p>
    against the mean over pairs of fp64 autograd of the restatement run on each pair alone"""
    cfg, sd, _ = models(cfg_name)
    model = _fresh(cfg, sd)
    data = _collate(cfg, [_pair(workload, i) for i in range(B)], workload)
    with torch.no_grad():
        feats_c = model.backbone(data['features'], data)[-1]
    pts = data['points'][-1]
    cn = [int(v) for v in data['lengths_host'][-1]]
    fc = feats_c.clone().requires_grad_(True)
    tr = model.transformer
    y = tr.forward_stacked(pts, fc, cn)
    c_out = y.shape[1]
    shapes = [[(cn[p], c_out), (cn[B + p], c_out)] for p in range(B)]
    up = torch.zeros_like(y)
    for p in range(B):
        g0, g1 = BV.upstream(shapes[p])
        r, s = _pair_rows(cn, B, p)
        up[r], up[s] = g0.cuda() / B, g1.cuda() / B
    (y * up).sum().backward()
    keys = [k for k, _ in tr.named_parameters()]
    got = dict({k: q.grad for k, q in tr.named_parameters()}, feats=fc.grad)
    want = {k: torch.zeros(g.shape, dtype=torch.float64, device='cuda') for k, g in got.items()}
    for p in range(B):
        r, s = _pair_rows(cn, B, p)
        w = TG.restatement_grads(sd, cfg, pts[r], pts[s], feats_c[r], feats_c[s], keys, torch.float64, device='cuda')
        for k in keys:
            want[k] += w[k] / B
        want['feats'][r], want['feats'][s] = w['ref_feats'] / B, w['src_feats'] / B
    # the single-pair path on the same pairs and features (GeometricTransformer.forward), averaged: batching must not change it, and
    # its own deviation from fp64 on these pairs is what the single-pair bar allows here (the single-pair test measures pair 0 only)
    singles = {k: torch.zeros_like(g) for k, g in got.items()}
    for p in range(B):
        r, s = _pair_rows(cn, B, p)
        rf, sf = feats_c[r].clone().requires_grad_(True), feats_c[s].clone().requires_grad_(True)
        tr.zero_grad(set_to_none=True)
        y0, y1 = tr(pts[r].contiguous(), pts[s].contiguous(), rf, sf)
        g0, g1 = BV.upstream(shapes[p])
        ((y0 * g0.cuda()).sum() + (y1 * g1.cuda()).sum()).backward()
        for k, q in tr.named_parameters():
            singles[k] += q.grad / B
        singles['feats'][r], singles['feats'][s] = rf.grad / B, sf.grad / B
    worst = _worst(got, want)
    worst_single = _worst(singles, want)
    same = _worst(got, singles)
    print(f'{workload} B={B}: batched transformer vs fp64 autograd of the mean over pairs {worst[0]:.2e} ({worst[1]}); the single-pair '
          f'path {worst_single[0]:.2e} ({worst_single[1]}); batched vs single-pair {same[0]:.2e} ({same[1]})')
    assert same[0] <= 1e-4, same
    assert worst[0] <= max(TRANSFORMER_TOL, 1.5 * worst_single[0]), (worst, worst_single)


@pytest.mark.parametrize('workload,cfg_name,B', CASES[1:])
def test_gradient_is_the_mean_of_the_single_pair_gradients(workload, cfg_name, B, models):
    """the whole chain: every parameter's gradient of the batched loss (the mean over pairs) against the mean of the single-pair
    forward_train gradients under the same targets, each gradient relative to its own largest value"""
    cfg, sd, _ = models(cfg_name)
    model = _fresh(cfg, sd)
    pairs = [_pair(workload, i) for i in range(B)]
    data = _collate(cfg, pairs, workload)
    out = model.forward_train_batch(dict(data), 7351, 1)
    rows = model_loss(cfg)(out, data)
    w, _ = GF.batch_loss_weights(rows)
    assert torch.equal(w, torch.full((B,), 1.0 / B, device='cuda'))
    up = torch.zeros_like(rows)
    up[:, 0] = w
    rows.backward(up)
    got = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
    model.zero_grad(set_to_none=True)
    counts, corr, sc = out['_counts']['node_corr'].tolist(), out['target_corr'], out['node_corr_scores']
    want = {k: torch.zeros_like(g) for k, g in got.items()}
    single = []
    for p in range(B):
        dp = _collate(cfg, [pairs[p]], workload)
        n = counts[p]
        o1 = model.forward_train(dp, 7351, 1, targets=(corr[p, :n].contiguous(), corr[B + p, :n].contiguous(), sc[p, :n].contiguous()))
        r1 = model_loss(cfg)(o1, dp)
        single.append(r1.detach())
        r1[0, 0].backward()
        for k, q in model.named_parameters():
            want[k] += q.grad / B
        model.zero_grad(set_to_none=True)
    single = torch.cat(single)
    assert torch.allclose(rows.detach(), single, rtol=1e-4, atol=1e-6), (rows, single)
    worst = _worst(got, want)
    worst_tr = _worst({k: g for k, g in got.items() if k.startswith('transformer.')},
                      {k: g for k, g in want.items() if k.startswith('transformer.')})
    print(f'{workload} B={B}: batched vs mean of single-pair gradients {worst[0]:.2e} ({worst[1]}), transformer {worst_tr[0]:.2e} '
          f'({worst_tr[1]})')
    assert worst[0] <= OVERALL_TOL and worst_tr[0] <= OVERALL_TRANSFORMER_TOL, (worst, worst_tr)


def model_loss(cfg):
    from geotransformer_b200.loss import OverallLoss
    loss = OverallLoss(cfg)
    return loss.graph_rows


def test_loss_weight_kernel_equals_its_restatement():
    g = torch.Generator().manual_seed(3)
    for B, bad in ((1, []), (3, [1]), (4, [0, 3]), (5, [0, 1, 2, 3, 4]), (16, [7])):
        rows = (torch.rand((B, 4), generator=g) * 3).float()
        for p in bad:
            rows[p, p % 3] = float('nan') if p % 2 == 0 else float('inf')
        dev = rows.cuda()
        n_valid = torch.zeros(1, device='cuda')
        found = torch.zeros((), device='cuda')
        w, mean = GF.batch_loss_weights(dev, n_valid=n_valid, found_inf=found)
        ww, wm, wn, wf = loss_weights_restated(rows.numpy())
        assert np.array_equal(w.cpu().numpy().view(np.int32), ww.view(np.int32))
        m = mean.cpu().numpy()
        assert (np.array_equal(m.view(np.int32), wm.view(np.int32)) if wn else np.all(np.isnan(m)))
        assert int(n_valid.item()) == wn and (found.item() == 1.0) == wf


def test_a_pair_far_away_is_masked_not_skipped(models):
    cfg, sd, _ = models('3dmatch')
    model = _fresh(cfg, sd)
    eng = TrainingEngine(model, cfg, cfg.neighbor_limits, batch_size=3)
    pairs = [_pair('demo2k', i) for i in range(3)]
    pairs[1]['transform'] = pairs[1]['transform'].copy()
    pairs[1]['transform'][:3, 3] += 1000.0
    res = eng.train_batch(pairs)
    assert res['masked_pairs'] == 1 and not res['skipped'], res
    a, b = (np.float32(res['per_pair'][p]['loss']) for p in (0, 2))
    assert not np.isfinite(res['per_pair'][1]['loss'])
    assert np.float32(res['loss']) == np.float32(np.float32(0.5) * a + np.float32(0.5) * b)
    assert len(res['per_pair']) == 3 and res['lr'] == cfg.optim.lr * 3


def test_a_batch_without_a_valid_pair_is_skipped(models):
    cfg, sd, _ = models('3dmatch')
    model = _fresh(cfg, sd)
    eng = TrainingEngine(model, cfg, cfg.neighbor_limits, batch_size=2)
    eng.train_batch([_pair('demo2k', 0), _pair('demo2k', 1)])
    bad = [_pair('demo2k', i) for i in range(2)]
    for p in bad:
        p['transform'] = p['transform'].copy()
        p['transform'][:3, 3] += 1000.0
    before = _opt_state(eng.optimizer)
    res = eng.train_batch(bad)
    assert res['skipped'] and res['masked_pairs'] == 2 and res['loss'] != res['loss'], res
    for x, y in zip(before, _opt_state(eng.optimizer)):
        for a, c in zip(x, y):
            assert torch.equal(a, c)


def test_one_nan_gradient_element_skips_the_batched_step(models):
    cfg, sd, _ = models('3dmatch')
    model = _fresh(cfg, sd)
    eng = TrainingEngine(model, cfg, cfg.neighbor_limits, batch_size=2)
    pairs = [_pair('demo2k', 0), _pair('demo2k', 1)]
    assert not eng.train_batch(pairs)['skipped']
    p_bad = dict(model.named_parameters())['backbone.encoder2_1.KPConv.weights']

    def poison(g):
        g = g.clone()
        g.view(-1)[17] = float('nan')
        return g
    h = p_bad.register_hook(poison)
    before = _opt_state(eng.optimizer)
    try:
        res = eng.train_batch(pairs)
    finally:
        h.remove()
    assert res['skipped'] and res['masked_pairs'] == 0, res
    for x, y in zip(before, _opt_state(eng.optimizer)):
        for a, c in zip(x, y):
            assert torch.equal(a, c)


def test_batched_step_does_not_synchronise(models):
    cfg, sd, _ = models('3dmatch')
    model = _fresh(cfg, sd)
    eng = TrainingEngine(model, cfg, cfg.neighbor_limits, batch_size=2)
    pairs = [_pair('demo2k', 0), _pair('demo2k', 1)]
    eng.train_batch(pairs)                                           # caches, workspaces and guard tables exist
    data = _collate(cfg, pairs, 'demo2k')
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = model.forward_train_batch(data, eng.seed, 9)
        rows = eng.loss_func.graph_rows(out, data)
        w, mean = GF.batch_loss_weights(rows, found_inf=eng.found_inf)
        up = torch.zeros_like(rows)
        up[:, 0].copy_(w)
        rows.backward(up)
        GF.nonfinite_check([p.grad for p in model.parameters() if p.grad is not None] + [mean], eng.found_inf)
        optimizer_step(eng.optimizer, eng.found_inf)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert eng.found_inf.item() == 0.0


def _params(model):
    return [_bits(p).clone() for p in model.parameters()]


def test_two_batched_runs_from_one_seed_end_bit_identical(models):
    cfg, sd, _ = models('3dmatch')
    pairs = [_pair('demo2k', i % 3) for i in range(5)]
    ends = []
    for _ in range(2):
        model = _fresh(cfg, sd)
        eng = TrainingEngine(model, cfg, cfg.neighbor_limits, seed=11, batch_size=2)
        res = eng.train_epoch(pairs)
        assert [len(r['per_pair']) for r in res] == [2, 2, 1] and eng.iteration == 3
        ends.append(_params(model))
    assert all(torch.equal(a, b) for a, b in zip(*ends))


def test_resume_after_a_batched_step_equals_an_uninterrupted_run(models, tmp_path):
    cfg, sd, _ = models('3dmatch')
    pairs = [_pair('demo2k', i % 3) for i in range(5)]
    model = _fresh(cfg, sd)
    eng = TrainingEngine(model, cfg, cfg.neighbor_limits, batch_size=2)
    straight = [eng.train_batch(pairs[i:i + 2]) for i in (0, 2, 4)]
    want = _params(model)
    model = _fresh(cfg, sd)
    eng = TrainingEngine(model, cfg, cfg.neighbor_limits, batch_size=2)
    first = [eng.train_batch(pairs[:2])]
    path = str(tmp_path / 'snapshot.pth.tar')
    eng.save_snapshot(path)
    model2 = _fresh(cfg, sd)
    eng2 = TrainingEngine(model2, cfg, cfg.neighbor_limits, batch_size=2)
    eng2.load_snapshot(path)
    assert eng2.iteration == 1
    rest = [eng2.train_batch(pairs[i:i + 2]) for i in (2, 4)]
    assert all(torch.equal(a, b) for a, b in zip(want, _params(model2)))
    assert [r['loss'] for r in straight] == [r['loss'] for r in first + rest]


def test_thirty_batched_steps_lower_the_loss(models):
    cfg, sd, _ = models('3dmatch')
    cfg = copy.deepcopy(cfg)
    cfg.optim.lr = 5e-4 / 4
    model = _fresh(cfg, sd)
    eng = TrainingEngine(model, cfg, cfg.neighbor_limits, batch_size=4)
    pairs = [_pair('demo2k', i) for i in range(4)]
    losses = [eng.train_batch(pairs)['loss'] for _ in range(30)]
    print('losses', [round(v, 4) for v in losses])
    assert np.mean(losses[-5:]) < np.mean(losses[:5]), losses
