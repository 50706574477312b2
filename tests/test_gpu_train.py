"""The training step on the device: the ground-truth superpoint target sampler against its numpy restatement (both branches, empty
input, uniformity), the gradient guard, ``forward_train`` against the eval forward and the hand-built OverallLoss chain of
tests/test_gpu_transformer_grads.py (and through it the reference's fixture digests), the skipped step, the rebuild of cached and
native weights after a step, and the TrainingEngine's determinism, resumption and convergence."""
import copy
import os

import numpy as np
import pytest
import torch

from geotransformer_b200 import functional as GF
from geotransformer_b200.loss import OverallLoss
from geotransformer_b200.synth import make_pair
from geotransformer_b200.train import TrainingEngine, make_optimizer, optimizer_step
from oracle import backbone_grad_oracle as BV
from oracle import train_oracle as TO
from oracle import transformer_grad_oracle as TG

pytestmark = pytest.mark.gpu

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'transformer_grads.npz')
# the digest tolerances of test_gpu_transformer_grads.py::test_overall_loss_fills_every_parameter, restated: every parameter gradient
# per digest part against the reference's OverallLoss backward, and the transformer parameters alone
OVERALL_TOL = 0.25
OVERALL_TRANSFORMER_TOL = 5e-3


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def _fresh(cfg, sd):
    from geotransformer_b200.model import create_model
    model = create_model(cfg)
    model.load_state_dict(sd, strict=True)
    return model.cuda()


def _cuda_data(data):
    return {k: ([x.cuda() if isinstance(x, torch.Tensor) else x for x in v] if isinstance(v, list) else
                (v.cuda() if isinstance(v, torch.Tensor) else v)) for k, v in data.items()}


def _pair(workload, i=0):
    p = make_pair(workload, i)
    return {k: p[k] for k in ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')}


# ------------------------------------------------------------------------------------------------ sampler

def _gt_rows(rng, cloud_nodes, frac_above):
    """random gt rows of B pairs in the stacked layout of node_correspondences_batched"""
    B = len(cloud_nodes) // 2
    idx, ov = [], []
    for p in range(B):
        nr, ns = cloud_nodes[p], cloud_nodes[B + p]
        e = rng.permutation(nr * ns)                         # every (ref, src) node pair once, in a random order
        r, s = e // ns, e % ns
        o = np.where(rng.random(nr * ns) < frac_above[p], rng.uniform(0.1, 1.0, nr * ns), rng.uniform(0.0, 0.1, nr * ns))
        o[:3] = 0.1                                          # exactly at the threshold: not a candidate (strict)
        idx.append(np.stack([r, s], 1))
        ov.append(o.astype(np.float32))
    return np.concatenate(idx).astype(np.int64), np.concatenate(ov)


def _run_sampler(idx, ov, counts, cloud_nodes, k, seed, iteration, pair_base=0):
    c, s, n = GF.superpoint_targets_batched(torch.from_numpy(idx).cuda(), torch.from_numpy(ov).cuda(),
                                            torch.tensor(counts, dtype=torch.int32).cuda(), cloud_nodes, 0.1, k, seed, iteration,
                                            pair_base=pair_base)
    return c.cpu().numpy(), s.cpu().numpy(), n.cpu().numpy()


def _want(idx, ov, counts, cloud_nodes, k, seed, iteration, pair_base=0):
    B = len(cloud_nodes) // 2
    g0, out = 0, []
    for p in range(B):
        g1 = g0 + cloud_nodes[p] * cloud_nodes[B + p]
        c = counts[p]
        out.append(TO.select_targets(idx[g0:g0 + c], ov[g0:g0 + c], 0.1, k, seed, iteration, pair=pair_base + p))
        g0 = g1
    return out


def _check_sampler(got, want, k):
    c, s, n = got
    B = len(want)
    for p, (wr, ws, wo) in enumerate(want):
        m = len(wr)
        assert n[p] == min(m, k) == m
        assert np.array_equal(c[p, :m], wr) and np.array_equal(c[B + p, :m], ws), p
        assert np.array_equal(s[p, :m].view(np.int32), wo.view(np.int32)), p
        assert np.all(c[p, m:] == -1) and np.all(c[B + p, m:] == -1) and np.all(s[p, m:] == 0)


def test_sampler_keeps_all_candidates_in_gt_order():
    """n <= num_targets: the filtered gt rows in order, bit for bit, honouring the device counts"""
    rng = np.random.default_rng(1)
    cloud_nodes = [20, 31, 30, 17]
    idx, ov = _gt_rows(rng, cloud_nodes, [0.15, 0.2])
    counts = [600, 17 * 31 - 40]
    got = _run_sampler(idx, ov, counts, cloud_nodes, 128, 7351, 1)
    want = _want(idx, ov, counts, cloud_nodes, 128, 7351, 1)
    assert all(0 < len(w[0]) <= 128 for w in want), [len(w[0]) for w in want]
    _check_sampler(got, want, 128)


@pytest.mark.parametrize('seed,iteration,pair_base', [(7351, 1, 0), (7351, 2, 0), (1 << 40, (1 << 33) + 5, 0), (12345, 77, 9)])
def test_sampler_random_branch_matches_the_restatement(seed, iteration, pair_base):
    """n > num_targets: num_targets distinct candidates above the threshold, ascending, bit-identical to oracle/train_oracle.py"""
    rng = np.random.default_rng(seed % 1000 + iteration % 1000)
    cloud_nodes = [40, 64, 3, 50, 70, 5]
    idx, ov = _gt_rows(rng, cloud_nodes, [0.3, 0.5, 1.0])
    counts = [40 * 50, 64 * 70, 3 * 5]
    got = _run_sampler(idx, ov, counts, cloud_nodes, 128, seed, iteration, pair_base)
    want = _want(idx, ov, counts, cloud_nodes, 128, seed, iteration, pair_base)
    assert len(want[0][0]) == 128 and len(want[1][0]) == 128 and len(want[2][0]) < 128
    _check_sampler(got, want, 128)
    c, s, _ = got
    for p in range(2):
        g0 = sum(cloud_nodes[q] * cloud_nodes[3 + q] for q in range(p))
        keys = [tuple(r) for r in idx[g0:g0 + counts[p]].tolist()]
        assert np.all(s[p] > 0.1)
        rows = [keys.index((a, b)) for a, b in zip(c[p].tolist(), c[3 + p].tolist())]
        assert len(set(rows)) == 128 and rows == sorted(rows)


def test_sampler_without_candidates_gives_count_zero():
    rng = np.random.default_rng(3)
    cloud_nodes = [10, 12]
    idx, ov = _gt_rows(rng, cloud_nodes, [0.0])
    ov[:] = 0.05
    c, s, n = _run_sampler(idx, ov, [120], cloud_nodes, 128, 7351, 1)
    assert n[0] == 0 and np.all(c == -1) and np.all(s == 0)
    c, s, n = _run_sampler(idx, ov, [0], cloud_nodes, 128, 7351, 1)
    assert n[0] == 0 and np.all(c == -1)


def test_sampler_draws_uniform_subsets():
    """inclusion frequencies of 300 candidates over 2048 draws of 128 (64 launches of 32 pairs, distinct seeds and pair ids): the
    chi-square statistic with the without-replacement variance N p (1 - p) per cell stays within its 1e-4 tails"""
    from scipy.stats import chi2
    n, k, B = 300, 128, 32
    cloud_nodes = [15] * B + [20] * B
    idx1 = np.stack([np.arange(n) // 20, np.arange(n) % 20], 1).astype(np.int64)
    ov1 = np.full(n, 0.5, dtype=np.float32)
    idx, ov = np.tile(idx1, (B, 1)), np.tile(ov1, B)
    hits = np.zeros(n, dtype=np.int64)
    draws = 0
    for launch in range(64):
        got = _run_sampler(idx, ov, [n] * B, cloud_nodes, k, 1000 + launch, 1, pair_base=launch * B)
        _check_sampler(got, _want(idx, ov, [n] * B, cloud_nodes, k, 1000 + launch, 1, pair_base=launch * B), k)
        c = got[0]
        for p in range(B):
            hits[c[p] * 20 + c[B + p]] += 1
        draws += B
    pr = k / n
    stat = float((((hits - draws * pr) ** 2) / (draws * pr * (1 - pr))).sum())
    lo, hi = chi2.ppf(1e-4, n - 1), chi2.isf(1e-4, n - 1)
    print(f'chi2 {stat:.1f} in [{lo:.1f}, {hi:.1f}]')
    assert lo < stat < hi


# ------------------------------------------------------------------------------------------------ gradient guard

def test_nonfinite_check_finds_every_nan_and_inf():
    g = torch.Generator(device='cuda').manual_seed(5)
    base = [torch.randn(n, device='cuda', generator=g) for n in (1, 3, 1000, 4097, 300001)]
    views = base + [base[3][1:], base[4][2:-3]]                 # unaligned heads and ragged tails
    found = GF.nonfinite_check(views)
    assert found.item() == 0.0
    for t_i, pos in ((0, 0), (2, 999), (3, 1), (4, 150000), (4, 300000), (5, 0), (6, 0)):
        for bad in (float('nan'), float('inf'), float('-inf')):
            t = views[t_i]
            keep = t[pos].clone()
            t[pos] = bad
            assert GF.nonfinite_check(views, found).item() == 1.0, (t_i, pos, bad)
            t[pos] = keep
    assert GF.nonfinite_check(views, found).item() == 0.0


# ------------------------------------------------------------------------------------------------ forward_train

def _eval_corr(model, dc):
    with torch.no_grad():
        out = model(dict(dc))
    kk = out['ref_node_corr_indices'].shape[0]
    return out, (out['ref_node_corr_indices'][:kk].clone(), out['src_node_corr_indices'][:kk].clone(), out['node_corr_scores'][:kk].clone())


@pytest.mark.parametrize('workload,cfg_name', BV.WORKLOADS)
def test_forward_train_gradients_equal_the_hand_built_chain(workload, cfg_name, models):
    """teacher-forced on the eval forward's own coarse correspondences: the loss and every parameter gradient of forward_train equal
    the hand-built chain of test_overall_loss_fills_every_parameter bit for bit, and so agree with the reference's OverallLoss
    backward (fixture digests) under that test's tolerances"""
    cfg, sd, _ = models(cfg_name)
    model = _fresh(cfg, sd).eval()
    data = BV.collate(workload, cfg)
    dc = _cuda_data(data)
    _, forced = _eval_corr(model, dc)
    loss_fn = OverallLoss(cfg)
    out_t = model.forward_train(dict(dc), 7351, 1, targets=forced)
    lt = loss_fn(out_t, dc)
    lt['loss'].backward()
    got = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
    model.zero_grad(set_to_none=True)

    # the hand-built chain
    taps = {}
    with torch.no_grad():
        out = model(dict(dc, forced_node_corr=forced), taps=taps)
    ri = taps['ref_node_knn_indices'][forced[0]].contiguous()
    si = taps['src_node_knn_indices'][forced[1]].contiguous()
    fl = cfg.model.fine_level
    n_ref_f, n_all_f = int(data['lengths'][fl][0]), data['points'][fl].shape[0]
    n0 = int(data['lengths'][-1][0])
    pts = dc['points'][-1]
    feats_list = model.backbone(dc['features'], dc)
    rc, sc = model.transformer(pts[:n0].contiguous(), pts[n0:].contiguous(), feats_list[-1][:n0], feats_list[-1][n0:])
    y = GF.l2_normalize(torch.cat([rc, sc]))
    ms = GF.sinkhorn(GF.patch_scores_batched(feats_list[0], [n_ref_f, n_all_f - n_ref_f], ri, si), out['ref_node_corr_knn_masks'],
                     out['src_node_corr_knn_masks'], model.optimal_transport.alpha, cfg.model.num_sinkhorn_iterations)
    lh = loss_fn(dict(out, ref_feats_c=y[:n0], src_feats_c=y[n0:], matching_scores=ms), dc)
    lh['loss'].backward()
    for key in ('loss', 'c_loss', 'f_loss'):
        assert torch.equal(_bits(lt[key]), _bits(lh[key])), key
    for k, p in model.named_parameters():
        assert torch.equal(_bits(got[k]), _bits(p.grad)), k
    fx = np.load(FIXTURE)
    mine = {k: g for k, g in got.items() if f'overall/{workload}/{k}' in fx}
    assert len(mine) == len(got)
    gmax = max(float(g.abs().max()) for g in mine.values())
    errs = {k: TG.digest_err(g, fx[f'overall/{workload}/{k}'], k, gmax) for k, g in mine.items()}
    worst = max((e, k) for k, e in errs.items())
    worst_tr = max((e, k) for k, e in errs.items() if k.startswith('transformer.'))
    print(f'{workload}: loss {float(lt["loss"]):.6f}; gradients vs the reference fixture per digest part {worst[0]:.2e} ({worst[1]}), '
          f'transformer {worst_tr[0]:.2e} ({worst_tr[1]})')
    assert worst[0] <= OVERALL_TOL and worst_tr[0] <= OVERALL_TRANSFORMER_TOL, (worst, worst_tr)


@pytest.mark.parametrize('workload,cfg_name', BV.WORKLOADS)
def test_forward_train_values_equal_forward(workload, cfg_name, models):
    """grad mode runs the same forward kernels: coarse and fine features, the coarse matching and the gt correspondences of
    forward_train equal the eval forward's bit for bit; the sampled targets are the restatement's draw from the same gt rows"""
    cfg, sd, _ = models(cfg_name)
    model = _fresh(cfg, sd)
    dc = _cuda_data(BV.collate(workload, cfg))
    out, _ = _eval_corr(model, dc)
    t = model.forward_train(dict(dc), 7351, 3)
    cnt = {k: (None if v is None else int(v)) for k, v in t['_counts'].items()}
    for key in ('ref_feats_c', 'src_feats_c', 'ref_feats_f', 'src_feats_f'):
        assert torch.equal(_bits(t[key]), _bits(out[key])), key
    kc = cnt['coarse']
    assert kc == out['ref_node_corr_indices'].shape[0]
    assert torch.equal(t['ref_node_corr_indices'][:kc], out['ref_node_corr_indices'])
    assert torch.equal(t['src_node_corr_indices'][:kc], out['src_node_corr_indices'])
    g = cnt['gt']
    assert torch.equal(t['gt_node_corr_indices'][:g], out['gt_node_corr_indices'])
    assert torch.equal(_bits(t['gt_node_corr_overlaps'][:g]), _bits(out['gt_node_corr_overlaps']))
    wr, ws, wo = TO.select_targets(out['gt_node_corr_indices'].cpu().numpy(), out['gt_node_corr_overlaps'].cpu().numpy(),
                                   cfg.coarse_matching.overlap_threshold, cfg.coarse_matching.num_targets, 7351, 3)
    k = cnt['node_corr']
    assert k == len(wr)
    assert t['ref_node_corr_knn_points'].shape[0] == cfg.coarse_matching.num_targets
    assert np.array_equal(t['node_corr_scores'][:k].cpu().numpy(), wo)
    assert t['matching_scores'].requires_grad and t['ref_feats_c'].requires_grad


def test_forward_train_refuses_several_pairs(models):
    cfg, sd, _ = models('3dmatch')
    model = _fresh(cfg, sd)
    with pytest.raises(ValueError):
        model.forward_train({'batch_size': 2, 'features': torch.zeros(1, device='cuda')}, 1, 1)


# ------------------------------------------------------------------------------------------------ guard and optimizer

def _opt_state(opt):
    return [(_bits(p), _bits(opt.state[p]['exp_avg']), _bits(opt.state[p]['exp_avg_sq']), _bits(opt.state[p]['step']))
            for g in opt.param_groups for p in g['params'] if p in opt.state]


@pytest.mark.parametrize('bad', [float('nan'), float('inf')])
def test_one_nonfinite_gradient_element_skips_the_step(bad, models):
    cfg, sd, _ = models('3dmatch')
    model = _fresh(cfg, sd)
    eng = TrainingEngine(model, cfg, cfg.neighbor_limits)
    pair = _pair('demo2k')
    assert not eng.train_step(pair)['skipped']
    b = cfg.backbone
    from geotransformer_b200.utils.data import registration_collate_fn_stack_mode
    data = registration_collate_fn_stack_mode([pair], b.num_stages, b.init_voxel_size, b.init_radius, cfg.neighbor_limits)
    out = model.forward_train(data, eng.seed, 2)
    eng.loss_func(out, data)['loss'].backward()
    p_bad = dict(model.named_parameters())['transformer.transformer.layers.2.attention.attention.proj_v.weight']
    p_bad.grad[3, 5] = bad
    before = _opt_state(eng.optimizer)
    found = GF.nonfinite_check([p.grad for p in model.parameters()], eng.found_inf)
    optimizer_step(eng.optimizer, found)
    assert found.item() == 1.0
    after = _opt_state(eng.optimizer)
    assert len(before) == len(after) == len(list(model.parameters()))
    for x, y in zip(before, after):
        for a, c in zip(x, y):
            assert torch.equal(a, c)


def test_pair_without_targets_is_skipped_without_fault(models):
    """a ground-truth transform that leaves no overlapping superpoints: zero targets, a NaN fine loss as in the reference, and the
    step is skipped"""
    cfg, sd, _ = models('3dmatch')
    model = _fresh(cfg, sd)
    eng = TrainingEngine(model, cfg, cfg.neighbor_limits)
    eng.train_step(_pair('demo2k'))
    pair = _pair('demo2k')
    pair['transform'] = pair['transform'].copy()
    pair['transform'][:3, 3] += 1000.0
    before = _opt_state(eng.optimizer)
    res = eng.train_step(pair)
    assert res['skipped'] and not np.isfinite(res['f_loss']), res
    assert res['loss'] != res['loss']
    for x, y in zip(before, _opt_state(eng.optimizer)):
        for a, c in zip(x, y):
            assert torch.equal(a, c)
    assert not eng.train_step(_pair('demo2k'))['skipped']


def test_sampler_guard_and_optimizer_step_do_not_synchronise(models):
    cfg, sd, _ = models('3dmatch')
    model = _fresh(cfg, sd)
    opt = make_optimizer(model, cfg)
    for p in model.parameters():
        p.grad = torch.randn_like(p) * 1e-3
    found = torch.zeros((), device='cuda')
    rng = np.random.default_rng(0)
    idx, ov = _gt_rows(rng, [30, 40], [0.5])
    gi, go, gc = torch.from_numpy(idx).cuda(), torch.from_numpy(ov).cuda(), torch.tensor([1200], dtype=torch.int32, device='cuda')
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        GF.superpoint_targets_batched(gi, go, gc, [30, 40], 0.1, 128, 7351, 1)
        GF.nonfinite_check([p.grad for p in model.parameters()], found)
        optimizer_step(opt, found)
        optimizer_step(opt, found)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert found.item() == 0.0


def test_step_then_module_and_native_forwards_equal_a_fresh_model(models):
    """after a step the module forward (version-keyed caches) and validate's native forward (rebuilt drivers) both equal, bit for
    bit, a fresh model loaded with the stepped state_dict"""
    cfg, sd, _ = models('3dmatch')
    model = _fresh(cfg, sd)
    eng = TrainingEngine(model, cfg, cfg.neighbor_limits)
    pairs = [_pair('demo2k', 0), _pair('demo2k', 1)]
    v0 = eng.validate(pairs)                                     # native drivers built on the initial weights
    eng.train_step(pairs[0])
    v1 = eng.validate(pairs)
    fresh = _fresh(cfg, sd)
    fresh.load_state_dict(model.state_dict())
    from geotransformer_b200.engine import RegistrationEngine
    ref = RegistrationEngine(fresh, cfg, cfg.neighbor_limits, loss_func=eng.loss_func, evaluator=eng.evaluator)
    v2 = ref.register(pairs)
    ref.close()
    assert not torch.equal(v0[0]['estimated_transform'], v1[0]['estimated_transform']) or v0[0]['loss'] != v1[0]['loss']
    for a, b in zip(v1, v2):
        assert torch.equal(_bits(a['estimated_transform']), _bits(b['estimated_transform']))
        assert a['loss'] == b['loss'] and a['metrics'] == b['metrics']
    b = cfg.backbone
    from geotransformer_b200.utils.data import registration_collate_fn_stack_mode
    data = registration_collate_fn_stack_mode([pairs[1]], b.num_stages, b.init_voxel_size, b.init_radius, cfg.neighbor_limits)
    native = model.__dict__.pop('_native')
    try:
        with torch.no_grad():
            m = model(dict(data))
    finally:
        model._native = native
    fresh2 = _fresh(cfg, sd)
    fresh2.load_state_dict(model.state_dict())
    with torch.no_grad():
        f = fresh2(dict(data))
    for key in ('ref_feats_c', 'src_feats_c', 'estimated_transform'):
        assert torch.equal(_bits(m[key]), _bits(f[key])), key


# ------------------------------------------------------------------------------------------------ engine

def _params(model):
    return [_bits(p).clone() for p in model.parameters()]


def test_two_runs_from_one_seed_end_bit_identical(models):
    cfg, sd, _ = models('3dmatch')
    pairs = [_pair('demo2k', i % 2) for i in range(5)]
    ends = []
    for _ in range(2):
        model = _fresh(cfg, sd)
        eng = TrainingEngine(model, cfg, cfg.neighbor_limits, seed=11)
        for p in pairs:
            eng.train_step(p)
        ends.append(_params(model))
    assert all(torch.equal(a, b) for a, b in zip(*ends))
    assert not all(torch.equal(a, _bits(b)) for a, b in zip(ends[0], _fresh(cfg, sd).parameters()))


def test_resume_from_a_snapshot_equals_an_uninterrupted_run(models, tmp_path):
    cfg, sd, _ = models('3dmatch')
    pairs = [_pair('demo2k', i % 2) for i in range(4)]
    model = _fresh(cfg, sd)
    eng = TrainingEngine(model, cfg, cfg.neighbor_limits)
    straight = [eng.train_step(p) for p in pairs]
    want = _params(model)
    model = _fresh(cfg, sd)
    eng = TrainingEngine(model, cfg, cfg.neighbor_limits)
    first = [eng.train_step(p) for p in pairs[:2]]
    path = str(tmp_path / 'snapshot.pth.tar')
    eng.save_snapshot(path)
    snap = torch.load(path, map_location='cpu', weights_only=False)
    assert set(snap) == {'epoch', 'iteration', 'model', 'optimizer', 'scheduler'} and snap['iteration'] == 2
    model2 = _fresh(cfg, sd)
    eng2 = TrainingEngine(model2, cfg, cfg.neighbor_limits)
    eng2.load_snapshot(path)
    rest = [eng2.train_step(p) for p in pairs[2:]]
    assert all(torch.equal(a, b) for a, b in zip(want, _params(model2)))
    assert [r['loss'] for r in straight] == [r['loss'] for r in first + rest]


def test_optimizer_state_round_trips_through_a_plain_adam(models):
    cfg, sd, _ = models('3dmatch')
    model = _fresh(cfg, sd)
    eng = TrainingEngine(model, cfg, cfg.neighbor_limits)
    eng.train_step(_pair('demo2k'))
    state = copy.deepcopy(eng.optimizer.state_dict())
    plain = torch.optim.Adam(model.parameters(), lr=cfg.optim.lr, weight_decay=cfg.optim.weight_decay)
    plain.load_state_dict(state)
    back = plain.state_dict()
    # the reference's form: step counts on the host, unfused
    back = dict(back, state={i: dict(s, step=s['step'].cpu()) for i, s in back['state'].items()},
                param_groups=[dict(g, fused=None) for g in back['param_groups']])
    model2 = _fresh(cfg, sd)
    model2.load_state_dict(model.state_dict())
    eng2 = TrainingEngine(model2, cfg, cfg.neighbor_limits)
    from geotransformer_b200.train import fused_optimizer_state
    eng2.optimizer.load_state_dict(fused_optimizer_state(back))
    eng2.iteration = eng.iteration
    a, b = eng.train_step(_pair('demo2k', 1)), eng2.train_step(_pair('demo2k', 1))
    assert a['loss'] == b['loss']
    assert all(torch.equal(x, y) for x, y in zip(_params(model), _params(model2)))


def test_thirty_steps_on_one_pair_lower_the_loss(models):
    cfg, sd, _ = models('3dmatch')
    cfg = copy.deepcopy(cfg)
    cfg.optim.lr = 5e-4
    model = _fresh(cfg, sd)
    eng = TrainingEngine(model, cfg, cfg.neighbor_limits)
    pair = _pair('demo2k')
    losses = [eng.train_step(pair)['loss'] for _ in range(30)]
    print('losses', [round(v, 4) for v in losses])
    assert np.mean(losses[-5:]) < np.mean(losses[:5]), losses
