"""Gradients of the matching heads on the device (Sinkhorn, patch scores, coarse / fine losses): the kernels against torch fp64 autograd
of the oracle restatements (oracle/head_grad_oracle.py) run live on the same inputs, end to end on the product's forward outputs, and
the determinism / padding / bit-identity properties of the backward entry points."""
import numpy as np
import pytest
import torch

from geotransformer_b200 import functional as GF
from geotransformer_b200.loss import OverallLoss
from geotransformer_b200.synth import make_pair
from geotransformer_b200.utils.data import registration_collate_fn_stack_mode
from oracle import head_grad_oracle as HG
from oracle import loss_oracle as LO

pytestmark = pytest.mark.gpu
KEYS = ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')
LIMITS = {'3dmatch': [38, 36, 36, 38], 'modelnet': [13, 21, 27], 'kitti': [27, 75, 147, 157, 119]}


def _bits(t):
    return t.contiguous().view(torch.int32)


def _ref_grads(fn, inputs, dtype):
    """torch autograd of fn on CPU copies of the inputs (floating ones cast to dtype, requiring grad)"""
    leaves = [x.detach().cpu().to(dtype).requires_grad_(True) for x in inputs]
    out = fn(*leaves)
    out.backward()
    return [x.grad for x in leaves]


def _check(name, got, want64, want32, floor=None):
    """max |got - fp64| <= 10 x the fp32 reference autograd's own max error on the input, floor 1e-6 * max |g| (or ``floor``)"""
    got, w64, w32 = got.detach().cpu().double(), want64.double(), want32.double()
    assert torch.isfinite(got).all(), name
    scale = float(w64.abs().max())
    e32 = float((w32 - w64).abs().max()) if torch.isfinite(w32).all() else float('inf')
    tol = max(10.0 * e32, 1e-6 * scale if floor is None else floor)
    if e32 == float('inf'):
        tol = 1e-6 * scale if floor is None else floor
    err = float((got - w64).abs().max())
    print(f'{name}: max err {err:.2e} (fp32 autograd {e32:.2e}, max |g| {scale:.2e})')
    assert err <= tol, (name, err, tol)
    return err


@pytest.mark.parametrize('case', HG.SINKHORN_CASES, ids=lambda c: f'{c[0]}-{c[2][1]}-{c[1]}')
def test_sinkhorn_backward_matches_fp64_autograd(case):
    kind, seed, shape = case
    scores, rm, cm, alpha, g = HG.sinkhorn_case(kind, seed, shape)
    live = ~(~rm).all(1) | ~(~cm).all(1)            # padding patches excluded from the oracle (the reference never builds them)

    def loss(s, a):
        return (HG.sinkhorn(a, s[live], rm[live], cm[live]) * g[live].to(s.dtype)).sum()

    w64 = _ref_grads(loss, [scores, alpha], torch.float64)
    w32 = _ref_grads(loss, [scores, alpha], torch.float32)
    gs, ga = GF.sinkhorn_backward(scores.cuda(), rm.cuda(), cm.cuda(), alpha.cuda(), HG.ITERS, g.cuda())
    if kind == 'upstream':                          # the fp32 reference autograd is NaN here; the kernel follows fp64
        assert not (torch.isfinite(w32[0]).all() and torch.isfinite(w32[1]).all())
    # upstream on masked entries: the fp32 reference is NaN, fp64 carries its rounding of 1e12; measured <= 8.5e-6 of max |g|
    upstream_tol = 2e-5 * float(w64[0].abs().max()) if kind == 'upstream' else None
    _check(f'{kind} dscores', gs[live], w64[0][live], w32[0][live], upstream_tol)
    # dalpha: the same rule; with a NaN fp32 reference (upstream) fp64's rounding of 1e12 bounds it (measured <= 3.9e-4 relative)
    _check(f'{kind} dalpha', ga.reshape(1), w64[1].reshape(1), w32[1].reshape(1), 1e-3 * abs(float(w64[1])) if kind == 'upstream' else None)
    assert not gs[~live].any(), 'padding patches get zero gradient'
    # the hand-derived sweep in fp64 is the same computation as the kernel (same limit on masked lines)
    ds_np, da_np = HG.sinkhorn_backward_np(float(alpha), scores.double().numpy(), rm.numpy(), cm.numpy(), g.double().numpy())
    e_np = np.abs(gs.cpu().double().numpy() - ds_np).max() / np.abs(ds_np).max()
    print(f'{kind} dscores vs the fp64 sweep: {e_np:.2e} of max |g|')
    assert e_np <= 1e-5


def test_sinkhorn_autograd_padding_batch_and_determinism():
    scores, rm, cm, alpha, g = HG.sinkhorn_case('padding', 305, (6, 64))
    scores, rm, cm, alpha, g = (t.cuda() for t in (scores, rm, cm, alpha, g))
    s = scores.clone().requires_grad_(True)
    a = alpha.clone().requires_grad_(True)
    out = GF.sinkhorn(s, rm, cm, a, HG.ITERS)
    with torch.no_grad():
        ref = GF.sinkhorn(scores, rm, cm, alpha, HG.ITERS)
    assert torch.equal(_bits(out.detach()), _bits(ref)), 'forward bits change with grad mode'
    out.backward(g)
    gs, ga = GF.sinkhorn_backward(scores, rm, cm, alpha, HG.ITERS, g)
    gs2, ga2 = GF.sinkhorn_backward(scores, rm, cm, alpha, HG.ITERS, g)
    assert torch.equal(_bits(gs), _bits(s.grad)) and torch.equal(_bits(ga.reshape(1)), _bits(a.grad.reshape(1)))
    assert torch.equal(_bits(gs), _bits(gs2)) and torch.equal(_bits(ga.reshape(1)), _bits(ga2.reshape(1))), 'two runs differ'
    assert not gs[1:3].any() and torch.isfinite(gs).all() and torch.isfinite(ga).all()
    for p in (0, 4):                                # a patch alone gives the bits it gives in the batch
        one, _ = GF.sinkhorn_backward(scores[p:p + 1].contiguous(), rm[p:p + 1].contiguous(), cm[p:p + 1].contiguous(), alpha, HG.ITERS,
                                      g[p:p + 1].contiguous())
        assert torch.equal(_bits(one[0]), _bits(gs[p]))
    ga_pad, = [GF.sinkhorn_backward(scores[1:3].contiguous(), rm[1:3].contiguous(), cm[1:3].contiguous(), alpha, HG.ITERS,
                                    g[1:3].contiguous())[1]]
    assert float(ga_pad) == 0.0


@pytest.mark.parametrize('case', HG.PATCH_CASES, ids=lambda c: f'{c[0]}-{c[1]}')
def test_patch_scores_backward_matches_fp64_autograd(case):
    kind, seed, shape = case
    B, P, k, C, nr, ns = shape
    rf, sf, cp, ri, si, g = HG.patch_case(kind, seed, shape)
    # pair b's indices are local to its cloud: shift them into the stacked tables for the oracle (sentinels to the zero row)
    off_r, off_s = torch.arange(B).repeat_interleave(P)[:, None] * nr, torch.arange(B).repeat_interleave(P)[:, None] * ns
    ri_g = torch.where(ri >= nr, B * nr, ri + off_r)
    si_g = torch.where(si >= ns, B * ns, si + off_s)

    def loss(a, b):
        return (HG.patch_scores(a, b, ri_g, si_g) * g.to(a.dtype)).sum()

    w64 = _ref_grads(loss, [rf, sf], torch.float64)
    w32 = _ref_grads(loss, [rf, sf], torch.float32)
    gr, gs = GF.patch_scores_backward_batched(rf.cuda(), sf.cuda(), cp, ri.cuda(), si.cuda(), g.cuda())
    _check(f'{kind} dref', gr, w64[0], w32[0])
    _check(f'{kind} dsrc', gs, w64[1], w32[1])
    gr2, gs2 = GF.patch_scores_backward_batched(rf.cuda(), sf.cuda(), cp, ri.cuda(), si.cuda(), g.cuda())
    assert torch.equal(_bits(gr), _bits(gr2)) and torch.equal(_bits(gs), _bits(gs2)), 'two runs differ'
    if B > 1:                                       # batched equals per pair, bit for bit
        for b in range(B):
            one_r, one_s = GF.patch_scores_backward_batched(rf[b * nr:(b + 1) * nr].cuda(), sf[b * ns:(b + 1) * ns].cuda(), [nr, ns],
                                                            ri[b * P:(b + 1) * P].cuda(), si[b * P:(b + 1) * P].cuda(),
                                                            g[b * P:(b + 1) * P].cuda())
            assert torch.equal(_bits(one_r), _bits(gr[b * nr:(b + 1) * nr])) and torch.equal(_bits(one_s), _bits(gs[b * ns:(b + 1) * ns]))
    # forward bits with grad on and off
    rfc, sfc = rf.cuda().requires_grad_(True), sf.cuda().requires_grad_(True)
    out = GF.patch_scores_batched(torch.cat([rfc, sfc]), cp, ri.cuda(), si.cuda())
    with torch.no_grad():
        ref = GF.patch_scores_batched(torch.cat([rf, sf]).cuda(), cp, ri.cuda(), si.cuda())
    assert torch.equal(_bits(out.detach()), _bits(ref))
    out.backward(g.cuda())
    assert torch.equal(_bits(rfc.grad), _bits(gr)) and torch.equal(_bits(sfc.grad), _bits(gs))


def _coarse_inputs():
    for kind, seed, shape, ls in LO.COARSE_CASES:
        yield f'{kind}-{seed}', LO.coarse_case(kind, seed, shape), LO.coarse_params(ls)
    yield 'duplicated', HG.duplicated_coarse_case(), LO.coarse_params(24)


def test_coarse_loss_backward_matches_fp64_autograd():
    for name, (rf, sf, gi, go), p in _coarse_inputs():
        w64 = _ref_grads(lambda a, b: HG.coarse_loss(p, a, b, gi, go), [rf, sf], torch.float64)
        w32 = _ref_grads(lambda a, b: HG.coarse_loss(p, a, b, gi, go), [rf, sf], torch.float32)
        a, b = rf.cuda().requires_grad_(True), sf.cuda().requires_grad_(True)
        params = (p.positive_margin, p.negative_margin, p.positive_optimal, p.negative_optimal, p.log_scale, p.positive_overlap)
        val = GF.coarse_matching_loss(a, b, gi.cuda(), go.cuda(), *params)[1]
        with torch.no_grad():
            ref = GF.coarse_matching_loss(rf.cuda(), sf.cuda(), gi.cuda(), go.cuda(), *params)[1]
        assert torch.equal(_bits(val.detach().reshape(1)), _bits(ref.reshape(1))), name
        val.backward()
        for got, want, w_32, side in ((a.grad, w64[0], w32[0], 'ref'), (b.grad, w64[1], w32[1], 'src')):
            got = got.cpu().double()
            fin = torch.isfinite(want)
            assert torch.equal(torch.isfinite(got), fin), (name, side, 'finite / NaN pattern')
            assert torch.equal(torch.isnan(got), torch.isnan(want)), (name, side, 'NaN pattern')
            if fin.any():
                e32 = float((w_32.double() - want)[fin].abs().max())
                err = float((got - want)[fin].abs().max())
                tol = max(10.0 * e32, 1e-6 * float(want[fin].abs().max()))
                print(f'coarse {name} {side}: max err {err:.2e} (fp32 autograd {e32:.2e})')
                assert err <= tol, (name, side, err, tol)
        if name == 'duplicated':
            assert not torch.isfinite(a.grad).all(), 'd = 0 gives a non-finite gradient, as torch autograd does'


def test_fine_loss_backward_matches_fp64_autograd():
    for kind, seed, shape in LO.FINE_CASES:
        rp, sp, rm, sm, sc, T = LO.fine_case(kind, seed, shape)
        w64 = _ref_grads(lambda s: HG.fine_loss(shape[2], rp, sp, rm, sm, s, T), [sc], torch.float64)[0]
        x = sc.cuda().requires_grad_(True)
        val = GF.fine_matching_loss(rp.cuda(), sp.cuda(), rm.cuda(), sm.cuda(), x, T.cuda(), shape[2])[2]
        val.backward()
        err = float((x.grad.cpu().double() - w64).abs().max())
        print(f'fine {kind}-{seed}: max err {err:.2e}')
        assert err <= 1e-6 * max(float(w64.abs().max()), 1e-30) or (err == 0.0), (kind, seed, err)
        want_np = HG.fine_backward_np(shape[2], rp, sp, rm, sm, shape[1] + 1, T)
        assert np.abs(x.grad.cpu().double().numpy() - want_np).max() <= 1e-6 * max(np.abs(want_np).max(), 1e-30) + 0.0


def _collate(dicts, cfg, limits):
    b = cfg.backbone
    return registration_collate_fn_stack_mode(dicts, b.num_stages, b.init_voxel_size, b.init_radius, limits)


@pytest.mark.parametrize('workload,cfg_name', [('demo2k', '3dmatch'), ('modelnet717', 'modelnet'), ('kitti4k', 'kitti'),
                                               ('3dmatch20k', '3dmatch')])
def test_end_to_end_head_gradients_on_forward_outputs(workload, cfg_name, models):
    """features of the product's forward as leaves: patch_scores -> sinkhorn -> OverallLoss -> backward, against the same chain in
    torch fp64 autograd of the oracle on CPU"""
    cfg, _, model = models(cfg_name)
    model = model.cuda().eval()
    pair = make_pair(workload, 0)
    data = _collate([{k: pair[k] for k in KEYS}], cfg, LIMITS[cfg_name])
    taps = {}
    with torch.no_grad():
        out = model(data, taps=taps)
    kk = out['ref_node_corr_indices'].shape[0]
    ri = taps['ref_node_knn_indices'][out['ref_node_corr_indices'][:kk]].contiguous()
    si = taps['src_node_knn_indices'][out['src_node_corr_indices'][:kk]].contiguous()
    rm, sm = out['ref_node_corr_knn_masks'], out['src_node_corr_knn_masks']
    alpha0 = model.optimal_transport.alpha.detach()
    iters = cfg.model.num_sinkhorn_iterations
    T = data['transform']
    leaves0 = [out['ref_feats_c'], out['src_feats_c'], out['ref_feats_f'], out['src_feats_f'], alpha0]

    def chain_gpu(rfc, sfc, rff, sff, a):
        ms = GF.sinkhorn(GF.patch_scores(rff, sff, ri, si), rm, sm, a, iters)
        o = dict(out, ref_feats_c=rfc, src_feats_c=sfc, matching_scores=ms)
        return OverallLoss(cfg)(o, data)['loss']

    leaves = [x.detach().clone().requires_grad_(True) for x in leaves0]
    loss = chain_gpu(*leaves)
    with torch.no_grad():
        loss_ng = chain_gpu(*[x.detach() for x in leaves0])
    assert torch.equal(_bits(loss.detach().reshape(1)), _bits(loss_ng.reshape(1))), 'forward bits change with grad mode'
    loss.backward()
    got = [x.grad for x in leaves]
    leaves2 = [x.detach().clone().requires_grad_(True) for x in leaves0]
    chain_gpu(*leaves2).backward()
    for a, b in zip(got, leaves2):
        assert torch.equal(_bits(a.reshape(-1)), _bits(b.grad.reshape(-1))), 'two runs differ'

    cpu = {k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in out.items()}
    nrf, nsf = out['ref_feats_f'].shape[0], out['src_feats_f'].shape[0]
    ri_c, si_c = ri.cpu().clamp(max=nrf), si.cpu().clamp(max=nsf)

    def chain_cpu(rfc, sfc, rff, sff, a):
        ms = HG.sinkhorn(a, HG.patch_scores(rff, sff, ri_c, si_c), rm.cpu(), sm.cpu(), iters)
        c = HG.coarse_loss(cfg.coarse_loss, rfc, sfc, cpu['gt_node_corr_indices'], cpu['gt_node_corr_overlaps'])
        f = HG.fine_loss(cfg.fine_loss.positive_radius, cpu['ref_node_corr_knn_points'], cpu['src_node_corr_knn_points'],
                         cpu['ref_node_corr_knn_masks'], cpu['src_node_corr_knn_masks'], ms, T.cpu())
        return cfg.loss.weight_coarse_loss * c + cfg.loss.weight_fine_loss * f

    w64 = _ref_grads(chain_cpu, leaves0, torch.float64)
    w32 = _ref_grads(chain_cpu, leaves0, torch.float32)
    for name, g, a, b in zip(('ref_feats_c', 'src_feats_c', 'ref_feats_f', 'src_feats_f', 'alpha'), got, w64, w32):
        _check(f'{workload} {name}', g.reshape(-1), a.reshape(-1), b.reshape(-1))


def test_batched_loss_backward_equals_per_pair():
    """two pairs of fine-loss / coarse-loss inputs in one batched backward give each pair's single-pair gradient bit for bit"""
    cases = [LO.fine_case('random', 200, (6, 64, 0.05)), LO.fine_case('random', 203, (6, 64, 0.6))]
    grads = torch.tensor([[0.3, 1.0, 1.0], [-0.7, 2.0, 0.5]], device='cuda')
    cat = [torch.cat([c[i] for c in cases]).cuda() for i in range(4)]
    Ts = torch.stack([c[5] for c in cases]).cuda()
    gb = GF.fine_matching_loss_backward_batched(2, *cat, Ts, 0.05, grads, loss_weights=(1.0, 1.0))
    for p, c in enumerate(cases):
        g1 = GF.fine_matching_loss_backward_batched(1, *[t.cuda() for t in c[:4]], c[5].cuda(), 0.05, grads[p:p + 1].contiguous(),
                                                    loss_weights=(1.0, 1.0))
        assert torch.equal(_bits(g1), _bits(gb[6 * p:6 * (p + 1)]))
    cc = [LO.coarse_case('mixed', 100, (40, 37, 128)), LO.coarse_case('sparse', 109, (90, 70, 128))]
    p = LO.coarse_params(24)
    params = (p.positive_margin, p.negative_margin, p.positive_optimal, p.negative_optimal, p.log_scale, p.positive_overlap)
    nodes = [40, 90, 37, 70]
    rf = torch.cat([cc[0][0], cc[1][0]]).cuda()
    sf = torch.cat([cc[0][1], cc[1][1]]).cuda()
    gi = torch.zeros((40 * 37 + 90 * 70, 2), dtype=torch.int64)
    go = torch.zeros((40 * 37 + 90 * 70,))
    gi[:cc[0][2].shape[0]], go[:cc[0][3].shape[0]] = cc[0][2], cc[0][3]
    gi[1480:1480 + cc[1][2].shape[0]], go[1480:1480 + cc[1][3].shape[0]] = cc[1][2], cc[1][3]
    cnt = torch.tensor([cc[0][2].shape[0], cc[1][2].shape[0]], dtype=torch.int32, device='cuda')
    gr, gs = GF.coarse_matching_loss_backward_batched(rf, sf, nodes, gi.cuda(), go.cuda(), cnt, params, grads, loss_weights=(1.0, 1.0))
    for q, c in enumerate(cc):
        r1, s1 = GF.coarse_matching_loss_backward_batched(c[0].cuda(), c[1].cuda(), [c[0].shape[0], c[1].shape[0]], c[2].cuda(),
                                                          c[3].cuda(), cnt[q:q + 1].contiguous(), params, grads[q:q + 1].contiguous(),
                                                          loss_weights=(1.0, 1.0))
        r0, s0 = (0, 0) if q == 0 else (40, 37)
        assert torch.equal(_bits(r1), _bits(gr[r0:r0 + c[0].shape[0]])) and torch.equal(_bits(s1), _bits(gs[s0:s0 + c[1].shape[0]]))


def _digest_err(got, want):
    """largest deviation over the parts of a fixture digest, relative to each part's largest magnitude"""
    e = 0.0
    for k, w in want.items():
        g = got[k]
        assert np.array_equal(np.isnan(g), np.isnan(w)), k
        fin = ~np.isnan(w)
        if fin.any():
            e = max(e, float(np.abs(g[fin] - w[fin]).max() / max(np.abs(w[fin]).max(), 1e-30)))
    return e


@pytest.mark.parametrize('workload,cfg_name', [('demo2k', '3dmatch'), ('modelnet717', 'modelnet'), ('kitti4k', 'kitti')])
def test_teacher_forced_head_gradients_match_reference_fixture(workload, cfg_name, golden, models):
    """the reference's coarse correspondences forced and its ground-truth pairs substituted (as test_gpu_loss does for the values):
    the device gradients of OverallLoss w.r.t. the coarse / fine features and alpha against the reference's fp32 autograd on its own
    forward (tests/golden/head_grads.npz).  What remains between them is the forward's features (<= 1e-4 abs vs the reference)."""
    import os
    fx = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'head_grads.npz'))
    cfg, _, model = models(cfg_name)
    model = model.cuda().eval()
    gold = golden(workload)
    pair = make_pair(workload, 0)
    data = _collate([{k: pair[k] for k in KEYS}], cfg, gold['neighbor_limits'].tolist())
    data['forced_node_corr'] = tuple(torch.from_numpy(gold[k]).cuda() for k in ('ref_node_corr_indices', 'src_node_corr_indices',
                                                                                 'node_corr_scores'))
    taps = {}
    with torch.no_grad():
        out = model(data, taps=taps)
    out['gt_node_corr_indices'] = torch.from_numpy(gold['gt_node_corr_indices'].astype(np.int64)).cuda()
    out['gt_node_corr_overlaps'] = torch.from_numpy(gold['gt_node_corr_overlaps'].astype(np.float32)).cuda()
    ri = taps['ref_node_knn_indices'][out['ref_node_corr_indices']].contiguous()
    si = taps['src_node_knn_indices'][out['src_node_corr_indices']].contiguous()
    names = ('ref_feats_c', 'src_feats_c', 'ref_feats_f', 'src_feats_f')
    leaves = [out[k].detach().clone().requires_grad_(True) for k in names]
    alpha = model.optimal_transport.alpha.detach().clone().requires_grad_(True)
    ms = GF.sinkhorn(GF.patch_scores(leaves[2], leaves[3], ri, si), out['ref_node_corr_knn_masks'], out['src_node_corr_knn_masks'], alpha,
                     cfg.model.num_sinkhorn_iterations)
    loss = OverallLoss(cfg)(dict(out, ref_feats_c=leaves[0], src_feats_c=leaves[1], matching_scores=ms), data)['loss']
    loss.backward()
    want_loss = float(fx[f'e2e/{workload}/loss'])
    assert abs(float(loss) - want_loss) <= 1e-5 * abs(want_loss)
    for name, t in zip(names + ('alpha',), [x.grad for x in leaves] + [alpha.grad.reshape(1)]):
        want = {k.split(':')[1]: fx[k] for k in fx.files if k.split(':')[0] == f'e2e/{workload}/{name}'}
        e = _digest_err(HG.digest(t), want)
        print(f'{workload} {name}: max deviation from the reference fixture {e:.2e} of max |g|')
        assert e <= 1e-4, (workload, name, e)        # measured <= 3.8e-5 (H100): the forward's feature differences
