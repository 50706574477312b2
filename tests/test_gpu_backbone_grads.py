"""Gradients of the KPConv-FPN backbone on the device (KPConv, Linear, GroupNorm, max-pool, upsample + concat): every kernel against
torch fp64 autograd of the oracle restatement (oracle/geo_oracle.py) on the same inputs, the whole backbone of three configs against
fp64 autograd and against the reference's fixture (tests/golden/backbone_grads.npz), the fine-matching path end to end, and the
determinism / bit-identity properties of the backward entry points."""
import copy
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from geotransformer_b200 import functional as GF
from geotransformer_b200.modules.kpconv.modules import default_kernel_points
from oracle import geo_oracle as G
from oracle import head_grad_oracle as HG
from oracle import backbone_grad_oracle as BV

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.contiguous().view(torch.int32)


def _ref_grads(fn, inputs, dtype):
    """torch autograd of fn on CPU copies of the inputs (floating ones cast to dtype, requiring grad)"""
    leaves = [x.detach().cpu().to(dtype).requires_grad_(True) for x in inputs]
    fn(*leaves).backward()
    return [x.grad for x in leaves]


def _check(name, got, want64, want32, floor=None):
    """max |got - fp64| <= 10 x the fp32 reference autograd's own max error on the input, floor 1e-6 * max |g| (or ``floor``)"""
    got, w64, w32 = got.detach().cpu().double(), want64.double(), want32.double()
    assert got.shape == w64.shape, (name, tuple(got.shape), tuple(w64.shape))
    assert torch.isfinite(got).all(), name
    scale = float(w64.abs().max())
    e32 = float((w32 - w64).abs().max())
    tol = max(10.0 * e32, 1e-6 * scale if floor is None else floor)
    err = float((got - w64).abs().max())
    print(f'{name}: max err {err:.2e} (fp32 autograd {e32:.2e}, max |g| {scale:.2e})')
    assert err <= tol, (name, err, tol)
    return err


def _neighbours(seed, m, ns, h, n_far=0, pad_rows=0):
    """q (m, 3), s (ns + n_far, 3), nbr (m, h): the h nearest support points of each query; the last ``pad_rows`` rows keep only
    their first 5 neighbours and pad with the sentinel; the n_far support rows lie far away and are never referenced"""
    g = torch.Generator().manual_seed(seed)
    s = torch.rand(ns, 3, generator=g)
    q = s[torch.randperm(ns, generator=g)[:m]] + 0.01 * torch.randn(m, 3, generator=g)
    nbr = torch.cdist(q.double(), s.double()).topk(h, largest=False).indices
    s = torch.cat([s, 10.0 + torch.rand(n_far, 3, generator=g)])
    ntot = s.shape[0]
    if pad_rows:
        nbr[-pad_rows:, 5:] = ntot
    return q, s, nbr.contiguous(), ntot


@pytest.mark.parametrize('case', [('tc', 200, 64, 64), ('fallback', 40, 32, 32), ('c1', 150, 1, 64), ('tc-wide', 96, 128, 256)],
                         ids=lambda c: c[0])
def test_kpconv_backward_matches_fp64_autograd(case):
    kind, m, cin, cout = case
    h, radius, sigma = 20, 0.25, 0.2
    q, s, nbr, ns = _neighbours(11 + cin, m, 500, h, n_far=7, pad_rows=9)
    g = torch.Generator().manual_seed(5 + cout)
    feats = torch.randn(ns, cin, generator=g) if cin > 1 else torch.rand(ns, 1, generator=g) + 0.5
    W = torch.randn(15, cin, cout, generator=g) / (15 * cin) ** 0.5
    b = 0.1 * torch.randn(cout, generator=g)
    kp = default_kernel_points(15, radius, seed=3)
    up = torch.randn(m, cout, generator=g)

    def loss(f, w, bb):
        sd = {'kernel_points': kp.to(f.dtype), 'weights': w, 'bias': bb}
        return (G.kpconv(sd, '', f, q.to(f.dtype), s.to(f.dtype), nbr, sigma) * up.to(f.dtype)).sum()

    w64 = _ref_grads(loss, [feats, W, b], torch.float64)
    w32 = _ref_grads(loss, [feats, W, b], torch.float32)
    fc, Wc, bc = (x.cuda().requires_grad_(True) for x in (feats, W, b))
    out = GF.kpconv(fc, q.cuda(), s.cuda(), nbr.cuda(), kp.cuda(), Wc, bc, sigma)
    with torch.no_grad():
        ref = GF.kpconv(fc, q.cuda(), s.cuda(), nbr.cuda(), kp.cuda(), Wc, bc, sigma)
    assert torch.equal(_bits(out.detach()), _bits(ref)), 'forward bits change with grad mode'
    out.backward(up.cuda())
    _check(f'kpconv {kind} dW', Wc.grad, w64[1], w32[1])
    _check(f'kpconv {kind} db', bc.grad, w64[2], w32[2])
    _check(f'kpconv {kind} dfeats', fc.grad, w64[0], w32[0])
    assert not fc.grad[500:].any(), 'support rows no query references get zero gradient'
    gf, gw, gb = GF.kpconv_backward(fc, q.cuda(), s.cuda(), nbr.cuda(), kp.cuda(), Wc, sigma, up.cuda())
    assert torch.equal(_bits(gw), _bits(Wc.grad)) and torch.equal(_bits(gb), _bits(bc.grad)), 'two runs differ'
    assert torch.equal(_bits(gf), _bits(fc.grad)), 'two runs differ'


def test_linear_backward_column_slice():
    g = torch.Generator().manual_seed(21)
    xf = torch.randn(300, 96, generator=g)
    W = torch.randn(48, 64, generator=g) / 8
    b = torch.randn(48, generator=g)
    up = torch.randn(300, 48, generator=g)

    def loss(x, w, bb):
        return (F.linear(x[:, 16:80], w, bb) * up.to(x.dtype)).sum()

    w64 = _ref_grads(loss, [xf, W, b], torch.float64)
    w32 = _ref_grads(loss, [xf, W, b], torch.float32)
    xc, Wc, bc = (t.cuda().requires_grad_(True) for t in (xf, W, b))
    out = GF.linear(xc[:, 16:80], Wc, bc)
    with torch.no_grad():
        ref = GF.linear(xc[:, 16:80], Wc, bc)
    assert torch.equal(_bits(out.detach()), _bits(ref))
    out.backward(up.cuda())
    for name, got, a, c in (('dx', xc.grad, w64[0], w32[0]), ('dW', Wc.grad, w64[1], w32[1]), ('db', bc.grad, w64[2], w32[2])):
        _check(f'linear {name}', got, a, c)


def test_linear_backward_relu_and_out():
    """the ReLU variant is differentiable (the gradient passes where the output is positive), and ``out=`` carries the graph"""
    g = torch.Generator().manual_seed(23)
    x = torch.randn(200, 64, generator=g)
    W = torch.randn(96, 64, generator=g) / 8
    b = torch.randn(96, generator=g)
    up = torch.randn(200, 96, generator=g)
    w64 = _ref_grads(lambda a, w, bb: (F.relu(F.linear(a, w, bb)) * up.to(a.dtype)).sum(), [x, W, b], torch.float64)
    w32 = _ref_grads(lambda a, w, bb: (F.relu(F.linear(a, w, bb)) * up.to(a.dtype)).sum(), [x, W, b], torch.float32)
    xc, Wc, bc = (t.cuda().requires_grad_(True) for t in (x, W, b))
    out = GF.linear(xc, Wc, bc, relu=True)
    with torch.no_grad():
        ref = GF.linear(xc, Wc, bc, relu=True)
    assert torch.equal(_bits(out.detach()), _bits(ref))
    out.backward(up.cuda())
    for name, got, a, c in (('dx', xc.grad, w64[0], w32[0]), ('dW', Wc.grad, w64[1], w32[1]), ('db', bc.grad, w64[2], w32[2])):
        _check(f'linear relu {name}', got, a, c)
    grads = [t.grad.clone() for t in (xc, Wc, bc)]
    for t in (xc, Wc, bc):
        t.grad = None
    buf = torch.zeros(300, 96, device='cuda')
    GF.linear(xc, Wc, bc, relu=True, out=buf[50:250])
    assert torch.equal(_bits(buf[50:250].detach()), _bits(ref)) and buf.requires_grad
    (buf[50:250] * up.cuda()).sum().backward()
    for a, t in zip(grads, (xc, Wc, bc)):
        assert torch.equal(_bits(a), _bits(t.grad)), 'out= gives the same gradients'


@pytest.mark.parametrize('workload,cfg_name', BV.WORKLOADS)
def test_head_gradient_at_fine_features_matches_reference_fixture(workload, cfg_name, golden, models):
    """the gradient the matching heads hand to the backbone's fine output: the reference's coarse correspondences forced (as
    test_gpu_head_grads does), OverallLoss backward to ref_feats_f / src_feats_f, stacked as feats_list[0], against the reference's
    OverallLoss backward at feats_list[0] (tests/golden/backbone_grads.npz), every digest part relative to its own largest value"""
    from geotransformer_b200.loss import OverallLoss
    cfg, _, model0 = models(cfg_name)
    model = copy.deepcopy(model0).cuda().eval()
    gold = golden(workload)
    data = BV.collate(workload, cfg)
    data['forced_node_corr'] = tuple(torch.from_numpy(gold[k]).cuda() for k in ('ref_node_corr_indices', 'src_node_corr_indices',
                                                                                 'node_corr_scores'))
    taps = {}
    with torch.no_grad():
        out = model(_cuda_data(data), taps=taps)
    out['gt_node_corr_indices'] = torch.from_numpy(gold['gt_node_corr_indices'].astype(np.int64)).cuda()
    out['gt_node_corr_overlaps'] = torch.from_numpy(gold['gt_node_corr_overlaps'].astype(np.float32)).cuda()
    ri = taps['ref_node_knn_indices'][out['ref_node_corr_indices']].contiguous()
    si = taps['src_node_knn_indices'][out['src_node_corr_indices']].contiguous()
    rf, sf = (out[k].detach().clone().requires_grad_(True) for k in ('ref_feats_f', 'src_feats_f'))
    ms = GF.sinkhorn(GF.patch_scores(rf, sf, ri, si), out['ref_node_corr_knn_masks'], out['src_node_corr_knn_masks'],
                     model.optimal_transport.alpha.detach(), cfg.model.num_sinkhorn_iterations)
    OverallLoss(cfg)(dict(out, matching_scores=ms), dict(data, transform=data['transform'].cuda()))['loss'].backward()
    fx = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'backbone_grads.npz'))
    g = torch.cat([rf.grad, sf.grad])
    e = BV.digest_err(g, fx[f'overall/{workload}/feats_f'], 1e-6 * float(g.abs().max()))
    print(f'{workload}: gradient at feats_list[0] vs the reference fixture, per digest part {e:.2e}')
    assert e <= 1e-4, (workload, e)         # measured <= 3.6e-6 (H100): what remains is the forward's features


@pytest.mark.parametrize('channels,groups,residual,slope', [(32, 32, True, 0.1), (32, 32, False, None), (128, 32, True, 0.1),
                                                            (128, 32, False, 0.1), (256, 8, True, None)])
def test_group_norm_backward_matches_fp64_autograd(channels, groups, residual, slope):
    g = torch.Generator().manual_seed(channels + groups)
    n = 700
    x = 2.0 * torch.randn(n, channels, generator=g) + 0.5
    w = 1.0 + 0.3 * torch.randn(channels, generator=g)
    b = 0.2 * torch.randn(channels, generator=g)
    r = torch.randn(n, channels, generator=g)
    up = torch.randn(n, channels, generator=g)

    def loss(xx, ww, bb, rr):
        y = G.group_norm({'norm.weight': ww, 'norm.bias': bb}, '', xx, groups)
        if residual:
            y = y + rr
        if slope is not None:
            y = F.leaky_relu(y, slope)
        return (y * up.to(xx.dtype)).sum()

    w64 = _ref_grads(loss, [x, w, b, r], torch.float64)
    w32 = _ref_grads(loss, [x, w, b, r], torch.float32)
    xc, wc, bc, rc = (t.cuda().requires_grad_(True) for t in (x, w, b, r))
    out = GF.group_norm(xc, wc, bc, groups, negative_slope=slope, residual=rc if residual else None)
    with torch.no_grad():
        ref = GF.group_norm(xc, wc, bc, groups, negative_slope=slope, residual=rc if residual else None)
    assert torch.equal(_bits(out.detach()), _bits(ref))
    out.backward(up.cuda())
    tag = f'gn C={channels} G={groups}'
    _check(f'{tag} dx', xc.grad, w64[0], w32[0])
    _check(f'{tag} dgamma', wc.grad, w64[1], w32[1])
    _check(f'{tag} dbeta', bc.grad, w64[2], w32[2])
    if residual:
        _check(f'{tag} dres', rc.grad, w64[3], w32[3])


def test_group_norm_backward_two_pairs_equal_one_pair_calls():
    g = torch.Generator().manual_seed(77)
    rows = [300, 170, 260, 90]                      # [ref_1, ref_2, src_1, src_2]
    x = torch.randn(sum(rows), 64, generator=g).cuda()
    w = (1.0 + 0.2 * torch.randn(64, generator=g)).cuda()
    b = torch.randn(64, generator=g).cuda()
    dy = torch.randn(sum(rows), 64, generator=g).cuda()
    y = GF.group_norm_batched(x, w, b, 16, rows, negative_slope=0.1)
    gx, gw, gb, gr = GF.group_norm_backward_batched(x, y, w, 16, rows, dy, negative_slope=0.1, need_residual=True)
    starts = np.cumsum([0] + rows)
    gw_sum = torch.zeros(64, dtype=torch.float64, device='cuda')
    for p in range(2):
        sl = [slice(starts[p], starts[p + 1]), slice(starts[2 + p], starts[3 + p])]
        xp, yp, dyp = (torch.cat([t[s] for s in sl]).contiguous() for t in (x, y, dy))
        gx1, gw1, _, gr1 = GF.group_norm_backward_batched(xp, yp, w, 16, [rows[p], rows[2 + p]], dyp, negative_slope=0.1, need_residual=True)
        assert torch.equal(_bits(gx1), _bits(torch.cat([gx[s] for s in sl])))
        assert torch.equal(_bits(gr1), _bits(torch.cat([gr[s] for s in sl])))
        gw_sum += gw1.double()
    assert float((gw_sum - gw.double()).abs().max()) <= 1e-5 * float(gw.abs().max())
    gx2, gw2, gb2, _ = GF.group_norm_backward_batched(x, y, w, 16, rows, dy, negative_slope=0.1)
    assert torch.equal(_bits(gx2), _bits(gx)) and torch.equal(_bits(gw2), _bits(gw)) and torch.equal(_bits(gb2), _bits(gb))


def test_maxpool_backward_shadow_winner_and_pair_cut():
    q, s, nbr, ns = _neighbours(41, 120, 300, 12, n_far=3, pad_rows=20)
    g = torch.Generator().manual_seed(42)
    x = torch.randn(ns, 64, generator=g)
    x[nbr[-20:, :5].reshape(-1)] = -x[nbr[-20:, :5].reshape(-1)].abs() - 0.1   # padded rows: every real entry < 0, the shadow wins
    up = torch.randn(120, 64, generator=g)
    w64 = _ref_grads(lambda t: (G.maxpool(t, nbr) * up.to(t.dtype)).sum(), [x], torch.float64)[0]
    w32 = _ref_grads(lambda t: (G.maxpool(t, nbr) * up.to(t.dtype)).sum(), [x], torch.float32)[0]
    xc = x.cuda().requires_grad_(True)
    out = GF.maxpool(xc, nbr.cuda())
    out.backward(up.cuda())
    _check('maxpool', xc.grad, w64, w32)
    # two pairs in one table: pair 0's rows may only use its own width (8 columns), pair 1's all 12
    rows = [30, 40, 20, 30]
    nb2 = nbr.clone()
    p0 = torch.cat([torch.arange(0, 30), torch.arange(70, 90)])
    nb2[p0, 8:] = ns
    nb2[p0[:10], 8:] = nbr[p0[:10], 8:]               # ... except that these rows carry entries past the cut, which must not exist
    cloud_max = torch.tensor([8, 12, 8, 12], dtype=torch.int32, device='cuda')

    def cut_pool(t):
        pooled = G.maxpool(t, nb2)
        pooled0 = G.maxpool(t, nb2[:, :8])
        mask = torch.zeros(120, 1, dtype=torch.bool)
        mask[p0] = True
        return (torch.where(mask, pooled0, pooled) * up.to(t.dtype)).sum()

    c64 = _ref_grads(cut_pool, [x], torch.float64)[0]
    c32 = _ref_grads(cut_pool, [x], torch.float32)[0]
    gx = GF.maxpool_backward_batched(x.cuda(), nb2.cuda(), rows, up.cuda(), cloud_max=cloud_max)
    _check('maxpool cut', gx, c64, c32)
    assert torch.equal(_bits(gx), _bits(GF.maxpool_backward_batched(x.cuda(), nb2.cuda(), rows, up.cuda(), cloud_max=cloud_max)))


def test_upsample_concat_backward_with_sentinels():
    g = torch.Generator().manual_seed(61)
    ns, m = 90, 400
    x = torch.randn(ns, 48, generator=g)
    skip = torch.randn(m, 16, generator=g)
    up = torch.randint(0, ns - 10, (m, 3), generator=g)          # coarse rows ns-10.. are never copied
    up[::17, 0] = ns                                             # sentinel: the zero row
    gy = torch.randn(m, 64, generator=g)

    def loss(a, b):
        return (torch.cat([G.nearest_upsample(a, up), b], 1) * gy.to(a.dtype)).sum()

    w64 = _ref_grads(loss, [x, skip], torch.float64)
    w32 = _ref_grads(loss, [x, skip], torch.float32)
    xc, sc = x.cuda().requires_grad_(True), skip.cuda().requires_grad_(True)
    out = GF.upsample_concat(xc, up.cuda(), sc)
    out.backward(gy.cuda())
    _check('upsample dx', xc.grad, w64[0], w32[0])
    assert torch.equal(sc.grad.cpu(), gy[:, 48:]), 'the skip half is a copy'
    assert not xc.grad[ns - 10:].any()


def _cuda_data(data):
    return {k: ([x.cuda() if isinstance(x, torch.Tensor) else x for x in v] if isinstance(v, list) else
                (v.cuda() if isinstance(v, torch.Tensor) else v)) for k, v in data.items()}


@pytest.mark.parametrize('workload,cfg_name', BV.WORKLOADS)
def test_backbone_gradients_match_fp64_autograd_and_reference_fixture(workload, cfg_name, models):
    cfg, sd, model0 = models(cfg_name)
    model = copy.deepcopy(model0).cuda()
    data = BV.collate(workload, cfg)
    dc = _cuda_data(data)
    feats_list = model.backbone(dc['features'], dc)
    with torch.no_grad():
        ref = model.backbone(dc['features'], dc)
    for a, b in zip(feats_list, ref):
        assert torch.equal(_bits(a.detach()), _bits(b)), 'forward bits change with grad mode'
    ups = BV.upstream([tuple(f.shape) for f in feats_list])
    sum(((f * u.cuda()).sum() for f, u in zip(feats_list, ups))).backward()
    params = _backbone_params(model)
    assert all(p.grad is not None for _, p in params)
    got = {k: p.grad.detach().clone() for k, p in params}
    for _, p in params:                             # two runs give the same bits
        p.grad = None
    sum(((f * u.cuda()).sum() for f, u in zip(model.backbone(dc['features'], dc), ups))).backward()
    for k, p in params:
        assert torch.equal(_bits(p.grad), _bits(got[k])), ('two runs differ', k)
    # a third run with the blocks tapped (their inputs aliased: autograd then sums a skip connection's gradients in another order)
    taps = _tap_blocks(model)
    for _, p in params:
        p.grad = None
    sum(((f * u.cuda()).sum() for f, u in zip(model.backbone(dc['features'], dc), ups))).backward()
    blocks = {name: (t['args'], t['out'], t['inner'], t['out'].grad, t['args'][0].grad) for name, t in taps['blocks'].items()}
    tapped = {k: p.grad.detach().clone() for k, p in params}
    _check_blocks_in_chain(workload, model, sd, cfg, blocks, tapped)
    # the whole backbone against fp64 autograd of the restatement and against the reference's own fp32 autograd (fixture digests).
    # Both run their own forward: where a pre-activation of the LeakyReLU lies within the forwards' rounding difference the
    # derivative itself differs, so these bound the sum of those, not rounding.  fp64: deviations relative to the parameter's largest
    # gradient, and at least 1e-2 of the backbone's largest.  Fixture: every digest part (sums, samples, slice sums or the whole
    # tensor) relative to its own largest value, at least FIXTURE_FLOOR of the backbone's largest gradient (the gradients of the
    # biases feeding a GroupNorm with one channel per group are rounding noise around zero).
    keys = [k for k, _ in params]
    w64 = BV.restatement_grads(sd, cfg, data, keys, torch.float64)
    fx = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'backbone_grads.npz'))
    gmax = max(float(g.abs().max()) for g in got.values())
    worst64 = max(_whole_err(got[k], w64[k], 1e-2 * gmax) for k in keys)
    worst_fx = max((BV.digest_err(got[k], fx[f'{workload}/{k}'], FIXTURE_FLOOR * gmax), k) for k in keys)
    print(f'{workload}: whole backbone vs fp64 autograd {worst64:.2e}, vs the reference fixture per digest part {worst_fx[0]:.2e} '
          f'({worst_fx[1]})')
    assert worst64 <= WHOLE_TOL, (workload, worst64)
    assert worst_fx[0] <= FIXTURE_TOL, (workload, worst_fx)


def _check_blocks_in_chain(workload, model, sd, cfg, blocks, got):
    """every block inside the chain, at the product's own activations and upstream gradient: its parameter gradients and its input
    gradient against fp64 autograd of the restatement's block, under the 10 x fp32-autograd rule.  The restated block runs its own
    forward, so an element whose LeakyReLU pre-activation lies within the two forwards' rounding difference would take the other
    slope (measured on kitti4k's level 4: one element at |t| = 7e-7, 0.69 of a max |g| of 4.9 in d input); so every LeakyReLU of
    the restated block takes the branch the product's took.  The max-pool reads the same input in both, so its winners agree.
    The bias of a layer feeding a GroupNorm receives a row sum whose group sums cancel exactly, so its error follows the block's
    gradient scale rather than its own: the floor is BIAS_FLOOR of the block's largest parameter gradient (measured on an H100: one
    parameter of 632 above 10 x the fp32 autograd error, kitti4k decoder4.mlp.bias at 12.9 x = 6.4e-7 of the block's largest)."""
    for name, (args, y_prod, inner, g_out, g_in) in blocks.items():
        pre = f'backbone.{name}.'
        keys = [k for k in got if k.startswith(name + '.')]

        def block_loss(x, *ws, args=args, y_prod=y_prod, inner=inner, g_out=g_out, pre=pre, keys=keys, name=name):
            sdb = {k: (v.to(x.dtype) if v.is_floating_point() else v) for k, v in sd.items() if k.startswith(pre)}
            sdb.update({'backbone.' + k: w for k, w in zip(keys, ws)})
            return (_restated_block(model, name, sdb, pre, x, args, cfg, y_prod, inner) * g_out.cpu().to(x.dtype)).sum()

        leaves = [args[0].detach()] + [sd['backbone.' + k] for k in keys]
        w64 = _ref_grads(block_loss, leaves, torch.float64)
        w32 = _ref_grads(block_loss, leaves, torch.float32)
        block_max = max(float(a.abs().max()) for a in w64[1:])
        for k, a, b in zip(keys, w64[1:], w32[1:]):
            _check(f'{workload} {k}', got[k], a, b, max(1e-6 * float(a.abs().max()), BIAS_FLOOR * block_max))
        if g_in is not None:
            _check(f'{workload} {name} d input', g_in, w64[0], w32[0])


def _whole_err(got, want, scale):
    return float((got.cpu().double() - want).abs().max()) / max(float(want.abs().max()), scale)


BIAS_FLOOR = 1e-5
WHOLE_TOL = 5e-2
FIXTURE_FLOOR = 1e-4
# measured on an H100: 2.3e-2 (demo2k), 6.1e-2 (modelnet717), 1.7e-1 (kitti4k, the GroupNorm bias of encoder4_3.unary2, the block
# holding the LeakyReLU element at |t| = 7e-7 of _check_blocks_in_chain); the per-block checks are the rounding-level ones
FIXTURE_TOL = 0.25


def _tap_blocks(model):
    """forward hooks on the backbone's blocks: inputs and outputs (retaining their gradients) of the first forward with grad, and the
    outputs of a residual block's two inner activations; the block reads an alias of its input, whose gradient is the block's own
    contribution"""
    taps = {'blocks': {}}
    for name, mod in model.backbone.named_children():
        def pre(m, args, name=name):
            if torch.is_grad_enabled() and name not in taps['blocks']:
                if args[0].requires_grad:      # an alias of the input: its gradient is this block's share only (skip connections)
                    args = (args[0].view_as(args[0]),) + tuple(args[1:])
                    args[0].retain_grad()
                taps['blocks'][name] = {'args': args, 'inner': {}}
                return args

        def post(m, args, out, name=name):
            if torch.is_grad_enabled() and 'out' not in taps['blocks'][name]:
                out.retain_grad()
                taps['blocks'][name]['out'] = out

        mod.register_forward_pre_hook(pre)
        mod.register_forward_hook(post)
        if type(mod).__name__ == 'ResidualBlock':
            def inner(key, t, name=name):
                d = taps['blocks'].get(name, {}).get('inner')
                if torch.is_grad_enabled() and d is not None and key not in d:
                    d[key] = t.detach()
            if not isinstance(mod.unary1, torch.nn.Identity):
                mod.unary1.register_forward_hook(lambda m, a, o, inner=inner: inner('unary1', o))
            mod.unary2.register_forward_pre_hook(lambda m, a, inner=inner: inner('conv', a[0]))
    return taps


def _restated_block(model, name, sdb, pre, x, args, cfg, y_prod, inner):
    """the restatement of backbone block ``name`` on input x (the other forward arguments as the product's block received them).
    Every LeakyReLU takes the branch the product's took: that of its output ``y_prod`` / ``inner`` (see _check_blocks_in_chain)."""
    blk = getattr(model.backbone, name)
    g = cfg.backbone.group_norm
    cpu = [a.cpu() for a in args[1:]]
    if len(cpu) == 3:
        cpu[0], cpu[1] = cpu[0].to(x.dtype), cpu[1].to(x.dtype)

    def leaky_as(t, y=y_prod):
        return torch.where(y.detach().cpu() > 0, t, 0.1 * t)

    kind = type(blk).__name__
    if kind == 'ConvBlock':
        return leaky_as(G.group_norm(sdb, pre + 'norm.', G.kpconv(sdb, pre + 'KPConv.', x, *cpu, blk.KPConv.sigma), g))
    if kind == 'ResidualBlock':                     # geo_oracle.residual_block up to its last activation
        h = leaky_as(G.unary(sdb, pre + 'unary1.', x, g, relu=False), inner['unary1']) if 'unary1' in inner else x
        h = G.kpconv(sdb, pre + 'KPConv.', h, *cpu, blk.KPConv.sigma)
        h = leaky_as(G.group_norm(sdb, pre + 'norm_conv.', h, g), inner['conv'])
        h = G.unary(sdb, pre + 'unary2.', h, g, relu=False)
        sc = G.maxpool(x, cpu[2]) if blk.strided else x
        if (pre + 'unary_shortcut.mlp.weight') in sdb:
            sc = G.unary(sdb, pre + 'unary_shortcut.', sc, g, relu=False)
        return leaky_as(h + sc)
    if kind == 'UnaryBlock':
        return leaky_as(G.unary(sdb, pre, x, g, relu=False))
    return G.unary(sdb, pre, x, g, relu=False, norm=False)


def _backbone_params(model):
    return list(model.backbone.named_parameters())


def test_weights_t_rebuilt_after_in_place_update(models):
    cfg, _, model0 = models('modelnet')
    model = copy.deepcopy(model0).cuda()
    conv = model.backbone.encoder1_2.KPConv
    wt0 = conv._weights_t().clone()
    opt = torch.optim.SGD([conv.weights], lr=0.5)
    conv.weights.grad = torch.ones_like(conv.weights)
    opt.step()
    wt1 = conv._weights_t()
    want = conv.weights.detach().reshape(-1, conv.weights.shape[2]).t()
    assert torch.equal(wt1, want) and not torch.equal(wt1, wt0)
    with torch.no_grad():
        conv.weights.mul_(2.0)
    assert torch.equal(conv._weights_t(), conv.weights.detach().reshape(-1, conv.weights.shape[2]).t())


@pytest.mark.parametrize('workload,cfg_name', [('demo2k', '3dmatch'), ('modelnet717', 'modelnet')])
def test_fine_path_end_to_end(workload, cfg_name, models):
    """forced coarse correspondences: model.backbone with grad -> patch scores -> Sinkhorn -> fine matching loss -> backward.  Every
    block inside the chain against fp64 autograd of the restatement's block, and the whole chain against fp64 autograd of the
    restatement chain"""
    cfg, sd, model0 = models(cfg_name)
    model = copy.deepcopy(model0).cuda().eval()
    data = BV.collate(workload, cfg)
    dc = _cuda_data(data)
    taps = {}
    with torch.no_grad():
        out = model(dict(dc), taps=taps)
    kk = out['ref_node_corr_indices'].shape[0]
    forced = (out['ref_node_corr_indices'][:kk].clone(), out['src_node_corr_indices'][:kk].clone(), out['node_corr_scores'][:kk].clone())
    taps = {}
    with torch.no_grad():
        out = model(dict(dc, forced_node_corr=forced), taps=taps)
    ri = taps['ref_node_knn_indices'][forced[0]].contiguous()
    si = taps['src_node_knn_indices'][forced[1]].contiguous()
    rm, sm = out['ref_node_corr_knn_masks'], out['src_node_corr_knn_masks']
    fine = 1 if cfg_name in ('3dmatch', 'kitti') else 0       # level of the fine features (the finest decoder's output)
    n_ref = int(data['lengths'][fine][0])
    n_all = data['points'][fine].shape[0]
    iters = cfg.model.num_sinkhorn_iterations
    alpha = model.optimal_transport.alpha.detach()
    T = data['transform']

    taps = _tap_blocks(model)
    feats_f = model.backbone(dc['features'], dc)[0]
    ms = GF.sinkhorn(GF.patch_scores_batched(feats_f, [n_ref, n_all - n_ref], ri, si), rm, sm, alpha, iters)
    f_loss = GF.fine_matching_loss(out['ref_node_corr_knn_points'], out['src_node_corr_knn_points'], rm, sm, ms, T.cuda(),
                                   cfg.fine_loss.positive_radius)[2]
    f_loss.backward()
    params = _backbone_params(model)
    keys = [k for k, _ in params]
    got = {k: p.grad.detach().clone() for k, p in params}
    blocks = {name: (t['args'], t['out'], t['inner'], t['out'].grad, t['args'][0].grad) for name, t in taps['blocks'].items()
              if t['out'].grad is not None}
    _check_blocks_in_chain(f'fine path {workload}', model, sd, cfg, blocks, got)
    ri_c, si_c = ri.cpu().clamp(max=n_ref), si.cpu().clamp(max=n_all - n_ref)
    cpu = {k: out[k].cpu() for k in ('ref_node_corr_knn_points', 'src_node_corr_knn_points')}

    def head(ff, dtype):
        ms_ = HG.sinkhorn(alpha.cpu().to(dtype), HG.patch_scores(ff[:n_ref], ff[n_ref:], ri_c, si_c), rm.cpu(), sm.cpu(), iters)
        return HG.fine_loss(cfg.fine_loss.positive_radius, cpu['ref_node_corr_knn_points'], cpu['src_node_corr_knn_points'], rm.cpu(),
                            sm.cpu(), ms_, T)

    # the whole chain against fp64 autograd of the restatement chain (its own forward: see the whole-backbone test)
    w64 = BV.restatement_grads(sd, cfg, data, keys, torch.float64, head=head)
    scale = 1e-2 * max(float(g.abs().max()) for g in got.values())
    worst = max(_whole_err(got[k], w64[k], scale) for k in keys)
    print(f'fine path {workload}: whole chain vs fp64 autograd {worst:.2e}')
    assert worst <= WHOLE_TOL, (workload, worst)
