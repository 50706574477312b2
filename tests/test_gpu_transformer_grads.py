"""Gradients of the geometric transformer on the device (residual LayerNorm, L2 normalisation, head_project, attention with and
without the structure term, the structure embedding): every op against torch fp64 autograd of a restatement on the same inputs, the
whole GeometricTransformer of three configs against fp64 autograd of oracle/geo_oracle.py, OverallLoss end to end through backbone and
transformer, the determinism / bit-identity properties of the backward entry points, and the rebuild of the cached weights after an
optimiser step."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from geotransformer_b200 import functional as GF
from geotransformer_b200.loss import OverallLoss
from oracle import geo_oracle as G
from oracle import backbone_grad_oracle as BV
from oracle import transformer_grad_oracle as TG

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'transformer_grads.npz')

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.contiguous().view(torch.int32)


def _ref_grads(fn, inputs, dtype):
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


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _fresh(cfg, sd):
    """a new model with the state dict, on the GPU (the session's shared models carry caches of other tests)"""
    from geotransformer_b200.model import create_model
    model = create_model(cfg)
    model.load_state_dict(sd, strict=True)
    return model.cuda()


@pytest.mark.parametrize('channels', [128, 256])
@pytest.mark.parametrize('with_b', [True, False])
def test_add_layernorm_backward_matches_fp64_autograd(channels, with_b):
    g = _gen(channels + with_b)
    n = 450
    a = 2.0 * torch.randn(n, channels, generator=g) + 0.3
    b = torch.randn(n, channels, generator=g)
    w = 1.0 + 0.3 * torch.randn(channels, generator=g)
    bb = 0.2 * torch.randn(channels, generator=g)
    up = torch.randn(n, channels, generator=g)

    def loss(x, y, ww, bias):
        return (F.layer_norm(x + y if with_b else x, (channels,), ww, bias) * up.to(x.dtype)).sum()

    w64 = _ref_grads(loss, [a, b, w, bb], torch.float64)
    w32 = _ref_grads(loss, [a, b, w, bb], torch.float32)
    ac, bc, wc, bbc = (t.cuda().requires_grad_(True) for t in (a, b, w, bb))
    out = GF.add_layernorm(ac, bc if with_b else None, wc, bbc)
    with torch.no_grad():
        ref = GF.add_layernorm(ac, bc if with_b else None, wc, bbc)
    assert torch.equal(_bits(out.detach()), _bits(ref)), 'forward bits change with grad mode'
    out.backward(up.cuda())
    tag = f'layernorm C={channels} b={with_b}'
    _check(f'{tag} da', ac.grad, w64[0], w32[0])
    if with_b:
        _check(f'{tag} db', bc.grad, w64[1], w32[1])
    _check(f'{tag} dgamma', wc.grad, w64[2], w32[2])
    _check(f'{tag} dbeta', bbc.grad, w64[3], w32[3])
    gx, gw, gb = GF.add_layernorm_backward(ac, bc if with_b else None, wc, up.cuda())
    assert torch.equal(_bits(gx), _bits(ac.grad)) and torch.equal(_bits(gw), _bits(wc.grad)) and torch.equal(_bits(gb), _bits(bbc.grad))


def test_l2_normalize_backward_matches_fp64_autograd():
    g = _gen(3)
    x = torch.randn(500, 256, generator=g) * torch.rand(500, 1, generator=g) * 3
    up = torch.randn(500, 256, generator=g)
    w64 = _ref_grads(lambda t: (F.normalize(t, p=2, dim=1) * up.to(t.dtype)).sum(), [x], torch.float64)[0]
    w32 = _ref_grads(lambda t: (F.normalize(t, p=2, dim=1) * up.to(t.dtype)).sum(), [x], torch.float32)[0]
    xc = x.cuda().requires_grad_(True)
    out = GF.l2_normalize(xc)
    assert torch.equal(_bits(out.detach()), _bits(GF.l2_normalize(xc.detach())))
    out.backward(up.cuda())
    _check('l2_normalize', xc.grad, w64, w32)


def _head_project_ref(q, wp, bp, heads):
    n, c = q.shape
    d = c // heads
    qh = q.view(n, heads, d)
    qp = torch.einsum('nht,htc->nhc', qh, wp.view(heads, d, c))
    qb = (qh * bp.view(heads, d)).sum(-1)
    return qp, qb


@pytest.mark.parametrize('channels', [128, 256])
def test_head_project_backward_matches_fp64_autograd(channels):
    heads = 4
    g = _gen(40 + channels)
    n = 300
    qkv = torch.randn(n, 3 * channels, generator=g)
    wp = torch.randn(channels, channels, generator=g) / channels ** 0.5
    bp = 0.1 * torch.randn(channels, generator=g)
    up_p = torch.randn(n, heads, channels, generator=g)
    up_b = torch.randn(n, heads, generator=g)

    def loss(x, w, b):
        qp, qb = _head_project_ref(x[:, :channels], w, b, heads)
        return (qp * up_p.to(x.dtype)).sum() + (qb * up_b.to(x.dtype)).sum()

    w64 = _ref_grads(loss, [qkv, wp, bp], torch.float64)
    w32 = _ref_grads(loss, [qkv, wp, bp], torch.float32)
    xc, wc, bc = (t.cuda().requires_grad_(True) for t in (qkv, wp, bp))
    qp, qb = GF.head_project(xc[:, :channels], wc.t(), bc, heads)
    with torch.no_grad():
        qp0, qb0 = GF.head_project(xc[:, :channels], wc.t().contiguous(), bc, heads)
    assert torch.equal(_bits(qp.detach()), _bits(qp0)) and torch.equal(_bits(qb.detach()), _bits(qb0))
    ((qp * up_p.cuda()).sum() + (qb * up_b.cuda()).sum()).backward()
    tag = f'head_project C={channels}'
    _check(f'{tag} dq', xc.grad, w64[0], w32[0])
    _check(f'{tag} dWp', wc.grad, w64[1], w32[1])
    _check(f'{tag} dbp', bc.grad, w64[2], w32[2])


def _attention_ref(q, k, v, heads, qp=None, qb=None, e=None):
    n, c = q.shape
    m = k.shape[0]
    d = c // heads
    qh, kh, vh = q.view(n, heads, d), k.view(m, heads, d), v.view(m, heads, d)
    s = torch.einsum('nhd,mhd->hnm', qh, kh)
    if e is not None:
        s = s + torch.einsum('nhc,nmc->hnm', qp, e) + qb.t().unsqueeze(-1)
    p = torch.softmax(s / d ** 0.5, dim=-1)
    return torch.einsum('hnm,mhd->nhd', p, vh).reshape(n, c)


def _attention_inputs(seed, n, m, c, heads, self_att):
    g = _gen(seed)
    qkv = torch.randn(n, 3 * c, generator=g) * 0.5
    kv = torch.randn(m, 2 * c, generator=g) * 0.5
    up = torch.randn(n, c, generator=g)
    if not self_att:
        return [qkv, kv], up
    qp = torch.randn(n, heads, c, generator=g) * 0.1
    qb = torch.randn(n, heads, generator=g) * 0.5
    e = torch.randn(n, n, c, generator=g)
    return [qkv, qp, qb, e], up


@pytest.mark.parametrize('channels', [128, 256])
def test_cross_attention_backward_column_slices(channels):
    """cross-attention with N != M, q a column slice of a (N, 3C) buffer and k / v of a (M, 2C) one"""
    heads, n, m = 4, 230, 170
    (qkv, kv), up = _attention_inputs(60 + channels, n, m, channels, heads, False)
    c = channels

    def loss(a, b):
        return (_attention_ref(a[:, :c], b[:, :c], b[:, c:], heads) * up.to(a.dtype)).sum()

    w64 = _ref_grads(loss, [qkv, kv], torch.float64)
    w32 = _ref_grads(loss, [qkv, kv], torch.float32)
    ac, bc = (t.cuda().requires_grad_(True) for t in (qkv, kv))
    out = GF.attention(ac[:, :c], bc[:, :c], bc[:, c:], heads)
    with torch.no_grad():
        ref = GF.attention(ac[:, :c], bc[:, :c], bc[:, c:], heads)
    assert torch.equal(_bits(out.detach()), _bits(ref)), 'forward bits change with grad mode'
    out.backward(up.cuda())
    _check(f'cross C={c} dq', ac.grad, w64[0], w32[0])
    _check(f'cross C={c} dk|dv', bc.grad, w64[1], w32[1])


@pytest.mark.parametrize('channels', [128, 256])
def test_self_attention_backward_with_embedding(channels):
    """the structure term with E an input of both sides (so the table's interpolation error does not enter)"""
    heads, n = 4, 150
    (qkv, qp, qb, e), up = _attention_inputs(80 + channels, n, n, channels, heads, True)
    c = channels

    def loss(a, p, b, ee):
        return (_attention_ref(a[:, :c], a[:, c:2 * c], a[:, 2 * c:], heads, p, b, ee) * up.to(a.dtype)).sum()

    w64 = _ref_grads(loss, [qkv, qp, qb, e], torch.float64)
    w32 = _ref_grads(loss, [qkv, qp, qb, e], torch.float32)
    ac, pc, bc, ec = (t.cuda().requires_grad_(True) for t in (qkv, qp, qb, e))
    out = GF.attention(ac[:, :c], ac[:, c:2 * c], ac[:, 2 * c:], heads, qp=pc, qb=bc, embed=ec)
    with torch.no_grad():
        ref = GF.attention(ac[:, :c], ac[:, c:2 * c], ac[:, 2 * c:], heads, qp=pc, qb=bc, embed=ec)
    assert torch.equal(_bits(out.detach()), _bits(ref)), 'forward bits change with grad mode'
    out.backward(up.cuda())
    tag = f'self C={c}'
    _check(f'{tag} dq|dk|dv', ac.grad, w64[0], w32[0])
    _check(f'{tag} dqp', pc.grad, w64[1], w32[1])
    _check(f'{tag} dqb', bc.grad, w64[2], w32[2])
    _check(f'{tag} dE', ec.grad, w64[3], w32[3])
    grads = [t.grad.clone() for t in (ac, pc, bc, ec)]
    for t in (ac, pc, bc, ec):
        t.grad = None
    GF.attention(ac[:, :c], ac[:, c:2 * c], ac[:, 2 * c:], heads, qp=pc, qb=bc, embed=ec).backward(up.cuda())
    for a, t in zip(grads, (ac, pc, bc, ec)):
        assert torch.equal(_bits(a), _bits(t.grad)), 'two backward runs differ'


def test_attention_backward_after_the_lanes_channels_forward():
    """the other streaming forward (geob200_set_attention_tma(0)) also leaves the probabilities for the backward"""
    from geotransformer_b200 import _lib as L
    L.lib().geob200_set_attention_tma(0)
    try:
        test_self_attention_backward_with_embedding(256)
        test_cross_attention_backward_column_slices(128)
    finally:
        L.lib().geob200_set_attention_tma(1)


def test_attention_backward_batch_of_two_equals_per_item_calls():
    heads, c = 4, 256
    items, singles = [], []
    for seed, n in ((5, 140), (6, 97)):
        (qkv, qp, qb, e), up = _attention_inputs(seed, n, n, c, heads, True)
        qkv, qp, qb, e, up = (t.cuda() for t in (qkv, qp, qb, e, up))
        buf, probs = GF.attention_probs(n, n, heads, qkv.device)
        out = GF._attention(qkv[:, :c], qkv[:, c:2 * c], qkv[:, 2 * c:], heads, qp, qb, e, probs=buf)
        it = dict(q=qkv[:, :c], k=qkv[:, c:2 * c], v=qkv[:, 2 * c:], out=out, probs=probs, grad_out=up, qp=qp, qb=qb, embed=e)
        items.append(it)
        singles.append(GF.attention_backward_batched([it], heads)[0])
    both = GF.attention_backward_batched(items, heads)
    for one, two in zip(singles, both):
        for a, b in zip(one, two):
            assert torch.equal(_bits(a), _bits(b))


def _near_ties(a, div, wa, ba):
    """(rows..., C) mask of the entries whose angle max has a near-tie: the two largest terms, with different arguments, within 1e-4
    in the fp64 restatement.  Near such a tie the restatement and the tabulated forward may pick different terms, so the tests give
    these entries no upstream gradient; what they check then has a clear winner everywhere (gap >= 1e-4, asserted).  Inputs without
    any near-tie cannot be chosen: the diagonal (i, i) has all angle indices equal (an exact tie, harmless: equal arguments give the
    same gradient whichever term wins), and among ~10^6 (row, channel) entries a few fall within 1e-4 by chance."""
    with torch.no_grad():
        ga = F.linear(G.sinusoid(a, div), wa.detach().cpu().double(), ba.detach().cpu().double())
        top2 = ga.topk(2, dim=-2)
        args = torch.gather(a.unsqueeze(-1).expand_as(ga), -2, top2.indices)
        gap = top2.values[..., 0, :] - top2.values[..., 1, :]
        near = (gap < 1e-4) & (args[..., 0, :] != args[..., 1, :])
        assert float(near.double().mean()) < 1e-2, float(near.double().mean())
        assert float(gap[~near & (args[..., 0, :] != args[..., 1, :])].min()) >= 1e-4
    return near


def _gse_ref(d, a, div, wd, bd, wa, ba):
    return F.linear(G.sinusoid(d, div), wd, bd) + F.linear(G.sinusoid(a, div), wa, ba).max(dim=-2)[0]


@pytest.mark.parametrize('cfg_name', ['3dmatch', 'kitti'])
def test_flat_structure_embedding_backward_matches_fp64_autograd(cfg_name, models):
    """forward_flat of one cloud: its graph's backward against fp64 autograd; its values are those of forward, which carries no graph"""
    cfg, sd, _ = models(cfg_name)
    emb = _fresh(cfg, sd).transformer.embedding
    c = emb.proj_d.out_features
    g = _gen(90 + c)
    scale = 0.4 if cfg_name == '3dmatch' else 12.0
    pts = (torch.rand(60, 3, generator=g) * scale).cuda()
    d, a = GF.gse_indices(pts, emb.sigma_d, emb.sigma_a, emb.angle_k)
    div = emb.embedding.div_term.detach().cpu().double()
    params = [emb.proj_d.weight, emb.proj_d.bias, emb.proj_a.weight, emb.proj_a.bias]
    dc, ac = d.cpu().double(), a.cpu().double()
    up = torch.randn(60, 60, c, generator=g)
    up[_near_ties(ac, div, params[2], params[3])] = 0.0

    def loss(wd, bd, wa, ba):
        return (_gse_ref(dc.to(wd.dtype), ac.to(wd.dtype), div.to(wd.dtype), wd, bd, wa, ba) * up.to(wd.dtype)).sum()

    w64 = _ref_grads(loss, params, torch.float64)
    w32 = _ref_grads(loss, params, torch.float32)
    out = emb.forward_flat(pts, [60]).view(60, 60, c)
    ref = emb(pts)
    assert not ref.requires_grad
    assert torch.equal(_bits(out.detach()), _bits(ref)), 'forward bits change with the graph'
    out.backward(up.cuda())
    names = ('dWd', 'dbd', 'dWa', 'dba')
    for name, p, a64, a32 in zip(names, params, w64, w32):
        _check(f'gse C={c} {name}', p.grad, a64, a32)
    grads = [p.grad.clone() for p in params]
    for p in params:
        p.grad = None
    emb.forward_flat(pts, [60]).view(60, 60, c).backward(up.cuda())
    for a_, p in zip(grads, params):
        assert torch.equal(_bits(a_), _bits(p.grad)), 'two backward runs differ'


def _cuda_data(data):
    return {k: ([x.cuda() if isinstance(x, torch.Tensor) else x for x in v] if isinstance(v, list) else
                (v.cuda() if isinstance(v, torch.Tensor) else v)) for k, v in data.items()}


def _transformer_inputs(model, data):
    """the transformer's inputs of pair 0: coarse points and the backbone's coarse features, split [ref; src]"""
    dc = _cuda_data(data)
    with torch.no_grad():
        feats_c = model.backbone(dc['features'], dc)[-1]
    pts = dc['points'][-1]
    n0 = int(data['lengths'][-1][0])
    return pts[:n0].contiguous(), pts[n0:].contiguous(), feats_c[:n0].contiguous(), feats_c[n0:].contiguous()


# Whole transformer against fp64 autograd of the restatement: deviation relative to each gradient's largest value, at least 1e-2
# of the largest gradient (see _whole_err).  Measured on an H100: 2.6e-4 (demo2k), 2.0e-4 (modelnet717), 4.0e-6 (kitti4k), all at
# embedding.proj_a.weight: the tabulated forward's interpolation error in E and the fp32 structure-embedding indices.  No LeakyReLU
# kinks here, so the bound sits far inside the backbone's 5e-2.
WHOLE_TOL = 2e-3
# Against the reference's fp32 autograd (fixture digests, oracle/transformer_grad_oracle.digest_err), each side on its own backbone
# features.  Measured on an H100: 2.2e-4 (demo2k), 7.6e-4 (modelnet717), 4.7e-4 (kitti4k), all at embedding.proj_a.weight.
FIXTURE_TOL = 1e-2
# OverallLoss at every model parameter: measured 0.18 (demo2k), 0.22 (modelnet717), 0.23 (kitti4k), all at the backbone's
# encoder1_2.KPConv.bias: the LeakyReLU kinks of the backbone (its own fixture's bound is 0.25); the transformer's parameters agree
# like the whole-transformer check above.
OVERALL_TOL = 0.25
# ... and its transformer parameters alone: measured 4.8e-4 (demo2k), 1.1e-3 (modelnet717), 1.0e-3 (kitti4k), at the embedding weights
OVERALL_TRANSFORMER_TOL = 5e-3
# per layer in the chain: the 10 x fp32-autograd rule with a floor of LAYER_FLOOR x the layer's largest parameter gradient.  Measured
# on an H100: the worst err / (10 x fp32 error) is 0.54 (demo2k), 0.89 (modelnet717); on kitti4k two parameters of 116 pass through
# the floor only: layers.5 proj_k.bias at 1.18 (its gradient is zero in exact arithmetic, max |g| 7e-16: rounding noise, see
# oracle/transformer_grad_oracle.py) and layers.5 proj_q.bias at 1.02 (2.3e-6 of a max |g| of 0.2).
LAYER_FLOOR = 1e-5


def _whole_err(got, want, scale):
    return float((got.detach().cpu().double() - want).abs().max()) / max(float(want.abs().max()), scale)


@pytest.mark.parametrize('workload,cfg_name', BV.WORKLOADS)
def test_transformer_gradients_match_fp64_autograd(workload, cfg_name, models):
    cfg, sd, _ = models(cfg_name)
    model = _fresh(cfg, sd)
    data = BV.collate(workload, cfg)
    rp, sp, rf, sf = _transformer_inputs(model, data)
    tr = model.transformer
    rfc, sfc = rf.clone().requires_grad_(True), sf.clone().requires_grad_(True)
    y0, y1 = tr(rp, sp, rfc, sfc)
    with torch.no_grad():
        z0, z1 = tr(rp, sp, rf, sf)
    assert torch.equal(_bits(y0.detach()), _bits(z0)) and torch.equal(_bits(y1.detach()), _bits(z1)), 'forward bits change with grad mode'
    ups = [u.cuda() for u in BV.upstream([tuple(y0.shape), tuple(y1.shape)])]
    ((y0 * ups[0]).sum() + (y1 * ups[1]).sum()).backward()
    params = list(tr.named_parameters())
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for _, p in params), [k for k, p in params if p.grad is None]
    got = {k: p.grad.detach().clone() for k, p in params}
    got['ref_feats'], got['src_feats'] = rfc.grad.clone(), sfc.grad.clone()
    for _, p in params:                     # two runs give the same bits
        p.grad = None
    rfc.grad = sfc.grad = None
    y0, y1 = tr(rp, sp, rfc, sfc)
    ((y0 * ups[0]).sum() + (y1 * ups[1]).sum()).backward()
    for k, p in params:
        assert torch.equal(_bits(p.grad), _bits(got[k])), ('two runs differ', k)
    # fp64 autograd of the restatement (its own forward: fp64 structure-embedding indices, direct projections)
    keys = [k for k, _ in params]
    sd64 = {k: (v.detach().double() if v.is_floating_point() else v) for k, v in sd.items() if k.startswith('transformer.')}
    leaves = {k: sd64['transformer.' + k].clone().requires_grad_(True) for k in keys}
    sd64.update({'transformer.' + k: v for k, v in leaves.items()})
    f64 = [t.detach().cpu().double().requires_grad_(True) for t in (rf, sf)]
    o0, o1 = G.geometric_transformer(sd64, cfg, rp.cpu().double(), sp.cpu().double(), f64[0], f64[1])
    ((o0 * ups[0].cpu().double()).sum() + (o1 * ups[1].cpu().double()).sum()).backward()
    want = {k: leaves[k].grad for k in keys}
    want['ref_feats'], want['src_feats'] = f64[0].grad, f64[1].grad
    gmax = max(float(g.abs().max()) for g in want.values())
    errs = {k: _whole_err(got[k], want[k], 1e-2 * gmax) for k in want}
    worst = max(errs.items(), key=lambda kv: kv[1])
    # against the reference's fp32 autograd (fixture digests, oracle/transformer_grad_oracle.digest_err); the reference ran on its own
    # backbone features
    fx = np.load(FIXTURE)
    gmax_got = max(float(g.abs().max()) for g in got.values())
    worst_fx = max((TG.digest_err(got[k], fx[f'{workload}/{k}'], k, gmax_got), k) for k in got)
    print(f'{workload}: whole transformer vs fp64 autograd {worst[1]:.2e} ({worst[0]}), vs the reference fixture per digest part '
          f'{worst_fx[0]:.2e} ({worst_fx[1]})')
    assert worst[1] <= WHOLE_TOL, (workload, worst)
    assert worst_fx[0] <= FIXTURE_TOL, (workload, worst_fx)


@pytest.mark.parametrize('workload,cfg_name', BV.WORKLOADS)
def test_overall_loss_fills_every_parameter(workload, cfg_name, models):
    """teacher-forced on the forward's own coarse correspondences: backbone -> transformer -> l2_normalize -> coarse + fine loss ->
    backward gives every parameter of GeoTransformer a finite gradient, which agrees with the reference's OverallLoss backward
    (fixture digests)"""
    cfg, sd, _ = models(cfg_name)
    model = _fresh(cfg, sd).eval()
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
    fine = 1 if cfg_name in ('3dmatch', 'kitti') else 0
    n_ref_f = int(data['lengths'][fine][0])
    n_all_f = data['points'][fine].shape[0]
    n0 = int(data['lengths'][-1][0])
    pts = dc['points'][-1]
    feats_list = model.backbone(dc['features'], dc)
    feats_c, feats_f = feats_list[-1], feats_list[0]
    rc, sc = model.transformer(pts[:n0].contiguous(), pts[n0:].contiguous(), feats_c[:n0], feats_c[n0:])
    y = GF.l2_normalize(torch.cat([rc, sc]))
    ms = GF.sinkhorn(GF.patch_scores_batched(feats_f, [n_ref_f, n_all_f - n_ref_f], ri, si), out['ref_node_corr_knn_masks'],
                     out['src_node_corr_knn_masks'], model.optimal_transport.alpha, cfg.model.num_sinkhorn_iterations)
    loss = OverallLoss(cfg)(dict(out, ref_feats_c=y[:n0], src_feats_c=y[n0:], matching_scores=ms),
                            dict(data, transform=data['transform'].cuda()))['loss']
    assert torch.isfinite(loss)
    loss.backward()
    missing = [k for k, p in model.named_parameters() if p.grad is None or not torch.isfinite(p.grad).all()]
    assert not missing, missing
    assert all(float(p.grad.abs().max()) > 0 for k, p in model.named_parameters() if k.startswith('transformer.')), 'zero gradients'
    fx = np.load(FIXTURE)
    got = {k: p.grad for k, p in model.named_parameters() if f'overall/{workload}/{k}' in fx}
    gmax = max(float(g.abs().max()) for g in got.values())
    errs = {k: TG.digest_err(g, fx[f'overall/{workload}/{k}'], k, gmax) for k, g in got.items()}
    worst = max((e, k) for k, e in errs.items())
    worst_tr = max((e, k) for k, e in errs.items() if k.startswith('transformer.'))
    print(f'{workload}: OverallLoss gradients of {len(got)} parameters vs the reference fixture per digest part {worst[0]:.2e} ({worst[1]}); '
          f'transformer parameters {worst_tr[0]:.2e} ({worst_tr[1]})')
    assert len(got) == len(list(model.parameters()))
    assert worst[0] <= OVERALL_TOL, (workload, worst)
    assert worst_tr[0] <= OVERALL_TRANSFORMER_TOL, (workload, worst_tr)


def test_sgd_step_rebuilds_cached_weights(models):
    """one SGD step on every parameter: the next forward equals, bit for bit, that of a fresh model loaded with the stepped
    state_dict (the version-keyed caches -- structure-embedding table, wd_t / wa_t, fused q|k|v and k|v weights, wp_t -- rebuild)"""
    cfg, sd, _ = models('3dmatch')
    model = _fresh(cfg, sd).eval()
    data = BV.collate('demo2k', cfg)
    rp, sp, rf, sf = _transformer_inputs(model, data)
    tr = model.transformer
    with torch.no_grad():
        tr(rp, sp, rf, sf)                                    # fills every cache with the current weights
    y0, y1 = tr(rp, sp, rf, sf)
    ups = [u.cuda() for u in BV.upstream([tuple(y0.shape), tuple(y1.shape)])]
    ((y0 * ups[0]).sum() + (y1 * ups[1]).sum()).backward()
    torch.optim.SGD(model.parameters(), lr=0.05).step()
    fresh = _fresh(cfg, sd).eval()
    fresh.load_state_dict(model.state_dict())
    with torch.no_grad():
        a0, a1 = tr(rp, sp, rf, sf)
        b0, b1 = fresh.transformer(rp, sp, rf, sf)
        o0, _ = _fresh(cfg, sd).transformer(rp, sp, rf, sf)
    assert not torch.equal(a0, o0), 'the step changed nothing'
    assert torch.equal(_bits(a0), _bits(b0)) and torch.equal(_bits(a1), _bits(b1))


@pytest.mark.parametrize('workload,cfg_name', BV.WORKLOADS)
def test_every_stacked_layer_matches_fp64_autograd(workload, cfg_name, models):
    """every piece of the whole transformer at the product's own activations and upstream gradients against fp64 autograd of its
    restatement, under the 10 x fp32-autograd rule: in_proj, each self / cross layer (parameters and input), out_proj, and the
    structure embedding's backward at the product's dE (near-ties of the angle max masked, see _near_ties)"""
    cfg, sd, _ = models(cfg_name)
    model = _fresh(cfg, sd)
    data = BV.collate(workload, cfg)
    rp, sp, rf, sf = _transformer_inputs(model, data)
    tr = model.transformer
    st = tr.transformer
    heads = cfg.geotransformer.num_heads
    xs, flat = [], []
    layer = st._layer

    def tapped(i, x, rows, E):
        if i == 0:
            x.retain_grad()
            xs.append(x)
            E.retain_grad()
            flat.append(E)
        y = layer(i, x, rows, E)
        y.retain_grad()
        xs.append(y)
        return y

    st._layer = tapped
    rfc, sfc = rf.clone().requires_grad_(True), sf.clone().requires_grad_(True)
    y0, y1 = tr(rp, sp, rfc, sfc)
    ups = [u.cuda() for u in BV.upstream([tuple(y0.shape), tuple(y1.shape)])]
    ((y0 * ups[0]).sum() + (y1 * ups[1]).sum()).backward()
    del st._layer
    n0, n1 = rp.shape[0], sp.shape[0]
    E, dE = flat[0].detach(), flat[0].grad
    # each cloud's E and dE: its row block of the flat E
    embs = [(E[o:o + n * n].view(n, n, -1), dE[o:o + n * n].view(n, n, -1)) for o, n in ((0, n0), (n0 * n0, n1))]
    grads = dict(tr.named_parameters())
    up_all = torch.cat(ups).cpu()
    feats = torch.cat([rf, sf]).cpu()

    def check(tag, keys, fn, x, g_x):
        leaves = [x.detach().cpu()] + [sd['transformer.' + k] for k in keys]
        w64 = _ref_grads(fn, leaves, torch.float64)
        w32 = _ref_grads(fn, leaves, torch.float32)
        block_max = max(float(a.abs().max()) for a in w64[1:])
        for k, a, b in zip(keys, w64[1:], w32[1:]):
            _check(f'{workload} {k}', grads[k].grad, a, b, max(1e-6 * float(a.abs().max()), LAYER_FLOOR * block_max))
        if g_x is not None:
            _check(f'{workload} {tag} d input', g_x, w64[0], w32[0])

    def lin(pre):
        return lambda x, w, b: (F.linear(x, w, b) * (xs[0].grad if pre == 'in_proj' else up_all).cpu().to(x.dtype)).sum()

    check('in_proj', ['in_proj.weight', 'in_proj.bias'], lin('in_proj'), feats, torch.cat([rfc.grad, sfc.grad]))
    check('out_proj', ['out_proj.weight', 'out_proj.bias'], lin('out_proj'), xs[-1], None)
    e_cpu = [e.cpu() for e, _ in embs]
    for i, block in enumerate(cfg.geotransformer.blocks):
        pre = f'transformer.layers.{i}.'
        keys = [k for k in grads if k.startswith(pre)]

        def layer_loss(x, *ws, i=i, block=block, keys=keys):
            sdl = {'transformer.' + k: w for k, w in zip(keys, ws)}
            lp = f'transformer.transformer.layers.{i}.'
            if block == 'self':
                out = torch.cat([G.rpe_self_layer(sdl, lp, x[:n0], e_cpu[0].to(x.dtype), heads),
                                 G.rpe_self_layer(sdl, lp, x[n0:], e_cpu[1].to(x.dtype), heads)])
            else:
                f0 = G.cross_layer(sdl, lp, x[:n0], x[n0:], heads)
                out = torch.cat([f0, G.cross_layer(sdl, lp, x[n0:], f0, heads)])
            return (out * xs[i + 1].grad.cpu().to(x.dtype)).sum()

        check(f'layer {i} ({block})', keys, layer_loss, xs[i], xs[i].grad)
    # the structure embedding's backward at the product's dE of each cloud
    emb = tr.embedding
    div = emb.embedding.div_term.detach().cpu().double()
    table = emb._weights_table()
    ekeys = ['embedding.proj_d.weight', 'embedding.proj_d.bias', 'embedding.proj_a.weight', 'embedding.proj_a.bias']
    got = [torch.zeros_like(grads[k]) for k in ekeys]
    ups_e, idx = [], []
    for pts, (_, de) in zip((rp, sp), embs):
        d, a = GF.gse_indices(pts, emb.sigma_d, emb.sigma_a, emb.angle_k)
        de = de.clone()
        de[_near_ties(a.cpu().double(), div, emb.proj_a.weight, emb.proj_a.bias).cuda()] = 0.0
        n = pts.shape[0]
        gwd, gbd, gwa, gba = GF.gse_embed_backward(d, a, n * n, emb.embedding.div_term, emb.proj_a.weight, emb.proj_a.bias, table,
                                                   de.reshape(n * n, -1))
        for t, gk in zip(got, (gwd, gbd, gwa, gba)):
            t += gk
        ups_e.append(de.cpu())
        idx.append((d.cpu().double(), a.cpu().double()))

    def emb_loss(wd, bd, wa, ba):
        return sum((_gse_ref(d.to(wd.dtype), a.to(wd.dtype), div.to(wd.dtype), wd, bd, wa, ba) * u.to(wd.dtype)).sum()
                   for (d, a), u in zip(idx, ups_e))

    leaves = [sd['transformer.' + k] for k in ekeys]
    w64 = _ref_grads(emb_loss, leaves, torch.float64)
    w32 = _ref_grads(emb_loss, leaves, torch.float32)
    block_max = max(float(a.abs().max()) for a in w64)
    for k, t, a, b in zip(ekeys, got, w64, w32):
        _check(f'{workload} {k}', t, a, b, max(1e-6 * float(a.abs().max()), LAYER_FLOOR * block_max))


def test_frozen_embedding_two_forwards_before_backward(models):
    """with the structure embedding frozen (its parameters not requiring grad), the graph still keeps fresh E tensors: a second
    forward before the first one's backward leaves the first one's gradients unchanged, bit for bit"""
    cfg, sd, _ = models('3dmatch')
    model = _fresh(cfg, sd)
    model.transformer.embedding.requires_grad_(False)
    data = BV.collate('demo2k', cfg)
    rp, sp, rf, sf = _transformer_inputs(model, data)
    tr = model.transformer
    params = [p for p in tr.parameters() if p.requires_grad]

    def loss(a, b):
        y0, y1 = tr(a, b, rf, sf)
        ups = [u.cuda() for u in BV.upstream([tuple(y0.shape), tuple(y1.shape)])]
        return (y0 * ups[0]).sum() + (y1 * ups[1]).sum()

    loss(rp, sp).backward()
    want = [p.grad.clone() for p in params]
    for p in params:
        p.grad = None
    first = loss(rp, sp)
    loss(rp * 1.5, sp * 0.5)                        # overwrites any scratch the first graph might still read
    first.backward()
    for p, w in zip(params, want):
        assert torch.equal(_bits(p.grad), _bits(w))
