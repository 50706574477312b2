"""TEST INFRASTRUCTURE ONLY -- gradients of the matching heads.

* Torch restatements whose autograd is the reference's: ``sinkhorn`` (learnable_sinkhorn.py:13-66 via geo_oracle), ``patch_scores``
  (the 'bnd,bmd->bnm' einsum over zero-padded feature tables, model.py:176-188), ``coarse_loss`` (loss.py:10-40 with circle_loss.py:44-86,
  the weights and the kept-line masks DETACHED as there -- loss_oracle.coarse_loss restates the value only) and loss_oracle.fine_loss.
* numpy fp64 restatements of the hand-derived reverse sweeps the kernels implement (``*_backward_np``); tests check them against torch
  fp64 autograd of the restatements above.
* Seeded Sinkhorn / patch-score inputs (``SINKHORN_CASES``, ``PATCH_CASES``) and the coarse case with a duplicated feature row.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import loss_oracle as LO
from oracle.geo_oracle import optimal_transport, pairwise_distance

ITERS = 100


# ------------------------------------------------------------------------------------------------ torch restatements (autograd)
def sinkhorn(alpha, scores, row_masks, col_masks, num_iter=ITERS, inf=1e12):
    """every tensor in the dtype of ``scores``: the reference builds log_mu / log_nu with torch.empty (the default dtype), so an fp64
    run with fp32 marginals would put the masked marginals (fp32(1e12)) 4096 above the masked scores (1e12) -- not the arithmetic of
    either precision"""
    prev = torch.get_default_dtype()
    torch.set_default_dtype(scores.dtype)
    try:
        return optimal_transport(alpha, scores, row_masks, col_masks, num_iter, inf)
    finally:
        torch.set_default_dtype(prev)


def patch_scores(ref_feats, src_feats, ref_idx, src_idx):
    """sentinel index = the cloud's row count selects the padded zero row"""
    rp = torch.cat([ref_feats, torch.zeros_like(ref_feats[:1])], dim=0)
    sp = torch.cat([src_feats, torch.zeros_like(src_feats[:1])], dim=0)
    return torch.einsum('bnd,bmd->bnm', rp[ref_idx], sp[src_idx]) / ref_feats.shape[1] ** 0.5


def coarse_loss(c, ref_feats, src_feats, gt_indices, gt_overlaps):
    d = torch.sqrt(pairwise_distance(ref_feats, src_feats, normalized=True))
    o = torch.zeros_like(d)
    o[gt_indices[:, 0], gt_indices[:, 1]] = gt_overlaps.to(d.dtype)
    pos, neg = torch.gt(o, c.positive_overlap), torch.eq(o, 0)
    scales = torch.sqrt(o * pos.to(d.dtype))
    rows = (torch.gt(pos.sum(-1), 0) & torch.gt(neg.sum(-1), 0)).detach()
    cols = (torch.gt(pos.sum(-2), 0) & torch.gt(neg.sum(-2), 0)).detach()
    wp = torch.maximum(torch.zeros_like(d), d - 1e5 * (~pos).to(d.dtype) - c.positive_optimal) * scales
    wn = torch.maximum(torch.zeros_like(d), c.negative_optimal - (d + 1e5 * (~neg).to(d.dtype)))
    wp, wn = wp.detach(), wn.detach()
    lp = c.log_scale * (d - c.positive_margin) * wp
    ln = c.log_scale * (c.negative_margin - d) * wn
    l_row = F.softplus(torch.logsumexp(lp, dim=-1) + torch.logsumexp(ln, dim=-1)) / c.log_scale
    l_col = F.softplus(torch.logsumexp(lp, dim=-2) + torch.logsumexp(ln, dim=-2)) / c.log_scale
    return (l_row[rows].mean() + l_col[cols].mean()) / 2


fine_loss = LO.fine_loss


# ------------------------------------------------------------------------------------------------ numpy fp64 reverse sweeps
def _lse(x, axis):
    m = np.max(x, axis=axis, keepdims=True)
    return np.squeeze(m, axis) + np.log(np.sum(np.exp(x - m), axis=axis))


def sinkhorn_backward_np(alpha, scores, row_masks, col_masks, grad, num_iter=ITERS, inf=1e12):
    """(dscores, dalpha) by the reverse sweep of the kernel: the forward's log-sum-exps kept per half-step, masked lines in the
    inf -> infinity limit (a masked row's logits are v_j, its potential -LSE), padding patches zero"""
    P, K, _ = scores.shape
    K1 = K + 1
    ds = np.zeros((P, K, K))
    da = 0.0
    with np.errstate(divide='ignore'):
        for p in range(P):
            r, c = np.asarray(row_masks[p], bool), np.asarray(col_masks[p], bool)
            nr, nc = int(r.sum()), int(c.sum())
            if nr == 0 and nc == 0:
                continue
            rmk, cmk = np.r_[~r, False], np.r_[~c, False]
            mask = rmk[:, None] | cmk[None, :]
            Z = np.full((K1, K1), float(alpha))
            Z[:K, :K] = scores[p]
            Z[mask] = -inf
            norm = -np.log(nr + nc)
            lmu = np.r_[np.full(K, norm), np.log(nc) + norm]
            lnu = np.r_[np.full(K, norm), np.log(nr) + norm]
            u, v = np.zeros(K1), np.zeros(K1)
            hist = []
            for _ in range(num_iter):
                v_prev = v
                X = np.where(rmk[:, None], v[None, :], Z + v[None, :])
                Lu = _lse(X, 1)
                u = np.where(rmk, -Lu, lmu - Lu)
                Y = np.where(cmk[None, :], u[:, None], Z + u[:, None])
                Lv = _lse(Y, 0)
                v = np.where(cmk, -Lv, lnu - Lv)
                hist.append((X, Lu, Y, Lv, v_prev))
            G = np.asarray(grad[p], np.float64)
            dZ = G.copy()
            gu, gv = G.sum(1), G.sum(0)
            for t in range(num_iter - 1, -1, -1):
                X, Lu, Y, Lv, _ = hist[t]
                Pv = np.exp(Y - Lv[None, :])
                dZ -= gv[None, :] * Pv
                gu = (gu if t == num_iter - 1 else 0.0) - (gv[None, :] * Pv).sum(1)
                Pu = np.exp(X - Lu[:, None])
                dZ -= gu[:, None] * Pu
                gv = -(gu[:, None] * Pu).sum(0)
            ds[p] = np.where(mask[:K, :K], 0.0, dZ[:K, :K])
            dust = np.zeros((K1, K1), bool)
            dust[:, K] = True
            dust[K, :] = True
            da += dZ[dust & ~mask].sum()
    return ds, da


def patch_scores_backward_np(ref_feats, src_feats, ref_idx, src_idx, grad):
    """(dref, dsrc): per-patch products scattered to the rows; sentinel (>= row count) slots dropped"""
    fr, fs = np.asarray(ref_feats, np.float64), np.asarray(src_feats, np.float64)
    c = fr.shape[1]
    rp = np.vstack([fr, np.zeros((1, c))])
    sp = np.vstack([fs, np.zeros((1, c))])
    g = np.asarray(grad, np.float64) / np.sqrt(c)
    dr_p = np.einsum('pab,pbc->pac', g, sp[src_idx])
    ds_p = np.einsum('pab,pac->pbc', g, rp[ref_idx])
    dr, ds = np.zeros((fr.shape[0] + 1, c)), np.zeros((fs.shape[0] + 1, c))
    np.add.at(dr, np.minimum(ref_idx, fr.shape[0]).reshape(-1), dr_p.reshape(-1, c))
    np.add.at(ds, np.minimum(src_idx, fs.shape[0]).reshape(-1), ds_p.reshape(-1, c))
    return dr[:-1], ds[:-1]


def coarse_backward_np(c, ref_feats, src_feats, gt_indices, gt_overlaps, g=1.0):
    """(dref, dsrc) of c_loss: softmax-weighted detached weights per kept line, sqrt and clamp as torch differentiates them"""
    fr, fs = np.asarray(ref_feats, np.float64), np.asarray(src_feats, np.float64)
    y = 2.0 - 2.0 * fr @ fs.T
    d = np.sqrt(np.maximum(y, 0.0))
    o = np.zeros_like(d)
    gi = np.asarray(gt_indices)
    o[gi[:, 0], gi[:, 1]] = np.asarray(gt_overlaps, np.float64)
    pos, neg = o > c.positive_overlap, o == 0
    wp = np.where(pos, np.maximum(d - c.positive_optimal, 0.0) * np.sqrt(o), 0.0)
    wn = np.where(neg, np.maximum(c.negative_optimal - d, 0.0), 0.0)
    s = c.log_scale
    lp, ln = s * (d - c.positive_margin) * wp, s * (c.negative_margin - d) * wn
    gd = np.zeros_like(d)
    for axis in (1, 0):
        kept = pos.any(axis) & neg.any(axis)
        if not kept.any():
            continue
        Lp, Ln = _lse(lp, axis), _lse(ln, axis)
        x = Lp + Ln
        gx = np.where(kept, (g / 2.0) / kept.sum() / s / (1.0 + np.exp(-x)), 0.0)
        ex = (lambda a: a[:, None]) if axis == 1 else (lambda a: a[None, :])
        gd += ex(gx) * (np.exp(lp - ex(Lp)) * s * wp - np.exp(ln - ex(Ln)) * s * wn)
    with np.errstate(divide='ignore', invalid='ignore'):
        gxy = np.where(y >= 0.0, -2.0 * gd / (2.0 * d), 0.0)
        return gxy @ fs, gxy.T @ fr


def fine_backward_np(positive_radius, ref_pts, src_pts, ref_masks, src_masks, k1, transform, g=1.0):
    """d f_loss / d scores: -g / #labels on the label entries"""
    lab = np.zeros((ref_pts.shape[0], k1, k1), bool)
    d = pairwise_distance(torch.as_tensor(ref_pts), LO.apply_transform(torch.as_tensor(src_pts), torch.as_tensor(transform))).numpy()
    rm, sm = np.asarray(ref_masks, bool), np.asarray(src_masks, bool)
    hit = (d < positive_radius ** 2) & rm[:, :, None] & sm[:, None, :]
    lab[:, :-1, :-1] = hit
    lab[:, :-1, -1] = (hit.sum(2) == 0) & rm
    lab[:, -1, :-1] = (hit.sum(1) == 0) & sm
    n = lab.sum()
    return np.where(lab, -g / n, 0.0) if n else np.zeros(lab.shape)


# ------------------------------------------------------------------------------------------------ seeded inputs
# kind, seed, (patches, k): masks at 20 % per line ('masked'), none ('nomask'), a patch without a valid ref row but with valid columns
# ('norows'), padding patches without any valid line ('padding'); 'upstream' puts the upstream gradient on masked entries too.
SINKHORN_CASES = [(kind, seed, shape) for seed, (kind, shape) in enumerate([
    ('nomask', (8, 64)), ('masked', (32, 64)), ('nomask', (4, 128)), ('masked', (16, 128)), ('norows', (6, 64)), ('padding', (6, 64)),
    ('masked', (8, 32)), ('upstream', (32, 64)), ('upstream', (8, 128))], start=300)]
# kind, seed, (pairs, patches per pair, k, channels, ref rows, src rows): 'dup' repeats nodes across patches (shared rows), 'sentinel'
# pads patches with the sentinel index
PATCH_CASES = [(kind, seed, shape) for seed, (kind, shape) in enumerate([
    ('dup', (1, 12, 64, 32, 300, 280)), ('sentinel', (2, 8, 64, 64, 200, 260)), ('dup', (2, 6, 128, 32, 500, 400)),
    ('sentinel', (1, 5, 32, 16, 90, 70))], start=400)]


def sinkhorn_case(kind, seed, shape):
    """(scores (P,k,k) fp32, row_masks, col_masks (P,k) bool, alpha (0-dim), grad (P,k+1,k+1)) as torch tensors"""
    P, k = shape
    rng = np.random.default_rng(seed)
    scores = rng.normal(0.0, 1.0, size=(P, k, k)).astype(np.float32)
    rm, cm = np.ones((P, k), bool), np.ones((P, k), bool)
    if kind in ('masked', 'upstream', 'norows', 'padding'):
        rm, cm = rng.random((P, k)) >= 0.2, rng.random((P, k)) >= 0.2
    if kind == 'norows':
        rm[0] = False
    if kind == 'padding':
        rm[1:3], cm[1:3] = False, False
    g = rng.normal(0.0, 1.0, size=(P, k + 1, k + 1)).astype(np.float32)
    if kind != 'upstream':
        pad_r, pad_c = np.c_[~rm, np.zeros(P, bool)], np.c_[~cm, np.zeros(P, bool)]
        g[pad_r[:, :, None] | pad_c[:, None, :]] = 0.0
    alpha = np.float32(rng.uniform(0.5, 1.5))
    t = torch.from_numpy
    return t(scores), t(rm), t(cm), torch.tensor(alpha), t(g)


def patch_case(kind, seed, shape):
    """(ref_feats, src_feats (rows, C), cloud_points [ref counts..., src counts...], ref_idx, src_idx (B*P, k) int64 local to the pair's
    cloud, grad (B*P, k, k))"""
    B, P, k, C, nr, ns = shape
    rng = np.random.default_rng(seed)
    rf = rng.normal(size=(B * nr, C)).astype(np.float32)
    sf = rng.normal(size=(B * ns, C)).astype(np.float32)
    ri, si = np.empty((B * P, k), np.int64), np.empty((B * P, k), np.int64)
    for b in range(B):
        rnodes = [rng.choice(nr, size=k, replace=False) for _ in range(3)]    # few nodes: each appears in several patches
        snodes = [rng.choice(ns, size=k, replace=False) for _ in range(3)]
        for q in range(P):
            ri[b * P + q] = rnodes[rng.integers(3)] if kind == 'dup' else rng.choice(nr, size=k, replace=False)
            si[b * P + q] = snodes[rng.integers(3)] if kind == 'dup' else rng.choice(ns, size=k, replace=False)
            if kind == 'sentinel':
                ri[b * P + q, rng.random(k) < 0.3] = nr
                si[b * P + q, rng.random(k) < 0.3] = ns
    g = rng.normal(size=(B * P, k, k)).astype(np.float32)
    t = torch.from_numpy
    return t(rf), t(sf), [nr] * B + [ns] * B, t(ri), t(si), t(g)


def duplicated_coarse_case():
    """a coarse case with a ref and a src superpoint of identical one-hot features (d = 0 exactly in any summation order) next to
    random unit rows whose component on that axis is exact too: the torch finite / NaN pattern at d = 0 is determined"""
    rf, sf, gi, go = LO.coarse_case('mixed', 150, (20, 18, 128))
    rf, sf = rf.clone(), sf.clone()
    rf[3] = 0.0
    rf[3, 0] = 1.0
    sf[5] = 0.0
    sf[5, 0] = 1.0
    return rf, sf, gi, go


# ------------------------------------------------------------------------------------------------ fixture digests
def digest(t):
    """compact, comparable summary of a gradient tensor: the whole tensor when it has <= 2048 entries, else the sums and absolute sums
    over each leading-dimension slice plus 512 seeded flat samples (NaN kept)"""
    a = np.asarray(t.detach().cpu() if isinstance(t, torch.Tensor) else t, np.float64)
    if a.size <= 2048:
        return {'full': a}
    r = a.reshape(a.shape[0], -1)
    pos = np.random.default_rng(a.size).choice(a.size, size=512, replace=False)
    return {'rowsum': r.sum(1), 'rowabs': np.abs(r).sum(1), 'samples': a.reshape(-1)[pos]}


def digest_close(got, want, rtol):
    """every part of the digests agrees to rtol of its largest magnitude, with the same NaN positions"""
    for k, w in want.items():
        g = got[k]
        if g.shape != w.shape or not np.array_equal(np.isnan(g), np.isnan(w)):
            return False
        fin = ~np.isnan(w)
        if fin.any() and np.abs(g[fin] - w[fin]).max() > rtol * max(np.abs(w[fin]).max(), 1e-30):
            return False
    return True
