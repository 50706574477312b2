"""TEST INFRASTRUCTURE ONLY -- torch-CPU restatement of the validation losses (reference experiments/<exp>/loss.py:10-92 with
modules/loss/circle_loss.py:44-86) and the seeded inputs of tests/golden/losses.npz.

The inputs of the stored loss vectors are regenerated here from (kind, seed, shape) with numpy default_rng; the generator
(oracle/loss_vectors.py, run where the reference checkout exists) stores the reference's outputs next to those parameters.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.geo_oracle import apply_transform, pairwise_distance


def coarse_loss(c, ref_feats, src_feats, gt_indices, gt_overlaps):
    """CoarseMatchingLoss over all n_ref x n_src superpoints; c = cfg.coarse_loss"""
    d = torch.sqrt(pairwise_distance(ref_feats, src_feats, normalized=True))
    o = torch.zeros_like(d)
    o[gt_indices[:, 0], gt_indices[:, 1]] = gt_overlaps
    pos, neg = o > c.positive_overlap, o == 0
    pos_scales = torch.sqrt(o * pos.float())
    wp = torch.clamp(d - 1e5 * (~pos).float() - c.positive_optimal, min=0.0) * pos_scales
    wn = torch.clamp(c.negative_optimal - (d + 1e5 * (~neg).float()), min=0.0)
    lp = c.log_scale * (d - c.positive_margin) * wp
    ln = c.log_scale * (c.negative_margin - d) * wn
    rows = pos.any(-1) & neg.any(-1)
    cols = pos.any(-2) & neg.any(-2)
    l_row = F.softplus(torch.logsumexp(lp, dim=-1) + torch.logsumexp(ln, dim=-1)) / c.log_scale
    l_col = F.softplus(torch.logsumexp(lp, dim=-2) + torch.logsumexp(ln, dim=-2)) / c.log_scale
    return (l_row[rows].mean() + l_col[cols].mean()) / 2


def fine_loss(positive_radius, ref_pts, src_pts, ref_masks, src_masks, scores, transform):
    """FineMatchingLoss: labels of the (K+1)^2 Sinkhorn blocks, negative mean labelled score over all patches"""
    d = pairwise_distance(ref_pts, apply_transform(src_pts, torch.as_tensor(transform)))
    hit = (d < positive_radius ** 2) & ref_masks[:, :, None] & src_masks[:, None, :]
    labels = torch.zeros_like(scores, dtype=torch.bool)
    labels[:, :-1, :-1] = hit
    labels[:, :-1, -1] = (hit.sum(2) == 0) & ref_masks
    labels[:, -1, :-1] = (hit.sum(1) == 0) & src_masks
    return -scores[labels].mean()


def overall_loss(cfg, out, transform):
    """OverallLoss.forward on a forward's output dict: {'loss', 'c_loss', 'f_loss'} (0-dim tensors)"""
    c = coarse_loss(cfg.coarse_loss, out['ref_feats_c'], out['src_feats_c'], out['gt_node_corr_indices'], out['gt_node_corr_overlaps'])
    f = fine_loss(cfg.fine_loss.positive_radius, out['ref_node_corr_knn_points'], out['src_node_corr_knn_points'],
                  out['ref_node_corr_knn_masks'], out['src_node_corr_knn_masks'], out['matching_scores'], transform)
    return {'loss': cfg.loss.weight_coarse_loss * c + cfg.loss.weight_fine_loss * f, 'c_loss': c, 'f_loss': f}


# ------------------------------------------------------------------------------------------------ seeded inputs
# kind, seed, (m, n, channels) for the coarse loss / (patches, k, radius) for the fine loss.  Each kind targets quirks of the
# reference: weight-0 entries inside the logsumexp, softplus above/below its threshold, rows / columns with only positives or
# only negatives, no ground-truth pair at all (NaN), positives closer than positive_optimal, point pairs at exactly the radius,
# patches without a valid point.
COARSE_CASES = [(kind, seed, shape, ls) for seed, (kind, shape, ls) in enumerate([
    ('mixed', (40, 37, 128), 24), ('mixed', (64, 80, 256), 40), ('mixed', (7, 5, 128), 24), ('close', (50, 50, 128), 24),
    ('close', (33, 61, 256), 40), ('onlypos', (12, 9, 128), 24), ('onlypos', (30, 30, 256), 40), ('nogt', (20, 25, 128), 24),
    ('nogt', (1, 1, 128), 40), ('sparse', (90, 70, 128), 24), ('sparse', (45, 120, 256), 40), ('dense', (16, 16, 128), 24),
    ('dense', (24, 18, 256), 40), ('weak', (40, 40, 128), 24), ('weak', (25, 35, 256), 40)], start=100)]
FINE_CASES = [(kind, seed, shape) for seed, (kind, shape) in enumerate([
    ('random', (6, 64, 0.05)), ('random', (5, 128, 0.05)), ('random', (4, 128, 0.6)), ('random', (7, 64, 0.6)),
    ('lattice', (3, 64, 0.05)), ('lattice', (2, 128, 0.05)), ('lattice', (2, 64, 0.6)), ('empty', (4, 64, 0.05)),
    ('empty', (3, 128, 0.6)), ('allempty', (3, 64, 0.05)), ('sparse', (5, 128, 0.05)), ('dense', (4, 64, 0.05)),
    ('rotated', (4, 128, 0.05)), ('rotated', (3, 64, 0.6)), ('halfmask', (6, 128, 0.05))], start=200)]


def _unit(x):
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def coarse_case(kind, seed, shape):
    """(ref_feats (m,c), src_feats (n,c), gt_indices (g,2) int64 row-major, gt_overlaps (g,)) as torch tensors"""
    m, n, c = shape
    rng = np.random.default_rng(seed)
    src = _unit(rng.standard_normal((n, c)))
    ref = _unit(rng.standard_normal((m, c)))
    ov = np.zeros((m, n), dtype=np.float32)
    if kind != 'nogt':
        partner = rng.integers(0, n, size=m)
        noise = {'close': 0.02, 'dense': 0.3, 'weak': 1.5}.get(kind, 0.4)
        take = rng.random(m) < (0.3 if kind == 'sparse' else 0.8)
        ref[take] = _unit(src[partner[take]] + noise * rng.standard_normal((int(take.sum()), c)))
        for i in np.nonzero(take)[0]:
            ov[i, partner[i]] = rng.uniform(0.1, 1.0)
        extra = rng.random((m, n)) < {'dense': 0.5, 'sparse': 0.02}.get(kind, 0.08)
        ov[extra] = rng.choice(np.array([0.05, 0.1, 0.1000001, 0.3, 0.9], dtype=np.float32), size=int(extra.sum()))
        if kind == 'onlypos':
            ov[0, :] = rng.uniform(0.2, 1.0, size=n)          # row 0: positives only
            ov[:, -1] = 0.0                                   # last column: negatives only
        if kind == 'close':                                   # positives closer than positive_optimal
            ref[: m // 2] = _unit(src[partner[: m // 2]] + 1e-3 * rng.standard_normal((m // 2, c)))
    gi = np.stack(np.nonzero(ov), axis=1).astype(np.int64)
    go = ov[gi[:, 0], gi[:, 1]].astype(np.float32)
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    return f(ref), f(src), torch.from_numpy(gi.reshape(-1, 2)), torch.from_numpy(go)


def fine_case(kind, seed, shape):
    """(ref_pts (P,k,3), src_pts (P,k,3), ref_masks, src_masks (P,k) bool, scores (P,k+1,k+1), transform (4,4)) as torch tensors"""
    P, k, r = shape
    rng = np.random.default_rng(seed)
    T = np.eye(4)
    if kind in ('rotated', 'random', 'sparse', 'halfmask'):
        a = rng.uniform(-np.pi, np.pi)
        T[:3, :3] = [[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]]
        T[:3, 3] = rng.uniform(-1.0, 1.0, size=3)
    T = T.astype(np.float32)
    if kind == 'lattice':                                     # grid spacing = radius: many pairs at exactly the radius
        g = np.stack(np.meshgrid(*[np.arange(4)] * 3, indexing='ij'), -1).reshape(-1, 3)
        base = np.resize(g, (k, 3)).astype(np.float32) * np.float32(r)
        ref = np.broadcast_to(base, (P, k, 3)).copy()
        src = ref + np.array([r, 0, 0], dtype=np.float32) * rng.integers(0, 2, size=(P, k, 1)).astype(np.float32)
    else:
        spread = {'dense': 1.0, 'sparse': 6.0}.get(kind, 3.0) * r
        ref = rng.uniform(0, spread, size=(P, k, 3)).astype(np.float32)
        src_world = ref[:, rng.permutation(k)] + rng.normal(0, 0.6 * r, size=(P, k, 3)).astype(np.float32)
        Ti = np.linalg.inv(T.astype(np.float64))
        src = (src_world @ Ti[:3, :3].T + Ti[:3, 3]).astype(np.float32)
    rm, sm = rng.random((P, k)) < 0.85, rng.random((P, k)) < 0.85
    if kind == 'halfmask':
        rm[:, k // 2:] = False
    if kind == 'empty':
        rm[1], sm[1] = False, False                           # a patch without a valid point
        sm[0] = False
    if kind == 'allempty':
        rm[:], sm[:] = False, False                           # no label at all: NaN
    scores = (rng.normal(-4.0, 2.0, size=(P, k + 1, k + 1))).astype(np.float32)
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    return f(ref), f(src), torch.from_numpy(rm), torch.from_numpy(sm), f(scores), f(T)


def coarse_params(log_scale):
    from geotransformer_b200.config import Cfg
    return Cfg(positive_margin=0.1, negative_margin=1.4, positive_optimal=0.1, negative_optimal=1.4, log_scale=log_scale,
               positive_overlap=0.1)
