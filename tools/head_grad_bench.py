"""Time the backward of the matching heads (patch scores -> Sinkhorn -> OverallLoss) for a batch of pairs, split by stage, against
eager torch autograd of the same chain on the same device tensors.

    python tools/head_grad_bench.py [--batch 8] [--reps 20]

For a batch of 3dmatch20k pairs and a batch of kitti4k pairs it runs the forward of each pair for real coarse / fine features,
masks, patch points, ground truth and the patch index tables (node knn tables of the superpoint correspondences, from the
forward's taps), so the per-row reduce of the patch-score backward sees the forward's real row sharing.  Reported per batch:
CUDA-event time (median and min over --reps after warm-up) of each backward stage -- fine loss, Sinkhorn, patch scores, coarse loss -- of the whole autograd backward, and of torch autograd's
backward through an eager restatement of patch scores + Sinkhorn (the stages that dominate).  The card name and power limit are
read in the same run and printed with the numbers; writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from geotransformer_b200 import functional as GF                        # noqa: E402
from geotransformer_b200.config import make_cfg                         # noqa: E402
from geotransformer_b200.loss import OverallLoss                        # noqa: E402
from geotransformer_b200.model import create_model, enable_native       # noqa: E402
from geotransformer_b200.synth import make_pair                         # noqa: E402
from geotransformer_b200.utils.data import registration_collate_fn_stack_mode  # noqa: E402
from geotransformer_b200.weights import synthetic_state_dict            # noqa: E402
from loss_bench import KEYS, LIMITS, card, timed                       # noqa: E402


def eager_sinkhorn(alpha, scores, rm, cm, iters, inf=1e12):
    """learnable_sinkhorn.py:20-66 as eager device ops (the reference's own formulation)"""
    b, n, m = scores.shape
    dev = scores.device
    prm = torch.zeros((b, n + 1), dtype=torch.bool, device=dev)
    prm[:, :n] = ~rm
    pcm = torch.zeros((b, m + 1), dtype=torch.bool, device=dev)
    pcm[:, :m] = ~cm
    ps = torch.cat([torch.cat([scores, alpha.expand(b, n, 1)], -1), alpha.expand(b, 1, m + 1)], 1)
    ps = ps.masked_fill(prm[:, :, None] | pcm[:, None, :], -inf)
    nvr, nvc = rm.float().sum(1), cm.float().sum(1)
    norm = -torch.log(nvr + nvc)
    lmu = torch.cat([norm[:, None].expand(b, n), (torch.log(nvc) + norm)[:, None]], 1).masked_fill(prm, -inf)
    lnu = torch.cat([norm[:, None].expand(b, m), (torch.log(nvr) + norm)[:, None]], 1).masked_fill(pcm, -inf)
    u, v = torch.zeros_like(lmu), torch.zeros_like(lnu)
    for _ in range(iters):
        u = lmu - torch.logsumexp(ps + v[:, None, :], dim=2)
        v = lnu - torch.logsumexp(ps + u[:, :, None], dim=1)
    return ps + u[:, :, None] + v[:, None, :] - norm[:, None, None]


def run(workload, cfg_name, batch, reps):
    cfg = make_cfg(cfg_name)
    model = create_model(cfg)
    model.load_state_dict(synthetic_state_dict(model, 7351), strict=True)
    model = enable_native(model.cuda().eval())
    pairs = [{k: make_pair(workload, i % 4)[k] for k in KEYS} for i in range(batch)]
    b = cfg.backbone
    data = {'transform': [torch.from_numpy(p['transform']).cuda() for p in pairs]}
    outs, tables = [], []
    with torch.no_grad():
        for p in range(batch):
            taps = {}
            one = registration_collate_fn_stack_mode([pairs[p]], b.num_stages, b.init_voxel_size, b.init_radius, LIMITS[cfg_name])
            outs.append(model(one, taps=taps))
            o = outs[-1]
            tables.append((taps['ref_node_knn_indices'][o['ref_node_corr_indices']],
                           taps['src_node_knn_indices'][o['src_node_corr_indices']]))
    torch.cuda.synchronize()
    B = len(outs)
    P = min(o['matching_scores'].shape[0] for o in outs)
    K = outs[0]['ref_node_corr_knn_masks'].shape[1]
    iters = cfg.model.num_sinkhorn_iterations
    cp = [o['ref_feats_f'].shape[0] for o in outs] + [o['src_feats_f'].shape[0] for o in outs]
    rm = torch.cat([o['ref_node_corr_knn_masks'][:P] for o in outs])
    sm = torch.cat([o['src_node_corr_knn_masks'][:P] for o in outs])
    ri = torch.cat([t[0][:P] for t in tables]).contiguous()
    si = torch.cat([t[1][:P] for t in tables]).contiguous()
    rff = torch.cat([o['ref_feats_f'] for o in outs])
    sff = torch.cat([o['src_feats_f'] for o in outs])
    rfc = torch.cat([o['ref_feats_c'] for o in outs])
    sfc = torch.cat([o['src_feats_c'] for o in outs])
    cn = [o['ref_feats_c'].shape[0] for o in outs] + [o['src_feats_c'].shape[0] for o in outs]
    nn = [cn[p] * cn[B + p] for p in range(B)]
    gi = torch.zeros((sum(nn), 2), dtype=torch.int64, device='cuda')
    go = torch.zeros((sum(nn),), dtype=torch.float32, device='cuda')
    cnt = torch.zeros((B,), dtype=torch.int32, device='cuda')
    g0 = 0
    for p, o in enumerate(outs):
        n = o['gt_node_corr_indices'].shape[0]
        gi[g0:g0 + n], go[g0:g0 + n], cnt[p] = o['gt_node_corr_indices'], o['gt_node_corr_overlaps'], n
        g0 += nn[p]
    rp = torch.cat([o['ref_node_corr_knn_points'][:P] for o in outs])
    sp = torch.cat([o['src_node_corr_knn_points'][:P] for o in outs])
    T = torch.stack(list(data['transform'])).reshape(B, 4, 4).contiguous()
    alpha = model.optimal_transport.alpha.detach()
    loss = OverallLoss(cfg)
    c = loss.coarse_loss
    coarse = dict(cloud_nodes=cn, gt_indices=gi, gt_overlaps=go, gt_count=cnt, params=c.params())
    fine = dict(n_pairs=B, ref_knn_points=rp, src_knn_points=sp, ref_knn_masks=rm, src_knn_masks=sm, transforms=T,
                positive_radius=loss.fine_loss.positive_radius, patch_count=None)
    weights = (loss.weight_coarse_loss, loss.weight_fine_loss)
    raw = GF._patch_scores(rff, sff, cp, ri, si)
    ms = GF.sinkhorn(raw, rm, sm, alpha, iters)
    grad_rows = torch.ones((B, 3), device='cuda')
    g_ms = GF.fine_matching_loss_backward_batched(grad_rows=grad_rows, loss_weights=weights, **fine)
    g_raw, _ = GF.sinkhorn_backward(raw, rm, sm, alpha, iters, g_ms)

    stages = {
        'fine_loss': lambda: GF.fine_matching_loss_backward_batched(grad_rows=grad_rows, loss_weights=weights, **fine),
        'sinkhorn': lambda: GF.sinkhorn_backward(raw, rm, sm, alpha, iters, g_ms),
        'patch_scores': lambda: GF.patch_scores_backward_batched(rff, sff, cp, ri, si, g_raw),
        'coarse_loss': lambda: GF.coarse_matching_loss_backward_batched(rfc, sfc, grad_rows=grad_rows, loss_weights=weights, **coarse),
    }
    res = {'workload': workload, 'batch': B, 'patches_per_pair': P, 'k': K, 'channels_fine': rff.shape[1]}
    for name, fn in stages.items():
        med, mn = timed(fn, reps)
        res[f'{name}_backward_ms_median'], res[f'{name}_backward_ms_min'] = round(med, 4), round(mn, 4)

    leaves = [t.detach().clone().requires_grad_(True) for t in (rfc, sfc, rff, sff, alpha)]

    def graph():
        s = GF.sinkhorn(GF._patch_scores(leaves[2], leaves[3], cp, ri, si), rm, sm, leaves[4], iters)
        return GF.matching_losses_batched(leaves[0], leaves[1], s, coarse, fine, weights)[:, 0].sum()
    g = [graph()]

    def backward():
        g[0].backward(retain_graph=True)
    med, mn = timed(backward, reps)
    res['autograd_backward_total_ms_median'], res['autograd_backward_total_ms_min'] = round(med, 4), round(mn, 4)

    # eager torch: patch scores + Sinkhorn on the same tensors, backward from the same upstream gradient
    el = [t.detach().clone().requires_grad_(True) for t in (rff, sff, alpha)]
    zr = torch.zeros((1, rff.shape[1]), device='cuda')
    off_r = torch.tensor(np.repeat(np.cumsum([0] + cp[:B - 1]), P), device='cuda')[:, None]
    off_s = torch.tensor(np.repeat(np.cumsum([0] + cp[B:2 * B - 1]), P), device='cuda')[:, None]
    eri = torch.where(ri < torch.tensor(cp[:B], device='cuda').repeat_interleave(P)[:, None], ri + off_r, rff.shape[0])
    esi = torch.where(si < torch.tensor(cp[B:], device='cuda').repeat_interleave(P)[:, None], si + off_s, sff.shape[0])
    e_out = [eager_sinkhorn(el[2], torch.einsum('bnd,bmd->bnm', torch.cat([el[0], zr])[eri], torch.cat([el[1], zr])[esi]) /
                            rff.shape[1] ** 0.5, rm, sm, iters)]

    def eager_backward():
        e_out[0].backward(g_ms, retain_graph=True)
    med, mn = timed(eager_backward, reps)
    res['eager_torch_patch_scores_sinkhorn_backward_ms_median'], res['eager_torch_patch_scores_sinkhorn_backward_ms_min'] = \
        round(med, 4), round(mn, 4)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--reps', type=int, default=20)
    a = ap.parse_args()
    name, pl = card()
    print(json.dumps({'card': name, 'power_limit': pl}))
    for workload, cfg_name in (('3dmatch20k', '3dmatch'), ('kitti4k', 'kitti')):
        print(json.dumps(run(workload, cfg_name, a.batch, max(20, a.reps))))


if __name__ == '__main__':
    main()
