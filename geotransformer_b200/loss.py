"""Evaluator (reference ``experiments/<exp>/loss.py:95-159``): PIR, IR, RRE, RTE, RMSE, RR of one registered pair; and the
validation losses CoarseMatchingLoss / FineMatchingLoss / OverallLoss (``loss.py:10-92``).

Same constructor/forward contract as the reference's three Evaluator classes (3DMatch, KITTI, ModelNet differ in how
RMSE and RR are defined; ``cfg.name`` selects).  All six numbers come from ONE kernel launch (`geob200_evaluate_counts`); the
result dict holds 0-dim device tensors like the reference's.  KITTI has no RMSE entry (loss.py:140-151 there).

The losses are the values the reference's ``val_step`` reports on the eval-mode forward.  When grad mode is on and the coarse
features (``ref_feats_c`` / ``src_feats_c``) or the Sinkhorn ``matching_scores`` require grad, the loss modules return 0-dim tensors
carrying the graph back to them (the backward runs on the device: ``functional.*_backward_batched``); the values are the same kernels'
bits either way.  There is no CPU path: non-CUDA inputs raise RuntimeError.
"""
import torch
import torch.nn as nn

from . import functional as GF


class Evaluator(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.mode = GF.EVAL_MODES[cfg.name]
        e = cfg.eval
        self.acceptance_overlap = e.acceptance_overlap
        self.acceptance_radius = e.acceptance_radius
        self.acceptance_rmse = getattr(e, 'rmse_threshold', 0.0) if self.mode == 0 else 0.0
        self.acceptance_rre = e.rre_threshold
        self.acceptance_rte = e.rte_threshold

    @torch.no_grad()
    def metrics_tensor(self, output_dict, data_dict, out=None):
        """(8,) device tensor [PIR, IR, RRE, RTE, RMSE, RR, #corr, #gt_node_corr] -- no host sync."""
        return GF.evaluate(output_dict['gt_node_corr_indices'], output_dict['gt_node_corr_overlaps'],
                           output_dict['ref_node_corr_indices'], output_dict['src_node_corr_indices'],
                           output_dict['ref_corr_points'], output_dict['src_corr_points'], data_dict['transform'],
                           output_dict['estimated_transform'], output_dict['src_points'], self.mode,
                           self.acceptance_overlap, self.acceptance_radius, self.acceptance_rmse, self.acceptance_rre,
                           self.acceptance_rte, out=out)

    def forward(self, output_dict, data_dict):
        m = self.metrics_tensor(output_dict, data_dict)
        res = {'PIR': m[0], 'IR': m[1], 'RRE': m[2], 'RTE': m[3], 'RMSE': m[4], 'RR': m[5]}
        if self.mode == 1:
            del res['RMSE']
        return res


def _counts(output_dict):
    """device counts of the valid rows when the output dict holds full-capacity buffers (forward_batch without a host sync)"""
    return output_dict.get('_counts') or {}


class CoarseMatchingLoss(nn.Module):
    """Weighted circle loss over all superpoint pairs (reference loss.py:10-40); forward returns a 0-dim device tensor."""

    def __init__(self, cfg):
        super().__init__()
        c = cfg.coarse_loss
        self.positive_margin, self.negative_margin = c.positive_margin, c.negative_margin
        self.positive_optimal, self.negative_optimal = c.positive_optimal, c.negative_optimal
        self.log_scale, self.positive_overlap = c.log_scale, c.positive_overlap

    def params(self):
        return (self.positive_margin, self.negative_margin, self.positive_optimal, self.negative_optimal, self.log_scale,
                self.positive_overlap)

    @torch.no_grad()
    def write(self, output_dict, out):
        """c_loss into column 1 of the (>= 3,) device row ``out``"""
        return GF.coarse_matching_loss(output_dict['ref_feats_c'], output_dict['src_feats_c'], output_dict['gt_node_corr_indices'],
                                       output_dict['gt_node_corr_overlaps'], *self.params(), out=out, n_gt=_counts(output_dict).get('gt'))

    def forward(self, output_dict):
        rf, sf = output_dict['ref_feats_c'], output_dict['src_feats_c']
        if GF._needs_grad(rf, sf):
            return GF.coarse_matching_loss(rf, sf, output_dict['gt_node_corr_indices'], output_dict['gt_node_corr_overlaps'], *self.params(),
                                           n_gt=_counts(output_dict).get('gt'))[1]
        return self.write(output_dict, None)[1]


class FineMatchingLoss(nn.Module):
    """Negative mean Sinkhorn score of the ground-truth labels of all patches (reference loss.py:43-71); 0-dim device tensor."""

    def __init__(self, cfg):
        super().__init__()
        self.positive_radius = cfg.fine_loss.positive_radius

    @torch.no_grad()
    def write(self, output_dict, data_dict, out, loss_weights=None):
        """f_loss into column 2 of ``out``; with ``loss_weights`` also the weighted total into column 0 (from column 1)"""
        return GF.fine_matching_loss(output_dict['ref_node_corr_knn_points'], output_dict['src_node_corr_knn_points'],
                                     output_dict['ref_node_corr_knn_masks'], output_dict['src_node_corr_knn_masks'],
                                     output_dict['matching_scores'], data_dict['transform'], self.positive_radius,
                                     loss_weights=loss_weights, out=out, n_patches=_counts(output_dict).get('node_corr'))

    def forward(self, output_dict, data_dict):
        if GF._needs_grad(output_dict['matching_scores']):
            return GF.fine_matching_loss(*self.inputs(output_dict, data_dict), self.positive_radius,
                                         n_patches=_counts(output_dict).get('node_corr'))[2]
        return self.write(output_dict, data_dict, None)[2]

    @staticmethod
    def inputs(output_dict, data_dict):
        return (output_dict['ref_node_corr_knn_points'], output_dict['src_node_corr_knn_points'], output_dict['ref_node_corr_knn_masks'],
                output_dict['src_node_corr_knn_masks'], output_dict['matching_scores'], data_dict['transform'])


class OverallLoss(nn.Module):
    """weight_coarse_loss * c_loss + weight_fine_loss * f_loss (reference loss.py:74-92): {'loss', 'c_loss', 'f_loss'} as 0-dim
    device tensors, differentiable w.r.t. the coarse features and the matching scores when they require grad."""

    def __init__(self, cfg):
        super().__init__()
        self.coarse_loss = CoarseMatchingLoss(cfg)
        self.fine_loss = FineMatchingLoss(cfg)
        self.weight_coarse_loss = cfg.loss.weight_coarse_loss
        self.weight_fine_loss = cfg.loss.weight_fine_loss

    @torch.no_grad()
    def loss_tensor(self, output_dict, data_dict, out=None):
        """(3,) device tensor [loss, c_loss, f_loss] -- no host sync"""
        if out is None:
            out = torch.empty((3,), dtype=torch.float32, device=output_dict['matching_scores'].device)
        self.coarse_loss.write(output_dict, out)
        self.fine_loss.write(output_dict, data_dict, out, loss_weights=(self.weight_coarse_loss, self.weight_fine_loss))
        return out

    @torch.no_grad()
    def write_batched(self, feats_c, cloud_nodes, gt, ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, scores,
                      transforms, patch_count, out):
        """rows [loss, c_loss, f_loss] of all pairs of a batched forward (GeoTransformer.forward_batch) into ``out`` (B, >= 3)"""
        B = len(cloud_nodes) // 2
        n_ref = sum(int(c) for c in cloud_nodes[:B])
        c = self.coarse_loss
        GF.coarse_matching_loss_batched(feats_c, feats_c[n_ref:], cloud_nodes, gt[0], gt[1], gt[2], *c.params(), out=out)
        GF.fine_matching_loss_batched(B, ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, scores, transforms,
                                      self.fine_loss.positive_radius, patch_count=patch_count,
                                      loss_weights=(self.weight_coarse_loss, self.weight_fine_loss), out=out)
        return out

    def forward(self, output_dict, data_dict):
        rf, sf, sc = output_dict['ref_feats_c'], output_dict['src_feats_c'], output_dict['matching_scores']
        if GF._needs_grad(rf, sf, sc):
            t = self.graph_rows(output_dict, data_dict)[0]
        else:
            t = self.loss_tensor(output_dict, data_dict)
        return {'loss': t[0], 'c_loss': t[1], 'f_loss': t[2]}

    def graph_rows(self, output_dict, data_dict):
        """(B, 3) [loss, c_loss, f_loss] of the B pairs of the output dict with gradients to the coarse features and the matching
        scores (the value kernels' bits).  One pair, or the stacked output of ``GeoTransformer.forward_train_batch`` (its
        ``_cloud_nodes`` give B and the pairs' superpoint rows, ``_stacked['gt_transforms']`` the (B, 4, 4) transforms)."""
        rf, sf = output_dict['ref_feats_c'], output_dict['src_feats_c']
        counts = _counts(output_dict)
        gi = output_dict['gt_node_corr_indices']
        cloud_nodes = output_dict.get('_cloud_nodes') or (rf.shape[0], sf.shape[0])
        B = len(cloud_nodes) // 2
        n_gt = counts.get('gt')
        n_gt = n_gt.reshape(B) if n_gt is not None else torch.full((1,), gi.shape[0], dtype=torch.int32, device=rf.device)
        coarse = dict(cloud_nodes=cloud_nodes, gt_indices=gi, gt_overlaps=output_dict['gt_node_corr_overlaps'], gt_count=n_gt,
                      params=self.coarse_loss.params())
        rp, sp, rm, sm, scores, T = FineMatchingLoss.inputs(output_dict, data_dict)
        if B > 1:
            T = output_dict['_stacked']['gt_transforms']
        n_p = counts.get('node_corr')
        fine = dict(n_pairs=B, ref_knn_points=rp, src_knn_points=sp, ref_knn_masks=rm, src_knn_masks=sm, transforms=T,
                    positive_radius=self.fine_loss.positive_radius, patch_count=None if n_p is None else n_p.reshape(B))
        return GF.matching_losses_batched(rf, sf, scores, coarse, fine, (self.weight_coarse_loss, self.weight_fine_loss))
