"""reference ``geotransformer/modules/registration/procrustes.py:6-91`` and ``metrics.py:8-161``."""
import torch
import torch.nn as nn

from ... import functional as GF


def weighted_procrustes(src_points, ref_points, weights=None, weight_thresh=0.0, eps=1e-5, return_transform=False):
    squeeze_first = src_points.ndim == 2
    if squeeze_first:
        src_points, ref_points = src_points.unsqueeze(0), ref_points.unsqueeze(0)
        if weights is not None:
            weights = weights.unsqueeze(0)
    T = GF.weighted_procrustes(src_points.contiguous(), ref_points.contiguous(),
                               None if weights is None else weights.contiguous(), weight_thresh, eps)
    if return_transform:
        return T.squeeze(0) if squeeze_first else T
    R, t = T[:, :3, :3], T[:, :3, 3]
    return (R.squeeze(0), t.squeeze(0)) if squeeze_first else (R, t)


class WeightedProcrustes(nn.Module):
    def __init__(self, weight_thresh=0.0, eps=1e-5, return_transform=False):
        super().__init__()
        self.weight_thresh, self.eps, self.return_transform = weight_thresh, eps, return_transform

    def forward(self, src_points, tgt_points, weights=None):
        return weighted_procrustes(src_points, tgt_points, weights=weights, weight_thresh=self.weight_thresh, eps=self.eps,
                                   return_transform=self.return_transform)


@torch.no_grad()
def get_node_correspondences(ref_nodes, src_nodes, ref_knn_points, src_knn_points, transform, pos_radius, ref_masks=None,
                             src_masks=None, ref_knn_masks=None, src_knn_masks=None):
    """reference ``geotransformer/modules/registration/matching.py:231-315``: ``(corr_indices (C,2), corr_overlaps (C,))``."""
    res = GF.node_correspondences(ref_nodes.contiguous(), src_nodes.contiguous(), ref_knn_points.contiguous(),
                                  src_knn_points.contiguous(), transform.contiguous(), pos_radius, ref_masks, src_masks,
                                  ref_knn_masks, src_knn_masks)
    return GF.finish_node_correspondences(*res)


# Registration metrics (reference modules/registration/metrics.py:8-161).  modified_chamfer_distance and anisotropic_transform_error
# are RPMNet's ModelNet metrics through functional.rpmnet_metrics_batched (32 pairs per call; contract in DESIGN.md section 8a); the
# isotropic errors come from functional.registration_error_batched in double.  All return float32 tensors on the inputs' device.

def _reduce(x, reduction):
    if reduction not in ('mean', 'sum', 'none'):
        raise ValueError(f"reduction must be 'mean', 'sum' or 'none', got {reduction!r}")
    return x.mean() if reduction == 'mean' else (x.sum() if reduction == 'sum' else x)


def _rpmnet_rows(raw_points, ref_points, src_points, gt_transforms, transforms):
    B = gt_transforms.shape[0]
    rows = []
    for b in range(0, B, GF.RPMNET_MAX_PAIRS):
        e = min(B, b + GF.RPMNET_MAX_PAIRS)
        clouds = [x[b:e].detach().to(torch.float32) for x in (raw_points, ref_points, src_points)]
        args = []
        for c in clouds:
            args += [c.reshape(-1, 3).contiguous(), [c.shape[1]] * (e - b)]
        rows.append(GF.rpmnet_metrics_batched(*args, gt_transforms[b:e].detach().float().contiguous(),
                                              transforms[b:e].detach().float().contiguous()))
    return torch.cat(rows)


def modified_chamfer_distance(raw_points, ref_points, src_points, gt_transform, transform, reduction='mean'):
    """RPMNet's modified Chamfer distance of (B, N, 3) raw / ref / src batches under (B, 4, 4) transforms.  Differs from the
    reference's fp32 xx + yy - 2xy expansion and torch.inverse: exact nearest neighbours, fp64 distances (INTEGRATION.md section 3)."""
    with torch.no_grad():
        B = gt_transform.shape[0]
        d = torch.zeros((B,), dtype=torch.float64, device=gt_transform.device)
        if B:
            d = _rpmnet_rows(raw_points, ref_points, src_points, gt_transform, transform)[:, 0]
    return _reduce(d.float(), reduction)


def anisotropic_transform_error(gt_transforms, transforms, reduction='mean'):
    """(r_mse, r_mae, t_mse, t_mae) per pair of (B, 4, 4) transforms: scipy's from_matrix / as_euler('xyz', degrees) errors, on the
    device.  ValueError (naming the pair) if a rotation has det <= 0."""
    with torch.no_grad():
        B = gt_transforms.shape[0]
        p = torch.zeros((B, 1, 3), dtype=torch.float32, device=gt_transforms.device)
        rows = _rpmnet_rows(p, p, p, gt_transforms, transforms)
    return tuple(_reduce(rows[:, c].float(), reduction) for c in (3, 4, 5, 6))


def _isotropic_rows(gt_transforms, transforms):
    gt = gt_transforms.detach().float().reshape(-1, 16).contiguous()
    est = transforms.detach().float().reshape(-1, 16).contiguous()
    return GF.registration_error_batched(gt, est, rre_threshold=0.0, rte_threshold=0.0)


def _with_rotation(R):
    T = torch.eye(4, dtype=torch.float32, device=R.device).repeat(*R.shape[:-2], 1, 1)
    T[..., :3, :3] = R
    return T


def _with_translation(t):
    T = torch.eye(4, dtype=torch.float32, device=t.device).repeat(*t.shape[:-1], 1, 1)
    T[..., :3, 3] = t
    return T


def relative_rotation_error(gt_rotations, rotations):
    """RRE in degrees of (*, 3, 3) rotations"""
    shape = gt_rotations.shape[:-2]
    return _isotropic_rows(_with_rotation(gt_rotations), _with_rotation(rotations))[:, 0].float().reshape(shape)


def relative_translation_error(gt_translations, translations):
    """RTE of (*, 3) translations"""
    shape = gt_translations.shape[:-1]
    return _isotropic_rows(_with_translation(gt_translations), _with_translation(translations))[:, 1].float().reshape(shape)


def isotropic_transform_error(gt_transforms, transforms, reduction='mean'):
    """(rre, rte) of (*, 4, 4) transforms"""
    shape = gt_transforms.shape[:-2]
    rows = _isotropic_rows(gt_transforms, transforms)
    return _reduce(rows[:, 0].float().reshape(shape), reduction), _reduce(rows[:, 1].float().reshape(shape), reduction)
