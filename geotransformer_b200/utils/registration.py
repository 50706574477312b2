"""Per-pair evaluation functions of ``geotransformer/utils/registration.py`` with the reference's names and signatures, on the device.

Inputs are numpy arrays or CUDA tensors; numpy inputs run on the current CUDA device.  Each call is the batched kernel with one
pair; ``geotransformer_b200.evaluate`` runs whole chunks of pairs instead.
"""
import numpy as np
import torch

from .. import functional as GF


def _device(*xs):
    for x in xs:
        if isinstance(x, torch.Tensor):
            if not x.is_cuda:
                raise RuntimeError('inputs must be numpy arrays or CUDA tensors (geotransformer_b200 has no CPU path)')
            return x.device
    return torch.device('cuda', torch.cuda.current_device())


def _dev(x, dtype, device):
    if isinstance(x, torch.Tensor):
        return x.detach().to(device=device, dtype=dtype).contiguous()
    return torch.from_numpy(np.ascontiguousarray(x)).to(device=device, dtype=dtype).contiguous()


def _feats(x, name, device):
    if isinstance(x, torch.Tensor):
        return x.detach().to(device=device, dtype=torch.float32).reshape(x.shape[0], -1).contiguous()
    x = np.asarray(x)
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(device).reshape(x.shape[0], -1).contiguous()


def extract_corr_indices_from_feats(ref_feats, src_feats, mutual=False, bilateral=False):
    r"""Correspondence indices from descriptor nearest neighbours (exact, csrc/feature_match.cu): plain (every ref row with its
    nearest src row), ``mutual`` (only pairs that are each other's nearest; increasing ref row) or ``bilateral`` (plain, then every
    src row with its nearest ref row; ignored when ``mutual``).  Returns (ref_corr_indices, src_corr_indices) int64, numpy for
    numpy inputs and device tensors for CUDA tensors."""
    return _corr_from_feats(ref_feats, src_feats, mutual, bilateral)[:2]


def _corr_from_feats(ref_feats, src_feats, mutual, bilateral):
    device = _device(ref_feats, src_feats)
    on_device = isinstance(ref_feats, torch.Tensor) or isinstance(src_feats, torch.Tensor)
    ref, src = _feats(ref_feats, 'ref_feats', device), _feats(src_feats, 'src_feats', device)
    if ref.shape[1] != src.shape[1]:
        raise ValueError('extract_corr_indices_from_feats: ref_feats and src_feats need the same width')
    mode = 'mutual' if mutual else ('bilateral' if bilateral else 'plain')
    if mode == 'plain':
        ref_nn, ref_dist = GF.feature_nearest_neighbor(ref, src)
        src_nn = src_dist = None
    else:
        ref_nn, ref_dist, src_nn, src_dist = GF.feature_nearest_neighbor(ref, src, bidirectional=True)
    out = GF.feature_correspondences(ref_nn, ref_dist, src_nn, src_dist, mode=mode)
    return out if on_device else tuple(v.cpu().numpy() for v in out)


def extract_correspondences_from_feats(ref_points, src_points, ref_feats, src_feats, mutual=False, return_feat_dist=False):
    r"""[ref_corr_points, src_corr_points] (+ the descriptor distance of every pair, float32, with ``return_feat_dist``) of the
    plain or ``mutual`` correspondences of extract_corr_indices_from_feats."""
    ref_idx, src_idx, dist = _corr_from_feats(ref_feats, src_feats, mutual, False)
    if isinstance(ref_idx, torch.Tensor):
        device = ref_idx.device
        ref_pts, src_pts = _feats(ref_points, 'ref_points', device), _feats(src_points, 'src_points', device)
        outputs = [GF.gather_rows(ref_pts, ref_idx), GF.gather_rows(src_pts, src_idx)]
    else:
        outputs = [np.asarray(ref_points)[ref_idx], np.asarray(src_points)[src_idx]]
    if return_feat_dist:
        outputs.append(dist)
    return outputs


def evaluate_sparse_correspondences(ref_points, src_points, ref_corr_indices, src_corr_indices, gt_corr_indices):
    """Precision, recall and hit ratio of the superpoint correspondences against the ground-truth pairs (duplicates count once);
    the values equal numpy's evaluation bit for bit."""
    device = _device(ref_corr_indices, src_corr_indices, gt_corr_indices)
    ref_idx = _dev(ref_corr_indices, torch.int64, device).reshape(1, -1)
    src_idx = _dev(src_corr_indices, torch.int64, device).reshape(1, -1)
    gt = _dev(gt_corr_indices, torch.int64, device).reshape(1, -1, 2)
    if ref_idx.shape != src_idx.shape:
        raise ValueError('evaluate_sparse_correspondences: ref_corr_indices and src_corr_indices need the same length')
    out = GF.sparse_correspondence_eval_batched(ref_idx, src_idx, gt, ref_points.shape[0], src_points.shape[0])[0].cpu().numpy()
    return {'precision': out[0], 'recall': out[1], 'hit_ratio': out[2]}


def compute_registration_error(gt_transform, est_transform):
    """(rre in degrees, rte) between two 4x4 rigid transforms, computed in double on the device."""
    device = _device(gt_transform, est_transform)
    gt = _dev(gt_transform, torch.float32, device).reshape(1, 16)
    est = _dev(est_transform, torch.float32, device).reshape(1, 16)
    out = GF.registration_error_batched(gt, est, rre_threshold=0.0, rte_threshold=0.0)[0].cpu().numpy()
    return float(out[0]), float(out[1])


def evaluate_correspondences(ref_points, src_points, transform, positive_radius=0.1):
    """Overlap, inlier ratio, mean residual and count of the correspondences ``ref_points[i] <-> src_points[i]`` under ``transform``
    (fp32 on the device)."""
    device = _device(ref_points, src_points, transform)
    ref = _dev(ref_points, torch.float32, device).reshape(-1, 3)
    src = _dev(src_points, torch.float32, device).reshape(-1, 3)
    T = _dev(transform, torch.float32, device).reshape(1, 16)
    v = GF.evaluate_correspondences(ref, src, T, positive_radius=positive_radius).cpu().numpy()
    return {'overlap': float(v[1]), 'inlier_ratio': float(v[0]), 'residual': float(v[2]), 'num_corr': int(ref.shape[0])}
