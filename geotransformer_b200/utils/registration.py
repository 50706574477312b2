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


# RPMNet's ModelNet metrics (reference utils/registration.py:17-130) through ``functional.rpmnet_metrics_batched`` (contract in
# DESIGN.md section 8a).  Numpy in gives numpy out (np.float64, and np.float32 for the translation errors, the reference's types);
# CUDA tensors give 0-d device tensors.

def _rpmnet_one(raw, ref, src, gt, est, on_device=None):
    """(8,) float64 device row of one pair, and whether to answer with device tensors (any input one, unless given)"""
    device = _device(raw, ref, src, gt, est)
    if on_device is None:
        on_device = any(isinstance(x, torch.Tensor) for x in (raw, ref, src, gt, est))
    clouds = [_dev(x, torch.float32, device).reshape(-1, 3) for x in (raw, ref, src)]
    T = [_dev(x, torch.float32, device).reshape(1, 4, 4) for x in (gt, est)]
    row = GF.rpmnet_metrics_batched(clouds[0], [clouds[0].shape[0]], clouds[1], [clouds[1].shape[0]], clouds[2], [clouds[2].shape[0]],
                                    *T)[0]
    return row, on_device


def _as_transform(rotation=None, translation=None):
    T = np.eye(4, dtype=np.float32)
    if rotation is not None:
        T[:3, :3] = np.asarray(rotation, np.float32)
    if translation is not None:
        T[:3, 3] = np.asarray(translation, np.float32)
    return T


def _out(row, on_device, cols, dtypes):
    if on_device:
        return tuple(row[c].to(torch.float32 if d == np.float32 else torch.float64) for c, d in zip(cols, dtypes))
    v = row.cpu().numpy()
    return tuple(d(v[c]) for c, d in zip(cols, dtypes))


def _one_point(device):
    return torch.zeros((1, 3), dtype=torch.float32, device=device)


def compute_transform_mse_and_mae(gt_transform, est_transform):
    """(r_mse, r_mae, t_mse, t_mae): the Euler angles ('xyz', degrees) of scipy's ``Rotation.from_matrix`` of both rotations,
    their unwrapped differences' MSE and MAE, and the translations' MSE and MAE in fp32.  ValueError if a rotation has det <= 0."""
    device = _device(gt_transform, est_transform)
    p = _one_point(device)
    row, on_device = _rpmnet_one(p, p, p, gt_transform, est_transform,
                                 on_device=isinstance(gt_transform, torch.Tensor) or isinstance(est_transform, torch.Tensor))
    return _out(row, on_device, (3, 4, 5, 6), (np.float64, np.float64, np.float32, np.float32))


def compute_rotation_mse_and_mae(gt_rotation, est_rotation):
    """(mse, mae) of the Euler angles ('xyz', degrees) of two rotation matrices, as compute_transform_mse_and_mae"""
    if isinstance(gt_rotation, torch.Tensor) or isinstance(est_rotation, torch.Tensor):
        device = _device(gt_rotation, est_rotation)
        T = [torch.eye(4, dtype=torch.float32, device=device) for _ in range(2)]
        T[0][:3, :3] = _dev(gt_rotation, torch.float32, device)
        T[1][:3, :3] = _dev(est_rotation, torch.float32, device)
        return compute_transform_mse_and_mae(*T)[:2]
    return compute_transform_mse_and_mae(_as_transform(gt_rotation), _as_transform(est_rotation))[:2]


def compute_translation_mse_and_mae(gt_translation, est_translation):
    """(mse, mae) of two translations in fp32"""
    if isinstance(gt_translation, torch.Tensor) or isinstance(est_translation, torch.Tensor):
        device = _device(gt_translation, est_translation)
        T = [torch.eye(4, dtype=torch.float32, device=device) for _ in range(2)]
        T[0][:3, 3] = _dev(gt_translation, torch.float32, device)
        T[1][:3, 3] = _dev(est_translation, torch.float32, device)
        return compute_transform_mse_and_mae(*T)[2:]
    return compute_transform_mse_and_mae(_as_transform(translation=gt_translation), _as_transform(translation=est_translation))[2:]


def compute_modified_chamfer_distance(raw_points, ref_points, src_points, gt_transform, est_transform):
    """RPMNet's modified Chamfer distance: the mean exact nearest-neighbour distance from the estimate-aligned src points to the raw
    shape, plus the mean from the ref points to the raw shape aligned by est gt^-1 (fp64 distances over fp32 coordinates)"""
    row, on_device = _rpmnet_one(raw_points, ref_points, src_points, gt_transform, est_transform)
    return _out(row, on_device, (0,), (np.float64,))[0]


def compute_relative_rotation_error(gt_rotation, est_rotation):
    """RRE = acos((trace(R^T gt) - 1) / 2) in degrees, in double on the device (registration_error_batched)"""
    device = _device(gt_rotation, est_rotation)
    T = [torch.eye(4, dtype=torch.float32, device=device).reshape(1, 16) for _ in range(2)]
    for t, r in zip(T, (gt_rotation, est_rotation)):
        t.view(4, 4)[:3, :3] = _dev(r, torch.float32, device)
    v = GF.registration_error_batched(T[0], T[1], rre_threshold=0.0, rte_threshold=0.0)[0, 0]
    return v if isinstance(gt_rotation, torch.Tensor) or isinstance(est_rotation, torch.Tensor) else float(v)


def compute_relative_translation_error(gt_translation, est_translation):
    """RTE = |gt - est|, in double on the device (registration_error_batched)"""
    device = _device(gt_translation, est_translation)
    T = [torch.eye(4, dtype=torch.float32, device=device).reshape(1, 16) for _ in range(2)]
    for t, x in zip(T, (gt_translation, est_translation)):
        t.view(4, 4)[:3, 3] = _dev(x, torch.float32, device).reshape(3)
    v = GF.registration_error_batched(T[0], T[1], rre_threshold=0.0, rte_threshold=0.0)[0, 1]
    return v if isinstance(gt_translation, torch.Tensor) or isinstance(est_translation, torch.Tensor) else float(v)


def compute_registration_rmse(src_points, gt_transform, est_transform):
    """mean |T_gt p - T_est p| over the src points: the Evaluator's ModelNet RMSE (fp32 transforms, double sum) of one pair"""
    device = _device(src_points, gt_transform, est_transform)
    src = _dev(src_points, torch.float32, device).reshape(-1, 3)
    gt, est = _dev(gt_transform, torch.float32, device).reshape(4, 4), _dev(est_transform, torch.float32, device).reshape(4, 4)
    z_i, z_f = torch.zeros((1, 2), dtype=torch.int64, device=device), torch.zeros((1, 3), dtype=torch.float32, device=device)
    n0 = torch.zeros((1,), dtype=torch.int32, device=device)
    # no correspondences (device counts 0): only the RMSE column is read
    v = GF.evaluate(z_i, z_f[0, :1], z_i[:, 0], z_i[:, 1], z_f, z_f, gt, est, src, 2, 0.1, 0.1, n_gt=n0, n_node_corr=n0, n_corr=n0)[4]
    return v if any(isinstance(x, torch.Tensor) for x in (src_points, gt_transform, est_transform)) else float(v)
