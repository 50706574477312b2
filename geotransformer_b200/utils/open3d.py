"""Voxel downsampling, normal estimation, correspondence RANSAC and feature-matching RANSAC with the reference's interface
(geotransformer/utils/open3d.py:49-65 and 133-198), on the device, without Open3D.

``voxel_downsample`` follows Open3D's ``PointCloud::VoxelDownSample`` in double, values and order, and ``estimate_normals``
Open3D's ``PointCloud::EstimateNormals`` (DESIGN.md section 8a); both are pinned to restatements of those functions, not checked
against an Open3D build.

The estimates follow Open3D's registration_ransac_based_on_correspondence and (0.11's) registration_ransac_based_on_feature_matching
as the reference calls them; the sampler, the tie rule and the fp32 scoring differ from Open3D (DESIGN.md section 3b), so the
transform is not Open3D's bit for bit.
"""
import numpy as np
import torch

from .. import functional as GF


def _points(x, name, device):
    if isinstance(x, torch.Tensor):
        if not x.is_cuda:
            raise RuntimeError(f'{name} must be a numpy array or a CUDA tensor (geotransformer_b200 has no CPU path)')
        return x.detach().to(torch.float32).contiguous()
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(device)


def voxel_downsample(points, voxel_size, normals=None):
    r"""Open3D's ``voxel_down_sample(voxel_size)`` of one cloud, with the reference's signature.

    numpy input gives float64 numpy arrays, as ``np.asarray(pcd.points)`` does; a CUDA tensor gives float64 CUDA tensors.  float32
    input is widened exactly, as ``Vector3dVector`` does.  Returns ``points``, or ``(points, normals)`` when normals are given
    (averaged, not renormalised, as Open3D)."""
    on_device = isinstance(points, torch.Tensor)
    if on_device and not points.is_cuda:
        raise RuntimeError('points must be a numpy array or a CUDA tensor (geotransformer_b200 has no CPU path)')
    device = points.device if on_device else torch.device('cuda', torch.cuda.current_device())

    def _f64(x, name):
        if isinstance(x, torch.Tensor):
            if not x.is_cuda:
                raise RuntimeError(f'{name} must be a numpy array or a CUDA tensor (geotransformer_b200 has no CPU path)')
            return x.detach().to(device=device, dtype=torch.float64).reshape(-1, 3).contiguous()
        return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64).reshape(-1, 3)).to(device)

    pts = _f64(points, 'points')
    nrm = None if normals is None else _f64(normals, 'normals')
    res = GF.voxel_down_sample_batched(pts, [pts.shape[0]], voxel_size, normals=nrm)
    out = (res[0],) if normals is None else (res[0], res[2])
    if not on_device:
        out = tuple(x.cpu().numpy() for x in out)
    return out[0] if normals is None else out


def registration_with_ransac_from_correspondences(src_points, ref_points, correspondences=None, distance_threshold=0.05, ransac_n=3,
                                                  num_iterations=10000, seed=0):
    r"""Compute the transformation matrix from src_points to ref_points.

    ``correspondences``: optional (K, 2) [src index, ref index] pairs (Open3D's order); without them row i of src_points
    corresponds to row i of ref_points.  numpy inputs give a float64 (4, 4) numpy array, as Open3D returns; CUDA tensors give a
    float32 (4, 4) device tensor.  Correspondence indices are range-checked on the host (for a device tensor this costs one
    read-back of its minimum and maximum).  ``seed`` keys the sampler."""
    on_device = isinstance(src_points, torch.Tensor)
    device = src_points.device if on_device else torch.device('cuda', torch.cuda.current_device())
    src = _points(src_points, 'src_points', device).reshape(-1, 3)
    ref = _points(ref_points, 'ref_points', device).reshape(-1, 3)
    if correspondences is not None:
        if isinstance(correspondences, torch.Tensor):
            corr = correspondences.to(device=device, dtype=torch.int64).reshape(-1, 2)
            lo, hi = (corr.amin(0).tolist(), corr.amax(0).tolist()) if corr.numel() else ((0, 0), (-1, -1))
        else:
            corr = np.asarray(correspondences, dtype=np.int64).reshape(-1, 2)
            lo, hi = (corr.min(0), corr.max(0)) if corr.size else ((0, 0), (-1, -1))
            corr = torch.from_numpy(corr).to(device)
        # gather_rows zero-fills rows past the table: an unchecked index would give a wrong transform, not an error
        if min(lo) < 0 or hi[0] >= src.shape[0] or hi[1] >= ref.shape[0]:
            raise IndexError('registration_with_ransac_from_correspondences: correspondence index out of range')
        src = GF.gather_rows(src, corr[:, 0].contiguous())
        ref = GF.gather_rows(ref, corr[:, 1].contiguous())
    elif src.shape[0] != ref.shape[0]:
        raise ValueError('registration_with_ransac_from_correspondences: without correspondences src and ref need the same rows')
    res = GF.ransac_correspondences(src, ref, distance_threshold, ransac_n, num_iterations, seed=seed)
    if on_device:
        return res['transform']
    return res['transform'].cpu().numpy().astype(np.float64)


def registration_with_ransac_from_feats(src_points, ref_points, src_feats, ref_feats, distance_threshold=0.05, ransac_n=3,
                                        num_iterations=50000, val_iterations=1000, seed=0):
    r"""Compute the transformation matrix from src_points to ref_points by RANSAC on descriptor matches.

    Follows Open3D 0.11's registration_ransac_based_on_feature_matching as the reference calls it (every src point matched to its
    nearest ref descriptor, edge-length checker 0.9, distance checker ``distance_threshold``, ``num_iterations`` iterations of which
    at most ``val_iterations`` passing ones are scored against the whole ref cloud); the sampler, the validated set (the first
    passing iterations) and the fp32 scoring are the package's (DESIGN.md section 3b).  numpy inputs give a float64 (4, 4) numpy
    array; CUDA tensors give a float32 (4, 4) device tensor.  ``seed`` keys the sampler."""
    on_device = any(isinstance(x, torch.Tensor) for x in (src_points, ref_points, src_feats, ref_feats))
    device = torch.device('cuda', torch.cuda.current_device())
    for x in (src_points, ref_points, src_feats, ref_feats):
        if isinstance(x, torch.Tensor):
            device = x.device
            break
    src = _points(src_points, 'src_points', device).reshape(-1, 3)
    ref = _points(ref_points, 'ref_points', device).reshape(-1, 3)
    sf = _points(src_feats, 'src_feats', device)
    rf = _points(ref_feats, 'ref_feats', device)
    sf, rf = sf.reshape(sf.shape[0], -1), rf.reshape(rf.shape[0], -1)
    if sf.shape[0] != src.shape[0] or rf.shape[0] != ref.shape[0]:
        raise ValueError('registration_with_ransac_from_feats: one descriptor row per point')
    res = GF.ransac_features(src, ref, sf, rf, distance_threshold, ransac_n, num_iterations, val_iterations, seed=seed)
    if on_device:
        return res['transform']
    return res['transform'].cpu().numpy().astype(np.float64)


def estimate_normals(points, knn=30, radius=None):
    r"""Open3D's ``pcd.estimate_normals()`` of one cloud, with the reference's signature (``knn`` and ``radius`` select
    ``KDTreeSearchParamKNN(knn)`` or ``KDTreeSearchParamHybrid(radius, knn)``; the reference calls the default, knn 30).

    numpy input gives a float64 numpy array, as ``np.asarray(pcd.normals)`` does; a CUDA tensor gives a float64 CUDA tensor.
    float32 input is widened exactly, as ``Vector3dVector`` does.  Normals are not oriented (Open3D orients only against normals
    the cloud already has)."""
    on_device = isinstance(points, torch.Tensor)
    if on_device and not points.is_cuda:
        raise RuntimeError('points must be a numpy array or a CUDA tensor (geotransformer_b200 has no CPU path)')
    if on_device:
        pts = points.detach().to(torch.float64).reshape(-1, 3).contiguous()
    else:
        pts = torch.from_numpy(np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)).to(
            torch.device('cuda', torch.cuda.current_device()))
    out = GF.estimate_normals_batched(pts, [pts.shape[0]], knn=knn, radius=radius)
    return out if on_device else out.cpu().numpy()
