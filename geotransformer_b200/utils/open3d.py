"""Correspondence RANSAC with the reference's interface (geotransformer/utils/open3d.py:169-198), on the device, without Open3D.

The estimate follows Open3D's registration_ransac_based_on_correspondence as the reference calls it; the sampler, the tie rule
and the fp32 scoring differ from Open3D (DESIGN.md section 3b), so the transform is not Open3D's bit for bit.
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
