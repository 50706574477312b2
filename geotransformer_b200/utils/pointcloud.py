"""``get_nearest_neighbor`` and ``regularize_normals`` of ``geotransformer/utils/pointcloud.py:11-37`` on the device
(``get_nearest_neighbor``: exact brute force, csrc/feature_match.cu; ``regularize_normals``: csrc/normals.cu).

Inputs are numpy arrays or CUDA tensors of points or descriptors (any width C in 1..1024), rounded to float32.  numpy inputs run
on the current CUDA device and give numpy outputs; CUDA tensors give device tensors; a CPU tensor raises RuntimeError.
"""
import numpy as np
import torch

from .. import functional as GF


def _rows(x, name, device):
    if isinstance(x, torch.Tensor):
        if not x.is_cuda:
            raise RuntimeError(f'{name} must be a numpy array or a CUDA tensor (geotransformer_b200 has no CPU path)')
        x = x.detach().to(torch.float32)
    else:
        x = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(device)
    return x.reshape(x.shape[0], -1).contiguous()


def _device(*xs):
    for x in xs:
        if isinstance(x, torch.Tensor):
            if not x.is_cuda:
                raise RuntimeError('inputs must be numpy arrays or CUDA tensors (geotransformer_b200 has no CPU path)')
            return x.device, True
    return torch.device('cuda', torch.cuda.current_device()), False


def get_nearest_neighbor(q_points, s_points, return_index=False):
    r"""Nearest support row of every query row, as ``cKDTree(s_points).query(q_points, k=1)``: float64 Euclidean distances and,
    with ``return_index``, int64 indices.  The index is the argmin of the fp64 squared distance (lowest index on exact ties)."""
    device, on_device = _device(q_points, s_points)
    q, s = _rows(q_points, 'q_points', device), _rows(s_points, 's_points', device)
    if q.shape[1] != s.shape[1]:
        raise ValueError('get_nearest_neighbor: q_points and s_points need the same width')
    index, dist = GF.feature_nearest_neighbor(q, s)
    if not on_device:
        index, dist = index.cpu().numpy(), dist.cpu().numpy()
    return (dist, index) if return_index else dist


def regularize_type(points_dtype, normals_dtype):
    """the type in which the drop-in takes the point-normal dot products: numpy's type of ``points * normals`` for float inputs,
    float32 only when both are float32 (the result is float64 either way)"""
    both32 = np.dtype(points_dtype) == np.float32 and np.dtype(normals_dtype) == np.float32
    return np.dtype(np.float32) if both32 else np.dtype(np.float64)


def regularize_normals(points, normals, positive=True):
    r"""Orient each normal by the sign of s_i = p_i . n_i, with the reference's signature.  ``positive=True`` makes the normals
    face the origin: n_i is kept when s_i < 0 and negated otherwise.  ``positive=False`` makes them face away from it: n_i is
    negated when s_i < 0 and kept otherwise.  The values, signed zeros included, and the float64 result type are those of the
    reference's numpy code (DESIGN.md section 8a).  numpy inputs give a numpy array; CUDA tensors give a device tensor."""
    device, on_device = _device(points, normals)
    if on_device:
        return GF.regularize_normals(points, normals, positive)
    p, n = np.asarray(points), np.asarray(normals)
    dt = regularize_type(p.dtype, n.dtype)
    out = GF.regularize_normals(torch.from_numpy(np.ascontiguousarray(p, dtype=dt)).to(device),
                                torch.from_numpy(np.ascontiguousarray(n, dtype=dt)).to(device), positive)
    return out.cpu().numpy()
