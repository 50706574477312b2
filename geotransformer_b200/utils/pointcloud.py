"""``get_nearest_neighbor`` of ``geotransformer/utils/pointcloud.py:11-22`` on the device (exact brute force, csrc/feature_match.cu).

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
