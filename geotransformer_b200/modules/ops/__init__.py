"""Op surface of ``geotransformer.modules.ops`` (reference ``modules/ops/__init__.py:1-21``) on the H100 path."""
import torch

from ... import ext as _ext
from ... import functional as GF


def grid_subsample(points, lengths, voxel_size):
    """reference ``modules/ops/grid_subsample.py:7-22``."""
    s_points, s_lengths = _ext.grid_subsampling(points, lengths, voxel_size)
    return s_points, s_lengths


def radius_search(q_points, s_points, q_lengths, s_lengths, radius, neighbor_limit):
    """reference ``modules/ops/radius_search.py:7-27``; returns a CONTIGUOUS (N, min(limit, max_count)) table (the
    reference returns a strided view that ``to_cuda`` later densifies, ``utils/torch.py:113-123``)."""
    return _ext.radius_neighbors(q_points, s_points, q_lengths, s_lengths, radius, neighbor_limit=max(int(neighbor_limit), 0))


def radius_search_deferred(q_points, s_points, q_lengths, s_lengths, radius, neighbor_limit):
    """radius_search without the host read-back: returns (table (N, limit), max_count device int32[1]); the caller cuts
    the table to min(limit, max_count) columns once it has read the counts (one sync for many searches)."""
    return _ext.radius_neighbors_deferred(q_points, s_points, q_lengths, s_lengths, radius, int(neighbor_limit))


def point_to_node_partition(points, nodes, point_limit, return_count=False):
    """reference ``modules/ops/pointcloud_partition.py:60-107``."""
    return GF.point_to_node_partition(points, nodes, point_limit, return_count)


def knn_partition(points, nodes, k, return_distance=False):
    """reference ``modules/ops/pointcloud_partition.py:35-57``."""
    return GF.knn_partition(points, nodes, k, return_distance)


def get_point_to_node_indices(points, nodes, return_counts=False):
    """reference ``modules/ops/pointcloud_partition.py:9-32``."""
    return GF.point_to_node_indices(points, nodes, return_counts)


def ball_query_partition(points, nodes, radius, point_limit, return_count=False):
    """reference ``modules/ops/pointcloud_partition.py:159-175``."""
    node_knn_distances, node_knn_indices = GF.knn_partition(points, nodes, point_limit, return_distance=True)
    node_knn_masks = torch.lt(node_knn_distances, radius)
    node_knn_indices = torch.where(node_knn_masks, node_knn_indices, torch.full_like(node_knn_indices, points.shape[0]))
    if return_count:
        return node_knn_indices, node_knn_masks, node_knn_masks.sum(1)
    return node_knn_indices, node_knn_masks


def pairwise_distance(x, y, normalized=False, channel_first=False):
    """reference ``modules/ops/pairwise_distance.py:4-31``."""
    return GF.pairwise_distance(x, y, normalized, channel_first)


def index_select(data, index, dim):
    """reference ``modules/ops/index_select.py:4-31`` (pure indexing; dim 0 on float tables uses the gather kernel)."""
    if dim == 0 and data.is_cuda and data.dtype == torch.float32 and data.ndim == 2 and data.is_contiguous():
        return GF.gather_rows(data, index.contiguous())
    out = data.index_select(dim, index.reshape(-1))
    if index.ndim > 1:
        out = out.view(*data.shape[:dim], *index.shape, *data.shape[dim:][1:])
    return out


def apply_transform(points, transform):
    """reference ``modules/ops/transformation.py:7-60`` (points only): Q = P R^T + t."""
    if transform.ndim == 2:
        return GF.apply_transform(points, transform.contiguous())
    return torch.stack([GF.apply_transform(p, t.contiguous()) for p, t in zip(points, transform)])
