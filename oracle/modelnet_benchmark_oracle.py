"""CPU restatement (numpy) of the ModelNet validation / test pairs of geotransformer_b200/csrc/augment.cu
(``geob200_modelnet_benchmark_pairs_batched``).

TEST INFRASTRUCTURE ONLY.  The reference's ``ModelNetPairDataset.__getitem__`` with ``deterministic=True`` and the shipped options
(twice_sample, plane crop, no twice_transform, jitter), written as plain numpy calls on ``np.random.RandomState(index)``: the draws
come in the reference's order from the same generator, so this restatement reproduces the reference bit for bit
(tests/test_modelnet_benchmark_oracle.py pins it to the fixture written from the reference itself).  It also reports what the
device cannot take from numpy: the shape row of every output point and the smallest gap between two crop distances.
"""
import numpy as np
from scipy.spatial.transform import Rotation


def crop_count(n, keep_ratio):
    return int(np.floor(n * keep_ratio + 0.5))


def _crop(points, rs, keep_ratio):
    """random_crop_point_cloud_with_plane: (kept points, their rows, smallest gap between sorted distances)"""
    phi = rs.uniform(0.0, 2 * np.pi)
    theta = rs.uniform(0.0, np.pi)
    normal = np.asarray([np.sin(theta) * np.cos(phi), np.sin(theta) * np.sin(phi), np.cos(theta)])
    k = crop_count(points.shape[0], keep_ratio)
    d = np.dot(points, normal)
    order = np.argsort(-d, kind='stable')[:k]               # ties to the lowest row; numpy's default sort leaves them open
    ds = np.sort(d)
    gap = float(np.min(np.diff(ds))) if len(ds) > 1 else np.inf
    return points[order], order, gap


def _sample(points, rows, rs, num_points):
    """random_sample_points"""
    n = points.shape[0]
    sel = rs.permutation(n)
    if n > num_points:
        sel = sel[:num_points]
    elif n < num_points:
        parts = [sel] * (num_points // n)
        if num_points % n:
            parts.append(sel[:num_points % n])
        sel = np.concatenate(parts, axis=0)
    return points[sel], rows[sel]


def benchmark_pair(shape, index, num_points=717, keep_ratio=0.7, rotation_magnitude=45.0, translation_magnitude=0.5,
                   noise_magnitude=0.05):
    """the pair of dataset index ``index`` from the raw shape (N, 3) fp32: dict(ref_points, src_points (num_points, 3) fp32,
    transform (4, 4) fp32, ref_origin, src_origin (the shape row of every output point), gap (smallest crop-distance gap of the
    two clouds))"""
    rs = np.random.RandomState(int(index))
    points = np.asarray(shape, dtype=np.float32)
    points = points - points.mean(axis=0)                   # normalize_points, fp32
    points = points / np.max(np.linalg.norm(points, axis=1))
    euler = rs.rand(3) * np.pi * rotation_magnitude / 180.0  # random_sample_transform
    R = Rotation.from_euler('zyx', euler).as_matrix()
    t = rs.uniform(-translation_magnitude, translation_magnitude, 3)
    inv_R = R.T
    inv_t = -np.matmul(inv_R, t)
    ref = points
    src = np.matmul(points, inv_R.T) + inv_t
    rows = np.arange(points.shape[0])
    ref, ref_rows, g0 = _crop(ref, rs, keep_ratio)
    src, src_rows, g1 = _crop(src, rs, keep_ratio)
    ref, ref_rows = _sample(ref, ref_rows, rs, num_points)
    src, src_rows = _sample(src, src_rows, rs, num_points)
    ref = ref + np.clip(rs.normal(scale=0.01, size=ref.shape), a_min=-noise_magnitude, a_max=noise_magnitude)
    src = src + np.clip(rs.normal(scale=0.01, size=src.shape), a_min=-noise_magnitude, a_max=noise_magnitude)
    a = rs.permutation(num_points)
    b = rs.permutation(num_points)
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return dict(ref_points=ref[a].astype(np.float32), src_points=src[b].astype(np.float32), transform=T.astype(np.float32),
                ref_origin=rows[ref_rows[a]], src_origin=rows[src_rows[b]], gap=min(g0, g1))


def synthetic_shapes(n, seed, small_every=5, small=(600, 1100), labels=(0, 1, 2, 3, 4, 5, 7, 8, 11)):
    """seeded raw shapes: 2 048 points, and ``small`` points for every ``small_every``-th one (shapes small_every - 1, 2 small_every - 1,
    ...; a crop of fewer than 717 points); labels cycle through ``labels`` (5 is a symmetric class, which the asymmetric split drops)"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        m = int(rng.integers(*small)) if small_every and i % small_every == small_every - 1 else 2048
        p = (rng.standard_normal((m, 3)) * [0.3, 0.5, 0.2] + rng.uniform(-1, 1, 3)).astype(np.float32)
        out.append({'points': p, 'normals': np.zeros_like(p), 'label': labels[i % len(labels)]})
    return out
