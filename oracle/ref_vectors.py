"""TEST INFRASTRUCTURE ONLY -- the reference outputs the oracle restatements are pinned against, on seeded inputs, stored as
SHA-256 digests in tests/golden/reference_ops.npz (bit-for-bit equality of an output is equality of its digest):

  collate:<case>   grid_subsampling / radius_neighbors of the reference's C++ ext (oracle/_ref) vs oracle/collate_oracle.c
  ops:<case>       pairwise_distance, knn_partition, get_point_to_node_indices, point_to_node_partition, ball_query_partition,
                   apply_transform of geotransformer.modules.ops (pointcloud_partition.py:9-107,159-175, pairwise_distance.py:4-31,
                   transformation.py:7-60) vs oracle/geo_oracle.py

Regenerate where the reference exists (it also checks the restatements against the reference live):
    python -m oracle.ref_vectors
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import geo_oracle as G  # noqa: E402
from oracle.fixture import _digest  # noqa: E402

PATH = os.path.join(ROOT, 'tests', 'golden', 'reference_ops.npz')
COLLATE_WORKLOADS = (('demo2k', 0.05), ('3dmatch20k', 0.05), ('modelnet717', 0.1))
REHASH_SIZES = (1, 2, 12, 13, 14, 28, 29, 30, 58, 59, 60, 126, 127, 128, 129, 257, 258, 542)


def adversarial_inputs(n_cases=60):
    """several ragged clouds per batch, coordinates quantised to a coarse lattice (many points per voxel, exact-distance ties,
    duplicated points), negative coordinates, 1-point clouds; (lengths, points, voxel) per case"""
    rng = np.random.default_rng(7351)
    cases = [([1], 0.0, 0.3), ([1, 1, 1, 1], 0.25, 0.5), ([40, 40, 40, 40], 0.25, 1.0), ([40, 1], 0.05, 0.3)]
    while len(cases) < n_cases:
        cases.append(([int(x) for x in rng.integers(1, 41, size=int(rng.integers(1, 5)))], float(rng.choice([0.0, 0.05, 0.25])),
                      float(rng.choice([0.3, 0.5, 1.0]))))
    out = []
    for i, (lengths, lattice, voxel) in enumerate(cases):
        g = torch.Generator().manual_seed(i)
        pts = (torch.rand(sum(lengths), 3, generator=g) - 0.5) * 4.0
        if lattice > 0:
            pts = torch.round(pts / lattice) * lattice
        out.append((torch.tensor(lengths), pts.contiguous(), voxel))
    return out


def collate_results(impl, workload, voxel=None):
    """the outputs of ``impl`` (oracle.ref_ext or oracle.collate_oracle) that must be bit-identical to the reference's; for the
    three collate workloads ``voxel`` is the first-level voxel size (default: the one of COLLATE_WORKLOADS, which the stored
    digests were made with)"""
    from geotransformer_b200.synth import make_pair
    res = {}
    if workload == 'rehash':
        # clouds whose voxel counts straddle the libstdc++ rehash thresholds (13/14, 29/30, 59/60, 127/128)
        g = torch.Generator().manual_seed(0)
        for n in REHASH_SIZES:
            pts = torch.rand(n, 3, generator=g) * 100.0          # one point per voxel with high probability
            res[f'rehash_{n}'] = impl.grid_subsampling(pts, torch.tensor([n]), 0.5)[0]
        return res
    if workload == 'adversarial':
        # grid_subsampling: values AND unordered_map order; radius_neighbors: rows up to the order inside exact-distance tie
        # groups (std::sort is unstable in both), for the self search and for the sub-sampled queries against the full support
        for i, (lens, pts, voxel) in enumerate(adversarial_inputs()):
            a, al = impl.grid_subsampling(pts, lens, voxel)
            r = voxel * 1.5
            res[f'adv{i}_points'], res[f'adv{i}_lengths'] = a, al
            res[f'adv{i}_self'] = G.canonical_neighbors(pts, pts, impl.radius_neighbors(pts, pts, lens, lens, r))
            res[f'adv{i}_sub'] = G.canonical_neighbors(a, pts, impl.radius_neighbors(a, pts, al, lens, r))
        return res
    voxel = dict(COLLATE_WORKLOADS)[workload] if voxel is None else voxel
    pair = make_pair(workload, 1)
    pts = torch.from_numpy(np.concatenate([pair['ref_points'], pair['src_points']]))
    lens = torch.tensor([len(pair['ref_points']), len(pair['src_points'])])
    for level in range(3):
        pts, lens = impl.grid_subsampling(pts, lens, voxel)
        res[f'{workload}_points_{level}'], res[f'{workload}_lengths_{level}'] = pts, lens
        voxel = voxel * 2
    res[f'{workload}_neighbors'] = impl.radius_neighbors(pts, pts, lens, lens, voxel * 1.25)     # raw: values AND order
    return res


def ops_results(ops):
    """outputs of the Boundary-2 ops of ``ops`` (geotransformer.modules.ops or oracle.geo_oracle) on seeded inputs"""
    res = {}
    for seed, n, m in ((0, 500, 40), (1, 64, 64), (2, 2000, 7)):
        g = torch.Generator().manual_seed(seed)
        pts = torch.rand(n, 3, generator=g) * 2.0
        nodes = pts[torch.randperm(n, generator=g)[:m]].contiguous() + 0.01 * torch.randn(m, 3, generator=g)
        feats_a = torch.nn.functional.normalize(torch.randn(m, 32, generator=g), dim=1)
        feats_b = torch.nn.functional.normalize(torch.randn(n, 32, generator=g), dim=1)
        c = f's{seed}'
        res[f'{c}_pairwise_distance'] = ops.pairwise_distance(nodes, pts)
        res[f'{c}_pairwise_distance_normalized'] = ops.pairwise_distance(feats_a, feats_b, normalized=True)
        for k in (1, 8, 33):
            kk = min(k, n)
            res[f'{c}_knn_{k}'] = ops.knn_partition(pts, nodes, kk)
            res[f'{c}_knn_{k}_distance'], res[f'{c}_knn_{k}_indices'] = ops.knn_partition(pts, nodes, kk, return_distance=True)
        res[f'{c}_point_to_node'] = ops.get_point_to_node_indices(pts, nodes)
        res[f'{c}_point_to_node_idx'], res[f'{c}_point_to_node_counts'] = ops.get_point_to_node_indices(pts, nodes, return_counts=True)
        for limit in (4, 16):
            for j, t in enumerate(ops.point_to_node_partition(pts, nodes, limit)):
                res[f'{c}_p2n_partition_{limit}_{j}'] = t
            for radius in (0.05, 0.3):
                for j, t in enumerate(ops.ball_query_partition(pts, nodes, radius, limit, return_count=True)):
                    res[f'{c}_ball_query_{limit}_{radius}_{j}'] = t
        T = torch.eye(4)
        q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g))
        T[:3, :3], T[:3, 3] = q, torch.randn(3, generator=g)
        res[f'{c}_apply_transform'] = ops.apply_transform(pts, T)
    return res


def digests(results):
    return {k: _digest(v.numpy()) for k, v in results.items()}


def mismatches(results, stored, prefix):
    """names whose digest differs from the stored reference digest (and stored names the results do not cover)"""
    got = digests(results)
    want = {k[len(prefix):]: str(stored[k]) for k in stored.files if k.startswith(prefix) and k[len(prefix):] in got}
    return sorted(k for k in got if want.get(k) != got[k])


def main():
    from oracle import collate_oracle, ref_ext, ref_harness
    assert ref_ext.available() and ref_harness.available(), 'needs the reference (oracle/_ref and the reference package)'
    out = {}
    for w in [w for w, _ in COLLATE_WORKLOADS] + ['rehash', 'adversarial']:
        ref, mine = digests(collate_results(ref_ext, w)), digests(collate_results(collate_oracle, w))
        assert ref == mine, f'collate restatement differs from the reference build: {w}'
        out.update({'collate:' + k: np.array(v) for k, v in ref.items()})
    ref_harness.install()
    from geotransformer.modules import ops as R
    ref, mine = digests(ops_results(R)), digests(ops_results(G))
    assert ref == mine, f'op restatements differ from the reference: {sorted(k for k in ref if ref[k] != mine[k])}'
    out.update({'ops:' + k: np.array(v) for k, v in ref.items()})
    np.savez_compressed(os.environ.get('GEOB200_REF_VECTORS_OUT') or PATH, **out)
    print(f'pinned: {len(out)} reference outputs, restatements equal')


if __name__ == '__main__':
    main()
