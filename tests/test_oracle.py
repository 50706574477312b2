"""The oracle itself (CPU): plain-C collate restatement and op restatements vs the stored outputs of the real reference
(tests/golden/reference_ops.npz), and the torch restatement of the forward vs the committed reference fixtures."""
import numpy as np
import pytest
import torch

from geotransformer_b200.synth import make_pair
from oracle import collate_oracle as co
from oracle import geo_oracle as G


def _stack(pair):
    pts = torch.from_numpy(np.concatenate([pair['ref_points'], pair['src_points']]))
    return pts, torch.tensor([len(pair['ref_points']), len(pair['src_points'])])


@pytest.fixture(scope='module')
def reference_ops():
    """digests of the reference's outputs on the seeded inputs of oracle/ref_vectors.py (tests/golden/reference_ops.npz)"""
    import os
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_ops.npz'))


@pytest.mark.parametrize('workload,voxel', [('demo2k', 0.05), ('3dmatch20k', 0.05), ('modelnet717', 0.1)])
def test_c_restatement_matches_reference_build(workload, voxel, reference_ops):
    """three grid_subsampling levels (values AND unordered_map order) and the radius_neighbors table of the last level (values
    AND order) of the plain-C restatement, bit for bit equal to the reference build's on pair 1 of the workload"""
    from oracle import ref_vectors
    assert not ref_vectors.mismatches(ref_vectors.collate_results(co, workload, voxel), reference_ops, 'collate:')


def test_grid_subsample_golden_order(golden):
    """against the committed fixture (reference output), no reference build needed"""
    gold = golden('demo2k')
    pts, lens = _stack(make_pair('demo2k', 0))
    v = 0.05
    for i in range(1, 4):
        pts, lens = co.grid_subsampling(pts, lens, v)
        assert np.array_equal(pts.numpy(), gold[f'points_{i}']) and lens.tolist() == gold[f'lengths_{i}'].tolist()
        v *= 2


def test_rehash_schedule_edge_sizes(reference_ops):
    """clouds whose voxel counts straddle the libstdc++ rehash thresholds (13/14, 29/30, 59/60, 127/128): grid_subsampling of
    the restatement bit for bit equal to the reference build's"""
    from oracle import ref_vectors
    assert not ref_vectors.mismatches(ref_vectors.collate_results(co, 'rehash'), reference_ops, 'collate:')


def test_forward_restatement_matches_reference_fixture(golden, models):
    """torch restatement vs the real reference on the ModelNet-shape pair (teacher-forced neighbour tables)"""
    cfg, sd, _ = models('modelnet')
    gold = golden('modelnet717')
    pair = make_pair('modelnet717', 0)
    data = G.collate_pair(pair, cfg, gold['neighbor_limits'].tolist())
    for i in range(1, cfg.backbone.num_stages):
        assert np.array_equal(data['points'][i].numpy(), gold[f'points_{i}'])
    for key in ('neighbors', 'subsampling', 'upsampling'):
        for i in range(len(data[key])):
            want = torch.from_numpy(gold[f'{key}_{i}'].astype(np.int64))
            q = data['points'][i + (1 if key == 'subsampling' else 0)]
            s = data['points'][i + (1 if key == 'upsampling' else 0)]
            assert torch.equal(G.canonical_neighbors(q, s, data[key][i]), G.canonical_neighbors(q, s, want))
            data[key][i] = want
    with torch.no_grad():
        out = G.forward(sd, cfg, data)
    assert np.abs(out['ref_feats_c'].numpy() - gold['ref_feats_c']).max() < 1e-5
    assert np.array_equal(out['ref_node_corr_indices'].numpy(), gold['ref_node_corr_indices'])
    assert np.array_equal(out['ref_corr_points'].numpy(), gold['ref_corr_points'])
    assert np.abs(out['estimated_transform'].numpy() - gold['estimated_transform']).max() < 1e-5
    # ground-truth superpoint correspondences (matching.py:231-315) and the Evaluator (loss.py:95-159)
    assert np.array_equal(out['gt_node_corr_indices'].numpy(), gold['gt_node_corr_indices'])
    assert np.abs(out['gt_node_corr_overlaps'].numpy() - gold['gt_node_corr_overlaps']).max() < 1e-6
    metrics = G.evaluate(cfg, out, data['transform'])
    assert sorted(metrics) == gold['metric_names'].tolist()
    for name, v in zip(gold['metric_names'].tolist(), gold['metric_values']):
        assert abs(float(metrics[name]) - v) < (1e-3 if name == 'RRE' else 1e-5), name


def test_evaluator_variants_match_reference_fixture(golden, models):
    """the three Evaluator variants (3DMatch / KITTI / ModelNet, loss.py:95-159) of the restatement on the demo pair vs the
    numbers the real reference Evaluators produced on the same outputs"""
    from geotransformer_b200.config import make_cfg
    cfg, sd, _ = models('3dmatch')
    gold = golden('demo2k')
    pair = make_pair('demo2k', 0)
    data = G.collate_pair(pair, cfg, gold['neighbor_limits'].tolist())
    for key in ('neighbors', 'subsampling', 'upsampling'):
        for i in range(len(data[key])):
            data[key][i] = torch.from_numpy(gold[f'{key}_{i}'].astype(np.int64))      # the reference's exact-tie order
    with torch.no_grad():
        out = G.forward(sd, cfg, data)
    assert np.array_equal(out['gt_node_corr_indices'].numpy(), gold['gt_node_corr_indices'])
    for variant, suffix in (('3dmatch', ''), ('kitti', '_kitti'), ('modelnet', '_modelnet')):
        metrics = G.evaluate(make_cfg(variant), out, data['transform'])
        assert sorted(metrics) == gold['metric_names' + suffix].tolist()
        for name, v in zip(gold['metric_names' + suffix].tolist(), gold['metric_values' + suffix]):
            assert abs(float(metrics[name]) - v) < (1e-3 if name == 'RRE' else 1e-5), (variant, name)


def test_calibration_restatement_matches_reference_fixture(golden, models):
    """calibrate_neighbors_stack_mode (utils/data.py:190-217): restatement vs the limits the real reference computed"""
    cfg, _, _ = models('3dmatch')
    keys = ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')
    pairs = [{k: make_pair('demo2k', i)[k] for k in keys} for i in range(3)]
    gold = golden('calibration')
    for thr in (2000, 150):
        assert np.array_equal(G.calibrate_neighbors(pairs, cfg, sample_threshold=thr), gold[f'limits_threshold_{thr}'])


def test_sinkhorn_marginals_property():
    g = torch.Generator().manual_seed(1)
    s = torch.randn(3, 20, 20, generator=g)
    rm, cm = torch.rand(3, 20, generator=g) > 0.2, torch.rand(3, 20, generator=g) > 0.2
    out = G.optimal_transport(torch.tensor(1.0), s, rm, cm, 100).exp()
    rows = out[:, :-1, :].sum(dim=2)
    assert (rows[rm] - 1).abs().max() < 1e-3


def test_procrustes_degenerate_cases():
    src = torch.randn(1, 10, 3)
    T = G.weighted_procrustes(src, src + 1.0, torch.zeros(1, 10))
    assert torch.equal(T[0], torch.eye(4))


@pytest.mark.parametrize('c,n,sigma_d,extent', [(256, 100, 0.2, 2.0), (128, 90, 4.8, 20.0)])
def test_tabulated_structure_embedding_model_vs_oracle(c, n, sigma_d, extent):
    """oracle/gse_table_model.py (the arithmetic of csrc/gse_table.cu: fp64-built table of proj(sinusoid(x)) on a 1/256 grid,
    fp16 forward differences, fp32 lerp) reproduces GeometricStructureEmbedding.forward to ~3e-6: the tabulation error is an
    order of magnitude below the 2e-5 of the split-precision tensor-core kernels it replaces"""
    import math
    from oracle.gse_table_model import structure_embedding_tabulated
    g = torch.Generator().manual_seed(n)
    pts = torch.rand(n, 3, generator=g) * extent
    sd = {'e.embedding.div_term': torch.exp(torch.arange(0, c, 2).float() * (-np.log(10000.0) / c)),
          'e.proj_d.weight': torch.randn(c, c, generator=g) / math.sqrt(c), 'e.proj_d.bias': torch.randn(c, generator=g) * 0.1,
          'e.proj_a.weight': torch.randn(c, c, generator=g) / math.sqrt(c), 'e.proj_a.bias': torch.randn(c, generator=g) * 0.1}
    want = G.structure_embedding(sd, 'e.', pts, sigma_d, 15, 3)
    got = structure_embedding_tabulated(sd, 'e.', pts, sigma_d, 15, 3)
    assert float((got - want).abs().max()) < 1e-5
    coarse = structure_embedding_tabulated(sd, 'e.', pts, sigma_d, 15, 3, inv_step=64)
    assert float((coarse - want).abs().max()) < 5e-5


def test_c_restatement_matches_reference_build_on_adversarial_small_inputs(reference_ops):
    """60 seeded cases: several ragged clouds per batch, coordinates quantised to a coarse lattice (many points per voxel,
    exact-distance ties, duplicated points), negative coordinates, 1-point clouds.  grid_subsampling: values AND unordered_map
    order bit for bit; radius_neighbors (self and sub-sampled queries): identical rows up to the order inside exact-distance
    tie groups (std::sort is unstable in both) -- all against the reference build's outputs"""
    from oracle import ref_vectors
    assert not ref_vectors.mismatches(ref_vectors.collate_results(co, 'adversarial'), reference_ops, 'collate:')


def test_boundary_2_op_restatements_match_the_reference(reference_ops):
    """the oracle's pairwise_distance / knn_partition / get_point_to_node_indices / point_to_node_partition / ball_query_partition /
    apply_transform are bit-identical to geotransformer.modules.ops on seeded inputs (oracle/ref_vectors.py)"""
    from oracle import ref_vectors
    assert not ref_vectors.mismatches(ref_vectors.ops_results(G), reference_ops, 'ops:')


def test_restatement_matches_the_reference_on_other_pairs(models):
    """the committed fixtures pin the restatement on pair 0 of each workload; here oracle/geo_oracle.py runs on further seeded
    pairs of all three models (tests/golden/other_pairs.npz, written by ``python -m oracle.make_golden other_pairs``) and is
    compared with the reference's outputs on them: collate tables up to tie order (the reference's tie order teacher-forced),
    features, matching scores, correspondences (as a set when two coarse scores tie to 1e-5), transform, gt superpoint pairs,
    all three Evaluator variants"""
    import os
    from geotransformer_b200.config import make_cfg
    from oracle import fixture
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'other_pairs.npz'))
    cases = z['cases'].tolist()
    assert len(cases) == 5
    for case in cases:
        workload, index = case.split(':')
        g = {k[len(case) + 1:]: z[k] for k in z.files if k.startswith(case + '/')}
        pair = make_pair(workload, int(index))
        cfg, sd, _ = models(pair['config'])
        ref = fixture.expand(workload, g, int(index))                      # the reference's level points and tables
        data = G.collate_pair(pair, cfg, g['neighbor_limits'].tolist())
        for i in range(1, cfg.backbone.num_stages):
            assert np.array_equal(data['points'][i].numpy(), ref[f'points_{i}']), (case, i)
        for key in fixture.TABLE_KEYS:
            data[key] = [torch.from_numpy(ref[f'{key}_{i}'].astype(np.int64)) for i in range(len(data[key]))]
        with torch.no_grad():
            out = G.forward(sd, cfg, data)
        variants = [k[len('metric_names_'):] for k in g if k.startswith('metric_names_')]
        metrics = {v: {k: float(x) for k, x in G.evaluate(make_cfg(v), out, data['transform']).items()} for v in variants}
        assert len(variants) == 3
        assert not fixture.compare_outputs(out, g, metrics), (case, fixture.compare_outputs(out, g, metrics))
