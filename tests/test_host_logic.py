"""Host-side logic that needs no GPU: configs, synthetic data, weight schema, loud failure without CUDA tensors."""
import numpy as np
import pytest
import torch

from geotransformer_b200.config import make_cfg
from geotransformer_b200.synth import make_pair, WORKLOADS


def test_configs_match_reference_hyperparameters():
    c = make_cfg('3dmatch')
    assert c.backbone.num_stages == 4 and abs(c.backbone.init_radius - 0.0625) < 1e-12 and abs(c.backbone.init_sigma - 0.05) < 1e-12
    assert c.geotransformer.input_dim == 1024 and c.geotransformer.hidden_dim == 256 and c.model.num_points_in_patch == 64
    k = make_cfg('kitti')
    assert k.backbone.num_stages == 5 and k.geotransformer.hidden_dim == 128 and k.fine_matching.topk == 2
    assert abs(k.backbone.init_radius - 1.275) < 1e-12 and k.geotransformer.sigma_d == 4.8
    m = make_cfg('modelnet')
    assert m.backbone.num_stages == 3 and m.model.fine_level == 0 and m.coarse_matching.num_correspondences == 128


def test_state_dict_schema(models):
    """key names / shapes of SURVEY.md appendix A (the weight interchange contract)"""
    cfg, sd, model = models('3dmatch')
    assert len(sd) == 269
    assert sum(v.numel() for k, v in sd.items() if not k.endswith('kernel_points') and not k.endswith('div_term')) == 9829377
    assert tuple(sd['backbone.encoder1_1.KPConv.weights'].shape) == (15, 1, 64)
    assert tuple(sd['backbone.encoder1_1.KPConv.kernel_points'].shape) == (15, 3)
    assert tuple(sd['backbone.encoder1_2.unary1.mlp.weight'].shape) == (32, 64)
    assert tuple(sd['backbone.decoder3.mlp.weight'].shape) == (512, 1536)
    assert tuple(sd['backbone.decoder2.mlp.weight'].shape) == (256, 768)
    assert 'backbone.decoder2.norm.norm.weight' not in sd            # LastUnaryBlock has no norm
    assert 'backbone.encoder1_2.unary_shortcut.mlp.weight' in sd and 'backbone.encoder2_3.unary_shortcut.mlp.weight' not in sd
    assert tuple(sd['transformer.embedding.embedding.div_term'].shape) == (128,)
    assert tuple(sd['transformer.in_proj.weight'].shape) == (256, 1024)
    assert 'transformer.transformer.layers.0.attention.attention.proj_p.weight' in sd
    assert 'transformer.transformer.layers.1.attention.attention.proj_p.weight' not in sd
    assert tuple(sd['transformer.transformer.layers.5.output.expand.weight'].shape) == (512, 256)
    assert sd['optimal_transport.alpha'].shape == ()
    _, ksd, _ = models('kitti')
    assert tuple(ksd['backbone.decoder4.mlp.weight'].shape) == (1024, 3072) and 'backbone.encoder5_3.KPConv.weights' in ksd
    _, msd, _ = models('modelnet')
    assert tuple(msd['backbone.decoder1.mlp.weight'].shape) == (256, 384) and 'backbone.encoder4_1.KPConv.weights' not in msd


def test_synthetic_pairs_are_deterministic_and_consistent():
    for w in WORKLOADS:
        if w == 'kitti60k':
            continue
        a, b = make_pair(w, 3), make_pair(w, 3)
        assert all(np.array_equal(a[k], b[k]) for k in ('ref_points', 'src_points', 'transform'))
        assert not np.array_equal(a['ref_points'], make_pair(w, 4)['ref_points'])
        T = a['transform'].astype(np.float64)
        R = T[:3, :3]
        assert np.allclose(R @ R.T, np.eye(3), atol=1e-6) and abs(np.linalg.det(R) - 1) < 1e-6
        assert a['ref_points'].dtype == np.float32 and a['ref_feats'].shape == (a['ref_points'].shape[0], 1)
    p = make_pair('3dmatch20k', 0)
    assert p['ref_points'].shape == (20000, 3)


def test_ops_fail_loudly_on_cpu_tensors():
    """no silent CPU fallback: the functional layer refuses non-CUDA tensors"""
    from geotransformer_b200 import functional as GF
    x = torch.randn(8, 4)
    with pytest.raises(RuntimeError):
        GF.linear(x, torch.randn(3, 4))
    with pytest.raises(RuntimeError):
        GF.l2_normalize(x)
    with pytest.raises(RuntimeError):
        GF.point_to_node_partition(torch.rand(10, 3), torch.rand(2, 3), 4)
    from geotransformer_b200.modules import ops
    for call in (lambda: ops.knn_partition(torch.rand(10, 3), torch.rand(2, 3), 4),
                 lambda: ops.pairwise_distance(torch.rand(10, 3), torch.rand(2, 3)),
                 lambda: ops.get_point_to_node_indices(torch.rand(10, 3), torch.rand(2, 3)),
                 lambda: ops.ball_query_partition(torch.rand(10, 3), torch.rand(2, 3), 0.5, 4),
                 lambda: ops.apply_transform(torch.rand(10, 3), torch.eye(4)),
                 lambda: GF.group_norm_batched(torch.rand(8, 32), torch.ones(32), torch.zeros(32), 32, (2, 2, 2, 2))):
        with pytest.raises(RuntimeError):
            call()


def test_boundary_2_op_surface_is_complete():
    """every name geotransformer/modules/ops/__init__.py:1-21 exports on the registration path exists here"""
    from geotransformer_b200.modules import ops
    for name in ('grid_subsample', 'radius_search', 'index_select', 'pairwise_distance', 'get_point_to_node_indices',
                 'point_to_node_partition', 'knn_partition', 'ball_query_partition', 'apply_transform'):
        assert callable(getattr(ops, name)), name


def test_forward_batch_needs_the_native_drivers(models):
    """the batched forward has no per-op fallback: it fails loudly instead of silently running something else"""
    cfg, sd, model = models('3dmatch')
    if hasattr(model, '_native'):
        del model._native
    with pytest.raises(RuntimeError, match='native'):
        model.forward_batch({'batch_size': 2})


def test_forward_batch_test_hooks_are_for_one_pair(models):
    """taps and forced coarse correspondences describe one pair: a batch of two is refused before anything touches the device"""
    cfg, sd, model = models('3dmatch')
    if hasattr(model, '_native'):
        del model._native
    with pytest.raises(ValueError, match='one pair'):
        model.forward_batch({'batch_size': 2}, taps={})
    forced = (torch.zeros(4, dtype=torch.int64), torch.zeros(4, dtype=torch.int64), torch.zeros(4))
    with pytest.raises(ValueError, match='one pair'):
        model.forward_batch({'batch_size': 2, 'forced_node_corr': forced})


def test_unsupported_module_options_are_rejected():
    from geotransformer_b200.modules.geotransformer import LocalGlobalRegistration, GeometricStructureEmbedding
    with pytest.raises(NotImplementedError):
        LocalGlobalRegistration(3, 0.1, use_dustbin=True)
    with pytest.raises(NotImplementedError):
        GeometricStructureEmbedding(256, 0.2, 15, 3, reduction_a='mean')
