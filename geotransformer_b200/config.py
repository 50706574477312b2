"""Hot-path hyper-parameters of the three shipped GeoTransformer experiments.

Only the fields that fix shapes/arithmetic on the registration forward are kept (SURVEY.md section 8 table);
values restate reference ``experiments/*/config.py``:
  3DMatch  ``geotransformer.3dmatch.stage4.gse.k3.max.oacl.stage2.sinkhorn/config.py:76-125``
  KITTI    ``geotransformer.kitti.stage5.gse.k3.max.oacl.stage2.sinkhorn/config.py:76-125``
  ModelNet ``geotransformer.modelnet.rpmnet.stage4.gse.k3.max.oacl.stage2.sinkhorn/config.py:81-130``
"""


class Cfg(dict):
    """Attribute dict (the reference uses easydict.EasyDict; same access pattern)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v


def _base(seed=7351):
    c = Cfg()
    c.seed = seed
    c.backbone = Cfg(kernel_size=15, base_sigma=2.0, group_norm=32, input_dim=1, init_dim=64, output_dim=256)
    c.model = Cfg(num_sinkhorn_iterations=100)
    c.coarse_matching = Cfg(num_targets=128, overlap_threshold=0.1, dual_normalization=True)
    c.geotransformer = Cfg(output_dim=256, num_heads=4, blocks=['self', 'cross', 'self', 'cross', 'self', 'cross'],
                           sigma_a=15, angle_k=3, reduction_a='max')
    c.fine_matching = Cfg(mutual=True, confidence_threshold=0.05, use_dustbin=False, use_global_score=False,
                          correspondence_threshold=3, correspondence_limit=None, num_refinement_steps=5)
    c.eval = Cfg(acceptance_overlap=0.0, inlier_ratio_threshold=0.05)
    # validation losses (OverallLoss, experiments/*/config.py:127-143; ModelNet 132-148)
    c.coarse_loss = Cfg(positive_margin=0.1, negative_margin=1.4, positive_optimal=0.1, negative_optimal=1.4, log_scale=24,
                        positive_overlap=0.1)
    c.fine_loss = Cfg(positive_radius=0.05)
    c.loss = Cfg(weight_coarse_loss=1.0, weight_fine_loss=1.0)
    # correspondence RANSAC of eval.py --method ransac (experiments/*/config.py, _C.ransac); seed keys the sampler
    c.ransac = Cfg(distance_threshold=0.05, num_points=3, num_iterations=1000, seed=0)
    return c


def make_cfg(name='3dmatch'):
    c = _base()
    c.name = name
    if name == '3dmatch':
        c.backbone.update(num_stages=4, init_voxel_size=0.025, base_radius=2.5)
        c.model.update(ground_truth_matching_radius=0.05, num_points_in_patch=64, fine_level=1)
        c.coarse_matching.num_correspondences = 256
        c.geotransformer.update(input_dim=1024, hidden_dim=256, sigma_d=0.2)
        c.fine_matching.update(topk=3, acceptance_radius=0.1)
        c.eval.update(acceptance_radius=0.1, rmse_threshold=0.2, rre_threshold=15.0, rte_threshold=0.3)
        c.neighbor_limits = [38, 36, 36, 38]  # reference demo.py:52
    elif name == 'kitti':
        c.backbone.update(num_stages=5, init_voxel_size=0.3, base_radius=4.25)
        c.model.update(ground_truth_matching_radius=0.6, num_points_in_patch=128, fine_level=1)
        c.coarse_matching.num_correspondences = 256
        c.geotransformer.update(input_dim=2048, hidden_dim=128, sigma_d=4.8)
        c.fine_matching.update(topk=2, acceptance_radius=0.6)
        c.eval.update(acceptance_radius=1.0, rre_threshold=5.0, rte_threshold=2.0)
        c.coarse_loss.log_scale = 40
        c.fine_loss.positive_radius = 0.6
        c.ransac.update(distance_threshold=0.3, num_points=4, num_iterations=50000)
        c.neighbor_limits = None  # calibrated (reference utils/data.py:192-217)
    elif name == 'modelnet':
        c.backbone.update(num_stages=3, init_voxel_size=0.05, base_radius=2.5)
        c.model.update(ground_truth_matching_radius=0.05, num_points_in_patch=128, fine_level=0)
        c.coarse_matching.num_correspondences = 128
        c.geotransformer.update(input_dim=512, hidden_dim=256, sigma_d=0.2)
        c.fine_matching.update(topk=3, acceptance_radius=0.1)
        c.eval.update(acceptance_radius=0.1, rre_threshold=1.0, rte_threshold=0.1)
        c.neighbor_limits = None
    else:
        raise ValueError(f'unknown config {name}')
    c.backbone.init_radius = c.backbone.base_radius * c.backbone.init_voxel_size
    c.backbone.init_sigma = c.backbone.base_sigma * c.backbone.init_voxel_size
    return c
