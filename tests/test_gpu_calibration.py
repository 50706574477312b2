"""Neighbour calibration of the augmented training set in chunks of pairs (``calibrate_neighbors_augmented``) against the existing
per-pair ``calibrate_neighbors_stack_mode`` run on the same augmented pairs, one at a time."""
import numpy as np
import pytest
import torch

from geotransformer_b200.augment import augment_stacked
from geotransformer_b200.config import make_cfg
from geotransformer_b200.synth import make_pair
from geotransformer_b200.utils.data import (CALIBRATION_ITERATION, calibrate_neighbors_augmented, calibrate_neighbors_stack_mode,
                                            registration_collate_fn_stack_mode)

pytestmark = pytest.mark.gpu


def _sequential(pairs, cfg, seed, sample_threshold):
    """the augmented pairs one at a time (streams (seed, CALIBRATION_ITERATION, p)), the reference loop's limits, and its stop"""
    dev = torch.device('cuda', torch.cuda.current_device())
    items = []
    for p, pair in enumerate(pairs):
        pts, lengths, T, _, _ = augment_stacked([pair], cfg, seed, CALIBRATION_ITERATION, dev, pair_base=p)
        pts = pts.cpu()
        items.append({'ref_points': pts[:lengths[0]], 'src_points': pts[lengths[0]:],
                      'ref_feats': torch.ones((lengths[0], 1)), 'src_feats': torch.ones((lengths[1], 1)), 'transform': T[0].cpu()})
    b = cfg.backbone
    limits = calibrate_neighbors_stack_mode(items, registration_collate_fn_stack_mode, b.num_stages, b.init_voxel_size, b.init_radius,
                                            sample_threshold=sample_threshold)
    hist_n = int(np.ceil(4 / 3 * np.pi * (b.init_radius / b.init_voxel_size + 1) ** 3))
    rows = np.zeros(b.num_stages, dtype=np.int64)
    used = len(items)
    for p, it in enumerate(items):
        data = registration_collate_fn_stack_mode([it], b.num_stages, b.init_voxel_size, b.init_radius, [hist_n] * b.num_stages)
        for s, nb in enumerate(data['neighbors']):
            counts = (nb < nb.shape[0]).sum(dim=1)
            rows[s] += int((counts < hist_n).sum())
        if rows.min() > sample_threshold:
            used = p + 1
            break
    return limits, used


@pytest.mark.parametrize('name,workload,n,chunk,threshold', [
    ('3dmatch', 'demo2k', 12, 5, 500),
    ('3dmatch', 'demo2k', 6, 4, 10 ** 6),   # never stops: every pair counts
    ('kitti', 'kitti4k', 10, 3, 400),
])
def test_batched_calibration_equals_per_pair(name, workload, n, chunk, threshold):
    cfg = make_cfg(name)
    pairs = [make_pair(workload, i) for i in range(n)]
    want, want_used = _sequential(pairs, cfg, 5, threshold)
    got, used = calibrate_neighbors_augmented(pairs, cfg, 5, sample_threshold=threshold, chunk=chunk)
    assert used == want_used, (used, want_used)
    assert np.array_equal(np.asarray(got), np.asarray(want)), (got, want)
