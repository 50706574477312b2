"""Validation losses on the CPU side: the torch restatement (oracle/loss_oracle.py) against what the real reference's
OverallLoss / CoarseMatchingLoss / FineMatchingLoss produced (tests/golden/losses.npz), and the error behaviour of the loss
modules and entry points (no GPU needed)."""
import ctypes
import os

import numpy as np
import pytest
import torch

from geotransformer_b200 import _lib as L
from geotransformer_b200.config import make_cfg
from geotransformer_b200.synth import make_pair
from oracle import geo_oracle as G
from oracle import loss_oracle as LO

NAMES = ('loss', 'c_loss', 'f_loss')


@pytest.fixture(scope='module')
def losses():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'losses.npz'))


def _rel(a, b):
    a, b = float(a), float(b)
    if np.isnan(a) or np.isnan(b):
        return 0.0 if (np.isnan(a) and np.isnan(b)) else float('inf')
    return abs(a - b) / max(abs(b), 1e-30)


@pytest.mark.parametrize('workload,cfg_name', [('demo2k', '3dmatch'), ('modelnet717', 'modelnet')])
def test_restatement_matches_reference_scalars(workload, cfg_name, golden, losses, models):
    """restated forward (teacher-forced neighbour tables) + restated losses vs the reference's OverallLoss on its own forward"""
    cfg, sd, _ = models(cfg_name)
    gold = golden(workload)
    data = G.collate_pair(make_pair(workload, 0), cfg, gold['neighbor_limits'].tolist())
    for key in ('neighbors', 'subsampling', 'upsampling'):
        for i in range(len(data[key])):
            data[key][i] = torch.from_numpy(gold[f'{key}_{i}'].astype(np.int64))      # the reference's exact-tie order
    with torch.no_grad():
        out = G.forward(sd, cfg, data)
        got = LO.overall_loss(cfg, out, data['transform'])
    want = losses['scalars'][list(losses['pairs']).index(f'{workload}:0')]
    errs = [_rel(got[k], want[i]) for i, k in enumerate(NAMES)]
    print(f'{workload}: max rel deviation from the reference {max(errs):.2e}')
    assert max(errs) <= 1e-6, errs


def test_restatement_matches_reference_loss_vectors(losses):
    for kind, seed, shape, ls, want in zip(losses['coarse_kind'], losses['coarse_seed'], losses['coarse_shape'], losses['coarse_log_scale'],
                                           losses['coarse_value']):
        rf, sf, gi, go = LO.coarse_case(str(kind), int(seed), tuple(int(v) for v in shape))
        got = LO.coarse_loss(LO.coarse_params(float(ls)), rf, sf, gi, go)
        assert _rel(got, want) <= 1e-6, ('coarse', str(kind), int(seed), float(got), float(want))
    for kind, seed, shape, want in zip(losses['fine_kind'], losses['fine_seed'], losses['fine_shape'], losses['fine_value']):
        shape = (int(shape[0]), int(shape[1]), float(shape[2]))
        got = LO.fine_loss(shape[2], *LO.fine_case(str(kind), int(seed), shape))
        assert _rel(got, want) <= 1e-6, ('fine', str(kind), int(seed), float(got), float(want))
    assert np.isnan(losses['coarse_value']).any() and np.isnan(losses['fine_value']).any()
    assert len(losses['coarse_value']) + len(losses['fine_value']) >= 30


def test_loss_config_fields():
    for name, ls, r in (('3dmatch', 24, 0.05), ('kitti', 40, 0.6), ('modelnet', 24, 0.05)):
        c = make_cfg(name)
        assert c.coarse_loss.log_scale == ls and c.fine_loss.positive_radius == r
        assert (c.coarse_loss.positive_margin, c.coarse_loss.negative_margin, c.coarse_loss.positive_optimal,
                c.coarse_loss.negative_optimal, c.coarse_loss.positive_overlap) == (0.1, 1.4, 0.1, 1.4, 0.1)
        assert (c.loss.weight_coarse_loss, c.loss.weight_fine_loss) == (1.0, 1.0)


def test_loss_modules_raise_on_cpu_tensors():
    from geotransformer_b200.loss import CoarseMatchingLoss, FineMatchingLoss, OverallLoss
    cfg = make_cfg('3dmatch')
    rf, sf, gi, go = LO.coarse_case('mixed', 100, (8, 6, 128))
    rp, sp, rm, sm, sc, T = LO.fine_case('random', 200, (2, 64, 0.05))
    out = {'ref_feats_c': rf, 'src_feats_c': sf, 'gt_node_corr_indices': gi, 'gt_node_corr_overlaps': go, 'ref_node_corr_knn_points': rp,
           'src_node_corr_knn_points': sp, 'ref_node_corr_knn_masks': rm, 'src_node_corr_knn_masks': sm, 'matching_scores': sc}
    with pytest.raises(RuntimeError, match='CUDA'):
        CoarseMatchingLoss(cfg)(out)
    with pytest.raises(RuntimeError, match='CUDA'):
        FineMatchingLoss(cfg)(out, {'transform': T})
    with pytest.raises(RuntimeError, match='CUDA'):
        OverallLoss(cfg)(out, {'transform': T})


def test_loss_entry_points_reject_bad_arguments_before_any_launch():
    lib = L.lib()
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.addressof(buf)
    nodes = (ctypes.c_int64 * 2)(5, 4)
    neg = (ctypes.c_int64 * 2)(5, -1)

    def err():
        return lib.geob200_last_error().decode()

    def coarse(cloud, log_scale=24.0, n_pairs=1):
        return lib.geob200_coarse_matching_loss_batched(p, p, 128, n_pairs, cloud, p, p, p, 0.1, 1.4, 0.1, 1.4, log_scale, 0.1, p, 3, p,
                                                        1 << 16, None)

    def fine(k=64, radius=0.05, patches=4):
        return lib.geob200_fine_matching_loss_batched(p, p, p, p, p, p, 1, patches, k, None, radius, None, p, 3, p, 1 << 16, None)

    assert coarse(nodes, log_scale=0.0) < 0 and 'log_scale' in err()
    assert coarse(nodes, log_scale=-24.0) < 0 and 'log_scale' in err()
    assert coarse(neg) < 0 and 'negative' in err()
    assert coarse(nodes, n_pairs=0) < 0 and 'pairs' in err()
    assert fine(k=96) < 0 and 'k must be 64 or 128' in err()
    assert fine(radius=0.0) < 0 and 'positive_radius' in err()
    assert fine(patches=-1) < 0 and 'negative' in err()
    assert lib.geob200_coarse_matching_loss_batched_workspace_bytes(100, 10000) >= 2 * 4 * 10000
    assert lib.geob200_launch_count() == 0
