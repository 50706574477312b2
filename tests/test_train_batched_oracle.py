"""Batched training without a GPU: the numpy restatement of the loss-weight kernel's contract (``geob200_batch_loss_weights``), the
argument checks of the new batched entry points (rejected before any launch), and the learning-rate scaling of a batched engine
against the reference's order (``register_optimizer`` scales, then the experiment builds its scheduler)."""
import ctypes

import numpy as np
import pytest
import torch

from geotransformer_b200 import _lib as L
from geotransformer_b200.config import make_cfg
from geotransformer_b200.model import create_model
from geotransformer_b200.train import make_optimizer, make_optimizer_and_scheduler, make_scheduler


def loss_weights_restated(rows):
    """(w (B,), mean (3,), n_valid, found) of geob200_batch_loss_weights for (B, >= 3) float32 rows: a pair is valid when its three
    losses are finite, w_p = valid_p / n_valid in fp32, the mean is the pair-order fp32 sum of the rounded products w_p * row_p over
    the valid pairs, NaN (and found = 1) when none is valid"""
    rows = np.asarray(rows, dtype=np.float32)[:, :3]
    valid = np.isfinite(rows).all(axis=1)
    n = int(valid.sum())
    inv = np.float32(1.0) / np.float32(n) if n else np.float32(0.0)
    w = np.where(valid, inv, np.float32(0.0)).astype(np.float32)
    mean = np.zeros(3, dtype=np.float32)
    for p in np.flatnonzero(valid):
        mean = (mean + (inv * rows[p]).astype(np.float32)).astype(np.float32)
    if n == 0:
        mean[:] = np.nan
    return w, mean, n, n == 0


def test_restatement_weights_and_mean():
    rows = np.array([[1.5, 0.5, 1.0], [np.nan, 0.2, np.nan], [2.5, 1.0, 1.5], [0.25, np.inf, 0.1]], dtype=np.float32)
    w, mean, n, found = loss_weights_restated(rows)
    assert n == 2 and not found
    assert w.tolist() == [0.5, 0.0, 0.5, 0.0]
    assert mean.tolist() == [2.0, 0.75, 1.25]                      # the mean of the two finite rows, exact here
    w3, mean3, n3, _ = loss_weights_restated(np.array([[1, 1, 1], [2, 2, 2], [4, 4, 4]], dtype=np.float32))
    assert n3 == 3 and np.all(w3 == np.float32(1) / np.float32(3))
    third = np.float32(1) / np.float32(3)
    want = np.float32(np.float32(np.float32(third * np.float32(1)) + np.float32(third * np.float32(2))) + np.float32(third * np.float32(4)))
    assert mean3[0] == want


def test_restatement_without_a_valid_pair():
    w, mean, n, found = loss_weights_restated(np.full((3, 3), np.nan, dtype=np.float32))
    assert n == 0 and found and np.all(w == 0) and np.all(np.isnan(mean))


def test_batched_entry_points_reject_bad_arguments_before_any_launch():
    lib = L.lib()
    launches = lib.geob200_launch_count()
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.addressof(buf)

    def err():
        return lib.geob200_last_error().decode()

    assert lib.geob200_batch_loss_weights(p, 3, 0, p, p, p, p, None) < 0 and 'pairs' in err()
    assert lib.geob200_batch_loss_weights(p, 3, 33, p, p, p, p, None) < 0 and 'pairs' in err()
    assert lib.geob200_batch_loss_weights(p, 2, 4, p, p, p, p, None) < 0 and 'ld_rows' in err()
    assert lib.geob200_batch_loss_weights(None, 3, 4, p, p, p, p, None) < 0 and 'null pointer' in err()
    assert lib.geob200_batch_loss_weights(p, 3, 4, p, None, p, p, None) < 0 and 'null pointer' in err()
    assert lib.geob200_batch_loss_weights(p, 3, 4, p, p, p, None, None) < 0 and 'null pointer' in err()

    rows = np.array([40, 30, 50, 20], dtype=np.int64)                 # 2 pairs, 140 query rows
    r = rows.ctypes.data
    assert lib.geob200_maxpool_batched(p, p, 141, 200, 8, 64, p, 2, r, p, None) < 0 and 'add up' in err()
    assert lib.geob200_maxpool_batched(p, p, 140, 200, 8, 64, p, 0, r, p, None) < 0 and 'pairs' in err()
    assert lib.geob200_maxpool_batched(p, p, 140, 200, 8, 64, None, 2, r, p, None) < 0 and 'null pointer' in err()
    assert lib.geob200_maxpool_batched(p, p, 140, 200, 0, 64, p, 2, r, p, None) < 0 and 'empty' in err()
    neg = np.array([-1, 30, 50, 61], dtype=np.int64)
    assert lib.geob200_maxpool_batched(p, p, 140, 200, 8, 64, p, 2, neg.ctypes.data, p, None) < 0 and 'negative' in err()

    def kpgn(n_query=140, n_pairs=2, cloud_rows=r, c_in=64, groups=32, out=p, gn_bytes=1 << 16):
        return lib.geob200_kpconv_group_norm_batched(p, p, p, p, n_query, 200, 8, p, 15, p, p, c_in, 64, 1.0, groups, p, p, 1e-5, 1, 0.1,
                                                     out, out, p, gn_bytes, p, 1 << 16, None, n_pairs, cloud_rows)
    assert kpgn(n_query=139) < 0 and 'add up' in err()
    assert kpgn(n_pairs=40) < 0 and 'pairs' in err()
    assert kpgn(cloud_rows=None) < 0
    assert kpgn(out=None) < 0 and 'null output' in err()
    assert kpgn(c_in=48) < 0 and 'unsupported shape' in err()
    assert kpgn(groups=7) < 0 and 'group count' in err()
    assert kpgn(gn_bytes=16) < 0 and 'workspace' in err()
    assert lib.geob200_launch_count() == launches


@pytest.mark.parametrize('name', ['3dmatch', 'kitti', 'modelnet'])
@pytest.mark.parametrize('batch_size', [1, 2, 4, 8])
def test_lr_scaled_before_the_scheduler_as_the_reference(name, batch_size):
    """the reference: optimizer built with cfg.optim.lr, register_optimizer multiplies every group's lr by the world size, then the
    scheduler is built on it (its base lrs are the scaled ones); the schedule's first steps follow"""
    cfg = make_cfg(name)
    model = create_model(cfg)
    opt, sched = make_optimizer_and_scheduler(model, cfg, batch_size)
    ref = torch.optim.Adam(model.parameters(), lr=cfg.optim.lr, weight_decay=cfg.optim.weight_decay)
    for g in ref.param_groups:
        g['lr'] = g['lr'] * batch_size
    ref_sched = make_scheduler(ref, cfg)
    assert sched.base_lrs == ref_sched.base_lrs == [cfg.optim.lr * batch_size]
    for _ in range(3):
        assert [g['lr'] for g in opt.param_groups] == [g['lr'] for g in ref.param_groups]
        opt.step()
        ref.step()
        sched.step()
        ref_sched.step()
    _, unscaled = make_optimizer_and_scheduler(model, cfg, batch_size, scale_lr=False)
    assert unscaled.base_lrs == [cfg.optim.lr]


@pytest.mark.parametrize('name', ['3dmatch', 'kitti', 'modelnet'])
def test_batch_size_one_builds_todays_optimizer_and_scheduler(name):
    cfg = make_cfg(name)
    model = create_model(cfg)
    opt, sched = make_optimizer_and_scheduler(model, cfg, 1)
    want = make_optimizer(model, cfg)
    want_sched = make_scheduler(want, cfg)
    assert opt.state_dict() == want.state_dict()
    assert sched.state_dict() == want_sched.state_dict()
