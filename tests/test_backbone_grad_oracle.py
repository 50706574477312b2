"""Backbone gradients without a GPU: the restatement's fp32 autograd (oracle/backbone_grad_oracle.py) reproduces the reference's
(tests/golden/backbone_grads.npz), and the backward entry points reject bad arguments before any launch and size their workspaces
on the host."""
import ctypes
import os

import numpy as np
import pytest
import torch

from geotransformer_b200 import _lib as L
from oracle import backbone_grad_oracle as BG

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'backbone_grads.npz')


@pytest.fixture(scope='module')
def fixture():
    return np.load(FIXTURE)


@pytest.mark.parametrize('workload,cfg_name', BG.WORKLOADS)
def test_restatement_autograd_reproduces_reference_fixture(workload, cfg_name, models, fixture):
    cfg, sd, model = models(cfg_name)
    keys = [k for k, _ in model.backbone.named_parameters()]
    got = BG.restatement_grads(sd, cfg, BG.collate(workload, cfg), keys, torch.float32)
    # every digest part relative to its own largest value; the floor covers the gradients that are rounding noise around zero
    # (a bias feeding a GroupNorm with one channel per group)
    floor = 1e-6 * max(float(g.abs().max()) for g in got.values())
    for k in keys:
        e = BG.digest_err(got[k], fixture[f'{workload}/{k}'], floor)
        assert e <= 1e-4, (workload, k, e)


def _h(*v):
    return (ctypes.c_int64 * len(v))(*v)


def test_backward_entry_points_reject_bad_arguments_before_any_launch():
    lib = L.lib()
    fake = 4096                               # never dereferenced: every call below fails its host-side checks
    ws, big = fake, 1 << 40
    before = lib.geob200_launch_count()
    calls = [
        # kpconv: kernel size, c_in not 1 / multiple of 32, grad_feats without the weights, small workspace, empty input
        lib.geob200_kpconv_backward(fake, fake, fake, fake, 100, 80, 20, fake, 14, fake, 32, 32, 0.2, fake, fake, fake, fake, ws, big, None),
        lib.geob200_kpconv_backward(fake, fake, fake, fake, 100, 80, 20, fake, 15, fake, 48, 32, 0.2, fake, fake, fake, fake, ws, big, None),
        lib.geob200_kpconv_backward(fake, fake, fake, fake, 100, 80, 20, fake, 15, None, 32, 32, 0.2, fake, fake, fake, fake, ws, big, None),
        lib.geob200_kpconv_backward(fake, fake, fake, fake, 100, 80, 20, fake, 15, fake, 32, 32, 0.2, fake, fake, fake, fake, ws, 16, None),
        lib.geob200_kpconv_backward(fake, fake, fake, fake, 0, 80, 20, fake, 15, fake, 32, 32, 0.2, fake, fake, fake, fake, ws, big, None),
        # linear: empty problem, ldx < k, grad_x without weight_t, small workspace (with and without the ReLU's mask)
        lib.geob200_linear_backward(fake, 64, fake, None, 0, 32, 64, fake, fake, fake, fake, ws, big, None),
        lib.geob200_linear_backward(fake, 32, fake, None, 100, 32, 64, fake, fake, fake, fake, ws, big, None),
        lib.geob200_linear_backward(fake, 64, None, None, 100, 32, 64, fake, fake, fake, fake, ws, big, None),
        lib.geob200_linear_backward(fake, 64, fake, None, 100, 32, 64, fake, fake, fake, fake, ws, 8, None),
        lib.geob200_linear_backward(fake, 64, fake, fake, 100, 32, 64, fake, fake, fake, fake, ws,
                                    lib.geob200_linear_backward_workspace_bytes(100, 32, 64, 0), None),
        # group norm: channels not a multiple of groups, rows not adding up, too many pairs, negative slope, no y with leaky
        lib.geob200_group_norm_backward_batched(fake, fake, 100, 30, 8, fake, 1e-5, 1, 0.1, fake, fake, fake, fake, None, ws, big, None,
                                                1, _h(100, 0)),
        lib.geob200_group_norm_backward_batched(fake, fake, 100, 32, 8, fake, 1e-5, 1, 0.1, fake, fake, fake, fake, None, ws, big, None,
                                                1, _h(60, 30)),
        lib.geob200_group_norm_backward_batched(fake, fake, 100, 32, 8, fake, 1e-5, 1, 0.1, fake, fake, fake, fake, None, ws, big, None,
                                                33, _h(*([100] + [0] * 65))),
        lib.geob200_group_norm_backward_batched(fake, fake, 100, 32, 8, fake, 1e-5, 1, -0.1, fake, fake, fake, fake, None, ws, big, None,
                                                1, _h(100, 0)),
        lib.geob200_group_norm_backward_batched(fake, None, 100, 32, 8, fake, 1e-5, 1, 0.1, fake, fake, fake, fake, None, ws, big, None,
                                                1, _h(100, 0)),
        lib.geob200_group_norm_backward_batched(fake, fake, 100, 32, 8, fake, 1e-5, 1, 0.1, fake, fake, fake, fake, None, ws, 64, None,
                                                1, _h(100, 0)),
        # max-pool: segments, empty input, small workspace
        lib.geob200_maxpool_backward_batched(fake, fake, 100, 80, 20, 64, None, 1, _h(50, 40), fake, fake, ws, big, None),
        lib.geob200_maxpool_backward_batched(fake, fake, 100, 0, 20, 64, None, 1, _h(100, 0), fake, fake, ws, big, None),
        lib.geob200_maxpool_backward_batched(fake, fake, 100, 80, 20, 64, None, 1, _h(100, 0), fake, fake, ws, 32, None),
        # upsample: bad stride, grad_skip without skip columns, small workspace
        lib.geob200_upsample_concat_backward(fake, 0, 100, 40, 32, 16, fake, fake, fake, ws, big, None),
        lib.geob200_upsample_concat_backward(fake, 3, 100, 40, 32, 0, fake, fake, fake, ws, big, None),
        lib.geob200_upsample_concat_backward(fake, 3, 100, 40, 32, 16, fake, fake, fake, ws, 16, None),
    ]
    assert all(rc != 0 for rc in calls), calls
    assert lib.geob200_launch_count() == before


def test_workspace_queries_work_without_gpu():
    lib = L.lib()
    kp = lib.geob200_kpconv_backward_workspace_bytes(20000, 20000, 38, 64, 64)
    assert kp >= 20000 * 15 * 64 * 4                              # the recomputed gathered features
    assert lib.geob200_kpconv_backward_workspace_bytes(20000, 20000, 38, 1, 64) < kp
    assert lib.geob200_linear_backward_workspace_bytes(20000, 128, 64, 0) >= 79 * 128 * 64 * 4   # the 256-row chunk partials
    assert lib.geob200_linear_backward_workspace_bytes(200, 128, 64, 1) >= 200 * 128 * 4           # the ReLU-masked gradient
    assert lib.geob200_group_norm_backward_batched_workspace_bytes(20000, 128, 32, 2) >= 2 * (20000 // 128) * 128 * 16
    assert lib.geob200_maxpool_backward_batched_workspace_bytes(5000, 20000, 38, 128) >= 5000 * 128 * 4 + 2 * 5000 * 38 * 4
    assert lib.geob200_upsample_concat_backward_workspace_bytes(20000, 5000) >= 2 * 20000 * 4
