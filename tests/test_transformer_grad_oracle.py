"""Transformer gradients without a GPU: the restatement's fp32 autograd (oracle/transformer_grad_oracle.py) reproduces the reference's
(tests/golden/transformer_grads.npz), and the backward entry points reject bad arguments before any launch and size their workspaces on
the host."""
import ctypes
import os

import numpy as np
import pytest
import torch

from geotransformer_b200 import _lib as L
from geotransformer_b200 import functional as GF
from oracle import backbone_grad_oracle as BG
from oracle import geo_oracle as G
from oracle import transformer_grad_oracle as TG

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'transformer_grads.npz')


@pytest.mark.parametrize('workload,cfg_name', BG.WORKLOADS)
def test_restatement_autograd_reproduces_reference_fixture(workload, cfg_name, models):
    cfg, sd, model = models(cfg_name)
    fx = np.load(FIXTURE)
    data = BG.collate(workload, cfg)
    with torch.no_grad():
        feats_c = G.backbone(sd, cfg, data['features'], data)[-1]
    n0 = int(data['lengths'][-1][0])
    pts = data['points'][-1]
    keys = [k for k, _ in model.transformer.named_parameters()]
    got = TG.restatement_grads(sd, cfg, pts[:n0], pts[n0:], feats_c[:n0], feats_c[n0:], keys, torch.float32)
    gmax = max(float(g.abs().max()) for g in got.values())
    for k, g in got.items():
        e = TG.digest_err(g, fx[f'{workload}/{k}'], k, gmax)
        assert e <= 1e-4, (workload, k, e)


def _items(*shapes, embed=False):
    fake = 4096
    arr = (GF._AttItem * len(shapes))()
    grads = (GF._AttGradItem * len(shapes))()
    for i, (n, m) in enumerate(shapes):
        e = fake if embed else None
        arr[i] = GF._AttItem(fake, fake, fake, e, e, e, fake, n, m)
        grads[i] = GF._AttGradItem(fake, fake, fake, fake, fake, e, e, e)
    return arr, grads


def test_transformer_backward_entry_points_reject_bad_arguments_before_any_launch():
    lib = L.lib()
    fake = 4096                               # never dereferenced: every call below fails its host-side checks
    ws, big = fake, 1 << 40
    before = lib.geob200_launch_count()
    ok_items, ok_grads = _items((320, 320), embed=True)
    cross, cross_grads = _items((300, 280))
    cross_bad = (GF._AttGradItem * 1)(GF._AttGradItem(fake, fake, fake, fake, fake, fake, fake, fake))    # structure grads, no E
    calls = [
        # add_layernorm: empty, channels > 1024, no grad_x, small workspace
        lib.geob200_add_layernorm_backward(fake, None, fake, 0, 256, 1e-5, fake, fake, fake, fake, ws, big, None),
        lib.geob200_add_layernorm_backward(fake, None, fake, 100, 2048, 1e-5, fake, fake, fake, fake, ws, big, None),
        lib.geob200_add_layernorm_backward(fake, None, fake, 100, 256, 1e-5, fake, None, fake, fake, ws, big, None),
        lib.geob200_add_layernorm_backward(fake, fake, fake, 100, 256, 1e-5, fake, fake, fake, fake, ws, 64, None),
        # l2_normalize: empty, null output
        lib.geob200_l2_normalize_backward(fake, 0, 256, fake, fake, None),
        lib.geob200_l2_normalize_backward(fake, 100, 256, fake, None, None),
        # head_project: channels not a multiple of heads, ldq < channels, grad_q without wp, small workspace
        lib.geob200_head_project_backward(fake, 768, fake, fake, 100, 250, 4, fake, fake, fake, 250, fake, fake, ws, big, None),
        lib.geob200_head_project_backward(fake, 128, fake, fake, 100, 256, 4, fake, fake, fake, 256, fake, fake, ws, big, None),
        lib.geob200_head_project_backward(fake, 768, None, fake, 100, 256, 4, fake, fake, fake, 256, fake, fake, ws, big, None),
        lib.geob200_head_project_backward(fake, 768, fake, fake, 1000, 256, 4, fake, fake, fake, 256, fake, fake, ws, 16, None),
        # attention: channels, heads, strides, structure gradients of a cross item, small workspace, no items
        lib.geob200_attention_backward_batched(ok_items, ok_grads, 1, 768, 768, 768, 192, 768, 768, 768, 192, 4, ws, big, None),
        lib.geob200_attention_backward_batched(ok_items, ok_grads, 1, 768, 768, 768, 256, 768, 768, 768, 256, 3, ws, big, None),
        lib.geob200_attention_backward_batched(ok_items, ok_grads, 1, 128, 768, 768, 256, 768, 768, 768, 256, 4, ws, big, None),
        lib.geob200_attention_backward_batched(cross, cross_bad, 1, 256, 512, 512, 256, 256, 512, 512, 256, 4, ws, big, None),
        lib.geob200_attention_backward_batched(ok_items, ok_grads, 1, 768, 768, 768, 256, 768, 768, 768, 256, 4, ws, 1024, None),
        lib.geob200_attention_backward_batched(ok_items, ok_grads, 0, 768, 768, 768, 256, 768, 768, 768, 256, 4, ws, big, None),
        # structure embedding: channels, angle_k, table too small, inv_step not a power of two, small workspace
        lib.geob200_gse_embed_backward(fake, fake, 1000, 3, 192, fake, big, 256, 96.0, 12.25, fake, fake, fake, fake, fake, fake, fake,
                                       fake, ws, big, None),
        lib.geob200_gse_embed_backward(fake, fake, 1000, 4, 256, fake, big, 256, 96.0, 12.25, fake, fake, fake, fake, fake, fake, fake,
                                       fake, ws, big, None),
        lib.geob200_gse_embed_backward(fake, fake, 1000, 3, 256, fake, 1024, 256, 96.0, 12.25, fake, fake, fake, fake, fake, fake, fake,
                                       fake, ws, big, None),
        lib.geob200_gse_embed_backward(fake, fake, 1000, 3, 256, fake, big, 200, 96.0, 12.25, fake, fake, fake, fake, fake, fake, fake,
                                       fake, ws, big, None),
        lib.geob200_gse_embed_backward(fake, fake, 1000, 3, 256, fake, big, 256, 96.0, 12.25, fake, fake, fake, fake, fake, fake, fake,
                                       fake, ws, 4096, None),
        # ... a non-positive table range, more rows than the bias column sums take
        lib.geob200_gse_embed_backward(fake, fake, 1000, 3, 256, fake, big, 256, -1.0, 12.25, fake, fake, fake, fake, fake, fake, fake,
                                       fake, ws, big, None),
        lib.geob200_gse_embed_backward(fake, fake, 1000, 3, 256, fake, big, 256, 96.0, 0.0, fake, fake, fake, fake, fake, fake, fake,
                                       fake, ws, big, None),
        lib.geob200_gse_embed_backward(fake, fake, 256 * 65535 + 1, 3, 256, fake, big, 256, 96.0, 12.25, fake, fake, fake, fake, fake, fake,
                                       fake, fake, ws, big, None),
    ]
    assert all(rc != 0 for rc in calls), calls
    assert lib.geob200_launch_count() == before
    assert cross_grads is not None


def test_transformer_workspace_queries_work_without_gpu():
    lib = L.lib()
    assert lib.geob200_add_layernorm_backward_workspace_bytes(640, 256) >= 640 * 256 * 4      # dy * xhat for dgamma
    assert lib.geob200_head_project_backward_workspace_bytes(20000, 256, 4) >= 78 * 64 * 256 * 4  # 256-row chunk partials
    items, _ = _items((320, 320), (300, 300), embed=True)
    assert lib.geob200_attention_backward_batched_workspace_bytes(items, 2, 4) >= 320 * 320 * 4 * 4   # dS' of the largest item
    n = 320 * 320
    need = lib.geob200_gse_embed_backward_workspace_bytes(n, 256)
    assert need >= n * 256 + 50 * 2 * 256 * 256 * 4                  # k* bytes and the 2048-row chunk partials of dWd, dWa
    assert lib.geob200_gse_embed_backward_workspace_bytes(n, 128) < need
    assert ctypes.sizeof(GF._AttGradItem) == 8 * ctypes.sizeof(ctypes.c_void_p)
