"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/backbone_grads.npz from the REAL reference's KPConvFPN (imported through
oracle/ref_harness.py, CPU, fp32 autograd) and checks the restatement's autograd (oracle/backbone_grad_oracle.py) against it.
Run where the reference checkout exists:   python -m oracle.backbone_grad_vectors

Stored (every gradient as an oracle/backbone_grad_oracle.packed_digest):
  <workload>/<param>            d/d param of sum_i <feats_list[i], G_i> (G_i = backbone_grad_oracle.upstream) for every backbone
                                parameter, on the reference's collate of pair 0 with the synthetic weights (seed 7351)
  overall/<workload>/feats_f    OverallLoss(out, data)['loss'].backward() on the reference's eval-mode forward: the gradient at
                                feats_list[0], what the matching heads hand to the backbone's fine output (the coarse output's
                                passes through the transformer first)
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from geotransformer_b200.config import make_cfg                     # noqa: E402
from geotransformer_b200.model import create_model                  # noqa: E402
from geotransformer_b200.synth import make_pair                     # noqa: E402
from geotransformer_b200.weights import synthetic_state_dict        # noqa: E402
from oracle import backbone_grad_oracle as BG, head_grad_oracle as HG, ref_harness   # noqa: E402
from oracle.head_grad_vectors import _ref_module                    # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')


def _put(g, key, t):
    g[key] = BG.packed_digest(t)


def _ref_data(pair, rcfg, limits):
    from geotransformer.utils.data import registration_collate_fn_stack_mode
    dd = {k: pair[k] for k in ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')}
    data = registration_collate_fn_stack_mode([dd], rcfg.backbone.num_stages, rcfg.backbone.init_voxel_size, rcfg.backbone.init_radius,
                                              limits)
    return {k: ([x.clone() if isinstance(x, torch.Tensor) else x for x in v] if isinstance(v, list) else
                (v.clone() if isinstance(v, torch.Tensor) else v)) for k, v in data.items()}


def backbone_case(g, workload, which):
    pair = make_pair(workload, 0)
    cfg = make_cfg(pair['config'])
    sd = synthetic_state_dict(create_model(cfg), BG.SEED)
    rcfg, rcreate = ref_harness.load_experiment(which)
    model = rcreate(rcfg).eval()
    model.load_state_dict(sd, strict=True)
    data = _ref_data(pair, rcfg, BG.limits(workload))
    feats_list = model.backbone(data['features'], data)
    ups = BG.upstream([tuple(f.shape) for f in feats_list])
    sum((f * u).sum() for f, u in zip(feats_list, ups)).backward()
    keys = [k for k, _ in model.backbone.named_parameters()]
    mine = BG.restatement_grads(sd, cfg, BG.collate(workload, cfg), keys, torch.float32)
    worst = 0.0
    for k, p in model.backbone.named_parameters():
        assert HG.digest_close(BG.digest(mine[k]), BG.digest(p.grad), 1e-4), (workload, k)
        worst = max(worst, float((mine[k] - p.grad).abs().max() / p.grad.abs().max().clamp_min(1e-30)))
        _put(g, f'{workload}/{k}', p.grad)
    print(f'  {workload}: {len(keys)} parameter gradients, restatement within {worst:.2e} of max |g|')
    # the whole OverallLoss: the gradients the heads hand to the backbone
    model.zero_grad()
    data = _ref_data(pair, rcfg, BG.limits(workload))
    kept = {}

    def keep(_m, _i, outs):
        outs[0].retain_grad()
        kept['f'] = outs[0]

    h = model.backbone.register_forward_hook(keep)
    out = model(data)
    h.remove()
    _ref_module(which, 'loss').OverallLoss(rcfg)(out, data)['loss'].backward()
    t = kept['f'].grad
    print(f'  overall/{workload}/feats_f: {tuple(t.shape)}, max |g| {float(t.abs().max()):.4g}')
    _put(g, f'overall/{workload}/feats_f', t)


def main():
    assert ref_harness.available(), 'needs the reference checkout'
    ref_harness.install()
    g = {}
    for workload, which in BG.WORKLOADS:
        backbone_case(g, workload, which)
    path = os.path.join(GOLD, 'backbone_grads.npz')
    np.savez_compressed(path, **g)
    print(f'wrote {path} ({os.path.getsize(path) / 1e3:.1f} kB)')


if __name__ == '__main__':
    main()
