"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/transformer_grads.npz from the REAL reference's GeometricTransformer (imported
through oracle/ref_harness.py, CPU, fp32 autograd) and checks the restatement's autograd (oracle/geo_oracle.geometric_transformer)
against it.  Run where the reference checkout exists:   python -m oracle.transformer_grad_vectors

Stored (every gradient as an oracle/transformer_grad_oracle.packed_digest):
  <workload>/<param>              d/d param of <ref_out, G_0> + <src_out, G_1> (G_i = backbone_grad_oracle.upstream) for every
                                  transformer parameter, on the reference's coarse points and backbone features of pair 0 with the
                                  synthetic weights (seed 7351)
  <workload>/ref_feats, src_feats the same gradient at the transformer's two input feature tensors
  overall/<workload>/<param>      OverallLoss(out, data)['loss'].backward() on the reference's eval-mode forward, every model parameter
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
from oracle import backbone_grad_oracle as BG, ref_harness        # noqa: E402
from oracle import transformer_grad_oracle as TG                    # noqa: E402
from oracle.backbone_grad_vectors import _ref_data                  # noqa: E402
from oracle.head_grad_vectors import _ref_module                    # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')


def transformer_case(g, workload, which):
    pair = make_pair(workload, 0)
    cfg = make_cfg(pair['config'])
    sd = synthetic_state_dict(create_model(cfg), BG.SEED)
    rcfg, rcreate = ref_harness.load_experiment(which)
    model = rcreate(rcfg).eval()
    model.load_state_dict(sd, strict=True)
    data = _ref_data(pair, rcfg, BG.limits(workload))
    with torch.no_grad():
        feats_c = model.backbone(data['features'], data)[-1]
    n0 = int(data['lengths'][-1][0])
    pts = data['points'][-1]
    rf, sf = feats_c[:n0].clone().requires_grad_(True), feats_c[n0:].clone().requires_grad_(True)
    o0, o1 = model.transformer(pts[:n0].unsqueeze(0), pts[n0:].unsqueeze(0), rf.unsqueeze(0), sf.unsqueeze(0))
    ups = BG.upstream([tuple(o0.shape[1:]), tuple(o1.shape[1:])])
    ((o0[0] * ups[0]).sum() + (o1[0] * ups[1]).sum()).backward()
    keys = [k for k, _ in model.transformer.named_parameters()]
    mine = TG.restatement_grads(sd, cfg, pts[:n0], pts[n0:], feats_c[:n0], feats_c[n0:], keys, torch.float32)
    ref = dict({k: p.grad for k, p in model.transformer.named_parameters()}, ref_feats=rf.grad, src_feats=sf.grad)
    # every digest part relative to its own largest value (transformer_grad_oracle.digest_err)
    gmax = max(float(t.abs().max()) for t in ref.values())
    worst = 0.0
    for k, t in ref.items():
        g[f'{workload}/{k}'] = TG.packed_digest(t)
        e = TG.digest_err(mine[k], g[f'{workload}/{k}'], k, gmax)
        assert e <= 1e-4, (workload, k, e)
        worst = max(worst, e)
    print(f'  {workload}: {len(ref)} transformer gradients, restatement within {worst:.2e} per digest part')
    # the whole OverallLoss at every model parameter
    model.zero_grad()
    data = _ref_data(pair, rcfg, BG.limits(workload))
    out = model(data)
    _ref_module(which, 'loss').OverallLoss(rcfg)(out, data)['loss'].backward()
    n = 0
    for k, p in model.named_parameters():
        if p.grad is not None:
            g[f'overall/{workload}/{k}'] = TG.packed_digest(p.grad)
            n += 1
    print(f'  overall/{workload}: {n} parameter gradients')


def main():
    assert ref_harness.available(), 'needs the reference checkout'
    ref_harness.install()
    g = {}
    for workload, which in BG.WORKLOADS:
        transformer_case(g, workload, which)
    path = os.path.join(GOLD, 'transformer_grads.npz')
    np.savez_compressed(path, **g)
    print(f'wrote {path} ({os.path.getsize(path) / 1e3:.1f} kB)')


if __name__ == '__main__':
    main()
