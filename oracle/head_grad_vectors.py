"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/head_grads.npz from the REAL reference's modules (imported through
oracle/ref_harness.py, CPU, fp32 autograd) and checks the restatements of oracle/head_grad_oracle.py against them.
Run where the reference checkout exists:   python -m oracle.head_grad_vectors

Stored (every gradient as an oracle/head_grad_oracle.digest):
  coarse/<i>, fine/<i>        CoarseMatchingLoss / FineMatchingLoss gradients on loss_oracle.COARSE_CASES / FINE_CASES (and the
                              duplicated-feature coarse case, index len(COARSE_CASES))
  sinkhorn/<i>                LearnableLogOptimalTransport gradients (scores, alpha) of sum(out * g) on head_grad_oracle.SINKHORN_CASES
                              without their padding patches; sinkhorn_nan/<i> = the NaN count of the reference's fp32 dscores
  e2e/<workload>/<name>       OverallLoss(out, data)['loss'].backward() on the reference's eval-mode forward of pair 0 with the
                              synthetic weights: ref/src_feats_c, ref/src_feats_f, optimal_transport.alpha
"""
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from geotransformer_b200.config import Cfg, make_cfg                # noqa: E402
from geotransformer_b200.model import create_model                  # noqa: E402
from geotransformer_b200.synth import make_pair                     # noqa: E402
from geotransformer_b200.weights import synthetic_state_dict        # noqa: E402
from oracle import head_grad_oracle as HG, loss_oracle as LO, ref_harness   # noqa: E402
from oracle.make_golden import GOLD, LIMITS                         # noqa: E402

E2E = (('demo2k', '3dmatch'), ('modelnet717', 'modelnet'), ('kitti4k', 'kitti'))
E2E_NAMES = ('ref_feats_c', 'src_feats_c', 'ref_feats_f', 'src_feats_f', 'alpha')


def _ref_module(which, name):
    exp_dir = os.path.join(ref_harness.REF_ROOT, 'experiments', ref_harness.EXP[which])
    sys.modules.pop(name, None)
    sys.path.insert(0, exp_dir)
    try:
        return importlib.import_module(name)
    finally:
        sys.path.remove(exp_dir)


def _put(g, key, dig):
    for k, v in dig.items():
        g[f'{key}:{k}'] = v


def _grads(fn, inputs):
    leaves = [x.detach().clone().requires_grad_(True) for x in inputs]
    fn(*leaves).backward()
    return [x.grad for x in leaves]


def _check(key, got, ref, rtol):
    ok = HG.digest_close(HG.digest(got), HG.digest(ref), rtol)
    print(f'  {key}: restatement {"matches" if ok else "DIFFERS"} (rtol {rtol})')
    assert ok, key


def coarse_and_fine(g, loss):
    cases = [(LO.coarse_case(k, s, sh), LO.coarse_params(ls)) for k, s, sh, ls in LO.COARSE_CASES]
    cases.append((HG.duplicated_coarse_case(), LO.coarse_params(24)))
    for i, ((rf, sf, gi, go), p) in enumerate(cases):
        m = loss.CoarseMatchingLoss(Cfg(coarse_loss=p))
        ref = _grads(lambda a, b: m({'ref_feats_c': a, 'src_feats_c': b, 'gt_node_corr_indices': gi, 'gt_node_corr_overlaps': go}),
                     [rf, sf])
        mine = _grads(lambda a, b: HG.coarse_loss(p, a, b, gi, go), [rf, sf])
        for side, r, x in zip(('ref', 'src'), ref, mine):
            _check(f'coarse/{i}/{side}', x, r, 1e-5)
            _put(g, f'coarse/{i}/{side}', HG.digest(r))
    for i, (kind, seed, shape) in enumerate(LO.FINE_CASES):
        rp, sp, rm, sm, sc, T = LO.fine_case(kind, seed, shape)
        m = loss.FineMatchingLoss(Cfg(fine_loss=Cfg(positive_radius=shape[2])))
        od = {'ref_node_corr_knn_points': rp, 'src_node_corr_knn_points': sp, 'ref_node_corr_knn_masks': rm,
              'src_node_corr_knn_masks': sm}
        ref, = _grads(lambda s: m(dict(od, matching_scores=s), {'transform': T}), [sc])
        mine, = _grads(lambda s: HG.fine_loss(shape[2], rp, sp, rm, sm, s, T), [sc])
        _check(f'fine/{i}', mine, ref, 1e-6)
        _put(g, f'fine/{i}', HG.digest(ref))


def sinkhorn_cases(g):
    from geotransformer.modules.sinkhorn import LearnableLogOptimalTransport
    for i, (kind, seed, shape) in enumerate(HG.SINKHORN_CASES):
        scores, rm, cm, alpha, gr = HG.sinkhorn_case(kind, seed, shape)
        live = ~(~rm).all(1) | ~(~cm).all(1)
        ot = LearnableLogOptimalTransport(HG.ITERS)
        with torch.no_grad():
            ot.alpha.fill_(float(alpha))
        s = scores[live].clone().requires_grad_(True)
        (ot(s, rm[live], cm[live]) * gr[live]).sum().backward()
        ds, da = s.grad, ot.alpha.grad.reshape(1)
        nan = int(torch.isnan(ds).sum())
        print(f'  sinkhorn/{i} {kind} {shape}: reference fp32 dscores NaN entries {nan} of {ds.numel()}, dalpha {float(da):.6g}')
        if kind == 'upstream':
            assert nan > 0 and torch.isnan(da).all(), 'the reference fp32 autograd is expected to give NaN here'
        else:
            mine = _grads(lambda x, a: (HG.sinkhorn(a, x, rm[live], cm[live]) * gr[live]).sum(), [scores[live], alpha])
            _check(f'sinkhorn/{i}/scores', mine[0], ds, 1e-5)
        _put(g, f'sinkhorn/{i}/scores', HG.digest(ds))
        _put(g, f'sinkhorn/{i}/alpha', HG.digest(da))
        g[f'sinkhorn_nan/{i}'] = np.array(nan)


def e2e(g, workload, which):
    pair = make_pair(workload, 0)
    cfg = make_cfg(pair['config'])
    limits = cfg.neighbor_limits or LIMITS[workload]
    sd = synthetic_state_dict(create_model(cfg), 7351)
    rcfg, rcreate = ref_harness.load_experiment(which)
    from geotransformer.utils.data import registration_collate_fn_stack_mode
    model = rcreate(rcfg).eval()
    model.load_state_dict(sd, strict=True)
    dd = {k: pair[k] for k in ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')}
    data = registration_collate_fn_stack_mode([dd], rcfg.backbone.num_stages, rcfg.backbone.init_voxel_size, rcfg.backbone.init_radius,
                                              limits)
    data = {k: ([x.clone() if isinstance(x, torch.Tensor) else x for x in v] if isinstance(v, list) else
                (v.clone() if isinstance(v, torch.Tensor) else v)) for k, v in data.items()}
    out = model(data)
    for k in E2E_NAMES[:4]:
        out[k].retain_grad()
    loss = _ref_module(which, 'loss').OverallLoss(rcfg)(out, data)['loss']
    loss.backward()
    grads = [out[k].grad for k in E2E_NAMES[:4]] + [model.optimal_transport.alpha.grad.reshape(1)]
    for name, t in zip(E2E_NAMES, grads):
        print(f'  e2e/{workload}/{name}: {tuple(t.shape)}, max |g| {float(t.abs().max()):.4g}')
        _put(g, f'e2e/{workload}/{name}', HG.digest(t))
    g[f'e2e/{workload}/loss'] = np.array(float(loss.detach()))


def main():
    assert ref_harness.available(), 'needs the reference checkout'
    ref_harness.install()
    g = {}
    coarse_and_fine(g, _ref_module('3dmatch', 'loss'))
    sinkhorn_cases(g)
    for workload, which in E2E:
        e2e(g, workload, which)
    path = os.path.join(GOLD, 'head_grads.npz')
    np.savez_compressed(path, **g)
    print(f'wrote {path} ({os.path.getsize(path) / 1e3:.1f} kB)')


if __name__ == '__main__':
    main()
