"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/losses.npz from the REAL reference's loss modules (imported through
oracle/ref_harness.py, CPU) and checks the restatement oracle/loss_oracle.py against them.
Run where the reference checkout exists:   python -m oracle.loss_vectors

Stored:
  scalars/<workload>:<pair>   (loss, c_loss, f_loss) of the reference's OverallLoss on the reference's own eval-mode forward of the
                              pair with the synthetic weights (demo2k, modelnet717, kitti4k pair 0 and make_golden.OTHER_PAIRS)
  coarse / fine case tables   kind, seed, shape of every seeded input (oracle/loss_oracle.py regenerates them) and the reference's
                              CoarseMatchingLoss / FineMatchingLoss value on it
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
from oracle import loss_oracle as LO, ref_harness                   # noqa: E402
from oracle.make_golden import GOLD, LIMITS, OTHER_PAIRS            # noqa: E402

PAIRS = (('demo2k', 0), ('modelnet717', 0), ('kitti4k', 0)) + OTHER_PAIRS


def _ref_loss_module(which):
    exp_dir = os.path.join(ref_harness.REF_ROOT, 'experiments', ref_harness.EXP[which])
    sys.modules.pop('loss', None)
    sys.path.insert(0, exp_dir)
    try:
        return importlib.import_module('loss')
    finally:
        sys.path.remove(exp_dir)


def _rel(a, b):
    a, b = float(a), float(b)
    if np.isnan(a) or np.isnan(b):
        return 0.0 if (np.isnan(a) and np.isnan(b)) else float('inf')
    return abs(a - b) / max(abs(b), 1e-30)


def scalars(workload, index):
    pair = make_pair(workload, index)
    cfg = make_cfg(pair['config'])
    limits = cfg.neighbor_limits or LIMITS[workload]
    sd = synthetic_state_dict(create_model(cfg), 7351)
    rcfg, rcreate = ref_harness.load_experiment(pair['config'])
    from geotransformer.utils.data import registration_collate_fn_stack_mode
    ref_model = rcreate(rcfg).eval()
    ref_model.load_state_dict(sd, strict=True)
    dd = {k: pair[k] for k in ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')}
    data = registration_collate_fn_stack_mode([dd], rcfg.backbone.num_stages, rcfg.backbone.init_voxel_size, rcfg.backbone.init_radius,
                                              limits)
    data = {k: ([x.clone() if isinstance(x, torch.Tensor) else x for x in v] if isinstance(v, list) else
                (v.clone() if isinstance(v, torch.Tensor) else v)) for k, v in data.items()}       # dense neighbour tables, as to_cuda
    loss = _ref_loss_module(pair['config'])
    with torch.no_grad():
        out = ref_model(data)
        ref = {k: float(v) for k, v in loss.OverallLoss(rcfg)(out, data).items()}
        mine = {k: float(v) for k, v in LO.overall_loss(cfg, out, data['transform']).items()}
    worst = max(_rel(mine[k], ref[k]) for k in ref)
    print(f'[{workload}:{index}] reference {ref}; restatement max rel diff {worst:.2e}')
    assert worst <= 1e-6, (ref, mine)
    return np.array([ref['loss'], ref['c_loss'], ref['f_loss']], dtype=np.float64)


def main():
    assert ref_harness.available(), 'needs the reference checkout'
    g = {'pairs': np.array([f'{w}:{i}' for w, i in PAIRS])}
    g['scalars'] = np.stack([scalars(w, i) for w, i in PAIRS])
    loss = _ref_loss_module('3dmatch')
    cvals, fvals = [], []
    for kind, seed, shape, ls in LO.COARSE_CASES:
        rf, sf, gi, go = LO.coarse_case(kind, seed, shape)
        p = LO.coarse_params(ls)
        m = loss.CoarseMatchingLoss(Cfg(coarse_loss=p))
        with torch.no_grad():
            v = float(m({'ref_feats_c': rf, 'src_feats_c': sf, 'gt_node_corr_indices': gi, 'gt_node_corr_overlaps': go}))
        assert _rel(float(LO.coarse_loss(p, rf, sf, gi, go)), v) <= 1e-6, (kind, seed)
        cvals.append(v)
    for kind, seed, shape in LO.FINE_CASES:
        rp, sp, rm, sm, sc, T = LO.fine_case(kind, seed, shape)
        m = loss.FineMatchingLoss(Cfg(fine_loss=Cfg(positive_radius=shape[2])))
        od = {'ref_node_corr_knn_points': rp, 'src_node_corr_knn_points': sp, 'ref_node_corr_knn_masks': rm,
              'src_node_corr_knn_masks': sm, 'matching_scores': sc}
        with torch.no_grad():
            v = float(m(od, {'transform': T}))
        assert _rel(float(LO.fine_loss(shape[2], rp, sp, rm, sm, sc, T)), v) <= 1e-6, (kind, seed)
        fvals.append(v)
    g['coarse_kind'] = np.array([c[0] for c in LO.COARSE_CASES])
    g['coarse_seed'] = np.array([c[1] for c in LO.COARSE_CASES])
    g['coarse_shape'] = np.array([c[2] for c in LO.COARSE_CASES])
    g['coarse_log_scale'] = np.array([c[3] for c in LO.COARSE_CASES], dtype=np.float64)
    g['coarse_value'] = np.array(cvals, dtype=np.float64)
    g['fine_kind'] = np.array([c[0] for c in LO.FINE_CASES])
    g['fine_seed'] = np.array([c[1] for c in LO.FINE_CASES])
    g['fine_shape'] = np.array([c[2] for c in LO.FINE_CASES], dtype=np.float64)
    g['fine_value'] = np.array(fvals, dtype=np.float64)
    print('coarse values', np.round(cvals, 5).tolist())
    print('fine values', np.round(fvals, 5).tolist())
    path = os.path.join(GOLD, 'losses.npz')
    np.savez_compressed(path, **g)
    print(f'wrote {path} ({os.path.getsize(path) / 1e3:.1f} kB)')


if __name__ == '__main__':
    main()
