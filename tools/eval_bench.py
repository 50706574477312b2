"""Times the device stages of the benchmark evaluation (geotransformer_b200.evaluate) on a synthetic benchmark at real size.

    python tools/eval_bench.py [--chunk 64] [--out DIR]

Workloads: 1 700 pairs of ~5 000 correspondences (a 3DMatch / 3DLoMatch run, ~300 superpoints per cloud) and 550 pairs (the KITTI
test split, ~1 078 superpoints per cloud), resident on the device in chunks of --chunk pairs.  Per stage: CUDA-event time summed over
the chunks (median of 3 passes after a warm-up pass); the sweep is the five-setting --num_corr 250,500,1000,2500,5000 (one order,
five selections, metrics per setting).  RANSAC runs at the config iterations.  Prints one JSON line with the card's name and power
limit; the host side (npz loading, meters) is not timed.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from geotransformer_b200 import functional as GF  # noqa: E402
from geotransformer_b200.config import make_cfg    # noqa: E402

SWEEP = (250, 500, 1000, 2500, 5000)


def _chunk(g, B, n, nodes, scale):
    cnt = torch.randint(int(0.8 * n), int(1.2 * n), (B,), generator=g, dtype=torch.int32).cuda()
    cap = int(1.2 * n)
    src = (torch.rand((B, cap, 3), generator=g) * scale).cuda()
    ref = src + torch.randn((B, cap, 3), generator=g).cuda() * 0.02 * scale
    sc = torch.rand((B, cap), generator=g).cuda()
    P = 256
    idx = torch.randint(0, nodes, (B, P), generator=g).cuda()
    gt = torch.randint(0, nodes, (B, 4 * nodes, 2), generator=g).cuda()
    T = torch.eye(4).repeat(B, 1, 1).cuda()
    cov = torch.eye(6).repeat(B, 1, 1).cuda()
    return dict(ref=ref, src=src, sc=sc, cnt=cnt, idx=idx, gt=gt, T=T, cov=cov, nodes=nodes)


def _stages(d, cfg, method, ks, first_pair):
    """list of (stage, callable) for one chunk"""
    B = d['ref'].shape[0]
    st = [('sparse_eval', lambda: GF.sparse_correspondence_eval_batched(d['idx'], d['idx'], d['gt'], d['nodes'], d['nodes']))]
    state = {}
    if ks:
        st.append(('order', lambda: state.__setitem__('order', GF.corr_order_batched(d['sc'], max(ks), num_corr=d['cnt']))))
    for k in ks or [None]:
        def sel(k=k):
            state[k] = (d['ref'], d['src'], d['sc'], d['cnt']) if k is None else GF.corr_select_batched(d['ref'], d['src'], d['sc'], state['order'], k,
                                                                                                       num_corr=d['cnt'])
        st.append(('select', sel))
        st.append(('corr_metrics', lambda k=k: GF.correspondence_metrics_batched(state[k][0], state[k][1], d['T'], cfg.eval.acceptance_radius,
                                                                                 num_corr=state[k][3])))
        if method == 'ransac':
            st.append(('ransac', lambda k=k: GF.ransac_correspondences_batched(state[k][1], state[k][0], cfg.ransac.distance_threshold,
                                                                               cfg.ransac.num_points, cfg.ransac.num_iterations,
                                                                               num_corr=state[k][3], first_pair=first_pair)))
        elif method == 'svd':
            st.append(('svd', lambda k=k: GF.weighted_procrustes_counts(state[k][1], state[k][0], state[k][2], state[k][3])))
        st.append(('registration_error', lambda: GF.registration_error_batched(d['T'], d['T'], covariances=d['cov'], rmse_threshold=0.2)))
    return st


def run(config, pairs, n, nodes, scale, method, ks, chunk, g):
    cfg = make_cfg(config)
    chunks = [_chunk(g, min(chunk, pairs - b), n, nodes, scale) for b in range(0, pairs, chunk)]
    passes = []
    for rep in range(4):
        times = {}
        ev = []
        for ci, d in enumerate(chunks):
            for name, fn in _stages(d, cfg, method, ks, ci * chunk):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                fn()
                e.record()
                ev.append((name, s, e))
        torch.cuda.synchronize()
        for name, s, e in ev:
            times[name] = times.get(name, 0.0) + s.elapsed_time(e)
        if rep:
            passes.append(times)
    med = {k: float(np.median([p[k] for p in passes])) for k in passes[0]}
    total = sum(med.values())
    return {'config': config, 'pairs': pairs, 'corr_per_pair': n, 'method': method, 'num_corr': list(ks) or None,
            'stage_ms': {k: round(v, 3) for k, v in med.items()}, 'total_ms': round(total, 3), 'pairs_per_s': round(pairs / total * 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--chunk', type=int, default=64)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'eval_bench needs a GPU'
    g = torch.Generator().manual_seed(0)
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    res = {'gpu': smi.split('\n')[0], 'chunk': a.chunk, 'runs': []}
    for config, pairs, nodes, scale in (('3dmatch', 1700, 300, 3.0), ('kitti', 550, 1078, 60.0)):
        for method, ks in (('lgr', ()), ('svd', ()), ('ransac', ()), ('lgr', SWEEP), ('ransac', (5000,))):
            res['runs'].append(run(config, pairs, 5000, nodes, scale, method, ks, a.chunk, g))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'eval_bench.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
