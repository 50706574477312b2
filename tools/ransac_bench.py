"""Time the batched correspondence RANSAC (csrc/ransac.cu) at the reference configs on the correspondences of real forwards.

    python tools/ransac_bench.py [--batch 8] [--reps 20] [--oracle-iterations 200]

For a batch of 3dmatch20k pairs (3DMatch config: tau 0.05 m, 3 points, 1 000 iterations) and a batch of kitti4k pairs (KITTI
config: tau 0.3 m, 4 points, 50 000 iterations) it runs one forward_batch, pads the LGR correspondences into the (B, capacity, 3)
layout with device counts, and reports: CUDA-event time of the RANSAC launches (median and min over --reps after warm-up), the
work counted from shapes (B * I * n residual evaluations, 26 fp32 operations each: 9 mul + 9 add for R x + t, 3 sub, 3 mul + 2 add
for the squared norm), the achieved rate against the FP32 data-sheet peak of the H100 SXM (67 TFLOP/s, which counts an FMA as
two operations; the pinned residual issues no FMA), and, as the CPU yardstick, the numpy restatement (oracle/ransac_oracle.py)
timed on the host for the first pair at --oracle-iterations.  Open3D is not installed, so no Open3D time is given.  The card
name and power limit are read in the same run and printed with the numbers; writes nothing.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from geotransformer_b200 import _lib                                    # noqa: E402
from geotransformer_b200 import functional as GF                        # noqa: E402
from geotransformer_b200.config import make_cfg                         # noqa: E402
from geotransformer_b200.model import create_model, enable_native       # noqa: E402
from geotransformer_b200.synth import make_pair                         # noqa: E402
from geotransformer_b200.utils.data import registration_collate_fn_stack_mode  # noqa: E402
from geotransformer_b200.weights import synthetic_state_dict            # noqa: E402
from oracle import ransac_oracle as RO                                  # noqa: E402
from tools.loss_bench import KEYS, LIMITS, card, timed                  # noqa: E402

OPS_PER_RESIDUAL = 26
FP32_PEAK = 67e12


def run(workload, cfg_name, batch, reps, oracle_iterations):
    cfg = make_cfg(cfg_name)
    rc = cfg.ransac
    model = create_model(cfg)
    model.load_state_dict(synthetic_state_dict(model, 7351), strict=True)
    model = enable_native(model.cuda().eval())
    pairs = [{k: make_pair(workload, i % 4)[k] for k in KEYS} for i in range(batch)]
    b = cfg.backbone
    data = registration_collate_fn_stack_mode(pairs, b.num_stages, b.init_voxel_size, b.init_radius, LIMITS[cfg_name])
    outs = model.forward_batch(data, side_streams=[torch.cuda.Stream() for _ in range(4)])
    torch.cuda.synchronize()
    ns = [int(o['ref_corr_points'].shape[0]) for o in outs]
    B, cap = len(outs), max(ns)
    src = torch.zeros((B, cap, 3), dtype=torch.float32, device='cuda')
    ref = torch.zeros((B, cap, 3), dtype=torch.float32, device='cuda')
    for p, o in enumerate(outs):
        src[p, :ns[p]], ref[p, :ns[p]] = o['src_corr_points'], o['ref_corr_points']
    cnt = torch.tensor(ns, dtype=torch.int32, device='cuda')

    def kernels():
        return GF.ransac_correspondences_batched(src, ref, rc.distance_threshold, rc.num_points, rc.num_iterations, seed=rc.seed,
                                                 num_corr=cnt)
    lib = _lib.lib()
    before = lib.geob200_launch_count()
    res = kernels()
    launches = lib.geob200_launch_count() - before
    torch.cuda.synchronize()
    med, mn = timed(kernels, reps)
    evals = rc.num_iterations * sum(ns)
    s0, r0 = outs[0]['src_corr_points'].cpu().numpy(), outs[0]['ref_corr_points'].cpu().numpy()
    t0 = time.perf_counter()
    RO.ransac(s0, r0, rc.distance_threshold, rc.num_points, oracle_iterations, seed=rc.seed)
    host_s = time.perf_counter() - t0
    return {'workload': workload, 'config': cfg_name, 'batch': B, 'num_iterations': rc.num_iterations, 'ransac_n': rc.num_points,
            'distance_threshold': rc.distance_threshold, 'correspondences_per_pair': ns, 'launches_per_batch': int(launches),
            'ransac_ms_median': round(med, 4), 'ransac_ms_min': round(mn, 4), 'residual_evaluations': evals,
            'fp32_ops': evals * OPS_PER_RESIDUAL, 'achieved_tops_median': round(evals * OPS_PER_RESIDUAL / (med * 1e-3) / 1e12, 3),
            'share_of_fp32_datasheet_peak': round(evals * OPS_PER_RESIDUAL / (med * 1e-3) / FP32_PEAK, 4),
            'fitness': [round(float(v), 4) for v in res['fitness'].cpu()],
            'oracle_host_s_pair0': round(host_s, 3), 'oracle_iterations_pair0': oracle_iterations,
            'open3d_time': 'not measured (Open3D is not installed)'}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--oracle-iterations', type=int, default=200)
    a = ap.parse_args()
    name, pl = card()
    print(json.dumps({'card': name, 'power_limit': pl}))
    for workload, cfg_name in (('3dmatch20k', '3dmatch'), ('kitti4k', 'kitti')):
        print(json.dumps(run(workload, cfg_name, a.batch, max(20, a.reps), a.oracle_iterations)))


if __name__ == '__main__':
    main()
