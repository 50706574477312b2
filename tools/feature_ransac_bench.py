"""Time the descriptor nearest neighbour (csrc/feature_match.cu) and the feature-matching RANSAC (csrc/ransac.cu).

    python tools/feature_ransac_bench.py [--batch 8] [--reps 10]

1. Nearest neighbour at the fine level of a batch of 3dmatch20k pairs (one forward_batch; ref_feats_f / src_feats_f, both
   directions) and at 20 000 x 20 000 x 32 (seeded normal descriptors, both directions).  FLOP counted from shapes: 2 n_q n_s C per
   direction (one screening GEMM; the kernel runs it twice, the second pass collecting candidates), over the FP32 data-sheet peak
   of the H100 SXM (67 TFLOP/s).  Yardstick: torch.cdist + argmin on the same tensors, per pair and direction (measurement only).
2. RANSAC at the reference defaults (tau 0.05, 3 points, 50 000 iterations, 1 000 validations) on the same batch of fine-level
   pairs, one call for the batch.
CUDA-event times, median and min over --reps after warm-up; the card name and power limit are read in the same run and printed
with the numbers.  Writes nothing.
"""
import argparse
import json
import os
import sys

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
from tools.loss_bench import KEYS, LIMITS, card, timed                  # noqa: E402

FP32_PEAK = 67e12


def fine_batch(batch):
    cfg = make_cfg('3dmatch')
    model = create_model(cfg)
    model.load_state_dict(synthetic_state_dict(model, 7351), strict=True)
    model = enable_native(model.cuda().eval())
    pairs = [{k: make_pair('3dmatch20k', i % 4)[k] for k in KEYS} for i in range(batch)]
    b = cfg.backbone
    data = registration_collate_fn_stack_mode(pairs, b.num_stages, b.init_voxel_size, b.init_radius, LIMITS['3dmatch'])
    with torch.no_grad():
        outs = model.forward_batch(data, side_streams=[torch.cuda.Stream() for _ in range(4)])
    torch.cuda.synchronize()
    del model
    return outs


def pad(tensors):
    cap = max(int(t.shape[0]) for t in tensors)
    out = torch.zeros((len(tensors), cap, tensors[0].shape[1]), dtype=torch.float32, device='cuda')
    for p, t in enumerate(tensors):
        out[p, :t.shape[0]] = t
    return out, torch.tensor([int(t.shape[0]) for t in tensors], dtype=torch.int32, device='cuda')


def nn_case(label, q_list, s_list, reps):
    Q, nq = pad(q_list)
    S, ns = pad(s_list)
    C = int(Q.shape[2])
    flop = sum(2 * 2 * int(q.shape[0]) * int(s.shape[0]) * C for q, s in zip(q_list, s_list))        # both directions

    def kernels():
        return GF.feature_nearest_neighbor_batched(Q, S, nq, ns, bidirectional=True)

    def yardstick():
        for q, s in zip(q_list, s_list):
            d = torch.cdist(q, s)
            d.argmin(1)
            d.argmin(0)
    lib = _lib.lib()
    before = lib.geob200_launch_count()
    kernels()
    launches = lib.geob200_launch_count() - before
    med, mn = timed(kernels, reps)
    ymed, _ = timed(yardstick, reps)
    # the yardstick's answer vs the kernel's (cdist is not exact: rows it gets wrong are counted, not asserted)
    qi = kernels()[0]
    diff = sum(int((torch.cdist(q, s).argmin(1) != qi[p, :q.shape[0]]).sum()) for p, (q, s) in enumerate(zip(q_list, s_list)))
    return {'case': label, 'pairs': len(q_list), 'rows_query': [int(q.shape[0]) for q in q_list],
            'rows_support': [int(s.shape[0]) for s in s_list], 'channels': C, 'launches': int(launches),
            'nn_ms_median': round(med, 3), 'nn_ms_min': round(mn, 3), 'flop_both_directions': flop,
            'achieved_tflops': round(flop / (med * 1e-3) / 1e12, 2), 'share_of_fp32_datasheet_peak': round(flop / (med * 1e-3) / FP32_PEAK, 3),
            'torch_cdist_argmin_ms_median': round(ymed, 3), 'rows_where_cdist_argmin_differs': diff}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--reps', type=int, default=10)
    a = ap.parse_args()
    name, pl = card()
    print(json.dumps({'card': name, 'power_limit': pl}))
    outs = fine_batch(a.batch)
    rf = [o['ref_feats_f'].contiguous() for o in outs]
    sf = [o['src_feats_f'].contiguous() for o in outs]
    print(json.dumps(nn_case('3dmatch20k fine level (src -> ref and ref -> src)', sf, rf, a.reps)))
    g = torch.Generator(device='cuda').manual_seed(0)
    q = torch.randn((20000, 32), device='cuda', generator=g)
    s = torch.randn((20000, 32), device='cuda', generator=g)
    print(json.dumps(nn_case('20000 x 20000 x 32', [q], [s], a.reps)))
    sp, ns = pad([o['src_points_f'].contiguous() for o in outs])
    rp, nr = pad([o['ref_points_f'].contiguous() for o in outs])
    SF, _ = pad(sf)
    RF, _ = pad(rf)

    def ransac():
        return GF.ransac_features_batched(sp, rp, SF, RF, 0.05, 3, 50000, 1000, num_src=ns, num_ref=nr)
    lib = _lib.lib()
    before = lib.geob200_launch_count()
    res = ransac()
    launches = lib.geob200_launch_count() - before
    med, mn = timed(ransac, max(3, a.reps // 2), warmup=2)
    print(json.dumps({'case': 'feature RANSAC, 3dmatch20k fine level', 'pairs': len(outs), 'num_iterations': 50000, 'val_iterations': 1000,
                      'distance_threshold': 0.05, 'ransac_n': 3, 'launches': int(launches), 'ransac_ms_median': round(med, 3),
                      'ransac_ms_min': round(mn, 3), 'num_validated': res['num_validated'].tolist(),
                      'fitness': [round(float(v), 4) for v in res['fitness'].cpu()]}))


if __name__ == '__main__':
    main()
