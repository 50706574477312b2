"""Time the validation-loss launches of a batched forward (OverallLoss.write_batched: coarse circle loss + fine matching loss)
against the same losses computed as eager torch ops on the device.

    python tools/loss_bench.py [--batch 8] [--reps 50]

For a batch of 3dmatch20k pairs and a batch at the KITTI shape (kitti4k pairs) it runs one forward_batch to get real inputs,
then reports per batch: CUDA-event time of the loss launches (after warm-up, median over --reps), the launches they add
(geob200_launch_count), and the eager-torch time of the restatement run on the same device tensors.  The card name and
power limit are read in the same run and printed with the numbers; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from geotransformer_b200 import _lib                                    # noqa: E402
from geotransformer_b200.config import make_cfg                         # noqa: E402
from geotransformer_b200.loss import OverallLoss                        # noqa: E402
from geotransformer_b200.model import create_model, enable_native       # noqa: E402
from geotransformer_b200.synth import make_pair                         # noqa: E402
from geotransformer_b200.utils.data import registration_collate_fn_stack_mode  # noqa: E402
from geotransformer_b200.weights import synthetic_state_dict            # noqa: E402
from oracle import loss_oracle as LO                                    # noqa: E402

KEYS = ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')
LIMITS = {'3dmatch': [38, 36, 36, 38], 'kitti': [27, 75, 147, 157, 119]}


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:          # noqa: BLE001
        pl = f'unavailable ({e})'
    return name, pl


def timed(fn, reps, warmup=5):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts))


def run(workload, cfg_name, batch, reps):
    cfg = make_cfg(cfg_name)
    model = create_model(cfg)
    model.load_state_dict(synthetic_state_dict(model, 7351), strict=True)
    model = enable_native(model.cuda().eval())
    pairs = [{k: make_pair(workload, i % 4)[k] for k in KEYS} for i in range(batch)]
    b = cfg.backbone
    data = registration_collate_fn_stack_mode(pairs, b.num_stages, b.init_voxel_size, b.init_radius, LIMITS[cfg_name])
    outs = model.forward_batch(data, side_streams=[torch.cuda.Stream() for _ in range(4)])
    torch.cuda.synchronize()
    # the batched inputs forward_batch hands to the loss (full-capacity buffers + device counts)
    loss = OverallLoss(cfg)
    B = len(outs)
    cn = [o['ref_feats_c'].shape[0] for o in outs] + [o['src_feats_c'].shape[0] for o in outs]
    feats = torch.cat([o['ref_feats_c'] for o in outs] + [o['src_feats_c'] for o in outs])
    nn = [cn[p] * cn[B + p] for p in range(B)]
    gi = torch.zeros((sum(nn), 2), dtype=torch.int64, device='cuda')
    go = torch.zeros((sum(nn),), dtype=torch.float32, device='cuda')
    cnt = torch.zeros((B,), dtype=torch.int32, device='cuda')
    g0 = 0
    for p, o in enumerate(outs):
        n = o['gt_node_corr_indices'].shape[0]
        gi[g0:g0 + n], go[g0:g0 + n], cnt[p] = o['gt_node_corr_indices'], o['gt_node_corr_overlaps'], n
        g0 += nn[p]
    P = max(o['matching_scores'].shape[0] for o in outs)
    K = outs[0]['ref_node_corr_knn_masks'].shape[1]

    def pad(t, fill=0):
        x = torch.full((P,) + tuple(t.shape[1:]), fill, dtype=t.dtype, device='cuda')
        x[:t.shape[0]] = t
        return x
    rp = torch.cat([pad(o['ref_node_corr_knn_points']) for o in outs])
    sp = torch.cat([pad(o['src_node_corr_knn_points']) for o in outs])
    rm = torch.cat([pad(o['ref_node_corr_knn_masks'], False) for o in outs])
    sm = torch.cat([pad(o['src_node_corr_knn_masks'], False) for o in outs])
    sc = torch.cat([pad(o['matching_scores']) for o in outs])
    pc = torch.tensor([o['matching_scores'].shape[0] for o in outs], dtype=torch.int32, device='cuda')
    T = torch.stack(list(data["transform"])).reshape(B, 4, 4).contiguous()
    rows = torch.empty((B, 3), device='cuda')

    def kernels():
        loss.write_batched(feats, cn, (gi, go, cnt), rp, sp, rm, sm, sc, T, pc, rows)

    def eager():
        return [LO.overall_loss(cfg, o, data['transform'][p]) for p, o in enumerate(outs)]
    lib = _lib.lib()
    before = lib.geob200_launch_count()
    kernels()
    launches = lib.geob200_launch_count() - before
    torch.cuda.synchronize()
    k_med, k_min = timed(kernels, reps)
    e_med, e_min = timed(eager, reps)
    want = eager()
    dev = max(abs(float(rows[p, i]) - float(w[k])) / max(abs(float(w[k])), 1e-30)
              for p, w in enumerate(want) for i, k in enumerate(('loss', 'c_loss', 'f_loss')) if not np.isnan(float(w[k])))
    return {'workload': workload, 'batch': B, 'superpoints_per_cloud_mean': float(np.mean(cn)), 'patches_per_pair': P, 'k': K,
            'loss_kernels_ms_median': round(k_med, 4), 'loss_kernels_ms_min': round(k_min, 4), 'launches_per_batch': int(launches),
            'eager_torch_ms_median': round(e_med, 4), 'eager_torch_ms_min': round(e_min, 4), 'max_rel_diff_vs_eager': dev}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--reps', type=int, default=50)
    a = ap.parse_args()
    name, pl = card()
    print(json.dumps({'card': name, 'power_limit': pl}))
    for workload, cfg_name in (('3dmatch20k', '3dmatch'), ('kitti4k', 'kitti')):
        print(json.dumps(run(workload, cfg_name, a.batch, max(20, a.reps))))


if __name__ == '__main__':
    main()
