"""Device time of the training-data augmentation and its share of a batched training step.

For each workload and batch size B: the median CUDA-event time of the augmentation launches on a device-resident raw batch
(``augment.augment_stacked`` minus its copies: ``functional.augment_pairs_batched`` / ``modelnet_pairs_batched``), the median
CUDA-event time of one ``TrainingEngine.train_batch`` step with ``augment=True`` on the same pairs, and the share.  Also the host
time per pair of the numpy restatement (oracle/augment_oracle.py), the CPU work the kernels replace, and the card's name and power
limit, read in the same run.  One JSON line per measurement.

    python tools/augment_bench.py [--batch 1 4 8] [--steps 10] [--warmup 3] [--limit3dm 15000]
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from geotransformer_b200 import functional as GF                    # noqa: E402
from geotransformer_b200.config import make_cfg                     # noqa: E402
from geotransformer_b200.model import create_model                  # noqa: E402
from geotransformer_b200.synth import make_pair                     # noqa: E402
from geotransformer_b200.train import TrainingEngine                # noqa: E402
from geotransformer_b200.weights import synthetic_state_dict        # noqa: E402
from oracle import augment_oracle as AO                             # noqa: E402
from oracle import backbone_grad_oracle as BG                       # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                            # noqa: BLE001
        q = f'{torch.cuda.get_device_name()}, power limit unavailable ({e})'
    return q


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    out = []
    for _ in range(steps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        out.append(s.elapsed_time(e))
    return float(np.median(out))


def registration(workload, B, limit, steps, warmup):
    pairs = []
    for i in range(B):
        p = make_pair(workload, i)
        pairs.append({k: p[k] for k in ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')})
    cfg = copy.deepcopy(make_cfg(make_pair(workload, 0)['config']))
    cfg.train.point_limit = limit
    clouds = [torch.from_numpy(p['ref_points']) for p in pairs] + [torch.from_numpy(p['src_points']) for p in pairs]
    raw = torch.cat(clouds).cuda()
    T = torch.from_numpy(np.stack([p['transform'] for p in pairs])).cuda()
    lens = [len(c) for c in clouds]
    tr, kitti = cfg.train, cfg.name == 'kitti'
    kw = dict(min_scale=tr.augmentation_min_scale, max_scale=tr.augmentation_max_scale, shift=tr.augmentation_shift) if kitti else {}
    it = [0]

    def aug():
        it[0] += 1
        GF.augment_pairs_batched(raw, lens, T, GF.AUGMENT_KITTI if kitti else GF.AUGMENT_3DMATCH, limit, tr.augmentation_noise,
                                 tr.augmentation_rotation, seed=7351, iteration=it[0], **kw)
    aug_ms = timed(aug, steps, warmup)
    model = create_model(cfg)
    model.load_state_dict(synthetic_state_dict(model, 7351), strict=True)
    # the synthetic KITTI scenes share one neighbour calibration (kitti4k's)
    limits = BG.limits('kitti4k' if cfg.name == 'kitti' else workload)
    eng = TrainingEngine(model.cuda(), cfg, limits, batch_size=B, augment=True)
    step_ms = timed(lambda: eng.train_batch(pairs), steps, warmup)
    t = time.perf_counter()
    for p in range(B):
        AO.augment_pair(pairs[p]['ref_points'], pairs[p]['src_points'], pairs[p]['transform'], AO.KITTI if kitti else AO.THREEDMATCH,
                        limit, tr.augmentation_noise, tr.augmentation_rotation, seed=7351, iteration=1, pair=p, **kw)
    host_ms = (time.perf_counter() - t) * 1e3 / B
    return dict(workload=workload, B=B, point_limit=limit, raw_points=sum(lens), augment_ms=round(aug_ms, 4),
                train_batch_ms=round(step_ms, 2), share_percent=round(100 * aug_ms / step_ms, 3), restatement_host_ms_per_pair=round(host_ms, 2))


def modelnet(B, steps, warmup):
    cfg = make_cfg('modelnet')
    rng = np.random.default_rng(0)
    shapes = [(rng.normal(size=(2048, 3)) * np.array([1.0, 0.6, 0.3])).astype(np.float32) for _ in range(B)]
    raw = torch.from_numpy(np.concatenate(shapes)).cuda()
    d = cfg.data
    it = [0]

    def aug():
        it[0] += 1
        GF.modelnet_pairs_batched(raw, [2048] * B, d.num_points, d.keep_ratio, d.rotation_magnitude, d.translation_magnitude,
                                  cfg.train.noise_magnitude, 7351, it[0])
    aug_ms = timed(aug, steps, warmup)
    t = time.perf_counter()
    for p in range(B):
        AO.modelnet_pair(shapes[p], d.num_points, d.keep_ratio, d.rotation_magnitude, d.translation_magnitude, cfg.train.noise_magnitude,
                         seed=7351, iteration=1, pair=p)
    host_ms = (time.perf_counter() - t) * 1e3 / B
    return dict(workload='modelnet2048', B=B, augment_ms=round(aug_ms, 4), restatement_host_ms_per_pair=round(host_ms, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, nargs='+', default=[1, 4, 8])
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--limit3dm', type=int, default=15000, help='a point limit that binds on the 20k-point 3DMatch clouds')
    a = ap.parse_args()
    print(json.dumps(dict(card=card())), flush=True)
    for B in a.batch:
        for workload, limit in (('3dmatch20k', a.limit3dm), ('kitti60k', 30000)):
            try:
                print(json.dumps(registration(workload, B, limit, a.steps, a.warmup)), flush=True)
            except torch.cuda.OutOfMemoryError:
                print(json.dumps(dict(workload=workload, B=B, point_limit=limit, error='out of memory')), flush=True)
            except RuntimeError as e:              # a batch beyond a limit of the training step itself
                print(json.dumps(dict(workload=workload, B=B, point_limit=limit, error=str(e))), flush=True)
            torch.cuda.empty_cache()
        print(json.dumps(modelnet(B, a.steps, a.warmup)), flush=True)


if __name__ == '__main__':
    main()
