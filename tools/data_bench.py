"""Times of the data-side pieces of training, one JSON line each:
  kernel_points   the device disposition optimisation (geob200_kernel_point_optimize, 100 candidates of 15 points) against the numpy
                  restatement (tests/kernel_points_oracle.py) of the reference's descent
  calibration     calibrate_neighbors_augmented (chunks of pairs) against the per-pair calibrate_neighbors_stack_mode on the same
                  augmented pairs, 3DMatch demo-size pairs
  loader          PrefetchLoader steps per second from a 3DMatch tree of 3dmatch20k-size clouds and a KITTI tree of kitti20k-size clouds
                  in a temporary directory (warm page cache: every file is read once before the timed epochs), beside the
                  steps per second of TrainingEngine.train_batch (augmented, random-init weights) at the same B and cloud size:
                  prefetch hides the file reads when the loader's rate is the higher one
Every number is the median of --repeats runs, with min and max.  Usage: python tools/data_bench.py [--repeats R]
"""
import argparse
import json
import os
import pickle
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def _stats(xs):
    return {'median': statistics.median(xs), 'min': min(xs), 'max': max(xs), 'n': len(xs)}


def _gpu():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def bench_kernel_points(repeats):
    import kernel_points_oracle as O
    from geotransformer_b200.modules.kpconv import kernel_points as KP
    KP.optimize_dispositions(15)
    dev = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t = time.perf_counter()
        KP.optimize_dispositions(15)
        torch.cuda.synchronize()
        dev.append(time.perf_counter() - t)
    init = O.accept(O.philox_uniforms(0, 12000), 1500)
    t = time.perf_counter()
    O.optimize(init, 100, 15)
    host = time.perf_counter() - t
    return {'bench': 'kernel_points', 'device_s': _stats(dev), 'numpy_s': host}


def bench_calibration(repeats, n=24):
    from geotransformer_b200.augment import augment_stacked
    from geotransformer_b200.config import make_cfg
    from geotransformer_b200.synth import make_pair
    from geotransformer_b200.utils.data import (CALIBRATION_ITERATION, calibrate_neighbors_augmented, calibrate_neighbors_stack_mode,
                                                registration_collate_fn_stack_mode)
    cfg = make_cfg('3dmatch')
    b = cfg.backbone
    pairs = [make_pair('demo2k', i) for i in range(n)]
    dev = torch.device('cuda', torch.cuda.current_device())
    threshold = 10 ** 9          # no early exit: every pair is histogrammed in both
    batched, per_pair = [], []
    calibrate_neighbors_augmented(pairs[:4], cfg, 1, sample_threshold=threshold)
    for _ in range(repeats):
        torch.cuda.synchronize()
        t = time.perf_counter()
        calibrate_neighbors_augmented(pairs, cfg, 1, sample_threshold=threshold)
        torch.cuda.synchronize()
        batched.append(time.perf_counter() - t)
        t = time.perf_counter()
        items = []
        for p, pair in enumerate(pairs):
            pts, lengths, T, _, _ = augment_stacked([pair], cfg, 1, CALIBRATION_ITERATION, dev, pair_base=p)
            items.append({'ref_points': pts[:lengths[0]], 'src_points': pts[lengths[0]:], 'ref_feats': torch.ones((lengths[0], 1), device=dev),
                          'src_feats': torch.ones((lengths[1], 1), device=dev), 'transform': T[0]})
        calibrate_neighbors_stack_mode(items, registration_collate_fn_stack_mode, b.num_stages, b.init_voxel_size, b.init_radius,
                                       sample_threshold=threshold)
        torch.cuda.synchronize()
        per_pair.append(time.perf_counter() - t)
    return {'bench': 'calibration', 'pairs': n, 'batched_s': _stats(batched), 'per_pair_s': _stats(per_pair)}


def bench_loader(repeats, workload, n=64, batch=4):
    from geotransformer_b200.datasets.kitti import KittiPairs
    from geotransformer_b200.datasets.loader import PrefetchLoader
    from geotransformer_b200.datasets.threedmatch import ThreeDMatchPairs
    from geotransformer_b200.synth import make_pair
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, 'metadata'))
        meta = []
        kitti = workload.startswith('kitti')
        for i in range(n):
            pair = make_pair(workload, i % 4)
            names = [f'downsampled/00/{2 * i:06d}.npy', f'downsampled/00/{2 * i + 1:06d}.npy'] if kitti else \
                [f'train/scene/cloud_bin_{2 * i}.pth', f'train/scene/cloud_bin_{2 * i + 1}.pth']
            for name, key in zip(names, ('ref_points', 'src_points')):
                path = os.path.join(tmp, name) if kitti else os.path.join(tmp, 'data', name)
                os.makedirs(os.path.dirname(path), exist_ok=True)
                np.save(path, pair[key]) if kitti else torch.save(pair[key], path)
            T = pair['transform'].astype(np.float64)
            meta.append({'seq_id': 0, 'frame0': 2 * i, 'frame1': 2 * i + 1, 'pcd0': names[0], 'pcd1': names[1], 'transform': T} if kitti else
                        {'pcd0': names[0], 'pcd1': names[1], 'rotation': T[:3, :3], 'translation': T[:3, 3], 'overlap': 0.5,
                         'scene_name': 'scene', 'frag_id0': 2 * i, 'frag_id1': 2 * i + 1})
        with open(os.path.join(tmp, 'metadata', 'train.pkl'), 'wb') as f:
            pickle.dump(meta, f)
        ds = KittiPairs(tmp, 'train') if kitti else ThreeDMatchPairs(tmp, 'train')
        loader = PrefetchLoader(ds, batch, seed=0)
        for _ in loader.epoch(0):
            pass
        rates = []
        for r in range(repeats):
            t = time.perf_counter()
            steps = sum(1 for _ in loader.epoch(r + 1))
            rates.append(steps / (time.perf_counter() - t))
    return {'bench': 'loader', 'workload': workload, 'pairs': n, 'batch_size': batch, 'steps_per_s': _stats(rates)}


def bench_train_step(repeats, workload, batch=4, steps=5):
    from geotransformer_b200.config import make_cfg
    from geotransformer_b200.model import create_model
    from geotransformer_b200.synth import make_pair
    from geotransformer_b200.train import TrainingEngine
    from geotransformer_b200.utils.data import calibrate_neighbors_augmented
    cfg = make_cfg('kitti' if workload.startswith('kitti') else '3dmatch')
    pairs = [make_pair(workload, i) for i in range(4)]
    limits, _ = calibrate_neighbors_augmented(pairs, cfg, 0)
    torch.manual_seed(0)
    engine = TrainingEngine(create_model(cfg).cuda(), cfg, [int(x) for x in limits], seed=0, batch_size=batch, augment=True)
    group = [pairs[i % 4] for i in range(batch)]
    for _ in range(2):
        engine.train_batch(group)
    rates = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t = time.perf_counter()
        for _ in range(steps):
            engine.train_batch(group)
        torch.cuda.synchronize()
        rates.append(steps / (time.perf_counter() - t))
    return {'bench': 'train_batch', 'workload': workload, 'batch_size': batch, 'steps_per_s': _stats(rates)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('data_bench.py needs a CUDA device')
    gpu = _gpu()
    benches = (lambda: bench_kernel_points(args.repeats), lambda: bench_calibration(args.repeats),
               lambda: bench_loader(args.repeats, '3dmatch20k'), lambda: bench_train_step(args.repeats, '3dmatch20k'),
               lambda: bench_loader(args.repeats, 'kitti20k'), lambda: bench_train_step(args.repeats, 'kitti20k'))
    for bench in benches:
        res = bench()
        res['gpu'] = gpu
        print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
