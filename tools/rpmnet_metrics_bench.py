"""Times RPMNet's ModelNet metrics: ``functional.rpmnet_metrics_batched`` on the device against the reference's numpy / cKDTree
path on the host, and the ModelNet tester with and without ``rpmnet_metrics``.

    python tools/rpmnet_metrics_bench.py [--iters 20] [--rounds 2] [--out FILE]

- ``op``: 256 test pairs (717 + 717 points, 2 048-point raw shapes, random estimates) already on the device, in calls of 32 pairs
  (the entry point's maximum); CUDA events around ``--iters`` passes over the 256 pairs after two warm-up passes.  ``numpy_ms`` is
  the same 256 pairs on the host: the contract's restatement (oracle/rpmnet_metrics_oracle.py: fp64 transforms, cKDTree,
  scipy-equivalent Euler angles), one pass.
- ``tester``: ``RegistrationTester.run`` (synthetic weights, the ModelNet fixture's neighbour limits) over 64 ModelNet pairs of a temporary
  tree, without and with ``rpmnet_metrics`` alternately for ``--rounds`` rounds after one warm-up pass of each; pairs/s per pass.
Prints one JSON line with the GPU's name and power limit.
"""
import argparse
import json
import os
import pickle
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
from scipy.spatial.transform import Rotation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from geotransformer_b200 import functional as GF  # noqa: E402
from geotransformer_b200 import trainval  # noqa: E402
from geotransformer_b200.datasets.modelnet import ModelNetPairs  # noqa: E402
from geotransformer_b200.tester import RegistrationTester  # noqa: E402
from oracle import backbone_grad_oracle as BV  # noqa: E402
from oracle import modelnet_benchmark_oracle as MB  # noqa: E402
from oracle import rpmnet_metrics_oracle as O  # noqa: E402

PAIRS, TESTER_PAIRS = 256, 64


def synthetic_pairs(rng, n):
    shapes = [s['points'][:2048] for s in MB.synthetic_shapes(n, seed=5, small_every=0)]
    shapes = [s if len(s) == 2048 else np.resize(s, (2048, 3)) for s in shapes]
    dev = torch.device('cuda', torch.cuda.current_device())
    stacked = torch.from_numpy(np.concatenate(shapes).astype(np.float32)).to(dev)
    pts, _, T, _ = GF.modelnet_benchmark_pairs_batched(stacked, [2048] * n, list(range(n)), 717, 0.7, 45.0, 0.5, 0.05)
    raw = GF.modelnet_raw_points_batched(stacked, [2048] * n)
    est = np.stack([np.eye(4, dtype=np.float32)] * n)
    est[:, :3, :3] = Rotation.random(n, random_state=1).as_matrix()
    est[:, :3, 3] = rng.uniform(-0.5, 0.5, (n, 3))
    return raw, pts[:n * 717], pts[n * 717:], T, torch.from_numpy(est).to(dev)


def time_op(raw, ref, src, gt, est, iters):
    n = gt.shape[0]
    calls = [(raw[b * 2048:(b + 32) * 2048], ref[b * 717:(b + 32) * 717], src[b * 717:(b + 32) * 717], gt[b:b + 32], est[b:b + 32])
             for b in range(0, n, 32)]

    def one_pass():
        for r, f, s, g, e in calls:
            k = g.shape[0]
            GF.rpmnet_metrics_batched(r, [2048] * k, f, [717] * k, s, [717] * k, g, e, check=False)

    for _ in range(2):
        one_pass()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        one_pass()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def numpy_path(raw, ref, src, gt, est):
    raw, ref, src, gt, est = (x.cpu().numpy() for x in (raw, ref, src, gt, est))
    t0 = time.perf_counter()
    for p in range(gt.shape[0]):
        O.metrics(raw[p * 2048:(p + 1) * 2048], ref[p * 717:(p + 1) * 717], src[p * 717:(p + 1) * 717], gt[p], est[p])
    return (time.perf_counter() - t0) * 1e3


def time_tester(rounds):
    cfg = trainval.make_cfg('modelnet')
    device = torch.device('cuda', torch.cuda.current_device())
    model = trainval.build_model(cfg, 5, device)
    model.eval()
    res = {'without': [], 'with': []}
    with tempfile.TemporaryDirectory() as root:
        rows = MB.synthetic_shapes(TESTER_PAIRS, seed=11, small_every=0, labels=(0,))
        with open(os.path.join(root, 'test.pkl'), 'wb') as f:
            pickle.dump(rows, f)
        ds = ModelNetPairs(root, 'test', cfg)
        testers = {'without': RegistrationTester(cfg, model, BV.limits('modelnet717'), device=device),
                   'with': RegistrationTester(cfg, model, BV.limits('modelnet717'), device=device, rpmnet_metrics=True)}
        try:
            for r in range(rounds + 1):
                for name, tester in testers.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    tester.run(ds)
                    torch.cuda.synchronize()
                    if r > 0:
                        res[name].append(round(len(ds) / (time.perf_counter() - t0), 2))
        finally:
            for t in testers.values():
                t.close()
    return res


def gpu_info():
    name = torch.cuda.get_device_name()
    try:
        limit = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                               timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001 - the figure is reported as unknown
        limit = 'unknown'
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('rpmnet_metrics_bench needs a GPU')
    name, limit = gpu_info()
    data = synthetic_pairs(np.random.default_rng(0), PAIRS)
    ms = time_op(*data, args.iters)
    res = {'gpu': name, 'power_limit': limit,
           'op': {'pairs': PAIRS, 'points': '717 + 717, raw 2048', 'calls_per_pass': (PAIRS + 31) // 32, 'device_ms': round(ms, 4),
                  'numpy_ms': round(numpy_path(*data), 2)},
           'tester_pairs_per_s': time_tester(args.rounds)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
