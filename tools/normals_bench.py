"""Times normal estimation (geob200_estimate_normals) on the device and the single-threaded C++ oracle on the same clouds.

    python tools/normals_bench.py [--iters 20] [--oracle-rows 200] [--bench-steps 20] [--out FILE]

- ``kitti16``: one batched call on 16 KITTI-size synthetic ring scans (120 k points each, float32-origin), knn 30.
- ``3dmatch``: one call on a 3DMatch-size synthetic fragment (300 k points), knn 30.
- ``modelnet64``: one call on 64 ModelNet-size shapes (1 024 points each), knn 30.
- ``hybrid``: the fragment with ``KDTreeSearchParamHybrid(0.05, 30)``.
- ``outlier``: a 100 k-point fragment alone and with one point 100 m away diagonally, which inflates the grid's cell edge
  (DESIGN.md section 8a names this limit); one warm-up and ``--outlier-iters`` timed calls each.
- ``kernels``: the device time per kernel of one fragment call under ``torch.profiler``, in a run of its own.
Device time per call comes from CUDA events around ``--iters`` calls after three warm-up calls (each includes the status
read-back of ``functional.estimate_normals_batched``).  The oracle is a brute-force restatement (a full sort per query), so it is
timed on ``--oracle-rows`` queries per case and scaled to all points; it stands in for no Open3D figure.  Then ``bench.py`` runs
in the same session, to show its figure beside these.  Prints one JSON line with the GPU's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from geotransformer_b200 import functional as GF  # noqa: E402
from oracle import normals_oracle as NO  # noqa: E402


def time_device(clouds, iters, radius=None, warmup=3):
    lengths = [c.shape[0] for c in clouds]
    pts = torch.from_numpy(np.concatenate(clouds).astype(np.float64)).cuda()
    for _ in range(warmup):
        GF.estimate_normals_batched(pts, lengths, knn=30, radius=radius)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        GF.estimate_normals_batched(pts, lengths, knn=30, radius=radius)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def time_oracle(clouds, rows, rng, radius=None):
    """ms for every point of every cloud, extrapolated from ``rows`` queries per cloud"""
    total = 0.0
    for c in clouds:
        r = rng.choice(c.shape[0], min(rows, c.shape[0]), replace=False)
        t0 = time.perf_counter()
        NO.estimate_normals(c, 30, radius, rows=r)
        total += (time.perf_counter() - t0) * 1e3 * c.shape[0] / len(r)
    return total


def kernel_times(cloud, calls=5):
    """ms per call of each kernel, from torch.profiler's CUDA activity over ``calls`` calls after a warm-up"""
    from torch.profiler import ProfilerActivity, profile
    pts = torch.from_numpy(cloud.astype(np.float64)).cuda()
    GF.estimate_normals_batched(pts, [pts.shape[0]])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            GF.estimate_normals_batched(pts, [pts.shape[0]])
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        t = getattr(ev, 'device_time_total', None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            name = ev.key.replace('(anonymous namespace)::', '').split('(')[0].split('::')[-1][:60]
            out[name] = round(out.get(name, 0.0) + t / 1e3 / calls, 4)
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def gpu_info():
    name = torch.cuda.get_device_name()
    try:
        limit = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                               timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001 - the figure is reported as unknown
        limit = 'unknown'
    return name, limit


def run_bench(steps):
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--gpus', '1', '--steps', str(steps), '--warmup', '3'],
                         capture_output=True, text=True, cwd=ROOT, timeout=1800)
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith('{')]
    return json.loads(lines[-1]) if lines else {'error': out.stderr[-500:]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--oracle-rows', type=int, default=200)
    ap.add_argument('--bench-steps', type=int, default=20)
    ap.add_argument('--outlier-iters', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    name, limit = gpu_info()
    res = {'gpu': name, 'power_limit': limit}
    kitti = [NO.ring_scan(rng).astype(np.float64) for _ in range(16)]
    frag = [NO.fragment(rng)]
    shapes = [rng.standard_normal((1024, 3)) * 0.3 for _ in range(64)]
    shapes = [s / np.linalg.norm(s, axis=1, keepdims=True) * rng.uniform(0.5, 1.0, (1024, 1)) for s in shapes]
    for key, clouds, radius in (('kitti16', kitti, None), ('3dmatch', frag, None), ('modelnet64', shapes, None),
                                ('hybrid', frag, 0.05)):
        ms = time_device(clouds, args.iters, radius)
        res[key] = {'points': int(sum(c.shape[0] for c in clouds)), 'clouds': len(clouds), 'radius': radius,
                    'device_ms': round(ms, 3), 'oracle_ms_extrapolated': round(time_oracle(clouds, args.oracle_rows, rng, radius), 1)}
    small = NO.fragment(rng, 100000)
    far = np.concatenate([small, [[100.0, 100.0, 100.0]]])
    res['outlier'] = {'points': int(small.shape[0]),
                      'device_ms_without': round(time_device([small], args.outlier_iters, warmup=1), 3),
                      'device_ms_with_one_outlier': round(time_device([far], args.outlier_iters, warmup=1), 3)}
    res['kernels_3dmatch_ms'] = kernel_times(frag[0])
    res['bench'] = run_bench(args.bench_steps)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
