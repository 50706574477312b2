"""Times voxel downsampling (geob200_voxel_down_sample) on the device and the single-threaded C++ oracle on the same clouds.

    python tools/voxel_bench.py [--iters 20] [--files 64] [--out FILE]

- ``kitti16``: one batched call on 16 KITTI-size synthetic ring scans (120 k points each, float32-origin) at 0.3 m.
- ``3dmatch``: one call on a 3DMatch-size synthetic fragment (300 k points, float64) at 2.5 cm.
Device time per call comes from CUDA events around ``--iters`` calls after three warm-up calls (one includes the status read-back
and the output slicing of ``functional.voxel_down_sample_batched``).  The oracle (oracle/liboracle_voxel.so) is timed once per
cloud on the host; it stands in for Open3D's single-threaded loop and is not Open3D.  ``driver`` runs
``python -m geotransformer_b200.datasets.kitti_downsample`` on a synthetic tree of ``--files`` scans in a temporary directory and
compares its files per second with reading the same files alone.  Prints one JSON line with the GPU's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from geotransformer_b200 import functional as GF  # noqa: E402
from geotransformer_b200.datasets import kitti_downsample  # noqa: E402
from oracle import voxel_oracle as VO  # noqa: E402


def ring_scan(rng, n=120000):
    az = rng.uniform(0, 2 * np.pi, n)
    elev = np.deg2rad(rng.integers(0, 64, n) * (28.0 / 64) - 25.0)
    r = rng.uniform(3.0, 80.0, n)
    xyz = np.stack([r * np.cos(az) * np.cos(elev), r * np.sin(az) * np.cos(elev), r * np.sin(elev) + 1.73], 1)
    return xyz.astype(np.float32)


def fragment(rng, n=300000):
    k = n // 4
    a = np.stack([rng.uniform(0, 3, k), rng.uniform(0, 3, k), np.zeros(k)], 1)
    b = np.stack([np.zeros(k), rng.uniform(0, 3, k), rng.uniform(0, 3, k)], 1)
    c = np.stack([rng.uniform(0, 3, k), np.full(k, 3.0), rng.uniform(0, 3, k)], 1)
    d = rng.standard_normal((n - 3 * k, 3))
    d = d / np.linalg.norm(d, axis=1, keepdims=True) * 0.7 + 1.5
    return np.concatenate([a, b, c, d]) + rng.normal(0, 0.003, (n, 3))


def time_device(clouds, voxel, iters):
    lengths = [c.shape[0] for c in clouds]
    pts = torch.from_numpy(np.concatenate(clouds).astype(np.float64)).cuda()
    for _ in range(3):
        out = GF.voxel_down_sample_batched(pts, lengths, voxel)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        GF.voxel_down_sample_batched(pts, lengths, voxel)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters, int(out[1].sum())


def time_oracle(clouds, voxel):
    t0 = time.perf_counter()
    for c in clouds:
        VO.voxel_down_sample(c.astype(np.float64), voxel)
    return (time.perf_counter() - t0) * 1e3


def time_driver(n_files, rng):
    with tempfile.TemporaryDirectory() as root:
        vel = os.path.join(root, 'sequences', '00', 'velodyne')
        os.makedirs(vel)
        for f in range(n_files):
            xyz = ring_scan(rng)
            np.concatenate([xyz, np.zeros((xyz.shape[0], 1), np.float32)], 1).tofile(os.path.join(vel, f'{f:06d}.bin'))
        t0 = time.perf_counter()
        for f in range(n_files):
            np.fromfile(os.path.join(vel, f'{f:06d}.bin'), dtype=np.float32).reshape(-1, 4)[:, :3].copy()
        read_s = time.perf_counter() - t0
        kitti_downsample.run(root, sequences=[0], batch=16, threads=4, log=None)   # warm-up (module load, workspace)
        t0 = time.perf_counter()
        kitti_downsample.run(root, sequences=[0], batch=16, threads=4, log=None)
        drive_s = time.perf_counter() - t0
    return n_files / drive_s, n_files / read_s


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
    ap.add_argument('--files', type=int, default=64)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    name, limit = gpu_info()
    res = {'gpu': name, 'power_limit': limit}
    kitti = [ring_scan(rng) for _ in range(16)]
    ms, m = time_device(kitti, 0.3, args.iters)
    res['kitti16'] = {'points': int(sum(c.shape[0] for c in kitti)), 'voxels': m, 'device_ms': round(ms, 3),
                      'oracle_ms': round(time_oracle(kitti, 0.3), 1)}
    frag = [fragment(rng)]
    ms, m = time_device(frag, 0.025, args.iters)
    res['3dmatch'] = {'points': int(frag[0].shape[0]), 'voxels': m, 'device_ms': round(ms, 3),
                      'oracle_ms': round(time_oracle(frag, 0.025), 1)}
    files_s, read_s = time_driver(args.files, rng)
    res['driver'] = {'files': args.files, 'files_per_s': round(files_s, 1), 'read_only_files_per_s': round(read_s, 1)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
