"""Times the rotated 3DMatch benchmark pairs: ``functional.rotated_pairs_batched`` on the device against the reference's numpy path,
and the tester on rotated against un-rotated pairs.

    python tools/rotated_bench.py [--iters 50] [--rounds 2] [--out FILE]

- ``op``: one call on 16 pairs of 20 000 + 20 000 fp32 points already on the device; CUDA events around ``--iters`` calls after three
  warm-up calls.  Bytes are the points read and written (24 per row; the draws and transforms are negligible), over the time, and
  that rate over the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  ``numpy_ms`` is the reference's host path for the same 16
  pairs (np.random.seed, two random_sample_rotation_v2, the numpy matmuls and the fp32 casts), one pass.
- ``tester``: ``RegistrationTester.run`` (synthetic weights, the config's neighbour limits, no output files) over the same 16 pairs
  from a temporary dataset tree, un-rotated and rotated alternately for ``--rounds`` rounds after one warm-up pass of each; pairs/s
  per pass, including the file reads.
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
from geotransformer_b200.datasets.threedmatch import ThreeDMatchPairs, transform_from_rotation_translation  # noqa: E402
from geotransformer_b200.tester import RegistrationTester  # noqa: E402

PAIRS, POINTS = 16, 20000


def fragment(rng, n=POINTS):
    """three walls and a ball in a 3 m room, 3 mm noise"""
    k = n // 4
    a = np.stack([rng.uniform(0, 3, k), rng.uniform(0, 3, k), np.zeros(k)], 1)
    b = np.stack([np.zeros(k), rng.uniform(0, 3, k), rng.uniform(0, 3, k)], 1)
    c = np.stack([rng.uniform(0, 3, k), np.full(k, 3.0), rng.uniform(0, 3, k)], 1)
    d = rng.standard_normal((n - 3 * k, 3))
    d = d / np.linalg.norm(d, axis=1, keepdims=True) * 0.7 + 1.5
    return (np.concatenate([a, b, c, d]) + rng.normal(0, 0.003, (n, 3))).astype(np.float32)


def synthetic_pairs(rng):
    pairs = []
    for _ in range(PAIRS):
        ref = fragment(rng)
        R = Rotation.from_euler('zyx', rng.uniform(-0.3, 0.3, 3)).as_matrix()
        t = rng.uniform(-0.2, 0.2, 3)
        src = ((fragment(rng).astype(np.float64) - t) @ R).astype(np.float32)       # ref ~= R src + t
        pairs.append((ref, src, R, t))
    return pairs


def rotation_v2():
    axis = np.random.rand(3) - 0.5
    axis = axis / np.linalg.norm(axis) + 1e-8
    theta = np.pi * np.random.rand()
    return Rotation.from_euler('zyx', axis * theta).as_matrix()


def numpy_path(pairs):
    t0 = time.perf_counter()
    for i, (ref, src, R, t) in enumerate(pairs):
        np.random.seed(i)
        Rr = rotation_v2()
        ref_r, rot, tr = np.matmul(ref, Rr.T), np.matmul(Rr, R), np.matmul(Rr, t)
        Rs = rotation_v2()
        src_r, rot = np.matmul(src, Rs.T), np.matmul(rot, Rs.T)
        ref_r.astype(np.float32), src_r.astype(np.float32), transform_from_rotation_translation(rot, tr).astype(np.float32)
    return (time.perf_counter() - t0) * 1e3


def time_op(pairs, iters):
    stacked = [p[0] for p in pairs] + [p[1] for p in pairs]
    lengths = [len(c) for c in stacked]
    pts = torch.from_numpy(np.concatenate(stacked)).cuda()
    T = np.stack([transform_from_rotation_translation(p[2], p[3]) for p in pairs])
    for _ in range(3):
        GF.rotated_pairs_batched(pts, lengths, range(PAIRS), T)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        GF.rotated_pairs_batched(pts, lengths, range(PAIRS), T)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / iters
    nbytes = 24 * sum(lengths)
    return ms, nbytes


def write_tree(root, pairs):
    meta = []
    for j, (ref, src, R, t) in enumerate(pairs):
        names = [f'test/7-scenes-redkitchen/cloud_bin_{2 * j + k}.pth' for k in (0, 1)]
        for name, pts in zip(names, (ref, src)):
            os.makedirs(os.path.join(root, 'data', os.path.dirname(name)), exist_ok=True)
            torch.save(pts, os.path.join(root, 'data', name))
        meta.append({'pcd0': names[0], 'pcd1': names[1], 'rotation': R, 'translation': t, 'overlap': 0.5,
                     'scene_name': '7-scenes-redkitchen', 'frag_id0': 2 * j, 'frag_id1': 2 * j + 1})
    os.makedirs(os.path.join(root, 'metadata'), exist_ok=True)
    with open(os.path.join(root, 'metadata', '3DMatch.pkl'), 'wb') as f:
        pickle.dump(meta, f)


def time_tester(pairs, rounds):
    cfg = trainval.make_cfg('3dmatch')
    device = torch.device('cuda', torch.cuda.current_device())
    model = trainval.build_model(cfg, 5, device)
    model.eval()
    tester = RegistrationTester(cfg, model, list(cfg.neighbor_limits), output_dir=None, device=device)
    res = {'unrotated': [], 'rotated': []}
    try:
        with tempfile.TemporaryDirectory() as root:
            write_tree(root, pairs)
            sets = {'unrotated': ThreeDMatchPairs(root, '3DMatch'), 'rotated': ThreeDMatchPairs(root, '3DMatch', rotated=True)}
            for r in range(rounds + 1):
                for name, ds in sets.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    tester.run(ds)
                    torch.cuda.synchronize()
                    if r > 0:                                   # round 0 warms both paths up
                        res[name].append(round(len(ds) / (time.perf_counter() - t0), 2))
    finally:
        tester.close()
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
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    name, limit = gpu_info()
    pairs = synthetic_pairs(rng)
    ms, nbytes = time_op(pairs, args.iters)
    res = {'gpu': name, 'power_limit': limit,
           'op': {'pairs': PAIRS, 'points_per_cloud': POINTS, 'device_ms': round(ms, 4), 'bytes': nbytes,
                  'GB_per_s': round(nbytes / ms / 1e6, 1), 'share_of_hbm': round(nbytes / ms / 1e6 / 3350, 4),
                  'numpy_ms': round(numpy_path(pairs), 2)},
           'tester_pairs_per_s': time_tester(pairs, args.rounds)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
