"""Prepare the KITTI tree the reference's ``data/Kitti/downsample_pcd.py`` writes, on the device and without Open3D.

    python -m geotransformer_b200.datasets.kitti_downsample --root DIR [--sequences 0 ... 10] [--batch 16] [--threads 4]

For every ``{root}/sequences/{seq}/velodyne/{frame}.bin`` scan: read it as (-1, 4) float32, keep ``[:, :3]``, voxel-downsample it
at 0.3 m with Open3D's semantics (``functional.voxel_down_sample_batched``, DESIGN.md section 8a) and save the float32 result as
``{root}/downsampled/{seq}/{frame}.npy``, the files ``datasets.kitti.KittiPairs`` reads.  Host threads read the next batch of scans
into pinned memory while the device downsamples the current one in a single call, and write the finished batch's files.
"""
import argparse
import glob
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from .. import functional as GF

VOXEL_SIZE = 0.3


def scan_files(root, sequences):
    """(seq_id, frame, path) of every velodyne scan of ``sequences``, in sequence then file-name order"""
    out = []
    for s in sequences:
        seq_id = '{:02d}'.format(int(s))
        for path in sorted(glob.glob(os.path.join(root, 'sequences', seq_id, 'velodyne', '*.bin'))):
            out.append((seq_id, os.path.basename(path)[:-4], path))
    return out


def _read(path):
    points = np.fromfile(path, dtype=np.float32).reshape(-1, 4)[:, :3]
    return torch.from_numpy(np.ascontiguousarray(points)).pin_memory()


def _save(path, points):
    np.save(path, points)


def run(root, sequences=range(11), batch=16, threads=4, voxel_size=VOXEL_SIZE, log=print):
    """downsample every scan of ``sequences`` under ``root``; returns the number of files written"""
    if not 1 <= batch <= GF.VOXEL_MAX_CLOUDS:
        raise ValueError(f'batch must be in 1..{GF.VOXEL_MAX_CLOUDS}')
    files = scan_files(root, sequences)
    for seq_id in sorted({f[0] for f in files}):
        os.makedirs(os.path.join(root, 'downsampled', seq_id), exist_ok=True)
    groups = [files[i:i + batch] for i in range(0, len(files), batch)]
    device = torch.device('cuda', torch.cuda.current_device())
    with ThreadPoolExecutor(max(1, int(threads))) as pool:
        pending = [pool.submit(_read, f[2]) for f in groups[0]] if groups else []
        writes = []
        for g, group in enumerate(groups):
            clouds = [f.result() for f in pending]
            # the next batch is read while this one is on the device
            pending = [pool.submit(_read, f[2]) for f in groups[g + 1]] if g + 1 < len(groups) else []
            lengths = [c.shape[0] for c in clouds]
            points = torch.cat([c.to(device, non_blocking=True) for c in clouds]) if clouds else None
            out, out_len = GF.voxel_down_sample_batched(points, lengths, voxel_size)[:2]
            out = out.to(torch.float32).cpu().numpy()          # np.array(pcd.points).astype(np.float32)
            start = 0
            for (seq_id, frame, _), m in zip(group, out_len.tolist()):
                writes.append(pool.submit(_save, os.path.join(root, 'downsampled', seq_id, frame + '.npy'), out[start:start + m]))
                start += m
            if log is not None:
                log(f'batch {g + 1}/{len(groups)}: {len(group)} scans, {sum(lengths)} points -> {start} points')
        for w in writes:
            w.result()
    return len(files)


def main(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    parser.add_argument('--root', required=True, help='the KITTI odometry root holding sequences/')
    parser.add_argument('--sequences', type=int, nargs='+', default=list(range(11)))
    parser.add_argument('--batch', type=int, default=16, help='scans per device call (1..64)')
    parser.add_argument('--threads', type=int, default=4, help='host threads reading and writing files')
    args = parser.parse_args(argv)
    n = run(args.root, args.sequences, args.batch, args.threads)
    print(f'{n} scans downsampled into {os.path.join(args.root, "downsampled")}')


if __name__ == '__main__':
    main()
