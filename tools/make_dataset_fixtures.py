"""Writes two data fixtures from a checkout of the reference GeoTransformer (path as the first argument):
  tests/golden/dataset_metadata.pkl     the first 32 entries of every 3DMatch / 3DLoMatch and KITTI metadata split, as the reference
                                        pickles them ({'3DMatch/train': [...], ..., 'Kitti/test': [...]})
  tests/golden/kernel_disposition.npz   the reference's k_015_center_3D.ply points (15 x 3 fp64), their potential energy and mean
                                        radius of the non-centre points
"""
import os
import pickle
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import kernel_points_oracle as O  # noqa: E402


def main(ref):
    out = {}
    for dataset, splits in (('3DMatch', ('train', 'val', '3DMatch', '3DLoMatch')), ('Kitti', ('train', 'val', 'test'))):
        for split in splits:
            with open(os.path.join(ref, 'data', dataset, 'metadata', f'{split}.pkl'), 'rb') as f:
                out[f'{dataset}/{split}'] = pickle.load(f)[:32]
    with open(os.path.join(ROOT, 'tests', 'golden', 'dataset_metadata.pkl'), 'wb') as f:
        pickle.dump(out, f, protocol=4)
    pts = O.read_ply_points(os.path.join(ref, 'geotransformer', 'modules', 'kpconv', 'dispositions', 'k_015_center_3D.ply'))
    np.savez(os.path.join(ROOT, 'tests', 'golden', 'kernel_disposition.npz'), points=pts, energy=O.energy(pts),
             mean_radius=np.linalg.norm(pts[1:], axis=1).mean())


if __name__ == '__main__':
    main(sys.argv[1])
