"""KITTI odometry pairs from the reference's dataset tree (``datasets/registration/kitti/dataset.py``).

``{root}/metadata/{subset}.pkl`` lists the pairs (``seq_id``, ``frame0``, ``frame1``, ``pcd0``, ``pcd1``, ``transform``); ``pcd0`` /
``pcd1`` are paths relative to ``root`` of downsampled (N, 3) ``.npy`` clouds.  An item is the reference dataset's dict without
augmentation: training pairs go raw to ``augment.augmented_collate``, which augments them on the device.
"""
import os
import pickle

import numpy as np

from .threedmatch import check_host_options

SUBSETS = ('train', 'val', 'test')


class KittiPairs:
    def __init__(self, root, subset, point_limit=None):
        if subset not in SUBSETS:
            raise ValueError(f'subset must be one of {SUBSETS}, got {subset!r}')
        check_host_options(point_limit, False)
        self.root, self.subset = root, subset
        with open(os.path.join(root, 'metadata', f'{subset}.pkl'), 'rb') as f:
            self.metadata = pickle.load(f)

    def __len__(self):
        return len(self.metadata)

    def files(self, index):
        """the two cloud files of pair ``index``"""
        m = self.metadata[index]
        return os.path.join(self.root, m['pcd0']), os.path.join(self.root, m['pcd1'])

    def __getitem__(self, index):
        m = self.metadata[index]
        ref_points, src_points = (np.load(p) for p in self.files(index))
        return {'seq_id': m['seq_id'], 'ref_frame': m['frame0'], 'src_frame': m['frame1'],
                'ref_points': ref_points.astype(np.float32), 'src_points': src_points.astype(np.float32),
                'ref_feats': np.ones((ref_points.shape[0], 1), dtype=np.float32),
                'src_feats': np.ones((src_points.shape[0], 1), dtype=np.float32),
                'transform': m['transform'].astype(np.float32)}
