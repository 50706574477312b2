"""3DMatch / 3DLoMatch pairs from the reference's dataset tree (``datasets/registration/threedmatch/dataset.py``).

``{root}/metadata/{subset}.pkl`` lists the pairs (``pcd0``, ``pcd1``, ``rotation``, ``translation``, ``overlap``, ``scene_name``,
``frag_id0``, ``frag_id1``); ``{root}/data/{pcd}`` holds each cloud as a ``torch.save``d (N, 3) array.  An item is the reference
dataset's dict without augmentation: training pairs go raw to ``augment.augmented_collate``, which applies the point limit, the
rotation and the noise on the device.
"""
import os
import pickle

import numpy as np
import torch

SUBSETS = ('train', 'val', '3DMatch', '3DLoMatch')


def transform_from_rotation_translation(rotation, translation):
    """reference ``utils/pointcloud.py`` get_transform_from_rotation_translation: (4, 4) float64"""
    transform = np.eye(4)
    transform[:3, :3] = rotation
    transform[:3, 3] = translation
    return transform


def check_host_options(point_limit, rotated):
    if point_limit is not None:
        raise NotImplementedError('point_limit on the host (None in every shipped test / val config; training pairs get the limit '
                                  'on the device in augment.augmented_collate)')
    if rotated:
        raise NotImplementedError('rotated=True (the rotated benchmark draws its rotations on the host)')


class ThreeDMatchPairs:
    def __init__(self, root, subset, overlap_threshold=None, point_limit=None, rotated=False):
        if subset not in SUBSETS:
            raise ValueError(f'subset must be one of {SUBSETS}, got {subset!r}')
        check_host_options(point_limit, rotated)
        self.root, self.subset = root, subset
        self.data_root = os.path.join(root, 'data')
        with open(os.path.join(root, 'metadata', f'{subset}.pkl'), 'rb') as f:
            self.metadata_list = pickle.load(f)
        if overlap_threshold is not None:
            self.metadata_list = [x for x in self.metadata_list if x['overlap'] > overlap_threshold]

    def __len__(self):
        return len(self.metadata_list)

    def files(self, index):
        """the two cloud files of pair ``index``"""
        m = self.metadata_list[index]
        return os.path.join(self.data_root, m['pcd0']), os.path.join(self.data_root, m['pcd1'])

    def __getitem__(self, index):
        m = self.metadata_list[index]
        # the clouds are numpy arrays pickled by torch.save, so they need the full unpickler
        ref_points, src_points = (np.asarray(torch.load(p, weights_only=False)) for p in self.files(index))
        transform = transform_from_rotation_translation(m['rotation'], m['translation'])
        return {'scene_name': m['scene_name'], 'ref_frame': m['frag_id0'], 'src_frame': m['frag_id1'], 'overlap': m['overlap'],
                'ref_points': ref_points.astype(np.float32), 'src_points': src_points.astype(np.float32),
                'ref_feats': np.ones((ref_points.shape[0], 1), dtype=np.float32),
                'src_feats': np.ones((src_points.shape[0], 1), dtype=np.float32),
                'transform': transform.astype(np.float32)}
