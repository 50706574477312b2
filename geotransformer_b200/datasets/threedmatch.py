"""3DMatch / 3DLoMatch pairs from the reference's dataset tree (``datasets/registration/threedmatch/dataset.py``).

``{root}/metadata/{subset}.pkl`` lists the pairs (``pcd0``, ``pcd1``, ``rotation``, ``translation``, ``overlap``, ``scene_name``,
``frag_id0``, ``frag_id1``); ``{root}/data/{pcd}`` holds each cloud as a ``torch.save``d (N, 3) array.  An item is the reference
dataset's dict without augmentation: training pairs go raw to ``augment.augmented_collate``, which applies the point limit, the
rotation and the noise on the device.

``rotated=True`` (every subset but 'train') is the reference's rotated benchmark: ref and src each get a random rotation from
``random_sample_rotation_v2`` and the transform follows them.  The reference draws them from numpy's unseeded global stream, so its
rotated benchmark changes from run to run; here pair i draws from ``np.random.seed(i)``, the convention of the ModelNet val / test
pairs, so the benchmark is fixed.  The rotations, points and transform come from ``functional.rotated_pairs_batched`` on the device
and equal the reference's item after ``np.random.seed(i)`` bit for bit wherever the host libm rounds the half-angles' sin and cos
correctly (the device rounds them correctly; DESIGN.md section 8a).  ``rotated_batch`` builds a chunk of pairs as device tensors.
"""
import os
import pickle

import numpy as np
import torch

from .. import functional as GF

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
        raise NotImplementedError('rotated=True for training pairs (the device augmentation would have to rotate after it augments; '
                                  'no shipped config trains on rotated pairs)')


class ThreeDMatchPairs:
    def __init__(self, root, subset, overlap_threshold=None, point_limit=None, rotated=False):
        if subset not in SUBSETS:
            raise ValueError(f'subset must be one of {SUBSETS}, got {subset!r}')
        check_host_options(point_limit, rotated and subset == 'train')
        self.root, self.subset, self.rotated = root, subset, bool(rotated)
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

    def _clouds(self, index):
        # the clouds are numpy arrays pickled by torch.save, so they need the full unpickler
        return [np.asarray(torch.load(p, weights_only=False)) for p in self.files(index)]

    def _meta(self, index):
        m = self.metadata_list[index]
        return {'scene_name': m['scene_name'], 'ref_frame': m['frag_id0'], 'src_frame': m['frag_id1'], 'overlap': m['overlap']}

    def __getitem__(self, index):
        if self.rotated:
            d = self.rotated_batch([index], device='cuda')[0]
            return {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}
        m = self.metadata_list[index]
        ref_points, src_points = self._clouds(index)
        transform = transform_from_rotation_translation(m['rotation'], m['translation'])
        return dict(self._meta(index), ref_points=ref_points.astype(np.float32), src_points=src_points.astype(np.float32),
                    ref_feats=np.ones((ref_points.shape[0], 1), dtype=np.float32),
                    src_feats=np.ones((src_points.shape[0], 1), dtype=np.float32), transform=transform.astype(np.float32))

    def rotated_batch(self, indices, device='cuda'):
        """The rotated items of ``indices`` as dicts of device tensors (points, feats, transform) and the metadata fields: the
        clouds are packed into one pinned buffer, copied to the device once and rotated by one ``rotated_pairs_batched`` call.
        Returns after the rotation has finished, because the engines read their inputs on streams that do not wait for this one."""
        if not self.rotated:
            raise ValueError('rotated_batch needs rotated=True')
        indices = [int(i) for i in indices]
        device = torch.device(device)
        if device.type == 'cuda' and device.index is None:
            device = torch.device('cuda', torch.cuda.current_device())
        clouds = [self._clouds(i) for i in indices]
        dtype = np.float64 if any(c.dtype == np.float64 for pair in clouds for c in pair) else np.float32
        stacked = [c for pair in clouds for c in pair[:1]] + [c for pair in clouds for c in pair[1:]]
        lengths = [int(c.shape[0]) for c in stacked]
        host = torch.empty((sum(lengths), 3), dtype=torch.float64 if dtype == np.float64 else torch.float32, pin_memory=True)
        hv, row = host.numpy(), 0
        for c in stacked:
            hv[row:row + c.shape[0]] = c              # a float32 cloud widens exactly when another cloud of the chunk is float64
            row += c.shape[0]
        transforms = np.stack([transform_from_rotation_translation(self.metadata_list[i]['rotation'], self.metadata_list[i]['translation'])
                               for i in indices])
        with torch.cuda.device(device):
            points = host.to(device, non_blocking=True)
            out, T, _ = GF.rotated_pairs_batched(points, lengths, indices, transforms)
            torch.cuda.current_stream(device).synchronize()
        B, starts = len(indices), np.concatenate([[0], np.cumsum(lengths)])
        items = []
        for p, i in enumerate(indices):
            ref, src = out[starts[p]:starts[p + 1]], out[starts[B + p]:starts[B + p + 1]]
            items.append(dict(self._meta(i), ref_points=ref, src_points=src,
                              ref_feats=torch.ones((ref.shape[0], 1), dtype=torch.float32, device=device),
                              src_feats=torch.ones((src.shape[0], 1), dtype=torch.float32, device=device), transform=T[p]))
        return items
