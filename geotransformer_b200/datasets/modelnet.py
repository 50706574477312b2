"""ModelNet validation and test pairs built on the device.

The reference's ``ModelNetPairDataset(subset, deterministic=True)`` (``datasets/registration/modelnet/dataset.py``, with the val /
test options of ``EXPMN/dataset.py``) seeds numpy's global generator with each pair's index, so its val and test splits are fixed
sets of pairs.  ``ModelNetPairs`` reads the same ``{root}/{subset}.pkl``, applies the same class filter, and builds those pairs
with ``functional.modelnet_benchmark_pairs_batched``, which reproduces the reference's random stream on the device.  Pairs are
built a chunk at a time and stay on the device, so ``RegistrationEngine.register``, ``TrainingEngine.validate`` and
``RegistrationTester.run`` take them without a copy through the host.  Building a chunk waits for its launch to finish, because
the engines read their inputs on worker streams that do not wait for the caller's stream.
"""
import os
import pickle

import numpy as np
import torch

from .. import functional as GF
from ..utils.data import _stack_to_device

# ModelNetPairDataset.ASYMMETRIC_INDICES: the 32 of the 40 ModelNet40 classes that are not rotationally symmetric
ASYMMETRIC_INDICES = (0, 1, 2, 3, 4, 7, 8, 11, 12, 13, 14, 16, 17, 18, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 35, 36,
                      38, 39)


def get_class_indices(class_indices, asymmetric):
    """'all' -> the 40 classes, 'seen' -> the first 20, 'unseen' -> the last 20, a list or tuple as given; ``asymmetric`` then
    drops the symmetric classes (ModelNetPairDataset.get_class_indices)"""
    if isinstance(class_indices, str):
        if class_indices not in ('all', 'seen', 'unseen'):
            raise ValueError(f"class_indices must be 'all', 'seen', 'unseen' or a list, got {class_indices!r}")
        class_indices = {'all': range(40), 'seen': range(20), 'unseen': range(20, 40)}[class_indices]
    class_indices = list(class_indices)
    if asymmetric:
        class_indices = [x for x in class_indices if x in ASYMMETRIC_INDICES]
    return class_indices


def check_options(cfg):
    """NotImplementedError for the reference's val / test switches that no shipped experiment turns on"""
    d = cfg.data
    if d.get('crop_method', 'plane') != 'plane':
        raise NotImplementedError("ModelNet crop_method='point' (every shipped config crops with a plane)")
    if not d.get('twice_sample', True):
        raise NotImplementedError('ModelNet twice_sample=False (True in every shipped config)')
    if d.get('twice_transform', False):
        raise NotImplementedError('ModelNet twice_transform=True (False in every shipped config)')
    if d.get('voxel_size') is not None:
        raise NotImplementedError('ModelNet voxel_size (None in every shipped config)')
    if d.get('keep_ratio') is None:
        raise NotImplementedError('ModelNet keep_ratio=None (0.7 in every shipped config)')
    for k in ('min_overlap', 'max_overlap', 'overfitting_index'):
        if d.get(k) is not None:
            raise NotImplementedError(f'ModelNet {k} (None in every shipped config)')
    for k in ('estimate_normal', 'return_normals'):
        if d.get(k, False):
            raise NotImplementedError(f'ModelNet {k} (off in every shipped val / test loader)')
    if cfg.test.get('noise_magnitude') is None:
        raise NotImplementedError('ModelNet test.noise_magnitude=None (0.05 in every shipped config)')


class ModelNetPairs:
    """The val or test split of ModelNet as the reference's deterministic dataset makes it: ``len(pairs)`` pairs, pair i built
    from the i-th shape of ``{root}/{subset}.pkl`` whose label passes the class filter, with the stream seeded by i.

    ``pairs[i]`` is a dict of device tensors ``ref_points`` / ``src_points`` (num_points, 3), ``ref_feats`` / ``src_feats``
    (ones), ``transform`` (4, 4) and the ints ``label`` and ``index``; ``chunks()`` yields them as lists of up to ``chunk_size``.
    Indexing builds (once) the chunk that holds the pair, so a sequential pass builds every pair once.  ``data_list`` stands in for
    the pkl's list of ``{'points', 'normals', 'label'}`` when given."""

    def __init__(self, root, subset, cfg, device='cuda', chunk_size=256, data_list=None):
        if subset not in ('train', 'val', 'test'):
            raise ValueError(f"subset must be 'train', 'val' or 'test', got {subset!r}")
        check_options(cfg)
        self.cfg = cfg
        self.device = torch.device(device)
        if self.device.type == 'cuda' and self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        self.chunk_size = int(chunk_size)
        if self.chunk_size < 1:
            raise ValueError('chunk_size must be positive')
        self.class_indices = get_class_indices(cfg.test.class_indices, cfg.data.asymmetric)
        if data_list is None:
            with open(os.path.join(root, f'{subset}.pkl'), 'rb') as f:
                data_list = pickle.load(f)
        self.data_list = [x for x in data_list if x['label'] in self.class_indices]
        self._chunk = (None, None)

    def __len__(self):
        return len(self.data_list)

    def build(self, start, stop):
        """the pairs start .. stop-1 as a list of dicts, built in one call"""
        if not 0 <= start < stop <= len(self):
            raise IndexError(f'pairs {start}..{stop} of {len(self)}')
        d, m = self.cfg.data, self.cfg.data.num_points
        shapes = [torch.from_numpy(np.ascontiguousarray(x['points'], dtype=np.float32)) for x in self.data_list[start:stop]]
        lengths = [int(s.shape[0]) for s in shapes]
        raw = _stack_to_device(shapes, self.device)
        points, _, T, _ = GF.modelnet_benchmark_pairs_batched(raw, lengths, range(start, stop), m, d.keep_ratio, d.rotation_magnitude,
                                                              d.translation_magnitude, self.cfg.test.noise_magnitude)
        B = stop - start
        ones = torch.ones((m, 1), dtype=torch.float32, device=self.device)
        # the engines read their inputs on worker streams that do not wait for this one: the chunk is complete on return
        torch.cuda.current_stream(self.device).synchronize()
        return [{'ref_points': points[p * m:(p + 1) * m], 'src_points': points[(B + p) * m:(B + p + 1) * m], 'ref_feats': ones,
                 'src_feats': ones, 'transform': T[p], 'label': int(self.data_list[start + p]['label']), 'index': start + p}
                for p in range(B)]

    def chunks(self):
        for start in range(0, len(self), self.chunk_size):
            yield self.build(start, min(len(self), start + self.chunk_size))

    def __getitem__(self, i):
        if not -len(self) <= i < len(self):
            raise IndexError(i)
        i %= len(self)
        start = i - i % self.chunk_size
        if self._chunk[0] != start:
            self._chunk = (start, self.build(start, min(len(self), start + self.chunk_size)))
        return self._chunk[1][i - start]
