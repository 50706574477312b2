"""Training-data augmentation on the device, in front of the stack-mode collate.

The reference augments every training pair in its DataLoader workers, in numpy at float64 (``datasets/registration/threedmatch/
dataset.py:60-88``, ``kitti/dataset.py:57-92``, ``modelnet/dataset.py:120-240``).  Here the raw pair goes to the device in one
stacked copy, as the plain collate sends it, and ``functional.augment_pairs_batched`` / ``functional.modelnet_pairs_batched`` write
the augmented clouds straight into the collate's input.  Every draw comes from Philox streams keyed by (seed, iteration, pair), so
a resumed run draws the augmented pairs an uninterrupted run would, and no step waits for the device before the collate's own
read-back.
"""
import numpy as np
import torch

from . import functional as GF
from .utils.data import _stack_to_device, precompute_data_stack_mode

_RAW_KEYS = ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform', 'points', 'normals')


def _t(v):
    return torch.from_numpy(v) if isinstance(v, np.ndarray) else v


def check_options(cfg):
    """NotImplementedError for the reference's switches that no shipped experiment turns on"""
    tr, data = cfg.get('train', {}), cfg.get('data', {})
    if cfg.name == 'modelnet':
        if data.get('crop_method', 'plane') != 'plane':
            raise NotImplementedError("ModelNet crop_method='point' (every shipped config crops with a plane)")
        if not data.get('twice_sample', True):
            raise NotImplementedError('ModelNet twice_sample=False (True in every shipped config)')
        if data.get('twice_transform', False):
            raise NotImplementedError('ModelNet twice_transform=True (False in every shipped config)')
        if data.get('voxel_size') is not None:
            raise NotImplementedError('ModelNet voxel_size (None in every shipped config)')
        for k in ('min_overlap', 'max_overlap'):
            if data.get(k) is not None:
                raise NotImplementedError(f'ModelNet {k} (None in every shipped config)')
        for k in ('estimate_normal', 'return_normals'):
            if data.get(k, False):
                raise NotImplementedError(f'ModelNet {k} (off in every shipped config)')
    else:
        if not tr.get('use_augmentation', True):
            raise NotImplementedError('use_augmentation=False: train on the pairs as given (TrainingEngine(augment=False))')
        if tr.get('rotated', False):
            raise NotImplementedError('3DMatch rotated=True (off in every shipped training config)')


def augment_stacked(pairs, cfg, seed, iteration, device, pair_base=0):
    """the augmented clouds of ``pairs`` on the device: (points stacked [ref..., src...], lengths_host, transforms (B, 4, 4), origin,
    record), from ``functional.augment_pairs_batched`` (3DMatch, KITTI) or ``functional.modelnet_pairs_batched`` (ModelNet).  Pair p
    draws from the streams (seed, iteration, pair_base + p)."""
    check_options(cfg)
    if cfg.name == 'modelnet':
        shapes = [_t(d['points']) for d in pairs]
        lengths = [int(s.shape[0]) for s in shapes]
        raw = _stack_to_device([s.float() for s in shapes], device)
        d, tr = cfg.data, cfg.train
        return GF.modelnet_pairs_batched(raw, lengths, d.num_points, d.keep_ratio, d.rotation_magnitude, d.translation_magnitude,
                                         tr.noise_magnitude, seed, iteration, pair_base)
    clouds = [_t(d['ref_points']) for d in pairs] + [_t(d['src_points']) for d in pairs]
    lengths = [int(c.shape[0]) for c in clouds]
    raw = _stack_to_device([c.float() for c in clouds], device)
    T = torch.stack([_t(d['transform']).float().reshape(4, 4) for d in pairs]).to(device, non_blocking=True)
    tr = cfg.train
    if cfg.name == 'kitti':
        return GF.augment_pairs_batched(raw, lengths, T, GF.AUGMENT_KITTI, tr.point_limit, tr.augmentation_noise, tr.augmentation_rotation,
                                        tr.augmentation_min_scale, tr.augmentation_max_scale, tr.augmentation_shift, seed, iteration,
                                        pair_base)
    return GF.augment_pairs_batched(raw, lengths, T, GF.AUGMENT_3DMATCH, tr.point_limit, tr.augmentation_noise, tr.augmentation_rotation,
                                    seed=seed, iteration=iteration, pair_base=pair_base)


def augmented_collate(pairs, cfg, neighbor_limits, seed, iteration, device='cuda'):
    """``registration_collate_fn_stack_mode`` of the augmented ``pairs``: the reference's training pipeline of ``cfg.name`` (point
    limit, rotation, noise, and for KITTI scale and shift; for ModelNet the pair synthesis from a raw shape ``{'points': (N, 3)}``)
    on the device, then the multi-level precompute on its output.  ``features`` are ones, as every reference dataset makes them;
    ``transform`` is the augmented ground truth, (4, 4) for one pair and (B, 4, 4) for more."""
    pairs = list(pairs)
    B = len(pairs)
    if B < 1:
        raise ValueError('augmented_collate: no pairs')
    device = torch.device(device)
    if device.type == 'cuda' and device.index is None:
        device = torch.device('cuda', torch.cuda.current_device())
    points, lengths, T, _, _ = augment_stacked(pairs, cfg, seed, iteration, device)
    collated = {}
    for d in pairs:
        for key, value in d.items():
            if key not in _RAW_KEYS:
                collated.setdefault(key, []).append(_t(value))
    if B == 1:
        collated = {k: v[0] for k, v in collated.items()}
    collated = {k: (v.to(device, non_blocking=True) if isinstance(v, torch.Tensor) else v) for k, v in collated.items()}
    collated['transform'] = T[0] if B == 1 else T
    collated['features'] = torch.ones((points.shape[0], 1), dtype=torch.float32, device=device)
    b = cfg.backbone
    collated.update(precompute_data_stack_mode(points, torch.LongTensor(lengths), b.num_stages, b.init_voxel_size, b.init_radius,
                                               neighbor_limits))
    collated['batch_size'] = B
    return collated
