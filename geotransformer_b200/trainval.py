"""Training with validation from the dataset files, the experiments' ``trainval.py`` with ``EpochBasedTrainer``.

    python -m geotransformer_b200.trainval --config {3dmatch,kitti,modelnet} --dataset-root DIR --output-dir DIR
        [--batch-size B] [--resume] [--seed S] [--max-epoch E]

A fresh run seeds torch with ``--seed``, builds the model with PyTorch's default initialisation and gives every KPConv its kernel
points (``initialize_kernel_points``).  The neighbour limits are calibrated on the augmented training set and logged.  Every epoch
trains on the ``PrefetchLoader``'s steps of B pairs (order keyed by (seed, epoch); augmentation keyed by (seed, iteration, pair) on
the device), validates through ``TrainingEngine.validate`` and writes ``snapshots/epoch-{e}.pth.tar`` (epoch, iteration, model) and
``snapshots/snapshot.pth.tar`` (plus optimizer and scheduler), as the reference's trainer does.  ``--resume`` continues from
``snapshots/snapshot.pth.tar``; the pairs and draws of the remaining epochs are those an uninterrupted run would use.

3DMatch and KITTI train on ``{root}/metadata/train.pkl`` and validate on ``val.pkl``; ModelNet trains on the raw shapes of
``{root}/train.pkl`` and validates on ``ModelNetPairs(root, 'val')``.  For ModelNet an epoch is one pass over the training shapes,
and training stops once ``cfg.optim.max_iteration`` steps are done (the reference's iteration-based trainer; its warm-up cosine
schedule steps every iteration).
"""
import argparse
import math
import os
import pickle
import time

import numpy as np
import torch

from .config import make_cfg
from .datasets.loader import PrefetchLoader
from .train import LOSS_KEYS, MAX_BATCH, TrainingEngine

VAL_CHUNK = 64


def _log(path, message):
    print(message, flush=True)
    with open(path, 'a') as f:
        f.write(message + '\n')


def log_string(result, epoch=None, max_epoch=None, iteration=None, max_iteration=None, lr=None):
    """the reference's get_log_string (utils/common.py:46-71): 'Epoch: e/E, iter: i/I, key: value, ..., lr: x'"""
    parts = []
    if epoch is not None:
        parts.append(f'Epoch: {epoch}' + (f'/{max_epoch}' if max_epoch is not None else ''))
    if iteration is not None:
        s = f'iter: {iteration}' + (f'/{max_iteration}' if max_iteration is not None else '')
        parts.append(s if epoch is not None else s.capitalize())
    for k, v in result.items():
        parts.append(f'{k}: {v:d}' if isinstance(v, int) else f'{k}: {v:.3f}')
    if lr is not None:
        parts.append(f'lr: {lr:.3e}')
    return ', '.join(parts)


def training_set(cfg, root):
    """the training pairs of ``cfg.name`` read from ``root`` (raw shapes for ModelNet)"""
    if cfg.name == '3dmatch':
        from .datasets.threedmatch import ThreeDMatchPairs
        return ThreeDMatchPairs(root, 'train')
    if cfg.name == 'kitti':
        from .datasets.kitti import KittiPairs
        return KittiPairs(root, 'train')
    from .datasets.modelnet import get_class_indices
    with open(os.path.join(root, 'train.pkl'), 'rb') as f:
        shapes = pickle.load(f)
    keep = get_class_indices(cfg.train.class_indices, cfg.data.asymmetric)
    return [{'points': np.asarray(x['points'], dtype=np.float32)} for x in shapes if x['label'] in keep]


def validation_set(cfg, root):
    if cfg.name == '3dmatch':
        from .datasets.threedmatch import ThreeDMatchPairs
        return ThreeDMatchPairs(root, 'val')
    if cfg.name == 'kitti':
        from .datasets.kitti import KittiPairs
        return KittiPairs(root, 'val')
    from .datasets.modelnet import ModelNetPairs
    return ModelNetPairs(root, 'val', cfg)


def build_model(cfg, seed, device):
    """a fresh model: PyTorch's default initialisation under ``torch.manual_seed(seed)``, then the reference's kernel points"""
    from .model import create_model
    from .modules.kpconv import initialize_kernel_points
    torch.manual_seed(seed)
    model = create_model(cfg).to(device)
    initialize_kernel_points(model, seed)
    return model


def _tensors(item):
    return {k: v for k, v in item.items() if isinstance(v, (np.ndarray, torch.Tensor))}


def validate(engine, dataset):
    """the means of the reference's val_step results (losses and Evaluator metrics) over ``dataset``, a chunk of pairs at a time"""
    sums, n = {}, 0
    for start in range(0, len(dataset), VAL_CHUNK):
        chunk = [_tensors(dataset[i]) for i in range(start, min(len(dataset), start + VAL_CHUNK))]
        for res in engine.validate(chunk):
            for k, v in list(res.get('loss', {}).items()) + list(res['metrics'].items()):
                sums[k] = sums.get(k, 0.0) + float(v)
            n += 1
    return {k: v / max(n, 1) for k, v in sums.items()}


def run(config, dataset_root, output_dir, batch_size=1, resume=False, seed=None, max_epoch=None, num_threads=4, log_steps=10):
    """the training loop of the module docstring; returns the engine after the last epoch"""
    from .utils.data import calibrate_neighbors_augmented
    cfg = make_cfg(config)
    seed = int(cfg.seed if seed is None else seed)
    if not 1 <= batch_size <= MAX_BATCH:
        raise ValueError(f'--batch-size must be in 1..{MAX_BATCH}')
    device = torch.device('cuda', torch.cuda.current_device())
    snap_dir = os.path.join(output_dir, 'snapshots')
    os.makedirs(snap_dir, exist_ok=True)
    log_file = os.path.join(output_dir, 'train.log')
    train_set, val_set = training_set(cfg, dataset_root), validation_set(cfg, dataset_root)

    model = build_model(cfg, seed, device)
    limits, used = calibrate_neighbors_augmented(train_set, cfg, seed)
    limits = [int(x) for x in limits]
    _log(log_file, f'Calibrate neighbors: {limits} (from {used} augmented training pairs).')

    engine = TrainingEngine(model, cfg, limits, seed=seed, device=device, batch_size=batch_size, augment=True)
    if resume:
        path = os.path.join(snap_dir, 'snapshot.pth.tar')
        engine.load_snapshot(path)
        _log(log_file, f'Snapshot loaded from "{path}" (epoch {engine.epoch}, iteration {engine.iteration}).')
    loader = PrefetchLoader(train_set, batch_size, seed, num_threads=num_threads)
    steps = len(loader)
    if cfg.name == 'modelnet':
        max_iteration = int(cfg.optim.max_iteration)
        epochs = math.ceil(max_iteration / steps) if max_epoch is None else int(max_epoch)
    else:
        max_iteration = None
        epochs = int(cfg.optim.max_epoch if max_epoch is None else max_epoch)

    while engine.epoch < epochs and (max_iteration is None or engine.iteration < max_iteration):
        epoch = engine.epoch + 1
        left = steps if max_iteration is None else min(steps, max_iteration - engine.iteration)
        groups = (g for i, g in zip(range(left), loader.epoch(epoch)))
        t0 = time.perf_counter()
        step = [0]

        def log_step(res):
            step[0] += 1
            if step[0] % log_steps == 0 or step[0] == left:
                shown = {k: res[k] for k in LOSS_KEYS}
                shown.update({k: v for k, v in res.items() if k not in LOSS_KEYS and isinstance(v, float) and k != 'lr'})
                _log(log_file, log_string(shown, epoch, epochs, step[0], steps, lr=res['lr']))
        engine.train_groups(groups, log=log_step)
        _log(log_file, f'Epoch {epoch} trained in {time.perf_counter() - t0:.1f}s, iteration {engine.iteration}.')
        _log(log_file, '[Val] ' + log_string(validate(engine, val_set), epoch))
        state = {'epoch': engine.epoch, 'iteration': engine.iteration, 'model': model.state_dict()}
        torch.save(state, os.path.join(snap_dir, f'epoch-{engine.epoch}.pth.tar'))
        engine.save_snapshot(os.path.join(snap_dir, 'snapshot.pth.tar'))
    return engine


def make_parser():
    p = argparse.ArgumentParser(prog='python -m geotransformer_b200.trainval', description=__doc__.split('\n\n')[0])
    p.add_argument('--config', choices=['3dmatch', 'kitti', 'modelnet'], required=True)
    p.add_argument('--dataset-root', required=True, help="the reference's dataset directory of the config")
    p.add_argument('--output-dir', required=True, help='snapshots/ and train.log go here')
    p.add_argument('--batch-size', type=int, default=1, help=f'pairs per optimisation step (1..{MAX_BATCH})')
    p.add_argument('--resume', action='store_true', help='continue from <output-dir>/snapshots/snapshot.pth.tar')
    p.add_argument('--seed', type=int, default=None, help='model initialisation, data order and augmentation (default cfg.seed)')
    p.add_argument('--max-epoch', type=int, default=None, help="epochs to train (default the config's max_epoch)")
    return p


def main(argv=None):
    a = make_parser().parse_args(argv)
    run(a.config, a.dataset_root, a.output_dir, batch_size=a.batch_size, resume=a.resume, seed=a.seed, max_epoch=a.max_epoch)


if __name__ == '__main__':
    main()
