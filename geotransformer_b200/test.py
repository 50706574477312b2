"""Testing a snapshot on a benchmark from the dataset files, the experiments' ``test.py``.

    python -m geotransformer_b200.test --config 3dmatch --benchmark {3DMatch,3DLoMatch} --snapshot FILE --dataset-root DIR \\
        --output-dir DIR [--neighbor-limits calibrate|config] [--seed S] [--rotated]
    python -m geotransformer_b200.test --config kitti --snapshot FILE --dataset-root DIR --output-dir DIR
    python -m geotransformer_b200.test --config modelnet --snapshot FILE --dataset-root DIR --output-dir DIR [--rpmnet-metrics]

``RegistrationTester`` runs the model over the benchmark's pairs and logs the reference's per-pair and summary lines.  3DMatch
writes ``<output-dir>/features/<benchmark>/<scene>/<ref>_<src>.npz`` and KITTI ``<output-dir>/features/<seq>_<src>_<ref>.npz``, the
tree ``python -m geotransformer_b200.evaluate --features <output-dir>/features`` reads; ModelNet reports the metrics only, as the
reference's ModelNet ``test.py`` does.  By default the neighbour limits are calibrated on the augmented training set, as the
reference's ``test_data_loader`` does; ``--neighbor-limits config`` takes the config's limits instead (3DMatch only).
``--rotated`` (3DMatch only) tests on the rotated benchmark: pair i's clouds get the rotations drawn from ``np.random.seed(i)``, and
the ``.npz`` files hold the rotated points and transform; score them with ``evaluate --protocol dgr``, since gt.log is in the frame
of the un-rotated fragments.  ``--rpmnet-metrics`` (ModelNet only) also scores every pair with RPMNet's metrics (modified Chamfer
distance, anisotropic rotation and translation MSE / MAE) and logs their means as ``rpmnet_<name>``.
"""
import argparse
import os

import torch

from .config import make_cfg
from .trainval import _log, log_string, training_set


def benchmark_set(cfg, root, benchmark, rotated=False):
    if rotated and cfg.name != '3dmatch':
        raise ValueError('--rotated is a 3dmatch benchmark')
    if cfg.name == '3dmatch':
        from .datasets.threedmatch import ThreeDMatchPairs
        if benchmark not in ('3DMatch', '3DLoMatch'):
            raise ValueError("--benchmark must be '3DMatch' or '3DLoMatch' for 3dmatch")
        return ThreeDMatchPairs(root, benchmark, rotated=rotated)
    if cfg.name == 'kitti':
        from .datasets.kitti import KittiPairs
        return KittiPairs(root, 'test')
    from .datasets.modelnet import ModelNetPairs
    return ModelNetPairs(root, 'test', cfg)


def run(config, snapshot, dataset_root, output_dir, benchmark=None, neighbor_limits='calibrate', seed=None, rotated=False,
        rpmnet_metrics=False):
    """the test of the module docstring; returns (summary, per-pair results)"""
    from .model import create_model
    from .tester import RegistrationTester
    from .utils.data import calibrate_neighbors_augmented
    cfg = make_cfg(config)
    if rpmnet_metrics and cfg.name != 'modelnet':
        raise ValueError('--rpmnet-metrics is a modelnet benchmark')
    seed = int(cfg.seed if seed is None else seed)
    device = torch.device('cuda', torch.cuda.current_device())
    os.makedirs(output_dir, exist_ok=True)
    log_file = os.path.join(output_dir, 'test.log')
    test_set = benchmark_set(cfg, dataset_root, benchmark, rotated=rotated)
    if neighbor_limits == 'calibrate':
        limits, used = calibrate_neighbors_augmented(training_set(cfg, dataset_root), cfg, seed)
        limits = [int(x) for x in limits]
        _log(log_file, f'Calibrate neighbors: {limits} (from {used} augmented training pairs).')
    elif neighbor_limits == 'config':
        if cfg.neighbor_limits is None:
            raise ValueError(f'config {config} has no fixed neighbor limits: use --neighbor-limits calibrate')
        limits = list(cfg.neighbor_limits)
    else:
        raise ValueError("--neighbor-limits must be 'calibrate' or 'config'")
    model = create_model(cfg).to(device)
    state = torch.load(snapshot, map_location='cpu', weights_only=False)
    model.load_state_dict(state['model'], strict=True)
    model.eval()
    _log(log_file, f'Model loaded from "{snapshot}".')
    if cfg.name == 'modelnet':
        feature_dir, layout = None, '3dmatch'
    else:
        feature_dir = os.path.join(output_dir, 'features', benchmark) if cfg.name == '3dmatch' else os.path.join(output_dir, 'features')
        layout = cfg.name
    tester = RegistrationTester(cfg, model, limits, output_dir=feature_dir, device=device, layout=layout, rpmnet_metrics=rpmnet_metrics)
    try:
        summary, per_pair = tester.run(test_set, log=lambda m: _log(log_file, m))
    finally:
        tester.close()
    _log(log_file, log_string(summary))
    return summary, per_pair


def make_parser():
    p = argparse.ArgumentParser(prog='python -m geotransformer_b200.test', description=__doc__.split('\n\n')[0])
    p.add_argument('--config', choices=['3dmatch', 'kitti', 'modelnet'], required=True)
    p.add_argument('--benchmark', choices=['3DMatch', '3DLoMatch'], default=None, help='3dmatch only')
    p.add_argument('--snapshot', required=True, help='a snapshot of trainval (or the reference) holding "model"')
    p.add_argument('--dataset-root', required=True)
    p.add_argument('--output-dir', required=True)
    p.add_argument('--neighbor-limits', choices=['calibrate', 'config'], default='calibrate')
    p.add_argument('--seed', type=int, default=None, help='seed of the calibration draws (default cfg.seed)')
    p.add_argument('--rotated', action='store_true', help='3dmatch only: the rotated benchmark (pair i rotated from np.random.seed(i))')
    p.add_argument('--rpmnet-metrics', action='store_true',
                   help="modelnet only: also report RPMNet's metrics (Chamfer distance, anisotropic MSE / MAE) as rpmnet_<name>")
    return p


def main(argv=None):
    a = make_parser().parse_args(argv)
    if a.rotated and a.config != '3dmatch':
        make_parser().error('--rotated is a 3dmatch benchmark')
    if a.rpmnet_metrics and a.config != 'modelnet':
        raise ValueError('--rpmnet-metrics is a modelnet benchmark')
    run(a.config, a.snapshot, a.dataset_root, a.output_dir, benchmark=a.benchmark, neighbor_limits=a.neighbor_limits, seed=a.seed,
        rotated=a.rotated, rpmnet_metrics=a.rpmnet_metrics)


if __name__ == '__main__':
    main()
