"""Test-time loop over a dataset of pairs (SURVEY.md section 8f next #2).

Reference: ``geotransformer/engine/single_tester.py:39-74`` (the loop: to_cuda -> test_step -> eval_step -> after_test_step ->
summary) and ``experiments/*/test.py:40-92`` (test_step = model forward, eval_step = Evaluator, after_test_step = one
``<output_dir>/<scene_name>/<ref_frame>_<src_frame>.npz`` per pair with the arrays ``eval.py`` consumes).  Differences: the
collate runs on the GPU in this process (CUDA cannot be used in forked DataLoader workers), ``num_streams`` pairs are in
flight at once (`RegistrationEngine`), and the six metrics come from one device kernel per pair.
"""
import os

import numpy as np
import torch

from .engine import RegistrationEngine
from .loss import Evaluator, OverallLoss

# arrays written per pair, in the order of experiments/geotransformer.3dmatch.*/test.py:73-92
NPZ_OUTPUT_KEYS = ('ref_points', 'src_points', 'ref_points_f', 'src_points_f', 'ref_points_c', 'src_points_c', 'ref_feats_c',
                   'src_feats_c', 'ref_node_corr_indices', 'src_node_corr_indices', 'ref_corr_points', 'src_corr_points',
                   'corr_scores', 'gt_node_corr_indices', 'gt_node_corr_overlaps', 'estimated_transform')
METRICS = ('PIR', 'IR', 'RRE', 'RTE', 'RMSE', 'RR')
LOSSES = ('loss', 'c_loss', 'f_loss')
RPMNET = ('CD', 'r_mse', 'r_mae', 't_mse', 't_mae')


def _np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


class RegistrationTester:
    def __init__(self, cfg, model, neighbor_limits, output_dir=None, num_streams=4, chunk=16, device=None, batch_size=1, with_loss=False,
                 with_ransac=False, layout='3dmatch', rpmnet_metrics=False):
        """batch_size > 1: that many pairs per forward (GeoTransformer.forward_batch) on each of the num_streams lanes.
        with_loss: also report the validation losses loss / c_loss / f_loss (OverallLoss) per pair and as means in the summary,
        as the reference's val_step does (trainval.py: loss_dict.update(result_dict)).
        with_ransac: also run correspondence RANSAC (cfg.ransac) on every pair's correspondences; each entry gains 'ransac'
        (transform, fitness, inlier_rmse, metrics of the RANSAC transform) and the summary the means as ransac_<name>.
        layout: '3dmatch' writes <output_dir>/<scene_name>/<ref_frame>_<src_frame>.npz with 'overlap' (3DMatch test.py); 'kitti'
        writes <output_dir>/<seq_id>_<src_frame>_<ref_frame>.npz without it (KITTI test.py:60-85).
        rpmnet_metrics (ModelNet only): also score every pair with RPMNet's metrics (``functional.rpmnet_metrics_batched``, one call
        per 32 pairs, on the items' ``raw_points`` / ``ref_points`` / ``src_points`` / ``transform`` and the estimate); each entry
        gains 'rpmnet' {CD, r_mse, r_mae, t_mse, t_mae} and the summary their means as rpmnet_<name>"""
        if layout not in ('3dmatch', 'kitti'):
            raise ValueError(f"layout must be '3dmatch' or 'kitti', got {layout!r}")
        if rpmnet_metrics and cfg.name != 'modelnet':
            raise ValueError(f'rpmnet_metrics is a modelnet benchmark, got config {cfg.name!r}')
        self.rpmnet_metrics = bool(rpmnet_metrics)
        self.layout = layout
        self.cfg, self.output_dir, self.chunk = cfg, output_dir, max(1, int(chunk), int(batch_size) * int(num_streams))
        self.with_loss = bool(with_loss)
        self.with_ransac = bool(with_ransac)
        self.engine = RegistrationEngine(model, cfg, neighbor_limits, num_streams=num_streams, device=device, evaluator=Evaluator(cfg),
                                         batch_size=batch_size, loss_func=OverallLoss(cfg) if self.with_loss else None,
                                         ransac=cfg.ransac if self.with_ransac else None)

    def after_test_step(self, data_dict, output_dict):
        """experiments/*/test.py:65-92"""
        ref_id, src_id = data_dict.get('ref_frame', 0), data_dict.get('src_frame', 1)
        arrays = {k: _np(output_dict[k]) for k in NPZ_OUTPUT_KEYS}
        arrays['transform'] = _np(data_dict['transform'])
        if self.layout == 'kitti':
            os.makedirs(self.output_dir, exist_ok=True)
            path = os.path.join(self.output_dir, f"{data_dict.get('seq_id', 0)}_{src_id}_{ref_id}.npz")
            np.savez_compressed(path, **arrays)
            return path
        scene = data_dict.get('scene_name', 'scene')
        os.makedirs(os.path.join(self.output_dir, str(scene)), exist_ok=True)
        arrays['overlap'] = data_dict.get('overlap', np.float32('nan'))
        path = os.path.join(self.output_dir, str(scene), f'{ref_id}_{src_id}.npz')
        np.savez_compressed(path, **arrays)
        return path

    def run(self, dataset, log=None):
        """dataset: indexable of dicts with ref_points/src_points/ref_feats/src_feats/transform (+ scene_name, ref_frame,
        src_frame, overlap as the reference datasets provide).  A rotated ``ThreeDMatchPairs`` builds each chunk on the device with
        ``rotated_batch``, which the engine takes without a copy through the host.  Returns (summary of mean metrics, per-pair
        results)."""
        per_pair = []
        n = len(dataset)
        device_chunk = getattr(dataset, 'rotated_batch', None) if getattr(dataset, 'rotated', False) else None
        for base in range(0, n, self.chunk):
            stop = min(n, base + self.chunk)
            if device_chunk is not None:
                items = device_chunk(range(base, stop), device=self.engine.device)
            else:
                items = [dataset[i] for i in range(base, stop)]
            tensors = [{k: v for k, v in it.items() if isinstance(v, (np.ndarray, torch.Tensor)) and k != 'raw_points'} for it in items]
            results = self.engine.register(tensors, keep_outputs=self.output_dir is not None)
            scores = self._rpmnet(items, results) if self.rpmnet_metrics else None
            for j, (it, res) in enumerate(zip(items, results)):
                entry = {'metrics': res['metrics'], 'num_corr': res['num_corr'], 'estimated_transform': res['estimated_transform']}
                if self.with_loss:
                    entry.update(res['loss'])
                if self.with_ransac:
                    entry['ransac'] = res['ransac']
                if scores is not None:
                    entry['rpmnet'] = scores[j]
                if self.output_dir is not None:
                    entry['file'] = self.after_test_step(it, res.pop('output_dict'))
                per_pair.append(entry)
                if log is not None:       # single_tester.py:62-66 / test.py:55-63 summary string
                    msg = ', '.join(f'{k}: {res["metrics"][k]:.3f}' for k in METRICS)
                    log(f"{it.get('scene_name', 'scene')}, id0: {it.get('ref_frame', 0)}, id1: {it.get('src_frame', 1)}, {msg}, "
                        f"nCorr: {res['num_corr']}" + (''.join(f", {k}: {res['loss'][k]:.3f}" for k in LOSSES) if self.with_loss else '')
                        + (''.join(f", {k}: {scores[j][k]:.6f}" for k in RPMNET) if scores is not None else ''))
        summary = {k: float(np.mean([p['metrics'][k] for p in per_pair])) for k in METRICS} if per_pair else {}
        if self.with_loss and per_pair:
            summary.update({k: float(np.mean([p[k] for p in per_pair])) for k in LOSSES})
        if self.with_ransac and per_pair:
            summary.update({f'ransac_{k}': float(np.mean([p['ransac']['metrics'][k] for p in per_pair])) for k in METRICS})
            summary.update({f'ransac_{k}': float(np.mean([p['ransac'][k] for p in per_pair])) for k in ('fitness', 'inlier_rmse')})
        if self.rpmnet_metrics and per_pair:
            summary.update({f'rpmnet_{k}': float(np.mean([p['rpmnet'][k] for p in per_pair])) for k in RPMNET})
        return summary, per_pair

    def _rpmnet(self, items, results):
        """RPMNet's metrics of a chunk: one device call per 32 pairs, one read-back each"""
        from . import functional as GF
        dev = self.engine.device
        out = []
        for b in range(0, len(items), GF.RPMNET_MAX_PAIRS):
            its, res = items[b:b + GF.RPMNET_MAX_PAIRS], results[b:b + GF.RPMNET_MAX_PAIRS]
            if any('raw_points' not in it for it in its):
                raise ValueError('rpmnet_metrics needs items with raw_points (datasets.modelnet.ModelNetPairs)')
            clouds = {k: [torch.as_tensor(it[k], dtype=torch.float32).to(dev) for it in its] for k in ('raw_points', 'ref_points', 'src_points')}
            gt = torch.stack([torch.as_tensor(it['transform'], dtype=torch.float32).to(dev) for it in its])
            est = torch.stack([r['estimated_transform'] for r in res]).to(dev, torch.float32)
            m = GF.rpmnet_metrics_batched(*(x for k in ('raw_points', 'ref_points', 'src_points')
                                            for x in (torch.cat(clouds[k]).contiguous(), [c.shape[0] for c in clouds[k]])),
                                          gt, est).cpu().numpy()
            out.extend({k: float(row[GF.RPMNET_COLUMNS.index(k)]) for k in RPMNET} for row in m)
        return out

    def close(self):
        self.engine.close()
