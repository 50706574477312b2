"""The benchmark evaluation of the experiments' ``eval.py`` (3DMatch / 3DLoMatch and KITTI) with the per-pair stages on the device.

    python -m geotransformer_b200.evaluate --config 3dmatch --benchmark 3DMatch --method lgr \\
        --features FEATURES --gt-root METADATA/benchmarks --registration-dir OUT [--num_corr 250,500,1000,2500,5000] [--verbose]
    python -m geotransformer_b200.evaluate --config kitti --method ransac --features FEATURES [--num_corr 5000]
    python -m geotransformer_b200.evaluate --config 3dmatch --benchmark 3DMatch --method lgr --features FEATURES --protocol dgr \\
        [--test-epoch E] [--num_corr 1000]

It reads the ``.npz`` tree ``test.py`` (or ``RegistrationTester``) writes: 3DMatch ``<features>/<benchmark>/<scene>/<ref>_<src>.npz``,
KITTI ``<features>/<seq>_<src>_<ref>.npz``, in the order ``eval.py`` visits them.  Per chunk of pairs the arrays are packed into one
pinned buffer and copied to the device once; the top-k selection (``--num_corr``), the sparse coarse precision, the correspondence
metrics, the estimator (``lgr``: the stored transform, ``ransac``: correspondence RANSAC, ``svd``: weighted Procrustes) and the
registration error run there for the whole chunk, and one copy brings the per-pair rows back.  The meters and log lines are the
reference's, on the host.  ``--gt-root`` is the directory holding ``<benchmark>/<scene>/gt.log`` and ``gt.info``; with
``--registration-dir`` each scene's estimates go to ``<dir>/<benchmark>/<scene>/est.log`` (``<dir>/num_corr_<k>/...`` per setting
of a sweep).

``--protocol dgr`` (3dmatch) is the experiments' ``eval_dgr.py`` instead: a pair is accepted when its RRE and RTE against the
npz ``transform`` are under ``cfg.eval.rre_threshold`` / ``rte_threshold``, so it needs no ``--gt-root`` and writes no est.log.
It is the protocol that can score the rotated benchmark (``test --rotated``), whose transforms are not gt.log's.  Its meters and
lines are eval_dgr's, quirks included: a scene's RRE / RTE average its accepted pairs only and are NaN without one, the NaN reaches
``mean_RRE`` / ``mean_RTE``, and the summary opens with ``Epoch {--test-epoch}``.  It reads the same ``<features>/<benchmark>/<scene>``
layout as ``gtlog``.  Scoring a rotated tree with ``gtlog`` is meaningless: gt.log holds the un-rotated fragments' transforms.

A sweep ``--num_corr 250,500`` orders each pair's correspondences once and selects once per setting; its results equal separate
runs.  Where this differs from ``eval.py`` (DESIGN.md section 3b): ``--num_corr`` works for 3DMatch too (the reference's 3DMatch
script raises NameError there), rows with tied scores at the selection boundary go by row index, and RANSAC draws from its own
counter-based sampler keyed by ``cfg.ransac.seed`` and the pair's position in the benchmark.
"""
import argparse
import glob
import logging
import os
import sys
import warnings

import numpy as np
import torch

from . import functional as GF
from .config import make_cfg
from .datasets.threedmatch_utils import get_gt_logs_and_infos, get_num_fragments, get_scene_abbr, write_log_file

_LOG = logging.getLogger('geotransformer_b200.evaluate')
INFO, CRITICAL = logging.INFO, logging.CRITICAL


class AverageMeter:
    """Records of Python floats; mean / median / std as numpy takes them (NaN for no record)."""

    def __init__(self):
        self.records = []

    def update(self, value):
        self.records.append(value)

    def reset(self):
        self.records.clear()

    def _stat(self, fn):
        with warnings.catch_warnings():
            warnings.simplefilter('ignore', RuntimeWarning)
            return float(fn(self.records))

    def mean(self):
        return self._stat(np.mean)

    def median(self):
        return self._stat(np.median)

    def std(self):
        return self._stat(np.std)


def _meters(names):
    return {n: AverageMeter() for n in names}


def _ids(path):
    return [int(x) for x in os.path.splitext(os.path.basename(path))[0].split('_')]


def discover(config, features, benchmark=None):
    """[(scene name or None, [npz path, ...])] in eval.py's order: 3DMatch scenes sorted by name, files by their integer ids."""
    if config == '3dmatch':
        scenes = sorted(glob.glob(os.path.join(features, benchmark, '*')))
        return [(os.path.basename(s), sorted(glob.glob(os.path.join(s, '*.npz')), key=_ids)) for s in scenes]
    return [(None, sorted(glob.glob(os.path.join(features, '*.npz')), key=_ids))]


def parse_num_corr(text):
    """'250,500' -> [250, 500]; None -> [None] (no selection)."""
    if text is None:
        return [None]
    values = [int(v) for v in str(text).split(',') if v.strip()]
    if not values or min(values) < 1 or max(values) > GF.CORR_ORDER_KMAX:
        raise ValueError(f'--num_corr: one or more integers in 1..{GF.CORR_ORDER_KMAX}')
    return values


_TORCH = {np.dtype(np.float32): torch.float32, np.dtype(np.int64): torch.int64, np.dtype(np.int32): torch.int32}


def _upload(arrays, device):
    """One pinned host buffer, one host-to-device copy; device views of the arrays, in order."""
    offsets, total = [], 0
    for a in arrays:
        total = (total + 255) // 256 * 256
        offsets.append(total)
        total += a.nbytes
    host = torch.empty(max(total, 1), dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    for a, o in zip(arrays, offsets):
        hv[o:o + a.nbytes] = a.reshape(-1).view(np.uint8)
    dev = host.to(device, non_blocking=True)
    return [dev[o:o + a.nbytes].view(_TORCH[a.dtype]).view(a.shape) for a, o in zip(arrays, offsets)]


def _ragged(rows, width, dtype):
    cap = max([r.shape[0] for r in rows] + [1])
    out = np.zeros((len(rows), cap) + width, dtype=dtype)
    for i, r in enumerate(rows):
        out[i, :r.shape[0]] = r
    return out, np.array([r.shape[0] for r in rows], dtype=np.int32)


class _Run:
    """Meters, log lines, per-pair values and estimates of one --num_corr setting."""

    def __init__(self, label, log):
        self.label, self.log, self.lines, self.pairs, self.estimates = label, log, [], [], []
        self.coarse = _meters(['precision', 'PMR>0', 'PMR>=0.1', 'PMR>=0.3', 'PMR>=0.5'])
        self.fine = _meters(['recall', 'inlier_ratio', 'overlap'])
        self.reg = _meters(['recall', 'rre', 'rte', 'mean_rre', 'mean_rte', 'median_rre', 'median_rte', 'overall_recall', 'overall_rre',
                            'overall_rte'])
        self.scene_coarse, self.scene_fine, self.scene_reg = {}, {}, {}

    def emit(self, level, message):
        self.lines.append((level, message))
        if self.log is not None:
            self.log(level, message if self.label is None else f'[num_corr={self.label}] {message}')


def _load(path, config, gt, dgr=False):
    d = np.load(path)
    item = {k: d[k] for k in ('ref_points_c', 'src_points_c', 'ref_node_corr_indices', 'src_node_corr_indices', 'ref_corr_points',
                              'src_corr_points', 'corr_scores', 'gt_node_corr_indices', 'transform', 'estimated_transform')}
    item['overlap'] = d['overlap'] if 'overlap' in d.files else np.float32('nan')
    ids = _ids(path)
    if config == '3dmatch' and dgr:                     # --protocol dgr: scored against the npz transform, gt.log is not read
        item['ids'] = ids
        item['has_cov'] = False
        item['reg_gt'] = item['transform']
        item['cov'] = np.zeros((6, 6), np.float32)
    elif config == '3dmatch':
        item['ids'] = ids                                 # ref, src
        gt_indices, gt_logs, gt_infos = gt
        index = gt_indices[ids[0], ids[1]]
        item['has_cov'] = index != -1
        item['reg_gt'] = gt_logs[index]['transform'] if index != -1 else item['transform']
        item['cov'] = gt_infos[index]['covariance'] if index != -1 else np.zeros((6, 6), np.float32)
    else:
        item['ids'] = ids                                 # seq, src, ref
        item['has_cov'] = False
        item['reg_gt'] = item['transform']
        item['cov'] = np.zeros((6, 6), np.float32)
    return item


def _device_rows(items, cfg, method, settings, first_pair, device, rre_rte=False):
    """All device stages of a chunk; one (B, 3 + 24 * settings) float64 host array: sparse eval, then per setting the correspondence
    metrics (4), the estimate (16) and the registration error (4).  rre_rte: accept by RRE / RTE for 3dmatch too (--protocol dgr)."""
    f32 = np.float32
    ref, cnt = _ragged([np.asarray(it['ref_corr_points'], f32).reshape(-1, 3) for it in items], (3,), f32)
    src, _ = _ragged([np.asarray(it['src_corr_points'], f32).reshape(-1, 3) for it in items], (3,), f32)
    sc, _ = _ragged([np.asarray(it['corr_scores'], f32).reshape(-1) for it in items], (), f32)
    nref, pcnt = _ragged([np.asarray(it['ref_node_corr_indices'], np.int64).reshape(-1) for it in items], (), np.int64)
    nsrc, _ = _ragged([np.asarray(it['src_node_corr_indices'], np.int64).reshape(-1) for it in items], (), np.int64)
    gt, gcnt = _ragged([np.asarray(it['gt_node_corr_indices'], np.int64).reshape(-1, 2) for it in items], (2,), np.int64)
    mats = [np.stack([np.asarray(it[k], f32).reshape(-1) for it in items]) for k in ('transform', 'reg_gt', 'estimated_transform', 'cov')]
    has_cov = np.array([it['has_cov'] for it in items], dtype=np.int32)
    (ref, src, sc, cnt, nref, nsrc, pcnt, gt, gcnt, corr_T, reg_T, est_T, cov, has_cov) = _upload(
        [ref, src, sc, cnt, nref, nsrc, pcnt, gt, gcnt] + mats + [has_cov], device)
    m_cap = max(max(it['ref_points_c'].shape[0] for it in items), 1)
    n_cap = max(max(it['src_points_c'].shape[0] for it in items), 1)
    rows = [GF.sparse_correspondence_eval_batched(nref, nsrc, gt, m_cap, n_cap, pred_count=pcnt, gt_count=gcnt)]
    ks = [k for k in settings if k is not None]
    order = GF.corr_order_batched(sc, max(ks), num_corr=cnt) if ks else None
    B = len(items)
    for k in settings:
        r, s, w, c = (ref, src, sc, cnt) if k is None else GF.corr_select_batched(ref, src, sc, order, k, num_corr=cnt)
        metrics = GF.correspondence_metrics_batched(r, s, corr_T, cfg.eval.acceptance_radius, num_corr=c)
        if method == 'lgr':
            T = est_T
        elif method == 'ransac':
            T = GF.ransac_correspondences_batched(s, r, cfg.ransac.distance_threshold, cfg.ransac.num_points, cfg.ransac.num_iterations,
                                                  seed=cfg.ransac.seed, num_corr=c, first_pair=first_pair)['transform'].reshape(B, 16)
        elif method == 'svd':
            T = GF.weighted_procrustes_counts(s, r, w, c).reshape(B, 16)
        else:
            raise ValueError(f'Unsupported registration method: {method}.')
        if cfg.name == '3dmatch' and not rre_rte:
            err = GF.registration_error_batched(reg_T, T, covariances=cov, has_covariance=has_cov, rmse_threshold=cfg.eval.rmse_threshold)
        else:
            err = GF.registration_error_batched(reg_T, T, rre_threshold=cfg.eval.rre_threshold, rte_threshold=cfg.eval.rte_threshold)
        rows += [metrics.double(), T.double(), err]
    return torch.cat(rows, 1).cpu().numpy()


def _pair_values(row, j, item, method):
    base = 3 + 24 * j
    ir, ov, rs, nu = row[base:base + 4]
    T = row[base + 4:base + 20].reshape(4, 4)
    rre, rte, perr, acc = row[base + 20:base + 24]
    # lgr / svd estimates are float32 as the reference's; its RANSAC estimate is Open3D's float64
    est = T.astype(np.float64) if method == 'ransac' else T.astype(np.float32)
    # the kernel's ratios are count / n rounded to fp32; the count is exact below 2^22 rows, so form count / n in double as numpy does
    # (the fp32 value can print differently at 3 decimals, e.g. 0.3825)
    n = int(nu)
    if 0 < n < 1 << 22:
        ir, ov = round(float(ir) * n) / n, round(float(ov) * n) / n
    return dict(precision=float(row[0]), recall=float(row[1]), hit_ratio=float(row[2]), inlier_ratio=float(ir), overlap=float(ov),
                residual=float(rs), num_corr=int(nu), estimated_transform=est, rre=float(rre), rte=float(rte), error=float(perr),
                accepted=bool(acc))


def _pair_3dmatch(run, cfg, scene_abbr, item, v):
    ref_frame, src_frame = item['ids']
    c = v['precision']
    msg = '{}, id0: {}, id1: {}, OV: {:.3f}'.format(scene_abbr, ref_frame, src_frame, item['overlap'])
    run.scene_meters['precision'].update(c)
    for name, ok in (('PMR>0', c > 0), ('PMR>=0.1', c >= 0.1), ('PMR>=0.3', c >= 0.3), ('PMR>=0.5', c >= 0.5)):
        run.scene_meters[name].update(float(ok))
    run.scene_meters['inlier_ratio'].update(v['inlier_ratio'])
    run.scene_meters['overlap'].update(v['overlap'])
    run.scene_meters['fmr'].update(float(v['inlier_ratio'] >= cfg.eval.inlier_ratio_threshold))
    msg += ', c_PIR: {:.3f}, f_IR: {:.3f}, f_OV: {:.3f}, f_RS: {:.3f}, f_NU: {}'.format(c, v['inlier_ratio'], v['overlap'], v['residual'],
                                                                                      v['num_corr'])
    if item['has_cov']:
        msg += ', r_RMSE: {:.3f}'.format(np.sqrt(v['error']))
        run.scene_meters['rr'].update(float(v['accepted']))
        if v['accepted']:
            run.scene_meters['rre'].update(v['rre'])
            run.scene_meters['rte'].update(v['rte'])
            msg += ', r_RRE: {:.3f}, r_RTE: {:.3f}'.format(v['rre'], v['rte'])
    else:
        v['accepted'] = None                              # not in the benchmark: never counted in the recall
    return msg


def _scene_end_3dmatch(run, scene_name, scene_abbr):
    sm = run.scene_meters
    c = {k: sm[k].mean() for k in ('precision', 'PMR>0', 'PMR>=0.1', 'PMR>=0.3', 'PMR>=0.5')}
    for k, val in c.items():
        run.coarse[k].update(val)
    run.scene_coarse[scene_abbr] = c
    f = {'recall': sm['fmr'].mean(), 'inlier_ratio': sm['inlier_ratio'].mean(), 'overlap': sm['overlap'].mean()}
    for k, val in f.items():
        run.fine[k].update(val)
    run.scene_fine[scene_abbr] = {'recall': f['recall'], 'inlier_ratio': f['inlier_ratio']}
    r = {'recall': sm['rr'].mean(), 'mean_rre': sm['rre'].mean(), 'mean_rte': sm['rte'].mean(), 'median_rre': sm['rre'].median(),
         'median_rte': sm['rte'].median()}
    for k, val in r.items():
        run.reg[k].update(val)
    run.scene_reg[scene_abbr] = r
    run.emit(INFO, f'Scene_name: {scene_name}')
    run.emit(INFO, '  Correspondence, , c_PIR: {:.3f}, c_PMR>0: {:.3f}, c_PMR>=0.1: {:.3f}, c_PMR>=0.3: {:.3f}, c_PMR>=0.5: {:.3f}, '
                   'f_FMR: {:.3f}, f_IR: {:.3f}, f_OV: {:.3f}'.format(c['precision'], c['PMR>0'], c['PMR>=0.1'], c['PMR>=0.3'],
                                                                      c['PMR>=0.5'], f['recall'], f['inlier_ratio'], f['overlap']))
    run.emit(INFO, '  Registration, RR: {:.3f}, mean_RRE: {:.3f}, mean_RTE: {:.3f}, median_RRE: {:.3f}, median_RTE: {:.3f}'.format(
        r['recall'], r['mean_rre'], r['mean_rte'], r['median_rre'], r['median_rte']))


def _pair_dgr(run, cfg, scene_abbr, item, v):
    """eval_dgr.py's per-pair meters and line: every pair is scored by RRE / RTE against the npz transform"""
    ref_frame, src_frame = item['ids']
    c = v['precision']
    sm = run.scene_meters
    sm['precision'].update(c)
    for name, ok in (('PMR>0', c > 0), ('PMR>=0.1', c >= 0.1), ('PMR>=0.3', c >= 0.3), ('PMR>=0.5', c >= 0.5)):
        sm[name].update(float(ok))
    sm['inlier_ratio'].update(v['inlier_ratio'])
    sm['overlap'].update(v['overlap'])
    sm['fmr'].update(float(v['inlier_ratio'] >= cfg.eval.inlier_ratio_threshold))
    if v['accepted']:
        for name in ('rre', 'rte'):
            sm[name].update(v[name])
            run.reg[f'overall_{name}'].update(v[name])
    sm['rr'].update(float(v['accepted']))
    run.reg['overall_recall'].update(float(v['accepted']))
    return ('{}, id0: {}, id1: {}, OV: {:.3f}, c_PIR: {:.3f}, f_IR: {:.3f}, f_OV: {:.3f}, f_RS: {:.3f}, f_NU: {}, r_RRE: {:.3f}, '
            'r_RTE: {:.3f}'.format(scene_abbr, ref_frame, src_frame, item['overlap'], c, v['inlier_ratio'], v['overlap'], v['residual'],
                                   v['num_corr'], v['rre'], v['rte']))


def _scene_end_dgr(run, scene_name, scene_abbr):
    sm = run.scene_meters
    c = {k: sm[k].mean() for k in ('precision', 'PMR>0', 'PMR>=0.1', 'PMR>=0.3', 'PMR>=0.5')}
    for k, val in c.items():
        run.coarse[k].update(val)
    run.scene_coarse[scene_abbr] = c
    f = {'recall': sm['fmr'].mean(), 'inlier_ratio': sm['inlier_ratio'].mean(), 'overlap': sm['overlap'].mean()}
    for k, val in f.items():
        run.fine[k].update(val)
    run.scene_fine[scene_abbr] = {'recall': f['recall'], 'inlier_ratio': f['inlier_ratio']}
    r = {'recall': sm['rr'].mean(), 'rre': sm['rre'].mean(), 'rte': sm['rte'].mean()}
    for k, val in r.items():
        run.reg[k].update(val)
    run.scene_reg[scene_abbr] = r
    run.emit(INFO, f'Scene_name: {scene_name}')
    run.emit(INFO, '  Correspondence, , c_PIR: {:.3f}, c_PMR>0: {:.3f}, c_PMR>=0.1: {:.3f}, c_PMR>=0.3: {:.3f}, c_PMR>=0.5: {:.3f}, '
                   'f_FMR: {:.3f}, f_IR: {:.3f}, f_OV: {:.3f}'.format(c['precision'], c['PMR>0'], c['PMR>=0.1'], c['PMR>=0.3'],
                                                                      c['PMR>=0.5'], f['recall'], f['inlier_ratio'], f['overlap']))
    run.emit(INFO, '  Registration, RR: {:.3f}, RRE: {:.3f}, RTE: {:.3f}'.format(r['recall'], r['rre'], r['rte']))


def _final_dgr(run, test_epoch):
    """eval_dgr.py's summary, its trailing ', ' included"""
    run.emit(CRITICAL, 'Epoch {}'.format(test_epoch))
    coarse = {k: m.mean() for k, m in run.coarse.items()}
    fine = {'recall': run.fine['recall'].mean(), 'inlier_ratio': run.fine['inlier_ratio'].mean(),
            'overlap': run.fine['overlap'].mean(), 'std': run.fine['recall'].std()}
    run.emit(CRITICAL, _pmr('  Coarse Matching, ', coarse))
    for abbr, m in run.scene_coarse.items():
        run.emit(CRITICAL, _pmr(f'    {abbr}', m))
    run.emit(CRITICAL, '  Fine Matching, FMR: {:.3f}, IR: {:.3f}, OV: {:.3f}, std: {:.3f}'.format(
        fine['recall'], fine['inlier_ratio'], fine['overlap'], fine['std']))
    for abbr, m in run.scene_fine.items():
        run.emit(CRITICAL, '    {}, FMR: {:.3f}, IR: {:.3f}'.format(abbr, m['recall'], m['inlier_ratio']))
    reg = {'recall': run.reg['overall_recall'].mean(), 'rre': run.reg['overall_rre'].mean(), 'rte': run.reg['overall_rte'].mean(),
           'mean_recall': run.reg['recall'].mean(), 'mean_rre': run.reg['rre'].mean(), 'mean_rte': run.reg['rte'].mean()}
    run.emit(CRITICAL, '  Registration, RR: {:.3f}, RRE: {:.3f}, RTE: {:.3f}, mean_RR: {:.3f}, mean_RRE: {:.3f}, mean_RTE: {:.3f}, '
             .format(*reg.values()))
    for abbr, m in run.scene_reg.items():
        run.emit(CRITICAL, '    {}, RR: {:.3f}, RRE: {:.3f}, RTE: {:.3f}'.format(abbr, m['recall'], m['rre'], m['rte']))
    return {'coarse': coarse, 'fine': fine, 'registration': reg, 'scenes': {'coarse': run.scene_coarse, 'fine': run.scene_fine,
                                                                            'registration': run.scene_reg}}


def _pmr(prefix, m):
    return ('{}, PIR: {:.3f}, PMR>0: {:.3f}, PMR>=0.1: {:.3f}, PMR>=0.3: {:.3f}, PMR>=0.5: {:.3f}'
            .format(prefix, m['precision'], m['PMR>0'], m['PMR>=0.1'], m['PMR>=0.3'], m['PMR>=0.5']))


def _final(run, config):
    coarse = {k: m.mean() for k, m in run.coarse.items()}
    fine = {'recall': run.fine['recall'].mean(), 'inlier_ratio': run.fine['inlier_ratio'].mean(),
            'overlap': run.fine['overlap'].mean(), 'std': run.fine['recall'].std()}
    run.emit(CRITICAL, _pmr('  Coarse Matching', coarse))
    if config == '3dmatch':
        for abbr, m in run.scene_coarse.items():
            run.emit(CRITICAL, _pmr(f'    {abbr}', m))
    run.emit(CRITICAL, '  Fine Matching, FMR: {:.3f}, IR: {:.3f}, OV: {:.3f}, std: {:.3f}'.format(
        fine['recall'], fine['inlier_ratio'], fine['overlap'], fine['std']))
    if config == '3dmatch':
        for abbr, m in run.scene_fine.items():
            run.emit(CRITICAL, '    {}, FMR: {:.3f}, IR: {:.3f}'.format(abbr, m['recall'], m['inlier_ratio']))
        reg = {k: run.reg[k].mean() for k in ('recall', 'mean_rre', 'mean_rte', 'median_rre', 'median_rte')}
        fmt = ', RR: {:.3f}, mean_RRE: {:.3f}, mean_RTE: {:.3f}, median_RRE: {:.3f}, median_RTE: {:.3f}'
        run.emit(CRITICAL, '  Registration' + fmt.format(*reg.values()))
        for abbr, m in run.scene_reg.items():
            run.emit(CRITICAL, f'    {abbr}' + fmt.format(m['recall'], m['mean_rre'], m['mean_rte'], m['median_rre'], m['median_rte']))
    else:
        reg = {'recall': run.reg['recall'].mean(), 'rre': run.reg['rre'].mean(), 'rte': run.reg['rte'].mean()}
        run.emit(CRITICAL, '  Registration, RR: {:.3f}, RRE: {:.3f}, RTE: {:.3f}'.format(reg['recall'], reg['rre'], reg['rte']))
    return {'coarse': coarse, 'fine': fine, 'registration': reg, 'scenes': {'coarse': run.scene_coarse, 'fine': run.scene_fine,
                                                                            'registration': run.scene_reg}}


def evaluate(config, method, features, benchmark=None, gt_root=None, num_corr=None, registration_dir=None, verbose=False, chunk=64,
             log=None, device=None, protocol='gtlog', test_epoch=None):
    """Runs the evaluation; returns ``{setting: {'summary', 'lines', 'pairs'}}`` with one entry per --num_corr value (key None
    without --num_corr).  ``lines`` are the (logging level, message) pairs eval.py (protocol 'gtlog') or eval_dgr.py (protocol
    'dgr', 3dmatch only; ``test_epoch`` is printed in its Epoch line) logs; ``pairs`` the per-pair values in evaluation order.
    ``log(level, message)`` receives the lines as they are produced."""
    if config not in ('3dmatch', 'kitti'):
        raise ValueError(f'unsupported config {config!r} (3dmatch or kitti)')
    if method not in ('lgr', 'ransac', 'svd'):
        raise ValueError(f'Unsupported registration method: {method}.')
    if protocol not in ('gtlog', 'dgr'):
        raise ValueError(f"protocol must be 'gtlog' or 'dgr', got {protocol!r}")
    dgr = protocol == 'dgr'
    if dgr and config != '3dmatch':
        raise ValueError("--protocol dgr is a 3dmatch evaluation (KITTI's eval.py already scores by RRE / RTE)")
    if dgr and registration_dir is not None:
        raise ValueError('--protocol dgr writes no est.log: drop --registration-dir')
    if config == '3dmatch' and (benchmark not in ('3DMatch', '3DLoMatch') or (gt_root is None and not dgr)):
        raise ValueError('3dmatch needs --benchmark 3DMatch or 3DLoMatch, and --gt-root unless --protocol dgr')
    cfg = make_cfg(config)
    settings = parse_num_corr(num_corr) if not isinstance(num_corr, list) else num_corr
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    runs = [_Run(k if len(settings) > 1 else None, log) for k in settings]
    scenes = discover(config, features, benchmark)
    n_total = sum(len(files) for _, files in scenes)
    pair_id = 0
    for scene_name, files in scenes:
        gt, abbr = None, None
        if config == '3dmatch':
            abbr = get_scene_abbr(scene_name)
            num_fragments = get_num_fragments(scene_name)
            if not dgr:
                gt = get_gt_logs_and_infos(os.path.join(gt_root, benchmark, scene_name), num_fragments)
            for run in runs:
                run.scene_meters = _meters(['precision', 'PMR>0', 'PMR>=0.1', 'PMR>=0.3', 'PMR>=0.5', 'fmr', 'inlier_ratio', 'overlap',
                                            'rr', 'rre', 'rte'])
                run.estimates = []
        for base in range(0, len(files), max(int(chunk), 1)):
            items = [_load(f, config, gt, dgr) for f in files[base:base + max(int(chunk), 1)]]
            rows = _device_rows(items, cfg, method, settings, pair_id, device, rre_rte=dgr)
            for i, item in enumerate(items):
                for j, run in enumerate(runs):
                    v = _pair_values(rows[i], j, item, method)
                    if dgr:
                        msg = _pair_dgr(run, cfg, abbr, item, v)
                        v.update(scene=scene_name, id0=item['ids'][0], id1=item['ids'][1])
                    elif config == '3dmatch':
                        msg = _pair_3dmatch(run, cfg, abbr, item, v)
                        run.estimates.append({'test_pair': item['ids'], 'num_fragments': num_fragments,
                                              'transform': v['estimated_transform']})
                        v.update(scene=scene_name, id0=item['ids'][0], id1=item['ids'][1])
                    else:
                        msg = _pair_kitti(run, cfg, item, v, pair_id + i, n_total)
                    run.pairs.append(v)
                    if verbose:
                        run.emit(INFO, msg)
            pair_id += len(items)
        if dgr:
            for run in runs:
                _scene_end_dgr(run, scene_name, abbr)
        elif config == '3dmatch':
            for k, run in zip(settings, runs):
                if registration_dir is not None:
                    sub = registration_dir if len(settings) == 1 else os.path.join(registration_dir, f'num_corr_{k}')
                    write_log_file(os.path.join(sub, benchmark, scene_name, 'est.log'), run.estimates)
                _scene_end_3dmatch(run, scene_name, abbr)
    return {k: {'summary': _final_dgr(run, test_epoch) if dgr else _final(run, config), 'lines': run.lines, 'pairs': run.pairs}
            for k, run in zip(settings, runs)}


def _pair_kitti(run, cfg, item, v, index, n_total):
    seq_id, src_frame, ref_frame = item['ids']
    c = v['precision']
    run.coarse['precision'].update(c)
    for name, ok in (('PMR>0', c > 0), ('PMR>=0.1', c >= 0.1), ('PMR>=0.3', c >= 0.3), ('PMR>=0.5', c >= 0.5)):
        run.coarse[name].update(float(ok))
    run.fine['inlier_ratio'].update(v['inlier_ratio'])
    run.fine['overlap'].update(v['overlap'])
    run.fine['recall'].update(float(v['inlier_ratio'] >= cfg.eval.inlier_ratio_threshold))
    if v['accepted']:
        run.reg['rre'].update(v['rre'])
        run.reg['rte'].update(v['rte'])
    run.reg['recall'].update(float(v['accepted']))
    v.update(seq=seq_id, id0=src_frame, id1=ref_frame)
    return ('{}/{}, seq_id: {}, id0: {}, id1: {}, c_PIR: {:.3f}, f_IR: {:.3f}, f_OV: {:.3f}, f_RS: {:.3f}, f_NU: {}, r_RRE: {:.3f}, '
            'r_RTE: {:.3f}'.format(index + 1, n_total, seq_id, src_frame, ref_frame, c, v['inlier_ratio'], v['overlap'], v['residual'],
                                   v['num_corr'], v['rre'], v['rte']))


def make_parser():
    parser = argparse.ArgumentParser(prog='python -m geotransformer_b200.evaluate', description=__doc__.split('\n\n')[0])
    parser.add_argument('--config', choices=['3dmatch', 'kitti'], required=True)
    parser.add_argument('--benchmark', choices=['3DMatch', '3DLoMatch'], help='3dmatch only')
    parser.add_argument('--method', choices=['lgr', 'ransac', 'svd'], required=True, help='registration method')
    parser.add_argument('--num_corr', default=None, help='number of correspondences for registration: one value or a comma list')
    parser.add_argument('--features', required=True, help='the tester\'s npz tree')
    parser.add_argument('--protocol', choices=['gtlog', 'dgr'], default='gtlog',
                        help="3dmatch: 'gtlog' scores against gt.log (eval.py), 'dgr' by RRE / RTE against the npz transform (eval_dgr.py)")
    parser.add_argument('--test-epoch', type=int, default=None, help='dgr: the epoch its Epoch line prints')
    parser.add_argument('--gt-root', default=None, help='3dmatch gtlog: the directory holding <benchmark>/<scene>/gt.log and gt.info')
    parser.add_argument('--registration-dir', default=None, help='3dmatch: where est.log files go')
    parser.add_argument('--verbose', action='store_true', help='log every pair')
    return parser


def main(argv=None):
    args = make_parser().parse_args(argv)
    if args.protocol == 'dgr' and args.config != '3dmatch':
        make_parser().error("--protocol dgr is a 3dmatch evaluation (KITTI's eval.py already scores by RRE / RTE)")
    if args.protocol == 'dgr' and args.registration_dir is not None:
        make_parser().error('--protocol dgr writes no est.log: drop --registration-dir')
    if args.config == '3dmatch' and (args.benchmark is None or (args.gt_root is None and args.protocol == 'gtlog')):
        make_parser().error('--config 3dmatch needs --benchmark, and --gt-root unless --protocol dgr')
    try:
        settings = parse_num_corr(args.num_corr)
    except ValueError as e:
        make_parser().error(str(e))
    logging.basicConfig(level=logging.INFO, format='[%(asctime)s] %(message)s', stream=sys.stdout)
    return evaluate(args.config, args.method, args.features, benchmark=args.benchmark, gt_root=args.gt_root, num_corr=settings,
                    registration_dir=args.registration_dir, verbose=args.verbose, log=lambda level, msg: _LOG.log(level, msg),
                    protocol=args.protocol, test_epoch=args.test_epoch)


if __name__ == '__main__':
    main()
