"""Training front end: the reference's training step (``engine/epoch_based_trainer.py::train_epoch`` and
``engine/iter_based_trainer.py``) on the device, one pair per step as the reference trains (``train.batch_size = 1``).

A step is: device collate -> ``GeoTransformer.forward_train`` -> ``OverallLoss`` -> ``backward`` -> the non-finite gradient guard
(``functional.nonfinite_check``) -> ``torch.optim.Adam.step`` -> ``zero_grad``.  The optimizer is the reference's class and
settings (Adam, L2 weight decay), so its ``state_dict`` and the snapshot ``{'epoch', 'iteration', 'model', 'optimizer',
'scheduler'}`` are interchangeable with the reference's ``snapshot.pth.tar``.  It runs fused; the guard's flag is handed to it as
``optimizer.found_inf``, so a step with a NaN or Inf gradient leaves parameters, moments and step counts untouched without a host
read-back (the reference applies such an update unless ``run_grad_check`` is set, which stops in a debugger).

The loss, the Evaluator's metrics and the skip flag of a step come back in one packed device-to-host copy and one event wait.

``batch_size`` B > 1 trains B pairs per step on one device (``train_batch``): the step the reference takes with B-rank
DistributedDataParallel.  One forward over the collated batch (``GeoTransformer.forward_train_batch``), the (B, 3) loss rows of
all pairs, and one backward of their mean over the valid pairs (``functional.batch_loss_weights``: a pair whose loss row is not
finite -- no ground truth or no targets -- is dropped from the mean instead of skipping the step).  With all pairs valid the
gradient is DDP's (1/B) sum_p g_p; with ``scale_lr`` the learning rates are multiplied by B as the reference's
``register_optimizer`` multiplies them by the world size.
"""
import math

import torch
from torch.autograd.graph import increment_version

from . import functional as GF
from .engine import LOSS_KEYS, METRIC_KEYS, RegistrationEngine
from .loss import Evaluator, OverallLoss
from .utils.data import registration_collate_fn_stack_mode


def make_optimizer(model, cfg):
    """the reference's optimizer (experiments/*/trainval.py): Adam(lr, weight_decay) with L2 weight decay, fused on the device.
    Its fused step writes the parameters without bumping their version counters: call ``optimizer_step`` rather than ``step``, so
    the caches keyed on parameter versions (structure-embedding table, transposed and fused weights) see the update."""
    return torch.optim.Adam(model.parameters(), lr=cfg.optim.lr, weight_decay=cfg.optim.weight_decay, fused=True)


def optimizer_step(optimizer, found_inf):
    """``optimizer.step()`` skipped on the device when ``found_inf`` (0-dim fp32, from ``functional.nonfinite_check``) is 1, then
    the version counters of its parameters are bumped (no kernel): torch's fused Adam leaves them unchanged, and every weight cache
    of the model is keyed on them"""
    optimizer.found_inf = found_inf
    optimizer.step()
    increment_version([p for g in optimizer.param_groups for p in g['params']])


def warmup_cosine(total_steps, warmup_steps, eta_init, eta_min):
    """LR factor of the reference's warm-up cosine (``utils/torch.py::WarmUpCosineAnnealingFunction``) as a function of
    LambdaLR's ``last_step``: linear from eta_init to 1 over ``warmup_steps``, then cosine down to eta_min at ``total_steps``"""
    normal_steps = total_steps - warmup_steps

    def factor(last_step):
        step = last_step + 1
        if step < warmup_steps:
            return eta_init + (1.0 - eta_init) / warmup_steps * step
        if step > total_steps:
            return eta_min
        return eta_min + 0.5 * (1.0 - eta_min) * (1.0 + math.cos(math.pi * (step - warmup_steps) / normal_steps))
    return factor


def make_scheduler(optimizer, cfg):
    """3DMatch and KITTI: StepLR(lr_decay_steps, lr_decay), stepped per epoch; ModelNet: the warm-up cosine, stepped per iteration"""
    o = cfg.optim
    if cfg.name == 'modelnet':
        return torch.optim.lr_scheduler.LambdaLR(optimizer, warmup_cosine(o.max_iteration, o.warmup_steps, o.eta_init, o.eta_min))
    return torch.optim.lr_scheduler.StepLR(optimizer, o.lr_decay_steps, gamma=o.lr_decay)


def make_optimizer_and_scheduler(model, cfg, batch_size=1, scale_lr=True):
    """``make_optimizer``, then (``scale_lr``) every param group's lr multiplied by ``batch_size``, then ``make_scheduler``: the
    reference's order (``register_optimizer`` scales by the DDP world size before the experiment builds its scheduler), so the
    scheduler's base lrs are the scaled ones.  ``batch_size`` 1 gives ``make_optimizer`` / ``make_scheduler`` unchanged."""
    optimizer = make_optimizer(model, cfg)
    if scale_lr:
        for g in optimizer.param_groups:
            g['lr'] = g['lr'] * batch_size
    return optimizer, make_scheduler(optimizer, cfg)


def fused_optimizer_state(state):
    """an Adam ``state_dict`` (the reference saves an unfused one: step counts on the host) made loadable into ``make_optimizer``'s
    fused Adam: ``load_state_dict`` takes the saved group options, so they are set to fused here, and with them it moves the step
    counts to the parameters' device"""
    groups = [dict(g, fused=True, foreach=None, capturable=False) for g in state['param_groups']]
    return dict(state, param_groups=groups)


# packed per-step row on the device: [loss, c_loss, f_loss | PIR, IR, RRE, RTE, RMSE, RR, #corr, #gt | found_inf]
_ROW = 12
# a batched step appends [n_valid] and per pair [loss, c_loss, f_loss | the 8 metrics]
_PAIR_ROW = 11
# attention items of one batched launch pair whose probabilities the backward reads (GEOB200_ATT_MAX_ITEMS): one per cloud
MAX_BATCH = GF.ATT_MAX_ITEMS // 2


class TrainingEngine:
    def __init__(self, model, cfg, neighbor_limits, seed=None, device=None, batch_size=1, scale_lr=True, augment=False):
        """``model``: a GeoTransformer on its device with its weights loaded.  ``seed`` keys the target sampler's Philox stream
        (default ``cfg.seed``); target draws depend on (seed, iteration, pair) only, so a resumed run draws what an uninterrupted one
        would.  ``batch_size``: pairs per ``train_batch`` step (1 .. MAX_BATCH); with ``scale_lr`` every param group's lr is
        multiplied by it before the scheduler is built (the reference scales by the DDP world size in ``register_optimizer``).
        ``augment``: every step trains on its pairs augmented on the device as the reference's training set does
        (``augment.augmented_collate`` with (seed, iteration); pair p of a step draws from stream p); for ModelNet a pair is then a raw
        shape ``{'points': (N, 3)}``.  Off: the pairs are trained on as given."""
        if cfg.optim.grad_acc_steps != 1:
            raise NotImplementedError('grad_acc_steps > 1 (1 in every shipped config)')
        if not 1 <= int(batch_size) <= MAX_BATCH:
            raise ValueError(f'batch_size must be in 1..{MAX_BATCH}')
        self.model, self.cfg, self.limits = model, cfg, neighbor_limits
        self.batch_size = int(batch_size)
        self.augment = bool(augment)
        if self.augment:
            from .augment import check_options
            check_options(cfg)
        self.seed = int(cfg.seed if seed is None else seed)
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self.loss_func = OverallLoss(cfg)
        self.evaluator = Evaluator(cfg)
        self.optimizer, self.scheduler = make_optimizer_and_scheduler(model, cfg, self.batch_size, scale_lr)
        self.per_iteration = cfg.name == 'modelnet'
        self.epoch, self.iteration = 0, 0
        self.found_inf = torch.zeros((), dtype=torch.float32, device=self.device)   # 0-dim: fused Adam subtracts it from its 0-dim step counts
        self.no_valid = torch.zeros((), dtype=torch.float32, device=self.device)    # a batched step's "no valid pair" flag
        self.row_dev = torch.zeros((_ROW,), dtype=torch.float32, device=self.device)
        self.row_host = torch.zeros((_ROW,), dtype=torch.float32).pin_memory()
        self.stage_events = None       # set to a list to receive (label, CUDA event) marks of every step (tools/train_bench.py)
        self._native_versions = None

    def _mark(self, label):
        if self.stage_events is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self.stage_events.append((label, e))

    def train_step(self, pair):
        """one optimisation step on ``pair`` (dict with ref_points / src_points / ref_feats / src_feats / transform); returns the
        reference's train_step result: loss, c_loss, f_loss and the Evaluator's metrics (no RMSE for KITTI), plus ``lr`` (of this
        step) and ``skipped`` (a non-finite gradient: no update)"""
        model = self.model
        self.iteration += 1
        self._mark('start')
        data = self._collate([pair])
        self._mark('collate')
        out = model.forward_train(data, self.seed, self.iteration)
        self._mark('forward')
        rows = self.loss_func.graph_rows(out, data)
        self._mark('loss')
        rows[0, 0].backward()
        self._mark('backward')
        # a non-finite loss also skips the step: with no ground truth or no targets the losses are NaN, as in the reference,
        # while the gradients of their empty sums are zero
        checked = [p.grad for p in model.parameters() if p.grad is not None] + [rows.detach()]
        GF.nonfinite_check(checked, self.found_inf)
        self._mark('guard')
        lr = self.optimizer.param_groups[0]['lr']
        optimizer_step(self.optimizer, self.found_inf)
        self.optimizer.zero_grad(set_to_none=True)
        self._mark('optimizer')
        with torch.no_grad():
            row = self.row_dev
            row[:3].copy_(rows.detach()[0])
            st, ev = out['_stacked'], self.evaluator
            gt_idx, gt_ov, gt_cnt = st['gt']
            (m_corr, m_cnt), (rcp, scp, n_corr) = st['coarse'], st['lgr']
            GF.evaluate_batched(gt_idx, gt_ov, gt_cnt, m_corr, m_cnt, rcp, scp, n_corr, data['transform'].reshape(1, 4, 4),
                                st['transforms'], st['points'], st['cloud_nodes'], st['cloud_points'], ev.mode, ev.acceptance_overlap,
                                ev.acceptance_radius, row[3:11].view(1, 8), ev.acceptance_rmse, ev.acceptance_rre, ev.acceptance_rte)
            row[11].copy_(self.found_inf)
        self._mark('metrics')
        self.row_host.copy_(self.row_dev, non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        if self.per_iteration:
            self.scheduler.step()
        done.synchronize()
        v = self.row_host.tolist()
        res = dict(zip(LOSS_KEYS, v[:3]))
        res.update(zip(METRIC_KEYS, v[3:9]))
        if self.evaluator.mode == 1:
            del res['RMSE']
        res['lr'] = lr
        res['skipped'] = v[11] != 0.0
        return res

    def train_batch(self, pairs):
        """one optimisation step on 1 .. batch_size pairs: the mean over the valid pairs of their losses (a pair is valid when its
        [loss, c_loss, f_loss] row is finite).  Returns loss, c_loss, f_loss (that mean) and the Evaluator's metrics averaged over
        all pairs, ``per_pair`` (one dict of losses and metrics per pair), ``lr``, ``skipped`` (a non-finite gradient or no valid
        pair: no update) and ``masked_pairs`` (pairs left out of the mean).  Everything comes back in one packed device-to-host
        copy and one event wait; nothing else waits for the device after the collate."""
        B = len(pairs)
        if not 1 <= B <= self.batch_size:
            raise ValueError(f'train_batch: 1..{self.batch_size} pairs per step, got {B}')
        model = self.model
        self.iteration += 1
        self._mark('start')
        data = self._collate(list(pairs))
        self._mark('collate')
        out = model.forward_train_batch(data, self.seed, self.iteration)
        self._mark('forward')
        rows = self.loss_func.graph_rows(out, data)
        packed = self._packed(B)
        self.no_valid.zero_()
        w, _ = GF.batch_loss_weights(rows, mean_row=packed[:3], n_valid=packed[_ROW:_ROW + 1], found_inf=self.no_valid)
        upstream = torch.zeros_like(rows)
        upstream[:, 0].copy_(w)
        self._mark('loss')
        rows.backward(upstream)
        self._mark('backward')
        checked = [p.grad for p in model.parameters() if p.grad is not None] + [packed[:3]]
        GF.nonfinite_check(checked, self.found_inf)
        torch.maximum(self.found_inf, self.no_valid, out=self.found_inf)     # a step without a valid pair is skipped too
        self._mark('guard')
        lr = self.optimizer.param_groups[0]['lr']
        optimizer_step(self.optimizer, self.found_inf)
        self.optimizer.zero_grad(set_to_none=True)
        self._mark('optimizer')
        with torch.no_grad():
            per = packed[_ROW + 1:].view(B, _PAIR_ROW)
            per[:, :3].copy_(rows.detach())
            st, ev = out['_stacked'], self.evaluator
            gt_idx, gt_ov, gt_cnt = st['gt']
            (m_corr, m_cnt), (rcp, scp, n_corr) = st['coarse'], st['lgr']
            GF.evaluate_batched(gt_idx, gt_ov, gt_cnt, m_corr, m_cnt, rcp, scp, n_corr, st['gt_transforms'], st['transforms'], st['points'],
                                st['cloud_nodes'], st['cloud_points'], ev.mode, ev.acceptance_overlap, ev.acceptance_radius, per[:, 3:],
                                ev.acceptance_rmse, ev.acceptance_rre, ev.acceptance_rte)
            torch.mean(per[:, 3:], dim=0, out=packed[3:11])          # the metrics of all pairs, as the reference's all_reduce_tensors
            packed[11].copy_(self.found_inf)
        self._mark('metrics')
        host = self._host[:packed.numel()]
        host.copy_(packed, non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        if self.per_iteration:
            self.scheduler.step()
        done.synchronize()
        v = host.tolist()
        res = self._result(v[:_ROW])
        res['lr'] = lr
        n_valid = int(v[_ROW])
        res['masked_pairs'] = B - n_valid
        res['skipped'] = v[11] != 0.0
        res['per_pair'] = [self._result(v[_ROW + 1 + p * _PAIR_ROW:_ROW + 1 + (p + 1) * _PAIR_ROW]) for p in range(B)]
        return res

    def _collate(self, pairs):
        """the step's collate: the plain stack-mode collate, or with ``augment`` the device augmentation keyed by (seed, iteration)"""
        if self.augment:
            from .augment import augmented_collate
            return augmented_collate(pairs, self.cfg, self.limits, self.seed, self.iteration, device=self.device)
        b = self.cfg.backbone
        return registration_collate_fn_stack_mode(pairs, b.num_stages, b.init_voxel_size, b.init_radius, self.limits, device=self.device)

    def _packed(self, B):
        """the device buffer of one batched step's results: [the step row (_ROW) | n_valid | B per-pair rows], and its pinned mirror"""
        n = _ROW + 1 + B * _PAIR_ROW
        if getattr(self, '_packed_dev', None) is None or self._packed_dev.numel() < n:
            self._packed_dev = torch.zeros((_ROW + 1 + self.batch_size * _PAIR_ROW,), dtype=torch.float32, device=self.device)
            self._host = torch.zeros((self._packed_dev.numel(),), dtype=torch.float32).pin_memory()
        return self._packed_dev[:n]

    def _result(self, v):
        res = dict(zip(LOSS_KEYS, v[:3]))
        res.update(zip(METRIC_KEYS, v[3:9]))
        if self.evaluator.mode == 1:
            del res['RMSE']
        return res

    def train_epoch(self, pairs):
        """one epoch over ``pairs``, then the per-epoch scheduler step (3DMatch, KITTI); returns the step results.  With
        batch_size 1: ``train_step`` per pair; otherwise ``train_batch`` on consecutive groups of batch_size pairs, a trailing
        partial group being a step of fewer pairs (``iteration`` counts steps)."""
        self.epoch += 1
        if self.batch_size == 1:
            results = [self.train_step(p) for p in pairs]
        else:
            pairs = list(pairs)
            results = [self.train_batch(pairs[i:i + self.batch_size]) for i in range(0, len(pairs), self.batch_size)]
        if not self.per_iteration:
            self.scheduler.step()
        return results

    def train_groups(self, groups, log=None):
        """one epoch over the steps of an iterable of pair groups (``datasets.loader.PrefetchLoader.epoch``), pulled one at a time so
        that only the loader's prefetched steps are held in memory; then the per-epoch scheduler step (3DMatch, KITTI).  As in
        ``train_epoch``, steps are ``train_step`` with batch_size 1 and ``train_batch`` otherwise.  ``log(result)`` is called after
        every step; returns the step results."""
        self.epoch += 1
        results = []
        for group in groups:
            res = self.train_step(group[0]) if self.batch_size == 1 else self.train_batch(group)
            results.append(res)
            if log is not None:
                log(res)
        if not self.per_iteration:
            self.scheduler.step()
        return results

    def _param_versions(self):
        return tuple((p.data_ptr(), p._version) for p in self.model.parameters())

    def validate(self, pairs, **engine_kwargs):
        """the reference's val_step on ``pairs`` through ``RegistrationEngine`` (native stage drivers, OverallLoss and Evaluator on
        the device).  The drivers hold derived copies of the weights (tf32 images, fused projections, transposes), so they are
        rebuilt first when any parameter changed since they were built."""
        from .model import enable_native
        from .native import NativeModel
        if getattr(self.model, '_native', None) is None:
            enable_native(self.model)
        elif self._native_versions != self._param_versions():
            self.model._native = NativeModel(self.model)
        self._native_versions = self._param_versions()
        eng = RegistrationEngine(self.model, self.cfg, self.limits, device=self.device, loss_func=self.loss_func,
                                 evaluator=self.evaluator, **engine_kwargs)
        try:
            return eng.register(pairs)
        finally:
            eng.close()

    def state_dict(self):
        """the reference's snapshot: {'epoch', 'iteration', 'model', 'optimizer', 'scheduler'}"""
        return {'epoch': self.epoch, 'iteration': self.iteration, 'model': self.model.state_dict(),
                'optimizer': self.optimizer.state_dict(), 'scheduler': self.scheduler.state_dict()}

    def save_snapshot(self, path):
        torch.save(self.state_dict(), path)

    def load_snapshot(self, path):
        """a snapshot of ``save_snapshot`` or the reference's ``snapshot.pth.tar``; training continues at its epoch / iteration"""
        sd = torch.load(path, map_location='cpu', weights_only=False)
        self.model.load_state_dict(sd['model'], strict=True)
        self.epoch = int(sd.get('epoch', 0))
        self.iteration = int(sd.get('iteration', 0))
        if 'optimizer' in sd:
            self.optimizer.load_state_dict(fused_optimizer_state(sd['optimizer']))
        if 'scheduler' in sd:
            self.scheduler.load_state_dict(sd['scheduler'])
