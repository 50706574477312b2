"""Training front end: the reference's training step (``engine/epoch_based_trainer.py::train_epoch`` and
``engine/iter_based_trainer.py``) on the device, one pair per step as the reference trains (``train.batch_size = 1``).

A step is: device collate -> ``GeoTransformer.forward_train`` -> ``OverallLoss`` -> ``backward`` -> the non-finite gradient guard
(``functional.nonfinite_check``) -> ``torch.optim.Adam.step`` -> ``zero_grad``.  The optimizer is the reference's class and
settings (Adam, L2 weight decay), so its ``state_dict`` and the snapshot ``{'epoch', 'iteration', 'model', 'optimizer',
'scheduler'}`` are interchangeable with the reference's ``snapshot.pth.tar``.  It runs fused; the guard's flag is handed to it as
``optimizer.found_inf``, so a step with a NaN or Inf gradient leaves parameters, moments and step counts untouched without a host
read-back (the reference applies such an update unless ``run_grad_check`` is set, which stops in a debugger).

The loss, the Evaluator's metrics and the skip flag of a step come back in one packed device-to-host copy and one event wait.
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


def fused_optimizer_state(state):
    """an Adam ``state_dict`` (the reference saves an unfused one: step counts on the host) made loadable into ``make_optimizer``'s
    fused Adam: ``load_state_dict`` takes the saved group options, so they are set to fused here, and with them it moves the step
    counts to the parameters' device"""
    groups = [dict(g, fused=True, foreach=None, capturable=False) for g in state['param_groups']]
    return dict(state, param_groups=groups)


# packed per-step row on the device: [loss, c_loss, f_loss | PIR, IR, RRE, RTE, RMSE, RR, #corr, #gt | found_inf]
_ROW = 12


class TrainingEngine:
    def __init__(self, model, cfg, neighbor_limits, seed=None, device=None):
        """``model``: a GeoTransformer on its device with its weights loaded.  ``seed`` keys the target sampler's Philox stream
        (default ``cfg.seed``); target draws depend on (seed, iteration) only, so a resumed run draws what an uninterrupted one
        would."""
        if cfg.optim.grad_acc_steps != 1:
            raise NotImplementedError('grad_acc_steps > 1 (1 in every shipped config)')
        self.model, self.cfg, self.limits = model, cfg, neighbor_limits
        self.seed = int(cfg.seed if seed is None else seed)
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self.loss_func = OverallLoss(cfg)
        self.evaluator = Evaluator(cfg)
        self.optimizer = make_optimizer(model, cfg)
        self.scheduler = make_scheduler(self.optimizer, cfg)
        self.per_iteration = cfg.name == 'modelnet'
        self.epoch, self.iteration = 0, 0
        self.found_inf = torch.zeros((), dtype=torch.float32, device=self.device)   # 0-dim: fused Adam subtracts it from its 0-dim step counts
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
        model, b = self.model, self.cfg.backbone
        self.iteration += 1
        self._mark('start')
        data = registration_collate_fn_stack_mode([pair], b.num_stages, b.init_voxel_size, b.init_radius, self.limits, device=self.device)
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

    def train_epoch(self, pairs):
        """``train_step`` over ``pairs``, then the per-epoch scheduler step (3DMatch, KITTI); returns the step results"""
        self.epoch += 1
        results = [self.train_step(p) for p in pairs]
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
