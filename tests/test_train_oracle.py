"""The training step without a GPU: the numpy restatement of the ground-truth superpoint target sampler against the reference's
SuperPointTargetGenerator, the argument checks of the two training entry points (rejected before any launch), and the learning-rate
schedules of make_scheduler against the reference's formulas, restated here."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

from geotransformer_b200 import _lib as L
from geotransformer_b200.config import make_cfg
from geotransformer_b200.train import make_scheduler
from oracle import ransac_oracle as RO
from oracle import ref_harness
from oracle import train_oracle as TO

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
REF_TARGET = os.path.join(ref_harness.REF_ROOT, 'geotransformer', 'modules', 'geotransformer', 'superpoint_target.py')
WORKLOADS = ['demo2k', 'modelnet717', 'kitti4k']


def _gt(workload):
    g = np.load(os.path.join(GOLD, f'{workload}.npz'))
    return g['gt_node_corr_indices'], g['gt_node_corr_overlaps']


@pytest.mark.parametrize('workload', WORKLOADS)
def test_sampler_keeps_every_candidate_in_gt_order_up_to_num_targets(workload):
    """the reference's deterministic branch: at most num_targets candidates -> all rows with overlap > threshold, in gt order"""
    idx, ov = _gt(workload)
    keep = ov > np.float32(0.1)
    n = int(keep.sum())
    assert n > 0
    for k in (n, n + 7):
        r, s, o = TO.select_targets(idx, ov, 0.1, k, seed=7351, iteration=3)
        assert np.array_equal(r, idx[keep, 0]) and np.array_equal(s, idx[keep, 1]) and np.array_equal(o, ov[keep])


@pytest.mark.skipif(not os.path.exists(REF_TARGET), reason='reference checkout not present')
@pytest.mark.parametrize('workload', WORKLOADS)
def test_sampler_matches_the_reference_generator(workload):
    """the reference's SuperPointTargetGenerator on the fixture's gt correspondences: same rows in its deterministic branch, and in
    the random branch a subset of the same size drawn from the same candidates"""
    spec = importlib.util.spec_from_file_location('ref_superpoint_target', REF_TARGET)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    idx, ov = _gt(workload)
    n = int((ov > np.float32(0.1)).sum())
    gen = mod.SuperPointTargetGenerator(n, 0.1)
    r, s, o = gen(torch.from_numpy(idx), torch.from_numpy(ov))
    mr, ms, mo = TO.select_targets(idx, ov, 0.1, n, seed=1, iteration=1)
    assert np.array_equal(r.numpy(), mr) and np.array_equal(s.numpy(), ms) and np.array_equal(o.numpy(), mo)
    mr, ms, mo = TO.select_targets(idx, ov, 0.1, 128, seed=1, iteration=1)
    cands = set(map(tuple, idx[ov > np.float32(0.1)].tolist()))
    assert len(mr) == 128 and len(set(zip(mr.tolist(), ms.tolist()))) == 128
    assert set(zip(mr.tolist(), ms.tolist())) <= cands


def test_sampler_random_branch_is_sorted_distinct_and_keyed():
    """n > num_targets: num_targets distinct candidates in ascending gt order, a function of (seed, iteration, pair) only"""
    idx, ov = _gt('demo2k')
    cand = np.nonzero(ov > np.float32(0.1))[0]
    a = TO.select_targets(idx, ov, 0.1, 128, seed=7351, iteration=5, pair=0)
    pos = np.array([np.nonzero((idx[cand, 0] == r) & (idx[cand, 1] == s))[0][0] for r, s in zip(a[0], a[1])])
    assert len(pos) == 128 and np.all(np.diff(pos) > 0)
    assert np.all(a[2] > np.float32(0.1))
    again = TO.select_targets(idx, ov, 0.1, 128, seed=7351, iteration=5, pair=0)
    assert all(np.array_equal(x, y) for x, y in zip(a, again))
    others = [TO.select_targets(idx, ov, 0.1, 128, seed=sd, iteration=it, pair=p)[0] for sd, it, p in ((7352, 5, 0), (7351, 6, 0), (7351, 5, 1))]
    assert sum(np.array_equal(a[0], o) for o in others) == 0


def test_target_words_use_the_ransac_philox():
    """word 0 of Philox4x32-10 with counter (j, iteration lo, iteration hi, pair) and the 64-bit seed as key"""
    seed, it = (5 << 32) | 77, (3 << 32) | 9
    w = TO.target_words(4, seed, it, 2)
    ctr = np.array([[j, 9, 3, 2] for j in range(4)], dtype=np.uint64)
    assert np.array_equal(w, RO.philox4x32_10(ctr, (77, 5))[:, 0])


def test_training_entry_points_reject_bad_arguments_before_any_launch():
    lib = L.lib()
    launches = lib.geob200_launch_count()
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.addressof(buf)
    nodes = np.array([10, 12], dtype=np.int64)
    ws = lib.geob200_superpoint_targets_batched_workspace_bytes(120)
    assert ws >= 2 * 4 * 120

    def err():
        return lib.geob200_last_error().decode()

    def targets(n_pairs=1, cloud_nodes=nodes.ctypes.data, thr=0.1, k=128, pair_base=0, gt=p, ws_bytes=1 << 16, out=p):
        return lib.geob200_superpoint_targets_batched(gt, p, p, n_pairs, cloud_nodes, thr, k, 7351, 1, pair_base, out, p, p, p, ws_bytes, None)

    assert targets(n_pairs=0) < 0 and 'pairs' in err()
    assert targets(n_pairs=33) < 0 and 'pairs' in err()
    assert targets(k=0) < 0 and 'num_targets' in err()
    assert targets(thr=float('nan')) < 0 and 'overlap_threshold' in err()
    assert targets(pair_base=-1) < 0 and 'pair_base' in err()
    assert targets(cloud_nodes=None) < 0 and 'cloud_nodes' in err()
    assert targets(gt=None) < 0 and 'null pointer' in err()
    assert targets(out=None) < 0 and 'null pointer' in err()
    assert targets(ws_bytes=16) < 0 and 'workspace' in err()
    bad_nodes = np.array([-1, 12], dtype=np.int64)
    assert targets(cloud_nodes=bad_nodes.ctypes.data) < 0
    assert lib.geob200_nonfinite_check(p, p, 0, 10, p, None) < 0 and 'tensors' in err()
    assert lib.geob200_nonfinite_check(p, p, 70000, 10, p, None) < 0 and 'tensors' in err()
    assert lib.geob200_nonfinite_check(p, p, 3, -1, p, None) < 0 and 'max_numel' in err()
    assert lib.geob200_nonfinite_check(None, p, 3, 10, p, None) < 0 and 'null pointer' in err()
    assert lib.geob200_nonfinite_check(p, p, 3, 10, None, None) < 0 and 'null pointer' in err()
    assert lib.geob200_launch_count() == launches


def _ref_step_lr(lr, gamma, step_size, epoch):
    return lr * gamma ** (epoch // step_size)


def _ref_warmup_cosine(total, warmup, eta_init, eta_min, last_step):
    nxt = last_step + 1
    if nxt < warmup:
        return eta_init + (1.0 - eta_init) / warmup * nxt
    if nxt > total:
        return eta_min
    nxt -= warmup
    return eta_min + 0.5 * (1.0 - eta_min) * (1 + np.cos(np.pi * nxt / (total - warmup)))


def _lrs(cfg, n):
    opt = torch.optim.Adam([torch.nn.Parameter(torch.zeros(1))], lr=cfg.optim.lr)
    sched = make_scheduler(opt, cfg)
    out = []
    for _ in range(n):
        out.append(opt.param_groups[0]['lr'])
        opt.step()
        sched.step()
    return out


@pytest.mark.parametrize('name', ['3dmatch', 'kitti'])
def test_step_lr_per_epoch_matches_the_reference(name):
    cfg = make_cfg(name)
    o = cfg.optim
    got = _lrs(cfg, 20)
    want = [_ref_step_lr(o.lr, o.lr_decay, o.lr_decay_steps, e) for e in range(20)]
    assert np.allclose(got, want, rtol=1e-12, atol=0), (got, want)


@pytest.mark.parametrize('warmup,total', [(10000, 400000), (5, 12)])
def test_warmup_cosine_per_iteration_matches_the_reference(warmup, total):
    """ModelNet's warm-up cosine over the first 20 iterations at the shipped setting, and on a short schedule that reaches the cosine
    and its floor within 20 iterations"""
    cfg = make_cfg('modelnet')
    cfg.optim.update(warmup_steps=warmup, max_iteration=total)
    o = cfg.optim
    got = _lrs(cfg, 20)
    # LambdaLR evaluates the factor at last_step = 0 on construction, then once per scheduler step
    want = [o.lr * _ref_warmup_cosine(total, warmup, o.eta_init, o.eta_min, i) for i in range(20)]
    assert np.allclose(got, want, rtol=1e-12, atol=0), (got, want)


def test_grad_acc_steps_other_than_one_is_refused():
    from geotransformer_b200.train import TrainingEngine
    cfg = make_cfg('3dmatch')
    cfg.optim.grad_acc_steps = 2
    with pytest.raises(NotImplementedError):
        TrainingEngine(torch.nn.Linear(1, 1), cfg, None, device='cpu')


def test_make_optimizer_is_the_reference_adam_and_round_trips():
    """Adam with the config's lr and L2 weight decay, fused; its state_dict loads into a plain Adam and back"""
    from geotransformer_b200.train import fused_optimizer_state, make_optimizer
    cfg = make_cfg('3dmatch')
    model = torch.nn.Linear(3, 2)
    opt = make_optimizer(model, cfg)
    assert type(opt) is torch.optim.Adam
    g = opt.param_groups[0]
    assert g['lr'] == cfg.optim.lr and g['weight_decay'] == cfg.optim.weight_decay and g['fused'] and not g['decoupled_weight_decay']
    model(torch.ones(4, 3)).sum().backward()
    opt.step()
    plain = torch.optim.Adam(model.parameters())
    plain.load_state_dict(opt.state_dict())
    back = make_optimizer(model, cfg)
    back.load_state_dict(fused_optimizer_state(plain.state_dict()))
    for p in model.parameters():
        for key in ('exp_avg', 'exp_avg_sq', 'step'):
            assert torch.equal(back.state[p][key], opt.state[p][key])
    assert back.param_groups[0]['fused']
