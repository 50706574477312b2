"""Training-step throughput on the device: TrainingEngine.train_step on one pair per step (synthetic weights, seed 7351).

Prints, per workload, steps/s over --steps timed steps after --warmup, the host time per step (wall clock of train_step, which ends
in its one event wait), and the median CUDA-event time of each stage: collate, forward_train, OverallLoss, backward, the gradient
guard, the fused Adam step and the metrics.  The card name and power limit are read in the same run.

    python tools/train_bench.py [--workloads 3dmatch20k kitti4k] [--steps 20] [--warmup 5]

With ``--batch 1 2 4 8`` it also times TrainingEngine.train_batch on B distinct pairs per step (B = 1 included, through the
batched path) and adds pairs/s and torch.cuda.max_memory_allocated of each batch size; a batch size that does not fit is reported
as out of memory.  ``--repeat R`` runs every configuration R times, the configurations interleaved (train_step, then each B, R
rounds), and reports the median of each number with the min and max of pairs/s.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from geotransformer_b200.config import make_cfg                     # noqa: E402
from geotransformer_b200.model import create_model                  # noqa: E402
from geotransformer_b200.synth import make_pair                     # noqa: E402
from geotransformer_b200.train import TrainingEngine                # noqa: E402
from geotransformer_b200.weights import synthetic_state_dict        # noqa: E402
from oracle import backbone_grad_oracle as BG                       # noqa: E402


def run(workload, steps, warmup, extra=False):
    pair = make_pair(workload, 0)
    cfg = make_cfg(pair['config'])
    model = create_model(cfg)
    model.load_state_dict(synthetic_state_dict(model, 7351), strict=True)
    model = model.cuda()
    eng = TrainingEngine(model, cfg, BG.limits(workload))
    torch.cuda.reset_peak_memory_stats()
    dd = {k: pair[k] for k in ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')}
    for _ in range(warmup):
        eng.train_step(dd)
    torch.cuda.synchronize()
    eng.stage_events = []
    host, skipped = [], 0
    t0 = time.perf_counter()
    for _ in range(steps):
        t = time.perf_counter()
        skipped += eng.train_step(dd)['skipped']
        host.append(time.perf_counter() - t)
    wall = time.perf_counter() - t0
    torch.cuda.synchronize()
    stages = {}
    marks = eng.stage_events
    for (_, e0), (label, e1) in zip(marks[:-1], marks[1:]):
        if label != 'start':
            stages.setdefault(label, []).append(e0.elapsed_time(e1))
    med = {k: sorted(v)[len(v) // 2] for k, v in stages.items()}
    host.sort()
    n_params = sum(p.numel() for p in model.parameters())
    res = dict(workload=workload, config=cfg.name, parameters=n_params, steps=steps, skipped=int(skipped), steps_per_s=steps / wall,
               host_ms_per_step_median=1e3 * host[len(host) // 2], stage_ms_median={k: round(v, 4) for k, v in med.items()})
    if extra:          # the fields of the batched runs, for the train_step baseline beside them
        res.update(pairs_per_s=steps / wall, max_memory_allocated_mib=torch.cuda.max_memory_allocated() / 2 ** 20)
    return res


def run_batch(workload, B, steps, warmup):
    pairs = [make_pair(workload, i) for i in range(B)]
    cfg = make_cfg(pairs[0]['config'])
    model = create_model(cfg)
    model.load_state_dict(synthetic_state_dict(model, 7351), strict=True)
    model = model.cuda()
    eng = TrainingEngine(model, cfg, BG.limits(workload), batch_size=B)
    dd = [{k: p[k] for k in ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')} for p in pairs]
    torch.cuda.reset_peak_memory_stats()
    for _ in range(warmup):
        eng.train_batch(dd)
    torch.cuda.synchronize()
    eng.stage_events = []
    host, skipped, masked = [], 0, 0
    t0 = time.perf_counter()
    for _ in range(steps):
        t = time.perf_counter()
        r = eng.train_batch(dd)
        host.append(time.perf_counter() - t)
        skipped += r['skipped']
        masked += r['masked_pairs']
    wall = time.perf_counter() - t0
    torch.cuda.synchronize()
    stages = {}
    marks = eng.stage_events
    for (_, e0), (label, e1) in zip(marks[:-1], marks[1:]):
        if label != 'start':
            stages.setdefault(label, []).append(e0.elapsed_time(e1))
    med = {k: sorted(v)[len(v) // 2] for k, v in stages.items()}
    host.sort()
    return dict(workload=workload, config=cfg.name, batch=B, steps=steps, skipped=int(skipped), masked_pairs=int(masked),
                steps_per_s=steps / wall, pairs_per_s=B * steps / wall, host_ms_per_step_median=1e3 * host[len(host) // 2],
                stage_ms_median={k: round(v, 4) for k, v in med.items()}, max_memory_allocated_mib=torch.cuda.max_memory_allocated() / 2 ** 20)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', nargs='+', default=['3dmatch20k', 'kitti4k'])
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--batch', type=int, nargs='+', default=None, help='pairs per step: time train_batch at each of these batch sizes')
    ap.add_argument('--repeat', type=int, default=1, help='runs per configuration; medians are reported')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'train_bench needs a GPU'
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    print(json.dumps({'device': q.stdout.strip() or torch.cuda.get_device_name()}))
    if a.batch is None and a.repeat == 1:
        for w in a.workloads:
            print(json.dumps(run(w, a.steps, a.warmup)))
        return
    for w in a.workloads:
        configs = ['train_step'] + list(a.batch or [])
        runs = {c: [] for c in configs}
        for _ in range(a.repeat):
            for c in configs:
                try:
                    runs[c].append(run(w, a.steps, a.warmup, extra=True) if c == 'train_step' else run_batch(w, c, a.steps, a.warmup))
                except torch.cuda.OutOfMemoryError:
                    runs[c].append(None)
                torch.cuda.empty_cache()
        for c in configs:
            print(json.dumps(summarise(w, c, runs[c])), flush=True)


def summarise(workload, config, runs):
    """one run as it is; several: the median of every number, the min and max of pairs/s"""
    if any(r is None for r in runs):
        return dict(workload=workload, mode=config if config == 'train_step' else 'train_batch', batch=config if config != 'train_step'
                    else 1, out_of_memory=True)
    med = lambda xs: sorted(xs)[len(xs) // 2]
    r = dict(runs[0], mode='train_step' if config == 'train_step' else 'train_batch', repeats=len(runs))
    for k in ('steps_per_s', 'pairs_per_s', 'host_ms_per_step_median', 'max_memory_allocated_mib'):
        r[k] = med([x[k] for x in runs])
    r['stage_ms_median'] = {k: med([x['stage_ms_median'][k] for x in runs]) for k in runs[0]['stage_ms_median']}
    r['pairs_per_s_min'], r['pairs_per_s_max'] = min(x['pairs_per_s'] for x in runs), max(x['pairs_per_s'] for x in runs)
    r['skipped'] = sum(x['skipped'] for x in runs)
    return r


if __name__ == '__main__':
    main()
