"""Training-step throughput on the device: TrainingEngine.train_step on one pair per step (synthetic weights, seed 7351).

Prints, per workload, steps/s over --steps timed steps after --warmup, the host time per step (wall clock of train_step, which ends
in its one event wait), and the median CUDA-event time of each stage: collate, forward_train, OverallLoss, backward, the gradient
guard, the fused Adam step and the metrics.  The card name and power limit are read in the same run.

    python tools/train_bench.py [--workloads 3dmatch20k kitti4k] [--steps 20] [--warmup 5]
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


def run(workload, steps, warmup):
    pair = make_pair(workload, 0)
    cfg = make_cfg(pair['config'])
    model = create_model(cfg)
    model.load_state_dict(synthetic_state_dict(model, 7351), strict=True)
    model = model.cuda()
    eng = TrainingEngine(model, cfg, BG.limits(workload))
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
    return dict(workload=workload, config=cfg.name, parameters=n_params, steps=steps, skipped=int(skipped), steps_per_s=steps / wall,
                host_ms_per_step_median=1e3 * host[len(host) // 2], stage_ms_median={k: round(v, 4) for k, v in med.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', nargs='+', default=['3dmatch20k', 'kitti4k'])
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'train_bench needs a GPU'
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    print(json.dumps({'device': q.stdout.strip() or torch.cuda.get_device_name()}))
    for w in a.workloads:
        print(json.dumps(run(w, a.steps, a.warmup)))


if __name__ == '__main__':
    main()
