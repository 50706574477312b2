"""Cost of building ModelNet validation / test pairs on the device against the reference's numpy path.

Times ``functional.modelnet_benchmark_pairs_batched`` on a split-sized list of synthetic 2 048-point shapes already on the device
(CUDA events, median of repeats), and the numpy restatement (oracle/modelnet_benchmark_oracle.py, the reference's per-pair numpy
work) per pair on one host core.  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/modelnet_benchmark_bench.py [--pairs 1200] [--repeat 5] [--host-pairs 50]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from geotransformer_b200 import functional as GF                    # noqa: E402
from oracle import modelnet_benchmark_oracle as MB                  # noqa: E402
from tools.augment_bench import card                                # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', type=int, default=1200)
    ap.add_argument('--repeat', type=int, default=5)
    ap.add_argument('--host-pairs', type=int, default=50)
    a = ap.parse_args()
    shapes = [s['points'] for s in MB.synthetic_shapes(a.pairs, seed=1, small_every=0)]
    raw = torch.from_numpy(np.concatenate(shapes)).cuda()
    lengths, indices = [len(s) for s in shapes], list(range(a.pairs))

    def build():
        return GF.modelnet_benchmark_pairs_batched(raw, lengths, indices, 717, 0.7, 45.0, 0.5, 0.05)

    build()
    times = []
    for _ in range(a.repeat):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        build()
        e.record()
        e.synchronize()
        times.append(s.elapsed_time(e))
    os.sched_setaffinity(0, {sorted(os.sched_getaffinity(0))[0]})
    t0 = time.perf_counter()
    for i in range(a.host_pairs):
        MB.benchmark_pair(shapes[i], i)
    host_ms = (time.perf_counter() - t0) * 1e3 / a.host_pairs
    dev_ms = float(np.median(times))
    print(json.dumps({'card': card(), 'pairs': a.pairs, 'device_ms': round(dev_ms, 3), 'device_ms_per_pair': round(dev_ms / a.pairs, 5),
                      'device_ms_spread': [round(min(times), 3), round(max(times), 3)], 'host_ms_per_pair_one_core': round(host_ms, 3),
                      'host_ms_split_one_core': round(host_ms * a.pairs, 1)}))


if __name__ == '__main__':
    main()
