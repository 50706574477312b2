"""Host-side cost of one pair (dev tool): cProfile of RegistrationEngine with one stream + throughput vs number of streams."""
import cProfile
import os
import pstats
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from geotransformer_b200.config import make_cfg
from geotransformer_b200.engine import RegistrationEngine
from geotransformer_b200.loss import Evaluator
from geotransformer_b200.model import create_model
from geotransformer_b200.synth import make_pair
from geotransformer_b200.weights import synthetic_state_dict

cfg = make_cfg('3dmatch')
model = create_model(cfg)
model.load_state_dict(synthetic_state_dict(model, 7351))
model = model.cuda().eval()
limits = [38, 36, 36, 38]
keys = ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')
n = int(sys.argv[1]) if len(sys.argv) > 1 else 48
pairs = [{k: torch.from_numpy(make_pair('3dmatch20k', i)[k]).pin_memory() for k in keys} for i in range(n)]
ev = Evaluator(cfg)

for s in (1, 4, 6, 8):
    eng = RegistrationEngine(model, cfg, limits, num_streams=s, evaluator=ev)
    eng.register(pairs[:max(8, 2 * s)])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    eng.register(pairs)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print(f'streams {s:2d}: {n / dt:7.1f} pairs/s  ({dt / n * 1e3:.2f} ms per pair)')
    eng.close()

# per-stage GPU time of a pair, alone and with 4 pairs in flight
for s in (1, 4):
    eng = RegistrationEngine(model, cfg, limits, num_streams=s, evaluator=ev)
    eng.register(pairs[:16])
    eng.stage_times = {}
    eng.register(pairs)
    print(f'streams {s}: per-stage ms per pair:', {k: round(sum(v) / len(v), 3) for k, v in eng.stage_times.items()},
          'total', round(sum(sum(v) / len(v) for v in eng.stage_times.values()), 3))
    eng.close()

# is the GPU the limit?  triple the Sinkhorn work (more full-GPU kernel time per pair) and compare
it0 = model.optimal_transport.num_iterations
for s, iters in ((4, it0), (4, 3 * it0), (6, it0), (6, 3 * it0)):
    model.optimal_transport.num_iterations = iters
    eng = RegistrationEngine(model, cfg, limits, num_streams=s, evaluator=ev)
    eng.register(pairs[:16])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    eng.register(pairs)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print(f'streams {s:2d}, sinkhorn iterations {iters}: {n / dt:7.1f} pairs/s  ({dt / n * 1e3:.2f} ms per pair)')
    eng.close()
model.optimal_transport.num_iterations = it0

eng = RegistrationEngine(model, cfg, limits, num_streams=1, evaluator=ev)
eng.register(pairs[:8])
torch.cuda.synchronize()
pr = cProfile.Profile()
# profile the worker body directly in this thread (cProfile does not follow pool threads)
from geotransformer_b200 import _lib
stream = eng.streams[0]
with torch.cuda.stream(stream), _lib.stream_scope(stream.cuda_stream):
    t0 = time.perf_counter()
    pr.enable()
    for p in pairs[:16]:
        eng._one(0, p, False)
    pr.disable()
    dt = time.perf_counter() - t0
print(f'single stream, profiled: {dt / 16 * 1e3:.2f} ms per pair wall')
st = pstats.Stats(pr)
st.sort_stats('tottime').print_stats(28)
