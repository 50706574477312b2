"""Per-kernel GPU time per pair in batch mode (torch.profiler, CUDA activities), with the share of the per-pair stages
(grouping, ground-truth correspondences, matching, patches, Sinkhorn, LGR, Evaluator).  Dev tool.
    python tools/tail_profile.py [batch] [batches] [lanes]"""
import collections
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile

from geotransformer_b200.config import make_cfg
from geotransformer_b200.engine import RegistrationEngine
from geotransformer_b200.loss import Evaluator
from geotransformer_b200.model import create_model
from geotransformer_b200.synth import make_pair
from geotransformer_b200.weights import synthetic_state_dict

B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
NB = int(sys.argv[2]) if len(sys.argv) > 2 else 4
LANES = int(sys.argv[3]) if len(sys.argv) > 3 else 1

# kernels of the per-pair stages: everything defined in these sources except the generic helpers used by other stages too
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'geotransformer_b200', 'csrc')
TAIL = set()
for f in ('partition.cu', 'matching.cu', 'lgr.cu', 'evaluation.cu'):
    TAIL |= set(re.findall(r'__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)', open(os.path.join(CSRC, f)).read()))
TAIL -= {'gather_rows_kernel', 'pairwise_distance_kernel', 'apply_transform_kernel'}

cfg = make_cfg('3dmatch')
model = create_model(cfg)
model.load_state_dict(synthetic_state_dict(model, 7351))
model = model.cuda().eval()
keys = ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')
pairs = [{k: torch.from_numpy(make_pair('3dmatch20k', i)[k]).cuda() for k in keys} for i in range(B * (NB + 2))]
eng = RegistrationEngine(model, cfg, cfg.neighbor_limits, num_streams=LANES, evaluator=Evaluator(cfg), batch_size=B, pin_cpu=True)
eng.register(pairs[:B * 2])
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    eng.register(pairs[B * 2:])
    torch.cuda.synchronize()
eng.close()
n = B * NB
agg = collections.defaultdict(lambda: [0, 0.0])
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time > 0:
        name = re.sub(r'^void ', '', e.name).split('(')[0].split('<')[0].split('::')[-1]
        agg[name][0] += 1
        agg[name][1] += e.device_time
tot = sum(t for _, t in agg.values())
tail = sum(t for k, (_, t) in agg.items() if k in TAIL)
tail_launches = sum(c for k, (c, _) in agg.items() if k in TAIL)
print(f'{torch.cuda.get_device_name()}: batch {B}, {NB} batches, {LANES} lane(s); kernel time summed over all streams')
print(f'total {tot / n:8.1f} us/pair over {sum(c for c, _ in agg.values()) / n:.1f} kernels/pair')
print(f'per-pair stages {tail / n:8.1f} us/pair = {100 * tail / tot:.1f} % of kernel time, {tail_launches / n:.1f} kernels/pair')
for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print(f'{t / n:9.1f} us/pair {100 * t / tot:5.1f} %  {c / n:5.2f}/pair  avg {t / c:8.1f} us  {"*" if k in TAIL else " "} {k}')
