"""Tabulated structure embedding (GSE mode 5, csrc/gse_table.cu) on the GPU: accuracy against the CPU oracle next to the
tensor-core contraction (mode 3), the direct-evaluation path for arguments beyond the table, and the time of one batch-sized
launch next to the wgmma 3xFP16 kernel.  Prints one JSON line per check.  A CHECKER (lives under tests/ because it imports oracle/), not a
pytest module: ``python tests/gse_table_check.py``."""
import json
import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from geotransformer_b200 import functional as GF  # noqa: E402
from oracle import geo_oracle as G  # noqa: E402


def weights(c, g):
    return {'e.embedding.div_term': torch.exp(torch.arange(0, c, 2).float() * (-np.log(10000.0) / c)),
            'e.proj_d.weight': torch.randn(c, c, generator=g) / math.sqrt(c), 'e.proj_d.bias': torch.randn(c, generator=g) * 0.1,
            'e.proj_a.weight': torch.randn(c, c, generator=g) / math.sqrt(c), 'e.proj_a.bias': torch.randn(c, generator=g) * 0.1}


def args_of(sd, d, a):
    cu = {k: v.cuda() for k, v in sd.items()}
    return cu, (d, a, cu['e.embedding.div_term'], cu['e.proj_d.weight'], cu['e.proj_a.weight'], cu['e.proj_d.bias'], cu['e.proj_a.bias'],
                cu['e.proj_d.weight'].t().contiguous(), cu['e.proj_a.weight'].t().contiguous())


def table_of(cu, sigma_a=15, **kw):
    return GF.gse_table(cu['e.embedding.div_term'], cu['e.proj_d.weight'].t().contiguous(), cu['e.proj_a.weight'].t().contiguous(),
                        cu['e.proj_d.bias'], cu['e.proj_a.bias'], sigma_a, **kw)


def accuracy(c, n, sigma_d, extent, seed):
    g = torch.Generator().manual_seed(seed)
    pts = torch.rand(n, 3, generator=g) * extent
    sd = weights(c, g)
    want = G.structure_embedding(sd, 'e.', pts, sigma_d, 15, 3)
    d, a = GF.gse_indices(pts.cuda(), sigma_d, 15, 3)
    cu, args = args_of(sd, d, a)
    out = {'check': 'accuracy', 'channels': c, 'n': n, 'max_d_index': float(d.max())}
    for name, kw in (('table', {}), ('table_inv_step_64', {'inv_step': 64}), ('table_mostly_direct', {'d_max': float(d.max()) * 0.5})):
        got = GF.gse_embed(*args, mode=5, table=table_of(cu, **kw)).cpu()
        out[name + '_vs_oracle'] = float((got - want).abs().max())
    out['tensor_core_3xfp16_vs_oracle'] = float((GF.gse_embed(*args, mode=3).cpu() - want).abs().max())
    out['scale'] = float(want.abs().max())
    print(json.dumps(out), flush=True)


def timing(c, clouds, n, reps=5):
    g = torch.Generator().manual_seed(3)
    sd = weights(c, g)
    pts = (torch.rand(clouds * n, 3, generator=g) * 4.0).cuda()
    tot = clouds * n * n
    d_all, a_all = torch.empty(tot, device='cuda'), torch.empty(tot, 3, device='cuda')
    GF.gse_indices_batched(pts, [n] * clouds, 0.2, 15, 3, d_all, a_all)
    cu, args = args_of(sd, d_all, a_all)
    E3, E5 = torch.empty(tot, c, device='cuda'), torch.empty(tot, c, device='cuda')
    tab = table_of(cu)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    res = {'check': 'timing', 'channels': c, 'clouds': clouds, 'n': n, 'rows': tot, 'table_MB': tab.blob.numel() / 1e6}
    for mode, E, kw in ((3, E3, {}), (5, E5, {'table': tab})):
        ms = []
        for r in range(reps + 1):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            GF.gse_embed_flat(d_all, a_all, tot, *args[2:], E, mode=mode, **kw)
            e.record()
            e.synchronize()
            if r:
                ms.append(s.elapsed_time(e))
        res[f'mode{mode}_ms'] = sorted(ms)[len(ms) // 2]
    res['max_abs_diff_table_vs_tensor_core'] = float((E3 - E5).abs().max())
    res['E_write_GBps_table'] = tot * c * 4 / (res['mode5_ms'] * 1e-3) / 1e9
    res['node_read_GBps_table'] = tot * 4 * c * 6 / (res['mode5_ms'] * 1e-3) / 1e9
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    accuracy(256, 100, 0.2, 2.0, 1)
    accuracy(128, 173, 4.8, 20.0, 9)
    accuracy(256, 7, 0.2, 2.0, 7)
    timing(256, 16, 317)
    timing(128, 8, 1000, reps=3)
