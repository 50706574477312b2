"""Times of the geometric transformer's backward on the device, one pair: the transformer forward without grad, forward with grad
and backward of <ref_out, G_0> + <src_out, G_1> (CUDA events, median of repeats), the backward by op (kernel times from
torch.profiler in a run of its own: attention per layer, the E pass per layer and cloud, the structure-embedding backward per cloud),
and eager torch autograd of the restatement (oracle/geo_oracle.geometric_transformer) on the same GPU in fp32 with TF32 off.

    python tools/transformer_grad_bench.py [--workloads 3dmatch20k kitti20k] [--reps 10]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from geotransformer_b200.config import make_cfg                     # noqa: E402
from geotransformer_b200.model import create_model                  # noqa: E402
from geotransformer_b200.synth import make_pair                     # noqa: E402
from geotransformer_b200.utils.data import registration_collate_fn_stack_mode   # noqa: E402
from geotransformer_b200.weights import synthetic_state_dict        # noqa: E402
from oracle import backbone_grad_oracle as BG, geo_oracle as G       # noqa: E402

# kernel name fragments of the backward, by op
OPS = {'attention (q.k, softmax, P.v products)': ('att_gemm_kernel', 'att_softmax_grad_kernel'),
       'E pass': ('att_embed_grad_kernel',),
       'structure-embedding backward': ('gse_kstar_kernel', 'gse_dw_partial_kernel', 'gse_dw_fold_kernel')}


def _cuda(data):
    return {k: ([x.cuda() if isinstance(x, torch.Tensor) else x for x in v] if isinstance(v, list) else
                (v.cuda() if isinstance(v, torch.Tensor) else v)) for k, v in data.items()}


def _median_ms(fn, reps):
    ts = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def _op_times(fn, reps):
    """device ms per run of every OPS entry, all kernels together and the ten largest kernels by device time, and the kernel count
    per run, from the kernel records of ``reps`` profiled runs"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    tot = {k: 0.0 for k in OPS}
    kernels, launches, every = [], 0, 0.0
    for ev in prof.key_averages():
        if ev.device_time_total <= 0:
            continue
        ms = ev.device_time_total / 1e3 / reps
        kernels.append((ms, ev.count // reps, ev.key))
        launches += ev.count
        every += ms
        for op, frags in OPS.items():
            if any(f in ev.key for f in frags):
                tot[op] += ms
    kernels.sort(reverse=True)
    return tot, every, launches // reps, kernels[:10]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', nargs='+', default=['3dmatch20k', 'kitti20k'])
    ap.add_argument('--reps', type=int, default=10)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    print(f'device: {q.stdout.strip() or torch.cuda.get_device_name()}')
    for workload in args.workloads:
        pair = make_pair(workload, 0)
        cfg = make_cfg(pair['config'])
        model = create_model(cfg)
        sd = synthetic_state_dict(model, BG.SEED)
        model.load_state_dict(sd, strict=True)
        model = model.cuda()
        b = cfg.backbone
        limits = cfg.neighbor_limits or BG.LIMITS.get(workload) or [64] * b.num_stages
        dd = {k: pair[k] for k in ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')}
        data = _cuda(registration_collate_fn_stack_mode([dd], b.num_stages, b.init_voxel_size, b.init_radius, limits))
        with torch.no_grad():
            feats_c = model.backbone(data['features'], data)[-1]
        pts = data['points'][-1]
        n0 = int(data['lengths'][-1][0])
        rp, sp, rf, sf = pts[:n0].contiguous(), pts[n0:].contiguous(), feats_c[:n0].contiguous(), feats_c[n0:].contiguous()
        tr = model.transformer
        with torch.no_grad():
            o0, o1 = tr(rp, sp, rf, sf)
        ups = [u.cuda() for u in BG.upstream([tuple(o0.shape), tuple(o1.shape)])]

        def fwd_nograd():
            with torch.no_grad():
                tr(rp, sp, rf, sf)

        def fwd_grad():
            return tr(rp, sp, rf, sf)

        def fwd_bwd():
            model.zero_grad(set_to_none=True)
            y0, y1 = tr(rp, sp, rf, sf)
            ((y0 * ups[0]).sum() + (y1 * ups[1]).sum()).backward()

        for _ in range(3):
            fwd_nograd()
            fwd_bwd()
        t_fwd = _median_ms(fwd_nograd, args.reps)
        t_fg = _median_ms(fwd_grad, args.reps)
        t_fb = _median_ms(fwd_bwd, args.reps)
        ops, dev_fb, n_fb, top = _op_times(fwd_bwd, args.reps)
        _, dev_fg, n_fg, _ = _op_times(fwd_grad, args.reps)

        sdc = {k: (v.cuda().requires_grad_(True) if v.is_floating_point() and 'div_term' not in k else v.cuda())
               for k, v in sd.items() if k.startswith('transformer.')}

        def eager():
            for v in sdc.values():
                v.grad = None
            y0, y1 = G.geometric_transformer(sdc, cfg, rp, sp, rf, sf)
            ((y0 * ups[0]).sum() + (y1 * ups[1]).sum()).backward()

        eager()
        t_eager = _median_ms(eager, max(3, args.reps // 2))
        blocks = cfg.geotransformer.blocks
        n_self, n_cross = blocks.count('self'), blocks.count('cross')
        print(f'\n{workload}: {n0} + {pts.shape[0] - n0} superpoints, C = {tr.in_proj.out_features}, median of {args.reps}:')
        print(f'  transformer forward no_grad {t_fwd:.2f} ms | forward with grad {t_fg:.2f} ms | forward + backward {t_fb:.2f} ms '
              f'(backward ~{t_fb - t_fg:.2f} ms) | eager torch autograd of the restatement (fp32, TF32 off) {t_eager:.2f} ms')
        print(f'  backward by op (kernel time per backward): attention products {ops[list(OPS)[0]]:.3f} ms over {n_self + n_cross} '
              f'layers ({ops[list(OPS)[0]] / (n_self + n_cross):.3f} ms per layer, both clouds); E pass {ops["E pass"]:.3f} ms over '
              f'{n_self} layers x 2 clouds ({ops["E pass"] / (2 * n_self):.3f} ms each); structure-embedding backward '
              f'{ops["structure-embedding backward"]:.3f} ms for 2 clouds')
        print(f'  device time of all kernels: forward with grad {dev_fg:.2f} ms ({n_fg} kernels), forward + backward {dev_fb:.2f} ms '
              f'({n_fb} kernels); the rest of the wall time is host-side (Python, autograd, launches)')
        print('  largest kernels of forward + backward (ms per run, launches per run):')
        for ms, cnt, name in top:
            print(f'    {ms:8.3f} {cnt:5d}  {name[:110]}')


if __name__ == '__main__':
    main()
