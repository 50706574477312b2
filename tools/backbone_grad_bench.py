"""Times of the backbone backward on the device: KPConvFPN forward (no grad), forward with grad and backward of
sum_i <feats_list[i], G_i>, per block (CUDA events around each block's forward and, through autograd hooks, its backward) and
whole, against eager torch autograd of the restatement (oracle/geo_oracle.backbone) on the same GPU in fp32 with TF32 off.

    python tools/backbone_grad_bench.py [--workloads 3dmatch20k kitti20k] [--reps 10]
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


def _block_times(model, run, reps):
    """median per-block forward / backward ms of one forward-with-grad + backward"""
    fwd, bwd, ev = {}, {}, {}
    hooks = []
    for name, mod in model.backbone.named_children():
        def pre(m, inp, name=name):
            ev[name] = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ev[name][0].record()

        def post(m, inp, out, name=name):
            ev[name][1].record()
            if out.requires_grad:
                out.register_hook(lambda g, name=name: ev[name][2].record())

        hooks += [mod.register_forward_pre_hook(pre), mod.register_forward_hook(post)]
        hooks.append(mod.register_full_backward_hook(lambda m, gi, go, name=name: ev[name][3].record()))
    for _ in range(reps):
        run()
        torch.cuda.synchronize()
        for name, e in ev.items():
            fwd.setdefault(name, []).append(e[0].elapsed_time(e[1]))
            try:                                    # the first block's input takes no gradient: no backward hook there
                bwd.setdefault(name, []).append(e[2].elapsed_time(e[3]))
            except RuntimeError:
                bwd.setdefault(name, []).append(float('nan'))
    for h in hooks:
        h.remove()
    med = {n: sorted(v)[len(v) // 2] for n, v in fwd.items()}
    medb = {n: sorted(v)[len(v) // 2] for n, v in bwd.items()}
    medb = {n: (v if v > 0 else float('nan')) for n, v in medb.items()}   # the first block's input takes no gradient
    return med, medb


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
        feats = data['features']
        with torch.no_grad():
            outs = model.backbone(feats, data)
        ups = [u.cuda() for u in BG.upstream([tuple(o.shape) for o in outs])]

        def fwd_nograd():
            with torch.no_grad():
                model.backbone(feats, data)

        def fwd_bwd():
            model.zero_grad(set_to_none=True)
            sum((o * u).sum() for o, u in zip(model.backbone(feats, data), ups)).backward()

        for _ in range(3):
            fwd_nograd()
            fwd_bwd()
        t_fwd = _median_ms(fwd_nograd, args.reps)
        t_fb = _median_ms(fwd_bwd, args.reps)
        blk_f, blk_b = _block_times(model, fwd_bwd, args.reps)

        sdc = {k: (v.cuda().requires_grad_(True) if v.is_floating_point() and 'kernel_points' not in k else v.cuda())
               for k, v in sd.items() if k.startswith('backbone.')}
        dcpu = {k: v for k, v in data.items()}

        def eager():
            for v in sdc.values():
                v.grad = None
            o = G.backbone(sdc, cfg, feats, dcpu)
            sum((x * u).sum() for x, u in zip(o, ups)).backward()

        eager()
        t_eager = _median_ms(eager, max(3, args.reps // 2))
        n = data['points'][0].shape[0]
        print(f'\n{workload} ({n} points at level 1), median of {args.reps}:')
        print(f'  forward no_grad {t_fwd:.2f} ms | forward + backward {t_fb:.2f} ms (backward ~{t_fb - t_fwd:.2f} ms) | '
              f'eager torch autograd of the restatement (fp32, TF32 off) {t_eager:.2f} ms')
        print(f'  {"block":<14}{"fwd ms":>9}{"bwd ms":>9}')
        for name in blk_f:
            print(f'  {name:<14}{blk_f[name]:>9.3f}{blk_b.get(name, float("nan")):>9.3f}')


if __name__ == '__main__':
    main()
