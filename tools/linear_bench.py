"""Micro-benchmark of the tensor-core (wgmma) Linear (dev tool): CUDA-event time per call for the GEMM shapes of the 3DMatch model.
Run from any checkout: uses the package next to this file's parent directory (or GEOB_ROOT).

    python tools/linear_bench.py                  time the shapes below
    python tools/linear_bench.py --save F.npz     write the outputs of the GEMM paths on seeded inputs (see cases())
    python tools/linear_bench.py --compare F.npz  recompute them and compare bit for bit with F.npz (exit 1 on any difference)

--save with GEOB_ROOT pointing at another checkout records that build's outputs, so two builds can be compared bitwise."""
import argparse
import os
import sys

ROOT = os.environ.get('GEOB_ROOT', os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from geotransformer_b200 import functional as GF

SHAPES = [(40000, 64, 32), (40000, 480, 32), (40000, 32, 128), (40000, 64, 128), (12000, 960, 64), (12000, 64, 256), (3400, 1920, 128),
          (3400, 128, 512), (640, 3840, 256), (640, 256, 1024), (640, 1024, 256), (640, 256, 768), (320, 256, 256), (640, 256, 512)]

# (m, k, n) of every GEMM weight shape of the 3DMatch forward at batch 8 (m = the largest row count it runs at)
FORWARD_SHAPES = [(27945, 1536, 512), (98729, 960, 64), (27945, 1920, 128), (98729, 768, 256), (27945, 256, 512), (320000, 480, 32),
                  (5158, 3840, 256), (5158, 256, 256), (5158, 512, 256), (98729, 64, 256), (27945, 128, 512), (98729, 256, 64)]


def _lib():
    from geotransformer_b200 import _lib
    return _lib.lib()


def _gen(seed):
    g = torch.Generator(device='cuda')
    g.manual_seed(seed)
    return g


def _randn(g, *shape):
    return torch.randn(*shape, device='cuda', generator=g)


def _linear_case(seed, m, k, n, relu=False, ldx=None):
    g = _gen(seed)
    x = _randn(g, m, ldx or k)[:, :k]
    w = _randn(g, n, k) * (1.0 / k ** 0.5)
    b = _randn(g, n)
    return {'y': GF.linear(x, w, b, relu=relu)}


def _linear_gn_case(seed, m, k, n, groups, leaky):
    g = _gen(seed)
    x = _randn(g, m, k)
    w = _randn(g, n, k) * (1.0 / k ** 0.5)
    b, gamma, beta = _randn(g, n), _randn(g, n), _randn(g, n)
    y = GF.linear_group_norm(x, w, b, gamma, beta, groups, negative_slope=0.1 if leaky else None)
    return {'y': y, 'pre_norm': GF.scratch((m, n), x.device, 'pre_norm')}


def _kpconv_inputs(g, m, ns, cin, cout, h=24):
    s_points = torch.rand(ns, 3, device='cuda', generator=g) * 2.0
    q_points = s_points[:m].contiguous() if m <= ns else torch.rand(m, 3, device='cuda', generator=g) * 2.0
    nbr = torch.randint(0, ns + 1, (m, h), device='cuda', generator=g)         # ns = no neighbour (sentinel)
    s_feats = torch.relu(_randn(g, ns, cin))
    kp = (torch.rand(15, 3, device='cuda', generator=g) - 0.5) * 0.2
    weights = _randn(g, 15, cin, cout) * (1.0 / (15 * cin) ** 0.5)
    bias = _randn(g, cout)
    return s_feats, q_points, s_points, nbr, kp, weights, bias


def _kpconv_case(seed, m, ns, cin, cout):
    g = _gen(seed)
    s_feats, q_points, s_points, nbr, kp, weights, bias = _kpconv_inputs(g, m, ns, cin, cout)
    return {'y': GF.kpconv(s_feats, q_points, s_points, nbr, kp, weights, bias, 0.5)}


def _kpconv_gn_case(seed, m, ns, cin, cout, groups):
    g = _gen(seed)
    s_feats, q_points, s_points, nbr, kp, weights, bias = _kpconv_inputs(g, m, ns, cin, cout)
    gamma, beta = _randn(g, cout), _randn(g, cout)
    y = GF.kpconv_group_norm(s_feats, q_points, s_points, nbr, kp, weights, bias, 0.5, gamma, beta, groups)
    return {'y': y, 'pre_norm': GF.scratch((m, cout), s_feats.device, 'pre_norm')}


class _setting:
    """geob200_set_linear_persistent / geob200_set_split_k for the duration of a case (both default to on)"""

    def __init__(self, persistent=True, split_k=True):
        self.p, self.s = persistent, split_k

    def __enter__(self):
        _lib().geob200_set_linear_persistent(int(self.p))
        _lib().geob200_set_split_k(int(self.s))

    def __exit__(self, *a):
        _lib().geob200_set_linear_persistent(1)
        _lib().geob200_set_split_k(1)


def cases():
    """name -> (setting, callable returning a dict of tensors); seeded inputs, so every build computes the same problems"""
    c = {}
    for i, (m, k, n) in enumerate(FORWARD_SHAPES):
        c[f'fwd_{m}x{k}->{n}'] = (_setting(), lambda i=i, m=m, k=k, n=n: _linear_case(100 + i, m, k, n))
        c[f'fwd_{m}x{k}->{n}_persistent_off'] = (_setting(persistent=False), lambda i=i, m=m, k=k, n=n: _linear_case(100 + i, m, k, n))
    for n in (32, 48, 64, 96, 128, 256, 512, 1024):
        c[f'n{n}'] = (_setting(), lambda n=n: _linear_case(200 + n, 3001, 96, n))
        c[f'n{n}_relu'] = (_setting(), lambda n=n: _linear_case(300 + n, 20000, 160, n, relu=True))
    for k in (4, 36, 100, 250, 1000):                       # K not a multiple of the 32-wide chunk
        c[f'k{k}'] = (_setting(), lambda k=k: _linear_case(400 + k, 4099, k, 128))
    for m in (64, 65, 127, 129, 200, 1037):                 # M tails
        c[f'm{m}'] = (_setting(), lambda m=m: _linear_case(500 + m, m, 256, 256))
    for ldx in (132, 200):                                  # column slices of a wider row-major tensor
        c[f'ldx{ldx}'] = (_setting(), lambda ldx=ldx: _linear_case(600 + ldx, 5000, 128, 96, ldx=ldx))
    for (m, k, n) in ((640, 3840, 256), (320, 1024, 256), (640, 1024, 64), (200, 2000, 128)):   # split-K shapes
        c[f'splitk_{m}x{k}->{n}'] = (_setting(), lambda m=m, k=k, n=n: _linear_case(700 + k, m, k, n))
        c[f'splitk_off_{m}x{k}->{n}'] = (_setting(split_k=False), lambda m=m, k=k, n=n: _linear_case(700 + k, m, k, n))
    for (m, k, n, groups, leaky) in ((27945, 256, 512, 32, True), (98729, 64, 256, 32, False), (5000, 128, 64, 32, True),
                                     (3001, 96, 32, 8, True), (640, 1024, 256, 32, False)):
        c[f'linear_gn_{m}x{k}->{n}_g{groups}'] = (_setting(), lambda m=m, k=k, n=n, g=groups, l=leaky: _linear_gn_case(800 + n, m, k, n, g, l))
    for (m, ns, cin, cout) in ((20000, 24000, 32, 32), (8000, 20000, 64, 64), (3000, 8000, 128, 128), (1000, 3000, 256, 256),
                               (1037, 2000, 32, 64), (700, 1000, 64, 128)):
        c[f'kpconv_{m}_{cin}->{cout}'] = (_setting(), lambda m=m, ns=ns, a=cin, b=cout: _kpconv_case(900 + a + b, m, ns, a, b))
        c[f'kpconv_gn_{m}_{cin}->{cout}'] = (_setting(), lambda m=m, ns=ns, a=cin, b=cout: _kpconv_gn_case(950 + a + b, m, ns, a, b, 32))
    return c


def run_cases():
    out = {}
    for name, (setting, fn) in cases().items():
        with setting:
            res = fn()
            torch.cuda.synchronize()
        for key, t in res.items():
            out[f'{name}/{key}'] = t.detach().contiguous().cpu().numpy().copy()
    return out


def compare(path):
    want = np.load(path)
    got = run_cases()
    bad = 0
    for key in sorted(set(want.files) | set(got)):
        if key not in want.files or key not in got:
            print(f'{key}: missing in {"saved" if key not in want.files else "this build"}')
            bad += 1
            continue
        a, b = want[key], got[key]
        if a.shape != b.shape or a.dtype != b.dtype:
            print(f'{key}: shape/dtype {a.shape} {a.dtype} vs {b.shape} {b.dtype}')
            bad += 1
            continue
        ndiff = int(np.count_nonzero(np.any(a.view(np.uint8).reshape(a.size, -1) != b.view(np.uint8).reshape(b.size, -1), axis=1)) if a.size else 0)
        if ndiff:
            bad += 1
        print(f'{key}: {a.size} values, {ndiff} with differing bits')
    print(f'compared {len(got)} arrays: {"all bit-identical" if bad == 0 else f"{bad} differ"}')
    return bad == 0


def bench():
    if os.environ.get('GEOB200_LINEAR_PERSISTENT'):
        _lib().geob200_set_linear_persistent(1)
        print('persistent tile loop ON')
    for m, k, n in SHAPES:
        x = torch.randn(m, k, device='cuda')
        w = torch.randn(n, k, device='cuda')
        b = torch.randn(n, device='cuda')
        out = torch.empty(m, n, device='cuda')
        for _ in range(5):
            GF.linear(x, w, b, out=out)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(50):
            GF.linear(x, w, b, out=out)
        e1.record()
        torch.cuda.synchronize()
        print(f'{m:6d} x {k:5d} -> {n:5d}: {e0.elapsed_time(e1) / 50 * 1e3:8.1f} us')


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--save', metavar='FILE.npz')
    ap.add_argument('--compare', metavar='FILE.npz')
    args = ap.parse_args()
    print('root', ROOT)
    if args.save:
        np.savez(args.save, **run_cases())
        print('saved', args.save)
    elif args.compare:
        sys.exit(0 if compare(args.compare) else 1)
    else:
        bench()
