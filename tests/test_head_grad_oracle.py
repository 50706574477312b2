"""CPU checks of the matching-head gradients: the numpy fp64 restatements of the hand-derived reverse sweeps (what the kernels
compute) equal torch fp64 autograd of the oracle restatements, and the backward entry points reject bad arguments before any launch."""
import ctypes

import numpy as np
import pytest
import torch

from geotransformer_b200 import _lib as L
from oracle import head_grad_oracle as HG
from oracle import loss_oracle as LO


def _autograd64(fn, inputs):
    leaves = [x.detach().double().requires_grad_(True) for x in inputs]
    fn(*leaves).backward()
    return [x.grad.numpy() for x in leaves]


def _close(got, want, rtol):
    scale = max(np.abs(want).max(), 1e-300)
    return np.abs(got - want).max() <= rtol * scale


@pytest.mark.parametrize('case', [c for c in HG.SINKHORN_CASES if c[2][0] * c[2][1] <= 1024], ids=lambda c: f'{c[0]}-{c[1]}')
def test_sinkhorn_sweep_equals_fp64_autograd(case):
    kind, seed, shape = case
    scores, rm, cm, alpha, g = HG.sinkhorn_case(kind, seed, shape)
    live = ~(~rm).all(1) | ~(~cm).all(1)
    ds, da = _autograd64(lambda s, a: (HG.sinkhorn(a, s[live], rm[live], cm[live]) * g[live].double()).sum(), [scores, alpha])
    ds_np, da_np = HG.sinkhorn_backward_np(float(alpha), scores.double().numpy(), rm.numpy(), cm.numpy(), g.double().numpy())
    # on masked lines fp64 autograd carries the rounding of 1e12 (ulp 1.2e-4) into the potentials; the sweep takes the exact limit
    rtol = 1e-3 if kind == 'upstream' else 1e-6
    assert _close(ds_np[live.numpy()], ds[live.numpy()], rtol) and abs(da_np - float(da)) <= rtol * max(abs(float(da)), 1.0)
    assert not ds_np[~live.numpy()].any()


@pytest.mark.parametrize('case', HG.PATCH_CASES, ids=lambda c: f'{c[0]}-{c[1]}')
def test_patch_scores_sweep_equals_fp64_autograd(case):
    kind, seed, shape = case
    B, P, k, C, nr, ns = shape
    rf, sf, _, ri, si, g = HG.patch_case(kind, seed, shape)
    off = torch.arange(B).repeat_interleave(P)[:, None]
    ri_g, si_g = torch.where(ri >= nr, B * nr, ri + off * nr), torch.where(si >= ns, B * ns, si + off * ns)
    want = _autograd64(lambda a, b: (HG.patch_scores(a, b, ri_g, si_g) * g.double()).sum(), [rf, sf])
    got = HG.patch_scores_backward_np(rf.numpy(), sf.numpy(), ri_g.numpy(), si_g.numpy(), g.numpy())
    assert _close(got[0], want[0], 1e-12) and _close(got[1], want[1], 1e-12)


def test_coarse_loss_sweep_equals_fp64_autograd():
    cases = [(LO.coarse_case(kind, seed, shape), LO.coarse_params(ls)) for kind, seed, shape, ls in LO.COARSE_CASES]
    cases.append((HG.duplicated_coarse_case(), LO.coarse_params(24)))
    for (rf, sf, gi, go), p in cases:
        want = _autograd64(lambda a, b: HG.coarse_loss(p, a, b, gi, go), [rf, sf])
        got = HG.coarse_backward_np(p, rf.numpy(), sf.numpy(), gi.numpy(), go.numpy())
        for w, x in zip(want, got):
            assert np.array_equal(np.isfinite(w), np.isfinite(x)) and np.array_equal(np.isnan(w), np.isnan(x))
            fin = np.isfinite(w)
            if fin.any():
                assert _close(x[fin], w[fin], 1e-9)


def test_fine_loss_sweep_equals_fp64_autograd():
    for kind, seed, shape in LO.FINE_CASES:
        rp, sp, rm, sm, sc, T = LO.fine_case(kind, seed, shape)
        want, = _autograd64(lambda s: HG.fine_loss(shape[2], rp, sp, rm, sm, s, T), [sc])
        got = HG.fine_backward_np(shape[2], rp, sp, rm, sm, shape[1] + 1, T)
        assert np.array_equal(got, want) or _close(got, want, 1e-15)


def test_backward_entry_points_reject_bad_arguments_before_any_launch():
    lib = L.lib()
    before = lib.geob200_launch_count()
    err = lambda: lib.geob200_last_error().decode()
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.addressof(buf)
    big = 1 << 40

    def sk(k=64, iters=100, inf=1e12, ws=big, g=p):
        return lib.geob200_sinkhorn_backward(p, p, p, p, 4, k, iters, inf, g, p, p, p, ws, None)
    assert sk(k=48) < 0 and 'k must be' in err()
    assert sk(iters=0) < 0 and 'num_iterations' in err()
    assert sk(inf=0.0) < 0 and 'inf' in err()
    assert sk(g=None) < 0 and 'null' in err()
    assert sk(ws=16) < 0 and 'workspace' in err()
    counts = (ctypes.c_int64 * 2)(100, 90)

    def ps(k=64, C=32, ws=big, B=1, gr=p):
        return lib.geob200_patch_scores_backward_batched(p, p, C, B, counts, p, p, 4, k, p, gr, p, p, ws, None)
    assert ps(k=48) < 0 and 'num_points_in_patch' in err()
    assert ps(C=0) < 0 and 'channels' in err()
    assert ps(B=0) < 0 and 'pairs' in err()
    assert ps(gr=None) < 0 and 'null' in err()
    assert ps(ws=16) < 0 and 'workspace' in err()
    nodes = (ctypes.c_int64 * 2)(10, 12)

    def cl(C=32, ls=24.0, ld=3, ws=big, grad=p):
        return lib.geob200_coarse_matching_loss_backward_batched(p, p, C, 1, nodes, p, p, p, 0.1, 1.4, 0.1, 1.4, ls, 0.1, grad, ld, None, p,
                                                                 p, p, ws, None)
    assert cl(C=0) < 0 and 'channels' in err()
    assert cl(ls=0.0) < 0 and 'log_scale' in err()
    assert cl(ld=2) < 0 and 'grad_ld' in err()
    assert cl(grad=None) < 0 and 'null' in err()
    assert cl(ws=16) < 0 and 'workspace' in err()

    def fl(k=64, r=0.05, ld=3, ws=big, grad=p):
        return lib.geob200_fine_matching_loss_backward_batched(p, p, p, p, p, 1, 4, k, None, r, grad, ld, None, p, p, ws, None)
    assert fl(k=32) < 0 and 'k must be' in err()
    assert fl(r=0.0) < 0 and 'positive_radius' in err()
    assert fl(ld=1) < 0 and 'grad_ld' in err()
    assert fl(grad=None) < 0 and 'null' in err()
    assert fl(ws=0) < 0 and 'workspace' in err()
    assert lib.geob200_launch_count() == before
    assert lib.geob200_sinkhorn_backward_workspace_bytes(2048, 64, 100) >= 2048 * 2 * 100 * 65 * 4


# ------------------------------------------------------------------------------------------------ against the real reference
# tests/golden/head_grads.npz holds the reference's fp32 autograd gradients (oracle/head_grad_vectors.py).  The restatements' fp32
# autograd must reproduce them (same arithmetic up to summation order); their fp64 autograd must agree to the fp32 rounding the
# reference carries, except where the reference's fp32 result is NaN (upstream gradient on masked Sinkhorn entries): there fp64 is finite.

@pytest.fixture(scope='module')
def head_grads():
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'head_grads.npz'))
    return {k: g[k] for k in g.files}


def _want(fx, key):
    return {k.split(':')[1]: v for k, v in fx.items() if k.split(':')[0] == key}


def _grads(fn, inputs, dtype):
    leaves = [x.detach().to(dtype).requires_grad_(True) for x in inputs]
    fn(*leaves).backward()
    return [x.grad for x in leaves]


def test_restatements_reproduce_reference_gradient_fixture(head_grads):
    cases = [(LO.coarse_case(k, s, sh), LO.coarse_params(ls)) for k, s, sh, ls in LO.COARSE_CASES]
    cases.append((HG.duplicated_coarse_case(), LO.coarse_params(24)))
    for i, ((rf, sf, gi, go), p) in enumerate(cases):
        g32 = _grads(lambda a, b: HG.coarse_loss(p, a, b, gi, go), [rf, sf], torch.float32)
        g64 = _grads(lambda a, b: HG.coarse_loss(p, a, b, gi, go), [rf, sf], torch.float64)
        for side, x32, x64 in zip(('ref', 'src'), g32, g64):
            want = _want(head_grads, f'coarse/{i}/{side}')
            assert HG.digest_close(HG.digest(x32), want, 1e-5), ('coarse fp32', i, side)
            # fp64 differs from the fp32 reference by the reference's own rounding (up to a few % of a row near d = 0, where the sqrt
            # backward amplifies it; the GPU tests bound the kernels by it), so here only the finite / NaN pattern must agree
            d64 = HG.digest(x64)
            assert all(np.array_equal(np.isnan(d64[k]), np.isnan(v)) for k, v in want.items()), ('coarse fp64 NaN pattern', i, side)
    for i, (kind, seed, shape) in enumerate(LO.FINE_CASES):
        rp, sp, rm, sm, sc, T = LO.fine_case(kind, seed, shape)
        for dt in (torch.float32, torch.float64):
            x, = _grads(lambda s: HG.fine_loss(shape[2], rp, sp, rm, sm, s, T), [sc], dt)
            assert HG.digest_close(HG.digest(x), _want(head_grads, f'fine/{i}'), 1e-6), ('fine', i, dt)
    for i, (kind, seed, shape) in enumerate(HG.SINKHORN_CASES):
        scores, rm, cm, alpha, g = HG.sinkhorn_case(kind, seed, shape)
        live = ~(~rm).all(1) | ~(~cm).all(1)
        ws, wa = _want(head_grads, f'sinkhorn/{i}/scores'), _want(head_grads, f'sinkhorn/{i}/alpha')
        s32 = _grads(lambda s, a: (HG.sinkhorn(a, s, rm[live], cm[live]) * g[live].to(s.dtype)).sum(), [scores[live], alpha],
                     torch.float32)
        if kind == 'upstream':
            assert int(head_grads[f'sinkhorn_nan/{i}']) > 0 and np.isnan(wa['full']).all()
            assert HG.digest_close(HG.digest(s32[0]), ws, 1e-5), 'the restatement reproduces the reference NaN pattern'
            continue
        assert int(head_grads[f'sinkhorn_nan/{i}']) == 0
        s64 = _grads(lambda s, a: (HG.sinkhorn(a, s, rm[live], cm[live]) * g[live].to(s.dtype)).sum(), [scores[live], alpha],
                     torch.float64)
        for x, tol in ((s32, 1e-5), (s64, 1e-5)):
            assert HG.digest_close(HG.digest(x[0]), ws, tol), ('sinkhorn dscores', i, kind)
            assert HG.digest_close(HG.digest(x[1].reshape(1)), wa, tol), ('sinkhorn dalpha', i, kind)
