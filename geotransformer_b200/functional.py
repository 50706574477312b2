"""Thin torch-tensor wrappers over the C ABI (``include/geob200.h``).

PyTorch is used here only for device memory and the current stream; every computation is a hand-written
sm_90a kernel inside ``libgeob200.so``.  All functions require CUDA tensors and raise ``RuntimeError`` otherwise
(there is no CPU path in the product).
"""
import ctypes
import math

import torch

from . import _lib as L

_f32, _i64, _u8, _i32 = torch.float32, torch.int64, torch.uint8, torch.int32

# default ``mode`` of the structure embedding: 5 = tabulated projections (geob200_gse_embed_table: no contraction at all) when
# the caller passes the ``table`` of the weights (``gse_table``; the modules build and cache it), the contraction without one;
# 3 = always the contraction (geob200_gse_embed_pairs: wgmma 3xFP16 for C = 128 and 256, a generic fp32 kernel for other
# widths).  tests/gse_table_check.py compares the accuracy and launch time of the two.
GSE_MODE = 5
# tabulation grid of mode 5: step 1 / GSE_TABLE_INV_STEP index units (power of two), distance indices up to GSE_TABLE_D_MAX
# (larger ones are evaluated directly inside the kernel: correct, slow)
GSE_TABLE_INV_STEP = 256
GSE_TABLE_D_MAX = 96.0

# Optional per-op CUDA-event timing on the launching stream (bench.py sets EVENTS = {} to collect
# {op name: [(start_event, end_event), ...]}; None = off, zero overhead).
EVENTS = None


class _timed:
    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if EVENTS is not None:
            self.s = torch.cuda.Event(enable_timing=True)
            self.e = torch.cuda.Event(enable_timing=True)
            self.s.record()
        return self

    def __exit__(self, *a):
        if EVENTS is not None:
            self.e.record()
            EVENTS.setdefault(self.name, []).append((self.s, self.e))
        return False


def _f(t, name):
    L.require_cuda(t, name, _f32)
    return t


def _detach(t):
    return t.detach() if t is not None and t.requires_grad else t


def _needs_grad(*ts):
    """the autograd path of the differentiable ops: grad mode on and an input requiring grad (else the value-only path, same kernels)"""
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in ts)


_GN_WS = {}


def _gn_workspace(device, groups, rows=0, channels=0, n_pairs=1):
    """zero-initialised (ticket) GroupNorm scratch per (device, stream, groups); large enough for the statistics of a
    (rows, channels) activation produced by the GEMM epilogue (geob200_fused_group_norm_workspace_bytes) and the per-pair
    mean / rstd of a batch of n_pairs pairs"""
    key = (device.index, L.stream_ptr(), groups)
    lib = L.lib()
    need = lib.geob200_fused_group_norm_workspace_bytes(rows, channels, groups) if rows else lib.geob200_group_norm_workspace_bytes(groups)
    need += 8 * groups * max(int(n_pairs), 1) + 1024
    ws = _GN_WS.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.zeros(max(int(need * 1.5), 1 << 20), dtype=_u8, device=device)
        _GN_WS[key] = ws
    return ws


# ------------------------------------------------------------------------------------------------ backbone

# KPConv formulation: 'tc' = gather kernel + wgmma 3xTF32 GEMM (default where the shape allows), 'fused' = single fp32 kernel
KPCONV_MODE = 'tc'


def kpconv(s_feats, q_points, s_points, neighbor_indices, kernel_points, weights, bias, sigma, weights_t=None):
    """weights_t: optional cached (c_out, 15*c_in) transpose of the weights for the tensor-core path.  Differentiable w.r.t.
    ``s_feats``, ``weights`` and ``bias`` (``kpconv_backward``)."""
    if _needs_grad(s_feats, weights, bias):
        return _KPConv.apply(s_feats, weights, bias, q_points, s_points, neighbor_indices, kernel_points, float(sigma), weights_t)
    return _kpconv(s_feats, q_points, s_points, neighbor_indices, kernel_points, weights, bias, sigma, weights_t)


def _kpconv(s_feats, q_points, s_points, neighbor_indices, kernel_points, weights, bias, sigma, weights_t=None):
    s_feats, weights, bias = _detach(s_feats), _detach(weights), _detach(bias)
    _f(s_feats, 's_feats'); _f(q_points, 'q_points'); _f(s_points, 's_points')
    L.require_cuda(neighbor_indices, 'neighbor_indices', _i64)
    m, h = neighbor_indices.shape
    ns = s_points.shape[0]
    k, cin, cout = weights.shape
    out = torch.empty((m, cout), dtype=_f32, device=s_feats.device)
    lib = L.lib()
    if (KPCONV_MODE == 'tc' and cin % 32 == 0 and cout % 16 == 0 and cout >= 32 and (cout <= 128 or cout % 128 == 0) and m >= 64):
        if weights_t is None:
            weights_t = weights.reshape(k * cin, cout).t().contiguous()
        ws = L.workspace(lib.geob200_kpconv_tc_workspace_bytes(m, ns, cin), s_feats.device, 'kpconv_tc')
        L.check(lib.geob200_kpconv_tc(s_feats.data_ptr(), q_points.data_ptr(), s_points.data_ptr(), neighbor_indices.data_ptr(), m, ns,
                                      h, kernel_points.data_ptr(), k, weights_t.data_ptr(), L.ptr(bias), cin, cout, float(sigma),
                                      out.data_ptr(), ws.data_ptr(), ws.numel(), L.stream_ptr()), 'kpconv_tc')
        return out
    ws = L.workspace(lib.geob200_kpconv_workspace_bytes(ns), s_feats.device, 'kpconv')
    L.check(lib.geob200_kpconv(s_feats.data_ptr(), q_points.data_ptr(), s_points.data_ptr(),
                               neighbor_indices.data_ptr(), m, ns, h, kernel_points.data_ptr(), k,
                               weights.data_ptr(), L.ptr(bias), cin, cout, float(sigma), out.data_ptr(),
                               ws.data_ptr(), ws.numel(), L.stream_ptr()), 'kpconv')
    return out


def kpconv_backward(s_feats, q_points, s_points, neighbor_indices, kernel_points, weights, sigma, grad_out, need_feats=True,
                    need_weights=True, need_bias=True):
    """(grad_s_feats, grad_weights, grad_bias) of ``kpconv`` for the upstream gradient ``grad_out`` (n_query, c_out); the neighbour
    count n_valid is the forward's, a constant.  A gradient not requested is None."""
    for t, name in ((s_feats, 's_feats'), (q_points, 'q_points'), (s_points, 's_points'), (kernel_points, 'kernel_points'),
                    (weights, 'weights'), (grad_out, 'grad_out')):
        _f(_detach(t), name)
    L.require_cuda(neighbor_indices, 'neighbor_indices', _i64)
    s_feats, weights = _detach(s_feats), _detach(weights)
    m, h = neighbor_indices.shape
    ns = s_points.shape[0]
    k, cin, cout = weights.shape
    if tuple(grad_out.shape) != (m, cout) or tuple(s_feats.shape) != (ns, cin):
        raise RuntimeError(f'kpconv_backward: grad_out must be ({m}, {cout}) and s_feats ({ns}, {cin})')
    dev = s_feats.device
    gf = torch.empty((ns, cin), dtype=_f32, device=dev) if need_feats else None
    gw = torch.empty((k, cin, cout), dtype=_f32, device=dev) if need_weights else None
    gb = torch.empty((cout,), dtype=_f32, device=dev) if need_bias else None
    lib = L.lib()
    ws = L.workspace(lib.geob200_kpconv_backward_workspace_bytes(m, ns, h, cin, cout), dev, 'kpconv_backward')
    L.check(lib.geob200_kpconv_backward(s_feats.data_ptr(), q_points.data_ptr(), s_points.data_ptr(), neighbor_indices.data_ptr(), m, ns, h,
                                        kernel_points.data_ptr(), k, weights.data_ptr(), cin, cout, float(sigma), grad_out.data_ptr(),
                                        L.ptr(gf), L.ptr(gw), L.ptr(gb), ws.data_ptr(), ws.numel(), L.stream_ptr()), 'kpconv_backward')
    return gf, gw, gb


class _KPConv(torch.autograd.Function):
    @staticmethod
    def forward(ctx, s_feats, weights, bias, q_points, s_points, neighbor_indices, kernel_points, sigma, weights_t):
        ctx.save_for_backward(s_feats, weights, q_points, s_points, neighbor_indices, kernel_points)
        ctx.sigma = sigma
        return _kpconv(s_feats, q_points, s_points, neighbor_indices, kernel_points, weights, bias, sigma, weights_t)

    @staticmethod
    def backward(ctx, grad):
        s_feats, weights, q, s, nbr, kp = ctx.saved_tensors
        nf, nw, nb = ctx.needs_input_grad[:3]
        gf, gw, gb = kpconv_backward(s_feats, q, s, nbr, kp, weights, ctx.sigma, grad.contiguous(), nf, nw, nb)
        return gf, gw, gb, None, None, None, None, None, None


def linear(x, weight, bias=None, relu=False, out=None):
    """y = x @ weight.T + bias (ReLU'd with ``relu``); x may be a column slice of a wider row-major tensor (stride(1) == 1).
    Differentiable w.r.t. ``x``, ``weight`` and ``bias`` (``linear_backward``); with ``out`` the result is copied into it, which
    then carries the graph."""
    if _needs_grad(x, weight, bias):
        y = _Linear.apply(x, weight, bias, bool(relu))
        return y if out is None else out.copy_(y)
    return _linear(x, weight, bias, relu, out)


def _linear(x, weight, bias=None, relu=False, out=None):
    x, weight, bias = _detach(x), _detach(weight), _detach(bias)
    if not x.is_cuda or x.dtype != _f32 or x.stride(1) != 1:
        raise RuntimeError('linear: x must be a float32 CUDA tensor with unit inner stride')
    L.require_cuda(weight, 'weight', _f32)
    m, k = x.shape
    n = weight.shape[0]
    if out is None:
        out = torch.empty((m, n), dtype=_f32, device=x.device)
    L.check(L.lib().geob200_linear(x.data_ptr(), x.stride(0), weight.data_ptr(), L.ptr(bias), out.data_ptr(),
                                   out.stride(0), m, n, k, int(relu), L.stream_ptr()), 'linear')
    return out


def linear_backward(x, weight, grad_y, need_x=True, need_weight=True, need_bias=True, relu_y=None):
    """(grad_x (m, k), grad_weight (n, k), grad_bias (n,)) of ``linear`` for the upstream gradient ``grad_y`` (m, n); x may be a column
    slice; ``relu_y``: the forward's output when it applied the ReLU.  grad_x runs through the forward's GEMM (3xTF32 on the tensor
    cores where the shape allows), grad_weight / grad_bias are fp32 sums over the rows in a fixed order.  An output not requested is
    None."""
    x, weight = _detach(x), _detach(weight)
    if not x.is_cuda or x.dtype != _f32 or x.stride(1) != 1:
        raise RuntimeError('linear_backward: x must be a float32 CUDA tensor with unit inner stride')
    L.require_cuda(weight, 'weight', _f32); _f(grad_y, 'grad_y')
    m, k = x.shape
    n = weight.shape[0]
    if tuple(grad_y.shape) != (m, n) or weight.shape[1] != k:
        raise RuntimeError(f'linear_backward: grad_y must be ({m}, {n}) and weight ({n}, {k})')
    if relu_y is not None:
        _f(relu_y, 'relu_y')
        if tuple(relu_y.shape) != (m, n):
            raise RuntimeError(f'linear_backward: relu_y must be ({m}, {n})')
    dev = x.device
    wt = weight.t().contiguous() if need_x else None
    gx = torch.empty((m, k), dtype=_f32, device=dev) if need_x else None
    gw = torch.empty((n, k), dtype=_f32, device=dev) if need_weight else None
    gb = torch.empty((n,), dtype=_f32, device=dev) if need_bias else None
    lib = L.lib()
    ws = L.workspace(lib.geob200_linear_backward_workspace_bytes(m, n, k, int(relu_y is not None)), dev, 'linear_backward')
    L.check(lib.geob200_linear_backward(x.data_ptr(), x.stride(0), L.ptr(wt), L.ptr(_detach(relu_y)), m, n, k, grad_y.data_ptr(), L.ptr(gx),
                                        L.ptr(gw), L.ptr(gb), ws.data_ptr(), ws.numel(), L.stream_ptr()), 'linear_backward')
    return gx, gw, gb


class _Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, relu):
        y = _linear(x, weight, bias, relu)
        ctx.save_for_backward(x, weight, y if relu else None)
        return y

    @staticmethod
    def backward(ctx, grad):
        x, weight, y = ctx.saved_tensors
        return (*linear_backward(x, weight, grad.contiguous(), *ctx.needs_input_grad[:3], relu_y=y), None)


def split_tf32(weight):
    """(n, k) fp32 weight -> (2n, k) image [hi; lo]: hi = weight rounded to tf32 (nearest, ties away from zero), lo = weight - hi.
    The operand layout in which the tensor-core GEMM reads its weights."""
    weight = _detach(weight)
    if not weight.is_cuda or weight.dtype != _f32 or weight.dim() != 2 or weight.stride(1) != 1:
        raise RuntimeError('split_tf32: weight must be a 2-D float32 CUDA tensor with unit inner stride')
    n, k = weight.shape
    out = torch.empty((2 * n, k), dtype=_f32, device=weight.device)
    L.check(L.lib().geob200_split_tf32(weight.data_ptr(), weight.stride(0), n, k, out.data_ptr(), L.stream_ptr()), 'split_tf32')
    return out


def group_norm(x, weight, bias, groups, eps=1e-5, negative_slope=None, residual=None, cloud_rows=None):
    """leaky(GroupNorm(x) + residual) over all rows (one pair), or with per-pair statistics given ``cloud_rows`` (2B host ints, as
    ``group_norm_batched``); differentiable w.r.t. x, weight, bias and residual"""
    if _needs_grad(x, weight, bias, residual):
        return _GroupNorm.apply(x, weight, bias, residual, int(groups), float(eps), negative_slope, cloud_rows)
    if cloud_rows is not None:
        return group_norm_batched(x, weight, bias, groups, cloud_rows, eps, negative_slope, _detach(residual))
    return _group_norm(x, weight, bias, groups, eps, negative_slope, residual)


def group_norm_backward_batched(x, y, weight, groups, cloud_rows, grad_y, eps=1e-5, negative_slope=None, need_residual=False,
                                need_weight=True, need_bias=True):
    """(grad_x, grad_weight, grad_bias, grad_residual) of ``leaky(GroupNorm(x) + residual)`` with per-pair statistics (``cloud_rows``:
    2B host ints, as ``group_norm_batched``; one pair: ``[n_rows, 0]``).  ``x`` is the pre-norm input and ``y`` the forward's output
    (its sign gives the LeakyReLU's derivative).  The statistics are recomputed from x; every sum runs in a fixed order."""
    x, y, weight = _detach(x), _detach(y), _detach(weight)
    _f(x, 'x'); _f(weight, 'weight'); _f(grad_y, 'grad_y')
    leaky = negative_slope is not None
    if leaky:
        _f(y, 'y')
    n, c = x.shape
    if tuple(grad_y.shape) != (n, c) or (leaky and tuple(y.shape) != (n, c)):
        raise RuntimeError(f'group_norm_backward_batched: grad_y and y must be ({n}, {c})')
    dev = x.device
    np_ = len(cloud_rows) // 2
    gx = torch.empty_like(x)
    gw = torch.empty((c,), dtype=_f32, device=dev) if need_weight else None
    gb = torch.empty((c,), dtype=_f32, device=dev) if need_bias else None
    gr = torch.empty_like(x) if need_residual else None
    lib = L.lib()
    ws = L.workspace(lib.geob200_group_norm_backward_batched_workspace_bytes(n, c, groups, np_), dev, 'group_norm_backward')
    L.check(lib.geob200_group_norm_backward_batched(x.data_ptr(), L.ptr(y) if leaky else None, n, c, groups, weight.data_ptr(), float(eps),
                                                    int(leaky), float(negative_slope or 0.0), grad_y.data_ptr(), gx.data_ptr(), L.ptr(gw),
                                                    L.ptr(gb), L.ptr(gr), ws.data_ptr(), ws.numel(), L.stream_ptr(), np_,
                                                    _host_i64(cloud_rows)), 'group_norm_backward_batched')
    return gx, gw, gb, gr


class _GroupNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, residual, groups, eps, negative_slope, cloud_rows):
        if cloud_rows is None:
            y = _group_norm(x, weight, bias, groups, eps, negative_slope, residual)
        else:
            y = group_norm_batched(x, weight, bias, groups, cloud_rows, eps, negative_slope, _detach(residual))
        ctx.save_for_backward(x, y, weight)
        ctx.args = (groups, eps, negative_slope, _seg_rows(cloud_rows, x.shape[0]))
        return y

    @staticmethod
    def backward(ctx, grad):
        x, y, weight = ctx.saved_tensors
        groups, eps, slope, rows = ctx.args
        need = ctx.needs_input_grad
        gx, gw, gb, gr = group_norm_backward_batched(x, y, weight, groups, rows, grad.contiguous(), eps, slope, need[3], need[1], need[2])
        return gx if need[0] else None, gw, gb, gr, None, None, None, None


def _seg_rows(cloud_rows, n_rows):
    """the per-pair row layout the backward entry points take: ``cloud_rows``, or one pair of all rows"""
    return [n_rows, 0] if cloud_rows is None else [int(r) for r in cloud_rows]


def _group_norm(x, weight, bias, groups, eps=1e-5, negative_slope=None, residual=None):
    x, weight, bias, residual = _detach(x), _detach(weight), _detach(bias), _detach(residual)
    _f(x, 'x')
    n, c = x.shape
    ws = _gn_workspace(x.device, groups)
    y = torch.empty_like(x)
    L.check(L.lib().geob200_group_norm(x.data_ptr(), n, c, groups, weight.data_ptr(), bias.data_ptr(), float(eps),
                                       L.ptr(residual), int(negative_slope is not None),
                                       float(negative_slope or 0.0), y.data_ptr(), ws.data_ptr(), ws.numel(),
                                       L.stream_ptr()), 'group_norm')
    return y


def linear_group_norm(x, weight, bias, gn_weight, gn_bias, groups, eps=1e-5, negative_slope=None, residual=None, cloud_rows=None):
    """UnaryBlock: leaky(GroupNorm(x @ weight.T + bias) + residual); statistics from the GEMM epilogue on the wgmma path, per pair
    with ``cloud_rows`` (``linear_group_norm_batched``).  Differentiable w.r.t. every float input (the autograd path keeps its own
    copy of the pre-norm activation)."""
    if _needs_grad(x, weight, bias, gn_weight, gn_bias, residual):
        return _LinearGroupNorm.apply(x, weight, bias, gn_weight, gn_bias, residual, int(groups), float(eps), negative_slope, cloud_rows)
    if cloud_rows is not None:
        return linear_group_norm_batched(x, weight, bias, gn_weight, gn_bias, groups, cloud_rows, eps, negative_slope, _detach(residual))
    return _linear_group_norm(x, weight, bias, gn_weight, gn_bias, groups, eps, negative_slope, residual)


class _LinearGroupNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, gn_weight, gn_bias, residual, groups, eps, negative_slope, cloud_rows):
        pre = torch.empty((x.shape[0], weight.shape[0]), dtype=_f32, device=x.device)
        if cloud_rows is None:
            y = _linear_group_norm(x, weight, bias, gn_weight, gn_bias, groups, eps, negative_slope, residual, pre=pre)
        else:
            y = linear_group_norm_batched(x, weight, bias, gn_weight, gn_bias, groups, cloud_rows, eps, negative_slope, _detach(residual),
                                          pre=pre)
        ctx.save_for_backward(x, weight, gn_weight, pre, y)
        ctx.args = (groups, eps, negative_slope, _seg_rows(cloud_rows, pre.shape[0]))
        return y

    @staticmethod
    def backward(ctx, grad):
        x, weight, gn_weight, pre, y = ctx.saved_tensors
        groups, eps, slope, rows = ctx.args
        need = ctx.needs_input_grad
        gpre, ggw, ggb, gr = group_norm_backward_batched(pre, y, gn_weight, groups, rows, grad.contiguous(), eps, slope, need[5], need[3],
                                                         need[4])
        gx, gw, gb = linear_backward(x, weight, gpre, need[0], need[1], need[2]) if any(need[:3]) else (None, None, None)
        return gx, gw, gb, ggw, ggb, gr, None, None, None, None


def _linear_group_norm(x, weight, bias, gn_weight, gn_bias, groups, eps=1e-5, negative_slope=None, residual=None, pre=None):
    """``pre``: tensor to receive the pre-norm activation (default: a shared scratch buffer)"""
    x, weight, bias, gn_weight, gn_bias = _detach(x), _detach(weight), _detach(bias), _detach(gn_weight), _detach(gn_bias)
    residual = _detach(residual)
    if not x.is_cuda or x.dtype != _f32 or x.stride(1) != 1:
        raise RuntimeError('linear_group_norm: x must be a float32 CUDA tensor with unit inner stride')
    L.require_cuda(weight, 'weight', _f32)
    m, k = x.shape
    n = weight.shape[0]
    if pre is None:
        pre = scratch((m, n), x.device, 'pre_norm')
    y = torch.empty((m, n), dtype=_f32, device=x.device)
    ws = _gn_workspace(x.device, groups, m, n)
    L.check(L.lib().geob200_linear_group_norm(x.data_ptr(), x.stride(0), weight.data_ptr(), L.ptr(bias), m, n, k, groups,
                                              gn_weight.data_ptr(), gn_bias.data_ptr(), float(eps), L.ptr(residual),
                                              int(negative_slope is not None), float(negative_slope or 0.0), pre.data_ptr(),
                                              y.data_ptr(), ws.data_ptr(), ws.numel(), L.stream_ptr()), 'linear_group_norm')
    return y


def kpconv_group_norm(s_feats, q_points, s_points, neighbor_indices, kernel_points, weights, bias, sigma, gn_weight, gn_bias, groups,
                      eps=1e-5, negative_slope=0.1, weights_t=None, cloud_rows=None):
    """ConvBlock / conv part of ResidualBlock: leaky(GroupNorm(KPConv(...))), with per-pair statistics given ``cloud_rows`` (query
    rows per cloud).  Differentiable w.r.t. s_feats, the weights, the biases and the GroupNorm affine (the autograd path keeps its
    own copy of the pre-norm activation)."""
    m, h = neighbor_indices.shape
    k, cin, cout = weights.shape
    if not (KPCONV_MODE == 'tc' and cin % 32 == 0 and cout % 16 == 0 and cout >= 32 and (cout <= 128 or cout % 128 == 0) and m >= 64):
        x = kpconv(s_feats, q_points, s_points, neighbor_indices, kernel_points, weights, bias, sigma, weights_t=weights_t)
        return group_norm(x, gn_weight, gn_bias, groups, eps, negative_slope=negative_slope, cloud_rows=cloud_rows)
    if _needs_grad(s_feats, weights, bias, gn_weight, gn_bias):
        return _KPConvGroupNorm.apply(s_feats, weights, bias, gn_weight, gn_bias, q_points, s_points, neighbor_indices, kernel_points,
                                      float(sigma), int(groups), float(eps), negative_slope, weights_t, cloud_rows)
    return _kpconv_group_norm(s_feats, q_points, s_points, neighbor_indices, kernel_points, weights, bias, sigma, gn_weight, gn_bias,
                              groups, eps, negative_slope, weights_t, cloud_rows=cloud_rows)


class _KPConvGroupNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, s_feats, weights, bias, gn_weight, gn_bias, q_points, s_points, neighbor_indices, kernel_points, sigma, groups, eps,
                negative_slope, weights_t, cloud_rows):
        pre = torch.empty((neighbor_indices.shape[0], weights.shape[2]), dtype=_f32, device=s_feats.device)
        y = _kpconv_group_norm(s_feats, q_points, s_points, neighbor_indices, kernel_points, weights, bias, sigma, gn_weight, gn_bias,
                               groups, eps, negative_slope, weights_t, pre=pre, cloud_rows=cloud_rows)
        ctx.save_for_backward(s_feats, weights, gn_weight, q_points, s_points, neighbor_indices, kernel_points, pre, y)
        ctx.args = (sigma, groups, eps, negative_slope, _seg_rows(cloud_rows, pre.shape[0]))
        return y

    @staticmethod
    def backward(ctx, grad):
        s_feats, weights, gn_weight, q, s, nbr, kp, pre, y = ctx.saved_tensors
        sigma, groups, eps, slope, rows = ctx.args
        need = ctx.needs_input_grad
        gpre, ggw, ggb, _ = group_norm_backward_batched(pre, y, gn_weight, groups, rows, grad.contiguous(), eps, slope, False, need[3],
                                                        need[4])
        gf, gw, gb = kpconv_backward(s_feats, q, s, nbr, kp, weights, sigma, gpre, need[0], need[1], need[2])
        return gf, gw, gb, ggw, ggb, None, None, None, None, None, None, None, None, None, None


def _kpconv_group_norm(s_feats, q_points, s_points, neighbor_indices, kernel_points, weights, bias, sigma, gn_weight, gn_bias, groups,
                       eps=1e-5, negative_slope=0.1, weights_t=None, pre=None, cloud_rows=None):
    """``cloud_rows``: per-pair statistics (``geob200_kpconv_group_norm_batched``)"""
    m, h = neighbor_indices.shape
    k, cin, cout = weights.shape
    s_feats, weights, bias, gn_weight, gn_bias = _detach(s_feats), _detach(weights), _detach(bias), _detach(gn_weight), _detach(gn_bias)
    _f(s_feats, 's_feats'); _f(q_points, 'q_points'); _f(s_points, 's_points')
    L.require_cuda(neighbor_indices, 'neighbor_indices', _i64)
    ns = s_points.shape[0]
    dev = s_feats.device
    if weights_t is None:
        weights_t = weights.reshape(k * cin, cout).t().contiguous()
    lib = L.lib()
    if pre is None:
        pre = scratch((m, cout), dev, 'pre_norm')
    y = torch.empty((m, cout), dtype=_f32, device=dev)
    ws = L.workspace(lib.geob200_kpconv_tc_workspace_bytes(m, ns, cin), dev, 'kpconv_tc')
    if cloud_rows is not None:
        gws = _gn_workspace(dev, groups, m, cout, n_pairs=len(cloud_rows) // 2)
        L.check(lib.geob200_kpconv_group_norm_batched(
            s_feats.data_ptr(), q_points.data_ptr(), s_points.data_ptr(), neighbor_indices.data_ptr(), m, ns, h, kernel_points.data_ptr(), k,
            weights_t.data_ptr(), L.ptr(bias), cin, cout, float(sigma), groups, gn_weight.data_ptr(), gn_bias.data_ptr(), float(eps),
            int(negative_slope is not None), float(negative_slope or 0.0), pre.data_ptr(), y.data_ptr(), gws.data_ptr(), gws.numel(),
            ws.data_ptr(), ws.numel(), L.stream_ptr(), len(cloud_rows) // 2, _host_i64(cloud_rows)), 'kpconv_group_norm_batched')
        return y
    gws = _gn_workspace(dev, groups, m, cout)
    L.check(lib.geob200_kpconv_group_norm(s_feats.data_ptr(), q_points.data_ptr(), s_points.data_ptr(), neighbor_indices.data_ptr(),
                                          m, ns, h, kernel_points.data_ptr(), k, weights_t.data_ptr(), L.ptr(bias), cin, cout,
                                          float(sigma), groups, gn_weight.data_ptr(), gn_bias.data_ptr(), float(eps),
                                          int(negative_slope is not None), float(negative_slope or 0.0), pre.data_ptr(),
                                          y.data_ptr(), gws.data_ptr(), gws.numel(), ws.data_ptr(), ws.numel(), L.stream_ptr()),
            'kpconv_group_norm')
    return y


def _host_i64(values):
    values = [int(v) for v in values]
    return (ctypes.c_int64 * len(values))(*values)


def group_norm_batched(x, weight, bias, groups, cloud_rows, eps=1e-5, negative_slope=None, residual=None):
    """GroupNorm with per-PAIR statistics for rows in stack order [ref_1..ref_B, src_1..src_B] (``cloud_rows``: 2B host ints)"""
    x, weight, bias = _detach(x), _detach(weight), _detach(bias)
    _f(x, 'x')
    n, c = x.shape
    np_ = len(cloud_rows) // 2
    ws = _gn_workspace(x.device, groups, n, c, n_pairs=np_)
    y = torch.empty_like(x)
    L.check(L.lib().geob200_group_norm_batched(x.data_ptr(), n, c, groups, weight.data_ptr(), bias.data_ptr(), float(eps), L.ptr(residual),
                                               int(negative_slope is not None), float(negative_slope or 0.0), y.data_ptr(), ws.data_ptr(),
                                               ws.numel(), L.stream_ptr(), np_, _host_i64(cloud_rows)), 'group_norm_batched')
    return y


def linear_group_norm_batched(x, weight, bias, gn_weight, gn_bias, groups, cloud_rows, eps=1e-5, negative_slope=None, residual=None,
                              pre=None):
    """linear_group_norm with per-pair GroupNorm statistics (see group_norm_batched); ``pre``: tensor to receive the pre-norm
    activation (default: a shared scratch buffer)"""
    x, weight, bias, gn_weight, gn_bias = _detach(x), _detach(weight), _detach(bias), _detach(gn_weight), _detach(gn_bias)
    m, k = x.shape
    n = weight.shape[0]
    np_ = len(cloud_rows) // 2
    if pre is None:
        pre = scratch((m, n), x.device, 'pre_norm')
    y = torch.empty((m, n), dtype=_f32, device=x.device)
    ws = _gn_workspace(x.device, groups, m, n, n_pairs=np_)
    L.check(L.lib().geob200_linear_group_norm_batched(x.data_ptr(), x.stride(0), weight.data_ptr(), L.ptr(bias), m, n, k, groups,
                                                      gn_weight.data_ptr(), gn_bias.data_ptr(), float(eps), L.ptr(residual),
                                                      int(negative_slope is not None), float(negative_slope or 0.0), pre.data_ptr(),
                                                      y.data_ptr(), ws.data_ptr(), ws.numel(), L.stream_ptr(), np_, _host_i64(cloud_rows)),
            'linear_group_norm_batched')
    return y


def maxpool(x, neighbor_indices, cloud_rows=None, cloud_max=None):
    """differentiable w.r.t. x (``maxpool_backward_batched``).  A batch of pairs (``cloud_rows``: query rows per cloud, 2B host ints;
    ``cloud_max``: ``cloud_max_count`` of the table) pools pair p's rows over its own table width only (``geob200_maxpool_batched``)."""
    if (cloud_rows is None) != (cloud_max is None):
        raise RuntimeError('maxpool: cloud_rows and cloud_max come together')
    if _needs_grad(x):
        return _Maxpool.apply(x, neighbor_indices, cloud_rows, cloud_max)
    return _maxpool(x, neighbor_indices, cloud_rows, cloud_max)


def _maxpool(x, neighbor_indices, cloud_rows=None, cloud_max=None):
    x = _detach(x)
    _f(x, 'x'); L.require_cuda(neighbor_indices, 'neighbor_indices', _i64)
    m, h = neighbor_indices.shape
    y = torch.empty((m, x.shape[1]), dtype=_f32, device=x.device)
    if cloud_rows is not None:
        L.require_cuda(cloud_max, 'cloud_max', _i32)
        if cloud_max.numel() != len(cloud_rows):
            raise RuntimeError('maxpool: cloud_max needs one entry per cloud')
        L.check(L.lib().geob200_maxpool_batched(x.data_ptr(), neighbor_indices.data_ptr(), m, x.shape[0], h, x.shape[1], cloud_max.data_ptr(),
                                                len(cloud_rows) // 2, _host_i64(cloud_rows), y.data_ptr(), L.stream_ptr()), 'maxpool_batched')
        return y
    L.check(L.lib().geob200_maxpool(x.data_ptr(), neighbor_indices.data_ptr(), m, x.shape[0], h, x.shape[1],
                                    y.data_ptr(), L.stream_ptr()), 'maxpool')
    return y


def cloud_max_count(neighbor_indices, n_support, cloud_rows):
    """(2B,) device int32: per cloud the widest row (number of real neighbours) of the (n_query, H) table ``neighbor_indices`` whose
    query rows are laid out by ``cloud_rows`` (2B host ints) -- the per-pair widths of the batched max-pool"""
    L.require_cuda(neighbor_indices, 'neighbor_indices', _i64)
    out = torch.empty((len(cloud_rows),), dtype=_i32, device=neighbor_indices.device)
    L.check(L.lib().geob200_cloud_max_count(neighbor_indices.data_ptr(), neighbor_indices.shape[0], int(n_support), neighbor_indices.shape[1],
                                            len(cloud_rows) // 2, _host_i64(cloud_rows), out.data_ptr(), L.stream_ptr()), 'cloud_max_count')
    return out


def maxpool_backward_batched(x, neighbor_indices, cloud_rows, grad_y, cloud_max=None):
    """grad_x of the max-pool for the upstream gradient ``grad_y`` (n_query, C): each output's gradient goes to the neighbour column
    that won the forward's max (ties: the lowest column), none when the zero shadow row won.  ``cloud_rows``: query rows per cloud
    (2B host ints); ``cloud_max`` (device int32 (2B,), ``geob200_cloud_max_count``): cut pair p's rows to the batched forward's width,
    None = every column (``maxpool``)."""
    x = _detach(x)
    _f(x, 'x'); _f(grad_y, 'grad_y'); L.require_cuda(neighbor_indices, 'neighbor_indices', _i64)
    if cloud_max is not None:
        L.require_cuda(cloud_max, 'cloud_max', _i32)
        if cloud_max.numel() != len(cloud_rows):
            raise RuntimeError('maxpool_backward_batched: cloud_max needs one entry per cloud')
    m, h = neighbor_indices.shape
    ns, c = x.shape
    if tuple(grad_y.shape) != (m, c):
        raise RuntimeError(f'maxpool_backward_batched: grad_y must be ({m}, {c})')
    gx = torch.empty_like(x)
    lib = L.lib()
    ws = L.workspace(lib.geob200_maxpool_backward_batched_workspace_bytes(m, ns, h, c), x.device, 'maxpool_backward')
    L.check(lib.geob200_maxpool_backward_batched(x.data_ptr(), neighbor_indices.data_ptr(), m, ns, h, c, L.ptr(cloud_max), len(cloud_rows) // 2,
                                                 _host_i64(cloud_rows), grad_y.data_ptr(), gx.data_ptr(), ws.data_ptr(), ws.numel(),
                                                 L.stream_ptr()), 'maxpool_backward_batched')
    return gx


class _Maxpool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, neighbor_indices, cloud_rows, cloud_max):
        ctx.save_for_backward(x, neighbor_indices, cloud_max)
        ctx.rows = _seg_rows(cloud_rows, neighbor_indices.shape[0])
        return _maxpool(x, neighbor_indices, cloud_rows, cloud_max)

    @staticmethod
    def backward(ctx, grad):
        x, nbr, cloud_max = ctx.saved_tensors
        return maxpool_backward_batched(x, nbr, ctx.rows, grad.contiguous(), cloud_max), None, None, None


def upsample_concat(x, upsample_indices, skip=None):
    """[nearest_upsample(x, upsample_indices) | skip]; ``upsample_indices`` (M, H) -- only column 0 is used.  Differentiable w.r.t.
    x and skip (``upsample_concat_backward``)."""
    if _needs_grad(x, skip):
        return _UpsampleConcat.apply(x, skip, upsample_indices)
    return _upsample_concat(x, upsample_indices, skip)


def upsample_concat_backward(upsample_indices, n_support, c1, grad_y, need_skip=True):
    """(grad_x (n_support, c1), grad_skip (n_query, C - c1) or None) of ``upsample_concat``: each coarse row sums the gradient rows of
    the fine rows that copied it, in fine-row order; sentinel indices contribute nothing"""
    _f(grad_y, 'grad_y')
    if not upsample_indices.is_cuda or upsample_indices.dtype != _i64:
        raise RuntimeError('upsample_indices must be an int64 CUDA tensor')
    m = upsample_indices.shape[0]
    stride = upsample_indices.stride(0) if upsample_indices.ndim == 2 else 1
    c2 = grad_y.shape[1] - c1
    if grad_y.shape[0] != m or c2 < 0:
        raise RuntimeError(f'upsample_concat_backward: grad_y must have {m} rows and at least {c1} columns')
    dev = grad_y.device
    gx = torch.empty((n_support, c1), dtype=_f32, device=dev)
    gs = torch.empty((m, c2), dtype=_f32, device=dev) if need_skip and c2 > 0 else None
    lib = L.lib()
    ws = L.workspace(lib.geob200_upsample_concat_backward_workspace_bytes(m, n_support), dev, 'upsample_concat_backward')
    L.check(lib.geob200_upsample_concat_backward(upsample_indices.data_ptr(), stride, m, n_support, c1, c2, grad_y.data_ptr(), gx.data_ptr(),
                                                 L.ptr(gs), ws.data_ptr(), ws.numel(), L.stream_ptr()), 'upsample_concat_backward')
    return gx, gs


class _UpsampleConcat(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, skip, upsample_indices):
        ctx.save_for_backward(upsample_indices)
        ctx.shape = tuple(x.shape)
        return _upsample_concat(x, upsample_indices, skip)

    @staticmethod
    def backward(ctx, grad):
        up, = ctx.saved_tensors
        ns, c1 = ctx.shape
        gx, gs = upsample_concat_backward(up, ns, c1, grad.contiguous(), ctx.needs_input_grad[1])
        return gx if ctx.needs_input_grad[0] else None, gs, None


def _upsample_concat(x, upsample_indices, skip=None):
    x, skip = _detach(x), _detach(skip)
    _f(x, 'x')
    if not upsample_indices.is_cuda or upsample_indices.dtype != _i64:
        raise RuntimeError('upsample_indices must be an int64 CUDA tensor')
    m = upsample_indices.shape[0]
    stride = upsample_indices.stride(0) if upsample_indices.ndim == 2 else 1
    c1 = x.shape[1]
    c2 = 0 if skip is None else skip.shape[1]
    y = torch.empty((m, c1 + c2), dtype=_f32, device=x.device)
    L.check(L.lib().geob200_upsample_concat(x.data_ptr(), upsample_indices.data_ptr(), stride, x.shape[0],
                                            L.ptr(skip), m, c1, c2, y.data_ptr(), L.stream_ptr()), 'upsample_concat')
    return y


def nearest_upsample(x, upsample_indices):
    return upsample_concat(x, upsample_indices, None)


# ------------------------------------------------------------------------------------------------ partition

def point_to_node_partition(points, nodes, point_limit, return_count=False):
    return point_to_node_partition_batched(points, nodes, [points.shape[0]], [nodes.shape[0]], point_limit, return_count)


def knn_partition(points, nodes, k, return_distance=False):
    """reference ``pointcloud_partition.py:35-57``: (n_nodes, k) nearest point indices per node [and their distances]"""
    _f(points, 'points'); _f(nodes, 'nodes')
    n, m = points.shape[0], nodes.shape[0]
    k = min(int(k), n)
    idx = torch.empty((m, k), dtype=_i64, device=points.device)
    d2 = torch.empty((m, k), dtype=_f32, device=points.device) if return_distance else None
    L.check(L.lib().geob200_knn_partition(points.data_ptr(), n, nodes.data_ptr(), m, k, idx.data_ptr(), L.ptr(d2), L.stream_ptr()),
            'knn_partition')
    if return_distance:
        return d2.sqrt_(), idx
    return idx


def pairwise_distance(x, y, normalized=False, channel_first=False):
    """reference ``pairwise_distance.py:4-31`` for 2-D (or batched 3-D) inputs"""
    if channel_first:
        x, y = x.transpose(-1, -2), y.transpose(-1, -2)
    if x.ndim == 3:
        return torch.stack([pairwise_distance(a, b, normalized) for a, b in zip(x, y)])
    x, y = x.contiguous(), y.contiguous()
    _f(x, 'x'); _f(y, 'y')
    if x.ndim != 2 or y.ndim != 2 or x.shape[1] != y.shape[1]:
        raise RuntimeError('pairwise_distance: x (N, C) and y (M, C) expected')
    out = torch.empty((x.shape[0], y.shape[0]), dtype=_f32, device=x.device)
    L.check(L.lib().geob200_pairwise_distance(x.data_ptr(), x.shape[0], y.data_ptr(), y.shape[0], x.shape[1], int(normalized),
                                              out.data_ptr(), L.stream_ptr()), 'pairwise_distance')
    return out


def point_to_node_indices(points, nodes, return_counts=False):
    """reference ``pointcloud_partition.py:9-32`` (get_point_to_node_indices)"""
    _f(points, 'points'); _f(nodes, 'nodes')
    idx = torch.empty((points.shape[0],), dtype=_i64, device=points.device)
    sizes = torch.empty((nodes.shape[0],), dtype=_i32, device=points.device) if return_counts else None
    L.check(L.lib().geob200_point_to_node_indices(points.data_ptr(), points.shape[0], nodes.data_ptr(), nodes.shape[0], idx.data_ptr(),
                                                  L.ptr(sizes), L.stream_ptr()), 'get_point_to_node_indices')
    return (idx, sizes.long()) if return_counts else idx


def apply_transform(points, transform):
    """reference ``ops/transformation.py:7-60`` (points only) for a single (4, 4) transform: Q = P R^T + t"""
    _f(transform, 'transform')
    p = points.reshape(-1, 3).contiguous()
    _f(p, 'points')
    out = torch.empty_like(p)
    L.check(L.lib().geob200_apply_transform(p.data_ptr(), p.shape[0], transform.data_ptr(), out.data_ptr(), L.stream_ptr()),
            'apply_transform')
    return out.reshape(points.shape)


def gather_rows(table, indices):
    """index_select on a zero-padded table: rows with index >= len(table) come back as zeros."""
    table = _detach(table)
    _f(table, 'table'); L.require_cuda(indices, 'indices', _i64)
    c = table.shape[1]
    out = torch.empty((*indices.shape, c), dtype=_f32, device=table.device)
    L.check(L.lib().geob200_gather_rows(table.data_ptr(), table.shape[0], c, indices.data_ptr(), indices.numel(),
                                        out.data_ptr(), L.stream_ptr()), 'gather_rows')
    return out


# ------------------------------------------------------------------------------------------------ transformer

def gse_indices(points, sigma_d, sigma_a, angle_k, out=None):
    """``out``: optional (d, a) contiguous float buffers of n*n and n*n*angle_k elements to write into"""
    _f(points, 'points')
    n = points.shape[0]
    if out is not None:
        d, a = out[0].view(n, n), out[1].view(n, n, angle_k)
    else:
        d = torch.empty((n, n), dtype=_f32, device=points.device)
        a = torch.empty((n, n, angle_k), dtype=_f32, device=points.device)
    return gse_indices_batched(points, [n], sigma_d, sigma_a, angle_k, d, a)


def gse_indices_batched(points, cloud_rows, sigma_d, sigma_a, angle_k, d_out, a_out):
    """get_embedding_indices of several stacked clouds in ONE launch; d_out (sum n^2,), a_out (sum n^2, angle_k) receive the
    clouds' index arrays one after the other (the layout ``gse_embed_flat`` consumes)"""
    _f(points, 'points')
    factor_a = 180.0 / (sigma_a * math.pi)
    L.check(L.lib().geob200_gse_indices_batched(points.data_ptr(), len(cloud_rows), _host_i64(cloud_rows), float(sigma_d), float(factor_a),
                                                angle_k, d_out.data_ptr(), a_out.data_ptr(), L.stream_ptr()), 'gse_indices_batched')
    return d_out, a_out


def scratch(shape, device, tag):
    """View of a grow-only per-(device, stream, tag) float buffer: for big intermediates whose size changes from pair to
    pair (the N x N x C structure embedding), so that the caching allocator never has to cudaMalloc inside the timed loop.
    The result aliases the buffer: it is only valid until the next call with the same tag on the same stream."""
    numel = 1
    for s in shape:
        numel *= int(s)
    key = (device.index if device.index is not None else torch.cuda.current_device(), L.stream_ptr(), tag)
    buf = _SCRATCH.get(key)
    if buf is None or buf.numel() < numel:
        buf = torch.empty(int(numel * 1.3) + 1024, dtype=_f32, device=device)
        _SCRATCH[key] = buf
    return buf[:numel].view(*shape)


_SCRATCH = {}


class GseTable:
    """Tabulated proj_d(sinusoid(x)) / proj_a(sinusoid(x)) (``geob200_gse_table_build``): the device blob and the grid it was
    built on."""
    __slots__ = ('blob', 'channels', 'inv_step', 'd_max', 'a_max')

    def __init__(self, blob, channels, inv_step, d_max, a_max):
        self.blob, self.channels, self.inv_step, self.d_max, self.a_max = blob, channels, inv_step, d_max, a_max


def gse_table(div_term, wd_t, wa_t, bd, ba, sigma_a, inv_step=None, d_max=None, sync=True):
    """Tabulate the two projections of GeometricStructureEmbedding for the given weights (wd_t / wa_t: transposed nn.Linear
    weights (in, out)).  Angle indices lie in [0, 180 / sigma_a]; distance indices above ``d_max`` fall back to the direct
    evaluation inside ``gse_embed*``.  Returns after the build has COMPLETED, so any stream may use the table; ``sync=False``
    returns at once (only the current stream may use it before the caller waits for it)."""
    for t, name in ((div_term, 'div_term'), (wd_t, 'wd_t'), (wa_t, 'wa_t'), (bd, 'bd'), (ba, 'ba')):
        L.require_cuda(t, name, _f32)
    c = int(wd_t.shape[0])
    inv_step = GSE_TABLE_INV_STEP if inv_step is None else int(inv_step)
    d_max = GSE_TABLE_D_MAX if d_max is None else float(d_max)
    a_max = 180.0 / float(sigma_a) + 0.25
    lib = L.lib()
    nbytes = lib.geob200_gse_table_bytes(c, inv_step, d_max, a_max)
    if nbytes == 0:
        raise RuntimeError(f'gse_table: bad grid (channels {c}, inv_step {inv_step}, d_max {d_max}, a_max {a_max})')
    blob = torch.empty(nbytes, dtype=_u8, device=wd_t.device)
    L.check(lib.geob200_gse_table_build(div_term.data_ptr(), wd_t.data_ptr(), wa_t.data_ptr(), bd.data_ptr(), ba.data_ptr(), c,
                                        inv_step, d_max, a_max, blob.data_ptr(), nbytes, L.stream_ptr()), 'gse_table_build')
    if sync:
        torch.cuda.current_stream(wd_t.device).synchronize()
    return GseTable(blob, c, inv_step, d_max, a_max)


def _gse_embed_table(d_indices, a_indices, n_rows, div_term, wd, wa, bd, ba, table, out):
    c = wd.shape[0]
    if table is None or table.channels != c:
        raise RuntimeError('gse_embed mode 5 (tabulated projections) needs the GseTable of these weights (functional.gse_table)')
    with _timed('gse_embed'):
        L.check(L.lib().geob200_gse_embed_table(d_indices.data_ptr(), a_indices.data_ptr(), int(n_rows), c, table.blob.data_ptr(),
                                                table.blob.numel(), table.inv_step, table.d_max, table.a_max, div_term.data_ptr(),
                                                wd.data_ptr(), wa.data_ptr(), bd.data_ptr(), ba.data_ptr(), out.data_ptr(),
                                                L.stream_ptr()), 'gse_embed_table')
    return out


def _gse_mode(mode, table):
    """mode None, 3 or 5: an explicit mode wins (mode 5 without a table is an error, raised by ``_gse_embed_table``); the default
    is GSE_MODE, except that the tabulated mode without a table means the caller has none: the contraction (mode 3)"""
    if mode is None:
        mode = 3 if (GSE_MODE == 5 and table is None) else GSE_MODE
    if mode not in (3, 5):
        raise ValueError(f'gse_embed: mode {mode!r} unsupported (None, 3 = contraction or 5 = tabulated projections)')
    return mode


def gse_embed_flat(d_indices, a_indices, n_rows, div_term, wd, wa, bd, ba, wd_t, wa_t, out, mode=None, table=None):
    """structure embedding of ``n_rows`` (anchor, point) pairs given as flat index arrays -- the (i, j) pairs of SEVERAL clouds
    concatenated (d (n_rows,), a (n_rows, k)) -> out (n_rows, C): one launch for a whole batch of clouds.  Differentiable w.r.t.
    ``wd``, ``wa``, ``bd`` and ``ba`` (``gse_embed_backward``; C = 128 or 256), which then needs the ``table`` of these weights
    whatever the mode; with ``out`` the result is copied into it, which then carries the graph."""
    if _needs_grad(wd, wa, bd, ba):
        y = _GseEmbed.apply(wd, wa, bd, ba, d_indices, a_indices, int(n_rows), div_term, wd_t, wa_t, mode, table)
        return y if out is None else out.copy_(y)
    return _gse_embed_flat(d_indices, a_indices, n_rows, div_term, wd, wa, bd, ba, wd_t, wa_t, out, mode, table)


def _gse_embed_flat(d_indices, a_indices, n_rows, div_term, wd, wa, bd, ba, wd_t, wa_t, out, mode=None, table=None):
    wd, wa, bd, ba = _detach(wd), _detach(wa), _detach(bd), _detach(ba)
    c = wd.shape[0]
    mode = _gse_mode(mode, table)
    if mode == 5 and c in (128, 256):
        return _gse_embed_table(d_indices, a_indices, n_rows, div_term, wd, wa, bd, ba, table, out)
    lib = L.lib()
    ws = L.workspace(lib.geob200_gse_embed_workspace_bytes(1, c), d_indices.device, 'gse')
    with _timed('gse_embed'):
        L.check(lib.geob200_gse_embed_pairs(d_indices.data_ptr(), a_indices.data_ptr(), int(n_rows), c, div_term.data_ptr(),
                                            wd_t.data_ptr(), wa_t.data_ptr(), wd.data_ptr(), wa.data_ptr(), bd.data_ptr(),
                                            ba.data_ptr(), out.data_ptr(), ws.data_ptr(), ws.numel(), L.stream_ptr()),
                'gse_embed_pairs')
    return out


def gse_embed_backward(d_indices, a_indices, n_rows, div_term, wa, ba, table, grad_embed):
    """(grad_wd, grad_bd, grad_wa, grad_ba) of the structure embedding for the upstream gradient ``grad_embed`` (n_rows, C), C = 128 or
    256.  The winning angle term of every (row, channel) is the one the tabulated forward picks: it comes from the lookups into
    ``table`` (the GseTable of the current weights).  The sinusoid is evaluated on the fly, never stored."""
    wa, ba = _detach(wa), _detach(ba)
    for t, name in ((d_indices, 'd_indices'), (a_indices, 'a_indices'), (div_term, 'div_term'), (wa, 'wa'), (ba, 'ba'),
                    (grad_embed, 'grad_embed')):
        _f(t, name)
    c = int(wa.shape[0])
    if table is None or table.channels != c:
        raise RuntimeError('gse_embed_backward needs the GseTable of these weights (functional.gse_table)')
    n_rows = int(n_rows)
    if grad_embed.numel() != n_rows * c or d_indices.numel() < n_rows or a_indices.numel() % max(n_rows, 1) != 0:
        raise RuntimeError(f'gse_embed_backward: grad_embed must hold ({n_rows}, {c}) values and the indices {n_rows} rows')
    dev = grad_embed.device
    gwd, gwa = (torch.empty((c, c), dtype=_f32, device=dev) for _ in range(2))
    gbd, gba = (torch.empty((c,), dtype=_f32, device=dev) for _ in range(2))
    lib = L.lib()
    ws = L.workspace(lib.geob200_gse_embed_backward_workspace_bytes(n_rows, c), dev, 'gse_embed_backward')
    with _timed('gse_embed_backward'):
        L.check(lib.geob200_gse_embed_backward(d_indices.data_ptr(), a_indices.data_ptr(), n_rows, a_indices.numel() // n_rows, c,
                                               table.blob.data_ptr(), table.blob.numel(), table.inv_step, table.d_max, table.a_max,
                                               div_term.data_ptr(), wa.data_ptr(), ba.data_ptr(), grad_embed.data_ptr(), gwd.data_ptr(),
                                               gbd.data_ptr(), gwa.data_ptr(), gba.data_ptr(), ws.data_ptr(), ws.numel(), L.stream_ptr()),
                'gse_embed_backward')
    return gwd, gbd, gwa, gba


class _GseEmbed(torch.autograd.Function):
    @staticmethod
    def forward(ctx, wd, wa, bd, ba, d_indices, a_indices, n_rows, div_term, wd_t, wa_t, mode, table):
        if table is None:
            raise RuntimeError('gse_embed: the backward needs the GseTable of these weights (functional.gse_table)')
        out = torch.empty((n_rows, wd.shape[0]), dtype=_f32, device=d_indices.device)
        _gse_embed_flat(d_indices, a_indices, n_rows, div_term, wd, wa, bd, ba, wd_t, wa_t, out, mode, table)
        ctx.save_for_backward(d_indices, a_indices, div_term, wa, ba)
        ctx.n_rows, ctx.table = n_rows, table
        return out

    @staticmethod
    def backward(ctx, grad):
        d, a, div_term, wa, ba = ctx.saved_tensors
        gwd, gbd, gwa, gba = gse_embed_backward(d, a, ctx.n_rows, div_term, wa, ba, ctx.table, grad.contiguous())
        return gwd, gwa, gbd, gba, None, None, None, None, None, None, None, None


def gse_embed(d_indices, a_indices, div_term, wd, wa, bd, ba, wd_t, wa_t, mode=None, out=None, table=None):
    """structure embedding of one cloud: d (n, n), a (n, n, k) -> (n, n, C)"""
    n = d_indices.shape[0]
    c = wd.shape[0]
    if _needs_grad(wd, wa, bd, ba):
        emb = gse_embed_flat(d_indices, a_indices, n * n, div_term, wd, wa, bd, ba, wd_t, wa_t, None, mode=mode, table=table)
        emb = emb.view(n, n, c)
        return emb if out is None else out.copy_(emb)
    emb = torch.empty((n, n, c), dtype=_f32, device=d_indices.device) if out is None else out
    return gse_embed_flat(d_indices, a_indices, n * n, div_term, wd, wa, bd, ba, wd_t, wa_t, emb, mode=mode, table=table)


def _rows(t, name):
    if not t.is_cuda or t.dtype != _f32 or t.ndim != 2 or t.stride(1) != 1:
        raise RuntimeError(f'{name} must be a 2-D float32 CUDA tensor with unit inner stride')
    return t


def attention(q, k, v, heads, qp=None, qb=None, embed=None, out=None, streaming=True):
    """q, k, v may be column slices of a fused projection buffer (row stride != channels).  streaming=False forces the
    single-kernel path (the only one for channel counts other than 128 / 256).  Differentiable w.r.t. q, k, v, qp, qb and embed
    (``attention_backward_batched``; C = 128 or 256, streaming): the forward then leaves its softmax probabilities in a tensor owned
    by the autograd node; with ``out`` the result is copied into it, which then carries the graph."""
    if _needs_grad(q, k, v, qp, qb, embed):
        if not streaming:
            raise RuntimeError('attention: the backward needs the probabilities of the streaming forward')
        srcs, where = _att_sources(q, k, v)
        y = _Attention.apply(int(heads), int(q.shape[1]), where, qp, qb, embed, *srcs)
        return y if out is None else out.copy_(y)
    return _attention(q, k, v, heads, qp, qb, embed, out, streaming)


def _attention(q, k, v, heads, qp=None, qb=None, embed=None, out=None, streaming=True, probs=None):
    """``probs``: a uint8 tensor of geob200_attention_workspace_bytes to run the streaming path in, instead of the shared scratch;
    it holds the (n, heads, m) probabilities afterwards"""
    q, k, v, qp, qb, embed = (_detach(t) for t in (q, k, v, qp, qb, embed))
    _rows(q, 'q'); _rows(k, 'k'); _rows(v, 'v')
    n, c = q.shape
    m = k.shape[0]
    if out is None:
        out = torch.empty((n, c), dtype=_f32, device=q.device)
    lib = L.lib()
    ws = probs if probs is not None else (
        L.workspace(lib.geob200_attention_workspace_bytes(n, m, heads), q.device, tag='attention') if streaming else None)
    L.check(lib.geob200_attention(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
                                  L.ptr(qp), L.ptr(qb), L.ptr(embed), n, m, c, heads, out.data_ptr(), out.stride(0),
                                  L.ptr(ws), 0 if ws is None else ws.numel(), L.stream_ptr()), 'attention')
    return out


def _column_source(t):
    """(base, r0, col): ``t`` is rows r0 .. r0 + t.shape[0], columns col .. col + t.shape[1] of the 2-D tensor ``base`` it is a view
    of (or of itself).  The backward writes the gradient of every slice of one row block into one (rows, base width) tensor, so a
    fused projection (q|k|v, k|v) gets one contiguous upstream gradient."""
    base = t._base if t._base is not None else t
    if base.dim() != 2 or base.stride(1) != 1 or t.stride(1) != 1 or t.stride(0) != base.stride(0):
        return t, 0, 0
    r0, col = divmod(t.storage_offset() - base.storage_offset(), base.stride(0))
    return base, r0, col


class _AttItem(ctypes.Structure):
    """geob200_att_item_t"""
    _fields_ = [(n, ctypes.c_void_p) for n in ('q', 'k', 'v', 'qp', 'qb', 'embed', 'out')] + [('n_query', ctypes.c_int64),
                                                                                            ('n_key', ctypes.c_int64)]


class _AttGradItem(ctypes.Structure):
    """geob200_att_grad_item_t"""
    _fields_ = [(n, ctypes.c_void_p) for n in ('probs', 'grad_out', 'grad_q', 'grad_k', 'grad_v', 'grad_qp', 'grad_qb', 'grad_embed')]


def attention_probs(n, m, heads, device):
    """buffer for the (n, heads, m) probabilities of one ``attention`` forward (its streaming workspace) and the float view of them"""
    buf = torch.empty(L.lib().geob200_attention_workspace_bytes(n, m, heads), dtype=_u8, device=device)
    return buf, buf[:n * m * heads * 4].view(_f32).view(n, heads, m)


def attention_backward_batched(items, heads):
    """Gradients of ``attention`` for a list of items in one call.  Every item is a dict with the forward's q, k, v (column slices
    allowed), out (its output), probs ((n, heads, m) probabilities of that forward, ``attention_probs``), grad_out (n, C) and, for
    self-attention, qp, qb and embed; optionally grad_q / grad_k / grad_v, (n, C) / (m, C) views to write the gradients into (column
    slices of one fused gradient allowed), and structure=False to skip grad_qp / grad_embed (the E pass).  The items share channels and
    row strides.  Returns per item (grad_q, grad_k, grad_v, grad_qp, grad_qb, grad_embed), the last three None for cross-attention."""
    if not items:
        raise RuntimeError('attention_backward_batched: no items')
    arr, garr, res = (_AttItem * len(items))(), (_AttGradItem * len(items))(), []
    strides = gstrides = None
    for j, it in enumerate(items):
        q, k, v, o = (_rows(_detach(it[name]), name) for name in ('q', 'k', 'v', 'out'))
        qp, qb, e = (_detach(it.get(name)) for name in ('qp', 'qb', 'embed'))
        probs, go = _detach(it['probs']), _f(_detach(it['grad_out']), 'grad_out')
        n, c = q.shape
        m = k.shape[0]
        st = (q.stride(0), k.stride(0), v.stride(0), o.stride(0), c)
        if strides is not None and st != strides:
            raise RuntimeError('attention_backward_batched: the items must share channels and row strides')
        strides = st
        if tuple(go.shape) != (n, c) or tuple(o.shape) != (n, c) or tuple(v.shape) != (m, c) or probs.numel() < n * m * heads:
            raise RuntimeError(f'attention_backward_batched: item {j}: out / grad_out must be ({n}, {c}), v ({m}, {c}), probs {n * m * heads} values')
        if probs.dtype != _f32 or not probs.is_contiguous():
            raise RuntimeError('attention_backward_batched: probs must be a contiguous float32 view (attention_probs)')
        if e is not None:
            _f(qp, 'qp'); _f(qb, 'qb'); _f(e, 'embed')
            if tuple(qp.shape) != (n, heads, c) or tuple(qb.shape) != (n, heads) or e.numel() != n * m * c:
                raise RuntimeError(f'attention_backward_batched: item {j}: qp ({n}, {heads}, {c}), qb ({n}, {heads}), embed ({n}, {m}, {c})')
        dev = q.device
        g = []
        for name, rows in (('grad_q', n), ('grad_k', m), ('grad_v', m)):
            t = it.get(name)
            if t is None:
                t = torch.empty((rows, c), dtype=_f32, device=dev)
            elif not t.is_cuda or t.dtype != _f32 or tuple(t.shape) != (rows, c) or t.stride(1) != 1:
                raise RuntimeError(f'attention_backward_batched: item {j}: {name} must be a ({rows}, {c}) float32 CUDA view with unit inner stride')
            g.append(t)
        gst = tuple(t.stride(0) for t in g)
        if gstrides is not None and gst != gstrides:
            raise RuntimeError('attention_backward_batched: the items\' gradients must share row strides')
        gstrides = gst
        structure = e is not None and it.get('structure', True)
        if structure:
            for name, shape in (('grad_qp', (n, heads, c)), ('grad_qb', (n, heads)), ('grad_embed', (n, m, c))):
                t = it.get(name)
                if t is None:
                    t = torch.empty(shape, dtype=_f32, device=dev)
                elif not t.is_cuda or t.dtype != _f32 or t.numel() != math.prod(shape) or not t.is_contiguous():
                    raise RuntimeError(f'attention_backward_batched: item {j}: {name} must be a contiguous float32 CUDA view of {shape} values')
                g.append(t)
        else:
            g += [None, None, None]
        arr[j] = _AttItem(q.data_ptr(), k.data_ptr(), v.data_ptr(), L.ptr(qp), L.ptr(qb), L.ptr(e), o.data_ptr(), n, m)
        garr[j] = _AttGradItem(probs.data_ptr(), go.data_ptr(), *(L.ptr(t) for t in g))
        res.append(tuple(g))
    lib = L.lib()
    ldq, ldk, ldv, ldo, c = strides
    ws = L.workspace(lib.geob200_attention_backward_batched_workspace_bytes(arr, len(items), heads), dev, 'attention_backward')
    with _timed('attention_backward'):
        L.check(lib.geob200_attention_backward_batched(arr, garr, len(items), ldq, ldk, ldv, ldo, *gstrides, c, heads, ws.data_ptr(),
                                                       ws.numel(), L.stream_ptr()), 'attention_backward_batched')
    return res


def _source_grads(srcs, where, c):
    """one gradient per source (zero where no slice of it reads) and the (rows, c) views of it at the given column offsets"""
    covered = [set() for _ in srcs]
    for i, col in where:
        covered[i].update(range(col, col + c))
    gs = [(torch.empty if len(cov) == s.shape[1] else torch.zeros)(tuple(s.shape), dtype=_f32, device=s.device)
          for s, cov in zip(srcs, covered)]
    return gs, [gs[i][:, col:col + c] for i, col in where]


class _Attention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, heads, c, where, qp, qb, embed, *srcs):
        q, k, v = (srcs[i][:, col:col + c] for i, col in where)
        n, m = q.shape[0], k.shape[0]
        # only the streaming forward leaves the probabilities in its workspace (geob200_attention_batched_keeps_probs)
        if not _keeps_probs([(n, m)], c, heads):
            raise RuntimeError(f'attention backward: channels {c} (128 or 256) or keys {m} outside the streaming forward')
        buf, probs = attention_probs(n, m, heads, q.device)
        out = _attention(q, k, v, heads, qp, qb, embed, probs=buf)
        ctx.save_for_backward(qp, qb, embed, out, probs, *srcs)
        ctx.heads, ctx.c, ctx.where = heads, c, where
        return out

    @staticmethod
    def backward(ctx, grad):
        qp, qb, embed, out, probs, *srcs = ctx.saved_tensors
        c, where = ctx.c, ctx.where
        q, k, v = (srcs[i][:, col:col + c] for i, col in where)
        gsrc, (gq, gk, gv) = _source_grads(srcs, where, c)
        n_qp, n_qb, n_e = ctx.needs_input_grad[3:6]
        item = dict(q=q, k=k, v=v, out=out, probs=probs, grad_out=grad.contiguous(), qp=qp, qb=qb, embed=embed, grad_q=gq, grad_k=gk,
                    grad_v=gv, structure=n_qp or n_qb or n_e)
        g = attention_backward_batched([item], ctx.heads)[0]
        return (None, None, None, g[3] if n_qp else None, g[4] if n_qb else None, g[5] if n_e else None,
                *(gs if need else None for gs, need in zip(gsrc, ctx.needs_input_grad[6:])))


ATT_MAX_ITEMS = 32          # GEOB200_ATT_MAX_ITEMS: items whose probabilities one geob200_attention_batched call leaves in place


def _keeps_probs(rows, c, heads):
    """whether the streaming forward takes every (n_query, n_key) item of ``rows`` in one launch pair, leaving its probabilities in
    the workspace (geob200_attention_batched_keeps_probs)"""
    arr = (_AttItem * len(rows))(*[_AttItem(None, None, None, None, None, None, None, n, m) for n, m in rows])
    return L.lib().geob200_attention_batched_keeps_probs(arr, len(rows), c, heads) == 1


def _att_sources(q, k, v):
    """the row blocks q, k and v are column slices of (one per distinct block) and where each reads: (srcs, ((src, col) x 3))"""
    srcs, keys, where = [], [], []
    for t in (q, k, v):
        base, r0, col = _column_source(t)
        key = (id(base), r0, t.shape[0])
        if key not in keys:
            keys.append(key)
            srcs.append(base if (r0 == 0 and t.shape[0] == base.shape[0]) else base[r0:r0 + t.shape[0]])
        where.append((keys.index(key), col))
    return srcs, tuple(where)


def attention_batched(q, k, v, heads, q_rows, k_rows, qp=None, qb=None, embed=None):
    """Several attention items in one launch pair (``geob200_attention_batched``, the batched transformer's kernels): item i is
    query rows sum(q_rows[:i]) .. + q_rows[i] of q (and of qp (N, heads, C) / qb (N, heads)) against key rows sum(k_rows[:i]) .. +
    k_rows[i] of k and v (column slices allowed); a self-attention item reads its (q_rows[i], k_rows[i], C) structure embedding at
    rows sum_{j<i} q_rows[j] * k_rows[j] of the flat ``embed`` (sum q_rows * k_rows, C).  Returns the (N, C) output of all items.
    Differentiable w.r.t. q, k, v, qp, qb and embed: the forward leaves every item's probabilities in a buffer owned by the autograd
    node (at most ATT_MAX_ITEMS items, C = 128 or 256, streaming path), and the backward is one ``attention_backward_batched`` call."""
    q_rows, k_rows = [int(r) for r in q_rows], [int(r) for r in k_rows]
    if _needs_grad(q, k, v, qp, qb, embed):
        srcs, where = _att_sources(q, k, v)
        return _AttentionBatched.apply(int(heads), int(q.shape[1]), where, tuple(q_rows), tuple(k_rows), qp, qb, embed, *srcs)
    return _attention_batched(q, k, v, heads, q_rows, k_rows, qp, qb, embed)[0]


def _attention_batched(q, k, v, heads, q_rows, k_rows, qp=None, qb=None, embed=None, probs=False):
    """(out, probability buffer or None, per-item byte offsets into it); ``probs``: run in a fresh buffer whose item layout is
    the documented one of geob200_attention_batched, instead of the shared scratch"""
    q, k, v, qp, qb, embed = (_detach(t) for t in (q, k, v, qp, qb, embed))
    _rows(q, 'q'); _rows(k, 'k'); _rows(v, 'v')
    n_items, c = len(q_rows), q.shape[1]
    if n_items < 1 or len(k_rows) != n_items or min(q_rows) < 1 or min(k_rows) < 1:
        raise RuntimeError('attention_batched: one positive query and key row count per item')
    if sum(q_rows) != q.shape[0] or sum(k_rows) != k.shape[0] or v.shape[0] != k.shape[0]:
        raise RuntimeError(f'attention_batched: the items must cover the {q.shape[0]} query and {k.shape[0]} key rows')
    self_att = embed is not None
    if self_att:
        for t, name in ((qp, 'qp'), (qb, 'qb'), (embed, 'embed')):
            if t is None or not t.is_contiguous():
                raise RuntimeError(f'attention_batched: {name} must be a contiguous tensor')
            _f(t, name)
        if embed.numel() != sum(a * b for a, b in zip(q_rows, k_rows)) * c:
            raise RuntimeError('attention_batched: embed must hold sum(q_rows * k_rows) rows of C values')
    dev = q.device
    out = torch.empty((q.shape[0], c), dtype=_f32, device=dev)
    arr = (_AttItem * n_items)()
    qo = ko = eo = 0
    for i, (n, m) in enumerate(zip(q_rows, k_rows)):
        arr[i] = _AttItem(q.data_ptr() + 4 * qo * q.stride(0), k.data_ptr() + 4 * ko * k.stride(0), v.data_ptr() + 4 * ko * v.stride(0),
                          qp.data_ptr() + 4 * qo * heads * c if self_att else None, qb.data_ptr() + 4 * qo * heads if self_att else None,
                          embed.data_ptr() + 4 * eo * c if self_att else None, out.data_ptr() + 4 * qo * c, n, m)
        qo, ko, eo = qo + n, ko + m, eo + n * m
    lib = L.lib()
    nbytes = lib.geob200_attention_batched_workspace_bytes(arr, n_items, heads)
    buf, offs = None, None
    if probs:
        if not lib.geob200_attention_batched_keeps_probs(arr, n_items, c, heads):
            raise RuntimeError(f'attention backward: {n_items} items (<= {ATT_MAX_ITEMS}), channels {c} (128 or 256) or keys outside the '
                               'streaming forward')
        buf = torch.empty(nbytes, dtype=_u8, device=dev)
        offs, o = [], 0
        for n, m in zip(q_rows, k_rows):
            offs.append(o)
            o += (n * m * heads * 4 + 255) // 256 * 256
        ws = buf
    else:
        ws = L.workspace(nbytes, dev, tag='attention')
    L.check(lib.geob200_attention_batched(arr, n_items, q.stride(0), k.stride(0), v.stride(0), c, c, heads, ws.data_ptr(), ws.numel(),
                                          L.stream_ptr()), 'attention_batched')
    return out, buf, offs


class _AttentionBatched(torch.autograd.Function):
    @staticmethod
    def forward(ctx, heads, c, where, q_rows, k_rows, qp, qb, embed, *srcs):
        q, k, v = (srcs[i][:, col:col + c] for i, col in where)
        out, buf, offs = _attention_batched(q, k, v, heads, q_rows, k_rows, qp, qb, embed, probs=True)
        ctx.save_for_backward(qp, qb, embed, out, buf, *srcs)
        ctx.heads, ctx.c, ctx.where, ctx.q_rows, ctx.k_rows, ctx.offs = heads, c, where, q_rows, k_rows, offs
        return out

    @staticmethod
    def backward(ctx, grad):
        qp, qb, embed, out, buf, *srcs = ctx.saved_tensors
        c, H = ctx.c, ctx.heads
        q, k, v = (srcs[i][:, col:col + c] for i, col in ctx.where)
        gsrc, (gq, gk, gv) = _source_grads(srcs, ctx.where, c)
        n_qp, n_qb, n_e = ctx.needs_input_grad[5:8]
        grad = grad.contiguous()
        structure = embed is not None and (n_qp or n_qb or n_e)
        if structure:          # one gradient tensor per input, the items write their rows of it
            gqp, gqb, ge = torch.empty_like(qp), torch.empty_like(qb), torch.empty_like(embed)
        items, qo, ko, eo = [], 0, 0, 0
        for n, m, off in zip(ctx.q_rows, ctx.k_rows, ctx.offs):
            rq, rk = slice(qo, qo + n), slice(ko, ko + m)
            it = dict(q=q[rq], k=k[rk], v=v[rk], out=out[rq], probs=buf[off:off + n * m * H * 4].view(_f32).view(n, H, m), grad_out=grad[rq],
                      grad_q=gq[rq], grad_k=gk[rk], grad_v=gv[rk])
            if embed is not None:
                it.update(qp=qp[rq], qb=qb[rq], embed=embed.view(-1, c)[eo:eo + n * m], structure=structure)
                if structure:
                    it.update(grad_qp=gqp[rq], grad_qb=gqb[rq], grad_embed=ge.view(-1, c)[eo:eo + n * m])
            items.append(it)
            qo, ko, eo = qo + n, ko + m, eo + n * m
        attention_backward_batched(items, H)
        if not structure:
            gqp = gqb = ge = None
        return (None, None, None, None, None, gqp if n_qp else None, gqb if n_qb else None, ge if n_e else None,
                *(gs if need else None for gs, need in zip(gsrc, ctx.needs_input_grad[8:])))


def head_project(q, wp_t, bp, heads):
    """qp[n,h,:] = Wp[h*d:(h+1)*d, :]^T q[n,h*d:(h+1)*d]  and  qb[n,h] = q_h . bp_h   (proj_p moved onto q).  Differentiable w.r.t. q,
    wp_t and bp (``head_project_backward``); wp_t may then be the transposed view ``proj_p.weight.t()``."""
    if _needs_grad(q, wp_t, bp):
        base, r0, col = _column_source(q)
        src = base if (r0 == 0 and q.shape[0] == base.shape[0]) else base[r0:r0 + q.shape[0]]
        return _HeadProject.apply(src, col, int(q.shape[1]), wp_t, bp, int(heads))
    return _head_project(q, wp_t, bp, heads)


def _head_project(q, wp_t, bp, heads):
    q, wp_t, bp = _detach(q), _detach(wp_t), _detach(bp)
    _rows(q, 'q')
    n, c = q.shape
    d = c // heads
    qp = torch.empty((n, heads, c), dtype=_f32, device=q.device)
    qb = torch.empty((n, heads), dtype=_f32, device=q.device)
    lib = L.lib()
    # batched over heads: x = q[:, h*d:(h+1)*d] (ldx=row stride, stride d), W' = wp_t[:, h*d:(h+1)*d] (ldw=c, stride d),
    # y = qp[:, h, :] (ldy=heads*c, stride c)
    L.check(lib.geob200_linear_batched(q.data_ptr(), q.stride(0), d, wp_t.data_ptr(), c, d, None, 0, qp.data_ptr(), heads * c, c,
                                       n, c, d, heads, 0, L.stream_ptr()), 'head_project')
    L.check(lib.geob200_head_bias(q.data_ptr(), q.stride(0), bp.data_ptr(), n, c, heads, qb.data_ptr(), L.stream_ptr()), 'head_bias')
    return qp, qb


def head_project_backward(q, wp, bp, heads, grad_qp, grad_qb, need_q=True, need_wp=True, need_bp=True, grad_q=None):
    """(grad_q (n, C), grad_wp (C, C), grad_bp (C,)) of ``head_project`` with wp = proj_p.weight (the transpose of its wp_t).  grad_q
    runs through the forward's batched GEMM (into the given ``grad_q`` view, a column slice allowed), grad_wp / grad_bp are
    fixed-order sums over the rows.  An output not requested is None."""
    q, wp, bp = _rows(_detach(q), 'q'), _detach(wp), _detach(bp)
    _f(wp, 'wp'); _f(bp, 'bp'); _f(grad_qp, 'grad_qp'); _f(grad_qb, 'grad_qb')
    n, c = q.shape
    if tuple(wp.shape) != (c, c) or tuple(grad_qp.shape) != (n, heads, c) or tuple(grad_qb.shape) != (n, heads):
        raise RuntimeError(f'head_project_backward: wp must be ({c}, {c}), grad_qp ({n}, {heads}, {c}) and grad_qb ({n}, {heads})')
    dev = q.device
    gq = (torch.empty((n, c), dtype=_f32, device=dev) if grad_q is None else grad_q) if need_q else None
    if gq is not None and (tuple(gq.shape) != (n, c) or gq.dtype != _f32 or gq.stride(1) != 1 or not gq.is_cuda):
        raise RuntimeError(f'head_project_backward: grad_q must be a ({n}, {c}) float32 CUDA view with unit inner stride')
    gw = torch.empty((c, c), dtype=_f32, device=dev) if need_wp else None
    gb = torch.empty((c,), dtype=_f32, device=dev) if need_bp else None
    lib = L.lib()
    ws = L.workspace(lib.geob200_head_project_backward_workspace_bytes(n, c, heads), dev, 'head_project_backward')
    L.check(lib.geob200_head_project_backward(q.data_ptr(), q.stride(0), wp.data_ptr(), bp.data_ptr(), n, c, heads, grad_qp.data_ptr(),
                                              grad_qb.data_ptr(), L.ptr(gq), c if gq is None else gq.stride(0), L.ptr(gw), L.ptr(gb),
                                              ws.data_ptr(), ws.numel(),
                                              L.stream_ptr()), 'head_project_backward')
    return gq, gw, gb


class _HeadProject(torch.autograd.Function):
    @staticmethod
    def forward(ctx, src, col, c, wp_t, bp, heads):
        qp, qb = _head_project(src[:, col:col + c], wp_t.contiguous(), bp, heads)
        ctx.save_for_backward(src, wp_t, bp)
        ctx.col, ctx.c, ctx.heads = col, c, heads
        return qp, qb

    @staticmethod
    def backward(ctx, grad_qp, grad_qb):
        src, wp_t, bp = ctx.saved_tensors
        col, c = ctx.col, ctx.c
        q = src[:, col:col + c]
        n = q.shape[0]
        grad_qp = torch.zeros((n, ctx.heads, c), dtype=_f32, device=q.device) if grad_qp is None else grad_qp.contiguous()
        grad_qb = torch.zeros((n, ctx.heads), dtype=_f32, device=q.device) if grad_qb is None else grad_qb.contiguous()
        nq, nw, nb = ctx.needs_input_grad[0], ctx.needs_input_grad[3], ctx.needs_input_grad[4]
        gsrc, (gq,) = _source_grads([src], [(0, col)], c) if nq else ([None], [None])
        _, gw, gb = head_project_backward(q, wp_t.t().contiguous(), bp, ctx.heads, grad_qp, grad_qb, nq, nw, nb, grad_q=gq)
        return gsrc[0], None, None, (gw.t() if gw is not None else None), gb, None


def add_layernorm(a, b, weight, bias, eps=1e-5, out=None):
    """y = LayerNorm(a + b) (b may be None).  Differentiable w.r.t. a, b, weight and bias (``add_layernorm_backward``); with ``out``
    the result is copied into it, which then carries the graph."""
    if _needs_grad(a, b, weight, bias):
        y = _AddLayerNorm.apply(a, b, weight, bias, float(eps))
        return y if out is None else out.copy_(y)
    return _add_layernorm(a, b, weight, bias, eps, out)


def _add_layernorm(a, b, weight, bias, eps=1e-5, out=None):
    a, b, weight, bias = _detach(a), _detach(b), _detach(weight), _detach(bias)
    L.require_cuda(a, 'a', _f32)
    if b is not None:
        L.require_cuda(b, 'b', _f32)
    n, c = a.shape
    y = torch.empty_like(a) if out is None else out
    if not y.is_contiguous():
        raise RuntimeError('add_layernorm: out must be contiguous')
    L.check(L.lib().geob200_add_layernorm(a.data_ptr(), L.ptr(b), weight.data_ptr(), bias.data_ptr(), n, c, float(eps),
                                          y.data_ptr(), L.stream_ptr()), 'add_layernorm')
    return y


def add_layernorm_backward(a, b, weight, grad_y, eps=1e-5, need_weight=True, need_bias=True):
    """(grad_x, grad_weight, grad_bias) of ``add_layernorm``: grad_x is the gradient of both summands; the statistics are recomputed
    from a + b.  grad_weight / grad_bias are fixed-order sums over the rows (None when not requested)."""
    a, b, weight = _detach(a), _detach(b), _detach(weight)
    L.require_cuda(a, 'a', _f32); _f(weight, 'weight'); _f(grad_y, 'grad_y')
    if b is not None:
        L.require_cuda(b, 'b', _f32)
    n, c = a.shape
    if tuple(grad_y.shape) != (n, c) or (b is not None and tuple(b.shape) != (n, c)) or weight.numel() != c:
        raise RuntimeError(f'add_layernorm_backward: b and grad_y must be ({n}, {c}), weight ({c},)')
    dev = a.device
    gx = torch.empty((n, c), dtype=_f32, device=dev)
    gw = torch.empty((c,), dtype=_f32, device=dev) if need_weight else None
    gb = torch.empty((c,), dtype=_f32, device=dev) if need_bias else None
    lib = L.lib()
    ws = L.workspace(lib.geob200_add_layernorm_backward_workspace_bytes(n, c), dev, 'add_layernorm_backward')
    L.check(lib.geob200_add_layernorm_backward(a.data_ptr(), L.ptr(b), weight.data_ptr(), n, c, float(eps), grad_y.data_ptr(),
                                               gx.data_ptr(), L.ptr(gw), L.ptr(gb), ws.data_ptr(), ws.numel(), L.stream_ptr()),
            'add_layernorm_backward')
    return gx, gw, gb


class _AddLayerNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b, weight, bias, eps):
        ctx.save_for_backward(a, b, weight)
        ctx.eps = eps
        return _add_layernorm(a, b, weight, bias, eps)

    @staticmethod
    def backward(ctx, grad):
        a, b, weight = ctx.saved_tensors
        na, nb, nw, nbias = ctx.needs_input_grad[:4]
        gx, gw, gb = add_layernorm_backward(a, b, weight, grad.contiguous(), ctx.eps, nw, nbias)
        return (gx if na else None), (gx if (nb and b is not None) else None), gw, gb, None


def l2_normalize(x):
    """F.normalize(x, p=2, dim=1).  Differentiable w.r.t. x (``l2_normalize_backward``)."""
    if _needs_grad(x):
        return _L2Normalize.apply(x)
    return _l2_normalize(x)


def _l2_normalize(x):
    x = _detach(x)
    _f(x, 'x')
    y = torch.empty_like(x)
    L.check(L.lib().geob200_l2_normalize(x.data_ptr(), x.shape[0], x.shape[1], y.data_ptr(), L.stream_ptr()), 'l2_normalize')
    return y


def l2_normalize_backward(x, grad_y):
    """grad_x of ``l2_normalize``, with the max(|x|, 1e-12) clamp of F.normalize (below it the gradient is grad_y / 1e-12)"""
    x = _detach(x)
    _f(x, 'x'); _f(grad_y, 'grad_y')
    if grad_y.shape != x.shape or x.dim() != 2:
        raise RuntimeError('l2_normalize_backward: x and grad_y must be the same (n, C) shape')
    gx = torch.empty_like(x)
    L.check(L.lib().geob200_l2_normalize_backward(x.data_ptr(), x.shape[0], x.shape[1], grad_y.data_ptr(), gx.data_ptr(), L.stream_ptr()),
            'l2_normalize_backward')
    return gx


class _L2Normalize(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return _l2_normalize(x)

    @staticmethod
    def backward(ctx, grad):
        return l2_normalize_backward(ctx.saved_tensors[0], grad.contiguous())


# ------------------------------------------------------------------------------------------------ matching

def superpoint_matching(ref_feats, src_feats, ref_masks, src_masks, num_correspondences, dual_normalization=True, defer_count=False):
    """reference ``superpoint_matching.py:13-50``.  The number of rows is min(k, #valid ref x #valid src): it is read back
    from the device (one small D2H) unless ``defer_count`` -- then the full-capacity tensors (padding rows: index -1, score 0,
    which ``gather_patches`` turns into empty patches) and the device count are returned and the caller trims later."""
    corr, sc, cnt = _superpoint_matching(ref_feats, src_feats, ref_masks, src_masks, [ref_feats.shape[0], src_feats.shape[0]],
                                         num_correspondences, dual_normalization)
    ri, si, sc = corr[0], corr[1], sc[0]
    if defer_count:
        return ri, si, sc, cnt
    kk = int(cnt.item())
    return ri[:kk], si[:kk], sc[:kk]


def gather_patches(corr_indices, node_knn_indices, node_knn_masks, points):
    return gather_patches_batched(corr_indices.reshape(1, -1), corr_indices.shape[0], [node_knn_indices.shape[0]], [points.shape[0]],
                                  node_knn_indices, node_knn_masks, points)


def patch_scores(ref_feats, src_feats, ref_knn_indices, src_knn_indices):
    """differentiable w.r.t. ``ref_feats`` / ``src_feats`` (see ``patch_scores_backward_batched``)"""
    return _patch_scores(ref_feats, src_feats, [ref_feats.shape[0], src_feats.shape[0]], ref_knn_indices, src_knn_indices)


def sinkhorn(scores, row_masks, col_masks, alpha, num_iterations, inf=1e12):
    """learnable_sinkhorn.py:20-66; differentiable w.r.t. ``scores`` and ``alpha`` (``sinkhorn_backward``)"""
    p, k = scores.shape[0], scores.shape[1]
    dev = scores.device
    if row_masks is None:
        row_masks = torch.ones((p, k), dtype=torch.bool, device=dev)
    if col_masks is None:
        col_masks = torch.ones((p, k), dtype=torch.bool, device=dev)
    if _needs_grad(scores, alpha):
        return _Sinkhorn.apply(scores, row_masks, col_masks, alpha, int(num_iterations), float(inf))
    return _sinkhorn(scores, row_masks, col_masks, alpha, num_iterations, inf)


def _sinkhorn(scores, row_masks, col_masks, alpha, num_iterations, inf):
    scores, alpha = _detach(scores), _detach(alpha)
    _f(scores, 'scores')
    p, k, k2 = scores.shape
    if k != k2:
        raise RuntimeError('sinkhorn: the CUDA kernel handles square patch score matrices')
    out = torch.empty((p, k + 1, k + 1), dtype=_f32, device=scores.device)
    L.check(L.lib().geob200_sinkhorn(scores.data_ptr(), row_masks.data_ptr(), col_masks.data_ptr(), alpha.data_ptr(), p, k,
                                     int(num_iterations), float(inf), out.data_ptr(), L.stream_ptr()), 'sinkhorn')
    return out


def sinkhorn_backward(scores, row_masks, col_masks, alpha, num_iterations, grad_out, inf=1e12):
    """(grad_scores (P, k, k), grad_alpha (0-dim)) of ``sinkhorn`` for the upstream gradient ``grad_out`` (P, k+1, k+1); k = 32, 64
    or 128.  Masked entries get zero; masked lines follow the inf -> infinity limit, so any finite ``grad_out`` gives a finite result."""
    for t, name in ((scores, 'scores'), (alpha, 'alpha'), (grad_out, 'grad_out')):
        _f(t, name)
    L.require_cuda(row_masks, 'row_masks', torch.bool); L.require_cuda(col_masks, 'col_masks', torch.bool)
    p, k, _ = scores.shape
    if tuple(grad_out.shape) != (p, k + 1, k + 1):
        raise RuntimeError(f'sinkhorn_backward: grad_out must be ({p}, {k + 1}, {k + 1}), got {tuple(grad_out.shape)}')
    dev = scores.device
    lib = L.lib()
    gs = torch.empty((p, k, k), dtype=_f32, device=dev)
    ga = torch.empty((), dtype=_f32, device=dev)
    ws = L.workspace(lib.geob200_sinkhorn_backward_workspace_bytes(p, k, int(num_iterations)), dev, tag='sinkhorn_backward')
    L.check(lib.geob200_sinkhorn_backward(scores.data_ptr(), row_masks.data_ptr(), col_masks.data_ptr(), alpha.data_ptr(), p, k,
                                          int(num_iterations), float(inf), grad_out.data_ptr(), gs.data_ptr(), ga.data_ptr(),
                                          ws.data_ptr(), ws.numel(), L.stream_ptr()), 'sinkhorn_backward')
    return gs, ga


class _Sinkhorn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, scores, row_masks, col_masks, alpha, num_iterations, inf):
        ctx.save_for_backward(scores, row_masks, col_masks, alpha)
        ctx.args = (num_iterations, inf)
        return _sinkhorn(scores, row_masks, col_masks, alpha, num_iterations, inf)

    @staticmethod
    def backward(ctx, grad):
        scores, row_masks, col_masks, alpha = ctx.saved_tensors
        num_iterations, inf = ctx.args
        gs, ga = sinkhorn_backward(scores, row_masks, col_masks, alpha, num_iterations, grad.contiguous(), inf)
        return (gs if ctx.needs_input_grad[0] else None, None, None, ga.reshape(alpha.shape) if ctx.needs_input_grad[3] else None,
                None, None)


def local_global_registration(ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, score_mat, k, acceptance_radius,
                              mutual, confidence_threshold, correspondence_threshold, num_refinement_steps,
                              return_details=False, defer_count=False, transform_out=None):
    """``defer_count``: no host read-back -- returns the full-capacity correspondence tensors and the device count
    ``(ref_c, src_c, scores, T, n)``; rows ``[:n]`` are valid.  ``transform_out``: (16,) float view to write T into."""
    T = torch.empty((4, 4), dtype=_f32, device=score_mat.device) if transform_out is None else transform_out
    res = local_global_registration_batched(1, ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, score_mat, k, acceptance_radius,
                                            mutual, confidence_threshold, correspondence_threshold, num_refinement_steps,
                                            transform_out=T.view(1, 16), details=return_details)
    ref_c, src_c, sc, n = res[0][0], res[1][0], res[2][0], res[4]
    if defer_count:
        return ref_c, src_c, sc, T, n
    c = int(n.item())    # the one D2H of the stage: the number of correspondences sizes the returned tensors
    if return_details:
        det = res[5]
        return ref_c[:c], src_c[:c], sc[:c], T, dict(det, corr_patch=det['corr_patch'][0][:c])
    return ref_c[:c], src_c[:c], sc[:c], T


def weighted_procrustes(src_points, ref_points, weights=None, weight_thresh=0.0, eps=1e-5):
    b, n = src_points.shape[0], src_points.shape[1]
    T = torch.empty((b, 4, 4), dtype=_f32, device=src_points.device)
    L.check(L.lib().geob200_weighted_procrustes(src_points.data_ptr(), ref_points.data_ptr(), L.ptr(weights), b, n,
                                                float(weight_thresh), float(eps), T.data_ptr(), L.stream_ptr()),
            'weighted_procrustes')
    return T


def node_correspondences(ref_nodes, src_nodes, ref_knn_points, src_knn_points, transform, pos_radius, ref_masks=None,
                         src_masks=None, ref_knn_masks=None, src_knn_masks=None):
    """Ground-truth superpoint pairs (reference matching.py:231-315).  Asynchronous: returns full-capacity
    ``(indices (M*N,2), overlaps (M*N,), count (1,) int32)``; rows ``[:count]`` are valid (see ``finish_node_correspondences``)."""
    for t, name in ((ref_nodes, 'ref_nodes'), (src_nodes, 'src_nodes'), (ref_knn_points, 'ref_knn_points'),
                    (src_knn_points, 'src_knn_points'), (transform, 'transform')):
        _f(t, name)
    m, n, k = ref_nodes.shape[0], src_nodes.shape[0], ref_knn_points.shape[1]
    if src_knn_points.shape[1] != k or tuple(transform.shape) != (4, 4):
        raise ValueError('node_correspondences: patches must share K and transform must be (4, 4)')
    for t, shape, name in ((ref_masks, (m,), 'ref_masks'), (src_masks, (n,), 'src_masks'),
                           (ref_knn_masks, (m, k), 'ref_knn_masks'), (src_knn_masks, (n, k), 'src_knn_masks')):
        if t is not None:
            L.require_cuda(t, name, torch.bool)
            if tuple(t.shape) != shape:
                raise ValueError('node_correspondences: %s must have shape %s' % (name, shape))
    cap = (m * n + 65535) // 65536 * 65536          # rounded: same block sizes from pair to pair (no allocator churn)
    return _node_correspondences(ref_nodes, src_nodes, ref_knn_points, src_knn_points, ref_masks, src_masks, ref_knn_masks, src_knn_masks,
                                 [m, n], transform, pos_radius, capacity=cap)


def finish_node_correspondences(idx, ov, cnt):
    c = int(cnt.item())
    return idx[:c], ov[:c]


EVAL_MODES = {'3dmatch': 0, 'kitti': 1, 'modelnet': 2}


def evaluate(gt_node_corr_indices, gt_node_corr_overlaps, ref_node_corr_indices, src_node_corr_indices, ref_corr_points,
             src_corr_points, gt_transform, est_transform, src_points, mode, acceptance_overlap, acceptance_radius,
             rmse_threshold=0.0, rre_threshold=0.0, rte_threshold=0.0, out=None, n_gt=None, n_node_corr=None, n_corr=None):
    """Evaluator.forward (reference experiments/<exp>/loss.py:95-159) as one launch; returns a device tensor
    ``[PIR, IR, RRE, RTE, RMSE, RR, #corr, #gt_node_corr]``.  ``n_gt / n_node_corr / n_corr``: optional device int32 counts
    of valid rows when the index / point tensors are full-capacity buffers (no host read-back in between)."""
    dev = est_transform.device
    if out is None:
        out = torch.empty((8,), dtype=_f32, device=dev)
    for t, name in ((ref_corr_points, 'ref_corr_points'), (src_corr_points, 'src_corr_points'), (gt_transform, 'transform'),
                    (est_transform, 'estimated_transform'), (src_points, 'src_points'), (gt_node_corr_overlaps, 'overlaps')):
        _f(t, name)
    for t, name in ((gt_node_corr_indices, 'gt_node_corr_indices'), (ref_node_corr_indices, 'ref_node_corr_indices'),
                    (src_node_corr_indices, 'src_node_corr_indices')):
        L.require_cuda(t, name, _i64)
    L.check(L.lib().geob200_evaluate_counts(gt_node_corr_indices.data_ptr(), gt_node_corr_overlaps.data_ptr(),
                                            gt_node_corr_indices.shape[0], L.ptr(n_gt), float(acceptance_overlap),
                                            ref_node_corr_indices.data_ptr(), src_node_corr_indices.data_ptr(),
                                            ref_node_corr_indices.shape[0], L.ptr(n_node_corr), ref_corr_points.data_ptr(),
                                            src_corr_points.data_ptr(), ref_corr_points.shape[0], L.ptr(n_corr),
                                            float(acceptance_radius), gt_transform.data_ptr(),
                                            est_transform.data_ptr(), src_points.data_ptr(), src_points.shape[0], int(mode),
                                            float(rmse_threshold), float(rre_threshold), float(rte_threshold), out.data_ptr(),
                                            L.stream_ptr()), 'evaluate')
    return out


# ------------------------------------------------------------------------------------------------ batched per-pair stages
# One launch per stage for all pairs of a batch (GeoTransformer.forward_batch); the single-pair ops above are these with B = 1.
# Clouds are stacked [ref_1..ref_B, src_1..src_B]; ``cloud_nodes`` / ``cloud_points`` are the host lists of the 2B per-cloud row
# counts.  A pair gets the same bits alone and in any batch.

def point_to_node_partition_batched(points, nodes, cloud_points, cloud_nodes, point_limit, return_count=False):
    """stacked ``point_to_node_partition``: (point_to_node[, node_sizes], node_masks, knn_indices, knn_masks), indices local to each
    cloud"""
    _f(points, 'points'); _f(nodes, 'nodes')
    n, m = points.shape[0], nodes.shape[0]
    dev = points.device
    p2n = torch.empty((n,), dtype=_i64, device=dev)
    node_masks = torch.empty((m,), dtype=torch.bool, device=dev)
    node_sizes = torch.empty((m,), dtype=_i32, device=dev)
    knn = torch.empty((m, point_limit), dtype=_i64, device=dev)
    knn_masks = torch.empty((m, point_limit), dtype=torch.bool, device=dev)
    L.check(L.lib().geob200_point_to_node_partition_batched(points.data_ptr(), nodes.data_ptr(), len(cloud_nodes), _host_i64(cloud_points),
                                                            _host_i64(cloud_nodes), point_limit, p2n.data_ptr(), node_masks.data_ptr(),
                                                            node_sizes.data_ptr(), knn.data_ptr(), knn_masks.data_ptr(), L.stream_ptr()),
            'point_to_node_partition_batched')
    if return_count:
        return p2n, node_sizes.long(), node_masks, knn, knn_masks
    return p2n, node_masks, knn, knn_masks


def _min_rows(t, rows, name):
    """host check before a launch: the stacked tensor ``t`` holds the ``rows`` rows its clouds address"""
    if t.shape[0] < rows:
        raise RuntimeError(f'{name} has {t.shape[0]} rows, its clouds need {rows}')


def _patch_tables(name, rows, k, *tables):
    """host check before a launch: the (rows, k[, ...]) patch tensors of one call agree"""
    for t in tables:
        if tuple(t.shape[:2]) != (rows, k):
            raise RuntimeError(f'{name}: patch tensors must all have ({rows}, {k}) leading dimensions, got {tuple(t.shape)}')


def gather_patches_batched(corr_indices, n_corr, cloud_nodes, cloud_points, node_knn_indices, node_knn_masks, points):
    """``corr_indices`` (n_clouds, n_corr) int64 local node indices, cloud after cloud -> (n_clouds * n_corr, k) patches; ``None``:
    every node of every cloud is a patch (rows at the superpoint offsets)"""
    _f(points, 'points'); L.require_cuda(node_knn_indices, 'node_knn_indices', _i64); L.require_cuda(node_knn_masks, 'node_knn_masks', torch.bool)
    k = node_knn_indices.shape[1]
    _patch_tables('gather_patches_batched', node_knn_indices.shape[0], k, node_knn_masks)
    _min_rows(node_knn_indices, sum(int(c) for c in cloud_nodes), 'node_knn_indices')
    _min_rows(points, sum(int(c) for c in cloud_points), 'points')
    if corr_indices is not None:
        L.require_cuda(corr_indices, 'corr_indices', _i64)
        if tuple(corr_indices.shape) != (len(cloud_nodes), n_corr):
            raise RuntimeError(f'gather_patches_batched: corr_indices must be ({len(cloud_nodes)}, {n_corr}), got {tuple(corr_indices.shape)}')
    rows = len(cloud_nodes) * n_corr if corr_indices is not None else node_knn_indices.shape[0]
    dev = points.device
    idx = torch.empty((rows, k), dtype=_i64, device=dev)
    msk = torch.empty((rows, k), dtype=torch.bool, device=dev)
    pts = torch.empty((rows, k, 3), dtype=_f32, device=dev)
    L.check(L.lib().geob200_gather_patches_batched(L.ptr(corr_indices), n_corr, len(cloud_nodes), _host_i64(cloud_nodes),
                                                   _host_i64(cloud_points), node_knn_indices.data_ptr(), node_knn_masks.data_ptr(), k,
                                                   points.data_ptr(), idx.data_ptr(), msk.data_ptr(), pts.data_ptr(), L.stream_ptr()),
            'gather_patches_batched')
    return idx, msk, pts


def _ref_rows(cloud_rows):
    """rows of the B ref clouds at the head of a stack [ref_1..ref_B, src_1..src_B]: where the src block starts"""
    return sum(int(c) for c in cloud_rows[:len(cloud_rows) // 2])


def node_correspondences_batched(nodes, knn_points, node_masks, knn_masks, cloud_nodes, transforms, pos_radius):
    """stacked ``node_correspondences``: (indices (R, 2), overlaps (R,), counts (B,) int32) with pair p's rows at
    ``sum_{q<p} n_ref(q) * n_src(q)``"""
    r = _ref_rows(cloud_nodes)
    return _node_correspondences(nodes[:r], nodes[r:], knn_points[:r], knn_points[r:], node_masks[:r], node_masks[r:], knn_masks[:r],
                                 knn_masks[r:], cloud_nodes, transforms, pos_radius)


def _node_correspondences(ref_nodes, src_nodes, ref_knn_points, src_knn_points, ref_masks, src_masks, ref_knn_masks, src_knn_masks,
                          cloud_nodes, transforms, pos_radius, capacity=None):
    """``node_correspondences_batched`` with the ref clouds' nodes / (rows, k, 3) patch points / masks (None = all valid) in the
    ref_* tensors and the src clouds' in the src_* tensors (the two blocks of the C entry point); ``capacity``: rows of the outputs
    (default: the sum of n_ref * n_src over all pairs)."""
    _f(ref_nodes, 'ref_nodes'); _f(src_nodes, 'src_nodes'); _f(ref_knn_points, 'ref_knn_points'); _f(src_knn_points, 'src_knn_points')
    _f(transforms, 'transforms')
    B = len(cloud_nodes) // 2
    k = ref_knn_points.shape[1]
    nn = sum(int(cloud_nodes[p]) * int(cloud_nodes[B + p]) for p in range(B))
    rows = sum(int(c) for c in cloud_nodes)
    cap = max(nn, 1) if capacity is None else capacity
    dev = ref_nodes.device
    lib = L.lib()
    ws = L.workspace(lib.geob200_node_correspondences_batched_workspace_bytes(rows, nn, k), dev, tag='node_corr')
    idx = torch.empty((cap, 2), dtype=_i64, device=dev)
    ov = torch.empty((cap,), dtype=_f32, device=dev)
    cnt = torch.empty((B,), dtype=_i32, device=dev)
    L.check(lib.geob200_node_correspondences_batched(ref_nodes.data_ptr(), src_nodes.data_ptr(), ref_knn_points.data_ptr(),
                                                     src_knn_points.data_ptr(), L.ptr(ref_masks), L.ptr(src_masks), L.ptr(ref_knn_masks),
                                                     L.ptr(src_knn_masks), B, _host_i64(cloud_nodes), k, transforms.data_ptr(),
                                                     float(pos_radius), idx.data_ptr(), ov.data_ptr(), cnt.data_ptr(), ws.data_ptr(),
                                                     ws.numel(), L.stream_ptr()), 'node_correspondences_batched')
    return idx, ov, cnt


def superpoint_matching_batched(feats, masks, cloud_nodes, num_correspondences, dual_normalization=True):
    """stacked ``superpoint_matching`` (deferred counts): (corr (2B, k) int64 -- row p ref / row B + p src indices of pair p,
    scores (B, k), counts (B,) int32)"""
    r = _ref_rows(cloud_nodes)
    return _superpoint_matching(feats[:r], feats[r:], masks[:r], masks[r:], cloud_nodes, num_correspondences, dual_normalization)


def _superpoint_matching(ref_feats, src_feats, ref_masks, src_masks, cloud_nodes, num_correspondences, dual_normalization):
    """``superpoint_matching_batched`` with the ref clouds' rows in ``ref_feats`` / ``ref_masks`` and the src clouds' in
    ``src_feats`` / ``src_masks`` (masks None = all valid)"""
    _f(ref_feats, 'ref_feats'); _f(src_feats, 'src_feats')
    B = len(cloud_nodes) // 2
    k = int(num_correspondences)
    nn = sum(int(cloud_nodes[p]) * int(cloud_nodes[B + p]) for p in range(B))
    rows = sum(int(c) for c in cloud_nodes)
    dev = ref_feats.device
    lib = L.lib()
    ws = L.workspace(lib.geob200_superpoint_matching_batched_workspace_bytes(rows, nn, B), dev)
    corr = torch.empty((2 * B, k), dtype=_i64, device=dev)
    sc = torch.empty((B, k), dtype=_f32, device=dev)
    cnt = torch.empty((B,), dtype=_i32, device=dev)
    L.check(lib.geob200_superpoint_matching_batched(ref_feats.data_ptr(), src_feats.data_ptr(), ref_feats.shape[1], L.ptr(ref_masks),
                                                    L.ptr(src_masks), B, _host_i64(cloud_nodes), k, int(dual_normalization), corr.data_ptr(),
                                                    sc.data_ptr(), cnt.data_ptr(), ws.data_ptr(), ws.numel(), L.stream_ptr()),
            'superpoint_matching_batched')
    return corr, sc, cnt


def patch_scores_batched(feats, cloud_points, ref_knn_indices, src_knn_indices):
    """stacked ``patch_scores``: pair p's patches at rows p * (rows / B) of both index tensors"""
    r = _ref_rows(cloud_points)
    return _patch_scores(feats[:r], feats[r:], cloud_points, ref_knn_indices, src_knn_indices)


def _patch_scores(ref_feats, src_feats, cloud_points, ref_knn_indices, src_knn_indices):
    """``patch_scores_batched`` with the ref clouds' fine rows in ``ref_feats`` and the src clouds' in ``src_feats``"""
    if _needs_grad(ref_feats, src_feats):
        return _PatchScores.apply(ref_feats, src_feats, tuple(int(c) for c in cloud_points), ref_knn_indices, src_knn_indices)
    ref_feats, src_feats = _detach(ref_feats), _detach(src_feats)
    _f(ref_feats, 'ref_feats'); _f(src_feats, 'src_feats')
    L.require_cuda(ref_knn_indices, 'ref_knn_indices', _i64); L.require_cuda(src_knn_indices, 'src_knn_indices', _i64)
    B = len(cloud_points) // 2
    p, k = ref_knn_indices.shape
    if B < 1 or p % B:
        raise RuntimeError(f'patch_scores_batched: {p} patch rows are not a multiple of {B} pairs')
    _patch_tables('patch_scores_batched', p, k, src_knn_indices)
    _min_rows(ref_feats, _ref_rows(cloud_points), 'ref_feats')
    _min_rows(src_feats, sum(int(c) for c in cloud_points[B:]), 'src_feats')
    out = torch.empty((p, k, k), dtype=_f32, device=ref_feats.device)
    L.check(L.lib().geob200_patch_scores_batched(ref_feats.data_ptr(), src_feats.data_ptr(), ref_feats.shape[1], B, _host_i64(cloud_points),
                                                 ref_knn_indices.data_ptr(), src_knn_indices.data_ptr(), p // B, k, out.data_ptr(),
                                                 L.stream_ptr()), 'patch_scores_batched')
    return out


def patch_scores_backward_batched(ref_feats, src_feats, cloud_points, ref_knn_indices, src_knn_indices, grad_scores):
    """(grad_ref_feats, grad_src_feats) of ``_patch_scores`` (ref / src blocks as there) for the upstream gradient ``grad_scores``
    (P, k, k): each feature row sums its (patch, slot) contributions in (patch, slot) order; rows no patch reads get zeros."""
    _f(ref_feats, 'ref_feats'); _f(src_feats, 'src_feats'); _f(grad_scores, 'grad_scores')
    L.require_cuda(ref_knn_indices, 'ref_knn_indices', _i64); L.require_cuda(src_knn_indices, 'src_knn_indices', _i64)
    B = len(cloud_points) // 2
    p, k = ref_knn_indices.shape
    if tuple(grad_scores.shape) != (p, k, k) or tuple(src_knn_indices.shape) != (p, k):
        raise RuntimeError(f'patch_scores_backward_batched: grad_scores must be ({p}, {k}, {k}) and the index tensors ({p}, {k})')
    dev = ref_feats.device
    lib = L.lib()
    gr, gs = torch.empty_like(ref_feats), torch.empty_like(src_feats)
    rows = ref_feats.shape[0] + src_feats.shape[0]
    ws = L.workspace(lib.geob200_patch_scores_backward_batched_workspace_bytes(rows, p, k, ref_feats.shape[1]), dev,
                     tag='patch_scores_backward')
    L.check(lib.geob200_patch_scores_backward_batched(ref_feats.data_ptr(), src_feats.data_ptr(), ref_feats.shape[1], B,
                                                      _host_i64(cloud_points), ref_knn_indices.data_ptr(), src_knn_indices.data_ptr(),
                                                      p // B, k, grad_scores.data_ptr(), gr.data_ptr(), gs.data_ptr(), ws.data_ptr(),
                                                      ws.numel(), L.stream_ptr()), 'patch_scores_backward_batched')
    return gr, gs


class _PatchScores(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ref_feats, src_feats, cloud_points, ref_knn_indices, src_knn_indices):
        ctx.save_for_backward(ref_feats, src_feats, ref_knn_indices, src_knn_indices)
        ctx.cloud_points = cloud_points
        return _patch_scores(ref_feats, src_feats, cloud_points, ref_knn_indices, src_knn_indices)

    @staticmethod
    def backward(ctx, grad):
        ref_feats, src_feats, ri, si = ctx.saved_tensors
        gr, gs = patch_scores_backward_batched(ref_feats, src_feats, ctx.cloud_points, ri, si, grad.contiguous())
        return gr if ctx.needs_input_grad[0] else None, gs if ctx.needs_input_grad[1] else None, None, None, None


def local_global_registration_batched(n_pairs, ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, score_mat, k,
                                      acceptance_radius, mutual, confidence_threshold, correspondence_threshold, num_refinement_steps,
                                      transform_out=None, details=False):
    """stacked ``local_global_registration`` (deferred counts): (ref_c (B, cap, 3), src_c, scores (B, cap), T, counts (B,) int32).
    ``transform_out``: (B, >= 16) float rows (row stride = its stride(0)) to write the transforms into; else T is (B, 16).
    ``details``: also a dict corr_patch (B, cap), patch_transforms (B * P, 4, 4), patch_inliers (B * P,), best (B,)."""
    for t, name in ((ref_knn_points, 'ref_knn_points'), (src_knn_points, 'src_knn_points'), (score_mat, 'score_mat')):
        _f(t, name)
    L.require_cuda(ref_knn_masks, 'ref_knn_masks', torch.bool); L.require_cuda(src_knn_masks, 'src_knn_masks', torch.bool)
    pt, kk = ref_knn_masks.shape
    B = int(n_pairs)
    if B < 1 or pt % B:
        raise RuntimeError(f'local_global_registration_batched: {pt} patch rows are not a multiple of {B} pairs')
    _patch_tables('local_global_registration_batched', pt, kk, src_knn_masks, ref_knn_points, src_knn_points)
    if ref_knn_points.shape[2:] != (3,) or src_knn_points.shape[2:] != (3,):
        raise RuntimeError('local_global_registration_batched: patch points must be (rows, k, 3)')
    if score_mat.shape[0] != pt:
        raise RuntimeError(f'local_global_registration_batched: score_mat must have {pt} patch rows, got {tuple(score_mat.shape)}')
    P = pt // B
    dev = score_mat.device
    lib = L.lib()
    cap = P * kk * k * (1 if mutual else 2)
    ref_c = torch.empty((B, cap, 3), dtype=_f32, device=dev)
    src_c = torch.empty((B, cap, 3), dtype=_f32, device=dev)
    sc = torch.empty((B, cap), dtype=_f32, device=dev)
    cp = torch.empty((B, cap), dtype=_i32, device=dev)
    n = torch.empty((B,), dtype=_i32, device=dev)
    T = torch.empty((B, 16), dtype=_f32, device=dev) if transform_out is None else transform_out
    det = None
    if details:
        det = dict(corr_patch=cp, patch_transforms=torch.empty((pt, 4, 4), dtype=_f32, device=dev),
                   patch_inliers=torch.empty((pt,), dtype=_i32, device=dev), best=torch.empty((B,), dtype=_i32, device=dev))
    ws = L.workspace(lib.geob200_lgr_batched_workspace_bytes(B, P, kk, k), dev)
    L.check(lib.geob200_local_global_registration_batched(
        ref_knn_points.data_ptr(), src_knn_points.data_ptr(), ref_knn_masks.data_ptr(), src_knn_masks.data_ptr(), score_mat.data_ptr(),
        B, P, kk, score_mat.shape[1], k, float(acceptance_radius), int(mutual), float(confidence_threshold), int(correspondence_threshold),
        int(num_refinement_steps), ref_c.data_ptr(), src_c.data_ptr(), sc.data_ptr(), cp.data_ptr(), n.data_ptr(), T.data_ptr(),
        T.stride(0), *(None if det is None else det[key].data_ptr() for key in ('patch_transforms', 'patch_inliers', 'best')),
        ws.data_ptr(), ws.numel(), L.stream_ptr()), 'local_global_registration_batched')
    if details:
        return ref_c, src_c, sc, T, n, det
    return ref_c, src_c, sc, T, n


def evaluate_batched(gt_indices, gt_overlaps, n_gt, corr_indices, n_node_corr, ref_corr_points, src_corr_points, n_corr, gt_transforms,
                     est_transforms, points, cloud_nodes, cloud_points, mode, acceptance_overlap, acceptance_radius, out,
                     rmse_threshold=0.0, rre_threshold=0.0, rte_threshold=0.0):
    """stacked ``evaluate``: row p of ``out`` (B, >= 8 columns, any row stride) = the metrics of pair p; inputs as returned by
    node_correspondences_batched / superpoint_matching_batched / local_global_registration_batched, ``points`` = the stacked
    input clouds (``cloud_points`` their 2B counts)"""
    B = len(cloud_nodes) // 2
    L.require_cuda(gt_indices, 'gt_indices', _i64); L.require_cuda(corr_indices, 'corr_indices', _i64); _f(gt_overlaps, 'gt_overlaps')
    _f(ref_corr_points, 'ref_corr_points'); _f(src_corr_points, 'src_corr_points'); _f(points, 'points')
    for t, name in ((n_gt, 'n_gt'), (n_node_corr, 'n_node_corr'), (n_corr, 'n_corr')):
        L.require_cuda(t, name, _i32)
        if t.numel() < B:
            raise RuntimeError(f'evaluate_batched: {name} must hold {B} counts')
    if corr_indices.ndim != 2 or corr_indices.shape[0] != 2 * B:
        raise RuntimeError(f'evaluate_batched: corr_indices must be ({2 * B}, k), got {tuple(corr_indices.shape)}')
    if ref_corr_points.ndim != 3 or ref_corr_points.shape[0] != B or ref_corr_points.shape[2] != 3 or src_corr_points.shape != ref_corr_points.shape:
        raise RuntimeError(f'evaluate_batched: correspondence points must both be ({B}, capacity, 3)')
    nn = sum(int(cloud_nodes[p]) * int(cloud_nodes[B + p]) for p in range(B))
    _min_rows(gt_indices, nn, 'gt_indices')
    _min_rows(gt_overlaps, nn, 'gt_overlaps')
    _min_rows(points, sum(int(c) for c in cloud_points), 'points')
    k = corr_indices.shape[1]
    L.check(L.lib().geob200_evaluate_batched(
        gt_indices.data_ptr(), gt_overlaps.data_ptr(), n_gt.data_ptr(), float(acceptance_overlap), corr_indices.data_ptr(),
        corr_indices[B:].data_ptr(), k, n_node_corr.data_ptr(), ref_corr_points.data_ptr(), src_corr_points.data_ptr(),
        ref_corr_points.shape[1], n_corr.data_ptr(), float(acceptance_radius), gt_transforms.data_ptr(), est_transforms.data_ptr(),
        est_transforms.stride(0), points.data_ptr(), B, _host_i64(cloud_nodes), _host_i64(cloud_points), int(mode), float(rmse_threshold),
        float(rre_threshold), float(rte_threshold), out.data_ptr(), out.stride(0), L.stream_ptr()), 'evaluate_batched')
    return out


# ------------------------------------------------------------------------------------------------ validation losses
# OverallLoss values (reference experiments/<exp>/loss.py:10-92).  ``out``: (B, >= 3 columns, any row stride)
# rows [loss, c_loss, f_loss]; the coarse call writes column 1, the fine call column 2 and, given ``loss_weights``, column 0 from
# column 1 -- so run the fine call after the coarse one on the same stream.  Counts are optional DEVICE int32 tensors: no read-back.
# When gradients are required (grad mode on and the features / scores require grad) the calls return fresh (B, 3) rows (zeros in the
# columns they do not write) carrying the graph to ``ref_feats`` / ``src_feats`` (coarse) and ``matching_scores`` (fine); ``out`` must
# then be None.  The values are the same kernels' either way.

def _loss_rows(out, B, dev):
    if out is None:
        out = torch.empty((B, 3), dtype=_f32, device=dev)
    view = out.reshape(1, -1) if out.ndim == 1 else out
    if view.shape[0] != B or view.shape[1] < 3 or view.stride(1) != 1 or view.dtype != _f32 or not view.is_cuda:
        raise RuntimeError(f'loss out must be a float32 CUDA tensor of {B} rows with >= 3 contiguous columns')
    return out, view


def coarse_matching_loss_batched(ref_feats, src_feats, cloud_nodes, gt_indices, gt_overlaps, gt_count, positive_margin, negative_margin,
                                 positive_optimal, negative_optimal, log_scale, positive_overlap, out=None):
    """CoarseMatchingLoss of B pairs: pair p's superpoints at rows sum_{q<p} n_ref(q) of ``ref_feats`` / sum_{q<p} n_src(q) of
    ``src_feats`` (``cloud_nodes``: 2B host counts, ref clouds first), its ground-truth rows at sum_{q<p} n_ref(q) * n_src(q) of
    ``gt_indices`` / ``gt_overlaps`` with ``gt_count[p]`` (device int32) valid.  Writes column 1 of ``out``."""
    coarse = dict(cloud_nodes=tuple(int(c) for c in cloud_nodes), gt_indices=gt_indices, gt_overlaps=gt_overlaps, gt_count=gt_count,
                  params=(positive_margin, negative_margin, positive_optimal, negative_optimal, log_scale, positive_overlap))
    if _needs_grad(ref_feats, src_feats):
        _no_out(out)
        return _LossRows.apply(ref_feats, src_feats, None, coarse, None, None)
    return _coarse_loss_values(ref_feats, src_feats, out=out, **coarse)


def _no_out(out):
    if out is not None:
        raise RuntimeError('loss out= is a value-only buffer: pass out=None when gradients are required')


def _coarse_loss_values(ref_feats, src_feats, cloud_nodes, gt_indices, gt_overlaps, gt_count, params, out):
    ref_feats, src_feats = _detach(ref_feats), _detach(src_feats)
    positive_margin, negative_margin, positive_optimal, negative_optimal, log_scale, positive_overlap = params
    _f(ref_feats, 'ref_feats'); _f(src_feats, 'src_feats'); _f(gt_overlaps, 'gt_node_corr_overlaps')
    L.require_cuda(gt_indices, 'gt_node_corr_indices', _i64); L.require_cuda(gt_count, 'gt_count', _i32)
    B = len(cloud_nodes) // 2
    dev = ref_feats.device
    out, view = _loss_rows(out, B, dev)
    rows = sum(int(c) for c in cloud_nodes)
    nn = sum(int(cloud_nodes[p]) * int(cloud_nodes[B + p]) for p in range(B))
    lib = L.lib()
    ws = L.workspace(lib.geob200_coarse_matching_loss_batched_workspace_bytes(rows, nn), dev, tag='coarse_loss')
    L.check(lib.geob200_coarse_matching_loss_batched(
        ref_feats.data_ptr(), src_feats.data_ptr(), ref_feats.shape[1], B, _host_i64(cloud_nodes), gt_indices.data_ptr(),
        gt_overlaps.data_ptr(), gt_count.data_ptr(), float(positive_margin), float(negative_margin), float(positive_optimal),
        float(negative_optimal), float(log_scale), float(positive_overlap), view.data_ptr(), view.stride(0), ws.data_ptr(), ws.numel(),
        L.stream_ptr()), 'coarse_matching_loss_batched')
    return out


def fine_matching_loss_batched(n_pairs, ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, matching_scores, transforms,
                               positive_radius, patch_count=None, loss_weights=None, out=None):
    """FineMatchingLoss of B pairs: patch q of pair p at row p * P + q of the (B * P, k, 3) points, (B * P, k) masks and
    (B * P, k+1, k+1) Sinkhorn scores; ``transforms`` (B, 4, 4); ``patch_count`` (B,) device int32 or None (all P).  Writes column 2
    of ``out``; with ``loss_weights`` = (w_coarse, w_fine) also column 0 from column 1."""
    fine = dict(n_pairs=int(n_pairs), ref_knn_points=ref_knn_points, src_knn_points=src_knn_points, ref_knn_masks=ref_knn_masks,
                src_knn_masks=src_knn_masks, transforms=transforms, positive_radius=positive_radius, patch_count=patch_count)
    if _needs_grad(matching_scores):
        _no_out(out)
        return _LossRows.apply(None, None, matching_scores, None, fine, loss_weights)
    return _fine_loss_values(matching_scores=_detach(matching_scores), loss_weights=loss_weights, out=out, **fine)


def _fine_loss_values(n_pairs, ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, matching_scores, transforms, positive_radius,
                      patch_count, loss_weights, out):
    for t, name in ((ref_knn_points, 'ref_node_corr_knn_points'), (src_knn_points, 'src_node_corr_knn_points'),
                    (matching_scores, 'matching_scores'), (transforms, 'transform')):
        _f(t, name)
    L.require_cuda(ref_knn_masks, 'ref_node_corr_knn_masks', torch.bool); L.require_cuda(src_knn_masks, 'src_node_corr_knn_masks', torch.bool)
    if patch_count is not None:
        L.require_cuda(patch_count, 'patch_count', _i32)
    B = int(n_pairs)
    rows, k = ref_knn_masks.shape
    dev = matching_scores.device
    out, view = _loss_rows(out, B, dev)
    lib = L.lib()
    ws = L.workspace(lib.geob200_fine_matching_loss_batched_workspace_bytes(B, rows // B), dev, tag='fine_loss')
    w = None if loss_weights is None else (ctypes.c_float * 2)(float(loss_weights[0]), float(loss_weights[1]))
    L.check(lib.geob200_fine_matching_loss_batched(
        ref_knn_points.data_ptr(), src_knn_points.data_ptr(), ref_knn_masks.data_ptr(), src_knn_masks.data_ptr(),
        matching_scores.data_ptr(), transforms.data_ptr(), B, rows // B, k, L.ptr(patch_count), float(positive_radius), w,
        view.data_ptr(), view.stride(0), ws.data_ptr(), ws.numel(), L.stream_ptr()), 'fine_matching_loss_batched')
    return out


def _grad_rows(grad_rows, B):
    _f(grad_rows, 'grad_rows')
    if grad_rows.dim() != 2 or grad_rows.shape[0] != B or grad_rows.shape[1] < 3:
        raise RuntimeError(f'grad_rows must be ({B}, >= 3)')
    return grad_rows


def _host_weights(loss_weights):
    return None if loss_weights is None else (ctypes.c_float * 2)(float(loss_weights[0]), float(loss_weights[1]))


def coarse_matching_loss_backward_batched(ref_feats, src_feats, cloud_nodes, gt_indices, gt_overlaps, gt_count, params, grad_rows,
                                          loss_weights=None):
    """(grad_ref_feats, grad_src_feats) of ``coarse_matching_loss_batched`` (``params``: its six float arguments in order) for the
    upstream gradient ``grad_rows`` (B, >= 3) of the [loss, c_loss, f_loss] rows; column 0 reaches c_loss through loss_weights[0]."""
    _f(ref_feats, 'ref_feats'); _f(src_feats, 'src_feats'); _f(gt_overlaps, 'gt_node_corr_overlaps')
    L.require_cuda(gt_indices, 'gt_node_corr_indices', _i64); L.require_cuda(gt_count, 'gt_count', _i32)
    B = len(cloud_nodes) // 2
    grad_rows = _grad_rows(grad_rows, B)
    dev = ref_feats.device
    rows = sum(int(c) for c in cloud_nodes)
    nn = sum(int(cloud_nodes[p]) * int(cloud_nodes[B + p]) for p in range(B))
    lib = L.lib()
    gr, gs = torch.empty_like(ref_feats), torch.empty_like(src_feats)
    ws = L.workspace(lib.geob200_coarse_matching_loss_backward_batched_workspace_bytes(rows, nn, B), dev, tag='coarse_loss_backward')
    L.check(lib.geob200_coarse_matching_loss_backward_batched(
        ref_feats.data_ptr(), src_feats.data_ptr(), ref_feats.shape[1], B, _host_i64(cloud_nodes), gt_indices.data_ptr(),
        gt_overlaps.data_ptr(), gt_count.data_ptr(), *(float(v) for v in params), grad_rows.data_ptr(), grad_rows.stride(0),
        _host_weights(loss_weights), gr.data_ptr(), gs.data_ptr(), ws.data_ptr(), ws.numel(), L.stream_ptr()),
        'coarse_matching_loss_backward_batched')
    return gr, gs


def fine_matching_loss_backward_batched(n_pairs, ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, transforms, positive_radius,
                                        grad_rows, patch_count=None, loss_weights=None):
    """grad of ``fine_matching_loss_batched`` w.r.t. its (B * P, k+1, k+1) matching scores for the upstream gradient ``grad_rows``
    (B, >= 3): -g_p / #labels of pair p on the label entries, 0 elsewhere; column 0 reaches f_loss through loss_weights[1]."""
    for t, name in ((ref_knn_points, 'ref_node_corr_knn_points'), (src_knn_points, 'src_node_corr_knn_points'), (transforms, 'transform')):
        _f(t, name)
    L.require_cuda(ref_knn_masks, 'ref_node_corr_knn_masks', torch.bool); L.require_cuda(src_knn_masks, 'src_node_corr_knn_masks', torch.bool)
    if patch_count is not None:
        L.require_cuda(patch_count, 'patch_count', _i32)
    B = int(n_pairs)
    grad_rows = _grad_rows(grad_rows, B)
    rows, k = ref_knn_masks.shape
    dev = ref_knn_points.device
    lib = L.lib()
    g = torch.empty((rows, k + 1, k + 1), dtype=_f32, device=dev)
    ws = L.workspace(lib.geob200_fine_matching_loss_backward_batched_workspace_bytes(B, rows // B), dev, tag='fine_loss_backward')
    L.check(lib.geob200_fine_matching_loss_backward_batched(
        ref_knn_points.data_ptr(), src_knn_points.data_ptr(), ref_knn_masks.data_ptr(), src_knn_masks.data_ptr(), transforms.data_ptr(), B,
        rows // B, k, L.ptr(patch_count), float(positive_radius), grad_rows.data_ptr(), grad_rows.stride(0), _host_weights(loss_weights),
        g.data_ptr(), ws.data_ptr(), ws.numel(), L.stream_ptr()), 'fine_matching_loss_backward_batched')
    return g


class _LossRows(torch.autograd.Function):
    """[loss, c_loss, f_loss] rows (B, 3) of the coarse loss (``coarse``: the arguments of _coarse_loss_values), the fine loss
    (``fine``) or both, from the value kernels; backward through the loss backward kernels.  With ``weights`` (w_coarse, w_fine)
    column 0 is the weighted total, as the fine value kernel writes it."""

    @staticmethod
    def forward(ctx, ref_feats, src_feats, scores, coarse, fine, weights):
        B = len(coarse['cloud_nodes']) // 2 if coarse is not None else fine['n_pairs']
        dev = (scores if scores is not None else ref_feats).device
        out = torch.zeros((B, 3), dtype=_f32, device=dev)
        if coarse is not None:
            _coarse_loss_values(ref_feats, src_feats, out=out, **coarse)
        if fine is not None:
            _fine_loss_values(matching_scores=scores, loss_weights=weights, out=out, **fine)
        ctx.save_for_backward(ref_feats, src_feats)
        ctx.coarse, ctx.fine, ctx.weights = coarse, fine, weights
        return out

    @staticmethod
    def backward(ctx, grad):
        ref_feats, src_feats = ctx.saved_tensors
        grad = grad.contiguous()
        gr = gs = gsc = None
        if ctx.coarse is not None and (ctx.needs_input_grad[0] or ctx.needs_input_grad[1]):
            gr, gs = coarse_matching_loss_backward_batched(ref_feats, src_feats, grad_rows=grad, loss_weights=ctx.weights, **ctx.coarse)
        if ctx.fine is not None and ctx.needs_input_grad[2]:
            gsc = fine_matching_loss_backward_batched(grad_rows=grad, loss_weights=ctx.weights, **ctx.fine)
        return gr, gs, gsc, None, None, None


def matching_losses_batched(ref_feats, src_feats, matching_scores, coarse, fine, loss_weights):
    """OverallLoss rows (B, 3) [loss, c_loss, f_loss] with gradients: ``coarse`` / ``fine`` are the keyword arguments of
    ``coarse_matching_loss_batched`` (cloud_nodes, gt_indices, gt_overlaps, gt_count, params = the six floats) and
    ``fine_matching_loss_batched`` (n_pairs, ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, transforms, positive_radius,
    patch_count) without the differentiable inputs."""
    coarse = dict(coarse, cloud_nodes=tuple(int(c) for c in coarse['cloud_nodes']))
    return _LossRows.apply(ref_feats, src_feats, matching_scores, coarse, fine, tuple(loss_weights))


def _one_count(n, count, dev):
    return count.reshape(1) if count is not None else torch.full((1,), int(n), dtype=_i32, device=dev)


def coarse_matching_loss(ref_feats, src_feats, gt_node_corr_indices, gt_node_corr_overlaps, positive_margin, negative_margin,
                         positive_optimal, negative_optimal, log_scale, positive_overlap, out=None, n_gt=None):
    """CoarseMatchingLoss of one pair (the batched kernels with B = 1); ``out``: (>= 3,) row, column 1 written.
    ``n_gt``: optional device int32 count of valid ground-truth rows (full-capacity buffers)."""
    dev = ref_feats.device
    cnt = _one_count(gt_node_corr_indices.shape[0], n_gt, dev)
    args = ([ref_feats.shape[0], src_feats.shape[0]], gt_node_corr_indices, gt_node_corr_overlaps, cnt, positive_margin, negative_margin,
            positive_optimal, negative_optimal, log_scale, positive_overlap)
    if _needs_grad(ref_feats, src_feats):
        _no_out(out)
        return coarse_matching_loss_batched(ref_feats, src_feats, *args).reshape(3)
    if out is None:
        out = torch.empty((3,), dtype=_f32, device=dev)
    coarse_matching_loss_batched(ref_feats, src_feats, *args, out=out)
    return out


def fine_matching_loss(ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, matching_scores, transform, positive_radius,
                       loss_weights=None, out=None, n_patches=None):
    """FineMatchingLoss of one pair; ``out``: (>= 3,) row, column 2 (and column 0 given ``loss_weights``) written.
    ``n_patches``: optional device int32 count of valid patches (full-capacity buffers)."""
    dev = matching_scores.device
    kw = dict(patch_count=None if n_patches is None else n_patches.reshape(1), loss_weights=loss_weights)
    args = (1, ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, matching_scores, transform, positive_radius)
    if _needs_grad(matching_scores):
        _no_out(out)
        return fine_matching_loss_batched(*args, **kw).reshape(3)
    if out is None:
        out = torch.empty((3,), dtype=_f32, device=dev)
    fine_matching_loss_batched(*args, **kw, out=out)
    return out


# ------------------------------------------------------------------------------------------------ correspondence RANSAC
# Open3D's registration_ransac_based_on_correspondence as the reference calls it (utils/open3d.py:169-198); semantics and the
# deviations from Open3D (sampler, tie rule, fp32 scoring) in DESIGN.md section 3b.  Pair p's correspondences are rows
# [0, num_corr[p]) of (B, capacity, 3) tensors -- the layout local_global_registration_batched returns.

RANSAC_KEYS = ('transform', 'fitness', 'inlier_rmse', 'inliers', 'iteration')


def ransac_correspondences_batched(src_corr_points, ref_corr_points, distance_threshold, ransac_n, num_iterations, seed=0, num_corr=None,
                                   records=False, first_pair=0):
    """RANSAC of B pairs in one launch pair, no host synchronisation.  ``num_corr``: (B,) device int32 counts or None (all rows).
    Pair p draws its samples from the stream (seed, first_pair + p): a pair gives the same result alone (``first_pair`` = its id)
    as inside any batch.
    Returns a dict: transform (B, 4, 4), fitness (B,), inlier_rmse (B,), inliers (B,) int32, iteration (B,) int32 (-1: no
    hypothesis with an inlier, or fewer than ransac_n correspondences: identity, fitness 0).  ``records``: also the
    per-hypothesis hyp_transforms (B, I, 4, 4), hyp_inliers (B, I), hyp_rmse (B, I), hyp_samples (B, I, ransac_n) int32."""
    _f(src_corr_points, 'src_corr_points'); _f(ref_corr_points, 'ref_corr_points')
    if src_corr_points.ndim != 3 or src_corr_points.shape[2] != 3 or ref_corr_points.shape != src_corr_points.shape:
        raise ValueError('ransac_correspondences_batched: src / ref must both be (B, capacity, 3)')
    if not 0 <= int(seed) < 1 << 64:
        raise ValueError('ransac_correspondences_batched: seed must be a 64-bit unsigned integer')
    B, cap = src_corr_points.shape[0], src_corr_points.shape[1]
    I = int(num_iterations)
    dev = src_corr_points.device
    if ref_corr_points.device != dev:
        raise RuntimeError('ransac_correspondences_batched: src and ref must be on one device')
    if num_corr is not None:
        L.require_cuda(num_corr, 'num_corr', _i32)
        if num_corr.numel() != B or num_corr.device != dev:
            raise ValueError('ransac_correspondences_batched: num_corr must hold one count per pair, on the points\' device')
    lib = L.lib()
    T = torch.empty((B, 4, 4), dtype=_f32, device=dev)
    fit = torch.empty((B,), dtype=_f32, device=dev)
    rmse = torch.empty((B,), dtype=_f32, device=dev)
    inl = torch.empty((B,), dtype=_i32, device=dev)
    it = torch.empty((B,), dtype=_i32, device=dev)
    rec = None
    if records:
        rec = dict(hyp_transforms=torch.empty((B, max(I, 1), 4, 4), dtype=_f32, device=dev),
                   hyp_inliers=torch.empty((B, max(I, 1)), dtype=_i32, device=dev),
                   hyp_rmse=torch.empty((B, max(I, 1)), dtype=_f32, device=dev),
                   hyp_samples=torch.empty((B, max(I, 1), 8), dtype=_i32, device=dev))
    ws = L.workspace(lib.geob200_ransac_correspondences_batched_workspace_bytes(B, I), dev, tag='ransac')
    L.check(lib.geob200_ransac_correspondences_batched(
        ref_corr_points.data_ptr(), src_corr_points.data_ptr(), B, cap, L.ptr(num_corr), float(distance_threshold), int(ransac_n), I,
        ctypes.c_uint64(int(seed)), int(first_pair), T.data_ptr(), fit.data_ptr(), rmse.data_ptr(), inl.data_ptr(), it.data_ptr(),
        *(None if rec is None else rec[k].data_ptr() for k in ('hyp_transforms', 'hyp_inliers', 'hyp_rmse', 'hyp_samples')),
        ws.data_ptr(), ws.numel(), L.stream_ptr()), 'ransac_correspondences_batched')
    res = dict(transform=T, fitness=fit, inlier_rmse=rmse, inliers=inl, iteration=it)
    if rec is not None:
        rec['hyp_samples'] = rec['hyp_samples'][:, :, :int(ransac_n)]
        res.update(rec)
    return res


def ransac_correspondences(src_corr_points, ref_corr_points, distance_threshold, ransac_n, num_iterations, seed=0, num_corr=None,
                           records=False, pair=0):
    """RANSAC of one pair: (N, 3) src / ref correspondence points (``num_corr``: optional (1,) device int32 count of valid rows;
    ``pair``: the pair id of the random stream, see the batched op).
    Same dict as the batched op without the pair dimension: transform (4, 4), fitness, inlier_rmse, inliers, iteration."""
    res = ransac_correspondences_batched(src_corr_points.unsqueeze(0), ref_corr_points.unsqueeze(0), distance_threshold, ransac_n,
                                         num_iterations, seed=seed, num_corr=None if num_corr is None else num_corr.reshape(1),
                                         records=records, first_pair=pair)
    return {k: v[0] for k, v in res.items()}


# ------------------------------------------------------------------------------------------------ feature matching
# get_nearest_neighbor / extract_corr_indices_from_feats (utils/pointcloud.py:11-22, utils/registration.py:179-234) and Open3D 0.11's
# registration_ransac_based_on_feature_matching as utils/open3d.py:133-166 calls it (csrc/feature_match.cu, csrc/ransac.cu;
# semantics and deviations in DESIGN.md section 3b).  Ragged layout: pair p's rows are [0, count[p]) of (B, capacity, .) tensors.

def _ragged(x, name, B=None, width=None):
    _f(x, name)
    if x.ndim != 3 or (B is not None and x.shape[0] != B) or (width is not None and x.shape[2] != width):
        raise ValueError(f'{name} must be (B, capacity, {width or "C"})')
    return x


def feature_nearest_neighbor_batched(query, support, num_query=None, num_support=None, bidirectional=False):
    """Exact nearest support row of every query row: (B, cap_q, C) and (B, cap_s, C) float32, C in 1..1024; counts (B,) device int32
    or None.  Returns (index (B, cap_q) int64, distance (B, cap_q) float64) -- index = argmin of the fp64 squared distance (lowest
    index on exact ties), distance = its sqrt; rows past the count: -1 / NaN.  ``bidirectional``: also the nearest query row of
    every support row, as a second (index, distance) pair."""
    _ragged(query, 'query'); _ragged(support, 'support', query.shape[0], query.shape[2])
    B, cq, C = query.shape
    cs = support.shape[1]
    dev = query.device
    if support.device != dev:
        raise RuntimeError('feature_nearest_neighbor_batched: query and support must be on one device')
    _counts(num_query, B, dev, 'feature_nearest_neighbor_batched')
    _counts(num_support, B, dev, 'feature_nearest_neighbor_batched')
    lib = L.lib()
    qi = torch.empty((B, cq), dtype=_i64, device=dev)
    qd = torch.empty((B, cq), dtype=torch.float64, device=dev)
    si = torch.empty((B, cs), dtype=_i64, device=dev) if bidirectional else None
    sd = torch.empty((B, cs), dtype=torch.float64, device=dev) if bidirectional else None
    ws = L.workspace(lib.geob200_feature_nn_batched_workspace_bytes(B, cq, cs), dev, tag='feature_nn')
    L.check(lib.geob200_feature_nn_batched(query.data_ptr(), support.data_ptr(), B, cq, cs, C, L.ptr(num_query), L.ptr(num_support),
                                           qi.data_ptr(), qd.data_ptr(), L.ptr(si), L.ptr(sd), ws.data_ptr(), ws.numel(), L.stream_ptr()),
            'feature_nearest_neighbor_batched')
    return (qi, qd, si, sd) if bidirectional else (qi, qd)


def feature_nearest_neighbor(query, support, bidirectional=False):
    """One pair: (N, C) query, (M, C) support -> (index (N,) int64, distance (N,) float64)[, (M,) support -> query pair]."""
    res = feature_nearest_neighbor_batched(query.unsqueeze(0), support.unsqueeze(0), bidirectional=bidirectional)
    return tuple(v[0] for v in res)


CORR_MODES = {'plain': 0, 'mutual': 1, 'bilateral': 2}


def feature_correspondences(ref_nn, ref_dist, src_nn=None, src_dist=None, mode='plain'):
    """extract_corr_indices_from_feats from the two nearest-neighbour directions of one pair (ref -> src: ref_nn / ref_dist (N,);
    src -> ref: src_nn / src_dist (M,), needed for 'mutual' and 'bilateral').  Returns (ref indices, src indices) int64 and the
    listed pairs' descriptor distances (float32).  The mutual count is read back to the host (the lists' length)."""
    m = CORR_MODES[mode]
    for t, name in ((ref_nn, 'ref_nn'), (src_nn, 'src_nn')):
        if t is not None:
            L.require_cuda(t, name, _i64)
    for t, name in ((ref_dist, 'ref_dist'), (src_dist, 'src_dist')):
        if t is not None:
            L.require_cuda(t, name, torch.float64)
    if m and (src_nn is None or src_dist is None):
        raise ValueError(f'feature_correspondences: mode {mode!r} needs both directions')
    n, k = ref_nn.numel(), (0 if src_nn is None else src_nn.numel())
    dev = ref_nn.device
    rows = n + k if m == 2 else n
    ref_corr = torch.empty((rows,), dtype=_i64, device=dev)
    src_corr = torch.empty((rows,), dtype=_i64, device=dev)
    dist = torch.empty((rows,), dtype=_f32, device=dev)
    cnt = torch.empty((1,), dtype=_i32, device=dev)
    L.check(L.lib().geob200_feature_corr_indices(ref_nn.data_ptr(), ref_dist.data_ptr(), L.ptr(src_nn), L.ptr(src_dist), n, k, m,
                                                 ref_corr.data_ptr(), src_corr.data_ptr(), dist.data_ptr(), cnt.data_ptr(),
                                                 L.stream_ptr()), 'feature_correspondences')
    if m == 1:
        c = int(cnt.item())
        ref_corr, src_corr, dist = ref_corr[:c], src_corr[:c], dist[:c]
    return ref_corr, src_corr, dist


FEATURE_RANSAC_KEYS = RANSAC_KEYS + ('num_validated',)


def ransac_features_batched(src_points, ref_points, src_feats, ref_feats, distance_threshold, ransac_n, num_iterations, val_iterations,
                            seed=0, num_src=None, num_ref=None, records=False, first_pair=0):
    """Feature-matching RANSAC of B pairs in one call, no host synchronisation: src (B, cap_src, 3) points and (B, cap_src, C)
    descriptors, ref likewise; num_src / num_ref (B,) device int32 or None.  Pair p draws from the stream (seed, first_pair + p), so
    a pair gives the same bits alone (``first_pair`` = its id) as inside any batch.
    Returns a dict: transform (B, 4, 4), fitness, inlier_rmse, inliers int32, iteration int32 (the winning iteration, -1 for the
    default result: identity, fitness 0), num_validated int32.  ``records``: also matches (B, cap_src) int64, samples
    (B, I, ransac_n) int32, pass_flags (B, I) int32, val_ids (B, V') int32 (-1 past num_validated), val_transforms (B, V', 4, 4),
    val_inliers (B, V'), val_rmse (B, V') with V' = min(val_iterations, num_iterations)."""
    _ragged(src_points, 'src_points', width=3)
    B = src_points.shape[0]
    _ragged(ref_points, 'ref_points', B, 3)
    _ragged(src_feats, 'src_feats', B); _ragged(ref_feats, 'ref_feats', B, src_feats.shape[2])
    if src_feats.shape[1] != src_points.shape[1] or ref_feats.shape[1] != ref_points.shape[1]:
        raise ValueError('ransac_features_batched: points and descriptors need the same capacity')
    if not 0 <= int(seed) < 1 << 64:
        raise ValueError('ransac_features_batched: seed must be a 64-bit unsigned integer')
    dev = src_points.device
    if any(t.device != dev for t in (ref_points, src_feats, ref_feats)):
        raise RuntimeError('ransac_features_batched: all inputs must be on one device')
    _counts(num_src, B, dev, 'ransac_features_batched')
    _counts(num_ref, B, dev, 'ransac_features_batched')
    cs, cr, C = src_points.shape[1], ref_points.shape[1], src_feats.shape[2]
    I, V = int(num_iterations), int(val_iterations)
    Vr = max(min(I, V), 1)
    lib = L.lib()
    T = torch.empty((B, 4, 4), dtype=_f32, device=dev)
    fit = torch.empty((B,), dtype=_f32, device=dev)
    rmse = torch.empty((B,), dtype=_f32, device=dev)
    inl = torch.empty((B,), dtype=_i32, device=dev)
    it = torch.empty((B,), dtype=_i32, device=dev)
    nv = torch.empty((B,), dtype=_i32, device=dev)
    rec = None
    if records:
        rec = dict(matches=torch.full((B, max(cs, 1)), -1, dtype=_i64, device=dev),
                   samples=torch.full((B, max(I, 1), 8), -1, dtype=_i32, device=dev),
                   pass_flags=torch.zeros((B, max(I, 1)), dtype=_i32, device=dev),
                   val_ids=torch.full((B, Vr), -1, dtype=_i32, device=dev),
                   val_transforms=torch.zeros((B, Vr, 4, 4), dtype=_f32, device=dev),
                   val_inliers=torch.zeros((B, Vr), dtype=_i32, device=dev),
                   val_rmse=torch.zeros((B, Vr), dtype=_f32, device=dev))
    ws = L.workspace(lib.geob200_ransac_features_batched_workspace_bytes(B, cs, cr, I, V), dev, tag='ransac_features')
    L.check(lib.geob200_ransac_features_batched(
        src_points.data_ptr(), ref_points.data_ptr(), src_feats.data_ptr(), ref_feats.data_ptr(), B, cs, cr, C, L.ptr(num_src),
        L.ptr(num_ref), float(distance_threshold), int(ransac_n), I, V, ctypes.c_uint64(int(seed)), int(first_pair), T.data_ptr(),
        fit.data_ptr(), rmse.data_ptr(), inl.data_ptr(), it.data_ptr(), nv.data_ptr(),
        *(None if rec is None else rec[k].data_ptr() for k in ('matches', 'samples', 'pass_flags', 'val_ids', 'val_transforms',
                                                                'val_inliers', 'val_rmse')),
        ws.data_ptr(), ws.numel(), L.stream_ptr()), 'ransac_features_batched')
    res = dict(transform=T, fitness=fit, inlier_rmse=rmse, inliers=inl, iteration=it, num_validated=nv)
    if rec is not None:
        rec['samples'] = rec['samples'][:, :, :max(int(ransac_n), 0)]
        res.update(rec)
    return res


def ransac_features(src_points, ref_points, src_feats, ref_feats, distance_threshold, ransac_n, num_iterations, val_iterations, seed=0,
                    records=False, pair=0):
    """Feature-matching RANSAC of one pair: (N, 3) / (N, C) src, (M, 3) / (M, C) ref (``pair``: the pair id of the random stream).
    Same dict as the batched op without the pair dimension."""
    res = ransac_features_batched(src_points.unsqueeze(0), ref_points.unsqueeze(0), src_feats.unsqueeze(0), ref_feats.unsqueeze(0),
                                  distance_threshold, ransac_n, num_iterations, val_iterations, seed=seed, records=records,
                                  first_pair=pair)
    return {k: v[0] for k, v in res.items()}


CORRESPONDENCE_METRICS = ('f_IR', 'f_OV', 'f_RS', 'f_NU')


def correspondence_metrics_batched(ref_corr_points, src_corr_points, transforms, positive_radius, num_corr=None, out=None):
    """evaluate_correspondences (utils/registration.py:240-250) of B pairs in the RANSAC layout under ``transforms`` (B, 4, 4) or
    (B, >= 16) rows: row p of ``out`` (B, >= 4, any row stride) = [f_IR, f_OV, f_RS, f_NU] (inlier ratio, overlap, mean residual,
    count; the means of an empty pair are NaN)."""
    _f(ref_corr_points, 'ref_corr_points'); _f(src_corr_points, 'src_corr_points')
    if src_corr_points.ndim != 3 or src_corr_points.shape[2] != 3 or ref_corr_points.shape != src_corr_points.shape:
        raise ValueError('correspondence_metrics_batched: src / ref must both be (B, capacity, 3)')
    B, cap = src_corr_points.shape[0], src_corr_points.shape[1]
    tr = transforms.reshape(B, -1) if transforms.is_contiguous() else transforms
    if tr.dtype != _f32 or not tr.is_cuda or tr.shape[1] < 12 or tr.stride(1) != 1:
        raise RuntimeError('correspondence_metrics_batched: transforms must be float32 CUDA rows of >= 12 contiguous values')
    dev = src_corr_points.device
    if ref_corr_points.device != dev or tr.device != dev:
        raise RuntimeError('correspondence_metrics_batched: points and transforms must be on one device')
    if num_corr is not None:
        L.require_cuda(num_corr, 'num_corr', _i32)
        if num_corr.numel() != B or num_corr.device != dev:
            raise ValueError('correspondence_metrics_batched: num_corr must hold one count per pair, on the points\' device')
    if out is None:
        out = torch.empty((B, 4), dtype=_f32, device=dev)
    if out.shape[0] != B or out.shape[1] < 4 or out.stride(1) != 1 or out.dtype != _f32 or out.device != dev:
        raise RuntimeError('correspondence_metrics_batched: out must be float32 CUDA rows of >= 4 contiguous columns')
    lib = L.lib()
    ws = L.workspace(lib.geob200_correspondence_metrics_batched_workspace_bytes(B, cap), dev, tag='corr_metrics')
    L.check(lib.geob200_correspondence_metrics_batched(ref_corr_points.data_ptr(), src_corr_points.data_ptr(), B, cap, L.ptr(num_corr),
                                                       tr.data_ptr(), tr.stride(0), float(positive_radius), out.data_ptr(), out.stride(0),
                                                       ws.data_ptr(), ws.numel(), L.stream_ptr()), 'correspondence_metrics_batched')
    return out


def evaluate_correspondences(ref_corr_points, src_corr_points, transform, positive_radius=0.1):
    """one pair: (4,) device tensor [f_IR, f_OV, f_RS, f_NU]"""
    return correspondence_metrics_batched(ref_corr_points.unsqueeze(0), src_corr_points.unsqueeze(0), transform.reshape(1, 16).contiguous(),
                                          positive_radius)[0]


# ------------------------------------------------------------------------------------------------ benchmark evaluation
# The per-pair stages of eval.py that RANSAC and the correspondence metrics above do not cover (csrc/benchmark.cu).  Same
# ragged layout: pair p's rows are [0, count[p]) of (B, capacity, ...) tensors, counts are (B,) device int32 or None (all rows).

CORR_ORDER_KMAX = 8192


def _counts(counts, B, dev, what):
    if counts is not None:
        L.require_cuda(counts, 'counts', _i32)
        if counts.numel() != B or counts.device != dev:
            raise ValueError(f'{what}: counts must hold one int32 count per pair, on the inputs\' device')
    return counts


def corr_order_batched(corr_scores, kmax, num_corr=None):
    """(B, kmax) int32: row p = np.argsort(-scores[p, :n], kind='stable')[:kmax] (score descending, then row; NaN last), -1 past
    min(n, kmax).  kmax <= CORR_ORDER_KMAX."""
    _f(corr_scores, 'corr_scores')
    if corr_scores.ndim != 2:
        raise ValueError('corr_order_batched: corr_scores must be (B, capacity)')
    if not 1 <= int(kmax) <= CORR_ORDER_KMAX:
        raise ValueError(f'corr_order_batched: kmax must be in 1..{CORR_ORDER_KMAX}')
    B, cap = corr_scores.shape
    dev = corr_scores.device
    _counts(num_corr, B, dev, 'corr_order_batched')
    order = torch.empty((B, int(kmax)), dtype=_i32, device=dev)
    L.check(L.lib().geob200_corr_order_batched(corr_scores.data_ptr(), B, cap, L.ptr(num_corr), int(kmax), order.data_ptr(),
                                               L.stream_ptr()), 'corr_order_batched')
    return order


def corr_select_batched(ref_corr_points, src_corr_points, corr_scores, order, k, num_corr=None):
    """eval.py's top-k selection with an ``order`` from corr_order_batched: returns (ref (B, K, 3), src (B, K, 3), scores (B, K),
    count (B,) int32) with K = min(k, capacity) and count = min(n, k).  A pair with n <= k keeps its rows in their order."""
    _f(ref_corr_points, 'ref_corr_points'); _f(src_corr_points, 'src_corr_points'); _f(corr_scores, 'corr_scores')
    L.require_cuda(order, 'order', _i32)
    B, cap = corr_scores.shape
    if ref_corr_points.shape != (B, cap, 3) or src_corr_points.shape != (B, cap, 3) or order.ndim != 2 or order.shape[0] != B:
        raise ValueError('corr_select_batched: ref / src must be (B, capacity, 3), scores (B, capacity), order (B, kmax)')
    dev = corr_scores.device
    if any(t.device != dev for t in (ref_corr_points, src_corr_points, order)):
        raise RuntimeError('corr_select_batched: inputs must be on one device')
    _counts(num_corr, B, dev, 'corr_select_batched')
    K = min(int(k), cap)
    ref_o = torch.empty((B, K, 3), dtype=_f32, device=dev)
    src_o = torch.empty((B, K, 3), dtype=_f32, device=dev)
    sc_o = torch.empty((B, K), dtype=_f32, device=dev)
    cnt = torch.empty((B,), dtype=_i32, device=dev)
    L.check(L.lib().geob200_corr_select_batched(ref_corr_points.data_ptr(), src_corr_points.data_ptr(), corr_scores.data_ptr(), B, cap,
                                                L.ptr(num_corr), order.data_ptr(), order.shape[1], int(k), ref_o.data_ptr(),
                                                src_o.data_ptr(), sc_o.data_ptr(), cnt.data_ptr(), L.stream_ptr()), 'corr_select_batched')
    return ref_o, src_o, sc_o, cnt


def sparse_correspondence_eval_batched(ref_node_corr_indices, src_node_corr_indices, gt_node_corr_indices, num_ref_nodes, num_src_nodes,
                                       pred_count=None, gt_count=None):
    """evaluate_sparse_correspondences (utils/registration.py:253-281) of B pairs: (B, 3) float64 [precision, recall, hit_ratio],
    bit-identical to numpy.  Indices: (B, P) int64 ref / src node indices and (B, G, 2) int64 gt pairs; ``num_ref_nodes`` /
    ``num_src_nodes``: host upper bounds of the node indices (the M x N of the reference's dense matrices)."""
    for t, name in ((ref_node_corr_indices, 'ref_node_corr_indices'), (src_node_corr_indices, 'src_node_corr_indices'),
                    (gt_node_corr_indices, 'gt_node_corr_indices')):
        L.require_cuda(t, name, _i64)
    B, pcap = ref_node_corr_indices.shape
    if src_node_corr_indices.shape != (B, pcap) or gt_node_corr_indices.ndim != 3 or gt_node_corr_indices.shape[0] != B \
            or gt_node_corr_indices.shape[2] != 2:
        raise ValueError('sparse_correspondence_eval_batched: indices must be (B, P), (B, P) and (B, G, 2)')
    dev = ref_node_corr_indices.device
    if src_node_corr_indices.device != dev or gt_node_corr_indices.device != dev:
        raise RuntimeError('sparse_correspondence_eval_batched: inputs must be on one device')
    _counts(pred_count, B, dev, 'sparse_correspondence_eval_batched')
    _counts(gt_count, B, dev, 'sparse_correspondence_eval_batched')
    lib = L.lib()
    m, n = int(num_ref_nodes), int(num_src_nodes)
    out = torch.empty((B, 3), dtype=torch.float64, device=dev)
    need = lib.geob200_sparse_correspondence_eval_batched_workspace_bytes(B, m, n)
    ws = L.workspace(need, dev, tag='sparse_eval') if need else None
    L.check(lib.geob200_sparse_correspondence_eval_batched(
        ref_node_corr_indices.data_ptr(), src_node_corr_indices.data_ptr(), pcap, L.ptr(pred_count), gt_node_corr_indices.data_ptr(),
        gt_node_corr_indices.shape[1], L.ptr(gt_count), B, m, n, out.data_ptr(), L.ptr(ws), 0 if ws is None else ws.numel(),
        L.stream_ptr()), 'sparse_correspondence_eval_batched')
    return out


def _transform_rows(t, B, what):
    tr = t.reshape(B, -1) if t.is_contiguous() else t
    if tr.dtype != _f32 or not tr.is_cuda or tr.ndim != 2 or tr.shape[1] < 16 or tr.stride(1) != 1:
        raise RuntimeError(f'{what}: transforms must be float32 CUDA rows of >= 16 contiguous values')
    return tr


def registration_error_batched(gt_transforms, est_transforms, covariances=None, has_covariance=None, rmse_threshold=None,
                               rre_threshold=None, rte_threshold=None):
    """(B, 4) float64 rows [rre (deg), rte, p, accepted], computed in double.  p = compute_transform_error of 3DMatch
    (threedmatch/utils.py:130-136) with the (B, 6, 6) ``covariances`` where ``has_covariance`` (B,) int32 is set, NaN elsewhere.
    Acceptance: ``rmse_threshold`` given = p < rmse_threshold**2 (3DMatch); otherwise rre < rre_threshold and rte < rte_threshold
    (KITTI)."""
    B = gt_transforms.shape[0]
    gt = _transform_rows(gt_transforms, B, 'registration_error_batched')
    est = _transform_rows(est_transforms, B, 'registration_error_batched')
    dev = gt.device
    if est.device != dev or est.shape[0] != B:
        raise RuntimeError('registration_error_batched: gt and est transforms must be B rows on one device')
    if covariances is not None:
        _f(covariances, 'covariances')
        if covariances.numel() != 36 * B or covariances.device != dev:
            raise ValueError('registration_error_batched: covariances must be (B, 6, 6) on the transforms\' device')
    _counts(has_covariance, B, dev, 'registration_error_batched')
    if rmse_threshold is not None:
        if covariances is None:
            raise ValueError('registration_error_batched: the rmse acceptance needs covariances')
        mode, t0, t1 = 0, float(rmse_threshold) ** 2, 0.0
    elif rre_threshold is not None and rte_threshold is not None:
        mode, t0, t1 = 1, float(rre_threshold), float(rte_threshold)
    else:
        raise ValueError('registration_error_batched: give rmse_threshold, or rre_threshold and rte_threshold')
    out = torch.empty((B, 4), dtype=torch.float64, device=dev)
    L.check(L.lib().geob200_registration_error_batched(gt.data_ptr(), gt.stride(0), est.data_ptr(), est.stride(0), L.ptr(covariances),
                                                       L.ptr(has_covariance), B, mode, t0, t1, out.data_ptr(), L.stream_ptr()),
            'registration_error_batched')
    return out


def weighted_procrustes_counts(src_points, ref_points, weights, counts, weight_thresh=0.0, eps=1e-5):
    """weighted_procrustes over ragged problems: problem b = rows [0, counts[b]) of (B, capacity, 3) src / ref and (B, capacity)
    weights (or None); (B, 4, 4), bit-identical to weighted_procrustes on the trimmed rows."""
    _f(src_points, 'src_points'); _f(ref_points, 'ref_points')
    if src_points.ndim != 3 or src_points.shape[2] != 3 or ref_points.shape != src_points.shape:
        raise ValueError('weighted_procrustes_counts: src / ref must both be (B, capacity, 3)')
    B, cap = src_points.shape[0], src_points.shape[1]
    dev = src_points.device
    if weights is not None:
        _f(weights, 'weights')
        if weights.shape != (B, cap) or weights.device != dev:
            raise ValueError('weighted_procrustes_counts: weights must be (B, capacity) on the points\' device')
    if ref_points.device != dev:
        raise RuntimeError('weighted_procrustes_counts: src and ref must be on one device')
    if counts is None:
        raise ValueError('weighted_procrustes_counts: counts are required (weighted_procrustes takes full problems)')
    _counts(counts, B, dev, 'weighted_procrustes_counts')
    T = torch.empty((B, 4, 4), dtype=_f32, device=dev)
    L.check(L.lib().geob200_weighted_procrustes_counts(src_points.data_ptr(), ref_points.data_ptr(), L.ptr(weights), B, cap, counts.data_ptr(),
                                                       float(weight_thresh), float(eps), T.data_ptr(), L.stream_ptr()),
            'weighted_procrustes_counts')
    return T


# ------------------------------------------------------------------------------------------------ training step
# The ground-truth superpoint targets of the training-mode forward and the non-finite gradient guard (csrc/train.cu).  Neither
# reads anything back to the host.

def superpoint_targets_batched(gt_indices, gt_overlaps, gt_count, cloud_nodes, overlap_threshold, num_targets, seed, iteration,
                               pair_base=0):
    """SuperPointTargetGenerator of B pairs on the stacked output of ``node_correspondences_batched``: (corr (2B, num_targets) int64
    -- row p ref / row B + p src indices of pair p, scores (B, num_targets) = the selected overlaps, counts (B,) device int32), the
    layout of ``superpoint_matching_batched``.  Pair p takes all of its gt rows with overlap > ``overlap_threshold`` in gt order when
    there are at most ``num_targets``, else a uniform subset of ``num_targets`` of them drawn from the Philox stream
    (seed, iteration, pair_base + p), in gt order."""
    L.require_cuda(gt_indices, 'gt_indices', _i64); _f(gt_overlaps, 'gt_overlaps'); L.require_cuda(gt_count, 'gt_count', _i32)
    B = len(cloud_nodes) // 2
    if B < 1 or len(cloud_nodes) != 2 * B:
        raise RuntimeError('superpoint_targets_batched: cloud_nodes must hold 2B counts')
    if gt_indices.ndim != 2 or gt_indices.shape[1] != 2:
        raise RuntimeError(f'superpoint_targets_batched: gt_indices must be (R, 2), got {tuple(gt_indices.shape)}')
    if gt_count.numel() < B:
        raise RuntimeError(f'superpoint_targets_batched: gt_count must hold {B} counts')
    nn = sum(int(cloud_nodes[p]) * int(cloud_nodes[B + p]) for p in range(B))
    _min_rows(gt_indices, nn, 'gt_indices')
    _min_rows(gt_overlaps, nn, 'gt_overlaps')
    seed, iteration = int(seed), int(iteration)
    if not (0 <= seed < 1 << 64 and 0 <= iteration < 1 << 64):
        raise ValueError('superpoint_targets_batched: seed and iteration must be 64-bit unsigned integers')
    k = int(num_targets)
    dev = gt_indices.device
    lib = L.lib()
    ws = L.workspace(lib.geob200_superpoint_targets_batched_workspace_bytes(nn), dev, tag='superpoint_targets')
    corr = torch.empty((2 * B, k), dtype=_i64, device=dev)
    sc = torch.empty((B, k), dtype=_f32, device=dev)
    cnt = torch.empty((B,), dtype=_i32, device=dev)
    L.check(lib.geob200_superpoint_targets_batched(gt_indices.data_ptr(), gt_overlaps.data_ptr(), gt_count.data_ptr(), B,
                                                   _host_i64(cloud_nodes), float(overlap_threshold), k, seed, iteration, int(pair_base),
                                                   corr.data_ptr(), sc.data_ptr(), cnt.data_ptr(), ws.data_ptr(), ws.numel(),
                                                   L.stream_ptr()), 'superpoint_targets_batched')
    return corr, sc, cnt


_NF_TABLES = {}


def nonfinite_check(tensors, found_inf=None):
    """0-dim (or 1-element) fp32 device tensor ``found_inf`` = 1.0 when any element of the fp32 CUDA ``tensors`` is NaN or +-Inf, else 0.0; one
    launch.  The device table of (pointer, numel) is cached per set of tensors and refreshed by a non-blocking copy when their
    storage moves, so the call never waits for the device."""
    tensors = list(tensors)
    if not tensors:
        raise ValueError('nonfinite_check: no tensors')
    for i, t in enumerate(tensors):
        _f(t, f'tensors[{i}]')
    dev = tensors[0].device
    if any(t.device != dev for t in tensors):
        raise RuntimeError('nonfinite_check: all tensors must be on one device')
    if found_inf is None:
        found_inf = torch.empty((), dtype=_f32, device=dev)        # 0-dim: the form torch's fused Adam takes as ``found_inf``
    _f(found_inf, 'found_inf')
    if found_inf.numel() != 1 or found_inf.device != dev:
        raise RuntimeError('nonfinite_check: found_inf must be a 1-element float32 tensor on the tensors\' device')
    key = (dev, tuple((t.data_ptr(), t.numel()) for t in tensors))
    table = _NF_TABLES.get(key)
    if table is None:
        host = torch.tensor([p for p, _ in key[1]] + [n for _, n in key[1]], dtype=_i64).pin_memory()
        table = host.to(dev, non_blocking=True)          # the pinned block is held by the host allocator until the copy is done
        if len(_NF_TABLES) > 64:
            _NF_TABLES.clear()
        _NF_TABLES[key] = table
    n = len(tensors)
    L.check(L.lib().geob200_nonfinite_check(table.data_ptr(), table[n:].data_ptr(), n, max(t.numel() for t in tensors),
                                            found_inf.data_ptr(), L.stream_ptr()), 'nonfinite_check')
    return found_inf


def batch_loss_weights(loss_rows, mean_row=None, n_valid=None, found_inf=None):
    """Loss weights of a batched training step (``geob200_batch_loss_weights``, one launch): pair p of the (B, >= 3) [loss, c_loss,
    f_loss] rows is valid when its row is finite.  Returns (w (B,) = valid_p / n_valid, mean_row (3,) = the fixed-order sum over
    the valid pairs of w_p * row p, NaN without one).  ``n_valid`` (1-element fp32) receives the count; ``found_inf`` (1-element fp32)
    is set to 1 when no pair is valid and left alone otherwise.  No host synchronisation."""
    loss_rows = _detach(loss_rows)
    _f(loss_rows, 'loss_rows')
    if loss_rows.dim() != 2 or loss_rows.shape[1] < 3 or loss_rows.stride(1) != 1:
        raise RuntimeError('batch_loss_weights: loss_rows must be (B, >= 3) with unit inner stride')
    B, dev = loss_rows.shape[0], loss_rows.device
    w = torch.empty((B,), dtype=_f32, device=dev)
    if mean_row is None:
        mean_row = torch.empty((3,), dtype=_f32, device=dev)
    if found_inf is None:
        found_inf = torch.zeros((), dtype=_f32, device=dev)
    for t, name, n in ((mean_row, 'mean_row', 3), (n_valid, 'n_valid', 1), (found_inf, 'found_inf', 1)):
        if t is not None and (_f(t, name).numel() != n or not t.is_contiguous() or t.device != dev):
            raise RuntimeError(f'batch_loss_weights: {name} must be a contiguous float32 tensor of {n} values on {dev}')
    L.check(L.lib().geob200_batch_loss_weights(loss_rows.data_ptr(), loss_rows.stride(0), B, w.data_ptr(), mean_row.data_ptr(), L.ptr(n_valid),
                                               found_inf.data_ptr(), L.stream_ptr()), 'batch_loss_weights')
    return w, mean_row


AUGMENT_3DMATCH, AUGMENT_KITTI = 0, 1
AUGMENT_RECORD = 20


def _seed_iteration(seed, iteration, what):
    seed, iteration = int(seed), int(iteration)
    if not (0 <= seed < 1 << 64 and 0 <= iteration < 1 << 64):
        raise ValueError(f'{what}: seed and iteration must be 64-bit unsigned integers')
    return seed, iteration


def augment_pairs_batched(points, lengths, transforms, mode, point_limit, noise, rotation_factor=1.0, min_scale=1.0, max_scale=1.0,
                          shift=0.0, seed=0, iteration=0, pair_base=0):
    """3DMatch (``mode`` AUGMENT_3DMATCH) / KITTI (AUGMENT_KITTI) training-pair augmentation of B pairs (``geob200_augment_pairs_batched``,
    two launches).  ``points``: raw clouds stacked [ref_0..ref_{B-1}, src_0..src_{B-1}] with ``lengths`` (2B host ints);
    ``transforms`` (B, 4, 4) fp32 ground truth.  Pair p draws from the streams (seed, iteration, pair_base + p).  Returns (points,
    lengths_host (list of min(n, point_limit)), transforms (B, 4, 4) fp32, origin (rows,) int32 = each row's row in its input cloud,
    record (B, 20) fp64 = [u0..u10 | R]).  No host synchronisation."""
    _f(points, 'points'); _f(transforms, 'transforms')
    lengths = [int(v) for v in lengths]
    B = len(lengths) // 2
    if B < 1 or len(lengths) != 2 * B:
        raise RuntimeError('augment_pairs_batched: lengths must hold 2B counts')
    if points.dim() != 2 or points.shape[1] != 3 or points.shape[0] != sum(lengths):
        raise RuntimeError(f'augment_pairs_batched: points must be (sum(lengths), 3), got {tuple(points.shape)}')
    if transforms.numel() != 16 * B:
        raise RuntimeError(f'augment_pairs_batched: transforms must be ({B}, 4, 4)')
    seed, iteration = _seed_iteration(seed, iteration, 'augment_pairs_batched')
    limit = int(point_limit)
    out_len = [min(n, limit) for n in lengths]
    dev = points.device
    lib = L.lib()
    ws = L.workspace(lib.geob200_augment_pairs_batched_workspace_bytes(sum(lengths)), dev, tag='augment')
    out = torch.empty((sum(out_len), 3), dtype=_f32, device=dev)
    origin = torch.empty((sum(out_len),), dtype=_i32, device=dev)
    T = torch.empty((B, 4, 4), dtype=_f32, device=dev)
    record = torch.empty((B, AUGMENT_RECORD), dtype=torch.float64, device=dev)
    L.check(lib.geob200_augment_pairs_batched(points.data_ptr(), _host_i64(lengths), B, transforms.data_ptr(), int(mode), limit, float(noise),
                                              float(rotation_factor), float(min_scale), float(max_scale), float(shift), seed, iteration,
                                              int(pair_base), out.data_ptr(), origin.data_ptr(), T.data_ptr(), record.data_ptr(),
                                              ws.data_ptr(), ws.numel(), L.stream_ptr()), 'augment_pairs_batched')
    return out, out_len, T, origin, record


def modelnet_pairs_batched(shapes, lengths, num_points, keep_ratio, rotation_magnitude, translation_magnitude, noise_magnitude, seed=0,
                           iteration=0, pair_base=0):
    """ModelNet training pairs from B raw shapes (``geob200_modelnet_pairs_batched``, one launch): ``shapes`` stacked with ``lengths``
    (B host ints, each <= 8192 with round(keep_ratio N) >= num_points).  Returns (points (2B num_points, 3) stacked [ref..., src...],
    lengths_host, transforms (B, 4, 4) fp32, origin (int32, the raw shape row of every output row), record (B, 20) fp64).  No host
    synchronisation."""
    _f(shapes, 'shapes')
    lengths = [int(v) for v in lengths]
    B = len(lengths)
    if B < 1:
        raise RuntimeError('modelnet_pairs_batched: no shapes')
    if shapes.dim() != 2 or shapes.shape[1] != 3 or shapes.shape[0] != sum(lengths):
        raise RuntimeError(f'modelnet_pairs_batched: shapes must be (sum(lengths), 3), got {tuple(shapes.shape)}')
    seed, iteration = _seed_iteration(seed, iteration, 'modelnet_pairs_batched')
    m = int(num_points)
    dev = shapes.device
    lib = L.lib()
    ws = L.workspace(lib.geob200_modelnet_pairs_batched_workspace_bytes(sum(lengths)), dev, tag='augment')
    out = torch.empty((2 * B * max(m, 0), 3), dtype=_f32, device=dev)
    origin = torch.empty((2 * B * max(m, 0),), dtype=_i32, device=dev)
    T = torch.empty((B, 4, 4), dtype=_f32, device=dev)
    record = torch.empty((B, AUGMENT_RECORD), dtype=torch.float64, device=dev)
    L.check(lib.geob200_modelnet_pairs_batched(shapes.data_ptr(), _host_i64(lengths), B, m, float(keep_ratio), float(rotation_magnitude),
                                               float(translation_magnitude), float(noise_magnitude), seed, iteration, int(pair_base),
                                               out.data_ptr(), origin.data_ptr(), T.data_ptr(), record.data_ptr(), ws.data_ptr(),
                                               ws.numel(), L.stream_ptr()), 'modelnet_pairs_batched')
    return out, [m] * (2 * B), T, origin, record


def modelnet_benchmark_pairs_batched(shapes, lengths, indices, num_points, keep_ratio, rotation_magnitude, translation_magnitude,
                                     noise_magnitude):
    """ModelNet validation / test pairs (``geob200_modelnet_benchmark_pairs_batched``): pair p is the reference's
    ``ModelNetPairDataset(deterministic=True)`` item of dataset index ``indices[p]`` (0 .. 2^32-1), built from raw shape p of
    ``shapes`` (stacked fp32, ``lengths`` host ints of 1 .. 8192) with numpy's legacy stream seeded by that index.  Returns (points
    (2B num_points, 3) fp32 stacked [ref..., src...], lengths_host, transforms (B, 4, 4) fp32, origin (int32, the raw shape row of
    every output row)).  No host synchronisation."""
    _f(shapes, 'shapes')
    lengths = [int(v) for v in lengths]
    indices = [int(v) for v in indices]
    B = len(lengths)
    if B < 1 or len(indices) != B:
        raise RuntimeError('modelnet_benchmark_pairs_batched: lengths and indices must hold one value per pair')
    if shapes.dim() != 2 or shapes.shape[1] != 3 or shapes.shape[0] != sum(lengths) or not shapes.is_contiguous():
        raise RuntimeError(f'modelnet_benchmark_pairs_batched: shapes must be contiguous (sum(lengths), 3), got {tuple(shapes.shape)}')
    if any(not 0 <= i < 1 << 32 for i in indices):
        raise RuntimeError('modelnet_benchmark_pairs_batched: indices must be in 0..2^32-1')
    m = int(num_points)
    dev = shapes.device
    lib = L.lib()
    ws = L.workspace(lib.geob200_modelnet_benchmark_pairs_batched_workspace_bytes(B, m), dev, tag='augment')
    out = torch.empty((2 * B * max(m, 0), 3), dtype=_f32, device=dev)
    origin = torch.empty((2 * B * max(m, 0),), dtype=_i32, device=dev)
    T = torch.empty((B, 4, 4), dtype=_f32, device=dev)
    L.check(lib.geob200_modelnet_benchmark_pairs_batched(shapes.data_ptr(), _host_i64(lengths), _host_i64(indices), B, m, float(keep_ratio),
                                                         float(rotation_magnitude), float(translation_magnitude), float(noise_magnitude),
                                                         out.data_ptr(), origin.data_ptr(), T.data_ptr(), ws.data_ptr(), ws.numel(),
                                                         L.stream_ptr()), 'modelnet_benchmark_pairs_batched')
    return out, [m] * (2 * B), T, origin


def rotated_pairs_batched(points, lengths, indices, transforms):
    """Rotated 3DMatch / 3DLoMatch test pairs (``geob200_rotated_pairs_batched``): pair p is the reference's
    ``ThreeDMatchPairDataset(rotated=True)`` item of dataset index ``indices[p]`` (0 .. 2^32-1) with numpy's legacy stream seeded by
    that index.  ``points``: CUDA (sum(lengths), 3) float32 or float64 (the clouds' file type: numpy rotates either in fp64), stacked [ref_0..ref_{B-1}, src_0..src_{B-1}]; ``lengths``: 2B host ints
    (each >= 1); ``transforms``: (B, 4, 4) float64 [R | t] from the metadata (ref = T src).  Returns (points (sum(lengths), 3) fp32
    in the input's layout, transforms (B, 4, 4) fp32, rotations (B, 2, 3, 3) float64: R_ref, R_src).  The half-angles' sin and cos are
    correctly rounded, which the host libm that the reference calls is except in rare near-tie cases (DESIGN.md section 8a).  No
    host synchronisation."""
    if not isinstance(points, torch.Tensor) or not points.is_cuda or points.dtype not in (torch.float32, torch.float64):
        raise RuntimeError('rotated_pairs_batched: points must be a CUDA float32 or float64 tensor (geotransformer_b200 has no CPU path)')
    lengths = [int(v) for v in lengths]
    indices = [int(v) for v in indices]
    B = len(indices)
    if B < 1 or len(lengths) != 2 * B:
        raise RuntimeError('rotated_pairs_batched: indices must hold one value per pair and lengths two')
    if points.dim() != 2 or points.shape[1] != 3 or points.shape[0] != sum(lengths) or not points.is_contiguous():
        raise RuntimeError(f'rotated_pairs_batched: points must be contiguous (sum(lengths), 3), got {tuple(points.shape)}')
    if any(not 0 <= i < 1 << 32 for i in indices):
        raise RuntimeError('rotated_pairs_batched: indices must be in 0..2^32-1')
    dev = points.device
    T_in = torch.as_tensor(transforms, dtype=torch.float64).to(dev, non_blocking=True).contiguous()
    if tuple(T_in.shape) != (B, 4, 4):
        raise RuntimeError(f'rotated_pairs_batched: transforms must be ({B}, 4, 4), got {tuple(T_in.shape)}')
    out = torch.empty(points.shape, dtype=_f32, device=dev)
    T = torch.empty((B, 4, 4), dtype=_f32, device=dev)
    rot = torch.empty((B, 2, 3, 3), dtype=torch.float64, device=dev)
    L.check(L.lib().geob200_rotated_pairs_batched(points.data_ptr(), int(points.dtype == torch.float64), _host_i64(lengths), _host_i64(indices), B, T_in.data_ptr(),
                                                  out.data_ptr(), T.data_ptr(), rot.data_ptr(), L.stream_ptr()), 'rotated_pairs_batched')
    return out, T, rot


VOXEL_MAX_CLOUDS = 64
_VOXEL_ERRORS = {1: 'a coordinate is NaN or infinite',
                 2: 'voxel_size is too small (voxel_size * INT_MAX < the extent of the bounding box, as Open3D checks)',
                 3: 'an axis spans 2^21 voxels or more (the limit of the packed voxel key): use a larger voxel_size'}


def voxel_down_sample_batched(points, lengths, voxel_size, normals=None):
    """Open3D's ``PointCloud::VoxelDownSample`` of up to 64 stacked clouds in one call (``geob200_voxel_down_sample``), in double.
    ``points``: CUDA (sum(lengths), 3) float64, or float32 (widened exactly, as Open3D's ``Vector3dVector`` does); ``lengths``: B
    host ints (empty clouds allowed); ``normals``: optional, like ``points``.  Each voxel's value is the input-order double sum of
    its points divided by their count (normals likewise, not renormalised), in the iteration order of Open3D's voxel map (DESIGN.md
    section 8a).  Returns (points (M, 3) float64, lengths (B,) int64[, normals (M, 3) float64]) on the device; M and the error
    status are read back in one 8 (B + 1) byte copy.  Raises RuntimeError on a non-finite coordinate, a voxel size Open3D calls too
    small, or an axis of 2^21 voxels or more."""
    lengths = [int(v) for v in lengths]
    B = len(lengths)
    if not 1 <= B <= VOXEL_MAX_CLOUDS:
        raise RuntimeError(f'voxel_down_sample_batched: 1..{VOXEL_MAX_CLOUDS} clouds per call, got {B}')
    voxel_size = float(voxel_size)
    if not (voxel_size > 0 and math.isfinite(voxel_size)):
        raise RuntimeError(f'voxel_down_sample_batched: voxel_size must be positive and finite, got {voxel_size}')

    def _as_f64(t, name):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise RuntimeError(f'{name} must be a CUDA tensor (geotransformer_b200 has no CPU path)')
        if t.dtype not in (torch.float32, torch.float64):
            raise RuntimeError(f'{name} must be float32 or float64, got {t.dtype}')
        t = t.to(torch.float64).contiguous()
        if t.dim() != 2 or t.shape[1] != 3 or t.shape[0] != sum(lengths):
            raise RuntimeError(f'voxel_down_sample_batched: {name} must be (sum(lengths), 3), got {tuple(t.shape)}')
        return t

    pts = _as_f64(points, 'points')
    nrm = None if normals is None else _as_f64(normals, 'normals')
    if nrm is not None and nrm.device != pts.device:
        raise RuntimeError('voxel_down_sample_batched: points and normals must be on one device')
    n, dev = pts.shape[0], pts.device
    lib = L.lib()
    ws = L.workspace(lib.geob200_voxel_down_sample_workspace_bytes(n, B), dev, tag='voxel')
    out = torch.empty((n, 3), dtype=torch.float64, device=dev)
    out_n = torch.empty((n, 3), dtype=torch.float64, device=dev) if nrm is not None else None
    out_len = torch.empty((B + 1,), dtype=_i64, device=dev)
    L.check(lib.geob200_voxel_down_sample(pts.data_ptr(), L.ptr(nrm), n, _host_i64(lengths), B, voxel_size, out.data_ptr(),
                                          L.ptr(out_n), out_len.data_ptr(), ws.data_ptr(), ws.numel(), L.stream_ptr()),
            'voxel_down_sample_batched')
    host = out_len.cpu().tolist()
    if host[B] != 0:
        raise RuntimeError(f'voxel_down_sample_batched: {_VOXEL_ERRORS.get(host[B], f"error {host[B]}")}')
    m = sum(host[:B])
    res = (out[:m].clone(), out_len[:B])
    if nrm is not None:
        res = res + (out_n[:m].clone(),)
    return res
