"""KPConv building blocks with the reference's class names, constructor signatures and ``state_dict`` keys
(reference ``geotransformer/modules/kpconv/kpconv.py:10-122`` and ``modules.py:33-225``); every forward
runs hand-written sm_90a kernels through the C ABI (``geotransformer_b200.functional``)."""
import math

import torch
import torch.nn as nn

from ... import functional as GF


class KPConv(nn.Module):
    """reference ``kpconv.py:10-122``.  ``kernel_points`` is a buffer: real values come from a checkpoint
    (the reference draws a randomly rotated, noised disposition per instance, ``kernel_points.py:423-455``)."""

    def __init__(self, in_channels, out_channels, kernel_size, radius, sigma, bias=False, dimension=3, inf=1e6,
                 eps=1e-9):
        super().__init__()
        self.kernel_size, self.in_channels, self.out_channels = kernel_size, in_channels, out_channels
        self.radius, self.sigma, self.dimension, self.inf, self.eps = radius, sigma, dimension, inf, eps
        self.weights = nn.Parameter(torch.zeros(kernel_size, in_channels, out_channels))
        if bias:
            self.bias = nn.Parameter(torch.zeros(out_channels))
        else:
            self.register_parameter('bias', None)
        nn.init.kaiming_uniform_(self.weights, a=math.sqrt(5))
        if self.bias is not None:
            nn.init.uniform_(self.bias, -1 / math.sqrt(in_channels * out_channels), 1 / math.sqrt(in_channels * out_channels))
        self.register_buffer('kernel_points', default_kernel_points(kernel_size, radius))

    def _weights_t(self):
        w = self.weights
        key = (w.data_ptr(), w._version)
        if getattr(self, '_wt_key', None) != key:     # (c_out, 15*c_in) copy for the tensor-core GEMM, rebuilt if weights change
            self._wt = w.detach().reshape(-1, w.shape[2]).t().contiguous()
            self._wt_key = key
        return self._wt

    def forward(self, s_feats, q_points, s_points, neighbor_indices):
        return GF.kpconv(s_feats, q_points, s_points, neighbor_indices, self.kernel_points, self.weights, self.bias,
                         self.sigma, weights_t=self._weights_t())

    def forward_norm(self, s_feats, q_points, s_points, neighbor_indices, norm, negative_slope, cloud_rows=None):
        """KPConv -> GroupNorm -> LeakyReLU as one fused op (GroupNorm statistics from the GEMM epilogue; per pair with
        ``cloud_rows``, the query rows per cloud of a batch)"""
        return GF.kpconv_group_norm(s_feats, q_points, s_points, neighbor_indices, self.kernel_points, self.weights, self.bias,
                                    self.sigma, norm.norm.weight, norm.norm.bias, norm.num_groups, norm.norm.eps,
                                    negative_slope=negative_slope, weights_t=self._weights_t(), cloud_rows=cloud_rows)

    def __repr__(self):
        return (f'KPConv(kernel_size: {self.kernel_size}, in_channels: {self.in_channels}, out_channels: '
                f'{self.out_channels}, radius: {self.radius:g}, sigma: {self.sigma:g}, bias: {self.bias is not None})')


def default_kernel_points(k, radius, seed=None):
    """Centre + (k-1) quasi-uniform points on a sphere of 0.66*radius (Fibonacci lattice).  Stand-in used only
    when no checkpoint provides the buffer; optionally rotated by a seeded random rotation."""
    pts = torch.zeros(k, 3, dtype=torch.float64)
    m = k - 1
    for i in range(m):
        z = 1 - 2 * (i + 0.5) / m
        r = math.sqrt(max(0.0, 1 - z * z))
        phi = math.pi * (1 + 5 ** 0.5) * i
        pts[i + 1] = torch.tensor([r * math.cos(phi), r * math.sin(phi), z], dtype=torch.float64) * 0.66
    if seed is not None:
        g = torch.Generator().manual_seed(seed)
        q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
        pts = pts @ q + 0.01 * torch.randn(k, 3, generator=g, dtype=torch.float64)
        pts[0] = 0.01 * torch.randn(3, generator=g, dtype=torch.float64)
    return (pts * radius).float()


class GroupNorm(nn.Module):
    """reference ``modules.py:33-50``: statistics span ALL stacked points of the pair."""

    def __init__(self, num_groups, num_channels):
        super().__init__()
        self.num_groups, self.num_channels = num_groups, num_channels
        self.norm = nn.GroupNorm(num_groups, num_channels)

    def forward(self, x, negative_slope=None, residual=None):
        return GF.group_norm(x, self.norm.weight, self.norm.bias, self.num_groups, self.norm.eps,
                             negative_slope=negative_slope, residual=residual)


class UnaryBlock(nn.Module):
    """reference ``modules.py:53-86``: Linear -> GroupNorm -> LeakyReLU(0.1)."""

    def __init__(self, in_channels, out_channels, group_norm, has_relu=True, bias=True, layer_norm=False):
        super().__init__()
        if layer_norm:
            raise NotImplementedError('layer_norm=True is not used by any shipped model')
        self.in_channels, self.out_channels, self.group_norm = in_channels, out_channels, group_norm
        self.mlp = nn.Linear(in_channels, out_channels, bias=bias)
        self.norm = GroupNorm(group_norm, out_channels)
        self.leaky_relu = nn.LeakyReLU(0.1) if has_relu else None

    def forward(self, x, residual=None, residual_slope=None, cloud_rows=None):
        """``cloud_rows``: rows per cloud of a batch of pairs (per-pair GroupNorm statistics), None for one pair"""
        slope = self.leaky_relu.negative_slope if self.leaky_relu is not None else None
        if residual is not None:      # fused tail of ResidualBlock: leaky(norm(x) + shortcut)
            slope = residual_slope
        n = self.norm
        return GF.linear_group_norm(x, self.mlp.weight, self.mlp.bias, n.norm.weight, n.norm.bias, n.num_groups, n.norm.eps,
                                    negative_slope=slope, residual=residual, cloud_rows=cloud_rows)


class LastUnaryBlock(nn.Module):
    """reference ``modules.py:89-104``."""

    def __init__(self, in_channels, out_channels, bias=True):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.mlp = nn.Linear(in_channels, out_channels, bias=bias)

    def forward(self, x):
        return GF.linear(x, self.mlp.weight, self.mlp.bias)


class ConvBlock(nn.Module):
    """reference ``modules.py:107-148``."""

    def __init__(self, in_channels, out_channels, kernel_size, radius, sigma, group_norm, negative_slope=0.1,
                 bias=True, layer_norm=False):
        super().__init__()
        if layer_norm:
            raise NotImplementedError('layer_norm=True is not used by any shipped model')
        self.in_channels, self.out_channels = in_channels, out_channels
        self.KPConv = KPConv(in_channels, out_channels, kernel_size, radius, sigma, bias=bias)
        self.norm = GroupNorm(group_norm, out_channels)
        self.leaky_relu = nn.LeakyReLU(negative_slope=negative_slope)

    def forward(self, s_feats, q_points, s_points, neighbor_indices, cloud_rows=None):
        return self.KPConv.forward_norm(s_feats, q_points, s_points, neighbor_indices, self.norm, self.leaky_relu.negative_slope,
                                        cloud_rows=cloud_rows)


class ResidualBlock(nn.Module):
    """reference ``modules.py:151-225`` (bottleneck)."""

    def __init__(self, in_channels, out_channels, kernel_size, radius, sigma, group_norm, strided=False, bias=True,
                 layer_norm=False):
        super().__init__()
        if layer_norm:
            raise NotImplementedError('layer_norm=True is not used by any shipped model')
        self.in_channels, self.out_channels, self.strided = in_channels, out_channels, strided
        mid = out_channels // 4
        self.unary1 = UnaryBlock(in_channels, mid, group_norm, bias=bias) if in_channels != mid else nn.Identity()
        self.KPConv = KPConv(mid, mid, kernel_size, radius, sigma, bias=bias)
        self.norm_conv = GroupNorm(group_norm, mid)
        self.unary2 = UnaryBlock(mid, out_channels, group_norm, has_relu=False, bias=bias)
        if in_channels != out_channels:
            self.unary_shortcut = UnaryBlock(in_channels, out_channels, group_norm, has_relu=False, bias=bias)
        else:
            self.unary_shortcut = nn.Identity()
        self.leaky_relu = nn.LeakyReLU(0.1)

    def forward(self, s_feats, q_points, s_points, neighbor_indices, s_rows=None, q_rows=None, cloud_max=None):
        """``s_rows`` / ``q_rows``: support / query rows per cloud of a batch of pairs (per-pair GroupNorm statistics), and for a
        strided block ``cloud_max`` (``GF.cloud_max_count`` of its table): the max-pool's per-pair widths.  None for one pair."""
        x = s_feats if isinstance(self.unary1, nn.Identity) else self.unary1(s_feats, cloud_rows=s_rows)
        x = self.KPConv.forward_norm(x, q_points, s_points, neighbor_indices, self.norm_conv, self.leaky_relu.negative_slope,
                                     cloud_rows=q_rows)
        if self.strided:
            shortcut = GF.maxpool(s_feats, neighbor_indices, q_rows, cloud_max) if q_rows is not None else GF.maxpool(s_feats, neighbor_indices)
        else:
            shortcut = s_feats
        if not isinstance(self.unary_shortcut, nn.Identity):
            shortcut = self.unary_shortcut(shortcut, cloud_rows=q_rows)
        # unary2 (Linear+GroupNorm) + shortcut add + LeakyReLU in one normalisation pass
        return self.unary2(x, residual=shortcut, residual_slope=self.leaky_relu.negative_slope, cloud_rows=q_rows)


def maxpool(x, neighbor_indices):
    """reference ``functional.py:54-67``."""
    return GF.maxpool(x, neighbor_indices)


def nearest_upsample(x, upsample_indices):
    """reference ``functional.py:6-22``."""
    return GF.nearest_upsample(x, upsample_indices)
