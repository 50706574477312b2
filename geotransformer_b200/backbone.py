"""KPConv-FPN backbones of the three shipped experiments as one class (same child-module names, so reference
checkpoints load strict): reference ``experiments/*/backbone.py`` (3DMatch :8-87, KITTI :7-124, ModelNet :8-73)."""
import torch.nn as nn

from . import functional as GF
from .modules.kpconv import ConvBlock, ResidualBlock, UnaryBlock, LastUnaryBlock


class KPConvFPN(nn.Module):
    """``num_stages`` encoder levels; decoders from level ``num_stages-1`` down to ``finest_decoder`` (2 for
    3DMatch/KITTI, 1 for ModelNet); the last decoder is a LastUnaryBlock (no norm/activation)."""

    def __init__(self, input_dim, output_dim, init_dim, kernel_size, init_radius, init_sigma, group_norm, num_stages=4,
                 finest_decoder=2):
        super().__init__()
        self.num_stages, self.finest_decoder = num_stages, finest_decoder
        r, s, d = init_radius, init_sigma, init_dim
        self.encoder1_1 = ConvBlock(input_dim, d, kernel_size, r, s, group_norm)
        self.encoder1_2 = ResidualBlock(d, d * 2, kernel_size, r, s, group_norm)
        for lvl in range(2, num_stages + 1):
            cin = d * 2 ** (lvl - 1)
            setattr(self, f'encoder{lvl}_1', ResidualBlock(cin, cin, kernel_size, r, s, group_norm, strided=True))
            r, s = r * 2, s * 2
            setattr(self, f'encoder{lvl}_2', ResidualBlock(cin, cin * 2, kernel_size, r, s, group_norm))
            setattr(self, f'encoder{lvl}_3', ResidualBlock(cin * 2, cin * 2, kernel_size, r, s, group_norm))
        for lvl in range(num_stages - 1, finest_decoder - 1, -1):
            cin = d * 2 ** (lvl + 1) + d * 2 ** lvl          # upsampled latent (level lvl+1 width) + skip (level lvl width)
            if lvl == finest_decoder:
                setattr(self, f'decoder{lvl}', LastUnaryBlock(cin, output_dim))
            else:
                setattr(self, f'decoder{lvl}', UnaryBlock(cin, d * 2 ** lvl, group_norm))

    def forward(self, feats, data_dict):
        """A batch of several pairs (``data_dict['batch_size']`` > 1, stack order [ref_1..ref_B, src_1..src_B]) normalises per pair
        and max-pools each pair over its own subsampling width, as the batched native backbone does: the per-level cloud rows come
        from ``lengths_host``, the widths from ``GF.cloud_max_count``."""
        pts, nb = data_dict['points'], data_dict['neighbors']
        sub, up = data_dict['subsampling'], data_dict['upsampling']
        S = self.num_stages
        # per level: the rows of every cloud and (strided blocks) the per-cloud table widths; None for one pair.  They go to the blocks
        # as keyword arguments, so a block's positional arguments are the same for one pair and for a batch.
        rows, cmax = [None] * S, [None] * (S - 1)
        if int(data_dict.get('batch_size', 1)) > 1:
            rows = [[int(v) for v in lv] for lv in data_dict['lengths_host']]
            cmax = [GF.cloud_max_count(sub[lv], pts[lv].shape[0], rows[lv + 1]) for lv in range(S - 1)]
        x = self.encoder1_1(feats, pts[0], pts[0], nb[0], cloud_rows=rows[0])
        x = self.encoder1_2(x, pts[0], pts[0], nb[0], s_rows=rows[0], q_rows=rows[0])
        enc = [x]
        for lvl in range(2, S + 1):
            r, rq = rows[lvl - 2], rows[lvl - 1]
            x = getattr(self, f'encoder{lvl}_1')(x, pts[lvl - 1], pts[lvl - 2], sub[lvl - 2], s_rows=r, q_rows=rq, cloud_max=cmax[lvl - 2])
            x = getattr(self, f'encoder{lvl}_2')(x, pts[lvl - 1], pts[lvl - 1], nb[lvl - 1], s_rows=rq, q_rows=rq)
            x = getattr(self, f'encoder{lvl}_3')(x, pts[lvl - 1], pts[lvl - 1], nb[lvl - 1], s_rows=rq, q_rows=rq)
            enc.append(x)
        feats_list = [enc[-1]]
        latent = enc[-1]
        for lvl in range(S - 1, self.finest_decoder - 1, -1):
            latent = GF.upsample_concat(latent, up[lvl - 1], enc[lvl - 1])
            dec = getattr(self, f'decoder{lvl}')
            latent = dec(latent) if lvl == self.finest_decoder else dec(latent, cloud_rows=rows[lvl - 1])
            feats_list.append(latent)
        feats_list.reverse()
        return feats_list
