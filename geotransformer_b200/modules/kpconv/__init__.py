from .modules import (KPConv, GroupNorm, UnaryBlock, LastUnaryBlock, ConvBlock, ResidualBlock, maxpool,
                      nearest_upsample, default_kernel_points)
from .kernel_points import initialize_kernel_points
