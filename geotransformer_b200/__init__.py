"""geotransformer_b200 -- H100-native (sm_90a) implementation of GeoTransformer's per-pair registration
hot path behind the reference's own op/module surface.  See DESIGN.md for the scope and INTEGRATION.md for
the drop-in boundary."""
__version__ = '0.1.0'
