"""TEST INFRASTRUCTURE ONLY (and only usable where the reference checkout exists).

Imports the UNMODIFIED reference Python package from ``/root/reference`` so that
``oracle/make_golden.py`` can run the real reference forward on CPU and dump golden vectors into
``tests/golden/``.  No test imports this module.

What has to be faked for the import to succeed (SURVEY.md section 8c):
  * debug-only third-party imports that are not installed: IPython, ipdb, matplotlib.pyplot,
    coloredlogs, easydict, open3d (only ``io.read_point_cloud`` of the 15-vertex kernel PLY is real);
  * ``geotransformer.ext``: served by ``oracle/ref_ext.py`` = the reference C++ cores behind a C shim;
  * hard-coded ``.cuda()`` calls: ``Tensor.cuda`` is replaced by a clone on CPU (clone, not identity, so
    that ``to_cuda`` keeps its densifying effect on the sliced neighbour tables);
  * ``config.py`` creates output dirs on import: ``os.makedirs`` is made a no-op for the read-only tree.
"""
import importlib
import os
import struct
import sys
import types

import numpy as np
import torch

REF_ROOT = '/root/reference'
EXP = {
    '3dmatch': 'geotransformer.3dmatch.stage4.gse.k3.max.oacl.stage2.sinkhorn',
    'kitti': 'geotransformer.kitti.stage5.gse.k3.max.oacl.stage2.sinkhorn',
    'modelnet': 'geotransformer.modelnet.rpmnet.stage4.gse.k3.max.oacl.stage2.sinkhorn',
}


def available():
    return os.path.isdir(os.path.join(REF_ROOT, 'geotransformer'))


def _read_ply_points(path):
    with open(path, 'rb') as f:
        data = f.read()
    header_end = data.index(b'end_header\n') + len(b'end_header\n')
    header = data[:header_end].decode()
    n = int([ln for ln in header.split('\n') if ln.startswith('element vertex')][0].split()[-1])
    vals = struct.unpack('<' + 'd' * (3 * n), data[header_end:header_end + 24 * n])
    return np.asarray(vals, dtype=np.float64).reshape(n, 3)


class _AttrDict(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v


_installed = False


def install():
    """Make ``import geotransformer`` resolve to the real reference, CPU-runnable."""
    global _installed
    if _installed:
        return
    assert available(), 'reference tree not present'

    def stub(name, **attrs):
        m = types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
        return m

    stub('IPython', embed=lambda *a, **k: None)
    stub('ipdb', set_trace=lambda *a, **k: None)
    mpl = stub('matplotlib')
    mpl.pyplot = stub('matplotlib.pyplot')
    stub('coloredlogs', install=lambda *a, **k: None)
    stub('easydict', EasyDict=_AttrDict)

    class _PCD:
        def __init__(self, pts):
            self.points = pts

    o3d = stub('open3d')
    o3d.io = stub('open3d.io', read_point_cloud=lambda p: _PCD(_read_ply_points(p)))
    o3d.geometry = stub('open3d.geometry')
    o3d.utility = stub('open3d.utility')

    from oracle import ref_ext
    sys.path.insert(0, REF_ROOT)
    pkg = importlib.import_module('geotransformer')
    ext = types.ModuleType('geotransformer.ext')
    ext.grid_subsampling = ref_ext.grid_subsampling
    ext.radius_neighbors = ref_ext.radius_neighbors
    sys.modules['geotransformer.ext'] = ext
    pkg.ext = ext

    torch.Tensor.cuda = lambda self, *a, **k: self.clone(memory_format=torch.preserve_format)
    _installed = True


def load_experiment(which):
    """Returns (cfg, create_model) of one of the reference experiments."""
    install()
    exp_dir = os.path.join(REF_ROOT, 'experiments', EXP[which])
    for name in ('config', 'model', 'backbone'):
        sys.modules.pop(name, None)
    sys.path.insert(0, exp_dir)
    real_makedirs = os.makedirs
    os.makedirs = lambda *a, **k: None
    try:
        config = importlib.import_module('config')
        model = importlib.import_module('model')
    finally:
        os.makedirs = real_makedirs
        sys.path.remove(exp_dir)
    return config.make_cfg(), model.create_model


def load_evaluator(which, cfg):
    """The reference Evaluator (experiments/<exp>/loss.py) of the experiment; call after load_experiment(which).
    Its .cuda() allocations resolve to CPU clones through install()."""
    exp_dir = os.path.join(REF_ROOT, 'experiments', EXP[which])
    sys.modules.pop('loss', None)
    sys.path.insert(0, exp_dir)
    try:
        loss = importlib.import_module('loss')
    finally:
        sys.path.remove(exp_dir)
    return loss.Evaluator(cfg)


def kernel_disposition():
    """The 15x3 float64 kernel-point disposition shipped with the reference (a data fixture)."""
    return _read_ply_points(os.path.join(REF_ROOT, 'geotransformer/modules/kpconv/dispositions/k_015_center_3D.ply'))
