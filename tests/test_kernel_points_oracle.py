"""Kernel-point dispositions without a GPU: the numpy restatement (tests/kernel_points_oracle.py) against the reference's
``kernel_point_optimization_debug`` and ``load_kernels`` with ``np.random`` patched to return the restatement's draws, the Philox
draws against the generator's published known answer, the committed disposition fixture, and the argument checks of the two
entry points (rejected before any launch)."""
import importlib.util
import os
import sys
import types

import numpy as np
import pytest

import kernel_points_oracle as O
from geotransformer_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = '/root/reference'
REF_KP = os.path.join(REF, 'geotransformer', 'modules', 'kpconv', 'kernel_points.py')
needs_ref = pytest.mark.skipif(not os.path.exists(REF_KP), reason='reference checkout not present')


def _ref_kernel_points(monkeypatch):
    """the reference's kernel_points.py as a module; its plotting and .ply imports are stubbed (neither runs on these paths)"""
    monkeypatch.setitem(sys.modules, 'matplotlib', types.ModuleType('matplotlib'))
    monkeypatch.setitem(sys.modules, 'matplotlib.pyplot', types.ModuleType('matplotlib.pyplot'))
    monkeypatch.setitem(sys.modules, 'open3d', types.ModuleType('open3d'))
    spec = importlib.util.spec_from_file_location('ref_kernel_points', REF_KP)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class _Rand:
    """np.random.rand stand-in: consecutive rows of a fixed (n, 3) array of uniforms"""

    def __init__(self, uniforms):
        self.u, self.pos = uniforms, 0

    def __call__(self, *shape):
        rows = shape[0]
        assert shape[1:] == (3,) and self.pos + rows <= self.u.shape[0]
        v = self.u[self.pos:self.pos + rows].copy()
        self.pos += rows
        return v


@needs_ref
@pytest.mark.parametrize('num_kernels', [1, 12])
def test_optimization_equals_reference_from_patched_draws(monkeypatch, num_kernels):
    ref = _ref_kernel_points(monkeypatch)
    uniforms = O.philox_uniforms(11, 200 * num_kernels * 15)
    monkeypatch.setattr(np.random, 'rand', _Rand(uniforms))
    want, want_norms = ref.kernel_point_optimization_debug(1.0, 15, num_kernels=num_kernels, dimension=3, fixed='center')
    want_best = int(np.argmin(want_norms[-1, :]))
    want_stop = int(np.count_nonzero(want_norms[:, 0])) - 1
    got, norms, stop, best = O.optimize(O.accept(uniforms, num_kernels * 15), num_kernels, 15)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
    np.testing.assert_array_equal(norms, want_norms)
    assert (best, stop) == (want_best, want_stop)
    assert stop < O.MAX_ITER


@needs_ref
def test_instance_equals_load_kernels_from_patched_draws(monkeypatch):
    ref = _ref_kernel_points(monkeypatch)
    disp = np.load(os.path.join(ROOT, 'tests', 'golden', 'kernel_disposition.npz'))['points']
    rng = np.random.default_rng(3)
    theta_u, noise = float(rng.random()), rng.normal(scale=0.01, size=(15, 3))

    class PointCloud:
        points = disp
    monkeypatch.setattr(ref, 'exists', lambda p: True)
    monkeypatch.setattr(ref, 'o3d', types.SimpleNamespace(io=types.SimpleNamespace(read_point_cloud=lambda f: PointCloud())),
                        raising=False)
    monkeypatch.setattr(np.random, 'rand', lambda: theta_u)
    monkeypatch.setattr(np.random, 'normal', lambda scale, size: noise)
    want = ref.load_kernels(0.0625, 15, dimension=3, fixed='center')
    got = O.instance(disp, 0.0625, theta_u, noise)
    assert got.dtype == np.float32 and want.dtype == np.float32
    np.testing.assert_array_equal(got, want)


def test_philox_known_answer():
    """Random123's published Philox4x32-10 answers for counter 0 / key 0 and counter = key = all ones"""
    z = O.philox4x32_10(np.zeros((1, 4), dtype=np.uint64), 0, 0)[0]
    assert [int(v) for v in z] == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    o = O.philox4x32_10(np.full((1, 4), 0xFFFFFFFF, dtype=np.uint64), 0xFFFFFFFF, 0xFFFFFFFF)[0]
    assert [int(v) for v in o] == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]


def test_disposition_fixture():
    f = np.load(os.path.join(ROOT, 'tests', 'golden', 'kernel_disposition.npz'))
    pts = f['points']
    assert pts.shape == (15, 3) and pts.dtype == np.float64
    assert np.all(pts[0] == 0)
    assert abs(float(f['mean_radius']) - 0.66) < 1e-6
    assert float(f['energy']) == pytest.approx(O.energy(pts), rel=1e-15)


def test_bad_arguments_are_rejected_before_any_launch():
    import ctypes
    lib = L.lib()
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf)

    def err():
        return lib.geob200_last_error().decode()
    assert lib.geob200_kernel_point_optimize(None, 100, 31, 0, 0.66, p, p, None) < 0 and 'num_points' in err()
    assert lib.geob200_kernel_point_optimize(None, 0, 15, 0, 0.66, p, p, None) < 0 and 'num_kernels' in err()
    assert lib.geob200_kernel_point_optimize(None, 200, 15, 0, 0.66, p, p, None) < 0 and 'num_kernels * num_points' in err()
    assert lib.geob200_kernel_point_optimize(None, 100, 15, 0, 0.0, p, p, None) < 0 and 'ratio' in err()
    assert lib.geob200_kernel_point_optimize(None, 100, 15, 0, 0.66, None, p, None) < 0 and 'null' in err()
    assert lib.geob200_kernel_point_instances(p, 0, p, p, 1, 0, p, None) < 0 and 'num_points' in err()
    assert lib.geob200_kernel_point_instances(p, 15, p, p, 0, 0, p, None) < 0 and 'num_layers' in err()
    assert lib.geob200_kernel_point_instances(p, 15, None, p, 1, 0, p, None) < 0 and 'null' in err()
    assert lib.geob200_launch_count() == 0
