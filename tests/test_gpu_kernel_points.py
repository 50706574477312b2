"""Kernel-point dispositions on the device against the numpy restatement (tests/kernel_points_oracle.py) and the reference's
shipped disposition (tests/golden/kernel_disposition.npz), and the per-instance buffers of ``initialize_kernel_points``."""
import math
import os

import numpy as np
import pytest
import torch

import kernel_points_oracle as O
from geotransformer_b200.modules.kpconv import kernel_points as KP

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ply():
    return np.load(os.path.join(ROOT, 'tests', 'golden', 'kernel_disposition.npz'))


def test_optimizer_equals_restatement_from_given_points():
    init = O.accept(O.philox_uniforms(5, 12000), 1500)
    want, _, want_stop, want_best = O.optimize(init, 100, 15)
    got, best, stop = KP.optimize_dispositions(15, init=init)
    assert (best, stop) == (want_best, want_stop)
    assert float((got.cpu() - torch.from_numpy(want)).abs().max()) < 1e-9


def test_optimizer_draws_and_shipped_disposition():
    """from its own Philox draws (the restatement of those draws gives the same run) the disposition's potential equals the
    reference file's to 1e-6 relative; the points agree after alignment to the level the descent's stopping test allows"""
    got, best, stop = KP.optimize_dispositions(15)
    init = O.accept(O.philox_uniforms(KP.DISPOSITION_SEED, 12000), 1500)
    want, _, want_stop, want_best = O.optimize(init, 100, 15)
    assert (best, stop) == (want_best, want_stop)
    assert float((got.cpu() - torch.from_numpy(want)).abs().max()) < 1e-9
    d = got[best].cpu().numpy()
    f = _ply()
    assert abs(O.energy(d) - float(f['energy'])) / float(f['energy']) < 1e-6
    assert abs(np.linalg.norm(got[:, 1:].cpu().numpy(), axis=-1).mean() - 0.66) < 1e-12     # one scale for all candidates
    # after the best rotation (or reflection) and point assignment: 5.5e-4 measured; both descents stop on a change-of-gradient
    # test, not at the exact minimum, so the 1e-4 the two files would share at the minimum is not reached
    assert _aligned_max_diff(d, f['points']) < 6e-4


def _aligned_max_diff(A, B, starts=300):
    """min over proper and improper rotations of the largest point distance after an optimal assignment, Kabsch-refined from
    ``starts`` fixed random rotations"""
    from scipy.optimize import linear_sum_assignment
    from scipy.spatial.transform import Rotation
    best = np.inf
    for R0 in Rotation.random(starts, random_state=0).as_matrix():
        for refl in (1.0, -1.0):
            X, R = A * np.array([1.0, 1.0, refl]), R0
            for _ in range(10):
                r, c = linear_sum_assignment(np.linalg.norm((X @ R.T)[:, None] - B[None], axis=-1))
                U, _, Vt = np.linalg.svd(X[r].T @ B[c])
                R = Vt.T @ np.diag([1.0, 1.0, np.sign(np.linalg.det(Vt.T @ U.T))]) @ U.T
            best = min(best, float(np.abs(X[r] @ R.T - B[c]).max()))
    return best


def test_instances_are_noised_rotations_scaled_by_radius():
    disp = KP.disposition(15)
    d32 = disp.float().double().cpu().numpy()
    ids = list(range(8))
    a = KP.kernel_point_instances(disp, [1.0] * 8, ids, seed=42).double().cpu().numpy()
    b = KP.kernel_point_instances(disp, [2.0] * 8, ids, seed=42).double().cpu().numpy()
    again = KP.kernel_point_instances(disp, [1.0] * 8, ids, seed=42).cpu().numpy()
    other = KP.kernel_point_instances(disp, [1.0] * 8, ids, seed=43).cpu().numpy()
    assert np.array_equal(a.astype(np.float32), again) and not np.array_equal(again, other)
    assert np.array_equal(b, a * 2.0)      # the radius scales the fp64 points before the one rounding to fp32
    for l in range(8):
        # undo the rotation about z: the in-plane angle that best maps the disposition onto the instance
        x, y = a[l, :, 0], a[l, :, 1]
        theta = math.atan2(np.sum(y * d32[:, 0] - x * d32[:, 1]), np.sum(x * d32[:, 0] + y * d32[:, 1]))
        c, s = math.cos(theta), math.sin(theta)
        back = np.stack([x * c + y * s, y * c - x * s, a[l, :, 2]], axis=1)
        noise = back - d32
        assert np.abs(noise).max() < 0.06 and 0.004 < noise.std() < 0.02, (l, noise.std())
    assert len({a[l].tobytes() for l in range(8)}) == 8


def test_initialize_kernel_points_is_reproducible_per_seed():
    from geotransformer_b200.config import make_cfg
    from geotransformer_b200.model import create_model
    cfg = make_cfg('3dmatch')
    m1, m2 = create_model(cfg).cuda(), create_model(cfg).cuda()
    n = KP.initialize_kernel_points(m1, 7)
    assert n == sum(1 for m in m1.modules() if m.__class__.__name__ == 'KPConv') and n > 1
    KP.initialize_kernel_points(m2, 7)
    convs1 = [m for m in m1.modules() if m.__class__.__name__ == 'KPConv']
    convs2 = [m for m in m2.modules() if m.__class__.__name__ == 'KPConv']
    for c1, c2 in zip(convs1, convs2):
        assert torch.equal(c1.kernel_points, c2.kernel_points)
        r = c1.kernel_points.norm(dim=1)[1:].mean().item() / c1.radius
        assert abs(r - 0.66) < 0.02
