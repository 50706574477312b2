"""Normal estimation on the device (geob200_estimate_normals) against the C++ oracle (oracle/normals_oracle.cpp): neighbour lists
and covariances bit for bit, normals bit for bit or, where the device's acos / cos differ from the host libm's in the last bit,
within 1e-12 with the same sign wherever the two smallest eigenvalues are separated, and in the near-repeated eigenspace
elsewhere (DESIGN.md section 8a); regularize_normals bit for bit against the restatement of its numpy expression in
oracle/normals_oracle.py, which the CPU tests pin to the reference's own function; the drop-ins and the demo's PLY."""

import numpy as np
import pytest
import torch

from geotransformer_b200 import _lib as L
from geotransformer_b200 import functional as GF
from oracle import normals_oracle as NO

pytestmark = pytest.mark.gpu

CASES = NO.cases()


def _full(c):
    return np.array([[c[0], c[1], c[2]], [c[1], c[3], c[4]], [c[2], c[4], c[5]]])


def _separated(cov6):
    w = np.linalg.eigvalsh(_full(cov6))
    return w[1] - w[0] >= 1e-6 * max(abs(w).max(), 1e-300)


def _device(clouds, knn=30, radius=None, dtype=np.float64):
    lengths = [c.shape[0] for c in clouds]
    pts = torch.from_numpy(np.ascontiguousarray(np.concatenate([np.asarray(c, dtype) .reshape(-1, 3) for c in clouds]))).cuda()
    n, nbr, cov = GF.estimate_normals_batched(pts, lengths, knn=knn, radius=radius, return_neighbors=True)
    assert n.dtype == torch.float64 and n.shape == (sum(lengths), 3)
    split = np.cumsum([0] + lengths)
    n, nbr, cov = n.cpu().numpy(), nbr.cpu().numpy(), cov.cpu().numpy()
    return [(n[a:b], nbr[a:b], cov[a:b]) for a, b in zip(split[:-1], split[1:])]


def _compare(points, knn, radius, got, rows=None):
    """neighbours and covariances bit for bit; normals bit for bit or within 1e-12 with the same sign where separated.
    Returns the number of normals that are not bit-identical."""
    want_n, want_nbr, want_cov = NO.estimate_normals(points, knn, radius, rows=rows)
    g_n, g_nbr, g_cov = got if rows is None else (got[0][rows], got[1][rows], got[2][rows])
    assert np.array_equal(g_nbr, want_nbr), np.argwhere(g_nbr != want_nbr)[:5]
    assert np.array_equal(g_cov, want_cov), np.argwhere(g_cov != want_cov)[:5]
    diff = np.flatnonzero(np.any(g_n != want_n, 1))
    for i in diff:
        # the device's acos / cos are not the host libm's in every last bit: where the two smallest eigenvalues are separated
        # the normals agree within 1e-12 with the same sign; where they are not (collinear points), any unit vector of the
        # near-repeated eigenspace is an answer, and a last-bit difference can move the normal inside it
        if _separated(want_cov[i]):
            assert np.abs(g_n[i] - want_n[i]).max() <= 1e-12 and float(g_n[i] @ want_n[i]) > 0, (i, g_n[i], want_n[i])
        else:
            w = np.linalg.eigvalsh(_full(want_cov[i]))
            assert abs(np.linalg.norm(g_n[i]) - 1) <= 1e-12, (i, g_n[i])
            assert np.linalg.norm(_full(want_cov[i]) @ g_n[i]) <= w[1] + 1e-9 * abs(w).max(), (i, g_n[i], w)
    return len(diff)


@pytest.mark.parametrize('name', sorted(CASES))
def test_device_equals_oracle(name):
    pts, knn, radius = CASES[name]
    got = _device([pts], knn, radius, dtype=np.asarray(pts).dtype)[0]
    _compare(pts, knn, radius, got)


def test_fp32_and_fp64_input_agree():
    pts = CASES['float32'][0]
    a = _device([pts], dtype=np.float32)[0]
    b = _device([pts.astype(np.float64)], dtype=np.float64)[0]
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_kitti_ring_scan_and_fragment():
    rng = np.random.default_rng(5)
    scan = NO.ring_scan(rng)
    got = _device([scan], dtype=np.float32)[0]
    _compare(scan.astype(np.float64), 30, None, got, rows=rng.choice(scan.shape[0], 150, replace=False))
    frag = NO.fragment(rng)
    got = _device([frag])[0]
    _compare(frag, 30, None, got, rows=rng.choice(frag.shape[0], 100, replace=False))
    got = _device([frag], knn=30, radius=0.05)[0]
    _compare(frag, 30, 0.05, got, rows=rng.choice(frag.shape[0], 100, replace=False))


def test_ragged_batch_of_64_equals_single_calls_and_repeats():
    rng = np.random.default_rng(7)
    clouds = []
    for b in range(64):
        kind = b % 8
        if kind == 0:
            clouds.append(np.zeros((0, 3)))
        elif kind == 1:
            clouds.append(rng.uniform(-1, 1, (int(rng.integers(1, 30)), 3)))      # shorter than knn
        else:
            clouds.append(rng.uniform(-1, 1, (int(rng.integers(100, 3000)), 3)) * rng.uniform(0.1, 10) + rng.uniform(-50, 50, 3))
    batch = _device(clouds)
    again = _device(clouds)
    for b, c in enumerate(clouds):
        for x, y in zip(batch[b], again[b]):
            assert np.array_equal(x, y), b
        single = _device([c])[0]
        for x, y in zip(batch[b], single):
            assert np.array_equal(x, y), b
        if c.shape[0]:
            _compare(c, 30, None, batch[b], rows=None if c.shape[0] <= 600 else np.arange(0, c.shape[0], 7))


def test_errors_raise_and_write_nothing():
    p = torch.from_numpy(np.random.default_rng(0).uniform(-1, 1, (100, 3))).cuda()
    for knn in (0, -1, 65):
        with pytest.raises(ValueError):
            GF.estimate_normals_batched(p, [100], knn=knn)
    for radius in (0.0, -1.0, float('nan')):
        with pytest.raises(ValueError):
            GF.estimate_normals_batched(p, [100], radius=radius)
    for bad in (float('nan'), float('inf'), -float('inf')):
        q = p.clone()
        q[57, 2] = bad
        with pytest.raises(ValueError, match='NaN or infinite'):
            GF.estimate_normals_batched(q, [40, 60])
        # the entry point itself: status set, outputs untouched
        lib = L.lib()
        ws = torch.empty(lib.geob200_estimate_normals_workspace_bytes(100, 2), dtype=torch.uint8, device='cuda')
        out = torch.full((100, 3), 7.0, dtype=torch.float64, device='cuda')
        nbr = torch.full((100, 30), 7, dtype=torch.int32, device='cuda')
        cov = torch.full((100, 6), 7.0, dtype=torch.float64, device='cuda')
        st = torch.full((1,), -5, dtype=torch.int64, device='cuda')
        lengths = np.array([40, 60], dtype=np.int64)
        rc = lib.geob200_estimate_normals(q.data_ptr(), 100, lengths.ctypes.data, 2, 30, 0.0, out.data_ptr(), nbr.data_ptr(),
                                          cov.data_ptr(), st.data_ptr(), ws.data_ptr(), ws.numel(), L.stream_ptr())
        assert rc == 0 and int(st.item()) == 1
        assert bool((out == 7.0).all()) and bool((nbr == 7).all()) and bool((cov == 7.0).all())


def test_empty_cloud_and_drop_in():
    from geotransformer_b200.utils.open3d import estimate_normals
    e = GF.estimate_normals_batched(torch.zeros((0, 3), dtype=torch.float64, device='cuda'), [0])
    assert e.shape == (0, 3)
    pts = CASES['random'][0]
    n_np = estimate_normals(pts)
    assert isinstance(n_np, np.ndarray) and n_np.dtype == np.float64
    n_t = estimate_normals(torch.from_numpy(pts).cuda())
    assert n_t.is_cuda and n_t.dtype == torch.float64
    assert np.array_equal(n_np, n_t.cpu().numpy())
    assert np.array_equal(n_np, _device([pts])[0][0])


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_regularize_normals_bit_for_bit(dtype):
    from geotransformer_b200.utils.pointcloud import regularize_normals
    rng = np.random.default_rng(11)
    p = rng.standard_normal((5000, 3)).astype(dtype)
    n = rng.standard_normal((5000, 3)).astype(dtype)
    # zeros of both signs, dot products of exactly 0, and points orthogonal to their normals
    n[:50] = np.array([0.0, -0.0, 0.0], dtype)
    n[50:100] = np.array([-0.0, -0.0, -0.0], dtype)
    p[100:150] = 0.0
    n[150:200, 2] = -0.0
    p[200:250] = np.array([1.0, 0.0, 0.0], dtype)
    n[200:250] = np.array([0.0, 1.0, -0.0], dtype)
    for positive in (True, False):
        want = NO.regularize_normals(p, n, positive)
        got = regularize_normals(p, n, positive)
        assert got.dtype == want.dtype
        assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), positive
        got_t = regularize_normals(torch.from_numpy(p).cuda(), torch.from_numpy(n).cuda(), positive)
        assert np.array_equal(got_t.cpu().numpy().view(np.uint8), want.view(np.uint8))
    # mixed types promote to float64, as numpy does
    want = NO.regularize_normals(p.astype(np.float32), n.astype(np.float64))
    got = regularize_normals(p.astype(np.float32), n.astype(np.float64))
    assert got.dtype == np.float64 and np.array_equal(got.view(np.uint8), want.view(np.uint8))


def _old_ply(path, ref_points, src_points):
    """the PLY the demo wrote before normals existed"""
    rows = [(p, (255, 204, 102)) for p in ref_points] + [(p, (102, 153, 255)) for p in src_points]
    with open(path, 'w') as f:
        f.write('ply\nformat ascii 1.0\n')
        f.write(f'element vertex {len(rows)}\n')
        f.write('property float x\nproperty float y\nproperty float z\n')
        f.write('property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n')
        for p, c in rows:
            f.write(f'{float(p[0]):.9g} {float(p[1]):.9g} {float(p[2]):.9g} {c[0]} {c[1]} {c[2]}\n')


def test_demo_normals_ply(tmp_path):
    from geotransformer_b200 import demo
    from geotransformer_b200.config import make_cfg
    from geotransformer_b200.model import create_model
    from geotransformer_b200.synth import make_pair
    from geotransformer_b200.utils.open3d import estimate_normals
    from geotransformer_b200.weights import synthetic_state_dict
    cfg = make_cfg('3dmatch')
    model = create_model(cfg)
    state = synthetic_state_dict(model, 7351)
    pair = make_pair('demo2k', 0)
    files = {}
    for name, key in (('src', 'src_points'), ('ref', 'ref_points')):
        files[name] = str(tmp_path / f'{name}.npy')
        np.save(files[name], pair[key])
    weights = str(tmp_path / 'snapshot.pth.tar')
    torch.save({'model': state}, weights)
    base = ['--src-file', files['src'], '--ref-file', files['ref'], '--weights', weights]
    demo.main(base + ['--output', str(tmp_path / 'plain')])
    demo.main(base + ['--output', str(tmp_path / 'shaded'), '--normals'])
    T = np.load(str(tmp_path / 'plain' / 'estimated_transform.npy'))
    assert np.array_equal(T, np.load(str(tmp_path / 'shaded' / 'estimated_transform.npy')))
    ref = pair['ref_points'].astype(np.float32)
    src = pair['src_points'].astype(np.float32).astype(np.float64)
    aligned = src @ T[:3, :3].T.astype(np.float64) + T[:3, 3].astype(np.float64)
    _old_ply(str(tmp_path / 'old.ply'), ref, aligned)
    with open(str(tmp_path / 'old.ply'), 'rb') as a, open(str(tmp_path / 'plain' / 'registration.ply'), 'rb') as b:
        assert a.read() == b.read()
    with open(str(tmp_path / 'shaded' / 'registration.ply')) as f:
        text = f.read()
    head, body = text.split('end_header\n')
    assert 'property double nx\nproperty double ny\nproperty double nz\n' in head
    rows = np.array([[float(v) for v in line.split()] for line in body.strip().splitlines()])
    want_ref = estimate_normals(ref)
    want_src = estimate_normals(pair['src_points'].astype(np.float32)) @ T[:3, :3].astype(np.float64).T
    assert np.array_equal(rows[:ref.shape[0], 3:6], want_ref)
    assert np.array_equal(rows[ref.shape[0]:, 3:6], want_src)
    assert np.array_equal(rows[:, :3], np.array([[float(v) for v in line.split()[:3]] for line in
                                                 open(str(tmp_path / 'old.ply')).read().split('end_header\n')[1].strip().splitlines()]))
