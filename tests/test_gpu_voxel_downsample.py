"""Voxel downsampling on the device (geob200_voxel_down_sample) against the C++ oracle (oracle/voxel_oracle.cpp), bit for bit in
values and order, and the entry points built on it: utils.open3d.voxel_downsample, the KITTI preparation driver and the demo."""
import io
import os
import pickle
import re
import time

import numpy as np
import pytest
import torch

from geotransformer_b200 import functional as GF
from oracle import voxel_oracle as VO

pytestmark = pytest.mark.gpu

GROWTH = [13, 29, 59, 127, 257, 541, 1109, 2357, 5087, 10273, 20753, 42043, 85229, 172933]


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).cuda()


def _device_clouds(clouds, voxel, normals=None):
    """one batched call; returns per-cloud (points[, normals]) numpy float64"""
    lengths = [c.shape[0] for c in clouds]
    pts = _dev(np.concatenate(clouds).reshape(-1, 3))
    nrm = None if normals is None else _dev(np.concatenate(normals).reshape(-1, 3))
    res = GF.voxel_down_sample_batched(pts, lengths, voxel, normals=nrm)
    out_len = res[1].cpu().tolist()
    assert res[0].dtype == torch.float64 and res[0].shape[0] == sum(out_len)
    split = np.cumsum([0] + out_len)
    p = res[0].cpu().numpy()
    n = None if normals is None else res[2].cpu().numpy()
    return [(p[split[i]:split[i + 1]], None if n is None else n[split[i]:split[i + 1]]) for i in range(len(clouds))]


def _check(clouds, voxel, with_normals=True, seed=0):
    rng = np.random.default_rng(seed)
    normals = [rng.standard_normal(c.shape) for c in clouds] if with_normals else None
    got = _device_clouds(clouds, voxel, normals)
    for i, c in enumerate(clouds):
        if with_normals:
            want_p, want_n = VO.voxel_down_sample(c, voxel, normals[i])
            assert np.array_equal(got[i][1], want_n), f'cloud {i}: normals differ'
        else:
            want_p = VO.voxel_down_sample(c, voxel)
        assert got[i][0].shape == want_p.shape, (i, got[i][0].shape, want_p.shape)
        assert np.array_equal(got[i][0], want_p), f'cloud {i}: points differ'
    return got


def lattice(m, voxel, rng, dup=0.3):
    """a cloud with exactly m voxels: one jittered point per lattice cell (a fraction twice) in the cell's upper half, and a point
    at 0.5 voxel on every axis, so that lo = 0 and cell i is voxel i"""
    g = rng.permutation(m)
    side = 64
    cells = np.stack([g % side, (g // side) % side, g // (side * side)], 1).astype(np.float64)
    pts = (cells + 0.5 + rng.uniform(0.0, 0.45, cells.shape)) * voxel
    extra = pts[rng.random(m) < dup] + rng.uniform(0.0, 0.04, (1, 3)) * voxel
    pts = np.concatenate([np.full((1, 3), 0.5 * voxel), pts, extra])
    return pts


def ring_scan(rng, n=120000):
    """a KITTI-like velodyne sweep: 64 rings, ranges 3..80 m, float32 as stored in the .bin files"""
    rings = 64
    az = rng.uniform(0, 2 * np.pi, n)
    elev = np.deg2rad(rng.integers(0, rings, n) * (28.0 / rings) - 25.0)
    r = rng.uniform(3.0, 80.0, n)
    xyz = np.stack([r * np.cos(az) * np.cos(elev), r * np.sin(az) * np.cos(elev), r * np.sin(elev) + 1.73], 1)
    return xyz.astype(np.float32).astype(np.float64)


def fragment(rng, n=300000):
    """a dense RGB-D-like fragment: points on a few planes and a sphere in a 3 m box, genuinely float64"""
    k = n // 4
    a = np.stack([rng.uniform(0, 3, k), rng.uniform(0, 3, k), np.zeros(k)], 1)
    b = np.stack([np.zeros(k), rng.uniform(0, 3, k), rng.uniform(0, 3, k)], 1)
    c = np.stack([rng.uniform(0, 3, k), np.full(k, 3.0), rng.uniform(0, 3, k)], 1)
    d = rng.standard_normal((n - 3 * k, 3))
    d = d / np.linalg.norm(d, axis=1, keepdims=True) * 0.7 + 1.5
    return np.concatenate([a, b, c, d]) + rng.normal(0, 0.003, (n, 3))


@pytest.mark.parametrize('with_normals', [False, True])
def test_lattices_at_every_bucket_growth(with_normals):
    """voxel counts exactly at and one past every libstdc++ bucket growth up to 172933"""
    rng = np.random.default_rng(1)
    counts = [1] + [c + d for c in GROWTH for d in (0, 1)]
    clouds = [lattice(m, 0.3, rng) for m in counts]
    got = _check(clouds, 0.3, with_normals)
    assert [g[0].shape[0] for g in got] == counts


@pytest.mark.parametrize('with_normals', [False, True])
def test_kitti_ring_scans(with_normals):
    rng = np.random.default_rng(2)
    _check([ring_scan(rng) for _ in range(16)], 0.3, with_normals)


@pytest.mark.parametrize('with_normals', [False, True])
def test_dense_fragment(with_normals):
    rng = np.random.default_rng(3)
    _check([fragment(rng)], 0.025, with_normals)


def test_one_voxel_of_100k_points_is_linear():
    rng = np.random.default_rng(4)
    cloud = rng.uniform(0.0, 0.1, (100000, 3))
    got = _check([cloud], 0.3)
    assert got[0][0].shape == (1, 3)
    pts = _dev(cloud)
    GF.voxel_down_sample_batched(pts, [100000], 0.3)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    GF.voxel_down_sample_batched(pts, [100000], 0.3)
    torch.cuda.synchronize()
    assert time.perf_counter() - t0 < 0.25       # a quadratic reduce would take seconds here


def test_points_exactly_on_voxel_faces():
    clouds = []
    # v = 0.25: p - lo = k v exactly (lo = -0.125 from the point at 0)
    k = np.arange(0, 40, dtype=np.float64)
    face = 0.25 * k - 0.125
    face[0] = 0.0
    g = np.stack(np.meshgrid(face, face[:7], face[:5], indexing='ij'), -1).reshape(-1, 3)
    clouds.append(g)
    # v = 0.3: points at lo + k v rounded in double, on either side of the face
    lo = -0.15
    f = lo + 0.3 * k[1:]
    g2 = np.concatenate([np.stack([f, f, f], 1), np.stack([np.nextafter(f, -np.inf)] * 3, 1), np.zeros((1, 3))])
    clouds.append(g2)
    _check(clouds[:1], 0.25)
    _check(clouds[1:], 0.3)


def test_negative_and_far_from_origin():
    rng = np.random.default_rng(5)
    base = rng.uniform(-3, 3, (50000, 3))
    _check([base - 7.0, base + 1e5, base - np.array([1e5, -1e5, 3e5])], 0.05)
    _check([(base + 1e5).astype(np.float32).astype(np.float64)], 0.3)


def test_float32_input_is_widened_exactly():
    rng = np.random.default_rng(6)
    c32 = rng.uniform(-10, 10, (40000, 3)).astype(np.float32)
    want = VO.voxel_down_sample(c32.astype(np.float64), 0.3)
    got, _ = GF.voxel_down_sample_batched(torch.from_numpy(c32).cuda(), [c32.shape[0]], 0.3)
    assert np.array_equal(got.cpu().numpy(), want)


def test_ragged_batch_of_64_equals_single_calls():
    rng = np.random.default_rng(7)
    sizes = [int(s) for s in rng.integers(0, 20000, 64)]
    sizes[3], sizes[10], sizes[40], sizes[63] = 0, 1, 0, 1
    clouds = [rng.uniform(-5, 5, (s, 3)) * rng.uniform(0.5, 3) for s in sizes]
    got = _check(clouds, 0.2)
    normals = [rng.standard_normal(c.shape) for c in clouds]
    batched = _device_clouds(clouds, 0.2, normals)
    for i, c in enumerate(clouds):
        single = _device_clouds([c], 0.2, [normals[i]])[0]
        assert np.array_equal(batched[i][0], single[0]) and np.array_equal(batched[i][1], single[1])
        assert np.array_equal(batched[i][0], got[i][0])
    assert [g[0].shape[0] for g in got][3] == 0 and [g[0].shape[0] for g in got][10] == 1


def test_errors_produce_no_output():
    good = np.random.default_rng(8).uniform(0, 1, (100, 3))
    cases = [([good, np.array([[0.0, np.nan, 0.0]])], 0.1, 'NaN or infinite'),
             ([np.array([[0.0, 0.0, np.inf]]), good], 0.1, 'NaN or infinite'),
             ([np.array([[0.0, 0, 0], [1e9, 0, 0]])], 1e-9, 'too small'),
             ([good, np.array([[0.0, 0, 0], [3e6, 0, 0]])], 1.0, '2^21')]
    for clouds, voxel, word in cases:
        with pytest.raises(RuntimeError, match=re.escape(word)):
            _device_clouds(clouds, voxel)
    for voxel in (0.0, -1.0):
        with pytest.raises(RuntimeError, match='voxel_size'):
            _device_clouds([good], voxel)
    with pytest.raises(RuntimeError, match='1..64'):
        _device_clouds([good] * 65, 0.1)
    # at the C entry point: every count is 0 and the status word names the error
    from geotransformer_b200 import _lib as L
    lib = L.lib()
    pts = _dev(np.concatenate([good, [[0.0, np.nan, 0.0]]]))
    out = torch.full((101, 3), -1.0, dtype=torch.float64, device='cuda')
    lens = torch.full((3,), -7, dtype=torch.int64, device='cuda')
    ws = torch.empty(lib.geob200_voxel_down_sample_workspace_bytes(101, 2), dtype=torch.uint8, device='cuda')
    L.check(lib.geob200_voxel_down_sample(pts.data_ptr(), None, 101, GF._host_i64([100, 1]), 2, 0.1, out.data_ptr(), None,
                                          lens.data_ptr(), ws.data_ptr(), ws.numel(), L.stream_ptr()), 'voxel')
    assert lens.cpu().tolist() == [0, 0, 1]
    assert bool((out == -1.0).all())


def test_open3d_voxel_downsample_kinds():
    from geotransformer_b200.utils.open3d import voxel_downsample
    rng = np.random.default_rng(9)
    p = rng.uniform(0, 2, (5000, 3)).astype(np.float32)
    n = rng.standard_normal((5000, 3))
    want_p, want_n = VO.voxel_down_sample(p.astype(np.float64), 0.1, n)
    got = voxel_downsample(p, 0.1)
    assert isinstance(got, np.ndarray) and got.dtype == np.float64 and np.array_equal(got, want_p)
    gp, gn = voxel_downsample(p, 0.1, normals=n)
    assert gp.dtype == gn.dtype == np.float64 and np.array_equal(gp, want_p) and np.array_equal(gn, want_n)
    t = voxel_downsample(torch.from_numpy(p).cuda(), 0.1)
    assert isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float64 and np.array_equal(t.cpu().numpy(), want_p)
    tp, tn = voxel_downsample(torch.from_numpy(p).cuda(), 0.1, normals=torch.from_numpy(n).cuda())
    assert tn.is_cuda and np.array_equal(tn.cpu().numpy(), want_n)
    with pytest.raises(RuntimeError, match='CUDA'):
        voxel_downsample(torch.from_numpy(p), 0.1)


def test_kitti_driver_writes_the_reference_files(tmp_path):
    from geotransformer_b200.datasets import kitti_downsample
    from geotransformer_b200.datasets.kitti import KittiPairs
    rng = np.random.default_rng(10)
    root = str(tmp_path)
    scans = {}
    for seq in ('00', '03'):
        os.makedirs(os.path.join(root, 'sequences', seq, 'velodyne'))
        for f in range(3):
            xyz = ring_scan(rng, 30000).astype(np.float32)
            rec = np.concatenate([xyz, rng.uniform(0, 1, (xyz.shape[0], 1)).astype(np.float32)], 1)
            rec.tofile(os.path.join(root, 'sequences', seq, 'velodyne', f'{f:06d}.bin'))
            scans[(seq, f'{f:06d}')] = xyz
    assert kitti_downsample.run(root, sequences=[0, 3], batch=4, threads=2, log=None) == 6
    for (seq, frame), xyz in scans.items():
        want = io.BytesIO()
        np.save(want, VO.voxel_down_sample(xyz.astype(np.float64), 0.3).astype(np.float32))
        with open(os.path.join(root, 'downsampled', seq, frame + '.npy'), 'rb') as fh:
            assert fh.read() == want.getvalue(), (seq, frame)
    os.makedirs(os.path.join(root, 'metadata'))
    meta = [{'seq_id': 3, 'frame0': 0, 'frame1': 2, 'pcd0': 'downsampled/03/000000.npy', 'pcd1': 'downsampled/03/000002.npy',
             'transform': np.eye(4)}]
    with open(os.path.join(root, 'metadata', 'test.pkl'), 'wb') as fh:
        pickle.dump(meta, fh)
    item = KittiPairs(root, 'test')[0]
    want = VO.voxel_down_sample(scans[('03', '000000')].astype(np.float64), 0.3).astype(np.float32)
    assert np.array_equal(item['ref_points'], want)


@pytest.mark.parametrize('voxel_size', [None, 0.025])
def test_demo_prints_the_reference_line_and_saves_the_model_estimate(tmp_path, capsys, voxel_size):
    from geotransformer_b200 import demo
    from geotransformer_b200.config import make_cfg
    from geotransformer_b200.model import create_model
    from geotransformer_b200.synth import make_pair
    from geotransformer_b200.utils.data import registration_collate_fn_stack_mode
    from geotransformer_b200.utils.open3d import voxel_downsample
    from geotransformer_b200.weights import synthetic_state_dict
    cfg = make_cfg('3dmatch')
    model = create_model(cfg)
    state = synthetic_state_dict(model, 7351)
    model.load_state_dict(state, strict=True)
    model = model.cuda().eval()
    pair = make_pair('demo2k', 0)
    files = {}
    for name, key in (('src', 'src_points'), ('ref', 'ref_points'), ('gt', 'transform')):
        files[name] = str(tmp_path / f'{name}.npy')
        np.save(files[name], pair[key])
    weights = str(tmp_path / 'snapshot.pth.tar')
    torch.save({'model': state}, weights)
    argv = ['--src-file', files['src'], '--ref-file', files['ref'], '--gt-file', files['gt'], '--weights', weights,
            '--output', str(tmp_path / 'out')]
    if voxel_size is not None:
        argv += ['--voxel-size', str(voxel_size)]
    demo.main(argv)
    line = capsys.readouterr().out.strip().splitlines()[-1]
    assert re.fullmatch(r'RRE\(deg\): \d+\.\d{3}, RTE\(m\): \d+\.\d{3}', line), line

    src, ref = np.load(files['src']), np.load(files['ref'])
    if voxel_size is not None:
        src, ref = voxel_downsample(src, voxel_size), voxel_downsample(ref, voxel_size)
        assert src.shape[0] < pair['src_points'].shape[0]
    dd = {'ref_points': ref.astype(np.float32), 'src_points': src.astype(np.float32),
          'ref_feats': np.ones((ref.shape[0], 1), np.float32), 'src_feats': np.ones((src.shape[0], 1), np.float32),
          'transform': pair['transform'].astype(np.float32)}
    data = registration_collate_fn_stack_mode([dd], cfg.backbone.num_stages, cfg.backbone.init_voxel_size, cfg.backbone.init_radius,
                                              [38, 36, 36, 38])
    want = model(data)['estimated_transform'].cpu().numpy()
    got = np.load(str(tmp_path / 'out' / 'estimated_transform.npy'))
    assert got.dtype == np.float32 and np.array_equal(got, want)
    with open(str(tmp_path / 'out' / 'registration.ply')) as fh:
        head = [next(fh) for _ in range(10)]
        body = fh.readlines()
    n_vertex = int(head[2].split()[-1])
    assert head[0] == 'ply\n' and head[-1] == 'end_header\n' and len(body) == n_vertex
    assert body[0].rstrip().endswith('255 204 102') and body[-1].rstrip().endswith('102 153 255')
