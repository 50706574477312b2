"""Training-data augmentation on the device: both entry points against the numpy restatement (oracle/augment_oracle.py) under the
parity contract of DESIGN.md section 3b, the geometry of the augmented ground truth, the distributions of every draw, the
independence of the streams, and the engine with ``augment=True``."""
import copy

import numpy as np
import pytest
import torch
from scipy import stats
from scipy.spatial.transform import Rotation

from geotransformer_b200 import functional as GF
from geotransformer_b200.augment import augment_stacked, augmented_collate
from geotransformer_b200.synth import make_pair
from geotransformer_b200.train import TrainingEngine
from geotransformer_b200.utils.data import registration_collate_fn_stack_mode
from oracle import augment_oracle as AO
from oracle import backbone_grad_oracle as BV

pytestmark = pytest.mark.gpu
LIMIT = 700


def _pairs(B, seed, limit=LIMIT):
    """ragged synthetic pairs, some clouds above and some below the point limit; src row j maps onto ref row j under T"""
    rng = np.random.default_rng(seed)
    out = []
    for p in range(B):
        n = int(rng.integers(limit // 2, 2 * limit))
        R = Rotation.from_euler('zyx', rng.uniform(0, 2 * np.pi, 3)).as_matrix()
        t = rng.normal(size=3)
        ref = rng.normal(size=(n, 3)).astype(np.float32)
        src = ((ref.astype(np.float64) - t) @ R).astype(np.float32)
        m = int(rng.integers(limit // 2, 2 * limit))
        src = np.concatenate([src, rng.normal(size=(max(m - n, 0), 3)).astype(np.float32)])[:m] if m > n else src[:m]
        T = np.eye(4, dtype=np.float32)
        T[:3, :3], T[:3, 3] = R, t
        out.append(dict(ref_points=ref, src_points=src, transform=T))
    return out


def _run(pairs, mode, limit, noise, seed, it, pair_base=0, **kw):
    clouds = [torch.from_numpy(p['ref_points']) for p in pairs] + [torch.from_numpy(p['src_points']) for p in pairs]
    pts = torch.cat(clouds).cuda()
    T = torch.from_numpy(np.stack([p['transform'] for p in pairs])).cuda()
    out, lens, To, origin, rec = GF.augment_pairs_batched(pts, [len(c) for c in clouds], T, mode, limit, noise, seed=seed, iteration=it,
                                                          pair_base=pair_base, **kw)
    return out.cpu().numpy(), lens, To.cpu().numpy(), origin.cpu().numpy(), rec.cpu().numpy()


def _split(a, lens):
    o = np.cumsum([0] + list(lens))
    return [a[o[i]:o[i + 1]] for i in range(len(lens))]


def _ulp_close(a, b, n=1):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    tol = n * np.spacing(np.maximum(np.abs(a), np.abs(b)).astype(np.float32))
    return bool(np.all(np.abs(a.astype(np.float64) - b.astype(np.float64)) <= tol))


KW = {AO.THREEDMATCH: dict(rotation_factor=1.0), AO.KITTI: dict(rotation_factor=1.0, min_scale=0.8, max_scale=1.2, shift=2.0)}


@pytest.mark.parametrize('mode', [AO.THREEDMATCH, AO.KITTI])
@pytest.mark.parametrize('B', [1, 3, 8])
def test_pairs_match_the_restatement(mode, B):
    pairs = _pairs(B, 10 + B)
    noise = 0.005 if mode == AO.THREEDMATCH else 0.01
    out, lens, To, origin, rec = _run(pairs, mode, LIMIT, noise, 7351, 12, **KW[mode])
    assert lens == [min(len(p['ref_points']), LIMIT) for p in pairs] + [min(len(p['src_points']), LIMIT) for p in pairs]
    assert any(len(p['ref_points']) > LIMIT for p in pairs) or B == 1
    pts, org = _split(out, lens), _split(origin, lens)
    for p in range(B):
        w = AO.augment_pair(pairs[p]['ref_points'], pairs[p]['src_points'], pairs[p]['transform'], mode, LIMIT, noise, seed=7351,
                            iteration=12, pair=p, R=rec[p, 11:], **KW[mode])
        assert np.array_equal(rec[p, :11].view(np.int64), w['record'][:11].view(np.int64)), p
        u = rec[p, :3]
        np.testing.assert_allclose(rec[p, 11:].reshape(3, 3), Rotation.from_euler('zyx', (u * np.pi) * 2 / 1.0).as_matrix(), rtol=0,
                                   atol=1e-14)
        assert np.array_equal(org[p], w['ref_origin']) and np.array_equal(org[B + p], w['src_origin'])
        assert np.array_equal(pts[p].view(np.int32), w['ref'].view(np.int32)), p
        assert np.array_equal(pts[B + p].view(np.int32), w['src'].view(np.int32)), p
        assert _ulp_close(To[p], w['transform']), (To[p], w['transform'])


@pytest.mark.parametrize('mode', [AO.THREEDMATCH, AO.KITTI])
def test_augmented_transform_maps_src_onto_ref_without_noise(mode):
    """noise 0 and no point limit: row j of the augmented src maps onto row j of the augmented ref as the original did"""
    B = 4
    pairs = _pairs(B, 3, limit=10 ** 6)
    for p in pairs:
        n = min(len(p['ref_points']), len(p['src_points']))
        p['ref_points'], p['src_points'] = p['ref_points'][:n], p['src_points'][:n]
    out, lens, To, _, _ = _run(pairs, mode, 10 ** 6, 0.0, 5, 3, **KW[mode])
    pts = _split(out, lens)
    for p in range(B):
        T = To[p].astype(np.float64)
        mapped = pts[B + p].astype(np.float64) @ T[:3, :3].T + T[:3, 3]
        T0 = pairs[p]['transform'].astype(np.float64)
        base = np.abs(pairs[p]['src_points'].astype(np.float64) @ T0[:3, :3].T + T0[:3, 3] - pairs[p]['ref_points']).max()
        scale = np.abs(pts[p]).max() + 1.0
        assert np.abs(mapped - pts[p]).max() <= base * 1.3 + 8 * scale * 2.0 ** -23, p


def _shapes(B, seed, n=2048):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(B):
        p = rng.normal(size=(n, 3)) * np.array([1.0, 0.6, 0.3])
        out.append((p + 0.1 * np.sin(3 * p[:, [1, 2, 0]])).astype(np.float32))
    return out


def _run_mn(shapes, noise, seed, it, pair_base=0, num_points=717, keep=0.7):
    s = torch.from_numpy(np.concatenate(shapes)).cuda()
    out, lens, To, origin, rec = GF.modelnet_pairs_batched(s, [len(x) for x in shapes], num_points, keep, 45.0, 0.5, noise, seed, it,
                                                           pair_base)
    return out.cpu().numpy(), lens, To.cpu().numpy(), origin.cpu().numpy(), rec.cpu().numpy()


@pytest.mark.parametrize('B', [1, 3])
def test_modelnet_matches_the_restatement(B):
    shapes = _shapes(B, 40 + B)
    out, lens, To, origin, rec = _run_mn(shapes, 0.05, 9, 4)
    pts, org = _split(out, lens), _split(origin, lens)
    for p in range(B):
        w = AO.modelnet_pair(shapes[p], 717, 0.7, 45.0, 0.5, 0.05, seed=9, iteration=4, pair=p)
        for name in ('ref', 'src'):
            d = np.sort(w[name + '_d'])[::-1]
            k = AO.crop_count(2048, 0.7)
            assert d[k - 1] - d[k] > 1e-6                          # no near tie decides the crop
        assert np.array_equal(rec[p, :11].view(np.int64), w['record'][:11].view(np.int64))
        np.testing.assert_allclose(rec[p, 11:], w['record'][11:], rtol=0, atol=1e-14)
        assert np.array_equal(org[p], w['ref_origin']) and np.array_equal(org[B + p], w['src_origin'])
        assert _ulp_close(pts[p], w['ref']) and _ulp_close(pts[B + p], w['src'])
        assert _ulp_close(To[p], w['transform'])


def test_modelnet_without_jitter_keeps_the_normalised_rows():
    shapes = _shapes(2, 7)
    out, lens, _, origin, _ = _run_mn(shapes, 0.0, 1, 1)
    pts, org = _split(out, lens), _split(origin, lens)
    for p in range(2):
        norm = AO.normalize(shapes[p])
        assert _ulp_close(pts[p], norm[org[p]].astype(np.float32))
        assert len(set(org[p].tolist())) == 717


def test_draw_distributions():
    B, n, limit, iters = 8, 40, 12, 150
    pairs = [dict(ref_points=np.zeros((n, 3), np.float32), src_points=np.zeros((n, 3), np.float32), transform=np.eye(4, dtype=np.float32))
             for _ in range(B)]
    hits, coins, angles, noises, scales, shifts = np.zeros(n), [], [], [], [], []
    for it in range(iters):
        out, lens, _, origin, rec = _run(pairs, AO.KITTI, limit, 1.0, 3, it, **KW[AO.KITTI])
        np.add.at(hits, origin, 1)
        coins += list(rec[:, 3] > 0.5)
        angles += list(rec[:, :3].ravel())
        scales += list(rec[:, 4])
        shifts += list(rec[:, 5:11].ravel())
    assert stats.chisquare(hits).pvalue > 1e-3                                     # subset membership
    assert stats.binomtest(int(np.sum(coins)), len(coins)).pvalue > 1e-3          # the coin
    for x in (angles, scales, shifts):
        assert stats.kstest(x, 'uniform').pvalue > 1e-3
    # noise: zero clouds, 3DMatch order, noise 1: every output coordinate is (u - 0.5) (rotation of 0 is 0)
    out, _, _, _, _ = _run(pairs, AO.THREEDMATCH, 10 ** 6, 1.0, 3, 1)
    assert stats.kstest(out.ravel(), 'uniform', args=(-0.5, 1.0)).pvalue > 1e-3
    # KITTI: zero clouds, noise 0 -> the shift itself
    out, lens, _, _, rec = _run(pairs, AO.KITTI, 10 ** 6, 0.0, 3, 2, **KW[AO.KITTI])
    first = np.cumsum([0] + lens)[:-1]
    assert np.allclose(out[first[:B]], -2.0 + 4.0 * rec[:, 5:8], atol=1e-6)
    # jitter: clip(N(0, 0.01), +-0.05) around the normalised row
    shapes = _shapes(2, 3)
    out, lens, _, origin, _ = _run_mn(shapes, 0.05, 1, 1)
    j = np.concatenate([(pts.astype(np.float64) - AO.normalize(s)[o]).ravel()
                        for pts, o, s in zip(_split(out, lens)[:2], _split(origin, lens)[:2], shapes)])     # ref clouds
    assert np.abs(j).max() <= 0.05 + 1e-6
    assert stats.kstest(j / 0.01, 'norm').pvalue > 1e-3


def test_modelnet_sample_order_is_a_uniform_permutation():
    shapes = _shapes(8, 5, n=10)
    pos = np.zeros(10)
    for it in range(200):
        _, lens, _, origin, _ = _run_mn(shapes, 0.0, 2, it, num_points=10, keep=1.0)
        for o in _split(origin, lens):
            assert sorted(o.tolist()) == list(range(10))
            pos[int(np.nonzero(o == 0)[0][0])] += 1
    assert stats.chisquare(pos).pvalue > 1e-3


def test_streams_are_keyed_by_seed_iteration_and_pair():
    pairs = _pairs(4, 1)
    a = _run(pairs, AO.KITTI, LIMIT, 0.01, 5, 7, **KW[AO.KITTI])
    b = _run(pairs, AO.KITTI, LIMIT, 0.01, 5, 7, **KW[AO.KITTI])
    assert all(np.array_equal(x, y) for x, y in zip(a[::2] + (a[3], a[4]), b[::2] + (b[3], b[4])))
    lens = a[1]
    for p in range(4):
        one = _run([pairs[p]], AO.KITTI, LIMIT, 0.01, 5, 7, pair_base=p, **KW[AO.KITTI])
        pts = _split(a[0], lens)
        assert np.array_equal(one[0], np.concatenate([pts[p], pts[4 + p]]))
        assert np.array_equal(one[4][0], a[4][p]) and np.array_equal(one[2][0], a[2][p])
    c = _run(pairs, AO.KITTI, LIMIT, 0.01, 5, 8, **KW[AO.KITTI])
    assert not np.array_equal(a[4], c[4]) and not np.array_equal(a[0], c[0])
    shapes = _shapes(3, 2)
    m = _run_mn(shapes, 0.05, 5, 7)
    assert np.array_equal(m[0], _run_mn(shapes, 0.05, 5, 7)[0])
    one = _run_mn(shapes[2:], 0.05, 5, 7, pair_base=2)
    pts = _split(m[0], m[1])
    assert np.array_equal(one[0], np.concatenate([pts[2], pts[5]]))
    assert not np.array_equal(m[3], _run_mn(shapes, 0.05, 5, 8)[3])


def _train_pairs(n):
    out = []
    for i in range(n):
        p = make_pair('demo2k', i)
        out.append({k: p[k] for k in ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')})
    return out


def _cfg(models, name='3dmatch', limit=1500):
    cfg, sd, _ = models(name)
    cfg = copy.deepcopy(cfg)
    if name != 'modelnet':
        cfg.train.point_limit = limit
    return cfg, sd


def _fresh(cfg, sd):
    from geotransformer_b200.model import create_model
    model = create_model(cfg)
    model.load_state_dict(sd, strict=True)
    return model.cuda()


@pytest.mark.parametrize('B', [1, 3])
def test_augmented_collate_equals_the_plain_collate_of_the_augmented_pairs(models, B):
    cfg, _ = _cfg(models)
    pairs = _train_pairs(B)
    data = augmented_collate(pairs, cfg, cfg.neighbor_limits, 11, 4)
    pts, lens, T, _, _ = augment_stacked(pairs, cfg, 11, 4, torch.device('cuda', torch.cuda.current_device()))
    clouds = _split(pts.cpu().numpy(), lens)
    host = [dict(ref_points=clouds[p], src_points=clouds[B + p], ref_feats=np.ones((len(clouds[p]), 1), np.float32),
                 src_feats=np.ones((len(clouds[B + p]), 1), np.float32), transform=T[p].cpu().numpy()) for p in range(B)]
    b = cfg.backbone
    want = registration_collate_fn_stack_mode(host, b.num_stages, b.init_voxel_size, b.init_radius, cfg.neighbor_limits)
    assert set(data) == set(want)
    for k in want:
        x, y = data[k], want[k]
        if k == 'transform' and isinstance(y, list):
            y = torch.stack(y)
        if isinstance(y, torch.Tensor):
            assert torch.equal(x.cpu(), y.cpu()), k
        elif isinstance(y, list) and y and isinstance(y[0], torch.Tensor):
            assert all(torch.equal(u.cpu(), v.cpu()) for u, v in zip(x, y)), k
        else:
            assert x == y, k


def test_augmentation_does_not_synchronise(models):
    """the augmentation itself (H2D of the raw clouds and transforms, the kernels) never waits for the device; the collate's one
    read-back of the neighbour counts comes after it, as in the plain collate"""
    cfg, sd = _cfg(models)
    eng = TrainingEngine(_fresh(cfg, sd), cfg, cfg.neighbor_limits, batch_size=4, augment=True)
    pairs = [{k: torch.from_numpy(v).pin_memory() for k, v in p.items()} for p in _train_pairs(4)]
    eng.train_batch(pairs)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        augment_stacked(pairs, cfg, eng.seed, 9, eng.device)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert eng.iteration == 1


def _params(model):
    return [p.detach().contiguous().view(torch.int32).clone() for p in model.parameters()]


def test_resumed_augmented_run_equals_an_uninterrupted_run(models, tmp_path):
    cfg, sd = _cfg(models)
    pairs = _train_pairs(5)
    eng = TrainingEngine(_fresh(cfg, sd), cfg, cfg.neighbor_limits, batch_size=2, augment=True)
    straight = [eng.train_batch(pairs[i:i + 2]) for i in (0, 2, 4)]
    want = _params(eng.model)
    eng = TrainingEngine(_fresh(cfg, sd), cfg, cfg.neighbor_limits, batch_size=2, augment=True)
    first = [eng.train_batch(pairs[:2])]
    path = str(tmp_path / 'snapshot.pth.tar')
    eng.save_snapshot(path)
    eng2 = TrainingEngine(_fresh(cfg, sd), cfg, cfg.neighbor_limits, batch_size=2, augment=True)
    eng2.load_snapshot(path)
    rest = [eng2.train_batch(pairs[i:i + 2]) for i in (2, 4)]
    assert all(torch.equal(a, b) for a, b in zip(want, _params(eng2.model)))
    assert [r['loss'] for r in straight] == [r['loss'] for r in first + rest]
    # augmentation changes what is trained on
    plain = TrainingEngine(_fresh(cfg, sd), cfg, cfg.neighbor_limits, batch_size=2)
    assert plain.train_batch(pairs[:2])['loss'] != straight[0]['loss']


def test_modelnet_trains_from_raw_shapes(models):
    cfg, sd = _cfg(models, 'modelnet')
    eng = TrainingEngine(_fresh(cfg, sd), cfg, BV.limits('modelnet717'), batch_size=4, augment=True)
    shapes = [{'points': s} for s in _shapes(4, 11)]
    losses = [eng.train_batch(shapes)['loss'] for _ in range(3)]
    one = eng.train_step(shapes[0])['loss']
    print('modelnet losses', losses, one)
    assert all(np.isfinite(losses)) and np.isfinite(one)
