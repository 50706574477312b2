"""ModelNet validation / test pairs on the device (``functional.modelnet_benchmark_pairs_batched``, ``datasets.modelnet``) against
the reference's deterministic dataset (tests/golden/modelnet_benchmark.npz, written by oracle/modelnet_benchmark_vectors.py) and
its numpy restatement (oracle/modelnet_benchmark_oracle.py).

Exactness: the shape row of every output point is exactly the reference's.  Coordinates and transforms are bit-identical except
where the host's float64 BLAS dot products / libm and the device's pinned operation order round differently in the last float64
bit; such an element may then round to the neighbouring float32, so up to 1 float32 ulp is allowed and the count is reported."""
import copy
import os
import pickle

import numpy as np
import pytest
import torch

from geotransformer_b200 import _lib as L
from geotransformer_b200 import functional as GF
from geotransformer_b200.config import make_cfg
from geotransformer_b200.datasets.modelnet import ModelNetPairs
from oracle import modelnet_benchmark_oracle as MB

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'modelnet_benchmark.npz')
OPT = (0.7, 45.0, 0.5, 0.05)                 # keep_ratio, rotation, translation, noise


def _gold():
    g = np.load(GOLD)
    starts = np.concatenate([[0], np.cumsum(g['length'])])
    shapes = [g['shape'][starts[i]:starts[i + 1]] for i in range(len(g['length']))]
    return g, shapes


def _build(shapes, indices, m=717, opt=OPT):
    raw = torch.from_numpy(np.concatenate(shapes).astype(np.float32)).cuda()
    pts, _, T, origin = GF.modelnet_benchmark_pairs_batched(raw, [len(s) for s in shapes], indices, m, *opt)
    B = len(shapes)
    pts, T, origin = pts.cpu().numpy(), T.cpu().numpy(), origin.cpu().numpy()
    return [dict(ref_points=pts[p * m:(p + 1) * m], src_points=pts[(B + p) * m:(B + p + 1) * m], transform=T[p],
                 ref_origin=origin[p * m:(p + 1) * m], src_origin=origin[(B + p) * m:(B + p + 1) * m]) for p in range(B)]


def _ulps(a, b):
    """elementwise distance in float32 ulps"""
    def ordered(x):
        i = np.ascontiguousarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(a) - ordered(b))


def _compare(got, want, what):
    """origin exactly equal; points and transform within 1 ulp; returns the count of 1-ulp elements"""
    n1 = 0
    for k in ('ref_origin', 'src_origin'):
        assert np.array_equal(got[k], want[k]), (what, k)
    for k in ('ref_points', 'src_points', 'transform'):
        u = _ulps(got[k], want[k])
        assert u.max() <= 1, (what, k, int(u.max()))
        n1 += int((u == 1).sum())
    return n1


def test_pairs_match_the_reference_fixture():
    g, shapes = _gold()
    got = _build(shapes, g['index'].tolist())
    total = 0
    for p in range(len(shapes)):
        want = {k: g[k][p] for k in ('ref_points', 'src_points', 'transform', 'ref_origin', 'src_origin')}
        total += _compare(got[p], want, f'index {int(g["index"][p])}')
    n = sum(x.size for p in range(len(shapes)) for x in (g['ref_points'][p], g['src_points'][p], g['transform'][p]))
    print(f'fixture: {total} of {n} elements 1 ulp from the reference, the rest bit-identical')
    assert total <= n // 1000


@pytest.mark.parametrize('m', [717, 716])
def test_pairs_match_the_restatement(m):
    shapes = [s['points'] for s in MB.synthetic_shapes(240, seed=31 + m)]
    rng = np.random.default_rng(m)
    indices = [int(v) for v in rng.integers(0, 1 << 32, len(shapes))]
    indices[:3] = [0, 1, (1 << 32) - 1]
    got = _build(shapes, indices, m)
    total, n, undecided = 0, 0, 0
    for p, (s, i) in enumerate(zip(shapes, indices)):
        want = MB.benchmark_pair(s, i, m, *OPT)
        if want['gap'] < 1e-12:            # a near-tie of two crop distances: the crop order may legitimately differ
            undecided += 1
            continue
        total += _compare(got[p], want, f'index {i}')
        n += 2 * m * 3 + 16
    print(f'num_points {m}: {total} of {n} elements 1 ulp from the restatement; {undecided} pairs with a near-tied crop skipped')
    assert undecided <= 2 and total <= n // 1000


def test_each_pair_is_the_same_alone_and_in_any_batch():
    g, shapes = _gold()
    idx = g['index'].tolist()
    together = _build(shapes, idx)
    for p in range(len(shapes)):
        alone = _build([shapes[p]], [idx[p]])[0]
        assert all(np.array_equal(alone[k], together[p][k]) for k in alone), p
    order = list(range(len(shapes)))[::-1]
    rev = _build([shapes[p] for p in order], [idx[p] for p in order])
    assert all(np.array_equal(rev[i][k], together[p][k]) for i, p in enumerate(order) for k in rev[i])
    # more pairs than one launch takes: the host splits the call; pairs across the split are unchanged
    small = [s['points'][:300] for s in MB.synthetic_shapes(5, seed=3, small_every=0)]
    many = [small[i % 5] for i in range(1030)]
    many_idx = list(range(1030))
    big = _build(many, many_idx, 64)
    for p in (0, 1023, 1024, 1029):
        one = _build([many[p]], [p], 64)[0]
        assert all(np.array_equal(one[k], big[p][k]) for k in one), p


def _write_pkl(tmp_path, g, shapes):
    """the fixture's pkl: its filtered shapes with a symmetric-class shape (label 5) at row 1"""
    labels = g['labels'].tolist()
    n = len(labels) - 1
    rows = [shapes[0], shapes[0][::2].copy()] + shapes[1:n]
    data = [{'points': r, 'normals': np.zeros_like(r), 'label': l} for r, l in zip(rows, labels)]
    assert labels[1] == 5
    with open(tmp_path / 'test.pkl', 'wb') as f:
        pickle.dump(data, f)
    return n


def test_reader_yields_the_reference_split(tmp_path):
    g, shapes = _gold()
    n = _write_pkl(tmp_path, g, shapes)
    cfg = make_cfg('modelnet')
    ds = ModelNetPairs(str(tmp_path), 'test', cfg, chunk_size=4)
    assert len(ds) == n
    seen = []
    for chunk in ds.chunks():
        assert len(chunk) <= 4
        for d in chunk:
            assert d['ref_points'].is_cuda and d['transform'].is_cuda and d['ref_feats'].shape == (717, 1)
            seen.append(d)
    for i, d in enumerate(seen):
        assert d['index'] == i and int(g['index'][i]) == i
        for k in ('ref_points', 'src_points', 'transform'):
            assert _ulps(d[k].cpu().numpy(), g[k][i]).max() <= 1
        assert torch.equal(ds[i]['ref_points'], d['ref_points'])
    cfg2 = copy.deepcopy(cfg)
    cfg2.test.class_indices = 'unseen'            # labels 0..7 are all 'seen'
    assert len(ModelNetPairs(str(tmp_path), 'test', cfg2)) == 0
    cfg3 = copy.deepcopy(cfg)
    cfg3.data.twice_transform = True
    with pytest.raises(NotImplementedError):
        ModelNetPairs(str(tmp_path), 'test', cfg3)


def test_validate_and_register_take_the_device_pairs(tmp_path, models):
    from geotransformer_b200.engine import RegistrationEngine
    from geotransformer_b200.model import create_model
    from geotransformer_b200.train import TrainingEngine
    from oracle import backbone_grad_oracle as BV
    g, shapes = _gold()
    _write_pkl(tmp_path, g, shapes)
    cfg, sd, _ = models('modelnet')
    cfg = copy.deepcopy(cfg)
    pairs = list(ModelNetPairs(str(tmp_path), 'test', cfg))
    # the fixture's pairs, written by the reference on the host, uploaded by the engine
    ones = np.ones((717, 1), np.float32)
    host = [{'ref_points': g['ref_points'][i], 'src_points': g['src_points'][i], 'ref_feats': ones, 'src_feats': ones,
             'transform': g['transform'][i]} for i in range(len(pairs))]
    for d, h in zip(pairs, host):
        assert all(np.array_equal(d[k].cpu().numpy(), h[k]) for k in ('ref_points', 'src_points', 'transform'))
    model = create_model(cfg)
    model.load_state_dict(sd, strict=True)
    eng = TrainingEngine(model.cuda(), cfg, BV.limits('modelnet717'))
    a, b = eng.validate(pairs), eng.validate(host)
    for x, y in zip(a, b):
        np.testing.assert_equal((x['metrics'], x['loss']), (y['metrics'], y['loss']))     # NaN-aware
        assert np.array_equal(np.asarray(x['estimated_transform']), np.asarray(y['estimated_transform']))
    reg = RegistrationEngine(eng.model, cfg, BV.limits('modelnet717'))
    try:
        c, d = reg.register(pairs), reg.register(host)
    finally:
        reg.close()
    for x, y in zip(c, d):
        assert np.array_equal(np.asarray(x['estimated_transform']), np.asarray(y['estimated_transform']))
    # the tester indexes the reader like any dataset
    from geotransformer_b200.tester import RegistrationTester
    tester = RegistrationTester(cfg, eng.model, BV.limits('modelnet717'), chunk=4, with_loss=True)
    try:
        summary, per_pair = tester.run(ModelNetPairs(str(tmp_path), 'test', cfg, chunk_size=4))
        ref_summary, ref_per_pair = tester.run(host)
    finally:
        tester.close()
    np.testing.assert_equal((summary, [p['metrics'] for p in per_pair]), (ref_summary, [p['metrics'] for p in ref_per_pair]))
    print('validate', [round(float(x['loss']['loss']), 4) for x in a])


def test_argument_errors_are_raised_before_any_launch():
    shapes = [np.zeros((100, 3), np.float32) + np.arange(100, dtype=np.float32)[:, None]]
    raw = torch.from_numpy(shapes[0]).cuda()
    lib = L.lib()
    torch.cuda.synchronize()
    n0 = lib.geob200_launch_count()
    for kwargs, msg in ((dict(indices=[-1]), 'indices'), (dict(indices=[1 << 32]), 'indices'), (dict(indices=[0, 1]), 'indices'),
                        (dict(m=0), 'num_points'), (dict(m=4097), 'num_points'), (dict(keep=0.0), 'keep_ratio'),
                        (dict(keep=float('nan')), 'keep_ratio'), (dict(noise=-1.0), 'magnitudes'), (dict(keep=0.001), 'keeps no point')):
        args = dict(indices=[0], m=64, keep=0.7, noise=0.05)
        args.update(kwargs)
        with pytest.raises(RuntimeError, match=msg):
            GF.modelnet_benchmark_pairs_batched(raw, [100], args['indices'], args['m'], args['keep'], 45.0, 0.5, args['noise'])
    with pytest.raises(RuntimeError, match='8192'):
        GF.modelnet_benchmark_pairs_batched(torch.zeros((8193, 3), device='cuda'), [8193], [0], 64, 0.7, 45.0, 0.5, 0.05)
    assert lib.geob200_launch_count() == n0
