"""Benchmark evaluation on the device (csrc/benchmark.cu, geotransformer_b200.evaluate) against numpy restatements, the golden values
of the reference's eval_one_epoch (tests/golden/eval_benchmark.npz) and the existing single-pair ops."""
import os
import re

import numpy as np
import pytest
import torch

from geotransformer_b200 import _lib as L
from geotransformer_b200 import evaluate as EV
from geotransformer_b200 import functional as GF
from geotransformer_b200.datasets import threedmatch_utils as TU
from oracle import eval_vectors as V

pytestmark = pytest.mark.gpu
GOLD = np.load(V.GOLD_PATH)
DEV = 'cuda'


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    return V.make_tree(str(tmp_path_factory.mktemp('bench')))


def _pack(rows, width=()):
    cap = max([len(r) for r in rows] + [1])
    out = np.zeros((len(rows), cap) + width, np.float32)
    for i, r in enumerate(rows):
        out[i, :len(r)] = r
    return torch.from_numpy(out).to(DEV), torch.tensor([len(r) for r in rows], dtype=torch.int32, device=DEV)


def test_order_and_select_equal_stable_argsort():
    rng = np.random.default_rng(3)
    cases = []
    s = rng.integers(0, 50, 6000).astype(np.float32)                 # heavy ties
    cases.append(s)
    s = rng.random(7000).astype(np.float32)
    s[rng.integers(0, 7000, 300)] = np.nan
    s[rng.integers(0, 7000, 50)] = -0.0
    s[rng.integers(0, 7000, 50)] = 0.0
    s[:3] = [np.inf, -np.inf, np.nan]
    cases.append(s)
    cases.append(rng.random(300).astype(np.float32))                  # n <= k
    cases.append(np.zeros(0, np.float32))                             # n = 0
    cases.append(rng.random(49152).astype(np.float32))               # LGR's capacity at the 3DMatch config
    s = rng.random(5003).astype(np.float32)
    s[np.argsort(-s, kind='stable')[4990:5010]] = 0.5                 # ties straddling k = 5000
    cases.append(s)
    pts = [rng.normal(size=(len(c), 3)).astype(np.float32) for c in cases]
    sc, cnt = _pack(cases)
    ref, _ = _pack(pts, (3,))
    src, _ = _pack([p * 2 for p in pts], (3,))
    kmax = 5000
    order = GF.corr_order_batched(sc, kmax, num_corr=cnt).cpu().numpy()
    for i, c in enumerate(cases):
        want = np.argsort(-c, kind='stable')[:kmax]
        assert np.array_equal(order[i, :len(want)], want) and (order[i, len(want):] == -1).all(), i
    for k in (250, 1000, 5000):
        r, s2, w, c2 = GF.corr_select_batched(ref, src, sc, GF.corr_order_batched(sc, max(k, 250), num_corr=cnt), k, num_corr=cnt)
        r, w, c2 = r.cpu().numpy(), w.cpu().numpy(), c2.cpu().numpy()
        for i, c in enumerate(cases):
            sel = np.argsort(-c, kind='stable')[:k] if len(c) > k else np.arange(len(c))
            assert c2[i] == len(sel)
            assert np.array_equal(r[i, :len(sel)], pts[i][sel])
            assert np.array_equal(w[i, :len(sel)].view(np.uint32), c[sel].view(np.uint32)), (i, k)
    # one pair alone gives the same rows as in the batch
    alone = GF.corr_order_batched(sc[1:2].contiguous(), kmax, num_corr=cnt[1:2].contiguous()).cpu().numpy()
    assert np.array_equal(alone[0], order[1])


def test_order_rejects_kmax_above_8192_before_any_launch():
    lib = L.lib()
    torch.cuda.synchronize()
    before = lib.geob200_launch_count()
    buf = torch.zeros(16, device=DEV)
    assert lib.geob200_corr_order_batched(buf.data_ptr(), 1, 16, None, 8193, buf.data_ptr(), None) < 0
    assert 'kmax' in lib.geob200_last_error().decode()
    assert lib.geob200_launch_count() == before
    with pytest.raises(ValueError):
        GF.corr_order_batched(buf.reshape(1, 16), 9000)


def _sparse_np(M, N, ref_idx, src_idx, gt):
    g = np.zeros((M, N))
    g[gt[:, 0], gt[:, 1]] = 1.0
    p = np.zeros_like(g)
    p[ref_idx, src_idx] = 1.0
    pos = g * p
    prec = pos.sum() / (p.sum() + 1e-12)
    rec = pos.sum() / (g.sum() + 1e-12)
    pos, g = pos > 0, g > 0
    hit = 0.5 * (np.any(pos, 1).sum() / (np.any(g, 1).sum() + 1e-12) + np.any(pos, 0).sum() / (np.any(g, 0).sum() + 1e-12))
    return np.array([prec, rec, hit])


@pytest.mark.parametrize('big', [False, True])
def test_sparse_eval_bit_identical_to_numpy(big):
    rng = np.random.default_rng(11 + big)
    pairs = []
    for i in range(7):
        M, N = (int(rng.integers(900, 1100)), int(rng.integers(900, 1100))) if big else (int(rng.integers(1, 80)), int(rng.integers(1, 80)))
        G = 0 if i == 2 else int(rng.integers(1, 3 * max(M, N)))
        gt = np.stack([rng.integers(0, M, G), rng.integers(0, N, G)], 1)
        P = 0 if i == 4 else int(rng.integers(1, 2 * max(M, N)))
        pred = np.stack([rng.integers(0, M, P), rng.integers(0, N, P)], 1)
        if G and P:
            pred[:P // 2] = gt[rng.integers(0, G, P // 2)]
        pairs.append((M, N, pred, gt))
    B = len(pairs)
    pcap, gcap = max(len(p[2]) for p in pairs) or 1, max(len(p[3]) for p in pairs) or 1
    pr, ps, gg = np.zeros((B, pcap), np.int64), np.zeros((B, pcap), np.int64), np.zeros((B, gcap, 2), np.int64)
    for b, (M, N, pred, gt) in enumerate(pairs):
        pr[b, :len(pred)], ps[b, :len(pred)], gg[b, :len(gt)] = pred[:, 0], pred[:, 1], gt
    t = lambda a: torch.from_numpy(a).to(DEV)
    pc = torch.tensor([len(p[2]) for p in pairs], dtype=torch.int32, device=DEV)
    gc = torch.tensor([len(p[3]) for p in pairs], dtype=torch.int32, device=DEV)
    m_cap, n_cap = max(p[0] for p in pairs), max(p[1] for p in pairs)
    if big:
        assert L.lib().geob200_sparse_correspondence_eval_batched_workspace_bytes(B, m_cap, n_cap) > 0      # global-memory bitmaps
    out = GF.sparse_correspondence_eval_batched(t(pr), t(ps), t(gg), m_cap, n_cap, pred_count=pc, gt_count=gc).cpu().numpy()
    for b, (M, N, pred, gt) in enumerate(pairs):
        assert np.array_equal(out[b], _sparse_np(M, N, pred[:, 0], pred[:, 1], gt)), b


def _tree_items(tree, config, benchmark=None):
    scenes = EV.discover(config, tree['features'] if config == '3dmatch' else tree['kitti'], benchmark)
    items = []
    for scene, files in scenes:
        gt = TU.get_gt_logs_and_infos(os.path.join(tree['gt_root'], benchmark, scene), 37) if config == '3dmatch' else None
        items += [EV._load(f, config, gt) for f in files]
    return items


def test_sparse_eval_and_registration_error_against_the_reference(tree):
    for config, bench, name in (('3dmatch', '3DMatch', '3DMatch_lgr'), ('3dmatch', '3DLoMatch', '3DLoMatch_lgr'), ('kitti', None, 'kitti_lgr')):
        items = _tree_items(tree, config, bench)
        res = EV.evaluate(config, 'lgr', tree['features'] if config == '3dmatch' else tree['kitti'], benchmark=bench, gt_root=tree['gt_root'],
                          chunk=5)[None]['pairs']
        sparse, reg, terr = GOLD[f'{name}/sparse'], GOLD[f'{name}/reg'], GOLD[f'{name}/terr']
        for i, (it, v) in enumerate(zip(items, res)):
            assert np.array_equal([v['precision'], v['recall'], v['hit_ratio']], sparse[i]), (name, i)
            if not np.isnan(reg[i, 0]):
                # the reference's rre is fp32 arccos of an fp32 trace: a few ulp of x = cos(rre) near 1 move it by ~ulp / sin(rre)
                tol = 1e-4 + np.degrees(8 * 2.0 ** -24 / np.sin(np.radians(max(reg[i, 0], 0.05))))
                assert abs(v['rre'] - reg[i, 0]) <= tol and abs(v['rte'] - reg[i, 1]) <= 1e-6 * max(1.0, reg[i, 1]), \
                    (name, i, v['rre'], v['rte'], reg[i])
                want = V._rre_rte(it['reg_gt'].astype(np.float64), it['estimated_transform'].astype(np.float64))
                assert abs(v['rre'] - want[0]) <= 1e-9 and abs(v['rte'] - want[1]) <= 1e-12, (name, i)   # the double restatement
            if config == '3dmatch':
                assert np.isnan(terr[i]) == (not it['has_cov'])
                if it['has_cov']:
                    assert abs(v['error'] - terr[i]) <= 1e-5 * abs(terr[i]) + 1e-9, (name, i, v['error'], terr[i])
                    assert v['accepted'] == (terr[i] < 0.04)
                else:
                    assert v['accepted'] is None                   # absent from gt.log or adjacent: never in the recall
            else:
                assert v['accepted'] == (reg[i, 0] < 5.0 and reg[i, 1] < 2.0)


def test_procrustes_counts_bit_identical_to_weighted_procrustes():
    rng = np.random.default_rng(5)
    ns = [3, 40, 1000, 1, 777]
    src = [rng.normal(size=(n, 3)).astype(np.float32) for n in ns]
    R = V._rotation(rng, 30)
    ref = [(s @ R.T + 0.5 + rng.normal(scale=0.01, size=s.shape)).astype(np.float32) for s in src]
    w = [rng.random(n).astype(np.float32) for n in ns]
    S, cnt = _pack(src, (3,))
    Rf, _ = _pack(ref, (3,))
    W, _ = _pack(w)
    got = GF.weighted_procrustes_counts(S, Rf, W, cnt).cpu()
    for b in range(len(ns)):
        want = GF.weighted_procrustes(torch.from_numpy(src[b])[None].to(DEV), torch.from_numpy(ref[b])[None].to(DEV),
                                      torch.from_numpy(w[b])[None].to(DEV)).cpu()
        assert torch.equal(got[b], want[0]), b


def _same_lines(got, want):
    """equal line for line; RRE / RTE fields may differ by one unit of the last printed digit (the reference computes them in
    float32, this driver in double: DESIGN.md section 3b)"""
    got = [f'{"INFO" if lv == 20 else "CRITICAL"}\t{m}' for lv, m in got]
    assert len(got) == len(want)
    for a, b in zip(got, want):
        if a == b:
            continue
        fa, fb = re.split(r'(RRE: |RTE: )(-?[0-9.]+|nan)', a), re.split(r'(RRE: |RTE: )(-?[0-9.]+|nan)', str(b))
        assert len(fa) == len(fb), (a, b)
        for i, (x, y) in enumerate(zip(fa, fb)):
            if i % 3 == 2:
                assert abs(float(x) - float(y)) <= 1.0001e-3, (a, b)
            else:
                assert x == y, (a, b)


def test_driver_lgr_matches_the_reference(tree, tmp_path):
    for bench in ('3DMatch', '3DLoMatch'):
        name = f'{bench}_lgr'
        out = EV.evaluate('3dmatch', 'lgr', tree['features'], benchmark=bench, gt_root=tree['gt_root'], registration_dir=str(tmp_path),
                          verbose=True)[None]
        corr = GOLD[f'{name}/corr']
        for i, v in enumerate(out['pairs']):
            assert v['num_corr'] == int(corr[i, 3])
            assert abs(v['overlap'] - corr[i, 0]) <= 1e-6 and abs(v['inlier_ratio'] - corr[i, 1]) <= 1e-6
            assert abs(v['residual'] - corr[i, 2]) <= 1e-6 * max(1.0, corr[i, 2])
        assert [f'{"INFO" if lv == 20 else "CRITICAL"}\t{m}' for lv, m in out['lines']] == list(GOLD[f'{name}/lines'])   # exact
        for scene in V.SCENES:
            assert open(os.path.join(tmp_path, bench, scene, 'est.log'), 'rb').read() == GOLD[f'{name}/estlog/{scene}'].tobytes()
    for k, name in ((None, 'kitti_lgr'), (1000, 'kitti_lgr_k1000')):
        out = EV.evaluate('kitti', 'lgr', tree['kitti'], num_corr=None if k is None else str(k), verbose=True)[k]
        _same_lines(out['lines'], list(GOLD[f'{name}/lines']))


def test_driver_svd_matches_the_reference_svd(tree):
    runs = [('3dmatch', '3DMatch', None, '3DMatch_svd', 1.5), ('kitti', None, None, 'kitti_svd', 30.0), ('kitti', None, '1000', 'kitti_svd_k1000', 30.0)]
    for config, bench, k, name, scale in runs:
        root = tree['features'] if config == '3dmatch' else tree['kitti']
        out = EV.evaluate(config, 'svd', root, benchmark=bench, gt_root=tree['gt_root'], num_corr=k)
        pairs = next(iter(out.values()))['pairs']
        want = GOLD[f'{name}/est']
        for i, v in enumerate(pairs):
            assert np.abs(v['estimated_transform'] - want[i]).max() <= 1e-5 * scale, (name, i)


def test_driver_ransac_equals_the_single_pair_op(tree):
    from geotransformer_b200.config import make_cfg
    res = EV.evaluate('kitti', 'ransac', tree['kitti'], num_corr='1000', chunk=4)[1000]['pairs']
    items = _tree_items(tree, 'kitti')
    for pid, (it, v) in enumerate(zip(items, res)):
        s = it['corr_scores']
        sel = np.argsort(-s, kind='stable')[:1000] if len(s) > 1000 else np.arange(len(s))
        src = torch.from_numpy(it['src_corr_points'][sel]).to(DEV)
        ref = torch.from_numpy(it['ref_corr_points'][sel]).to(DEV)
        c = make_cfg('kitti').ransac
        want = GF.ransac_correspondences(src, ref, c.distance_threshold, c.num_points, c.num_iterations, seed=c.seed, pair=pid)['transform']
        assert np.array_equal(v['estimated_transform'].astype(np.float32), want.cpu().numpy()), pid


def test_sweep_and_chunking_do_not_change_results(tree):
    def strip(pairs):          # repr: NaN entries (no covariance on KITTI) compare equal
        return repr([{k: (x.tolist() if isinstance(x, np.ndarray) else x) for k, x in p.items()} for p in pairs])
    for method in ('ransac', 'svd'):
        both = EV.evaluate('kitti', method, tree['kitti'], num_corr='250,1000', chunk=64)
        for k in (250, 1000):
            alone = EV.evaluate('kitti', method, tree['kitti'], num_corr=str(k), chunk=1)[k]
            assert strip(both[k]['pairs']) == strip(alone['pairs'])
            assert repr(both[k]['summary']) == repr(alone['summary'])


def test_tester_kitti_layout_feeds_the_driver(tmp_path):
    from geotransformer_b200.config import make_cfg
    from geotransformer_b200.model import create_model
    from geotransformer_b200.synth import make_pair
    from geotransformer_b200.tester import RegistrationTester
    from geotransformer_b200.weights import synthetic_state_dict
    from geotransformer_b200.utils.registration import evaluate_sparse_correspondences
    cfg = make_cfg('3dmatch')
    model = create_model(cfg)
    model.load_state_dict(synthetic_state_dict(model, 7351), strict=True)
    model = model.cuda().eval()
    data = []
    for i in range(2):
        p = make_pair('demo2k', i)
        d = {k: p[k] for k in ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')}
        d.update(seq_id=3, ref_frame=10 + i, src_frame=i, scene_name='7-scenes-redkitchen', overlap=np.float32(0.5))
        data.append(d)
    files = {}
    for layout in ('3dmatch', 'kitti'):
        t = RegistrationTester(cfg, model, cfg.neighbor_limits, output_dir=str(tmp_path / layout), num_streams=1, layout=layout)
        _, per_pair = t.run(data)
        t.close()
        files[layout] = [p['file'] for p in per_pair]
    assert [os.path.basename(f) for f in files['kitti']] == ['3_0_10.npz', '3_1_11.npz']
    for a, b in zip(files['3dmatch'], files['kitti']):
        da, db = np.load(a), np.load(b)
        assert set(da.files) - set(db.files) == {'overlap'}
        for k in db.files:
            assert np.array_equal(da[k], db[k]), k
    res = EV.evaluate('kitti', 'lgr', str(tmp_path / 'kitti'))[None]['pairs']
    for f, v in zip(files['3dmatch'], res):
        d = np.load(f)
        want = evaluate_sparse_correspondences(d['ref_points_c'], d['src_points_c'], d['ref_node_corr_indices'], d['src_node_corr_indices'],
                                               d['gt_node_corr_indices'])
        assert v['precision'] == want['precision'] and v['recall'] == want['recall']
        assert np.array_equal(v['estimated_transform'], d['estimated_transform'])
