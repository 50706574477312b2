"""Descriptor nearest neighbours and the feature-matching RANSAC on the device against the reference fixture
(tests/golden/feature_match.npz) and the numpy restatement (oracle/feature_ransac_oracle.py)."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from oracle import feature_match_vectors as V
from oracle import feature_ransac_oracle as FO
from oracle import ransac_oracle as RO

pytestmark = pytest.mark.gpu

GOLD = np.load(V.GOLD_PATH)


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _check_nn(q, s, idx, dist):
    want_d, want_i = FO.nearest_neighbor(q, s)
    assert np.array_equal(idx, want_i)
    assert np.all(np.abs(dist - want_d) <= 1e-12 * np.maximum(want_d, 1e-300))


@pytest.mark.parametrize('name', list(V.CASES))
def test_nearest_neighbor_equals_fixture_and_fp64_brute_force(name):
    from geotransformer_b200 import functional as GF
    q, s = V.inputs(name)
    qi, qd, si, sd = (v.cpu().numpy() for v in GF.feature_nearest_neighbor(_cuda(q), _cuda(s), bidirectional=True))
    assert np.array_equal(qi, GOLD[f'{name}/nn_index'])
    assert np.all(np.abs(qd - GOLD[f'{name}/nn_dist']) <= 1e-12 * np.maximum(GOLD[f'{name}/nn_dist'], 1e-300))
    _check_nn(q, s, qi, qd)
    _check_nn(s, q, si, sd)


@pytest.mark.parametrize('C', [3, 32, 256, 1000])
def test_ragged_batch_both_directions(C):
    """row counts off the 64-row tile, 1-row clouds, rows past the count (-1 / NaN), channel counts off the 32-channel chunk"""
    from geotransformer_b200 import functional as GF
    rng = np.random.default_rng(C)
    sizes = [(1, 1), (65, 130), (200, 63), (129, 1), (1, 97)]
    cq, cs = max(a for a, _ in sizes), max(b for _, b in sizes)
    Q = np.zeros((len(sizes), cq, C), np.float32)
    S = np.zeros((len(sizes), cs, C), np.float32)
    for p, (a, b) in enumerate(sizes):
        Q[p, :a] = rng.normal(size=(a, C))
        S[p, :b] = rng.normal(size=(b, C))
    nq = torch.tensor([a for a, _ in sizes], dtype=torch.int32, device='cuda')
    ns = torch.tensor([b for _, b in sizes], dtype=torch.int32, device='cuda')
    qi, qd, si, sd = (v.cpu().numpy() for v in GF.feature_nearest_neighbor_batched(_cuda(Q), _cuda(S), nq, ns, bidirectional=True))
    for p, (a, b) in enumerate(sizes):
        _check_nn(Q[p, :a], S[p, :b], qi[p, :a], qd[p, :a])
        _check_nn(S[p, :b], Q[p, :a], si[p, :b], sd[p, :b])
        assert np.all(qi[p, a:] == -1) and np.all(np.isnan(qd[p, a:]))
        assert np.all(si[p, b:] == -1) and np.all(np.isnan(sd[p, b:]))


def test_exact_ties_and_crowded_bands():
    """exact duplicates: the lowest index; rows with more than 8 supports inside the screening band: the fp64 fallback scan"""
    from geotransformer_b200 import functional as GF
    rng = np.random.default_rng(5)
    C = 32
    s = rng.normal(size=(300, C)).astype(np.float32)
    s[250:260] = s[40]                                          # exact ties with row 40
    q = np.concatenate([s[40:41] + np.float32(1e-3), rng.normal(size=(20, C)).astype(np.float32)])
    # a crowded row: 40 supports at distance ~1 from the query, differing in the last bits only
    base = rng.normal(size=C)
    base /= np.linalg.norm(base)
    crowd = np.tile(base, (40, 1)) + rng.normal(size=(40, C)) * 1e-7
    s[100:140] = crowd.astype(np.float32)
    q = np.concatenate([q, np.zeros((1, C), np.float32)])
    qi, qd = (v.cpu().numpy() for v in GF.feature_nearest_neighbor(_cuda(q), _cuda(s)))
    _check_nn(q, s, qi, qd)
    assert qi[0] == 40
    assert 100 <= qi[-1] < 140


def test_mutual_and_bilateral_equal_the_reference():
    from geotransformer_b200.utils.pointcloud import get_nearest_neighbor
    from geotransformer_b200.utils.registration import extract_corr_indices_from_feats, extract_correspondences_from_feats
    for name in V.CASES:
        ref, src = V.inputs(name)
        d, i = get_nearest_neighbor(ref, src, return_index=True)
        assert d.dtype == np.float64 and i.dtype == np.int64 and np.array_equal(i, GOLD[f'{name}/nn_index'])
        for mode in V.MODES:
            r, c = extract_corr_indices_from_feats(ref, src, mutual=mode == 'mutual', bilateral=mode == 'bilateral')
            assert r.dtype == np.int64 and c.dtype == np.int64
            assert np.array_equal(r, GOLD[f'{name}/{mode}/ref']) and np.array_equal(c, GOLD[f'{name}/{mode}/src']), (name, mode)
            rt, ct = extract_corr_indices_from_feats(_cuda(ref), _cuda(src), mutual=mode == 'mutual', bilateral=mode == 'bilateral')
            assert rt.is_cuda and np.array_equal(rt.cpu().numpy(), r) and np.array_equal(ct.cpu().numpy(), c)
        rng = np.random.default_rng(1)
        rp, sp = rng.normal(size=(len(ref), 3)).astype(np.float32), rng.normal(size=(len(src), 3)).astype(np.float32)
        for mutual in (False, True):
            a, b, fd = extract_correspondences_from_feats(rp, sp, ref, src, mutual=mutual, return_feat_dist=True)
            r, c = GOLD[f'{name}/{"mutual" if mutual else "plain"}/ref'], GOLD[f'{name}/{"mutual" if mutual else "plain"}/src']
            assert np.array_equal(a, rp[r]) and np.array_equal(b, sp[c])
            want = np.linalg.norm(ref[r] - src[c], axis=1)
            assert fd.dtype == np.float32 and np.allclose(fd, want, rtol=1e-5, atol=1e-7)
            at, bt, fdt = extract_correspondences_from_feats(_cuda(rp), _cuda(sp), _cuda(ref), _cuda(src), mutual=mutual, return_feat_dist=True)
            assert np.array_equal(at.cpu().numpy(), a) and np.array_equal(bt.cpu().numpy(), b) and np.array_equal(fdt.cpu().numpy(), fd)
    with pytest.raises(RuntimeError):
        get_nearest_neighbor(torch.zeros(4, 3), torch.zeros(4, 3))


def _synthetic(n_src, n_ref, wrong, rng, C=32, noise=0.002, scale=2.0):
    """src points, ref = R src + t on a shuffled order (+ extra ref points); descriptors: ref rows carry a unit code per point, a
    right src row its partner's code plus noise, a wrong src row a random code (so its match is some random ref point)"""
    R = Rotation.random(random_state=rng).as_matrix()
    t = rng.normal(size=3) * scale * 0.5
    src = rng.uniform(-1, 1, size=(n_src, 3)) * scale
    perm = rng.permutation(n_ref)
    ref = rng.uniform(-1, 1, size=(n_ref, 3)) * scale @ R.T + t
    ref[perm[:n_src]] = src @ R.T + t + rng.normal(size=(n_src, 3)) * noise
    code = rng.normal(size=(n_ref, C))
    code /= np.linalg.norm(code, axis=1, keepdims=True)
    sf = code[perm[:n_src]] + rng.normal(size=(n_src, C)) * 0.05 / np.sqrt(C)
    bad = rng.random(n_src) < wrong
    sf[bad] = rng.normal(size=(int(bad.sum()), C))
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return (src.astype(np.float32), ref.astype(np.float32), sf.astype(np.float32), code.astype(np.float32), T)


def _batch(pairs):
    B = len(pairs)
    cs, cr, C = max(len(p[0]) for p in pairs), max(len(p[1]) for p in pairs), pairs[0][2].shape[1]
    out = [np.zeros((B, cs, 3), np.float32), np.zeros((B, cr, 3), np.float32), np.zeros((B, cs, C), np.float32),
           np.zeros((B, cr, C), np.float32)]
    for b, p in enumerate(pairs):
        for k in range(4):
            out[k][b, :len(p[k])] = p[k]
    ns = torch.tensor([len(p[0]) for p in pairs], dtype=torch.int32, device='cuda')
    nr = torch.tensor([len(p[1]) for p in pairs], dtype=torch.int32, device='cuda')
    return [_cuda(x) for x in out] + [ns, nr]


def _rre_rte(T_gt, T):
    T = np.asarray(T, np.float64)
    R = T_gt[:3, :3].T @ T[:3, :3]
    return np.degrees(np.arccos(np.clip((np.trace(R) - 1) / 2, -1, 1))), np.linalg.norm(T_gt[:3, 3] - T[:3, 3])


def test_records_match_the_restatement():
    """samples, matches, pass flags, validated ids and inlier counts equal the restatement's (which scores the device's own
    validated transforms); rmse within 1e-6 relative; the winner is the best slot under the stated order.  The pass flags of the
    distance check compare double residuals with tau: they could differ only for a residual within ~1e-15 of tau."""
    from geotransformer_b200 import functional as GF
    rng = np.random.default_rng(17)
    pairs = [_synthetic(a, b, w, rng)[:4] for a, b, w in ((600, 700, 0.5), (333, 420, 0.7), (900, 900, 0.6))]
    sp, rp, sf, rf, ns, nr = _batch(pairs)
    tau, rn, I, Vv, seed = 0.05, 3, 3000, 40, 0xfeed_5eed
    res = GF.ransac_features_batched(sp, rp, sf, rf, tau, rn, I, Vv, seed=seed, num_src=ns, num_ref=nr, records=True)
    rec = {k: v.cpu().numpy() for k, v in res.items()}
    for p, (s, r, a, b) in enumerate(pairs):
        nv = int(rec['num_validated'][p])
        Tv = rec['val_transforms'][p, :nv]
        want = FO.ransac_features(s, r, a, b, tau, rn, I, Vv, seed=seed, pair=p, transforms=Tv)
        assert np.array_equal(rec['matches'][p, :len(s)], want['matches'])
        assert np.array_equal(rec['samples'][p], want['samples'])
        assert np.array_equal(rec['pass_flags'][p].astype(bool), want['pass_flags'])
        assert nv == want['num_validated'] and nv > 0
        assert np.array_equal(rec['val_ids'][p, :nv], want['val_ids']) and np.all(rec['val_ids'][p, nv:] == -1)
        assert np.array_equal(rec['val_inliers'][p, :nv], want['counts'])
        rm, wr = rec['val_rmse'][p, :nv].astype(np.float64), want['rmse'].astype(np.float64)
        assert np.all(np.abs(rm - wr) <= 1e-6 * np.maximum(wr, 1e-30))
        best = RO.winner(rec['val_inliers'][p, :nv], rec['val_rmse'][p, :nv])
        assert rec['iteration'][p] == rec['val_ids'][p, best] and rec['inliers'][p] == rec['val_inliers'][p, best]
        assert np.array_equal(rec['transform'][p], rec['val_transforms'][p, best])
        assert rec['fitness'][p] == np.float32(rec['inliers'][p] / len(s)) and rec['inlier_rmse'][p] == rec['val_rmse'][p, best]
        # the device's Kabsch agrees with the restatement's float64 SVD on the validated samples
        for k in range(nv):
            idx = want['samples'][want['val_ids'][k]]
            if len(set(idx)) < rn or np.linalg.svd(s[idx] - s[idx].mean(0), compute_uv=False)[1] < 0.2:
                continue                                        # degenerate sample: the rotation is not unique
            R64, t64 = want['hyps'][k]
            assert np.abs(Tv[k, :3, :3] - R64).max() <= 1e-5 and np.abs(Tv[k, :3, 3] - t64).max() <= 1e-5 * max(1.0, np.abs(t64).max())


@pytest.mark.parametrize('wrong', [0.5, 0.8])
def test_recovers_synthetic_transforms(wrong):
    """50 % and 80 % wrong matches at the reference defaults (tau 0.05, 3 points, 50 000 iterations, 1 000 validations)"""
    from geotransformer_b200 import functional as GF
    rng = np.random.default_rng(int(wrong * 10))
    s, r, a, b, T = _synthetic(3000, 3500, wrong, rng)
    res = GF.ransac_features(_cuda(s), _cuda(r), _cuda(a), _cuda(b), 0.05, 3, 50000, 1000)
    rre, rte = _rre_rte(T, res['transform'].cpu().numpy())
    assert rre < 1.0 and rte < 0.05, (rre, rte)
    assert 0 < int(res['num_validated']) <= 1000 and float(res['fitness']) > 0.9 * (1 - wrong)


def test_alone_equals_batch_and_runs_are_identical():
    from geotransformer_b200 import functional as GF
    rng = np.random.default_rng(23)
    pairs = [_synthetic(a, b, 0.6, rng)[:4] for a, b in ((500, 640), (2, 50), (900, 1200), (1, 1), (700, 700))]
    sp, rp, sf, rf, ns, nr = _batch(pairs)
    args = (0.05, 3, 4000, 200)
    x = GF.ransac_features_batched(sp, rp, sf, rf, *args, seed=7, num_src=ns, num_ref=nr)
    y = GF.ransac_features_batched(sp, rp, sf, rf, *args, seed=7, num_src=ns, num_ref=nr)
    for k in x:
        assert torch.equal(x[k], y[k]), k
    for p, (s, r, a, b) in enumerate(pairs):
        one = GF.ransac_features(_cuda(s), _cuda(r), _cuda(a), _cuda(b), *args, seed=7, pair=p)
        for k in x:
            assert torch.equal(one[k], x[k][p]), (p, k)
    assert int(x['iteration'][1]) == -1 and int(x['num_validated'][1]) == 0          # 2 src points < ransac_n
    assert float(x['fitness'][0]) > 0.3 and float(x['fitness'][4]) > 0.3


def test_default_results_on_the_device():
    from geotransformer_b200 import functional as GF
    rng = np.random.default_rng(2)
    s, r, a, b, _ = _synthetic(100, 100, 0.0, rng)
    for args in ((0.05, 2, 100, 10), (0.0, 3, 100, 10), (0.05, 3, 0, 10), (0.05, 3, 100, 0)):
        res = GF.ransac_features(_cuda(s), _cuda(r), _cuda(a), _cuda(b), *args)
        assert torch.equal(res['transform'].cpu(), torch.eye(4)) and float(res['fitness']) == 0.0 and int(res['iteration']) == -1
        assert int(res['num_validated']) == 0 and float(res['inlier_rmse']) == 0.0
    # nothing validates: the ref cloud is 3x the src cloud, so every edge fails the 0.9 check
    res = GF.ransac_features(_cuda(s), _cuda(r * 3), _cuda(a), _cuda(b), 0.05, 3, 200, 10, records=True)
    assert int(res['num_validated']) == 0 and int(res['iteration']) == -1 and int(res['pass_flags'].sum()) == 0


def test_open3d_drop_in_on_fine_features(models):
    """registration_with_ransac_from_feats on ref_feats_f / src_feats_f of a demo2k forward: numpy in gives a float64 (4, 4) array
    equal to the CUDA-tensor call's float32 device tensor"""
    from geotransformer_b200.synth import make_pair
    from geotransformer_b200.utils.data import registration_collate_fn_stack_mode
    from geotransformer_b200.utils.open3d import registration_with_ransac_from_feats
    cfg, _, model = models('3dmatch')
    model = model.cuda().eval()
    pair = make_pair('demo2k', 0)
    dd = {k: pair[k] for k in ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')}
    data = registration_collate_fn_stack_mode([dd], cfg.backbone.num_stages, cfg.backbone.init_voxel_size, cfg.backbone.init_radius,
                                              cfg.neighbor_limits)
    with torch.no_grad():
        out = model(data)
    keys = ('src_points_f', 'ref_points_f', 'src_feats_f', 'ref_feats_f')
    T_dev = registration_with_ransac_from_feats(*(out[k] for k in keys), distance_threshold=0.05, num_iterations=5000, val_iterations=200)
    assert T_dev.is_cuda and T_dev.dtype == torch.float32 and T_dev.shape == (4, 4)
    T_np = registration_with_ransac_from_feats(*(out[k].cpu().numpy() for k in keys), distance_threshold=0.05, num_iterations=5000,
                                               val_iterations=200)
    assert isinstance(T_np, np.ndarray) and T_np.dtype == np.float64 and np.array_equal(T_np, T_dev.cpu().numpy().astype(np.float64))
    R = T_np[:3, :3]
    assert np.abs(R @ R.T - np.eye(3)).max() < 1e-4
    with pytest.raises(RuntimeError):
        registration_with_ransac_from_feats(*(out[k].cpu() for k in keys))
