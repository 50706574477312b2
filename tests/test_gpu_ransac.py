"""Correspondence RANSAC and correspondence metrics on the device against the numpy restatement (oracle/ransac_oracle.py)."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from oracle import ransac_oracle as RO

pytestmark = pytest.mark.gpu


def _synthetic(n, inlier_ratio, rng, noise=0.0, scale=1.0):
    R = Rotation.random(random_state=rng).as_matrix()
    t = rng.normal(size=3) * scale
    src = (rng.uniform(-1, 1, size=(n, 3)) * scale).astype(np.float32)
    ref = (src.astype(np.float64) @ R.T + t + rng.normal(size=(n, 3)) * noise).astype(np.float32)
    out = rng.random(n) >= inlier_ratio
    ref[out] = (rng.uniform(-1, 1, size=(int(out.sum()), 3)) * scale + t).astype(np.float32)
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return src, ref, T


def _batch(pairs, cap):
    B = len(pairs)
    src = np.zeros((B, cap, 3), np.float32)
    ref = np.zeros((B, cap, 3), np.float32)
    for p, (s, r) in enumerate(pairs):
        src[p, :len(s)], ref[p, :len(r)] = s, r
    cnt = torch.tensor([len(s) for s, _ in pairs], dtype=torch.int32, device='cuda')
    return torch.from_numpy(src).cuda(), torch.from_numpy(ref).cuda(), cnt


def _rre_rte(T_gt, T):
    R = T_gt[:3, :3].T @ np.asarray(T, np.float64)[:3, :3]
    rre = np.degrees(np.arccos(np.clip((np.trace(R) - 1) / 2, -1, 1)))
    return rre, np.linalg.norm(T_gt[:3, 3] - np.asarray(T, np.float64)[:3, 3])


def test_sampler_scoring_and_winner_match_the_oracle():
    """per-hypothesis records: the device's samples are the oracle's bit for bit; the oracle scores the device's own (R, t) to the
    same inlier counts (rmse within 1e-6 relative); the winner is the records' best under the stated rule; on well-conditioned
    samples the device Kabsch agrees with a float64 SVD Kabsch within 1e-5"""
    from geotransformer_b200 import functional as GF
    rng = np.random.default_rng(11)
    pairs = [_synthetic(n, r, rng, noise=0.004, scale=2.0)[:2] for n, r in ((1500, 0.3), (777, 0.5), (2100, 0.1))]
    src, ref, cnt = _batch(pairs, 2200)
    tau, rn, I, seed = 0.05, 3, 600, 0x1234_5678_9abc_def0
    res = GF.ransac_correspondences_batched(src, ref, tau, rn, I, seed=seed, num_corr=cnt, records=True)
    torch.cuda.synchronize()
    rec = {k: v.cpu().numpy() for k, v in res.items()}
    worst_rmse, worst_kabsch, checked = 0.0, 0.0, 0
    for p, (s, r) in enumerate(pairs):
        n = len(s)
        idx = RO.sample_indices(seed, p, n, rn, I)
        assert np.array_equal(rec['hyp_samples'][p], idx), f'pair {p}: samples differ'
        for i in range(I):
            Tdev = rec['hyp_transforms'][p, i]
            c, rm = RO.score(Tdev[:3, :3], Tdev[:3, 3], s, r, tau)
            assert c == rec['hyp_inliers'][p, i], (p, i, c, rec['hyp_inliers'][p, i])
            worst_rmse = max(worst_rmse, abs(float(rm) - float(rec['hyp_rmse'][p, i])) / max(float(rm), 1e-30))
            sv = np.linalg.svd(s[idx[i]] - s[idx[i]].mean(0), compute_uv=False)
            if len(set(idx[i])) == rn and sv[1] > 0.2:
                R64, t64 = RO.kabsch(s[idx[i]], r[idx[i]])
                worst_kabsch = max(worst_kabsch, np.abs(Tdev[:3, :3] - R64).max(), np.abs(Tdev[:3, 3] - t64).max() / max(1.0, np.abs(t64).max()))
                checked += 1
        best = RO.winner(rec['hyp_inliers'][p], rec['hyp_rmse'][p])
        assert rec['iteration'][p] == best and rec['inliers'][p] == rec['hyp_inliers'][p, best]
        assert np.array_equal(rec['transform'][p], rec['hyp_transforms'][p, best])
        assert rec['inlier_rmse'][p] == rec['hyp_rmse'][p, best]
        assert rec['fitness'][p] == np.float32(rec['inliers'][p] / n)
    assert worst_rmse <= 1e-6, worst_rmse
    assert checked > 500 and worst_kabsch <= 1e-5, (checked, worst_kabsch)


@pytest.mark.parametrize('config,ratio', [('3dmatch', 0.25), ('3dmatch', 0.5), ('kitti', 0.15), ('kitti', 0.5)])
def test_recovers_synthetic_transforms(config, ratio):
    """at the reference configs: RRE < 1 deg, RTE < tau / 2; the fitness is the oracle's for the same transform.
    The lowest inlier ratios are the ones the configs can meet: an all-inlier sample needs ratio^n * I >> 1, i.e. about 10
    expected clean samples at 0.22 (3DMatch: 3 points, 1 000 iterations) and 0.12 (KITTI: 4 points, 50 000 iterations).  At 5 %
    inliers the expectation is 0.125 and 0.3 clean samples, so no RANSAC at these configs recovers such a pair reliably."""
    from geotransformer_b200 import functional as GF
    from geotransformer_b200.config import make_cfg
    rc = make_cfg(config).ransac
    scale, noise = (2.0, 0.005) if config == '3dmatch' else (20.0, 0.03)
    rng = np.random.default_rng(int(ratio * 100) + len(config))
    s, r, T = _synthetic(3000, ratio, rng, noise=noise, scale=scale)
    res = GF.ransac_correspondences(torch.from_numpy(s).cuda(), torch.from_numpy(r).cuda(), rc.distance_threshold, rc.num_points,
                                    rc.num_iterations, seed=rc.seed)
    Tdev = res['transform'].cpu().numpy()
    rre, rte = _rre_rte(T, Tdev)
    assert rre < 1.0 and rte < rc.distance_threshold / 2, (rre, rte)
    c, _ = RO.score(Tdev[:3, :3], Tdev[:3, 3], s, r, rc.distance_threshold)
    assert int(res['inliers']) == c and float(res['fitness']) == float(np.float32(c / len(s)))


def test_deterministic_and_batch_independent():
    """same seed: bit-identical; a ragged batch (0, 1, ransac_n - 1 correspondences, full capacity) equals single-pair calls"""
    from geotransformer_b200 import functional as GF
    rng = np.random.default_rng(3)
    cap, rn, I, tau = 1500, 4, 2000, 0.3
    sizes = [0, 1, rn - 1, 640, cap, 37]
    pairs = [_synthetic(n, 0.4, rng, noise=0.02, scale=10.0)[:2] for n in sizes]
    src, ref, cnt = _batch(pairs, cap)
    a = GF.ransac_correspondences_batched(src, ref, tau, rn, I, seed=99, num_corr=cnt)
    b = GF.ransac_correspondences_batched(src, ref, tau, rn, I, seed=99, num_corr=cnt)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    for p, n in enumerate(sizes):
        one = GF.ransac_correspondences(src[p, :max(n, 1)].contiguous(), ref[p, :max(n, 1)].contiguous(), tau, rn, I, seed=99, pair=p,
                                        num_corr=cnt[p:p + 1])
        for k in a:
            assert torch.equal(one[k], a[k][p]), (p, k)
        if n < rn:
            assert torch.equal(a['transform'][p], torch.eye(4, device='cuda')) and float(a['fitness'][p]) == 0.0
            assert int(a['iteration'][p]) == -1 and float(a['inlier_rmse'][p]) == 0.0
    assert float(a['fitness'][4]) > 0.3


def test_correspondence_metrics_match_the_restatement():
    from geotransformer_b200 import functional as GF
    rng = np.random.default_rng(8)
    pairs, Ts = [], []
    for n in (900, 0, 1, 2500):
        s, r, T = _synthetic(n, 0.4, rng, noise=0.03, scale=1.5)
        pairs.append((s, r))
        Ts.append(T.astype(np.float32))
    # residuals exactly at the radius: src = ref - (0.1, 0, 0) under the identity
    r = rng.uniform(-1, 1, size=(64, 3)).astype(np.float32)
    s = r.copy()
    s[:, 0] = r[:, 0] - np.float32(0.1)
    pairs.append((s, r))
    Ts.append(np.eye(4, dtype=np.float32))
    src, ref, cnt = _batch(pairs, 2500)
    out = GF.correspondence_metrics_batched(ref, src, torch.from_numpy(np.stack(Ts)).cuda(), 0.1, num_corr=cnt).cpu().numpy()
    for p, ((s, r), T) in enumerate(zip(pairs, Ts)):
        ir, ov, rs, nu, nn = RO.correspondence_metrics(r, s, T, 0.1)
        assert out[p, 3] == nu
        if nu == 0:
            assert np.isnan(out[p, :3]).all()
            continue
        # counts may differ only where the float64 distance lies within 1e-6 relative of the radius
        res = np.linalg.norm(r.astype(np.float64) - (s.astype(np.float64) @ T[:3, :3].T.astype(np.float64) + T[:3, 3]), axis=1)
        near_res, near_nn = int(np.sum(np.abs(res - 0.1) <= 1e-7)), int(np.sum(np.abs(nn - 0.1) <= 1e-7))
        assert abs(out[p, 0] - ir) <= near_res / nu + 1e-6, (p, out[p, 0], ir, near_res)
        assert abs(out[p, 1] - ov) <= near_nn / nu + 1e-6, (p, out[p, 1], ov, near_nn)
        assert abs(out[p, 2] - rs) <= 1e-6 * max(1.0, rs), (p, out[p, 2], rs)


def test_open3d_drop_in():
    """numpy in: float64 (4, 4) equal to the functional op; the index form equals a pre-gathered call"""
    from geotransformer_b200 import functional as GF
    from geotransformer_b200.utils.open3d import registration_with_ransac_from_correspondences as ransac_o3d
    rng = np.random.default_rng(21)
    s, r, _ = _synthetic(800, 0.5, rng, noise=0.003, scale=1.0)
    T = ransac_o3d(s, r, distance_threshold=0.05, ransac_n=3, num_iterations=1000)
    assert isinstance(T, np.ndarray) and T.dtype == np.float64 and T.shape == (4, 4)
    want = GF.ransac_correspondences(torch.from_numpy(s).cuda(), torch.from_numpy(r).cuda(), 0.05, 3, 1000)['transform'].cpu().numpy()
    assert np.array_equal(T, want.astype(np.float64))
    perm_s, perm_r = rng.permutation(800), rng.permutation(800)
    S, Rr = np.empty_like(s), np.empty_like(r)
    S[perm_s], Rr[perm_r] = s, r
    corr = np.stack([perm_s, perm_r], axis=1)
    T_idx = ransac_o3d(S, Rr, correspondences=corr, distance_threshold=0.05, ransac_n=3, num_iterations=1000)
    assert np.array_equal(T_idx, T)
    T_dev = ransac_o3d(torch.from_numpy(S).cuda(), torch.from_numpy(Rr).cuda(), correspondences=torch.from_numpy(corr).cuda(),
                       distance_threshold=0.05, ransac_n=3, num_iterations=1000)
    assert T_dev.is_cuda and np.array_equal(T_dev.cpu().numpy().astype(np.float64), T)


def test_argument_checks():
    from geotransformer_b200 import functional as GF
    from geotransformer_b200.utils.open3d import registration_with_ransac_from_correspondences as ransac_o3d
    src = torch.zeros((2, 8, 3), device='cuda')
    T = torch.eye(4, device='cuda').expand(2, 4, 4).contiguous()
    one = torch.full((1,), 8, dtype=torch.int32, device='cuda')
    with pytest.raises(ValueError, match='one count per pair'):
        GF.correspondence_metrics_batched(src, src, T, 0.1, num_corr=one)
    with pytest.raises(ValueError, match='one count per pair'):
        GF.ransac_correspondences_batched(src, src, 0.1, 3, 10, num_corr=one)
    with pytest.raises(RuntimeError, match='CUDA'):
        GF.correspondence_metrics_batched(src, src, T.cpu(), 0.1)
    pts = torch.rand((10, 3), device='cuda')
    for bad in ([[0, 0], [10, 1]], [[0, 0], [1, 10]], [[-1, 0]]):
        with pytest.raises(IndexError):
            ransac_o3d(pts, pts, correspondences=torch.tensor(bad, device='cuda'))
        with pytest.raises(IndexError):
            ransac_o3d(pts.cpu().numpy(), pts.cpu().numpy(), correspondences=np.array(bad))


def _close(a, b):
    return all(abs(a[k] - b[k]) <= (2e-3 if k == 'RRE' else 1e-5) * max(1.0, abs(b[k])) for k in b)


def test_engine_and_tester_run_ransac_after_lgr(models):
    """RegistrationEngine(ransac=cfg.ransac): batch mode (device counts, no host sync) gives per pair the single-pair op's RANSAC on
    the trimmed correspondences, bit for bit; the metrics of the RANSAC transform match the Evaluator's; turning RANSAC on leaves
    the LGR transform and metrics bit-identical; the tester reports the means"""
    from geotransformer_b200 import functional as GF
    from geotransformer_b200.engine import RegistrationEngine
    from geotransformer_b200.loss import Evaluator
    from geotransformer_b200.model import enable_native
    from geotransformer_b200.synth import make_pair
    from geotransformer_b200.tester import METRICS, RegistrationTester
    cfg, _, model = models('3dmatch')
    model = model.cuda().eval()
    enable_native(model)
    keys = ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')
    pairs = [{k: make_pair('demo2k', i)[k] for k in keys} for i in range(4)]
    ev, rc = Evaluator(cfg), cfg.ransac
    eng = RegistrationEngine(model, cfg, cfg.neighbor_limits, num_streams=1, batch_size=4, evaluator=ev)
    off = eng.register(pairs)
    eng.close()
    for bs in (4, 1):
        eng = RegistrationEngine(model, cfg, cfg.neighbor_limits, num_streams=1, batch_size=bs, evaluator=ev, ransac=rc)
        on = eng.register(pairs)
        kept = eng.register(pairs, keep_outputs=True)
        eng.close()
        for p in range(4):
            if bs == 4:
                assert torch.equal(on[p]['estimated_transform'], off[p]['estimated_transform']) and on[p]['metrics'] == off[p]['metrics']
            o = kept[p]['output_dict']
            pid = p if bs == 4 else 0
            want = GF.ransac_correspondences(o['src_corr_points'], o['ref_corr_points'], rc.distance_threshold, rc.num_points,
                                             rc.num_iterations, seed=rc.seed, pair=pid)
            for got in (on[p]['ransac'], kept[p]['ransac']):
                assert torch.equal(got['estimated_transform'], want['transform'].cpu()), (bs, p)
                assert got['fitness'] == float(want['fitness']) and got['inlier_rmse'] == float(want['inlier_rmse'])
            m = ev(dict(o, estimated_transform=want['transform']), {'transform': torch.from_numpy(pairs[p]['transform']).cuda()})
            m = {k: float(v) for k, v in m.items()}
            assert _close(on[p]['ransac']['metrics'], m) and _close(kept[p]['ransac']['metrics'], m), (bs, p, on[p]['ransac']['metrics'], m)
    tester = RegistrationTester(cfg, model, cfg.neighbor_limits, num_streams=1, batch_size=4, with_ransac=True)
    summary, per_pair = tester.run(pairs)
    tester.close()
    for k in METRICS:
        assert summary['ransac_' + k] == float(np.mean([e['ransac']['metrics'][k] for e in per_pair]))
    assert summary['ransac_fitness'] == float(np.mean([e['ransac']['fitness'] for e in per_pair]))
