"""End-to-end parity of the CUDA path against the committed golden fixtures (outputs of the REAL reference run in the
reference checkout by oracle/make_golden.py) on the deterministic pairs/weights.  Stage-wise with teacher forcing where
the reference itself is ill-conditioned (coarse top-k on random-weight features, SURVEY.md 'hard parts')."""
import numpy as np
import pytest
import torch

from geotransformer_b200.synth import make_pair
from geotransformer_b200.utils.data import registration_collate_fn_stack_mode
from oracle import geo_oracle as G

pytestmark = pytest.mark.gpu

CASES = [('demo2k', '3dmatch'), ('modelnet717', 'modelnet'), ('kitti4k', 'kitti')]


def _collate(pair, cfg, limits):
    dd = {k: pair[k] for k in ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')}
    return registration_collate_fn_stack_mode([dd], cfg.backbone.num_stages, cfg.backbone.init_voxel_size,
                                              cfg.backbone.init_radius, limits)


def _rows(t, idx):
    return t.reshape(-1, t.shape[-1])[torch.from_numpy(idx).to(t.device)].cpu().numpy()


def check_collate(workload, cfg, pair, gold):
    """GPU collate vs the gold dict (reference fixture or live oracle): lengths, level points (values AND order) and all
    3S-2 neighbour tables, bit-exact up to the order inside exact-distance tie groups"""
    limits = np.asarray(gold['neighbor_limits']).tolist()
    data = _collate(pair, cfg, limits)
    S = cfg.backbone.num_stages
    for i in range(S):
        assert data['lengths'][i].tolist() == gold[f'lengths_{i}'].tolist()
        if i > 0:
            assert np.array_equal(data['points'][i].cpu().numpy(), gold[f'points_{i}']), f'points level {i} (values/order)'
    n_tie = 0
    for key, qi, si in (('neighbors', 0, 0), ('subsampling', 1, 0), ('upsampling', 0, 1)):
        for i, t in enumerate(data[key]):
            want = torch.from_numpy(gold[f'{key}_{i}'].astype(np.int64))
            got = t.cpu()
            assert got.shape == want.shape, f'{key}[{i}] shape {tuple(got.shape)} vs {tuple(want.shape)}'
            if not torch.equal(got, want):     # only the order inside exact-distance tie groups may differ
                q, s = data['points'][i + qi].cpu(), data['points'][i + si].cpu()
                assert torch.equal(G.canonical_neighbors(q, s, got), G.canonical_neighbors(q, s, want)), f'{key}[{i}]'
                n_tie += int((got != want).any(dim=1).sum())
    print(f'{workload}: {n_tie} rows differ from the reference only by exact-tie order')
    return data


@pytest.mark.parametrize('workload,cfg_name', CASES)
def test_collate_matches_reference(workload, cfg_name, golden, models):
    cfg, sd, model = models(cfg_name)
    check_collate(workload, cfg, make_pair(workload, 0), golden(workload))


def check_forward(workload, cfg, model, pair, gold, native=False):
    """stage-wise parity of the CUDA forward against the gold dict (teacher forcing where the reference itself is
    ill-conditioned); native=True runs the C++ stage drivers (what bench.py measures)"""
    model = model.cuda().eval()
    if native:
        from geotransformer_b200.model import enable_native
        enable_native(model)
    elif hasattr(model, '_native'):
        del model._native
    limits = np.asarray(gold['neighbor_limits']).tolist()
    data = _collate(pair, cfg, limits)
    # teacher-force the reference's neighbour tables (identical up to exact-tie order, previous test)
    for key in ('neighbors', 'subsampling', 'upsampling'):
        data[key] = [torch.from_numpy(gold[f'{key}_{i}'].astype(np.int64)).cuda() for i in range(len(data[key]))]
    taps = {}
    out = model(data, taps=taps)
    tol = 1e-4
    for k in ('feats_c', 'feats_f'):
        got = _rows(taps[k], gold[k + '_rows'])
        err = np.abs(got - gold[k + '_sample']).max() / max(np.abs(gold[k + '_sample']).max(), 1.0)
        assert err < tol, f'{k}: rel err {err:.2e}'
    # structure embedding of the reference cloud (sampled (i, j) rows): E rms ~0.6, budget 2e-5 (3-term split on the tensor cores)
    nc = data['lengths_host'][-1][0]
    emb = model.transformer.embedding(data['points'][-1][:nc].contiguous())
    got = _rows(emb, gold['ref_embeddings_rows'])
    err = np.abs(got - gold['ref_embeddings_sample']).max()
    assert err < 5e-5, f'structure embedding: abs err {err:.2e}'
    del emb
    fl = cfg.model.fine_level
    for side, sl in (('ref', slice(0, data['lengths_host'][fl][0])), ('src', slice(data['lengths_host'][fl][0], None))):
        got = taps[f'{side}_node_knn_indices'].cpu()
        want = torch.from_numpy(gold[f'{side}_node_knn_indices'].astype(np.int64))
        if not torch.equal(got, want):
            # a differing index is accepted only if the reference's own matmul-form distances of the two candidates are
            # within a few ulp of each other (pairwise_distance is x2 - 2xy + y2: BLAS accumulation order is unspecified)
            nc = data['lengths_host'][-1][0]
            nodes = data['points'][-1].cpu()[:nc] if side == 'ref' else data['points'][-1].cpu()[nc:]
            sq = G.pairwise_distance(nodes, data['points'][fl].cpu()[sl])
            bad = (got != want).nonzero()
            npts = sq.shape[1]
            for r, c in bad.tolist():
                a = sq[r, got[r, c]].item() if got[r, c] < npts else float('inf')
                b = sq[r, want[r, c]].item() if want[r, c] < npts else float('inf')
                assert abs(a - b) <= 8 * np.spacing(np.float32(max(a, b))), f'{side} node {r} slot {c}: {got[r, c]} (d2={a}) vs {want[r, c]} (d2={b})'
            print(f'{workload}: {len(bad)} {side} patch slots differ between near-tied distances')
    for k in ('ref_feats_c', 'src_feats_c'):
        err = np.abs(out[k].cpu().numpy() - gold[k]).max()
        assert err < tol, f'{k}: abs err {err:.2e} (unit-norm features)'
    # coarse matching: same SET of node correspondences; order may differ between near-equal scores
    got_pairs = set(zip(out['ref_node_corr_indices'].tolist(), out['src_node_corr_indices'].tolist()))
    want_pairs = set(zip(gold['ref_node_corr_indices'].tolist(), gold['src_node_corr_indices'].tolist()))
    missing = want_pairs - got_pairs
    assert len(missing) <= max(2, len(want_pairs) // 50), f'{len(missing)} coarse correspondences differ'
    # second pass with the reference's coarse correspondences forced: fine matching must then agree
    data['forced_node_corr'] = (torch.from_numpy(gold['ref_node_corr_indices']).cuda(), torch.from_numpy(gold['src_node_corr_indices']).cuda(),
                                torch.from_numpy(gold['node_corr_scores']).cuda())
    out = model(data)
    ms = out['matching_scores'].reshape(out['matching_scores'].shape[0], -1)[torch.from_numpy(gold['matching_scores_rows']).cuda()].cpu().numpy()
    want = gold['matching_scores_sample']
    # a sampled patch is comparable element by element only if both of its point lists are the reference's (a patch slot that
    # flipped between near-tied distances above permutes a row / column of its assignment matrix)
    same_r = (taps['ref_node_knn_indices'].cpu() == torch.from_numpy(gold['ref_node_knn_indices'].astype(np.int64))).all(dim=1)
    same_s = (taps['src_node_knn_indices'].cpu() == torch.from_numpy(gold['src_node_knn_indices'].astype(np.int64))).all(dim=1)
    keep = np.array([bool(same_r[gold['ref_node_corr_indices'][p]]) and bool(same_s[gold['src_node_corr_indices'][p]])
                     for p in gold['matching_scores_rows']])
    assert keep.sum() >= len(keep) // 2, 'too many sampled patches have permuted point lists'
    ms, want = ms[keep], want[keep]
    live = want > -1e11
    assert np.abs(ms[live] - want[live]).max() < 2e-4, f'matching_scores {np.abs(ms[live] - want[live]).max():.2e}'
    # fine correspondences: identical rows in identical order, except entries whose acceptance is decided by a value
    # within float noise of a threshold (score > 0.05, mutual top-k near ties): at most 0.5% may differ
    def rows(a, b, s):
        return {(tuple(np.round(x, 6)), tuple(np.round(y, 6))): float(z) for x, y, z in zip(a, b, s)}
    got_c = rows(out['ref_corr_points'].cpu().numpy(), out['src_corr_points'].cpu().numpy(), out['corr_scores'].cpu().numpy())
    want_c = rows(gold['ref_corr_points'], gold['src_corr_points'], gold['corr_scores'])
    only = set(got_c) ^ set(want_c)
    print(f'{workload}: {len(got_c)} vs {len(want_c)} fine correspondences, {len(only)} differ')
    assert len(only) <= max(2, len(want_c) // 200), f'{len(only)} correspondences differ'
    common = set(got_c) & set(want_c)
    assert max(abs(got_c[k] - want_c[k]) for k in common) < 1e-4
    if not only:
        assert np.array_equal(out['ref_corr_points'].cpu().numpy(), gold['ref_corr_points'])      # same order too
    T = out['estimated_transform'].cpu().numpy()
    # LGR given OUR assignment matrix must agree with the oracle run on the very same matrix (hypothesis selection by
    # inlier count is discontinuous: one borderline correspondence can legitimately change the winning hypothesis on a
    # near-symmetric shape such as the ModelNet-shape sphere, so the fixture comparison above is only made when the
    # correspondence sets are identical)
    cpu = {k: out[k].cpu() for k in ('ref_node_corr_knn_points', 'src_node_corr_knn_points', 'ref_node_corr_knn_masks',
                                     'src_node_corr_knn_masks', 'matching_scores')}
    otaps = {}
    o_rc, o_sc, o_cs, o_T = G.local_global_registration(cfg, cpu['ref_node_corr_knn_points'], cpu['src_node_corr_knn_points'],
                                                        cpu['ref_node_corr_knn_masks'], cpu['src_node_corr_knn_masks'],
                                                        cpu['matching_scores'][:, :-1, :-1], taps=otaps)
    rc, sc, cs, T2, det = model.fine_matching(out['ref_node_corr_knn_points'], out['src_node_corr_knn_points'],
                                              out['ref_node_corr_knn_masks'], out['src_node_corr_knn_masks'],
                                              out['matching_scores'], None, return_details=True)
    assert torch.equal(T2, out['estimated_transform'])                      # deterministic
    assert o_rc.shape[0] == rc.shape[0]
    assert torch.equal(o_rc, rc.cpu()) and torch.equal(o_sc, sc.cpu())
    # hypotheses: a patch with 3-5 nearly collinear correspondences has an ill-conditioned Kabsch problem, so the
    # per-patch transforms are compared in the bulk (median) and through what they are used for: their inlier counts
    inl = det['patch_inliers'].cpu()
    valid = (inl >= 0).nonzero().flatten()
    assert valid.numel() == otaps['patch_transforms'].shape[0]
    dT = (det['patch_transforms'].cpu()[valid] - otaps['patch_transforms']).abs().flatten(1).max(dim=1)[0]
    # absolute tolerances are stated for metre-scale scenes (3DMatch / ModelNet); the translation error of a Kabsch solution
    # scales with the coordinates (KITTI: tens of metres), so they are scaled by the extent of the patch coordinates
    scale = max(1.0, float(out['ref_node_corr_knn_points'].abs().max()) / 2.0)
    # ... and the bulk criterion is applied to the well-conditioned problems only (second singular value of the centred
    # source points >= 20 % of the first; the oracle reports it): a near-collinear patch leaves the rotation about its line
    # to the SVD implementation (fp32 LAPACK there, double Jacobi here)
    well = otaps['patch_conditioning'] > 0.2
    assert dT.median() < 1e-4 * scale, f'patch transforms: median {dT.median():.2e}'
    assert (dT[well] < 1e-3 * scale).float().mean() > 0.9, \
        f'patch transforms: {(dT[well] >= 1e-3 * scale).sum()} of {int(well.sum())} well-conditioned patches differ by more than {1e-3 * scale:.1e}'
    dcount = (inl[valid].long() - otaps['inlier_counts']).abs()
    assert (dcount <= 2).float().mean() > 0.8, f'inlier counts differ: {dcount.tolist()}'
    good = (dT < 1e-4 * scale)
    assert int(dcount[good].max()) <= 2
    best = int(det['best'].item())
    o_best = int(valid[int(otaps['best_index'])])
    if best == o_best:
        dT_final = float((o_T - T2.cpu()).abs().max())
        if dT_final >= 1e-4 * scale:
            # legitimate only when a residual sits on the hard inlier threshold (within the propagated float noise of the
            # hypothesis transform, ~1e-4 of the cloud scale): the refinement then re-selects a different inlier set
            assert otaps['threshold_margin'] < 2e-4 * cfg.fine_matching.acceptance_radius / 0.1 + 1e-6, \
                f'{o_T} vs {T2} (closest residual is {otaps["threshold_margin"]:.2e} from the threshold)'
            print(f'{workload}: a residual lies {otaps["threshold_margin"]:.1e} from the inlier threshold; refined transforms '
                  f'differ by {dT_final:.1e} and are not compared')
        if not only:
            # same correspondences and same winning hypothesis as the reference run.  The refinement re-selects inliers
            # with a hard distance threshold, so the fixture is only reproducible when the oracle LGR, fed OUR assignment
            # matrix (which differs from the reference's by ~1e-5), still lands on the fixture itself
            if float(np.abs(o_T.numpy() - gold['estimated_transform']).max()) < 1e-4 * scale and dT_final < 1e-4 * scale:
                assert np.abs(T - gold['estimated_transform']).max() < 1e-4 * scale, f'transform\n{T}\nvs\n{gold["estimated_transform"]}'
            else:
                print(f'{workload}: oracle LGR on our scores leaves the fixture transform (threshold flip in the refinement); '
                      f'compared against the oracle only')
    else:
        # either two hypotheses within the count noise, or the oracle's winner is one of the ill-conditioned patches
        # (its fp32 LAPACK Kabsch solution differs from our double-precision one by more than 1e-3)
        o_pos = int(otaps['best_index'])
        near_tie = abs(int(inl[best]) - int(inl[o_best])) <= 2
        b_pos = int((valid == best).nonzero()[0])
        assert near_tie or dT[o_pos] > 1e-3 * scale or dT[b_pos] > 1e-3 * scale, \
            f'best hypothesis {best} ({inl[best]}) vs oracle {o_best} ({inl[o_best]}), dT {dT[o_pos]:.2e} / {dT[b_pos]:.2e}'
        print(f'{workload}: hypotheses {best} / {o_best} (inliers {int(inl[best])} / {int(inl[o_best])}, near tie {near_tie}); '
              f'final transform not compared')
    return out


@pytest.mark.parametrize('workload,cfg_name', CASES)
def test_forward_matches_reference(workload, cfg_name, golden, models):
    cfg, sd, model = models(cfg_name)
    check_forward(workload, cfg, model, make_pair(workload, 0), golden(workload))


# ---- BASELINE.json configs 3 and 4 at full size: the pinned restatement (oracle/geo_oracle.py == the real reference with 0.0
# difference on the committed fixtures, KITTI branch included: tests/golden/kitti4k.npz) is run LIVE on the host cores
# and packed into the fixture layout, so the headline workload goes through exactly the same stage-wise checks.
FULL = [('3dmatch20k', '3dmatch'), ('kitti20k', 'kitti')]
_LIVE = {}


def _live_gold(workload, cfg, sd):
    if workload not in _LIVE:
        from oracle import fixture
        torch.set_num_threads(min(16, torch.get_num_threads()))
        pair = make_pair(workload, 0)
        limits = cfg.neighbor_limits or [27, 75, 147, 157, 119][:cfg.backbone.num_stages]
        odata = G.collate_pair(pair, cfg, limits)
        taps = {}
        with torch.no_grad():
            o = G.forward(sd, cfg, odata, taps=taps)
        _LIVE[workload] = (pair, fixture.pack(odata, taps, o, o['node_corr_scores'], limits))
    return _LIVE[workload]


@pytest.mark.parametrize('workload,cfg_name', FULL)
def test_full_size_collate_matches_oracle(workload, cfg_name, models):
    cfg, sd, model = models(cfg_name)
    pair, gold = _live_gold(workload, cfg, sd)
    check_collate(workload, cfg, pair, gold)


@pytest.mark.parametrize('workload,cfg_name', FULL)
@pytest.mark.parametrize('native', [False, True])
def test_full_size_forward_matches_oracle(workload, cfg_name, native, models):
    cfg, sd, model = models(cfg_name)
    pair, gold = _live_gold(workload, cfg, sd)
    out = check_forward(workload, cfg, model, pair, gold, native=native)
    # ground-truth superpoint pairs (model.py:112-126) against the oracle's: identical up to overlaps within float noise of 0
    got = set(map(tuple, out['gt_node_corr_indices'].cpu().tolist()))
    want = set(map(tuple, gold['gt_node_corr_indices'].tolist()))
    assert len(got ^ want) <= max(2, len(want) // 500), f'{len(got ^ want)} of {len(want)} gt superpoint pairs differ'


def test_full_size_properties_3dmatch20k(models):
    """BASELINE size (20k+20k points): size-independent properties instead of an oracle run"""
    cfg, sd, model = models('3dmatch')
    model = model.cuda().eval()
    pair = make_pair('3dmatch20k', 0)
    data = _collate(pair, cfg, cfg.neighbor_limits)
    lens = data['lengths_host']
    assert lens[0] == [20000, 20000]
    for i, nb in enumerate(data['neighbors']):
        n = data['points'][i].shape[0]
        assert nb.shape[0] == n and nb.shape[1] <= cfg.neighbor_limits[i]
        assert torch.equal(nb[:, 0].cpu(), torch.arange(n)), 'self is the nearest neighbour of a self search'
        assert int(nb.min()) >= 0 and int(nb.max()) <= n
        # every row: real indices first, sentinels last; neighbours stay inside the row's own cloud
        is_sent = nb == n
        assert not bool((is_sent[:, :-1] & ~is_sent[:, 1:]).any())
        n_ref = lens[i][0]
        ref_rows = torch.arange(n, device=nb.device) < n_ref
        real = ~is_sent
        assert not bool(((nb >= n_ref) & real & ref_rows[:, None]).any())
        assert not bool(((nb < n_ref) & real & ~ref_rows[:, None]).any())
    out = model(data)
    T = out['estimated_transform'].cpu().double()
    R = T[:3, :3]
    assert (R @ R.t() - torch.eye(3, dtype=torch.double)).abs().max() < 1e-5 and abs(torch.det(R).item() - 1) < 1e-5
    ms = out['matching_scores']
    assert ms.shape == (256, 65, 65) and bool(torch.isfinite(ms).all())
    fc = out['ref_feats_c']
    assert (fc.norm(dim=1) - 1).abs().max() < 1e-4
    rre, rte = G.registration_error(pair['transform'], T.numpy())
    print(f'3dmatch20k random-weight registration: RRE {rre:.3f} deg, RTE {rte:.4f} m, {out["ref_corr_points"].shape[0]} correspondences')
    # determinism: a second run gives identical outputs
    out2 = model(data)
    assert torch.equal(out2['estimated_transform'], out['estimated_transform'])
    assert torch.equal(out2['ref_corr_points'], out['ref_corr_points'])


def test_kitti_shape_runs(models):
    """5-stage backbone, hidden 128, K_patch 128, topk 2 (config 4 shape at reduced point count to stay fast)"""
    from geotransformer_b200.synth import WORKLOADS, _ground
    cfg, sd, model = models('kitti')
    model = model.cuda().eval()
    WORKLOADS['kitti8k'] = ('kitti', _ground, dict(n=8000, R=25.0, sigma=0.05), 10.0)
    pair = make_pair('kitti8k', 0)
    data = _collate(pair, cfg, [27, 75, 147, 157, 119])
    out = model(data)
    assert out['matching_scores'].shape[1:] == (129, 129)
    assert bool(torch.isfinite(out['estimated_transform']).all())
