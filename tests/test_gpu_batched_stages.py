"""The batched per-pair stages (one launch for all pairs of a batch) give every pair exactly what the single-pair entry points
give it, bit for bit, on a ragged batch: clouds of different sizes and a pair with fewer valid superpoint pairs than
num_correspondences (its rows past the count are padding)."""
import pytest
import torch

from geotransformer_b200 import functional as GF

pytestmark = pytest.mark.gpu

B, K, KC, C = 3, 64, 12, 32
N_FINE = [900, 400, 70, 700, 500, 90]          # ref_1..ref_3, src_1..src_3
N_NODES = [40, 25, 3, 35, 30, 3]               # pair 3: 3 x 3 = 9 < KC superpoint pairs


def _same(a, b):
    """bit-identical (NaN rows of fully masked padding patches included)"""
    if a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    return torch.equal(a, b)


def _cloud(t, counts, c):
    o = sum(counts[:c])
    return t[o:o + counts[c]]


def test_batched_stages_equal_single_pair_calls():
    g = torch.Generator().manual_seed(11)
    pts = [torch.rand(n, 3, generator=g) * 2.0 for n in N_FINE]
    nodes = [p[torch.randperm(p.shape[0], generator=g)[:m]] for p, m in zip(pts, N_NODES)]
    points_f, points_c = torch.cat(pts).cuda(), torch.cat(nodes).cuda()
    T = torch.eye(4).repeat(B, 1, 1)
    T[:, :3, 3] = torch.rand(B, 3, generator=g) * 0.05
    T = T.cuda()

    # grouping
    _, masks, knn, knn_masks = GF.point_to_node_partition_batched(points_f, points_c, N_FINE, N_NODES, K)
    single = [GF.point_to_node_partition(_cloud(points_f, N_FINE, c), _cloud(points_c, N_NODES, c), K) for c in range(2 * B)]
    for c, (_, m, kn, km) in enumerate(single):
        assert _same(_cloud(masks, N_NODES, c), m) and _same(_cloud(knn, N_NODES, c), kn)
        assert _same(_cloud(knn_masks, N_NODES, c), km)

    # ground-truth superpoint correspondences
    _, _, all_pts = GF.gather_patches_batched(None, 0, N_NODES, N_FINE, knn, knn_masks, points_f)
    gi, go, gc = GF.node_correspondences_batched(points_c, all_pts, masks, knn_masks, N_NODES, T, 0.1)
    g0 = 0
    for p in range(B):
        r, s = p, B + p
        pr = [GF.gather_patches(torch.arange(N_NODES[c], device='cuda'), single[c][2], single[c][3], _cloud(points_f, N_FINE, c))[2]
              for c in (r, s)]
        idx, ov, cnt = GF.node_correspondences(_cloud(points_c, N_NODES, r), _cloud(points_c, N_NODES, s), pr[0], pr[1], T[p].contiguous(),
                                               0.1, single[r][1], single[s][1], single[r][3], single[s][3])
        n = int(cnt.item())
        assert int(gc[p].item()) == n
        assert _same(gi[g0:g0 + n], idx[:n]) and _same(go[g0:g0 + n], ov[:n])
        g0 += N_NODES[r] * N_NODES[s]

    # superpoint matching, patches, scores, Sinkhorn, LGR, metrics
    feats_c = GF.l2_normalize(torch.randn(sum(N_NODES), C, generator=g).cuda())
    feats_f = torch.randn(sum(N_FINE), C, generator=g).cuda()
    corr, nsc, ncnt = GF.superpoint_matching_batched(feats_c, masks, N_NODES, KC)
    k_idx, k_masks, k_pts = GF.gather_patches_batched(corr, KC, N_NODES, N_FINE, knn, knn_masks, points_f)
    rs, ss = slice(0, B * KC), slice(B * KC, 2 * B * KC)
    scores = GF.patch_scores_batched(feats_f, N_FINE, k_idx[rs], k_idx[ss])
    alpha = torch.ones((), device='cuda')
    log_scores = GF.sinkhorn(scores, k_masks[rs], k_masks[ss], alpha, 100)
    rc, sc, cs, Tb, nb = GF.local_global_registration_batched(B, k_pts[rs], k_pts[ss], k_masks[rs], k_masks[ss], log_scores, 3, 0.1,
                                                              True, 0.05, 3, 5)
    res = torch.zeros((B, 24), device='cuda')
    GF.evaluate_batched(gi, go, gc, corr, ncnt, rc, sc, nb, T, Tb, points_f, N_NODES, N_FINE, 0, 0.1, 0.1, res[:, 16:], 0.2)
    assert int(ncnt[2].item()) == 9
    g0 = 0
    for p in range(B):
        r, s = p, B + p
        ri, si, sco, cnt = GF.superpoint_matching(_cloud(feats_c, N_NODES, r), _cloud(feats_c, N_NODES, s), single[r][1], single[s][1], KC,
                                                  defer_count=True)
        assert _same(corr[r], ri) and _same(corr[s], si) and _same(nsc[p], sco) and _same(ncnt[p], cnt[0])
        rk = GF.gather_patches(ri, single[r][2], single[r][3], _cloud(points_f, N_FINE, r))
        sk = GF.gather_patches(si, single[s][2], single[s][3], _cloud(points_f, N_FINE, s))
        pr = slice(p * KC, (p + 1) * KC)
        for a, b in zip(rk + sk, (k_idx[rs][pr], k_masks[rs][pr], k_pts[rs][pr], k_idx[ss][pr], k_masks[ss][pr], k_pts[ss][pr])):
            assert _same(a, b)
        sp = GF.patch_scores(_cloud(feats_f, N_FINE, r), _cloud(feats_f, N_FINE, s), rk[0], sk[0])
        assert _same(sp, scores[pr])
        ls = GF.sinkhorn(sp, rk[1], sk[1], alpha, 100)
        assert _same(ls, log_scores[pr])
        r1, s1, c1, T1, n1 = GF.local_global_registration(rk[2], sk[2], rk[1], sk[1], ls, 3, 0.1, True, 0.05, 3, 5, defer_count=True)
        n = int(n1.item())
        assert int(nb[p].item()) == n
        assert _same(rc[p][:n], r1[:n]) and _same(sc[p][:n], s1[:n]) and _same(cs[p][:n], c1[:n])
        assert _same(Tb[p].contiguous(), T1.reshape(16))
        gn = N_NODES[r] * N_NODES[s]
        m = GF.evaluate(gi[g0:g0 + gn], go[g0:g0 + gn], ri, si, r1, s1, T[p].contiguous(), T1, _cloud(points_f, N_FINE, s), 0, 0.1, 0.1,
                        0.2, n_gt=gc[p:p + 1], n_node_corr=cnt, n_corr=n1)
        assert _same(res[p, 16:].contiguous(), m)
        g0 += gn
