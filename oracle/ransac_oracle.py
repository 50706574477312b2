"""CPU restatement (numpy) of the correspondence RANSAC of geotransformer_b200/csrc/ransac.cu and of the correspondence metrics.

TEST INFRASTRUCTURE ONLY.  Restates, independently of the CUDA source:
  * the sampler: Philox4x32-10 (Salmon et al., SC'11) in uint32 arithmetic, key = 64-bit seed, counter = (iteration, pair,
    draw block, 0), index = umulhi(word, n);
  * the hypothesis: unweighted Kabsch in float64 (numpy SVD), (R, t) rounded to float32;
  * the pinned fp32 score: ((r0 x + r1 y) + r2 z) + t, (dx^2 + dy^2) + dz^2 < tau^2, numpy float32 rounds every operation;
  * the winner rule: most inliers, then lowest float32 rmse, then lowest iteration; no inlier at all -> identity, fitness 0.
"""
import numpy as np

M0, M1, W0, W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(counter, key):
    """counter (N, 4) uint32-valued, key (k0, k1) -> (N, 4) uint32"""
    c = [np.asarray(counter, dtype=np.uint64)[:, i] for i in range(4)]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for r in range(10):
        if r > 0:
            k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
        p0, p1 = M0 * c[0], M1 * c[2]                 # < 2^64: exact in uint64
        hi0, lo0 = p0 >> np.uint64(32), p0 & _MASK
        hi1, lo1 = p1 >> np.uint64(32), p1 & _MASK
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
    return np.stack(c, axis=1).astype(np.uint32)


def sample_indices(seed, pair, n, ransac_n, num_iterations):
    """(num_iterations, ransac_n) int64 correspondence indices of the hypotheses of pair ``pair`` with ``n`` correspondences"""
    seed = int(seed)
    key = (seed & 0xFFFFFFFF, seed >> 32)
    it = np.arange(num_iterations, dtype=np.uint64)
    words = []
    for blk in range((ransac_n + 3) // 4):
        ctr = np.stack([it, np.full_like(it, pair), np.full_like(it, blk), np.zeros_like(it)], axis=1)
        words.append(philox4x32_10(ctr, key))
    w = np.concatenate(words, axis=1)[:, :ransac_n].astype(np.uint64)
    return ((w * np.uint64(n)) >> np.uint64(32)).astype(np.int64)


def kabsch(src, ref):
    """unweighted Kabsch in float64: (R (3, 3), t (3,)) with ref ~ R src + t"""
    src, ref = np.asarray(src, np.float64), np.asarray(ref, np.float64)
    cs, cr = src.mean(0), ref.mean(0)
    H = (src - cs).T @ (ref - cr)
    U, _, Vt = np.linalg.svd(H)
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(Vt.T @ U.T))])
    R = Vt.T @ D @ U.T
    return R, cr - R @ cs


def residual2(R, t, src, ref):
    """pinned fp32 squared residuals of every correspondence under (R, t) (rounded to float32 first)"""
    R, t = np.asarray(R, np.float32), np.asarray(t, np.float32)
    src, ref = np.asarray(src, np.float32), np.asarray(ref, np.float32)
    x, y, z = src[:, 0], src[:, 1], src[:, 2]
    d = [(((R[i, 0] * x + R[i, 1] * y) + R[i, 2] * z) + t[i]) - ref[:, i] for i in range(3)]
    return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]


def score(R, t, src, ref, distance_threshold):
    """(inlier count, float32 inlier rmse) of one hypothesis"""
    tau = np.float32(distance_threshold)
    d2 = residual2(R, t, src, ref)
    inl = d2 < tau * tau
    c = int(inl.sum())
    rmse = np.float32(np.sqrt(d2[inl].astype(np.float64).sum() / c)) if c > 0 else np.float32(0.0)
    return c, rmse


def winner(counts, rmse):
    """index of the best hypothesis (most inliers, then lowest rmse, then lowest index), or -1 when none has an inlier"""
    counts, rmse = np.asarray(counts), np.asarray(rmse, np.float32)
    if counts.size == 0 or counts.max() <= 0:
        return -1
    cand = np.flatnonzero(counts == counts.max())
    cand = cand[rmse[cand] == rmse[cand].min()]
    return int(cand[0])


def ransac(src, ref, distance_threshold, ransac_n, num_iterations, seed=0, pair=0):
    """the whole RANSAC of one pair: dict(transform (4, 4) float32, fitness, inlier_rmse, inliers, iteration, counts, rmse)"""
    src, ref = np.asarray(src, np.float32), np.asarray(ref, np.float32)
    n = src.shape[0]
    out = dict(transform=np.eye(4, dtype=np.float32), fitness=0.0, inlier_rmse=0.0, inliers=0, iteration=-1)
    if n < ransac_n:
        return out
    idx = sample_indices(seed, pair, n, ransac_n, num_iterations)
    counts = np.zeros(num_iterations, np.int64)
    rmse = np.zeros(num_iterations, np.float32)
    hyps = []
    for i in range(num_iterations):
        R, t = kabsch(src[idx[i]], ref[idx[i]])
        R, t = R.astype(np.float32), t.astype(np.float32)
        hyps.append((R, t))
        counts[i], rmse[i] = score(R, t, src, ref, distance_threshold)
    best = winner(counts, rmse)
    out.update(counts=counts, rmse=rmse)
    if best >= 0:
        T = np.eye(4, dtype=np.float32)
        T[:3, :3], T[:3, 3] = hyps[best]
        out.update(transform=T, fitness=float(np.float32(counts[best] / n)), inlier_rmse=float(rmse[best]), inliers=int(counts[best]),
                   iteration=best)
    return out


def correspondence_metrics(ref, src, transform, positive_radius):
    """evaluate_correspondences (utils/registration.py:240-250) with a brute-force nearest neighbour in float64:
    (f_IR, f_OV, f_RS, f_NU, nearest distances)"""
    ref, src = np.asarray(ref, np.float64), np.asarray(src, np.float64)
    T = np.asarray(transform, np.float64)
    s = src @ T[:3, :3].T + T[:3, 3]
    res = np.linalg.norm(ref - s, axis=1)
    nn = np.sqrt(((ref[:, None, :] - s[None, :, :]) ** 2).sum(-1).min(1)) if len(ref) else np.zeros(0)
    with np.errstate(invalid='ignore', divide='ignore'):
        mean = (lambda a: float(a.mean()) if a.size else float('nan'))
        return mean(res < positive_radius), mean(nn < positive_radius), mean(res), len(ref), nn
