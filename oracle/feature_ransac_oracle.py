"""CPU restatement (numpy) of the feature matching and the feature-matching RANSAC of geotransformer_b200/csrc/feature_match.cu
and csrc/ransac.cu (DESIGN.md section 3b).

TEST INFRASTRUCTURE ONLY.  Restates, independently of the CUDA source, Open3D 0.11's registration_ransac_based_on_feature_matching
as the reference calls it (utils/open3d.py:133-166) with the package's deterministic deviations:
  1. match: m(s) = the nearest ref descriptor of src row s (nearest_neighbor below: fp64, channels summed in order, lowest index
     on exact ties);
  2. iteration i draws ransac_n src rows with ransac_oracle.sample_indices (Philox, keyed (seed, pair id, i));
  3. edge-length check 0.9 and 4. unweighted Kabsch and 5. distance check tau, all in double;
  6. the validated set is the first min(V, #passing) passing iterations in iteration order;
  7. score against the WHOLE ref cloud by brute force in pinned fp32: x' = ((r0 x + r1 y) + r2 z) + t, d^2 = (dx^2 + dy^2) + dz^2
     to the nearest ref point, inlier when d^2 < tau^2; rmse = sqrt(sum d^2 / inliers) with the sum in double;
  8. winner: ransac_oracle.winner (more inliers, then lower rmse, then lower slot = lower iteration); no final refit.
"""
import numpy as np

from oracle import ransac_oracle as RO


def sq_dist64(q, s):
    """(nq, ns) fp64 squared distances, channels summed in order with every operation rounded on its own"""
    q, s = np.asarray(q, np.float64), np.asarray(s, np.float64)
    acc = np.zeros((q.shape[0], s.shape[0]), np.float64)
    for c in range(q.shape[1]):
        d = q[:, c][:, None] - s[:, c][None, :]
        acc = acc + d * d
    return acc


def nearest_neighbor(q, s, block=512):
    """(distances float64, indices int64): argmin of sq_dist64 (np.argmin keeps the lowest index on ties) and its sqrt"""
    q, s = np.asarray(q, np.float32), np.asarray(s, np.float32)
    idx = np.empty(len(q), np.int64)
    dist = np.empty(len(q), np.float64)
    for b in range(0, len(q), block):
        d = sq_dist64(q[b:b + block], s)
        i = np.argmin(d, axis=1)
        idx[b:b + block] = i
        dist[b:b + block] = np.sqrt(d[np.arange(len(i)), i])
    return dist, idx


def edge_check(s, t, ratio=0.9):
    """CorrespondenceCheckerBasedOnEdgeLength: every pair j < k of the sample, d = sqrt((dx^2 + dy^2) + dz^2) in double"""
    s, t = np.asarray(s, np.float64), np.asarray(t, np.float64)
    for j in range(len(s)):
        for k in range(j + 1, len(s)):
            u, v = s[j] - s[k], t[j] - t[k]
            ds = np.sqrt((u[0] * u[0] + u[1] * u[1]) + u[2] * u[2])
            dt = np.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])
            if ds < ratio * dt or dt < ratio * ds:
                return False
    return True


def residuals64(R, t, s, tt):
    """|R s_j + t - t_j| in double, ((r0 x + r1 y) + r2 z) + t per row"""
    s, tt = np.asarray(s, np.float64), np.asarray(tt, np.float64)
    y = np.stack([((R[a, 0] * s[:, 0] + R[a, 1] * s[:, 1]) + R[a, 2] * s[:, 2]) + t[a] for a in range(3)], axis=1)
    e = y - tt
    return np.sqrt((e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2])


def distance_check(R, t, s, tt, tau):
    """CorrespondenceCheckerBasedOnDistance: reject when any residual exceeds tau"""
    return bool(np.all(residuals64(R, t, s, tt) <= np.float64(np.float32(tau))))


def validated(pass_flags, V):
    """the first min(V, #passing) passing iterations, in iteration order"""
    return np.flatnonzero(np.asarray(pass_flags))[:V]


def score(R, t, src, ref, tau):
    """(inliers, float32 rmse) of (R, t) (rounded to float32) over the whole src cloud against the whole ref cloud"""
    R, t = np.asarray(R, np.float32), np.asarray(t, np.float32)
    src, ref = np.asarray(src, np.float32), np.asarray(ref, np.float32)
    if len(src) == 0 or len(ref) == 0:
        return 0, np.float32(0.0)
    x, y, z = src[:, 0], src[:, 1], src[:, 2]
    a = [((R[i, 0] * x + R[i, 1] * y) + R[i, 2] * z) + t[i] for i in range(3)]
    best = np.full(len(src), np.inf, np.float32)
    for b in range(0, len(ref), 2048):
        r = ref[b:b + 2048]
        d = [a[i][:, None] - r[:, i][None, :] for i in range(3)]
        best = np.minimum(best, ((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]).min(1))
    tau2 = np.float32(tau) * np.float32(tau)
    inl = best < tau2
    c = int(inl.sum())
    return c, (np.float32(np.sqrt(best[inl].astype(np.float64).sum() / c)) if c > 0 else np.float32(0.0))


def ransac_features(src, ref, src_feats, ref_feats, tau, ransac_n, num_iterations, val_iterations, seed=0, pair=0, transforms=None):
    """The whole feature-matching RANSAC of one pair.  ``transforms``: optional (V', 4, 4) per-validated transforms to score instead
    of the restatement's own Kabsch (the device's hypotheses: the inlier counts then reproduce exactly).  Returns a dict:
    transform, fitness, inlier_rmse, inliers, iteration, num_validated, matches, samples, pass, val_ids, counts, rmse, hyps."""
    src, ref = np.asarray(src, np.float32), np.asarray(ref, np.float32)
    n = len(src)
    out = dict(transform=np.eye(4, dtype=np.float32), fitness=0.0, inlier_rmse=0.0, inliers=0, iteration=-1, num_validated=0)
    if ransac_n < 3 or not tau > 0 or num_iterations == 0 or val_iterations == 0 or n < ransac_n or len(ref) == 0:
        return out
    _, match = nearest_neighbor(src_feats, ref_feats)
    idx = RO.sample_indices(seed, pair, n, ransac_n, num_iterations)
    flags = np.zeros(num_iterations, bool)
    hyps = {}
    for i in range(num_iterations):
        s, t = src[idx[i]], ref[match[idx[i]]]
        if not edge_check(s, t):
            continue
        R, tr = RO.kabsch(s, t)
        if distance_check(R, tr, s, t, tau):
            flags[i] = True
            hyps[i] = (R, tr)
    vids = validated(flags, val_iterations)
    counts = np.zeros(len(vids), np.int64)
    rmse = np.zeros(len(vids), np.float32)
    for k, i in enumerate(vids):
        if transforms is not None:
            R, tr = transforms[k][:3, :3], transforms[k][:3, 3]
        else:
            R, tr = hyps[i]
        counts[k], rmse[k] = score(R, tr, src, ref, tau)
    out.update(matches=match, samples=idx, pass_flags=flags, val_ids=vids, counts=counts, rmse=rmse, num_validated=len(vids),
               hyps=[hyps[i] for i in vids])
    best = RO.winner(counts, rmse)
    if best >= 0:
        T = np.eye(4, dtype=np.float32)
        if transforms is not None:
            T = np.asarray(transforms[best], np.float32)
        else:
            T[:3, :3], T[:3, 3] = hyps[vids[best]][0], hyps[vids[best]][1]
        out.update(transform=T, fitness=float(np.float32(counts[best] / n)), inlier_rmse=float(rmse[best]), inliers=int(counts[best]),
                   iteration=int(vids[best]))
    return out
