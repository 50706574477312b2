"""CPU restatement (numpy) of the training-data augmentation of geotransformer_b200/csrc/augment.cu.

TEST INFRASTRUCTURE ONLY.  Restates, independently of the CUDA source, the random streams of include/geob200.h:
  * Philox4x32-10 of ransac_oracle with key (seed lo, seed hi ^ tag), tag = 0xA6000000 | stream << 4 | cloud, counter (index,
    iteration lo, iteration hi, pair);
  * pair uniforms ((w0 >> 5) 2^26 + (w1 >> 6)) 2^-53 from words (0, 1) and (2, 3) of calls 0, 1, ...; per-point uniforms w 2^-32;
  * R = Rx(c) Ry(b) Rz(a) (scipy's from_euler('zyx', (a, b, c)));
and the per-point arithmetic of the 3DMatch / KITTI modes in the kernel's fp64 operation order: numpy rounds every elementwise
operation, so given the device's R (from its record) the points are bit-identical.  The ModelNet mode is restated with numpy's
own reductions and libm, so its coordinates agree to fp32 rounding.
"""
import numpy as np

from oracle.ransac_oracle import philox4x32_10

TAG_BASE = 0xA6000000
PAIR, LIMIT, NOISE, SAMPLE, JITTER = 1, 2, 3, 4, 5
THREEDMATCH, KITTI = 0, 1


def tag(stream, cloud):
    return TAG_BASE | (stream << 4) | cloud


def words(index, seed, iteration, pair, stream, cloud):
    """(len(index), 4) uint32 Philox words of the given counter indices"""
    seed, iteration = int(seed), int(iteration)
    j = np.asarray(index, dtype=np.uint64).reshape(-1)
    ctr = np.stack([j, np.full_like(j, iteration & 0xFFFFFFFF), np.full_like(j, iteration >> 32), np.full_like(j, int(pair))], axis=1)
    return philox4x32_10(ctr, (seed & 0xFFFFFFFF, (seed >> 32) ^ tag(stream, cloud)))


def pair_uniforms(n, seed, iteration, pair):
    """u0 .. u10 (float64, slots >= n are 0)"""
    w = words(np.arange(6), seed, iteration, pair, PAIR, 0).astype(np.uint64)
    u = np.zeros(12)
    for i in range(6):
        for h in range(2):
            a, b = w[i, 2 * h], w[i, 2 * h + 1]
            u[2 * i + h] = float((a >> np.uint64(5)) * np.uint64(1 << 26) + (b >> np.uint64(6))) * 2.0 ** -53
    u = u[:11]
    u[n:] = 0.0
    return u


def u32(w):
    return np.asarray(w, dtype=np.float64) * 2.0 ** -32


def euler_zyx(a, b, c):
    """scipy Rotation.from_euler('zyx', (a, b, c)).as_matrix() = Rx(c) Ry(b) Rz(a)"""
    sa, ca, sb, cb, sc, cc = np.sin(a), np.cos(a), np.sin(b), np.cos(b), np.sin(c), np.cos(c)
    return np.array([[cb * ca, -(cb * sa), sb],
                     [cc * sa + (sc * sb) * ca, cc * ca - (sc * sb) * sa, -(sc * cb)],
                     [sc * sa - (cc * sb) * ca, sc * ca + (cc * sb) * sa, cc * cb]])


def _rows(M, x, y, z):
    """rows of M applied to the coordinate arrays, ((m0 x + m1 y) + m2 z)"""
    return [(M[i, 0] * x + M[i, 1] * y) + M[i, 2] * z for i in range(3)]


def limit_rows(n, point_limit, seed, iteration, pair, cloud):
    """rows kept by the point limit, ascending"""
    if n <= point_limit:
        return np.arange(n)
    w = words(np.arange(n), seed, iteration, pair, LIMIT, cloud)[:, 0].astype(np.uint64)
    keys = (w << np.uint64(32)) | np.arange(n, dtype=np.uint64)
    return np.sort(np.argsort(keys, kind='stable')[:point_limit])


def pair_draws(mode, rotation_factor, min_scale, max_scale, shift, seed, iteration, pair):
    """(u (11,), R, rotate_ref, scale, ref_shift (3,), src_shift (3,)) of one 3DMatch / KITTI pair"""
    u = pair_uniforms(11 if mode == KITTI else 4, seed, iteration, pair)
    ang = (u[:3] * np.pi) * 2 / rotation_factor
    R = euler_zyx(*ang)
    scale, rs, ss = 1.0, np.zeros(3), np.zeros(3)
    if mode == KITTI:
        scale = min_scale + (max_scale - min_scale) * u[4]
        rs = -shift + (shift - -shift) * u[5:8]
        ss = -shift + (shift - -shift) * u[8:11]
    return u, R, bool(u[3] > 0.5), scale, rs, ss


def augment_cloud64(points, rows, R, rotated, scale, shift_c, noise, mode, seed, iteration, pair, cloud):
    """the per-point pass of one cloud before the rounding to fp32: (len(rows), 3) float64"""
    p = np.asarray(points, np.float64)[rows]
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    w = words(rows, seed, iteration, pair, NOISE, cloud)
    n = [(u32(w[:, i]) + -0.5) * noise for i in range(3)]
    if mode == KITTI:
        x, y, z = x + n[0], y + n[1], z + n[2]
        if rotated:
            x, y, z = _rows(R, x, y, z)
        x, y, z = x * scale + shift_c[0], y * scale + shift_c[1], z * scale + shift_c[2]
    else:
        if rotated:
            x, y, z = _rows(R, x, y, z)
        x, y, z = x + n[0], y + n[1], z + n[2]
    return np.stack([x, y, z], axis=1)


def noise_uniforms(rows, seed, iteration, pair, cloud):
    """(len(rows), 3) the noise uniforms of the given rows"""
    return u32(words(rows, seed, iteration, pair, NOISE, cloud)[:, :3])


def compose_transform(T, R, rotate_ref, mode, scale, rs, ss):
    """the augmented ground truth in fp64 (4, 4)"""
    T = np.asarray(T, np.float64)
    G, g = T[:3, :3], T[:3, 3]
    if rotate_ref:
        N = np.array([_rows(R, G[0, j], G[1, j], G[2, j]) for j in range(3)]).T
        t = np.array(_rows(R, g[0], g[1], g[2]))
    else:
        N = np.array([_rows(G, R[j, 0], R[j, 1], R[j, 2]) for j in range(3)]).T
        t = g.copy()
    if mode == KITTI:
        t = t * scale
        m = np.array(_rows(N, ss[0], ss[1], ss[2]))
        t = (-m + t) + rs
    out = np.eye(4)
    out[:3, :3], out[:3, 3] = N, t
    return out


def augment_pair(ref, src, T, mode, point_limit, noise, rotation_factor=1.0, min_scale=1.0, max_scale=1.0, shift=0.0,
                 seed=0, iteration=0, pair=0, R=None):
    """one 3DMatch / KITTI pair: dict(ref, src (fp32), ref_origin, src_origin, transform (fp32), record (20,)).  R: the rotation to
    use (the device's record[11:]); default the restatement's own."""
    u, R0, rot_ref, scale, rs, ss = pair_draws(mode, rotation_factor, min_scale, max_scale, shift, seed, iteration, pair)
    R = R0 if R is None else np.asarray(R, np.float64).reshape(3, 3)
    out = dict(record=np.concatenate([u, R.reshape(9)]))
    for cloud, (name, pts, sh) in enumerate((('ref', ref, rs), ('src', src, ss))):
        rows = limit_rows(len(pts), point_limit, seed, iteration, pair, cloud)
        rotated = rot_ref if cloud == 0 else not rot_ref
        pts32 = np.asarray(pts, np.float32)
        out[name] = augment_cloud64(pts32, rows, R, rotated, scale, sh, noise, mode, seed, iteration, pair, cloud).astype(np.float32)
        out[name + '_origin'] = rows
    out['transform64'] = compose_transform(T, R, rot_ref, mode, scale, rs, ss)
    out['transform'] = out['transform64'].astype(np.float32)
    return out


# ---- ModelNet ------------------------------------------------------------------------------------------------------------------

def crop_count(n, keep_ratio):
    return int(np.floor(n * keep_ratio + 0.5))


def modelnet_draws(rotation_magnitude, translation_magnitude, seed, iteration, pair):
    """(u (11,), R, t, ref plane normal, src plane normal)"""
    u = pair_uniforms(10, seed, iteration, pair)
    R = euler_zyx(*((u[:3] * np.pi) * rotation_magnitude / 180.0))
    t = -translation_magnitude + (translation_magnitude - -translation_magnitude) * u[3:6]

    def normal(a, b):
        phi, theta = (2 * np.pi - 0.0) * a, (np.pi - 0.0) * b
        return np.array([np.sin(theta) * np.cos(phi), np.sin(theta) * np.sin(phi), np.cos(theta)])
    return u, R, t, normal(u[6], u[7]), normal(u[8], u[9])


def normalize(points):
    p = np.asarray(points, np.float32).astype(np.float64)
    p = p - p.mean(axis=0)
    return p / np.max(np.linalg.norm(p, axis=1))


def crop_rows(points, normal, keep_ratio):
    """the round(keep N) rows of largest plane distance (ties to the lowest row), ascending; and the distances"""
    d = points @ normal
    k = crop_count(len(points), keep_ratio)
    order = np.lexsort((np.arange(len(d)), -d))
    return np.sort(order[:k]), d


def sample_rows(cropped, num_points, seed, iteration, pair, cloud):
    """the num_points smallest keys (word << 32) | row of the cropped rows, in key order"""
    w = words(cropped, seed, iteration, pair, SAMPLE, cloud)[:, 0].astype(np.uint64)
    keys = (w << np.uint64(32)) | np.asarray(cropped, dtype=np.uint64)
    return np.asarray(cropped)[np.argsort(keys, kind='stable')[:num_points]]


def jitter(rows, noise_magnitude, seed, iteration, pair, cloud):
    """(len(rows), 3) clip(0.01 z, +-noise_magnitude), Box-Muller from the row's words"""
    w = words(rows, seed, iteration, pair, JITTER, cloud)
    r0, r1 = np.sqrt(-2.0 * np.log(1.0 - u32(w[:, 0]))), np.sqrt(-2.0 * np.log(1.0 - u32(w[:, 2])))
    a0, a1 = 2 * np.pi * u32(w[:, 1]), 2 * np.pi * u32(w[:, 3])
    z = np.stack([r0 * np.cos(a0), r0 * np.sin(a0), r1 * np.cos(a1)], axis=1)
    return np.clip(0.01 * z, -noise_magnitude, noise_magnitude)


def modelnet_pair(shape, num_points, keep_ratio, rotation_magnitude, translation_magnitude, noise_magnitude, seed=0, iteration=0,
                  pair=0):
    """one ModelNet pair from a raw shape: dict(ref, src (fp32), ref_origin, src_origin, transform (fp32), record (20,), and the
    crop distances ref_d / src_d)"""
    u, R, t, n_ref, n_src = modelnet_draws(rotation_magnitude, translation_magnitude, seed, iteration, pair)
    out = dict(record=np.concatenate([u, R.reshape(9)]))
    ref = normalize(shape)
    inv_R, inv_t = R.T, -(R.T @ t)
    src = ref @ inv_R.T + inv_t
    for cloud, (name, pts, nrm) in enumerate((('ref', ref, n_ref), ('src', src, n_src))):
        cropped, d = crop_rows(pts, nrm, keep_ratio)
        rows = sample_rows(cropped, num_points, seed, iteration, pair, cloud)
        out[name] = (pts[rows] + jitter(rows, noise_magnitude, seed, iteration, pair, cloud)).astype(np.float32)
        out[name + '_origin'] = rows
        out[name + '_d'] = d
        out[name + '_points64'] = pts
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    out['transform'] = T.astype(np.float32)
    out['transform64'] = T
    return out
