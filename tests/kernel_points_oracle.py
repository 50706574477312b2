"""numpy restatement of the reference's kernel-point disposition (``modules/kpconv/kernel_points.py``):
``kernel_point_optimization_debug`` (lines 247-386) for ``fixed='center'`` in 3-D, the candidate choice of ``load_kernels``
(lines 389-421) and its per-instance rotation about z, noise and scaling (lines 423-455).  The random draws are inputs, so the
same draws can be fed to the reference (with ``np.random`` patched) and to the device optimiser."""
import numpy as np

MAX_ITER = 10000


TAG_INIT = 0x4B500001


def philox4x32_10(ctr, k0, k1):
    """Philox4x32-10 on (n, 4) uint32 counters with key (k0, k1)"""
    c = [np.asarray(ctr[:, i], dtype=np.uint64) for i in range(4)]
    k0, k1 = np.uint64(k0), np.uint64(k1)
    m32 = np.uint64(0xFFFFFFFF)
    for r in range(10):
        if r > 0:
            k0, k1 = (k0 + np.uint64(0x9E3779B9)) & m32, (k1 + np.uint64(0xBB67AE85)) & m32
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & m32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & m32]
    return np.stack(c, axis=1)


def philox_uniforms(seed, n):
    """the device optimiser's draws (csrc/kernel_points.cu): point i from counters (i, 0, TAG_INIT, 0) (x, y) and (i, 1, TAG_INIT, 0)
    (z), u = (64-bit word >> 11) * 2^-53"""
    idx = np.arange(n, dtype=np.uint64)
    k0, k1 = seed & 0xFFFFFFFF, seed >> 32
    a = philox4x32_10(np.stack([idx, 0 * idx, 0 * idx + TAG_INIT, 0 * idx], axis=1), k0, k1)
    b = philox4x32_10(np.stack([idx, 0 * idx + 1, 0 * idx + TAG_INIT, 0 * idx], axis=1), k0, k1)

    def u(lo, hi):
        return ((hi << np.uint64(32)) | lo) >> np.uint64(11)
    return np.stack([u(a[:, 0], a[:, 1]), u(a[:, 2], a[:, 3]), u(b[:, 0], b[:, 1])], axis=1).astype(np.float64) * 2.0 ** -53


def accept(uniforms, count):
    """the reference's rejection step: rows of ``uniforms`` (U[0, 1)^3) map to 2u - 1 and the first ``count`` with d2 < 0.5 are
    kept in draw order"""
    pts = np.asarray(uniforms, dtype=np.float64) * 2 - 1
    pts = pts[np.sum(np.power(pts, 2), axis=1) < 0.5]
    if pts.shape[0] < count:
        raise ValueError(f'{pts.shape[0]} accepted points, {count} needed')
    return pts[:count]


def optimize(init, num_kernels, num_points, ratio=0.66):
    """``init``: (num_kernels * num_points, 3) accepted points.  Returns (points (K, N, 3) after the rescale, the per-candidate
    max gradient norm of every iteration (MAX_ITER, K), stop iteration, best candidate)."""
    kernel_points = np.array(init, dtype=np.float64).reshape(num_kernels, num_points, 3)
    kernel_points[:, 0, :] *= 0
    moving_factor, decay, thresh, clip = 1e-2, 0.9995, 1e-5, 0.05
    saved = np.zeros((MAX_ITER, num_kernels))
    old = np.zeros((num_kernels, num_points))
    stop = MAX_ITER
    for it in range(MAX_ITER):
        A = np.expand_dims(kernel_points, axis=2)
        B = np.expand_dims(kernel_points, axis=1)
        interd2 = np.sum(np.power(A - B, 2), axis=-1)
        inter = np.sum((A - B) / (np.power(np.expand_dims(interd2, -1), 3 / 2) + 1e-6), axis=1)
        grads = inter + 10 * kernel_points
        norms = np.sqrt(np.sum(np.power(grads, 2), axis=-1))
        saved[it, :] = np.max(norms, axis=1)
        if np.max(np.abs(old[:, 1:] - norms[:, 1:])) < thresh:
            stop = it
            break
        old = norms
        dists = np.minimum(moving_factor * norms, clip)
        dists[:, 0] = 0
        kernel_points -= np.expand_dims(dists, -1) * grads / np.expand_dims(norms + 1e-6, -1)
        moving_factor *= decay
    r = np.sqrt(np.sum(np.power(kernel_points, 2), axis=-1))
    kernel_points *= ratio / np.mean(r[:, 1:])
    # load_kernels: argmin of the LAST row of the saved norms, which is all zeros unless the descent ran MAX_ITER iterations
    best = int(np.argmin(saved[-1, :]))
    return kernel_points, saved, stop, best


def instance(disposition, radius, theta_u, noise):
    """load_kernels' per-instance buffer from the fp32 disposition: theta = 2 pi u, + noise (N(0, 0.01^2) draws, (N, 3)), * radius,
    rotated about z (row vectors times R), fp32"""
    kp = np.asarray(disposition).astype(np.float32)
    theta = theta_u * 2 * np.pi
    c, s = np.cos(theta), np.sin(theta)
    R = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], dtype=np.float32)
    kp = kp + noise
    kp = radius * kp
    return np.matmul(kp, R).astype(np.float32)


def energy(points):
    """the potential the descent lowers: sum over pairs of 1 / d plus 5 |x|^2 per point (gradient 10 x)"""
    p = np.asarray(points, dtype=np.float64)
    d = np.sqrt(np.sum((p[:, None, :] - p[None, :, :]) ** 2, axis=-1))
    iu = np.triu_indices(p.shape[0], 1)
    return float(np.sum(1.0 / d[iu]) + 5 * np.sum(p ** 2))


def read_ply_points(path):
    """the vertex block of a binary little-endian float64 x/y/z .ply (the reference's disposition file)"""
    raw = open(path, 'rb').read()
    head, body = raw.split(b'end_header\n', 1)
    n = int([ln for ln in head.decode().splitlines() if ln.startswith('element vertex')][0].split()[-1])
    return np.frombuffer(body, dtype='<f8', count=3 * n).reshape(n, 3).copy()
