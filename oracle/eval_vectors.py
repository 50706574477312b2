"""TEST INFRASTRUCTURE ONLY -- the seeded synthetic benchmark tree of the evaluation tests, and the generator of
tests/golden/eval_benchmark.npz from the REAL reference's ``eval_one_epoch`` (imported through oracle/ref_harness.py, CPU).
Run where the reference checkout exists:   python -m oracle.eval_vectors

``make_tree(root)`` writes (numpy only, from SEED):
  features/3DMatch|3DLoMatch/<scene>/<ref>_<src>.npz   two real 3DMatch scene names (get_num_fragments rejects others)
  gt/3DMatch|3DLoMatch/<scene>/gt.log, gt.info          covariances from calibrate_ground_truth's formula; adjacent pairs that the
                                                        benchmark skips, and tree pairs missing from gt.log
  kitti/<seq>_<src>_<ref>.npz                           one KITTI sequence
Per pair: node correspondences with duplicates (one pair with an empty gt set), correspondence scores with ties straddling the
num_corr boundaries (the tied rows are copies of one correspondence, so every tie rule gives the same metrics) and more than 5 000
rows for some pairs, estimated transforms on both sides of every acceptance threshold and none within 1e-3 relative of one.

Stored per run (3DMatch / 3DLoMatch x lgr / svd, KITTI x lgr / svd with and without --num_corr 1000):
  <run>/lines              'LEVEL<TAB>message' of every line the reference logs (verbose)
  <run>/estlog/<scene>     the est.log bytes (3DMatch)
  <run>/sparse             (pairs, 3) precision, recall, hit_ratio of the reference's evaluate_sparse_correspondences
  <run>/corr               (pairs, 4) overlap, inlier_ratio, residual, num_corr of its evaluate_correspondences
  <run>/reg                (pairs, 2) rre, rte of its compute_registration_error (NaN where it was not called)
  <run>/terr               (pairs,) compute_transform_error (NaN where it was not called)
  <run>/est                (pairs, 4, 4) the estimate the reference evaluated
"""
import importlib
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD_PATH = os.path.join(ROOT, 'tests', 'golden', 'eval_benchmark.npz')
SEED = 20261015
SCENES = ('7-scenes-redkitchen', 'sun3d-hotel_uc-scan3')
KITTI_SEQ = 8
RUNS = (('3dmatch', '3DMatch', 'lgr', None), ('3dmatch', '3DLoMatch', 'lgr', None), ('3dmatch', '3DMatch', 'svd', None),
        ('3dmatch', '3DLoMatch', 'svd', None), ('kitti', None, 'lgr', None), ('kitti', None, 'svd', None),
        ('kitti', None, 'lgr', 1000), ('kitti', None, 'svd', 1000))


def run_name(config, benchmark, method, num_corr):
    return f'{benchmark or config}_{method}' + ('' if num_corr is None else f'_k{num_corr}')


def mat2quat(M):
    """nibabel.quaternions.mat2quat restated: [w, x, y, z] = eigenvector of the largest eigenvalue of Bar-Itzhack's K (its lower
    triangle, / 3), w >= 0."""
    Qxx, Qyx, Qzx, Qxy, Qyy, Qzy, Qxz, Qyz, Qzz = np.asarray(M).flat
    K = np.array([[Qxx - Qyy - Qzz, 0, 0, 0],
                  [Qyx + Qxy, Qyy - Qxx - Qzz, 0, 0],
                  [Qzx + Qxz, Qzy + Qyz, Qzz - Qxx - Qyy, 0],
                  [Qyz - Qzy, Qzx - Qxz, Qxy - Qyx, Qxx + Qyy + Qzz]]) / 3.0
    vals, vecs = np.linalg.eigh(K)
    q = vecs[[3, 0, 1, 2], np.argmax(vals)]
    if q[0] < 0:
        q *= -1
    return q


def _rotation(rng, angle_deg):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    a = np.deg2rad(angle_deg)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K


def _transform(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def _covariance(rng, scale):
    pts = rng.uniform(-scale, scale, size=(400, 3))
    g = np.zeros((pts.shape[0], 3, 6))
    g[:, :3, :3] = np.eye(3)
    g[:, 0, 4], g[:, 0, 5] = pts[:, 2], -pts[:, 1]
    g[:, 1, 3], g[:, 1, 5] = -pts[:, 2], pts[:, 0]
    g[:, 2, 3], g[:, 2, 4] = pts[:, 1], -pts[:, 0]
    return np.matmul(g.transpose(0, 2, 1), g).sum(0)


def _transform_error(gt, cov, est):
    rel = np.linalg.inv(gt.astype(np.float64)) @ est.astype(np.float64)
    er = np.concatenate([rel[:3, 3], mat2quat(rel[:3, :3])[1:]])
    return float(er @ cov.astype(np.float64) @ er / cov[0, 0])


def _rre_rte(gt, est):
    x = np.clip(0.5 * (np.trace(est[:3, :3].T @ gt[:3, :3]) - 1.0), -1.0, 1.0)
    return float(np.degrees(np.arccos(x))), float(np.linalg.norm(gt[:3, 3] - est[:3, 3]))


def _far(v, thr):
    return abs(v - thr) > 1e-3 * thr


def _pair(rng, gt, scale, n, k_ties, est_ok, empty_gt=False):
    """npz arrays of one pair: gt (4, 4) float32; est_ok(est) says whether an estimate is far enough from every threshold."""
    M, N = int(rng.integers(20, 60)), int(rng.integers(20, 60))
    ref_c = rng.uniform(-scale, scale, size=(M, 3)).astype(np.float32)
    src_c = rng.uniform(-scale, scale, size=(N, 3)).astype(np.float32)
    G = 0 if empty_gt else int(rng.integers(10, 40))
    gt_nodes = np.stack([rng.integers(0, M, G), rng.integers(0, N, G)], 1).astype(np.int64).reshape(-1, 2)
    P = int(rng.integers(20, 80))
    pred = np.stack([rng.integers(0, M, P), rng.integers(0, N, P)], 1).astype(np.int64)
    if G:                                                # some hits, and duplicate predictions
        take = rng.integers(0, G, P // 3)
        pred[:take.shape[0]] = gt_nodes[take]
    pred[-5:] = pred[:5]
    src = rng.uniform(-scale, scale, size=(n, 3))
    R, t = gt[:3, :3].astype(np.float64), gt[:3, 3].astype(np.float64)
    ref = src @ R.T + t + rng.normal(scale=0.02 * scale, size=(n, 3))
    outl = rng.random(n) < 0.6
    ref[outl] = rng.uniform(-scale, scale, size=(int(outl.sum()), 3))
    scores = rng.random(n).astype(np.float32)
    for k in k_ties:                                     # rows k-2 .. k+1 of the order share one score and one correspondence
        if n > k + 2:
            order = np.argsort(-scores, kind='stable')
            rows = order[k - 2:k + 2]
            scores[rows] = scores[order[k - 2]]
            src[rows], ref[rows] = src[rows[0]], ref[rows[0]]
    while True:
        angle = float(rng.choice([0.5, 2.0, 4.0, 8.0, 20.0])) * float(rng.uniform(0.5, 1.5))
        dt = rng.normal(size=3)
        dt *= float(rng.choice([0.02, 0.1, 0.3, 1.0, 3.0])) * scale / 3.0 * float(rng.uniform(0.5, 1.5)) / np.linalg.norm(dt)
        est = (gt.astype(np.float64) @ _transform(_rotation(rng, angle), dt)).astype(np.float32)
        if est_ok(est):
            break
    return dict(ref_points_c=ref_c, src_points_c=src_c, ref_node_corr_indices=pred[:, 0].copy(), src_node_corr_indices=pred[:, 1].copy(),
                ref_corr_points=ref.astype(np.float32), src_corr_points=src.astype(np.float32), corr_scores=scores,
                gt_node_corr_indices=gt_nodes, gt_node_corr_overlaps=rng.random(G).astype(np.float32), estimated_transform=est,
                transform=gt.astype(np.float32))


def _fmt(v):
    return '{:.8e}'.format(v)


def make_tree(root, seed=SEED):
    """Writes the synthetic benchmark under root; returns {'features', 'gt_root', 'kitti'} paths."""
    rng = np.random.default_rng(seed)
    feat, gtr, kit = os.path.join(root, 'features'), os.path.join(root, 'gt'), os.path.join(root, 'kitti')
    for bi, bench in enumerate(('3DMatch', '3DLoMatch')):
        for scene in SCENES:
            sdir = os.path.join(feat, bench, scene)
            gdir = os.path.join(gtr, bench, scene)
            os.makedirs(sdir, exist_ok=True)
            os.makedirs(gdir, exist_ok=True)
            nfrag = 37
            pairs = [(0, 1), (0, 5), (1, 7), (2, 3), (3, 12), (4, 20), (5, 9), (10, 30)]
            log_lines, info_lines = [], []
            for pi, (i, j) in enumerate(pairs):
                gt = _transform(_rotation(rng, rng.uniform(5, 90)), rng.uniform(-2, 2, 3))
                gt_txt = np.array([[float(_fmt(v)) for v in row] for row in gt])
                cov = _covariance(rng, 1.5)
                in_log = pi != 6                          # pair 6 is missing from gt.log
                if in_log:
                    log_lines.append(f'{i}\t{j}\t{nfrag}\n' + ''.join('\t'.join(_fmt(v) for v in row) + '\n' for row in gt_txt))
                    info_lines.append(f'{i}\t{j}\t{nfrag}\n' + ''.join('\t'.join(_fmt(v) for v in row) + '\n' for row in cov))
                gt32 = gt_txt.astype(np.float32)
                cov32 = cov.astype(np.float32)
                n = int(rng.choice([800, 3000, 5600, 6200]))

                def ok(est, gt32=gt32, cov32=cov32):
                    p = _transform_error(gt32, cov32, est)
                    return _far(p, 0.04)

                d = _pair(rng, gt32, 1.5, n, (250, 1000, 5000), ok, empty_gt=(bi == 0 and pi == 2))
                d['overlap'] = np.float32(rng.uniform(0.1, 0.9) if bench == '3DMatch' else rng.uniform(0.1, 0.3))
                np.savez_compressed(os.path.join(sdir, f'{i}_{j}.npz'), **d)
            with open(os.path.join(gdir, 'gt.log'), 'w') as f:
                f.writelines(log_lines)
            with open(os.path.join(gdir, 'gt.info'), 'w') as f:
                f.writelines(info_lines)
    os.makedirs(kit, exist_ok=True)
    for src, ref in ((0, 11), (5, 17), (12, 25), (30, 44), (50, 61), (80, 95)):
        gt = _transform(_rotation(rng, rng.uniform(1, 10)), rng.uniform(-10, 10, 3)).astype(np.float32)

        def ok(est, gt=gt):
            rre, rte = _rre_rte(gt.astype(np.float64), est.astype(np.float64))
            return _far(rre, 5.0) and _far(rte, 2.0)

        n = int(rng.choice([900, 2600, 5400, 6400]))
        d = _pair(rng, gt, 30.0, n, (250, 1000, 5000), ok)
        np.savez_compressed(os.path.join(kit, f'{KITTI_SEQ}_{src}_{ref}.npz'), **d)
    return {'features': feat, 'gt_root': gtr, 'kitti': kit}


class _Capture:
    def __init__(self):
        self.lines = []

    def info(self, m):
        self.lines.append(f'INFO\t{m}')

    def critical(self, m):
        self.lines.append(f'CRITICAL\t{m}')


def _recorder(fn, sink):
    def wrapped(*a, **k):
        out = fn(*a, **k)
        sink.append(out)
        return out
    return wrapped


def run_reference(tree, config, benchmark, method, num_corr, out_dir):
    """The reference's eval_one_epoch on the tree; returns the stored record of the run."""
    from oracle import ref_harness
    ref_harness.install()
    sys.modules['nibabel'] = nb = types.ModuleType('nibabel')
    nb.quaternions = types.ModuleType('nibabel.quaternions')
    nb.quaternions.mat2quat = mat2quat
    sys.modules['nibabel.quaternions'] = nb.quaternions
    sys.modules['matplotlib.colors'] = sys.modules['matplotlib'].colors = types.ModuleType('matplotlib.colors')  # plotting helpers only
    import geotransformer.utils.pointcloud as pc            # the reference passes scipy's old n_jobs= (now workers=)
    from scipy.spatial import cKDTree

    class _Tree(cKDTree):
        def query(self, x, k=1, n_jobs=1, **kw):
            return super().query(x, k=k, workers=n_jobs, **kw)
    pc.cKDTree = _Tree
    rcfg, _ = ref_harness.load_experiment(config)
    exp_dir = os.path.join(ref_harness.REF_ROOT, 'experiments', ref_harness.EXP[config])
    sys.modules.pop('eval', None)
    sys.path.insert(0, exp_dir)
    try:
        ev = importlib.import_module('eval')
    finally:
        sys.path.remove(exp_dir)
    rec = {k: [] for k in ('sparse', 'corr', 'reg', 'terr', 'est')}
    ev.evaluate_sparse_correspondences = _recorder(ev.evaluate_sparse_correspondences, rec['sparse'])
    ev.evaluate_correspondences = _recorder(ev.evaluate_correspondences, rec['corr'])
    reg_calls, terr_calls = [], []
    ev.compute_registration_error = _recorder(ev.compute_registration_error, reg_calls)
    if config == '3dmatch':
        ev.compute_transform_error = _recorder(ev.compute_transform_error, terr_calls)
    ev.weighted_procrustes = _recorder(ev.weighted_procrustes, rec['est'])
    if config == '3dmatch':
        rcfg.feature_dir = tree['features']
        rcfg.data.dataset_root = os.path.join(out_dir, 'dataset')
        os.makedirs(os.path.join(rcfg.data.dataset_root, 'metadata'), exist_ok=True)
        link = os.path.join(rcfg.data.dataset_root, 'metadata', 'benchmarks')
        if not os.path.exists(link):
            os.symlink(tree['gt_root'], link)
        rcfg.registration_dir = os.path.join(out_dir, 'registration')
    else:
        rcfg.feature_dir = tree['kitti']
    args = types.SimpleNamespace(test_epoch=None, benchmark=benchmark, method=method, num_corr=num_corr, verbose=True)
    logger = _Capture()
    # which pairs the registration error / transform error were called for: the verbose per-pair line says it
    ev.eval_one_epoch(args, rcfg, logger)
    pair_lines = [ln for ln in logger.lines if ln.startswith('INFO\t') and ', id0: ' in ln]
    n = len(rec['sparse'])
    assert len(pair_lines) == n, (len(pair_lines), n)
    out = {'lines': np.array(logger.lines)}
    out['sparse'] = np.array([[d['precision'], d['recall'], d['hit_ratio']] for d in rec['sparse']], dtype=np.float64)
    out['corr'] = np.array([[d['overlap'], d['inlier_ratio'], d['residual'], d['num_corr']] for d in rec['corr']], dtype=np.float64)
    reg = np.full((n, 2), np.nan)
    terr = np.full((n,), np.nan)
    ri = ti = 0
    for i, ln in enumerate(pair_lines):
        if config == '3dmatch' and 'r_RMSE' in ln:
            terr[i] = terr_calls[ti]
            ti += 1
        if 'r_RRE' in ln:
            reg[i] = reg_calls[ri]
            ri += 1
    assert ri == len(reg_calls) and ti == len(terr_calls)
    out['reg'], out['terr'] = reg, terr
    if method == 'svd':
        out['est'] = np.stack([np.asarray(t.detach().cpu().numpy() if hasattr(t, 'detach') else t) for t in rec['est']])
    if config == '3dmatch':
        for scene in SCENES:
            with open(os.path.join(rcfg.registration_dir, benchmark, scene, 'est.log'), 'rb') as f:
                out[f'estlog/{scene}'] = np.frombuffer(f.read(), dtype=np.uint8)
    return out


def main():
    from oracle import ref_harness
    assert ref_harness.available(), 'needs the reference checkout'
    g = {}
    with tempfile.TemporaryDirectory() as tmp:
        tree = make_tree(os.path.join(tmp, 'tree'))
        for config, bench, method, k in RUNS:
            name = run_name(config, bench, method, k)
            res = run_reference(tree, config, bench, method, k, os.path.join(tmp, name))
            for key, v in res.items():
                g[f'{name}/{key}'] = v
            print(name, 'lines', len(res['lines']))
            for ln in res['lines']:
                if ln.startswith('CRITICAL'):
                    print('   ', ln.split('\t', 1)[1])
    np.savez_compressed(GOLD_PATH, **g)
    print(f'wrote {GOLD_PATH} ({os.path.getsize(GOLD_PATH) / 1e3:.1f} kB)')


if __name__ == '__main__':
    sys.path.insert(0, ROOT)
    main()
