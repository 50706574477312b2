"""TEST INFRASTRUCTURE ONLY -- packs the stage-boundary tensors of one forward (the real reference's, when run by
oracle/make_golden.py next to the reference checkout; the pinned restatement oracle/geo_oracle.py's, when a -m gpu parity test runs
it live at BASELINE.json's full sizes) into the flat dict layout of tests/golden/*.npz, so that fixture-based and live
parity tests share one checker (tests/test_gpu_e2e.py::check_forward)."""
import numpy as np


def sample_rows(t, n=64):
    t = t.detach()
    idx = np.unique(np.linspace(0, t.shape[0] - 1, num=min(n, t.shape[0])).astype(np.int64))
    return idx, t[idx].numpy()


def pack(data, taps, out, node_corr_scores, limits):
    """data: collated dict (CPU tensors); taps: geo_oracle.forward taps; out: output_dict the fixture is made of."""
    g = {}
    for i, (p, l) in enumerate(zip(data['points'], data['lengths'])):
        if i > 0:
            g[f'points_{i}'] = p.numpy()
        g[f'lengths_{i}'] = l.numpy()
    for key in ('neighbors', 'subsampling', 'upsampling'):
        for i, t in enumerate(data[key]):
            g[f'{key}_{i}'] = t.numpy().astype(np.uint16 if int(t.max()) < 65536 else np.int32)   # sentinel = number of support rows
    for k in ('feats_c', 'feats_f', 'ref_embeddings'):
        t = taps[k]
        idx, rows = sample_rows(t.reshape(t.shape[0], -1) if k != 'ref_embeddings' else t.reshape(-1, t.shape[-1]), 96)
        g[k + '_rows'], g[k + '_sample'] = idx, rows
        g[k + '_sum'] = np.array([t.double().sum().item(), t.double().abs().sum().item()])
    for k in ('ref_feats_c', 'src_feats_c', 'estimated_transform', 'corr_scores', 'ref_corr_points', 'src_corr_points',
              'ref_node_corr_indices', 'src_node_corr_indices'):
        g[k] = out[k].detach().numpy()
    g['gt_node_corr_indices'] = out['gt_node_corr_indices'].numpy()
    g['gt_node_corr_overlaps'] = out['gt_node_corr_overlaps'].numpy()
    g['node_corr_scores'] = node_corr_scores.numpy()
    idx, rows = sample_rows(out['matching_scores'].reshape(out['matching_scores'].shape[0], -1), 16)
    g['matching_scores_rows'], g['matching_scores_sample'] = idx, rows
    for k in ('ref_node_knn_indices', 'src_node_knn_indices'):
        g[k] = taps[k].numpy().astype(np.int32)
    g['neighbor_limits'] = np.array(limits)
    return g


# ---- compact storage of a fixture (tests/golden/*.npz stay small) -----------------------------------------------------------
# The level points and the neighbour tables of the reference's collate are what the C restatement (oracle/collate_oracle.c)
# computes, up to the order inside exact-distance tie groups of the neighbour rows.  A compact fixture stores, for each of them,
# the SHA-256 of the reference's array and the rows whose order differs from the restatement's; ``expand`` recomputes the array
# with the restatement, patches those rows back and checks the digest, so tests compare against the reference's exact bytes.
# Row samples of large float tensors keep every ``stride``-th sampled row (MAX_SAMPLE_BYTES per sample).
TABLE_KEYS = ('neighbors', 'subsampling', 'upsampling')
MAX_SAMPLE_BYTES = 160_000


def _digest(a):
    import hashlib
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f'{a.dtype.str}{a.shape}'.encode())
    h.update(a.tobytes())
    return h.hexdigest()


def _restated(workload, limits, index=0):
    """level points / lengths / neighbour tables of the C restatement for pair ``index`` of the workload"""
    from geotransformer_b200.config import make_cfg
    from geotransformer_b200.synth import make_pair
    from oracle import geo_oracle
    pair = make_pair(workload, index)
    return geo_oracle.collate_pair(pair, make_cfg(pair['config']), list(limits))


def compact(workload, g, index=0):
    """full fixture dict of pair ``index`` -> compact fixture dict (see above)"""
    c = dict(g)
    data = _restated(workload, g['neighbor_limits'].tolist(), index)
    arrays = {f'points_{i}': p.numpy() for i, p in enumerate(data['points']) if f'points_{i}' in g}
    for key in TABLE_KEYS:
        for i, t in enumerate(data[key]):
            arrays[f'{key}_{i}'] = t.numpy()
    for name, mine in arrays.items():
        ref = g[name]
        assert mine.shape == ref.shape, (workload, name)
        mine = mine.astype(ref.dtype)
        c[name + '_sha256'] = np.array(_digest(ref))
        if name.startswith('points_'):
            assert np.array_equal(mine, ref), (workload, name)
        else:
            rows = np.nonzero((mine != ref).any(axis=1))[0].astype(np.int32)
            c[name + '_tie_rows'], c[name + '_tie_values'] = rows, ref[rows]
        del c[name]
    for k in [k for k in g if k.endswith('_sample')]:
        stride = -(-g[k].nbytes // MAX_SAMPLE_BYTES)
        base = k[:-len('_sample')]
        c[k], c[base + '_rows'] = g[k][::stride], g[base + '_rows'][::stride]
    return c


def expand(workload, z, index=0):
    """compact fixture (npz or dict) of pair ``index`` -> dict with the full arrays of the reference; raises if the restatement
    no longer reproduces them"""
    g = dict(z) if isinstance(z, dict) else {k: z[k] for k in z.files}
    names = [k[:-len('_sha256')] for k in g if k.endswith('_sha256')]
    if not names:
        return g
    data = _restated(workload, g['neighbor_limits'].tolist(), index)
    for name in names:
        key, i = name.rsplit('_', 1)
        t = data[key][int(i)].numpy()
        if key == 'points':
            a = t
        else:
            a = t.astype(np.uint16 if t.max() < 65536 else np.int32)
            a[g.pop(name + '_tie_rows')] = g.pop(name + '_tie_values')
        if _digest(a) != str(g.pop(name + '_sha256')):
            raise RuntimeError(f'{workload}: {name} of the C restatement (tie rows patched) differs from the reference fixture')
        g[name] = a
    return g


# ---- reduced reference outputs of further pairs (tests/golden/other_pairs.npz) -------------------------------------------------
# What oracle/make_golden.py compares between the restatement and the reference on a pair, stored small: the collate tables as
# above, the integer outputs, the transform, the gt overlaps and the metrics in full, the float tensors as row samples plus
# float64 sum / abs-sum.  ``compare_outputs`` applies make_golden's tolerances to a restatement run of the same pair.
FLOAT_KEYS = ('ref_feats_c', 'src_feats_c', 'ref_feats_f', 'src_feats_f', 'matching_scores')
OTHER_SAMPLE_ROWS = {'matching_scores': 8}           # rows per float tensor (a matching-score row is a whole patch)
FEATURE_SAMPLE_ROWS = 24
CORR_SAMPLE_ROWS = 384


def corr_rows(out):
    """fine correspondences as rows [ref point, src point, score], sorted lexicographically (they come out patch after patch,
    so a permutation of near-tied coarse correspondences permutes them block-wise)"""
    r = np.concatenate([out['ref_corr_points'].numpy(), out['src_corr_points'].numpy(), out['corr_scores'].numpy()[:, None]], axis=1)
    r = r.astype(np.float64)
    return r[np.lexsort(r.T[::-1])]


def _sampled(name, a, n, g):
    a = a.reshape(a.shape[0], -1) if a.ndim > 1 else a[:, None]
    rows = np.unique(np.linspace(0, a.shape[0] - 1, num=min(n, a.shape[0])).astype(np.int64)) if a.shape[0] else np.zeros(0, np.int64)
    g[name + '_shape'] = np.array(a.shape)
    g[name + '_rows'], g[name + '_sample'] = rows, a[rows]
    g[name + '_sum'] = np.array([a.astype(np.float64).sum(), np.abs(a.astype(np.float64)).sum()])


def reduce_outputs(ref_out, metrics):
    """ref_out: the reference's output_dict; metrics: {evaluator variant: {name: value}}"""
    g = {}
    for k in FLOAT_KEYS:
        _sampled(k, ref_out[k].detach().numpy(), OTHER_SAMPLE_ROWS.get(k, FEATURE_SAMPLE_ROWS), g)
    _sampled('corr', corr_rows(ref_out), CORR_SAMPLE_ROWS, g)
    for k in ('estimated_transform', 'ref_node_corr_indices', 'src_node_corr_indices', 'gt_node_corr_indices', 'gt_node_corr_overlaps'):
        g[k] = ref_out[k].detach().numpy()
    for variant, m in metrics.items():
        g['metric_names_' + variant] = np.array(sorted(m))
        g['metric_values_' + variant] = np.array([m[k] for k in sorted(m)], dtype=np.float64)
    return g


def compare_outputs(o, g, metrics):
    """restatement output_dict ``o`` and its metrics {variant: {name: value}} vs the reduced reference outputs ``g``: the list of
    keys that deviate (empty = the restatement reproduces the reference within make_golden's tolerances)"""
    bad = []

    def close(name, a, tol=1e-5):
        a = a.reshape(a.shape[0], -1) if a.ndim > 1 else a[:, None]
        if tuple(a.shape) != tuple(g[name + '_shape']):
            bad.append(name + ' shape')
            return
        a64 = a.astype(np.float64)
        if len(g[name + '_rows']) and float(np.abs(a[g[name + '_rows']] - g[name + '_sample']).max()) > tol:
            bad.append(name)
        n = max(a.size, 1)              # |a - b| <= tol everywhere bounds the difference of the sums by tol * size
        if abs(a64.sum() - g[name + '_sum'][0]) > tol * n or abs(np.abs(a64).sum() - g[name + '_sum'][1]) > tol * n:
            bad.append(name + ' sum')

    mine = list(zip(o['ref_node_corr_indices'].tolist(), o['src_node_corr_indices'].tolist()))
    want = list(zip(g['ref_node_corr_indices'].tolist(), g['src_node_corr_indices'].tolist()))
    perm = np.arange(len(want))
    if mine != want:
        # adjacent coarse scores can sit within an ulp of each other: accept a permutation between scores that agree to 1e-5
        # relative and compare the per-patch tensors under it
        pos = {pr: i for i, pr in enumerate(mine)}
        if len(pos) != len(want) or set(pos) != set(want):
            return ['coarse correspondence sets']
        perm = np.array([pos[pr] for pr in want])
        sc = o['node_corr_scores'].numpy()
        if not np.allclose(sc[perm], sc, rtol=1e-5, atol=0):
            bad.append('coarse correspondences permuted between different scores')
    for k in FLOAT_KEYS:
        a = o[k].detach().numpy()
        close(k, a[perm] if k == 'matching_scores' else a)
    close('corr', corr_rows(o))
    if float(np.abs(o['estimated_transform'].numpy() - g['estimated_transform']).max()) > 1e-5:
        bad.append('estimated_transform')
    if not np.array_equal(o['gt_node_corr_indices'].numpy(), g['gt_node_corr_indices']):
        bad.append('gt_node_corr_indices')
    elif float(np.abs(o['gt_node_corr_overlaps'].numpy() - g['gt_node_corr_overlaps']).max(initial=0.0)) > 1e-5:
        bad.append('gt_node_corr_overlaps')
    for variant, m in metrics.items():
        names = g['metric_names_' + variant].tolist()
        if sorted(m) != names:
            bad.append(f'metric names {variant}')
            continue
        for name, v in zip(names, g['metric_values_' + variant]):
            if abs(float(m[name]) - float(v)) > (1e-3 if name == 'RRE' else 1e-5):       # RRE: acos of an fp32 3x3 product
                bad.append(f'metric {variant} {name}')
    return bad
