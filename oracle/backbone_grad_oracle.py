"""TEST INFRASTRUCTURE ONLY -- gradients of the KPConv-FPN backbone through torch autograd of the restatement
(oracle/geo_oracle.backbone), and the seeded upstream gradients G_i of the backbone fixture (oracle/backbone_grad_vectors.py).
No import of the reference: the GPU tests use this module."""
import numpy as np
import torch

from geotransformer_b200.config import make_cfg
from geotransformer_b200.synth import make_pair
from oracle import geo_oracle as G

WORKLOADS = (('demo2k', '3dmatch'), ('modelnet717', 'modelnet'), ('kitti4k', 'kitti'))
# neighbour limits of the fixture workloads (as oracle/make_golden.py: the config's own, else these)
LIMITS = {'demo2k': [38, 36, 36, 38], 'modelnet717': [13, 21, 27], 'kitti4k': [27, 75, 147, 157, 119]}
SEED = 7351


def limits(workload):
    return make_cfg(make_pair(workload, 0)['config']).neighbor_limits or LIMITS[workload]


def collate(workload, cfg):
    """collate of pair 0 of the workload through the reference's own neighbour search and subsampling (oracle/_ref, made by
    build()): bit-identical to the reference's collate, neighbour order inside distance ties included"""
    from oracle import ref_ext
    return G.collate_pair(make_pair(workload, 0), cfg, limits(workload), impl=ref_ext)


def digest(t):
    """compact summary of a gradient (a few hundred floats): the whole tensor up to 256 entries, else the sum, the absolute sum,
    192 seeded flat samples and, for a leading dimension of at most 64, the per-slice sums"""
    a = np.asarray(t.detach().cpu() if isinstance(t, torch.Tensor) else t, np.float64)
    if a.size <= 256:
        return {'full': a}
    d = {'sum': np.array([a.sum()]), 'abssum': np.array([np.abs(a).sum()]),
         'samples': a.reshape(-1)[np.random.default_rng(a.size).choice(a.size, size=192, replace=False)]}
    if a.ndim > 1 and a.shape[0] <= 64:
        d['rowsum'] = a.reshape(a.shape[0], -1).sum(1)
    return d


def packed_digest(t):
    """``digest`` as one float32 vector (its parts in key order): the fixture's storage form"""
    d = digest(t)
    return np.concatenate([d[k].ravel() for k in sorted(d)]).astype(np.float32)


def unpack(packed, t):
    """the parts of a packed digest of a tensor shaped like ``t`` (the inverse of ``packed_digest``)"""
    d, out, i = digest(t), {}, 0
    for k in sorted(d):
        out[k] = np.asarray(packed[i:i + d[k].size], np.float64)
        i += d[k].size
    assert i == len(packed), 'packed digest does not match the tensor shape'
    return out


def digest_err(got, packed, floor):
    """largest deviation between the digest of gradient ``got`` and a stored packed digest, part by part, each relative to
    max(that stored part's largest magnitude, floor)"""
    mine, want = digest(got), unpack(packed, got)
    return max(float(np.abs(mine[k] - w).max()) / max(float(np.abs(w).max()), floor) for k, w in want.items())


def upstream(shapes):
    """G_i of the loss sum_i <feats_list[i], G_i>: standard normal, one seeded CPU generator per output"""
    return [torch.randn(s, generator=torch.Generator().manual_seed(1000 + i)) for i, s in enumerate(shapes)]


def restatement_grads(sd, cfg, data, keys, dtype, head=None):
    """{key: d loss / d sd['backbone.' + key]} of geo_oracle.backbone in ``dtype`` on CPU; loss = head(feats_list[0], dtype) or
    sum_i <feats_list[i], G_i>"""
    sd2 = {k: (v.detach().to(dtype) if v.is_floating_point() else v) for k, v in sd.items() if k.startswith('backbone.')}
    leaves = {k: sd2['backbone.' + k].clone().requires_grad_(True) for k in keys}
    sd2.update({'backbone.' + k: v for k, v in leaves.items()})
    d = dict(data, points=[p.to(dtype) for p in data['points']])
    outs = G.backbone(sd2, cfg, data['features'].to(dtype), d)
    if head is not None:
        loss = head(outs[0], dtype)
    else:
        loss = sum((o * u.to(dtype)).sum() for o, u in zip(outs, upstream([tuple(o.shape) for o in outs])))
    loss.backward()
    return {k: leaves[k].grad for k in keys}
