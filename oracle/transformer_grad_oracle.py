"""TEST INFRASTRUCTURE ONLY -- gradients of the geometric transformer through torch autograd of the restatement
(oracle/geo_oracle.geometric_transformer), and the digests of tests/golden/transformer_grads.npz.  No import of the reference: the GPU
tests use this module."""
import numpy as np
import torch

from oracle import backbone_grad_oracle as BG
from oracle import geo_oracle as G

# Fixture comparisons: every digest part relative to max(its own largest value, FLOOR x the case's largest gradient).  Two kinds of
# gradient are rounding noise in part, and get a larger scale:
#   - a per-row constant of the attention scores drops out of the softmax, so the true gradients of proj_k.bias (q . bk), proj_p.bias
#     (q_h . bp_h) and the structure-embedding biases (added to every E[n, m]) are zero: ZERO_FLOOR x the largest gradient;
#   - the 'sum' part of a weight feeding a LayerNorm is zero (the norm drops a shift of its input): SUM_NOISE x the 'abssum' part.
FLOOR = 1e-6
ZERO_FLOOR = 1e-4
SUM_NOISE = 1e-3
ZERO_GRADS = ('proj_k.bias', 'proj_p.bias', 'embedding.proj_d.bias', 'embedding.proj_a.bias')


SAMPLES = 96


def digest(t):
    """backbone_grad_oracle.digest with SAMPLES seeded samples instead of 192: the fixture holds ~1100 gradients (every model
    parameter of OverallLoss on three workloads) and stays under 1 MB with them.  A copy rather than a parameter of the backbone's
    function: that module and the backbone fixture written with it are kept exactly as they are.  The whole tensor up to 256 entries,
    else the sum, the absolute sum, the samples and, for a leading dimension of at most 64, the per-slice sums"""
    a = np.asarray(t.detach().cpu() if isinstance(t, torch.Tensor) else t, np.float64)
    if a.size <= 256:
        return {'full': a}
    d = {'sum': np.array([a.sum()]), 'abssum': np.array([np.abs(a).sum()]),
         'samples': a.reshape(-1)[np.random.default_rng(a.size).choice(a.size, size=SAMPLES, replace=False)]}
    if a.ndim > 1 and a.shape[0] <= 64:
        d['rowsum'] = a.reshape(a.shape[0], -1).sum(1)
    return d


def packed_digest(t):
    """``digest`` as one float32 vector (its parts in key order): the fixture's storage form"""
    d = digest(t)
    return np.concatenate([d[k].ravel() for k in sorted(d)]).astype(np.float32)


def unpack(packed, t):
    d, out, i = digest(t), {}, 0
    for k in sorted(d):
        out[k] = np.asarray(packed[i:i + d[k].size], np.float64)
        i += d[k].size
    assert i == len(packed), 'packed digest does not match the tensor shape'
    return out


def digest_err(got, packed, key, gmax):
    """largest deviation between the digest of gradient ``got`` of parameter ``key`` and a stored packed digest, part by part"""
    mine, want = digest(got), unpack(packed, got)
    base = (ZERO_FLOOR if key.endswith(ZERO_GRADS) else FLOOR) * gmax
    err = 0.0
    for k, w in want.items():
        scale = max(float(np.abs(w).max()), base, SUM_NOISE * float(want['abssum'][0]) if k == 'sum' else 0.0)
        err = max(err, float(np.abs(mine[k] - w).max()) / scale)
    return err


def restatement_grads(sd, cfg, ref_points, src_points, ref_feats, src_feats, keys, dtype, device='cpu'):
    """{key: d loss / d sd['transformer.' + key]} plus 'ref_feats' / 'src_feats' of geo_oracle.geometric_transformer in ``dtype``,
    loss = <ref_out, G_0> + <src_out, G_1> with G_i = backbone_grad_oracle.upstream"""
    sd2 = {k: (v.detach().to(device, dtype) if v.is_floating_point() else v.to(device)) for k, v in sd.items()
           if k.startswith('transformer.')}
    leaves = {k: sd2['transformer.' + k].clone().requires_grad_(True) for k in keys}
    sd2.update({'transformer.' + k: v for k, v in leaves.items()})
    f = [t.detach().to(device, dtype).requires_grad_(True) for t in (ref_feats, src_feats)]
    o0, o1 = G.geometric_transformer(sd2, cfg, ref_points.detach().to(device, dtype), src_points.detach().to(device, dtype), f[0], f[1])
    ups = BG.upstream([tuple(o0.shape), tuple(o1.shape)])
    ((o0 * ups[0].to(device, dtype)).sum() + (o1 * ups[1].to(device, dtype)).sum()).backward()
    return dict({k: leaves[k].grad for k in keys}, ref_feats=f[0].grad, src_feats=f[1].grad)
