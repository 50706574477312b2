"""``geotransformer.modules.geotransformer`` on the H100 path: same class names, constructor/forward signatures and
``state_dict`` keys as the reference (``geotransformer/modules/geotransformer/{geotransformer.py:9-155,
superpoint_matching.py:7-50, local_global_registration.py:11-235}``)."""
import threading

import torch
import torch.nn as nn

from ... import functional as GF
from ..transformer.modules import SinusoidalPositionalEmbedding, RPEConditionalTransformer, _WeightCache


_TABLE_LOCK = threading.Lock()     # module-level: a lock inside the nn.Module would break deepcopy / pickling of the model


class GeometricStructureEmbedding(nn.Module):
    """reference ``geotransformer.py:9-72``."""

    def __init__(self, hidden_dim, sigma_d, sigma_a, angle_k, reduction_a='max'):
        super().__init__()
        if reduction_a != 'max':
            raise NotImplementedError("only reduction_a='max' (every shipped config) is implemented")
        self.sigma_d, self.sigma_a, self.angle_k, self.reduction_a = sigma_d, sigma_a, angle_k, reduction_a
        self.embedding = SinusoidalPositionalEmbedding(hidden_dim)
        self.proj_d = nn.Linear(hidden_dim, hidden_dim)
        self.proj_a = nn.Linear(hidden_dim, hidden_dim)
        self._cache = _WeightCache()
        self._table = None

    def table(self):
        """``functional.GseTable`` of the current projection weights when the tabulated mode (``GF.GSE_MODE == 5``) is on, else
        None.  Rebuilt when any of the four parameters changes (version counters) or the grid settings do; built once and
        complete before it is returned, so the engine's lanes (host thread + stream each) can share it."""
        c = self.proj_d.out_features
        if GF.GSE_MODE != 5 or c not in (128, 256):
            return None
        return self._weights_table()

    def _weights_table(self, sync=True):
        """the version-keyed table of ``table`` whatever GF.GSE_MODE: the structure embedding's backward picks the winning angle
        term with its lookups.  ``sync=False`` (the training forward, after every optimizer step) builds it without waiting for the
        device: it is then used on the current stream only, and the first ``sync`` caller waits for its build."""
        params = (self.proj_d.weight, self.proj_d.bias, self.proj_a.weight, self.proj_a.bias)
        key = tuple((p.data_ptr(), p._version) for p in params) + (GF.GSE_TABLE_INV_STEP, GF.GSE_TABLE_D_MAX, float(self.sigma_a))
        hit = self._table
        if hit is None or hit[0] != key or (sync and hit[2] is not None):
            with _TABLE_LOCK:
                hit = self._table
                if hit is None or hit[0] != key:
                    wd_t = self.proj_d.weight.detach().t().contiguous()
                    wa_t = self.proj_a.weight.detach().t().contiguous()
                    tab = GF.gse_table(self.embedding.div_term, wd_t, wa_t, self.proj_d.bias.detach().contiguous(),
                                       self.proj_a.bias.detach().contiguous(), self.sigma_a, sync=sync)
                    built = None
                    if not sync:
                        built = torch.cuda.Event()
                        built.record()
                    hit = (key, tab, built)
                    self._table = hit
                elif sync and hit[2] is not None:
                    hit[2].synchronize()
                    hit = (hit[0], hit[1], None)
                    self._table = hit
        return hit[1]

    @torch.no_grad()
    def get_embedding_indices(self, points):
        """points (B=1, N, 3) or (N, 3) -> d_indices (.., N, N), a_indices (.., N, N, k)."""
        squeeze = points.ndim == 3
        pts = points[0] if squeeze else points
        d, a = GF.gse_indices(pts.contiguous(), self.sigma_d, self.sigma_a, self.angle_k)
        return (d.unsqueeze(0), a.unsqueeze(0)) if squeeze else (d, a)

    def forward(self, points, scratch_tag=None):
        """``scratch_tag``: write E into the grow-only scratch buffer of that name (valid until the next call with the same
        tag on this stream) instead of a fresh allocation; used by GeometricTransformer for its two embeddings.  E carries no
        graph: ``forward_grad`` is the differentiable form."""
        squeeze = points.ndim == 3
        if squeeze and points.shape[0] != 1:
            raise NotImplementedError('one cloud per call (the reference model always passes B=1)')
        pts = (points[0] if squeeze else points).contiguous()
        d, a = GF.gse_indices(pts, self.sigma_d, self.sigma_a, self.angle_k)
        wd_t = self._cache.get('wd_t', self.proj_d.weight, lambda w: w.t().contiguous())
        wa_t = self._cache.get('wa_t', self.proj_a.weight, lambda w: w.t().contiguous())
        n, c = pts.shape[0], self.proj_d.out_features
        out = GF.scratch((n, n, c), pts.device, scratch_tag) if scratch_tag is not None else None
        emb = GF.gse_embed(d, a, self.embedding.div_term, self.proj_d.weight.detach(), self.proj_a.weight.detach(),
                           self.proj_d.bias.detach(), self.proj_a.bias.detach(), wd_t, wa_t, out=out, table=self.table())
        return emb.unsqueeze(0) if squeeze else emb

    def forward_grad(self, points):
        """``forward`` of one (N, 3) cloud with the graph to proj_d / proj_a (when they require grad in grad mode): E is a fresh tensor
        the backward keeps (not a scratch view), computed by the same kernels, so its values are ``forward``'s bit for bit.  GeometricTransformer uses it in grad
        mode; the backward takes the winning angle terms from the table of the current weights whatever GF.GSE_MODE."""
        pts = points.contiguous()
        d, a = GF.gse_indices(pts, self.sigma_d, self.sigma_a, self.angle_k)
        wd_t = self._cache.get('wd_t', self.proj_d.weight, lambda w: w.t().contiguous())
        wa_t = self._cache.get('wa_t', self.proj_a.weight, lambda w: w.t().contiguous())
        return GF.gse_embed(d, a, self.embedding.div_term, self.proj_d.weight, self.proj_a.weight, self.proj_d.bias, self.proj_a.bias,
                            wd_t, wa_t, table=self._weights_table())

    def forward_flat_grad(self, points, cloud_rows):
        """The structure embeddings of several stacked clouds (``cloud_rows``: their row counts) as ONE flat (sum n_c^2, C) tensor,
        cloud after cloud, with the graph to proj_d / proj_a: one ``gse_indices_batched`` and one ``gse_embed_flat`` launch, the
        kernels of the batched forward (``GeoTransformer.forward_batch``), so the values are its bits.  The backward
        (``geob200_gse_embed_backward``) sums over all rows of all clouds."""
        rows = [int(r) for r in cloud_rows]
        n2 = sum(r * r for r in rows)
        dev = points.device
        d = torch.empty((n2,), dtype=torch.float32, device=dev)
        a = torch.empty((n2, self.angle_k), dtype=torch.float32, device=dev)
        GF.gse_indices_batched(points, rows, self.sigma_d, self.sigma_a, self.angle_k, d, a)
        wd_t = self._cache.get('wd_t', self.proj_d.weight, lambda w: w.t().contiguous())
        wa_t = self._cache.get('wa_t', self.proj_a.weight, lambda w: w.t().contiguous())
        p = (self.proj_d.weight, self.proj_a.weight, self.proj_d.bias, self.proj_a.bias)
        if GF._needs_grad(*p):
            return GF.gse_embed_flat(d, a, n2, self.embedding.div_term, *p, wd_t, wa_t, None, table=self._weights_table(sync=False))
        out = torch.empty((n2, self.proj_d.out_features), dtype=torch.float32, device=dev)
        return GF.gse_embed_flat(d, a, n2, self.embedding.div_term, *(t.detach() for t in p), wd_t, wa_t, out, table=self.table())


class GeometricTransformer(nn.Module):
    """reference ``geotransformer.py:75-155``."""

    def __init__(self, input_dim, output_dim, hidden_dim, num_heads, blocks, sigma_d, sigma_a, angle_k, dropout=None,
                 activation_fn='ReLU', reduction_a='max'):
        super().__init__()
        self.embedding = GeometricStructureEmbedding(hidden_dim, sigma_d, sigma_a, angle_k, reduction_a=reduction_a)
        self.in_proj = nn.Linear(input_dim, hidden_dim)
        self.transformer = RPEConditionalTransformer(blocks, hidden_dim, num_heads, dropout=dropout,
                                                     activation_fn=activation_fn)
        self.out_proj = nn.Linear(hidden_dim, output_dim)

    def forward(self, ref_points, src_points, ref_feats, src_feats, ref_masks=None, src_masks=None):
        if ref_masks is not None or src_masks is not None:
            raise NotImplementedError('masks are None on the inference path (EXP*/model.py:135-140)')
        batched = ref_points.ndim == 3
        if batched:
            ref_points, src_points, ref_feats, src_feats = ref_points[0], src_points[0], ref_feats[0], src_feats[0]
        if GF._needs_grad(ref_feats, src_feats, *self.parameters()):
            # the graph's attention nodes keep E: fresh tensors, never the scratch the next forward overwrites (also with a frozen
            # embedding, when forward_grad runs the no-grad kernels into a fresh tensor)
            ref_emb, src_emb = self.embedding.forward_grad(ref_points), self.embedding.forward_grad(src_points)
        else:
            ref_emb = self.embedding(ref_points, scratch_tag='gse_ref')     # consumed inside this forward only
            src_emb = self.embedding(src_points, scratch_tag='gse_src')
        n0, n1 = ref_feats.shape[0], src_feats.shape[0]
        # both clouds share every weight: keep them stacked [ref; src] through the whole transformer
        x = torch.empty((n0 + n1, self.in_proj.out_features), dtype=torch.float32, device=ref_feats.device)
        GF.linear(ref_feats, self.in_proj.weight, self.in_proj.bias, out=x[:n0])
        GF.linear(src_feats, self.in_proj.weight, self.in_proj.bias, out=x[n0:])
        x = self.transformer.forward_stacked(x, n0, ref_emb, src_emb)
        y = GF.linear(x, self.out_proj.weight, self.out_proj.bias)
        rf, sf = y[:n0], y[n0:]
        if batched:
            return rf.unsqueeze(0), sf.unsqueeze(0)
        return rf, sf


    def forward_batched_grad(self, points_c, feats_c, cloud_rows):
        """The transformer (with in_proj and out_proj, before the L2 normalisation) over the stacked superpoints of B pairs (stack order
        [ref_1..ref_B, src_1..src_B], ``cloud_rows``: the 2B row counts), with the graph to every parameter and to ``feats_c``: the
        kernels of the batched native forward in its order (one structure-embedding launch for all clouds, one in_proj / out_proj
        GEMM over all rows, ``RPEConditionalTransformer.forward_batched_grad``)."""
        E = self.embedding.forward_flat_grad(points_c, cloud_rows)
        x = GF.linear(feats_c, self.in_proj.weight, self.in_proj.bias)
        x = self.transformer.forward_batched_grad(x, cloud_rows, E)
        return GF.linear(x, self.out_proj.weight, self.out_proj.bias)


class SuperPointMatching(nn.Module):
    """reference ``superpoint_matching.py:7-50``."""

    def __init__(self, num_correspondences, dual_normalization=True):
        super().__init__()
        self.num_correspondences, self.dual_normalization = num_correspondences, dual_normalization

    def forward(self, ref_feats, src_feats, ref_masks=None, src_masks=None):
        return GF.superpoint_matching(ref_feats, src_feats, ref_masks, src_masks, self.num_correspondences,
                                      self.dual_normalization)


class LocalGlobalRegistration(nn.Module):
    """reference ``local_global_registration.py:11-235``."""

    def __init__(self, k, acceptance_radius, mutual=True, confidence_threshold=0.05, use_dustbin=False,
                 use_global_score=False, correspondence_threshold=3, correspondence_limit=None, num_refinement_steps=5):
        super().__init__()
        if use_dustbin or use_global_score or correspondence_limit is not None:
            raise NotImplementedError('use_dustbin / use_global_score / correspondence_limit are off in every shipped config')
        self.k, self.acceptance_radius, self.mutual = k, acceptance_radius, mutual
        self.confidence_threshold, self.use_dustbin, self.use_global_score = confidence_threshold, use_dustbin, use_global_score
        self.correspondence_threshold, self.correspondence_limit = correspondence_threshold, correspondence_limit
        self.num_refinement_steps = num_refinement_steps

    def forward(self, ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, score_mat, global_scores,
                return_details=False):
        """score_mat: (B, K, K) or (B, K+1, K+1) log-assignment (a dustbin row/column is ignored in place, so the
        caller does not need to slice -- a slice is accepted too, it is made contiguous)."""
        return GF.local_global_registration(ref_knn_points.contiguous(), src_knn_points.contiguous(), ref_knn_masks.contiguous(),
                                            src_knn_masks.contiguous(), score_mat.contiguous(), self.k, self.acceptance_radius,
                                            self.mutual, self.confidence_threshold, self.correspondence_threshold,
                                            self.num_refinement_steps, return_details=return_details)
