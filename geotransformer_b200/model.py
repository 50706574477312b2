"""GeoTransformer registration model (inference forward) on the H100 path.

Reference: ``experiments/*/model.py:18-217``.  Same attribute names (``backbone``, ``transformer``,
``coarse_matching``, ``fine_matching``, ``optimal_transport``) and hence the same ``state_dict`` keys; same
``forward(data_dict) -> output_dict`` contract, including ``gt_node_corr_indices/overlaps`` (model.py:112-126, computed
whenever ``data_dict`` carries the ground-truth ``transform``; the reference requires it).
"""
import torch
import torch.nn as nn

from . import _lib
from . import functional as GF
from .backbone import KPConvFPN
from .modules.geotransformer import GeometricTransformer, SuperPointMatching, LocalGlobalRegistration
from .modules.sinkhorn import LearnableLogOptimalTransport


class GeoTransformer(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        self.num_points_in_patch = cfg.model.num_points_in_patch
        self.matching_radius = cfg.model.ground_truth_matching_radius
        self.fine_level = cfg.model.fine_level            # 1 for 3DMatch/KITTI (model.py:77,80), 0 for ModelNet
        b = cfg.backbone
        self.backbone = KPConvFPN(b.input_dim, b.output_dim, b.init_dim, b.kernel_size, b.init_radius, b.init_sigma,
                                  b.group_norm, num_stages=b.num_stages,
                                  finest_decoder=2 if self.fine_level == 1 else 1)
        g = cfg.geotransformer
        self.transformer = GeometricTransformer(g.input_dim, g.output_dim, g.hidden_dim, g.num_heads, g.blocks, g.sigma_d,
                                                g.sigma_a, g.angle_k, reduction_a=g.reduction_a)
        self.coarse_matching = SuperPointMatching(cfg.coarse_matching.num_correspondences,
                                                  cfg.coarse_matching.dual_normalization)
        f = cfg.fine_matching
        self.fine_matching = LocalGlobalRegistration(
            f.topk, f.acceptance_radius, mutual=f.mutual, confidence_threshold=f.confidence_threshold,
            use_dustbin=f.use_dustbin, use_global_score=f.use_global_score,
            correspondence_threshold=f.correspondence_threshold, correspondence_limit=f.correspondence_limit,
            num_refinement_steps=f.num_refinement_steps)
        self.optimal_transport = LearnableLogOptimalTransport(cfg.model.num_sinkhorn_iterations)

    @torch.no_grad()
    def forward_batch(self, data_dict, evaluator=None, results=None, side_streams=None, keep_outputs=True, loss_func=None, loss_out=None):
        """Several pairs per forward (``data_dict['batch_size'] = B > 1`` from ``registration_collate_fn_stack_mode``, stack
        order ``[ref_1..ref_B, src_1..src_B]`` at every level) -- the reference asserts batch_size == 1
        (``engine/single_tester.py:39-74``, README "only batch_size=1 is supported").  Backbone and transformer run ONCE over
        the stacked rows of all pairs (per-pair GroupNorm statistics, batched attention launches, one structure-embedding
        launch); the per-pair stages run once for all pairs too (one launch per stage, the pair index in the grid): grouping and
        ground-truth correspondences on the first of ``side_streams`` (overlapping the backbone), matching, Sinkhorn, LGR and the
        metrics on the current stream.  Per pair the arithmetic is the single-pair forward's.

        Returns a list of per-pair output dicts (``keep_outputs``), each like ``forward``'s.  With ``results`` (a (B, 24)
        float device tensor) the estimated transform (16) and, with ``evaluator``, the metrics (8) of pair p are written to
        row p WITHOUT any host synchronisation in this call (correspondence tensors then stay full-capacity).  With ``loss_func``
        (a geotransformer_b200.loss.OverallLoss) and ``loss_out`` (a (B, 3) float device tensor) the validation losses
        [loss, c_loss, f_loss] of pair p are written to row p of ``loss_out`` after LGR, also without a host synchronisation."""
        native = getattr(self, '_native', None)
        if native is None:
            raise RuntimeError('forward_batch needs the native stage drivers: call enable_native(model) first')
        marks = data_dict.get('_stage_events')            # profiling hook: list receiving (label, CUDA event) pairs

        def mark(label):
            if marks is not None:
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                marks.append((label, e))
        mark('start')
        B = int(data_dict['batch_size'])
        lens_h = data_dict.get('lengths_host') or [l.tolist() for l in data_dict['lengths']]
        fl, K = self.fine_level, self.num_points_in_patch
        dev = data_dict['features'].device
        offs = []
        for lv in lens_h:
            o = [0]
            for v in lv:
                o.append(o[-1] + int(v))
            offs.append(o)
        oc, of, o0 = offs[-1], offs[fl], offs[0]
        points_c, points_f, points0 = data_dict['points'][-1], data_dict['points'][fl], data_dict['points'][0]
        cloud = lambda t, o, c: t[o[c]:o[c + 1]]
        main = torch.cuda.current_stream()
        sides = side_streams or [main]
        no_sync = results is not None

        def fork():
            ev = torch.cuda.Event()
            ev.record(main)
            for s in sides:
                if s is not main:
                    s.wait_event(ev)

        def join():
            for s in sides:
                if s is not main:
                    ev = torch.cuda.Event()
                    ev.record(s)
                    main.wait_event(ev)

        class on:          # run the body on side stream i (also for the ctypes calls: thread-local stream pointer)
            def __init__(self, i):
                self.s = sides[i % len(sides)]
            def __enter__(self):
                self.a = torch.cuda.stream(self.s); self.a.__enter__()
                self.b = _lib.stream_scope(self.s.cuda_stream); self.b.__enter__()
            def __exit__(self, *e):
                self.b.__exit__(*e); self.a.__exit__(*e)

        # ---- grouping of all clouds and ground-truth superpoint correspondences of all pairs (one side stream: overlaps the backbone)
        cn, cf = [int(v) for v in lens_h[-1]], [int(v) for v in lens_h[fl]]
        transforms = data_dict.get('transform')
        if transforms is not None:
            transforms = (torch.stack(list(transforms)) if isinstance(transforms, (list, tuple)) else transforms).reshape(B, 4, 4).contiguous()
        gt = None
        fork()
        with on(0):
            _, node_masks, knn_idx, knn_masks = GF.point_to_node_partition_batched(points_f, points_c, cf, cn, K)
            if transforms is not None:
                _, _, all_pts = GF.gather_patches_batched(None, 0, cn, cf, knn_idx, knn_masks, points_f)
                gt = GF.node_correspondences_batched(points_c, all_pts, node_masks, knn_masks, cn, transforms, self.matching_radius)

        # ---- backbone over all pairs (main stream, overlaps the grouping)
        feats_list = native.backbone_forward(data_dict['features'], data_dict)
        feats_c, feats_f = feats_list[-1], feats_list[0]
        mark('backbone')

        # ---- structure embeddings of all clouds in one launch, transformer over all rows
        tr = self.transformer
        emb_mod = tr.embedding
        rows_c = [int(v) for v in lens_h[-1]]
        n2 = [r * r for r in rows_c]
        eo = [0]
        for v in n2:
            eo.append(eo[-1] + v)
        C = tr.in_proj.out_features
        d_all = GF.scratch((eo[-1],), dev, 'gse_d_all')
        a_all = GF.scratch((eo[-1], emb_mod.angle_k), dev, 'gse_a_all')
        E_all = GF.scratch((eo[-1], C), dev, 'gse_E_all')
        GF.gse_indices_batched(points_c, rows_c, emb_mod.sigma_d, emb_mod.sigma_a, emb_mod.angle_k, d_all, a_all)
        wd_t = emb_mod._cache.get('wd_t', emb_mod.proj_d.weight, lambda w: w.t().contiguous())
        wa_t = emb_mod._cache.get('wa_t', emb_mod.proj_a.weight, lambda w: w.t().contiguous())
        GF.gse_embed_flat(d_all, a_all, eo[-1], emb_mod.embedding.div_term, emb_mod.proj_d.weight.detach(), emb_mod.proj_a.weight.detach(),
                          emb_mod.proj_d.bias.detach(), emb_mod.proj_a.bias.detach(), wd_t, wa_t, E_all, table=emb_mod.table())
        embs = [E_all[eo[c]:eo[c + 1]] for c in range(2 * B)]
        mark('structure_embedding')
        x = GF.linear(feats_c, tr.in_proj.weight, tr.in_proj.bias)
        x = native.transformer_forward_batched(x, rows_c, embs)
        y = GF.linear(x, tr.out_proj.weight, tr.out_proj.bias)
        y_n = GF.l2_normalize(y)
        mark('transformer')

        # ---- matching, patches, Sinkhorn, LGR and metrics of all pairs: one launch per stage on the main stream
        join()
        mark('join_grouping+gt')
        cm, fm = self.coarse_matching, self.fine_matching
        kc = cm.num_correspondences
        corr, node_scores, corr_count = GF.superpoint_matching_batched(y_n, node_masks, cn, kc, cm.dual_normalization)
        k_idx, k_masks, k_pts = GF.gather_patches_batched(corr, kc, cn, cf, knn_idx, knn_masks, points_f)
        r, s = slice(0, B * kc), slice(B * kc, 2 * B * kc)          # patches of the ref clouds, then of the src clouds
        scores = GF.patch_scores_batched(feats_f, cf, k_idx[r], k_idx[s])
        scores = self.optimal_transport(scores, k_masks[r], k_masks[s])
        rc, sc, cs, T, n_corr = GF.local_global_registration_batched(
            B, k_pts[r], k_pts[s], k_masks[r], k_masks[s], scores, fm.k, fm.acceptance_radius, fm.mutual, fm.confidence_threshold,
            fm.correspondence_threshold, fm.num_refinement_steps, transform_out=results if no_sync else None)
        if gt is not None and evaluator is not None and no_sync:
            GF.evaluate_batched(gt[0], gt[1], gt[2], corr, corr_count, rc, sc, n_corr, transforms, results, points0,
                                cn, [int(v) for v in lens_h[0]], evaluator.mode, evaluator.acceptance_overlap, evaluator.acceptance_radius,
                                results[:, 16:], evaluator.acceptance_rmse, evaluator.acceptance_rre, evaluator.acceptance_rte)
        if gt is not None and loss_func is not None and loss_out is not None:
            loss_func.write_batched(y_n, cn, gt, k_pts[r], k_pts[s], k_masks[r], k_masks[s], scores, transforms, corr_count, loss_out)
        mark('matching+sinkhorn+lgr+metrics')
        if no_sync and not keep_outputs:
            return None
        outs = []
        g0 = 0
        for p in range(B):
            pr, ps = slice(p * kc, (p + 1) * kc), slice((B + p) * kc, (B + p + 1) * kc)
            o = dict(ref_points_c=cloud(points_c, oc, p), src_points_c=cloud(points_c, oc, B + p), ref_points_f=cloud(points_f, of, p),
                     src_points_f=cloud(points_f, of, B + p), ref_points=cloud(points0, o0, p), src_points=cloud(points0, o0, B + p),
                     ref_feats_c=cloud(y_n, oc, p), src_feats_c=cloud(y_n, oc, B + p), ref_feats_f=cloud(feats_f, of, p),
                     src_feats_f=cloud(feats_f, of, B + p), ref_node_corr_indices=corr[p], src_node_corr_indices=corr[B + p],
                     node_corr_scores=node_scores[p], ref_node_corr_knn_points=k_pts[pr], src_node_corr_knn_points=k_pts[ps],
                     ref_node_corr_knn_masks=k_masks[pr], src_node_corr_knn_masks=k_masks[ps], matching_scores=scores[pr],
                     ref_corr_points=rc[p], src_corr_points=sc[p], corr_scores=cs[p], estimated_transform=T[p, :16].reshape(4, 4),
                     _counts=dict(node_corr=corr_count[p], corr=n_corr[p], gt=None if gt is None else gt[2][p]))
            if gt is not None:
                g1 = g0 + cn[p] * cn[B + p]
                o['gt_node_corr_indices'], o['gt_node_corr_overlaps'] = gt[0][g0:g1], gt[1][g0:g1]
                g0 = g1
            outs.append(o)
        if no_sync:
            return outs
        # trim the capacity tensors to the counts (one host sync for the whole batch)
        main.synchronize()
        for o in outs:
            cnt = o.pop('_counts')
            kk, c = int(cnt['node_corr'].item()), int(cnt['corr'].item())
            for key in ('ref_node_corr_indices', 'src_node_corr_indices', 'node_corr_scores', 'ref_node_corr_knn_points',
                        'src_node_corr_knn_points', 'ref_node_corr_knn_masks', 'src_node_corr_knn_masks', 'matching_scores'):
                o[key] = o[key][:kk]
            for key in ('ref_corr_points', 'src_corr_points', 'corr_scores'):
                o[key] = o[key][:c]
            if cnt['gt'] is not None:
                g = int(cnt['gt'].item())
                o['gt_node_corr_indices'], o['gt_node_corr_overlaps'] = o['gt_node_corr_indices'][:g], o['gt_node_corr_overlaps'][:g]
        return outs

    @torch.no_grad()
    def forward(self, data_dict, taps=None):
        if int(data_dict.get('batch_size', 1)) > 1:
            return self.forward_batch(data_dict)
        out = {}
        marks = data_dict.get('_stage_events')            # profiling hook: list receiving (label, CUDA event) pairs
        def mark(label):
            if marks is not None:
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                marks.append((label, e))
        mark('start')
        feats = data_dict['features']
        lens = data_dict['lengths']
        fl = self.fine_level
        # lengths are needed on the host to slice ref/src (the reference does three .item() syncs, model.py:76-78);
        # the collate keeps host copies so no sync happens here
        lens_h = data_dict.get('lengths_host')
        if lens_h is None:
            lens_h = [l.tolist() for l in lens]
        nc, nf, n0 = int(lens_h[-1][0]), int(lens_h[fl][0]), int(lens_h[0][0])
        points_c, points_f, points = data_dict['points'][-1], data_dict['points'][fl], data_dict['points'][0]
        ref_c, src_c = points_c[:nc], points_c[nc:]
        ref_f, src_f = points_f[:nf], points_f[nf:]
        out.update(ref_points_c=ref_c, src_points_c=src_c, ref_points_f=ref_f, src_points_f=src_f,
                   ref_points=points[:n0], src_points=points[n0:])

        K = self.num_points_in_patch
        _, ref_node_masks, ref_knn_idx, ref_knn_masks = GF.point_to_node_partition(ref_f, ref_c, K)
        _, src_node_masks, src_knn_idx, src_knn_masks = GF.point_to_node_partition(src_f, src_c, K)
        if taps is not None:
            taps.update(ref_node_masks=ref_node_masks, src_node_masks=src_node_masks, ref_node_knn_indices=ref_knn_idx,
                        src_node_knn_indices=src_knn_idx, ref_node_knn_masks=ref_knn_masks, src_node_knn_masks=src_knn_masks)

        # ground-truth superpoint correspondences (reference model.py:106-126).  Launched here, read back after the last
        # host sync of the forward so that it costs no extra synchronisation.
        gt_pending = None
        transform = data_dict.get('transform')
        if transform is not None:
            ar_r = GF.scratch_arange(ref_c.shape[0], ref_c.device, 'ar_ref')
            ar_s = GF.scratch_arange(src_c.shape[0], src_c.device, 'ar_src')
            _, _, ref_all_pts = GF.gather_patches(ar_r, ref_knn_idx, ref_knn_masks, ref_f)
            _, _, src_all_pts = GF.gather_patches(ar_s, src_knn_idx, src_knn_masks, src_f)
            gt_pending = GF.node_correspondences(ref_c, src_c, ref_all_pts, src_all_pts, transform, self.matching_radius,
                                                 ref_node_masks, src_node_masks, ref_knn_masks, src_knn_masks)

        mark('partition+gt')
        native = getattr(self, '_native', None)          # NativeModel: backbone / transformer as one C call each
        feats_list = native.backbone_forward(feats, data_dict) if native is not None else self.backbone(feats, data_dict)
        feats_c, feats_f = feats_list[-1], feats_list[0]
        mark('backbone')
        if taps is not None:
            taps['feats_c'], taps['feats_f'] = feats_c, feats_f

        ref_fc, src_fc = self.transformer(ref_c, src_c, feats_c[:nc], feats_c[nc:], native=native)
        mark('transformer')
        ref_fc_n, src_fc_n = GF.l2_normalize(ref_fc), GF.l2_normalize(src_fc)
        ref_ff, src_ff = feats_f[:nf], feats_f[nf:]
        out.update(ref_feats_c=ref_fc_n, src_feats_c=src_fc_n, ref_feats_f=ref_ff, src_feats_f=src_ff)

        # fewer than num_correspondences rows exist only when #valid ref x #valid src superpoints is smaller (tiny clouds):
        # the count stays on the device, the padding rows become empty patches (no fine correspondences, so LGR is
        # unaffected) and the per-patch outputs are trimmed after the forward's last host sync
        ref_corr, src_corr, node_scores, corr_count = self.coarse_matching(ref_fc_n, src_fc_n, ref_node_masks, src_node_masks,
                                                                           defer_count=True)
        forced = data_dict.get('forced_node_corr')       # test hook: teacher-forced coarse correspondences
        if forced is not None:
            ref_corr, src_corr, node_scores = forced
            corr_count = None
        out.update(ref_node_corr_indices=ref_corr, src_node_corr_indices=src_corr, node_corr_scores=node_scores)

        rk_idx, rk_masks, rk_pts = GF.gather_patches(ref_corr, ref_knn_idx, ref_knn_masks, ref_f)
        sk_idx, sk_masks, sk_pts = GF.gather_patches(src_corr, src_knn_idx, src_knn_masks, src_f)
        out.update(ref_node_corr_knn_points=rk_pts, src_node_corr_knn_points=sk_pts, ref_node_corr_knn_masks=rk_masks,
                   src_node_corr_knn_masks=sk_masks)

        scores = GF.patch_scores(ref_ff, src_ff, rk_idx, sk_idx)
        if taps is not None:
            taps['matching_scores_raw'] = scores
        scores = self.optimal_transport(scores, rk_masks, sk_masks)
        out['matching_scores'] = scores
        mark('matching+sinkhorn')

        rc, sc, cs, T = self.fine_matching(rk_pts, sk_pts, rk_masks, sk_masks, scores, node_scores)
        out.update(ref_corr_points=rc, src_corr_points=sc, corr_scores=cs, estimated_transform=T)
        mark('lgr')
        if gt_pending is not None:
            out['gt_node_corr_indices'], out['gt_node_corr_overlaps'] = GF.finish_node_correspondences(*gt_pending)
        if corr_count is not None:
            kk = int(corr_count.item())          # already complete: LGR synchronised the stream
            if kk < ref_corr.shape[0]:
                for key in ('ref_node_corr_indices', 'src_node_corr_indices', 'node_corr_scores', 'ref_node_corr_knn_points',
                            'src_node_corr_knn_points', 'ref_node_corr_knn_masks', 'src_node_corr_knn_masks', 'matching_scores'):
                    out[key] = out[key][:kk]
        return out


def enable_native(model):
    """Attach the C++ stage drivers (geotransformer_b200.native): same kernels and results, ~10x less host time per pair.
    Call after the weights are loaded and the model is on its device."""
    from .native import NativeModel
    model._native = NativeModel(model)
    if not getattr(model, '_native_hook', False):
        # NativeModel snapshots pointers AND derived copies (fused q|k|v weights, transposes): rebuild it whenever new
        # weights are loaded, otherwise the raw parameters would update in place while the derived copies stayed stale
        def _rebuild(module, incompatible_keys):
            if getattr(module, '_native', None) is not None:
                module._native = NativeModel(module)
        model.register_load_state_dict_post_hook(_rebuild)
        model._native_hook = True
    return model


def create_model(cfg):
    return GeoTransformer(cfg)
