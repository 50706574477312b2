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
    def forward_batch(self, data_dict, evaluator=None, results=None, side_streams=None, keep_outputs=True, loss_func=None, loss_out=None,
                      ransac=None, ransac_out=None, taps=None):
        """B pairs per forward (``data_dict['batch_size']`` from ``registration_collate_fn_stack_mode``, stack order
        ``[ref_1..ref_B, src_1..src_B]`` at every level) -- the reference asserts batch_size == 1
        (``engine/single_tester.py:39-74``, README "only batch_size=1 is supported").  Backbone and transformer run ONCE over
        the stacked rows of all pairs (per-pair GroupNorm statistics, batched attention launches, one structure-embedding
        launch); the per-pair stages run once for all pairs too (one launch per stage, the pair index in the grid): grouping and
        ground-truth correspondences on the first of ``side_streams`` (overlapping the backbone; without side streams on the
        current stream), matching, Sinkhorn, LGR and the metrics on the current stream.  Backbone and transformer run through
        the native stage drivers after ``enable_native``, else through the modules (one pair only): the drivers' bit-for-bit
        reference.

        Returns a list of per-pair output dicts (``keep_outputs``), trimmed to their counts after one host synchronisation.
        With ``results`` (a (B, 24) float device tensor) the estimated transform (16), the number of LGR correspondences
        (column 22) and, with ``evaluator``, the metrics (8, from column 16) of pair p are written to row p WITHOUT any host
        synchronisation in this call; the output dicts then keep the full-capacity buffers and the device counts under
        ``_counts`` (``trim_outputs``).  With ``loss_func``
        (a geotransformer_b200.loss.OverallLoss) and ``loss_out`` (a (B, 3) float device tensor) the validation losses
        [loss, c_loss, f_loss] of pair p are written to row p of ``loss_out`` after LGR, also without a host synchronisation.
        With ``ransac`` (a config section: distance_threshold, num_points, num_iterations, seed) and ``ransac_out`` (a (B, 26)
        float device tensor) correspondence RANSAC runs on the LGR correspondences of every pair (pair p draws from the stream
        (seed, p)); row p receives [transform (16), fitness, inlier_rmse] and, with ``evaluator``, the metrics (8) of the RANSAC
        transform -- no host synchronisation either.

        Test hooks for one pair: ``taps`` (a dict) receives the pair's ref_/src_ node_masks, node_knn_indices and
        node_knn_masks, the backbone's ``feats_c`` / ``feats_f`` and ``matching_scores_raw`` (before Sinkhorn);
        ``data_dict['forced_node_corr']`` (ref indices, src indices, scores) replaces the superpoint matching."""
        B = int(data_dict.get('batch_size', 1))
        forced = data_dict.get('forced_node_corr')
        if B > 1 and (taps is not None or forced is not None):
            raise ValueError('forward_batch: taps and forced_node_corr apply to one pair per forward')
        native = getattr(self, '_native', None)
        if native is None and B > 1:
            raise RuntimeError('forward_batch of several pairs needs the native stage drivers: call enable_native(model) first')
        dev = data_dict['features'].device
        if forced is not None:
            forced = _forced_node_corr(forced, dev)
        marks = data_dict.get('_stage_events')            # profiling hook: list receiving (label, CUDA event) pairs

        def mark(label):
            if marks is not None:
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                marks.append((label, e))
        mark('start')
        lens_h = data_dict.get('lengths_host') or [l.tolist() for l in data_dict['lengths']]
        fl, K = self.fine_level, self.num_points_in_patch
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
        feats = data_dict['features']
        feats_list = native.backbone_forward(feats, data_dict) if native is not None else self.backbone(feats, data_dict)
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
        if native is not None:
            x = native.transformer_forward_batched(x, rows_c, embs)
        else:
            x = tr.transformer.forward_stacked(x, rows_c[0], embs[0], embs[1])
        y = GF.linear(x, tr.out_proj.weight, tr.out_proj.bias)
        y_n = GF.l2_normalize(y)
        mark('transformer')

        # ---- matching, patches, Sinkhorn, LGR and metrics of all pairs: one launch per stage on the main stream
        join()
        mark('join_grouping+gt')
        cm, fm = self.coarse_matching, self.fine_matching
        if forced is None:
            kc = cm.num_correspondences
            corr, node_scores, corr_count = GF.superpoint_matching_batched(y_n, node_masks, cn, kc, cm.dual_normalization)
        else:
            corr, node_scores = forced
            kc = corr.shape[1]
            corr_count = torch.full((1,), kc, dtype=torch.int32, device=dev)
        k_idx, k_masks, k_pts = GF.gather_patches_batched(corr, kc, cn, cf, knn_idx, knn_masks, points_f)
        r, s = slice(0, B * kc), slice(B * kc, 2 * B * kc)          # patches of the ref clouds, then of the src clouds
        raw_scores = GF.patch_scores_batched(feats_f, cf, k_idx[r], k_idx[s])
        scores = self.optimal_transport(raw_scores, k_masks[r], k_masks[s])
        rc, sc, cs, T, n_corr = GF.local_global_registration_batched(
            B, k_pts[r], k_pts[s], k_masks[r], k_masks[s], scores, fm.k, fm.acceptance_radius, fm.mutual, fm.confidence_threshold,
            fm.correspondence_threshold, fm.num_refinement_steps, transform_out=results if no_sync else None)
        if no_sync:
            if gt is not None and evaluator is not None:
                GF.evaluate_batched(gt[0], gt[1], gt[2], corr, corr_count, rc, sc, n_corr, transforms, results, points0,
                                    cn, [int(v) for v in lens_h[0]], evaluator.mode, evaluator.acceptance_overlap, evaluator.acceptance_radius,
                                    results[:, 16:], evaluator.acceptance_rmse, evaluator.acceptance_rre, evaluator.acceptance_rte)
            else:
                results[:, 22].copy_(n_corr)          # the metrics' #corr column
        if ransac is not None and ransac_out is not None:
            write_ransac_rows(ransac, sc, rc, n_corr, ransac_out)
            if gt is not None and evaluator is not None:
                GF.evaluate_batched(gt[0], gt[1], gt[2], corr, corr_count, rc, sc, n_corr, transforms, ransac_out, points0,
                                    cn, [int(v) for v in lens_h[0]], evaluator.mode, evaluator.acceptance_overlap, evaluator.acceptance_radius,
                                    ransac_out[:, 18:26], evaluator.acceptance_rmse, evaluator.acceptance_rre, evaluator.acceptance_rte)
        if gt is not None and loss_func is not None and loss_out is not None:
            loss_func.write_batched(y_n, cn, gt, k_pts[r], k_pts[s], k_masks[r], k_masks[s], scores, transforms, corr_count, loss_out)
        mark('matching+sinkhorn+lgr+metrics')
        if taps is not None:
            nr = cn[0]
            taps.update(ref_node_masks=node_masks[:nr], src_node_masks=node_masks[nr:], ref_node_knn_indices=knn_idx[:nr],
                        src_node_knn_indices=knn_idx[nr:], ref_node_knn_masks=knn_masks[:nr], src_node_knn_masks=knn_masks[nr:],
                        feats_c=feats_c, feats_f=feats_f, matching_scores_raw=raw_scores)
        if no_sync:
            if not keep_outputs:
                return None
            T = T[:, :16].clone()          # the output dicts outlive the caller's reuse of its result rows
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
        main.synchronize()
        return trim_outputs(outs)

    def forward_train(self, data_dict, seed, iteration, targets=None):
        """The reference's training-mode forward (``experiments/*/model.py``, step 7 "Random select ground truth node
        correspondences during training") of ONE pair (``data_dict['batch_size']`` must be 1, as the reference trains).

        Grouping and ground-truth superpoint correspondences as ``forward_batch``; the backbone and the transformer through the
        modules (the native drivers carry no graph), so ``ref_feats_c`` / ``src_feats_c`` / ``matching_scores`` carry the graph
        to every parameter.  ``ref_/src_node_corr_indices`` hold the superpoint matching (no graph, as the reference; the Evaluator's
        PIR reads them), while the fine-matching patches come from ``superpoint_targets_batched``: at most
        ``cfg.coarse_matching.num_targets`` gt correspondences with overlap > ``overlap_threshold``, drawn from the Philox stream
        (``seed``, ``iteration``, pair 0).  ``targets`` = (ref indices (k',), src indices (k',), overlaps (k',)) replaces the draw.
        LGR runs on the detached scores.  Returns one output dict with full-capacity buffers and the device counts under
        ``_counts``: ``node_corr`` = the target patches (rows of the patch tensors, ``node_corr_scores``, ``matching_scores``),
        ``coarse`` = the superpoint matching rows, ``corr`` = LGR, ``gt`` = ground truth.  No host synchronisation."""
        if int(data_dict.get('batch_size', 1)) != 1:
            raise ValueError('forward_train: one pair per training forward (data_dict["batch_size"] must be 1)')
        transform = data_dict.get('transform')
        if transform is None:
            raise ValueError('forward_train: the training forward needs the ground-truth transform')
        dev = data_dict['features'].device
        if targets is not None:
            targets = _forced_node_corr(targets, dev)
        lens_h = data_dict.get('lengths_host') or [l.tolist() for l in data_dict['lengths']]
        fl, K = self.fine_level, self.num_points_in_patch
        cn, cf, c0 = [int(v) for v in lens_h[-1]], [int(v) for v in lens_h[fl]], [int(v) for v in lens_h[0]]
        points_c, points_f, points0 = data_dict['points'][-1], data_dict['points'][fl], data_dict['points'][0]
        transforms = transform.reshape(1, 4, 4).contiguous()
        n0, nf, np0 = cn[0], cf[0], c0[0]

        _, node_masks, knn_idx, knn_masks = GF.point_to_node_partition_batched(points_f, points_c, cf, cn, K)
        _, _, all_pts = GF.gather_patches_batched(None, 0, cn, cf, knn_idx, knn_masks, points_f)
        gt_idx, gt_ov, gt_cnt = GF.node_correspondences_batched(points_c, all_pts, node_masks, knn_masks, cn, transforms,
                                                                self.matching_radius)

        feats_list = self.backbone(data_dict['features'], data_dict)
        feats_c, feats_f = feats_list[-1], feats_list[0]
        rc, sc = self.transformer(points_c[:n0].contiguous(), points_c[n0:].contiguous(), feats_c[:n0], feats_c[n0:])
        y_n = GF.l2_normalize(torch.cat([rc, sc]))

        cm, fm = self.coarse_matching, self.fine_matching
        with torch.no_grad():
            m_corr, _, m_count = GF.superpoint_matching_batched(y_n.detach(), node_masks, cn, cm.num_correspondences,
                                                                cm.dual_normalization)
            if targets is None:
                kc = self.cfg.coarse_matching.num_targets
                corr, node_scores, corr_count = GF.superpoint_targets_batched(
                    gt_idx, gt_ov, gt_cnt, cn, self.cfg.coarse_matching.overlap_threshold, kc, seed, iteration)
            else:
                corr, node_scores = targets
                kc = corr.shape[1]
                corr_count = torch.full((1,), kc, dtype=torch.int32, device=dev)
            k_idx, k_masks, k_pts = GF.gather_patches_batched(corr, kc, cn, cf, knn_idx, knn_masks, points_f)
        r, s = slice(0, kc), slice(kc, 2 * kc)
        raw_scores = GF.patch_scores_batched(feats_f, cf, k_idx[r], k_idx[s])
        scores = self.optimal_transport(raw_scores, k_masks[r], k_masks[s])
        with torch.no_grad():
            rcp, scp, cs, T, n_corr = GF.local_global_registration_batched(
                1, k_pts[r], k_pts[s], k_masks[r], k_masks[s], scores.detach(), fm.k, fm.acceptance_radius, fm.mutual,
                fm.confidence_threshold, fm.correspondence_threshold, fm.num_refinement_steps)
        return dict(ref_points_c=points_c[:n0], src_points_c=points_c[n0:], ref_points_f=points_f[:nf], src_points_f=points_f[nf:],
                    ref_points=points0[:np0], src_points=points0[np0:], ref_feats_c=y_n[:n0], src_feats_c=y_n[n0:],
                    ref_feats_f=feats_f[:nf], src_feats_f=feats_f[nf:], gt_node_corr_indices=gt_idx, gt_node_corr_overlaps=gt_ov,
                    ref_node_corr_indices=m_corr[0], src_node_corr_indices=m_corr[1], node_corr_scores=node_scores[0],
                    ref_node_corr_knn_points=k_pts[r], src_node_corr_knn_points=k_pts[s], ref_node_corr_knn_masks=k_masks[r],
                    src_node_corr_knn_masks=k_masks[s], matching_scores=scores, ref_corr_points=rcp[0], src_corr_points=scp[0],
                    corr_scores=cs[0], estimated_transform=T[0].reshape(4, 4),
                    _counts=dict(node_corr=corr_count[0], coarse=m_count[0], corr=n_corr[0], gt=gt_cnt[0]),
                    _stacked=dict(gt=(gt_idx, gt_ov, gt_cnt), coarse=(m_corr, m_count), lgr=(rcp, scp, n_corr), transforms=T,
                                  cloud_nodes=cn, cloud_points=c0, points=points0))

    def forward_train_batch(self, data_dict, seed, iteration, targets=None):
        """``forward_train`` of the B pairs of one collated batch (``registration_collate_fn_stack_mode``, stack order
        [ref_1..ref_B, src_1..src_B]), the step the reference gets from B-rank DistributedDataParallel.  Per pair it does what
        ``forward_train`` does; the backbone and the transformer run ONCE over the stacked rows, with a graph to every parameter
        and the kernel sequence of the native drivers' ``forward_batch`` (per-pair GroupNorm statistics, per-pair max-pool widths,
        one structure-embedding launch, batched attention, one in_proj / out_proj GEMM over all rows), so ``feats_c``,
        ``feats_f`` and ``y_n`` are its bits.  Pair p's targets come from the Philox stream (``seed``, ``iteration``, p): one
        ``superpoint_targets_batched`` launch for all pairs.  ``targets``: a list of B (ref indices, src indices, overlaps) tuples
        replacing the draw.

        Returns one dict of stacked full-capacity buffers: ``ref_feats_c`` / ``src_feats_c`` = the ref / src blocks of y_n, the
        gt rows of all pairs, the target patches (pair p's patch q at row p * K + q of the ref / src patch tensors and of
        ``matching_scores``), ``_cloud_nodes`` and the device counts under ``_counts`` ((B,) each), ``_stacked`` for the metrics
        and ``_features`` = (feats_c, feats_f, y_n).  No host synchronisation."""
        B = int(data_dict.get('batch_size', 1))
        transform = data_dict.get('transform')
        if transform is None:
            raise ValueError('forward_train_batch: the training forward needs the ground-truth transforms')
        dev = data_dict['features'].device
        lens_h = data_dict.get('lengths_host') or [l.tolist() for l in data_dict['lengths']]
        fl, K = self.fine_level, self.num_points_in_patch
        cn, cf, c0 = [int(v) for v in lens_h[-1]], [int(v) for v in lens_h[fl]], [int(v) for v in lens_h[0]]
        points_c, points_f, points0 = data_dict['points'][-1], data_dict['points'][fl], data_dict['points'][0]
        transforms = (torch.stack(list(transform)) if isinstance(transform, (list, tuple)) else transform).reshape(B, 4, 4).contiguous()
        R, Rf, R0 = sum(cn[:B]), sum(cf[:B]), sum(c0[:B])

        _, node_masks, knn_idx, knn_masks = GF.point_to_node_partition_batched(points_f, points_c, cf, cn, K)
        _, _, all_pts = GF.gather_patches_batched(None, 0, cn, cf, knn_idx, knn_masks, points_f)
        gt_idx, gt_ov, gt_cnt = GF.node_correspondences_batched(points_c, all_pts, node_masks, knn_masks, cn, transforms,
                                                                self.matching_radius)

        feats_list = self.backbone(data_dict['features'], data_dict)
        feats_c, feats_f = feats_list[-1], feats_list[0]
        y_n = GF.l2_normalize(self.transformer.forward_batched_grad(points_c, feats_c, cn))

        cm, fm = self.coarse_matching, self.fine_matching
        with torch.no_grad():
            m_corr, _, m_count = GF.superpoint_matching_batched(y_n.detach(), node_masks, cn, cm.num_correspondences,
                                                                cm.dual_normalization)
            if targets is None:
                kc = self.cfg.coarse_matching.num_targets
                corr, node_scores, corr_count = GF.superpoint_targets_batched(
                    gt_idx, gt_ov, gt_cnt, cn, self.cfg.coarse_matching.overlap_threshold, kc, seed, iteration)
            else:
                corr, node_scores, corr_count = _forced_targets(targets, B, dev)
                kc = corr.shape[1]
            k_idx, k_masks, k_pts = GF.gather_patches_batched(corr, kc, cn, cf, knn_idx, knn_masks, points_f)
        r, s = slice(0, B * kc), slice(B * kc, 2 * B * kc)
        raw_scores = GF.patch_scores_batched(feats_f, cf, k_idx[r], k_idx[s])
        scores = self.optimal_transport(raw_scores, k_masks[r], k_masks[s])
        with torch.no_grad():
            rcp, scp, cs, T, n_corr = GF.local_global_registration_batched(
                B, k_pts[r], k_pts[s], k_masks[r], k_masks[s], scores.detach(), fm.k, fm.acceptance_radius, fm.mutual,
                fm.confidence_threshold, fm.correspondence_threshold, fm.num_refinement_steps)
        return dict(ref_points_c=points_c[:R], src_points_c=points_c[R:], ref_points_f=points_f[:Rf], src_points_f=points_f[Rf:],
                    ref_points=points0[:R0], src_points=points0[R0:], ref_feats_c=y_n[:R], src_feats_c=y_n[R:],
                    ref_feats_f=feats_f[:Rf], src_feats_f=feats_f[Rf:], gt_node_corr_indices=gt_idx, gt_node_corr_overlaps=gt_ov,
                    node_corr_scores=node_scores, ref_node_corr_knn_points=k_pts[r], src_node_corr_knn_points=k_pts[s],
                    ref_node_corr_knn_masks=k_masks[r], src_node_corr_knn_masks=k_masks[s], matching_scores=scores,
                    matching_scores_raw=raw_scores, target_corr=corr, _cloud_nodes=cn, _features=(feats_c, feats_f, y_n),
                    _counts=dict(node_corr=corr_count, coarse=m_count, corr=n_corr, gt=gt_cnt),
                    _stacked=dict(gt=(gt_idx, gt_ov, gt_cnt), coarse=(m_corr, m_count), lgr=(rcp, scp, n_corr), transforms=T,
                                  gt_transforms=transforms, cloud_nodes=cn, cloud_points=c0, points=points0))

    def forward(self, data_dict, taps=None):
        """``forward_batch`` with its defaults: the output dict of a single pair (the reference's contract), the list of output
        dicts for a batch of several pairs.  ``taps`` and ``data_dict['forced_node_corr']``: see ``forward_batch``."""
        outs = self.forward_batch(data_dict, taps=taps)
        return outs[0] if int(data_dict.get('batch_size', 1)) == 1 else outs


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


def _forced_node_corr(forced, device):
    """teacher-forced coarse correspondences (ref indices (k',), src indices (k',), scores (k',)) -> the superpoint matching's
    layout for one pair: corr (2, k') int64, scores (1, k') float32"""
    ref, src, scores = forced
    for t, dtype, name in ((ref, torch.int64, 'ref indices'), (src, torch.int64, 'src indices'), (scores, torch.float32, 'scores')):
        if t.ndim != 1 or t.dtype != dtype or t.device != device:
            raise ValueError(f'forced_node_corr: the {name} must be a 1-D {dtype} tensor on {device}')
    if not ref.shape[0] == src.shape[0] == scores.shape[0]:
        raise ValueError('forced_node_corr: the ref indices, src indices and scores must have the same length')
    return torch.stack([ref, src]), scores.reshape(1, -1)


def _forced_targets(targets, B, device):
    """per-pair teacher-forced targets [(ref indices (k_p,), src indices (k_p,), overlaps (k_p,))] * B -> the layout of
    ``superpoint_targets_batched``: corr (2B, max k_p) int64 (-1 past a count), scores (B, max k_p) (0 past it), counts (B,) int32"""
    if len(targets) != B:
        raise ValueError(f'forward_train_batch: targets must hold one (ref, src, overlaps) tuple per pair ({B})')
    forced = [_forced_node_corr(t, device) for t in targets]
    k = max(max(c.shape[1] for c, _ in forced), 1)
    corr = torch.full((2 * B, k), -1, dtype=torch.int64, device=device)
    scores = torch.zeros((B, k), dtype=torch.float32, device=device)
    for p, (c, sc) in enumerate(forced):
        n = c.shape[1]
        corr[p, :n], corr[B + p, :n], scores[p, :n] = c[0], c[1], sc[0]
    counts = torch.tensor([c.shape[1] for c, _ in forced], dtype=torch.int32).to(device, non_blocking=True)
    return corr, scores, counts


def trim_outputs(outs):
    """Cut the per-pair output dicts of ``forward_batch(results=...)`` to their device counts and drop ``_counts`` (in place;
    returns ``outs``).  The rows past a count are uninitialised, so call it only after the forward's stream has been
    synchronised."""
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


def write_ransac_rows(ransac, src_corr_points, ref_corr_points, num_corr, out):
    """Correspondence RANSAC (``ransac``: distance_threshold, num_points, num_iterations, seed) of B pairs of (B, capacity, 3)
    correspondences (``num_corr``: (B,) device int32 or None) into columns 0..17 of the (B, >= 18) float rows ``out``:
    [transform (16), fitness, inlier_rmse]; pair p draws from the stream (seed, p).  No host synchronisation."""
    rr = GF.ransac_correspondences_batched(src_corr_points, ref_corr_points, ransac.distance_threshold, ransac.num_points,
                                           ransac.num_iterations, seed=ransac.get('seed', 0), num_corr=num_corr)
    B = out.shape[0]
    out[:, :16].copy_(rr['transform'].reshape(B, 16))
    out[:, 16].copy_(rr['fitness'])
    out[:, 17].copy_(rr['inlier_rmse'])
    return rr
