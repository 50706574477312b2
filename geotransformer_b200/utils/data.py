"""Stack-mode collate on the GPU (reference ``geotransformer/utils/data.py:13-77,139-189``).

The reference runs this on CPU inside DataLoader worker processes (single-threaded C++ ops); CUDA cannot be used in
forked workers, so here the raw pair is moved to the device and collated in the main process on the current stream
(the reference already has the switch for handing raw pairs through: ``precompute_data=False``, ``data.py:181-186``).
"""
import ctypes

import numpy as np
import torch

from ..modules.ops import grid_subsample, radius_search_deferred


def precompute_data_stack_mode(points, lengths, num_stages, voxel_size, radius, neighbor_limits):
    """reference ``utils/data.py:13-77``.  ``lengths`` may live on the host or the device; host copies of every level's
    lengths are returned under ``lengths_host`` so that later stages need no device->host sync."""
    assert num_stages == len(neighbor_limits)
    points_list, lengths_list, lengths_host = [], [], []
    for i in range(num_stages):
        if i > 0:
            points, lengths = grid_subsample(points, lengths_host[-1], voxel_size=voxel_size)
        lengths_h = lengths.cpu() if lengths.is_cuda else lengths
        points_list.append(points)
        lengths_host.append(lengths_h)
        lengths_list.append(lengths_h.to(points.device))
        voxel_size *= 2

    # all 3S-2 searches are launched back to back at their full `limit` width; the reference's row width is
    # min(limit, max neighbour count) (radius_search.py:25-26), so the max counts are read back ONCE at the end and only
    # the tables that are narrower than their limit are cut (rare: the coarsest level)
    pending = []
    for i in range(num_stages):
        cur_points, cur_lengths = points_list[i], lengths_host[i]
        pending.append(('n', radius_search_deferred(cur_points, cur_points, cur_lengths, cur_lengths, radius, neighbor_limits[i])))
        if i < num_stages - 1:
            sub_points, sub_lengths = points_list[i + 1], lengths_host[i + 1]
            pending.append(('s', radius_search_deferred(sub_points, cur_points, sub_lengths, cur_lengths, radius, neighbor_limits[i])))
            pending.append(('u', radius_search_deferred(cur_points, sub_points, cur_lengths, sub_lengths, radius * 2,
                                                        neighbor_limits[i + 1])))
        radius *= 2
    counts = torch.stack([p[1][1] for p in pending]).cpu().flatten().tolist()      # the single D2H of the searches
    neighbors_list, subsampling_list, upsampling_list = [], [], []
    for (kind, (table, _)), mc in zip(pending, counts):
        if mc < 0:
            raise RuntimeError('radius_search: more than 16384 neighbours for one query')
        if mc < table.shape[1]:
            table = table[:, :mc].contiguous()
        {'n': neighbors_list, 's': subsampling_list, 'u': upsampling_list}[kind].append(table)
    return {'points': points_list, 'lengths': lengths_list, 'lengths_host': [l.tolist() for l in lengths_host],
            'neighbors': neighbors_list, 'subsampling': subsampling_list, 'upsampling': upsampling_list}


def _stack_to_device(tensors, device):
    """torch.cat(tensors).to(device) without the host-side concatenation"""
    if all(t.is_cuda for t in tensors):
        return tensors[0] if len(tensors) == 1 else torch.cat(tensors, dim=0)
    total = sum(int(t.shape[0]) for t in tensors)
    out = torch.empty((total,) + tuple(tensors[0].shape[1:]), dtype=tensors[0].dtype, device=device)
    row = 0
    for t in tensors:
        out[row:row + t.shape[0]].copy_(t, non_blocking=True)
        row += t.shape[0]
    return out


def registration_collate_fn_stack_mode(data_dicts, num_stages, voxel_size, search_radius, neighbor_limits,
                                       precompute_data=True, device='cuda'):
    """reference ``utils/data.py:139-189``: points are stacked ``[ref_1..ref_B, src_1..src_B]``."""
    batch_size = len(data_dicts)
    collated = {}
    for d in data_dicts:
        for key, value in d.items():
            if isinstance(value, np.ndarray):
                value = torch.from_numpy(value)
            collated.setdefault(key, []).append(value)
    feats_list = collated.pop('ref_feats') + collated.pop('src_feats')
    points_list = collated.pop('ref_points') + collated.pop('src_points')
    lengths = torch.LongTensor([p.shape[0] for p in points_list])
    if batch_size == 1:
        for key, value in collated.items():
            collated[key] = value[0]
    # one H2D per tensor (asynchronous from pinned staging) straight into the stacked device tensors: no host-side
    # torch.cat (a pageable temporary would also make the copy synchronous).  The reference stacks on the host and
    # moves everything later in to_cuda (utils/torch.py:113-123).
    def _dev(v):
        if isinstance(v, torch.Tensor):
            return v.to(device, non_blocking=True)
        if isinstance(v, list) and v and all(isinstance(x, torch.Tensor) for x in v):      # batch_size > 1: one entry per pair
            return [x.to(device, non_blocking=True) for x in v]
        return v
    collated = {k: _dev(v) for k, v in collated.items()}
    points, feats = _stack_to_device(points_list, device), _stack_to_device(feats_list, device)
    collated['features'] = feats
    if precompute_data:
        collated.update(precompute_data_stack_mode(points, lengths, num_stages, voxel_size, search_radius, neighbor_limits))
    else:
        collated['points'] = points
        collated['lengths'] = lengths
    collated['batch_size'] = batch_size
    return collated


def calibrate_neighbors_stack_mode(dataset, collate_fn, num_stages, voxel_size, search_radius, keep_ratio=0.8, sample_threshold=2000):
    """reference ``utils/data.py:190-217``: neighbour limits = the keep_ratio quantile of the neighbourhood sizes per stage.
    The collate runs on the GPU at the histogram width and the row counts are histogrammed on the device
    (`geob200_neighbor_histogram`); only the (num_stages, hist_n) table comes back, once per sample, for the early exit."""
    from .. import _lib as L
    hist_n = int(np.ceil(4 / 3 * np.pi * (search_radius / voxel_size + 1) ** 3))
    max_neighbor_limits = [hist_n] * num_stages
    hists = None
    lib = L.lib()
    for i in range(len(dataset)):
        data_dict = collate_fn([dataset[i]], num_stages, voxel_size, search_radius, max_neighbor_limits, precompute_data=True)
        if hists is None:
            hists = torch.zeros((num_stages, hist_n), dtype=torch.int32, device=data_dict['neighbors'][0].device)
        for s, neighbors in enumerate(data_dict['neighbors']):
            # support = query cloud of the same stage: the sentinel is the number of rows (data.py:205)
            L.check(lib.geob200_neighbor_histogram(neighbors.data_ptr(), neighbors.shape[0], neighbors.shape[1], neighbors.shape[0],
                                                   hist_n, hists[s].data_ptr(), L.stream_ptr()), 'neighbor_histogram')
        if int(hists.sum(dim=1).min().item()) > sample_threshold:
            break
    neighbor_hists = hists.cpu().numpy()
    cum_sum = np.cumsum(neighbor_hists.T, axis=0)
    neighbor_limits = np.sum(cum_sum < (keep_ratio * cum_sum[hist_n - 1, :]), axis=0)
    return neighbor_limits


# the augmentation "iteration" of the calibration's draws: training iterations count up from 1, so they never reach it
CALIBRATION_ITERATION = (1 << 64) - 1
HIST_MAX_PAIRS = 32         # GEOB200_HIST_MAX_PAIRS


def calibrate_neighbors_augmented(pairs, cfg, seed, keep_ratio=0.8, sample_threshold=2000, chunk=16, device=None):
    """the reference's ``calibrate_neighbors_stack_mode(train_dataset, ...)`` on the AUGMENTED training set: pair p is augmented
    as ``augment.augment_stacked`` draws it from the streams (seed, CALIBRATION_ITERATION, p), and the histograms stop at the first
    pair after which every stage has more than ``sample_threshold`` rows, as the reference's loop does.  ``chunk`` pairs are
    augmented and collated at the histogram width in one go (``geob200_neighbor_histogram_batched``), with one read-back per
    chunk.  ``pairs``: an indexable of training pairs (raw shapes for ModelNet).  Returns (neighbor limits, pairs used)."""
    from .. import _lib as L
    from ..augment import augment_stacked
    if not 1 <= chunk <= HIST_MAX_PAIRS:
        raise ValueError(f'chunk must be in 1..{HIST_MAX_PAIRS}')
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    b = cfg.backbone
    S, voxel_size, radius = b.num_stages, b.init_voxel_size, b.init_radius
    hist_n = int(np.ceil(4 / 3 * np.pi * (radius / voxel_size + 1) ** 3))
    totals = torch.zeros((S, hist_n), dtype=torch.int32, device=device)
    hists = torch.empty((chunk, S, hist_n), dtype=torch.int32, device=device)
    stop = torch.empty((1,), dtype=torch.int32, device=device)
    lib = L.lib()
    n, used = len(pairs), len(pairs)
    with torch.cuda.device(device):
        for base in range(0, n, chunk):
            group = [pairs[i] for i in range(base, min(n, base + chunk))]
            B = len(group)
            points, lengths, _, _, _ = augment_stacked(group, cfg, seed, CALIBRATION_ITERATION, device, pair_base=base)
            data = precompute_data_stack_mode(points, torch.LongTensor(lengths), S, voxel_size, radius, [hist_n] * S)
            tables = data['neighbors']
            ptrs = (ctypes.c_void_p * S)(*[t.data_ptr() for t in tables])
            widths = np.array([t.shape[1] for t in tables], dtype=np.int64)
            rows = np.array(data['lengths_host'], dtype=np.int64).reshape(S, 2 * B)
            L.check(lib.geob200_neighbor_histogram_batched(ptrs, widths.ctypes.data, rows.ctypes.data, S, B, hist_n, sample_threshold,
                                                           hists.data_ptr(), totals.data_ptr(), stop.data_ptr(), L.stream_ptr()),
                    'neighbor_histogram_batched')
            p = int(stop.item())
            if p >= 0:
                used = base + p + 1
                break
    cum_sum = np.cumsum(totals.cpu().numpy().T, axis=0)
    return np.sum(cum_sum < (keep_ratio * cum_sum[hist_n - 1, :]), axis=0), used
