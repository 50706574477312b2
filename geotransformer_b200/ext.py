"""H100 (CUDA) replacement of the reference's native op module ``geotransformer.ext``.

Same two positional-argument functions as reference ``geotransformer/extensions/pybind.cpp:6-18``:

    grid_subsampling(points, lengths, voxel_size) -> [s_points, s_lengths]
    radius_neighbors(q_points, s_points, q_lengths, s_lengths, radius) -> LongTensor (Nq, max_count)

Differences, all deliberate: tensors live on the GPU (CPU tensors are moved to the current CUDA device and the
results moved back, so a literal drop-in of the reference's CPU call sites keeps working); empty clouds are
rejected explicitly (the reference reads ``points[0]``, ``extra/cloud/cloud.cpp:5``).
To install it in place of the reference module: ``sys.modules['geotransformer.ext'] = geotransformer_b200.ext``
(see INTEGRATION.md).
"""

import torch

from . import _lib as L


def _prep(points, lengths, pname, lname):
    if points.dtype != torch.float32:
        raise RuntimeError(f'{pname} must be a float tensor')
    if lengths.dtype != torch.int64:
        raise RuntimeError(f'{lname} must be an long tensor')
    if not points.is_contiguous():
        raise RuntimeError(f'{pname} must be contiguous')
    if not lengths.is_contiguous():
        raise RuntimeError(f'{lname} must be contiguous')
    was_cpu = not points.is_cuda
    if was_cpu:
        points = points.cuda()
    lengths_h = lengths.cpu() if lengths.is_cuda else lengths
    return points, lengths_h, was_cpu


def grid_subsampling(points, lengths, voxel_size):
    """reference ``cpu/grid_subsampling/grid_subsampling.cpp:5-62``."""
    dev_lengths = lengths.device
    points, lengths_h, was_cpu = _prep(points, lengths, 'points', 'lengths')
    n, b = points.shape[0], lengths_h.shape[0]
    lib = L.lib()
    ws_bytes = lib.geob200_grid_subsample_workspace_bytes(n, b)
    ws = L.workspace(ws_bytes, points.device)
    s_points = torch.empty((n, 3), dtype=torch.float32, device=points.device)
    s_lengths = torch.empty((b,), dtype=torch.int64, device=points.device)
    L.check(lib.geob200_grid_subsample(points.data_ptr(), n, lengths_h.data_ptr(), b, float(voxel_size),
                                       s_points.data_ptr(), s_lengths.data_ptr(), ws.data_ptr(), ws.numel(),
                                       L.stream_ptr()), 'grid_subsampling')
    s_lengths_h = s_lengths.cpu()               # one 8*B byte D2H: the row count sizes the returned tensor
    total = int(s_lengths_h.sum())
    s_points = s_points[:total].clone()
    if was_cpu:
        return [s_points.cpu(), s_lengths_h]
    return [s_points, s_lengths if dev_lengths.type == 'cuda' else s_lengths_h]


def _radius_call(q_points, s_points, ql_h, sl_h, radius, width, out, counts, max_count):
    lib = L.lib()
    nq, ns, b = q_points.shape[0], s_points.shape[0], ql_h.shape[0]
    ws_bytes = lib.geob200_radius_search_workspace_bytes(nq, ns, b)
    ws = L.workspace(ws_bytes, q_points.device)
    L.check(lib.geob200_radius_search(q_points.data_ptr(), nq, s_points.data_ptr(), ns, ql_h.data_ptr(),
                                      sl_h.data_ptr(), b, float(radius), int(width), L.ptr(out), L.ptr(counts),
                                      max_count.data_ptr(), ws.data_ptr(), ws.numel(), L.stream_ptr()),
            'radius_neighbors')


def radius_neighbors(q_points, s_points, q_lengths, s_lengths, radius, neighbor_limit=0):
    """reference ``cpu/radius_neighbors/radius_neighbors.cpp:5-68``.

    ``neighbor_limit`` is an extension (0 = reference behaviour, full ``max_count`` width): with a positive
    limit the kernel keeps only the ``limit`` nearest neighbours per row in a single pass and the result is
    ``(Nq, min(limit, max_count))`` -- exactly what ``radius_search`` slices out of the full table
    (reference ``modules/ops/radius_search.py:25-26``), but contiguous.
    """
    q_points, ql_h, was_cpu = _prep(q_points, q_lengths, 'q_points', 'q_lengths')
    s_points, sl_h, _ = _prep(s_points, s_lengths, 's_points', 's_lengths')
    nq = q_points.shape[0]
    dev = q_points.device
    max_count = torch.zeros((1,), dtype=torch.int32, device=dev)
    if neighbor_limit > 0:
        out = torch.empty((nq, neighbor_limit), dtype=torch.int64, device=dev)
        _radius_call(q_points, s_points, ql_h, sl_h, radius, neighbor_limit, out, None, max_count)
        mc = int(max_count.item())
        if mc < 0:
            raise RuntimeError('radius_neighbors: more than 16384 neighbours for one query')
        if mc < neighbor_limit:
            out = out[:, :mc].contiguous()
    else:
        _radius_call(q_points, s_points, ql_h, sl_h, radius, 0, None, None, max_count)   # count pass
        mc = int(max_count.item())
        if mc < 0:
            raise RuntimeError('radius_neighbors: more than 16384 neighbours for one query')
        out = torch.empty((nq, mc), dtype=torch.int64, device=dev)
        if mc > 0:
            _radius_call(q_points, s_points, ql_h, sl_h, radius, mc, out, None, max_count)
    return out.cpu() if was_cpu else out


def radius_neighbors_deferred(q_points, s_points, q_lengths, s_lengths, radius, neighbor_limit):
    """Limited-width search with NO host synchronisation: (table (Nq, limit) int64, max_count int32[1] on the device)."""
    q_points, ql_h, _ = _prep(q_points, q_lengths, 'q_points', 'q_lengths')
    s_points, sl_h, _ = _prep(s_points, s_lengths, 's_points', 's_lengths')
    dev = q_points.device
    max_count = torch.empty((1,), dtype=torch.int32, device=dev)
    out = torch.empty((q_points.shape[0], neighbor_limit), dtype=torch.int64, device=dev)
    _radius_call(q_points, s_points, ql_h, sl_h, radius, neighbor_limit, out, None, max_count)
    return out, max_count
