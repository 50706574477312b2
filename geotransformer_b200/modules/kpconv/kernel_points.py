"""KPConv kernel points as the reference builds them (``geotransformer/modules/kpconv/kernel_points.py``).

The reference loads one optimised disposition, ``dispositions/k_015_center_3D.ply``, which ``kernel_point_optimization_debug``
produced once from an unseeded draw, and gives every KPConv its own copy rotated about z, noised and scaled (``load_kernels``).
Here the disposition is generated on the device (``geob200_kernel_point_optimize``, the same fp64 potential descent from Philox
draws under ``DISPOSITION_SEED``) and the per-instance buffers come from ``geob200_kernel_point_instances``.
"""
import torch

from ... import _lib as L

NUM_CANDIDATES = 100        # load_kernels: kernel_point_optimization_debug(..., num_kernels=100)
RATIO = 0.66
DISPOSITION_SEED = 0        # key of the initial draws of the shipped disposition: every model shares it, as the reference's file

_dispositions = {}


def optimize_dispositions(num_points, num_kernels=NUM_CANDIDATES, seed=DISPOSITION_SEED, init=None, ratio=RATIO, device=None):
    """``kernel_point_optimization_debug(1.0, num_points, num_kernels, 3, fixed='center', ratio)`` on the device.  ``init``: optional
    (num_kernels * num_points, 3) initial points (the accepted draws); default: Philox draws keyed by ``seed``.  Returns (points
    (num_kernels, num_points, 3) fp64, the candidate ``load_kernels`` picks, the iteration the descent stopped at)."""
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    if init is not None:
        init = torch.as_tensor(init, dtype=torch.float64).to(device).contiguous()
        if init.shape != (num_kernels * num_points, 3):
            raise ValueError(f'init must be ({num_kernels * num_points}, 3), got {tuple(init.shape)}')
    points = torch.empty((num_kernels, num_points, 3), dtype=torch.float64, device=device)
    info = torch.empty((2,), dtype=torch.int32, device=device)
    with torch.cuda.device(device):
        L.check(L.lib().geob200_kernel_point_optimize(L.ptr(init), int(num_kernels), int(num_points), int(seed), float(ratio),
                                                      points.data_ptr(), info.data_ptr(), L.stream_ptr()), 'kernel_point_optimize')
    best, stop = info.tolist()
    return points, best, stop


def disposition(num_points=15, device=None):
    """the disposition every KPConv with ``num_points`` kernel points starts from (load_kernels' best candidate), (num_points, 3)
    fp64 on ``device``; computed once per process and size"""
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    key = (num_points, str(device))
    if key not in _dispositions:
        points, best, _ = optimize_dispositions(num_points, device=device)
        _dispositions[key] = points[best].contiguous()
    return _dispositions[key]


def kernel_point_instances(disp, radii, layer_ids, seed):
    """load_kernels' buffers: (len(radii), num_points, 3) fp32, layer l = rotation about z of (fp32(disp) + N(0, 0.01^2)) * radii[l],
    drawn from the stream (seed, layer_ids[l])"""
    device = disp.device
    disp = disp.to(torch.float64).contiguous()
    r = torch.as_tensor(radii, dtype=torch.float64).reshape(-1).to(device)
    ids = torch.as_tensor(layer_ids, dtype=torch.int64).reshape(-1).to(device)
    if r.numel() != ids.numel():
        raise ValueError('radii and layer_ids must have the same length')
    out = torch.empty((r.numel(), disp.shape[0], 3), dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        L.check(L.lib().geob200_kernel_point_instances(disp.data_ptr(), disp.shape[0], r.data_ptr(), ids.data_ptr(), r.numel(),
                                                       int(seed), out.data_ptr(), L.stream_ptr()), 'kernel_point_instances')
    return out


def initialize_kernel_points(model, seed):
    """give every KPConv of ``model`` the buffer the reference's constructor draws: the shared disposition rotated about z, noised
    and scaled by the layer's radius.  The KPConv with index i in ``named_modules`` order draws from the stream (seed, i), so a model
    initialised twice with one seed gets the same buffers.  Returns the number of KPConvs initialised."""
    convs = [m for _, m in model.named_modules() if m.__class__.__name__ == 'KPConv']
    if not convs:
        return 0
    device = convs[0].kernel_points.device
    if device.type != 'cuda':
        device = torch.device('cuda', torch.cuda.current_device())
    by_size = {}
    for i, m in enumerate(convs):
        by_size.setdefault(m.kernel_size, []).append(i)
    for k, idx in by_size.items():
        buf = kernel_point_instances(disposition(k, device), [convs[i].radius for i in idx], idx, seed)
        with torch.no_grad():
            for row, i in enumerate(idx):
                convs[i].kernel_points.copy_(buf[row])
    return len(convs)
