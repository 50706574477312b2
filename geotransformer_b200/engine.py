"""Throughput front end: registers a batch of point-cloud pairs, several pairs in flight at once.

Pairs are independent (SURVEY.md section 8e).  Most kernels of one pair leave SMs idle (a few hundred CTAs, deep levels
with ~600 points), so the engine runs ``num_streams`` pairs concurrently, each on its own CUDA stream driven by its own
host thread (ctypes and torch release the GIL while launching / synchronising) that pulls the next pair from a shared
cursor.  Per pair it performs: H2D of the raw
clouds (pinned staging) -> GPU collate -> model forward -> D2H of the estimated transform.  This is the caller-facing API
bench.py measures as `e2e` (SURVEY.md section 8f next #2, the SingleTester-compatible loop, is built on it).
"""
import threading
from concurrent.futures import ThreadPoolExecutor

import torch

from . import _lib
from .model import trim_outputs
from .utils.data import registration_collate_fn_stack_mode

LOSS_KEYS = ('loss', 'c_loss', 'f_loss')
METRIC_KEYS = ('PIR', 'IR', 'RRE', 'RTE', 'RMSE', 'RR')


def pin_host_threads_to_gpu(device):
    """Restrict the calling thread (and the threads it creates afterwards) to the CPUs NVML reports as local to `device`
    (same NUMA node / PCIe root).  On a two-socket host a launch thread running on the remote socket costs tens of percent of
    throughput.  Best effort: returns False when NVML or the affinity call is unavailable."""
    try:
        import os
        import pynvml
        pynvml.nvmlInit()
        uuid = str(torch.cuda.get_device_properties(device).uuid)
        handle = pynvml.nvmlDeviceGetHandleByUUID(('GPU-' + uuid) if not uuid.startswith('GPU-') else uuid)
        words = pynvml.nvmlDeviceGetCpuAffinity(handle, (os.cpu_count() + 63) // 64)
        cpus = {64 * i + b for i, w in enumerate(words) for b in range(64) if (int(w) >> b) & 1}
        cpus &= os.sched_getaffinity(0)
        if not cpus:
            return False
        os.sched_setaffinity(0, cpus)
        return True
    except Exception:
        return False


class RegistrationEngine:
    def __init__(self, model, cfg, neighbor_limits, num_streams=4, device=None, native=True, evaluator=None, pin_cpu=False,
                 batch_size=1, side_streams=4, loss_func=None, ransac=None):
        """pin_cpu: bind the calling thread and the worker threads to the CPUs local to the GPU (pin_host_threads_to_gpu).
        evaluator: optional geotransformer_b200.loss.Evaluator; its metrics (PIR, IR, RRE, RTE, RMSE, RR) are then computed
        on the device for every pair and travel back with the transform in the same D2H copy.
        batch_size: every worker registers up to ``batch_size`` pairs per forward (GeoTransformer.forward_batch: one collate,
        one backbone / transformer pass over the stacked rows of all pairs, per-pair stages on ``side_streams`` extra
        streams when batch_size > 1), with ONE host synchronisation per forward besides the collate's size read-backs.
        loss_func: optional geotransformer_b200.loss.OverallLoss; every result then gains 'loss': {'loss', 'c_loss', 'f_loss'}
        (the reference's val_step losses), computed on the device and read back with the same event.
        ransac: optional config section (cfg.ransac: distance_threshold, num_points, num_iterations, seed); every result then gains
        'ransac': {'estimated_transform', 'fitness', 'inlier_rmse'(, 'metrics' with an evaluator)} -- correspondence RANSAC on the
        LGR correspondences, run on the lane's stream after LGR (pair p of a forward draws from the stream (seed, p))."""
        self.model, self.cfg, self.limits = model, cfg, neighbor_limits
        if native and not hasattr(model, '_native'):
            from .model import enable_native
            enable_native(model)          # C++ stage drivers: same results, ~10x less host time per pair
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self.num_streams = num_streams
        self.pinned_cpu = pin_host_threads_to_gpu(self.device) if pin_cpu else False
        self.evaluator = evaluator
        self.loss_func = loss_func
        self.ransac = ransac
        self.stage_times = None          # set to {} to collect per-stage CUDA-event times (profiling; adds ~7 events per pair)
        self.streams = [torch.cuda.Stream(self.device) for _ in range(num_streams)]
        self.pool = ThreadPoolExecutor(max_workers=num_streams)
        # per slot: [estimated_transform (16) | metrics (8)] on the device and pinned on the host
        self.batch_size = max(1, int(batch_size))
        if self.batch_size > 32:
            raise ValueError('RegistrationEngine: at most 32 pairs per forward (the kernels carry the 2 x batch cloud offsets by value)')
        bs = self.batch_size
        self.r_dev = [torch.zeros((bs, 24), dtype=torch.float32, device=self.device) for _ in range(num_streams)]
        self.r_host = [torch.zeros((bs, 24), dtype=torch.float32).pin_memory() for _ in range(num_streams)]
        # per slot: [loss, c_loss, f_loss] rows on the device and pinned on the host (only with a loss function)
        self.l_dev = [torch.zeros((bs, 3), dtype=torch.float32, device=self.device) for _ in range(num_streams)]
        self.l_host = [torch.zeros((bs, 3), dtype=torch.float32).pin_memory() for _ in range(num_streams)]
        # per slot: [RANSAC transform (16) | fitness | inlier_rmse | metrics of the RANSAC transform (8)] (only with ransac)
        self.x_dev = [torch.zeros((bs, 26), dtype=torch.float32, device=self.device) if ransac is not None else None for _ in range(num_streams)]
        self.x_host = [torch.zeros((bs, 26), dtype=torch.float32).pin_memory() if ransac is not None else None for _ in range(num_streams)]
        self.sides = [[torch.cuda.Stream(self.device) for _ in range(side_streams)] if bs > 1 else [] for _ in range(num_streams)]

    def _ransac_result(self, row):
        v = row.tolist()
        r = {'estimated_transform': row[:16].reshape(4, 4).clone(), 'fitness': v[16], 'inlier_rmse': v[17]}
        if self.evaluator is not None:
            r['metrics'] = dict(zip(METRIC_KEYS, v[18:24]))
        return r

    def _batch(self, slot, chunk, keep):
        """``len(chunk)`` pairs in one forward"""
        stream = self.streams[slot]
        b = self.cfg.backbone
        n = len(chunk)
        marks = None
        if self.stage_times is not None:
            marks = []
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            marks.append(('begin', e))
        data = registration_collate_fn_stack_mode(chunk, b.num_stages, b.init_voxel_size, b.init_radius, self.limits, device=self.device)
        if marks is not None:
            data['_stage_events'] = marks
        r_dev, r_host = self.r_dev[slot][:n], self.r_host[slot][:n]
        l_dev, l_host, lf = self.l_dev[slot][:n], self.l_host[slot][:n], self.loss_func
        rs = self.ransac
        x_dev, x_host = (self.x_dev[slot][:n], self.x_host[slot][:n]) if rs is not None else (None, None)
        outs = self.model.forward_batch(data, evaluator=self.evaluator, results=r_dev, side_streams=self.sides[slot], keep_outputs=keep,
                                        loss_func=lf, loss_out=l_dev, ransac=rs, ransac_out=x_dev)
        r_host.copy_(r_dev, non_blocking=True)
        if lf is not None:
            l_host.copy_(l_dev, non_blocking=True)
        if rs is not None:
            x_host.copy_(x_dev, non_blocking=True)
        done = torch.cuda.Event()
        done.record(stream)
        done.synchronize()
        if keep:
            trim_outputs(outs)
        if marks is not None:          # per-stage GPU time of this batch on its main stream (label = the interval ending at that mark)
            for (_, e0), (label, e1) in zip(marks[:-1], marks[1:]):
                self.stage_times.setdefault('collate' if label == 'start' else label, []).append(e0.elapsed_time(e1))
        lens_c = data['lengths_host'][-1]
        res = []
        for p in range(n):
            row = r_host[p]
            m = row[16:].tolist()
            r = {'estimated_transform': row[:16].reshape(4, 4).clone(), 'num_superpoints': (int(lens_c[p]), int(lens_c[n + p])),
                 'num_corr': int(m[6])}
            if self.evaluator is not None:
                r['metrics'] = dict(zip(METRIC_KEYS, m[:6]))
            if lf is not None:
                r['loss'] = dict(zip(LOSS_KEYS, l_host[p].tolist()))
            if rs is not None:
                r['ransac'] = self._ransac_result(x_host[p])
            if keep:
                r['output_dict'] = outs[p]
            res.append(r)
        return res, done

    def _worker(self, slot, pairs, results, cursor, lock, start_event, keep):
        """one host thread per stream: pulls the next unregistered pair until none is left (no per-chunk barrier)"""
        torch.cuda.set_device(self.device)
        stream = self.streams[slot]
        last = None
        with torch.cuda.stream(stream), _lib.stream_scope(stream.cuda_stream):
            if start_event is not None:
                stream.wait_event(start_event)
            bs = self.batch_size
            while True:
                with lock:
                    i = cursor[0]
                    cursor[0] += bs
                if i >= len(pairs):
                    return last
                res, last = self._batch(slot, pairs[i:i + bs], keep)
                results[i:i + len(res)] = res

    def register(self, pairs, start_event=None, keep_outputs=False):
        """pairs: list of dicts with ref_points/src_points/ref_feats/src_feats/transform (numpy, CPU or CUDA tensors).
        Returns one result dict per pair, in order.  The current stream waits for all of them."""
        results = [None] * len(pairs)
        cursor, lock = [0], threading.Lock()
        n_jobs = (len(pairs) + self.batch_size - 1) // self.batch_size
        futs = [self.pool.submit(self._worker, s, pairs, results, cursor, lock, start_event, keep_outputs)
                for s in range(min(self.num_streams, max(1, n_jobs)))]
        for f in futs:
            done = f.result()
            if done is not None:
                torch.cuda.current_stream().wait_event(done)
        return results

    def close(self):
        self.pool.shutdown()
