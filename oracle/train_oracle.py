"""CPU restatement (numpy) of the ground-truth superpoint target sampler of geotransformer_b200/csrc/train.cu.

TEST INFRASTRUCTURE ONLY.  Restates, independently of the CUDA source:
  * candidates: the gt rows with overlap > overlap_threshold (strict), j = 0 .. n-1 in gt order;
  * n <= num_targets: all of them in gt order (the reference SuperPointTargetGenerator's deterministic branch);
  * otherwise the num_targets smallest keys (philox(seed; j, iteration, pair) << 32) | j, in ascending j, with the Philox4x32-10 of
    ransac_oracle: key = 64-bit seed, counter = (j, iteration lo, iteration hi, pair), word 0.
"""
import numpy as np

from oracle.ransac_oracle import philox4x32_10


def target_words(n, seed, iteration, pair):
    """(n,) uint32 Philox words of candidates 0 .. n-1"""
    seed, iteration = int(seed), int(iteration)
    j = np.arange(n, dtype=np.uint64)
    ctr = np.stack([j, np.full_like(j, iteration & 0xFFFFFFFF), np.full_like(j, iteration >> 32), np.full_like(j, pair)], axis=1)
    return philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))[:, 0]


def select_targets(gt_indices, gt_overlaps, overlap_threshold, num_targets, seed, iteration, pair=0):
    """(ref indices, src indices, overlaps) of one pair, as the device sampler returns them"""
    gt_indices, gt_overlaps = np.asarray(gt_indices), np.asarray(gt_overlaps, dtype=np.float32)
    keep = np.nonzero(gt_overlaps > np.float32(overlap_threshold))[0]
    n = keep.shape[0]
    if n > num_targets:
        keys = (target_words(n, seed, iteration, pair).astype(np.uint64) << np.uint64(32)) | np.arange(n, dtype=np.uint64)
        keep = keep[np.sort(np.argsort(keys, kind='stable')[:num_targets])]
    return gt_indices[keep, 0], gt_indices[keep, 1], gt_overlaps[keep]
