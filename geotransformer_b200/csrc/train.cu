// Pieces of the training step that run on the device: the ground-truth superpoint target sampler of the training-mode forward
// and the non-finite gradient guard in front of the optimizer.
//
// Reference: geotransformer/modules/geotransformer/superpoint_target.py (SuperPointTargetGenerator) and
//            geotransformer/engine/epoch_based_trainer.py (train_step / check_gradients).
// Sampler semantics (DESIGN.md section 3b):
//   * candidates: the gt rows of the pair with overlap > overlap_threshold (strict), j = 0 .. n-1 in gt order;
//   * n <= num_targets: all of them in gt order (the reference's deterministic branch);
//   * otherwise the num_targets smallest keys (philox(seed; j, iteration, pair) << 32) | j, written in ascending j -- a uniform
//     subset without replacement; Philox4x32-10 with key = 64-bit seed, counter = (j, iteration lo, iteration hi, pair id),
//     pair id = pair_base + p, word 0.  The draw of a pair depends on (seed, iteration, pair id, candidates) only.
// One CTA per pair; integer shared-memory counters only (no float atomics), so the result is a function of the inputs.
#include "common.cuh"
#include "compaction.cuh"
#include "geob200.h"
#include "philox.cuh"
#include "radix_select.cuh"

namespace geob200 {

constexpr int ST_THREADS = 1024;

__device__ __forceinline__ uint32_t target_word(uint32_t j, uint32_t it_lo, uint32_t it_hi, uint32_t pair, uint32_t k0, uint32_t k1) {
    uint32_t c[4] = {j, it_lo, it_hi, pair};
    philox4x32_10(c, k0, k1);
    return c[0];
}

// Grid (1, B), ST_THREADS threads.  Pair p reads its gt rows at G.start[p] (first min(gt_count[p], G.count[p]) valid) and writes
// row p (ref) / B + p (src) of corr (2B, K), row p of scores (B, K), count[p].  cand / word: workspace, G.start[p] + j.
__global__ void __launch_bounds__(ST_THREADS) superpoint_targets_kernel(
        const long long* __restrict__ gt_idx, const float* __restrict__ gt_ov, const int* __restrict__ gt_count,
        const __grid_constant__ Segs G, float thr_ov, int K, uint32_t key0, uint32_t key1, uint32_t it_lo, uint32_t it_hi,
        uint32_t pair_base, int* __restrict__ cand, uint32_t* __restrict__ word, long long* __restrict__ corr, float* __restrict__ scores,
        int* __restrict__ count) {
    __shared__ unsigned hist[256];
    __shared__ unsigned prefix_s, kth_s;
    __shared__ int warp_tot[32];
    const int p = blockIdx.y, B = gridDim.y;
    const int rows = min(max(gt_count[p], 0), G.count[p]);
    gt_idx += 2ll * G.start[p]; gt_ov += G.start[p]; cand += G.start[p]; word += G.start[p];
    long long* ref_out = corr + (long long)p * K;
    long long* src_out = corr + (long long)(B + p) * K;
    scores += (long long)p * K;
    const uint32_t pair = pair_base + (uint32_t)p;

    // candidates in gt order, with their Philox words
    int n = 0;
    for (int base = 0; base < rows; base += ST_THREADS) {
        const int t = base + threadIdx.x;
        const bool f = t < rows && gt_ov[t] > thr_ov;
        int tot;
        const int r = chunk_rank(f, warp_tot, &tot);
        if (f) {
            cand[n + r] = t;
            word[n + r] = target_word((uint32_t)(n + r), it_lo, it_hi, pair, key0, key1);
        }
        n += tot;
    }
    const int k = min(n, K);
    for (int i = k + threadIdx.x; i < K; i += ST_THREADS) { ref_out[i] = -1; src_out[i] = -1; scores[i] = 0.f; }
    if (threadIdx.x == 0) count[p] = k;
    __syncthreads();                       // cand / word of this CTA are visible to all its threads
    if (n <= K) {
        for (int j = threadIdx.x; j < n; j += ST_THREADS) {
            const int t = cand[j];
            ref_out[j] = gt_idx[2 * t]; src_out[j] = gt_idx[2 * t + 1]; scores[j] = gt_ov[t];
        }
        return;
    }
    // the K smallest (word, j) = the K largest ~word, ties at the threshold to the lowest j; written in ascending j
    unsigned thr;
    int need_eq;
    radix_select_kth((long long)n, K, [&](long long j) { return ~word[j]; }, hist, &prefix_s, &kth_s, thr, need_eq);
    int out = 0, eq = 0;
    for (int base = 0; base < n; base += ST_THREADS) {
        const int j = base + threadIdx.x;
        const unsigned b = j < n ? ~word[j] : 0u;
        const bool fe = j < n && b == thr;
        int te;
        const int re = chunk_rank(fe, warp_tot, &te);
        const bool f = j < n && (b > thr || (fe && eq + re < need_eq));
        int tot;
        const int r = chunk_rank(f, warp_tot, &tot);
        if (f) {
            const int t = cand[j];
            ref_out[out + r] = gt_idx[2 * t]; src_out[out + r] = gt_idx[2 * t + 1]; scores[out + r] = gt_ov[t];
        }
        out += tot; eq += te;
    }
}

// found_inf[0] = 1 when any element of any listed tensor is NaN or +-Inf.  Grid (x, n_tensors); found_inf was zeroed before.  Many
// threads may store the same 1.0f: a race-free plain store, the flag never goes back to 0.
__global__ void __launch_bounds__(256) nonfinite_check_kernel(const float* const* __restrict__ ptrs, const long long* __restrict__ numels,
                                                              float* __restrict__ found_inf) {
    const float* x = ptrs[blockIdx.y];
    const long long n = numels[blockIdx.y];
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool bad = false;
    // float4 body from the first 16-byte boundary, scalar head and tail
    const long long head = min(n, (long long)(((16 - ((uintptr_t)x & 15)) & 15) / 4));
    const long long n4 = (n - head) / 4;
    const float4* x4 = reinterpret_cast<const float4*>(x + head);
    for (long long i = t0; i < n4; i += stride) {
        const float4 v = x4[i];
        bad |= !isfinite(v.x) || !isfinite(v.y) || !isfinite(v.z) || !isfinite(v.w);
    }
    for (long long i = t0; i < head; i += stride) bad |= !isfinite(x[i]);
    for (long long i = head + 4 * n4 + t0; i < n; i += stride) bad |= !isfinite(x[i]);
    if (__syncthreads_or(bad) && threadIdx.x == 0) *found_inf = 1.0f;
}

// Loss weights of a batched step: one thread walks the B rows in pair order, so the mean is a fixed-order fp32 sum (no atomics).
// __fmul_rn / __fadd_rn keep the compiler from contracting the sum into FMAs: the numpy restatement rounds every product.
__global__ void __launch_bounds__(32) batch_loss_weights_kernel(const float* __restrict__ rows, int ld, int B, float* __restrict__ w,
                                                                float* __restrict__ mean_row, float* __restrict__ n_valid,
                                                                float* __restrict__ found_inf) {
    if (threadIdx.x != 0) return;
    int n = 0;
    for (int p = 0; p < B; ++p) {
        const float* r = rows + (long long)p * ld;
        n += (isfinite(r[0]) && isfinite(r[1]) && isfinite(r[2])) ? 1 : 0;
    }
    const float inv = n > 0 ? __fdiv_rn(1.0f, (float)n) : 0.0f;
    float acc0 = 0.0f, acc1 = 0.0f, acc2 = 0.0f;
    for (int p = 0; p < B; ++p) {
        const float* r = rows + (long long)p * ld;
        const bool ok = isfinite(r[0]) && isfinite(r[1]) && isfinite(r[2]);
        w[p] = ok ? inv : 0.0f;
        if (ok) {
            acc0 = __fadd_rn(acc0, __fmul_rn(inv, r[0]));
            acc1 = __fadd_rn(acc1, __fmul_rn(inv, r[1]));
            acc2 = __fadd_rn(acc2, __fmul_rn(inv, r[2]));
        }
    }
    if (n == 0) {
        acc0 = acc1 = acc2 = __int_as_float(0x7fc00000);      // the mean over no pair is NaN, and the step is skipped
        *found_inf = 1.0f;
    }
    mean_row[0] = acc0; mean_row[1] = acc1; mean_row[2] = acc2;
    if (n_valid != nullptr) *n_valid = (float)n;
}

}  // namespace geob200

using namespace geob200;

extern "C" {

size_t geob200_superpoint_targets_batched_workspace_bytes(int64_t n_gt_rows) {
    return 2 * align_up(4 * (size_t)(n_gt_rows > 0 ? n_gt_rows : 0), 256) + 256;
}

int geob200_superpoint_targets_batched(const int64_t* gt_indices, const float* gt_overlaps, const int32_t* gt_count, int64_t n_pairs,
                                       const int64_t* cloud_nodes, float overlap_threshold, int64_t num_targets, uint64_t seed,
                                       uint64_t iteration, int64_t pair_base, int64_t* corr_indices, float* corr_scores, int32_t* num_out,
                                       void* workspace, size_t workspace_bytes, void* stream) {
    GEOB_REQUIRE(n_pairs > 0 && 2 * n_pairs <= GEOB_MAX_CLOUDS, "superpoint_targets_batched: 1..%d pairs", GEOB_MAX_CLOUDS / 2);
    GEOB_REQUIRE(num_targets > 0 && num_targets <= (1 << 20), "superpoint_targets_batched: num_targets must be in 1..%d", 1 << 20);
    GEOB_REQUIRE(isfinite(overlap_threshold), "superpoint_targets_batched: overlap_threshold must be finite");
    GEOB_REQUIRE(pair_base >= 0 && pair_base + n_pairs <= 0xFFFFFFFFll, "superpoint_targets_batched: pair_base out of range");
    GEOB_REQUIRE(cloud_nodes != nullptr, "superpoint_targets_batched: null cloud_nodes");
    GEOB_REQUIRE(gt_indices != nullptr && gt_overlaps != nullptr && gt_count != nullptr && corr_indices != nullptr &&
                     corr_scores != nullptr && num_out != nullptr,
                 "superpoint_targets_batched: null pointer");
    const int B = (int)n_pairs;
    Segs R, Q, G;
    if (segs_from_counts(&R, n_pairs, cloud_nodes) || segs_from_counts(&Q, n_pairs, cloud_nodes + n_pairs) || segs_products(&G, R, Q))
        return -1;
    const int64_t rows = (int64_t)G.start[B - 1] + G.count[B - 1];
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= geob200_superpoint_targets_batched_workspace_bytes(rows),
                 "superpoint_targets_batched: workspace too small");
    Arena ar(workspace, workspace_bytes);
    int* cand = ar.take<int>((size_t)rows);
    uint32_t* word = ar.take<uint32_t>((size_t)rows);
    GEOB_REQUIRE(ar.ok(), "superpoint_targets_batched: workspace accounting error");
    superpoint_targets_kernel<<<dim3(1, B), ST_THREADS, 0, (cudaStream_t)stream>>>(
        (const long long*)gt_indices, gt_overlaps, gt_count, G, overlap_threshold, (int)num_targets, (uint32_t)seed, (uint32_t)(seed >> 32),
        (uint32_t)iteration, (uint32_t)(iteration >> 32), (uint32_t)pair_base, cand, word, (long long*)corr_indices, corr_scores, num_out);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_nonfinite_check(const float* const* ptrs, const int64_t* numels, int64_t n_tensors, int64_t max_numel, float* found_inf,
                            void* stream) {
    GEOB_REQUIRE(n_tensors >= 1 && n_tensors <= 65535, "nonfinite_check: 1..65535 tensors");
    GEOB_REQUIRE(max_numel >= 0, "nonfinite_check: max_numel must be non-negative");
    GEOB_REQUIRE(ptrs != nullptr && numels != nullptr && found_inf != nullptr, "nonfinite_check: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    // enough CTAs per tensor to stream the largest one with ~16 float4 per thread, at most 4 waves of the device
    const long long per = (max_numel + 256ll * 4 * 16 - 1) / (256ll * 4 * 16);
    const unsigned gx = (unsigned)max(1ll, min(per, 4ll * num_sms()));
    GEOB_CHECK_CUDA(cudaMemsetAsync(found_inf, 0, sizeof(float), st));
    nonfinite_check_kernel<<<dim3(gx, (unsigned)n_tensors), 256, 0, st>>>(ptrs, (const long long*)numels, found_inf);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_batch_loss_weights(const float* loss_rows, int64_t ld_rows, int64_t n_pairs, float* weights, float* mean_row, float* n_valid,
                               float* found_inf, void* stream) {
    GEOB_REQUIRE(n_pairs >= 1 && 2 * n_pairs <= GEOB_MAX_CLOUDS, "batch_loss_weights: 1..%d pairs", GEOB_MAX_CLOUDS / 2);
    GEOB_REQUIRE(ld_rows >= 3 && ld_rows <= (1ll << 30), "batch_loss_weights: ld_rows must be in 3..2^30");
    GEOB_REQUIRE(loss_rows != nullptr && weights != nullptr && mean_row != nullptr && found_inf != nullptr,
                 "batch_loss_weights: null pointer");
    batch_loss_weights_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(loss_rows, (int)ld_rows, (int)n_pairs, weights, mean_row, n_valid,
                                                                 found_inf);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

}  // extern "C"
