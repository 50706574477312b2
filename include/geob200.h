/* geob200 -- C ABI of the H100-native GeoTransformer registration hot path.
 *
 * Drop-in boundary (SURVEY.md section 8b).  Every entry point takes plain pointers and sizes; device
 * pointers unless the name ends in `_h`; `stream` is a cudaStream_t passed as void*.  All functions
 * return 0 on success and a negative code on failure, with a message available from geob200_last_error()
 * (the reference raises c10::Error -> RuntimeError through TORCH_CHECK, common/torch_helper.h:6-35; the
 * Python host layer turns a non-zero return into RuntimeError to keep that behaviour).
 *
 * Scratch memory is provided by the caller: each op has a *_workspace_bytes() query.
 * Index tables are int64 and sentinels equal the number of support rows, as in the reference.
 */
#ifndef GEOB200_H
#define GEOB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* geob200_last_error(void);
/* number of CUDA kernels this library has launched since it was loaded (bench.py: gpu_launches) */
uint64_t geob200_launch_count(void);

/* ---- collate -------------------------------------------------------------------------------------------- */

/* Replaces ext.grid_subsampling (reference geotransformer/extensions/pybind.cpp:13-17,
 * cpu/grid_subsampling/grid_subsampling.cpp:5-62): per-cloud voxel barycentres, bit-identical values AND order.
 * points (n_points,3) f32; lengths_h host int64[batch]; s_points must hold n_points*3 floats (upper bound);
 * s_lengths device int64[batch] receives the per-cloud counts (their sum = rows written). */
size_t geob200_grid_subsample_workspace_bytes(int64_t n_points, int64_t batch);
int geob200_grid_subsample(const float* points, int64_t n_points, const int64_t* lengths_h, int64_t batch, float voxel,
                           float* s_points, int64_t* s_lengths, void* workspace, size_t workspace_bytes, void* stream);

/* Replaces ext.radius_neighbors (reference pybind.cpp:8-12, cpu/radius_neighbors/radius_neighbors.cpp:5-68)
 * fused with the column slice of modules/ops/radius_search.py:25-26.
 * For every query row: indices (offset by the cloud start) of the support points of the same batch element with
 * d2 < r*r, ascending by d2, first `width` of them, padded with the sentinel n_support.
 * max_count (device int32) receives the global maximum neighbour count (the reference's row width); a negative
 * value signals an unsupported density (> 16384 neighbours for one query).  counts (device int32[n_query]) and
 * out may be NULL (count-only pass when width == 0). */
size_t geob200_radius_search_workspace_bytes(int64_t n_query, int64_t n_support, int64_t batch);
int geob200_radius_search(const float* q_points, int64_t n_query, const float* s_points, int64_t n_support,
                          const int64_t* q_lengths_h, const int64_t* s_lengths_h, int64_t batch, float radius,
                          int64_t width, int64_t* out, int32_t* counts, int32_t* max_count, void* workspace,
                          size_t workspace_bytes, void* stream);

/* calibrate_neighbors_stack_mode (utils/data.py:190-217): hist[c] += #rows of a neighbour table (n_rows, width) with
 * exactly c entries < n_support, for c < hist_n (int32 device histogram, accumulated across calls). */
int geob200_neighbor_histogram(const int64_t* neighbors, int64_t n_rows, int64_t width, int64_t n_support, int64_t hist_n,
                               int32_t* hist, void* stream);

/* calibrate_neighbors_stack_mode over a batch of `batch` pairs at once (two launches).  neighbors: host array of num_stages device
 * pointers to the batch's stacked neighbour tables (stage s: (sum of cloud_rows[s], widths[s]) int64, sentinel = its row count);
 * cloud_rows: host (num_stages, 2 * batch) rows per cloud, clouds ordered [ref_0..ref_{B-1}, src_0..src_{B-1}].  hists (device
 * int32 (batch, num_stages, hist_n)) receives one histogram per (pair, stage).  Then, in pair order, the pairs' row totals are
 * added to the running totals of earlier calls (device int32 (num_stages, hist_n), in / out); the first pair after which every
 * stage's total exceeds sample_threshold -- the reference's early exit -- is written to *stop (device int32, -1 if none), and
 * totals receive the histograms of the pairs up to and including it (all pairs if none). */
#define GEOB200_HIST_MAX_PAIRS 32
int geob200_neighbor_histogram_batched(const int64_t* const* neighbors, const int64_t* widths, const int64_t* cloud_rows,
                                       int64_t num_stages, int64_t batch, int64_t hist_n, int64_t sample_threshold, int32_t* hists,
                                       int32_t* totals, int32_t* stop, void* stream);

/* ---- voxel downsampling (Open3D PointCloud::VoxelDownSample; csrc/voxel.cu) ------------------------------------------------- */

/* Open3D's voxel downsampling of `batch` stacked clouds (lengths_h host int64[batch], empty clouds allowed), in double: voxel
 * averages of the points (and of the normals if given, not renormalised) summed in input order, in the iteration order of
 * Open3D's std::unordered_map keyed by hash_eigen (the contract is in DESIGN.md section 8a).  points / normals: device
 * (n_points, 3) fp64; out_points / out_normals: device fp64 with room for n_points rows (normals and out_normals both given or
 * both NULL); each cloud's voxels start at the sum of the earlier clouds' voxel counts.  out_lengths: device int64[batch + 1]
 * receives the per-cloud voxel counts and then the status word: 0, or a GEOB200_VOXEL_* code for an error found on the device
 * (every count is then 0 and no output is written).  Arguments are checked before any launch; no host synchronisation. */
#define GEOB200_VOXEL_MAX_CLOUDS 64
#define GEOB200_VOXEL_NONFINITE 1   /* a coordinate is NaN or infinite */
#define GEOB200_VOXEL_TOO_SMALL 2   /* voxel * INT_MAX < the largest extent of the padded bounding box (Open3D's check) */
#define GEOB200_VOXEL_AXIS_LIMIT 3  /* an axis spans 2^21 voxels or more (the packed voxel key holds 21 bits per axis) */
size_t geob200_voxel_down_sample_workspace_bytes(int64_t n_points, int64_t batch);
int geob200_voxel_down_sample(const double* points, const double* normals, int64_t n_points, const int64_t* lengths_h, int64_t batch,
                              double voxel, double* out_points, double* out_normals, int64_t* out_lengths, void* workspace,
                              size_t workspace_bytes, void* stream);

/* ---- kernel-point dispositions (reference modules/kpconv/kernel_points.py; csrc/kernel_points.cu) ----------------------------- */

/* kernel_point_optimization_debug(1.0, num_points, num_kernels, 3, fixed='center', ratio) in fp64, one launch of one CTA: the
 * potential descent of num_kernels candidates with the centre fixed and the reference's global stopping test, then the rescale to
 * a mean radius of `ratio`.  init: device (num_kernels * num_points, 3) fp64 initial points (the accepted draws, centre rows
 * included and zeroed), or NULL to draw them from Philox keyed by seed (the draw layout is documented in kernel_points.cu).
 * points: device (num_kernels, num_points, 3) fp64 out.  info: device int32 [2] = {the candidate load_kernels picks, the
 * iteration the descent stopped at (10000 if it never did)}. */
#define GEOB200_KP_MAX_POINTS 30
int geob200_kernel_point_optimize(const double* init, int64_t num_kernels, int64_t num_points, uint64_t seed, double ratio,
                                  double* points, int32_t* info, void* stream);

/* load_kernels' per-instance buffers: layer l gets (fp32(disposition) + N(0, 0.01^2) noise) * radii[l], rotated about z by
 * theta ~ U(0, 2 pi), as fp32 (num_layers, num_points, 3) in out.  Draws are keyed by (seed, layer_ids[l]).  disposition: device
 * (num_points, 3) fp64; radii: device fp64 [num_layers]; layer_ids: device int64 [num_layers]. */
int geob200_kernel_point_instances(const double* disposition, int64_t num_points, const double* radii, const int64_t* layer_ids,
                                   int64_t num_layers, uint64_t seed, float* out, void* stream);

/* ---- KPConv-FPN backbone --------------------------------------------------------------------------------- */

/* KPConv.forward (reference geotransformer/modules/kpconv/kpconv.py:79-122), fused gather -> kernel-point
 * influence -> contraction -> neighbour-count normalisation -> bias.  neighbors (n_query, n_neighbors) int64 with
 * sentinel n_support; kernel_points (15,3); weights (15, c_in, c_out); bias may be NULL.
 * c_in == 1, or c_in, c_out multiples of 32 with c_out <= 512. */
size_t geob200_kpconv_workspace_bytes(int64_t n_support);
int geob200_kpconv(const float* s_feats, const float* q_points, const float* s_points, const int64_t* neighbors,
                   int64_t n_query, int64_t n_support, int64_t n_neighbors, const float* kernel_points, int64_t n_kernel,
                   const float* weights, const float* bias, int64_t c_in, int64_t c_out, float sigma, float* out,
                   void* workspace, size_t workspace_bytes, void* stream);

/* nn.Linear: y[m,n] = x[m,k] . weight[n,k]^T + bias (UnaryBlock.mlp, modules.py:78; every transformer Linear).
 * ldx / ldy are row strides in floats (inputs may be column slices). */
/* Same op, two-stage tensor-core formulation: gather kernel (wf = influence-weighted neighbour features, M x 15 c_in) followed by
 * the 3xTF32 wgmma GEMM with the neighbour-count scale and bias in its epilogue.  weights_t is the (15*c_in, c_out) weight
 * matrix transposed to (c_out, 15*c_in). */
size_t geob200_kpconv_tc_workspace_bytes(int64_t n_query, int64_t n_support, int64_t c_in);
int geob200_kpconv_tc(const float* s_feats, const float* q_points, const float* s_points, const int64_t* neighbors, int64_t n_query,
                      int64_t n_support, int64_t n_neighbors, const float* kernel_points, int64_t n_kernel, const float* weights_t,
                      const float* bias, int64_t c_in, int64_t c_out, float sigma, float* out, void* workspace, size_t workspace_bytes,
                      void* stream);

/* tf32 split image of a row-major weight (n x k, row stride ld >= k), the operand layout of the tensor-core GEMM:
 * out (2n x k, contiguous) = [hi; lo] with hi = w rounded to tf32 (nearest, ties away from zero; low 13 bits zero) and
 * lo = w - hi in fp32. */
int geob200_split_tf32(const float* w, int64_t ld, int64_t n, int64_t k, float* out, void* stream);

/* 1 (default): Linears run on the tensor cores with 3xTF32 when the shape allows; 0: fp32 CUDA cores only */
void geob200_set_linear_mode(int mode);
int geob200_linear(const float* x, int64_t ldx, const float* weight, const float* bias, float* y, int64_t ldy, int64_t m,
                   int64_t n, int64_t k, int relu, void* stream);
int geob200_linear_batched(const float* x, int64_t ldx, int64_t stride_x, const float* weight, int64_t ldw, int64_t stride_w,
                           const float* bias, int64_t stride_b, float* y, int64_t ldy, int64_t stride_y, int64_t m, int64_t n,
                           int64_t k, int64_t batch, int relu, void* stream);

/* GroupNorm over all n_rows of the stacked pair (modules.py:33-50) + optional residual add + optional LeakyReLU:
 * y = leaky((x - mean_g) * rstd_g * gamma + beta + residual).  The first 256 bytes of the workspace must be zero
 * on first use (launch ticket; the kernel restores it). */
size_t geob200_group_norm_workspace_bytes(int64_t groups);
int geob200_group_norm(const float* x, int64_t n_rows, int64_t channels, int64_t groups, const float* gamma,
                       const float* beta, float eps, const float* residual, int leaky, float slope, float* y,
                       void* workspace, size_t workspace_bytes, void* stream);

/* Fused blocks: Linear -> GroupNorm (+ residual) (+ LeakyReLU) = UnaryBlock and the unary parts of ResidualBlock
 * (modules/kpconv/modules.py:33-104,150-225); KPConv -> GroupNorm -> LeakyReLU = ConvBlock and the conv part of
 * ResidualBlock (modules.py:107-147,205-207).  On the wgmma path the GroupNorm statistics are produced by the GEMM
 * epilogue, so the activations are not re-read for them.  pre_norm receives the Linear / KPConv output, y the result.
 * The GroupNorm workspace (>= geob200_fused_group_norm_workspace_bytes) must be zero-filled once before first use. */
size_t geob200_fused_group_norm_workspace_bytes(int64_t n_rows, int64_t channels, int64_t groups);
int geob200_linear_group_norm(const float* x, int64_t ldx, const float* weight, const float* bias, int64_t m, int64_t n, int64_t k,
                              int64_t groups, const float* gamma, const float* beta, float eps, const float* residual, int leaky,
                              float slope, float* pre_norm, float* y, void* workspace, size_t workspace_bytes, void* stream);
/* workspace: geob200_kpconv_tc_workspace_bytes(n_query, n_support, c_in) */
int geob200_kpconv_group_norm(const float* s_feats, const float* q_points, const float* s_points, const int64_t* neighbors,
                              int64_t n_query, int64_t n_support, int64_t n_neighbors, const float* kernel_points, int64_t n_kernel,
                              const float* weights_t, const float* bias, int64_t c_in, int64_t c_out, float sigma, int64_t groups,
                              const float* gamma, const float* beta, float eps, int leaky, float slope, float* pre_norm, float* y,
                              void* gn_workspace, size_t gn_workspace_bytes, void* workspace, size_t workspace_bytes, void* stream);

/* Batched forms (several pairs per forward, rows in stack order [ref_1..ref_B, src_1..src_B], cloud_rows_h[2 * n_pairs] host row
 * counts): the statistics are taken per PAIR (cloud c belongs to pair c % n_pairs), everything else is identical.
 * Workspace: geob200_fused_group_norm_workspace_bytes(n_rows, channels, groups) + 8 * groups * n_pairs + 512 bytes (the per-pair
 * statistics), zero-filled once. */
int geob200_group_norm_batched(const float* x, int64_t n_rows, int64_t channels, int64_t groups, const float* gamma, const float* beta,
                               float eps, const float* residual, int leaky, float slope, float* y, void* workspace, size_t workspace_bytes,
                               void* stream, int64_t n_pairs, const int64_t* cloud_rows_h);
int geob200_linear_group_norm_batched(const float* x, int64_t ldx, const float* weight, const float* bias, int64_t m, int64_t n, int64_t k,
                                      int64_t groups, const float* gamma, const float* beta, float eps, const float* residual, int leaky,
                                      float slope, float* pre_norm, float* y, void* workspace, size_t workspace_bytes, void* stream,
                                      int64_t n_pairs, const int64_t* cloud_rows_h);
/* geob200_kpconv_group_norm with per-pair statistics from the GEMM epilogue partials (the batched native backbone's kernels);
 * cloud_rows_h: query rows per cloud.  GroupNorm workspace as geob200_linear_group_norm_batched. */
int geob200_kpconv_group_norm_batched(const float* s_feats, const float* q_points, const float* s_points, const int64_t* neighbors,
                                      int64_t n_query, int64_t n_support, int64_t n_neighbors, const float* kernel_points, int64_t n_kernel,
                                      const float* weights_t, const float* bias, int64_t c_in, int64_t c_out, float sigma, int64_t groups,
                                      const float* gamma, const float* beta, float eps, int leaky, float slope, float* pre_norm, float* y,
                                      void* gn_workspace, size_t gn_workspace_bytes, void* workspace, size_t workspace_bytes, void* stream,
                                      int64_t n_pairs, const int64_t* cloud_rows_h);

/* maxpool over neighbour rows with a zero shadow row (functional.py:54-67) */
int geob200_maxpool(const float* x, const int64_t* neighbors, int64_t n_query, int64_t n_support, int64_t n_neighbors,
                    int64_t channels, float* y, void* stream);
/* maxpool of a batch of pairs: pair p's rows see the first min(n_neighbors, max(cloud_max[p], cloud_max[B + p])) columns only
 * (cloud_max: device int32[2 * n_pairs] of geob200_cloud_max_count; cloud_rows_h[2 * n_pairs]: query rows per cloud), as the
 * batched native backbone's strided blocks */
int geob200_maxpool_batched(const float* x, const int64_t* neighbors, int64_t n_query, int64_t n_support, int64_t n_neighbors,
                            int64_t channels, const int32_t* cloud_max, int64_t n_pairs, const int64_t* cloud_rows_h, float* y,
                            void* stream);

/* cloud_max[c] (device int32[2 * n_pairs]) = widest row (number of real neighbours) among the query rows of cloud c: the batched
 * backbone's maxpool ignores the columns of pair p past min(n_neighbors, max(cloud_max[p], cloud_max[B + p])), as
 * radius_search.py:25-26 cuts each pair's table to its own max count. */
int geob200_cloud_max_count(const int64_t* neighbors, int64_t n_query, int64_t n_support, int64_t n_neighbors, int64_t n_pairs,
                            const int64_t* cloud_rows_h, int32_t* cloud_max, void* stream);

/* y[m] = [ x_pad[up_indices[m*up_stride]] | skip[m] ]: nearest_upsample (functional.py:6-22) fused with the
 * torch.cat of the decoder (backbone.py:75-76).  skip may be NULL (c2 = 0). */
int geob200_upsample_concat(const float* x, const int64_t* up_indices, int64_t up_stride, int64_t n_support,
                            const float* skip, int64_t n_query, int64_t c1, int64_t c2, float* y, void* stream);

/* ---- backbone backward (kpconv_grad.cu) ---------------------------------------------------------------------------------------
 * Gradients of the ops above for an upstream gradient of their output.  No float atomics: every reduction has a fixed order, so
 * two calls give the same bits.  Support rows sum their (query row, column) entries in that order through a CSR transpose of the
 * index table; reductions over rows fold 256-row chunk partials in chunk order.  Index entries outside [0, n_support) are sentinels
 * and contribute nothing.  Every argument check runs before the first launch.  An output pointer may be NULL to skip that
 * gradient where noted. */

/* KPConv (c_in = 1 or a multiple of 32): grad_weights (15, c_in, c_out) = wf^T (grad_out / n_valid) with wf recomputed by the
 * forward's gather, grad_bias = column sums of grad_out, grad_feats (n_support, c_in) = the transposed gather of
 * (grad_out / n_valid) . W_flat^T with the forward's influences.  n_valid is the forward's count, a constant (it depends on the
 * signs of the feature-row sums only).  Each of the three may be NULL. */
size_t geob200_kpconv_backward_workspace_bytes(int64_t n_query, int64_t n_support, int64_t n_neighbors, int64_t c_in, int64_t c_out);
int geob200_kpconv_backward(const float* s_feats, const float* q_points, const float* s_points, const int64_t* neighbors, int64_t n_query,
                            int64_t n_support, int64_t n_neighbors, const float* kernel_points, int64_t n_kernel, const float* weights,
                            int64_t c_in, int64_t c_out, float sigma, const float* grad_out, float* grad_feats, float* grad_weights,
                            float* grad_bias, void* workspace, size_t workspace_bytes, void* stream);

/* Linear y = x . weight^T + b, optionally followed by a ReLU: grad_x (m, k) = grad_y . weight through the forward's GEMM with
 * weight_t = weight^T (k, n) contiguous; grad_weight (n, k) = grad_y^T x and grad_bias (n) in fp32 with the fixed-order fold.  relu_y:
 * the forward's output when it applied the ReLU (the gradient passes where it is positive), else NULL.  Each output may be NULL. */
size_t geob200_linear_backward_workspace_bytes(int64_t m, int64_t n, int64_t k, int relu);
int geob200_linear_backward(const float* x, int64_t ldx, const float* weight_t, const float* relu_y, int64_t m, int64_t n, int64_t k,
                            const float* grad_y, float* grad_x, float* grad_weight, float* grad_bias, void* workspace, size_t workspace_bytes,
                            void* stream);

/* y = leaky(GroupNorm(x) + residual) with per-pair statistics (layout of geob200_group_norm_batched; one pair: cloud_rows_h =
 * {n_rows, 0}).  x is the pre-norm input, y the forward's output (read for the LeakyReLU's derivative, which follows the sign of
 * the pre-activation: slope at 0; may be NULL without leaky; slope >= 0).  The statistics are recomputed from x in double.  grad_residual
 * receives the gradient after the LeakyReLU (NULL: no residual); grad_gamma / grad_beta may be NULL. */
size_t geob200_group_norm_backward_batched_workspace_bytes(int64_t n_rows, int64_t channels, int64_t groups, int64_t n_pairs);
int geob200_group_norm_backward_batched(const float* x, const float* y, int64_t n_rows, int64_t channels, int64_t groups, const float* gamma,
                                        float eps, int leaky, float slope, const float* grad_y, float* grad_x, float* grad_gamma,
                                        float* grad_beta, float* grad_residual, void* workspace, size_t workspace_bytes, void* stream,
                                        int64_t n_pairs, const int64_t* cloud_rows_h);

/* maxpool: the gradient of y[m][c] goes to the neighbour column that won the forward's max (ties: the lowest column); a winning
 * zero shadow row drops it.  cloud_max (device, may be NULL = all n_neighbors columns, as geob200_maxpool) cuts pair p's rows to
 * the width of the batched forward; cloud_rows_h[2 * n_pairs] are the query rows per cloud. */
size_t geob200_maxpool_backward_batched_workspace_bytes(int64_t n_query, int64_t n_support, int64_t n_neighbors, int64_t channels);
int geob200_maxpool_backward_batched(const float* x, const int64_t* neighbors, int64_t n_query, int64_t n_support, int64_t n_neighbors,
                                     int64_t channels, const int32_t* cloud_max, int64_t n_pairs, const int64_t* cloud_rows_h,
                                     const float* grad_y, float* grad_x, void* workspace, size_t workspace_bytes, void* stream);

/* upsample_concat: grad_x (n_support, c1) = per coarse row the sum, in fine-row order, of the first c1 columns of grad_y over the
 * fine rows that copied it; grad_skip (n_query, c2) = the last c2 columns (may be NULL). */
size_t geob200_upsample_concat_backward_workspace_bytes(int64_t n_query, int64_t n_support);
int geob200_upsample_concat_backward(const int64_t* up_indices, int64_t up_stride, int64_t n_query, int64_t n_support, int64_t c1, int64_t c2,
                                     const float* grad_y, float* grad_x, float* grad_skip, void* workspace, size_t workspace_bytes,
                                     void* stream);

/* ---- point-to-node grouping ------------------------------------------------------------------------------ */

/* The per-pair stages (grouping, structure-embedding indices, ground-truth correspondences, matching, patches, LGR, metrics) have
 * one entry point each, batched over the pairs of a forward: one launch per stage covers every cloud or pair, and one pair is
 * B = 1 (one cloud: n_clouds = 1).  Clouds are stacked [ref_1..ref_B, src_1..src_B] as in the batched collate; cloud_nodes /
 * cloud_points are HOST arrays of the 2B per-cloud row counts at the superpoint / fine (or, for geob200_evaluate_batched, input)
 * level.  Entry points with separate ref_* / src_* inputs take the B ref clouds stacked in the ref block and the B src clouds in
 * the src block.  A pair gets the same bits alone and in any batch.  Indices stay local to their cloud.  1 <= B <= 32. */
/* point_to_node_partition (reference geotransformer/modules/ops/pointcloud_partition.py:60-107) of n_clouds stacked clouds:
 * points / point_to_node at the fine offsets, nodes / node_masks / node_sizes and the (nodes, point_limit) knn tables at the
 * superpoint offsets.  node_masks / node_knn_masks are uint8 (torch.bool); node_sizes int32.  Exact for any number of points per
 * node (chunked selection).  point_limit <= 2048. */
int geob200_point_to_node_partition_batched(const float* points, const float* nodes, int64_t n_clouds, const int64_t* cloud_points,
                                            const int64_t* cloud_nodes, int64_t point_limit, int64_t* point_to_node, uint8_t* node_masks,
                                            int32_t* node_sizes, int64_t* node_knn_indices, uint8_t* node_knn_masks, void* stream);

/* knn_partition (pointcloud_partition.py:35-57): for every node the k nearest points, ascending by the matmul-form squared
 * distance pairwise_distance(nodes, points) (ties by index).  knn_sq_distances (n_nodes, k) may be NULL.  1 <= k <= min(n_points, 2048). */
int geob200_knn_partition(const float* points, int64_t n_points, const float* nodes, int64_t n_nodes, int64_t k,
                          int64_t* knn_indices, float* knn_sq_distances, void* stream);
/* pairwise_distance (ops/pairwise_distance.py:4-31) of row-major x (n, c), y (m, c): out (n, m) = clamp(x2 - 2xy + y2, 0),
 * or 2 - 2xy when normalized != 0 */
int geob200_pairwise_distance(const float* x, int64_t n, const float* y, int64_t m, int64_t channels, int normalized, float* out,
                              void* stream);
/* get_point_to_node_indices (pointcloud_partition.py:9-32): indices[i] = argmin_j pairwise_distance(points, nodes)[i, j];
 * node_sizes (int32[n_nodes], may be NULL) = points per node */
int geob200_point_to_node_indices(const float* points, int64_t n_points, const float* nodes, int64_t n_nodes, int64_t* indices,
                                  int32_t* node_sizes, void* stream);
/* apply_transform (ops/transformation.py:7-60) for one (4,4) device transform: out = points R^T + t */
int geob200_apply_transform(const float* points, int64_t n_points, const float* transform, float* out, void* stream);

/* out[r] = indices[r] < n_rows ? table[indices[r]] : 0  (index_select on a zero-padded table, ops/index_select.py) */
int geob200_gather_rows(const float* table, int64_t n_rows, int64_t channels, const int64_t* indices, int64_t n_indices,
                        float* out, void* stream);

/* ---- geometric transformer -------------------------------------------------------------------------------- */

/* GeometricStructureEmbedding.get_embedding_indices (geotransformer.py:27-55) of n_clouds stacked clouds in ONE launch
 * (cloud_rows_h: host row counts; points (sum rows, 3)): per cloud, d_indices (n,n) = sqrt(pairwise_distance)/sigma_d and
 * a_indices (n,n,3) = atan2(|ref x anc|, ref.anc) * factor_a, concatenated cloud after cloud: d_indices (sum n_c^2), a_indices
 * (sum n_c^2, 3) -- the layout geob200_gse_embed_pairs takes. */
int geob200_gse_indices_batched(const float* points, int64_t n_clouds, const int64_t* cloud_rows_h, float sigma_d, float factor_a,
                                int64_t angle_k, float* d_indices, float* a_indices, void* stream);

/* GeometricStructureEmbedding.forward (geotransformer.py:57-72) given the indices: sinusoid -> proj_d / proj_a ->
 * max over k -> sum, fused, over a flat list of n_rows (anchor, point) index rows -- the n*n (i, j) pairs of one cloud, or of several
 * clouds concatenated: d_indices (n_rows,), a_indices (n_rows, 3) -> embeddings (n_rows, channels).  wd/wa are the nn.Linear
 * weights (out,in); wd_t/wa_t their transposes (in,out).  channels 128 and 256 run a wgmma 3xFP16 split contraction
 * (fp32-accurate), any other multiple of 4 a generic fp32 CUDA-core kernel. */
size_t geob200_gse_embed_workspace_bytes(int64_t n, int64_t channels);
int geob200_gse_embed_pairs(const float* d_indices, const float* a_indices, int64_t n_rows, int64_t channels, const float* div_term,
                            const float* wd_t, const float* wa_t, const float* wd, const float* wa, const float* bd, const float* ba,
                            float* embeddings, void* workspace, size_t workspace_bytes, void* stream);

/* The same embedding through TABULATED projections (csrc/gse_table.cu).  proj_d(sinusoid(x)) and proj_a(sinusoid(x)) are
 * functions of one scalar, band-limited to 1 rad per index unit: geob200_gse_table_build tabulates both once per set of weights
 * on a uniform grid of step 1/inv_step (power of two) over [0, d_max] / [0, a_max] (fp64 accumulation; node = fp32 values + fp16
 * forward differences), geob200_gse_embed_table then needs 4 lookups + 3 max + 1 add per (row, channel) instead of the
 * 2 * (1 + 3) * C^2 flop contraction.  Linear-interpolation error <= max|g''| / (8 inv_step^2) (< 1e-6 at inv_step 256 for
 * unit-scale weights).  Index values outside the tabulated range are evaluated directly (sincosf + dot products with wd / wa),
 * so results never depend on d_max / a_max -- only the speed does.  channels: 128 or 256.  The same (channels, inv_step, d_max,
 * a_max) must be passed to both calls; table: geob200_gse_table_bytes(...) bytes of device memory, 16-byte aligned. */
size_t geob200_gse_table_bytes(int64_t channels, int64_t inv_step, float d_max, float a_max);
int geob200_gse_table_build(const float* div_term, const float* wd_t, const float* wa_t, const float* bd, const float* ba,
                            int64_t channels, int64_t inv_step, float d_max, float a_max, void* table, size_t table_bytes,
                            void* stream);
int geob200_gse_embed_table(const float* d_indices, const float* a_indices, int64_t n_rows, int64_t channels, const void* table,
                            size_t table_bytes, int64_t inv_step, float d_max, float a_max, const float* div_term, const float* wd,
                            const float* wa, const float* bd, const float* ba, float* embeddings, void* stream);

/* Fused multi-head attention: softmax((q.k + qp.E + qb)/sqrt(d)) v  (rpe_transformer.py:51-70 with proj_p moved onto
 * q; vanilla_transformer.py:50-68 when qp = qb = embed = NULL).  q (n_query,C), k,v (n_key,C), qp (n_query,H,C),
 * qb (n_query,H), embed (n_query,n_key,C).  With a workspace and C = 128 or 256 the streaming path runs (one coalesced
 * pass over embed on a (query, key-chunk) grid + a softmax/P.V kernel); workspace = NULL selects the single-kernel path. */
size_t geob200_attention_workspace_bytes(int64_t n_query, int64_t n_key, int64_t heads);
int geob200_attention(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv, const float* qp,
                      const float* qb, const float* embed, int64_t n_query, int64_t n_key, int64_t channels, int64_t heads,
                      float* out, int64_t ldo, void* workspace, size_t workspace_bytes, void* stream);
/* A batch of independent attention problems that share channels, heads and row strides (the clouds / pairs of a batched
 * forward) in ONE launch pair; all items with embed (self-attention) or all without (cross-attention).
 * Probability layout: with at most GEOB200_ATT_MAX_ITEMS items, C = 128 or 256 and every item on the streaming path, item i's
 * softmax probabilities (n_query, heads, n_key) fp32 are left in the workspace at byte offset
 * sum_{j < i} align_up(n_query_j * n_key_j * heads * 4, 256) (the backward reads them there).  Larger batches run in chunks of
 * GEOB200_ATT_MAX_ITEMS items that reuse the workspace from its start. */
#define GEOB200_ATT_MAX_ITEMS 32
typedef struct { const float* q; const float* k; const float* v; const float* qp; const float* qb; const float* embed; float* out;
                 int64_t n_query, n_key; } geob200_att_item_t;
size_t geob200_attention_batched_workspace_bytes(const geob200_att_item_t* items_h, int64_t n_items, int64_t heads);
int geob200_attention_batched(const geob200_att_item_t* items_h, int64_t n_items, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo,
                              int64_t channels, int64_t heads, void* workspace, size_t workspace_bytes, void* stream);
/* 1 when geob200_attention_batched with a workspace leaves every item's probabilities at the layout above (at most
 * GEOB200_ATT_MAX_ITEMS items, all on the streaming path), else 0 (host only, no launch) */
int geob200_attention_batched_keeps_probs(const geob200_att_item_t* items_h, int64_t n_items, int64_t channels, int64_t heads);
/* self-attention kernels: 1 (default) = TMA-staged E stream (cp.async.bulk ring, q.k and P.v as tiled passes), 0 = the
 * lanes<->channels cp.async kernels */
int geob200_set_attention_tma(int on);
int geob200_head_bias(const float* q, int64_t ldq, const float* bias_p, int64_t n, int64_t channels, int64_t heads, float* qb,
                      void* stream);
/* y = LayerNorm(a + b) (b may be NULL) */
int geob200_add_layernorm(const float* a, const float* b, const float* gamma, const float* beta, int64_t n, int64_t channels,
                          float eps, float* y, void* stream);
/* F.normalize(x, p=2, dim=1) */
int geob200_l2_normalize(const float* x, int64_t n, int64_t channels, float* y, void* stream);

/* ---- geometric transformer: backward ----------------------------------------------------------------------- */
/* No float atomics: two runs give the same bits.  Sums over rows run on fixed row chunks folded in chunk order in double. */

/* y = LayerNorm(a + b) gamma + beta: grad_x (n, C) is the gradient of both summands; the statistics are recomputed per row from
 * a + b (b may be NULL).  grad_gamma / grad_beta may be NULL.  channels <= 1024. */
size_t geob200_add_layernorm_backward_workspace_bytes(int64_t n, int64_t channels);
int geob200_add_layernorm_backward(const float* a, const float* b, const float* gamma, int64_t n, int64_t channels, float eps,
                                   const float* grad_y, float* grad_x, float* grad_gamma, float* grad_beta, void* workspace,
                                   size_t workspace_bytes, void* stream);
/* y = x / max(|x|, 1e-12) per row: grad_x (n, C); needs no workspace. */
int geob200_l2_normalize_backward(const float* x, int64_t n, int64_t channels, const float* grad_y, float* grad_x, void* stream);
/* head_project (qp[n,h,:] = Wp_h^T q_h, qb[n,h] = q_h . bp_h, Wp_h = rows h d .. h d + d - 1 of the nn.Linear weight wp (C, C)):
 * grad_q (row stride ldgq, may be a column slice) through geob200_linear_batched over heads, grad_wp (C, C) and grad_bp (C) as
 * fixed-order row sums.  Each output may be NULL. */
size_t geob200_head_project_backward_workspace_bytes(int64_t n, int64_t channels, int64_t heads);
int geob200_head_project_backward(const float* q, int64_t ldq, const float* wp, const float* bp, int64_t n, int64_t channels, int64_t heads,
                                  const float* grad_qp, const float* grad_qb, float* grad_q, int64_t ldgq, float* grad_wp, float* grad_bp,
                                  void* workspace, size_t workspace_bytes, void* stream);
/* Attention backward for the items of a forward (geob200_att_item_t: the forward's inputs, `out` its output with row stride ldo).
 * Per item: probs = the (n_query, H, n_key) softmax probabilities the streaming forward leaves in its workspace, grad_out the
 * (n_query, C) contiguous upstream gradient; grad_q / grad_k / grad_v (row strides ldgq / ldgk / ldgv: column slices of one fused
 * gradient allowed; each may be NULL) and, for self-attention items, grad_qp (n_query, H, C), grad_qb (n_query, H) and
 * grad_embed (n_query, n_key, C) (grad_qp and grad_embed together; NULL skips the E pass).  channels 128 or 256. */
typedef struct { const float* probs; const float* grad_out; float* grad_q; float* grad_k; float* grad_v; float* grad_qp; float* grad_qb;
                 float* grad_embed; } geob200_att_grad_item_t;
size_t geob200_attention_backward_batched_workspace_bytes(const geob200_att_item_t* items_h, int64_t n_items, int64_t heads);
int geob200_attention_backward_batched(const geob200_att_item_t* items_h, const geob200_att_grad_item_t* grads_h, int64_t n_items,
                                       int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo, int64_t ldgq, int64_t ldgk, int64_t ldgv,
                                       int64_t channels, int64_t heads, void* workspace, size_t workspace_bytes, void* stream);
/* Structure embedding E = proj_d(s(d)) + max_k proj_a(s(a_k)) given grad_embed (n_rows, C): grad_wd / grad_wa (C, C, nn.Linear
 * layout) and grad_bd = grad_ba (C).  The winning angle term of every (row, channel) comes from the lookups of
 * geob200_gse_embed_table with the table of the current weights (same table arguments); the sinusoid is evaluated with sincosf.
 * channels 128 or 256, angle_k 3. */
size_t geob200_gse_embed_backward_workspace_bytes(int64_t n_rows, int64_t channels);
int geob200_gse_embed_backward(const float* d_indices, const float* a_indices, int64_t n_rows, int64_t angle_k, int64_t channels,
                               const void* table, size_t table_bytes, int64_t inv_step, float d_max, float a_max, const float* div_term,
                               const float* wa, const float* ba, const float* grad_embed, float* grad_wd, float* grad_bd, float* grad_wa,
                               float* grad_ba, void* workspace, size_t workspace_bytes, void* stream);

/* ---- matching ---------------------------------------------------------------------------------------------- */

/* SuperPointMatching.forward (superpoint_matching.py:13-50): ref_feats / ref_masks hold the superpoint rows of the B ref clouds,
 * src_feats / src_masks those of the B src clouds; masks are uint8 (torch.bool) or NULL (= all valid).  corr_indices
 * (2B, num_correspondences): row p = ref indices of pair p, row B + p = its src indices; corr_scores (B, num_correspondences);
 * num_out[p] (device int32) = number of rows written = min(num_correspondences, #valid ref nodes x #valid src nodes); rows past it
 * receive index -1 / score 0.  num_correspondences in 1..1024.  Workspace for n_rows = all 2B clouds' rows and n_products = sum over
 * pairs of n_ref * n_src. */
size_t geob200_superpoint_matching_batched_workspace_bytes(int64_t n_rows, int64_t n_products, int64_t n_pairs);
int geob200_superpoint_matching_batched(const float* ref_feats, const float* src_feats, int64_t channels, const uint8_t* ref_masks,
                                        const uint8_t* src_masks, int64_t n_pairs, const int64_t* cloud_nodes, int64_t num_correspondences,
                                        int dual, int64_t* corr_indices, float* corr_scores, int32_t* num_out, void* workspace,
                                        size_t workspace_bytes, void* stream);

/* patch gathers of model.py:169-174 over n_clouds stacked clouds (knn tables at the superpoint offsets, points at the fine
 * offsets): indices/masks/points of the k points of each selected superpoint.  Cloud c gathers the n_corr patches
 * corr_indices[c * n_corr ..] to rows c * n_corr; a negative corr index (padding row of geob200_superpoint_matching_batched) yields
 * an empty patch (sentinel indices, masks 0).  With corr_indices = NULL every node of cloud c is a patch (corr = arange), written at
 * the cloud's superpoint offset. */
int geob200_gather_patches_batched(const int64_t* corr_indices, int64_t n_corr, int64_t n_clouds, const int64_t* cloud_nodes,
                                   const int64_t* cloud_points, const int64_t* node_knn_indices, const uint8_t* node_knn_masks, int64_t k,
                                   const float* points, int64_t* out_indices, uint8_t* out_masks, float* out_points, void* stream);

/* matching_scores = einsum('bnd,bmd->bnm') / sqrt(C) over zero-padded feature tables (model.py:176-188): ref_feats / src_feats hold
 * the fine rows of the B ref / src clouds; pair p's n_patches patches at p * n_patches of ref_knn_indices, src_knn_indices and
 * scores. */
int geob200_patch_scores_batched(const float* ref_feats, const float* src_feats, int64_t channels, int64_t n_pairs, const int64_t* cloud_points,
                                 const int64_t* ref_knn_indices, const int64_t* src_knn_indices, int64_t n_patches, int64_t k,
                                 float* scores, void* stream);

/* Backward of geob200_patch_scores_batched (same layout): grad_scores (n_pairs * n_patches, k, k) -> grad_ref_feats / grad_src_feats
 * with the shapes of ref_feats / src_feats, every row written (zero where no patch reads it).  dR_p = dS_p Fs_p / sqrt(C) and
 * dS'_p = dS_p^T Fr_p / sqrt(C) per patch, then each feature row sums its (patch, slot) entries in (patch, slot) order (counting sort
 * of the entries by row; no float atomics).  Sentinel indices (>= the cloud's row count) receive nothing.  n_rows of the workspace
 * query = all ref + src rows; n_patches_total = n_pairs * n_patches. */
size_t geob200_patch_scores_backward_batched_workspace_bytes(int64_t n_rows, int64_t n_patches_total, int64_t k, int64_t channels);
int geob200_patch_scores_backward_batched(const float* ref_feats, const float* src_feats, int64_t channels, int64_t n_pairs,
                                          const int64_t* cloud_points, const int64_t* ref_knn_indices, const int64_t* src_knn_indices,
                                          int64_t n_patches, int64_t k, const float* grad_scores, float* grad_ref_feats,
                                          float* grad_src_feats, void* workspace, size_t workspace_bytes, void* stream);

/* LearnableLogOptimalTransport.forward (learnable_sinkhorn.py:20-66): out (n_patches, k+1, k+1) */
int geob200_sinkhorn(const float* scores, const uint8_t* row_masks, const uint8_t* col_masks, const float* alpha,
                     int64_t n_patches, int64_t k, int64_t num_iterations, float inf, float* out, void* stream);

/* Backward of geob200_sinkhorn: grad_out (n_patches, k+1, k+1) -> grad_scores (n_patches, k, k), zero on masked entries, and
 * grad_alpha (one device float) = the sum of the gradient over the unmasked dustbin entries of all patches, summed per patch and then
 * over the patches in index order (no atomics: a patch gives the same bits alone and in any batch).  The CTA of a patch re-runs the
 * forward iterations and keeps their log-sum-exps in the workspace (2 * num_iterations * (k+1) floats per patch), then sweeps them in
 * reverse.  Masked lines follow the inf -> infinity limit (finite for any grad_out); a patch without a valid row and without a valid
 * column gets zeros.  k must be 32, 64 or 128. */
size_t geob200_sinkhorn_backward_workspace_bytes(int64_t n_patches, int64_t k, int64_t num_iterations);
int geob200_sinkhorn_backward(const float* scores, const uint8_t* row_masks, const uint8_t* col_masks, const float* alpha, int64_t n_patches,
                              int64_t k, int64_t num_iterations, float inf, const float* grad_out, float* grad_scores, float* grad_alpha,
                              void* workspace, size_t workspace_bytes, void* stream);

/* ---- local-to-global registration -------------------------------------------------------------------------- */

/* LocalGlobalRegistration.forward (local_global_registration.py:196-235), use_dustbin=False, use_global_score=False,
 * correspondence_limit=None, for n_pairs pairs of n_patches patches each (pair p at patch p * n_patches).  log_scores
 * (P, score_ld, score_ld) with score_ld = k or k+1 (dustbin row/col ignored).  Pair p's correspondence rows start at
 * p * n_patches * k * topk (x2 when not mutual); num_corr[p] (device int32) = rows written, in (patch,i,j) order.  Its transform goes
 * to estimated_transform + p * transform_ld (>= 16).  patch_transforms (P,4,4), patch_inliers (P, -1 = patch below
 * correspondence_threshold) and best_patch (n_pairs) may be NULL. */
size_t geob200_lgr_batched_workspace_bytes(int64_t n_pairs, int64_t n_patches, int64_t k, int64_t topk);
int geob200_local_global_registration_batched(const float* ref_knn_points, const float* src_knn_points, const uint8_t* ref_knn_masks,
                                              const uint8_t* src_knn_masks, const float* log_scores, int64_t n_pairs, int64_t n_patches,
                                              int64_t k, int64_t score_ld, int64_t topk, float acceptance_radius, int mutual,
                                              float confidence_threshold, int64_t correspondence_threshold, int64_t num_refinement_steps,
                                              float* ref_corr_points, float* src_corr_points, float* corr_scores, int32_t* corr_patch,
                                              int32_t* num_corr, float* estimated_transform, int64_t transform_ld, float* patch_transforms,
                                              int32_t* patch_inliers, int32_t* best_patch, void* workspace, size_t workspace_bytes,
                                              void* stream);

/* weighted_procrustes (modules/registration/procrustes.py:6-73): transforms (batch,4,4); weights may be NULL */
int geob200_weighted_procrustes(const float* src_points, const float* ref_points, const float* weights, int64_t batch,
                                int64_t n, float weight_thresh, float eps, float* transforms, void* stream);

/* get_node_correspondences (modules/registration/matching.py:231-315): ground-truth superpoint pairs and their overlap
 * ratios under transforms (B,4,4, device).  ref_nodes / ref_masks and the (rows, k, 3) patch points / (rows, k) masks of the B ref
 * clouds in the ref_* block, those of the B src clouds in the src_* block; masks are uint8 (torch.bool) or NULL (= all valid).
 * Pair p's rows start at sum_{q<p} n_ref(q) * n_src(q) of corr_indices (rows of 2 int64) / corr_overlaps (that many rows of
 * capacity) and receive the pairs with overlap > 0 in row-major (ref, src) order, count[p] (device int32) their number. */
size_t geob200_node_correspondences_batched_workspace_bytes(int64_t n_rows, int64_t n_products, int64_t k);
int geob200_node_correspondences_batched(const float* ref_nodes, const float* src_nodes, const float* ref_knn_points,
                                         const float* src_knn_points, const uint8_t* ref_masks, const uint8_t* src_masks,
                                         const uint8_t* ref_knn_masks, const uint8_t* src_knn_masks, int64_t n_pairs, const int64_t* cloud_nodes,
                                         int64_t k, const float* transforms, float pos_radius, int64_t* corr_indices, float* corr_overlaps,
                                         int32_t* count, void* workspace, size_t workspace_bytes, void* stream);

/* Evaluator.forward (experiments/<exp>/loss.py:95-159; metrics.py:47-112) of one pair: metrics[8] (device) =
 * {PIR, IR, RRE [deg], RTE, RMSE, RR, #correspondences, #gt superpoint pairs}.  mode 0 = 3DMatch (RMSE of the realigned
 * source cloud, RR = RMSE < rmse_threshold), 1 = KITTI (no RMSE: NaN; RR = RRE < rre_threshold and RTE < rte_threshold),
 * 2 = ModelNet (RMSE of T_est x - T_gt x; RR as KITTI).  Means over empty sets are NaN, as torch reports them.
 * The three row counts are optionally taken from DEVICE memory (int32, as geob200_node_correspondences_batched /
 * geob200_superpoint_matching_batched / geob200_local_global_registration_batched write them): a non-NULL *_dev pointer overrides
 * the host value (n_node_corr: the smaller of the two), so a whole forward can be enqueued without a host read-back in between. */
int geob200_evaluate_counts(const int64_t* gt_node_corr_indices, const float* gt_node_corr_overlaps, int64_t n_gt, const int32_t* n_gt_dev,
                            float acceptance_overlap, const int64_t* ref_node_corr_indices, const int64_t* src_node_corr_indices,
                            int64_t n_node_corr, const int32_t* n_node_corr_dev, const float* ref_corr_points, const float* src_corr_points,
                            int64_t n_corr, const int32_t* n_corr_dev, float acceptance_radius, const float* gt_transform,
                            const float* est_transform, const float* src_points, int64_t n_src_points, int mode, float rmse_threshold,
                            float rre_threshold, float rte_threshold, float* metrics, void* stream);
/* Batched, one CTA per pair, counts from device memory: ground-truth rows of pair p as laid out by
 * geob200_node_correspondences_batched (cloud_nodes), n_node_corr / n_corr rows of capacity per pair (pair p at p * that),
 * gt_transforms (B,4,4), est_transforms at p * transform_ld, the source cloud of pair p = stacked cloud B + p of `points`
 * (cloud_points: 2B counts), metrics at p * metrics_ld (>= 8). */
int geob200_evaluate_batched(const int64_t* gt_node_corr_indices, const float* gt_node_corr_overlaps, const int32_t* n_gt_dev,
                             float acceptance_overlap, const int64_t* ref_node_corr_indices, const int64_t* src_node_corr_indices,
                             int64_t n_node_corr, const int32_t* n_node_corr_dev, const float* ref_corr_points, const float* src_corr_points,
                             int64_t n_corr, const int32_t* n_corr_dev, float acceptance_radius, const float* gt_transforms,
                             const float* est_transforms, int64_t transform_ld, const float* points, int64_t n_pairs, const int64_t* cloud_nodes,
                             const int64_t* cloud_points, int mode, float rmse_threshold, float rre_threshold, float rte_threshold,
                             float* metrics, int64_t metrics_ld, void* stream);

/* Validation losses (OverallLoss, experiments/<exp>/loss.py:10-92 with modules/loss/circle_loss.py:44-86): the values the reference
 * computes in val_step, without gradients.  Pair p writes its row out[p * out_ld + {0: loss, 1: c_loss, 2: f_loss}] (out_ld >= 3).
 * Batched over B pairs like geob200_evaluate_batched (cloud_nodes: HOST array of the 2B per-cloud superpoint counts, ref clouds
 * first); one pair is B = 1.  Every reduction runs in a fixed order: results are bit-identical run to run, and a pair gets the same
 * bits alone and in a batch.  Means over empty selections are NaN, as torch reports them.  Bad arguments (unsupported k,
 * non-positive log_scale or radius, negative counts) are rejected before any launch.
 *
 * Coarse (CoarseMatchingLoss + WeightedCircleLoss) over ALL n_ref x n_src superpoints of each pair (no node mask): ref superpoints of
 * pair p at rows sum_{q<p} n_ref(q) of ref_feats, src superpoints at rows sum_{q<p} n_src(q) of src_feats (both (rows, channels),
 * L2-normalised).  Ground-truth rows of pair p at sum_{q<p} n_ref(q) * n_src(q) of gt_node_corr_indices / _overlaps as
 * geob200_node_correspondences_batched lays them out; the first gt_count[p] (device int32, required) are valid.  Writes column 1. */
size_t geob200_coarse_matching_loss_batched_workspace_bytes(int64_t n_rows, int64_t n_products);
int geob200_coarse_matching_loss_batched(const float* ref_feats, const float* src_feats, int64_t channels, int64_t n_pairs,
                                         const int64_t* cloud_nodes, const int64_t* gt_node_corr_indices, const float* gt_node_corr_overlaps,
                                         const int32_t* gt_count, float positive_margin, float negative_margin, float positive_optimal,
                                         float negative_optimal, float log_scale, float positive_overlap, float* out, int64_t out_ld,
                                         void* workspace, size_t workspace_bytes, void* stream);
/* Fine (FineMatchingLoss): n_patches patches of k (64 or 128) points per pair, patch q of pair p at row p * n_patches + q of the
 * (rows, k, 3) points, (rows, k) uint8 masks and (rows, k+1, k+1) Sinkhorn scores; transforms (B,4,4) device.  patch_count
 * (device int32 per pair, may be NULL = all) limits the patches read; padding patches beyond it are never read.  positive_radius is
 * squared in double and rounded to fp32 once, like the reference's comparison.  Writes column 2; with loss_weights (HOST
 * {w_coarse, w_fine}, may be NULL) also column 0 = w_coarse * column 1 + w_fine * column 2, so run it after the coarse loss on the
 * same stream. */
size_t geob200_fine_matching_loss_batched_workspace_bytes(int64_t n_pairs, int64_t n_patches);
int geob200_fine_matching_loss_batched(const float* ref_knn_points, const float* src_knn_points, const uint8_t* ref_knn_masks,
                                       const uint8_t* src_knn_masks, const float* matching_scores, const float* transforms, int64_t n_pairs,
                                       int64_t n_patches, int64_t k, const int32_t* patch_count, double positive_radius,
                                       const float* loss_weights, float* out, int64_t out_ld, void* workspace, size_t workspace_bytes,
                                       void* stream);

/* Backward of the two losses.  grad_rows (device, n_pairs rows of stride grad_ld >= 3) is the upstream gradient of the [loss, c_loss,
 * f_loss] rows; with loss_weights (HOST {w_coarse, w_fine}, may be NULL) column 0 reaches c_loss / f_loss through the weights.  The
 * arguments otherwise mirror the forward entry points.  Coarse: grad_ref_feats / grad_src_feats (shapes of ref_feats / src_feats); a
 * half (rows or columns) of a pair with no kept line contributes zero, as torch autograd gives on the NaN loss, and an entry at feature
 * distance 0 gives inf / NaN where torch's sqrt backward does.  Fine: grad_scores (n_pairs * n_patches, k+1, k+1) = -g / #labels of
 * the pair on the label entries, 0 elsewhere (and everywhere for a pair without labels or a patch at or beyond patch_count[p]). */
size_t geob200_coarse_matching_loss_backward_batched_workspace_bytes(int64_t n_rows, int64_t n_products, int64_t n_pairs);
int geob200_coarse_matching_loss_backward_batched(const float* ref_feats, const float* src_feats, int64_t channels, int64_t n_pairs,
                                                  const int64_t* cloud_nodes, const int64_t* gt_node_corr_indices,
                                                  const float* gt_node_corr_overlaps, const int32_t* gt_count, float positive_margin,
                                                  float negative_margin, float positive_optimal, float negative_optimal, float log_scale,
                                                  float positive_overlap, const float* grad_rows, int64_t grad_ld, const float* loss_weights,
                                                  float* grad_ref_feats, float* grad_src_feats, void* workspace, size_t workspace_bytes,
                                                  void* stream);
size_t geob200_fine_matching_loss_backward_batched_workspace_bytes(int64_t n_pairs, int64_t n_patches);
int geob200_fine_matching_loss_backward_batched(const float* ref_knn_points, const float* src_knn_points, const uint8_t* ref_knn_masks,
                                                const uint8_t* src_knn_masks, const float* transforms, int64_t n_pairs, int64_t n_patches,
                                                int64_t k, const int32_t* patch_count, double positive_radius, const float* grad_rows,
                                                int64_t grad_ld, const float* loss_weights, float* grad_scores, void* workspace,
                                                size_t workspace_bytes, void* stream);

/* Correspondence RANSAC (Open3D's registration_ransac_based_on_correspondence as utils/open3d.py:169-198 calls it) for B pairs:
 * pair p's correspondences are rows [0, num_corr[p]) of (B, capacity, 3) ref / src arrays (num_corr: device int32 or NULL = all
 * capacity rows).  All num_iterations hypotheses run; hypothesis i draws ransac_n indices with replacement from Philox4x32-10
 * (key = seed, counter = (i, pair_base + p, j / 4, 0), index = umulhi(word j % 4, n)), fits an unweighted Kabsch, and counts the inliers
 * ||R src + t - ref||^2 < tau^2 in pinned fp32 arithmetic.  Winner: most inliers, then lowest rmse, then lowest i.  Outputs per
 * pair: transforms (B, 16) row-major, fitness = inliers / n, inlier_rmse, inlier_count, best_iteration (-1 and identity when no
 * hypothesis has an inlier or n < ransac_n).  Optional per-hypothesis records (each NULL or (B, num_iterations, ...)):
 * hyp_transforms (16 floats), hyp_inliers, hyp_rmse, hyp_samples (8 int32, -1 past ransac_n).  ransac_n in 3..8. */
size_t geob200_ransac_correspondences_batched_workspace_bytes(int64_t n_pairs, int64_t num_iterations);
int geob200_ransac_correspondences_batched(const float* ref_corr_points, const float* src_corr_points, int64_t n_pairs, int64_t capacity,
                                           const int32_t* num_corr, float distance_threshold, int64_t ransac_n, int64_t num_iterations,
                                           uint64_t seed, int64_t pair_base, float* transforms, float* fitness, float* inlier_rmse,
                                           int32_t* inlier_count,
                                           int32_t* best_iteration, float* hyp_transforms, int32_t* hyp_inliers, float* hyp_rmse,
                                           int32_t* hyp_samples, void* workspace, size_t workspace_bytes, void* stream);

/* evaluate_correspondences (utils/registration.py:240-250) for B pairs in the RANSAC layout: row p of out (stride out_ld >= 4)
 * = [inlier ratio, overlap, mean residual, count] under transforms + p * transform_ld (row-major, >= 12 floats).  The overlap is
 * the fraction of ref correspondence points whose nearest transformed src correspondence point is closer than positive_radius
 * (brute force).  The means of an empty pair are NaN. */
size_t geob200_correspondence_metrics_batched_workspace_bytes(int64_t n_pairs, int64_t capacity);
int geob200_correspondence_metrics_batched(const float* ref_corr_points, const float* src_corr_points, int64_t n_pairs, int64_t capacity,
                                           const int32_t* num_corr, const float* transforms, int64_t transform_ld, float positive_radius,
                                           float* out, int64_t out_ld, void* workspace, size_t workspace_bytes, void* stream);

/* ---- feature matching (utils/pointcloud.py:11-22, utils/registration.py:179-234, utils/open3d.py:133-166) --------------------
 * Exact nearest neighbour in descriptor space for B pairs (feature_match.cu): query (B, cap_query, C) and support
 * (B, cap_support, C) fp32, device int32 counts n_query / n_support (NULL = all capacity rows), C in 1..1024.  For every query row
 * q: query_index = argmin over the support rows s of D(q, s) = sum_c (q_c - s_c)^2 in fp64 (c in order, no FMA), the lowest s on
 * exact ties, and query_dist = sqrt(D).  With support_index / support_dist (both or neither) also every support row's nearest
 * query row.  Rows past the count: index -1, distance NaN; an empty other side: index -1, distance +inf. */
size_t geob200_feature_nn_batched_workspace_bytes(int64_t n_pairs, int64_t cap_query, int64_t cap_support);
int geob200_feature_nn_batched(const float* query, const float* support, int64_t n_pairs, int64_t cap_query, int64_t cap_support,
                               int64_t channels, const int32_t* n_query, const int32_t* n_support, int64_t* query_index,
                               double* query_dist, int64_t* support_index, double* support_dist, void* workspace, size_t workspace_bytes,
                               void* stream);
/* Correspondence lists of one pair from its two nearest-neighbour directions (extract_corr_indices_from_feats): mode 0 plain
 * (r <-> ref_nn[r] for every ref row), 1 mutual (only the r with src_nn[ref_nn[r]] == r, increasing r), 2 bilateral (plain, then
 * src_nn[s] <-> s for every src row).  Outputs hold n_ref (+ n_src for bilateral) rows; count (device) = the rows written;
 * feat_dist (may be NULL) = the listed pairs' descriptor distances in fp32. */
int geob200_feature_corr_indices(const int64_t* ref_nn, const double* ref_dist, const int64_t* src_nn, const double* src_dist,
                                 int64_t n_ref, int64_t n_src, int32_t mode, int64_t* ref_corr, int64_t* src_corr, float* feat_dist,
                                 int32_t* count, void* stream);
/* Feature-matching RANSAC (Open3D 0.11's registration_ransac_based_on_feature_matching as utils/open3d.py:133-166 calls it:
 * edge-length checker 0.9, distance checker tau, RANSACConvergenceCriteria(num_iterations, val_iterations)) for B pairs:
 * src (B, cap_src, 3) points + (B, cap_src, C) descriptors, ref likewise, device counts n_src / n_ref (NULL = all).
 * Source row s matches m(s) = its nearest ref descriptor.  Iteration i draws ransac_n src rows with replacement (the Philox stream of
 * the correspondence RANSAC, counter (i, pair_base + p, j / 4, 0), index = umulhi(word, n_src)); it passes when every sampled edge
 * satisfies 0.9 d_tgt <= d_src and 0.9 d_src <= d_tgt and the unweighted Kabsch fit leaves every sample within tau (both in
 * double).  The first min(val_iterations, #passing) passing iterations in iteration order are scored against the WHOLE ref
 * cloud: a src point is an inlier when its transformed position's nearest ref point has pinned-fp32 d^2 < tau^2; fitness =
 * inliers / n_src, rmse = sqrt(sum d^2 / inliers).  Winner: higher fitness, then lower rmse, then lower iteration; none with an
 * inlier, ransac_n < 3, tau <= 0, num_iterations == 0 or val_iterations == 0: identity, fitness 0, rmse 0, iteration -1.
 * Outputs per pair: transforms (B, 16), fitness, inlier_rmse, inlier_count, best_iteration, num_validated.  Optional records
 * (each NULL or written): rec_matches (B, cap_src) int64 = m(s), rec_samples (B, I, 8) (-1 past ransac_n), rec_pass (B, I),
 * rec_val_ids (B, V') (-1 past num_validated), rec_transforms (B, V', 16), rec_inliers (B, V'), rec_rmse (B, V') with
 * V' = min(val_iterations, num_iterations).  ransac_n in 0..8, C in 1..1024. */
size_t geob200_ransac_features_batched_workspace_bytes(int64_t n_pairs, int64_t cap_src, int64_t cap_ref, int64_t num_iterations,
                                                       int64_t val_iterations);
int geob200_ransac_features_batched(const float* src_points, const float* ref_points, const float* src_feats, const float* ref_feats,
                                    int64_t n_pairs, int64_t cap_src, int64_t cap_ref, int64_t channels, const int32_t* n_src,
                                    const int32_t* n_ref, float distance_threshold, int64_t ransac_n, int64_t num_iterations,
                                    int64_t val_iterations, uint64_t seed, int64_t pair_base, float* transforms, float* fitness,
                                    float* inlier_rmse, int32_t* inlier_count, int32_t* best_iteration, int32_t* num_validated,
                                    int64_t* rec_matches, int32_t* rec_samples, int32_t* rec_pass, int32_t* rec_val_ids,
                                    float* rec_transforms, int32_t* rec_inliers, float* rec_rmse, void* workspace, size_t workspace_bytes,
                                    void* stream);

/* ---- benchmark evaluation (the experiments' eval.py; benchmark.cu) -------------------------------------------------------------
 * Ragged pairs in the (B, capacity, .) layout with device int32 counts (NULL = all capacity rows), one launch for B pairs, no host
 * sync; a pair gets the same bits alone and in any batch.
 *
 * Score order: order[p][0 .. min(n, kmax)) = np.argsort(-scores[p][:n], kind='stable')[:kmax] (score descending, then row
 * ascending; -0 == +0; NaN after every number), -1 beyond.  kmax in 1..8192.  order: (B, kmax) int32. */
int geob200_corr_order_batched(const float* scores, int64_t n_pairs, int64_t capacity, const int32_t* num_corr, int64_t kmax, int32_t* order,
                               void* stream);
/* Top-k selection as eval.py:125-129 does it: count_out[p] = min(n, k); row i of pair p in the (B, min(k, capacity), .) outputs is
 * row order[p][i] when n > k and row i (the original order) when n <= k; zeros beyond the count.  order from
 * geob200_corr_order_batched with the same kmax; k in 1..kmax. */
int geob200_corr_select_batched(const float* ref_corr_points, const float* src_corr_points, const float* corr_scores, int64_t n_pairs,
                                int64_t capacity, const int32_t* num_corr, const int32_t* order, int64_t kmax, int64_t k,
                                float* ref_out, float* src_out, float* scores_out, int32_t* count_out, void* stream);
/* evaluate_sparse_correspondences (utils/registration.py:253-281): out[p] = [precision, recall, hit_ratio] in double, equal to
 * numpy's bit for bit.  Predicted pairs: rows [0, pred_count[p]) of (B, pred_cap) int64 ref / src node indices; gt pairs: rows
 * [0, gt_count[p]) of (B, gt_cap, 2) int64.  Node indices are below m_cap (ref) / n_cap (src); pairs outside are ignored.  The gt
 * and predicted sets are bitmaps: in shared memory when they fit, otherwise in the workspace (0 bytes when they fit). */
size_t geob200_sparse_correspondence_eval_batched_workspace_bytes(int64_t n_pairs, int64_t m_cap, int64_t n_cap);
int geob200_sparse_correspondence_eval_batched(const int64_t* ref_node_corr_indices, const int64_t* src_node_corr_indices, int64_t pred_cap,
                                               const int32_t* pred_count, const int64_t* gt_node_corr_indices, int64_t gt_cap,
                                               const int32_t* gt_count, int64_t n_pairs, int64_t m_cap, int64_t n_cap, double* out,
                                               void* workspace, size_t workspace_bytes, void* stream);
/* Registration error in double: out[p] = [rre (deg), rte, p, accepted] for the row-major 4x4 transforms at gt_transforms + p * gt_ld
 * and est_transforms + p * est_ld.  p = compute_transform_error (threedmatch/utils.py:130-136: inv(gt) est, nibabel's mat2quat,
 * er^T C er / C[0][0]) with the (B, 36) covariances where has_covariance[p] != 0 (NULL = every pair), NaN elsewhere.
 * mode 0 (3DMatch): accepted = has a covariance and p < threshold0; mode 1 (KITTI): rre < threshold0 and rte < threshold1. */
int geob200_registration_error_batched(const float* gt_transforms, int64_t gt_ld, const float* est_transforms, int64_t est_ld,
                                       const float* covariances, const int32_t* has_covariance, int64_t n_pairs, int mode,
                                       double threshold0, double threshold1, double* out, void* stream);
/* geob200_weighted_procrustes over ragged problems: problem b = rows [0, counts[b]) of (batch, capacity, 3) src / ref and
 * (batch, capacity) weights (may be NULL); bit-identical to geob200_weighted_procrustes on the trimmed rows. */
int geob200_weighted_procrustes_counts(const float* src_points, const float* ref_points, const float* weights, int64_t batch,
                                       int64_t capacity, const int32_t* counts, float weight_thresh, float eps, float* transforms,
                                       void* stream);

/* Profiling aid (bench.py roofline): while enabled, every tensor-core GEMM launch (nn.Linear and the KPConv contraction) is
 * bracketed by CUDA events on its stream; _read synchronises them and returns the count, shapes[3i..] = (m, n, k), ms[i]. */
int geob200_linear_profile_enable(int on);
/* split-K for deep-K GEMMs on few tiles (default on); off = every tile runs its whole K loop in one CTA */
int geob200_set_split_k(int on);
/* persistent tile loop (one CTA per SM) for GEMMs of more than one wave of tiles (default on) */
int geob200_set_linear_persistent(int on);
int64_t geob200_linear_profile_read(int64_t capacity, int64_t* shapes, float* ms);

/* ---- native stage drivers (native.cu) ------------------------------------------------------------------------
 * The whole KPConv-FPN backbone / geometric transformer as ONE call for a batch of pairs (one pair: n_pairs = 1): same kernels in
 * the same order as the per-op entry points above (bitwise-identical results), driven from C++ so that the host cost per pair is a
 * few hundred microseconds instead of milliseconds.  All pointers are device pointers; the structs are plain C (built from a
 * state_dict by geotransformer_b200/native.py). */
#define GEOB200_MAX_STAGES 6
/* weight_img / weights_img / *_img: optional tf32 split images (geob200_split_tf32) of weight / weights_t / the fused
 * projection weights, read by the tensor-core GEMM; NULL = split on every call. */
typedef struct { const float* weight; const float* bias; int64_t c_in, c_out; const float* weight_img; } geob200_linear_t;
typedef struct { const float* gamma; const float* beta; } geob200_norm_t;
typedef struct { const float* weights; const float* weights_t; const float* bias; const float* kernel_points;
                 int64_t c_in, c_out; float sigma; const float* weights_img; } geob200_kpconv_t;
/* ResidualBlock (reference geotransformer/modules/kpconv/modules.py:151-225) */
typedef struct {
    int32_t has_unary1, has_shortcut, strided, reserved;
    int64_t c_in;
    geob200_linear_t unary1; geob200_norm_t norm1;
    geob200_kpconv_t conv;   geob200_norm_t norm_conv;
    geob200_linear_t unary2; geob200_norm_t norm2;
    geob200_linear_t shortcut; geob200_norm_t norm_sc;
} geob200_resblock_t;
/* KPConvFPN (reference experiments/.../backbone.py): encoder1_1 = conv1+norm1, blocks[0] = encoder1_2, then three blocks per
 * further level; decoders[0] is the coarsest decoder, the last one (level finest_decoder) has no norm/activation. */
typedef struct {
    int32_t num_stages, finest_decoder, groups, init_dim;
    geob200_kpconv_t conv1; geob200_norm_t norm1;
    geob200_resblock_t blocks[1 + 3 * (GEOB200_MAX_STAGES - 1)];
    geob200_linear_t decoders[GEOB200_MAX_STAGES];
    geob200_norm_t decoder_norms[GEOB200_MAX_STAGES];
} geob200_backbone_t;
size_t geob200_backbone_workspace_bytes(const geob200_backbone_t* net, const int64_t* level_rows);
/* KPConvFPN.forward over n_pairs pairs in stack order [ref_1..ref_B, src_1..src_B] at every level (the reference collate with
 * batch_size B, utils/data.py:144): identical kernels over the stacked rows; the GroupNorm statistics are taken per pair
 * (modules/kpconv/modules.py:46-50 normalises over the stacked rows of ONE pair).  n_pairs <= 32.  out_feats[0] = coarsest encoder
 * output (rows level_rows[S-1]); out_feats[i>0] = decoder outputs, coarse to fine.  The GroupNorm workspace
 * (geob200_fused_group_norm_workspace_bytes(level_rows[0], init_dim << num_stages, groups) + 8 * groups * n_pairs + 512 bytes) is
 * zero-filled once.  With n_pairs > 1: cloud_rows_h[level][2 * n_pairs] = host row counts per cloud, and
 * sub_cloud_max[level][2 * n_pairs] (device int32, geob200_cloud_max_count of the subsampling tables) lets the strided blocks'
 * maxpool see every pair's table at the width the pair's own collate would have cut it to; with one pair both may be NULL. */
int geob200_backbone_forward_batched(const geob200_backbone_t* net, const float* feats, const float* const* points,
                                     const int64_t* level_rows, const int64_t* const* neighbors, const int64_t* neighbor_width,
                                     const int64_t* const* subsampling, const int64_t* subsampling_width,
                                     const int64_t* const* upsampling, const int64_t* upsampling_width, float* const* out_feats,
                                     void* gn_workspace, size_t gn_workspace_bytes, void* workspace, size_t workspace_bytes, void* stream,
                                     int64_t n_pairs, const int64_t* const* cloud_rows_h, const int32_t* const* sub_cloud_max);

/* one transformer layer ('self' with the structure embedding, or 'cross'); w_qkv = [Wq;Wk;Wv] (3C,C), w_kv = [Wk;Wv], wp_t = Wp^T */
typedef struct {
    int32_t is_self, reserved;
    const float* w_qkv; const float* b_qkv; const float* w_q; const float* b_q; const float* w_kv; const float* b_kv;
    const float* wp_t; const float* bp;
    geob200_linear_t att_linear; geob200_norm_t att_norm;
    geob200_linear_t expand; geob200_linear_t squeeze; geob200_norm_t out_norm;
    const float* w_qkv_img; const float* w_q_img; const float* w_kv_img;
} geob200_tlayer_t;
/* RPEConditionalTransformer.forward (after in_proj, sequential cross updates) over n_pairs pairs: x rows in stack order
 * [ref_1..ref_B, src_1..src_B] (cloud_rows_h[2B], host; one pair: [ref; src]); embeddings_h[c] = device pointer of the structure
 * embedding (rows_c, rows_c, C) of cloud c.  Linears / LayerNorms run once over all rows; attention is one batched launch pair per
 * phase (geob200_attention_batched).  A pair gets the same bits alone and in any batch. */
size_t geob200_transformer_batched_workspace_bytes(int64_t n_pairs, const int64_t* cloud_rows_h, int64_t channels, int64_t heads,
                                                   int64_t num_layers);
int geob200_transformer_forward_batched(const geob200_tlayer_t* layers, int64_t num_layers, int64_t channels, int64_t heads,
                                        const float* x, int64_t n_pairs, const int64_t* cloud_rows_h, const float* const* embeddings_h,
                                        float* out, void* workspace, size_t workspace_bytes, void* stream);

/* Ground-truth superpoint targets of the training-mode forward (SuperPointTargetGenerator, modules/geotransformer/
 * superpoint_target.py), one CTA per pair.  Inputs: the gt rows of geob200_node_correspondences_batched (indices (R, 2), overlaps
 * (R,), the first gt_count[p] (device int32) of pair p's n_ref * n_src rows valid, laid out by cloud_nodes (2B counts)).  The
 * candidates j = 0 .. n-1 are the rows with overlap > overlap_threshold, in gt order.  n <= num_targets: all of them; otherwise the
 * num_targets smallest keys (philox(seed; j, iteration, pair_base + p) << 32) | j (Philox4x32-10, key = seed, counter = (j,
 * iteration lo, iteration hi, pair_base + p), word 0), in ascending j.  Outputs in the layout of
 * geob200_superpoint_matching_batched: corr_indices (2B, num_targets) int64 (row p ref / row B + p src indices of pair p, -1 past
 * the count), corr_scores (B, num_targets) = the selected overlaps (0 past the count), num_out (B,) device int32. */
size_t geob200_superpoint_targets_batched_workspace_bytes(int64_t n_gt_rows);
int geob200_superpoint_targets_batched(const int64_t* gt_indices, const float* gt_overlaps, const int32_t* gt_count, int64_t n_pairs,
                                       const int64_t* cloud_nodes, float overlap_threshold, int64_t num_targets, uint64_t seed,
                                       uint64_t iteration, int64_t pair_base, int64_t* corr_indices, float* corr_scores, int32_t* num_out,
                                       void* workspace, size_t workspace_bytes, void* stream);

/* Gradient guard of the training step: found_inf[0] (device fp32) = 1 when any element of the n_tensors fp32 tensors listed in the
 * DEVICE tables ptrs / numels is NaN or +-Inf, else 0.  max_numel (host) = the largest numel, sizes the grid.  One launch. */
int geob200_nonfinite_check(const float* const* ptrs, const int64_t* numels, int64_t n_tensors, int64_t max_numel, float* found_inf,
                            void* stream);

/* Loss weights of a batched training step, one launch: pair p is valid when row p of loss_rows (n_pairs, >= 3 at row stride
 * ld_rows: [loss, c_loss, f_loss]) is finite.  weights[p] = valid_p / n_valid (the upstream gradient of column 0), mean_row[0..2] =
 * sum over the valid pairs, in pair order, of weights[p] * row p (fp32, every product rounded), n_valid (may be NULL) = the count as
 * a float.  With no valid pair: weights 0, mean_row NaN and found_inf[0] = 1; otherwise found_inf is not written. */
int geob200_batch_loss_weights(const float* loss_rows, int64_t ld_rows, int64_t n_pairs, float* weights, float* mean_row, float* n_valid,
                               float* found_inf, void* stream);

/* ---- training-data augmentation (datasets/registration/{threedmatch,kitti,modelnet}/dataset.py) -------------------------------
 *
 * Random streams.  Every draw is Philox4x32-10 (the generator of the target sampler and RANSAC) with
 *   key     = (seed lo, seed hi ^ tag),  tag = GEOB200_AUGMENT_TAG_BASE | stream << 4 | cloud  (cloud 0 = ref, 1 = src),
 *             stream 1 pair draws (cloud 0 only), 2 point-limit keys, 3 noise, 4 sample keys, 5 jitter;
 *   counter = (index, iteration lo, iteration hi, pair_base + p).
 * The target sampler and RANSAC use tag 0, so no augmentation stream shares their key.
 * Pair draws: call i (index i) gives u_{2i} = ((w0 >> 5) 2^26 + (w1 >> 6)) 2^-53 and u_{2i+1} from (w2, w3) likewise.
 *   3DMatch: u0..u2 Euler angles 2 pi u / rotation_factor, u3 the coin (u3 > 0.5 rotates ref, else src);
 *   KITTI:   additionally u4 scale min + (max - min) u4, u5..u7 ref shift -s + 2s u, u8..u10 src shift;
 *   ModelNet: u0..u2 Euler angles pi rotation_magnitude / 180 u, u3..u5 translation -m + 2m u, (u6, u7) ref plane and (u8, u9) src
 *   plane: phi = 2 pi u, theta = pi u, normal (sin theta cos phi, sin theta sin phi, cos theta).
 *   R = scipy's Rotation.from_euler('zyx', (a, b, c)) = Rx(c) Ry(b) Rz(a).
 * Per-point words: index = the point's row in its input cloud (raw shape for ModelNet); uniforms w 2^-32.
 *   point limit: key (w0 << 32) | row;  noise: u = w0, w1, w2;  sample: key (w0 << 32) | row;  jitter: Box-Muller
 *   z0, z1 = sqrt(-2 ln(1 - u0)) (cos, sin)(2 pi u1), z2 = sqrt(-2 ln(1 - u2)) cos(2 pi u3).
 * record (n_pairs, 20) fp64: [u0 .. u10 | R row-major], unused slots 0.  transforms / out_transforms: (n_pairs, 4, 4) fp32. */
#define GEOB200_AUGMENT_3DMATCH 0
#define GEOB200_AUGMENT_KITTI 1
#define GEOB200_AUGMENT_TAG_BASE 0xA6000000u

/* 3DMatch / KITTI training-pair augmentation, two launches for any n_pairs (1 .. 32).  points: raw clouds stacked
 * [ref_0..ref_{B-1}, src_0..src_{B-1}] with host lengths_h[2B] (each >= 1); transforms (B, 4, 4) ground truth (ref = T src).
 * Cloud c keeps min(n_c, point_limit) rows: all in order when n_c <= point_limit, else the point_limit smallest point-limit keys
 * in ascending row (a uniform subset).  origin (int32, same rows as out_points): the row of each output point in its input cloud.
 * Per point, in fp64 with every operation rounded (no contraction) and one rounding to fp32:
 *   3DMATCH: rotate (rows of R, ((r0 x + r1 y) + r2 z)) if this cloud is the rotated one, then + (u - 0.5) noise;
 *   KITTI:   + (u - 0.5) noise, rotate if rotated, * scale, + this cloud's shift.
 * out_transforms: rotated ref -> (R R_gt, R t_gt); rotated src -> (R_gt R^T, t_gt); KITTI then t = (-(R' src_shift) + scale t)
 * + ref_shift; computed in fp64 and rounded once.  workspace: geob200_augment_pairs_batched_workspace_bytes(sum of lengths). */
size_t geob200_augment_pairs_batched_workspace_bytes(int64_t n_rows);
int geob200_augment_pairs_batched(const float* points, const int64_t* lengths_h, int64_t n_pairs, const float* transforms, int mode,
                                  int64_t point_limit, double noise, double rotation_factor, double min_scale, double max_scale,
                                  double shift, uint64_t seed, uint64_t iteration, int64_t pair_base, float* out_points, int32_t* origin,
                                  float* out_transforms, double* record, void* workspace, size_t workspace_bytes, void* stream);

/* ModelNet pair synthesis (twice_sample, plane crop), one launch with one CTA per cloud for any n_pairs (1 .. 32).  shapes: B raw
 * shapes stacked with host lengths_h[B], each 1 .. 8192 points with round(keep_ratio N) = floor(N keep_ratio + 0.5) >= num_points
 * (1 .. 4096).  Per cloud, in fp64: normalise (subtract the mean, divide by the largest norm); src only: apply the inverse of the
 * drawn transform; crop to the round(keep_ratio N) largest plane distances dot(p, n), ties to the lowest row; keep the num_points
 * smallest sample keys of the cropped points and write them in key order (a uniformly random ordered subset); add the jitter
 * clip(0.01 z, +-noise_magnitude); round to fp32.  out_points (2B num_points, 3) stacked [ref..., src...]; origin: the raw shape
 * row; out_transforms: the drawn transform (ref = T src).  workspace: geob200_modelnet_pairs_batched_workspace_bytes(sum of
 * lengths). */
size_t geob200_modelnet_pairs_batched_workspace_bytes(int64_t n_rows);
int geob200_modelnet_pairs_batched(const float* shapes, const int64_t* lengths_h, int64_t n_pairs, int64_t num_points, double keep_ratio,
                                   double rotation_magnitude, double translation_magnitude, double noise_magnitude, uint64_t seed,
                                   uint64_t iteration, int64_t pair_base, float* out_points, int32_t* origin, float* out_transforms,
                                   double* record, void* workspace, size_t workspace_bytes, void* stream);

/* ---- ModelNet validation and test pairs (datasets/registration/modelnet/dataset.py, deterministic=True) ------------------------
 *
 * Pair p is the reference's val / test item of dataset index indices_h[p] (0 .. 2^32-1; the position in the class-filtered list),
 * built from raw shape p (host lengths_h[p], 1 .. 8192 points, stacked in `shapes`) with twice_sample, a plane crop and no
 * twice_transform.  One stream serves both clouds: numpy's legacy generator (MT19937) seeded as np.random.seed(index), consumed in
 * the reference's order:
 *   1. rand(3) -> Euler angles ((u pi) rotation_magnitude) / 180, R = scipy's from_euler('zyx', .) in its quaternion arithmetic;
 *      uniform(-m, m) x 3 -> t (low + (high - low) u);
 *   2. ref plane, then src plane: phi = uniform(0, 2 pi), theta = uniform(0, pi), n = (sin theta cos phi, sin theta sin phi, cos theta);
 *   3. permutation(K) for ref, then src, K = floor(N keep_ratio + 0.5): the first num_points, or (K < num_points) the permutation
 *      repeated and its head; permutation = arange, then for i = K-1 .. 1 swap i with the masked-rejection interval(i);
 *   4. 3 num_points Gaussians for ref, then src (the polar method with its one-value cache, which carries from ref to src when
 *      3 num_points is odd): jitter clip(0 + 0.01 g, +-noise_magnitude);
 *   5. permutation(num_points) for ref, then src: the final order.
 * Arithmetic: normalise in fp32 (column sums in row order, / N; subtract; divide by the largest sqrt((x^2 + y^2) + z^2)); src =
 * ((R[0,i] x + R[1,i] y) + R[2,i] z) + t_inv[i] with t_inv = -(R^T t) alike, in fp64; distances (x nx + y ny) + z nz in fp64; crop
 * order descending distance, ties to the lowest row; point + jitter in fp64, rounded to fp32 once.  No contraction anywhere.
 * out_points (2B num_points, 3) stacked [ref_0..ref_{B-1}, src_0..src_{B-1}]; origin (int32, same rows): the raw shape row of each
 * output point; out_transforms (B, 4, 4) fp32 [R | t] (ref = T src).  Any n_pairs (1 .. 262143): launches of up to 1024 pairs, one
 * CTA per pair.  workspace: geob200_modelnet_benchmark_pairs_batched_workspace_bytes(n_pairs, num_points). */
size_t geob200_modelnet_benchmark_pairs_batched_workspace_bytes(int64_t n_pairs, int64_t num_points);
int geob200_modelnet_benchmark_pairs_batched(const float* shapes, const int64_t* lengths_h, const int64_t* indices_h, int64_t n_pairs,
                                             int64_t num_points, double keep_ratio, double rotation_magnitude, double translation_magnitude,
                                             double noise_magnitude, float* out_points, int32_t* origin, float* out_transforms,
                                             void* workspace, size_t workspace_bytes, void* stream);

/* ---- Rotated 3DMatch / 3DLoMatch benchmark pairs (datasets/registration/threedmatch/dataset.py, rotated=True) -------------------
 *
 * Pair p is the reference's rotated test item of dataset index indices_h[p] (0 .. 2^32-1).  Its clouds are rows of `points` (fp32,
 * or fp64 with points_fp64 = 1: the type the dataset's files hold, since numpy rotates them in fp64 either way; stacked [ref_0..ref_{B-1}, src_0..src_{B-1}] with host lengths_h[2B], each 1 .. 2^31-1 points, 2^31-1 rows in all) and its
 * transform is transforms[p] (fp64 (4, 4), [R | t], ref = T src, from the metadata's fp64 rotation and translation).  One stream
 * per pair: numpy's legacy generator seeded as np.random.seed(index), drawing random_sample_rotation_v2 for ref, then for src:
 *   axis = rand(3) - 0.5; axis = axis / sqrt(fma(a2, a2, fma(a1, a1, a0 a0))) + 1e-8 (added after the division); theta = pi rand();
 *   R = scipy's from_euler('zyx', axis theta) in its quaternion arithmetic.
 * Outputs, in the layout of the inputs: out_points = fp32(p R^T), fma(z, R[i,2], fma(y, R[i,1], x R[i,0])) in fp64, numpy's own
 * order (ref with R_ref, src with R_src); out_transforms (B, 4, 4) fp32 = fp32([R_ref R R_src^T | R_ref t]), the products in numpy's
 * (OpenBLAS's) fp64 order: (A B)[i, j] = fma(a_i2, b_2j, fma(a_i1, b_1j, a_i0 b_0j)), (A v)[i] = fma(a_i2, v2, fma(a_i0, v0,
 * a_i1 v1)); rotations (B, 2, 9) fp64: R_ref, R_src row-major.  The half-angles' sin and cos are correctly rounded (the host
 * libm's differ from that only in rare near-tie cases, DESIGN §8a).  Any n_pairs (1 .. 2^30): launches of up to 64 pairs, each a
 * one-warp-per-pair draw kernel and one grid over the rows.  No workspace. */
int geob200_rotated_pairs_batched(const void* points, int points_fp64, const int64_t* lengths_h, const int64_t* indices_h, int64_t n_pairs,
                                  const double* transforms, float* out_points, float* out_transforms, double* rotations, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GEOB200_H */
