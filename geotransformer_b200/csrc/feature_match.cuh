// Host-side launcher of the exact descriptor nearest neighbour (feature_match.cu), shared with the feature-matching RANSAC
// (ransac.cu).
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace geob200 {

// workspace of one feature_nn_launch call (both directions share the candidate buffers: they run one after the other)
size_t feature_nn_workspace(int64_t n_pairs, int64_t cap_q, int64_t cap_s);

// Arguments already checked.  Writes q_index / q_dist for every query row (and s_index / s_dist for every support row when
// s_index != nullptr); adds the launches it made to *launches.  Returns 0, or -1 with the error message set.
int feature_nn_launch(const float* query, const float* support, int n_pairs, int cap_q, int cap_s, int channels, const int32_t* n_query,
                      const int32_t* n_support, int64_t* q_index, double* q_dist, int64_t* s_index, double* s_dist, void* workspace,
                      size_t workspace_bytes, cudaStream_t stream, int* launches);

}  // namespace geob200
