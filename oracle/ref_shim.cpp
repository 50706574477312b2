// TEST INFRASTRUCTURE ONLY -- never linked into or called from the product path.
//
// C-ABI shim around the UNMODIFIED reference CPU ops so that the real reference code can be
// (a) used to validate the restatement in oracle/collate_oracle.c and (b) timed as the
// "reference" CPU baseline on machines where only the built .so is present.
//
// The reference sources are compiled where they lie (see oracle/Makefile):
//   geotransformer/extensions/extra/cloud/cloud.cpp
//   geotransformer/extensions/cpu/grid_subsampling/grid_subsampling_cpu.cpp   (core :3-75)
//   geotransformer/extensions/cpu/radius_neighbors/radius_neighbors_cpu.cpp   (core :3-91)
// This file only re-does what the ATen wrappers do around those cores
// (grid_subsampling.cpp:5-62, radius_neighbors.cpp:5-68): copy in, call, copy out.
#include <cstdint>
#include <cstring>
#include <vector>

#include "cpu/grid_subsampling/grid_subsampling_cpu.h"
#include "cpu/radius_neighbors/radius_neighbors_cpu.h"

extern "C" {

// Returns total number of subsampled points; writes at most `cap` points into s_points.
int64_t ref_grid_subsampling(const float* points, int64_t n_points, const int64_t* lengths, int64_t batch,
                             float voxel_size, float* s_points, int64_t cap, int64_t* s_lengths) {
  std::vector<PointXYZ> vp(reinterpret_cast<const PointXYZ*>(points),
                           reinterpret_cast<const PointXYZ*>(points) + n_points);
  std::vector<long> vl(lengths, lengths + batch);
  std::vector<PointXYZ> sp;
  std::vector<long> sl;
  grid_subsampling_cpu(vp, sp, vl, sl, voxel_size);
  int64_t total = static_cast<int64_t>(sp.size());
  int64_t ncopy = total < cap ? total : cap;
  std::memcpy(s_points, sp.data(), sizeof(float) * 3 * ncopy);
  for (int64_t b = 0; b < batch; ++b) s_lengths[b] = sl[b];
  return total;
}

// Two-phase: call with out == nullptr to get max_count (the row width), then with a buffer.
// The search is re-run on the second call; callers that time it should time one call.
int64_t ref_radius_neighbors(const float* q_points, int64_t nq, const float* s_points, int64_t ns,
                             const int64_t* q_lengths, const int64_t* s_lengths, int64_t batch, float radius,
                             int64_t* out, int64_t out_cols) {
  std::vector<PointXYZ> vq(reinterpret_cast<const PointXYZ*>(q_points),
                           reinterpret_cast<const PointXYZ*>(q_points) + nq);
  std::vector<PointXYZ> vs(reinterpret_cast<const PointXYZ*>(s_points),
                           reinterpret_cast<const PointXYZ*>(s_points) + ns);
  std::vector<long> ql(q_lengths, q_lengths + batch);
  std::vector<long> sl(s_lengths, s_lengths + batch);
  std::vector<long> idx;
  radius_neighbors_cpu(vq, vs, ql, sl, idx, radius);
  int64_t max_count = nq > 0 ? static_cast<int64_t>(idx.size()) / nq : 0;
  if (out != nullptr && out_cols == max_count) {
    std::memcpy(out, idx.data(), sizeof(int64_t) * idx.size());
  }
  return max_count;
}

// Single-search form (what the reference does: search, THEN allocate the tensor and copy, radius_neighbors.cpp:47-66):
// ref_radius_neighbors_search runs the reference search once and keeps the index list; ref_radius_neighbors_fetch copies it
// out.  Used by oracle/ref_ext.py so that a timed reference search is ONE search.
static thread_local std::vector<long> g_last_idx;

int64_t ref_radius_neighbors_search(const float* q_points, int64_t nq, const float* s_points, int64_t ns,
                                    const int64_t* q_lengths, const int64_t* s_lengths, int64_t batch, float radius) {
  std::vector<PointXYZ> vq(reinterpret_cast<const PointXYZ*>(q_points),
                           reinterpret_cast<const PointXYZ*>(q_points) + nq);
  std::vector<PointXYZ> vs(reinterpret_cast<const PointXYZ*>(s_points),
                           reinterpret_cast<const PointXYZ*>(s_points) + ns);
  std::vector<long> ql(q_lengths, q_lengths + batch);
  std::vector<long> sl(s_lengths, s_lengths + batch);
  g_last_idx.clear();
  radius_neighbors_cpu(vq, vs, ql, sl, g_last_idx, radius);
  return nq > 0 ? static_cast<int64_t>(g_last_idx.size()) / nq : 0;
}

int64_t ref_radius_neighbors_fetch(int64_t* out, int64_t n_values) {
  if (static_cast<int64_t>(g_last_idx.size()) != n_values) return -1;
  std::memcpy(out, g_last_idx.data(), sizeof(int64_t) * g_last_idx.size());
  g_last_idx.clear();
  g_last_idx.shrink_to_fit();
  return 0;
}

}  // extern "C"
