// TEST INFRASTRUCTURE ONLY.  A plain C++ restatement of Open3D's PointCloud::VoxelDownSample, the contract that
// geob200_voxel_down_sample (geotransformer_b200/csrc/voxel.cu) implements on the device:
//
//   p_i in double (float32 inputs are widened exactly), voxel size v;
//   lo = min_i p_i - 0.5 v, hi = max_i p_i + 0.5 v componentwise (0.5 v is exact);
//   error if v <= 0, if v * INT_MAX < max(hi - lo) (Open3D's "voxel_size is too small"), on a non-finite coordinate (Open3D does
//   not check), or when an axis spans 2^21 voxels or more (the device packs 21 bits per axis);
//   an empty cloud gives an empty result;
//   voxel of point i: k_a = int(floor((p_i[a] - lo[a]) / v)), IEEE double subtraction and division, no FMA;
//   points are grouped by the exact triple (k_x, k_y, k_z);
//   the value of a voxel is the double sum of its points added in input order from 0, divided by double(count); normals, if
//   given, the same, not renormalised (AccumulatedPoint::GetAveragePoint / GetAverageNormal);
//   the output order is the iteration order of a default-constructed std::unordered_map<triple, ...> filled by operator[] in
//   input order and hashed by Open3D's utility::hash_eigen: seed = 0, then for x, y, z in turn
//   seed ^= size_t(k) + 0x9e3779b9 + (seed << 6) + (seed >> 2), all in size_t, std::hash<int> being the identity cast.
//
// The map below is a real libstdc++ std::unordered_map, so on a libstdc++ system it is the ground truth for the order.  Parity
// with Open3D itself is not verified here: Open3D is not a dependency of this project.
// Built without -ffast-math and without -march=native (x86-64 baseline has no FMA).
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <limits>
#include <unordered_map>
#include <vector>

namespace {

struct Triple {
    int k[3];
    bool operator==(const Triple& o) const { return k[0] == o.k[0] && k[1] == o.k[1] && k[2] == o.k[2]; }
};

struct HashEigen {
    std::size_t operator()(const Triple& t) const {
        std::size_t seed = 0;
        for (int a = 0; a < 3; ++a) seed ^= std::hash<int>()(t.k[a]) + 0x9e3779b9 + (seed << 6) + (seed >> 2);
        return seed;
    }
};

struct Accumulated {
    double p[3] = {0.0, 0.0, 0.0};
    double n[3] = {0.0, 0.0, 0.0};
    long long count = 0;
};

}  // namespace

extern "C" {

enum { VOX_OK = 0, VOX_NONFINITE = 1, VOX_TOO_SMALL = 2, VOX_AXIS_LIMIT = 3, VOX_BAD_SIZE = 4 };

uint64_t voxel_oracle_hash(int x, int y, int z) {
    Triple t{{x, y, z}};
    return (uint64_t)HashEigen()(t);
}

// One cloud.  out_points / out_normals must hold n rows; *out_n receives the voxel count.  Returns 0 or an error code.
int voxel_oracle(const double* points, const double* normals, int64_t n, double voxel, double* out_points, double* out_normals,
                 int64_t* out_n) {
    *out_n = 0;
    if (!(voxel > 0.0)) return VOX_BAD_SIZE;
    if (n == 0) return VOX_OK;
    double mn[3], mx[3];
    for (int a = 0; a < 3; ++a) { mn[a] = points[a]; mx[a] = points[a]; }
    for (int64_t i = 0; i < n; ++i)
        for (int a = 0; a < 3; ++a) {
            const double x = points[3 * i + a];
            if (!std::isfinite(x)) return VOX_NONFINITE;
            if (x < mn[a]) mn[a] = x;
            if (x > mx[a]) mx[a] = x;
        }
    double lo[3], extent = 0.0;
    for (int a = 0; a < 3; ++a) {
        lo[a] = mn[a] - voxel * 0.5;
        const double hi = mx[a] + voxel * 0.5;
        if (hi - lo[a] > extent) extent = hi - lo[a];
    }
    if (voxel * std::numeric_limits<int>::max() < extent) return VOX_TOO_SMALL;
    for (int a = 0; a < 3; ++a)
        if (std::floor((mx[a] - lo[a]) / voxel) >= (double)(1 << 21)) return VOX_AXIS_LIMIT;

    std::unordered_map<Triple, Accumulated, HashEigen> map;
    for (int64_t i = 0; i < n; ++i) {
        Triple t;
        for (int a = 0; a < 3; ++a) t.k[a] = int(std::floor((points[3 * i + a] - lo[a]) / voxel));
        Accumulated& acc = map[t];
        for (int a = 0; a < 3; ++a) acc.p[a] += points[3 * i + a];
        if (normals != nullptr)
            for (int a = 0; a < 3; ++a) acc.n[a] += normals[3 * i + a];
        acc.count += 1;
    }
    int64_t q = 0;
    for (const auto& kv : map) {
        const double c = double(kv.second.count);
        for (int a = 0; a < 3; ++a) out_points[3 * q + a] = kv.second.p[a] / c;
        if (normals != nullptr)
            for (int a = 0; a < 3; ++a) out_normals[3 * q + a] = kv.second.n[a] / c;
        ++q;
    }
    *out_n = q;
    return VOX_OK;
}

// The bucket counts a default-constructed map of this kind takes while n_keys distinct triples are inserted by operator[]:
// writes each new bucket_count() (the first being the one after the first insertion) to out, returns how many were written.
int64_t voxel_oracle_bucket_growth(int64_t n_keys, uint64_t* out, int64_t cap) {
    std::unordered_map<Triple, Accumulated, HashEigen> map;
    std::size_t last = map.bucket_count();
    int64_t w = 0;
    for (int64_t i = 0; i < n_keys; ++i) {
        Triple t{{(int)(i % 1000), (int)(i / 1000), 0}};
        map[t].count += 1;
        if (map.bucket_count() != last) {
            last = map.bucket_count();
            if (w < cap) out[w] = (uint64_t)last;
            ++w;
        }
    }
    return w;
}

}  // extern "C"
