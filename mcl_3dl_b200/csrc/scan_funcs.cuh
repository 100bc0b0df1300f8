// scan_funcs.cuh — per-point pieces of scan preprocessing (mcl3dl_scan_prepare, scan_kernels.cuh): the VoxelGrid
// lattice and voxel key, the finiteness test, the centroid and label vote of one voxel, the models' clip and the uniform
// sampler's index.  They are also compiled for the host by tests/hostsim (scan_hostsim.cpp) and checked there against a
// numpy restatement of the same operations (tests/test_gpu_scan_exact.py).
//
// Float rules as in device_math.cuh: explicit round-to-nearest operations in the reference's operand order.
#pragma once
#ifndef MCL3DL_HOSTSIM
#include <cuda_runtime.h>
#endif
#include <math.h>
#include <stdint.h>

#include "../../include/mcl3dl_b200.h"
#include "pf_funcs.cuh"

namespace mcl3dl
{
// ---- VoxelGrid (pcl/filters/impl/voxel_grid.hpp: applyFilter)
struct VoxelGridDev
{
  float inv_leaf[3];  // float(1 / leaf), Eigen::Array4f inverse_leaf_size_
  int min_b[3];       // floor(min * inv_leaf)
  uint32_t div_b[3];  // floor(max * inv_leaf) - min_b + 1
  uint32_t cells;     // div_b[0] * div_b[1] * div_b[2]: real voxel keys are below it, non-finite points get key == cells
};

// pcl::isXYZFinite: no NaN and no infinity among x, y, z (exponent bits, so that no compiler flag can fold it away)
__device__ __forceinline__ bool scan_finite(float v) { return (__float_as_uint(v) & 0x7f800000u) != 0x7f800000u; }
__device__ __forceinline__ bool point_finite(const mcl3dl_point& p) { return scan_finite(p.x) && scan_finite(p.y) && scan_finite(p.z); }

// linear voxel index, x fastest; a cloud that is not dense has its non-finite points skipped, so they get a key past
// every real voxel (they sort last and form no voxel)
__device__ __forceinline__ uint32_t voxel_key(const VoxelGridDev& g, const mcl3dl_point& p)
{
  if (!point_finite(p))
    return g.cells;
  const int i = __float2int_rd(fmul(p.x, g.inv_leaf[0])) - g.min_b[0];
  const int j = __float2int_rd(fmul(p.y, g.inv_leaf[1])) - g.min_b[1];
  const int k = __float2int_rd(fmul(p.z, g.inv_leaf[2])) - g.min_b[2];
  return static_cast<uint32_t>(i) + static_cast<uint32_t>(j) * g.div_b[0] + static_cast<uint32_t>(k) * (g.div_b[0] * g.div_b[1]);
}

// the second sort key of the label vote: voxel, then label
__device__ __forceinline__ uint64_t voxel_key_label(uint32_t key, uint32_t label) { return (static_cast<uint64_t>(key) << 32) | label; }

// One output point: the voxel's `cnt` points are pts[order[0..cnt)] in input order (the key sort is stable) and
// key_label[0..cnt) holds the same points' voxel_key_label sorted ascending.  Centroid = float sums in input order over
// float(cnt) (PCL orders a voxel's points with an unstable std::sort, so its sums are defined only up to summation
// order).  Label = the majority label, lowest on ties (CentroidPoint / AccumulatorLabel: a std::map walked in key order,
// first maximum): the labels come ascending, so the first longest run wins.  Linear in cnt.
__device__ __forceinline__ mcl3dl_point scan_voxel_point(const mcl3dl_point* __restrict__ pts, const uint32_t* __restrict__ order,
                                                        const uint64_t* __restrict__ key_label, uint32_t cnt)
{
  float sx = 0.0f, sy = 0.0f, sz = 0.0f;
  for (uint32_t j = 0; j < cnt; ++j)
  {
    const mcl3dl_point p = pts[order[j]];
    sx = fadd(sx, p.x);
    sy = fadd(sy, p.y);
    sz = fadd(sz, p.z);
  }
  uint32_t best_label = 0, best_cnt = 0, run = 0, prev = 0;
  for (uint32_t j = 0; j < cnt; ++j)
  {
    const uint32_t l = static_cast<uint32_t>(key_label[j]);
    run = (j > 0 && l == prev) ? run + 1 : 1;
    prev = l;
    if (run > best_cnt)
    {
      best_cnt = run;
      best_label = l;
    }
  }
  mcl3dl_point o;
  const float fc = static_cast<float>(cnt);
  o.x = fdiv(sx, fc);
  o.y = fdiv(sy, fc);
  o.z = fdiv(sz, fc);
  o.label = best_label;
  return o;
}

// Host side, once per scan: the lattice of the finite points' bounding box [mn, mx] and whether to downsample at all.
// PCL's rule: dx = int64((max - min) * inv_leaf) + 1 per axis, and more than INT32_MAX voxels leave the cloud unfiltered.
// Where that rule passes but PCL's own int arithmetic would overflow (min_b / max_b beyond int, or div_b's product
// beyond 32 bits: possible only for extreme outliers, and undefined in PCL), the cloud is left unfiltered as well.
// end_bit: radix bits of the keys, the non-finite key (== cells) included.  Plain host float arithmetic, like
// pf_set_odoms.
inline bool scan_voxel_lattice(const float leaf[3], const float mn[3], const float mx[3], VoxelGridDev& g, int& end_bit)
{
  uint64_t voxels = 1, cells = 1;
  for (int k = 0; k < 3; ++k)
  {
    g.inv_leaf[k] = 1.0f / leaf[k];
    const float ext = (mx[k] - mn[k]) * g.inv_leaf[k];
    if (!(ext < 2147483648.0f))  // this axis alone is past the limit (or the extent is not a number)
      return false;
    voxels *= static_cast<uint64_t>(static_cast<int64_t>(ext) + 1);
    if (voxels > 2147483647u)
      return false;
    const float lo = floorf(mn[k] * g.inv_leaf[k]), hi = floorf(mx[k] * g.inv_leaf[k]);
    if (!(lo >= -2147483648.0f && hi < 2147483648.0f))
      return false;
    g.min_b[k] = static_cast<int>(lo);
    const int64_t div = static_cast<int64_t>(hi) - g.min_b[k] + 1;
    cells *= static_cast<uint64_t>(div);
    if (cells > 0xffffffffu)
      return false;
    g.div_b[k] = static_cast<uint32_t>(div);
  }
  g.cells = static_cast<uint32_t>(cells);
  end_bit = 1;
  while (end_bit < 32 && (uint64_t(1) << end_bit) <= cells) ++end_bit;
  return true;
}

// ---- the models' filter() clip (src/lidar_measurement_model_likelihood.cpp:79-103 == _beam.cpp:98-122)
struct ClipDev
{
  float near_sq, far_sq, z_min, z_max;  // clip_near_sq_ = clip_near * clip_near (float), likelihood.cpp:59-60
};

inline ClipDev scan_clip_window(float near, float far, float z_min, float z_max)
{
  return ClipDev{near * near, far * far, z_min, z_max};
}

// local_points_filter of filter(), likelihood.cpp:83-93 / beam.cpp:102-112: true = REMOVE
__device__ __forceinline__ bool clip_removes(const ClipDev& c, const mcl3dl_point& p)
{
  const float r2 = fadd(fmul(p.x, p.x), fmul(p.y, p.y));
  if (r2 > c.far_sq)
    return true;
  if (r2 < c.near_sq)
    return true;
  if (p.z < c.z_min || c.z_max < p.z)
    return true;
  return false;
}

// ---- PointCloudUniformSampler::sample: draw t of stream (0 likelihood, 1 beam) takes clipped point floor(u * n),
// u = the first Philox word / 2^32, counter (t, stream, 0x5ca11ab1, 0), key = the 64-bit seed's low and high words
__device__ __forceinline__ uint32_t scan_sample_index(uint64_t seed, uint32_t stream, uint32_t t, uint32_t n)
{
  uint32_t c[4] = {t, stream, 0x5ca11ab1u, 0u};
  philox4x32_10(c, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  return static_cast<uint32_t>((static_cast<uint64_t>(c[0]) * n) >> 32);
}

}  // namespace mcl3dl
