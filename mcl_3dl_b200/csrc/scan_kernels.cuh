// scan_kernels.cuh — scan preprocessing on the device (scope row f4, scan half): what the node does to the accumulated
// raw cloud before every measurement (src/mcl_3dl.cpp:363-383):
//   1. pcl::VoxelGrid downsample (leaf = params.downsample_x/y/z, :363-367).  PCL is a third-party dependency that is
//      absent from the reference tree (PCL >= 1.8, version unpinned); restated from its published algorithm
//      (pcl/filters/impl/voxel_grid.hpp: applyFilter): non-finite points are skipped (the cloud is treated as not
//      dense), the lattice comes from the finite points' bounding box, more than INT32_MAX voxels by PCL's own count
//      leave the cloud unfiltered, leaf index = floor(coord * float(1 / leaf)) - floor(min * ...), linear index x
//      fastest, output in ascending voxel index, one centroid per occupied voxel (float sums in input order; the label
//      is the majority label of the voxel, lowest on ties, as PCL's CentroidPoint / AccumulatorLabel does).  PCL
//      subtracts min_b in float, which equals the integer subtraction here while |coord / leaf| < 2^24.  "Parity
//      unpinned" for this piece (no reference test pins VoxelGrid output).  Per-point pieces: scan_funcs.cuh.
//   2. the models' filter(): clip by planar range^2 and z window, order kept
//      (src/lidar_measurement_model_likelihood.cpp:79-103 == _beam.cpp:98-122) — exact, checked against the oracle;
//   3. PointCloudUniformSampler::sample (point_cloud_random_samplers/point_cloud_uniform_sampler.h:56-74): `num` draws with
//      replacement, uniform over the clipped points.  The reference seeds std::default_random_engine from
//      std::random_device, i.e. its draws are not reproducible by construction; the device draws from Philox-4x32-10
//      keyed by (seed, stream, draw index).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/mcl3dl_b200.h"
#include "scan_funcs.cuh"

namespace mcl3dl
{
// bounding box of the finite points (getMinMax3D of a cloud that is not dense): bbox[0..2] min, [3..5] max, in the
// ordered-uint encoding; with no finite point the minimum stays +inf
__global__ void scan_bbox_kernel(const mcl3dl_point* __restrict__ pts, uint32_t n, uint32_t* __restrict__ bbox)
{
  float mn[3], mx[3];
#pragma unroll
  for (int k = 0; k < 3; ++k)
  {
    mn[k] = __int_as_float(0x7f800000);
    mx[k] = __int_as_float(0xff800000);
  }
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
  {
    const mcl3dl_point p = pts[i];
    if (!point_finite(p))
      continue;
    const float v[3] = {p.x, p.y, p.z};
#pragma unroll
    for (int k = 0; k < 3; ++k)
    {
      mn[k] = fminf(mn[k], v[k]);
      mx[k] = fmaxf(mx[k], v[k]);
    }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k)
  {
    for (int o = 16; o > 0; o >>= 1)
    {
      mn[k] = fminf(mn[k], __shfl_xor_sync(0xffffffffu, mn[k], o));
      mx[k] = fmaxf(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o));
    }
  }
  if ((threadIdx.x & 31) == 0)
  {
#pragma unroll
    for (int k = 0; k < 3; ++k)
    {
      atomicMin(bbox + k, f2ord(mn[k]));
      atomicMax(bbox + 3 + k, f2ord(mx[k]));
    }
  }
}

// keys / values of the voxel sort (input index) and the (voxel, label) keys of the vote
__global__ void scan_key_kernel(const mcl3dl_point* __restrict__ pts, uint32_t n, VoxelGridDev g, uint32_t* __restrict__ keys,
                                uint32_t* __restrict__ vals, uint64_t* __restrict__ key_label)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const mcl3dl_point p = pts[i];
  const uint32_t key = voxel_key(g, p);
  keys[i] = key;
  vals[i] = i;
  key_label[i] = voxel_key_label(key, p.label);
}

// heads of the runs of equal keys (sorted): flag[i] = 1 where a voxel starts
__global__ void scan_heads_kernel(const uint32_t* __restrict__ keys, uint32_t n, uint32_t* __restrict__ flags)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    flags[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1u : 0u;
}

// one thread per voxel head: scan_voxel_point over the run.  keys / order: sorted by voxel, input order inside one;
// key_label: sorted by (voxel, label), so the run covers the same positions.  The run of non-finite points (key ==
// nonfinite_key, last) is no voxel.
__global__ void scan_centroid_kernel(const mcl3dl_point* __restrict__ pts, const uint32_t* __restrict__ keys,
                                     const uint32_t* __restrict__ order, const uint64_t* __restrict__ key_label,
                                     const uint32_t* __restrict__ flags, const uint32_t* __restrict__ pos /* exclusive scan of flags */,
                                     uint32_t n, uint32_t nonfinite_key, mcl3dl_point* __restrict__ out, uint32_t* __restrict__ n_out)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const uint32_t key = keys[i];
  if (i == n - 1)
    *n_out = pos[i] + flags[i] - (key == nonfinite_key ? 1u : 0u);
  if (!flags[i] || key == nonfinite_key)
    return;
  uint32_t cnt = 1;
  while (i + cnt < n && keys[i + cnt] == key) ++cnt;
  out[pos[i]] = scan_voxel_point(pts, order + i, key_label + i, cnt);
}

__global__ void scan_clip_flags_kernel(const mcl3dl_point* __restrict__ pts, const uint32_t* __restrict__ n_ptr, ClipDev a, ClipDev b,
                                       uint32_t* __restrict__ flag_a, uint32_t* __restrict__ flag_b, uint32_t cap)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cap)
    return;
  const bool live = i < *n_ptr;
  const mcl3dl_point p = live ? pts[i] : mcl3dl_point{0, 0, 0, 0};
  flag_a[i] = (live && !clip_removes(a, p)) ? 1u : 0u;
  flag_b[i] = (live && !clip_removes(b, p)) ? 1u : 0u;
}

__global__ void scan_compact_kernel(const mcl3dl_point* __restrict__ pts, const uint32_t* __restrict__ flags,
                                    const uint32_t* __restrict__ pos, uint32_t cap, mcl3dl_point* __restrict__ out,
                                    uint32_t* __restrict__ n_out)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cap)
    return;
  if (i == cap - 1)
    *n_out = pos[i] + flags[i];
  if (flags[i])
    out[pos[i]] = pts[i];
}

// PointCloudUniformSampler::sample: draw t takes clipped point scan_sample_index(seed, stream, t, n)
__global__ void scan_sample_kernel(const mcl3dl_point* __restrict__ clipped, const uint32_t* __restrict__ n_ptr, uint32_t num,
                                   uint64_t seed, uint32_t stream, mcl3dl_point* __restrict__ out, uint32_t* __restrict__ n_out)
{
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t n = *n_ptr;
  if (t == 0)
    *n_out = n ? num : 0u;  // an empty clipped cloud gives an empty sample (:62-63)
  if (t >= num || n == 0)
    return;
  out[t] = clipped[scan_sample_index(seed, stream, t, n)];
}

}  // namespace mcl3dl
