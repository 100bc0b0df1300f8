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
// The node's other sampler, PointCloudSamplerWithNormal, replaces step 3 on demand (mcl3dl_scan_sample_with_normal,
// ns_*_kernel below): per clipped cloud a stable key sort into a neighbour grid, one thread per point for its normal
// and fixed-point weight, an exact uint64 inclusive sum, then rounds of weighted draws that keep each point's first
// draw.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/mcl3dl_b200.h"
#include "accum_funcs.cuh"
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

// ---- PointCloudSamplerWithNormal (mcl3dl_scan_sample_with_normal; the per-point pieces are ns_* of scan_funcs.cuh)
// keys / values of the neighbour grid's stable sort: voxel_key on the grid's lattice, clipped index
__global__ void ns_key_kernel(const mcl3dl_point* __restrict__ pts, uint32_t n, VoxelGridDev g, uint32_t* __restrict__ keys,
                              uint32_t* __restrict__ vals)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  keys[i] = voxel_key(g, pts[i]);
  vals[i] = i;
}

// the clipped points in sorted order
__global__ void ns_gather_kernel(const mcl3dl_point* __restrict__ pts, const uint32_t* __restrict__ order, uint32_t n,
                                 mcl3dl_point* __restrict__ spts)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    spts[i] = pts[order[i]];
}

// one thread per clipped point: its normal, neighbour count and fixed-point weight; n_finite counts the finite normals
__global__ void ns_normal_kernel(const mcl3dl_point* __restrict__ pts, uint32_t n, NsGridDev ng, const uint32_t* __restrict__ skeys,
                                 const mcl3dl_point* __restrict__ spts, float f0, float f1, float f2, double max_weight, double scale,
                                 float* __restrict__ normals, uint32_t* __restrict__ n_nb, uint64_t* __restrict__ q,
                                 uint32_t* __restrict__ n_finite)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  float nrm[3];
  n_nb[i] = ns_point_normal(ng, skeys, spts, n, pts[i], nrm);
  normals[3 * i + 0] = nrm[0];
  normals[3 * i + 1] = nrm[1];
  normals[3 * i + 2] = nrm[2];
  const float fpc[3] = {f0, f1, f2};
  q[i] = ns_weight_q(ns_weight(nrm, fpc, max_weight), scale);
  if (nrm[0] == nrm[0])
    atomicAdd(n_finite, 1u);
}

// draws d0 .. d0 + cnt - 1: their indices, and the first draw of each point (a 64-bit minimum over the draw numbers)
__global__ void ns_draw_kernel(const uint64_t* __restrict__ cum, uint32_t n, uint64_t seed, uint32_t stream, uint64_t d0, uint32_t cnt,
                               uint32_t* __restrict__ didx, unsigned long long* __restrict__ first)
{
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= cnt)
    return;
  const uint64_t t = d0 + k;
  const uint32_t i = ns_draw_index(cum, n, ns_draw_value(seed, stream, t, cum[n - 1]));
  didx[k] = i;
  atomicMin(first + i, static_cast<unsigned long long>(t));
}

// 1 where draw d0 + k is the first draw of its point
__global__ void ns_first_flag_kernel(const uint32_t* __restrict__ didx, const unsigned long long* __restrict__ first, uint64_t d0,
                                     uint32_t cnt, uint32_t* __restrict__ flags)
{
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < cnt)
    flags[k] = first[didx[k]] == d0 + k ? 1u : 0u;
}

// the round's first draws, in draw order, after the `carry` outputs of the earlier rounds (up to num); *carry_out =
// carry + the round's first draws
__global__ void ns_take_kernel(const mcl3dl_point* __restrict__ clipped, const uint32_t* __restrict__ didx, const uint32_t* __restrict__ flags,
                               const uint32_t* __restrict__ pos, uint32_t cnt, uint32_t carry, uint32_t num, mcl3dl_point* __restrict__ out,
                               uint32_t* __restrict__ carry_out)
{
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= cnt)
    return;
  const uint32_t j = carry + pos[k];
  if (k == cnt - 1)
    *carry_out = j + flags[k];
  if (flags[k] && j < num)
    out[j] = clipped[didx[k]];
}

// ---- cloud accumulation (mcl3dl_scan_accumulate / mcl3dl_scan_prepare_accumulated; per-point pieces: accum_funcs.cuh)
// accumCloud: point i of the uploaded PointCloud2 (row-major), moved into the odom frame and labelled with the
// accumulation index, at out[i]
__global__ void accum_cloud_kernel(const unsigned char* __restrict__ data, uint32_t width, uint32_t n, uint32_t row_step,
                                   uint32_t point_step, uint32_t ox, uint32_t oy, uint32_t oz, double tx, double ty, double tz,
                                   double qx, double qy, double qz, double qw, uint32_t label, mcl3dl_point* __restrict__ out)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const AccumXform m = accum_xform(tx, ty, tz, qx, qy, qz, qw);
  const F3 p = accum_apply(m, accum_read(data, i / width, i % width, row_step, point_step, ox, oy, oz));
  out[i] = mcl3dl_point{p.x, p.y, p.z, label};
}

// measure()'s pcl::transformPointCloud of the whole accumulation into base_link, labels kept
__global__ void accum_transform_kernel(const mcl3dl_point* __restrict__ in, uint32_t n, double tx, double ty, double tz, double qx,
                                       double qy, double qz, double qw, int dense, mcl3dl_point* __restrict__ out)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const AccumXform m = accum_xform(tx, ty, tz, qx, qy, qz, qw);
  const mcl3dl_point a = in[i];
  const F3 p = accum_second(m, dense != 0, F3{a.x, a.y, a.z});
  out[i] = mcl3dl_point{p.x, p.y, p.z, a.label};
}

// ---- map intake (mcl3dl_map_load / mcl3dl_map_update_set; per-point pieces: accum_funcs.cuh)
// fromROSMsg: point i of the uploaded map cloud (row-major) at pts[i], its intensity at inten[i]
__global__ void map_read_kernel(const unsigned char* __restrict__ data, uint32_t width, uint32_t n, uint32_t row_step, uint32_t point_step,
                                uint32_t ox, uint32_t oy, uint32_t oz, int32_t io, int32_t lo, mcl3dl_point* __restrict__ pts,
                                float* __restrict__ inten)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  float v;
  pts[i] = map_read(data, i / width, i % width, row_step, point_step, ox, oy, oz, io, lo, v);
  inten[i] = v;
}

// one thread per voxel head of voxel_grid's sorted runs (keys, order, flags, pos as scan_centroid_kernel reads them; see
// VoxelRuns in engine.cu): the voxel's intensity at out[pos[i]], the index its centroid has.  The run with key
// nonfinite_key (the non-finite points) is no voxel, as in scan_centroid_kernel.
__global__ void map_intensity_kernel(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ order,
                                     const uint32_t* __restrict__ flags, const uint32_t* __restrict__ pos, uint32_t n,
                                     uint32_t nonfinite_key, const float* __restrict__ inten, float* __restrict__ out)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !flags[i])
    return;
  const uint32_t key = keys[i];
  if (key == nonfinite_key)
    return;
  uint32_t cnt = 1;
  while (i + cnt < n && keys[i + cnt] == key) ++cnt;
  out[pos[i]] = map_voxel_intensity(inten, order + i, cnt);
}

// the unfiltered map (PCL's overflow rule, or no leaf): flag[i] = 1 for a finite point
__global__ void map_finite_flags_kernel(const mcl3dl_point* __restrict__ pts, uint32_t n, uint32_t* __restrict__ flags)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    flags[i] = point_finite(pts[i]) ? 1u : 0u;
}

// the flagged points and their intensities, order kept; *n_out = their count
__global__ void map_compact_kernel(const mcl3dl_point* __restrict__ pts, const float* __restrict__ inten,
                                   const uint32_t* __restrict__ flags, const uint32_t* __restrict__ pos, uint32_t n,
                                   mcl3dl_point* __restrict__ out, float* __restrict__ out_inten, uint32_t* __restrict__ n_out)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  if (i == n - 1)
    *n_out = pos[i] + flags[i];
  if (flags[i])
  {
    out[pos[i]] = pts[i];
    out_inten[pos[i]] = inten[i];
  }
}

}  // namespace mcl3dl
