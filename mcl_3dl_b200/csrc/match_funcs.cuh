// match_funcs.cuh — per-point pieces of the node's matched / unmatched output (mcl3dl_match_output,
// src/mcl_3dl.cpp:761-805): each point of the scan, transformed by the pose estimate, is looked up in the map index with
// ChunkedKdtree::radiusSearch(p, unmatch_output_dist, id, sqdist, 1) and classified.  Also compiled for the host by
// tests/hostsim (match_hostsim.cpp) and checked there against the CPU checkers.
//
// The search radius here (0.5 by default) exceeds the map index's max_search_radius, so the "global exact NN" that the
// likelihood searches rely on does not hold: which map points a query can see depends on its chunk
// (chunked_kdtree.h:124-263).  match_visible restates that rule exactly from the candidate's RAW coordinates.
// Float rules as in device_math.cuh: explicit round-to-nearest operations in the reference's operand order.
#pragma once
#include "device_funcs.cuh"
#include "scan_funcs.cuh"

namespace mcl3dl
{
enum
{
  MATCH_NEITHER = 0,
  MATCH_MATCHED = 1,
  MATCH_UNMATCHED = 2
};

struct MatchDev
{
  const float4* raw_pts;    // map points as handed to set_map, original order (the chunk rule needs raw coordinates)
  float r2;                 // float(double(r) * double(r)), r = float(unmatch_output_dist): KdTreeFLANN::radiusSearch
  float rpad;               // window half-width in the rescaled space: r plus a rounding guard
  double match_sq;          // match_output_dist * match_output_dist in double (src/mcl_3dl.cpp:777)
  float chunk_length;       // ChunkedKdtree::chunk_length_
  float pos_to_chunk;       // float(1.0 / double(chunk_length)) (chunked_kdtree.h:94)
  float max_search_radius;  // ChunkedKdtree::max_search_radius_
};

// getChunkId, chunked_kdtree.h:258-263 (finite coordinates only: the caller sends non-finite points elsewhere)
__device__ __forceinline__ int match_chunk(float v, float pos_to_chunk)
{
  return __float2int_rd(fmul(v, pos_to_chunk));
}

// Is the map point with raw coordinates `p` in the sub-cloud of chunk qc?  Its own chunk, or one of the halo copies
// setInputCloud makes (chunked_kdtree.h:138-199): per axis bound = -1 if in_chunk < max_search_radius, +1 if
// in_chunk > chunk_length - max_search_radius, and a copy goes to every chunk offset by a non-empty subset of the bounds.
__device__ __forceinline__ bool match_visible(const MatchDev& m, const float4& p, const int qc[3])
{
  const float v[3] = {p.x, p.y, p.z};
#pragma unroll
  for (int k = 0; k < 3; ++k)
  {
    const int pc = match_chunk(v[k], m.pos_to_chunk);
    const int d = qc[k] - pc;
    if (d == 0)
      continue;
    const float in_chunk = fsub(v[k], fmul(static_cast<float>(pc), m.chunk_length));
    int bound = 0;
    if (in_chunk < m.max_search_radius)
      bound = -1;
    else if (in_chunk > fsub(m.chunk_length, m.max_search_radius))
      bound = 1;
    if (bound == 0 || d != bound)
      return false;
  }
  return true;
}

// Class of one transformed point t (src/mcl_3dl.cpp:778-788).  The reference takes the nearest visible point within r
// and compares its sqdist with match_output_dist^2; as a question of existence that is:
//   matched:   some visible map point has d2 < r2 and double(d2) < match_sq (the nearest one then has too);
//   unmatched: no visible map point has d2 < r2;
//   neither:   otherwise.
// d2 is flann::L2_Simple in the rescaled space (same operation order as nn_search_arg).  Non-finite t is unmatched: the
// reference's floor(NaN) converts to INT_MIN on x86, no chunk has that id, and radiusSearch returns 0.
__device__ __forceinline__ int match_classify(const NnGridDev& g, const MatchDev& m, const F3& t)
{
  if (!scan_finite(t.x) || !scan_finite(t.y) || !scan_finite(t.z))
    return MATCH_UNMATCHED;
  const int qc[3] = {match_chunk(t.x, m.pos_to_chunk), match_chunk(t.y, m.pos_to_chunk), match_chunk(t.z, m.pos_to_chunk)};
  const float qx = fmul(t.x, g.wx), qy = fmul(t.y, g.wy), qz = fmul(t.z, g.wz);
  // same cell function as nn_key_kernel, applied to q -/+ rpad
  int lx = __float2int_rd(fmul(fsub(fsub(qx, m.rpad), g.ox), g.inv_cell));
  int ly = __float2int_rd(fmul(fsub(fsub(qy, m.rpad), g.oy), g.inv_cell));
  int lz = __float2int_rd(fmul(fsub(fsub(qz, m.rpad), g.oz), g.inv_cell));
  int hx = __float2int_rd(fmul(fsub(fadd(qx, m.rpad), g.ox), g.inv_cell));
  int hy = __float2int_rd(fmul(fsub(fadd(qy, m.rpad), g.oy), g.inv_cell));
  int hz = __float2int_rd(fmul(fsub(fadd(qz, m.rpad), g.oz), g.inv_cell));
  lx = max(lx, 0);
  ly = max(ly, 0);
  lz = max(lz, 0);
  hx = min(hx, g.nx - 1);
  hy = min(hy, g.ny - 1);
  hz = min(hz, g.nz - 1);
  bool near = false;  // some visible point within r seen
  for (int iz = lz; iz <= hz; ++iz)
    for (int iy = ly; iy <= hy; ++iy)
    {
      if (lx > hx)
        break;
      const int row = (iz * g.ny + iy) * g.nx;
      const uint32_t s0 = __ldg(g.cell_start + row + lx);
      const uint32_t s1 = __ldg(g.cell_start + row + hx + 1);
      for (uint32_t s = s0; s < s1; ++s)
      {
        const float4 p = __ldg(g.pts + s);
        const float dx = fsub(qx, p.x);
        const float dy = fsub(qy, p.y);
        const float dz = fsub(qz, p.z);
        const float d = fadd(fadd(fmul(dx, dx), fmul(dy, dy)), fmul(dz, dz));  // flann::L2_Simple
        if (!(d < m.r2))
          continue;
        const bool hit = static_cast<double>(d) < m.match_sq;
        if (!hit && near)
          continue;
        if (!match_visible(m, __ldg(m.raw_pts + __float_as_uint(p.w)), qc))
          continue;
        if (hit)
          return MATCH_MATCHED;
        near = true;
      }
    }
  return near ? MATCH_NEITHER : MATCH_UNMATCHED;
}

#ifndef MCL3DL_HOSTSIM
// One thread per scan point: the point transformed by the pose (label passed through) and one flag per output, which
// cub::DeviceScan + scan_compact_kernel turn into the two clouds in input order.
__global__ void match_classify_kernel(const mcl3dl_point* __restrict__ pts, uint32_t n, mcl3dl_pose pose, NnGridDev g, MatchDev m,
                                      mcl3dl_point* __restrict__ tf, uint32_t* __restrict__ flag_matched,
                                      uint32_t* __restrict__ flag_unmatched)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const mcl3dl_point p = pts[i];
  const Q4 rn = qnormalized(Q4{pose.qx, pose.qy, pose.qz, pose.qw});
  const F3 t = transform_point(rn, F3{pose.px, pose.py, pose.pz}, F3{p.x, p.y, p.z});
  const int cls = match_classify(g, m, t);
  tf[i] = mcl3dl_point{t.x, t.y, t.z, p.label};
  flag_matched[i] = cls == MATCH_MATCHED ? 1u : 0u;
  flag_unmatched[i] = cls == MATCH_UNMATCHED ? 1u : 0u;
}
#endif

}  // namespace mcl3dl
