// gl_funcs.cuh — per-thread pieces of global localisation and of resizing the resident particle set
// (mcl3dl_global_localization, mcl3dl_particles_resize): the node's free-space filter of the seed voxels
// (src/mcl_3dl.cpp:1058-1071), the particle fill (:1073-1096) and the pick of pf::ParticleFilter::resizeParticle
// (include/mcl_3dl/pf.h:399-436).  Also compiled for the host by tests/hostsim (gl_hostsim.cpp) and checked there against
// both CPU checkers (tests/test_global_localization_on_host.py).
//
// Float rules as in device_math.cuh: explicit round-to-nearest operations in the reference's operand order.  Nothing
// here draws a random number, so every output is exact.
#pragma once
#include <math.h>
#include <stdint.h>

#include <cmath>

#include "device_funcs.cuh"
#include "pf_funcs.cuh"
#include "scan_funcs.cuh"

namespace mcl3dl
{
// ---- free-space filter: a seed voxel p is dropped when kdtree->radiusSearch(p2, grid, id, sqdist, 1) finds a point,
// p2 = p raised by 0.01 + grid.  The tree holds the downsampled cloud vectorised by the node's point representation
// (xyz * dist_weight, float multiplies), so query and points live in the rescaled space and the test is
// flann::L2_Simple d2 < float(grid * grid) there (strict, as the shim KdTreeFLANN and FLANN's radius result set).
struct GlDev
{
  double z_off;  // 0.01 + grid, added to p.z in double: `p2.z += 0.01 + grid` (p2.z is a float)
  float r2;      // float(grid * grid): radiusSearch squares its double radius
  float rpad;    // window half-width in the rescaled space: the radius plus a rounding guard
};

// the rescaled query of p
__device__ __forceinline__ F3 gl_query(const NnGridDev& g, const GlDev& m, const mcl3dl_point& p)
{
  const float z2 = __double2float_rn(dadd(static_cast<double>(p.z), m.z_off));
  F3 q;
  q.x = fmul(p.x, g.wx);
  q.y = fmul(p.y, g.wy);
  q.z = fmul(z2, g.wz);
  return q;
}

// Does some point of the grid lie strictly within r2 of the rescaled query q?  The grid's cell edge is above rpad, so
// the window spans at most 3 cells per axis.  A non-finite query finds nothing (every distance to it is NaN or inf).
__device__ __forceinline__ bool gl_has_neighbour(const NnGridDev& g, const GlDev& m, const F3& q)
{
  if (!scan_finite(q.x) || !scan_finite(q.y) || !scan_finite(q.z))
    return false;
  // same cell function as nn_key_kernel, applied to q -/+ rpad
  int lx = __float2int_rd(fmul(fsub(fsub(q.x, m.rpad), g.ox), g.inv_cell));
  int ly = __float2int_rd(fmul(fsub(fsub(q.y, m.rpad), g.oy), g.inv_cell));
  int lz = __float2int_rd(fmul(fsub(fsub(q.z, m.rpad), g.oz), g.inv_cell));
  int hx = __float2int_rd(fmul(fsub(fadd(q.x, m.rpad), g.ox), g.inv_cell));
  int hy = __float2int_rd(fmul(fsub(fadd(q.y, m.rpad), g.oy), g.inv_cell));
  int hz = __float2int_rd(fmul(fsub(fadd(q.z, m.rpad), g.oz), g.inv_cell));
  lx = max(lx, 0);
  ly = max(ly, 0);
  lz = max(lz, 0);
  hx = min(hx, g.nx - 1);
  hy = min(hy, g.ny - 1);
  hz = min(hz, g.nz - 1);
  for (int iz = lz; iz <= hz; ++iz)
    for (int iy = ly; iy <= hy; ++iy)
    {
      if (lx > hx)
        break;
      const int row = (iz * g.ny + iy) * g.nx;
      const uint32_t s1 = __ldg(g.cell_start + row + hx + 1);
      for (uint32_t s = __ldg(g.cell_start + row + lx); s < s1; ++s)
      {
        const float4 p = __ldg(g.pts + s);
        const float dx = fsub(q.x, p.x);
        const float dy = fsub(q.y, p.y);
        const float dz = fsub(q.z, p.z);
        const float d = fadd(fadd(fmul(dx, dx), fmul(dy, dy)), fmul(dz, dz));  // flann::L2_Simple
        if (d < m.r2)
          return true;
      }
    }
  return false;
}

// ---- particle fill: particle i = State6DOF(seed[i / div_yaw], yaw[i % div_yaw]) with probability `prob`; the noise and
// odometry-error fields are those of the State6DOF(pos, rot) constructor, zero (state_6dof.h:192-200)
__device__ __forceinline__ PfState gl_particle(const mcl3dl_point* __restrict__ seeds, const Q4* __restrict__ yaw, uint32_t div_yaw,
                                               uint32_t i)
{
  const mcl3dl_point p = seeds[i / div_yaw];
  const Q4 r = yaw[i % div_yaw];
  PfState s;
  s.pos[0] = p.x;
  s.pos[1] = p.y;
  s.pos[2] = p.z;
  s.rot[0] = r.x;
  s.rot[1] = r.y;
  s.rot[2] = r.z;
  s.rot[3] = r.w;
  s.noise_ll = s.noise_la = s.noise_al = s.noise_aa = 0.0f;
  for (int k = 0; k < 3; ++k)
  {
    s.lin[k] = 0.0f;
    s.ang[k] = 0.0f;
  }
  return s;
}

// Host side, once per call: yaw[c] = (Quat(Vec3(0, 0, 2 pi c / div_yaw)) * imu_quat).normalized() for c < div_yaw, in the
// reference's operation order: the angle in double narrowed by Vec3's float constructor, Quat::setRPY (quat.h:196-209:
// float cos / sin of the half angles, every product written out, so that signed zeros come out as there), the Hamilton
// product (:131-138) and normalized() = operator*(float(1.0 / norm())) (:148-151,175-178).  Plain host arithmetic, like
// pf_set_odoms: x86-64 without FMA contraction rounds every operation like the reference's own build.
inline void gl_yaw_quats(int32_t div_yaw, const float imu[4], Q4* out)
{
  for (int32_t c = 0; c < div_yaw; ++c)
  {
    const float rpy[3] = {0.0f, 0.0f, static_cast<float>(2.0 * M_PI * c / div_yaw)};
    const float t2 = std::cos(rpy[0] / 2), t3 = std::sin(rpy[0] / 2);
    const float t4 = std::cos(rpy[1] / 2), t5 = std::sin(rpy[1] / 2);
    const float t0 = std::cos(rpy[2] / 2), t1 = std::sin(rpy[2] / 2);
    const Q4 a{t0 * t3 * t4 - t1 * t2 * t5, t0 * t2 * t5 + t1 * t3 * t4, t1 * t2 * t4 - t0 * t3 * t5, t0 * t2 * t4 + t1 * t3 * t5};
    const Q4 b{imu[0], imu[1], imu[2], imu[3]};
    const Q4 m{a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
               a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
    const float n = std::sqrt(m.x * m.x + m.y * m.y + m.z * m.z + m.w * m.w);
    const float inv = static_cast<float>(1.0 / n);
    out[c] = Q4{m.x * inv, m.y * inv, m.z * inv, m.w * inv};
  }
}

// `const float prob = 1.0 / static_cast<float>(points->size())` (src/mcl_3dl.cpp:1078): every particle gets it, so the
// set sums to div_yaw, not 1 (the reference's own quirk, kept: the next measurement normalises it away)
inline float gl_probability(uint64_t n_seeds) { return static_cast<float>(1.0 / static_cast<float>(n_seeds)); }

// ---- resizeParticle (pf.h:399-436).  accum[0..n) is the sequential float prefix sum of the probabilities (as for
// resampling), pstep = accum[n - 1] / float(num), and pscan[0..num) the sequential float chain pscan += pstep from 0,
// taken before each pick (so pscan[i] is NOT pstep * (i + 1) in float).  Output i takes lower_bound(pscan[i]) over accum
// (ties to the lowest index, the departure documented for resampling).  Past the end it copies it_prev: the last
// output's pick that was not past the end, or particle 0 when there is none.  pscan never decreases, so the outputs past
// the end form a suffix and a binary search finds its first member.
__device__ __forceinline__ uint32_t gl_resize_pick(const float* __restrict__ accum, uint32_t n, const float* __restrict__ pscan,
                                                   uint32_t i)
{
  const uint32_t it = pf_lower_bound(accum, n, __ldg(pscan + i));
  if (it < n)
    return it;
  uint32_t lo = 0, hi = i;  // first output whose pick is past the end
  while (lo < hi)
  {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (pf_lower_bound(accum, n, __ldg(pscan + mid)) < n)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo == 0 ? 0u : pf_lower_bound(accum, n, __ldg(pscan + lo - 1));
}

// the probability of every resized particle: `FLT_TYPE prob = 1.0 / num` (pf.h:418)
__device__ __forceinline__ float gl_resize_probability(uint32_t num) { return __double2float_rn(ddiv(1.0, static_cast<double>(num))); }

}  // namespace mcl3dl
