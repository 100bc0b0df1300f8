// device_funcs.cuh — the per-thread device functions of the measurement update (no warp or CTA cooperation):
// grid descriptors, the exact 1-NN searches, the DDA and KD-tree ray casts.  Kept free of anything but scalar
// intrinsics so that tests/hostsim can compile this very file for the host (with tests/hostsim/cuda_shim.h) and
// check every function against the oracle without a GPU.  The kernels that call them live in kernels.cuh.
#pragma once
#ifndef MCL3DL_HOSTSIM
#include <cuda_runtime.h>
#endif
#include <math.h>
#include <algorithm>
#include <cmath>
#include <stdint.h>

#include "device_math.cuh"

// MCL3DL_NEAR_BITS=1 (default) compiles the near-field screens below into the searches; -DMCL3DL_NEAR_BITS=0 builds
// the kernels without them.
#ifndef MCL3DL_NEAR_BITS
#define MCL3DL_NEAR_BITS 1
#endif
namespace mcl3dl
{
// ---- near field: one bit per FINE cubic cell (edge ef = 1.01 * r / k) of the rescaled space, set when some map
// point's fine cell lies within k cells (Chebyshev) of it.  A query whose bit is clear has no map point within r:
// |p - q| < r  =>  per axis |p_a - q_a| < r = 0.99 k ef  =>  the two cell indices differ by at most k (the 1 % margin
// covers the float rounding of the shared cell function below for up to ~65 k cells per axis).  The field is a
// conservative screen in front of the exact searches: a set bit decides nothing, a clear bit skips the search.
struct NearBitsDev
{
  const uint32_t* bits;  // nullptr = no field: every query is "maybe near"
  int nx, ny, nz;        // fine cells per axis
  int pitch;             // 32-bit words per x-row
  float ox, oy, oz;      // origin in the rescaled space: k + 0.5 cells below the map's bounding box
  float inv_cell;
};

__device__ __forceinline__ int near_cell(float v, float o, float inv_cell)
{
  return __float2int_rd(fmul(fsub(v, o), inv_cell));
}

// false only if no map point can be within the radius the field was built for (queries outside the field's extent
// are at least k cells away from every point's cell; a NaN coordinate lands in cell 0 and at worst runs the search)
__device__ __forceinline__ bool near_maybe(const NearBitsDev& f, float qx, float qy, float qz)
{
  if (!f.bits)
    return true;
  const int cx = near_cell(qx, f.ox, f.inv_cell), cy = near_cell(qy, f.oy, f.inv_cell), cz = near_cell(qz, f.oz, f.inv_cell);
  if (static_cast<unsigned>(cx) >= static_cast<unsigned>(f.nx) || static_cast<unsigned>(cy) >= static_cast<unsigned>(f.ny) ||
      static_cast<unsigned>(cz) >= static_cast<unsigned>(f.nz))
    return false;
  const uint32_t w = __ldg(f.bits + (static_cast<size_t>(cz) * f.ny + cy) * f.pitch + (cx >> 5));
  return (w >> (cx & 31)) & 1u;
}

// Build side, per map point (rescaled coordinates): set the bits of every fine cell within k cells of the point's.
// x is the bit index inside a row, so one (dy, dz) row is a run of <= 2k+1 <= 31 bits = at most two word updates.
__device__ __forceinline__ void near_mark_point(const NearBitsDev& f, uint32_t* bits, int k, float sx, float sy, float sz)
{
  const int cx = near_cell(sx, f.ox, f.inv_cell), cy = near_cell(sy, f.oy, f.inv_cell), cz = near_cell(sz, f.oz, f.inv_cell);
  const int x0 = max(cx - k, 0), x1 = min(cx + k, f.nx - 1);
  if (x0 > x1)
    return;
  const int w0 = x0 >> 5, w1 = x1 >> 5;
  const uint32_t lo = 0xffffffffu << (x0 & 31), hi = 0xffffffffu >> (31 - (x1 & 31));
  for (int iz = max(cz - k, 0); iz <= min(cz + k, f.nz - 1); ++iz)
    for (int iy = max(cy - k, 0); iy <= min(cy + k, f.ny - 1); ++iy)
    {
      uint32_t* row = bits + (static_cast<size_t>(iz) * f.ny + iy) * f.pitch;
      if (w0 == w1)
        atomicOr(row + w0, lo & hi);
      else
      {
        atomicOr(row + w0, lo);
        atomicOr(row + w1, hi);
      }
    }
}

// Host side: extent of a field for search radius r (> 0) and dilation k (1..15) over the rescaled bounding box.
// The cell edge is doubled until the field fits max_bytes and 16 384 * k cells per axis (coarser is still conservative).
inline bool near_layout(NearBitsDev& f, float r, int k, const float sc_min[3], const float sc_max[3], size_t max_bytes)
{
  if (!(r > 0.0f) || k < 1 || k > 15)
    return false;
  float ef = 1.01f * r / static_cast<float>(k);
  for (int tries = 0; tries < 40; ++tries, ef *= 2.0f)
  {
    double dims[3];
    float org[3];
    bool ok = true;
    for (int a = 0; a < 3; ++a)
    {
      org[a] = sc_min[a] - (static_cast<float>(k) + 0.5f) * ef;
      dims[a] = floor((static_cast<double>(sc_max[a]) - org[a]) / ef) + k + 2;
      // the 1 % margin of the cell edge must cover the float rounding of near_cell() (a subtraction and a multiplication:
      // ~1.2e-7 x the cell index each, twice for a difference of two cells) against 0.01 cells / k of slack per cell of
      // distance: indices up to 2^14 * k keep the error below 0.4 of the margin
      ok = ok && dims[a] >= 1.0 && dims[a] <= 16384.0 * k;
    }
    if (!ok)
      continue;
    const double pitch = floor((dims[0] + 31.0) / 32.0);
    if (pitch * dims[1] * dims[2] * 4.0 > static_cast<double>(max_bytes))
      continue;
    f.bits = nullptr;
    f.nx = static_cast<int>(dims[0]);
    f.ny = static_cast<int>(dims[1]);
    f.nz = static_cast<int>(dims[2]);
    f.pitch = static_cast<int>(pitch);
    f.ox = org[0];
    f.oy = org[1];
    f.oz = org[2];
    f.inv_cell = 1.0f / ef;
    return true;
  }
  return false;
}

// ---- NN field ("Voronoi voxels"): the exact 1-NN search turned into a two-hop gather.  The rescaled space is cut into
// FINE voxels of edge e ~ radius / 2 (the near-field lattice with k = 2).  For every voxel the build keeps the list of
// map points that can be the nearest neighbour (within `radius`) of SOME query inside the voxel: a point is dropped only
// when another point is PROVABLY closer for every position in the (slightly padded) voxel box — the difference of the
// two squared distances is affine in the query, so its minimum over the box is evaluated exactly from the box corners,
// and the proof keeps a relative margin of 1e-5, fifty times the rounding of the float distance evaluation of the query
// side.  A query therefore reads one 8-byte directory entry (2 x 2 x 2 voxels: first candidate + eight 4-bit counts)
// and then the few (typically 3-6, contiguous) candidates, instead of walking a 3 x 3 window of CSR rows; the minimum
// of the float distances over the candidates equals the minimum over ALL map points bit for bit whenever it is below
// radius^2 (ties included: points that tie can not dominate each other).  A voxel with more than kNnfMaxCand survivors
// makes its cell a wide cell (counts in a side table); more than kNnfMaxSurv (raw clouds): CSR window search there.
// No reference counterpart: ChunkedKdtree::radiusSearch (chunked_kdtree.h:218-251) descends a kd-tree per query.
constexpr int kNnfMaxCand = 14;  // per voxel in a regular directory cell (4-bit counts)
constexpr int kNnfMaxSurv = 40;  // per voxel in a wide cell (8-bit counts, side table); more: overflow cell
struct NnFieldDev
{
  const uint2* dir;    // nullptr = no field.  Per coarse cell: x = index of its first candidate, y = 8 nibbles = candidates
                       // per fine voxel (sub-index x | y<<1 | z<<2).  x with bit 31 set: 0xffffffff = overflow cell
                       // (generic search), else a WIDE cell = index into `wide` (some voxel has 15..40 candidates: three
                       // surfaces meeting; 41 of 22 M cells on the synthetic map — keeping them out of the overflow class
                       // lets regular maps run the kernel variant without any fallback code, 22 % faster on c2)
  const uint4* wide;   // wide cells: x = first candidate, y / z = byte counts of voxels 0..3 / 4..7
  const float4* cand;  // rescaled xyz, w = original map index (bits)
  int nx, ny, nz;      // FINE voxels per axis
  int cnx, cny, cnz;   // coarse cells per axis = (n + 1) / 2
  float ox, oy, oz;    // origin of the lattice (rescaled space)
  float inv_e, e;      // 1 / fine edge, fine edge
  float radius;        // searches of radius (window half-width) <= this are exact
  float pad;           // the build pads every voxel box by this much (float rounding of the voxel index of a query)
};

// ---- distance field ("field mode", BASELINE.json north_star): a dense Euclidean-distance volume over the NN field's
// fine lattice, looked up by trilinear interpolation.  NOT exact (a distance field is a cone around every point;
// interpolating it at 0.1 m voxels is off by 1e-1 relative, SURVEY hard part 1), so it is an opt-in, reported variant:
// the one kernel of this path that is a pure HBM gather — one 32-byte sector per eval.  Layout: every lattice cell
// stores its 8 corner distances itself (2 x float4, 32-byte aligned), i.e. the node volume replicated 8x, so an eval
// reads exactly one sector instead of four (the corner rows of a plain volume are nx and nx * ny floats apart).
struct FieldDev
{
  const float4* cells;  // nullptr = not staged.  [cell][2]: {d000, d100, d010, d110}, {d001, d101, d011, d111}
  int nx, ny, nz;       // cells per axis (nodes: n + 1)
  float ox, oy, oz;     // position of node (0, 0, 0) in the rescaled space
  float inv_e;          // 1 / lattice edge
  float clamp;          // node values are min(exact distance, clamp); queries outside the lattice read clamp
};

// ---- likelihood search grid: cubic cells over the RESCALED map points (p * dist_weight), CSR of
// cell -> contiguous run in `pts` (x fastest, so an x-row of cells is one contiguous run).
struct NnGridDev
{
  const uint32_t* cell_start;  // [nx*ny*nz + 1]
  const float4* pts;           // rescaled xyz, w = original map index (bits)
  // Window table for the likelihood kernel: entry (x, y, z) at ((z*nx + x)*nyp + y) = {start of cell (x,y,z),
  // packed point counts of the 1 / 2 / 3 cells starting there along x (10 | 11 | 11 bits, all-ones = overflow)}.
  // y is the fastest index, so the three y-rows of a query window are adjacent and one eval fetches its whole
  // 3x3 window with 6 aligned 16-byte loads instead of 18 scattered 4-byte ones (L1 wavefronts, see DESIGN.md).
  const uint2* row3;
  int nyp;  // padded (even) y pitch of row3
  int nx, ny, nz;
  float ox, oy, oz;  // grid origin in the rescaled space
  float inv_cell;
  float wx, wy, wz;  // dist_weight
#if MCL3DL_NEAR_BITS
  NearBitsDev near;  // built for the likelihood radius (LikDev::rpad)
#endif
  NnFieldDev field;  // exact candidate lists per fine voxel (field.dir == nullptr: not staged)
  FieldDev fld;      // trilinear distance volume of the opt-in field mode (fld.cells == nullptr: not staged)
};

struct LikDev
{
  float match_dist_min;   // R
  float match_dist_flat;  // F
  float match_weight;     // W
  float r2;               // float(double(R)*double(R)): what pcl::KdTreeFLANN::radiusSearch hands to FLANN
  float rpad;             // window half-width, R plus a rounding guard
};

// ---- DDA grid: exactly RaycastUsingDDA's lattice (min_p_, dda_grid_size_, map_size_), occupancy as
// one bit per cell + CSR of per-cell points in map order.
struct DdaGridDev
{
  const uint32_t* occ;         // bit c of word c>>5
  const uint32_t* cell_start;  // [cells + 1]
  const float4* pts;           // raw xyz, w = label bits; sorted by cell, map order inside a cell
  int nx, ny, nz;
  float min_x, min_y, min_z;
  float max_x, max_y, max_z;
  double grid;             // dda_grid_size_
  double ray_angle_half;   // ray_angle_half_
  double min_dist_thr_sq;  // min_dist_thr_sq_
  float hit_tolerance;     // float(hit_tolerance_): Vec3 * double narrows to float (vec3.h:119)
  float hit_range_sq;
  float sin_total_ref;
  float beam_likelihood;
  float beam_likelihood_min;
  uint32_t filter_label_max;
  int short_only;
};

// ---- KD-tree raycaster (RaycastUsingKDTree, the node's default caster): marches over the likelihood
// search grid; the colliding map point's raw coordinates / label are fetched by original index.
struct KdRayDev
{
  const float4* raw_pts;  // map points as handed to set_map: xyz + label bits, original order
  float grid_min;         // map_grid_min_ (raycast_using_kdtree.h:50)
  float hit_tolerance;    // hit_tolerance_ (:52)
  float r1, r1_sq, r1_pad;  // radius sqrt(2)*grid_max/2 narrowed to float (:83), float(double r * double r), window half-width
  float r2, r2_sq, r2_pad;  // radius grid_min*2 + sqrt(2)*grid_max/2 (:95)
  double sin_den;           // map_grid_min_ * 2.0 (:98)
#if MCL3DL_NEAR_BITS
  NearBitsDev near;  // built for the marching search radius (r1_pad)
#endif
};

enum
{
  ST_SHORT = 0,
  ST_HIT = 1,
  ST_LONG = 2,
  ST_TOTAL_REFLECTION = 3
};

// --------------------------------------------------------------------------------------------
// Exact nearest-neighbour distance^2 (rescaled metric) within the radius; returns r2 if none.
__device__ __forceinline__ float nn_dist2(const NnGridDev& g, const LikDev& lp, float qx, float qy, float qz,
                                          uint32_t& n_rows, uint32_t& n_pts)
{
#if MCL3DL_NEAR_BITS
  if (!near_maybe(g.near, qx, qy, qz))
    return lp.r2;
#endif
  // Same cell function as the build kernel (monotone in its argument), applied to q -/+ rpad.
  int lx = __float2int_rd(fmul(fsub(fsub(qx, lp.rpad), g.ox), g.inv_cell));
  int ly = __float2int_rd(fmul(fsub(fsub(qy, lp.rpad), g.oy), g.inv_cell));
  int lz = __float2int_rd(fmul(fsub(fsub(qz, lp.rpad), g.oz), g.inv_cell));
  int hx = __float2int_rd(fmul(fsub(fadd(qx, lp.rpad), g.ox), g.inv_cell));
  int hy = __float2int_rd(fmul(fsub(fadd(qy, lp.rpad), g.oy), g.inv_cell));
  int hz = __float2int_rd(fmul(fsub(fadd(qz, lp.rpad), g.oz), g.inv_cell));
  lx = max(lx, 0);
  ly = max(ly, 0);
  lz = max(lz, 0);
  hx = min(hx, g.nx - 1);
  hy = min(hy, g.ny - 1);
  hz = min(hz, g.nz - 1);
  float best = lp.r2;
  if (lx > hx || ly > hy || lz > hz)
    return best;
  n_rows += static_cast<uint32_t>((hz - lz + 1) * (hy - ly + 1));
  for (int iz = lz; iz <= hz; ++iz)
  {
    for (int iy = ly; iy <= hy; ++iy)
    {
      const int row = (iz * g.ny + iy) * g.nx;
      const uint32_t s0 = __ldg(g.cell_start + row + lx);
      const uint32_t s1 = __ldg(g.cell_start + row + hx + 1);
      n_pts += s1 - s0;
      for (uint32_t s = s0; s < s1; ++s)
      {
        const float4 m = __ldg(g.pts + s);
        // flann::L2_Simple: sequential float accumulate of squared differences
        const float dx = fsub(qx, m.x);
        const float dy = fsub(qy, m.y);
        const float dz = fsub(qz, m.z);
        const float d = fadd(fadd(fmul(dx, dx), fmul(dy, dy)), fmul(dz, dz));
        best = fminf(best, d);  // KNNRadiusResultSet: keep d < worst
      }
    }
  }
  return best;
}

// --------------------------------------------------------------------------------------------
__device__ __forceinline__ int dda_to_index(float v, float mn, double grid)
{
  // toIndex, raycast_using_dda.h:205-210: float difference, double division, truncation
  return __double2int_rz(ddiv(static_cast<double>(fsub(v, mn)), grid));
}

// One ray: RaycastUsingDDA::setRay + getNextCastResult loop + getBeamStatus's decision.
//
// Measured choices:
//   * the axis choice is evaluated branch-free (selects): the 3-way branch
//     diverges whenever the lanes of a warp cross different faces;
//   * t_max needs float(|index - begin|): kept as a float counter (+1.0f per step) instead of an
//     int->float conversion per step;
//   * the occupancy word is re-read only when the cell leaves the current 32-cell word;
//   * replacing the twelve fp64 divisions of the set-up by guarded reciprocal multiplications, caching
//     the per-sensor ray origin, or screening the cone test in float changed nothing measurable
//     (the kernel is latency/occupancy bound, not fp64 bound) and were dropped again;
//   * occupancy matters most: __launch_bounds__(256, 4) (<= 64 registers).
//
// The ray is cut into three pieces: dda_setup (setRay), dda_advance (getNextCastResult up to the next occupied cell: a
// tight stepping loop with nothing else in it) and dda_test_cell (hasIntersection + getBeamStatus, fp64).  With the cone
// test inside the stepping loop it executed with 2-3 live lanes and took a large share of the samples;
// as a loop of "advance, then test" the lanes of a warp reconverge after the walk and test together: same operations
// per lane, same bits.
struct DdaRay
{
  F3 b, e, dir;
  float e0x, e0y, e0z, tdx, tdy, tdz;  // initial_edges_, t_delta_
  float tx, ty, tz;                    // t_max_
  float kx, ky, kz;                    // float(|current - begin|): small integers, exact in float
  int cx, cy, cz, sx, sy, sz;
  int pos, max_movement;
  int last_w, cell;
  uint32_t word;
};

// setRay, :66-104.  Returns ST_LONG when the ray never starts (begin outside the map box, :70-75), else -1.
__device__ __forceinline__ int dda_setup(const DdaGridDev& g, const F3& b, const F3& e, DdaRay& r)
{
  r.b = b;
  r.e = e;
  r.pos = 1;
  r.max_movement = 0;
  // isPointWithinMap, :260-270
  if (b.x < g.min_x || g.max_x < b.x || b.y < g.min_y || g.max_y < b.y || b.z < g.min_z || g.max_z < b.z)
    return ST_LONG;
  F3 d;
  d.x = fsub(e.x, b.x);
  d.y = fsub(e.y, b.y);
  d.z = fsub(e.z, b.z);
  const float nrm = __fsqrt_rn(dot3(d, d));
  F3 dir;
  dir.x = fdiv(d.x, nrm);
  dir.y = fdiv(d.y, nrm);
  dir.z = fdiv(d.z, nrm);
  r.dir = dir;
  const float ex = fadd(e.x, fmul(dir.x, g.hit_tolerance));
  const float ey = fadd(e.y, fmul(dir.y, g.hit_tolerance));
  const float ez = fadd(e.z, fmul(dir.z, g.hit_tolerance));
  const int bx = dda_to_index(b.x, g.min_x, g.grid);
  const int by = dda_to_index(b.y, g.min_y, g.grid);
  const int bz = dda_to_index(b.z, g.min_z, g.grid);
  // (end indices are clamped to +-2^29 so that garbage end points — infinite or 1e30 coordinates, for which the
  // reference's own int conversion is undefined — cannot overflow the differences; the begin index is inside the grid)
  constexpr int kIdxLim = 1 << 29;
  const int dix = max(-kIdxLim, min(kIdxLim, dda_to_index(ex, g.min_x, g.grid))) - bx;
  const int diy = max(-kIdxLim, min(kIdxLim, dda_to_index(ey, g.min_y, g.grid))) - by;
  const int diz = max(-kIdxLim, min(kIdxLim, dda_to_index(ez, g.min_z, g.grid))) - bz;
  r.max_movement = abs(dix) + abs(diy) + abs(diz);
  r.sx = dix < 0 ? -1 : 1;
  r.sy = diy < 0 ? -1 : 1;
  r.sz = diz < 0 ? -1 : 1;
  const float inf = __int_as_float(0x7f800000);
  r.e0x = r.e0y = r.e0z = r.tdx = r.tdy = r.tdz = inf;
  if (dix != 0)
  {
    // nearest = index * grid + min_p in double; |(nearest - begin) / dir| and |grid / dir| stored as float (:94-99)
    const double nearest = dadd(dmul(static_cast<double>(dir.x < 0 ? bx : bx + 1), g.grid), static_cast<double>(g.min_x));
    r.e0x = __double2float_rn(fabs(ddiv(dsub(nearest, static_cast<double>(b.x)), static_cast<double>(dir.x))));
    r.tdx = __double2float_rn(fabs(ddiv(g.grid, static_cast<double>(dir.x))));
  }
  if (diy != 0)
  {
    const double nearest = dadd(dmul(static_cast<double>(dir.y < 0 ? by : by + 1), g.grid), static_cast<double>(g.min_y));
    r.e0y = __double2float_rn(fabs(ddiv(dsub(nearest, static_cast<double>(b.y)), static_cast<double>(dir.y))));
    r.tdy = __double2float_rn(fabs(ddiv(g.grid, static_cast<double>(dir.y))));
  }
  if (diz != 0)
  {
    const double nearest = dadd(dmul(static_cast<double>(dir.z < 0 ? bz : bz + 1), g.grid), static_cast<double>(g.min_z));
    r.e0z = __double2float_rn(fabs(ddiv(dsub(nearest, static_cast<double>(b.z)), static_cast<double>(dir.z))));
    r.tdz = __double2float_rn(fabs(ddiv(g.grid, static_cast<double>(dir.z))));
  }
  r.tx = r.e0x;
  r.ty = r.e0y;
  r.tz = r.e0z;
  r.cx = bx;
  r.cy = by;
  r.cz = bz;
  r.kx = r.ky = r.kz = 0.0f;
  r.last_w = -1;
  r.word = 0;
  r.cell = 0;
  return -1;
}

// getNextCastResult, :106-159, up to the next OCCUPIED cell: returns -1 with r.cell set, or ST_LONG when the ray is
// exhausted / leaves the grid.  At most max_movement-1 cells; begin and end cells are never tested.
__device__ __forceinline__ int dda_advance(const DdaGridDev& g, DdaRay& r, uint32_t& n_steps)
{
  const int nxy = g.nx * g.ny;
  for (; r.pos < r.max_movement;)
  {
    ++r.pos;
    ++n_steps;
    // strict-'<' ladder (:114-147): x if tx<ty && tx<tz; y if !(tx<ty) && ty<tz; else z (on ties z beats
    // y beats x).  incrementIndex (:192-203) recomputes t_max from the start:
    // float(edge0) + float(t_delta) * float(|index - begin|).
    const bool lt_xy = r.tx < r.ty;
    const bool ax = lt_xy && (r.tx < r.tz);
    const bool ay = !lt_xy && (r.ty < r.tz);
    const bool az = !ax && !ay;
    r.cx += ax ? r.sx : 0;
    r.cy += ay ? r.sy : 0;
    r.cz += az ? r.sz : 0;
    r.kx = ax ? fadd(r.kx, 1.0f) : r.kx;
    r.ky = ay ? fadd(r.ky, 1.0f) : r.ky;
    r.kz = az ? fadd(r.kz, 1.0f) : r.kz;
    r.tx = ax ? fadd(r.e0x, fmul(r.tdx, r.kx)) : r.tx;
    r.ty = ay ? fadd(r.e0y, fmul(r.tdy, r.ky)) : r.ty;
    r.tz = az ? fadd(r.e0z, fmul(r.tdz, r.kz)) : r.tz;
    if (static_cast<unsigned>(r.cx) >= static_cast<unsigned>(g.nx) || static_cast<unsigned>(r.cy) >= static_cast<unsigned>(g.ny) ||
        static_cast<unsigned>(r.cz) >= static_cast<unsigned>(g.nz))
    {
      r.pos = r.max_movement;
      return ST_LONG;  // left the grid (:197-201)
    }
    const int cell = r.cx + r.cy * g.nx + r.cz * nxy;
    const int w = cell >> 5;
    if (w != r.last_w)
    {
      r.word = __ldg(g.occ + w);
      r.last_w = w;
    }
    if ((r.word >> (cell & 31)) & 1u)
    {
      r.cell = cell;
      return -1;
    }
  }
  return ST_LONG;
}

// hasIntersection, :237-258 (first point of the cell, in map order, inside the cone) + getBeamStatus, beam.cpp:164-189.
// Returns the ray's status, or -1: no (unfiltered) collision in this cell, the walk continues.
__device__ __forceinline__ int dda_test_cell(const DdaGridDev& g, const DdaRay& r, uint32_t& n_occ, uint32_t& n_tested)
{
  const uint32_t s0 = __ldg(g.cell_start + r.cell);
  const uint32_t s1 = __ldg(g.cell_start + r.cell + 1);
  ++n_occ;
  for (uint32_t s = s0; s < s1; ++s)
  {
    ++n_tested;
    const float4 m = __ldg(g.pts + s);
    F3 rel;
    rel.x = fsub(m.x, r.b.x);
    rel.y = fsub(m.y, r.b.y);
    rel.z = fsub(m.z, r.b.z);
    const double foot = static_cast<double>(fabsf(dot3(rel, r.dir)));
    const double a0 = dmul(g.ray_angle_half, foot);
    const double thr = fmax(dmul(a0, a0), g.min_dist_thr_sq);
    const double dsq = dsub(static_cast<double>(dot3(rel, rel)), dmul(foot, foot));
    if (dsq < thr)
    {
      if (__float_as_uint(m.w) > g.filter_label_max)
        return -1;  // this cell's collision is filtered; the walk continues with the next cell
      if (1.0f > g.sin_total_ref)
      {
        const double ddx = static_cast<double>(fsub(r.e.x, m.x));
        const double ddy = static_cast<double>(fsub(r.e.y, m.y));
        const double ddz = static_cast<double>(fsub(r.e.z, m.z));
        const float dist_sq = __double2float_rn(dadd(dadd(dmul(ddx, ddx), dmul(ddy, ddy)), dmul(ddz, ddz)));
        return dist_sq < g.hit_range_sq ? ST_HIT : ST_SHORT;
      }
      return ST_TOTAL_REFLECTION;
    }
  }
  return -1;
}

__device__ __forceinline__ int cast_ray(const DdaGridDev& g, const F3& b, const F3& e, uint32_t& n_steps,
                                        uint32_t& n_occ, uint32_t& n_tested)
{
  DdaRay r;
  int st = dda_setup(g, b, e, r);
  while (st < 0)
  {
    st = dda_advance(g, r, n_steps);
    if (st < 0)
      st = dda_test_cell(g, r, n_occ, n_tested);
  }
  return st;
}

// 1-NN within a radius with the index of the winner (ChunkedKdtree::radiusSearch(p, r, id, d2, 1)); ties go to
// the lowest original index, like the CPU checkers.  General window (any radius below a few cells).
__device__ __forceinline__ bool nn_search_arg(const NnGridDev& g, float qx, float qy, float qz, float rpad, float r_sq,
                                              float& best, uint32_t& best_orig, uint32_t& n_tested)
{
  int lx = __float2int_rd(fmul(fsub(fsub(qx, rpad), g.ox), g.inv_cell));
  int ly = __float2int_rd(fmul(fsub(fsub(qy, rpad), g.oy), g.inv_cell));
  int lz = __float2int_rd(fmul(fsub(fsub(qz, rpad), g.oz), g.inv_cell));
  int hx = __float2int_rd(fmul(fsub(fadd(qx, rpad), g.ox), g.inv_cell));
  int hy = __float2int_rd(fmul(fsub(fadd(qy, rpad), g.oy), g.inv_cell));
  int hz = __float2int_rd(fmul(fsub(fadd(qz, rpad), g.oz), g.inv_cell));
  lx = max(lx, 0);
  ly = max(ly, 0);
  lz = max(lz, 0);
  hx = min(hx, g.nx - 1);
  hy = min(hy, g.ny - 1);
  hz = min(hz, g.nz - 1);
  best = r_sq;
  best_orig = 0xffffffffu;
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
        ++n_tested;
        const float4 m = __ldg(g.pts + s);
        const float dx = fsub(qx, m.x);
        const float dy = fsub(qy, m.y);
        const float dz = fsub(qz, m.z);
        const float d = fadd(fadd(fmul(dx, dx), fmul(dy, dy)), fmul(dz, dz));  // flann::L2_Simple
        const uint32_t orig = __float_as_uint(m.w);
        if (d < best || (d == best && orig < best_orig && best_orig != 0xffffffffu))
        {
          best = d;
          best_orig = orig;
        }
      }
    }
  return best_orig != 0xffffffffu;
}

// --------------------------------------------------------------------------------------------
// NN field: candidate count and first index of voxel `sub` of a directory entry; -1 in an overflow cell.
__device__ __forceinline__ int nnf_slot(const NnFieldDev& f, uint2 d, int sub, uint32_t& start)
{
  if (d.x & 0x80000000u)
  {
    if (d.x == 0xffffffffu)
      return -1;
    // wide cell (rare): byte counts from the side table
    const uint4 w = __ldg(f.wide + (d.x & 0x7fffffffu));
    const uint32_t word = sub < 4 ? w.y : w.z;
    const int sh8 = 8 * (sub & 3);
    const uint32_t part = word & ((1u << sh8) - 1u);  // bytes of this word before the voxel's
    const uint32_t full = sub < 4 ? 0u : w.y;        // the whole first word when the voxel sits in the second
    const uint32_t s0 = ((part & 0x00ff00ffu) + ((part >> 8) & 0x00ff00ffu)) * 0x00010001u >> 16;
    const uint32_t s1 = ((full & 0x00ff00ffu) + ((full >> 8) & 0x00ff00ffu)) * 0x00010001u >> 16;
    start = w.x + s0 + s1;
    return static_cast<int>((word >> sh8) & 255u);
  }
  const int sh = 4 * sub;
  const uint32_t below = d.y & ((1u << sh) - 1u);  // nibbles of the voxels stored before this one
  const uint32_t m = (below & 0x0f0f0f0fu) + ((below >> 4) & 0x0f0f0f0fu);
  start = d.x + ((m * 0x01010101u) >> 24);
  return static_cast<int>((d.y >> sh) & 15u);
}

// NN field, query side.  Returns the number of candidates of q's voxel and their first index, 0 when q lies outside the
// lattice (then no map point is within `radius`: the lattice extends 2.5 voxels > radius beyond the map's box) or -1 in
// an overflow cell.
__device__ __forceinline__ int nnf_lookup(const NnFieldDev& f, float qx, float qy, float qz, uint32_t& start)
{
  const int vx = near_cell(qx, f.ox, f.inv_e), vy = near_cell(qy, f.oy, f.inv_e), vz = near_cell(qz, f.oz, f.inv_e);
  if (static_cast<unsigned>(vx) >= static_cast<unsigned>(f.nx) || static_cast<unsigned>(vy) >= static_cast<unsigned>(f.ny) ||
      static_cast<unsigned>(vz) >= static_cast<unsigned>(f.nz))
    return 0;
  const uint2 d = __ldg(f.dir + (static_cast<size_t>(vz >> 1) * f.cny + (vy >> 1)) * f.cnx + (vx >> 1));
  return nnf_slot(f, d, (vx & 1) | ((vy & 1) << 1) | ((vz & 1) << 2), start);
}

// Warp-cooperative candidate scan (kernels.cuh: lik_kernel_nf, phase B).  The candidate lists of a warp's evals are laid
// end to end in one list of (eval, candidate) slots; the list of eval `e` occupies slots [base, base + count).  A pass
// covers slots [lo, hi): name `e` as the owner of its slots in that range (own[slot - lo]).
__device__ __forceinline__ void nnf_fill_owner(uint8_t* own, int lo, int hi, int base, int count, int e)
{
  const int a = max(base, lo), b = min(base + count, hi);
  for (int i = a; i < b; ++i) own[i - lo] = static_cast<uint8_t>(e);
}

// flann::L2_Simple of one candidate: sequential float accumulate of squared differences
__device__ __forceinline__ float nnf_cand_d2(float qx, float qy, float qz, const float4& m)
{
  const float dx = fsub(qx, m.x);
  const float dy = fsub(qy, m.y);
  const float dz = fsub(qz, m.z);
  return fadd(fadd(fmul(dx, dx), fmul(dy, dy)), fmul(dz, dz));
}

// Point-major likelihood kernel (kernels.cuh: lik_kernel_nf_pm).  The scan is cut into n_slices slices of `slice`
// points (a multiple of `unit`, the points of one warp trip): as many as put one CTA of every (particle block, slice)
// pair in the `slots` resident CTA slots, `blocks` particle blocks given.  Each slice adds one 64-bit word per particle
// into the particle's accumulator: [arr_bits: 1, the slice's arrival | cnt_bits: its matches | the rest, signed: the sum
// of its contributions in 2^-fx_shift fixed point].  The fields below the sum never carry (arrivals <= n_slices <
// 2^arr_bits, matches <= N < 2^cnt_bits), and fx_shift keeps N contributions of at most match_dist_min * |match_weight|
// each below a quarter of the sum field's range.  ok: the rounding of N terms stays below 2^-30 of that bound (scans of
// up to a few thousand points); otherwise the particle-major kernel runs.
struct NfPmShape
{
  int slice, n_slices, fx_shift, arr_bits, cnt_bits;
  bool ok;
};
inline int nf_bit_width(int v)
{
  int b = 0;
  while (b < 31 && (v >> b) != 0) ++b;
  return b;
}
inline NfPmShape nf_pm_shape(int N, int blocks, int slots, int unit, float match_dist_min, float match_weight)
{
  NfPmShape s;
  const int n = std::max(1, std::min(slots / std::max(blocks, 1), (N + unit - 1) / unit));
  s.slice = std::max(unit, ((N + n - 1) / n + unit - 1) / unit * unit);
  s.n_slices = std::max(1, (N + s.slice - 1) / s.slice);
  s.arr_bits = nf_bit_width(s.n_slices);
  s.cnt_bits = nf_bit_width(N);
  const int sum_bits = 64 - s.arr_bits - s.cnt_bits;
  const double bound = static_cast<double>(std::max(N, 1)) * std::fabs(static_cast<double>(match_dist_min)) *
                       std::fabs(static_cast<double>(match_weight));
  int e = 0;
  if (bound > 0.0)
    std::frexp(bound, &e);  // bound < 2^e
  s.fx_shift = std::max(-120, std::min(120, sum_bits - 3 - e));
  s.ok = sum_bits - 3 - nf_bit_width(N) >= 30;
  return s;
}
// one eval's contribution in fixed point (exact but for the bits below 2^-fx_shift: the scale is a power of two)
__device__ __forceinline__ long long nf_fx_term(float contribution, int fx_shift)
{
  return static_cast<long long>(rintf(fmul(contribution, ldexpf(1.0f, fx_shift))));
}
// the word one slice adds to a particle's accumulator
__device__ __forceinline__ unsigned long long nf_pm_word(long long sum, uint32_t cnt, const NfPmShape& s)
{
  return (static_cast<unsigned long long>(sum) << (s.arr_bits + s.cnt_bits)) +
         (static_cast<unsigned long long>(cnt) << s.arr_bits) + 1ull;
}
// the accumulator after a slice's addition: true when it was the particle's last slice, with the match count and the
// score (the fixed-point sum back in float, rounded once)
__device__ __forceinline__ bool nf_pm_done(unsigned long long v, const NfPmShape& s, uint32_t& cnt, float& score)
{
  if ((v & ((1ull << s.arr_bits) - 1ull)) != static_cast<unsigned long long>(s.n_slices))
    return false;
  cnt = static_cast<uint32_t>((v >> s.arr_bits) & ((1ull << s.cnt_bits) - 1ull));
  const long long sum = static_cast<long long>(v) >> (s.arr_bits + s.cnt_bits);  // arithmetic: the sum is signed
  score = fmul(static_cast<float>(sum), ldexpf(1.0f, -s.fx_shift));               // int64 -> float rounds to nearest
  return true;
}

// nn_dist2 through the field (likelihood model): min over the voxel's candidates, r2 if none is closer.
__device__ __forceinline__ float nnf_dist2(const NnGridDev& g, const LikDev& lp, float qx, float qy, float qz,
                                           uint32_t& n_rows, uint32_t& n_pts)
{
  uint32_t s = 0;
  const int c = nnf_lookup(g.field, qx, qy, qz, s);
  if (c < 0)
    return nn_dist2(g, lp, qx, qy, qz, n_rows, n_pts);
  ++n_rows;  // one 8-byte directory entry
  n_pts += static_cast<uint32_t>(c);
  float best = lp.r2;
  for (int i = 0; i < c; ++i)
  {
    const float4 m = __ldg(g.field.cand + s + i);
    // flann::L2_Simple: sequential float accumulate of squared differences
    const float dx = fsub(qx, m.x);
    const float dy = fsub(qy, m.y);
    const float dz = fsub(qz, m.z);
    best = fminf(best, fadd(fadd(fmul(dx, dx), fmul(dy, dy)), fmul(dz, dz)));  // KNNRadiusResultSet: keep d < worst
  }
  return best;
}

// nn_search_arg through the field (KD-tree raycaster's marching search); any radius the field does not cover, or an
// overflow cell, goes to the generic window search.  Same winner: smallest float d^2 below r_sq, lowest index on ties.
__device__ __forceinline__ bool nnf_search_arg(const NnGridDev& g, float qx, float qy, float qz, float rpad, float r_sq,
                                               float& best, uint32_t& best_orig, uint32_t& n_tested)
{
  if (!g.field.dir || rpad > g.field.radius)
    return nn_search_arg(g, qx, qy, qz, rpad, r_sq, best, best_orig, n_tested);
  uint32_t s = 0;
  const int c = nnf_lookup(g.field, qx, qy, qz, s);
  if (c < 0)
    return nn_search_arg(g, qx, qy, qz, rpad, r_sq, best, best_orig, n_tested);
  best = r_sq;
  best_orig = 0xffffffffu;
  for (int i = 0; i < c; ++i)
  {
    ++n_tested;
    const float4 m = __ldg(g.field.cand + s + i);
    const float dx = fsub(qx, m.x);
    const float dy = fsub(qy, m.y);
    const float dz = fsub(qz, m.z);
    const float d = fadd(fadd(fmul(dx, dx), fmul(dy, dy)), fmul(dz, dz));  // flann::L2_Simple
    const uint32_t orig = __float_as_uint(m.w);
    if (d < best || (d == best && orig < best_orig && best_orig != 0xffffffffu))
    {
      best = d;
      best_orig = orig;
    }
  }
  return best_orig != 0xffffffffu;
}

// --------------------------------------------------------------------------------------------
// Field mode: trilinearly interpolated distance at q (rescaled space); `clamp` outside the lattice.
__device__ __forceinline__ float field_dist(const FieldDev& f, float qx, float qy, float qz)
{
  const float tx = fmul(fsub(qx, f.ox), f.inv_e), ty = fmul(fsub(qy, f.oy), f.inv_e), tz = fmul(fsub(qz, f.oz), f.inv_e);
  const int ix = __float2int_rd(tx), iy = __float2int_rd(ty), iz = __float2int_rd(tz);
  if (static_cast<unsigned>(ix) >= static_cast<unsigned>(f.nx) || static_cast<unsigned>(iy) >= static_cast<unsigned>(f.ny) ||
      static_cast<unsigned>(iz) >= static_cast<unsigned>(f.nz))
    return f.clamp;
  const float fx = fsub(tx, static_cast<float>(ix)), fy = fsub(ty, static_cast<float>(iy)), fz = fsub(tz, static_cast<float>(iz));
  const size_t cell = (static_cast<size_t>(iz) * f.ny + iy) * f.nx + ix;
  const float4 a = __ldg(f.cells + 2 * cell), b = __ldg(f.cells + 2 * cell + 1);
  const float c00 = fadd(a.x, fmul(fx, fsub(a.y, a.x))), c10 = fadd(a.z, fmul(fx, fsub(a.w, a.z)));
  const float c01 = fadd(b.x, fmul(fx, fsub(b.y, b.x))), c11 = fadd(b.z, fmul(fx, fsub(b.w, b.z)));
  const float c0 = fadd(c00, fmul(fy, fsub(c10, c00))), c1 = fadd(c01, fmul(fy, fsub(c11, c01)));
  return fadd(c0, fmul(fz, fsub(c1, c0)));
}

// --------------------------------------------------------------------------------------------
// NN field, build side: the candidates of fine voxel (vx, vy, vz), as positions into the CSR point array g.pts, in CSR
// order (out holds kNnfMaxSurv entries).  Returns their number, or kNnfMaxSurv + 1 when more survive (overflow).  All geometry in double, relative to
// the voxel centre (magnitudes <= ~1, so double rounding is ~1e-16 against margins of >= 1e-8).
struct NnfPt
{
  double x, y, z;
};

// squared distance from p (centre-relative) to the box [-h, h]^3 / to its farthest corner
__device__ __forceinline__ double nnf_min2(const NnfPt& p, double h)
{
  const double ax = fmax(fabs(p.x) - h, 0.0), ay = fmax(fabs(p.y) - h, 0.0), az = fmax(fabs(p.z) - h, 0.0);
  return ax * ax + ay * ay + az * az;
}
__device__ __forceinline__ double nnf_max2(const NnfPt& p, double h)
{
  const double ax = fabs(p.x) + h, ay = fabs(p.y) + h, az = fabs(p.z) + h;
  return ax * ax + ay * ay + az * az;
}
// true when a is closer than p, with margin, for EVERY query in the box: min over the box of |q-p|^2 - |q-a|^2
// = 2 q.(a-p) + |p|^2 - |a|^2, affine in q, so the minimum sits at the corner that opposes (a - p) axis by axis
__device__ __forceinline__ bool nnf_dominates(const NnfPt& a, const NnfPt& p, double h)
{
  const double dx = a.x - p.x, dy = a.y - p.y, dz = a.z - p.z;
  const double fmin_ = -2.0 * h * (fabs(dx) + fabs(dy) + fabs(dz)) + (p.x * p.x + p.y * p.y + p.z * p.z) -
                       (a.x * a.x + a.y * a.y + a.z * a.z);
  return fmin_ > 1e-5 * nnf_max2(p, h) + 1e-12;
}

__device__ __forceinline__ int nnf_select(const NnGridDev& g, const NnFieldDev& f, int vx, int vy, int vz, uint32_t* out)
{
  // voxel centre and padded half edge; search reach = radius (already padded by the caller's 1.0001 factor) + pad
  const double e = static_cast<double>(f.e);
  const double cx = static_cast<double>(f.ox) + (static_cast<double>(vx) + 0.5) * e;
  const double cy = static_cast<double>(f.oy) + (static_cast<double>(vy) + 0.5) * e;
  const double cz = static_cast<double>(f.oz) + (static_cast<double>(vz) + 0.5) * e;
  const double h = 0.5 * e + static_cast<double>(f.pad);
  const double reach = static_cast<double>(f.radius) * 1.00001 + 1e-7;
  const double r2 = reach * reach;
  // CSR cells that can hold such points: the same (monotone) float cell function as the build, on widened float bounds
  const float w = static_cast<float>(h + reach) * 1.001f + 1e-5f;
  const float fx = static_cast<float>(cx), fy = static_cast<float>(cy), fz = static_cast<float>(cz);
  const int lx = max(__float2int_rd(fmul(fsub(fsub(fx, w), g.ox), g.inv_cell)), 0);
  const int ly = max(__float2int_rd(fmul(fsub(fsub(fy, w), g.oy), g.inv_cell)), 0);
  const int lz = max(__float2int_rd(fmul(fsub(fsub(fz, w), g.oz), g.inv_cell)), 0);
  const int hx = min(__float2int_rd(fmul(fsub(fadd(fx, w), g.ox), g.inv_cell)), g.nx - 1);
  const int hy = min(__float2int_rd(fmul(fsub(fadd(fy, w), g.oy), g.inv_cell)), g.ny - 1);
  const int hz = min(__float2int_rd(fmul(fsub(fadd(fz, w), g.oz), g.inv_cell)), g.nz - 1);
  if (lx > hx || ly > hy || lz > hz)
    return 0;
  // pass 1: the anchor = the in-reach point whose farthest corner is nearest (it bounds the NN distance of every query)
  double best_max2 = 1e300;
  NnfPt anchor;
  anchor.x = anchor.y = anchor.z = 0.0;
  uint32_t anchor_s = 0xffffffffu;
  for (int iz = lz; iz <= hz; ++iz)
    for (int iy = ly; iy <= hy; ++iy)
    {
      const int row = (iz * g.ny + iy) * g.nx;
      const uint32_t s0 = __ldg(g.cell_start + row + lx), s1 = __ldg(g.cell_start + row + hx + 1);
      for (uint32_t s = s0; s < s1; ++s)
      {
        const float4 m = __ldg(g.pts + s);
        NnfPt p;
        p.x = static_cast<double>(m.x) - cx;
        p.y = static_cast<double>(m.y) - cy;
        p.z = static_cast<double>(m.z) - cz;
        if (nnf_min2(p, h) < r2)
        {
          const double mx2 = nnf_max2(p, h);
          if (mx2 < best_max2)
          {
            best_max2 = mx2;
            anchor = p;
            anchor_s = s;
          }
        }
      }
    }
  if (anchor_s == 0xffffffffu)
    return 0;
  const double u2 = best_max2 * (1.0 + 2e-5) + 1e-12;
  // pass 2: survivors of the anchor test, in CSR order
  uint32_t surv_s[kNnfMaxSurv];
  NnfPt surv[kNnfMaxSurv];
  int ns = 0;
  bool too_many = false;
  for (int iz = lz; iz <= hz; ++iz)
    for (int iy = ly; iy <= hy; ++iy)
    {
      const int row = (iz * g.ny + iy) * g.nx;
      const uint32_t s0 = __ldg(g.cell_start + row + lx), s1 = __ldg(g.cell_start + row + hx + 1);
      for (uint32_t s = s0; s < s1; ++s)
      {
        const float4 m = __ldg(g.pts + s);
        NnfPt p;
        p.x = static_cast<double>(m.x) - cx;
        p.y = static_cast<double>(m.y) - cy;
        p.z = static_cast<double>(m.z) - cz;
        const double mn2 = nnf_min2(p, h);
        if (!(mn2 < r2) || mn2 > u2)
          continue;
        if (s != anchor_s && nnf_dominates(anchor, p, h))
          continue;
        if (ns < kNnfMaxSurv)
        {
          surv_s[ns] = s;
          surv[ns] = p;
          ++ns;
        }
        else
          too_many = true;
      }
    }
  if (too_many)
    return kNnfMaxSurv + 1;
  // pass 3: pairwise — drop what any other survivor dominates (dominance is transitive over the box, so testing
  // against survivors that are themselves dropped later is still sound)
  int n_out = 0;
  for (int i = 0; i < ns; ++i)
  {
    bool dead = false;
    for (int j = 0; j < ns && !dead; ++j)
      dead = (j != i) && nnf_dominates(surv[j], surv[i], h);
    if (dead)
      continue;
    out[n_out++] = surv_s[i];
  }
  return n_out;
}

// One ray with RaycastUsingKDTree (raycasts/raycast_using_kdtree.h:57-110) + getBeamStatus (beam.cpp:157-192), cut into
// pieces like the DDA caster: kd_setup (setRay), kd_march (the marching steps up to the next position whose near-field
// bit is set: a 1-NN search could succeed there) and kd_probe (the search and, on a collision, the second search +
// getBeamStatus), so that the lanes of a warp reconverge between marching and searching.
struct KdRay
{
  F3 e;        // end point
  F3 pos, inc; // pos_, inc_
  int count, length;
};

// setRay, :57-64
__device__ __forceinline__ void kd_setup(const KdRayDev& k, const F3& b, const F3& e, KdRay& r)
{
  F3 d;
  d.x = fsub(e.x, b.x);
  d.y = fsub(e.y, b.y);
  d.z = fsub(e.z, b.z);
  const float nrm = __fsqrt_rn(dot3(d, d));
  // The march is capped at 65 536 steps (6.5 km at the default 0.1 m step; the node clips scans at <= 10 m): an end
  // point at 1e30 or +inf must not keep a warp busy for 2^31 steps.  (The reference's float -> int conversion of such a
  // length is undefined; on x86 it yields INT_MIN, i.e. no march at all.)
  r.length = min(__float2int_rz(floorf(fdiv(fadd(nrm, k.hit_tolerance), k.grid_min))), 65536);
  r.inc.x = fmul(fdiv(d.x, nrm), k.grid_min);
  r.inc.y = fmul(fdiv(d.y, nrm), k.grid_min);
  r.inc.z = fmul(fdiv(d.z, nrm), k.grid_min);
  r.pos.x = fadd(b.x, r.inc.x);
  r.pos.y = fadd(b.y, r.inc.y);
  r.pos.z = fadd(b.z, r.inc.z);
  r.e = e;
  r.count = 1;
}

// getNextCastResult's loop, :66-110, over the steps that cannot collide (near-field bit clear: free space, most steps
// of most rays).  Returns -1 at a position that needs the search (r.pos / r.count stay on it), ST_LONG at the ray's end.
__device__ __forceinline__ int kd_march(const KdRayDev& k, const NnGridDev& nn, KdRay& r, uint32_t& n_steps)
{
  for (; r.count < r.length; ++r.count)
  {
    ++n_steps;
#if MCL3DL_NEAR_BITS
    if (near_maybe(k.near, fmul(r.pos.x, nn.wx), fmul(r.pos.y, nn.wy), fmul(r.pos.z, nn.wz)))
      return -1;
    r.pos.x = fadd(r.pos.x, r.inc.x);
    r.pos.y = fadd(r.pos.y, r.inc.y);
    r.pos.z = fadd(r.pos.z, r.inc.z);
#else
    return -1;
#endif
  }
  return ST_LONG;
}

// The search at the current marching position (:83) and, on a collision with an unfiltered point, the second search two
// steps back for sin_angle_ (:91-98) + getBeamStatus's decision.  Returns the status, or -1 after advancing one step.
__device__ __forceinline__ int kd_probe(const KdRayDev& k, const NnGridDev& nn, const DdaGridDev& g, KdRay& r, uint32_t& n_occ,
                                        uint32_t& n_tested)
{
  float d2;
  uint32_t id;
  const float qx = fmul(r.pos.x, nn.wx), qy = fmul(r.pos.y, nn.wy), qz = fmul(r.pos.z, nn.wz);
  if (nnf_search_arg(nn, qx, qy, qz, k.r1_pad, k.r1_sq, d2, id, n_tested))
  {
    ++n_occ;
    const float4 m = __ldg(k.raw_pts + id);
    if (!(__float_as_uint(m.w) > g.filter_label_max))  // beam.cpp:168
    {
      const float d0 = __fsqrt_rn(d2);
      // pos_prev = pos_ - inc_ * 2.0 (:91), second search radius grid_min*2 + sqrt(2)*grid_max/2 (:95)
      const float px = fsub(r.pos.x, fmul(r.inc.x, 2.0f)), py = fsub(r.pos.y, fmul(r.inc.y, 2.0f)),
                  pz = fsub(r.pos.z, fmul(r.inc.z, 2.0f));
      float d2b;
      uint32_t idb;
      float sin_ang = 1.0f;
      if (nnf_search_arg(nn, fmul(px, nn.wx), fmul(py, nn.wy), fmul(pz, nn.wz), k.r2_pad, k.r2_sq, d2b, idb, n_tested))
      {
        const float d1 = __fsqrt_rn(d2b);
        sin_ang = __double2float_rn(ddiv(fabs(static_cast<double>(fsub(d1, d0))), k.sin_den));  // :98
      }
      if (sin_ang > g.sin_total_ref)
      {
        const double ddx = static_cast<double>(fsub(r.e.x, m.x));
        const double ddy = static_cast<double>(fsub(r.e.y, m.y));
        const double ddz = static_cast<double>(fsub(r.e.z, m.z));
        const float dist_sq = __double2float_rn(dadd(dadd(dmul(ddx, ddx), dmul(ddy, ddy)), dmul(ddz, ddz)));
        return dist_sq < g.hit_range_sq ? ST_HIT : ST_SHORT;
      }
      return ST_TOTAL_REFLECTION;
    }
  }
  r.pos.x = fadd(r.pos.x, r.inc.x);
  r.pos.y = fadd(r.pos.y, r.inc.y);
  r.pos.z = fadd(r.pos.z, r.inc.z);
  ++r.count;
  return -1;
}

__device__ __forceinline__ int cast_ray_kd(const KdRayDev& k, const NnGridDev& nn, const DdaGridDev& g, const F3& b,
                                           const F3& e, uint32_t& n_steps, uint32_t& n_occ, uint32_t& n_tested)
{
  KdRay r;
  kd_setup(k, b, e, r);
  int st = -1;
  while (st < 0)
  {
    st = kd_march(k, nn, r, n_steps);
    if (st < 0)
      st = kd_probe(k, nn, g, r, n_occ, n_tested);
  }
  return st;
}

// begin = s.pos_ + s.rot_ * origins[label] with the RAW rot_ (beam.cpp:145)
__device__ __forceinline__ F3 ray_origin(const F3& pos, const Q4& q_raw, const float* __restrict__ origins_xyz,
                                         uint32_t label)
{
  F3 o;
  o.x = __ldg(origins_xyz + 3 * label);
  o.y = __ldg(origins_xyz + 3 * label + 1);
  o.z = __ldg(origins_xyz + 3 * label + 2);
  const F3 ro = qrot(q_raw, o);
  F3 begin;
  begin.x = fadd(pos.x, ro.x);
  begin.y = fadd(pos.y, ro.y);
  begin.z = fadd(pos.z, ro.z);
  return begin;
}

}  // namespace mcl3dl
