// scan_funcs.cuh — per-point pieces of scan preprocessing (mcl3dl_scan_prepare, scan_kernels.cuh): the VoxelGrid
// lattice and voxel key, the finiteness test, the centroid and label vote of one voxel, the models' clip, the uniform
// sampler's index, and the normal-weighted sampler's neighbour grid, normal, weight and draw (ns_*).  They are also
// compiled for the host by tests/hostsim (scan_hostsim.cpp, normal_sampler_hostsim.cpp) and checked there against a
// numpy restatement of the same operations (tests/test_gpu_scan_exact.py) and against the normal sampler's checkers
// (tests/test_normal_sampler_on_host.py).
//
// Float rules as in device_math.cuh: explicit round-to-nearest operations in the reference's operand order.
#pragma once
#ifndef MCL3DL_HOSTSIM
#include <cuda_runtime.h>
#endif
#include <math.h>
#include <stdint.h>

#include <cmath>

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

// ---- PointCloudSamplerWithNormal::sample (point_cloud_random_samplers/point_cloud_sampler_with_normal.h:91-185) on a
// clipped cloud, mcl3dl_scan_sample_with_normal (scan_kernels.cuh: ns_*_kernel).  Every piece is deterministic double /
// float arithmetic with explicit rounding, so that the host build (tests/hostsim/normal_sampler_hostsim.cpp) gives the
// same bits.
#ifdef MCL3DL_HOSTSIM
inline double ns_dsqrt(double a) { return sqrt(a); }
inline uint64_t ns_umulhi64(uint64_t a, uint64_t b) { return static_cast<uint64_t>((static_cast<unsigned __int128>(a) * b) >> 64); }
#else
__device__ __forceinline__ double ns_dsqrt(double a) { return __dsqrt_rn(a); }
__device__ __forceinline__ uint64_t ns_umulhi64(uint64_t a, uint64_t b) { return __umul64hi(a, b); }
#endif

// The neighbour grid: the VoxelGrid lattice (voxel_key) with cell edge `edge` on all three axes, and the radius test
// flann::L2_Simple d2 < r2 = float(double r * double r).
struct NsGridDev
{
  VoxelGridDev g;
  float r2;
};

// Host side, once per clipped cloud: the lattice of the finite points' bounding box [mn, mx] for search radius r, with
// cell edge = float(r * (1 + m)).  Every point within r of a query then has a cell index within 1 of the query's on
// every axis: with s = float(1 / edge), |fl(p s) - fl(q s)| <= |p - q| s + 2 M s 2^-24 (M = the largest |coordinate|),
// and |p - q| s <= (1 + 5 * 2^-24) / (1 + m) for a float d2 below r2, so 2 M s 2^-24 <= m / 4 leaves the difference
// below 1.  m starts at 2^-10 and doubles while far coordinates need more (up to m = 1).  false: no such lattice, or
// 2^31 cells or more.
inline bool ns_lattice(double r, const float mn[3], const float mx[3], VoxelGridDev& g, int& end_bit, float& edge)
{
  float big = 0.0f;
  for (int k = 0; k < 3; ++k) big = fmaxf(big, fmaxf(fabsf(mn[k]), fabsf(mx[k])));
  for (double m = 1.0 / 1024.0; m <= 1.0; m *= 2.0)
  {
    edge = static_cast<float>(r * (1.0 + m));
    const double s = static_cast<double>(1.0f / edge);
    if (2.0 * static_cast<double>(big) * s * 5.9604644775390625e-08 > m / 4.0)
      continue;
    const float leaf[3] = {edge, edge, edge};
    if (!scan_voxel_lattice(leaf, mn, mx, g, end_bit))
      return false;
    return g.cells < 0x80000000u;
  }
  return false;
}

// first position in keys[0..n) (ascending) whose key is >= key
__device__ __forceinline__ uint32_t ns_lower_bound(const uint32_t* __restrict__ keys, uint32_t n, uint32_t key)
{
  uint32_t lo = 0, hi = n;
  while (lo < hi)
  {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (keys[mid] < key)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}

// One cyclic-Jacobi rotation of the symmetric 3 x 3 matrix on the pair (P, Q) (the off-diagonal entry apq; arp / arq:
// the entries of the third row R against P and Q), accumulated into the eigenvector columns of v (row-major).  An
// exactly zero apq is never rotated.
template <int P, int Q>
__device__ __forceinline__ void ns_jacobi_rotate(double& app, double& aqq, double& apq, double& arp, double& arq, double v[9])
{
  if (apq == 0.0)
    return;
  const double theta = ddiv(dsub(aqq, app), dmul(2.0, apq));
  double t = ddiv(1.0, dadd(fabs(theta), ns_dsqrt(dadd(dmul(theta, theta), 1.0))));
  if (theta < 0.0)
    t = -t;
  const double c = ddiv(1.0, ns_dsqrt(dadd(dmul(t, t), 1.0)));
  const double s = dmul(t, c);
  app = dsub(app, dmul(t, apq));
  aqq = dadd(aqq, dmul(t, apq));
  apq = 0.0;
  const double rp = arp, rq = arq;
  arp = dsub(dmul(c, rp), dmul(s, rq));
  arq = dadd(dmul(s, rp), dmul(c, rq));
#pragma unroll
  for (int k = 0; k < 3; ++k)
  {
    const double vp = v[k * 3 + P], vq = v[k * 3 + Q];
    v[k * 3 + P] = dsub(dmul(c, vp), dmul(s, vq));
    v[k * 3 + Q] = dadd(dmul(s, vp), dmul(c, vq));
  }
}

// Unit eigenvector of the smallest eigenvalue of the symmetric matrix (a00 a11 a22 a01 a02 a12): ten sweeps of cyclic
// Jacobi in double over (0,1), (0,2), (1,2), then the column of the smallest diagonal entry (lowest index on ties),
// divided by its length.
__device__ __forceinline__ void ns_smallest_eigvec(double a[6], double out[3])
{
  double v[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0};
  for (int sweep = 0; sweep < 10; ++sweep)
  {
    ns_jacobi_rotate<0, 1>(a[0], a[1], a[3], a[4], a[5], v);
    ns_jacobi_rotate<0, 2>(a[0], a[2], a[4], a[3], a[5], v);
    ns_jacobi_rotate<1, 2>(a[1], a[2], a[5], a[3], a[4], v);
  }
  // column select without a dynamic index, so that v stays in registers
  double x = v[0], y = v[3], z = v[6], lo = a[0];
  if (a[1] < lo)
  {
    x = v[1];
    y = v[4];
    z = v[7];
    lo = a[1];
  }
  if (a[2] < lo)
  {
    x = v[2];
    y = v[5];
    z = v[8];
  }
  const double len = ns_dsqrt(dadd(dadd(dmul(x, x), dmul(y, y)), dmul(z, z)));
  out[0] = ddiv(x, len);
  out[1] = ddiv(y, len);
  out[2] = ddiv(z, len);
}

// pcl::NormalEstimation at the clipped point q, restated: the neighbours are every finite point p of the cloud with
// flann::L2_Simple d2(q, p) < r2 (the query itself included), visited cell by cell in the 3 x 3 x 3 block (z, then y
// rows; one row's three cells are one run of the sorted keys), each cell's points in ascending index (skeys / spts: the
// cloud stably sorted by voxel_key).  Count, sum d and sum d d^T with d = p - q are accumulated in double; C = S / n -
// m m^T and the normal is ns_smallest_eigvec(C) as float.  Fewer than 3 neighbours or a non-finite q: NaN normal.
// Returns the neighbour count (0 for a non-finite q).
__device__ __forceinline__ uint32_t ns_point_normal(const NsGridDev& ng, const uint32_t* __restrict__ skeys,
                                                    const mcl3dl_point* __restrict__ spts, uint32_t n, const mcl3dl_point& q,
                                                    float nrm[3])
{
  const float nan = __int_as_float(0x7fc00000);
  nrm[0] = nrm[1] = nrm[2] = nan;
  if (!point_finite(q))
    return 0;
  const VoxelGridDev& g = ng.g;
  const int ix = __float2int_rd(fmul(q.x, g.inv_leaf[0])) - g.min_b[0];
  const int iy = __float2int_rd(fmul(q.y, g.inv_leaf[1])) - g.min_b[1];
  const int iz = __float2int_rd(fmul(q.z, g.inv_leaf[2])) - g.min_b[2];
  const int nx = static_cast<int>(g.div_b[0]), ny = static_cast<int>(g.div_b[1]), nz = static_cast<int>(g.div_b[2]);
  const uint32_t x0 = static_cast<uint32_t>(max(ix - 1, 0)), x1 = static_cast<uint32_t>(min(ix + 1, nx - 1));
  const double qx = static_cast<double>(q.x), qy = static_cast<double>(q.y), qz = static_cast<double>(q.z);
  uint32_t cnt = 0;
  double s[3] = {0.0, 0.0, 0.0}, ss[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};  // xx yy zz xy xz yz
  for (int z = iz - 1; z <= iz + 1; ++z)
  {
    if (z < 0 || z >= nz)
      continue;
    for (int y = iy - 1; y <= iy + 1; ++y)
    {
      if (y < 0 || y >= ny)
        continue;
      const uint32_t row = static_cast<uint32_t>(y) * g.div_b[0] + static_cast<uint32_t>(z) * (g.div_b[0] * g.div_b[1]);
      const uint32_t end = ns_lower_bound(skeys, n, row + x1 + 1);
      for (uint32_t j = ns_lower_bound(skeys, n, row + x0); j < end; ++j)
      {
        const mcl3dl_point p = spts[j];
        const float dx = fsub(q.x, p.x), dy = fsub(q.y, p.y), dz = fsub(q.z, p.z);
        const float d2 = fadd(fadd(fmul(dx, dx), fmul(dy, dy)), fmul(dz, dz));  // flann::L2_Simple
        if (!(d2 < ng.r2))
          continue;
        ++cnt;
        const double ex = dsub(static_cast<double>(p.x), qx), ey = dsub(static_cast<double>(p.y), qy),
                     ez = dsub(static_cast<double>(p.z), qz);
        s[0] = dadd(s[0], ex);
        s[1] = dadd(s[1], ey);
        s[2] = dadd(s[2], ez);
        ss[0] = dadd(ss[0], dmul(ex, ex));
        ss[1] = dadd(ss[1], dmul(ey, ey));
        ss[2] = dadd(ss[2], dmul(ez, ez));
        ss[3] = dadd(ss[3], dmul(ex, ey));
        ss[4] = dadd(ss[4], dmul(ex, ez));
        ss[5] = dadd(ss[5], dmul(ey, ez));
      }
    }
  }
  if (cnt < 3)
    return cnt;
  const double fn = static_cast<double>(cnt);
  const double m[3] = {ddiv(s[0], fn), ddiv(s[1], fn), ddiv(s[2], fn)};
  double a[6] = {dsub(ddiv(ss[0], fn), dmul(m[0], m[0])), dsub(ddiv(ss[1], fn), dmul(m[1], m[1])),
                 dsub(ddiv(ss[2], fn), dmul(m[2], m[2])), dsub(ddiv(ss[3], fn), dmul(m[0], m[1])),
                 dsub(ddiv(ss[4], fn), dmul(m[0], m[2])), dsub(ddiv(ss[5], fn), dmul(m[1], m[2]))};
  double e[3];
  ns_smallest_eigvec(a, e);
  nrm[0] = __double2float_rn(e[0]);
  nrm[1] = __double2float_rn(e[1]);
  nrm[2] = __double2float_rn(e[2]);
  return cnt;
}

// asin(x) for 0 <= x <= 0.5: its Maclaurin series to x^55 (coefficients C(2k, k) / (4^k (2k + 1)) as doubles), Horner
// in x^2; truncation below 1e-17 relative.
__device__ __forceinline__ double ns_asin_half(double x)
{
  const double c[28] = {1.0, 0.16666666666666666, 0.075, 0.044642857142857144, 0.030381944444444444, 0.022372159090909092,
                        0.017352764423076924, 0.01396484375, 0.011551800896139705, 0.009761609529194078, 0.008390335809616815,
                        0.0073125258735988454, 0.006447210311889649, 0.005740037670841924, 0.005153309682319905,
                        0.004660143486915096, 0.004240907093679363, 0.003880964558837669, 0.0035692053938259347,
                        0.003297059503473485, 0.0030578216492580306, 0.002846178401108942, 0.00265787063820729,
                        0.0024894486782468836, 0.002338091892111975, 0.0022014739737101384, 0.0020776610325181676,
                        0.0019650336162772837};
  const double y = dmul(x, x);
  double h = c[27];
#pragma unroll
  for (int k = 26; k >= 0; --k) h = dadd(c[k], dmul(y, h));
  return dmul(x, h);
}

constexpr double kNsHalfPi = 1.5707963267948966;  // M_PI / 2

// acos(a) for 0 <= a <= 1 in double from +, -, *, / and sqrt only (the same bits on the device and the host; within a
// few ulp of libm's): pi/2 - asin(a) up to 0.5, 2 asin(sqrt((1 - a) / 2)) above.
__device__ __forceinline__ double ns_acos01(double a)
{
  if (a <= 0.5)
    return dsub(kNsHalfPi, ns_asin_half(a));
  return dmul(2.0, ns_asin_half(ns_dsqrt(dmul(dsub(1.0, a), 0.5))));
}

// Step 5 of sample(): the weight of one normal.  acos_angle = |nx fx + ny fy + nz fz| (float products and sums in that
// order, widened to double), clamped to 1; weight = 1 + (max_weight - 1) ((pi/2 - angle) / (pi/2)); a NaN normal: 1.
__device__ __forceinline__ double ns_weight(const float nrm[3], const float fpc[3], double max_weight)
{
  if (nrm[0] != nrm[0] || nrm[1] != nrm[1] || nrm[2] != nrm[2])
    return 1.0;
  const float dot = fadd(fadd(fmul(nrm[0], fpc[0]), fmul(nrm[1], fpc[1])), fmul(nrm[2], fpc[2]));
  double a = fabs(static_cast<double>(dot));
  if (a > 1.0)
    a = 1.0;
  const double angle = ns_acos01(a);
  return dadd(1.0, dmul(dsub(max_weight, 1.0), ddiv(dsub(kNsHalfPi, angle), kNsHalfPi)));
}

// the fixed-point weight q = max(1, rint(w * 2^F)), scale = 2^F
__device__ __forceinline__ uint64_t ns_weight_q(double w, double scale)
{
  const double v = rint(dmul(w, scale));
  return v < 1.0 ? 1ull : static_cast<uint64_t>(v);
}

// Draw t of stream (0 likelihood, 1 beam): Philox-4x32-10 keyed by the seed's two words at counter (t mod 2^32, stream,
// 0x6e6f726d, t >> 32); r = the high word of (w0 | w1 << 32) * total, uniform on [0, total) up to 2^-64 relative.
__device__ __forceinline__ uint64_t ns_draw_value(uint64_t seed, uint32_t stream, uint64_t t, uint64_t total)
{
  uint32_t c[4] = {static_cast<uint32_t>(t), stream, 0x6e6f726du, static_cast<uint32_t>(t >> 32)};
  philox4x32_10(c, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  return ns_umulhi64(static_cast<uint64_t>(c[0]) | (static_cast<uint64_t>(c[1]) << 32), total);
}

// the first i with cum[i] > r (cum: the inclusive sum of the q, cum[n - 1] = total > r), so i is drawn with probability
// q_i / total
__device__ __forceinline__ uint32_t ns_draw_index(const uint64_t* __restrict__ cum, uint32_t n, uint64_t r)
{
  uint32_t lo = 0, hi = n - 1;
  while (lo < hi)
  {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (cum[mid] > r)
      hi = mid;
    else
      lo = mid + 1;
  }
  return lo;
}

// Host side, once per call: steps 2 and 3 of sample() in the reference's operation order, and the weight shift.
//   ratio = sqrt(lambda2 / lambda1); below perform_weighting_ratio: 1; above max_weight_ratio: max_weight; otherwise
//   1 + (max_weight - 1) (ratio - pwr) / (mwr - pwr).  A non-finite result becomes 1 (the reference's is undefined
//   there).
//   fpc_local = mean_rot.inv() * Vec3(float(v)) in float Quat arithmetic (quat.h: inv() = conj() * float(1.0 / dot),
//   q * v = q * Quat(v, 0) * q.conj()).
//   F = 32 - ceil(log2(max(1, max_weight))), so every q <= 2^32 and a sum over < 2^30 points stays below 2^62.
struct NsHostQuat
{
  float x, y, z, w;
};
inline NsHostQuat ns_host_qmul(const NsHostQuat& a, const NsHostQuat& b)
{
  return NsHostQuat{a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
                    a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
inline void ns_host_consts(const mcl3dl_normal_sampler_params& p, double* max_weight, float fpc_local[3], int* shift)
{
  const double ratio = sqrt(p.eigen_values[2] / p.eigen_values[1]);
  double mw = 1.0;
  if (ratio < p.perform_weighting_ratio)
    mw = 1.0;
  else if (ratio > p.max_weight_ratio)
    mw = p.max_weight;
  else
    mw = 1.0 + (p.max_weight - 1.0) * ((ratio - p.perform_weighting_ratio) / (p.max_weight_ratio - p.perform_weighting_ratio));
  if (!std::isfinite(mw))
    mw = 1.0;
  *max_weight = mw;
  const NsHostQuat r{p.mean_rot[0], p.mean_rot[1], p.mean_rot[2], p.mean_rot[3]};
  const float dot = r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w;
  const float inv = static_cast<float>(1.0 / static_cast<double>(dot));
  const NsHostQuat iv{-r.x * inv, -r.y * inv, -r.z * inv, r.w * inv};
  const NsHostQuat v{static_cast<float>(p.eigen_vector[0]), static_cast<float>(p.eigen_vector[1]), static_cast<float>(p.eigen_vector[2]), 0.0f};
  const NsHostQuat o = ns_host_qmul(ns_host_qmul(iv, v), NsHostQuat{-iv.x, -iv.y, -iv.z, iv.w});
  fpc_local[0] = o.x;
  fpc_local[1] = o.y;
  fpc_local[2] = o.z;
  int e = 0;
  const double fr = frexp(mw > 1.0 ? mw : 1.0, &e);  // m = fr 2^e, fr in [0.5, 1)
  *shift = 32 - (fr == 0.5 ? e - 1 : e);
}

}  // namespace mcl3dl
