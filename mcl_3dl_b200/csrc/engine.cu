// engine.cu — host side of the C ABI (include/mcl3dl_b200.h): map staging on the device, the
// per-update launch sequence, multi-device sharding.  No CPU compute path exists here: every entry
// point either runs on a CUDA device or fails with an error code.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <limits>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

#include "gl_kernels.cuh"
#include "kernels.cuh"
#include "match_funcs.cuh"
#include "pf_kernels.cuh"
#include "scan_kernels.cuh"
#include "window_funcs.cuh"

using namespace mcl3dl;

namespace
{
constexpr int kMaxStagedBytes = 200 * 1024;
constexpr int kMaxStagedSorted = 160 * 1024;  // the sorted kernel also holds ~26 KB of static shared memory

// ---------------------------------------------------------------- device build kernels
inline float ord2f(uint32_t o)
{
  const uint32_t b = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
  float f;
  std::memcpy(&f, &b, 4);
  return f;
}

// bbox[0..2] = min raw, [3..5] = max raw, [6..8] = min rescaled, [9..11] = max rescaled (ordered-uint encoding)
__global__ void bbox_kernel(const mcl3dl_point* __restrict__ pts, size_t n, float wx, float wy, float wz,
                            uint32_t* __restrict__ bbox)
{
  float mn[6], mx[6];
#pragma unroll
  for (int k = 0; k < 6; ++k)
  {
    mn[k] = __int_as_float(0x7f800000);
    mx[k] = __int_as_float(0xff800000);
  }
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
  {
    const float4 p = __ldg(reinterpret_cast<const float4*>(pts) + i);
    const float v[6] = {p.x, p.y, p.z, fmul(p.x, wx), fmul(p.y, wy), fmul(p.z, wz)};
#pragma unroll
    for (int k = 0; k < 6; ++k)
    {
      mn[k] = fminf(mn[k], v[k]);
      mx[k] = fmaxf(mx[k], v[k]);
    }
  }
#pragma unroll
  for (int k = 0; k < 6; ++k)
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
      atomicMin(bbox + 6 + k, f2ord(mn[3 + k]));
      atomicMax(bbox + 9 + k, f2ord(mx[3 + k]));
    }
  }
}

// Likelihood grid: cell of a rescaled point.  MUST stay the same expression as nn_dist2's window bounds.
__global__ void nn_key_kernel(const mcl3dl_point* __restrict__ pts, uint32_t n, NnGridDev g,
                              uint32_t* __restrict__ keys, uint32_t* __restrict__ vals,
                              uint32_t* __restrict__ counts)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const float4 p = __ldg(reinterpret_cast<const float4*>(pts) + i);
  int cx = __float2int_rd(fmul(fsub(fmul(p.x, g.wx), g.ox), g.inv_cell));
  int cy = __float2int_rd(fmul(fsub(fmul(p.y, g.wy), g.oy), g.inv_cell));
  int cz = __float2int_rd(fmul(fsub(fmul(p.z, g.wz), g.oz), g.inv_cell));
  cx = min(max(cx, 0), g.nx - 1);
  cy = min(max(cy, 0), g.ny - 1);
  cz = min(max(cz, 0), g.nz - 1);
  const uint32_t c = static_cast<uint32_t>((cz * g.ny + cy) * g.nx + cx);
  keys[i] = c;
  vals[i] = i;
  atomicAdd(counts + c + 1, 1u);
}

__global__ void nn_gather_kernel(const mcl3dl_point* __restrict__ pts, uint32_t n, const uint32_t* __restrict__ order,
                                 float wx, float wy, float wz, float4* __restrict__ out)
{
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n)
    return;
  const uint32_t i = order[k];
  const float4 p = __ldg(reinterpret_cast<const float4*>(pts) + i);
  out[k] = make_float4(fmul(p.x, wx), fmul(p.y, wy), fmul(p.z, wz), __uint_as_float(i));
}

// ---- map window (window_funcs.cuh)
// What one call's queries need, folded into a zeroed WinNeed: the box of the finite particle positions, max(1, |q|^2) of
// their quaternions, the largest norm of a finite point of the two scans and of an origin.  Non-finite particles, points
// and origins are left out: their searches find nothing in any staging.
__global__ void window_need_kernel(const mcl3dl_pose* __restrict__ poses, uint32_t P, const mcl3dl_point* __restrict__ a,
                                   uint32_t na, const mcl3dl_point* __restrict__ b, uint32_t nb, const float* __restrict__ org,
                                   uint32_t norg, uint32_t* __restrict__ need)
{
  uint32_t w[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
  const size_t total = static_cast<size_t>(P) + na + nb + norg;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x)
  {
    if (i < P)
    {
      const mcl3dl_pose p = poses[i];
      if (isfinite(p.px) && isfinite(p.py) && isfinite(p.pz) && isfinite(p.qx) && isfinite(p.qy) && isfinite(p.qz) && isfinite(p.qw))
      {
        const float v[3] = {p.px, p.py, p.pz};
#pragma unroll
        for (int k = 0; k < 3; ++k)
        {
          w[k] = max(w[k], ~f2ord(v[k]));
          w[3 + k] = max(w[3 + k], f2ord(v[k]));
        }
        const double q2 = static_cast<double>(p.qx) * p.qx + static_cast<double>(p.qy) * p.qy + static_cast<double>(p.qz) * p.qz +
                          static_cast<double>(p.qw) * p.qw;
        w[7] = max(w[7], __float_as_uint(__double2float_ru(fmax(q2, 1.0))));
      }
      continue;
    }
    size_t j = i - P;
    float x, y, z;
    if (j < na)
    {
      x = a[j].x;
      y = a[j].y;
      z = a[j].z;
    }
    else if ((j -= na) < nb)
    {
      x = b[j].x;
      y = b[j].y;
      z = b[j].z;
    }
    else
    {
      j -= nb;
      x = org[3 * j];
      y = org[3 * j + 1];
      z = org[3 * j + 2];
    }
    if (isfinite(x) && isfinite(y) && isfinite(z))
    {
      const double n2 = static_cast<double>(x) * x + static_cast<double>(y) * y + static_cast<double>(z) * z;
      w[6] = max(w[6], __float_as_uint(__double2float_ru(__dsqrt_ru(n2) * (1.0 + 0x1p-40))));
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k)
  {
    const uint32_t m = __reduce_max_sync(0xffffffffu, w[k]);
    if ((threadIdx.x & 31) == 0 && m)
      atomicMax(need + k, m);
  }
}

// 1 for the map points inside the window box (the scan position of each comes from an exclusive sum)
__global__ void window_flag_kernel(const mcl3dl_point* __restrict__ pts, uint32_t n, WinBox box, uint32_t* __restrict__ flags)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const mcl3dl_point p = pts[i];
  flags[i] = win_point_inside(box, p.x, p.y, p.z) ? 1u : 0u;
}

// Appended points inside the window box (an append to a windowed map rebuilds the window only then)
__global__ void window_count_kernel(const mcl3dl_point* __restrict__ pts, uint32_t n, WinBox box, uint32_t* __restrict__ count)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const mcl3dl_point p = pts[i];
  if (win_point_inside(box, p.x, p.y, p.z))
    atomicAdd(count, 1u);
}

// The flagged points in map order and their original indices; n_out = their count
__global__ void window_compact_kernel(const mcl3dl_point* __restrict__ pts, const uint32_t* __restrict__ flags,
                                      const uint32_t* __restrict__ pos, uint32_t n, mcl3dl_point* __restrict__ out,
                                      uint32_t* __restrict__ idx, uint32_t* __restrict__ n_out)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  if (i == n - 1)
    *n_out = pos[i] + flags[i];
  if (flags[i])
  {
    out[pos[i]] = pts[i];
    idx[pos[i]] = i;
  }
}

// The window's CSR points carry their index into the window's point list: make it the map index (raw_pts)
__global__ void window_reindex_kernel(float4* __restrict__ pts, uint32_t n, const uint32_t* __restrict__ idx)
{
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n)
    return;
  pts[k].w = __uint_as_float(__ldg(idx + __float_as_uint(pts[k].w)));
}

// Window table of the likelihood grid (NnGridDev::row3), from the finished CSR.
__global__ void nn_row3_kernel(NnGridDev g, uint2* __restrict__ row3, size_t total)
{
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= total)
    return;
  const int y = static_cast<int>(i % g.nyp);
  const size_t zx = i / g.nyp;
  const int x = static_cast<int>(zx % g.nx);
  const int z = static_cast<int>(zx / g.nx);
  uint2 e = make_uint2(0u, 0u);
  if (y < g.ny)
  {
    const size_t cell = (static_cast<size_t>(z) * g.ny + y) * g.nx + x;
    const uint32_t s0 = g.cell_start[cell];
    const uint32_t c1 = g.cell_start[cell + min(1, g.nx - x)] - s0;
    const uint32_t c2 = g.cell_start[cell + min(2, g.nx - x)] - s0;
    const uint32_t c3 = g.cell_start[cell + min(3, g.nx - x)] - s0;
    e.x = s0;
    e.y = min(c1, 0x3ffu) | (min(c2, 0x7ffu) << 10) | (min(c3, 0x7ffu) << 21);  // all-ones field = "read the CSR"
  }
  row3[i] = e;
}

// Near field (NearBitsDev): every map point sets the bits of the fine cells within k cells of its own.
__global__ void near_mark_kernel(const mcl3dl_point* __restrict__ pts, uint32_t n, float wx, float wy, float wz, NearBitsDev f,
                                 uint32_t* __restrict__ bits, int k)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const float4 p = __ldg(reinterpret_cast<const float4*>(pts) + i);
  near_mark_point(f, bits, k, fmul(p.x, wx), fmul(p.y, wy), fmul(p.z, wz));
}

// NN field (device_funcs.cuh: NnFieldDev): one thread per FINE voxel, the 8 voxels of a directory cell in consecutive
// lanes.  Pass 1 counts the candidates (nibbles + per-cell totals); after an exclusive scan of the totals pass 2 repeats
// the selection and stores the candidates.  `bits` is the field's own k = 2 near field: a clear bit proves that no map
// point is within the radius of any query that maps to the voxel, so the (costly) selection only runs near surfaces.
// With `list` (after an append, update_nn_field) the threads cover the listed directory cells only: item i is cell
// list[i], and the per-item arrays (totals, base) are indexed by i; without it, item i is cell i.
__device__ __forceinline__ bool nnf_voxel_of_thread(const NnFieldDev& f, const uint32_t* list, size_t n_items, size_t t,
                                                    size_t& item, size_t& cell, int& sub, int& vx, int& vy, int& vz)
{
  item = t >> 3;
  sub = static_cast<int>(t & 7);
  if (item >= n_items)
    return false;
  cell = list ? list[item] : item;
  const int cx = static_cast<int>(cell % f.cnx);
  const size_t r = cell / f.cnx;
  const int cy = static_cast<int>(r % f.cny), cz = static_cast<int>(r / f.cny);
  vx = 2 * cx + (sub & 1);
  vy = 2 * cy + ((sub >> 1) & 1);
  vz = 2 * cz + (sub >> 2);
  return vx < f.nx && vy < f.ny && vz < f.nz;
}

__global__ void __launch_bounds__(256)
    nnf_count_kernel(NnGridDev g, NnFieldDev f, const uint32_t* __restrict__ bits, int pitch, uint2* __restrict__ dir,
                     uint32_t* __restrict__ totals, const uint32_t* __restrict__ list, size_t n_items, uint4* __restrict__ wide,
                     uint32_t wide_cap,
                     uint32_t* __restrict__ counters /* [0] wide cells used, [1] overflow cells; with a list also the
                                                         listed cells' old [2] candidates, [3] overflow and [4] wide cells */)
{
  const size_t t = blockIdx.x * static_cast<size_t>(256) + threadIdx.x;
  size_t item, cell = 0;
  int sub, vx, vy, vz, cnt = 0;
  if (nnf_voxel_of_thread(f, list, n_items, t, item, cell, sub, vx, vy, vz) &&
      ((__ldg(bits + (static_cast<size_t>(vz) * f.ny + vy) * pitch + (vx >> 5)) >> (vx & 31)) & 1u))
  {
    uint32_t tmp[kNnfMaxSurv];
    cnt = nnf_select(g, f, vx, vy, vz, tmp);
  }
  uint32_t ovf = cnt > kNnfMaxSurv ? 1u : 0u;
  uint32_t big = cnt > kNnfMaxCand ? 1u : 0u;
  const uint32_t c8 = static_cast<uint32_t>(min(cnt, 255));
  uint32_t lo = sub < 4 ? c8 << (8 * sub) : 0u, hi = sub >= 4 ? c8 << (8 * (sub - 4)) : 0u;
  uint32_t tot = static_cast<uint32_t>(cnt);
#pragma unroll
  for (int o = 1; o < 8; o <<= 1)
  {
    lo |= __shfl_xor_sync(0xffffffffu, lo, o);
    hi |= __shfl_xor_sync(0xffffffffu, hi, o);
    tot += __shfl_xor_sync(0xffffffffu, tot, o);
    ovf |= __shfl_xor_sync(0xffffffffu, ovf, o);
    big |= __shfl_xor_sync(0xffffffffu, big, o);
  }
  if (sub != 0 || item >= n_items)
    return;
  if (list)
  {
    // what the cell held before its re-selection (its old list becomes dead space)
    const uint2 d = dir[cell];
    if (d.x == 0xffffffffu)
      atomicAdd(counters + 3, 1u);
    else
    {
      uint32_t old = 0, start;
      for (int k = 0; k < 8; ++k) old += static_cast<uint32_t>(max(nnf_slot(f, d, k, start), 0));
      atomicAdd(counters + 2, old);
      if (d.x & 0x80000000u)
        atomicAdd(counters + 4, 1u);
    }
  }
  // dir[cell].y: nibbles | 0xfffffffe = wide cell (dir[cell].x already holds 0x80000000 | index) | 0xffffffff = overflow
  if (!ovf && big)
  {
    const uint32_t idx = atomicAdd(counters, 1u);
    if (idx < wide_cap)
    {
      wide[idx] = make_uint4(0u, lo, hi, 0u);  // x = first candidate, filled in by nnf_base_kernel
      dir[cell] = make_uint2(0x80000000u | idx, 0xfffffffeu);
      totals[item] = tot;
      return;
    }
    ovf = 1u;  // side table full: treat as an overflow cell
  }
  if (ovf)
  {
    dir[cell].y = 0xffffffffu;
    totals[item] = 0u;
    atomicAdd(counters + 1, 1u);
    return;
  }
  uint32_t nib = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) nib |= (((lo >> (8 * k)) & 15u) << (4 * k)) | (((hi >> (8 * k)) & 15u) << (4 * (k + 4)));
  dir[cell].y = nib;
  totals[item] = tot;
}

struct WidenU32
{
  __host__ __device__ unsigned long long operator()(uint32_t v) const { return v; }
};

// First candidate of every (listed) cell: the exclusive scan of the totals, plus `offset` (after an append: the end of
// the candidates already placed).
__global__ void nnf_base_kernel(uint2* __restrict__ dir, const uint32_t* __restrict__ base, uint32_t offset,
                                const uint32_t* __restrict__ list, size_t n_items, uint4* __restrict__ wide)
{
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n_items)
    return;
  const size_t c = list ? list[i] : i;
  const uint32_t y = dir[c].y;
  if (y == 0xffffffffu)
    dir[c].x = 0xffffffffu;
  else if (y == 0xfffffffeu)
    wide[dir[c].x & 0x7fffffffu].x = base[i] + offset;
  else
    dir[c].x = base[i] + offset;
}

__global__ void __launch_bounds__(256)
    nnf_fill_kernel(NnGridDev g, NnFieldDev f, const uint32_t* __restrict__ bits, int pitch, const uint2* __restrict__ dir,
                    float4* __restrict__ cand, const uint32_t* __restrict__ list, size_t n_items)
{
  const size_t t = blockIdx.x * static_cast<size_t>(256) + threadIdx.x;
  size_t item, cell;
  int sub, vx, vy, vz;
  if (!nnf_voxel_of_thread(f, list, n_items, t, item, cell, sub, vx, vy, vz))
    return;
  uint32_t start = 0;
  const int want = nnf_slot(f, dir[cell], sub, start);
  if (want <= 0)
    return;
  uint32_t pos[kNnfMaxSurv];
  const int cnt = nnf_select(g, f, vx, vy, vz, pos);
  for (int i = 0; i < cnt && i < want; ++i) cand[start + i] = g.pts[pos[i]];
}

// After an append: the directory cells the appended points pts[0..n) reach (device_funcs.cuh: nnf_mark_append), each
// listed once; count > cap tells the host that the list did not fit.
__global__ void nnf_mark_kernel(const mcl3dl_point* __restrict__ pts, uint32_t n, NnGridDev g, NnFieldDev f,
                                uint32_t* __restrict__ marks, uint32_t* __restrict__ list, uint32_t cap, uint32_t* __restrict__ count)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const float4 p = __ldg(reinterpret_cast<const float4*>(pts) + i);
  nnf_mark_append(g, f, p.x, p.y, p.z, [&](size_t cell) {
    const uint32_t bit = 1u << (cell & 31);
    if (atomicOr(marks + (cell >> 5), bit) & bit)
      return;
    const uint32_t k = atomicAdd(count, 1u);
    if (k < cap)
      list[k] = static_cast<uint32_t>(cell);
  });
}

// Field mode (device_funcs.cuh: FieldDev).  Node volume: exact distance (clamped) from every lattice node to the
// nearest map point, through the NN field; a pitched cudaMalloc3D volume so that cudaMemcpy3D moves it to / from the host.
__global__ void field_nodes_kernel(NnGridDev g, LikDev lp, cudaPitchedPtr vol, int nnx, int nny, int nnz, float clamp)
{
  const size_t t = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const size_t total = static_cast<size_t>(nnx) * nny * nnz;
  if (t >= total)
    return;
  const int i = static_cast<int>(t % nnx);
  const size_t r = t / nnx;
  const int j = static_cast<int>(r % nny), k = static_cast<int>(r / nny);
  const NnFieldDev& f = g.field;
  const float qx = fadd(f.ox, fmul(static_cast<float>(i), f.e)), qy = fadd(f.oy, fmul(static_cast<float>(j), f.e)),
              qz = fadd(f.oz, fmul(static_cast<float>(k), f.e));
  uint32_t a = 0, b = 0;
  const float d2 = nnf_dist2(g, lp, qx, qy, qz, a, b);
  float* row = reinterpret_cast<float*>(static_cast<char*>(vol.ptr) + (static_cast<size_t>(k) * nny + j) * vol.pitch);
  row[i] = d2 < lp.r2 ? fminf(__fsqrt_rn(d2), clamp) : clamp;
}

// cell (i, j, k) <- its 8 corner nodes, x fastest inside each float4
__global__ void field_expand_kernel(cudaPitchedPtr vol, int nx, int ny, int nz, float4* __restrict__ cells)
{
  const size_t t = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const size_t total = static_cast<size_t>(nx) * ny * nz;
  if (t >= total)
    return;
  const int i = static_cast<int>(t % nx);
  const size_t r = t / nx;
  const int j = static_cast<int>(r % ny), k = static_cast<int>(r / ny);
  const int nny = ny + 1;
  auto node = [&](int a, int b, int c) {
    return reinterpret_cast<const float*>(static_cast<const char*>(vol.ptr) + (static_cast<size_t>(c) * nny + b) * vol.pitch)[a];
  };
  cells[2 * t] = make_float4(node(i, j, k), node(i + 1, j, k), node(i, j + 1, k), node(i + 1, j + 1, k));
  cells[2 * t + 1] = make_float4(node(i, j, k + 1), node(i + 1, j, k + 1), node(i, j + 1, k + 1), node(i + 1, j + 1, k + 1));
}

// DDA grid: RaycastUsingDDA::setExists (raycast_using_dda.h:230-235) for every map point.
__global__ void dda_key_kernel(const mcl3dl_point* __restrict__ pts, uint32_t n, DdaGridDev g,
                               uint32_t* __restrict__ keys, uint32_t* __restrict__ vals,
                               uint32_t* __restrict__ counts, uint32_t* __restrict__ occ)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const float4 p = __ldg(reinterpret_cast<const float4*>(pts) + i);
  const int cx = dda_to_index(p.x, g.min_x, g.grid);
  const int cy = dda_to_index(p.y, g.min_y, g.grid);
  const int cz = dda_to_index(p.z, g.min_z, g.grid);
  const uint32_t c = static_cast<uint32_t>(cx + cy * g.nx + cz * (g.nx * g.ny));
  keys[i] = c;
  vals[i] = i;
  atomicAdd(counts + c + 1, 1u);
  atomicOr(occ + (c >> 5), 1u << (c & 31));
}

__global__ void dda_gather_kernel(const mcl3dl_point* __restrict__ pts, uint32_t n, const uint32_t* __restrict__ order,
                                  float4* __restrict__ out)
{
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n)
    return;
  out[k] = __ldg(reinterpret_cast<const float4*>(pts) + order[k]);  // xyz + label bits, map order kept by the stable sort
}

// Memory the engine owns: device memory (cudaMalloc) or a page-locked host block (cudaMallocHost).  Move-only; the
// destructor frees it.
template <bool kPinned>
struct Buf
{
  void* p = nullptr;
  size_t cap = 0;
  Buf() = default;
  Buf(Buf&& o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
  Buf& operator=(Buf&& o) noexcept
  {
    if (this != &o)
    {
      release();
      p = std::exchange(o.p, nullptr);
      cap = std::exchange(o.cap, 0);
    }
    return *this;
  }
  ~Buf() { release(); }
  // At least `bytes` (device memory: at least 256 B).  Grows only, by a new allocation: the contents are not kept.
  cudaError_t reserve(size_t bytes)
  {
    if (p && bytes <= cap)
      return cudaSuccess;
    if (const cudaError_t e = release())
      return e;
    const size_t want = kPinned ? bytes : std::max<size_t>(bytes, 256);
    if (const cudaError_t e = kPinned ? cudaMallocHost(&p, want) : cudaMalloc(&p, want))
      return e;
    cap = want;
    return cudaSuccess;
  }

 private:
  cudaError_t release()
  {
    const cudaError_t e = !p ? cudaSuccess : kPinned ? cudaFreeHost(p) : cudaFree(p);
    p = nullptr;
    cap = 0;
    return e;
  }
};
using DevBuf = Buf<false>;
using PinnedBuf = Buf<true>;

// Everything the engine holds on one device.  Not copyable or movable (the engine keeps its contexts where they were
// constructed); the destructor releases it all.
struct DeviceCtx
{
  DeviceCtx() = default;
  DeviceCtx(const DeviceCtx&) = delete;
  DeviceCtx& operator=(const DeviceCtx&) = delete;
  ~DeviceCtx()
  {
    cudaSetDevice(dev);
    for (cudaStream_t s : {stream, side})
      if (s)
        cudaStreamSynchronize(s);
    xchg_close();
    for (cudaEvent_t e : ev)
      if (e)
        cudaEventDestroy(e);
    for (cudaEvent_t e : {ev_fork, ev_join, ev_b0, ev_b1, ev_w0, ev_w1})
      if (e)
        cudaEventDestroy(e);
    for (cudaStream_t s : {side, stream})
      if (s)
        cudaStreamDestroy(s);
  }  // then the buffer members free themselves, on this device
  void xchg_close()
  {
    for (void*& o : x_opened)
      if (o)
      {
        cudaIpcCloseMemHandle(o);
        o = nullptr;
      }
    x_ready = false;
  }

  int dev = 0;
  cudaStream_t stream = nullptr;
  int sm_count = 132;
  // map
  DevBuf nn_cell_start, nn_pts, nn_row3, dda_occ, dda_cell_start, dda_pts;
  NnGridDev nn{};
  DdaGridDev dda{};
  KdRayDev kd{};
  DevBuf raw_pts;  // map points in original order (with a likelihood grid: KD-tree raycaster, matched / unmatched output)
  DevBuf near_lik, near_kd;  // near-field bits (MCL3DL_NEAR_BITS builds)
  DevBuf nnf_dir, nnf_cand, nnf_wide;  // NN field: directory, candidate lists, side table of the wide cells
  // NN field storage: candidates / wide entries placed so far (after appends: live and dead ones), wide-table capacity
  size_t nnf_cand_used = 0;
  uint32_t nnf_wide_used = 0, nnf_wide_cap = 0;
  uint32_t map_box[12] = {};  // bounding boxes of the staged map (bbox_kernel's encoding)
  DevBuf fld_cells;          // field mode: 8 corner distances per lattice cell
  DevBuf fld_mem;              // field mode: node volume (cudaMalloc3D), the owner of fld_nodes.ptr
  cudaPitchedPtr fld_nodes{};
  bool fld_nodes_valid = false;
  float near_kd_r = 0.0f;            // radius the KD field was built for
  size_t map_bytes = 0;
  size_t map_base = 0;  // the part of map_bytes a window rebuild keeps (raw points, DDA grid)
  // map window (window_funcs.cuh), when the whole map's likelihood lattice is refused: w_on = the map is staged windowed;
  // w_valid = the search structures hold the points inside w_box; w_stale = an append put points inside it since.  The
  // window's points in map order and their map indices, the reduction's block and its page-locked copy, the lattice,
  // the bytes of the window's structures, the rebuild count and the last rebuild's stream time (ev_w0 / ev_w1 around
  // the selection, then around the compaction and build).
  bool w_on = false, w_valid = false, w_stale = false;
  bool w_pending = false;  // window_need enqueued a reduction that window_settle has not read yet
  WinBox w_box{};
  int32_t w_dims[3] = {0, 0, 0};
  float w_org[3] = {0.0f, 0.0f, 0.0f};
  DevBuf w_pts, w_idx, w_need;
  PinnedBuf w_host;
  size_t w_bytes = 0;
  uint64_t w_rebuilds = 0;
  double w_ms = 0.0;
  cudaEvent_t ev_w0 = nullptr, ev_w1 = nullptr;
  // per-update I/O
  DevBuf d_poses /* whole input block of the host path */, d_out, d_status;
  PinnedBuf h_pinned;
  cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  // the two models are independent (disjoint fields of the record): the beam kernel runs on a side stream,
  // forked from / joined to the caller's stream with events
  cudaStream_t side = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_b0 = nullptr, ev_b1 = nullptr;
  DevBuf d_w, d_post, d_wpart, d_wticket;   // fused weight update: w_i, posterior, per-CTA partials, last-CTA tickets (2)
  DevBuf d_partial, d_tickets;  // lane-per-particle kernels: per-CTA partials + per-group ticket counters
  DevBuf d_tally, d_queue;      // dynamic-queue beam kernel: per-particle integer tallies, item counter (left at zero)
  DevBuf d_lacc;                // point-major likelihood kernel: per-particle accumulators (left at zero)
  std::vector<const void*> smem_opted;  // kernels already opted in to large dynamic shared memory on this device
  // resident particle set (mcl3dl_particles_*): two state buffers (resampling writes the other one), probabilities,
  // prefix sum + pstep, the packed poses / odometry-error factors the measurement kernels read
  // scan preprocessing (mcl3dl_scan_prepare): raw cloud, sort keys / values (x2), (voxel, label) keys of the vote (x2),
  // flags + scan positions (x2), the downsampled cloud, the two clipped clouds, the two sampled scans, cub scratch,
  // device-side counts
  DevBuf s_raw, s_keys[2], s_vals[2], s_key_label[2], s_flags[2], s_pos[2], s_ds, s_clip[2], s_out[2], s_tmp, s_counts;
  mcl3dl_scan_info s_info{};
  bool s_valid = false;
  // cloud accumulation (mcl3dl_scan_accumulate): the accumulated points in the odom frame, the last cloud's raw bytes;
  // points and clouds since the last clear, and whether every one of those clouds was dense
  DevBuf a_pts, a_raw;
  size_t a_n = 0;
  uint32_t a_clouds = 0;
  bool a_dense = true;
  // map intake (mcl3dl_map_load / mcl3dl_map_update_*): one intensity per staged point (mcl3dl_map_get; no kernel of the
  // models reads it); the pending patch and its intensities; the intake's raw bytes, converted cloud and intensities,
  // result and its intensities, VoxelGrid sort keys / values / (voxel, label) keys (x2), flags + scan positions, cub
  // scratch, device-side count
  DevBuf map_int, p_pts, p_int;
  DevBuf i_raw, i_cloud, i_cloud_int, i_pts, i_int, i_keys[2], i_vals[2], i_kl[2], i_flags, i_pos, i_tmp, i_count;
  // normal-weighted sampler (mcl3dl_scan_sample_with_normal): neighbour-grid sort keys / values (x2), sorted points; per
  // model the normals, neighbour counts and fixed-point weights of its clipped points (mcl3dl_scan_normals); the inclusive
  // sum of the weights, each point's first draw, a round's draw indices / flags / scan positions, the new sampled scans,
  // cub scratch, device-side words (bounding boxes, finite-normal counts, the round's carry)
  DevBuf n_keys[2], n_vals[2], n_spts, n_normals[2], n_nb[2], n_q[2], n_cum, n_first, n_didx, n_dflag, n_dpos, n_out[2], n_tmp, n_word;
  bool n_valid = false;
  // matched / unmatched output (mcl3dl_match_output), kept apart from the prepared scans it may read: host cloud,
  // transformed cloud, flags + scan positions per output, cub scratch; the page-locked block the compaction writes
  // both clouds and their counts into
  DevBuf m_in, m_tf, m_flags[2], m_pos[2], m_tmp;
  PinnedBuf m_host;
  // ray markers (mcl3dl_beam_cast): [pose | origins | host scan] on the device; the page-locked block holds the same
  // inputs for their one copy, the label error word and the records the kernel stores
  DevBuf b_in;
  PinnedBuf b_host;
  DevBuf r_states[2], r_prob, r_accum, r_poses, r_extra, r_est;  // r_est: EstHeader + per-CTA partial sums
  size_t r_n = 0;
  int r_cur = 0;
  uint32_t r_calls = 0;
  uint32_t r_redraw_calls = 0, r_noise_calls = 0;  // the Philox call words of the odometry-noise redraw and the expansion noise
  uint32_t r_init_calls = 0;                        // ... and of the initial seed
  // record exchange over peer memory (one process per GPU, mcl3dl_exchange_*): [world * n_local records | world flags]
  DevBuf xchg, x_ticket;  // x_ticket: [0] completed-step counter, [1] error word (device memory, local)
  PeerTable xt{};
  RecordSink xsink{};
  void* x_opened[kMaxPeers] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  size_t x_local = 0;   // records per rank
  uint32_t x_step = 0;
  bool x_ready = false;
  DevBuf d_stats;            // 5 x uint64 work counters, only written while stats collection is on
  bool stats_on = false;
  unsigned long long* stats_ptr() const { return stats_on ? static_cast<unsigned long long*>(d_stats.p) : nullptr; }
};
}  // namespace

struct mcl3dl_engine
{
  std::vector<DeviceCtx> devs;
  bool has_map = false;
  bool has_patch = false;  // mcl3dl_map_update_set left a pending patch (DeviceCtx::p_pts) of patch_n points
  size_t patch_n = 0;
  bool has_lik = false, has_beam = false;
  uint64_t stamp = 0;
  size_t n_points = 0;
  mcl3dl_lik_params lik{};
  mcl3dl_beam_params beam{};
  LikDev likdev{};
  mcl3dl_map_info info{};
  double t_h2d = 0, t_lik = 0, t_beam = 0, t_d2h = 0;
  uint64_t launches = 0;
  std::string err;
  float nn_cell_factor = 1.0f;
  int overlap = 1;  // run the beam and likelihood kernels concurrently (MCL3DL_OVERLAP=0 serialises them)
  int near_k = 2;     // near-field dilation of the likelihood screen (MCL3DL_NEAR_K, 0 = no field)
  int near_kd_k = 1;  // same for the KD-tree raycaster's marching search (MCL3DL_NEAR_KD_K)
  size_t near_max_bytes = size_t(256) << 20;  // MCL3DL_NEAR_MAX_MB
  int near_info_k[2] = {0, 0};
  uint64_t near_info_bytes[2] = {0, 0};
  // Host-path choices:
  int timing = 0;               // the per-call timing events of mcl3dl_last_timing cost tens of us per update: off unless
                                // mcl3dl_collect_timing(eng, 1) or MCL3DL_TIMING=1
  size_t zero_copy_max = 8192;  // the kernels of updates with <= this many particles per device store their records
                                // (or their posterior and weight summaries) straight into the pinned result block (no
                                // D2H copy launch); MCL3DL_ZEROCOPY_OUT
  int field_mode = 0;  // 1: the likelihood model reads the trilinear distance volume (opt-in, inexact; MCL3DL_LIK_MODE=field)
  size_t field_max_bytes = size_t(24) << 30;  // MCL3DL_FIELD_MAX_MB
  int beam_dq = 2;  // beam kernel: 2 = by job size, 1 = MCL3DL_BEAM=dq, 0 = MCL3DL_BEAM=pl
  int beam_dq_ppl = 0;  // MCL3DL_BEAM_DQ_PPL: rays per item (0 = chosen from the job size)
  int lik_share = 4;  // CTA slots per SM the likelihood kernel takes while the beam kernel runs next to it (MCL3DL_LIK_SHARE)
  int nnf_kd_r2 = 1;  // MCL3DL_NNF_KD_R2=0: the NN field also covers the KD-tree raycaster's second search radius
  int nnf = 1;  // stage the NN field (exact per-voxel candidate lists) and use lik_kernel_nf*; MCL3DL_NNF=0: lik_kernel_wi
  size_t nnf_max_bytes = size_t(32) << 30;  // MCL3DL_NNF_MAX_MB: directory + candidates above this -> no field
  // MCL3DL_MAP_MAX_CELLS: a map whose likelihood lattice has more cells is staged windowed, and no window may exceed it
  size_t map_max_cells = (size_t(1) << 31) - 1;
  uint64_t nnf_bytes = 0, nnf_cands = 0, nnf_overflow_cells = 0, nnf_wide_cells = 0;
  // page-locked blocks handed to the caller by mcl3dl_host_alloc: pose / record arrays that live in one of them are
  // DMA-ed (or, small updates, written by the kernels) in place instead of going through the engine's staging block
  std::vector<std::pair<char*, size_t>> host_blocks;
  size_t direct_min_bytes = size_t(64) << 10;  // smaller pose arrays ride in the staging block's single copy: a second DMA
                                               // operation costs more than their memcpy; MCL3DL_DIRECT_MIN_KB
};

static bool in_host_block(const mcl3dl_engine* eng, const void* p, size_t bytes)
{
  const char* q = static_cast<const char*>(p);
  for (const auto& b : eng->host_blocks)
    if (q >= b.first && q + bytes <= b.first + b.second)
      return true;
  return false;
}

namespace
{
#define CK(call)                                                                                     \
  do                                                                                                 \
  {                                                                                                  \
    cudaError_t e__ = (call);                                                                        \
    if (e__ != cudaSuccess)                                                                          \
    {                                                                                                \
      eng->err = std::string(#call) + ": " + cudaGetErrorString(e__) + " (" __FILE__ ":" + std::to_string(__LINE__) + ")"; \
      return MCL3DL_ERR_CUDA;                                                                        \
    }                                                                                                \
  } while (0)

template <bool kPinned>
int reserve(mcl3dl_engine* eng, Buf<kPinned>& b, size_t bytes)
{
  CK(b.reserve(bytes));
  return MCL3DL_OK;
}

// Scratch that the kernels leave at zero (tickets, counters, accumulators): when the buffer grows, its whole new capacity
// is zeroed on `st`, ahead of the kernels that read it there.
int reserve_zeroed(mcl3dl_engine* eng, DevBuf& b, size_t bytes, cudaStream_t st)
{
  if (b.p && bytes <= b.cap)
    return MCL3DL_OK;
  if (int rc = reserve(eng, b, bytes))
    return rc;
  CK(cudaMemsetAsync(b.p, 0, b.cap, st));
  return MCL3DL_OK;
}

// The weight update's grid for n particles and its scratch on one device: w_i, one slot set [nblk per-CTA partials |
// folded partial] per pass (0, 1) and a zeroed ticket per pass for its last-CTA fold
int weight_scratch(mcl3dl_engine* eng, DeviceCtx& c, size_t n, int pass, int* nblk, WeightPartial** slots, unsigned int** ticket)
{
  *nblk = static_cast<int>(std::min<size_t>((n + kBlockThreads - 1) / kBlockThreads, static_cast<size_t>(c.sm_count) * 4));
  int rc;
  if ((rc = reserve(eng, c.d_w, n * 4)) || (rc = reserve(eng, c.d_wpart, 2 * (*nblk + 1) * sizeof(WeightPartial))) ||
      (rc = reserve_zeroed(eng, c.d_wticket, 256, c.stream)))
    return rc;
  *slots = static_cast<WeightPartial*>(c.d_wpart.p) + pass * (*nblk + 1);
  *ticket = static_cast<unsigned int*>(c.d_wticket.p) + pass;
  return MCL3DL_OK;
}

int pick_tpp(size_t P, size_t N, int sm_count)
{
  // Enough threads to fill the chip (>= ~1024 per SM) but never more lanes than points.
  int tpp = 32;
  while (tpp < kBlockThreads && P * static_cast<size_t>(tpp) < static_cast<size_t>(sm_count) * 1024 &&
         static_cast<size_t>(tpp) < N)
    tpp *= 2;
  return tpp;
}

// launch(std::integral_constant<int, TPP>()) for the lanes per particle `tpp` chosen at run time: a power of two from
// LO to kBlockThreads, the kernels' template instances
template <int LO, typename F>
int with_tpp(int tpp, F&& launch)
{
  if constexpr (LO < kBlockThreads)
    if (tpp > LO)
      return with_tpp<2 * LO>(tpp, launch);
  return launch(std::integral_constant<int, LO>());
}

// cudaFuncSetAttribute is a driver call: opt each kernel instantiation in to the large dynamic shared memory
// size once per device instead of on every launch.
template <typename K>
int opt_in_smem(mcl3dl_engine* eng, DeviceCtx& c, K kernel, int bytes)
{
  // keyed by the kernel's address: instantiations with the same signature share one function-pointer type
  const void* key = reinterpret_cast<const void*>(kernel);
  for (const void* k : c.smem_opted)
    if (k == key)
      return MCL3DL_OK;
  CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  c.smem_opted.push_back(key);
  return MCL3DL_OK;
}

// ---- every kernel launch and every device-wide CUB call goes through launch / launch_pdl / cub_call: each returns its
// own error (CK at the call site names it) and counts one in mcl3dl_kernel_launches when it succeeded.  None of them
// allocates or synchronises, except that cub_call grows its scratch.
cudaError_t counted(mcl3dl_engine* eng, cudaError_t e)
{
  if (e == cudaSuccess)
    eng->launches++;
  return e;
}

template <typename... KArgs, typename... Args>
cudaError_t launch(mcl3dl_engine* eng, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                   Args... args)
{
  kernel<<<grid, block, smem, st>>>(static_cast<KArgs>(args)...);
  return counted(eng, cudaGetLastError());
}

// Launch with programmatic stream serialization (kernels.cuh: pdl_start): the kernel's launch and CTA dispatch overlap
// the drain of the grid before it in the stream; the kernel itself waits for that grid before its first global read.
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(mcl3dl_engine* eng, void (*kernel)(KArgs...), int grid, size_t smem, cudaStream_t st, Args... args)
{
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kBlockThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return counted(eng, cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...));
}

// A device-wide CUB call is a lambda f(void* temp, size_t& bytes) around one cub::Device* call.  cub_reserve grows `tmp`
// to the largest size query of the calls fs.  A function that runs several calls on one scratch sizes it for all of them
// before the first one, so that it never grows (and is freed, which waits for the device) between two of them.
template <typename... F>
cudaError_t cub_reserve(DevBuf& tmp, const F&... fs)
{
  cudaError_t e = cudaSuccess;
  size_t need = 0;
  const auto query = [&](const auto& f) {
    size_t bytes = 0;
    if (e == cudaSuccess)
      e = f(nullptr, bytes);
    need = std::max(need, bytes);
  };
  (query(fs), ...);
  return e != cudaSuccess ? e : tmp.reserve(need);
}

// One CUB call on scratch `tmp`, counted as one launch however many kernels CUB runs inside it
template <typename F>
cudaError_t cub_call(mcl3dl_engine* eng, DevBuf& tmp, const F& f)
{
  if (const cudaError_t e = cub_reserve(tmp, f))
    return e;
  size_t bytes = tmp.cap;
  return counted(eng, f(tmp.p, bytes));
}

// CSR-window likelihood kernel (no NN field staged)
template <int TPP>
int launch_lik_wi_t(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, int P, const float4* scan, int N,
                    mcl3dl_result* out, int beam_defaults, cudaStream_t st, const RecordSink& sink)
{
  constexpr int PPB = kBlockThreads / TPP;
  const int groups = (P + PPB - 1) / PPB;
  const int grid = std::max(1, std::min(groups, c.sm_count * 8));
  const size_t bytes = static_cast<size_t>(N) * 16;
  const bool staged = bytes <= static_cast<size_t>(kMaxStagedSorted);
  const auto kernel = staged ? lik_kernel_wi<TPP, true> : lik_kernel_wi<TPP, false>;
  if (staged)
    if (int rc = opt_in_smem(eng, c, kernel, kMaxStagedSorted)) return rc;
  CK(launch(eng, kernel, grid, kBlockThreads, staged ? bytes : 0, st, poses, P, scan, N, c.nn, eng->likdev, out, beam_defaults,
            c.stats_ptr(), sink));
  return MCL3DL_OK;
}

// ---- NN-field likelihood kernel: lanes per particle, staging and grid (kernels.cuh: lik_kernel_nf)
constexpr int kNfCtasPerSm = MCL3DL_NF_MINB;

int pick_tpp_nf(size_t P, size_t N, int sm_count)
{
  const size_t slots = static_cast<size_t>(sm_count) * kNfCtasPerSm;
  auto ctas = [&](int tpp) { return (P * tpp + kBlockThreads - 1) / kBlockThreads; };
  // ~kNfU evals per lane and particle ...
  int tpp = 8;
  while (tpp < kBlockThreads && static_cast<size_t>(tpp) * kNfU < N) tpp *= 2;
  // ... unless that leaves SMs without a CTA: then more lanes per particle (fewer evals per lane)
  while (tpp < kBlockThreads && static_cast<size_t>(tpp) < N && ctas(tpp) * 2 <= static_cast<size_t>(sm_count)) tpp *= 2;
  // a grid a little larger than the resident slots would run a mostly empty second wave: fewer, longer CTAs instead
  while (tpp > 8 && ctas(tpp) > slots && ctas(tpp) < 2 * slots) tpp /= 2;
  return tpp;
}

template <int TPP>
int launch_lik_nf_t(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, int P, const float4* scan, int N,
                    mcl3dl_result* out, int beam_defaults, cudaStream_t st, const RecordSink& sink)
{
  constexpr int PPB = kBlockThreads / TPP;
  const int groups = (P + PPB - 1) / PPB;
  // every CTA resident at once; CTAs loop when there are more particle groups than slots.  When the beam kernel runs
  // concurrently on the side stream (beam_defaults == 0: both models have a scan), the likelihood kernel takes only
  // `lik_share` of the 4 CTA slots per SM, so that beam CTAs become resident next to it instead of behind it.
  const int per_sm = beam_defaults ? kNfCtasPerSm : std::max(1, std::min(kNfCtasPerSm, eng->lik_share));
  const int grid = std::max(1, std::min(groups, c.sm_count * per_sm));
  const size_t bytes = static_cast<size_t>(N) * 16;
  const bool ovf = eng->nnf_overflow_cells != 0;
  // the tile pays when several particles of the CTA (or several loop trips) read it; otherwise the scan comes from L2
  const bool staged = bytes <= static_cast<size_t>(kMaxStagedBytes) / 2 && (PPB >= 4 || groups > grid);
  const auto kernel = staged ? (ovf ? lik_kernel_nf<TPP, true, true> : lik_kernel_nf<TPP, true, false>)
                             : (ovf ? lik_kernel_nf<TPP, false, true> : lik_kernel_nf<TPP, false, false>);
  if (staged)
    if (int rc = opt_in_smem(eng, c, kernel, kMaxStagedBytes / 2)) return rc;
  CK(launch_pdl(eng, kernel, grid, staged ? bytes : 0, st, poses, P, scan, N, c.nn, eng->likdev, out, beam_defaults,
                c.stats_ptr(), sink));
  return MCL3DL_OK;
}

// point-major mapping (kernels.cuh: lik_kernel_nf_pm): 256 particles per CTA, the scan cut into slices (nf_pm_shape)
int launch_lik_nf_pm(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, int P, const float4* scan, int N,
                     mcl3dl_result* out, int beam_defaults, cudaStream_t st, const RecordSink& sink, int blocks,
                     const NfPmShape& sh)
{
  // one accumulator per particle; zeroed once, the kernel leaves it at zero
  if (int rc = reserve_zeroed(eng, c.d_lacc, static_cast<size_t>(P) * 8, st))
    return rc;
  auto* acc = static_cast<unsigned long long*>(c.d_lacc.p);
  const auto kernel = eng->nnf_overflow_cells != 0 ? lik_kernel_nf_pm<true> : lik_kernel_nf_pm<false>;
  CK(launch_pdl(eng, kernel, blocks * sh.n_slices, 0, st, poses, P, scan, N, c.nn, eng->likdev, out, beam_defaults,
                c.stats_ptr(), sink, sh, acc));
  return MCL3DL_OK;
}

int launch_lik_nf(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* scan, size_t N,
                  mcl3dl_result* out, int beam_defaults, cudaStream_t st, const RecordSink& sink)
{
  const float4* s4 = reinterpret_cast<const float4*>(scan);
  const int p = static_cast<int>(P), n = static_cast<int>(N);
  if (P >= static_cast<size_t>(kBlockThreads))  // a full CTA of particles per scan point
  {
    const int blocks = (p + kBlockThreads - 1) / kBlockThreads;
    const int per_sm = beam_defaults ? kNfCtasPerSm : std::max(1, std::min(kNfCtasPerSm, eng->lik_share));
    const NfPmShape sh = nf_pm_shape(n, blocks, c.sm_count * per_sm, kNfU, eng->likdev.match_dist_min,
                                     eng->likdev.match_weight);
    if (sh.ok)
      return launch_lik_nf_pm(eng, c, poses, p, s4, n, out, beam_defaults, st, sink, blocks, sh);
  }
  return with_tpp<8>(pick_tpp_nf(P, N, c.sm_count), [&](auto tpp) {
    return launch_lik_nf_t<decltype(tpp)::value>(eng, c, poses, p, s4, n, out, beam_defaults, st, sink);
  });
}

// ---- field mode: staging and launch
// Stage (or re-stage from host node values) the distance volume of one device.  host_nodes == nullptr: the nodes are
// computed on the device from the NN field.  Either way the node volume is a cudaMalloc3D allocation and host <-> device
// moves go through cudaMemcpy3D (north_star: "staged once to HBM via cudaMemcpy3D").
int stage_field(mcl3dl_engine* eng, DeviceCtx& c, const float* host_nodes)
{
  const NnFieldDev& f = c.nn.field;
  if (!f.dir)
    return MCL3DL_ERR_INVALID_ARG;  // field mode sits on the NN field's lattice
  CK(cudaSetDevice(c.dev));
  const int nnx = f.nx + 1, nny = f.ny + 1, nnz = f.nz + 1;
  const size_t n_cells = static_cast<size_t>(f.nx) * f.ny * f.nz;
  if (n_cells * 32 > eng->field_max_bytes)
    return MCL3DL_ERR_TOO_LARGE;
  cudaStream_t st = c.stream;
  if (!c.fld_mem.p)
  {
    const cudaExtent ext = make_cudaExtent(static_cast<size_t>(nnx) * sizeof(float), nny, nnz);
    CK(cudaMalloc3D(&c.fld_nodes, ext));
    c.fld_mem.p = c.fld_nodes.ptr;
    c.fld_mem.cap = c.fld_nodes.pitch * nny * nnz;
  }
  int rc = reserve(eng, c.fld_cells, n_cells * 32);
  if (rc != MCL3DL_OK)
    return rc;
  const float clamp = f.radius;
  if (host_nodes)
  {
    cudaMemcpy3DParms cp{};
    cp.srcPtr = make_cudaPitchedPtr(const_cast<float*>(host_nodes), static_cast<size_t>(nnx) * sizeof(float), nnx, nny);
    cp.dstPtr = c.fld_nodes;
    cp.extent = make_cudaExtent(static_cast<size_t>(nnx) * sizeof(float), nny, nnz);
    cp.kind = cudaMemcpyHostToDevice;
    CK(cudaMemcpy3DAsync(&cp, st));
  }
  else
  {
    LikDev lp = eng->likdev;
    lp.rpad = f.radius;
    lp.r2 = static_cast<float>(static_cast<double>(clamp) * static_cast<double>(clamp));
    NnGridDev g = c.nn;
#if MCL3DL_NEAR_BITS
    // The likelihood screen is built for likdev.rpad, and the field's radius can be larger (the KD-tree raycaster's
    // search radius): in an overflow cell the window search must then run unscreened, or a node whose nearest point
    // lies between the two radii would read `clamp`.
    g.near.bits = nullptr;
#endif
    const size_t total = static_cast<size_t>(nnx) * nny * nnz;
    CK(launch(eng, field_nodes_kernel, static_cast<unsigned>((total + 255) / 256), 256, 0, st, g, lp, c.fld_nodes, nnx, nny, nnz,
              clamp));
  }
  CK(launch(eng, field_expand_kernel, static_cast<unsigned>((n_cells + 255) / 256), 256, 0, st, c.fld_nodes, f.nx, f.ny, f.nz,
            static_cast<float4*>(c.fld_cells.p)));
  CK(cudaStreamSynchronize(st));
  FieldDev d{};
  d.cells = static_cast<const float4*>(c.fld_cells.p);
  d.nx = f.nx;
  d.ny = f.ny;
  d.nz = f.nz;
  d.ox = f.ox;
  d.oy = f.oy;
  d.oz = f.oz;
  d.inv_e = f.inv_e;
  d.clamp = clamp;
  c.nn.fld = d;
  c.fld_nodes_valid = true;
  return MCL3DL_OK;
}

template <int TPP>
int launch_lik_field_t(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, int P, const float4* scan, int N,
                       mcl3dl_result* out, int beam_defaults, cudaStream_t st, const RecordSink& sink)
{
  constexpr int PPB = kBlockThreads / TPP;
  const int groups = (P + PPB - 1) / PPB;
  const int grid = std::max(1, std::min(groups, c.sm_count * kNfCtasPerSm));
  const size_t bytes = static_cast<size_t>(N) * 16;
  const bool staged = bytes <= static_cast<size_t>(kMaxStagedBytes) / 2 && (PPB >= 4 || groups > grid);
  const auto kernel = staged ? lik_kernel_field<TPP, true> : lik_kernel_field<TPP, false>;
  if (staged)
    if (int rc = opt_in_smem(eng, c, kernel, kMaxStagedBytes / 2)) return rc;
  CK(launch(eng, kernel, grid, kBlockThreads, staged ? bytes : 0, st, poses, P, scan, N, c.nn, eng->likdev, out, beam_defaults,
            c.stats_ptr(), sink));
  return MCL3DL_OK;
}

int launch_lik_field(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* scan, size_t N,
                     mcl3dl_result* out, int beam_defaults, cudaStream_t st, const RecordSink& sink)
{
  const float4* s4 = reinterpret_cast<const float4*>(scan);
  const int p = static_cast<int>(P), n = static_cast<int>(N);
  return with_tpp<8>(pick_tpp_nf(P, N, c.sm_count), [&](auto tpp) {
    return launch_lik_field_t<decltype(tpp)::value>(eng, c, poses, p, s4, n, out, beam_defaults, st, sink);
  });
}

PlShape pick_pl_shape(size_t P, size_t N, int sm_count)
{
  // Every warp walks `ppl` consecutive scan points for 32 particles.  The kernels hold 4 CTAs = 32 warps per SM
  // (64 registers), and a grid slightly larger than the resident slots runs a mostly empty second wave: size the chunks so that the whole grid is resident at once when
  // the job allows it, and otherwise make it many waves deep.
  const size_t groups = (P + 31) / 32;
  const size_t slots = static_cast<size_t>(sm_count) * 4;  // resident CTAs
  PlShape sh;
  auto ctas_for = [&](size_t ppl, PlShape& o) {
    const size_t chunks = std::max<size_t>((N + ppl - 1) / ppl, 1);
    int cpg = kPlWarps;
    while (cpg > 1 && static_cast<size_t>(cpg) / 2 >= chunks) cpg /= 2;  // smallest power of two >= chunks (<= 8)
    o.ppl = static_cast<int>(ppl);
    o.cpg = cpg;
    o.cb = cpg == kPlWarps ? static_cast<int>((chunks + kPlWarps - 1) / kPlWarps) : 1;
    const size_t gpc = kPlWarps / cpg;
    return (groups + gpc - 1) / gpc * o.cb;
  };
  size_t ppl = std::max<size_t>((N * groups + slots * kPlWarps - 1) / std::max<size_t>(slots * kPlWarps, 1), 1);
  ppl = std::min<size_t>(ppl, 64);
  size_t n = ctas_for(ppl, sh);
  while (n > slots && n < 3 * slots && ppl < 64) n = ctas_for(++ppl, sh);
  return sh;
}

int prepare_pl_scratch(mcl3dl_engine* eng, DeviceCtx& c, size_t P, const PlShape& sh, cudaStream_t st)
{
  const size_t groups = (P + 31) / 32;
  int rc = reserve(eng, c.d_partial, std::max<size_t>(P, 1) * sh.cb * 12);
  if (rc != MCL3DL_OK)
    return rc;
  return reserve_zeroed(eng, c.d_tickets, std::max<size_t>(groups * 4, 4096), st);
}

int launch_beam_pl(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* scan, size_t N,
                   const float* origins, int n_origins, mcl3dl_result* out, uint8_t* status, int lik_defaults, cudaStream_t st,
                   const RecordSink& sink)
{
  const PlShape sh = pick_pl_shape(P, N, c.sm_count);
  int rc = prepare_pl_scratch(eng, c, P, sh, st);
  if (rc != MCL3DL_OK)
    return rc;
  const int gpc = kPlWarps / sh.cpg;
  const int groups = static_cast<int>(((P + 31) / 32 + gpc - 1) / gpc);
  const size_t smem = static_cast<size_t>(kPlWarps) * sh.ppl * 16;
  const auto kernel = eng->beam.use_raycast_using_dda ? beam_kernel_pl<false> : beam_kernel_pl<true>;
  CK(launch(eng, kernel, groups * sh.cb, kBlockThreads, smem, st, poses, static_cast<int>(P), reinterpret_cast<const float4*>(scan),
            static_cast<int>(N), origins, c.dda, c.kd, c.nn, out, status, lik_defaults, c.stats_ptr(), sh,
            static_cast<uint32_t*>(c.d_partial.p), static_cast<unsigned int*>(c.d_tickets.p), sink));
  return MCL3DL_OK;
}

int launch_beam_dq(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* scan, size_t N,
                   const float* origins, mcl3dl_result* out, uint8_t* status, int lik_defaults, cudaStream_t st, const RecordSink& sink)
{
  const size_t groups = (P + 31) / 32;
  const int grid = c.sm_count * 4;  // the resident CTAs (64 registers)
  const size_t warps = static_cast<size_t>(grid) * kPlWarps;
  // ~4 items per resident warp so that the queue can balance, 1..16 rays per item
  size_t ppl = eng->beam_dq_ppl ? static_cast<size_t>(eng->beam_dq_ppl) : (N * groups + 4 * warps - 1) / (4 * warps);
  ppl = std::min<size_t>(std::max<size_t>(ppl, 1), 16);
  const int n_chunks = static_cast<int>(std::max<size_t>((N + ppl - 1) / ppl, 1));
  int rc;
  if ((rc = reserve_zeroed(eng, c.d_tally, std::max<size_t>(P, 1) * 12, st)) ||
      (rc = reserve_zeroed(eng, c.d_tickets, std::max<size_t>(groups * 4, 4096), st)) ||
      (rc = reserve_zeroed(eng, c.d_queue, 256, st)))
    return rc;
  const auto kernel = eng->beam.use_raycast_using_dda ? beam_kernel_dq<false> : beam_kernel_dq<true>;
  CK(launch(eng, kernel, grid, kBlockThreads, 0, st, poses, static_cast<int>(P), reinterpret_cast<const float4*>(scan),
            static_cast<int>(N), origins, c.dda, c.kd, c.nn, out, status, lik_defaults, c.stats_ptr(), static_cast<int>(ppl),
            n_chunks, static_cast<uint32_t*>(c.d_tally.p), static_cast<unsigned int*>(c.d_tickets.p),
            static_cast<unsigned int*>(c.d_queue.p), sink));
  return MCL3DL_OK;
}

int launch_lik(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* scan, size_t N,
               mcl3dl_result* out, int beam_defaults, cudaStream_t st, const RecordSink& sink)
{
  if (eng->field_mode && c.nn.fld.cells)
    return launch_lik_field(eng, c, poses, P, scan, N, out, beam_defaults, st, sink);
  if (c.nn.field.dir)
    return launch_lik_nf(eng, c, poses, P, scan, N, out, beam_defaults, st, sink);
  const float4* s4 = reinterpret_cast<const float4*>(scan);
  const int p = static_cast<int>(P), n = static_cast<int>(N);
  return with_tpp<32>(pick_tpp(P, N, c.sm_count), [&](auto tpp) {
    return launch_lik_wi_t<decltype(tpp)::value>(eng, c, poses, p, s4, n, out, beam_defaults, st, sink);
  });
}

int launch_beam(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* scan, size_t N,
                const float* origins, int n_origins, mcl3dl_result* out, uint8_t* status, int lik_defaults, cudaStream_t st,
                const RecordSink& sink)
{
  if (eng->beam_dq == 1 || (eng->beam_dq == 2 && P * N >= 262144))
    return launch_beam_dq(eng, c, poses, P, scan, N, origins, out, status, lik_defaults, st, sink);
  return launch_beam_pl(eng, c, poses, P, scan, N, origins, n_origins, out, status, lik_defaults, st, sink);
}

void derive_lik(mcl3dl_engine* eng)
{
  const float R = eng->lik.match_dist_min;
  eng->likdev.match_dist_min = R;
  eng->likdev.match_dist_flat = eng->lik.match_dist_flat;
  eng->likdev.match_weight = eng->lik.match_weight;
  eng->likdev.r2 = static_cast<float>(static_cast<double>(R) * static_cast<double>(R));
  eng->likdev.rpad = R * 1.0001f + 1e-6f;
}

void fill_dda_scalars(const mcl3dl_beam_params& b, DdaGridDev& g)
{
  g.grid = b.dda_grid_size;
  g.ray_angle_half = b.ray_angle_half;
  // ctor, raycast_using_dda.h:59 — y is used twice, as the reference does
  g.min_dist_thr_sq = b.map_grid_size[0] * b.map_grid_size[0] + b.map_grid_size[1] * b.map_grid_size[1] +
                      b.map_grid_size[1] * b.map_grid_size[1];
  g.hit_tolerance = static_cast<float>(b.hit_tolerance);
  g.hit_range_sq = b.hit_range_sq;
  g.sin_total_ref = b.sin_total_ref;
  g.beam_likelihood = b.beam_likelihood;
  g.beam_likelihood_min = b.beam_likelihood_min;
  g.filter_label_max = b.filter_label_max;
  g.short_only = b.add_penalty_short_only_mode ? 1 : 0;
}

void fill_kd_scalars(const mcl3dl_beam_params& b, KdRayDev& k)
{
  // RaycastUsingKDTree ctor takes floats (raycast_using_kdtree.h:48-55); refreshParameters passes the float params
  const float gx = static_cast<float>(b.map_grid_size[0]), gy = static_cast<float>(b.map_grid_size[1]),
              gz = static_cast<float>(b.map_grid_size[2]);
  const float gmin = std::min(gx, std::min(gy, gz)), gmax = std::max(gx, std::max(gy, gz));
  k.grid_min = gmin;
  k.hit_tolerance = static_cast<float>(b.hit_tolerance);
  k.r1 = static_cast<float>(std::sqrt(2.0) * gmax / 2.0);             // :83, narrowed by radiusSearch(const float radius)
  k.r2 = static_cast<float>(gmin * 2 + std::sqrt(2.0) * gmax / 2.0);  // :95
  k.r1_sq = static_cast<float>(static_cast<double>(k.r1) * static_cast<double>(k.r1));
  k.r2_sq = static_cast<float>(static_cast<double>(k.r2) * static_cast<double>(k.r2));
  k.r1_pad = k.r1 * 1.0001f + 1e-6f;
  k.r2_pad = k.r2 * 1.0001f + 1e-6f;
  k.sin_den = gmin * 2.0;  // :98
}

#if MCL3DL_NEAR_BITS
// Near field for search radius r over the rescaled map points (device_funcs.cuh: NearBitsDev).  k == 0, or a box that
// cannot be laid out within the byte cap, leaves `out.bits` null (the searches then run unscreened).
// first > 0: the bits of points [0, first) are already in `buf`, laid out for the same box (an append): only the rest are
// added (a bit is an OR over points).
int build_near_field(mcl3dl_engine* eng, DeviceCtx& c, cudaStream_t st, const mcl3dl_point* pts, uint32_t n, uint32_t first,
                     float wx, float wy, float wz, float r, int k, const float sc_min[3], const float sc_max[3], DevBuf& buf,
                     NearBitsDev& out, int slot)
{
  out = NearBitsDev{};
  eng->near_info_k[slot] = 0;
  eng->near_info_bytes[slot] = 0;
  NearBitsDev f{};
  if (k <= 0 || !near_layout(f, r, k, sc_min, sc_max, eng->near_max_bytes))
    return MCL3DL_OK;
  const size_t bytes = static_cast<size_t>(f.pitch) * f.ny * f.nz * 4;
  int rc = reserve(eng, buf, bytes);
  if (rc != MCL3DL_OK)
    return rc;
  if (first == 0)
    CK(cudaMemsetAsync(buf.p, 0, bytes, st));
  CK(launch(eng, near_mark_kernel, (n - first + 255) / 256, 256, 0, st, pts + first, n - first, wx, wy, wz, f,
            static_cast<uint32_t*>(buf.p), k));
  f.bits = static_cast<const uint32_t*>(buf.p);
  out = f;
  c.map_bytes += bytes;
  eng->near_info_k[slot] = k;
  eng->near_info_bytes[slot] = bytes;
  return MCL3DL_OK;
}
#endif

// NN field (device_funcs.cuh: NnFieldDev) over the finished CSR grid g.  Leaves g.field.dir null when the field is
// switched off, cannot be laid out, or would exceed the byte cap: the CSR-window kernels then serve the searches.
int build_nn_field(mcl3dl_engine* eng, DeviceCtx& c, cudaStream_t st, const mcl3dl_point* pts, uint32_t n, NnGridDev& g,
                   float radius, const float sc_min[3], const float sc_max[3])
{
  eng->nnf_bytes = eng->nnf_cands = eng->nnf_overflow_cells = eng->nnf_wide_cells = 0;
  NearBitsDev lay{};
  // the lattice of a k = 2 near field for this radius: fine edge 1.01 * radius / 2, origin 2.5 voxels below the box
  if (!near_layout(lay, radius, 2, sc_min, sc_max, size_t(1) << 40))
    return MCL3DL_OK;
  NnFieldDev f{};
  f.nx = lay.nx;
  f.ny = lay.ny;
  f.nz = lay.nz;
  f.cnx = (lay.nx + 1) / 2;
  f.cny = (lay.ny + 1) / 2;
  f.cnz = (lay.nz + 1) / 2;
  f.ox = lay.ox;
  f.oy = lay.oy;
  f.oz = lay.oz;
  f.inv_e = lay.inv_cell;
  f.e = 1.0f / lay.inv_cell;
  f.radius = radius;
  float ext = 0.0f;
  for (int k = 0; k < 3; ++k) ext = std::max(ext, std::max(std::fabs(sc_min[k]), std::fabs(sc_max[k])) + 4.0f * f.e);
  f.pad = 0.01f * f.e + 16.0f * std::numeric_limits<float>::epsilon() * ext;
  const size_t n_cells = static_cast<size_t>(f.cnx) * f.cny * f.cnz;
  const size_t bits_bytes = static_cast<size_t>(lay.pitch) * lay.ny * lay.nz * 4;
  if (n_cells >= (size_t(1) << 31) || n_cells * 8 + bits_bytes > eng->nnf_max_bytes)
    return MCL3DL_OK;
  DevBuf d_bits, d_tot, d_tmp;
  int rc = MCL3DL_OK;
  const uint32_t wide_cap = static_cast<uint32_t>(std::min<size_t>(n_cells, size_t(1) << 18));
  const size_t sum_at = (n_cells + 5) & ~size_t(1);  // 64-bit grand total, 8-byte aligned behind the tail words
  if ((rc = reserve(eng, d_bits, bits_bytes)) || (rc = reserve(eng, d_tot, (sum_at + 2) * 4)) ||
      (rc = reserve(eng, c.nnf_dir, n_cells * sizeof(uint2))) || (rc = reserve(eng, c.nnf_wide, static_cast<size_t>(wide_cap) * sizeof(uint4))))
    return rc;
  CK(cudaMemsetAsync(d_bits.p, 0, bits_bytes, st));
  CK(launch(eng, near_mark_kernel, (n + 255) / 256, 256, 0, st, pts, n, g.wx, g.wy, g.wz, lay, static_cast<uint32_t*>(d_bits.p), 2));
  const unsigned blocks = static_cast<unsigned>((n_cells * 8 + 255) / 256);
  uint2* dir = static_cast<uint2*>(c.nnf_dir.p);
  uint32_t* tot = static_cast<uint32_t*>(d_tot.p);
  CK(cudaMemsetAsync(tot + n_cells, 0, 16, st));  // [n_cells]: scan tail, [n_cells + 2] wide cells, [n_cells + 3] overflow cells
  f.wide = static_cast<const uint4*>(c.nnf_wide.p);
  CK(launch(eng, nnf_count_kernel, blocks, 256, 0, st, g, f, static_cast<const uint32_t*>(d_bits.p), lay.pitch, dir, tot, nullptr,
            n_cells, static_cast<uint4*>(c.nnf_wide.p), wide_cap, tot + n_cells + 2));
  // exclusive scan of the per-cell totals (in place); the grand total sizes the candidate array.  A candidate index
  // must stay below 2^31 (bit 31 of a directory entry marks wide / overflow cells): the total is first summed in 64 bits.
  cub::TransformInputIterator<unsigned long long, WidenU32, const uint32_t*> wide_in(tot, WidenU32());
  unsigned long long* d_sum = reinterpret_cast<unsigned long long*>(tot + sum_at);
  const auto scan = [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, tot, tot, static_cast<int>(n_cells + 1), st); };
  const auto sum = [&](void* t, size_t& b) { return cub::DeviceReduce::Sum(t, b, wide_in, d_sum, static_cast<int>(n_cells), st); };
  CK(cub_reserve(d_tmp, scan, sum));
  CK(cub_call(eng, d_tmp, sum));
  unsigned long long sum64 = 0;
  CK(cudaMemcpyAsync(&sum64, d_sum, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (sum64 >= (1ull << 31))
  {
    c.nnf_dir = DevBuf();
    c.nnf_wide = DevBuf();
    return MCL3DL_OK;
  }
  CK(cub_call(eng, d_tmp, scan));
  uint32_t tail[4] = {0, 0, 0, 0};
  CK(cudaMemcpyAsync(tail, tot + n_cells, sizeof(tail), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const uint32_t total = tail[0];
  eng->nnf_wide_cells = std::min<uint32_t>(tail[2], wide_cap);
  eng->nnf_overflow_cells = tail[3];
  const size_t cand_bytes = static_cast<size_t>(total) * sizeof(float4);
  if (n_cells * 8 + cand_bytes > eng->nnf_max_bytes)
  {
    c.nnf_dir = DevBuf();
    c.nnf_wide = DevBuf();
    return MCL3DL_OK;
  }
  if ((rc = reserve(eng, c.nnf_cand, std::max<size_t>(cand_bytes, 16))))
    return rc;
  CK(launch(eng, nnf_base_kernel, static_cast<unsigned>((n_cells + 255) / 256), 256, 0, st, dir, tot, 0u, nullptr, n_cells,
            static_cast<uint4*>(c.nnf_wide.p)));
  CK(launch(eng, nnf_fill_kernel, blocks, 256, 0, st, g, f, static_cast<const uint32_t*>(d_bits.p), lay.pitch, dir,
            static_cast<float4*>(c.nnf_cand.p), nullptr, n_cells));
  CK(cudaStreamSynchronize(st));
  f.dir = dir;
  f.cand = static_cast<const float4*>(c.nnf_cand.p);
  g.field = f;
  eng->nnf_bytes = n_cells * 8 + cand_bytes + static_cast<size_t>(wide_cap) * sizeof(uint4);
  eng->nnf_cands = total;
  c.nnf_cand_used = total;
  c.nnf_wide_used = std::min<uint32_t>(tail[2], wide_cap);
  c.nnf_wide_cap = wide_cap;
  c.map_bytes += eng->nnf_bytes;
  return MCL3DL_OK;
}

// NN field after an append that left every lattice as it was (same boxes, same parameters), over the re-sorted CSR grid
// g: only the directory cells an appended point pts[n_before..n) can reach are re-selected (nnf_mark_append), with the
// count / base / fill kernels of the build over that list; their new lists go after the candidates already placed, their
// new wide entries after the used ones.  The old lists become dead space.  The first append that needs room grows the
// candidate array; done = false when the lists or the wide entries do not fit, or the cap (MCL3DL_NNF_MAX_MB) would be
// exceeded: the caller then rebuilds the field, which compacts.
int update_nn_field(mcl3dl_engine* eng, DeviceCtx& c, cudaStream_t st, const mcl3dl_point* pts, uint32_t n_before, uint32_t n,
                    NnGridDev& g, const float sc_min[3], const float sc_max[3], bool& done, uint64_t& reselected)
{
  done = false;
  NnFieldDev f = c.nn.field;  // lattice, pad and radius are those of the staged map
  NearBitsDev lay{};
  if (!f.dir || !near_layout(lay, f.radius, 2, sc_min, sc_max, size_t(1) << 40))
    return MCL3DL_OK;
  const size_t n_cells = static_cast<size_t>(f.cnx) * f.cny * f.cnz;
  const uint32_t n_new = n - n_before;
  // list capacity: the directory cells one point can mark, per axis (nnf_mark_append's voxel interval, halved, + 2)
  const double w = static_cast<double>(static_cast<float>(0.5 * f.e + f.pad + f.radius * 1.00001 + 1e-7) * 1.001f + 1e-5f);
  const size_t per_axis = static_cast<size_t>((1.0 / g.inv_cell + 2.0 * w) / f.e + 7.0) / 2 + 2;
  const size_t list_cap = std::min(n_cells, static_cast<size_t>(n_new) * per_axis * per_axis * per_axis);
  const size_t bits_bytes = static_cast<size_t>(lay.pitch) * lay.ny * lay.nz * 4;
  const size_t mark_words = (n_cells + 31) / 32;
  DevBuf d_bits, d_mark, d_list, d_tot, d_cnt, d_tmp;
  int rc = MCL3DL_OK;
  if ((rc = reserve(eng, d_bits, bits_bytes)) || (rc = reserve(eng, d_mark, mark_words * 4)) ||
      (rc = reserve(eng, d_list, list_cap * 4)) || (rc = reserve(eng, d_tot, (list_cap + 1) * 4)) ||
      (rc = reserve(eng, d_cnt, 8 * 4)))
    return rc;
  uint32_t* cnt = static_cast<uint32_t*>(d_cnt.p);  // [0..4] nnf_count_kernel's counters, [5] marked cells
  uint32_t* list = static_cast<uint32_t*>(d_list.p);
  uint32_t* tot = static_cast<uint32_t*>(d_tot.p);
  // the field's k = 2 near field of the whole map, as the build makes it
  CK(cudaMemsetAsync(d_bits.p, 0, bits_bytes, st));
  CK(launch(eng, near_mark_kernel, (n + 255) / 256, 256, 0, st, pts, n, g.wx, g.wy, g.wz, lay, static_cast<uint32_t*>(d_bits.p), 2));
  CK(cudaMemsetAsync(d_mark.p, 0, mark_words * 4, st));
  const uint32_t init[8] = {c.nnf_wide_used, 0, 0, 0, 0, 0, 0, 0};
  CK(cudaMemcpyAsync(cnt, init, sizeof(init), cudaMemcpyHostToDevice, st));
  CK(launch(eng, nnf_mark_kernel, (n_new + 255) / 256, 256, 0, st, pts + n_before, n_new, g, f, static_cast<uint32_t*>(d_mark.p),
            list, static_cast<uint32_t>(list_cap), cnt + 5));
  uint32_t n_list = 0;
  CK(cudaMemcpyAsync(&n_list, cnt + 5, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (n_list > list_cap)
    return MCL3DL_OK;
  reselected = n_list;
  if (n_list == 0)
  {
    g.field = f;
    c.map_bytes += eng->nnf_bytes;
    done = true;
    return MCL3DL_OK;
  }
  uint2* dir = const_cast<uint2*>(f.dir);
  CK(cudaMemsetAsync(tot + n_list, 0, 4, st));
  const unsigned blocks = static_cast<unsigned>((static_cast<size_t>(n_list) * 8 + 255) / 256);
  CK(launch(eng, nnf_count_kernel, blocks, 256, 0, st, g, f, static_cast<const uint32_t*>(d_bits.p), lay.pitch, dir, tot, list,
            n_list, static_cast<uint4*>(c.nnf_wide.p), c.nnf_wide_cap, cnt));
  // at most 8 x 41 candidates per listed cell, fewer than 2^31 listed: the sum is taken in 64 bits
  cub::TransformInputIterator<unsigned long long, WidenU32, const uint32_t*> wide_in(tot, WidenU32());
  DevBuf d_sum;
  if ((rc = reserve(eng, d_sum, 8)))
    return rc;
  unsigned long long* sum = static_cast<unsigned long long*>(d_sum.p);
  const auto scan = [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, tot, tot, static_cast<int>(n_list + 1), st); };
  const auto reduce = [&](void* t, size_t& b) { return cub::DeviceReduce::Sum(t, b, wide_in, sum, static_cast<int>(n_list), st); };
  CK(cub_reserve(d_tmp, scan, reduce));
  CK(cub_call(eng, d_tmp, reduce));
  uint32_t h_cnt[5];
  unsigned long long added = 0;
  CK(cudaMemcpyAsync(h_cnt, cnt, sizeof(h_cnt), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(&added, sum, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const size_t need = c.nnf_cand_used + added;  // candidates placed once the new lists are in
  const size_t live = eng->nnf_cands - h_cnt[2] + added;
  if (h_cnt[0] > c.nnf_wide_cap || need >= (size_t(1) << 31))
    return MCL3DL_OK;  // (the directory entries the count pass rewrote are rebuilt with the rest)
  const size_t wide_bytes = static_cast<size_t>(c.nnf_wide_cap) * sizeof(uint4);
  if (need * sizeof(float4) > c.nnf_cand.cap)
  {
    // grow once, with room for more appends; not while dead lists would outweigh the live ones (rebuild then)
    const size_t cap = need + live / 4;
    if (need - live > live || n_cells * 8 + cap * sizeof(float4) + wide_bytes > eng->nnf_max_bytes)
      return MCL3DL_OK;
    DevBuf grown;
    if ((rc = reserve(eng, grown, cap * sizeof(float4))))
      return rc;
    CK(cudaMemcpyAsync(grown.p, c.nnf_cand.p, c.nnf_cand_used * sizeof(float4), cudaMemcpyDeviceToDevice, st));
    c.nnf_cand = std::move(grown);
    eng->nnf_bytes = n_cells * 8 + cap * sizeof(float4) + wide_bytes;
  }
  CK(cub_call(eng, d_tmp, scan));
  f.cand = static_cast<const float4*>(c.nnf_cand.p);
  CK(launch(eng, nnf_base_kernel, (n_list + 255) / 256, 256, 0, st, dir, tot, static_cast<uint32_t>(c.nnf_cand_used), list, n_list,
            static_cast<uint4*>(c.nnf_wide.p)));
  CK(launch(eng, nnf_fill_kernel, blocks, 256, 0, st, g, f, static_cast<const uint32_t*>(d_bits.p), lay.pitch, dir,
            static_cast<float4*>(c.nnf_cand.p), list, n_list));
  CK(cudaStreamSynchronize(st));
  eng->nnf_cands = live;
  eng->nnf_overflow_cells = eng->nnf_overflow_cells - h_cnt[3] + h_cnt[1];
  eng->nnf_wide_cells = eng->nnf_wide_cells - h_cnt[4] + (h_cnt[0] - c.nnf_wide_used);
  c.nnf_cand_used = need;
  c.nnf_wide_used = h_cnt[0];
  g.field = f;
  c.map_bytes += eng->nnf_bytes;
  done = true;
  return MCL3DL_OK;
}

// Build both grids on one device from the map points in d_pts (device memory, map order, n points, written on c.stream).
// On success the points become the context's raw_pts: the map stays on the device, so that mcl3dl_map_append uploads only
// the appended points.
//
// n_before > 0: d_pts is the staged map followed by appended points.  When the appended points leave both bounding boxes
// as they were, every lattice is unchanged: the grids are re-sorted, the near fields get the new points' bits and the NN
// field re-selects only the cells the new points reach (update_nn_field); `reselected` counts its re-selected cells
// (all of them on a full build) and `incremental` says which path ran.
// CSR order of a grid, once its key kernel has written the (cell, point) pairs to keys[0] / vals[0] and the per-cell
// counts to cell_start[1 .. cells]: the pairs sorted by cell into keys[1] / vals[1] (stable: input order inside a cell),
// then the inclusive scan that turns the counts into each cell's first index.  tmp: cub scratch.
int sort_csr(mcl3dl_engine* eng, cudaStream_t st, uint32_t n, size_t cells, uint32_t* cell_start, uint32_t* const keys[2],
             uint32_t* const vals[2], DevBuf& tmp)
{
  int end_bit = 1;
  while ((size_t(1) << end_bit) < cells && end_bit < 32) ++end_bit;
  const auto sort = [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(t, b, keys[0], keys[1], vals[0], vals[1], n, 0, end_bit, st);
  };
  const auto scan = [&](void* t, size_t& b) {
    return cub::DeviceScan::InclusiveSum(t, b, cell_start, cell_start, static_cast<int>(cells + 1), st);
  };
  CK(cub_reserve(tmp, sort, scan));
  CK(cub_call(eng, tmp, sort));
  CK(cub_call(eng, tmp, scan));
  return MCL3DL_OK;
}

// Lattice of a likelihood-style search grid with edge `cell` over the rescaled bounding box [sc_min, sc_max]: origin half
// a cell below the minimum, one spare cell above.  false: 2^31 cells or more.
bool nn_lattice(float cell, const float sc_min[3], const float sc_max[3], NnGridDev& g, size_t& cells)
{
  g.inv_cell = 1.0f / cell;
  int64_t total = 1;
  int dims[3];
  float org[3];
  for (int k = 0; k < 3; ++k)
  {
    org[k] = sc_min[k] - 0.5f * cell;
    dims[k] = static_cast<int>(std::floor((static_cast<double>(sc_max[k]) - org[k]) / cell)) + 2;
    total *= dims[k];
  }
  if (total >= (int64_t(1) << 31))
    return false;
  g.nx = dims[0];
  g.ny = dims[1];
  g.nz = dims[2];
  g.ox = org[0];
  g.oy = org[1];
  g.oz = org[2];
  cells = static_cast<size_t>(total);
  return true;
}

// The CSR of a likelihood-style grid g (lattice and dist_weight set) over pts[0..n): cell_start (cells + 1 entries) and
// the rescaled points in cell order, w = the point's index (nn_key_kernel / sort_csr / nn_gather_kernel).  keys / vals:
// two arrays of n each; tmp: cub scratch.
int build_nn_csr(mcl3dl_engine* eng, cudaStream_t st, const mcl3dl_point* pts, uint32_t n, const NnGridDev& g, size_t cells,
                 uint32_t* const keys[2], uint32_t* const vals[2], DevBuf& tmp, uint32_t* cell_start, float4* out)
{
  const int nb = static_cast<int>((static_cast<size_t>(n) + 255) / 256);
  CK(cudaMemsetAsync(cell_start, 0, (cells + 1) * 4, st));
  CK(launch(eng, nn_key_kernel, nb, 256, 0, st, pts, n, g, keys[0], vals[0], cell_start));
  if (int rc = sort_csr(eng, st, n, cells, cell_start, keys, vals, tmp))
    return rc;
  CK(launch(eng, nn_gather_kernel, nb, 256, 0, st, pts, n, vals[1], g.wx, g.wy, g.wz, out));
  return MCL3DL_OK;
}

// Cell edge of the likelihood search grid.  The window (q -/+ rpad) must span at most 3 cells per axis: cell edge
// strictly above rpad (1 % margin: the float cell function can be off by ~1e-7 x cells-per-axis, and the kernels rely on
// <= 3).
float lik_cell(const mcl3dl_engine* eng)
{
  return std::max(eng->lik.match_dist_min * eng->nn_cell_factor, eng->likdev.rpad * 1.01f);
}

// The likelihood search grid over pts[0..n) in lattice g (weights, dimensions and origin set; `cells` cells of edge
// `cell`) over the rescaled box [sc_min, sc_max]: its CSR, near field, NN field or window table, and the KD-tree
// raycaster's near field.  pts is the whole map, or the points of a map window: then idx gives each one's map index,
// which the gathered float4.w must carry (the KD caster's colliding point and the match output read raw_pts by it), and
// n may be 0.  keys / vals: two arrays of n each; tmp: cub scratch; n_before, first, reselected and incremental are
// build_map_on_device's.  The bytes staged are added to c.map_bytes.
int build_search(mcl3dl_engine* eng, DeviceCtx& c, cudaStream_t st, const mcl3dl_point* pts, uint32_t n32, size_t n_before,
                 uint32_t first, const float sc_min[3], const float sc_max[3], NnGridDev g, size_t cells, float cell,
                 uint32_t* const keys[2], uint32_t* const vals[2], DevBuf& d_tmp, const uint32_t* idx, uint64_t& reselected,
                 bool& incremental)
{
  int rc = MCL3DL_OK;
  const size_t n = n32;
  const float wx = g.wx, wy = g.wy, wz = g.wz;
  if ((rc = reserve(eng, c.nn_cell_start, (cells + 1) * 4)) || (rc = reserve(eng, c.nn_pts, std::max<size_t>(n, 1) * 16)))
    return rc;
  uint32_t* cell_start = static_cast<uint32_t*>(c.nn_cell_start.p);
  if (n32 == 0)
    CK(cudaMemsetAsync(cell_start, 0, (cells + 1) * 4, st));
  else if ((rc = build_nn_csr(eng, st, pts, n32, g, cells, keys, vals, d_tmp, cell_start, static_cast<float4*>(c.nn_pts.p))))
    return rc;
  if (idx && n32)
    CK(launch(eng, window_reindex_kernel, (n32 + 255) / 256, 256, 0, st, static_cast<float4*>(c.nn_pts.p), n32, idx));
  g.cell_start = cell_start;
  g.pts = static_cast<const float4*>(c.nn_pts.p);
#if MCL3DL_NEAR_BITS
  if (n32 && (rc = build_near_field(eng, c, st, pts, n32, first, wx, wy, wz, eng->likdev.rpad, eng->near_k, sc_min, sc_max, c.near_lik,
                                    g.near, 0)))
    return rc;
#endif
  // NN field: exact for the likelihood radius and, with the KD-tree raycaster, for its marching radius as well
  {
    float radius = eng->likdev.rpad;
    if (eng->has_beam && !eng->beam.use_raycast_using_dda)
    {
      KdRayDev tmp{};
      fill_kd_scalars(eng->beam, tmp);
      // the marching search always; the second (sin_angle_) search as well when asked for — it runs once per colliding
      // ray, through the CSR window search otherwise (a wider field means longer candidate lists for every query)
      radius = std::max(radius, eng->nnf_kd_r2 ? tmp.r2_pad : tmp.r1_pad);
    }
    g.field = NnFieldDev{};
    bool done = false;
    // (the field's radius follows the beam params, which set_params may have changed since the field was built)
    if (incremental && eng->nnf && radius == c.nn.field.radius &&
        (rc = update_nn_field(eng, c, st, pts, static_cast<uint32_t>(n_before), n32, g, sc_min, sc_max, done, reselected)))
      return rc;
    if (!done)
    {
      incremental = false;
      if (n_before > 0 || idx)
        c.nnf_cand = DevBuf();  // the rebuild compacts: no dead lists, no room kept from earlier appends
      if (n32 && eng->nnf && (rc = build_nn_field(eng, c, st, pts, n32, g, radius, sc_min, sc_max)))
        return rc;
      if (g.field.dir)
        reselected = static_cast<uint64_t>(g.field.cnx) * g.field.cny * g.field.cnz;
    }
  }
  // window table of the CSR-window kernel (lik_kernel_wi): only when the field is not staged
  size_t row3_total = 0;
  g.nyp = (g.ny + 4) & ~1;  // even pitch with room for the 4-entry fetch starting at (ly & ~1)
  if (!g.field.dir)
  {
    row3_total = static_cast<size_t>(g.nz) * g.nx * g.nyp;
    if ((rc = reserve(eng, c.nn_row3, (row3_total + 2) * sizeof(uint2))))
      return rc;
    g.row3 = static_cast<const uint2*>(c.nn_row3.p);
    CK(launch(eng, nn_row3_kernel, static_cast<unsigned>((row3_total + 255) / 256), 256, 0, st, g, static_cast<uint2*>(c.nn_row3.p),
              row3_total));
  }
  else
  {
    c.nn_row3 = DevBuf();
    g.row3 = nullptr;
  }
  c.nn = g;
  c.map_bytes += (cells + 1) * 4 + n * 16 + row3_total * sizeof(uint2);
  eng->info.nn_dims[0] = g.nx;
  eng->info.nn_dims[1] = g.ny;
  eng->info.nn_dims[2] = g.nz;
  eng->info.nn_cell = cell;
  eng->info.nn_origin[0] = g.ox;
  eng->info.nn_origin[1] = g.oy;
  eng->info.nn_origin[2] = g.oz;
  // the KD-tree raycaster's near field (its scalars are set)
  if (eng->has_beam && !eng->beam.use_raycast_using_dda)
  {
#if MCL3DL_NEAR_BITS
    // (set_params may have widened the marching radius since the field was built: then it is built anew)
    c.kd.near = NearBitsDev{};
    if (n32 && (rc = build_near_field(eng, c, st, pts, n32, c.near_kd_r == c.kd.r1_pad ? first : 0u, wx, wy, wz, c.kd.r1_pad,
                                      eng->near_kd_k, sc_min, sc_max, c.near_kd, c.kd.near, 1)))
      return rc;
    c.near_kd_r = c.kd.r1_pad;
#endif
  }
  return MCL3DL_OK;
}

int build_map_on_device(mcl3dl_engine* eng, DeviceCtx& c, DevBuf& d_pts, size_t n, size_t n_before, uint64_t& reselected,
                        bool& incremental)
{
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = c.stream;
  cudaEvent_t e0 = c.ev[0], e1 = c.ev[1];  // build time: the per-update timing events, unused between calls
  DevBuf d_bbox, d_keys[2], d_vals[2], d_tmp;  // keys / values: [0] per point, [1] sorted by cell
  int rc = MCL3DL_OK;
  const uint32_t n32 = static_cast<uint32_t>(n);
  const int tb = 256;
  const int nb = static_cast<int>((n + tb - 1) / tb);
  if ((rc = reserve(eng, d_bbox, 12 * sizeof(uint32_t))) || (rc = reserve(eng, d_keys[0], n * 4)) ||
      (rc = reserve(eng, d_vals[0], n * 4)) || (rc = reserve(eng, d_keys[1], n * 4)) || (rc = reserve(eng, d_vals[1], n * 4)))
    return rc;
  CK(cudaEventRecord(e0, st));
  const mcl3dl_point* pts = static_cast<const mcl3dl_point*>(d_pts.p);
  uint32_t* const keys[2] = {static_cast<uint32_t*>(d_keys[0].p), static_cast<uint32_t*>(d_keys[1].p)};
  uint32_t* const vals[2] = {static_cast<uint32_t*>(d_vals[0].p), static_cast<uint32_t*>(d_vals[1].p)};

  // ---- bounding boxes (raw: pcl::getMinMax3D, raycast_using_dda.h:175; rescaled: likelihood grid)
  uint32_t h_bbox[12];
  for (int k = 0; k < 3; ++k)
  {
    h_bbox[k] = 0xffffffffu;
    h_bbox[3 + k] = 0u;
    h_bbox[6 + k] = 0xffffffffu;
    h_bbox[9 + k] = 0u;
  }
  CK(cudaMemcpyAsync(d_bbox.p, h_bbox, sizeof(h_bbox), cudaMemcpyHostToDevice, st));
  const float wx = eng->has_lik ? eng->lik.dist_weight[0] : 1.0f;
  const float wy = eng->has_lik ? eng->lik.dist_weight[1] : 1.0f;
  const float wz = eng->has_lik ? eng->lik.dist_weight[2] : 1.0f;
  CK(launch(eng, bbox_kernel, std::min(nb, c.sm_count * 8), tb, 0, st, pts, n, wx, wy, wz, static_cast<uint32_t*>(d_bbox.p)));
  CK(cudaMemcpyAsync(h_bbox, d_bbox.p, sizeof(h_bbox), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  float raw_min[3], raw_max[3], sc_min[3], sc_max[3];
  for (int k = 0; k < 3; ++k)
  {
    raw_min[k] = ord2f(h_bbox[k]);
    raw_max[k] = ord2f(h_bbox[3 + k]);
    sc_min[k] = ord2f(h_bbox[6 + k]);
    sc_max[k] = ord2f(h_bbox[9 + k]);
  }
  incremental = n_before > 0 && std::memcmp(h_bbox, c.map_box, sizeof(h_bbox)) == 0;
  std::memcpy(c.map_box, h_bbox, sizeof(h_bbox));
  const uint32_t first = incremental ? static_cast<uint32_t>(n_before) : 0u;  // near fields: bits of points [first, n)
  reselected = 0;
  c.map_bytes = 0;
  if (eng->has_beam && !eng->beam.use_raycast_using_dda)
    fill_kd_scalars(eng->beam, c.kd);

  // ---- likelihood search grid over the whole map, or, when its lattice is refused or exceeds MCL3DL_MAP_MAX_CELLS, a
  // windowed staging: the points and boxes are kept and the search structures wait for the first call's window
  const bool was_windowed = c.w_on;
  c.w_on = false;
  size_t search_bytes = 0;
  if (eng->has_lik)
  {
    NnGridDev g{};
    const float cell = lik_cell(eng);
    if (!(cell > 0.0f))
      return MCL3DL_ERR_INVALID_ARG;
    g.wx = wx;
    g.wy = wy;
    g.wz = wz;
    size_t cells = 0;
    if (!nn_lattice(cell, sc_min, sc_max, g, cells) || cells > eng->map_max_cells)
      c.w_on = true;
    else if ((rc = build_search(eng, c, st, pts, n32, n_before, first, sc_min, sc_max, g, cells, cell, keys, vals, d_tmp, nullptr,
                                reselected, incremental)))
      return rc;
    search_bytes = c.map_bytes;
  }
  if (c.w_on)
  {
    incremental = false;
    if (!was_windowed || !c.w_valid || n_before == 0)
    {
      // a new map, or nothing staged yet: the first call that reads the map builds its window (a window of an earlier
      // map indexes that map's points and was laid out for its parameters)
      c.w_valid = false;
      c.w_stale = false;
      c.w_box = WinBox{};
      if (n_before == 0)
      {
        c.w_rebuilds = 0;
        c.w_ms = 0.0;
      }
      c.nn = NnGridDev{};
      c.nn_cell_start = DevBuf();
      c.nn_pts = DevBuf();
      c.nn_row3 = DevBuf();
      c.nnf_dir = DevBuf();
      c.nnf_cand = DevBuf();
      c.nnf_wide = DevBuf();
      c.near_lik = DevBuf();
      c.near_kd = DevBuf();
      c.kd.near = NearBitsDev{};
      eng->nnf_bytes = eng->nnf_cands = eng->nnf_overflow_cells = eng->nnf_wide_cells = 0;
      for (int k = 0; k < 3; ++k)
      {
        eng->info.nn_dims[k] = 0;
        eng->info.nn_origin[k] = 0.0f;
      }
      eng->info.nn_cell = lik_cell(eng);
    }
    else
    {
      // an append to a windowed map: the window is rebuilt when an appended point lies inside it
      DevBuf d_cnt;
      if ((rc = reserve(eng, d_cnt, 4)) || (rc = reserve(eng, c.w_host, 64)))
        return rc;
      uint32_t* cnt = static_cast<uint32_t*>(d_cnt.p);
      CK(cudaMemsetAsync(cnt, 0, 4, st));
      const uint32_t n_new = static_cast<uint32_t>(n - n_before);
      if (n_new)
        CK(launch(eng, window_count_kernel, (n_new + 255) / 256, 256, 0, st, pts + n_before, n_new, c.w_box, cnt));
      CK(cudaMemcpyAsync(c.w_host.p, cnt, 4, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      // (stays stale when an earlier append, not yet followed by a call that reads the map, put points inside)
      c.w_stale = c.w_stale || *static_cast<const uint32_t*>(c.w_host.p) != 0;
      for (int k = 0; k < 3; ++k)
      {
        eng->info.nn_dims[k] = c.w_dims[k];
        eng->info.nn_origin[k] = c.w_org[k];
      }
      eng->info.nn_cell = lik_cell(eng);
    }
  }
  // ---- the raw points by original index (the KD-tree raycaster's colliding point; the chunk rule of
  // mcl3dl_match_output; the base of mcl3dl_map_append; a window's point list).  device_bytes counts them where the
  // models read them: with a likelihood grid.
  c.raw_pts = std::move(d_pts);
  if (eng->has_lik)
    c.map_bytes += n * 16;

  // ---- KD-tree raycaster: marches over the likelihood grid; needs the raw points by original index
  if (eng->has_beam && !eng->beam.use_raycast_using_dda)
  {
    if (!eng->has_lik)
      return MCL3DL_ERR_INVALID_ARG;
    fill_dda_scalars(eng->beam, c.dda);
    c.kd.raw_pts = static_cast<const float4*>(c.raw_pts.p);
  }
  // ---- DDA grid: updatePointCloud, raycast_using_dda.h:162-190
  if (eng->has_beam && eng->beam.use_raycast_using_dda)
  {
    DdaGridDev g{};
    fill_dda_scalars(eng->beam, g);
    if (!(g.grid > 0.0))
      return MCL3DL_ERR_INVALID_ARG;
    int64_t total = 1;
    int dims[3];
    for (int k = 0; k < 3; ++k)
    {
      // map_size_[i] = static_cast<size_t>((max_p_[i] - min_p_[i]) / dda_grid_size_) + 1  (:179)
      const float diff = raw_max[k] - raw_min[k];
      dims[k] = static_cast<int>(static_cast<size_t>(static_cast<double>(diff) / g.grid) + 1);
      total *= dims[k];
    }
    if (total >= (int64_t(1) << 31))  // `int point_total` (:176)
      return MCL3DL_ERR_TOO_LARGE;
    g.nx = dims[0];
    g.ny = dims[1];
    g.nz = dims[2];
    g.min_x = raw_min[0];
    g.min_y = raw_min[1];
    g.min_z = raw_min[2];
    g.max_x = raw_max[0];
    g.max_y = raw_max[1];
    g.max_z = raw_max[2];
    const size_t cells = static_cast<size_t>(total);
    const size_t occ_words = (cells + 31) / 32 + 1;
    if ((rc = reserve(eng, c.dda_cell_start, (cells + 2) * 4)) || (rc = reserve(eng, c.dda_occ, occ_words * 4)) ||
        (rc = reserve(eng, c.dda_pts, n * 16)))
      return rc;
    uint32_t* cell_start = static_cast<uint32_t*>(c.dda_cell_start.p);
    CK(cudaMemsetAsync(cell_start, 0, (cells + 2) * 4, st));
    CK(cudaMemsetAsync(c.dda_occ.p, 0, occ_words * 4, st));
    CK(launch(eng, dda_key_kernel, nb, tb, 0, st, pts, n32, g, keys[0], vals[0], cell_start, static_cast<uint32_t*>(c.dda_occ.p)));
    if ((rc = sort_csr(eng, st, n32, cells, cell_start, keys, vals, d_tmp)))
      return rc;
    CK(launch(eng, dda_gather_kernel, nb, tb, 0, st, pts, n32, vals[1], static_cast<float4*>(c.dda_pts.p)));
    g.occ = static_cast<const uint32_t*>(c.dda_occ.p);
    g.cell_start = cell_start;
    g.pts = static_cast<const float4*>(c.dda_pts.p);
    c.dda = g;
    c.map_bytes += (cells + 2) * 4 + occ_words * 4 + n * 16;
    for (int k = 0; k < 3; ++k) eng->info.dda_dims[k] = dims[k];
    for (int k = 0; k < 3; ++k)
    {
      eng->info.dda_min[k] = raw_min[k];
      eng->info.dda_max[k] = raw_max[k];
    }
  }
  CK(cudaEventRecord(e1, st));
  CK(cudaStreamSynchronize(st));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  eng->info.build_ms = std::max(eng->info.build_ms, static_cast<double>(ms));
  c.map_base = c.map_bytes - search_bytes;  // what a window rebuild keeps: the raw points and the DDA grid
  if (c.w_on && c.w_valid)
    c.map_bytes += c.w_bytes;
  eng->info.device_bytes = c.map_bytes;
  return MCL3DL_OK;
}

// ---- map window (window_funcs.cuh)
// Stage the search structures over the map points inside box `b` (raw space): the points are selected in map order, the
// grids are built over them exactly as over a whole map, with the lattice laid over the box, and each gathered point
// keeps its map index.  Points outside the box never enter a cell.
int build_window(mcl3dl_engine* eng, DeviceCtx& c, const WinBox& b)
{
  cudaStream_t st = c.stream;
  const size_t n = eng->n_points;
  const uint32_t n32 = static_cast<uint32_t>(n);
  const float w[3] = {eng->lik.dist_weight[0], eng->lik.dist_weight[1], eng->lik.dist_weight[2]};
  const float cell = lik_cell(eng);
  NnGridDev g{};
  float org[3];
  int dims[3];
  size_t cells = 0;
  if (!win_box_lattice(b, w, cell, dims, org, cells) || cells > eng->map_max_cells)
    return MCL3DL_ERR_TOO_LARGE;
  g.wx = w[0];
  g.wy = w[1];
  g.wz = w[2];
  g.inv_cell = 1.0f / cell;
  g.nx = dims[0];
  g.ny = dims[1];
  g.nz = dims[2];
  g.ox = org[0];
  g.oy = org[1];
  g.oz = org[2];
  DevBuf d_flags, d_pos, d_cnt, d_keys[2], d_vals[2], d_tmp;
  int rc;
  if ((rc = reserve(eng, d_flags, n * 4)) || (rc = reserve(eng, d_pos, n * 4)) || (rc = reserve(eng, d_cnt, 4)) ||
      (rc = reserve(eng, c.w_host, 64)))
    return rc;
  // the selection's flags and scan positions first: the window's point list is sized by their count
  CK(cudaEventRecord(c.ev_w0, st));
  const mcl3dl_point* raw = static_cast<const mcl3dl_point*>(c.raw_pts.p);
  uint32_t* flags = static_cast<uint32_t*>(d_flags.p);
  uint32_t* pos = static_cast<uint32_t*>(d_pos.p);
  uint32_t* cnt = static_cast<uint32_t*>(d_cnt.p);
  const int nb = static_cast<int>((n + 255) / 256);
  CK(launch(eng, window_flag_kernel, nb, 256, 0, st, raw, n32, b, flags));
  CK(cub_call(eng, d_tmp, [&](void* t, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(t, bytes, flags, pos, n32, st); }));
  CK(cudaEventRecord(c.ev_w1, st));
  uint32_t* h = static_cast<uint32_t*>(c.w_host.p);
  CK(cudaMemcpyAsync(h, pos + (n32 - 1), 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(h + 1, flags + (n32 - 1), 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  float ms_select = 0;
  CK(cudaEventElapsedTime(&ms_select, c.ev_w0, c.ev_w1));
  const uint32_t m = h[0] + h[1];
  const size_t mk = std::max<uint32_t>(m, 1u);
  // the point list and map indices at the window's size (a much smaller window gives the larger buffers back)
  if (c.w_pts.cap > 2 * mk * 16)
    c.w_pts = DevBuf();
  if (c.w_idx.cap > 2 * mk * 4)
    c.w_idx = DevBuf();
  if ((rc = reserve(eng, c.w_pts, mk * 16)) || (rc = reserve(eng, c.w_idx, mk * 4)) || (rc = reserve(eng, d_keys[0], mk * 4)) ||
      (rc = reserve(eng, d_keys[1], mk * 4)) || (rc = reserve(eng, d_vals[0], mk * 4)) || (rc = reserve(eng, d_vals[1], mk * 4)))
    return rc;
  CK(cudaEventRecord(c.ev_w0, st));
  CK(launch(eng, window_compact_kernel, nb, 256, 0, st, raw, flags, pos, n32, static_cast<mcl3dl_point*>(c.w_pts.p),
            static_cast<uint32_t*>(c.w_idx.p), cnt));
  uint32_t* const keys[2] = {static_cast<uint32_t*>(d_keys[0].p), static_cast<uint32_t*>(d_keys[1].p)};
  uint32_t* const vals[2] = {static_cast<uint32_t*>(d_vals[0].p), static_cast<uint32_t*>(d_vals[1].p)};
  float sc_min[3], sc_max[3];
  for (int k = 0; k < 3; ++k)
  {
    sc_min[k] = b.lo[k] * w[k];
    sc_max[k] = b.hi[k] * w[k];
  }
  c.w_valid = false;
  c.map_bytes = 0;
  uint64_t reselected = 0;
  bool incremental = false;
  if ((rc = build_search(eng, c, st, static_cast<const mcl3dl_point*>(c.w_pts.p), m, 0, 0u, sc_min, sc_max, g, cells, cell, keys, vals,
                         d_tmp, static_cast<const uint32_t*>(c.w_idx.p), reselected, incremental)))
    return rc;
  CK(cudaEventRecord(c.ev_w1, st));
  CK(cudaStreamSynchronize(st));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, c.ev_w0, c.ev_w1));
  c.w_bytes = c.map_bytes + mk * 20;  // + the window's point list and map indices
  c.map_bytes = c.map_base + c.w_bytes;
  eng->info.device_bytes = c.map_bytes;
  c.w_box = b;
  for (int k = 0; k < 3; ++k)
  {
    c.w_dims[k] = dims[k];
    c.w_org[k] = org[k];
  }
  c.w_valid = true;
  c.w_stale = false;
  c.w_rebuilds++;
  c.w_ms = static_cast<double>(ms_select) + ms;
  return MCL3DL_OK;
}

// The window check of one call that reads the map, on a windowed map, in two steps so that a multi-device call enqueues
// every device's reduction before it waits for any.  window_need enqueues on c.stream the reduction of the particles
// [poses, +P) with the scans and origins given (device pointers) and its 32-byte copy back; window_settle synchronises,
// forms the required box for the search `s` and rebuilds the window when the box is not inside it.  TOO_LARGE: the
// required box alone exceeds the cap (or is not finite); the staged window is left as it was.  A whole-staged map
// returns at once from both.
int window_need(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* a, size_t na,
                const mcl3dl_point* b, size_t nb, const float* org, size_t norg, const WinSearch& s,
                const mcl3dl_pose* host_pose = nullptr)
{
  c.w_pending = false;
  if (!c.w_on || (c.w_valid && !c.w_stale && !(s.r_scaled > 0.0f)))
    return MCL3DL_OK;  // (no search of this call reads the window: DDA beam only)
  cudaStream_t st = c.stream;
  int rc;
  if ((rc = reserve(eng, c.w_need, 64)) || (rc = reserve(eng, c.w_host, 64)))
    return rc;
  CK(cudaMemsetAsync(c.w_need.p, 0, sizeof(WinNeed), st));
  if (host_pose)  // one pose from the host: behind the reduction's block
  {
    static_assert(sizeof(WinNeed) + sizeof(mcl3dl_pose) <= 64, "pose slot");
    std::memcpy(static_cast<char*>(c.w_host.p) + sizeof(WinNeed), host_pose, sizeof(mcl3dl_pose));
    CK(cudaMemcpyAsync(static_cast<char*>(c.w_need.p) + sizeof(WinNeed), static_cast<char*>(c.w_host.p) + sizeof(WinNeed),
                       sizeof(mcl3dl_pose), cudaMemcpyHostToDevice, st));
    poses = reinterpret_cast<const mcl3dl_pose*>(static_cast<char*>(c.w_need.p) + sizeof(WinNeed));
    P = 1;
  }
  const size_t total = P + na + nb + norg;
  const int grid = static_cast<int>(std::max<size_t>(1, std::min<size_t>((total + 255) / 256, static_cast<size_t>(c.sm_count) * 8)));
  CK(launch(eng, window_need_kernel, grid, 256, 0, st, poses, static_cast<uint32_t>(P), a, static_cast<uint32_t>(na), b,
            static_cast<uint32_t>(nb), org, static_cast<uint32_t>(norg), static_cast<uint32_t*>(c.w_need.p)));
  CK(cudaMemcpyAsync(c.w_host.p, c.w_need.p, sizeof(WinNeed), cudaMemcpyDeviceToHost, st));
  c.w_pending = true;
  return MCL3DL_OK;
}

int window_settle(mcl3dl_engine* eng, DeviceCtx& c, const WinSearch& s)
{
  if (!c.w_pending)
    return MCL3DL_OK;
  c.w_pending = false;
  CK(cudaSetDevice(c.dev));
  CK(cudaStreamSynchronize(c.stream));
  WinNeed need;
  std::memcpy(&need, c.w_host.p, sizeof(need));
  if (!win_has_particles(need))
  {
    // no finite particle: no search can find a point, so any staged window serves; the first one sits at the map's corner
    if (c.w_valid)
      return MCL3DL_OK;
    for (int k = 0; k < 3; ++k)
    {
      need.pmax[k] = c.map_box[k];
      need.pmin_c[k] = ~c.map_box[k];
    }
  }
  const float w[3] = {eng->lik.dist_weight[0], eng->lik.dist_weight[1], eng->lik.dist_weight[2]};
  WinBox req;
  if (!win_required(need, s, w, req))
  {
    eng->err = "map window: the required box is not finite";
    return MCL3DL_ERR_TOO_LARGE;
  }
  if (c.w_valid && !c.w_stale && win_contains(c.w_box, req))
    return MCL3DL_OK;
  WinBox win;
  if (!win_choose(req, win_reach(need), w, lik_cell(eng), eng->map_max_cells, win))
  {
    eng->err = "map window: the particles' required box exceeds the lattice cap";
    return MCL3DL_ERR_TOO_LARGE;
  }
  return build_window(eng, c, win);
}

// Both steps, for a call on one device
int ensure_window(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* a, size_t na,
                  const mcl3dl_point* b, size_t nb, const float* org, size_t norg, const WinSearch& s,
                  const mcl3dl_pose* host_pose = nullptr)
{
  if (int rc = window_need(eng, c, poses, P, a, na, b, nb, org, norg, s, host_pose))
    return rc;
  return window_settle(eng, c, s);
}

// The searches of a measure call: the likelihood radius, and with a beam scan and the KD caster its second radius and march
WinSearch measure_search(const mcl3dl_engine* eng, const DeviceCtx& c, size_t n_lik, size_t n_beam)
{
  WinSearch s{0.0f, 0.0f, 0.0f};
  if (n_lik)
    s.r_scaled = eng->likdev.rpad;
  if (n_beam && !eng->beam.use_raycast_using_dda)
  {
    s.r_scaled = std::max(s.r_scaled, std::max(c.kd.r1_pad, c.kd.r2_pad));
    s.grid_min = c.kd.grid_min;
    s.hit_tolerance = c.kd.hit_tolerance;
  }
  return s;
}

// After a build: a field-mode volume of the previous map is stale; in field mode the new one is staged.
int restage_field(mcl3dl_engine* eng, DeviceCtx& c)
{
  c.fld_nodes_valid = false;
  c.fld_mem = DevBuf();
  c.fld_nodes = cudaPitchedPtr{};
  if (eng->field_mode && eng->has_lik && c.w_on)
    return MCL3DL_ERR_TOO_LARGE;  // the volume covers the whole map
  return eng->field_mode && eng->has_lik ? stage_field(eng, c, nullptr) : MCL3DL_OK;
}

// The buffers of one VoxelGrid pass: sort keys / values (x2, at least n each, reserved by the caller), the (voxel, label)
// keys of the vote (x2), voxel-head flags and their scan positions (at least n each, reserved by the caller), cub scratch
struct VoxelBufs
{
  DevBuf* keys[2];
  DevBuf* vals[2];
  DevBuf* key_label[2];
  DevBuf* flags;
  DevBuf* pos;
  DevBuf* tmp;
};

// pcl::VoxelGrid with leaf `leaf` over the device cloud in[0..n) (scan_kernels.cuh: the finite points' bounding box,
// the lattice and PCL's overflow rule of scan_voxel_lattice, stable sort by voxel key, sort of the (voxel, label) keys,
// one centroid per voxel in ascending voxel index).  done: the pass wrote the downsampled cloud to out and its size to
// *d_count; false when the cloud passes unfiltered (out and *d_count untouched).  With no finite point, done is true and
// nothing is written: the caller's zeroed count stands.  cap: the capacity the vote's keys are reserved for (>= n).
// runs (may be NULL): when the pass sorted, the voxel runs stay for the caller (map_intensity_kernel): b.keys[1] the
// sorted keys, b.vals[1] the input index in that order, b.flags the run heads, b.pos their output positions, and the
// run with key runs->nonfinite_key holds the non-finite points (no voxel).
struct VoxelRuns
{
  bool sorted = false;
  uint32_t nonfinite_key = 0;
};
int voxel_grid(mcl3dl_engine* eng, DeviceCtx& c, cudaStream_t st, const mcl3dl_point* in, uint32_t n, size_t cap, const float leaf[3],
               const VoxelBufs& b, mcl3dl_point* out, uint32_t* d_count, bool& done, VoxelRuns* runs = nullptr)
{
  done = false;
  if (runs)
    *runs = VoxelRuns{};
  int rc;
  const int nb = static_cast<int>((n + 255) / 256);
  // bounding box of the finite points -> VoxelGrid lattice and PCL's overflow rule (scan_voxel_lattice)
  uint32_t h_bbox[6] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u};
  if ((rc = reserve(eng, *b.tmp, 4096)))
    return rc;
  uint32_t* bb = static_cast<uint32_t*>(b.tmp->p);
  CK(cudaMemcpyAsync(bb, h_bbox, sizeof(h_bbox), cudaMemcpyHostToDevice, st));
  CK(launch(eng, scan_bbox_kernel, std::min(nb, c.sm_count * 8), 256, 0, st, in, n, bb));
  CK(cudaMemcpyAsync(h_bbox, bb, sizeof(h_bbox), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const float mn[3] = {ord2f(h_bbox[0]), ord2f(h_bbox[1]), ord2f(h_bbox[2])};
  const float mx[3] = {ord2f(h_bbox[3]), ord2f(h_bbox[4]), ord2f(h_bbox[5])};
  VoxelGridDev g{};
  int end_bit = 0;
  if (!(mn[0] <= mx[0]))
  {
    done = true;  // no finite point: the voxel pass skips every point, the downsampled cloud is empty
    return MCL3DL_OK;
  }
  if (!scan_voxel_lattice(leaf, mn, mx, g, end_bit))
    return MCL3DL_OK;
  if ((rc = reserve(eng, *b.key_label[0], cap * 8)) || (rc = reserve(eng, *b.key_label[1], cap * 8)))
    return rc;
  uint32_t *k0 = static_cast<uint32_t*>(b.keys[0]->p), *k1 = static_cast<uint32_t*>(b.keys[1]->p);
  uint32_t *v0 = static_cast<uint32_t*>(b.vals[0]->p), *v1 = static_cast<uint32_t*>(b.vals[1]->p);
  uint64_t *kl0 = static_cast<uint64_t*>(b.key_label[0]->p), *kl1 = static_cast<uint64_t*>(b.key_label[1]->p);
  uint32_t *fl = static_cast<uint32_t*>(b.flags->p), *ps = static_cast<uint32_t*>(b.pos->p);
  CK(launch(eng, scan_key_kernel, nb, 256, 0, st, in, n, g, k0, v0, kl0));
  // stable: input order inside a voxel
  const auto sort = [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, k0, k1, v0, v1, n, 0, end_bit, st); };
  // labels ascending inside a voxel
  const auto sort_kl = [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortKeys(t, b, kl0, kl1, n, 0, 32 + end_bit, st); };
  const auto scan = [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, fl, ps, n, st); };
  CK(cub_reserve(*b.tmp, sort, sort_kl, scan));
  CK(cub_call(eng, *b.tmp, sort));
  CK(cub_call(eng, *b.tmp, sort_kl));
  CK(launch(eng, scan_heads_kernel, nb, 256, 0, st, k1, n, fl));
  CK(cub_call(eng, *b.tmp, scan));
  CK(launch(eng, scan_centroid_kernel, nb, 256, 0, st, in, k1, v1, kl1, fl, ps, n, g.cells, out, d_count));
  done = true;
  if (runs)
    *runs = VoxelRuns{true, g.cells};
  return MCL3DL_OK;
}

// PointCloudSamplerWithNormal on the clipped cloud k (n points, grid ng / end_bit checked by the caller): the normals,
// neighbour counts and fixed-point weights into n_normals[k] / n_nb[k] / n_q[k], then the distinct weighted draws into
// n_out[k] (include/mcl3dl_b200.h: mcl3dl_scan_sample_with_normal).  *n_sample, *rounds and *draws as the info reports.
constexpr uint64_t kNsMaxDraws = uint64_t(1) << 32;  // the documented cap on the draws of one call and model
constexpr uint32_t kNsMaxRound = 1u << 22;           // draws per round, at most
int ns_sample_model(mcl3dl_engine* eng, DeviceCtx& c, int k, uint32_t n, const NsGridDev& ng, int end_bit, const float fpc[3],
                    double max_weight, double scale, uint32_t num, uint64_t seed, uint32_t* n_sample, uint32_t* rounds, uint64_t* draws)
{
  cudaStream_t st = c.stream;
  int rc;
  *n_sample = 0;
  *rounds = 0;
  *draws = 0;
  const size_t cap = std::max<size_t>(n, 1);
  if ((rc = reserve(eng, c.n_normals[k], cap * 12)) || (rc = reserve(eng, c.n_nb[k], cap * 4)) || (rc = reserve(eng, c.n_q[k], cap * 8)) ||
      (rc = reserve(eng, c.n_out[k], std::max<size_t>(std::min<size_t>(num, n), 1) * 16)))
    return rc;
  if (n == 0)
    return MCL3DL_OK;
  for (int b = 0; b < 2; ++b)
    if ((rc = reserve(eng, c.n_keys[b], cap * 4)) || (rc = reserve(eng, c.n_vals[b], cap * 4)))
      return rc;
  if ((rc = reserve(eng, c.n_spts, cap * 16)) || (rc = reserve(eng, c.n_cum, cap * 8)))
    return rc;
  const mcl3dl_point* clipped = static_cast<const mcl3dl_point*>(c.s_clip[k].p);
  uint32_t* word = static_cast<uint32_t*>(c.n_word.p);  // [0, 12) bounding boxes, [12 + k] finite normals, [14] carry
  uint32_t *k0 = static_cast<uint32_t*>(c.n_keys[0].p), *k1 = static_cast<uint32_t*>(c.n_keys[1].p);
  uint32_t *v0 = static_cast<uint32_t*>(c.n_vals[0].p), *v1 = static_cast<uint32_t*>(c.n_vals[1].p);
  mcl3dl_point* spts = static_cast<mcl3dl_point*>(c.n_spts.p);
  uint64_t* q = static_cast<uint64_t*>(c.n_q[k].p);
  uint64_t* cum = static_cast<uint64_t*>(c.n_cum.p);
  const int nb = static_cast<int>((n + 255) / 256);
  CK(launch(eng, ns_key_kernel, nb, 256, 0, st, clipped, n, ng.g, k0, v0));
  // stable: ascending index in a cell
  const auto sort = [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, k0, k1, v0, v1, n, 0, end_bit, st); };
  // exact: the total stays below 2^62
  const auto scan = [&](void* t, size_t& b) { return cub::DeviceScan::InclusiveSum(t, b, q, cum, static_cast<int>(n), st); };
  CK(cub_reserve(c.n_tmp, sort, scan));
  CK(cub_call(eng, c.n_tmp, sort));
  CK(launch(eng, ns_gather_kernel, nb, 256, 0, st, clipped, v1, n, spts));
  CK(launch(eng, ns_normal_kernel, static_cast<int>((n + 127) / 128), 128, 0, st, clipped, n, ng, k1, spts, fpc[0], fpc[1], fpc[2],
            max_weight, scale, static_cast<float*>(c.n_normals[k].p), static_cast<uint32_t*>(c.n_nb[k].p), q, word + 12 + k));
  CK(cub_call(eng, c.n_tmp, scan));
  mcl3dl_point* out = static_cast<mcl3dl_point*>(c.n_out[k].p);
  if (num == 0)
    return MCL3DL_OK;
  if (n <= num)  // the whole clipped cloud, in order
  {
    CK(cudaMemcpyAsync(out, clipped, static_cast<size_t>(n) * 16, cudaMemcpyDeviceToDevice, st));
    *n_sample = n;
    return MCL3DL_OK;
  }
  if ((rc = reserve(eng, c.n_first, cap * 8)))
    return rc;
  unsigned long long* first = static_cast<unsigned long long*>(c.n_first.p);
  CK(cudaMemsetAsync(first, 0xff, static_cast<size_t>(n) * 8, st));
  const uint64_t r0 = std::max<uint64_t>(2048, 2 * static_cast<uint64_t>(num));
  uint32_t carry = 0;
  uint64_t d0 = 0;
  while (carry < num && d0 < kNsMaxDraws)
  {
    const uint32_t cnt = static_cast<uint32_t>(std::min(std::min(r0 << std::min<uint32_t>(*rounds, 16), uint64_t(kNsMaxRound)), kNsMaxDraws - d0));
    if ((rc = reserve(eng, c.n_didx, size_t(cnt) * 4)) || (rc = reserve(eng, c.n_dflag, size_t(cnt) * 4)) ||
        (rc = reserve(eng, c.n_dpos, size_t(cnt) * 4)))
      return rc;
    uint32_t *didx = static_cast<uint32_t*>(c.n_didx.p), *flags = static_cast<uint32_t*>(c.n_dflag.p), *pos = static_cast<uint32_t*>(c.n_dpos.p);
    const int db = static_cast<int>((cnt + 255) / 256);
    CK(launch(eng, ns_draw_kernel, db, 256, 0, st, cum, n, seed, static_cast<uint32_t>(k), d0, cnt, didx, first));
    CK(launch(eng, ns_first_flag_kernel, db, 256, 0, st, didx, first, d0, cnt, flags));
    CK(cub_call(eng, c.n_tmp,
                [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, flags, pos, static_cast<int>(cnt), st); }));
    CK(launch(eng, ns_take_kernel, db, 256, 0, st, clipped, didx, flags, pos, cnt, carry, num, out, word + 14));
    CK(cudaMemcpyAsync(c.h_pinned.p, word + 14, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    std::memcpy(&carry, c.h_pinned.p, 4);
    d0 += cnt;
    ++*rounds;
  }
  *draws = d0;
  *n_sample = std::min(carry, num);
  return MCL3DL_OK;
}
}  // namespace

extern "C" {

int mcl3dl_abi_version(void)
{
  return MCL3DL_ABI_VERSION;
}

const char* mcl3dl_strerror(int code)
{
  switch (code)
  {
    case MCL3DL_OK: return "ok";
    case MCL3DL_ERR_INVALID_ARG: return "invalid argument";
    case MCL3DL_ERR_NO_MAP: return "measure() before set_map()";
    case MCL3DL_ERR_CUDA: return "CUDA runtime error";
    case MCL3DL_ERR_NO_DEVICE: return "no usable CUDA device";
    case MCL3DL_ERR_TOO_LARGE: return "grid exceeds 2^31-1 cells";
    case MCL3DL_ERR_RADIUS: return "search radius exceeds the supported range";
    default: return "unknown error";
  }
}

const char* mcl3dl_last_error_detail(const mcl3dl_engine* eng)
{
  return eng ? eng->err.c_str() : "";
}

uint64_t mcl3dl_kernel_launches(const mcl3dl_engine* eng)
{
  return eng ? eng->launches : 0;
}

int mcl3dl_create(mcl3dl_engine** out, const int* device_ids, int n_devices)
{
  if (!out || n_devices < 1)
    return MCL3DL_ERR_INVALID_ARG;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count < 1)
    return MCL3DL_ERR_NO_DEVICE;
  mcl3dl_engine* eng = new mcl3dl_engine;
  if (const char* f = std::getenv("MCL3DL_NN_CELL_FACTOR"))
  {
    const float v = static_cast<float>(std::atof(f));
    if (v >= 1.0f && v <= 4.0f)
      eng->nn_cell_factor = v;
  }
  if (const char* v = std::getenv("MCL3DL_NEAR_K"))
    eng->near_k = std::min(std::max(std::atoi(v), 0), 15);
  if (const char* v = std::getenv("MCL3DL_NEAR_KD_K"))
    eng->near_kd_k = std::min(std::max(std::atoi(v), 0), 15);
  if (const char* v = std::getenv("MCL3DL_NEAR_MAX_MB"))
    eng->near_max_bytes = static_cast<size_t>(std::max(std::atoi(v), 1)) << 20;
  if (const char* v = std::getenv("MCL3DL_TIMING"))
    eng->timing = std::atoi(v) != 0;
  if (const char* v = std::getenv("MCL3DL_ZEROCOPY_OUT"))
    eng->zero_copy_max = static_cast<size_t>(std::max(std::atol(v), 0L));
  if (const char* v = std::getenv("MCL3DL_DIRECT_MIN_KB"))  // -1: never copy from / to the caller's page-locked arrays in place
    eng->direct_min_bytes = std::atoi(v) < 0 ? ~size_t(0) : static_cast<size_t>(std::atoi(v)) << 10;
  if (const char* v = std::getenv("MCL3DL_NNF"))
    eng->nnf = std::atoi(v) != 0;
  if (const char* v = std::getenv("MCL3DL_BEAM"))
    eng->beam_dq = std::strcmp(v, "dq") == 0 ? 1 : (std::strcmp(v, "pl") == 0 ? 0 : 2);
  if (const char* v = std::getenv("MCL3DL_BEAM_DQ_PPL"))
    eng->beam_dq_ppl = std::min(std::max(std::atoi(v), 0), 64);
  if (const char* v = std::getenv("MCL3DL_LIK_SHARE"))
    eng->lik_share = std::min(std::max(std::atoi(v), 1), 8);
  if (const char* v = std::getenv("MCL3DL_NNF_KD_R2"))
    eng->nnf_kd_r2 = std::atoi(v) != 0;
  if (const char* v = std::getenv("MCL3DL_LIK_MODE"))
    eng->field_mode = std::strcmp(v, "field") == 0;
  if (const char* v = std::getenv("MCL3DL_FIELD_MAX_MB"))
    eng->field_max_bytes = static_cast<size_t>(std::max(std::atol(v), 1L)) << 20;
  if (const char* v = std::getenv("MCL3DL_NNF_MAX_MB"))
    eng->nnf_max_bytes = static_cast<size_t>(std::max(std::atol(v), 1L)) << 20;
  if (const char* v = std::getenv("MCL3DL_MAP_MAX_CELLS"))
    eng->map_max_cells = std::min(std::max<size_t>(std::strtoull(v, nullptr, 10), 8), (size_t(1) << 31) - 1);
  if (const char* o = std::getenv("MCL3DL_OVERLAP"))
    eng->overlap = std::atoi(o) != 0;
  eng->devs = std::vector<DeviceCtx>(n_devices);  // at its final size: a context never moves
  for (int i = 0; i < n_devices; ++i)
  {
    DeviceCtx& c = eng->devs[i];
    c.dev = device_ids ? device_ids[i] : i;
    if (c.dev < 0 || c.dev >= count)
    {
      mcl3dl_destroy(eng);
      return MCL3DL_ERR_NO_DEVICE;
    }
    cudaDeviceProp prop;
    if (cudaSetDevice(c.dev) != cudaSuccess || cudaGetDeviceProperties(&prop, c.dev) != cudaSuccess ||
        prop.major != 9 || prop.minor != 0)
    {
      mcl3dl_destroy(eng);  // built for sm_90a only; anything else cannot run these kernels
      return MCL3DL_ERR_NO_DEVICE;
    }
    c.sm_count = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking) != cudaSuccess)
    {
      mcl3dl_destroy(eng);
      return MCL3DL_ERR_CUDA;
    }
    for (auto& e : c.ev)
      if (cudaEventCreate(&e) != cudaSuccess)
      {
        mcl3dl_destroy(eng);
        return MCL3DL_ERR_CUDA;
      }
    if (cudaStreamCreateWithFlags(&c.side, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&c.ev_fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c.ev_join, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreate(&c.ev_b0) != cudaSuccess || cudaEventCreate(&c.ev_b1) != cudaSuccess ||
        cudaEventCreate(&c.ev_w0) != cudaSuccess || cudaEventCreate(&c.ev_w1) != cudaSuccess)
    {
      mcl3dl_destroy(eng);
      return MCL3DL_ERR_CUDA;
    }
  }
  *out = eng;
  return MCL3DL_OK;
}

int mcl3dl_host_alloc(mcl3dl_engine* eng, size_t bytes, void** out)
{
  if (!eng || !out || bytes == 0 || eng->devs.empty())
    return MCL3DL_ERR_INVALID_ARG;
  *out = nullptr;
  CK(cudaSetDevice(eng->devs[0].dev));
  void* p = nullptr;
  // portable: page-locked for every device of a multi-device engine; mapped into the unified address space, so that the
  // kernels of small updates can store their records into it
  CK(cudaHostAlloc(&p, bytes, cudaHostAllocPortable | cudaHostAllocMapped));
  eng->host_blocks.emplace_back(static_cast<char*>(p), bytes);
  *out = p;
  return MCL3DL_OK;
}

int mcl3dl_host_free(mcl3dl_engine* eng, void* p)
{
  if (!eng || !p)
    return MCL3DL_ERR_INVALID_ARG;
  for (size_t i = 0; i < eng->host_blocks.size(); ++i)
    if (eng->host_blocks[i].first == p)
    {
      for (DeviceCtx& c : eng->devs)  // nothing of this engine may still be reading or writing the block
      {
        CK(cudaSetDevice(c.dev));
        if (c.stream) CK(cudaStreamSynchronize(c.stream));
      }
      eng->host_blocks.erase(eng->host_blocks.begin() + static_cast<std::ptrdiff_t>(i));
      CK(cudaFreeHost(p));
      return MCL3DL_OK;
    }
  return MCL3DL_ERR_INVALID_ARG;
}

void mcl3dl_destroy(mcl3dl_engine* eng)
{
  if (!eng)
    return;
  eng->devs.clear();  // each context waits for its streams before it releases anything
  for (auto& b : eng->host_blocks)  // (blocks the caller did not return; its pointers into them dangle from here on)
    cudaFreeHost(b.first);
  delete eng;
}

// mcl3dl_set_map from its points on: `fill(c, d_pts, d_int)` leaves the n points and their intensities in the two
// buffers of device c on c.stream (a host upload, or the map intake's result moved in), then the build on every device.
// fill is not called when the reference's rebuild trigger finds nothing to do.
extern "C++" {
template <typename Fill>
static int set_map_from(mcl3dl_engine* eng, size_t n, uint64_t stamp, const mcl3dl_lik_params* lik, const mcl3dl_beam_params* beam,
                        Fill fill)
{
  // the reference's rebuild trigger: same header.stamp (and a non-empty index) -> nothing to do
  // (raycast_using_dda.h:168)
  if (eng->has_map && eng->stamp == stamp && eng->n_points == n &&
      (!lik || (eng->has_lik && std::memcmp(lik, &eng->lik, sizeof(*lik)) == 0)) &&
      (!beam || (eng->has_beam && std::memcmp(beam, &eng->beam, sizeof(*beam)) == 0)))
    return MCL3DL_OK;
  if (lik)
  {
    if (!(lik->match_dist_min > 0.0f) || !(lik->dist_weight[0] > 0.0f) || !(lik->dist_weight[1] > 0.0f) ||
        !(lik->dist_weight[2] > 0.0f))
      return MCL3DL_ERR_INVALID_ARG;
    eng->lik = *lik;
  }
  if (beam)
    eng->beam = *beam;
  eng->has_lik = lik != nullptr;
  eng->has_beam = beam != nullptr;
  derive_lik(eng);
  eng->has_map = false;
  std::memset(&eng->info, 0, sizeof(eng->info));
  eng->info.n_points = n;
  for (DeviceCtx& c : eng->devs)
  {
    DevBuf d_pts, d_int;
    int rc = MCL3DL_OK;
    CK(cudaSetDevice(c.dev));
    if ((rc = fill(c, d_pts, d_int)))
      return rc;
    uint64_t reselected = 0;
    bool incremental = false;
    if ((rc = build_map_on_device(eng, c, d_pts, n, 0, reselected, incremental)) || (rc = restage_field(eng, c)))
      return rc;
    c.map_int = std::move(d_int);
  }
  eng->has_map = true;
  eng->stamp = stamp;
  eng->n_points = n;
  return MCL3DL_OK;
}

// mcl3dl_map_append from its count on: `fill(c, pts, inten)` writes the n new points and their intensities at the two
// device pointers (after the staged ones) on c.stream
template <typename Fill>
static int map_append_from(mcl3dl_engine* eng, size_t n, uint64_t stamp, mcl3dl_map_append_info* info, Fill fill)
{
  const size_t n_before = eng->n_points;
  mcl3dl_map_append_info r{};
  r.n_before = n_before;
  r.n_appended = n;
  r.n_after = n_before + n;
  r.incremental = 1;  // n == 0: only the stamp changes
  if (n > 0)
  {
    r.incremental = 0;
    eng->has_map = false;
    std::memset(&eng->info, 0, sizeof(eng->info));
    eng->info.n_points = r.n_after;
    for (DeviceCtx& c : eng->devs)
    {
      // the staged points followed by the new ones, joined on the device: the base map does not cross the bus again
      DevBuf d_pts, d_int;
      int rc = MCL3DL_OK;
      CK(cudaSetDevice(c.dev));
      if ((rc = reserve(eng, d_pts, r.n_after * sizeof(mcl3dl_point))) || (rc = reserve(eng, d_int, r.n_after * sizeof(float))))
        return rc;
      CK(cudaEventRecord(c.ev[2], c.stream));
      CK(cudaMemcpyAsync(d_pts.p, c.raw_pts.p, n_before * sizeof(mcl3dl_point), cudaMemcpyDeviceToDevice, c.stream));
      CK(cudaMemcpyAsync(d_int.p, c.map_int.p, n_before * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
      if ((rc = fill(c, static_cast<mcl3dl_point*>(d_pts.p) + n_before, static_cast<float*>(d_int.p) + n_before)))
        return rc;
      uint64_t reselected = 0;
      bool incremental = false;
      if ((rc = build_map_on_device(eng, c, d_pts, r.n_after, n_before, reselected, incremental)))
        return rc;
      c.map_int = std::move(d_int);
      r.incremental = &c == &eng->devs[0] ? incremental : r.incremental && incremental;
      r.cells_reselected = std::max(r.cells_reselected, reselected);
      float ms = 0;
      CK(cudaEventElapsedTime(&ms, c.ev[2], c.ev[1]));  // (ev[1]: the end of the build, synchronised)
      r.build_ms = std::max(r.build_ms, static_cast<double>(ms));
      if ((rc = restage_field(eng, c)))
        return rc;
    }
    eng->has_map = true;
    eng->n_points = r.n_after;
  }
  eng->stamp = stamp;
  if (info)
    *info = r;
  return MCL3DL_OK;
}
}  // extern "C++"

int mcl3dl_set_map(mcl3dl_engine* eng, const mcl3dl_point* pts, size_t n, uint64_t stamp, const mcl3dl_lik_params* lik,
                   const mcl3dl_beam_params* beam)
{
  if (!eng || !pts || n == 0 || (!lik && !beam))
    return MCL3DL_ERR_INVALID_ARG;
  if (n >= (size_t(1) << 31))
    return MCL3DL_ERR_TOO_LARGE;
  return set_map_from(eng, n, stamp, lik, beam, [&](DeviceCtx& c, DevBuf& d_pts, DevBuf& d_int) -> int {
    int rc;
    if ((rc = reserve(eng, d_pts, n * sizeof(mcl3dl_point))) || (rc = reserve(eng, d_int, n * sizeof(float))))
      return rc;
    CK(cudaMemcpyAsync(d_pts.p, pts, n * sizeof(mcl3dl_point), cudaMemcpyHostToDevice, c.stream));
    CK(cudaMemsetAsync(d_int.p, 0, n * sizeof(float), c.stream));  // host arrays carry no intensity
    return MCL3DL_OK;
  });
}

int mcl3dl_map_append(mcl3dl_engine* eng, const mcl3dl_point* pts, size_t n, uint64_t stamp, mcl3dl_map_append_info* info)
{
  if (!eng)
    return MCL3DL_ERR_INVALID_ARG;
  if (!eng->has_map)
    return MCL3DL_ERR_NO_MAP;
  if (!pts && n > 0)
    return MCL3DL_ERR_INVALID_ARG;
  if (n >= (size_t(1) << 31) || eng->n_points + n >= (size_t(1) << 31))
    return MCL3DL_ERR_TOO_LARGE;
  return map_append_from(eng, n, stamp, info, [&](DeviceCtx& c, mcl3dl_point* d_pts, float* d_int) -> int {
    CK(cudaMemcpyAsync(d_pts, pts, n * sizeof(mcl3dl_point), cudaMemcpyHostToDevice, c.stream));
    CK(cudaMemsetAsync(d_int, 0, n * sizeof(float), c.stream));
    return MCL3DL_OK;
  });
}

// ---- map intake (scan_kernels.cuh: map_*_kernel)
// The checks of mcl3dl_map_load / mcl3dl_map_update_set, all before data is read
static int check_map_cloud(const mcl3dl_engine* eng, const mcl3dl_map_cloud* m, const float* leaf)
{
  if (!eng || !m || !m->view.data || !leaf)
    return MCL3DL_ERR_INVALID_ARG;
  const mcl3dl_cloud_view& v = m->view;
  const uint64_t n = static_cast<uint64_t>(v.width) * v.height;
  if (n == 0 || static_cast<uint64_t>(v.row_step) < static_cast<uint64_t>(v.width) * v.point_step)
    return MCL3DL_ERR_INVALID_ARG;
  for (int k = 0; k < 3; ++k)
    if (static_cast<uint64_t>(v.offset[k]) + 4 > v.point_step)
      return MCL3DL_ERR_INVALID_ARG;
  for (const int32_t o : {m->intensity_offset, m->label_offset})
    if (o < -1 || (o >= 0 && static_cast<uint64_t>(o) + 4 > v.point_step))
      return MCL3DL_ERR_INVALID_ARG;
  if (n >= (uint64_t(1) << 30))
    return MCL3DL_ERR_TOO_LARGE;  // the VoxelGrid's key limit, as mcl3dl_scan_prepare's
  return MCL3DL_OK;
}

// One map cloud on device c: its bytes up, the conversion, then the VoxelGrid at `leaf` with the intensity centroid, or,
// when the cloud passes unfiltered, its finite points in order.  The result goes to c.i_pts / c.i_int (n_out points);
// downsampled: the VoxelGrid filtered.  Nothing but the intake's own buffers changes.
static int map_intake(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_map_cloud* m, const float leaf[3], uint32_t& n_out, bool& downsampled,
                      float& ms)
{
  const mcl3dl_cloud_view& v = m->view;
  const uint32_t n = v.width * v.height;
  const size_t bytes = static_cast<size_t>(v.height - 1) * v.row_step + static_cast<size_t>(v.width) * v.point_step;
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = c.stream;
  int rc;
  if ((rc = reserve(eng, c.i_raw, bytes)) || (rc = reserve(eng, c.i_cloud, size_t(n) * 16)) || (rc = reserve(eng, c.i_cloud_int, size_t(n) * 4)) ||
      (rc = reserve(eng, c.i_pts, size_t(n) * 16)) || (rc = reserve(eng, c.i_int, size_t(n) * 4)) ||
      (rc = reserve(eng, c.i_flags, size_t(n) * 4)) || (rc = reserve(eng, c.i_pos, size_t(n) * 4)) || (rc = reserve(eng, c.i_count, 64)) ||
      (rc = reserve(eng, c.h_pinned, 256)))
    return rc;
  for (int k = 0; k < 2; ++k)
    if ((rc = reserve(eng, c.i_keys[k], size_t(n) * 4)) || (rc = reserve(eng, c.i_vals[k], size_t(n) * 4)))
      return rc;
  CK(cudaEventRecord(c.ev[0], st));
  CK(cudaMemcpyAsync(c.i_raw.p, v.data, bytes, cudaMemcpyHostToDevice, st));
  mcl3dl_point* in = static_cast<mcl3dl_point*>(c.i_cloud.p);
  float* in_int = static_cast<float*>(c.i_cloud_int.p);
  const int nb = static_cast<int>((n + 255) / 256);
  CK(launch(eng, map_read_kernel, nb, 256, 0, st, static_cast<const unsigned char*>(c.i_raw.p), v.width, n, v.row_step, v.point_step,
            v.offset[0], v.offset[1], v.offset[2], m->intensity_offset, m->label_offset, in, in_int));
  uint32_t* count = static_cast<uint32_t*>(c.i_count.p);
  CK(cudaMemsetAsync(count, 0, 64, st));
  mcl3dl_point* out = static_cast<mcl3dl_point*>(c.i_pts.p);
  float* out_int = static_cast<float*>(c.i_int.p);
  bool done = false;
  VoxelRuns runs;
  if (leaf[0] > 0.0f && leaf[1] > 0.0f && leaf[2] > 0.0f)
  {
    const VoxelBufs vb{{&c.i_keys[0], &c.i_keys[1]}, {&c.i_vals[0], &c.i_vals[1]}, {&c.i_kl[0], &c.i_kl[1]}, &c.i_flags, &c.i_pos, &c.i_tmp};
    if ((rc = voxel_grid(eng, c, st, in, n, n, leaf, vb, out, count, done, &runs)))
      return rc;
  }
  if (runs.sorted)
  {
    CK(launch(eng, map_intensity_kernel, nb, 256, 0, st, static_cast<const uint32_t*>(c.i_keys[1].p),
              static_cast<const uint32_t*>(c.i_vals[1].p), static_cast<const uint32_t*>(c.i_flags.p),
              static_cast<const uint32_t*>(c.i_pos.p), n, runs.nonfinite_key, in_int, out_int));
  }
  downsampled = done;
  if (!done)
  {
    // unfiltered: the finite points in order (a KdTreeFLANN input drops the others; the grids would index them)
    uint32_t* fl = static_cast<uint32_t*>(c.i_flags.p);
    uint32_t* ps = static_cast<uint32_t*>(c.i_pos.p);
    CK(launch(eng, map_finite_flags_kernel, nb, 256, 0, st, in, n, fl));
    CK(cub_call(eng, c.i_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, fl, ps, n, st); }));
    CK(launch(eng, map_compact_kernel, nb, 256, 0, st, in, in_int, fl, ps, n, out, out_int, count));
  }
  CK(cudaMemcpyAsync(c.h_pinned.p, count, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaEventRecord(c.ev[1], st));
  CK(cudaStreamSynchronize(st));  // the caller may reuse data as soon as this returns
  CK(cudaEventElapsedTime(&ms, c.ev[0], c.ev[1]));
  n_out = *static_cast<const uint32_t*>(c.h_pinned.p);
  return MCL3DL_OK;
}

// The intake's result (c.i_pts / c.i_int, reserved for the raw count) into buffers of its own size
static int exact_copy(mcl3dl_engine* eng, DeviceCtx& c, size_t n, DevBuf& pts, DevBuf& inten)
{
  int rc;
  CK(cudaSetDevice(c.dev));
  if ((rc = reserve(eng, pts, std::max<size_t>(n, 1) * sizeof(mcl3dl_point))) || (rc = reserve(eng, inten, std::max<size_t>(n, 1) * sizeof(float))))
    return rc;
  CK(cudaMemcpyAsync(pts.p, c.i_pts.p, n * sizeof(mcl3dl_point), cudaMemcpyDeviceToDevice, c.stream));
  CK(cudaMemcpyAsync(inten.p, c.i_int.p, n * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  return MCL3DL_OK;
}

// map_intake on every device; an engine whose devices disagree on the count is a fault of the engine
static int map_intake_all(mcl3dl_engine* eng, const mcl3dl_map_cloud* m, const float leaf[3], mcl3dl_map_intake_info& info)
{
  info = mcl3dl_map_intake_info{};
  info.n_input = static_cast<uint64_t>(m->view.width) * m->view.height;
  for (DeviceCtx& c : eng->devs)
  {
    uint32_t n_out = 0;
    bool ds = false;
    float ms = 0;
    const int rc = map_intake(eng, c, m, leaf, n_out, ds, ms);
    if (rc)
      return rc;
    if (&c != &eng->devs[0] && (n_out != info.n_staged || (ds ? 1 : 0) != info.downsampled))
    {
      eng->err = "map intake: the devices disagree";
      return MCL3DL_ERR_CUDA;
    }
    info.n_staged = n_out;
    info.downsampled = ds ? 1 : 0;
    info.device_ms = std::max(info.device_ms, static_cast<double>(ms));
  }
  return MCL3DL_OK;
}

int mcl3dl_map_load(mcl3dl_engine* eng, const mcl3dl_map_cloud* map, const float leaf[3], uint64_t stamp, const mcl3dl_lik_params* lik,
                    const mcl3dl_beam_params* beam, mcl3dl_map_intake_info* info)
{
  int rc;
  if ((rc = check_map_cloud(eng, map, leaf)))
    return rc;
  if ((!lik && !beam) || (lik && (!(lik->match_dist_min > 0.0f) || !(lik->dist_weight[0] > 0.0f) ||
                                  !(lik->dist_weight[1] > 0.0f) || !(lik->dist_weight[2] > 0.0f))))
    return MCL3DL_ERR_INVALID_ARG;
  mcl3dl_map_intake_info r;
  if ((rc = map_intake_all(eng, map, leaf, r)))
    return rc;
  if (r.n_staged == 0)
    return MCL3DL_ERR_INVALID_ARG;  // no finite point: the previous map stays, as set_map refuses n == 0
  const size_t n = r.n_staged;
  rc = set_map_from(eng, n, stamp, lik, beam, [&](DeviceCtx& c, DevBuf& d_pts, DevBuf& d_int) -> int {
    return exact_copy(eng, c, n, d_pts, d_int);
  });
  if (rc)
    return rc;
  eng->has_patch = false;  // loadMapCloud: pc_update_.reset()
  if (info)
    *info = r;
  return MCL3DL_OK;
}

int mcl3dl_map_update_set(mcl3dl_engine* eng, const mcl3dl_map_cloud* patch, const float leaf[3], mcl3dl_map_intake_info* info)
{
  int rc;
  if ((rc = check_map_cloud(eng, patch, leaf)))
    return rc;
  mcl3dl_map_intake_info r;
  if ((rc = map_intake_all(eng, patch, leaf, r)))
    return rc;
  // the new patch replaces the pending one (copied first on every device: an error keeps the pending patch)
  std::vector<DevBuf> pts(eng->devs.size()), inten(eng->devs.size());
  for (size_t k = 0; k < eng->devs.size(); ++k)
    if ((rc = exact_copy(eng, eng->devs[k], r.n_staged, pts[k], inten[k])))
      return rc;
  for (size_t k = 0; k < eng->devs.size(); ++k)
  {
    eng->devs[k].p_pts = std::move(pts[k]);
    eng->devs[k].p_int = std::move(inten[k]);
  }
  eng->has_patch = true;
  eng->patch_n = r.n_staged;
  if (info)
    *info = r;
  return MCL3DL_OK;
}

int mcl3dl_map_update_commit(mcl3dl_engine* eng, uint64_t stamp, mcl3dl_map_append_info* info)
{
  if (!eng)
    return MCL3DL_ERR_INVALID_ARG;
  if (!eng->has_map)
    return MCL3DL_ERR_NO_MAP;  // the patch stays pending
  if (!eng->has_patch)
  {
    // cbMapUpdateTimer without pc_update_: nothing changes
    if (info)
    {
      *info = mcl3dl_map_append_info{};
      info->n_before = info->n_after = eng->n_points;
      info->incremental = 1;
    }
    return MCL3DL_OK;
  }
  const size_t n = eng->patch_n;
  if (eng->n_points + n >= (size_t(1) << 31))
    return MCL3DL_ERR_TOO_LARGE;
  const int rc = map_append_from(eng, n, stamp, info, [&](DeviceCtx& c, mcl3dl_point* d_pts, float* d_int) -> int {
    CK(cudaMemcpyAsync(d_pts, c.p_pts.p, n * sizeof(mcl3dl_point), cudaMemcpyDeviceToDevice, c.stream));
    CK(cudaMemcpyAsync(d_int, c.p_int.p, n * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
    return MCL3DL_OK;
  });
  if (rc)
    return rc;
  eng->has_patch = false;
  return MCL3DL_OK;
}

int mcl3dl_map_update_clear(mcl3dl_engine* eng)
{
  if (!eng)
    return MCL3DL_ERR_INVALID_ARG;
  eng->has_patch = false;
  return MCL3DL_OK;
}

int mcl3dl_map_get(mcl3dl_engine* eng, mcl3dl_point* out, float* intensity_out, size_t capacity, size_t* n_out)
{
  if (!eng || !n_out)
    return MCL3DL_ERR_INVALID_ARG;
  if (!eng->has_map)
    return MCL3DL_ERR_NO_MAP;
  const size_t n = eng->n_points;
  *n_out = n;
  if (!out)
    return MCL3DL_OK;
  if (capacity < n)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  CK(cudaSetDevice(c.dev));
  CK(cudaMemcpyAsync(out, c.raw_pts.p, n * sizeof(mcl3dl_point), cudaMemcpyDeviceToHost, c.stream));
  if (intensity_out)
    CK(cudaMemcpyAsync(intensity_out, c.map_int.p, n * sizeof(float), cudaMemcpyDeviceToHost, c.stream));
  CK(cudaStreamSynchronize(c.stream));
  return MCL3DL_OK;
}

int mcl3dl_set_params(mcl3dl_engine* eng, const mcl3dl_lik_params* lik, const mcl3dl_beam_params* beam)
{
  if (!eng || !eng->has_map)
    return MCL3DL_ERR_NO_MAP;
  if (lik)
  {
    if (!eng->has_lik || lik->match_dist_min != eng->lik.match_dist_min ||
        std::memcmp(lik->dist_weight, eng->lik.dist_weight, sizeof(lik->dist_weight)) != 0)
      return MCL3DL_ERR_INVALID_ARG;  // these fix the staged grid
    eng->lik = *lik;
    derive_lik(eng);
  }
  if (beam)
  {
    if (!eng->has_beam || beam->dda_grid_size != eng->beam.dda_grid_size ||
        beam->use_raycast_using_dda != eng->beam.use_raycast_using_dda)
      return MCL3DL_ERR_INVALID_ARG;
    eng->beam = *beam;
    for (DeviceCtx& c : eng->devs)
    {
      fill_dda_scalars(eng->beam, c.dda);
      const float4* keep = c.kd.raw_pts;
      fill_kd_scalars(eng->beam, c.kd);
      c.kd.raw_pts = keep;
#if MCL3DL_NEAR_BITS
      if (c.kd.r1_pad > c.near_kd_r)
        c.kd.near.bits = nullptr;  // the field was built for a smaller marching radius: search unscreened
#endif
    }
  }
  return MCL3DL_OK;
}

int mcl3dl_near_field_info(const mcl3dl_engine* eng, int32_t k_out[2], uint64_t bytes_out[2])
{
  if (!eng || !k_out || !bytes_out)
    return MCL3DL_ERR_INVALID_ARG;
  for (int i = 0; i < 2; ++i)
  {
    k_out[i] = eng->near_info_k[i];
    bytes_out[i] = eng->near_info_bytes[i];
  }
  return MCL3DL_OK;
}

int mcl3dl_field_mode(mcl3dl_engine* eng, int enable)
{
  if (!eng)
    return MCL3DL_ERR_INVALID_ARG;
  if (!enable)
  {
    eng->field_mode = 0;
    return MCL3DL_OK;
  }
  if (eng->has_map)
  {
    if (!eng->has_lik)
      return MCL3DL_ERR_INVALID_ARG;
    if (eng->devs[0].w_on)
      return MCL3DL_ERR_TOO_LARGE;
    for (DeviceCtx& c : eng->devs)
      if (!c.fld_nodes_valid)
      {
        const int rc = stage_field(eng, c, nullptr);
        if (rc != MCL3DL_OK)
          return rc;
      }
  }
  eng->field_mode = 1;  // (no map yet: the next set_map stages the volume)
  return MCL3DL_OK;
}

int mcl3dl_field_nodes(mcl3dl_engine* eng, float* nodes_out, int32_t dims_out[3], float origin_out[3], float* edge_out)
{
  if (!eng || !eng->has_map || eng->devs.empty())
    return MCL3DL_ERR_NO_MAP;
  DeviceCtx& c = eng->devs[0];
  if (c.w_on)
    return MCL3DL_ERR_TOO_LARGE;
  const NnFieldDev& f = c.nn.field;
  if (!f.dir)
    return MCL3DL_ERR_INVALID_ARG;
  const int nnx = f.nx + 1, nny = f.ny + 1, nnz = f.nz + 1;
  if (dims_out)
  {
    dims_out[0] = nnx;
    dims_out[1] = nny;
    dims_out[2] = nnz;
  }
  if (origin_out)
  {
    origin_out[0] = f.ox;
    origin_out[1] = f.oy;
    origin_out[2] = f.oz;
  }
  if (edge_out)
    *edge_out = f.e;
  if (!nodes_out)
    return MCL3DL_OK;
  if (!c.fld_nodes_valid)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  cudaMemcpy3DParms cp{};
  cp.srcPtr = c.fld_nodes;
  cp.dstPtr = make_cudaPitchedPtr(nodes_out, static_cast<size_t>(nnx) * sizeof(float), nnx, nny);
  cp.extent = make_cudaExtent(static_cast<size_t>(nnx) * sizeof(float), nny, nnz);
  cp.kind = cudaMemcpyDeviceToHost;
  CK(cudaMemcpy3DAsync(&cp, c.stream));
  CK(cudaStreamSynchronize(c.stream));
  return MCL3DL_OK;
}

int mcl3dl_field_upload(mcl3dl_engine* eng, const float* nodes, const int32_t dims[3])
{
  if (!eng || !nodes || !dims)
    return MCL3DL_ERR_INVALID_ARG;
  if (!eng->has_map || !eng->has_lik)
    return MCL3DL_ERR_NO_MAP;
  if (eng->devs[0].w_on)
    return MCL3DL_ERR_TOO_LARGE;
  for (DeviceCtx& c : eng->devs)
  {
    const NnFieldDev& f = c.nn.field;
    if (!f.dir || dims[0] != f.nx + 1 || dims[1] != f.ny + 1 || dims[2] != f.nz + 1)
      return MCL3DL_ERR_INVALID_ARG;
    const int rc = stage_field(eng, c, nodes);
    if (rc != MCL3DL_OK)
      return rc;
  }
  return MCL3DL_OK;
}

int mcl3dl_nn_field_info(const mcl3dl_engine* eng, uint64_t out[5])
{
  if (!eng || !out)
    return MCL3DL_ERR_INVALID_ARG;
  const bool on = !eng->devs.empty() && eng->devs[0].nn.field.dir != nullptr;
  out[0] = on ? eng->nnf_bytes : 0;
  out[1] = on ? eng->nnf_cands : 0;
  out[2] = on ? eng->nnf_overflow_cells : 0;
  out[3] = on ? static_cast<uint64_t>(eng->devs[0].nn.field.e * 1e6f) : 0;
  out[4] = on ? eng->nnf_wide_cells : 0;
  return MCL3DL_OK;
}

int mcl3dl_get_map_info(const mcl3dl_engine* eng, mcl3dl_map_info* out)
{
  if (!eng || !out)
    return MCL3DL_ERR_INVALID_ARG;
  if (!eng->has_map)
    return MCL3DL_ERR_NO_MAP;
  *out = eng->info;
  return MCL3DL_OK;
}

int mcl3dl_map_window_info(const mcl3dl_engine* eng, mcl3dl_window_info* out)
{
  if (!eng || !out)
    return MCL3DL_ERR_INVALID_ARG;
  if (!eng->has_map)
    return MCL3DL_ERR_NO_MAP;
  const DeviceCtx& c = eng->devs[0];
  *out = mcl3dl_window_info{};
  out->windowed = c.w_on ? 1 : 0;
  out->staged = c.w_on && c.w_valid ? 1 : 0;
  for (int k = 0; k < 3; ++k)
  {
    out->box_min[k] = c.w_box.lo[k];
    out->box_max[k] = c.w_box.hi[k];
    out->dims[k] = out->staged ? c.w_dims[k] : 0;
  }
  out->rebuilds = c.w_rebuilds;
  out->rebuild_ms = c.w_ms;
  return MCL3DL_OK;
}

int mcl3dl_last_timing(const mcl3dl_engine* eng, double* h2d_ms, double* lik_ms, double* beam_ms, double* d2h_ms)
{
  if (!eng)
    return MCL3DL_ERR_INVALID_ARG;
  if (h2d_ms) *h2d_ms = eng->t_h2d;
  if (lik_ms) *lik_ms = eng->t_lik;
  if (beam_ms) *beam_ms = eng->t_beam;
  if (d2h_ms) *d2h_ms = eng->t_d2h;
  return MCL3DL_OK;
}

// The arguments every measurement entry point shares.  `host_scans`: the scans are in host memory, so the beam labels,
// which index the origins (origins[p.label], beam.cpp:142-145), are checked too.
static int validate_measure(mcl3dl_engine* eng, size_t P, const mcl3dl_point* lik, size_t n_lik, const mcl3dl_point* beam,
                            size_t n_beam, const float* origins, size_t n_origins, bool host_scans)
{
  if (!eng)
    return MCL3DL_ERR_INVALID_ARG;
  if (!eng->has_map)
    return MCL3DL_ERR_NO_MAP;
  if (P >= (size_t(1) << 31) || n_lik >= (size_t(1) << 24) || n_beam >= (size_t(1) << 24))
    return MCL3DL_ERR_TOO_LARGE;
  if ((n_lik && !eng->has_lik) || (n_beam && !eng->has_beam))
    return MCL3DL_ERR_INVALID_ARG;  // that model's grid was never staged
  if (n_beam && n_origins == 0)
    return MCL3DL_ERR_INVALID_ARG;
  if ((n_lik && !lik) || (n_beam && (!beam || !origins)))
    return MCL3DL_ERR_INVALID_ARG;
  for (size_t j = 0; host_scans && j < n_beam; ++j)
    if (beam[j].label >= n_origins)
      return MCL3DL_ERR_INVALID_ARG;
  return MCL3DL_OK;
}

// Enqueue both models of one update for the particles [poses, poses+P) of one device.  Node order is "beam"
// then "likelihood" (src/mcl_3dl.cpp:409-415) but the two write disjoint fields, so when both have a scan the
// beam kernel goes to the side stream and overlaps the likelihood kernel.  A model without a scan costs no
// launch: the other kernel writes its (1, 0).  `timed` records ev[2]/ev[3] (likelihood) and ev_b0/ev_b1 (beam).
static int launch_models(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* lik,
                         size_t n_lik, const mcl3dl_point* beam, size_t n_beam, const float* origins, size_t n_origins,
                         mcl3dl_result* out, uint8_t* status, cudaStream_t st, bool timed, const RecordSink* sink_in = nullptr)
{
  int rc = MCL3DL_OK;
  const RecordSink sink = sink_in ? *sink_in : RecordSink{};
  const bool both = n_beam && n_lik && eng->overlap;
  cudaStream_t sb = both ? c.side : st;
  if (n_beam)
  {
    if (both)
    {
      CK(cudaEventRecord(c.ev_fork, st));
      CK(cudaStreamWaitEvent(sb, c.ev_fork, 0));
    }
    if (timed) CK(cudaEventRecord(c.ev_b0, sb));
    rc = launch_beam(eng, c, poses, P, beam, n_beam, origins, static_cast<int>(n_origins), out, status, n_lik == 0, sb, sink);
    if (rc != MCL3DL_OK)
      return rc;
    if (timed) CK(cudaEventRecord(c.ev_b1, sb));
    if (both) CK(cudaEventRecord(c.ev_join, sb));
  }
  if (timed) CK(cudaEventRecord(c.ev[2], st));
  if (n_lik || !n_beam)
  {
    rc = launch_lik(eng, c, poses, P, lik, n_lik, out, n_beam == 0, st, sink);
    if (rc != MCL3DL_OK)
    {
      if (both)
        cudaStreamWaitEvent(st, c.ev_join, 0);  // the side stream is joined on the error path as well
      return rc;
    }
  }
  if (timed) CK(cudaEventRecord(c.ev[3], st));
  if (both) CK(cudaStreamWaitEvent(st, c.ev_join, 0));
  return rc;
}

// One device's share of the particles of a host-array update and the layout of its pinned block: the inputs [poses |
// likelihood scan | beam scan | origins | prior | extra] (16-byte sections, as in d_poses), then the outputs [posterior |
// records | beam status | the WeightPartials of pass 1 and 2].  Absent sections have zero size.
struct Share
{
  size_t p0, n;  // the particles [p0, p0 + n)
  size_t o_lik, o_beam, o_org, o_prior, o_extra, in_bytes;
  size_t o_post, o_rec, o_status, o_part, total;
};

static size_t pad16(size_t b) { return (b + 15) & ~size_t(15); }

// Device d's block of P particles over G devices; per-particle sections in bytes per particle
static Share share_of(size_t P, size_t G, size_t d, size_t pose_b, size_t n_lik, size_t n_beam, size_t n_origins,
                      size_t prior_b, size_t extra_b, size_t post_b, size_t rec_b, size_t status_b)
{
  Share s;
  s.p0 = P * d / G;
  s.n = P * (d + 1) / G - s.p0;
  s.o_lik = s.n * pose_b;
  s.o_beam = s.o_lik + n_lik * 16;
  s.o_org = s.o_beam + n_beam * 16;
  s.o_prior = s.o_org + pad16(n_origins * 12);
  s.o_extra = s.o_prior + pad16(s.n * prior_b);
  s.in_bytes = s.o_extra + pad16(s.n * extra_b);
  s.o_post = s.in_bytes;
  s.o_rec = s.o_post + pad16(s.n * post_b);
  s.o_status = s.o_rec + s.n * rec_b;
  s.o_part = pad16(s.o_status + s.n * status_b);
  s.total = s.o_part + 2 * sizeof(WeightPartial) + 64;
  return s;
}

// The host inputs into their sections of the pinned block, then ONE H2D copy to d_poses.  Without `poses` the copy starts
// at the likelihood scan (resident poses, or a page-locked pose array DMA-ed in place).  `timed`: ev[0] before the copy.
static int stage_inputs(mcl3dl_engine* eng, DeviceCtx& c, const Share& s, const mcl3dl_pose* poses, const mcl3dl_point* lik,
                        const mcl3dl_point* beam, const float* origins, size_t n_origins, const float* prior, const float* extra,
                        bool timed)
{
  char* hp = static_cast<char*>(c.h_pinned.p);
  if (poses) std::memcpy(hp, poses + s.p0, s.o_lik);
  if (s.o_beam > s.o_lik) std::memcpy(hp + s.o_lik, lik, s.o_beam - s.o_lik);
  if (s.o_org > s.o_beam) std::memcpy(hp + s.o_beam, beam, s.o_org - s.o_beam);
  if (n_origins) std::memcpy(hp + s.o_org, origins, n_origins * 12);
  if (prior) std::memcpy(hp + s.o_prior, prior + s.p0, s.n * 4);
  if (extra) std::memcpy(hp + s.o_extra, extra + s.p0, s.n * 4);
  if (timed) CK(cudaEventRecord(c.ev[0], c.stream));
  const size_t from = poses ? 0 : s.o_lik;
  if (s.in_bytes > from)
    CK(cudaMemcpyAsync(static_cast<char*>(c.d_poses.p) + from, hp + from, s.in_bytes - from, cudaMemcpyHostToDevice, c.stream));
  return MCL3DL_OK;
}

// Pass 1 of the weight update: w_i into d_w; the folded partial is left at *folded (and stored by the kernel at h_part)
static int weight_pass1(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_result* rec, const float* prior, const float* extra,
                        size_t n, size_t n_lik, WeightPartial* h_part, const WeightPartial** folded)
{
  int nblk;
  WeightPartial* slots;
  unsigned int* tk;
  if (int rc = weight_scratch(eng, c, n, 0, &nblk, &slots, &tk))
    return rc;
  CK(launch(eng, weight_kernel, nblk, kBlockThreads, 0, c.stream, rec, prior, extra, static_cast<int>(n), static_cast<int>(n_lik),
            static_cast<float*>(c.d_w.p), slots, tk, h_part));
  *folded = slots + nblk;
  return MCL3DL_OK;
}

// Pass 2: p_i = w_i / total into `post`, the total read from `pass1` on the device when given; folded as pass 1
static int weight_pass2(mcl3dl_engine* eng, DeviceCtx& c, const WeightPartial* pass1, float total, size_t n, size_t index_offset,
                        float* post, WeightPartial* h_part, const WeightPartial** folded)
{
  int nblk;
  WeightPartial* slots;
  unsigned int* tk;
  if (int rc = weight_scratch(eng, c, n, 1, &nblk, &slots, &tk))
    return rc;
  CK(launch(eng, normalize_kernel, nblk, kBlockThreads, 0, c.stream, static_cast<const float*>(c.d_w.p), static_cast<int>(n), pass1,
            total, static_cast<int>(index_offset), post, slots, tk, h_part));
  *folded = slots + nblk;
  return MCL3DL_OK;
}

// The weight update of ONE device: both passes, the total read on the device.  The folded partials come back to
// h_part[0..1] and the posterior to h_post (if given): stored by the kernels up to zero_copy_max particles, else copied.
static int fold_weights(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_result* rec, const float* prior, const float* extra,
                        float* post, size_t n, size_t n_lik, size_t index_offset, WeightPartial* h_part, float* h_post)
{
  const bool zc = n <= eng->zero_copy_max;
  const WeightPartial *f1, *f2;
  int rc = weight_pass1(eng, c, rec, prior, extra, n, n_lik, zc ? h_part : nullptr, &f1);
  if (rc != MCL3DL_OK)
    return rc;
  rc = weight_pass2(eng, c, f1, 0.0f, n, index_offset, zc && h_post ? h_post : post, zc ? h_part + 1 : nullptr, &f2);
  if (rc != MCL3DL_OK)
    return rc;
  if (!zc)  // (behind both kernels, so that pass 2 does not wait for a copy)
  {
    CK(cudaMemcpyAsync(h_part, f1, sizeof(WeightPartial), cudaMemcpyDeviceToHost, c.stream));
    if (h_post)
      CK(cudaMemcpyAsync(h_post, post, n * 4, cudaMemcpyDeviceToHost, c.stream));
    CK(cudaMemcpyAsync(h_part + 1, f2, sizeof(WeightPartial), cudaMemcpyDeviceToHost, c.stream));
  }
  return MCL3DL_OK;
}

// The summary from the partials of pass 1 and 2, folded over the devices
static void make_summary(const WeightPartial& w1, const WeightPartial& w2, mcl3dl_update_summary* s)
{
  std::memset(s, 0, sizeof(*s));
  s->weight_sum = static_cast<float>(w1.sum);
  s->match_ratio_min = std::min(1.0f, w1.qmin);
  s->match_ratio_max = std::max(0.0f, w1.qmax);
  s->kept = s->weight_sum > 0.0f ? 1 : 0;
  s->entropy = s->kept ? static_cast<float>(-w2.sum) : 0.0f;
  s->max_index = s->kept && w2.best > -1.0f ? w2.best_i : 0;
}

int mcl3dl_measure_device(mcl3dl_engine* eng, const mcl3dl_pose* d_poses, size_t P, const mcl3dl_point* d_lik, size_t n_lik,
                          const mcl3dl_point* d_beam, size_t n_beam, const float* d_origins_xyz, size_t n_origins,
                          mcl3dl_result* d_out, void* cuda_stream)
{
  int rc = validate_measure(eng, P, d_lik, n_lik, d_beam, n_beam, d_origins_xyz, n_origins, false);
  if (rc != MCL3DL_OK)
    return rc;
  if (eng->devs.size() != 1 || (P && (!d_poses || !d_out)))
    return MCL3DL_ERR_INVALID_ARG;
  if (P == 0)
    return MCL3DL_OK;
  DeviceCtx& c = eng->devs[0];
  if (c.w_on)
    return MCL3DL_ERR_TOO_LARGE;  // a window check synchronises: not on the caller's stream
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  return launch_models(eng, c, d_poses, P, d_lik, n_lik, d_beam, n_beam, d_origins_xyz, n_origins, d_out, nullptr, st, false);
}

// ---- resident particle set (scope row f3; see include/mcl3dl_b200.h; tests/test_gpu_pf_exact.py holds it to its host
// restatement)
// Every per-particle buffer of the resident set with room for n particles: both state buffers, the probabilities, the
// prefix sum + pstep (n + 1), the packed poses and r_extra (the odometry-error factors of an update, the pscan chain of
// a resize).  reserve() drops a buffer's contents when it grows, so the buffers a kernel still has to read are named in
// `live` and left as they are (the caller reserves them again once that kernel has run); before anything grows, the
// stream's pending work is waited for.
static int reserve_resident(mcl3dl_engine* eng, DeviceCtx& c, size_t n, std::initializer_list<const DevBuf*> live = {})
{
  const std::pair<DevBuf*, size_t> want[] = {{&c.r_states[0], n * sizeof(mcl3dl_state)}, {&c.r_states[1], n * sizeof(mcl3dl_state)},
                                             {&c.r_prob, n * 4},  {&c.r_accum, (n + 1) * 4},
                                             {&c.r_poses, n * sizeof(mcl3dl_pose)}, {&c.r_extra, n * 4}};
  bool synced = false;
  for (const auto& w : want)
  {
    if (std::find(live.begin(), live.end(), w.first) != live.end() || (w.first->p && w.second <= w.first->cap))
      continue;
    if (!synced)
    {
      CK(cudaStreamSynchronize(c.stream));
      synced = true;
    }
    if (int rc = reserve(eng, *w.first, w.second))
      return rc;
  }
  return MCL3DL_OK;
}

int mcl3dl_particles_set(mcl3dl_engine* eng, const mcl3dl_state* states, const float* prob, size_t n)
{
  if (!eng || eng->devs.size() != 1 || !states || !prob || n == 0 || n >= (size_t(1) << 31))
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  CK(cudaSetDevice(c.dev));
  int rc;
  if ((rc = reserve_resident(eng, c, n)))
    return rc;
  CK(cudaMemcpyAsync(c.r_states[0].p, states, n * sizeof(mcl3dl_state), cudaMemcpyHostToDevice, c.stream));
  CK(cudaMemcpyAsync(c.r_prob.p, prob, n * 4, cudaMemcpyHostToDevice, c.stream));
  CK(cudaStreamSynchronize(c.stream));  // the caller's buffers are pageable and only read during the call
  c.r_n = n;
  c.r_cur = 0;
  return MCL3DL_OK;
}

int mcl3dl_particles_get(mcl3dl_engine* eng, mcl3dl_state* states, float* prob, size_t n)
{
  if (!eng || eng->devs.size() != 1)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (c.r_n == 0 || n != c.r_n)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  if (states)
    CK(cudaMemcpyAsync(states, c.r_states[c.r_cur].p, n * sizeof(mcl3dl_state), cudaMemcpyDeviceToHost, c.stream));
  if (prob)
    CK(cudaMemcpyAsync(prob, c.r_prob.p, n * 4, cudaMemcpyDeviceToHost, c.stream));
  CK(cudaStreamSynchronize(c.stream));
  return MCL3DL_OK;
}

int mcl3dl_particles_predict(mcl3dl_engine* eng, const mcl3dl_pose* a, const mcl3dl_pose* b, float time_diff, float tc_lin,
                             float tc_ang)
{
  if (!eng || eng->devs.size() != 1 || !a || !b)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (c.r_n == 0)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  const float pp[3] = {a->px, a->py, a->pz}, pq[4] = {a->qx, a->qy, a->qz, a->qw};
  const float cp[3] = {b->px, b->py, b->pz}, cq[4] = {b->qx, b->qy, b->qz, b->qw};
  const MotionDev m = pf_set_odoms(pp, pq, cp, cq, time_diff, tc_lin, tc_ang);
  const uint32_t n = static_cast<uint32_t>(c.r_n);
  CK(launch(eng, pf_predict_kernel, (n + 255) / 256, 256, 0, c.stream, static_cast<PfState*>(c.r_states[c.r_cur].p), n, m));
  return MCL3DL_OK;  // stream-ordered before whatever comes next; get() / measure_update() synchronise
}

int mcl3dl_particles_resample(mcl3dl_engine* eng, const float sigma_pos[3], const float sigma_rpy[3], float initial_frac,
                              uint64_t seed)
{
  if (!eng || eng->devs.size() != 1 || !sigma_pos || !sigma_rpy || !(initial_frac >= 0.0f) || !(initial_frac < 1.0f))
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (c.r_n == 0)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  const uint32_t n = static_cast<uint32_t>(c.r_n);
  float* accum = static_cast<float*>(c.r_accum.p);
  CK(launch(eng, pf_accum_kernel, 1, 32, 0, c.stream, static_cast<const float*>(c.r_prob.p), n, accum, accum + n));  // one warp, in order
  Sigma6 sg;
  for (int k = 0; k < 3; ++k)
  {
    sg.v[k] = sigma_pos[k];
    sg.v[k + 3] = sigma_rpy[k];
  }
  ++c.r_calls;
  CK(launch(eng, pf_resample_kernel, (n + 255) / 256, 256, 0, c.stream, static_cast<const PfState*>(c.r_states[c.r_cur].p), accum,
            accum + n, n, initial_frac, seed, c.r_calls, sg, static_cast<PfState*>(c.r_states[1 - c.r_cur].p),
            static_cast<float*>(c.r_prob.p)));
  c.r_cur = 1 - c.r_cur;
  return MCL3DL_OK;
}

// ---- the node's other particle events on the resident set: the odometry-noise redraw, expansion resetting and the
// IMU gravity update (pf_kernels.cuh)
static bool finite_nonneg(double v) { return v >= 0.0 && std::isfinite(v); }

int mcl3dl_particles_redraw_odom_noise(mcl3dl_engine* eng, double lin_lin, double lin_ang, double ang_lin, double ang_ang, uint64_t seed)
{
  if (!eng || eng->devs.size() != 1 || !finite_nonneg(lin_lin) || !finite_nonneg(lin_ang) || !finite_nonneg(ang_lin) ||
      !finite_nonneg(ang_ang))
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (c.r_n == 0)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  const uint32_t n = static_cast<uint32_t>(c.r_n);
  OdomNoiseSigma sg;
  sg.ll = lin_lin;
  sg.la = lin_ang;
  sg.aa = ang_ang;
  sg.al = ang_lin;
  ++c.r_redraw_calls;
  CK(launch(eng, pf_redraw_kernel, (n + 255) / 256, 256, 0, c.stream, static_cast<PfState*>(c.r_states[c.r_cur].p), n, seed,
            c.r_redraw_calls, sg));
  CK(cudaStreamSynchronize(c.stream));
  return MCL3DL_OK;
}

int mcl3dl_particles_noise(mcl3dl_engine* eng, const float sigma_pos[3], const float sigma_rpy[3], uint64_t seed)
{
  if (!eng || eng->devs.size() != 1 || !sigma_pos || !sigma_rpy)
    return MCL3DL_ERR_INVALID_ARG;
  Sigma6 sg;
  for (int k = 0; k < 3; ++k)
  {
    sg.v[k] = sigma_pos[k];
    sg.v[k + 3] = sigma_rpy[k];
  }
  for (float v : sg.v)
    if (!finite_nonneg(v))
      return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (c.r_n == 0)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  const uint32_t n = static_cast<uint32_t>(c.r_n);
  ++c.r_noise_calls;
  CK(launch(eng, pf_noise_kernel, (n + 255) / 256, 256, 0, c.stream, static_cast<PfState*>(c.r_states[c.r_cur].p), n, seed,
            c.r_noise_calls, sg));
  CK(cudaStreamSynchronize(c.stream));
  return MCL3DL_OK;
}

// An update of the resident set whose likelihood one thread-per-particle kernel computes (pf_imu_kernel,
// pf_landmark_kernel): kernel(d_rec, lik) launches the kernel that writes a unit record and the likelihood of every
// particle, and the weight fold takes the likelihood as the extra factor: w = prior * (((1 * 1) * 1) * lik) = prior * lik;
// n_lik = 0 makes every particle's match ratio 0.  The posterior replaces the resident probabilities unless the update is
// discarded.
extern "C++" {
template <typename Kernel>
static int resident_likelihood_update(mcl3dl_engine* eng, DeviceCtx& c, mcl3dl_update_summary* summary, Kernel kernel)
{
  const size_t P = c.r_n;
  CK(cudaSetDevice(c.dev));
  const Share s = share_of(P, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0);  // only the two WeightPartials come back
  int rc;
  if ((rc = reserve(eng, c.h_pinned, s.total)) || (rc = reserve(eng, c.d_out, P * sizeof(mcl3dl_result))))
    return rc;
  mcl3dl_result* d_rec = static_cast<mcl3dl_result*>(c.d_out.p);
  float* lik = static_cast<float*>(c.r_extra.p);
  CK(kernel(d_rec, lik));
  float* prob = static_cast<float*>(c.r_prob.p);
  WeightPartial* h_part = reinterpret_cast<WeightPartial*>(static_cast<char*>(c.h_pinned.p) + s.o_part);
  if ((rc = fold_weights(eng, c, d_rec, prob, lik, prob, P, 0, 0, h_part, nullptr)))
    return rc;
  CK(cudaStreamSynchronize(c.stream));
  make_summary(h_part[0], h_part[1], summary);
  return MCL3DL_OK;
}
}  // extern "C++"

int mcl3dl_particles_imu_update(mcl3dl_engine* eng, const float acc_measure[3], double acc_var, mcl3dl_update_summary* summary)
{
  if (!eng || eng->devs.size() != 1 || !acc_measure || !summary)
    return MCL3DL_ERR_INVALID_ARG;
  const float sigma = static_cast<float>(acc_var);  // ImuMeasurementModelGravity(const float acc_var)
  if (!(sigma > 0.0f) || !std::isfinite(sigma))
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (c.r_n == 0)
    return MCL3DL_ERR_INVALID_ARG;
  const ImuDev m = pf_imu_setup(acc_measure, sigma);
  const uint32_t n32 = static_cast<uint32_t>(c.r_n);
  return resident_likelihood_update(eng, c, summary, [&](mcl3dl_result* d_rec, float* lik) {
    return launch(eng, pf_imu_kernel, (n32 + 255) / 256, 256, 0, c.stream, static_cast<const PfState*>(c.r_states[c.r_cur].p), n32, m,
                  d_rec, lik);
  });
}

// ---- the landmark update, the odometry-error reset and the published poses on the resident set (pf_kernels.cuh)
int mcl3dl_particles_landmark_update(mcl3dl_engine* eng, const mcl3dl_landmark_params* params, mcl3dl_update_summary* summary)
{
  if (!eng || eng->devs.size() != 1 || !params || !summary)
    return MCL3DL_ERR_INVALID_ARG;
  const mcl3dl_pose& q = params->measured;
  const float pose[7] = {q.px, q.py, q.pz, q.qx, q.qy, q.qz, q.qw};
  for (float v : pose)
    if (!std::isfinite(v))
      return MCL3DL_ERR_INVALID_ARG;
  if (!std::isfinite(params->nd_a))
    return MCL3DL_ERR_INVALID_ARG;
  for (float v : params->sigma_inv)
    if (!std::isfinite(v))
      return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (c.r_n == 0)
    return MCL3DL_ERR_INVALID_ARG;
  LandmarkDev m;
  m.pos[0] = q.px;
  m.pos[1] = q.py;
  m.pos[2] = q.pz;
  m.rot = Q4{q.qx, q.qy, q.qz, q.qw};
  m.nd_a = params->nd_a;
  std::memcpy(m.sigma_inv, params->sigma_inv, sizeof(m.sigma_inv));
  const uint32_t n32 = static_cast<uint32_t>(c.r_n);
  return resident_likelihood_update(eng, c, summary, [&](mcl3dl_result* d_rec, float* lik) {
    return launch(eng, pf_landmark_kernel, (n32 + 255) / 256, 256, 0, c.stream, static_cast<const PfState*>(c.r_states[c.r_cur].p),
                  n32, m, d_rec, lik);
  });
}

int mcl3dl_particles_reset_odom_err_integ(mcl3dl_engine* eng)
{
  if (!eng || eng->devs.size() != 1)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (c.r_n == 0)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  const uint32_t n = static_cast<uint32_t>(c.r_n);
  CK(launch(eng, pf_reset_odom_err_kernel, (n + 255) / 256, 256, 0, c.stream, static_cast<PfState*>(c.r_states[c.r_cur].p), n));
  CK(cudaStreamSynchronize(c.stream));
  return MCL3DL_OK;
}

int mcl3dl_particles_get_poses(mcl3dl_engine* eng, mcl3dl_pose* out, size_t n)
{
  if (!eng || eng->devs.size() != 1 || !out)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (c.r_n == 0 || n != c.r_n)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  const uint32_t n32 = static_cast<uint32_t>(n);
  // r_poses (room for n poses since the set was sized) is the staging buffer; an update repacks it before it reads it
  CK(launch(eng, pf_poses_kernel, (n32 + 255) / 256, 256, 0, c.stream, static_cast<const PfState*>(c.r_states[c.r_cur].p), n32,
            static_cast<mcl3dl_pose*>(c.r_poses.p)));
  CK(cudaMemcpyAsync(out, c.r_poses.p, n * sizeof(mcl3dl_pose), cudaMemcpyDeviceToHost, c.stream));
  CK(cudaStreamSynchronize(c.stream));
  return MCL3DL_OK;
}

// ---- the initial seed of the resident set (pf_init_kernel): creates or replaces the set at count n
int mcl3dl_particles_init(mcl3dl_engine* eng, size_t n, const mcl3dl_init_params* params, uint64_t seed)
{
  if (!eng || eng->devs.size() != 1 || !params || n == 0 || n >= (size_t(1) << 31) ||
      (params->multivariate != 0 && params->multivariate != 1))
    return MCL3DL_ERR_INVALID_ARG;
  InitDev g;
  g.multivariate = params->multivariate;
  std::memcpy(g.mean, params->mean, sizeof(g.mean));
  std::memcpy(g.sigma, params->sigma, sizeof(g.sigma));
  std::memcpy(g.T, params->norm_transform, sizeof(g.T));
  for (float v : g.mean)
    if (!std::isfinite(v))
      return MCL3DL_ERR_INVALID_ARG;
  if (g.multivariate)
  {
    for (float v : g.T)
      if (!std::isfinite(v))
        return MCL3DL_ERR_INVALID_ARG;
  }
  else
  {
    for (float v : g.sigma)
      if (!finite_nonneg(v))
        return MCL3DL_ERR_INVALID_ARG;
  }
  DeviceCtx& c = eng->devs[0];
  CK(cudaSetDevice(c.dev));
  int rc;
  if ((rc = reserve_resident(eng, c, n)))
    return rc;
  const uint32_t n32 = static_cast<uint32_t>(n);
  ++c.r_init_calls;
  CK(launch(eng, pf_init_kernel, (n32 + 255) / 256, 256, 0, c.stream, static_cast<PfState*>(c.r_states[0].p),
            static_cast<float*>(c.r_prob.p), n32, seed, c.r_init_calls, g));
  CK(cudaStreamSynchronize(c.stream));
  c.r_n = n;
  c.r_cur = 0;
  return MCL3DL_OK;
}

// ---- resize and global localisation of the resident set (gl_kernels.cuh)
int mcl3dl_particles_resize(mcl3dl_engine* eng, size_t num)
{
  if (!eng || eng->devs.size() != 1 || num == 0 || num >= (size_t(1) << 31))
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (c.r_n == 0)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  const uint32_t n = static_cast<uint32_t>(c.r_n), num32 = static_cast<uint32_t>(num);
  float* accum = static_cast<float*>(c.r_accum.p);
  CK(launch(eng, pf_accum_kernel, 1, 32, 0, c.stream, static_cast<const float*>(c.r_prob.p), n, accum, accum + n));
  // the pick reads the current states and accum: they keep their storage until it has run
  int rc = reserve_resident(eng, c, num, {&c.r_states[c.r_cur], &c.r_accum});
  if (rc != MCL3DL_OK)
    return rc;
  float* pscan = static_cast<float*>(c.r_extra.p);
  CK(launch(eng, gl_pscan_kernel, 1, 32, 0, c.stream, accum, n, num32, pscan));
  CK(launch(eng, gl_resize_kernel, (num32 + 255) / 256, 256, 0, c.stream, static_cast<const PfState*>(c.r_states[c.r_cur].p), accum, n,
            pscan, num32, static_cast<PfState*>(c.r_states[1 - c.r_cur].p), static_cast<float*>(c.r_prob.p)));
  c.r_cur = 1 - c.r_cur;
  c.r_n = num;
  if ((rc = reserve_resident(eng, c, num)))  // now the other state buffer and accum as well
    return rc;
  CK(cudaStreamSynchronize(c.stream));
  return MCL3DL_OK;
}

int mcl3dl_global_localization(mcl3dl_engine* eng, const mcl3dl_point* pts, size_t n, const mcl3dl_global_localization_params* gp,
                               mcl3dl_global_localization_info* info)
{
  if (!eng || eng->devs.size() != 1 || !gp || !(gp->grid > 0.0) || !std::isfinite(gp->grid) || gp->div_yaw < 1 ||
      (pts && n >= (size_t(1) << 31)))
    return MCL3DL_ERR_INVALID_ARG;
  for (int k = 0; k < 3; ++k)
    if (!(gp->dist_weight[k] > 0.0f) || !std::isfinite(gp->dist_weight[k]))
      return MCL3DL_ERR_INVALID_ARG;
  if (!pts && !eng->has_map)
    return MCL3DL_ERR_NO_MAP;
  DeviceCtx& c = eng->devs[0];
  if (eng->has_map && c.w_on)
    return MCL3DL_ERR_TOO_LARGE;  // the seeds cover the whole map: no window holds them
  const size_t cnt = pts ? n : eng->n_points;
  mcl3dl_global_localization_info out{};
  out.n_input = cnt;
  if (info)
    *info = out;
  if (cnt == 0)
    return MCL3DL_OK;
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = c.stream;
  cudaEvent_t e0 = c.ev[0], e1 = c.ev[1];  // the per-update timing events, unused between calls
  // stage buffers of this call only: the uploaded cloud, the VoxelGrid's sort and scan buffers, the downsampled cloud,
  // the filter's CSR grid, the seeds, the yaw table, [0] downsampled / [1] seed counts
  DevBuf d_in, d_keys[2], d_vals[2], d_kl[2], d_flags, d_pos, d_tmp, d_ds, d_cell_start, d_grid, d_seeds, d_yaw, d_count, d_bbox;
  const uint32_t n32 = static_cast<uint32_t>(cnt);
  int rc;
  if ((rc = reserve(eng, d_keys[0], cnt * 4)) || (rc = reserve(eng, d_keys[1], cnt * 4)) || (rc = reserve(eng, d_vals[0], cnt * 4)) ||
      (rc = reserve(eng, d_vals[1], cnt * 4)) || (rc = reserve(eng, d_flags, cnt * 4)) || (rc = reserve(eng, d_pos, cnt * 4)) ||
      (rc = reserve(eng, d_ds, cnt * 16)) || (rc = reserve(eng, d_count, 64)) || (rc = reserve(eng, d_bbox, 12 * 4)) ||
      (pts && (rc = reserve(eng, d_in, cnt * 16))))
    return rc;
  CK(cudaEventRecord(e0, st));
  const mcl3dl_point* src = static_cast<const mcl3dl_point*>(c.raw_pts.p);
  if (pts)
  {
    CK(cudaMemcpyAsync(d_in.p, pts, cnt * 16, cudaMemcpyHostToDevice, st));
    src = static_cast<const mcl3dl_point*>(d_in.p);
  }
  uint32_t* count = static_cast<uint32_t*>(d_count.p);
  CK(cudaMemsetAsync(count, 0, 64, st));
  // 1. VoxelGrid at float(grid)
  const float g32 = static_cast<float>(gp->grid);
  const float leaf[3] = {g32, g32, g32};
  const VoxelBufs vb{{&d_keys[0], &d_keys[1]}, {&d_vals[0], &d_vals[1]}, {&d_kl[0], &d_kl[1]}, &d_flags, &d_pos, &d_tmp};
  bool filtered = false;
  if ((rc = voxel_grid(eng, c, st, src, n32, cnt, leaf, vb, static_cast<mcl3dl_point*>(d_ds.p), count, filtered)))
    return rc;
  const mcl3dl_point* ds = src;  // unfiltered (PCL's overflow rule): the cloud itself
  uint32_t n_ds = n32;
  if (filtered)
  {
    CK(cudaMemcpyAsync(&n_ds, count, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    ds = static_cast<const mcl3dl_point*>(d_ds.p);
  }
  out.n_downsampled = n_ds;
  if (n_ds == 0)
  {
    if (info)
      *info = out;
    return MCL3DL_OK;
  }
  // 2. free-space filter over a likelihood-style CSR grid of the downsampled cloud in the rescaled space
  const float wx = gp->dist_weight[0], wy = gp->dist_weight[1], wz = gp->dist_weight[2];
  const int nb = static_cast<int>((n_ds + 255) / 256);
  uint32_t h_bbox[12];
  for (int k = 0; k < 3; ++k)
  {
    h_bbox[k] = 0xffffffffu;
    h_bbox[3 + k] = 0u;
    h_bbox[6 + k] = 0xffffffffu;
    h_bbox[9 + k] = 0u;
  }
  CK(cudaMemcpyAsync(d_bbox.p, h_bbox, sizeof(h_bbox), cudaMemcpyHostToDevice, st));
  CK(launch(eng, bbox_kernel, std::min(nb, c.sm_count * 8), 256, 0, st, ds, n_ds, wx, wy, wz, static_cast<uint32_t*>(d_bbox.p)));
  CK(cudaMemcpyAsync(h_bbox, d_bbox.p, sizeof(h_bbox), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  float sc_min[3], sc_max[3];
  for (int k = 0; k < 3; ++k)
  {
    sc_min[k] = ord2f(h_bbox[6 + k]);
    sc_max[k] = ord2f(h_bbox[9 + k]);
    if (!std::isfinite(sc_min[k]) || !std::isfinite(sc_max[k]))
      return MCL3DL_ERR_TOO_LARGE;  // an infinite coordinate (only an unfiltered cloud keeps one): no finite lattice
  }
  GlDev m{};
  m.z_off = 0.01 + gp->grid;
  m.r2 = static_cast<float>(gp->grid * gp->grid);
  m.rpad = g32 * 1.0001f + 1e-6f;
  NnGridDev g{};
  g.wx = wx;
  g.wy = wy;
  g.wz = wz;
  size_t cells = 0;
  // the window (q -/+ rpad) spans at most 3 cells per axis: cell edge strictly above rpad (1 % margin, as for the map)
  if (!nn_lattice(m.rpad * 1.01f, sc_min, sc_max, g, cells))
    return MCL3DL_ERR_TOO_LARGE;
  if ((rc = reserve(eng, d_cell_start, (cells + 1) * 4)) || (rc = reserve(eng, d_grid, static_cast<size_t>(n_ds) * 16)) ||
      (rc = reserve(eng, d_seeds, static_cast<size_t>(n_ds) * 16)))
    return rc;
  uint32_t* const keys[2] = {static_cast<uint32_t*>(d_keys[0].p), static_cast<uint32_t*>(d_keys[1].p)};
  uint32_t* const vals[2] = {static_cast<uint32_t*>(d_vals[0].p), static_cast<uint32_t*>(d_vals[1].p)};
  if ((rc = build_nn_csr(eng, st, ds, n_ds, g, cells, keys, vals, d_tmp, static_cast<uint32_t*>(d_cell_start.p),
                         static_cast<float4*>(d_grid.p))))
    return rc;
  g.cell_start = static_cast<const uint32_t*>(d_cell_start.p);
  g.pts = static_cast<const float4*>(d_grid.p);
  uint32_t* flags = static_cast<uint32_t*>(d_flags.p);
  uint32_t* pos = static_cast<uint32_t*>(d_pos.p);
  CK(launch(eng, gl_flag_kernel, nb, 256, 0, st, ds, n_ds, g, m, flags));
  CK(cub_call(eng, d_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, flags, pos, n_ds, st); }));
  CK(launch(eng, scan_compact_kernel, nb, 256, 0, st, ds, flags, pos, n_ds, static_cast<mcl3dl_point*>(d_seeds.p), count + 1));
  uint32_t n_seeds = 0;
  CK(cudaMemcpyAsync(&n_seeds, count + 1, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  out.n_seeds = n_seeds;
  if (n_seeds == 0)
  {
    if (info)
      *info = out;
    return MCL3DL_OK;  // documented departure: the set stays as it was
  }
  const uint64_t n_particles = static_cast<uint64_t>(n_seeds) * static_cast<uint64_t>(gp->div_yaw);
  if (n_particles >= (uint64_t(1) << 31))
    return MCL3DL_ERR_TOO_LARGE;
  // 3. the particles: yaw table from the host, one thread per particle
  std::vector<Q4> yaw(static_cast<size_t>(gp->div_yaw));
  gl_yaw_quats(gp->div_yaw, gp->imu_quat, yaw.data());
  if ((rc = reserve(eng, d_yaw, yaw.size() * sizeof(Q4))))
    return rc;
  CK(cudaMemcpyAsync(d_yaw.p, yaw.data(), yaw.size() * sizeof(Q4), cudaMemcpyHostToDevice, st));
  if ((rc = reserve_resident(eng, c, n_particles)))
    return rc;
  const float prob = gl_probability(n_seeds);
  const uint32_t np32 = static_cast<uint32_t>(n_particles);
  CK(launch(eng, gl_fill_kernel, (np32 + 255) / 256, 256, 0, st, static_cast<const mcl3dl_point*>(d_seeds.p),
            static_cast<const Q4*>(d_yaw.p), static_cast<uint32_t>(gp->div_yaw), np32, prob, static_cast<PfState*>(c.r_states[0].p),
            static_cast<float*>(c.r_prob.p)));
  CK(cudaEventRecord(e1, st));
  CK(cudaStreamSynchronize(st));
  c.r_n = n_particles;
  c.r_cur = 0;
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  out.n_particles = n_particles;
  out.probability = prob;
  out.build_ms = ms;
  if (info)
    *info = out;
  return MCL3DL_OK;
}

// The resident update with every input already on the device: pose pack -> both models -> prior * likelihood * odometry
// term -> normalise; one synchronise.  `s`: the pinned block's layout, whose inputs are already on their way up.
static int resident_update(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_point* d_lik, size_t n_lik, const mcl3dl_point* d_beam,
                           size_t n_beam, const float* d_org, size_t n_origins, float odom_err_lin_sigma, const Share& s,
                           mcl3dl_update_summary* summary)
{
  const size_t P = c.r_n;
  cudaStream_t st = c.stream;
  int rc = reserve(eng, c.d_out, P * sizeof(mcl3dl_result));
  if (rc != MCL3DL_OK)
    return rc;
  // NormalLikelihood(sigma): a_ = float(1 / sqrt(2 pi s^2)), sq2_ = float(2 s^2) (include/mcl_3dl/nd.h:45-49)
  const bool with_odom = odom_err_lin_sigma > 0.0f;
  const double sg = static_cast<double>(odom_err_lin_sigma);
  const float nd_a = with_odom ? static_cast<float>(1.0 / std::sqrt(2.0 * M_PI * sg * sg)) : 1.0f;
  const float nd_sq2 = with_odom ? static_cast<float>(sg * sg * 2.0) : 1.0f;
  const uint32_t n32 = static_cast<uint32_t>(P);
  CK(launch(eng, pf_pack_kernel, (n32 + 255) / 256, 256, 0, st, static_cast<const PfState*>(c.r_states[c.r_cur].p), n32, nd_a, nd_sq2,
            static_cast<mcl3dl_pose*>(c.r_poses.p), with_odom ? static_cast<float*>(c.r_extra.p) : nullptr));
  // (the pack writes only the packed poses and factors: a refused window leaves the resident set as it was)
  if ((rc = ensure_window(eng, c, static_cast<const mcl3dl_pose*>(c.r_poses.p), P, d_lik, n_lik, d_beam, n_beam, d_org, n_origins,
                          measure_search(eng, c, n_lik, n_beam))))
    return rc;
  mcl3dl_result* d_rec = static_cast<mcl3dl_result*>(c.d_out.p);
  rc = launch_models(eng, c, static_cast<const mcl3dl_pose*>(c.r_poses.p), P, d_lik, n_lik, d_beam, n_beam, d_org, n_origins,
                     d_rec, nullptr, st, false);
  if (rc != MCL3DL_OK)
    return rc;
  // prior * likelihood from the resident probabilities; the posterior is written over them (the weights were read
  // into d_w first); a vanished total leaves them untouched = the reference's "restore" (pf.h:274-278)
  float* prob = static_cast<float*>(c.r_prob.p);
  WeightPartial* h_part = reinterpret_cast<WeightPartial*>(static_cast<char*>(c.h_pinned.p) + s.o_part);
  rc = fold_weights(eng, c, d_rec, prob, with_odom ? static_cast<const float*>(c.r_extra.p) : nullptr, prob, P, n_lik, 0, h_part,
                    nullptr);
  if (rc != MCL3DL_OK)
    return rc;
  CK(cudaStreamSynchronize(st));
  make_summary(h_part[0], h_part[1], summary);
  return MCL3DL_OK;
}

int mcl3dl_particles_measure_update(mcl3dl_engine* eng, const mcl3dl_point* lik_pts, size_t n_lik, const mcl3dl_point* beam_pts,
                                    size_t n_beam, const float* origins_xyz, size_t n_origins, float odom_err_lin_sigma,
                                    mcl3dl_update_summary* summary)
{
  if (!eng || eng->devs.size() != 1 || !summary)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  const size_t P = c.r_n;
  int rc = validate_measure(eng, P, lik_pts, n_lik, beam_pts, n_beam, origins_xyz, n_origins, true);
  if (rc != MCL3DL_OK)
    return rc;
  if (P == 0)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  // scans + origins up in one block (as in mcl3dl_measure); the poses come from the resident states
  const Share s = share_of(P, 1, 0, 0, n_lik, n_beam, n_origins, 0, 0, 0, 0, 0);
  if ((rc = reserve(eng, c.h_pinned, s.total)) || (rc = reserve(eng, c.d_poses, s.in_bytes)) ||
      (rc = stage_inputs(eng, c, s, nullptr, lik_pts, beam_pts, origins_xyz, n_origins, nullptr, nullptr, false)))
    return rc;
  const char* d_in = static_cast<const char*>(c.d_poses.p);
  return resident_update(eng, c, reinterpret_cast<const mcl3dl_point*>(d_in + s.o_lik), n_lik,
                         reinterpret_cast<const mcl3dl_point*>(d_in + s.o_beam), n_beam,
                         reinterpret_cast<const float*>(d_in + s.o_org), n_origins, odom_err_lin_sigma, s, summary);
}

int mcl3dl_particles_measure_update_prepared(mcl3dl_engine* eng, const float* origins_xyz, size_t n_origins, float odom_err_lin_sigma,
                                             mcl3dl_update_summary* summary)
{
  if (!eng || eng->devs.size() != 1 || !summary)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (!c.s_valid)
    return MCL3DL_ERR_INVALID_ARG;  // no mcl3dl_scan_prepare before
  const size_t P = c.r_n, n_lik = c.s_info.n_lik, n_beam = c.s_info.n_beam;
  const mcl3dl_point* d_lik = static_cast<const mcl3dl_point*>(c.s_out[0].p);
  const mcl3dl_point* d_beam = static_cast<const mcl3dl_point*>(c.s_out[1].p);
  int rc = validate_measure(eng, P, d_lik, n_lik, d_beam, n_beam, origins_xyz, n_origins, false);
  if (rc != MCL3DL_OK)
    return rc;
  if (P == 0)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  // only the origins go up; the scans are the prepared ones
  const Share s = share_of(P, 1, 0, 0, 0, 0, n_origins, 0, 0, 0, 0, 0);
  if ((rc = reserve(eng, c.h_pinned, s.total)) || (rc = reserve(eng, c.d_poses, s.in_bytes)) ||
      (rc = stage_inputs(eng, c, s, nullptr, nullptr, nullptr, origins_xyz, n_origins, nullptr, nullptr, false)))
    return rc;
  // (beam labels are the raw cloud's, voted per voxel: the caller's origins must cover them, as in the node)
  return resident_update(eng, c, d_lik, n_lik, d_beam, n_beam, static_cast<const float*>(c.d_poses.p), n_origins, odom_err_lin_sigma,
                         s, summary);
}

// ---- scan preprocessing on the device (scan_kernels.cuh)
// mcl3dl_scan_prepare from its raw cloud on: `fill(st)` writes the n_raw (< 2^30) raw points into c.s_raw on the stream
// (a host upload, or the accumulation's transform), then VoxelGrid, clip, uniform sample and the counts
extern "C++" {
template <typename Fill>
static int scan_prepare_from(mcl3dl_engine* eng, DeviceCtx& c, size_t n_raw, const mcl3dl_scan_params* sp, mcl3dl_scan_info* info,
                             Fill fill)
{
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = c.stream;
  c.s_valid = false;
  c.n_valid = false;
  c.s_info = mcl3dl_scan_info{};
  c.s_info.n_raw = static_cast<uint32_t>(n_raw);
  const uint32_t n = static_cast<uint32_t>(n_raw);
  const uint32_t num[2] = {sp->lik_num_points, sp->beam_num_points};
  int rc;
  const size_t cap = std::max<size_t>(n_raw, 1);
  if ((rc = reserve(eng, c.s_raw, cap * 16)) || (rc = reserve(eng, c.s_ds, cap * 16)) || (rc = reserve(eng, c.s_counts, 64)) ||
      (rc = reserve(eng, c.s_out[0], std::max<size_t>(num[0], 1) * 16)) || (rc = reserve(eng, c.s_out[1], std::max<size_t>(num[1], 1) * 16)))
    return rc;
  for (int k = 0; k < 2; ++k)
    if ((rc = reserve(eng, c.s_keys[k], cap * 4)) || (rc = reserve(eng, c.s_vals[k], cap * 4)) || (rc = reserve(eng, c.s_flags[k], cap * 4)) ||
        (rc = reserve(eng, c.s_pos[k], cap * 4)) || (rc = reserve(eng, c.s_clip[k], cap * 16)))
      return rc;
  uint32_t* counts = static_cast<uint32_t*>(c.s_counts.p);  // [0] downsampled, [1] [2] clipped, [3] [4] sampled
  CK(cudaMemsetAsync(counts, 0, 64, st));
  if (n == 0)
  {
    c.s_valid = true;
    if (info) *info = c.s_info;
    return MCL3DL_OK;
  }
  if ((rc = reserve(eng, c.h_pinned, 256)))
    return rc;
  if ((rc = fill(st)))
    return rc;
  const mcl3dl_point* d_raw = static_cast<const mcl3dl_point*>(c.s_raw.p);
  const mcl3dl_point* d_ds = d_raw;
  const int nb = static_cast<int>((n + 255) / 256);
  const bool downsample = sp->downsample[0] > 0.0f && sp->downsample[1] > 0.0f && sp->downsample[2] > 0.0f;
  bool ds_done = false;
  if (downsample)
  {
    const VoxelBufs vb{{&c.s_keys[0], &c.s_keys[1]}, {&c.s_vals[0], &c.s_vals[1]}, {&c.s_key_label[0], &c.s_key_label[1]},
                       &c.s_flags[0], &c.s_pos[0], &c.s_tmp};
    if ((rc = voxel_grid(eng, c, st, d_raw, n, cap, sp->downsample, vb, static_cast<mcl3dl_point*>(c.s_ds.p), counts + 0, ds_done)))
      return rc;
    d_ds = static_cast<const mcl3dl_point*>(c.s_ds.p);
  }
  if (!ds_done)
  {
    CK(cudaMemcpyAsync(c.s_ds.p, c.s_raw.p, n_raw * 16, cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(counts, &c.s_info.n_raw, 4, cudaMemcpyHostToDevice, st));
    d_ds = static_cast<const mcl3dl_point*>(c.s_ds.p);
  }
  // clip (both models at once), compaction in order, then the uniform sample
  const ClipDev ca = scan_clip_window(sp->lik_clip_near, sp->lik_clip_far, sp->lik_clip_z_min, sp->lik_clip_z_max);
  const ClipDev cb = scan_clip_window(sp->beam_clip_near, sp->beam_clip_far, sp->beam_clip_z_min, sp->beam_clip_z_max);
  uint32_t *fa = static_cast<uint32_t*>(c.s_flags[0].p), *fb = static_cast<uint32_t*>(c.s_flags[1].p);
  uint32_t *pa = static_cast<uint32_t*>(c.s_pos[0].p), *pb = static_cast<uint32_t*>(c.s_pos[1].p);
  CK(launch(eng, scan_clip_flags_kernel, nb, 256, 0, st, d_ds, counts + 0, ca, cb, fa, fb, n));
  CK(cub_call(eng, c.s_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, fa, pa, n, st); }));
  CK(cub_call(eng, c.s_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, fb, pb, n, st); }));
  CK(launch(eng, scan_compact_kernel, nb, 256, 0, st, d_ds, fa, pa, n, static_cast<mcl3dl_point*>(c.s_clip[0].p), counts + 1));
  CK(launch(eng, scan_compact_kernel, nb, 256, 0, st, d_ds, fb, pb, n, static_cast<mcl3dl_point*>(c.s_clip[1].p), counts + 2));
  for (int k = 0; k < 2; ++k)
    if (num[k])
      CK(launch(eng, scan_sample_kernel, (num[k] + 255) / 256, 256, 0, st, static_cast<const mcl3dl_point*>(c.s_clip[k].p),
                counts + 1 + k, num[k], sp->seed, static_cast<uint32_t>(k), static_cast<mcl3dl_point*>(c.s_out[k].p),
                counts + 3 + k));
  uint32_t h_counts[5];
  CK(cudaMemcpyAsync(c.h_pinned.p, counts, sizeof(h_counts), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  std::memcpy(h_counts, c.h_pinned.p, sizeof(h_counts));
  c.s_info.n_downsampled = h_counts[0];
  c.s_info.n_lik_clipped = h_counts[1];
  c.s_info.n_beam_clipped = h_counts[2];
  c.s_info.n_lik = h_counts[3];
  c.s_info.n_beam = h_counts[4];
  c.s_valid = true;
  if (info) *info = c.s_info;
  return MCL3DL_OK;
}
}  // extern "C++"

int mcl3dl_scan_prepare(mcl3dl_engine* eng, const mcl3dl_point* raw, size_t n_raw, const mcl3dl_scan_params* sp, mcl3dl_scan_info* info)
{
  if (!eng || eng->devs.size() != 1 || !sp || (n_raw && !raw) || n_raw >= (size_t(1) << 30))
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  return scan_prepare_from(eng, c, n_raw, sp, info, [&](cudaStream_t st) -> int {
    CK(cudaMemcpyAsync(c.s_raw.p, raw, n_raw * 16, cudaMemcpyHostToDevice, st));
    return MCL3DL_OK;
  });
}

// ---- cloud accumulation (scan_kernels.cuh: accum_*_kernel)
int mcl3dl_scan_accumulate(mcl3dl_engine* eng, const mcl3dl_cloud_view* v, const mcl3dl_transform* tf, uint32_t* n_clouds_out)
{
  if (!eng || eng->devs.size() != 1 || !v || !v->data || !tf)
    return MCL3DL_ERR_INVALID_ARG;
  const uint64_t n = static_cast<uint64_t>(v->width) * v->height;
  if (n == 0 || static_cast<uint64_t>(v->row_step) < static_cast<uint64_t>(v->width) * v->point_step)
    return MCL3DL_ERR_INVALID_ARG;
  for (int k = 0; k < 3; ++k)
    if (static_cast<uint64_t>(v->offset[k]) + 4 > v->point_step)
      return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  const uint64_t total = c.a_n + n;
  if (total >= (uint64_t(1) << 30))
    return MCL3DL_ERR_TOO_LARGE;
  // the bytes the points span (the last row ends at its last point)
  const size_t bytes = static_cast<size_t>(v->height - 1) * v->row_step + static_cast<size_t>(v->width) * v->point_step;
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = c.stream;
  int rc;
  if (!c.a_pts.p || total * 16 > c.a_pts.cap)
  {
    // reserve() drops the contents: grow into a new buffer and carry the accumulated points over on the device
    DevBuf grown;
    if ((rc = reserve(eng, grown, std::max<uint64_t>(total, std::min<uint64_t>(2 * c.a_n, uint64_t(1) << 30)) * 16)))
      return rc;
    if (c.a_n)
      CK(cudaMemcpyAsync(grown.p, c.a_pts.p, c.a_n * 16, cudaMemcpyDeviceToDevice, st));
    CK(cudaStreamSynchronize(st));
    c.a_pts = std::move(grown);
  }
  if ((rc = reserve(eng, c.a_raw, bytes)))
    return rc;
  CK(cudaMemcpyAsync(c.a_raw.p, v->data, bytes, cudaMemcpyHostToDevice, st));
  const uint32_t n32 = static_cast<uint32_t>(n);
  const double* t = tf->translation;
  const double* q = tf->rotation;
  CK(launch(eng, accum_cloud_kernel, (n32 + 255) / 256, 256, 0, st, static_cast<const unsigned char*>(c.a_raw.p), v->width, n32,
            v->row_step, v->point_step, v->offset[0], v->offset[1], v->offset[2], t[0], t[1], t[2], q[0], q[1], q[2], q[3], c.a_clouds,
            static_cast<mcl3dl_point*>(c.a_pts.p) + c.a_n));
  CK(cudaStreamSynchronize(st));  // the caller may reuse data as soon as this returns
  c.a_n = total;
  c.a_clouds++;
  c.a_dense = c.a_dense && v->is_dense;
  if (n_clouds_out)
    *n_clouds_out = c.a_clouds;
  return MCL3DL_OK;
}

int mcl3dl_scan_accumulate_clear(mcl3dl_engine* eng)
{
  if (!eng || eng->devs.size() != 1)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  c.a_n = 0;
  c.a_clouds = 0;
  c.a_dense = true;
  return MCL3DL_OK;
}

int mcl3dl_scan_accumulated_get(mcl3dl_engine* eng, mcl3dl_point* out, size_t capacity, size_t* n_out)
{
  if (!eng || eng->devs.size() != 1 || !n_out)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  *n_out = c.a_n;
  if (!out || c.a_n == 0)
    return MCL3DL_OK;
  if (capacity < c.a_n)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  CK(cudaMemcpyAsync(out, c.a_pts.p, c.a_n * 16, cudaMemcpyDeviceToHost, c.stream));
  CK(cudaStreamSynchronize(c.stream));
  return MCL3DL_OK;
}

int mcl3dl_scan_prepare_accumulated(mcl3dl_engine* eng, const mcl3dl_transform* tf, const mcl3dl_scan_params* sp, mcl3dl_scan_info* info)
{
  if (!eng || eng->devs.size() != 1 || !tf || !sp)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (c.a_clouds == 0)
    return MCL3DL_ERR_INVALID_ARG;  // "MCL measure function is called without available pointcloud" (:312-316)
  const uint32_t n = static_cast<uint32_t>(c.a_n);
  return scan_prepare_from(eng, c, c.a_n, sp, info, [&](cudaStream_t st) -> int {
    const double* t = tf->translation;
    const double* q = tf->rotation;
    CK(launch(eng, accum_transform_kernel, (n + 255) / 256, 256, 0, st, static_cast<const mcl3dl_point*>(c.a_pts.p), n, t[0], t[1], t[2],
              q[0], q[1], q[2], q[3], c.a_dense ? 1 : 0, static_cast<mcl3dl_point*>(c.s_raw.p)));
    return MCL3DL_OK;
  });
}

int mcl3dl_scan_get(mcl3dl_engine* eng, int which, mcl3dl_point* out, size_t capacity, size_t* n_out)
{
  if (!eng || eng->devs.size() != 1 || which < 0 || which > 4 || !n_out)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (!c.s_valid)
    return MCL3DL_ERR_INVALID_ARG;
  const uint32_t n[5] = {c.s_info.n_downsampled, c.s_info.n_lik_clipped, c.s_info.n_beam_clipped, c.s_info.n_lik, c.s_info.n_beam};
  const DevBuf* src[5] = {&c.s_ds, &c.s_clip[0], &c.s_clip[1], &c.s_out[0], &c.s_out[1]};
  *n_out = n[which];
  if (!out || n[which] == 0)
    return MCL3DL_OK;
  if (capacity < n[which])
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  CK(cudaMemcpyAsync(out, src[which]->p, static_cast<size_t>(n[which]) * 16, cudaMemcpyDeviceToHost, c.stream));
  CK(cudaStreamSynchronize(c.stream));
  return MCL3DL_OK;
}

// ---- PointCloudSamplerWithNormal on the prepared clipped clouds (scan_kernels.cuh: ns_*_kernel)
int mcl3dl_scan_sample_with_normal(mcl3dl_engine* eng, const mcl3dl_normal_sampler_params* p, mcl3dl_normal_sampler_info* info)
{
  if (!eng || !p || eng->devs.size() != 1)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (!c.s_valid)
    return MCL3DL_ERR_INVALID_ARG;  // no mcl3dl_scan_prepare before
  const double r = p->normal_search_range;
  bool ok = std::isfinite(r) && r > 0.0 && std::isfinite(p->max_weight) && p->max_weight > 0.0 &&
            std::isfinite(p->perform_weighting_ratio) && std::isfinite(p->max_weight_ratio);
  for (int k = 0; k < 3; ++k)
    ok = ok && std::isfinite(p->eigen_values[k]) && std::isfinite(p->eigen_vector[k]);
  for (int k = 0; k < 4; ++k)
    ok = ok && std::isfinite(p->mean_rot[k]);
  if (!ok)
    return MCL3DL_ERR_INVALID_ARG;
  mcl3dl_normal_sampler_info out{};
  int shift = 0;
  ns_host_consts(*p, &out.max_weight, out.fpc_local, &shift);
  out.weight_shift = shift;
  const double scale = std::ldexp(1.0, shift);
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = c.stream;
  const uint32_t n[2] = {c.s_info.n_lik_clipped, c.s_info.n_beam_clipped};
  const uint32_t num[2] = {p->lik_num_points, p->beam_num_points};
  int rc;
  if ((rc = reserve(eng, c.n_word, 256)) || (rc = reserve(eng, c.h_pinned, 256)))
    return rc;
  uint32_t* word = static_cast<uint32_t*>(c.n_word.p);
  // both clouds' neighbour grids first, so that TOO_LARGE leaves everything as it was
  uint32_t h_bbox[12];
  for (int k = 0; k < 12; ++k)
    h_bbox[k] = k % 6 < 3 ? 0xffffffffu : 0u;  // per model: minimum (x y z), maximum (x y z)
  CK(cudaMemcpyAsync(word, h_bbox, sizeof(h_bbox), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(word + 12, 0, 8, st));
  for (int k = 0; k < 2; ++k)
    if (n[k])
    {
      const int nb = static_cast<int>((n[k] + 255) / 256);
      CK(launch(eng, scan_bbox_kernel, std::min(nb, c.sm_count * 8), 256, 0, st, static_cast<const mcl3dl_point*>(c.s_clip[k].p), n[k],
                word + 6 * k));
    }
  CK(cudaMemcpyAsync(h_bbox, word, sizeof(h_bbox), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  NsGridDev ng[2] = {};
  int end_bit[2] = {1, 1};
  for (int k = 0; k < 2; ++k)
  {
    ng[k].r2 = static_cast<float>(r * r);
    const float mn[3] = {ord2f(h_bbox[6 * k]), ord2f(h_bbox[6 * k + 1]), ord2f(h_bbox[6 * k + 2])};
    const float mx[3] = {ord2f(h_bbox[6 * k + 3]), ord2f(h_bbox[6 * k + 4]), ord2f(h_bbox[6 * k + 5])};
    float edge = 0.0f;
    // no finite point: the zero lattice keys every point as non-finite (key 0 == cells)
    if (n[k] && mn[0] <= mx[0] && !ns_lattice(r, mn, mx, ng[k].g, end_bit[k], edge))
      return MCL3DL_ERR_TOO_LARGE;
  }
  c.n_valid = false;
  uint32_t n_sample[2];
  for (int k = 0; k < 2; ++k)
    if ((rc = ns_sample_model(eng, c, k, n[k], ng[k], end_bit[k], out.fpc_local, out.max_weight, scale, num[k], p->seed, n_sample + k,
                              out.rounds + k, out.draws + k)))
      return rc;
  CK(cudaMemcpyAsync(c.h_pinned.p, word + 12, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  std::memcpy(out.n_normal, c.h_pinned.p, 8);
  // the new samples replace the prepared ones
  std::swap(c.s_out[0], c.n_out[0]);
  std::swap(c.s_out[1], c.n_out[1]);
  out.n_lik = n_sample[0];
  out.n_beam = n_sample[1];
  c.s_info.n_lik = n_sample[0];
  c.s_info.n_beam = n_sample[1];
  c.n_valid = true;
  if (info)
    *info = out;
  return MCL3DL_OK;
}

int mcl3dl_scan_normals(mcl3dl_engine* eng, int which, float* normals_xyz, uint32_t* n_neighbours, uint64_t* weights_q, size_t capacity,
                        size_t* n_out)
{
  if (!eng || eng->devs.size() != 1 || which < 0 || which > 1 || !n_out)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (!c.s_valid || !c.n_valid)
    return MCL3DL_ERR_INVALID_ARG;
  const uint32_t n = which ? c.s_info.n_beam_clipped : c.s_info.n_lik_clipped;
  *n_out = n;
  if (n == 0 || (!normals_xyz && !n_neighbours && !weights_q))
    return MCL3DL_OK;
  if (capacity < n)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  if (normals_xyz)
    CK(cudaMemcpyAsync(normals_xyz, c.n_normals[which].p, size_t(n) * 12, cudaMemcpyDeviceToHost, c.stream));
  if (n_neighbours)
    CK(cudaMemcpyAsync(n_neighbours, c.n_nb[which].p, size_t(n) * 4, cudaMemcpyDeviceToHost, c.stream));
  if (weights_q)
    CK(cudaMemcpyAsync(weights_q, c.n_q[which].p, size_t(n) * 8, cudaMemcpyDeviceToHost, c.stream));
  CK(cudaStreamSynchronize(c.stream));
  return MCL3DL_OK;
}

int mcl3dl_match_output(mcl3dl_engine* eng, const mcl3dl_pose* pose, const mcl3dl_point* pts, size_t n, const mcl3dl_match_params* mp,
                        mcl3dl_point* matched, size_t* n_matched, mcl3dl_point* unmatched, size_t* n_unmatched)
{
  if (!eng || !pose || !mp || !n_matched || !n_unmatched)
    return MCL3DL_ERR_INVALID_ARG;
  if (!eng->has_map)
    return MCL3DL_ERR_NO_MAP;
  // radiusSearch takes the radius as a float and throws above the chunk length (chunked_kdtree.h:218-225)
  const float r = static_cast<float>(mp->unmatch_output_dist);
  if (!eng->has_lik || !(mp->chunk_length > 0.0f) || r > mp->chunk_length)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  const mcl3dl_point* src = pts;
  size_t cnt = n;
  if (!pts)
  {
    if (eng->devs.size() != 1 || !c.s_valid)
      return MCL3DL_ERR_INVALID_ARG;
    src = static_cast<const mcl3dl_point*>(c.s_ds.p);
    cnt = c.s_info.n_downsampled;
  }
  if (cnt >= (size_t(1) << 30))
    return MCL3DL_ERR_INVALID_ARG;
  *n_matched = 0;
  *n_unmatched = 0;
  if (cnt == 0)
    return MCL3DL_OK;
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = c.stream;
  const uint32_t n32 = static_cast<uint32_t>(cnt);
  int rc;
  if ((rc = reserve(eng, c.m_tf, cnt * 16)) || (pts && (rc = reserve(eng, c.m_in, cnt * 16))))
    return rc;
  for (int k = 0; k < 2; ++k)
    if ((rc = reserve(eng, c.m_flags[k], cnt * 4)) || (rc = reserve(eng, c.m_pos[k], cnt * 4)))
      return rc;
  // page-locked result block: [2 counts | 56 B pad | matched cloud | unmatched cloud], written by the compaction itself so
  // that one synchronise ends the call
  if ((rc = reserve(eng, c.m_host, 64 + 2 * cnt * 16)))
    return rc;
  if (pts)
  {
    CK(cudaMemcpyAsync(c.m_in.p, pts, cnt * 16, cudaMemcpyHostToDevice, st));
    src = static_cast<const mcl3dl_point*>(c.m_in.p);
  }
  MatchDev m{};
  m.raw_pts = static_cast<const float4*>(c.raw_pts.p);
  m.r2 = static_cast<float>(static_cast<double>(r) * static_cast<double>(r));
  m.rpad = r * 1.0001f + 1e-6f;
  m.match_sq = mp->match_output_dist * mp->match_output_dist;
  m.chunk_length = mp->chunk_length;
  m.pos_to_chunk = static_cast<float>(1.0 / static_cast<double>(mp->chunk_length));
  m.max_search_radius = mp->max_search_radius;
  const WinSearch ms{m.rpad, 0.0f, 0.0f};
  if ((rc = ensure_window(eng, c, nullptr, 0, src, cnt, nullptr, 0, nullptr, 0, ms, pose)))
    return rc;
  uint32_t* f[2] = {static_cast<uint32_t*>(c.m_flags[0].p), static_cast<uint32_t*>(c.m_flags[1].p)};
  uint32_t* ps[2] = {static_cast<uint32_t*>(c.m_pos[0].p), static_cast<uint32_t*>(c.m_pos[1].p)};
  mcl3dl_point* tf = static_cast<mcl3dl_point*>(c.m_tf.p);
  const int nb = static_cast<int>((cnt + 255) / 256);
  CK(launch(eng, match_classify_kernel, nb, 256, 0, st, src, n32, *pose, c.nn, m, tf, f[0], f[1]));
  char* hp = static_cast<char*>(c.m_host.p);
  uint32_t* h_counts = reinterpret_cast<uint32_t*>(hp);
  mcl3dl_point* h_out[2] = {reinterpret_cast<mcl3dl_point*>(hp + 64), reinterpret_cast<mcl3dl_point*>(hp + 64 + cnt * 16)};
  for (int k = 0; k < 2; ++k)
  {
    CK(cub_call(eng, c.m_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, f[k], ps[k], n32, st); }));
    CK(launch(eng, scan_compact_kernel, nb, 256, 0, st, tf, f[k], ps[k], n32, h_out[k], h_counts + k));
  }
  CK(cudaStreamSynchronize(st));
  *n_matched = h_counts[0];
  *n_unmatched = h_counts[1];
  if (matched)
    std::memcpy(matched, h_out[0], *n_matched * 16);
  if (unmatched)
    std::memcpy(unmatched, h_out[1], *n_unmatched * 16);
  return MCL3DL_OK;
}

int mcl3dl_particles_estimate(mcl3dl_engine* eng, const mcl3dl_pose* prev, float bias_var_dist, float bias_var_ang,
                              mcl3dl_estimate* out)
{
  if (!eng || eng->devs.size() != 1 || !out)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (c.r_n == 0)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = c.stream;
  const uint32_t n = static_cast<uint32_t>(c.r_n);
  const int grid = static_cast<int>(std::min<size_t>((c.r_n + 255) / 256, static_cast<size_t>(c.sm_count) * 4));
  const size_t part_doubles = static_cast<size_t>(grid) * (kEstSums + 2);
  const size_t hdr = (sizeof(EstHeader) + 255) & ~size_t(255);
  int rc;
  if ((rc = reserve(eng, c.r_est, hdr + part_doubles * sizeof(double))) || (rc = reserve(eng, c.h_pinned, sizeof(EstHeader) + sizeof(PfState) + 64)))
    return rc;
  BiasDev b{};
  if (prev)
  {
    b.enabled = 1;
    b.prev_pos[0] = prev->px;
    b.prev_pos[1] = prev->py;
    b.prev_pos[2] = prev->pz;
    // state_prev_.rot_.inv() = conj() / dot(*this), quat.h:187-190 (operator/(s) multiplies by float(1.0 / s))
    const float d = prev->qx * prev->qx + prev->qy * prev->qy + prev->qz * prev->qz + prev->qw * prev->qw;
    const float id = static_cast<float>(1.0 / d);
    b.prev_inv = Q4{-prev->qx * id, -prev->qy * id, -prev->qz * id, prev->qw * id};
    // NormalLikelihood<float>(sigma): a_ = float(1 / sqrt(2 pi s^2)), sq2_ = float(2 s^2), nd.h:45-49
    const double sl = bias_var_dist, sa = bias_var_ang;
    b.lin_a = static_cast<float>(1.0 / std::sqrt(2.0 * M_PI * sl * sl));
    b.lin_sq2 = static_cast<float>(sl * sl * 2.0);
    b.ang_a = static_cast<float>(1.0 / std::sqrt(2.0 * M_PI * sa * sa));
    b.ang_sq2 = static_cast<float>(sa * sa * 2.0);
  }
  EstHeader* h = static_cast<EstHeader*>(c.r_est.p);
  double* parts = reinterpret_cast<double*>(static_cast<char*>(c.r_est.p) + hdr);
  const PfState* states = static_cast<const PfState*>(c.r_states[c.r_cur].p);
  const float* probs = static_cast<const float*>(c.r_prob.p);
  CK(launch(eng, pf_est_pass1_kernel, grid, 256, 0, st, states, probs, n, b, parts));
  CK(launch(eng, pf_est_finish1_kernel, 1, 32, 0, st, parts, grid, h));
  CK(launch(eng, pf_est_pass2_kernel, grid, 256, 0, st, states, probs, n, h, parts));
  CK(launch(eng, pf_est_finish2_kernel, 1, 32, 0, st, parts, grid, h));
  char* hp = static_cast<char*>(c.h_pinned.p);
  CK(cudaMemcpyAsync(hp, h, sizeof(EstHeader), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  EstHeader hh;
  std::memcpy(&hh, hp, sizeof(hh));
  // the state of the best particle (one 68-byte read, after the index is known)
  PfState best{};
  if (hh.max_index < n)
  {
    CK(cudaMemcpyAsync(hp + sizeof(EstHeader), states + hh.max_index, sizeof(PfState), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    std::memcpy(&best, hp + sizeof(EstHeader), sizeof(best));
  }
  std::memset(out, 0, sizeof(*out));
  out->mean_biased = mcl3dl_pose{hh.mean_b_pos[0], hh.mean_b_pos[1], hh.mean_b_pos[2], 0.0f,
                                 hh.mean_b_rot[0], hh.mean_b_rot[1], hh.mean_b_rot[2], hh.mean_b_rot[3]};
  out->max_state = mcl3dl_pose{best.pos[0], best.pos[1], best.pos[2], 0.0f, best.rot[0], best.rot[1], best.rot[2], best.rot[3]};
  out->max_index = hh.max_index;
  out->weight_sum_biased = hh.weight_sum_biased;
  std::memcpy(out->cov, hh.cov, sizeof(hh.cov));
  return MCL3DL_OK;
}

// ---- record exchange over peer memory (one process per GPU, one device per engine; kernels.cuh: RecordSink +
// exchange_signal_kernel).  Buffer of a rank: [array 0: world * n_local records | array 1 | world flags]; the step
// counter and the error word live in x_ticket (local only).
static size_t xchg_flags_offset(size_t n_local, int world)
{
  return (2 * static_cast<size_t>(world) * n_local * sizeof(mcl3dl_result) + 255) & ~size_t(255);  // two arrays, by step parity
}

int mcl3dl_exchange_create(mcl3dl_engine* eng, size_t n_local, int world, int rank, void* ipc_handle_out)
{
  if (!eng || eng->devs.size() != 1 || n_local == 0 || world < 1 || world > kMaxPeers || rank < 0 || rank >= world ||
      !ipc_handle_out || static_cast<size_t>(world) * n_local >= (size_t(1) << 30))
    return MCL3DL_ERR_INVALID_ARG;
  static_assert(sizeof(cudaIpcMemHandle_t) == MCL3DL_IPC_HANDLE_BYTES, "ipc handle size");
  DeviceCtx& c = eng->devs[0];
  // one exchange per engine lifetime: a second create would free a buffer that the peers still have mapped
  if (c.xchg.p)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  const size_t flags_off = xchg_flags_offset(n_local, world);
  const size_t bytes = flags_off + 256;
  int rc = reserve(eng, c.xchg, bytes);  // a fresh cudaMalloc: IPC handles name whole allocations
  if (rc != MCL3DL_OK || (rc = reserve(eng, c.x_ticket, 256)) != MCL3DL_OK)
    return rc;
  CK(cudaMemset(c.xchg.p, 0, c.xchg.cap));
  CK(cudaMemset(c.x_ticket.p, 0, 256));
  CK(cudaDeviceSynchronize());
  cudaIpcMemHandle_t h;
  CK(cudaIpcGetMemHandle(&h, c.xchg.p));
  std::memcpy(ipc_handle_out, &h, sizeof(h));
  c.xt = PeerTable{};
  c.xt.world = world;
  c.xt.rank = rank;
  c.xsink = RecordSink{};
  c.x_local = n_local;
  c.x_step = 0;
  c.x_ready = false;
  return MCL3DL_OK;
}

int mcl3dl_exchange_open(mcl3dl_engine* eng, const void* ipc_handles /* world x MCL3DL_IPC_HANDLE_BYTES, rank order */)
{
  if (!eng || eng->devs.size() != 1 || !ipc_handles)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (!c.xchg.p || c.xt.world < 1 || c.x_ready)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  const size_t flags_off = xchg_flags_offset(c.x_local, c.xt.world);
  for (int g = 0; g < c.xt.world; ++g)
  {
    void* base = c.xchg.p;
    if (g != c.xt.rank)
    {
      cudaIpcMemHandle_t h;
      std::memcpy(&h, static_cast<const char*>(ipc_handles) + static_cast<size_t>(g) * sizeof(h), sizeof(h));
      const cudaError_t e = cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess)
      {
        eng->err = std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(e);
        c.xchg_close();
        return MCL3DL_ERR_CUDA;
      }
      c.x_opened[g] = base;
    }
    // this rank's slot inside rank g's array 0
    c.xsink.base[g] = static_cast<mcl3dl_result*>(base) + static_cast<size_t>(c.xt.rank) * c.x_local;
    c.xt.flags[g] = reinterpret_cast<uint32_t*>(static_cast<char*>(base) + flags_off);
  }
  c.xsink.step = static_cast<const uint32_t*>(c.x_ticket.p);
  c.xsink.parity_stride = static_cast<uint32_t>(static_cast<size_t>(c.xt.world) * c.x_local);
  c.xsink.world = c.xt.world;
  c.x_ready = true;
  return MCL3DL_OK;
}

int mcl3dl_measure_exchange_device(mcl3dl_engine* eng, const mcl3dl_pose* d_poses, size_t P, const mcl3dl_point* d_lik,
                                   size_t n_lik, const mcl3dl_point* d_beam, size_t n_beam, const float* d_origins_xyz,
                                   size_t n_origins, void* cuda_stream, const mcl3dl_result** d_all_out)
{
  int rc = validate_measure(eng, P, d_lik, n_lik, d_beam, n_beam, d_origins_xyz, n_origins, false);
  if (rc != MCL3DL_OK)
    return rc;
  if (eng->devs.size() != 1 || !d_poses)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (c.w_on)
    return MCL3DL_ERR_TOO_LARGE;
  if (!c.x_ready || P != c.x_local)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  rc = launch_models(eng, c, d_poses, P, d_lik, n_lik, d_beam, n_beam, d_origins_xyz, n_origins, nullptr, nullptr, st, false,
                     &c.xsink);
  if (rc != MCL3DL_OK)
    return rc;
  unsigned int* tk = static_cast<unsigned int*>(c.x_ticket.p);
  CK(launch(eng, exchange_signal_kernel, 1, 32, 0, st, c.xt, tk, tk + 1));
  ++c.x_step;  // host mirror of the device counter; exact for eager calls, resynchronised by mcl3dl_exchange_current
  if (d_all_out)
    *d_all_out = static_cast<const mcl3dl_result*>(c.xchg.p) + static_cast<size_t>(c.x_step & 1u) * c.xt.world * c.x_local;
  return MCL3DL_OK;
}

int mcl3dl_exchange_current(mcl3dl_engine* eng, void* cuda_stream, const mcl3dl_result** d_all_out, int* failed_out)
{
  if (!eng || eng->devs.size() != 1 || !eng->devs[0].x_ticket.p)
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  unsigned int w[2] = {0, 0};
  CK(cudaMemcpyAsync(w, c.x_ticket.p, sizeof(w), cudaMemcpyDeviceToHost, st));  // after everything enqueued on the stream
  CK(cudaStreamSynchronize(st));
  c.x_step = w[0];  // graph replays advance the device counter without the host mirror
  if (d_all_out)
    *d_all_out = static_cast<const mcl3dl_result*>(c.xchg.p) + static_cast<size_t>(c.x_step & 1u) * c.xt.world * c.x_local;
  if (failed_out)
    *failed_out = w[1] != 0;
  return MCL3DL_OK;
}

static int measure_host(mcl3dl_engine* eng, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* lik_pts, size_t n_lik,
                        const mcl3dl_point* beam_pts, size_t n_beam, const float* origins_xyz, size_t n_origins,
                        mcl3dl_result* out, uint8_t* status)
{
  int rc = validate_measure(eng, P, lik_pts, n_lik, beam_pts, n_beam, origins_xyz, n_origins, true);
  if (rc != MCL3DL_OK)
    return rc;
  if (P && (!poses || (!out && !status)))
    return MCL3DL_ERR_INVALID_ARG;
  if (P == 0)
    return MCL3DL_OK;
  const size_t G = eng->devs.size();
  std::vector<Share> sh(G);
  const bool timed = eng->timing != 0;
  // caller arrays inside a mcl3dl_host_alloc block are page-locked: a large pose array is DMA-ed from where it lies
  // and the records land where the caller reads them, without the staging memcpy on either side
  auto out_direct = [&](const Share& s) {
    return out && eng->direct_min_bytes != ~size_t(0) && in_host_block(eng, out + s.p0, s.n * sizeof(mcl3dl_result));
  };
  // enqueue everything on every device, then wait
  for (size_t d = 0; d < G; ++d)
  {
    DeviceCtx& c = eng->devs[d];
    const Share& s = sh[d] = share_of(P, G, d, sizeof(mcl3dl_pose), n_lik, n_beam, n_origins, 0, 0, 0, sizeof(mcl3dl_result),
                                      status ? n_beam : 0);
    if (s.n == 0)
      continue;
    CK(cudaSetDevice(c.dev));
    cudaStream_t st = c.stream;
    const size_t b_rec = s.n * sizeof(mcl3dl_result), b_status = status ? s.n * n_beam : 0;
    const bool poses_direct = s.o_lik >= eng->direct_min_bytes && in_host_block(eng, poses + s.p0, s.o_lik);
    if ((rc = reserve(eng, c.h_pinned, s.total)) || (rc = reserve(eng, c.d_poses, s.in_bytes)) ||
        (rc = reserve(eng, c.d_out, b_rec)) || (rc = reserve(eng, c.d_status, b_status)) ||
        (rc = stage_inputs(eng, c, s, poses_direct ? nullptr : poses, lik_pts, beam_pts, origins_xyz, n_origins, nullptr,
                           nullptr, timed)))
      return rc;
    if (poses_direct)
      CK(cudaMemcpyAsync(c.d_poses.p, poses + s.p0, s.o_lik, cudaMemcpyHostToDevice, st));
    if (timed) CK(cudaEventRecord(c.ev[1], st));
    const char* d_in = static_cast<const char*>(c.d_poses.p);
    if ((rc = window_need(eng, c, reinterpret_cast<const mcl3dl_pose*>(d_in), s.n, reinterpret_cast<const mcl3dl_point*>(d_in + s.o_lik),
                          n_lik, reinterpret_cast<const mcl3dl_point*>(d_in + s.o_beam), n_beam,
                          reinterpret_cast<const float*>(d_in + s.o_org), n_origins, measure_search(eng, c, n_lik, n_beam))))
      return rc;
  }
  // (a windowed map: every device's window check was enqueued above; each is read before that device's models launch)
  for (size_t d = 0; d < G; ++d)
  {
    DeviceCtx& c = eng->devs[d];
    const Share& s = sh[d];
    if (s.n == 0)
      continue;
    if ((rc = window_settle(eng, c, measure_search(eng, c, n_lik, n_beam))))
      return rc;
    CK(cudaSetDevice(c.dev));
    cudaStream_t st = c.stream;
    const size_t b_rec = s.n * sizeof(mcl3dl_result), b_status = status ? s.n * n_beam : 0;
    // small updates: the kernels store their records straight into the pinned block (cudaMallocHost memory is mapped
    // into the unified address space), which saves the D2H copy launch; large ones keep the bulk copy
    const bool zc = !status && s.n <= eng->zero_copy_max;  // (per-ray status bytes would be scattered 1-byte PCIe writes)
    char* hp = static_cast<char*>(c.h_pinned.p);
    mcl3dl_result* h_out = out_direct(s) ? out + s.p0 : reinterpret_cast<mcl3dl_result*>(hp + s.o_rec);
    mcl3dl_result* k_out = zc ? h_out : static_cast<mcl3dl_result*>(c.d_out.p);
    const char* d_in = static_cast<const char*>(c.d_poses.p);
    rc = launch_models(eng, c, reinterpret_cast<const mcl3dl_pose*>(d_in), s.n, reinterpret_cast<const mcl3dl_point*>(d_in + s.o_lik),
                       n_lik, reinterpret_cast<const mcl3dl_point*>(d_in + s.o_beam), n_beam,
                       reinterpret_cast<const float*>(d_in + s.o_org), n_origins, k_out,
                       status ? static_cast<uint8_t*>(c.d_status.p) : nullptr, st, timed);
    if (rc != MCL3DL_OK)
      return rc;
    if (timed) CK(cudaEventRecord(c.ev[5], st));
    if (!zc)
    {
      CK(cudaMemcpyAsync(h_out, c.d_out.p, b_rec, cudaMemcpyDeviceToHost, st));
      if (b_status) CK(cudaMemcpyAsync(hp + s.o_status, c.d_status.p, b_status, cudaMemcpyDeviceToHost, st));
    }
    if (timed) CK(cudaEventRecord(c.ev[4], st));
  }
  eng->t_h2d = eng->t_lik = eng->t_beam = eng->t_d2h = 0;
  for (size_t d = 0; d < G; ++d)
  {
    DeviceCtx& c = eng->devs[d];
    const Share& s = sh[d];
    if (s.n == 0)
      continue;
    CK(cudaSetDevice(c.dev));
    CK(cudaStreamSynchronize(c.stream));
    const char* hp = static_cast<const char*>(c.h_pinned.p);
    if (out && !out_direct(s))  // (else: already there)
      std::memcpy(out + s.p0, hp + s.o_rec, s.n * sizeof(mcl3dl_result));
    if (status) std::memcpy(status + s.p0 * n_beam, hp + s.o_status, s.n * n_beam);
    float ms_h2d = 0, ms_lik = 0, ms_beam = 0, ms_d2h = 0;
    if (timed)
    {
      CK(cudaEventElapsedTime(&ms_h2d, c.ev[0], c.ev[1]));
      CK(cudaEventElapsedTime(&ms_lik, c.ev[2], c.ev[3]));
      if (n_beam) CK(cudaEventElapsedTime(&ms_beam, c.ev_b0, c.ev_b1));
      CK(cudaEventElapsedTime(&ms_d2h, c.ev[5], c.ev[4]));
    }
    eng->t_h2d = std::max(eng->t_h2d, static_cast<double>(ms_h2d));
    eng->t_beam = std::max(eng->t_beam, static_cast<double>(ms_beam));
    eng->t_lik = std::max(eng->t_lik, static_cast<double>(ms_lik));
    eng->t_d2h = std::max(eng->t_d2h, static_cast<double>(ms_d2h));
  }
  return MCL3DL_OK;
}

int mcl3dl_measure_update(mcl3dl_engine* eng, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* lik_pts, size_t n_lik,
                          const mcl3dl_point* beam_pts, size_t n_beam, const float* origins_xyz, size_t n_origins,
                          const float* prior, const float* extra, float* posterior, mcl3dl_result* records,
                          mcl3dl_update_summary* summary)
{
  int rc = validate_measure(eng, P, lik_pts, n_lik, beam_pts, n_beam, origins_xyz, n_origins, true);
  if (rc != MCL3DL_OK)
    return rc;
  if (!summary || (P && (!poses || !prior || !posterior)))
    return MCL3DL_ERR_INVALID_ARG;
  const size_t G = eng->devs.size();
  std::vector<Share> sh(G);
  // ---- pass 1 on every device: inputs up, both models, w_i and its reduction.  One device: the whole weight update,
  // ONE synchronise.  Several devices: the total is a sum over devices, so pass 2 follows a host round trip.
  for (size_t d = 0; d < G; ++d)
  {
    DeviceCtx& c = eng->devs[d];
    const Share& s = sh[d] = share_of(P, G, d, sizeof(mcl3dl_pose), n_lik, n_beam, n_origins, 4, extra ? 4 : 0, 4,
                                      records ? sizeof(mcl3dl_result) : 0, 0);
    if (s.n == 0)
      continue;
    CK(cudaSetDevice(c.dev));
    cudaStream_t st = c.stream;
    if ((rc = reserve(eng, c.h_pinned, s.total)) || (rc = reserve(eng, c.d_poses, s.in_bytes)) ||
        (rc = reserve(eng, c.d_out, s.n * sizeof(mcl3dl_result))) || (rc = reserve(eng, c.d_post, s.n * 4)) ||
        (rc = stage_inputs(eng, c, s, poses, lik_pts, beam_pts, origins_xyz, n_origins, prior, extra, false)))
      return rc;
    const char* d_in = static_cast<const char*>(c.d_poses.p);
    if ((rc = window_need(eng, c, reinterpret_cast<const mcl3dl_pose*>(d_in), s.n, reinterpret_cast<const mcl3dl_point*>(d_in + s.o_lik),
                          n_lik, reinterpret_cast<const mcl3dl_point*>(d_in + s.o_beam), n_beam,
                          reinterpret_cast<const float*>(d_in + s.o_org), n_origins, measure_search(eng, c, n_lik, n_beam))))
      return rc;
  }
  // (a windowed map: every device's window check was enqueued above; each is read before that device's models launch)
  for (size_t d = 0; d < G; ++d)
  {
    DeviceCtx& c = eng->devs[d];
    const Share& s = sh[d];
    if (s.n == 0)
      continue;
    if ((rc = window_settle(eng, c, measure_search(eng, c, n_lik, n_beam))))
      return rc;
    CK(cudaSetDevice(c.dev));
    cudaStream_t st = c.stream;
    const char* d_in = static_cast<const char*>(c.d_poses.p);
    const float* d_prior = reinterpret_cast<const float*>(d_in + s.o_prior);
    const float* d_extra = extra ? reinterpret_cast<const float*>(d_in + s.o_extra) : nullptr;
    mcl3dl_result* d_rec = static_cast<mcl3dl_result*>(c.d_out.p);
    char* hp = static_cast<char*>(c.h_pinned.p);
    WeightPartial* h_part = reinterpret_cast<WeightPartial*>(hp + s.o_part);
    rc = launch_models(eng, c, reinterpret_cast<const mcl3dl_pose*>(d_in), s.n, reinterpret_cast<const mcl3dl_point*>(d_in + s.o_lik),
                       n_lik, reinterpret_cast<const mcl3dl_point*>(d_in + s.o_beam), n_beam,
                       reinterpret_cast<const float*>(d_in + s.o_org), n_origins, d_rec, nullptr, st, false);
    if (rc != MCL3DL_OK)
      return rc;
    if (G == 1)
    {
      if ((rc = fold_weights(eng, c, d_rec, d_prior, d_extra, static_cast<float*>(c.d_post.p), s.n, n_lik, s.p0, h_part,
                             reinterpret_cast<float*>(hp + s.o_post))))
        return rc;
      if (records)
        CK(cudaMemcpyAsync(hp + s.o_rec, d_rec, s.n * sizeof(mcl3dl_result), cudaMemcpyDeviceToHost, st));
    }
    else
    {
      const WeightPartial* f1;
      if ((rc = weight_pass1(eng, c, d_rec, d_prior, d_extra, s.n, n_lik, nullptr, &f1)))
        return rc;
      CK(cudaMemcpyAsync(h_part, f1, sizeof(WeightPartial), cudaMemcpyDeviceToHost, st));
    }
  }
  WeightPartial w1 = weight_identity(), w2 = weight_identity();  // each pass folded over the devices, in device order
  for (size_t d = 0; d < G; ++d)
  {
    DeviceCtx& c = eng->devs[d];
    if (sh[d].n == 0)
      continue;
    CK(cudaSetDevice(c.dev));
    CK(cudaStreamSynchronize(c.stream));
    const WeightPartial& wp = *reinterpret_cast<const WeightPartial*>(static_cast<const char*>(c.h_pinned.p) + sh[d].o_part);
    w1.sum += wp.sum;
    w1.qmin = std::min(w1.qmin, wp.qmin);
    w1.qmax = std::max(w1.qmax, wp.qmax);
  }
  const float total_f = static_cast<float>(w1.sum);
  const bool kept = total_f > 0.0f;
  // ---- pass 2 (several devices): normalise with the global total, entropy, arg max; only 4 B per particle come back
  for (size_t d = 0; d < G && G > 1; ++d)
  {
    DeviceCtx& c = eng->devs[d];
    const Share& s = sh[d];
    if (s.n == 0)
      continue;
    CK(cudaSetDevice(c.dev));
    cudaStream_t st = c.stream;
    char* hp = static_cast<char*>(c.h_pinned.p);
    if (kept)
    {
      const WeightPartial* f2;
      if ((rc = weight_pass2(eng, c, nullptr, total_f, s.n, s.p0, static_cast<float*>(c.d_post.p), nullptr, &f2)))
        return rc;
      CK(cudaMemcpyAsync(hp + s.o_post, c.d_post.p, s.n * 4, cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(hp + s.o_part + sizeof(WeightPartial), f2, sizeof(WeightPartial), cudaMemcpyDeviceToHost, st));
    }
    if (records)
      CK(cudaMemcpyAsync(hp + s.o_rec, c.d_out.p, s.n * sizeof(mcl3dl_result), cudaMemcpyDeviceToHost, st));
  }
  for (size_t d = 0; d < G; ++d)
  {
    DeviceCtx& c = eng->devs[d];
    const Share& s = sh[d];
    if (s.n == 0)
      continue;
    CK(cudaSetDevice(c.dev));
    if (G > 1)
      CK(cudaStreamSynchronize(c.stream));
    const char* hp = static_cast<const char*>(c.h_pinned.p);
    if (kept)
    {
      std::memcpy(posterior + s.p0, hp + s.o_post, s.n * 4);
      const WeightPartial& wp = reinterpret_cast<const WeightPartial*>(hp + s.o_part)[1];
      w2.sum += wp.sum;
      if (wp.best > w2.best)  // lower device = lower indices, so strict '>' keeps the first maximum
      {
        w2.best = wp.best;
        w2.best_i = wp.best_i;
      }
    }
    else
      std::memcpy(posterior + s.p0, prior + s.p0, s.n * 4);  // "No Particle alive, restoring." pf.h:274-278
    if (records)
      std::memcpy(records + s.p0, hp + s.o_rec, s.n * sizeof(mcl3dl_result));
  }
  make_summary(w1, w2, summary);
  return MCL3DL_OK;
}

int mcl3dl_measure(mcl3dl_engine* eng, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* lik_pts, size_t n_lik,
                   const mcl3dl_point* beam_pts, size_t n_beam, const float* origins_xyz, size_t n_origins,
                   mcl3dl_result* out)
{
  if (P && !out)
    return MCL3DL_ERR_INVALID_ARG;
  return measure_host(eng, poses, P, lik_pts, n_lik, beam_pts, n_beam, origins_xyz, n_origins, out, nullptr);
}

int mcl3dl_beam_status(mcl3dl_engine* eng, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* beam_pts, size_t n_beam,
                       const float* origins_xyz, size_t n_origins, uint8_t* status)
{
  if (P && n_beam && !status)
    return MCL3DL_ERR_INVALID_ARG;
  if (n_beam == 0)
    return MCL3DL_OK;
  return measure_host(eng, poses, P, nullptr, 0, beam_pts, n_beam, origins_xyz, n_origins, nullptr, status);
}

int mcl3dl_beam_cast(mcl3dl_engine* eng, const mcl3dl_pose* pose, const mcl3dl_point* beam_pts, size_t n_beam,
                     const float* origins_xyz, size_t n_origins, mcl3dl_beam_ray* out, size_t capacity, size_t* n_out)
{
  if (!eng || !pose || !n_out)
    return MCL3DL_ERR_INVALID_ARG;
  if (!eng->has_map)
    return MCL3DL_ERR_NO_MAP;
  const bool kd = !eng->beam.use_raycast_using_dda;
  if (!eng->has_beam || (kd && !eng->has_lik))
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  const mcl3dl_point* d_scan = nullptr;  // the prepared scan, or the host scan's copy in b_in
  size_t n = n_beam;
  if (!beam_pts)
  {
    if (eng->devs.size() != 1 || !c.s_valid)
      return MCL3DL_ERR_INVALID_ARG;
    d_scan = static_cast<const mcl3dl_point*>(c.s_out[1].p);
    n = c.s_info.n_beam;
  }
  if (n >= (size_t(1) << 24) || (n && (!out || capacity < n || !origins_xyz || n_origins == 0)))
    return MCL3DL_ERR_INVALID_ARG;
  if (n == 0)
  {
    *n_out = 0;
    return MCL3DL_OK;
  }
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = c.stream;
  // page-locked block: [label error word | pad to 64 | pose (32 B) | origins | host scan | records]; the inputs go up in
  // one copy to b_in (same layout from the pose on), the kernel stores the error word and the records in place
  const size_t o_org = 64 + sizeof(mcl3dl_pose), o_scan = o_org + pad16(n_origins * 12);
  const size_t in_end = o_scan + (beam_pts ? n * 16 : 0), o_rec = pad16(in_end);
  int rc;
  if ((rc = reserve(eng, c.b_host, o_rec + n * sizeof(mcl3dl_beam_ray))) || (rc = reserve(eng, c.b_in, in_end - 64)))
    return rc;
  char* hp = static_cast<char*>(c.b_host.p);
  char* dp = static_cast<char*>(c.b_in.p);
  unsigned int* bad = reinterpret_cast<unsigned int*>(hp);
  *bad = 0;
  std::memcpy(hp + 64, pose, sizeof(mcl3dl_pose));
  std::memcpy(hp + o_org, origins_xyz, n_origins * 12);
  if (beam_pts)
  {
    std::memcpy(hp + o_scan, beam_pts, n * 16);
    d_scan = reinterpret_cast<const mcl3dl_point*>(dp + o_scan - 64);
  }
  CK(cudaMemcpyAsync(dp, hp + 64, in_end - 64, cudaMemcpyHostToDevice, st));
  if (kd && (rc = ensure_window(eng, c, reinterpret_cast<const mcl3dl_pose*>(dp), 1, nullptr, 0, d_scan, n,
                                reinterpret_cast<const float*>(dp + o_org - 64), n_origins, measure_search(eng, c, 0, n))))
    return rc;
  mcl3dl_beam_ray* h_rec = reinterpret_cast<mcl3dl_beam_ray*>(hp + o_rec);
  const auto kernel = kd ? beam_cast_kernel<true> : beam_cast_kernel<false>;
  CK(launch(eng, kernel, static_cast<unsigned>((n + kBlockThreads - 1) / kBlockThreads), kBlockThreads, 0, st,
            reinterpret_cast<const mcl3dl_pose*>(dp), reinterpret_cast<const float4*>(d_scan), static_cast<int>(n),
            reinterpret_cast<const float*>(dp + o_org - 64), static_cast<uint32_t>(n_origins), c.dda, c.kd, c.nn, h_rec, bad));
  CK(cudaStreamSynchronize(st));
  if (*bad)
    return MCL3DL_ERR_INVALID_ARG;
  std::memcpy(out, h_rec, n * sizeof(mcl3dl_beam_ray));
  *n_out = n;
  return MCL3DL_OK;
}

int mcl3dl_collect_stats(mcl3dl_engine* eng, int enable)
{
  if (!eng)
    return MCL3DL_ERR_INVALID_ARG;
  for (DeviceCtx& c : eng->devs)
  {
    CK(cudaSetDevice(c.dev));
    int rc = reserve(eng, c.d_stats, 5 * sizeof(unsigned long long));
    if (rc != MCL3DL_OK)
      return rc;
    // every call restarts the counters: done before the call returns, so ahead of any later kernel on any stream
    CK(cudaMemsetAsync(c.d_stats.p, 0, 5 * sizeof(unsigned long long), c.stream));
    CK(cudaStreamSynchronize(c.stream));
    c.stats_on = enable != 0;
  }
  return MCL3DL_OK;
}

int mcl3dl_collect_timing(mcl3dl_engine* eng, int enable)
{
  if (!eng)
    return MCL3DL_ERR_INVALID_ARG;
  eng->timing = enable != 0;
  if (!enable)
    eng->t_h2d = eng->t_lik = eng->t_beam = eng->t_d2h = 0;
  return MCL3DL_OK;
}

int mcl3dl_read_stats(mcl3dl_engine* eng, mcl3dl_work_stats* out)
{
  if (!eng || !out)
    return MCL3DL_ERR_INVALID_ARG;
  std::memset(out, 0, sizeof(*out));
  for (DeviceCtx& c : eng->devs)
  {
    if (!c.d_stats.p)
      continue;
    unsigned long long h[5];
    CK(cudaSetDevice(c.dev));
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(h, c.d_stats.p, sizeof(h), cudaMemcpyDeviceToHost));
    out->lik_index_rows += h[0];
    out->lik_points_scanned += h[1];
    out->beam_cells_stepped += h[2];
    out->beam_cells_occupied += h[3];
    out->beam_points_tested += h[4];
  }
  return MCL3DL_OK;
}

void mcl3dl_beam_params_from_reference(mcl3dl_beam_params* o, float map_grid_x, float map_grid_y, float map_grid_z,
                                       size_t num_points_default, float beam_likelihood_min, float ang_total_ref,
                                       uint32_t filter_label_max, float hit_range, int add_penalty_short_only_mode,
                                       int use_raycast_using_dda, float ray_angle_half, float dda_grid_size)
{
  // LidarMeasurementModelBeam::refreshParameters, src/lidar_measurement_model_beam.cpp:58-80: the
  // float parameters are promoted to double where the RaycastUsingDDA constructor takes doubles.
  o->map_grid_size[0] = map_grid_x;
  o->map_grid_size[1] = map_grid_y;
  o->map_grid_size[2] = map_grid_z;
  o->dda_grid_size = dda_grid_size;
  o->ray_angle_half = ray_angle_half;
  o->hit_tolerance = hit_range;
  o->hit_range_sq = static_cast<float>(std::pow(static_cast<double>(hit_range), 2.0));
  o->sin_total_ref = sinf(ang_total_ref);
  o->beam_likelihood = static_cast<float>(
      std::pow(static_cast<double>(beam_likelihood_min), 1.0 / static_cast<double>(static_cast<float>(num_points_default))));
  o->beam_likelihood_min = beam_likelihood_min;
  o->filter_label_max = filter_label_max;
  o->add_penalty_short_only_mode = add_penalty_short_only_mode ? 1 : 0;
  o->use_raycast_using_dda = use_raycast_using_dda ? 1 : 0;
  o->_reserved = 0;
}

}  // extern "C"
