// engine.cu — host side of the C ABI (include/mcl3dl_b200.h): map staging on the device, the
// per-update launch sequence, multi-device sharding.  No CPU compute path exists here: every entry
// point either runs on a CUDA device or fails with an error code.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <string>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

#include "kernels.cuh"
#include "pf_kernels.cuh"
#include "scan_kernels.cuh"

using namespace mcl3dl;

namespace
{
constexpr int kMaxStagedBytes = 200 * 1024;
constexpr int kMaxStagedSorted = 160 * 1024;  // the sorted kernel also holds ~26 KB of static shared memory

// ---------------------------------------------------------------- device build kernels
__device__ __forceinline__ uint32_t f2ord(float f)
{
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
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
__device__ __forceinline__ bool nnf_voxel_of_thread(const NnFieldDev& f, size_t n_cells, size_t t, size_t& cell, int& sub, int& vx,
                                                    int& vy, int& vz)
{
  cell = t >> 3;
  sub = static_cast<int>(t & 7);
  if (cell >= n_cells)
    return false;
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
                     uint32_t* __restrict__ totals, size_t n_cells, uint4* __restrict__ wide, uint32_t wide_cap,
                     uint32_t* __restrict__ counters /* [0] wide cells used, [1] overflow cells */)
{
  const size_t t = blockIdx.x * static_cast<size_t>(256) + threadIdx.x;
  size_t cell;
  int sub, vx, vy, vz, cnt = 0;
  if (nnf_voxel_of_thread(f, n_cells, t, cell, sub, vx, vy, vz) &&
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
  if (sub != 0 || cell >= n_cells)
    return;
  // dir[cell].y: nibbles | 0xfffffffe = wide cell (dir[cell].x already holds 0x80000000 | index) | 0xffffffff = overflow
  if (!ovf && big)
  {
    const uint32_t idx = atomicAdd(counters, 1u);
    if (idx < wide_cap)
    {
      wide[idx] = make_uint4(0u, lo, hi, 0u);  // x = first candidate, filled in by nnf_base_kernel
      dir[cell] = make_uint2(0x80000000u | idx, 0xfffffffeu);
      totals[cell] = tot;
      return;
    }
    ovf = 1u;  // side table full: treat as an overflow cell
  }
  if (ovf)
  {
    dir[cell].y = 0xffffffffu;
    totals[cell] = 0u;
    atomicAdd(counters + 1, 1u);
    return;
  }
  uint32_t nib = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) nib |= (((lo >> (8 * k)) & 15u) << (4 * k)) | (((hi >> (8 * k)) & 15u) << (4 * (k + 4)));
  dir[cell].y = nib;
  totals[cell] = tot;
}

struct WidenU32
{
  __host__ __device__ unsigned long long operator()(uint32_t v) const { return v; }
};

__global__ void nnf_base_kernel(uint2* __restrict__ dir, const uint32_t* __restrict__ base, size_t n_cells, uint4* __restrict__ wide)
{
  const size_t c = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (c >= n_cells)
    return;
  const uint32_t y = dir[c].y;
  if (y == 0xffffffffu)
    dir[c].x = 0xffffffffu;
  else if (y == 0xfffffffeu)
    wide[dir[c].x & 0x7fffffffu].x = base[c];
  else
    dir[c].x = base[c];
}

__global__ void __launch_bounds__(256)
    nnf_fill_kernel(NnGridDev g, NnFieldDev f, const uint32_t* __restrict__ bits, int pitch, const uint2* __restrict__ dir,
                    float4* __restrict__ cand, size_t n_cells)
{
  const size_t t = blockIdx.x * static_cast<size_t>(256) + threadIdx.x;
  size_t cell;
  int sub, vx, vy, vz;
  if (!nnf_voxel_of_thread(f, n_cells, t, cell, sub, vx, vy, vz))
    return;
  uint32_t start = 0;
  const int want = nnf_slot(f, dir[cell], sub, start);
  if (want <= 0)
    return;
  uint32_t pos[kNnfMaxSurv];
  const int cnt = nnf_select(g, f, vx, vy, vz, pos);
  for (int i = 0; i < cnt && i < want; ++i) cand[start + i] = g.pts[pos[i]];
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

struct DevBuf
{
  void* p = nullptr;
  size_t cap = 0;
};

struct DeviceCtx
{
  int dev = 0;
  cudaStream_t stream = nullptr;
  int sm_count = 132;
  // map
  DevBuf nn_cell_start, nn_pts, nn_row3, dda_occ, dda_cell_start, dda_pts;
  NnGridDev nn{};
  DdaGridDev dda{};
  KdRayDev kd{};
  DevBuf raw_pts;  // map points in original order (KD-tree raycaster only)
  DevBuf near_lik, near_kd;  // near-field bits (MCL3DL_NEAR_BITS builds)
  DevBuf nnf_dir, nnf_cand, nnf_wide;  // NN field: directory, candidate lists, side table of the wide cells
  DevBuf fld_cells;          // field mode: 8 corner distances per lattice cell
  cudaPitchedPtr fld_nodes{};  // field mode: node volume (cudaMalloc3D)
  bool fld_nodes_valid = false;
  float near_kd_r = 0.0f;            // radius the KD field was built for
  size_t map_bytes = 0;
  // per-update I/O
  DevBuf d_poses /* whole input block of the host path */, d_out, d_status;
  void* h_pinned = nullptr;
  size_t h_pinned_cap = 0;
  cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  // the two models are independent (disjoint fields of the record): the beam kernel runs on a side stream,
  // forked from / joined to the caller's stream with events
  cudaStream_t side = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_b0 = nullptr, ev_b1 = nullptr;
  DevBuf d_w, d_post, d_wpart, d_wticket;   // fused weight update: w_i, posterior, per-CTA partials, last-CTA tickets (2)
  DevBuf d_partial, d_tickets;  // lane-per-particle kernels: per-CTA partials + per-group ticket counters
  DevBuf d_tally, d_queue;      // dynamic-queue beam kernel: per-particle integer tallies, item counter (left at zero)
  DevBuf d_lacc;                // point-major likelihood kernel: per-particle accumulators (left at zero)
  size_t tally_zeroed = 0;
  size_t tickets_zeroed = 0;
  std::vector<const void*> smem_opted;  // kernels already opted in to large dynamic shared memory on this device
  // resident particle set (mcl3dl_particles_*): two state buffers (resampling writes the other one), probabilities,
  // prefix sum + pstep, the packed poses / odometry-error factors the measurement kernels read
  // scan preprocessing (mcl3dl_scan_prepare): raw cloud, sort keys / values (x2), flags + scan positions (x2), the
  // downsampled cloud, the two clipped clouds, the two sampled scans, cub scratch, device-side counts
  DevBuf s_raw, s_keys[2], s_vals[2], s_flags[2], s_pos[2], s_ds, s_clip[2], s_out[2], s_tmp, s_counts;
  mcl3dl_scan_info s_info{};
  bool s_valid = false;
  DevBuf r_states[2], r_prob, r_accum, r_poses, r_extra, r_est;  // r_est: EstHeader + per-CTA partial sums
  size_t r_n = 0;
  int r_cur = 0;
  uint32_t r_calls = 0;
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
                                // straight into the pinned result block (no D2H copy launch); MCL3DL_ZEROCOPY_OUT
  int update_one_sync = 1;  // mcl3dl_measure_update on ONE device: normalise from the device-side total, one host
                            // synchronise instead of two (MCL3DL_UPDATE_ONE_SYNC=1; written without GPU time left in
                            // round 1: off until the f2 parity tests have run with it)
  int field_mode = 0;  // 1: the likelihood model reads the trilinear distance volume (opt-in, inexact; MCL3DL_LIK_MODE=field)
  size_t field_max_bytes = size_t(24) << 30;  // MCL3DL_FIELD_MAX_MB
  int beam_dq = 2;  // beam kernel: 2 = by job size, 1 = MCL3DL_BEAM=dq, 0 = MCL3DL_BEAM=pl
  int beam_dq_ppl = 0;  // MCL3DL_BEAM_DQ_PPL: rays per item (0 = chosen from the job size)
  int lik_share = 4;  // CTA slots per SM the likelihood kernel takes while the beam kernel runs next to it (MCL3DL_LIK_SHARE)
  int nnf_kd_r2 = 1;  // MCL3DL_NNF_KD_R2=0: the NN field also covers the KD-tree raycaster's second search radius
  int nnf = 1;  // stage the NN field (exact per-voxel candidate lists) and use lik_kernel_nf; MCL3DL_NNF=0: the CSR window kernels
  size_t nnf_max_bytes = size_t(32) << 30;  // MCL3DL_NNF_MAX_MB: directory + candidates above this -> no field
  uint64_t nnf_bytes = 0, nnf_cands = 0, nnf_overflow_cells = 0, nnf_wide_cells = 0;
  int mapping = 1;  // 1 = tuned kernels (lik_kernel_wi + beam_kernel_pl); 0 = the plain group kernels (MCL3DL_MAPPING=group)
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

int reserve(mcl3dl_engine* eng, DevBuf& b, size_t bytes)
{
  if (bytes <= b.cap && b.p)
    return MCL3DL_OK;
  if (b.p)
    CK(cudaFree(b.p));
  b.p = nullptr;
  b.cap = 0;
  const size_t want = std::max<size_t>(bytes, 256);
  CK(cudaMalloc(&b.p, want));
  b.cap = want;
  return MCL3DL_OK;
}

int reserve_pinned(mcl3dl_engine* eng, DeviceCtx& c, size_t bytes)
{
  if (bytes <= c.h_pinned_cap)
    return MCL3DL_OK;
  if (c.h_pinned)
    CK(cudaFreeHost(c.h_pinned));
  c.h_pinned = nullptr;
  c.h_pinned_cap = 0;
  CK(cudaMallocHost(&c.h_pinned, bytes));
  c.h_pinned_cap = bytes;
  return MCL3DL_OK;
}

void free_buf(DevBuf& b)
{
  if (b.p)
    cudaFree(b.p);
  b.p = nullptr;
  b.cap = 0;
}

// two zeroed ticket words for the last-CTA folds of the weight-update kernels (they leave them at zero)
int weight_tickets(mcl3dl_engine* eng, DeviceCtx& c, unsigned int** out)
{
  if (!c.d_wticket.p)
  {
    const int rc = reserve(eng, c.d_wticket, 256);
    if (rc != MCL3DL_OK)
      return rc;
    CK(cudaMemset(c.d_wticket.p, 0, 256));
  }
  *out = static_cast<unsigned int*>(c.d_wticket.p);
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

template <int TPP>
int launch_lik_t(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, int P, const float4* scan, int N,
                 mcl3dl_result* out, int beam_defaults, cudaStream_t st, const RecordSink& sink)
{
  constexpr int PPB = kBlockThreads / TPP;
  const int groups = (P + PPB - 1) / PPB;
  const int grid = std::max(1, std::min(groups, c.sm_count * 8));
  const size_t bytes = static_cast<size_t>(N) * 16;
  if (eng->mapping != 0)
  {
    if (bytes <= static_cast<size_t>(kMaxStagedSorted))
    {
      if (int rc = opt_in_smem(eng, c, lik_kernel_wi<TPP, true>, kMaxStagedSorted)) return rc;
      lik_kernel_wi<TPP, true><<<grid, kBlockThreads, bytes, st>>>(poses, P, scan, N, c.nn, eng->likdev, out, beam_defaults, c.stats_ptr(), sink);
    }
    else
    {
      lik_kernel_wi<TPP, false><<<grid, kBlockThreads, 0, st>>>(poses, P, scan, N, c.nn, eng->likdev, out, beam_defaults, c.stats_ptr(), sink);
    }
  }
  else if (bytes <= static_cast<size_t>(kMaxStagedBytes))
  {
    if (int rc = opt_in_smem(eng, c, lik_kernel<TPP, true>, kMaxStagedBytes)) return rc;
    lik_kernel<TPP, true><<<grid, kBlockThreads, bytes, st>>>(poses, P, scan, N, c.nn, eng->likdev, out, beam_defaults, c.stats_ptr(), sink);
  }
  else
  {
    lik_kernel<TPP, false><<<grid, kBlockThreads, 0, st>>>(poses, P, scan, N, c.nn, eng->likdev, out, beam_defaults, c.stats_ptr(), sink);
  }
  CK(cudaGetLastError());
  eng->launches++;
  return MCL3DL_OK;
}

template <int TPP>
int launch_beam_t(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, int P, const float4* scan, int N,
                  const float* origins, mcl3dl_result* out, uint8_t* status, int lik_defaults, cudaStream_t st, const RecordSink& sink)
{
  constexpr int PPB = kBlockThreads / TPP;
  const int groups = (P + PPB - 1) / PPB;
  const int grid = std::max(1, std::min(groups, c.sm_count * 8));
  const size_t bytes = static_cast<size_t>(N) * 16;
  if (bytes <= static_cast<size_t>(kMaxStagedBytes))
  {
    if (int rc = opt_in_smem(eng, c, beam_kernel<TPP, true>, kMaxStagedBytes)) return rc;
    beam_kernel<TPP, true><<<grid, kBlockThreads, bytes, st>>>(poses, P, scan, N, origins, c.dda, out, status, lik_defaults, c.stats_ptr(), sink);
  }
  else
  {
    beam_kernel<TPP, false><<<grid, kBlockThreads, 0, st>>>(poses, P, scan, N, origins, c.dda, out, status, lik_defaults, c.stats_ptr(), sink);
  }
  CK(cudaGetLastError());
  eng->launches++;
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
  if (const char* v = std::getenv("MCL3DL_NF_TPP"))  // experiments
  {
    const int t = std::atoi(v);
    if (t == 8 || t == 16 || t == 32 || t == 64 || t == 128 || t == 256)
      tpp = t;
  }
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
  bool staged = bytes <= static_cast<size_t>(kMaxStagedBytes) / 2 && (PPB >= 4 || groups > grid);
  if (const char* v = std::getenv("MCL3DL_NF_STAGE"))  // experiments
    staged = bytes <= static_cast<size_t>(kMaxStagedBytes) / 2 && std::atoi(v) != 0;
#define NF_LAUNCH(S, O)                                                                                                    \
  do                                                                                                                       \
  {                                                                                                                        \
    if (S)                                                                                                                 \
      if (int rc = opt_in_smem(eng, c, lik_kernel_nf<TPP, S, O>, kMaxStagedBytes / 2)) return rc;                          \
    lik_kernel_nf<TPP, S, O><<<grid, kBlockThreads, (S) ? bytes : 0, st>>>(poses, P, scan, N, c.nn, eng->likdev, out,       \
                                                                           beam_defaults, c.stats_ptr(), sink);            \
  } while (0)
  if (staged && ovf) NF_LAUNCH(true, true);
  else if (staged) NF_LAUNCH(true, false);
  else if (ovf) NF_LAUNCH(false, true);
  else NF_LAUNCH(false, false);
#undef NF_LAUNCH
  CK(cudaGetLastError());
  eng->launches++;
  return MCL3DL_OK;
}

// point-major mapping (kernels.cuh: lik_kernel_nf_pm): 256 particles per CTA, the scan cut into slices (nf_pm_shape)
int launch_lik_nf_pm(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, int P, const float4* scan, int N,
                     mcl3dl_result* out, int beam_defaults, cudaStream_t st, const RecordSink& sink, int blocks,
                     const NfPmShape& sh)
{
  // one accumulator per particle; zeroed once, the kernel leaves it at zero
  const size_t bytes = static_cast<size_t>(P) * 8;
  if (bytes > c.d_lacc.cap || !c.d_lacc.p)
  {
    if (int rc = reserve(eng, c.d_lacc, bytes))
      return rc;
    CK(cudaMemsetAsync(c.d_lacc.p, 0, c.d_lacc.cap, st));
  }
  auto* acc = static_cast<unsigned long long*>(c.d_lacc.p);
#define PM_LAUNCH(O)                                                                                                       \
  lik_kernel_nf_pm<O><<<blocks * sh.n_slices, kBlockThreads, 0, st>>>(poses, P, scan, N, c.nn, eng->likdev, out,           \
                                                                      beam_defaults, c.stats_ptr(), sink, sh, acc)
  if (eng->nnf_overflow_cells != 0)
    PM_LAUNCH(true);
  else
    PM_LAUNCH(false);
#undef PM_LAUNCH
  CK(cudaGetLastError());
  eng->launches++;
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
  switch (pick_tpp_nf(P, N, c.sm_count))
  {
    case 8: return launch_lik_nf_t<8>(eng, c, poses, p, s4, n, out, beam_defaults, st, sink);
    case 16: return launch_lik_nf_t<16>(eng, c, poses, p, s4, n, out, beam_defaults, st, sink);
    case 32: return launch_lik_nf_t<32>(eng, c, poses, p, s4, n, out, beam_defaults, st, sink);
    case 64: return launch_lik_nf_t<64>(eng, c, poses, p, s4, n, out, beam_defaults, st, sink);
    case 128: return launch_lik_nf_t<128>(eng, c, poses, p, s4, n, out, beam_defaults, st, sink);
    default: return launch_lik_nf_t<256>(eng, c, poses, p, s4, n, out, beam_defaults, st, sink);
  }
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
  if (!c.fld_nodes.ptr)
  {
    const cudaExtent ext = make_cudaExtent(static_cast<size_t>(nnx) * sizeof(float), nny, nnz);
    CK(cudaMalloc3D(&c.fld_nodes, ext));
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
    const size_t total = static_cast<size_t>(nnx) * nny * nnz;
    field_nodes_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(c.nn, lp, c.fld_nodes, nnx, nny, nnz, clamp);
    CK(cudaGetLastError());
    eng->launches++;
  }
  field_expand_kernel<<<static_cast<unsigned>((n_cells + 255) / 256), 256, 0, st>>>(c.fld_nodes, f.nx, f.ny, f.nz,
                                                                                    static_cast<float4*>(c.fld_cells.p));
  CK(cudaGetLastError());
  eng->launches++;
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
  if (staged)
  {
    if (int rc = opt_in_smem(eng, c, lik_kernel_field<TPP, true>, kMaxStagedBytes / 2)) return rc;
    lik_kernel_field<TPP, true><<<grid, kBlockThreads, bytes, st>>>(poses, P, scan, N, c.nn, eng->likdev, out, beam_defaults, c.stats_ptr(), sink);
  }
  else
    lik_kernel_field<TPP, false><<<grid, kBlockThreads, 0, st>>>(poses, P, scan, N, c.nn, eng->likdev, out, beam_defaults, c.stats_ptr(), sink);
  CK(cudaGetLastError());
  eng->launches++;
  return MCL3DL_OK;
}

int launch_lik_field(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* scan, size_t N,
                     mcl3dl_result* out, int beam_defaults, cudaStream_t st, const RecordSink& sink)
{
  const float4* s4 = reinterpret_cast<const float4*>(scan);
  const int p = static_cast<int>(P), n = static_cast<int>(N);
  switch (pick_tpp_nf(P, N, c.sm_count))
  {
    case 8: return launch_lik_field_t<8>(eng, c, poses, p, s4, n, out, beam_defaults, st, sink);
    case 16: return launch_lik_field_t<16>(eng, c, poses, p, s4, n, out, beam_defaults, st, sink);
    case 32: return launch_lik_field_t<32>(eng, c, poses, p, s4, n, out, beam_defaults, st, sink);
    case 64: return launch_lik_field_t<64>(eng, c, poses, p, s4, n, out, beam_defaults, st, sink);
    case 128: return launch_lik_field_t<128>(eng, c, poses, p, s4, n, out, beam_defaults, st, sink);
    default: return launch_lik_field_t<256>(eng, c, poses, p, s4, n, out, beam_defaults, st, sink);
  }
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
  if (groups * 4 > c.d_tickets.cap || !c.d_tickets.p)
  {
    rc = reserve(eng, c.d_tickets, std::max<size_t>(groups * 4, 4096));
    if (rc != MCL3DL_OK)
      return rc;
    CK(cudaMemsetAsync(c.d_tickets.p, 0, c.d_tickets.cap, st));  // the kernels leave them at zero afterwards
  }
  return MCL3DL_OK;
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
#define PL_LAUNCH(KD)                                                                                                             \
  beam_kernel_pl<KD><<<groups * sh.cb, kBlockThreads, smem, st>>>(                                                                \
      poses, static_cast<int>(P), reinterpret_cast<const float4*>(scan), static_cast<int>(N), origins, c.dda, c.kd, c.nn, out, status, \
      lik_defaults, c.stats_ptr(), sh, static_cast<uint32_t*>(c.d_partial.p), static_cast<unsigned int*>(c.d_tickets.p), sink)
  if (eng->beam.use_raycast_using_dda)
    PL_LAUNCH(false);
  else
    PL_LAUNCH(true);
#undef PL_LAUNCH
  CK(cudaGetLastError());
  eng->launches++;
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
  const size_t tally_bytes = std::max<size_t>(P, 1) * 12, ticket_bytes = std::max<size_t>(groups * 4, 4096);
  if (tally_bytes > c.d_tally.cap || !c.d_tally.p)
  {
    if ((rc = reserve(eng, c.d_tally, tally_bytes)))
      return rc;
    CK(cudaMemsetAsync(c.d_tally.p, 0, c.d_tally.cap, st));  // the kernel leaves them at zero afterwards
  }
  if (ticket_bytes > c.d_tickets.cap || !c.d_tickets.p)
  {
    if ((rc = reserve(eng, c.d_tickets, ticket_bytes)))
      return rc;
    CK(cudaMemsetAsync(c.d_tickets.p, 0, c.d_tickets.cap, st));
  }
  if (!c.d_queue.p)
  {
    if ((rc = reserve(eng, c.d_queue, 256)))
      return rc;
    CK(cudaMemsetAsync(c.d_queue.p, 0, 256, st));
  }
#define DQ_LAUNCH(KD)                                                                                                              \
  beam_kernel_dq<KD><<<grid, kBlockThreads, 0, st>>>(poses, static_cast<int>(P), reinterpret_cast<const float4*>(scan),             \
                                                     static_cast<int>(N), origins, c.dda, c.kd, c.nn, out, status, lik_defaults,   \
                                                     c.stats_ptr(), static_cast<int>(ppl), n_chunks,                               \
                                                     static_cast<uint32_t*>(c.d_tally.p), static_cast<unsigned int*>(c.d_tickets.p), \
                                                     static_cast<unsigned int*>(c.d_queue.p), sink)
  if (eng->beam.use_raycast_using_dda)
    DQ_LAUNCH(false);
  else
    DQ_LAUNCH(true);
#undef DQ_LAUNCH
  CK(cudaGetLastError());
  eng->launches++;
  return MCL3DL_OK;
}

int launch_lik(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* scan, size_t N,
               mcl3dl_result* out, int beam_defaults, cudaStream_t st, const RecordSink& sink)
{
  if (eng->field_mode && c.nn.fld.cells)
    return launch_lik_field(eng, c, poses, P, scan, N, out, beam_defaults, st, sink);
  if (eng->mapping != 0 && c.nn.field.dir)
    return launch_lik_nf(eng, c, poses, P, scan, N, out, beam_defaults, st, sink);
  const float4* s4 = reinterpret_cast<const float4*>(scan);
  switch (pick_tpp(P, N, c.sm_count))
  {
    case 32: return launch_lik_t<32>(eng, c, poses, static_cast<int>(P), s4, static_cast<int>(N), out, beam_defaults, st, sink);
    case 64: return launch_lik_t<64>(eng, c, poses, static_cast<int>(P), s4, static_cast<int>(N), out, beam_defaults, st, sink);
    case 128: return launch_lik_t<128>(eng, c, poses, static_cast<int>(P), s4, static_cast<int>(N), out, beam_defaults, st, sink);
    default: return launch_lik_t<256>(eng, c, poses, static_cast<int>(P), s4, static_cast<int>(N), out, beam_defaults, st, sink);
  }
}

int launch_beam(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* scan, size_t N,
                const float* origins, int n_origins, mcl3dl_result* out, uint8_t* status, int lik_defaults, cudaStream_t st,
                const RecordSink& sink)
{
  if (eng->mapping != 0 && (eng->beam_dq == 1 || (eng->beam_dq == 2 && P * N >= 262144)))
    return launch_beam_dq(eng, c, poses, P, scan, N, origins, out, status, lik_defaults, st, sink);
  if (eng->mapping != 0 || !eng->beam.use_raycast_using_dda)  // the KD-tree caster exists in the pl kernel only
    return launch_beam_pl(eng, c, poses, P, scan, N, origins, n_origins, out, status, lik_defaults, st, sink);
  const float4* s4 = reinterpret_cast<const float4*>(scan);
  switch (pick_tpp(P, N, c.sm_count))
  {
    case 32: return launch_beam_t<32>(eng, c, poses, static_cast<int>(P), s4, static_cast<int>(N), origins, out, status, lik_defaults, st, sink);
    case 64: return launch_beam_t<64>(eng, c, poses, static_cast<int>(P), s4, static_cast<int>(N), origins, out, status, lik_defaults, st, sink);
    case 128: return launch_beam_t<128>(eng, c, poses, static_cast<int>(P), s4, static_cast<int>(N), origins, out, status, lik_defaults, st, sink);
    default: return launch_beam_t<256>(eng, c, poses, static_cast<int>(P), s4, static_cast<int>(N), origins, out, status, lik_defaults, st, sink);
  }
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
int build_near_field(mcl3dl_engine* eng, DeviceCtx& c, cudaStream_t st, const mcl3dl_point* pts, uint32_t n, float wx,
                     float wy, float wz, float r, int k, const float sc_min[3], const float sc_max[3], DevBuf& buf,
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
  CK(cudaMemsetAsync(buf.p, 0, bytes, st));
  near_mark_kernel<<<(n + 255) / 256, 256, 0, st>>>(pts, n, wx, wy, wz, f, static_cast<uint32_t*>(buf.p), k);
  CK(cudaGetLastError());
  eng->launches++;
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
  auto cleanup = [&]() {
    free_buf(d_bits);
    free_buf(d_tot);
    free_buf(d_tmp);
  };
#define CKF(call)                                                                  \
  do                                                                               \
  {                                                                                \
    cudaError_t e__ = (call);                                                      \
    if (e__ != cudaSuccess)                                                        \
    {                                                                              \
      eng->err = std::string(#call) + ": " + cudaGetErrorString(e__);              \
      cleanup();                                                                   \
      return MCL3DL_ERR_CUDA;                                                      \
    }                                                                              \
  } while (0)
  const uint32_t wide_cap = static_cast<uint32_t>(std::min<size_t>(n_cells, size_t(1) << 18));
  const size_t sum_at = (n_cells + 5) & ~size_t(1);  // 64-bit grand total, 8-byte aligned behind the tail words
  if ((rc = reserve(eng, d_bits, bits_bytes)) || (rc = reserve(eng, d_tot, (sum_at + 2) * 4)) ||
      (rc = reserve(eng, c.nnf_dir, n_cells * sizeof(uint2))) || (rc = reserve(eng, c.nnf_wide, static_cast<size_t>(wide_cap) * sizeof(uint4))))
  {
    cleanup();
    return rc;
  }
  CKF(cudaMemsetAsync(d_bits.p, 0, bits_bytes, st));
  near_mark_kernel<<<(n + 255) / 256, 256, 0, st>>>(pts, n, g.wx, g.wy, g.wz, lay, static_cast<uint32_t*>(d_bits.p), 2);
  const unsigned blocks = static_cast<unsigned>((n_cells * 8 + 255) / 256);
  uint2* dir = static_cast<uint2*>(c.nnf_dir.p);
  uint32_t* tot = static_cast<uint32_t*>(d_tot.p);
  CKF(cudaMemsetAsync(tot + n_cells, 0, 16, st));  // [n_cells]: scan tail, [n_cells + 2] wide cells, [n_cells + 3] overflow cells
  f.wide = static_cast<const uint4*>(c.nnf_wide.p);
  nnf_count_kernel<<<blocks, 256, 0, st>>>(g, f, static_cast<const uint32_t*>(d_bits.p), lay.pitch, dir, tot, n_cells,
                                           static_cast<uint4*>(c.nnf_wide.p), wide_cap, tot + n_cells + 2);
  CKF(cudaGetLastError());
  // exclusive scan of the per-cell totals (in place); the grand total sizes the candidate array.  A candidate index
  // must stay below 2^31 (bit 31 of a directory entry marks wide / overflow cells): the total is first summed in 64 bits.
  cub::TransformInputIterator<unsigned long long, WidenU32, const uint32_t*> wide_in(tot, WidenU32());
  unsigned long long* d_sum = reinterpret_cast<unsigned long long*>(tot + sum_at);
  size_t tmp_bytes = 0, tmp_sum = 0;
  CKF(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, tot, tot, static_cast<int>(n_cells + 1), st));
  CKF(cub::DeviceReduce::Sum(nullptr, tmp_sum, wide_in, d_sum, static_cast<int>(n_cells), st));
  if ((rc = reserve(eng, d_tmp, std::max(tmp_bytes, tmp_sum))))
  {
    cleanup();
    return rc;
  }
  tmp_sum = d_tmp.cap;
  CKF(cub::DeviceReduce::Sum(d_tmp.p, tmp_sum, wide_in, d_sum, static_cast<int>(n_cells), st));
  unsigned long long sum64 = 0;
  CKF(cudaMemcpyAsync(&sum64, d_sum, 8, cudaMemcpyDeviceToHost, st));
  CKF(cudaStreamSynchronize(st));
  if (sum64 >= (1ull << 31))
  {
    cleanup();
    free_buf(c.nnf_dir);
    free_buf(c.nnf_wide);
    return MCL3DL_OK;
  }
  tmp_bytes = d_tmp.cap;
  CKF(cub::DeviceScan::ExclusiveSum(d_tmp.p, tmp_bytes, tot, tot, static_cast<int>(n_cells + 1), st));
  uint32_t tail[4] = {0, 0, 0, 0};
  CKF(cudaMemcpyAsync(tail, tot + n_cells, sizeof(tail), cudaMemcpyDeviceToHost, st));
  CKF(cudaStreamSynchronize(st));
  const uint32_t total = tail[0];
  eng->nnf_wide_cells = std::min<uint32_t>(tail[2], wide_cap);
  eng->nnf_overflow_cells = tail[3];
  const size_t cand_bytes = static_cast<size_t>(total) * sizeof(float4);
  if (n_cells * 8 + cand_bytes > eng->nnf_max_bytes)
  {
    cleanup();
    free_buf(c.nnf_dir);
    free_buf(c.nnf_wide);
    return MCL3DL_OK;
  }
  if ((rc = reserve(eng, c.nnf_cand, std::max<size_t>(cand_bytes, 16))))
  {
    cleanup();
    return rc;
  }
  nnf_base_kernel<<<static_cast<unsigned>((n_cells + 255) / 256), 256, 0, st>>>(dir, tot, n_cells, static_cast<uint4*>(c.nnf_wide.p));
  nnf_fill_kernel<<<blocks, 256, 0, st>>>(g, f, static_cast<const uint32_t*>(d_bits.p), lay.pitch, dir,
                                          static_cast<float4*>(c.nnf_cand.p), n_cells);
  CKF(cudaGetLastError());
  CKF(cudaStreamSynchronize(st));
  eng->launches += 4;
  f.dir = dir;
  f.cand = static_cast<const float4*>(c.nnf_cand.p);
  g.field = f;
  eng->nnf_bytes = n_cells * 8 + cand_bytes + static_cast<size_t>(wide_cap) * sizeof(uint4);
  eng->nnf_cands = total;
  c.map_bytes += eng->nnf_bytes;
  cleanup();
  return MCL3DL_OK;
#undef CKF
}

// Build both grids on one device from the uploaded points.
int build_map_on_device(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_point* h_pts, size_t n)
{
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = c.stream;
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  DevBuf d_pts, d_bbox, d_keys, d_vals, d_keys2, d_vals2, d_tmp;
  int rc = MCL3DL_OK;
  auto cleanup = [&]() {
    free_buf(d_pts);
    free_buf(d_bbox);
    free_buf(d_keys);
    free_buf(d_vals);
    free_buf(d_keys2);
    free_buf(d_vals2);
    free_buf(d_tmp);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
  };
#define CKB(x)            \
  do                      \
  {                       \
    rc = (x);             \
    if (rc != MCL3DL_OK)  \
    {                     \
      cleanup();          \
      return rc;          \
    }                     \
  } while (0)
#define CKC(call)                                                                       \
  do                                                                                    \
  {                                                                                     \
    cudaError_t e__ = (call);                                                           \
    if (e__ != cudaSuccess)                                                             \
    {                                                                                   \
      eng->err = std::string(#call) + ": " + cudaGetErrorString(e__);                   \
      cleanup();                                                                        \
      return MCL3DL_ERR_CUDA;                                                           \
    }                                                                                   \
  } while (0)

  const uint32_t n32 = static_cast<uint32_t>(n);
  const int tb = 256;
  const int nb = static_cast<int>((n + tb - 1) / tb);
  CKB(reserve(eng, d_pts, n * sizeof(mcl3dl_point)));
  CKB(reserve(eng, d_bbox, 12 * sizeof(uint32_t)));
  CKB(reserve(eng, d_keys, n * 4));
  CKB(reserve(eng, d_vals, n * 4));
  CKB(reserve(eng, d_keys2, n * 4));
  CKB(reserve(eng, d_vals2, n * 4));
  CKC(cudaMemcpyAsync(d_pts.p, h_pts, n * sizeof(mcl3dl_point), cudaMemcpyHostToDevice, st));
  CKC(cudaEventRecord(e0, st));
  const mcl3dl_point* pts = static_cast<const mcl3dl_point*>(d_pts.p);

  // ---- bounding boxes (raw: pcl::getMinMax3D, raycast_using_dda.h:175; rescaled: likelihood grid)
  uint32_t h_bbox[12];
  for (int k = 0; k < 3; ++k)
  {
    h_bbox[k] = 0xffffffffu;
    h_bbox[3 + k] = 0u;
    h_bbox[6 + k] = 0xffffffffu;
    h_bbox[9 + k] = 0u;
  }
  CKC(cudaMemcpyAsync(d_bbox.p, h_bbox, sizeof(h_bbox), cudaMemcpyHostToDevice, st));
  const float wx = eng->has_lik ? eng->lik.dist_weight[0] : 1.0f;
  const float wy = eng->has_lik ? eng->lik.dist_weight[1] : 1.0f;
  const float wz = eng->has_lik ? eng->lik.dist_weight[2] : 1.0f;
  bbox_kernel<<<std::min(nb, c.sm_count * 8), tb, 0, st>>>(pts, n, wx, wy, wz, static_cast<uint32_t*>(d_bbox.p));
  CKC(cudaGetLastError());
  eng->launches++;
  CKC(cudaMemcpyAsync(h_bbox, d_bbox.p, sizeof(h_bbox), cudaMemcpyDeviceToHost, st));
  CKC(cudaStreamSynchronize(st));
  float raw_min[3], raw_max[3], sc_min[3], sc_max[3];
  for (int k = 0; k < 3; ++k)
  {
    raw_min[k] = ord2f(h_bbox[k]);
    raw_max[k] = ord2f(h_bbox[3 + k]);
    sc_min[k] = ord2f(h_bbox[6 + k]);
    sc_max[k] = ord2f(h_bbox[9 + k]);
  }
  c.map_bytes = 0;

  // ---- likelihood search grid
  if (eng->has_lik)
  {
    NnGridDev g{};
    // the window (q -/+ rpad) must span at most 3 cells per axis: cell edge strictly above rpad
    // (1 % margin: the float cell function can be off by ~1e-7 x cells-per-axis, and the kernels rely on <= 3)
    const float cell = std::max(eng->lik.match_dist_min * eng->nn_cell_factor, eng->likdev.rpad * 1.01f);
    if (!(cell > 0.0f))
    {
      cleanup();
      return MCL3DL_ERR_INVALID_ARG;
    }
    g.inv_cell = 1.0f / cell;
    g.wx = wx;
    g.wy = wy;
    g.wz = wz;
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
    {
      cleanup();
      return MCL3DL_ERR_TOO_LARGE;
    }
    g.nx = dims[0];
    g.ny = dims[1];
    g.nz = dims[2];
    g.ox = org[0];
    g.oy = org[1];
    g.oz = org[2];
    const size_t cells = static_cast<size_t>(total);
    CKB(reserve(eng, c.nn_cell_start, (cells + 1) * 4));
    CKB(reserve(eng, c.nn_pts, n * 16));
    CKC(cudaMemsetAsync(c.nn_cell_start.p, 0, (cells + 1) * 4, st));
    nn_key_kernel<<<nb, tb, 0, st>>>(pts, n32, g, static_cast<uint32_t*>(d_keys.p), static_cast<uint32_t*>(d_vals.p),
                                     static_cast<uint32_t*>(c.nn_cell_start.p));
    CKC(cudaGetLastError());
    eng->launches++;
    size_t tmp_sort = 0, tmp_scan = 0;
    int end_bit = 1;
    while ((int64_t(1) << end_bit) < total && end_bit < 32) ++end_bit;
    CKC(cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, static_cast<uint32_t*>(d_keys.p),
                                        static_cast<uint32_t*>(d_keys2.p), static_cast<uint32_t*>(d_vals.p),
                                        static_cast<uint32_t*>(d_vals2.p), n32, 0, end_bit, st));
    CKC(cub::DeviceScan::InclusiveSum(nullptr, tmp_scan, static_cast<uint32_t*>(c.nn_cell_start.p),
                                      static_cast<uint32_t*>(c.nn_cell_start.p), static_cast<int>(cells + 1), st));
    CKB(reserve(eng, d_tmp, std::max(tmp_sort, tmp_scan)));
    size_t tsz = d_tmp.cap;
    CKC(cub::DeviceRadixSort::SortPairs(d_tmp.p, tsz, static_cast<uint32_t*>(d_keys.p), static_cast<uint32_t*>(d_keys2.p),
                                        static_cast<uint32_t*>(d_vals.p), static_cast<uint32_t*>(d_vals2.p), n32, 0,
                                        end_bit, st));
    tsz = d_tmp.cap;
    CKC(cub::DeviceScan::InclusiveSum(d_tmp.p, tsz, static_cast<uint32_t*>(c.nn_cell_start.p),
                                      static_cast<uint32_t*>(c.nn_cell_start.p), static_cast<int>(cells + 1), st));
    nn_gather_kernel<<<nb, tb, 0, st>>>(pts, n32, static_cast<uint32_t*>(d_vals2.p), wx, wy, wz,
                                        static_cast<float4*>(c.nn_pts.p));
    CKC(cudaGetLastError());
    eng->launches += 3;
    g.cell_start = static_cast<const uint32_t*>(c.nn_cell_start.p);
    g.pts = static_cast<const float4*>(c.nn_pts.p);
#if MCL3DL_NEAR_BITS
    CKB(build_near_field(eng, c, st, pts, n32, wx, wy, wz, eng->likdev.rpad, eng->near_k, sc_min, sc_max, c.near_lik, g.near, 0));
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
      if (eng->nnf && eng->mapping != 0)
        CKB(build_nn_field(eng, c, st, pts, n32, g, radius, sc_min, sc_max));
    }
    // window table of the CSR-window kernel (lik_kernel_wi): only when the field is not staged
    size_t row3_total = 0;
    g.nyp = (g.ny + 4) & ~1;  // even pitch with room for the 4-entry fetch starting at (ly & ~1)
    if (!g.field.dir)
    {
      row3_total = static_cast<size_t>(g.nz) * g.nx * g.nyp;
      CKB(reserve(eng, c.nn_row3, (row3_total + 2) * sizeof(uint2)));
      g.row3 = static_cast<const uint2*>(c.nn_row3.p);
      nn_row3_kernel<<<static_cast<unsigned>((row3_total + 255) / 256), 256, 0, st>>>(g, static_cast<uint2*>(c.nn_row3.p), row3_total);
      CKC(cudaGetLastError());
      eng->launches++;
    }
    else
    {
      free_buf(c.nn_row3);
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
  }

  // ---- KD-tree raycaster: marches over the likelihood grid; needs the raw points by original index
  if (eng->has_beam && !eng->beam.use_raycast_using_dda)
  {
    if (!eng->has_lik)
    {
      cleanup();
      return MCL3DL_ERR_INVALID_ARG;
    }
    fill_dda_scalars(eng->beam, c.dda);
    fill_kd_scalars(eng->beam, c.kd);
#if MCL3DL_NEAR_BITS
    CKB(build_near_field(eng, c, st, pts, n32, wx, wy, wz, c.kd.r1_pad, eng->near_kd_k, sc_min, sc_max, c.near_kd, c.kd.near, 1));
    c.near_kd_r = c.kd.r1_pad;
#endif
    free_buf(c.raw_pts);
    c.raw_pts = d_pts;  // keep the upload
    d_pts = DevBuf();
    c.kd.raw_pts = static_cast<const float4*>(c.raw_pts.p);
    c.map_bytes += n * 16;
  }
  // ---- DDA grid: updatePointCloud, raycast_using_dda.h:162-190
  if (eng->has_beam && eng->beam.use_raycast_using_dda)
  {
    DdaGridDev g{};
    fill_dda_scalars(eng->beam, g);
    if (!(g.grid > 0.0))
    {
      cleanup();
      return MCL3DL_ERR_INVALID_ARG;
    }
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
    {
      cleanup();
      return MCL3DL_ERR_TOO_LARGE;
    }
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
    CKB(reserve(eng, c.dda_cell_start, (cells + 2) * 4));
    CKB(reserve(eng, c.dda_occ, occ_words * 4));
    CKB(reserve(eng, c.dda_pts, n * 16));
    CKC(cudaMemsetAsync(c.dda_cell_start.p, 0, (cells + 2) * 4, st));
    CKC(cudaMemsetAsync(c.dda_occ.p, 0, occ_words * 4, st));
    dda_key_kernel<<<nb, tb, 0, st>>>(pts, n32, g, static_cast<uint32_t*>(d_keys.p), static_cast<uint32_t*>(d_vals.p),
                                      static_cast<uint32_t*>(c.dda_cell_start.p), static_cast<uint32_t*>(c.dda_occ.p));
    CKC(cudaGetLastError());
    size_t tmp_sort = 0, tmp_scan = 0;
    int end_bit = 1;
    while ((int64_t(1) << end_bit) < total && end_bit < 32) ++end_bit;
    CKC(cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, static_cast<uint32_t*>(d_keys.p),
                                        static_cast<uint32_t*>(d_keys2.p), static_cast<uint32_t*>(d_vals.p),
                                        static_cast<uint32_t*>(d_vals2.p), n32, 0, end_bit, st));
    CKC(cub::DeviceScan::InclusiveSum(nullptr, tmp_scan, static_cast<uint32_t*>(c.dda_cell_start.p),
                                      static_cast<uint32_t*>(c.dda_cell_start.p), static_cast<int>(cells + 1), st));
    CKB(reserve(eng, d_tmp, std::max(tmp_sort, tmp_scan)));
    size_t tsz = d_tmp.cap;
    CKC(cub::DeviceRadixSort::SortPairs(d_tmp.p, tsz, static_cast<uint32_t*>(d_keys.p), static_cast<uint32_t*>(d_keys2.p),
                                        static_cast<uint32_t*>(d_vals.p), static_cast<uint32_t*>(d_vals2.p), n32, 0,
                                        end_bit, st));
    tsz = d_tmp.cap;
    CKC(cub::DeviceScan::InclusiveSum(d_tmp.p, tsz, static_cast<uint32_t*>(c.dda_cell_start.p),
                                      static_cast<uint32_t*>(c.dda_cell_start.p), static_cast<int>(cells + 1), st));
    dda_gather_kernel<<<nb, tb, 0, st>>>(pts, n32, static_cast<uint32_t*>(d_vals2.p), static_cast<float4*>(c.dda_pts.p));
    CKC(cudaGetLastError());
    eng->launches += 4;
    g.occ = static_cast<const uint32_t*>(c.dda_occ.p);
    g.cell_start = static_cast<const uint32_t*>(c.dda_cell_start.p);
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
  CKC(cudaEventRecord(e1, st));
  CKC(cudaStreamSynchronize(st));
  float ms = 0;
  CKC(cudaEventElapsedTime(&ms, e0, e1));
  eng->info.build_ms = std::max(eng->info.build_ms, static_cast<double>(ms));
  eng->info.device_bytes = c.map_bytes;
  cleanup();
  return MCL3DL_OK;
#undef CKB
#undef CKC
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
  if (const char* v = std::getenv("MCL3DL_UPDATE_ONE_SYNC"))
    eng->update_one_sync = std::atoi(v) != 0;
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
  if (const char* o = std::getenv("MCL3DL_OVERLAP"))
    eng->overlap = std::atoi(o) != 0;
  if (const char* m = std::getenv("MCL3DL_MAPPING"))
    eng->mapping = (std::strcmp(m, "group") == 0) ? 0 : 1;
  eng->devs.resize(n_devices);
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
        cudaEventCreate(&c.ev_b0) != cudaSuccess || cudaEventCreate(&c.ev_b1) != cudaSuccess)
    {
      mcl3dl_destroy(eng);
      return MCL3DL_ERR_CUDA;
    }
  }
  *out = eng;
  return MCL3DL_OK;
}

static void xchg_close(DeviceCtx& c);

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
  for (DeviceCtx& c : eng->devs)
  {
    cudaSetDevice(c.dev);
    if (c.stream)
      cudaStreamSynchronize(c.stream);
    xchg_close(c);
    free_buf(c.xchg);
    free_buf(c.x_ticket);
    for (DevBuf* b : {&c.r_states[0], &c.r_states[1], &c.r_prob, &c.r_accum, &c.r_poses, &c.r_extra, &c.r_est, &c.s_raw, &c.s_keys[0],
                      &c.s_keys[1], &c.s_vals[0], &c.s_vals[1], &c.s_flags[0], &c.s_flags[1], &c.s_pos[0], &c.s_pos[1], &c.s_ds,
                      &c.s_clip[0], &c.s_clip[1], &c.s_out[0], &c.s_out[1], &c.s_tmp, &c.s_counts})
      free_buf(*b);
    for (DevBuf* b : {&c.nn_cell_start, &c.nn_pts, &c.nn_row3, &c.dda_occ, &c.dda_cell_start, &c.dda_pts, &c.raw_pts, &c.near_lik, &c.near_kd, &c.nnf_dir, &c.nnf_cand, &c.nnf_wide, &c.fld_cells, &c.d_poses,
                      &c.d_out, &c.d_status, &c.d_stats, &c.d_partial, &c.d_tickets, &c.d_tally, &c.d_queue, &c.d_lacc, &c.d_w, &c.d_post, &c.d_wpart, &c.d_wticket})
      free_buf(*b);
    if (c.fld_nodes.ptr)
      cudaFree(c.fld_nodes.ptr);
    if (c.h_pinned)
      cudaFreeHost(c.h_pinned);
    for (auto& e : c.ev)
      if (e)
        cudaEventDestroy(e);
    for (cudaEvent_t e : {c.ev_fork, c.ev_join, c.ev_b0, c.ev_b1})
      if (e)
        cudaEventDestroy(e);
    if (c.side)
    {
      cudaStreamSynchronize(c.side);
      cudaStreamDestroy(c.side);
    }
    if (c.stream)
      cudaStreamDestroy(c.stream);
  }
  for (auto& b : eng->host_blocks)  // (blocks the caller did not return; its pointers into them dangle from here on)
    cudaFreeHost(b.first);
  delete eng;
}

int mcl3dl_set_map(mcl3dl_engine* eng, const mcl3dl_point* pts, size_t n, uint64_t stamp, const mcl3dl_lik_params* lik,
                   const mcl3dl_beam_params* beam)
{
  if (!eng || !pts || n == 0 || (!lik && !beam))
    return MCL3DL_ERR_INVALID_ARG;
  if (n >= (size_t(1) << 31))
    return MCL3DL_ERR_TOO_LARGE;
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
    int rc = build_map_on_device(eng, c, pts, n);
    if (rc != MCL3DL_OK)
      return rc;
    c.fld_nodes_valid = false;  // a volume of the previous map is stale
    if (c.fld_nodes.ptr)
    {
      cudaFree(c.fld_nodes.ptr);
      c.fld_nodes = cudaPitchedPtr{};
    }
    if (eng->field_mode && eng->has_lik && (rc = stage_field(eng, c, nullptr)) != MCL3DL_OK)
      return rc;
  }
  eng->has_map = true;
  eng->stamp = stamp;
  eng->n_points = n;
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

static int validate_measure(mcl3dl_engine* eng, size_t P, size_t n_lik, size_t n_beam, size_t n_origins)
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

int mcl3dl_measure_device(mcl3dl_engine* eng, const mcl3dl_pose* d_poses, size_t P, const mcl3dl_point* d_lik, size_t n_lik,
                          const mcl3dl_point* d_beam, size_t n_beam, const float* d_origins_xyz, size_t n_origins,
                          mcl3dl_result* d_out, void* cuda_stream)
{
  int rc = validate_measure(eng, P, n_lik, n_beam, n_origins);
  if (rc != MCL3DL_OK)
    return rc;
  if (eng->devs.size() != 1 || (P && (!d_poses || !d_out)) || (n_lik && !d_lik) || (n_beam && (!d_beam || !d_origins_xyz)))
    return MCL3DL_ERR_INVALID_ARG;
  if (P == 0)
    return MCL3DL_OK;
  DeviceCtx& c = eng->devs[0];
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  return launch_models(eng, c, d_poses, P, d_lik, n_lik, d_beam, n_beam, d_origins_xyz, n_origins, d_out, nullptr, st, false);
}

// ---- resident particle set (scope row f3; prepared, not yet run on hardware — see include/mcl3dl_b200.h)
int mcl3dl_particles_set(mcl3dl_engine* eng, const mcl3dl_state* states, const float* prob, size_t n)
{
  if (!eng || eng->devs.size() != 1 || !states || !prob || n == 0 || n >= (size_t(1) << 31))
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  CK(cudaSetDevice(c.dev));
  int rc;
  if ((rc = reserve(eng, c.r_states[0], n * sizeof(mcl3dl_state))) || (rc = reserve(eng, c.r_states[1], n * sizeof(mcl3dl_state))) ||
      (rc = reserve(eng, c.r_prob, n * 4)) || (rc = reserve(eng, c.r_accum, (n + 1) * 4)) ||
      (rc = reserve(eng, c.r_poses, n * sizeof(mcl3dl_pose))) || (rc = reserve(eng, c.r_extra, n * 4)))
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
  pf_predict_kernel<<<(n + 255) / 256, 256, 0, c.stream>>>(static_cast<PfState*>(c.r_states[c.r_cur].p), n, m);
  CK(cudaGetLastError());
  eng->launches++;
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
  pf_accum_kernel<<<1, 32, 0, c.stream>>>(static_cast<const float*>(c.r_prob.p), n, accum, accum + n);  // one warp, in order
  Sigma6 sg;
  for (int k = 0; k < 3; ++k)
  {
    sg.v[k] = sigma_pos[k];
    sg.v[k + 3] = sigma_rpy[k];
  }
  ++c.r_calls;
  pf_resample_kernel<<<(n + 255) / 256, 256, 0, c.stream>>>(static_cast<const PfState*>(c.r_states[c.r_cur].p), accum, accum + n, n,
                                                           initial_frac, seed, c.r_calls, sg,
                                                           static_cast<PfState*>(c.r_states[1 - c.r_cur].p),
                                                           static_cast<float*>(c.r_prob.p));
  CK(cudaGetLastError());
  eng->launches += 2;
  c.r_cur = 1 - c.r_cur;
  return MCL3DL_OK;
}

// The resident update with every input already on the device: pose pack -> both models -> prior * likelihood * odometry
// term -> normalise; one synchronise.  `stage` = bytes of host inputs waiting in the pinned block for one H2D copy.
static int resident_update(mcl3dl_engine* eng, DeviceCtx& c, const mcl3dl_point* d_lik, size_t n_lik, const mcl3dl_point* d_beam,
                           size_t n_beam, const float* d_org, size_t n_origins, float odom_err_lin_sigma, size_t pinned_off,
                           mcl3dl_update_summary* summary)
{
  const size_t P = c.r_n;
  cudaStream_t st = c.stream;
  int rc;
  const int nblk = static_cast<int>(std::min<size_t>((P + kBlockThreads - 1) / kBlockThreads, static_cast<size_t>(c.sm_count) * 4));
  if ((rc = reserve(eng, c.d_out, P * sizeof(mcl3dl_result))) || (rc = reserve(eng, c.d_w, P * 4)) ||
      (rc = reserve(eng, c.d_wpart, 2 * (nblk + 1) * sizeof(WeightPartial))))
    return rc;
  // NormalLikelihood(sigma): a_ = float(1 / sqrt(2 pi s^2)), sq2_ = float(2 s^2) (include/mcl_3dl/nd.h:45-49)
  const bool with_odom = odom_err_lin_sigma > 0.0f;
  const double sg = static_cast<double>(odom_err_lin_sigma);
  const float nd_a = with_odom ? static_cast<float>(1.0 / std::sqrt(2.0 * M_PI * sg * sg)) : 1.0f;
  const float nd_sq2 = with_odom ? static_cast<float>(sg * sg * 2.0) : 1.0f;
  const uint32_t n32 = static_cast<uint32_t>(P);
  pf_pack_kernel<<<(n32 + 255) / 256, 256, 0, st>>>(static_cast<const PfState*>(c.r_states[c.r_cur].p), n32, nd_a, nd_sq2,
                                                  static_cast<mcl3dl_pose*>(c.r_poses.p),
                                                  with_odom ? static_cast<float*>(c.r_extra.p) : nullptr);
  CK(cudaGetLastError());
  eng->launches++;
  rc = launch_models(eng, c, static_cast<const mcl3dl_pose*>(c.r_poses.p), P, d_lik, n_lik, d_beam, n_beam, d_org, n_origins,
                     static_cast<mcl3dl_result*>(c.d_out.p), nullptr, st, false);
  if (rc != MCL3DL_OK)
    return rc;
  // prior * likelihood from the resident probabilities; the posterior is written over them (the weights were read
  // into d_w first); a vanished total leaves them untouched = the reference's "restore" (pf.h:274-278)
  WeightPartial* parts = static_cast<WeightPartial*>(c.d_wpart.p);
  WeightPartial* parts2 = parts + nblk + 1;
  unsigned int* tk;
  if ((rc = weight_tickets(eng, c, &tk)))
    return rc;
  weight_kernel<<<nblk, kBlockThreads, 0, st>>>(static_cast<const mcl3dl_result*>(c.d_out.p), static_cast<const float*>(c.r_prob.p),
                                               with_odom ? static_cast<const float*>(c.r_extra.p) : nullptr, static_cast<int>(P),
                                               static_cast<int>(n_lik), static_cast<float*>(c.d_w.p), parts, tk, nullptr);
  normalize_kernel_dev<<<nblk, kBlockThreads, 0, st>>>(static_cast<const float*>(c.d_w.p), static_cast<int>(P), parts + nblk, 0,
                                                      static_cast<float*>(c.r_prob.p), parts2, tk + 1, nullptr);
  CK(cudaGetLastError());
  eng->launches += 2;
  char* h_tot = static_cast<char*>(c.h_pinned) + pinned_off;
  CK(cudaMemcpyAsync(h_tot, parts + nblk, sizeof(WeightPartial), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(h_tot + sizeof(WeightPartial), parts2 + nblk, sizeof(WeightPartial), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  WeightPartial w1, w2;
  std::memcpy(&w1, h_tot, sizeof(w1));
  std::memcpy(&w2, h_tot + sizeof(w1), sizeof(w2));
  std::memset(summary, 0, sizeof(*summary));
  const float total_f = static_cast<float>(w1.sum);
  summary->weight_sum = total_f;
  summary->match_ratio_min = std::min(1.0f, w1.qmin);
  summary->match_ratio_max = std::max(0.0f, w1.qmax);
  summary->kept = total_f > 0.0f ? 1 : 0;
  summary->entropy = summary->kept ? static_cast<float>(-w2.sum) : 0.0f;
  summary->max_index = summary->kept ? w2.best_i : 0;
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
  int rc = validate_measure(eng, P, n_lik, n_beam, n_origins);
  if (rc != MCL3DL_OK)
    return rc;
  if (P == 0 || (n_lik && !lik_pts) || (n_beam && (!beam_pts || !origins_xyz)))
    return MCL3DL_ERR_INVALID_ARG;
  for (size_t j = 0; j < n_beam; ++j)
    if (beam_pts[j].label >= n_origins)
      return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  // scans + origins up in one block (as in mcl3dl_measure); the poses come from the resident states
  const size_t o_beam = n_lik * 16, o_org = o_beam + n_beam * 16, in_bytes = o_org + ((n_origins * 12 + 15) & ~size_t(15));
  if ((rc = reserve_pinned(eng, c, in_bytes + 2 * sizeof(WeightPartial) + 64)) || (rc = reserve(eng, c.d_poses, in_bytes + 16)))
    return rc;
  char* hp = static_cast<char*>(c.h_pinned);
  if (n_lik) std::memcpy(hp, lik_pts, n_lik * 16);
  if (n_beam) std::memcpy(hp + o_beam, beam_pts, n_beam * 16);
  if (n_origins) std::memcpy(hp + o_org, origins_xyz, n_origins * 12);
  if (in_bytes) CK(cudaMemcpyAsync(c.d_poses.p, hp, in_bytes, cudaMemcpyHostToDevice, c.stream));
  const char* d_in = static_cast<const char*>(c.d_poses.p);
  return resident_update(eng, c, reinterpret_cast<const mcl3dl_point*>(d_in), n_lik, reinterpret_cast<const mcl3dl_point*>(d_in + o_beam),
                         n_beam, reinterpret_cast<const float*>(d_in + o_org), n_origins, odom_err_lin_sigma, in_bytes, summary);
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
  int rc = validate_measure(eng, P, n_lik, n_beam, n_origins);
  if (rc != MCL3DL_OK)
    return rc;
  if (P == 0 || (n_beam && !origins_xyz))
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  const size_t in_bytes = (n_origins * 12 + 15) & ~size_t(15);
  if ((rc = reserve_pinned(eng, c, in_bytes + 2 * sizeof(WeightPartial) + 64)) || (rc = reserve(eng, c.d_poses, in_bytes + 16)))
    return rc;
  if (n_origins)
  {
    std::memcpy(c.h_pinned, origins_xyz, n_origins * 12);
    CK(cudaMemcpyAsync(c.d_poses.p, c.h_pinned, in_bytes, cudaMemcpyHostToDevice, c.stream));
  }
  // (beam labels are the raw cloud's, voted per voxel: the caller's origins must cover them, as in the node)
  return resident_update(eng, c, static_cast<const mcl3dl_point*>(c.s_out[0].p), n_lik, static_cast<const mcl3dl_point*>(c.s_out[1].p),
                         n_beam, static_cast<const float*>(c.d_poses.p), n_origins, odom_err_lin_sigma, in_bytes, summary);
}

// ---- scan preprocessing on the device (scan_kernels.cuh)
int mcl3dl_scan_prepare(mcl3dl_engine* eng, const mcl3dl_point* raw, size_t n_raw, const mcl3dl_scan_params* sp, mcl3dl_scan_info* info)
{
  if (!eng || eng->devs.size() != 1 || !sp || (n_raw && !raw) || n_raw >= (size_t(1) << 30))
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = c.stream;
  c.s_valid = false;
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
  if ((rc = reserve_pinned(eng, c, 256)))
    return rc;
  CK(cudaMemcpyAsync(c.s_raw.p, raw, n_raw * 16, cudaMemcpyHostToDevice, st));
  const mcl3dl_point* d_raw = static_cast<const mcl3dl_point*>(c.s_raw.p);
  const mcl3dl_point* d_ds = d_raw;
  const int nb = static_cast<int>((n + 255) / 256);
  const bool downsample = sp->downsample[0] > 0.0f && sp->downsample[1] > 0.0f && sp->downsample[2] > 0.0f;
  bool ds_done = false;
  if (downsample)
  {
    // bounding box -> VoxelGrid lattice (getMinMax3D; min_b / max_b / div_b of voxel_grid.hpp)
    uint32_t h_bbox[12];
    for (int k = 0; k < 3; ++k)
    {
      h_bbox[k] = 0xffffffffu;
      h_bbox[3 + k] = 0u;
      h_bbox[6 + k] = 0xffffffffu;
      h_bbox[9 + k] = 0u;
    }
    if ((rc = reserve(eng, c.s_tmp, 4096)))
      return rc;
    uint32_t* bb = static_cast<uint32_t*>(c.s_tmp.p);
    CK(cudaMemcpyAsync(bb, h_bbox, sizeof(h_bbox), cudaMemcpyHostToDevice, st));
    bbox_kernel<<<std::min(nb, c.sm_count * 8), 256, 0, st>>>(d_raw, n_raw, 1.0f, 1.0f, 1.0f, bb);
    CK(cudaGetLastError());
    eng->launches++;
    CK(cudaMemcpyAsync(h_bbox, bb, sizeof(h_bbox), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    VoxelGridDev g{};
    double cells = 1.0;
    for (int k = 0; k < 3; ++k)
    {
      g.inv_leaf[k] = 1.0f / sp->downsample[k];
      const float mn = ord2f(h_bbox[k]), mx = ord2f(h_bbox[3 + k]);
      g.min_b[k] = static_cast<int>(std::floor(mn * g.inv_leaf[k]));
      const int max_b = static_cast<int>(std::floor(mx * g.inv_leaf[k]));
      g.div_b[k] = max_b - g.min_b[k] + 1;
      cells *= static_cast<double>(g.div_b[k]);
    }
    if (cells < 4294967295.0)  // (PCL itself refuses above INT_MAX voxels and returns the cloud unfiltered)
    {
      uint32_t *k0 = static_cast<uint32_t*>(c.s_keys[0].p), *k1 = static_cast<uint32_t*>(c.s_keys[1].p);
      uint32_t *v0 = static_cast<uint32_t*>(c.s_vals[0].p), *v1 = static_cast<uint32_t*>(c.s_vals[1].p);
      uint32_t *fl = static_cast<uint32_t*>(c.s_flags[0].p), *ps = static_cast<uint32_t*>(c.s_pos[0].p);
      scan_key_kernel<<<nb, 256, 0, st>>>(d_raw, n, g, k0, v0);
      size_t t_sort = 0, t_scan = 0;
      int end_bit = 1;
      while ((1.0 * (uint64_t(1) << end_bit)) < cells && end_bit < 32) ++end_bit;
      CK(cub::DeviceRadixSort::SortPairs(nullptr, t_sort, k0, k1, v0, v1, n, 0, end_bit, st));
      CK(cub::DeviceScan::ExclusiveSum(nullptr, t_scan, fl, ps, n, st));
      if ((rc = reserve(eng, c.s_tmp, std::max(t_sort, t_scan) + 256)))
        return rc;
      size_t tsz = c.s_tmp.cap;
      CK(cub::DeviceRadixSort::SortPairs(c.s_tmp.p, tsz, k0, k1, v0, v1, n, 0, end_bit, st));  // stable: input order inside a voxel
      scan_heads_kernel<<<nb, 256, 0, st>>>(k1, n, fl);
      tsz = c.s_tmp.cap;
      CK(cub::DeviceScan::ExclusiveSum(c.s_tmp.p, tsz, fl, ps, n, st));
      scan_centroid_kernel<<<nb, 256, 0, st>>>(d_raw, k1, v1, fl, ps, n, static_cast<mcl3dl_point*>(c.s_ds.p), counts + 0);
      CK(cudaGetLastError());
      eng->launches += 5;
      d_ds = static_cast<const mcl3dl_point*>(c.s_ds.p);
      ds_done = true;
    }
  }
  if (!ds_done)
  {
    CK(cudaMemcpyAsync(c.s_ds.p, c.s_raw.p, n_raw * 16, cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(counts, &c.s_info.n_raw, 4, cudaMemcpyHostToDevice, st));
    d_ds = static_cast<const mcl3dl_point*>(c.s_ds.p);
  }
  // clip (both models at once), compaction in order, then the uniform sample
  const ClipDev ca{sp->lik_clip_near * sp->lik_clip_near, sp->lik_clip_far * sp->lik_clip_far, sp->lik_clip_z_min, sp->lik_clip_z_max};
  const ClipDev cb{sp->beam_clip_near * sp->beam_clip_near, sp->beam_clip_far * sp->beam_clip_far, sp->beam_clip_z_min, sp->beam_clip_z_max};
  uint32_t *fa = static_cast<uint32_t*>(c.s_flags[0].p), *fb = static_cast<uint32_t*>(c.s_flags[1].p);
  uint32_t *pa = static_cast<uint32_t*>(c.s_pos[0].p), *pb = static_cast<uint32_t*>(c.s_pos[1].p);
  scan_clip_flags_kernel<<<nb, 256, 0, st>>>(d_ds, counts + 0, ca, cb, fa, fb, n);
  size_t t_scan = 0;
  CK(cub::DeviceScan::ExclusiveSum(nullptr, t_scan, fa, pa, n, st));
  if ((rc = reserve(eng, c.s_tmp, t_scan + 256)))
    return rc;
  size_t tsz = c.s_tmp.cap;
  CK(cub::DeviceScan::ExclusiveSum(c.s_tmp.p, tsz, fa, pa, n, st));
  tsz = c.s_tmp.cap;
  CK(cub::DeviceScan::ExclusiveSum(c.s_tmp.p, tsz, fb, pb, n, st));
  scan_compact_kernel<<<nb, 256, 0, st>>>(d_ds, fa, pa, n, static_cast<mcl3dl_point*>(c.s_clip[0].p), counts + 1);
  scan_compact_kernel<<<nb, 256, 0, st>>>(d_ds, fb, pb, n, static_cast<mcl3dl_point*>(c.s_clip[1].p), counts + 2);
  for (int k = 0; k < 2; ++k)
    if (num[k])
      scan_sample_kernel<<<(num[k] + 255) / 256, 256, 0, st>>>(static_cast<const mcl3dl_point*>(c.s_clip[k].p), counts + 1 + k, num[k],
                                                             sp->seed, static_cast<uint32_t>(k),
                                                             static_cast<mcl3dl_point*>(c.s_out[k].p), counts + 3 + k);
  CK(cudaGetLastError());
  eng->launches += 5;
  uint32_t h_counts[5];
  CK(cudaMemcpyAsync(c.h_pinned, counts, sizeof(h_counts), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  std::memcpy(h_counts, c.h_pinned, sizeof(h_counts));
  c.s_info.n_downsampled = h_counts[0];
  c.s_info.n_lik_clipped = h_counts[1];
  c.s_info.n_beam_clipped = h_counts[2];
  c.s_info.n_lik = h_counts[3];
  c.s_info.n_beam = h_counts[4];
  c.s_valid = true;
  if (info) *info = c.s_info;
  return MCL3DL_OK;
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
  if ((rc = reserve(eng, c.r_est, hdr + part_doubles * sizeof(double))) || (rc = reserve_pinned(eng, c, sizeof(EstHeader) + sizeof(PfState) + 64)))
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
  pf_est_pass1_kernel<<<grid, 256, 0, st>>>(states, probs, n, b, parts);
  pf_est_finish1_kernel<<<1, 32, 0, st>>>(parts, grid, h);
  pf_est_pass2_kernel<<<grid, 256, 0, st>>>(states, probs, n, h, parts);
  pf_est_finish2_kernel<<<1, 32, 0, st>>>(parts, grid, h);
  CK(cudaGetLastError());
  eng->launches += 4;
  char* hp = static_cast<char*>(c.h_pinned);
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

static void xchg_close(DeviceCtx& c)
{
  for (void*& o : c.x_opened)
    if (o)
    {
      cudaIpcCloseMemHandle(o);
      o = nullptr;
    }
  c.x_ready = false;
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
        xchg_close(c);
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
  int rc = validate_measure(eng, P, n_lik, n_beam, n_origins);
  if (rc != MCL3DL_OK)
    return rc;
  if (eng->devs.size() != 1 || !d_poses || (n_lik && !d_lik) || (n_beam && (!d_beam || !d_origins_xyz)))
    return MCL3DL_ERR_INVALID_ARG;
  DeviceCtx& c = eng->devs[0];
  if (!c.x_ready || P != c.x_local)
    return MCL3DL_ERR_INVALID_ARG;
  CK(cudaSetDevice(c.dev));
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  rc = launch_models(eng, c, d_poses, P, d_lik, n_lik, d_beam, n_beam, d_origins_xyz, n_origins, nullptr, nullptr, st, false,
                     &c.xsink);
  if (rc != MCL3DL_OK)
    return rc;
  unsigned int* tk = static_cast<unsigned int*>(c.x_ticket.p);
  exchange_signal_kernel<<<1, 32, 0, st>>>(c.xt, tk, tk + 1);
  CK(cudaGetLastError());
  eng->launches++;
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
  int rc = validate_measure(eng, P, n_lik, n_beam, n_origins);
  if (rc != MCL3DL_OK)
    return rc;
  if ((P && (!poses || (!out && !status))) || (n_lik && !lik_pts) || (n_beam && (!beam_pts || !origins_xyz)))
    return MCL3DL_ERR_INVALID_ARG;
  for (size_t j = 0; j < n_beam; ++j)
    if (beam_pts[j].label >= n_origins)  // origins[p.label], beam.cpp:142-145
      return MCL3DL_ERR_INVALID_ARG;
  if (P == 0)
    return MCL3DL_OK;
  const size_t G = eng->devs.size();
  std::vector<size_t> p0(G + 1);
  for (size_t d = 0; d <= G; ++d) p0[d] = P * d / G;
  // enqueue everything on every device, then wait
  for (size_t d = 0; d < G; ++d)
  {
    DeviceCtx& c = eng->devs[d];
    const size_t Pd = p0[d + 1] - p0[d];
    if (Pd == 0)
      continue;
    CK(cudaSetDevice(c.dev));
    cudaStream_t st = c.stream;
    const size_t b_poses = Pd * sizeof(mcl3dl_pose), b_lik = n_lik * 16, b_beam = n_beam * 16, b_org = (n_origins * 12 + 15) & ~size_t(15);
    const size_t b_out = Pd * sizeof(mcl3dl_result), b_status = status ? Pd * n_beam : 0;
    const size_t o_lik = b_poses, o_beam = o_lik + b_lik, o_org = o_beam + b_beam, o_out = o_org + b_org;
    const size_t o_status = o_out + b_out;
    rc = reserve_pinned(eng, c, o_status + b_status + 64);
    if (rc != MCL3DL_OK) return rc;
    // one staging block, one H2D copy: [poses | likelihood scan | beam scan | origins] (all 16-byte multiples)
    if ((rc = reserve(eng, c.d_poses, o_out)) || (rc = reserve(eng, c.d_out, b_out)) || (rc = reserve(eng, c.d_status, b_status)))
      return rc;
    char* hp = static_cast<char*>(c.h_pinned);
    // caller arrays inside a mcl3dl_host_alloc block are page-locked: a large pose array is DMA-ed from where it lies
    // and the records land where the caller reads them, without the staging memcpy on either side
    const bool poses_direct = b_poses >= eng->direct_min_bytes && in_host_block(eng, poses + p0[d], b_poses);
    const bool out_direct = out && eng->direct_min_bytes != ~size_t(0) && in_host_block(eng, out + p0[d], b_out);
    if (!poses_direct) std::memcpy(hp, poses + p0[d], b_poses);
    if (b_lik) std::memcpy(hp + o_lik, lik_pts, b_lik);
    if (b_beam) std::memcpy(hp + o_beam, beam_pts, b_beam);
    if (n_origins) std::memcpy(hp + o_org, origins_xyz, n_origins * 12);
    const bool timed = eng->timing != 0;
    // small updates: the kernels store their records straight into the pinned block (cudaMallocHost memory is mapped
    // into the unified address space), which saves the D2H copy launch; large ones keep the bulk copy
    const bool zc = !status && Pd <= eng->zero_copy_max;  // (per-ray status bytes would be scattered 1-byte PCIe writes)
    if (timed) CK(cudaEventRecord(c.ev[0], st));
    if (poses_direct)
    {
      CK(cudaMemcpyAsync(c.d_poses.p, poses + p0[d], b_poses, cudaMemcpyHostToDevice, st));
      if (o_out > o_lik)
        CK(cudaMemcpyAsync(static_cast<char*>(c.d_poses.p) + o_lik, hp + o_lik, o_out - o_lik, cudaMemcpyHostToDevice, st));
    }
    else
      CK(cudaMemcpyAsync(c.d_poses.p, hp, o_out, cudaMemcpyHostToDevice, st));
    const char* d_in = static_cast<const char*>(c.d_poses.p);
    const mcl3dl_pose* d_poses = reinterpret_cast<const mcl3dl_pose*>(d_in);
    const mcl3dl_point* d_lik = reinterpret_cast<const mcl3dl_point*>(d_in + o_lik);
    const mcl3dl_point* d_beam = reinterpret_cast<const mcl3dl_point*>(d_in + o_beam);
    const float* d_org = reinterpret_cast<const float*>(d_in + o_org);
    if (timed) CK(cudaEventRecord(c.ev[1], st));
    mcl3dl_result* h_out = out_direct ? out + p0[d] : reinterpret_cast<mcl3dl_result*>(hp + o_out);
    mcl3dl_result* k_out = zc ? h_out : static_cast<mcl3dl_result*>(c.d_out.p);
    uint8_t* k_status = status ? static_cast<uint8_t*>(c.d_status.p) : nullptr;
    rc = launch_models(eng, c, d_poses, Pd, d_lik, n_lik, d_beam, n_beam, d_org, n_origins, k_out, k_status, st, timed);
    if (rc != MCL3DL_OK) return rc;
    if (timed) CK(cudaEventRecord(c.ev[5], st));
    if (!zc)
    {
      CK(cudaMemcpyAsync(h_out, c.d_out.p, b_out, cudaMemcpyDeviceToHost, st));
      if (b_status) CK(cudaMemcpyAsync(hp + o_status, c.d_status.p, b_status, cudaMemcpyDeviceToHost, st));
    }
    if (timed) CK(cudaEventRecord(c.ev[4], st));
  }
  eng->t_h2d = eng->t_lik = eng->t_beam = eng->t_d2h = 0;
  for (size_t d = 0; d < G; ++d)
  {
    DeviceCtx& c = eng->devs[d];
    const size_t Pd = p0[d + 1] - p0[d];
    if (Pd == 0)
      continue;
    CK(cudaSetDevice(c.dev));
    CK(cudaStreamSynchronize(c.stream));
    const size_t o_out = Pd * sizeof(mcl3dl_pose) + n_lik * 16 + n_beam * 16 + ((n_origins * 12 + 15) & ~size_t(15));
    const size_t o_status = o_out + Pd * sizeof(mcl3dl_result);
    const char* hp = static_cast<const char*>(c.h_pinned);
    if (out && !(eng->direct_min_bytes != ~size_t(0) && in_host_block(eng, out + p0[d], Pd * sizeof(mcl3dl_result))))  // (else: already there)
      std::memcpy(out + p0[d], hp + o_out, Pd * sizeof(mcl3dl_result));
    if (status) std::memcpy(status + p0[d] * n_beam, hp + o_status, Pd * n_beam);
    float ms_h2d = 0, ms_lik = 0, ms_beam = 0, ms_d2h = 0;
    if (eng->timing)
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
  int rc = validate_measure(eng, P, n_lik, n_beam, n_origins);
  if (rc != MCL3DL_OK)
    return rc;
  if (!summary || (P && (!poses || !prior || !posterior)) || (n_lik && !lik_pts) || (n_beam && (!beam_pts || !origins_xyz)))
    return MCL3DL_ERR_INVALID_ARG;
  for (size_t j = 0; j < n_beam; ++j)
    if (beam_pts[j].label >= n_origins)
      return MCL3DL_ERR_INVALID_ARG;
  std::memset(summary, 0, sizeof(*summary));
  summary->match_ratio_min = 1.0f;
  if (P == 0)
    return MCL3DL_OK;
  const size_t G = eng->devs.size();
  std::vector<size_t> p0(G + 1);
  for (size_t d = 0; d <= G; ++d) p0[d] = P * d / G;
  struct Lay
  {
    size_t o_lik, o_beam, o_org, o_prior, o_extra, in_bytes, o_post, o_rec, o_part, total;
    int nblk;
    bool zc;
  };
  std::vector<Lay> lay(G);
  // One device: the total never leaves the device (normalize_kernel_dev reads pass 1's folded slot) and everything comes
  // back after ONE synchronise; small updates store the posterior, the records and the two summaries straight into the
  // pinned block (no D2H copy launches).  Several devices: the total is a sum over devices, so two host round trips.
  const bool one_sync = eng->update_one_sync && G == 1;
  // ---- pass 1 on every device: inputs up, both models, w_i and its reduction
  for (size_t d = 0; d < G; ++d)
  {
    DeviceCtx& c = eng->devs[d];
    const size_t Pd = p0[d + 1] - p0[d];
    if (Pd == 0)
      continue;
    CK(cudaSetDevice(c.dev));
    cudaStream_t st = c.stream;
    Lay& L = lay[d];
    L.o_lik = Pd * sizeof(mcl3dl_pose);
    L.o_beam = L.o_lik + n_lik * 16;
    L.o_org = L.o_beam + n_beam * 16;
    L.o_prior = L.o_org + ((n_origins * 12 + 15) & ~size_t(15));
    L.o_extra = L.o_prior + ((Pd * 4 + 15) & ~size_t(15));
    L.in_bytes = L.o_extra + (extra ? ((Pd * 4 + 15) & ~size_t(15)) : 0);
    L.o_post = L.in_bytes;
    L.o_rec = L.o_post + ((Pd * 4 + 15) & ~size_t(15));
    L.o_part = (L.o_rec + (records ? Pd * sizeof(mcl3dl_result) : 0) + 15) & ~size_t(15);
    L.total = L.o_part + 2 * sizeof(WeightPartial) + 64;
    L.nblk = static_cast<int>(std::min<size_t>((Pd + kBlockThreads - 1) / kBlockThreads, static_cast<size_t>(c.sm_count) * 4));
    L.zc = one_sync && Pd <= eng->zero_copy_max;
    unsigned int* tk;
    if ((rc = reserve_pinned(eng, c, L.total)) || (rc = reserve(eng, c.d_poses, L.in_bytes)) ||
        (rc = reserve(eng, c.d_out, Pd * sizeof(mcl3dl_result))) || (rc = reserve(eng, c.d_w, Pd * 4)) ||
        (rc = reserve(eng, c.d_post, Pd * 4)) || (rc = reserve(eng, c.d_wpart, 2 * (L.nblk + 1) * sizeof(WeightPartial))) ||
        (rc = weight_tickets(eng, c, &tk)))
      return rc;
    char* hp = static_cast<char*>(c.h_pinned);
    std::memcpy(hp, poses + p0[d], Pd * sizeof(mcl3dl_pose));
    if (n_lik) std::memcpy(hp + L.o_lik, lik_pts, n_lik * 16);
    if (n_beam) std::memcpy(hp + L.o_beam, beam_pts, n_beam * 16);
    if (n_origins) std::memcpy(hp + L.o_org, origins_xyz, n_origins * 12);
    std::memcpy(hp + L.o_prior, prior + p0[d], Pd * 4);
    if (extra) std::memcpy(hp + L.o_extra, extra + p0[d], Pd * 4);
    CK(cudaMemcpyAsync(c.d_poses.p, hp, L.in_bytes, cudaMemcpyHostToDevice, st));
    const char* d_in = static_cast<const char*>(c.d_poses.p);
    // zero-copy: the model kernels store the records where the caller's copy is taken from (they are read again by
    // weight_kernel over PCIe only when they live in host memory, so that is limited to the case the caller wants them)
    mcl3dl_result* k_rec = (L.zc && records) ? reinterpret_cast<mcl3dl_result*>(hp + L.o_rec) : static_cast<mcl3dl_result*>(c.d_out.p);
    rc = launch_models(eng, c, reinterpret_cast<const mcl3dl_pose*>(d_in), Pd, reinterpret_cast<const mcl3dl_point*>(d_in + L.o_lik),
                       n_lik, reinterpret_cast<const mcl3dl_point*>(d_in + L.o_beam), n_beam,
                       reinterpret_cast<const float*>(d_in + L.o_org), n_origins, static_cast<mcl3dl_result*>(c.d_out.p),
                       nullptr, st, false);
    (void)k_rec;
    if (rc != MCL3DL_OK)
      return rc;
    WeightPartial* parts = static_cast<WeightPartial*>(c.d_wpart.p);
    WeightPartial* h_part = reinterpret_cast<WeightPartial*>(hp + L.o_part);
    weight_kernel<<<L.nblk, kBlockThreads, 0, st>>>(static_cast<const mcl3dl_result*>(c.d_out.p),
                                                   reinterpret_cast<const float*>(d_in + L.o_prior),
                                                   extra ? reinterpret_cast<const float*>(d_in + L.o_extra) : nullptr,
                                                   static_cast<int>(Pd), static_cast<int>(n_lik), static_cast<float*>(c.d_w.p), parts,
                                                   tk, L.zc ? h_part : nullptr);
    CK(cudaGetLastError());
    eng->launches += 1;
    if (!L.zc)
      CK(cudaMemcpyAsync(h_part, parts + L.nblk, sizeof(WeightPartial), cudaMemcpyDeviceToHost, st));
    if (one_sync)
    {
      // pass 2 right behind pass 1 (its partial slots live after pass 1's)
      WeightPartial* parts2 = parts + L.nblk + 1;
      float* k_post = L.zc ? reinterpret_cast<float*>(hp + L.o_post) : static_cast<float*>(c.d_post.p);
      normalize_kernel_dev<<<L.nblk, kBlockThreads, 0, st>>>(static_cast<const float*>(c.d_w.p), static_cast<int>(Pd), parts + L.nblk,
                                                            static_cast<int>(p0[d]), k_post, parts2, tk + 1,
                                                            L.zc ? h_part + 1 : nullptr);
      CK(cudaGetLastError());
      eng->launches += 1;
      if (!L.zc)
      {
        CK(cudaMemcpyAsync(hp + L.o_post, c.d_post.p, Pd * 4, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(h_part + 1, parts2 + L.nblk, sizeof(WeightPartial), cudaMemcpyDeviceToHost, st));
      }
      if (records)
        CK(cudaMemcpyAsync(hp + L.o_rec, c.d_out.p, Pd * sizeof(mcl3dl_result), cudaMemcpyDeviceToHost, st));
    }
  }
  double total = 0.0;
  float qmin = 1.0f, qmax = 0.0f;
  for (size_t d = 0; d < G; ++d)
  {
    DeviceCtx& c = eng->devs[d];
    if (p0[d + 1] == p0[d])
      continue;
    CK(cudaSetDevice(c.dev));
    CK(cudaStreamSynchronize(c.stream));
    WeightPartial wp;
    std::memcpy(&wp, static_cast<const char*>(c.h_pinned) + lay[d].o_part, sizeof(wp));
    total += wp.sum;  // device order: deterministic
    qmin = std::min(qmin, wp.qmin);
    qmax = std::max(qmax, wp.qmax);
  }
  const float total_f = static_cast<float>(total);
  summary->weight_sum = total_f;
  summary->match_ratio_min = qmin;
  summary->match_ratio_max = qmax;
  summary->kept = total_f > 0.0f ? 1 : 0;
  // ---- pass 2 (several devices): normalise with the global total, entropy, arg max; only 4 B per particle come back
  for (size_t d = 0; d < G && !one_sync; ++d)
  {
    DeviceCtx& c = eng->devs[d];
    const size_t Pd = p0[d + 1] - p0[d];
    if (Pd == 0)
      continue;
    CK(cudaSetDevice(c.dev));
    cudaStream_t st = c.stream;
    Lay& L = lay[d];
    char* hp = static_cast<char*>(c.h_pinned);
    WeightPartial* parts = static_cast<WeightPartial*>(c.d_wpart.p);
    unsigned int* tk;
    if ((rc = weight_tickets(eng, c, &tk)))
      return rc;
    if (summary->kept)
    {
      normalize_kernel<<<L.nblk, kBlockThreads, 0, st>>>(static_cast<const float*>(c.d_w.p), static_cast<int>(Pd), total_f,
                                                        static_cast<int>(p0[d]), static_cast<float*>(c.d_post.p), parts, tk, nullptr);
      CK(cudaGetLastError());
      eng->launches += 1;
      CK(cudaMemcpyAsync(hp + L.o_post, c.d_post.p, Pd * 4, cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(hp + L.o_part + sizeof(WeightPartial), parts + L.nblk, sizeof(WeightPartial), cudaMemcpyDeviceToHost, st));
    }
    if (records)
      CK(cudaMemcpyAsync(hp + L.o_rec, c.d_out.p, Pd * sizeof(mcl3dl_result), cudaMemcpyDeviceToHost, st));
  }
  double ent = 0.0;
  float best = -1.0f;
  uint32_t best_i = 0;
  for (size_t d = 0; d < G; ++d)
  {
    DeviceCtx& c = eng->devs[d];
    const size_t Pd = p0[d + 1] - p0[d];
    if (Pd == 0)
      continue;
    CK(cudaSetDevice(c.dev));
    if (!one_sync)
      CK(cudaStreamSynchronize(c.stream));
    const char* hp = static_cast<const char*>(c.h_pinned);
    if (summary->kept)
    {
      std::memcpy(posterior + p0[d], hp + lay[d].o_post, Pd * 4);
      WeightPartial wp;
      std::memcpy(&wp, hp + lay[d].o_part + sizeof(WeightPartial), sizeof(wp));
      ent += wp.sum;
      if (wp.best > best)  // lower device = lower indices, so strict '>' keeps the first maximum
      {
        best = wp.best;
        best_i = wp.best_i;
      }
    }
    else
    {
      std::memcpy(posterior + p0[d], prior + p0[d], Pd * 4);  // "No Particle alive, restoring." pf.h:274-278
    }
    if (records)
      std::memcpy(records + p0[d], hp + lay[d].o_rec, Pd * sizeof(mcl3dl_result));
  }
  summary->entropy = summary->kept ? static_cast<float>(-ent) : 0.0f;
  summary->max_index = best_i;
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
    CK(cudaMemset(c.d_stats.p, 0, 5 * sizeof(unsigned long long)));
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
