// kernels.cuh — the kernels of the measurement update, hand-written for sm_90a (H100).
//
//   likelihood model  LidarMeasurementModelLikelihood::measure (src/lidar_measurement_model_likelihood.cpp:105-139)
//                     + ChunkedKdtree::radiusSearch semantics (include/mcl_3dl/chunked_kdtree.h:217-237):
//       lik_kernel_nf_pm  NN field, point-major: a lane owns a particle, a warp 32 particles on one scan point
//       lik_kernel_nf     NN field, particle-major: TPP lanes (8 .. 256) own a particle and stride its scan points
//       lik_kernel_wi     no NN field staged: the CSR window search, particle-major (TPP >= 32)
//       lik_kernel_field  the opt-in, inexact field mode
//   beam model        LidarMeasurementModelBeam::measure / getBeamStatus (src/lidar_measurement_model_beam.cpp:124-192)
//                     + RaycastUsingDDA / RaycastUsingKDTree:
//       beam_kernel_pl    a lane owns a particle, a warp casts one chunk of rays; fixed CTA mapping
//       beam_kernel_dq    the same lanes, (particle group, ray chunk) items pulled from a global queue
//   weight_kernel / normalize_kernel*: the fused weight update; exchange_signal_kernel: the multi-GPU record exchange.
//
// The per-thread arithmetic (transform, searches, ray casts, likelihood term, beam score) lives in device_funcs.cuh,
// which tests/hostsim also compiles for the host.  Every reduction has a fixed order or sums integers, so results are
// deterministic run to run.  No tensor cores: there is no dense contraction anywhere on this path (HBM/L2 gather bound).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/mcl3dl_b200.h"
#include "device_funcs.cuh"
#include "device_math.cuh"

namespace mcl3dl
{
constexpr int kBlockThreads = 256;

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fadd(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ uint32_t warp_sum_u32(uint32_t v)
{
  return __reduce_add_sync(0xffffffffu, v);
}

// --------------------------------------------------------------------------------------------
// Where a kernel's writer lane stores its particle's record fields.  world == 0: the plain output array `out`.
// world >= 1 (one process per GPU, SURVEY 8e): the record exchange is folded into the kernels' epilogues — the writer
// stores the fields straight into slot `rank` of EVERY rank's gathered array over NVLink (peer memory mapped with CUDA
// IPC), so no collective and no copy kernel follows; exchange_signal_kernel then publishes "rank r finished step s".
// The gathered array is double-buffered by step parity (a peer may already be one step ahead); the parity of the
// upcoming step is read from the device-side step counter, so the launch sequence is identical every step (CUDA graph).
constexpr int kMaxPeers = 8;
struct RecordSink
{
  mcl3dl_result* base[kMaxPeers];  // every rank's array 0, already offset to this rank's slot (own buffer at [rank])
  const uint32_t* step;            // completed-step counter of this rank (device memory)
  uint32_t parity_stride;          // records between array 0 and array 1 (= world * n_local)
  int world;
};

// offset of particle p's record inside a rank's array 0 (world >= 1) — the parity of the step about to complete
__device__ __forceinline__ uint32_t sink_offset(const RecordSink& s, int p)
{
  return ((__ldcg(s.step) + 1u) & 1u) * s.parity_stride + static_cast<uint32_t>(p);
}

// likelihood-model fields (+ the beam model's (1, 0) when that model has no scan this update)
__device__ __forceinline__ void sink_store_lik(const RecordSink& s, mcl3dl_result* out, int p, float score_like,
                                               uint32_t match_cnt, int write_beam_defaults)
{
  const uint32_t off = s.world ? sink_offset(s, p) : 0u;
#pragma unroll
  for (int g = 0; g < kMaxPeers; ++g)
    if (g < max(s.world, 1))
    {
      mcl3dl_result* o = s.world ? s.base[g] + off : out + p;  // s.base[g]: a constant-bank read (unrolled)
      o->score_like = score_like;
      o->match_cnt = match_cnt;
      if (write_beam_defaults)
      {
        // no beam scan this update: LidarMeasurementResult(1, 0), beam.cpp:130-133
        o->score_beam = 1.0f;
        o->n_short = 0;
        o->n_hit = 0;
        o->n_long = 0;
      }
    }
}

__device__ __forceinline__ void sink_store_beam(const RecordSink& s, mcl3dl_result* out, int p, float score_beam, uint32_t n_short,
                                                uint32_t n_hit, uint32_t n_long, int write_lik_defaults)
{
  const uint32_t off = s.world ? sink_offset(s, p) : 0u;
#pragma unroll
  for (int g = 0; g < kMaxPeers; ++g)
    if (g < max(s.world, 1))
    {
      mcl3dl_result* o = s.world ? s.base[g] + off : out + p;
      o->score_beam = score_beam;
      o->n_short = n_short;
      o->n_hit = n_hit;
      o->n_long = n_long;
      if (write_lik_defaults)
      {
        // no likelihood scan this update: LidarMeasurementResult(1, 0), likelihood.cpp:111-114
        o->score_like = 1.0f;
        o->match_cnt = 0;
      }
    }
}

// --------------------------------------------------------------------------------------------
// Stage `bytes` (multiple of 16) from global to shared with one TMA bulk copy (cp.async.bulk + mbarrier): thread 0
// issues it, every thread waits for it.  stage_issue early and stage_wait late overlap the copy with other work.
__device__ __forceinline__ void stage_issue(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar)
{
  const uint32_t bar_a = static_cast<uint32_t>(__cvta_generic_to_shared(bar));
  const uint32_t dst_a = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  if (threadIdx.x == 0)
  {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_a),
        "l"(gsrc), "r"(bytes), "r"(bar_a)
        : "memory");
  }
}
__device__ __forceinline__ void stage_wait(uint64_t* bar)
{
  const uint32_t bar_a = static_cast<uint32_t>(__cvta_generic_to_shared(bar));
  __syncthreads();  // the barrier's initialisation (thread 0) is visible to every waiter
  uint32_t done = 0;
  while (!done)
  {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(bar_a)
        : "memory");
  }
}

__device__ __forceinline__ void stage_tile(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar)
{
  stage_issue(smem_dst, gsrc, bytes, bar);
  stage_wait(bar);
}

// Fold one value per lane over the TPP lanes that own a particle, in a fixed order.  TPP < 32: the particle's lanes
// are an aligned sub-group of the warp (xor-shuffle tree).  TPP >= 32: the warp's xor-shuffle tree, then the particle's
// warps in order through shared memory (red_f / red_u: one entry per warp).
template <int TPP>
__device__ __forceinline__ void particle_reduce(float& f, uint32_t& a, float* red_f, uint32_t* red_u)
{
  if (TPP >= 32)
  {
    f = warp_sum(f);
    a = warp_sum_u32(a);
    if (TPP > 32)
    {
      constexpr int WPP = TPP / 32;
      const int warp = threadIdx.x >> 5;
      __syncthreads();
      if ((threadIdx.x & 31) == 0)
      {
        red_f[warp] = f;
        red_u[warp] = a;
      }
      __syncthreads();
      const int w0 = (warp / WPP) * WPP;
      float sf = red_f[w0];
      uint32_t sa = red_u[w0];
#pragma unroll
      for (int k = 1; k < WPP; ++k)
      {
        sf = fadd(sf, red_f[w0 + k]);
        sa += red_u[w0 + k];
      }
      f = sf;
      a = sa;
    }
  }
  else
  {
#pragma unroll
    for (int o = TPP / 2; o > 0; o >>= 1)
    {
      f = fadd(f, __shfl_xor_sync(0xffffffffu, f, o));
      a += __shfl_xor_sync(0xffffffffu, a, o);
    }
  }
}

// add one per-thread work counter to stats[i] (SURVEY 5: the node's status path wants evals/steps): a warp sum and
// one atomic per warp
__device__ __forceinline__ void stats_add(unsigned long long* stats, int i, uint32_t v)
{
  v = warp_sum_u32(v);
  if ((threadIdx.x & 31) == 0)
    atomicAdd(stats + i, static_cast<unsigned long long>(v));
}

// --------------------------------------------------------------------------------------------
// Warp-item likelihood kernel (no NN field staged: MCL3DL_NNF=0, or a field above MCL3DL_NNF_MAX_MB).
//
// A kernel whose lanes each walk their own eval's window runs with few of its 32 lanes active: an eval next to a
// surface scans ~30 map points, one that misses scans ~2, and every lane waits for the slowest one, one dependent load
// at a time.  Here each warp works on 32 evals at a time in two warp-synchronous phases, no CTA barrier:
//   phase 1 (lane = eval, uniform): transform, window, ALL row bounds of the <=3x3 window issued back
//            to back (18 independent loads in flight per lane); the non-empty [s0,s1) runs go to
//            this warp's shared-memory slab;
//   phase 2 (lane = item): the warp's non-empty runs are enumerated with one prefix sum and dealt to
//            the lanes round-robin, so a lane that owns a surface-hugging eval gets help from the
//            lanes whose evals had nothing to scan; each item is one contiguous run of map points,
//            read 4 at a time; minima are merged with shared-memory atomicMin on the float bits
//            (order independent -> deterministic).
// The eval's owner lane then adds its contribution to its running sum in scan order.  Requires cell edge > window
// half-width (<= 3 cells/axis).
constexpr int kMaxWinRows = 9;
// map points fetched per batch of an item (4 was the fastest of 1/2/4/8 on c2);
// (before the window table) capping registers below 64 for more resident CTAs only spilled and lost
constexpr int kWiUnroll = 4;

struct LikWarpSmem
{
  uint2 rows[kMaxWinRows][32];  // non-empty runs of each lane's eval, compacted
  float qx[32], qy[32], qz[32];
  uint32_t best[32];                  // float bits of the running min d^2 (non-negative floats order as uints)
  uint16_t items[kMaxWinRows * 32];   // lane | run << 5
};

// __launch_bounds__(256, 4): with the window table the kernel wants 72 registers (3 CTAs/SM); capping at 64
// costs 24 bytes of spill and wins.
template <int TPP, bool STAGED>
__global__ void __launch_bounds__(kBlockThreads, 4)
    lik_kernel_wi(const mcl3dl_pose* __restrict__ poses, int P, const float4* __restrict__ scan, int N, NnGridDev g,
                  LikDev lp, mcl3dl_result* __restrict__ out, int write_beam_defaults,
                  unsigned long long* __restrict__ stats, RecordSink sink)
{
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ uint64_t bar;
  __shared__ float red_f[kBlockThreads / 32];
  __shared__ uint32_t red_u[3 * kBlockThreads / 32];
  __shared__ LikWarpSmem wsm_all[kBlockThreads / 32];
  const float4* pts = scan;
  if (STAGED && N > 0)
  {
    stage_tile(smem_raw, scan, static_cast<uint32_t>(N) * 16u, &bar);
    pts = reinterpret_cast<const float4*>(smem_raw);
  }
  constexpr int PPB = kBlockThreads / TPP;
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  LikWarpSmem& sm = wsm_all[tid >> 5];
  const int sub = tid / TPP;
  const int l = tid % TPP;
  const int n_groups = (P + PPB - 1) / PPB;
  const uint32_t r2_bits = __float_as_uint(lp.r2);
  uint32_t st_rows = 0, st_pts = 0;
  for (int grp = blockIdx.x; grp < n_groups; grp += gridDim.x)
  {
    const int p = grp * PPB + sub;
    const bool live = p < P;
    float score = 0.0f;
    uint32_t cnt = 0;
    F3 pos;
    Q4 rn;
    pos.x = pos.y = pos.z = 0.0f;
    rn.x = rn.y = rn.z = 0.0f;
    rn.w = 1.0f;
    if (live)
    {
      Q4 q;
      load_pose(poses + p, pos, q);
      rn = qnormalized(q);  // state_6dof.h:217
    }
    // a warp's 32 lanes always belong to one particle (TPP >= 32), so the trip count is warp-uniform
    for (int jbase = 0; jbase < N; jbase += TPP)
    {
      const int j = jbase + l;
      const bool valid = live && j < N;
      // ---------------- phase 1: lane = eval
      int nr = 0;
      sm.best[lane] = r2_bits;
      if (valid)
      {
        const float4 sp = pts[j];
        F3 v;
        v.x = sp.x;
        v.y = sp.y;
        v.z = sp.z;
        const F3 t = transform_point(rn, pos, v);
        // PointRepresentation::vectorize with rescale values (mcl_3dl.cpp:1270)
        const float qx = fmul(t.x, g.wx), qy = fmul(t.y, g.wy), qz = fmul(t.z, g.wz);
        sm.qx[lane] = qx;
        sm.qy[lane] = qy;
        sm.qz[lane] = qz;
        // same cell function as the build kernel (monotone), applied to q -/+ rpad
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
        hy = min(hy, min(g.ny - 1, ly + 2));
        hz = min(hz, min(g.nz - 1, lz + 2));
#if MCL3DL_NEAR_BITS
        // near-field screen: a far miss (most evals of a tracking update) costs one bit instead of the window fetch
        if (lx <= hx && ly <= hy && lz <= hz && near_maybe(g.near, qx, qy, qz))
#else
        if (lx <= hx && ly <= hy && lz <= hz)
#endif
        {
          st_rows += static_cast<uint32_t>((hz - lz + 1) * (hy - ly + 1));
          // the whole 3x3 window from the y-fastest window table: 2 aligned 16-byte loads per z layer
          const int width = hx - lx + 1;  // 1..3 cells along x
          const int yb = ly & ~1;
          const int odd = ly & 1;
          uint4 ea[3], eb[3];
#pragma unroll
          for (int dz = 0; dz < 3; ++dz)
          {
            const int iz = min(lz + dz, hz);
            const uint4* src = reinterpret_cast<const uint4*>(g.row3 + (static_cast<size_t>(iz) * g.nx + lx) * g.nyp + yb);
            ea[dz] = __ldg(src);
            eb[dz] = __ldg(src + 1);
          }
#pragma unroll
          for (int dz = 0; dz < 3; ++dz)
#pragma unroll
            for (int dy = 0; dy < 3; ++dy)
            {
              const int iy = ly + dy, iz = lz + dz;
              if (iy <= hy && iz <= hz)
              {
                // entry (iy - yb) of the four fetched ones
                uint32_t start, packed;
                if (dy == 0)
                {
                  start = odd ? ea[dz].z : ea[dz].x;
                  packed = odd ? ea[dz].w : ea[dz].y;
                }
                else if (dy == 1)
                {
                  start = odd ? eb[dz].x : ea[dz].z;
                  packed = odd ? eb[dz].y : ea[dz].w;
                }
                else
                {
                  start = odd ? eb[dz].z : eb[dz].x;
                  packed = odd ? eb[dz].w : eb[dz].y;
                }
                uint32_t cnt = width == 3 ? (packed >> 21) : (width == 2 ? ((packed >> 10) & 0x7ffu) : (packed & 0x3ffu));
                const uint32_t sat = width == 3 ? 0x7ffu : (width == 2 ? 0x7ffu : 0x3ffu);
                if (cnt == sat)
                {
                  // count did not fit the packed field (very dense cells): read the CSR bounds themselves
                  const int row = (iz * g.ny + iy) * g.nx;
                  start = __ldg(g.cell_start + row + lx);
                  cnt = __ldg(g.cell_start + row + hx + 1) - start;
                }
                if (cnt)
                {
                  sm.rows[nr][lane] = make_uint2(start, start + cnt);
                  ++nr;
                  st_pts += cnt;
                }
              }
            }
        }
      }
      // ---------------- deal the warp's runs to its lanes
      uint32_t incl = static_cast<uint32_t>(nr);
#pragma unroll
      for (int o = 1; o < 32; o <<= 1)
      {
        const uint32_t nbr = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o)
          incl += nbr;
      }
      const int n_items = static_cast<int>(__shfl_sync(0xffffffffu, incl, 31));
      const int first = static_cast<int>(incl) - nr;
      for (int k = 0; k < nr; ++k) sm.items[first + k] = static_cast<uint16_t>(lane | (k << 5));
      __syncwarp();
      // ---------------- phase 2: lane = item (one contiguous run of map points); a 4-lanes-per-item variant that
      // coalesces the point loads was measured and lost
      for (int it = lane; it < n_items; it += 32)
      {
        const uint32_t iv = sm.items[it];
        const int e = iv & 31;
        const uint2 run = sm.rows[iv >> 5][e];
        const float qx = sm.qx[e], qy = sm.qy[e], qz = sm.qz[e];
        float best = lp.r2;
        for (uint32_t s = run.x; s < run.y; s += kWiUnroll)
        {
          float4 mp[kWiUnroll];
#pragma unroll
          for (int u = 0; u < kWiUnroll; ++u)
            if (s + u < run.y)
              mp[u] = __ldg(g.pts + s + u);
#pragma unroll
          for (int u = 0; u < kWiUnroll; ++u)
            if (s + u < run.y)
            {
              // flann::L2_Simple: sequential float accumulate of squared differences
              const float dx = fsub(qx, mp[u].x);
              const float dy = fsub(qy, mp[u].y);
              const float dz = fsub(qz, mp[u].z);
              best = fminf(best, fadd(fadd(fmul(dx, dx), fmul(dy, dy)), fmul(dz, dz)));  // keep d < worst
            }
        }
        if (best < lp.r2)
          atomicMin(&sm.best[e], __float_as_uint(best));
      }
      __syncwarp();
      // ---------------- owner lane
      if (valid)
      {
        const float d2 = __uint_as_float(sm.best[lane]);
        float t;
        if (d2 < lp.r2 && lik_term(__fsqrt_rn(d2), lp, t))
        {
          score = fadd(score, t);
          cnt++;
        }
      }
      __syncwarp();
    }
    particle_reduce<TPP>(score, cnt, red_f, red_u);
    if (live && l == 0)  // empty scan -> LidarMeasurementResult(1, 0), likelihood.cpp:111-114
      sink_store_lik(sink, out, p, (N == 0) ? 1.0f : score, cnt, write_beam_defaults);
  }
  if (stats)
  {
    stats_add(stats, 0, st_rows);
    stats_add(stats, 1, st_pts);
  }
}


// --------------------------------------------------------------------------------------------
// NN-field likelihood kernel (the default when set_map staged the field, device_funcs.cuh: NnFieldDev).
//
// Profiled, lik_kernel_wi issues tens of warp instructions per eval at about half its lanes live, with L1/TEX the
// busiest unit and DRAM nearly idle: bound by the instructions and gather wavefronts of walking a 3 x 3 window of CSR
// rows per eval.  With the field an eval is: transform, one 8-byte directory entry, then
// the 0-14 (wide cells: up to 40) contiguous candidates of its voxel — two dependent loads and ~1/4 of the
// instructions.  What is left is latency, so the kernel is built around loads in flight:
//   * phase A: lane = eval, kNfU = 4 evals per lane (their directory loads overlap); the queries go to shared memory;
//   * phase B: the candidate lists of the warp's 32 * kNfU evals are flattened into one list of W (eval, candidate)
//     slots (a shuffle prefix sum of the lanes' candidate counts).  Lane k takes slots k, k + 32, ..., kNfB of them per
//     round with their loads in flight, and folds each distance into its eval's best with a shared atomicMin.  A warp
//     waits ~ceil(W / 32) / kNfB load latencies with every lane busy, instead of the longest of its 128 lists one
//     load after another with half the lanes idle; adjacent lanes read adjacent records of a list;
//   * TPP in {8 .. 256} lanes per particle, chosen on the host so that a particle's scan gives every lane ~4 evals and
//     the whole grid is resident in ONE wave where the job is small (c2: 128 lanes x 2 particles x 512 CTAs);
//   * the TMA copy of the scan tile is issued first and waited for only after the pose is loaded and normalised
//     (fp64 division); CTAs whose tile would be used by < 4 particles read the scan straight from L2 instead;
//   * the overflow fallback (raw clouds) is a template flag, so maps without overflow cells carry none of its code.
// Distances are sums of squares (non-negative, finite) and the best starts at r2 > 0, so the unsigned min over their
// bit patterns is fminf over the same set in any order: the best of an eval does not depend on which lane folded what.
// Per-lane accumulation runs in scan order (j = l, l + TPP, ...), lanes are folded by the xor-shuffle tree and warps in
// order: deterministic, and bit-identical to lik_kernel_wi whenever it runs with the same TPP.
#ifndef MCL3DL_NF_U
#define MCL3DL_NF_U 4
#endif
constexpr int kNfU = MCL3DL_NF_U;
constexpr int kNfEvals = 32 * kNfU;  // evals of one warp per trip; eval e = u * 32 + lane
static_assert(kNfEvals <= 256, "phase B names an eval by one byte");
// phase B: candidate loads in flight per lane, and (eval, candidate) slots per pass (longer flattened lists take passes)
#ifndef MCL3DL_NF_B
#define MCL3DL_NF_B 4
#endif
constexpr int kNfB = MCL3DL_NF_B;
constexpr int kNfSlots = 1024;
// resident CTAs per SM the compiler must allow (register cap): 3 -> 80 registers, 4 -> 64, 5 -> 48, 6 -> 40
#ifndef MCL3DL_NF_MINB
#define MCL3DL_NF_MINB 4
#endif

// per-warp shared memory of the NN-field kernels' candidate scan
struct NfWarpSmem
{
  float4 q[kNfEvals];       // query of eval e; .w = bits of (first candidate - first slot) of its list
  uint32_t best[kNfEvals];  // bits of the eval's best d^2 so far
  uint8_t own[kNfSlots];    // slot -> eval, for the pass's slots
};

// The candidate scan of one warp trip of the NN-field kernels (lik_kernel_nf, lik_kernel_nf_pm).  Phase A has left the
// query of this lane's eval u (eval e = u * 32 + lane) in ws.q[e].xyz, and its candidate count c[u] (-1: overflow cell)
// and first candidate s[u] from nnf_lookup; an eval without a query has c[u] = 0.  tot: the lane's candidates in all
// (the sum of max(c[u], 0), counted in phase A: summed here, it costs a spill).  Returns each eval's best d^2 in d2[u]
// (r2 when no map point is closer).  Every lane of the warp calls it: it shuffles and synchronises the whole warp.
template <bool OVF>
__device__ __forceinline__ void nf_warp_scan(NfWarpSmem& ws, const NnGridDev& g, const LikDev& lp, const int (&c)[kNfU],
                                             const uint32_t (&s)[kNfU], int tot, float (&d2)[kNfU], uint32_t& st_rows,
                                             uint32_t& st_pts)
{
  const int lane = threadIdx.x & 31;
  const NnFieldDev& f = g.field;
  // ---- flatten: the lanes' lists end to end (inclusive shuffle scan of the lane totals), W slots in all
  int incl = tot;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1)
  {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o)
      incl += v;
  }
  const int W = __shfl_sync(0xffffffffu, incl, 31);
  int b[kNfU];
  int base = incl - tot;
#pragma unroll
  for (int u = 0; u < kNfU; ++u)
  {
    b[u] = base;
    base += max(c[u], 0);
    ws.q[u * 32 + lane].w = __uint_as_float(s[u] - static_cast<uint32_t>(b[u]));  // slot + .w = candidate index
    ws.best[u * 32 + lane] = __float_as_uint(lp.r2);
  }
  // ---- phase B: kNfB candidates per lane in flight, folded into their evals' bests
  for (int lo = 0; lo < W; lo += kNfSlots)
  {
    const int hi = min(W, lo + kNfSlots);
#pragma unroll
    for (int u = 0; u < kNfU; ++u) nnf_fill_owner(ws.own, lo, hi, b[u], max(c[u], 0), u * 32 + lane);
    __syncwarp();
    for (int k = lo + lane; k < hi; k += 32 * kNfB)
    {
      int e[kNfB];
      float4 m[kNfB];
#pragma unroll
      for (int v = 0; v < kNfB; ++v)
        if (k + 32 * v < hi)
        {
          e[v] = ws.own[k + 32 * v - lo];
          m[v] = __ldg(f.cand + (__float_as_uint(ws.q[e[v]].w) + static_cast<uint32_t>(k + 32 * v)));
        }
#pragma unroll
      for (int v = 0; v < kNfB; ++v)
        if (k + 32 * v < hi)
        {
          const float4 qe = ws.q[e[v]];
          atomicMin(&ws.best[e[v]], __float_as_uint(nnf_cand_d2(qe.x, qe.y, qe.z, m[v])));
        }
    }
    __syncwarp();  // the bests are final, and the next pass may overwrite `own`
  }
  // ---- back to the owners
#pragma unroll
  for (int u = 0; u < kNfU; ++u)
  {
    d2[u] = __uint_as_float(ws.best[u * 32 + lane]);
    if (OVF && c[u] < 0)  // overflow cell (raw clouds): the CSR window search
    {
      const float4 qu = ws.q[u * 32 + lane];
      d2[u] = nn_dist2(g, lp, qu.x, qu.y, qu.z, st_rows, st_pts);
    }
    else
      st_pts += static_cast<uint32_t>(max(c[u], 0));
  }
}

template <int TPP, bool STAGED, bool OVF>
__global__ void __launch_bounds__(kBlockThreads, MCL3DL_NF_MINB)
    lik_kernel_nf(const mcl3dl_pose* __restrict__ poses, int P, const float4* __restrict__ scan, int N, NnGridDev g,
                  LikDev lp, mcl3dl_result* __restrict__ out, int write_beam_defaults,
                  unsigned long long* __restrict__ stats, RecordSink sink)
{
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ uint64_t bar;
  __shared__ float red_f[kBlockThreads / 32];
  __shared__ uint32_t red_u[kBlockThreads / 32];
  __shared__ NfWarpSmem nfw[kBlockThreads / 32];
  if (STAGED && N > 0)
    stage_issue(smem_raw, scan, static_cast<uint32_t>(N) * 16u, &bar);
  constexpr int PPB = kBlockThreads / TPP;
  const int sub = threadIdx.x / TPP;
  const int l = threadIdx.x % TPP;
  const int lane = threadIdx.x & 31;
  NfWarpSmem& ws = nfw[threadIdx.x >> 5];
  const int n_groups = (P + PPB - 1) / PPB;
  const NnFieldDev& f = g.field;
  uint32_t st_rows = 0, st_pts = 0;
  bool staged_ready = !(STAGED && N > 0);
  for (int grp = blockIdx.x; grp < n_groups; grp += gridDim.x)
  {
    const int p = grp * PPB + sub;
    const bool live = p < P;
    float score = 0.0f;
    uint32_t cnt = 0;
    F3 pos;
    Q4 rn;
    pos.x = pos.y = pos.z = 0.0f;
    rn.x = rn.y = rn.z = 0.0f;
    rn.w = 1.0f;
    if (live)
    {
      Q4 q;
      load_pose(poses + p, pos, q);
      rn = qnormalized(q);  // state_6dof.h:217
    }
    if (!staged_ready)
    {
      stage_wait(&bar);  // the tile has been in flight since the kernel started
      staged_ready = true;
    }
    const float4* pts = STAGED ? reinterpret_cast<const float4*>(smem_raw) : scan;
    // every lane of the warp runs every trip (dead particles and evals beyond N with no candidates): phase B shuffles
    // and synchronises the whole warp
    for (int j0 = 0; j0 < N; j0 += kNfU * TPP)
    {
      const int j = j0 + l;
      // ---- phase A: the queries and directory entries of up to kNfU evals (independent loads in flight)
      int c[kNfU];
      uint32_t s[kNfU];
      int tot = 0;
#pragma unroll
      for (int u = 0; u < kNfU; ++u)
      {
        c[u] = 0;
        s[u] = 0;
        float4 q = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (live && j + u * TPP < N)
        {
          const float4 sp = STAGED ? pts[j + u * TPP] : __ldg(pts + j + u * TPP);
          F3 v;
          v.x = sp.x;
          v.y = sp.y;
          v.z = sp.z;
          const F3 t = transform_point(rn, pos, v);
          // PointRepresentation::vectorize with rescale values (mcl_3dl.cpp:1270)
          q.x = fmul(t.x, g.wx);
          q.y = fmul(t.y, g.wy);
          q.z = fmul(t.z, g.wz);
          c[u] = nnf_lookup(f, q.x, q.y, q.z, s[u]);
          tot += max(c[u], 0);
        }
        ws.q[u * 32 + lane] = q;  // .w: nf_warp_scan's, once the eval's first slot is known
      }
      float d2[kNfU];
      nf_warp_scan<OVF>(ws, g, lp, c, s, tot, d2, st_rows, st_pts);
      // ---- the owners score their evals in scan order
#pragma unroll
      for (int u = 0; u < kNfU; ++u)
      {
        float t;
        if (d2[u] < lp.r2 && lik_term(__fsqrt_rn(d2[u]), lp, t))  // (evals beyond N keep d2 = r2)
        {
          score = fadd(score, t);
          cnt++;
        }
      }
    }
    if (live && l < N)
      st_rows += static_cast<uint32_t>((N - l + TPP - 1) / TPP);  // one directory entry per eval of this lane
    particle_reduce<TPP>(score, cnt, red_f, red_u);
    if (live && l == 0)  // empty scan -> LidarMeasurementResult(1, 0), likelihood.cpp:111-114
      sink_store_lik(sink, out, p, (N == 0) ? 1.0f : score, cnt, write_beam_defaults);
  }
  if (!staged_ready)
    stage_wait(&bar);  // never leave with the bulk copy in flight
  if (stats)
  {
    stats_add(stats, 0, st_rows);
    stats_add(stats, 1, st_pts);
  }
}

// --------------------------------------------------------------------------------------------
// Point-major mapping of the NN-field likelihood kernel (many particles per scan point).
//
// A lane owns one particle; the warp's 32 lanes are 32 consecutive particles on the SAME scan point, and the CTA's 8
// warps are 256 consecutive particles on the same slice of `slice` scan points.  In tracking mode the particles of a
// cloud see one scan point in nearly the same place, so their directory and candidate sectors coalesce within the
// load instruction and the CTA's other warps find them in L1, where lik_kernel_nf (a warp = one particle's points)
// sends every eval's sectors to L2 on its own.  The transform, the directory lookup (phase A) and the candidate scan
// (nf_warp_scan) are lik_kernel_nf's; only eval e = u * 32 + lane now means (particle lane, point j0 + u).
//
// A particle's points are spread over the grid's slices, so its score is folded across CTAs.  Each lane sums its
// slice's contributions in 2^-fx_shift fixed point and adds one word (device_funcs.cuh: nf_pm_word: the sum, the match
// count and an arrival) to the particle's 64-bit accumulator with one atomic.  Integer additions give the same total
// in any order, so the records are deterministic; the returned value tells the lane that brings the arrivals to
// n_slices, which stores the record and leaves the accumulator at zero.  No fence, ticket or read-back: the fold is one
// round trip to L2 after the candidate scan.  The score is the exact sum of the float contributions rounded once to
// float (to the fixed-point step, below 2^-30 / N of the largest possible score: nf_pm_shape).  A fold of the float contributions in scan
// order would be a chain of N dependent adds over N loads at the end of the kernel, after every other warp has finished.
template <bool OVF>
__global__ void __launch_bounds__(kBlockThreads, MCL3DL_NF_MINB)
    lik_kernel_nf_pm(const mcl3dl_pose* __restrict__ poses, int P, const float4* __restrict__ scan, int N, NnGridDev g,
                     LikDev lp, mcl3dl_result* __restrict__ out, int write_beam_defaults,
                     unsigned long long* __restrict__ stats, RecordSink sink, NfPmShape sh,
                     unsigned long long* __restrict__ acc)
{
  __shared__ NfWarpSmem nfw[kBlockThreads / 32];
  const int lane = threadIdx.x & 31;
  const int group = (blockIdx.x / sh.n_slices) * (kBlockThreads / 32) + (threadIdx.x >> 5);
  if (group * 32 >= P)
    return;  // warp-uniform: no CTA barrier below
  NfWarpSmem& ws = nfw[threadIdx.x >> 5];
  const int s0 = (blockIdx.x % sh.n_slices) * sh.slice, s1 = min(N, s0 + sh.slice);
  const int p = group * 32 + lane;
  const bool live = p < P;
  const NnFieldDev& f = g.field;
  uint32_t st_rows = 0, st_pts = 0;
  long long sum = 0;
  uint32_t cnt = 0;
  F3 pos;
  Q4 rn;
  pos.x = pos.y = pos.z = 0.0f;
  rn.x = rn.y = rn.z = 0.0f;
  rn.w = 1.0f;
  if (live)
  {
    Q4 q;
    load_pose(poses + p, pos, q);
    rn = qnormalized(q);  // state_6dof.h:217
  }
  // every lane of the warp runs every trip (dead particles: no candidates), as in lik_kernel_nf
  for (int j0 = s0; j0 < s1; j0 += kNfU)
  {
    // ---- phase A: one scan point per u, the same for every lane (one broadcast load)
    int c[kNfU];
    uint32_t s[kNfU];
    int tot = 0;
#pragma unroll
    for (int u = 0; u < kNfU; ++u)
    {
      c[u] = 0;
      s[u] = 0;
      float4 q = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      if (j0 + u < s1)
      {
        const float4 sp = __ldg(scan + j0 + u);
        if (live)
        {
          F3 v;
          v.x = sp.x;
          v.y = sp.y;
          v.z = sp.z;
          const F3 t = transform_point(rn, pos, v);
          // PointRepresentation::vectorize with rescale values (mcl_3dl.cpp:1270)
          q.x = fmul(t.x, g.wx);
          q.y = fmul(t.y, g.wy);
          q.z = fmul(t.z, g.wz);
          c[u] = nnf_lookup(f, q.x, q.y, q.z, s[u]);
          tot += max(c[u], 0);
          st_rows++;
        }
      }
      ws.q[u * 32 + lane] = q;
    }
    float d2[kNfU];
    nf_warp_scan<OVF>(ws, g, lp, c, s, tot, d2, st_rows, st_pts);
    // ---- the owners: this lane's particle at points j0 .. j0 + kNfU - 1
#pragma unroll
    for (int u = 0; u < kNfU; ++u)
    {
      float t;
      if (d2[u] < lp.r2 && lik_term(__fsqrt_rn(d2[u]), lp, t))  // (dead lanes and points beyond the slice keep d2 = r2)
      {
        sum += nf_fx_term(t, sh.fx_shift);
        cnt++;
      }
    }
    __syncwarp();  // the next trip overwrites q / best
  }
  // ---- fold across the slices: one atomic per particle and slice, whose result tells the last slice
  if (live)
  {
    const unsigned long long w = nf_pm_word(sum, cnt, sh);
    uint32_t n;
    float score;
    if (nf_pm_done(atomicAdd(acc + p, w) + w, sh, n, score))
    {
      acc[p] = 0ull;  // every slice has added: nothing else touches it in this launch
      // empty scan -> LidarMeasurementResult(1, 0), likelihood.cpp:111-114
      sink_store_lik(sink, out, p, (N == 0) ? 1.0f : score, n, write_beam_defaults);
    }
  }
  if (stats)
  {
    stats_add(stats, 0, st_rows);
    stats_add(stats, 1, st_pts);
  }
}

// --------------------------------------------------------------------------------------------
// Field-mode likelihood kernel (opt-in, mcl3dl_field_mode; device_funcs.cuh: FieldDev): same mapping and reductions as
// lik_kernel_nf, but an eval is the transform plus ONE 32-byte gather (the 8 corner distances of its lattice cell) and a
// trilinear blend — BASELINE.json north_star's literal kernel.  Its scores deviate from the reference's exact
// nearest-neighbour distances (reported by bench.py / tests, not gated); 32 algorithmic bytes per eval.
template <int TPP, bool STAGED>
__global__ void __launch_bounds__(kBlockThreads, MCL3DL_NF_MINB)
    lik_kernel_field(const mcl3dl_pose* __restrict__ poses, int P, const float4* __restrict__ scan, int N, NnGridDev g,
                     LikDev lp, mcl3dl_result* __restrict__ out, int write_beam_defaults,
                     unsigned long long* __restrict__ stats, RecordSink sink)
{
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ uint64_t bar;
  __shared__ float red_f[kBlockThreads / 32];
  __shared__ uint32_t red_u[3 * kBlockThreads / 32];
  if (STAGED && N > 0)
    stage_issue(smem_raw, scan, static_cast<uint32_t>(N) * 16u, &bar);
  constexpr int PPB = kBlockThreads / TPP;
  const int sub = threadIdx.x / TPP;
  const int l = threadIdx.x % TPP;
  const int n_groups = (P + PPB - 1) / PPB;
  uint32_t st_rows = 0;
  bool staged_ready = !(STAGED && N > 0);
  for (int grp = blockIdx.x; grp < n_groups; grp += gridDim.x)
  {
    const int p = grp * PPB + sub;
    const bool live = p < P;
    float score = 0.0f;
    uint32_t cnt = 0;
    F3 pos;
    Q4 rn;
    pos.x = pos.y = pos.z = 0.0f;
    rn.x = rn.y = rn.z = 0.0f;
    rn.w = 1.0f;
    if (live)
    {
      Q4 q;
      load_pose(poses + p, pos, q);
      rn = qnormalized(q);  // state_6dof.h:217
    }
    if (!staged_ready)
    {
      stage_wait(&bar);
      staged_ready = true;
    }
    const float4* pts = STAGED ? reinterpret_cast<const float4*>(smem_raw) : scan;
    if (live)
    {
      for (int j = l; j < N; j += kNfU * TPP)
      {
        float d[kNfU];
#pragma unroll
        for (int u = 0; u < kNfU; ++u)
        {
          d[u] = lp.match_dist_min;  // "no neighbour"
          if (j + u * TPP < N)
          {
            const float4 sp = STAGED ? pts[j + u * TPP] : __ldg(pts + j + u * TPP);
            F3 v;
            v.x = sp.x;
            v.y = sp.y;
            v.z = sp.z;
            const F3 t = transform_point(rn, pos, v);
            d[u] = field_dist(g.fld, fmul(t.x, g.wx), fmul(t.y, g.wy), fmul(t.z, g.wz));
            ++st_rows;
          }
        }
#pragma unroll
        for (int u = 0; u < kNfU; ++u)
        {
          float t;
          if (d[u] < lp.match_dist_min && lik_term(d[u], lp, t))  // the interpolated distance in place of sqrt(sqdist[0])
          {
            score = fadd(score, t);
            cnt++;
          }
        }
      }
    }
    particle_reduce<TPP>(score, cnt, red_f, red_u);
    if (live && l == 0)
      sink_store_lik(sink, out, p, (N == 0) ? 1.0f : score, cnt, write_beam_defaults);
  }
  if (!staged_ready)
    stage_wait(&bar);
  if (stats)
    stats_add(stats, 0, st_rows * 4u);  // counted as 8-byte index entries: 32 B per eval
}

// ============================================================================================
// Lane-per-particle mapping for the beam model ("pl" kernel).
//
// A warp takes 32 consecutive particles (one per lane) and a chunk of consecutive rays; every lane
// casts the SAME scan ray at the same time.  In tracking mode the 32 poses are within a few
// decimetres of each other, so the lanes walk nearly the same voxels for nearly the same number of
// steps: the occupancy words coalesce and the trip counts agree.  A CTA = one particle group x 8 chunks
// (8 warps); when a scan needs more than 8 chunks to fill the chip, several CTAs share a particle group and
// the last one to finish (ticket counter) folds the per-CTA partials in chunk order, so the result is still
// deterministic.
constexpr int kPlWarps = kBlockThreads / 32;

struct PlShape
{
  int ppl;  // scan points per lane (chunk length)
  int cb;   // CTAs per particle group (each covers kPlWarps chunks); > 1 only when cpg == kPlWarps
  int cpg;  // chunks (= warps) a CTA spends on one particle group: 1, 2, 4 or 8; the CTA covers kPlWarps / cpg groups
};

template <bool KD>
__global__ void __launch_bounds__(kBlockThreads, 4)
    beam_kernel_pl(const mcl3dl_pose* __restrict__ poses, int P, const float4* __restrict__ scan, int N,
                   const float* __restrict__ origins, DdaGridDev g, KdRayDev kd, NnGridDev nn,
                   mcl3dl_result* __restrict__ out,
                   uint8_t* __restrict__ status, int write_lik_defaults, unsigned long long* __restrict__ stats,
                   PlShape sh, uint32_t* __restrict__ partial, unsigned int* __restrict__ tickets, RecordSink sink)
{
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ uint64_t bar;
  __shared__ uint32_t red[kPlWarps][3][32];
  __shared__ unsigned int s_ticket;
  // short scans (few chunks per group): the CTA's warps are spread over kPlWarps / cpg particle groups, so that no warp
  // is left without rays (c5: 8 rays per particle = 4 chunks; half of every CTA used to idle at the barrier)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gpc = kPlWarps / sh.cpg;
  const int group = (blockIdx.x / sh.cb) * gpc + warp / sh.cpg;
  const int cblk = blockIdx.x % sh.cb;
  const int wchunk = warp % sh.cpg;
  const int base = cblk * kPlWarps * sh.ppl;
  const int slice = max(0, min(N - base, sh.cpg * sh.ppl));
  const float4* tile = reinterpret_cast<const float4*>(smem_raw);
  if (slice > 0)
    stage_tile(smem_raw, scan + base, static_cast<uint32_t>(slice) * 16u, &bar);
  const int j0 = wchunk * sh.ppl;
  const int j1 = min(slice, j0 + sh.ppl);
  const int p = group * 32 + lane;
  const bool live = p < P;
  uint32_t n_short = 0, n_hit = 0, n_long = 0, st_steps = 0, st_occ = 0, st_tested = 0;
  if (j0 < j1)  // warp-uniform
  {
    F3 pos;
    Q4 q;
    pos.x = pos.y = pos.z = 0.0f;
    q.x = q.y = q.z = 0.0f;
    q.w = 1.0f;
    if (live)
      load_pose(poses + p, pos, q);
    const Q4 rn = qnormalized(q);
    for (int j = j0; j < j1; ++j)
    {
      const float4 sp = tile[j];
      F3 v;
      v.x = sp.x;
      v.y = sp.y;
      v.z = sp.z;
      const F3 end = transform_point(rn, pos, v);  // beam.cpp:138-139
      const F3 begin = ray_origin(pos, q, origins, __float_as_uint(sp.w));
      // cast_ray / cast_ray_kd are loops of "walk to the next candidate cell / marching position" followed by the
      // expensive test (fp64 cone test / nearest-neighbour searches): the lanes of the warp reconverge after the walk, so
      // the tests of the lanes that found a candidate run together.
      int st = ST_LONG;
      if (live)
        st = KD ? cast_ray_kd(kd, nn, g, begin, end, st_steps, st_occ, st_tested) : cast_ray(g, begin, end, st_steps, st_occ, st_tested);
      if (live)
      {
        n_short += (st == ST_SHORT);
        n_hit += (st == ST_HIT);
        n_long += (st == ST_LONG);
        if (status)
          status[static_cast<size_t>(p) * N + base + j] = static_cast<uint8_t>(st);
      }
    }
  }
  red[warp][0][lane] = n_short;
  red[warp][1][lane] = n_hit;
  red[warp][2][lane] = n_long;
  __syncthreads();
  if (wchunk == 0)
  {
    uint32_t a = 0, b = 0, c = 0;
    for (int k = 0; k < sh.cpg; ++k)
    {
      a += red[warp + k][0][lane];
      b += red[warp + k][1][lane];
      c += red[warp + k][2][lane];
    }
    bool writer = sh.cb == 1;
    if (sh.cb > 1)
    {
      if (live)
      {
        uint32_t* dst = partial + (static_cast<size_t>(p) * sh.cb + cblk) * 3;
        dst[0] = a;
        dst[1] = b;
        dst[2] = c;
      }
      __threadfence();
      __syncwarp();  // every lane's partial is fenced before lane 0 takes the ticket
      if (lane == 0)
        s_ticket = atomicAdd(tickets + group, 1u);
      __syncwarp();
      if (s_ticket == static_cast<unsigned int>(sh.cb - 1))
      {
        __threadfence();
        writer = true;
        if (live)
        {
          a = b = c = 0;
          for (int k = 0; k < sh.cb; ++k)
          {
            const uint32_t* src = partial + (static_cast<size_t>(p) * sh.cb + k) * 3;
            a += __ldcg(src);
            b += __ldcg(src + 1);
            c += __ldcg(src + 2);
          }
        }
        if (lane == 0)
          tickets[group] = 0;
      }
    }
    if (writer && live)
      sink_store_beam(sink, out, p, beam_score(a, c, N, g), a, b, c, write_lik_defaults);
  }
  if (stats)
  {
    stats_add(stats, 2, st_steps);
    stats_add(stats, 3, st_occ);
    stats_add(stats, 4, st_tested);
  }
}


// ============================================================================================
// Dynamic-queue variant of the lane-per-particle beam kernel.
//
// beam_kernel_pl gives every CTA a fixed set of (particle group, ray chunk) pairs and folds the tallies at a CTA barrier:
// profiles show a large share of the samples of c3 waiting there (rays differ in length, the CTA waits for its slowest warp), and
// whole-wave grids leave nothing to fill the tail with.  Here the grid is the resident warps; every warp pulls
// (group, chunk) items from one global counter until the queue is empty, adds its integer tallies to the particles'
// global counters (integers: the order of the additions cannot change a bit) and the warp that completes a group's
// last chunk (per-group ticket) computes the score and stores the record.  No CTA barrier, no shared-memory tile (a
// chunk's scan points are read by one warp: L1/L2 serve them).  Queue, tickets and tallies are left at zero.
template <bool KD>
__global__ void __launch_bounds__(kBlockThreads, 4)
    beam_kernel_dq(const mcl3dl_pose* __restrict__ poses, int P, const float4* __restrict__ scan, int N,
                   const float* __restrict__ origins, DdaGridDev g, KdRayDev kd, NnGridDev nn, mcl3dl_result* __restrict__ out,
                   uint8_t* __restrict__ status, int write_lik_defaults, unsigned long long* __restrict__ stats, int ppl,
                   int n_chunks, uint32_t* __restrict__ tally /* [P][3] */, unsigned int* __restrict__ tickets /* [groups] */,
                   unsigned int* __restrict__ queue /* [0] next item, [1] warps finished */, RecordSink sink)
{
  const int lane = threadIdx.x & 31;
  const int n_groups = (P + 31) / 32;
  const unsigned int total = static_cast<unsigned int>(n_groups) * static_cast<unsigned int>(n_chunks);
  uint32_t st_steps = 0, st_occ = 0, st_tested = 0;
  for (;;)
  {
    unsigned int item = 0;
    if (lane == 0)
      item = atomicAdd(queue, 1u);
    item = __shfl_sync(0xffffffffu, item, 0);
    if (item >= total)
      break;
    // consecutive items = consecutive groups of the same chunk: neighbouring warps read the same scan points
    const int group = static_cast<int>(item % static_cast<unsigned int>(n_groups));
    const int chunk = static_cast<int>(item / static_cast<unsigned int>(n_groups));
    const int p = group * 32 + lane;
    const bool live = p < P;
    uint32_t n_short = 0, n_hit = 0, n_long = 0;
    if (live)
    {
      F3 pos;
      Q4 q;
      load_pose(poses + p, pos, q);
      const Q4 rn = qnormalized(q);
      const int j0 = chunk * ppl, j1 = min(N, j0 + ppl);
      for (int j = j0; j < j1; ++j)
      {
        const float4 sp = __ldg(scan + j);
        F3 v;
        v.x = sp.x;
        v.y = sp.y;
        v.z = sp.z;
        const F3 end = transform_point(rn, pos, v);  // beam.cpp:138-139
        const F3 begin = ray_origin(pos, q, origins, __float_as_uint(sp.w));
        const int st = KD ? cast_ray_kd(kd, nn, g, begin, end, st_steps, st_occ, st_tested) :
                            cast_ray(g, begin, end, st_steps, st_occ, st_tested);
        n_short += (st == ST_SHORT);
        n_hit += (st == ST_HIT);
        n_long += (st == ST_LONG);
        if (status)
          status[static_cast<size_t>(p) * N + j] = static_cast<uint8_t>(st);
      }
      uint32_t* t = tally + static_cast<size_t>(p) * 3;
      if (n_short) atomicAdd(t, n_short);
      if (n_hit) atomicAdd(t + 1, n_hit);
      if (n_long) atomicAdd(t + 2, n_long);
    }
    __threadfence();
    __syncwarp();
    unsigned int ticket = 0;
    if (lane == 0)
      ticket = atomicAdd(tickets + group, 1u);
    ticket = __shfl_sync(0xffffffffu, ticket, 0);
    if (ticket == static_cast<unsigned int>(n_chunks - 1))
    {
      __threadfence();
      if (live)
      {
        uint32_t* t = tally + static_cast<size_t>(p) * 3;
        const uint32_t a = __ldcg(t), b = __ldcg(t + 1), c = __ldcg(t + 2);
        t[0] = 0;
        t[1] = 0;
        t[2] = 0;
        sink_store_beam(sink, out, p, beam_score(a, c, N, g), a, b, c, write_lik_defaults);
      }
      if (lane == 0)
        tickets[group] = 0;
    }
  }
  // the last warp of the grid to leave resets the queue for the next launch
  if (lane == 0)
  {
    const unsigned int warps = gridDim.x * (kBlockThreads / 32);
    if (atomicAdd(queue + 1, 1u) == warps - 1)
    {
      queue[0] = 0;
      queue[1] = 0;
    }
  }
  if (stats)
  {
    stats_add(stats, 2, st_steps);
    stats_add(stats, 3, st_occ);
    stats_add(stats, 4, st_tested);
  }
}

// ============================================================================================
// Fused weight update (scope row f2): pf::ParticleFilter::measure's arithmetic on the records that
// the two kernels above left on the device.  Deterministic: every reduction has a fixed tree
// (warp shuffles -> per-CTA slot -> one finishing CTA walks the slots in order).
struct WeightPartial
{
  double sum;       // sum of w (pass 1) or of p*ln p (pass 2)
  float qmin, qmax; // likelihood-model quality extremes (pass 1)
  float best;       // largest posterior seen (pass 2)
  uint32_t best_i;  // its particle index (lowest index on ties)
};

// Per-CTA reduction into slots[blockIdx.x]; the LAST CTA to finish (ticket) then folds the slots in order into
// slots[gridDim.x] (and into *host_copy, mapped pinned memory, when given): deterministic, and no separate finishing launch.
__device__ __forceinline__ void weight_block_reduce(WeightPartial v, WeightPartial* slots, WeightPartial* sm, unsigned int* ticket,
                                                    WeightPartial* host_copy)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
  {
    v.sum = dadd(v.sum, __shfl_xor_sync(0xffffffffu, v.sum, o));
    v.qmin = fminf(v.qmin, __shfl_xor_sync(0xffffffffu, v.qmin, o));
    v.qmax = fmaxf(v.qmax, __shfl_xor_sync(0xffffffffu, v.qmax, o));
    const float ob = __shfl_xor_sync(0xffffffffu, v.best, o);
    const uint32_t oi = __shfl_xor_sync(0xffffffffu, v.best_i, o);
    if (ob > v.best || (ob == v.best && oi < v.best_i))
    {
      v.best = ob;
      v.best_i = oi;
    }
  }
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0)
    sm[warp] = v;
  __syncthreads();
  if (threadIdx.x == 0)
  {
    WeightPartial t = sm[0];
    for (int k = 1; k < kBlockThreads / 32; ++k)
    {
      t.sum = dadd(t.sum, sm[k].sum);
      t.qmin = fminf(t.qmin, sm[k].qmin);
      t.qmax = fmaxf(t.qmax, sm[k].qmax);
      if (sm[k].best > t.best || (sm[k].best == t.best && sm[k].best_i < t.best_i))
      {
        t.best = sm[k].best;
        t.best_i = sm[k].best_i;
      }
    }
    slots[blockIdx.x] = t;
    __threadfence();
    if (atomicAdd(ticket, 1u) == gridDim.x - 1)
    {
      __threadfence();
      const int n = static_cast<int>(gridDim.x);
      WeightPartial f;
      f.sum = __ldcg(&slots[0].sum);
      f.qmin = __ldcg(&slots[0].qmin);
      f.qmax = __ldcg(&slots[0].qmax);
      f.best = __ldcg(&slots[0].best);
      f.best_i = __ldcg(&slots[0].best_i);
      for (int k = 1; k < n; ++k)
      {
        f.sum = dadd(f.sum, __ldcg(&slots[k].sum));
        f.qmin = fminf(f.qmin, __ldcg(&slots[k].qmin));
        f.qmax = fmaxf(f.qmax, __ldcg(&slots[k].qmax));
        const float kb = __ldcg(&slots[k].best);
        const uint32_t ki = __ldcg(&slots[k].best_i);
        if (kb > f.best || (kb == f.best && ki < f.best_i))
        {
          f.best = kb;
          f.best_i = ki;
        }
      }
      slots[n] = f;
      if (host_copy)
        *host_copy = f;
      *ticket = 0;  // ready for the next launch (stream order)
    }
  }
}

// pass 1: w_i = prior_i * (((1 * beam) * like) * extra)   (src/mcl_3dl.cpp:406-424, pf.h:258)
__global__ void __launch_bounds__(kBlockThreads)
    weight_kernel(const mcl3dl_result* __restrict__ rec, const float* __restrict__ prior, const float* __restrict__ extra,
                  int P, int n_lik, float* __restrict__ w, WeightPartial* __restrict__ partials, unsigned int* __restrict__ ticket,
                  WeightPartial* __restrict__ host_copy)
{
  __shared__ WeightPartial sm[kBlockThreads / 32];
  WeightPartial v;
  v.sum = 0.0;
  v.qmin = 1.0f;
  v.qmax = 0.0f;
  v.best = -1.0f;
  v.best_i = 0xffffffffu;
  for (int i = blockIdx.x * kBlockThreads + threadIdx.x; i < P; i += gridDim.x * kBlockThreads)
  {
    const mcl3dl_result r = rec[i];
    float lk = fmul(1.0f, r.score_beam);  // map-key order: "beam" then "likelihood"
    lk = fmul(lk, r.score_like);
    if (extra)
      lk = fmul(lk, extra[i]);
    const float wi = fmul(prior[i], lk);
    w[i] = wi;
    v.sum = dadd(v.sum, static_cast<double>(wi));
    // quality of the likelihood model: match_cnt / N, (0 for an empty scan: likelihood.cpp:111-114)
    const float q = n_lik > 0 ? fdiv(static_cast<float>(r.match_cnt), static_cast<float>(n_lik)) : 0.0f;
    v.qmin = fminf(v.qmin, q);
    v.qmax = fmaxf(v.qmax, q);
  }
  weight_block_reduce(v, partials, sm, ticket, host_copy);
}

// pass 2: p_i = w_i / sum (pf.h:266), entropy terms p ln p (pf.h:267-270), arg max
__global__ void __launch_bounds__(kBlockThreads)
    normalize_kernel(const float* __restrict__ w, int P, float total, int index_offset, float* __restrict__ post,
                     WeightPartial* __restrict__ partials, unsigned int* __restrict__ ticket, WeightPartial* __restrict__ host_copy)
{
  __shared__ WeightPartial sm[kBlockThreads / 32];
  WeightPartial v;
  v.sum = 0.0;
  v.qmin = 1.0f;
  v.qmax = 0.0f;
  v.best = -1.0f;
  v.best_i = 0xffffffffu;
  for (int i = blockIdx.x * kBlockThreads + threadIdx.x; i < P; i += gridDim.x * kBlockThreads)
  {
    const float p = fdiv(w[i], total);
    post[i] = p;
    if (p > 0.0f)
      v.sum = dadd(v.sum, static_cast<double>(fmul(p, logf(p))));
    const uint32_t gi = static_cast<uint32_t>(index_offset + i);
    if (p > v.best || (p == v.best && gi < v.best_i))
    {
      v.best = p;
      v.best_i = gi;
    }
  }
  weight_block_reduce(v, partials, sm, ticket, host_copy);
}

// pass 2 without a host round trip (one device): the total comes from pass 1's folded slot instead of a kernel
// argument.  A non-positive total ("No Particle alive", pf.h:274-278) leaves `post` unwritten; the host restores the prior.
__global__ void __launch_bounds__(kBlockThreads)
    normalize_kernel_dev(const float* __restrict__ w, int P, const WeightPartial* __restrict__ pass1, int index_offset,
                         float* __restrict__ post, WeightPartial* __restrict__ partials, unsigned int* __restrict__ ticket,
                         WeightPartial* __restrict__ host_copy)
{
  __shared__ WeightPartial sm[kBlockThreads / 32];
  const float total = __double2float_rn(pass1->sum);
  WeightPartial v;
  v.sum = 0.0;
  v.qmin = 1.0f;
  v.qmax = 0.0f;
  v.best = -1.0f;
  v.best_i = 0xffffffffu;
  if (total > 0.0f)
  {
    for (int i = blockIdx.x * kBlockThreads + threadIdx.x; i < P; i += gridDim.x * kBlockThreads)
    {
      const float p = fdiv(w[i], total);
      post[i] = p;
      if (p > 0.0f)
        v.sum = dadd(v.sum, static_cast<double>(fmul(p, logf(p))));
      const uint32_t gi = static_cast<uint32_t>(index_offset + i);
      if (p > v.best || (p == v.best && gi < v.best_i))
      {
        v.best = p;
        v.best_i = gi;
      }
    }
  }
  weight_block_reduce(v, partials, sm, ticket, host_copy);
}

// --------------------------------------------------------------------------------------------
// Record exchange over peer memory, the signalling half (the data half is RecordSink: the measurement kernels store
// their records into every rank's gathered array).  Every rank owns one buffer [2 x world * n_local records | flags]
// that its peers have mapped (CUDA IPC over NVLink / NVSwitch).  After the two model kernels of step s have retired
// (stream order; their peer stores are performed by then), ONE warp of this kernel
//   (1) releases flag[rank] = s in every rank's buffer (fence.sys + st.release.sys), and
//   (2) spins (ld.acquire.sys, bounded) until all `world` flags of its OWN buffer show >= s,
// so when it retires this rank's copy of the whole array of step s is complete: no host involvement, no collective
// library, one 32-thread launch.  Double buffering by step parity: a peer that is already one step ahead writes the
// OTHER array; it cannot get two steps ahead because its next signal kernel waits for this rank's flag.
// The step number lives in device memory (this kernel increments it), so a captured CUDA graph replays unchanged.
struct PeerTable
{
  uint32_t* flags[kMaxPeers];  // base of every rank's flag array (this rank's own at [rank])
  int world, rank;
};

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v)
{
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p)
{
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__global__ void __launch_bounds__(32)
    exchange_signal_kernel(PeerTable t, uint32_t* __restrict__ step_ctr, unsigned int* __restrict__ err /* set to 1 on a timeout */)
{
  const uint32_t step = *step_ctr + 1u;
  __syncwarp();
  if (threadIdx.x < static_cast<unsigned>(t.world))
  {
    // st.release.sys = fence.acq_rel.sys + store: the records of the model kernels (visible to this kernel through the
    // kernel boundary) are ordered before the flag for the acquiring peer; no separate membar.sys in front of it
    st_release_sys(t.flags[threadIdx.x] + t.rank, step);
    const uint32_t* mine = t.flags[t.rank] + threadIdx.x;
    // steps increase monotonically; the difference is taken modulo 2^32.  Bounded: a peer that died must not hang
    // this GPU
    long polls = 0;
    while (static_cast<int32_t>(ld_acquire_sys(mine) - step) < 0)
      if (++polls > (1L << 22))
      {
        atomicExch(err, 1u);
        break;
      }
  }
  __syncwarp();
  if (threadIdx.x == 0)
    *step_ctr = step;
}

}  // namespace mcl3dl
