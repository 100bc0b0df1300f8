// gl_kernels.cuh — kernels of global localisation and of the resident set's resize (mcl3dl_global_localization,
// mcl3dl_particles_resize): one kernel per stage around the host-verified per-thread functions of gl_funcs.cuh.  The
// VoxelGrid, the CSR grid of the free-space filter and the compaction of its survivors reuse the kernels of scan
// preprocessing and of the map build.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/mcl3dl_b200.h"
#include "gl_funcs.cuh"

namespace mcl3dl
{
// one thread per downsampled point: flag = 1 where the point survives the free-space filter
__global__ void gl_flag_kernel(const mcl3dl_point* __restrict__ pts, uint32_t n, NnGridDev g, GlDev m, uint32_t* __restrict__ flags)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  flags[i] = gl_has_neighbour(g, m, gl_query(g, m, pts[i])) ? 0u : 1u;
}

// one thread per particle: the seeded set, written as the resident set's current states and probabilities
__global__ void gl_fill_kernel(const mcl3dl_point* __restrict__ seeds, const Q4* __restrict__ yaw, uint32_t div_yaw, uint32_t n,
                               float prob, PfState* __restrict__ states, float* __restrict__ probs)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  states[i] = gl_particle(seeds, yaw, div_yaw, i);
  probs[i] = prob;
}

// The pscan chain of resizeParticle (pf.h:415,421): pstep = accum[n - 1] / float(num), then pscan += pstep before each of
// the num picks — serial by definition, so it runs as pf_accum_kernel does: one warp, lane 0 on the dependent add chain
// in a shared tile, the lanes storing the tile coalesced.
__global__ void __launch_bounds__(32) gl_pscan_kernel(const float* __restrict__ accum, uint32_t n, uint32_t num, float* __restrict__ pscan)
{
  constexpr uint32_t kTile = 1024;
  __shared__ float tile[kTile];
  if (blockIdx.x != 0)
    return;
  const uint32_t lane = threadIdx.x;
  const float pstep = fdiv(accum[n - 1], static_cast<float>(num));
  float a = 0.0f;
  for (uint32_t base = 0; base < num; base += kTile)
  {
    const uint32_t m = min(kTile, num - base);
    if (lane == 0)
    {
      uint32_t i = 0;
      for (; i + 16 <= m; i += 16)
      {
        float v[16];
#pragma unroll
        for (int k = 0; k < 16; ++k)
        {
          a = fadd(a, pstep);
          v[k] = a;
        }
#pragma unroll
        for (int k = 0; k < 16; ++k) tile[i + k] = v[k];
      }
      for (; i < m; ++i)
      {
        a = fadd(a, pstep);
        tile[i] = a;
      }
    }
    __syncwarp();
    for (uint32_t i = lane; i < m; i += 32) pscan[base + i] = tile[i];
    __syncwarp();
  }
}

// one thread per output particle: the whole state of its pick, probability 1 / num
__global__ void gl_resize_kernel(const PfState* __restrict__ in, const float* __restrict__ accum, uint32_t n,
                                 const float* __restrict__ pscan, uint32_t num, PfState* __restrict__ out, float* __restrict__ out_probs)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= num)
    return;
  out[i] = in[gl_resize_pick(accum, n, pscan, i)];
  out_probs[i] = gl_resize_probability(num);
}

}  // namespace mcl3dl
