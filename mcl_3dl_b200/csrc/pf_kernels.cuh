// pf_kernels.cuh — kernels of the resident particle set (scope row f3, SURVEY.md §8f): one thread per particle around the
// host-verified per-particle functions of pf_funcs.cuh.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/mcl3dl_b200.h"
#include "pf_funcs.cuh"

namespace mcl3dl
{
static_assert(sizeof(PfState) == sizeof(mcl3dl_state), "mcl3dl_state is PfState");

// MotionPredictionModelDifferentialDrive::predict for every particle (pf::ParticleFilter::predict, pf.h:239-245)
__global__ void pf_predict_kernel(PfState* __restrict__ states, uint32_t n, MotionDev m)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    pf_predict(states[i], m);
}

// What the measurement kernels read: pos + RAW rot (they normalise it themselves, state_6dof.h:217), and the
// odometry-error factor of the node's lambda, NormalLikelihood(sigma)(|odom_err_integ_lin_|) (src/mcl_3dl.cpp:400,422-424,
// include/mcl_3dl/nd.h:45-53: a = float(1 / sqrt(2 pi s^2)), sq2 = float(2 s^2), a * expf(-x * x / sq2)).
__global__ void pf_pack_kernel(const PfState* __restrict__ states, uint32_t n, float nd_a, float nd_sq2, mcl3dl_pose* __restrict__ poses,
                               float* __restrict__ extra /* nullptr: no odometry-error factor */)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const PfState s = states[i];
  mcl3dl_pose p;
  p.px = s.pos[0];
  p.py = s.pos[1];
  p.pz = s.pos[2];
  p._pad = 0.0f;
  p.qx = s.rot[0];
  p.qy = s.rot[1];
  p.qz = s.rot[2];
  p.qw = s.rot[3];
  poses[i] = p;
  if (extra)
  {
    F3 l;
    l.x = s.lin[0];
    l.y = s.lin[1];
    l.z = s.lin[2];
    const float x = __fsqrt_rn(dot3(l, l));  // Vec3::norm, vec3.h:148-151
    extra[i] = fmul(nd_a, expf(fdiv(fmul(-x, x), nd_sq2)));
  }
}

// The sequential float prefix sum of pf.h:189-194 and pstep of :197 — strictly in order: a parallel scan rounds
// differently and would move picks at the interval boundaries.  One warp: the lanes stream the probabilities through
// shared memory in coalesced 1024-element tiles, lane 0 runs the dependent add chain on the tile (65 536 adds at the
// 4-cycle add latency ~ 0.15 ms; the first version read global memory inside the chain and took 1.1 ms), the lanes
// write the sums back coalesced.
__global__ void __launch_bounds__(32) pf_accum_kernel(const float* __restrict__ probs, uint32_t n, float* __restrict__ accum,
                                                      float* __restrict__ pstep)
{
  constexpr uint32_t kTile = 1024;
  __shared__ float tile[kTile];
  if (blockIdx.x != 0)
    return;
  const uint32_t lane = threadIdx.x;
  float a = 0.0f;
  for (uint32_t base = 0; base < n; base += kTile)
  {
    const uint32_t m = min(kTile, n - base);
    for (uint32_t i = lane; i < m; i += 32) tile[i] = probs[base + i];
    __syncwarp();
    if (lane == 0)
    {
      // 16 values at a time through registers: the loads and stores stay off the dependent add chain
      uint32_t i = 0;
      for (; i + 16 <= m; i += 16)
      {
        float v[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) v[k] = tile[i + k];
#pragma unroll
        for (int k = 0; k < 16; ++k)
        {
          a = fadd(a, v[k]);
          v[k] = a;
        }
#pragma unroll
        for (int k = 0; k < 16; ++k) tile[i + k] = v[k];
      }
      for (; i < m; ++i)
      {
        a = fadd(a, tile[i]);
        tile[i] = a;
      }
    }
    __syncwarp();
    for (uint32_t i = lane; i < m; i += 32) accum[base + i] = tile[i];
    __syncwarp();
  }
  if (lane == 0)
    *pstep = fdiv(a, static_cast<float>(n));
}

struct Sigma6
{
  float v[6];
};

// pf::ParticleFilter::resample (pf.h:182-225): systematic pick, noise on duplicates, probability 1 / n
__global__ void pf_resample_kernel(const PfState* __restrict__ in, const float* __restrict__ accum, const float* __restrict__ pstep,
                                   uint32_t n, float initial_frac, uint64_t seed, uint32_t call, Sigma6 sigma,
                                   PfState* __restrict__ out, float* __restrict__ out_probs)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const float ps = *pstep;
  bool dup;
  const uint32_t src = pf_pick(accum, n, ps, fmul(initial_frac, ps), i, dup);
  PfState s = in[src];
  if (dup)
  {
    float org[6];
    pf_noise6(seed, i, call, sigma.v, org);
    s = pf_add_noise(s, org);
  }
  out[i] = s;
  out_probs[i] = __double2float_rn(ddiv(1.0, static_cast<double>(n)));
}

// ---- pose estimate on the resident set (mcl3dl_particles_estimate): pf_->bias + expectationBiased + max + covariance
// (src/mcl_3dl.cpp:428-452,704-724; pf.h:246-251,281-374).  Two passes of double sums with a fixed tree (lanes by
// shuffles, warps and CTAs in order), so the result is deterministic; the reference sums sequentially in float, hence
// agreement to ~1e-5 relative, not bitwise.
constexpr int kEstSums = 20;  // biased: w, w*pos(3), w*front(3), w*up(3); unbiased: the same ten with p
constexpr int kCovSums = 22;  // p, 21 upper-triangle products p * d_j * d_k
struct EstHeader
{
  float mean_b_pos[3], mean_b_rot[4];  // expectationBiased()
  float mean_u_pos[3], mean_u_rpy[3];  // expectation(1.0): the centre of covariance()
  float weight_sum_biased, weight_sum;
  float max_prob;
  uint32_t max_index;
  float cov[36];
};

template <int NS>
__device__ __forceinline__ void est_block_reduce(double (&v)[NS], double* __restrict__ slot, double (*sm)[NS])
{
#pragma unroll
  for (int k = 0; k < NS; ++k)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] = dadd(v[k], __shfl_xor_sync(0xffffffffu, v[k], o));
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0)
    for (int k = 0; k < NS; ++k) sm[warp][k] = v[k];
  __syncthreads();
  if (threadIdx.x < NS)
  {
    double t = sm[0][threadIdx.x];
    for (int w = 1; w < 8; ++w) t = dadd(t, sm[w][threadIdx.x]);
    slot[threadIdx.x] = t;
  }
}

__global__ void __launch_bounds__(256)
    pf_est_pass1_kernel(const PfState* __restrict__ states, const float* __restrict__ probs, uint32_t n, BiasDev bias,
                        double* __restrict__ partials /* [grid][kEstSums + 2] */)
{
  __shared__ double sm[8][kEstSums];
  __shared__ float sm_best[8];
  __shared__ uint32_t sm_best_i[8];
  double v[kEstSums];
#pragma unroll
  for (int k = 0; k < kEstSums; ++k) v[k] = 0.0;
  float best = -1.0f;
  uint32_t best_i = 0xffffffffu;
  for (uint32_t i = blockIdx.x * 256u + threadIdx.x; i < n; i += gridDim.x * 256u)
  {
    const PfState s = states[i];
    const float p = probs[i];
    const float w = fmul(p, pf_bias(s, bias));  // mean.add(p.state_, p.probability_ * p.probability_bias_), pf.h:300
    float t[9];
    pf_mean_terms(s, t);
    v[0] = dadd(v[0], static_cast<double>(w));
    v[10] = dadd(v[10], static_cast<double>(p));
#pragma unroll
    for (int k = 0; k < 9; ++k)
    {
      v[1 + k] = dadd(v[1 + k], static_cast<double>(fmul(t[k], w)));   // e1.pos_ * prob etc.: float products, as the reference
      v[11 + k] = dadd(v[11 + k], static_cast<double>(fmul(t[k], p)));
    }
    if (p > best)  // pf.h:361-374: the first particle with the largest probability
    {
      best = p;
      best_i = i;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
  {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const uint32_t oi = __shfl_xor_sync(0xffffffffu, best_i, o);
    if (ob > best || (ob == best && oi < best_i))
    {
      best = ob;
      best_i = oi;
    }
  }
  if ((threadIdx.x & 31) == 0)
  {
    sm_best[threadIdx.x >> 5] = best;
    sm_best_i[threadIdx.x >> 5] = best_i;
  }
  double* slot = partials + static_cast<size_t>(blockIdx.x) * (kEstSums + 2);
  est_block_reduce<kEstSums>(v, slot, sm);
  if (threadIdx.x == 0)
  {
    float b = sm_best[0];
    uint32_t bi = sm_best_i[0];
    for (int w = 1; w < 8; ++w)
      if (sm_best[w] > b || (sm_best[w] == b && sm_best_i[w] < bi))
      {
        b = sm_best[w];
        bi = sm_best_i[w];
      }
    slot[kEstSums] = static_cast<double>(b);
    slot[kEstSums + 1] = static_cast<double>(bi);
  }
}

// fold the per-CTA slots: one thread per column, slots in order (deterministic), then thread 0 derives the means
__global__ void __launch_bounds__(32) pf_est_finish1_kernel(const double* __restrict__ partials, int n_slots, EstHeader* __restrict__ h)
{
  __shared__ double v[kEstSums];
  __shared__ double sm_best[2];
  if (blockIdx.x != 0)
    return;
  if (threadIdx.x < kEstSums)
  {
    double t = 0.0;
    for (int s = 0; s < n_slots; ++s) t = dadd(t, partials[static_cast<size_t>(s) * (kEstSums + 2) + threadIdx.x]);
    v[threadIdx.x] = t;
  }
  else if (threadIdx.x == kEstSums)
  {
    double best = -1.0, best_i = 4294967295.0;
    for (int s = 0; s < n_slots; ++s)
    {
      const double* slot = partials + static_cast<size_t>(s) * (kEstSums + 2);
      if (slot[kEstSums] > best || (slot[kEstSums] == best && slot[kEstSums + 1] < best_i))
      {
        best = slot[kEstSums];
        best_i = slot[kEstSums + 1];
      }
    }
    sm_best[0] = best;
    sm_best[1] = best_i;
  }
  __syncwarp();
  if (threadIdx.x != 0)
    return;
  for (int a = 0; a < 3; ++a)
  {
    h->mean_b_pos[a] = static_cast<float>(v[1 + a] / v[0]);   // e_.pos_ / p_sum_, state_6dof.h:347
    h->mean_u_pos[a] = static_cast<float>(v[11 + a] / v[10]);
  }
  pf_quat_from_front_up(v + 4, v + 7, h->mean_b_rot);
  float qu[4];
  pf_quat_from_front_up(v + 14, v + 17, qu);
  pf_rpy(qu, h->mean_u_rpy);
  h->weight_sum_biased = static_cast<float>(v[0]);
  h->weight_sum = static_cast<float>(v[10]);
  h->max_prob = static_cast<float>(sm_best[0]);
  h->max_index = static_cast<uint32_t>(sm_best[1]);
}

__global__ void __launch_bounds__(256)
    pf_est_pass2_kernel(const PfState* __restrict__ states, const float* __restrict__ probs, uint32_t n,
                        const EstHeader* __restrict__ h, double* __restrict__ partials /* [grid][kCovSums] */)
{
  __shared__ double sm[8][kCovSums];
  const float e_pos[3] = {h->mean_u_pos[0], h->mean_u_pos[1], h->mean_u_pos[2]};
  const float e_rpy[3] = {h->mean_u_rpy[0], h->mean_u_rpy[1], h->mean_u_rpy[2]};
  double v[kCovSums];
#pragma unroll
  for (int k = 0; k < kCovSums; ++k) v[k] = 0.0;
  for (uint32_t i = blockIdx.x * 256u + threadIdx.x; i < n; i += gridDim.x * 256u)
  {
    const PfState s = states[i];
    const float p = probs[i];
    float d[6];
    pf_cov_diff(s, e_pos, e_rpy, d);
    v[0] = dadd(v[0], static_cast<double>(p));
    int t = 1;
#pragma unroll
    for (int j = 0; j < 6; ++j)
#pragma unroll
      for (int k = j; k < 6; ++k)
      {
        v[t] = dadd(v[t], static_cast<double>(fmul(fmul(fmul(1.0f, d[j]), d[k]), p)));  // covElement(e, j, k) * probability_
        ++t;
      }
  }
  est_block_reduce<kCovSums>(v, partials + static_cast<size_t>(blockIdx.x) * kCovSums, sm);
}

__global__ void __launch_bounds__(32) pf_est_finish2_kernel(const double* __restrict__ partials, int n_slots, EstHeader* __restrict__ h)
{
  __shared__ double v[kCovSums];
  if (blockIdx.x != 0)
    return;
  if (threadIdx.x < kCovSums)
  {
    double t = 0.0;
    for (int s = 0; s < n_slots; ++s) t = dadd(t, partials[static_cast<size_t>(s) * kCovSums + threadIdx.x]);
    v[threadIdx.x] = t;
  }
  __syncwarp();
  if (threadIdx.x != 0)
    return;
  int t = 1;
  for (int j = 0; j < 6; ++j)
    for (int k = j; k < 6; ++k)
    {
      const float c = static_cast<float>(v[t++] / v[0]);  // cov[k][j] /= p_sum, pf.h:352-358
      h->cov[j * 6 + k] = c;
      h->cov[k * 6 + j] = c;
    }
}

}  // namespace mcl3dl
