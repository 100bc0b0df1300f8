// pf_compile_check.cu — TEST INFRASTRUCTURE ONLY: instantiates every function of mcl_3dl_b200/csrc/pf_funcs.cuh in device
// code, so that `nvcc -gencode arch=compute_90a,code=sm_90a -c` proves the f3 groundwork compiles for the H100
// (tests/test_hostsim.py::test_pf_funcs_compile_for_sm_90a).  The thin kernels below are also the shape the round-2
// kernels will take: one thread per particle around the host-verified per-thread functions.
#include <cuda_runtime.h>

#include "../../mcl_3dl_b200/csrc/pf_funcs.cuh"

using namespace mcl3dl;

__global__ void predict_kernel(PfState* __restrict__ states, uint32_t n, MotionDev m)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    pf_predict(states[i], m);
}

// the sequential float prefix sum of pf.h:189-194: one thread, in order (65 536 dependent adds ~ 0.15 ms)
__global__ void accum_kernel(const float* __restrict__ probs, uint32_t n, float* __restrict__ accum, float* __restrict__ pstep)
{
  if (blockIdx.x != 0 || threadIdx.x != 0)
    return;
  float a = 0.0f;
  for (uint32_t i = 0; i < n; ++i)
  {
    a = fadd(a, probs[i]);
    accum[i] = a;
  }
  *pstep = fdiv(a, static_cast<float>(n));
}

__global__ void resample_kernel(const PfState* __restrict__ in, const float* __restrict__ accum, const float* __restrict__ pstep,
                                uint32_t n, float initial_frac, uint64_t seed, uint32_t call, const float* __restrict__ sigma6,
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
    float sigma[6], org[6];
    for (int k = 0; k < 6; ++k) sigma[k] = sigma6[k];
    pf_noise6(seed, i, call, sigma, org);
    s = pf_add_noise(s, org);
  }
  out[i] = s;
  out_probs[i] = __double2float_rn(ddiv(1.0, static_cast<double>(n)));
}
