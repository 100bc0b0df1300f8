// Host model of lik_kernel_nf's warp-cooperative candidate scan (kernels.cuh, phase B), lane by lane, built from the
// device helpers in device_funcs.cuh.  TEST INFRASTRUCTURE ONLY (tests/test_nf_warp_scan.py).
#include "cuda_shim.h"

#include <algorithm>
#include <vector>

#include "../../include/mcl3dl_b200.h"
#include "../../mcl_3dl_b200/csrc/device_funcs.cuh"

using namespace mcl3dl;

// One warp trip of U evals per lane (eval e = u * 32 + lane): count[e] candidates from first[e] (count < 0: overflow
// cell, no candidates here), query q[e].  Slots are processed in passes of `pass_slots`, and within a pass in the order
// `perm` (a permutation of 0 .. pass_slots - 1; slots beyond a short pass are skipped) - any order the lanes' rounds and
// atomics may take.  best[e]: the bits the kernel's atomicMin leaves (r2 to start with).  Returns W.
extern "C" int hostsim_nf_warp_scan(int U, const int* count, const uint32_t* first, const float* q, const float4* cand,
                                    float r2, int pass_slots, const int* perm, float* best)
{
  const int E = 32 * U;
  std::vector<int> base(E);
  int W = 0;
  for (int lane = 0; lane < 32; ++lane)  // the shuffle scan: lanes in order, a lane's evals u = 0 .. U - 1
    for (int u = 0; u < U; ++u)
    {
      base[u * 32 + lane] = W;
      W += std::max(count[u * 32 + lane], 0);
    }
  std::vector<uint32_t> off(E), bits(E);
  for (int e = 0; e < E; ++e)
  {
    off[e] = first[e] - static_cast<uint32_t>(base[e]);
    bits[e] = __float_as_uint(r2);
  }
  std::vector<uint8_t> own(pass_slots);
  for (int lo = 0; lo < W; lo += pass_slots)
  {
    const int hi = std::min(W, lo + pass_slots);
    for (int e = 0; e < E; ++e) nnf_fill_owner(own.data(), lo, hi, base[e], std::max(count[e], 0), e);
    for (int i = 0; i < pass_slots; ++i)
    {
      const int k = lo + perm[i];
      if (k >= hi)
        continue;
      const int e = own[k - lo];
      const float4 m = cand[off[e] + static_cast<uint32_t>(k)];
      bits[e] = std::min(bits[e], __float_as_uint(nnf_cand_d2(q[3 * e], q[3 * e + 1], q[3 * e + 2], m)));
    }
  }
  for (int e = 0; e < E; ++e) best[e] = __uint_as_float(bits[e]);
  return W;
}
