// pf_init_hostsim.cpp — TEST INFRASTRUCTURE ONLY.
//
// Host driver for the per-particle function of the initial seed in mcl_3dl_b200/csrc/pf_funcs.cuh, compiled for the host
// through cuda_shim.h: one loop over the particles with the very function pf_init_kernel calls per thread.
// tests/test_pf_init_on_host.py compares it with the port and reference checkers of oracle/pf_init_api.h.
#include <cstring>

#include "cuda_shim.h"

#include "../../include/mcl3dl_b200.h"
#include "../../mcl_3dl_b200/csrc/pf_funcs.cuh"

using namespace mcl3dl;

static_assert(sizeof(PfState) == sizeof(mcl3dl_state), "PfState is mcl3dl_state");

// mcl3dl_particles_init's call `call` for n particles (the kernel's probability included); z [n][6] (may be NULL)
// receives each particle's standard normals
extern "C" void hostsim_pf_init(size_t n, int multivariate, const float mean[6], const float sigma[6], const float T[36],
                                uint64_t seed, uint32_t call, PfState* states, float* probs, float* z)
{
  InitDev g;
  g.multivariate = multivariate;
  std::memcpy(g.mean, mean, sizeof(g.mean));
  std::memcpy(g.sigma, sigma, sizeof(g.sigma));
  std::memcpy(g.T, T, sizeof(g.T));
  for (size_t i = 0; i < n; ++i)
  {
    states[i] = pf_init_state(seed, static_cast<uint32_t>(i), call, g);
    probs[i] = __double2float_rn(ddiv(1.0, static_cast<double>(n)));
    if (z)
      pf_normal6_event(seed, static_cast<uint32_t>(i), call, kPfEventInit, [&](int pair, float rad, float phi) {
        z[6 * i + 2 * pair] = fmul(rad, cosf(phi));
        z[6 * i + 2 * pair + 1] = fmul(rad, sinf(phi));
      });
  }
}
