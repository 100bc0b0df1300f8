// pf_landmark_hostsim.cpp — TEST INFRASTRUCTURE ONLY.
//
// Host drivers for the per-particle functions of the landmark update, the odometry-error reset and the published poses
// in mcl_3dl_b200/csrc/pf_funcs.cuh, compiled for the host through cuda_shim.h: one loop over the particles with the
// very functions pf_landmark_kernel, pf_reset_odom_err_kernel and pf_poses_kernel call per thread.
// tests/test_pf_landmark_on_host.py compares them with the port and reference checkers of oracle/pf_landmark_api.h.
#include <cstring>

#include "cuda_shim.h"

#include "../../include/mcl3dl_b200.h"
#include "../../mcl_3dl_b200/csrc/pf_funcs.cuh"

using namespace mcl3dl;

static_assert(sizeof(PfState) == sizeof(mcl3dl_state), "PfState is mcl3dl_state");

static LandmarkDev landmark_dev(const float measured[7], float nd_a, const float sigma_inv[36])
{
  LandmarkDev m;
  m.pos[0] = measured[0];
  m.pos[1] = measured[1];
  m.pos[2] = measured[2];
  m.rot = Q4{measured[3], measured[4], measured[5], measured[6]};
  m.nd_a = nd_a;
  std::memcpy(m.sigma_inv, sigma_inv, sizeof(m.sigma_inv));
  return m;
}

// pf_landmark_likelihood of states[0..n) for the measured pose (x y z, qx qy qz qw), a and sigma_inv (row-major); x (may
// be NULL) [n][6] receives each particle's pf_landmark_x
extern "C" void hostsim_pf_landmark(const PfState* states, size_t n, const float measured[7], float nd_a,
                                    const float sigma_inv[36], float* lik, float* x)
{
  const LandmarkDev m = landmark_dev(measured, nd_a, sigma_inv);
  for (size_t i = 0; i < n; ++i)
  {
    lik[i] = pf_landmark_likelihood(states[i], m);
    if (x)
      pf_landmark_x(states[i], m, x + 6 * i);
  }
}

// pf_nd6_exponent of one x
extern "C" float hostsim_pf_nd6_exponent(const float x[6], const float sigma_inv[36]) { return pf_nd6_exponent(x, sigma_inv); }

extern "C" void hostsim_pf_reset_odom_err(PfState* states, size_t n)
{
  for (size_t i = 0; i < n; ++i) pf_reset_odom_err_integ(states[i]);
}

// pf_published_pose of states[0..n) into out [n][8] (the mcl3dl_pose layout)
extern "C" void hostsim_pf_poses(const PfState* states, size_t n, float* out)
{
  for (size_t i = 0; i < n; ++i) pf_published_pose(states[i], out + 8 * i);
}
