// pf_events_hostsim.cpp — TEST INFRASTRUCTURE ONLY.
//
// Host drivers for the per-particle functions of the odometry-noise redraw, the expansion noise and the IMU gravity
// update in mcl_3dl_b200/csrc/pf_funcs.cuh, compiled for the host through cuda_shim.h: one loop over the particles with
// the very functions pf_redraw_kernel, pf_noise_kernel and pf_imu_kernel call per thread.
// tests/test_pf_events_on_host.py compares them with the port and reference checkers of oracle/pf_events_api.h.
#include "cuda_shim.h"

#include "../../include/mcl3dl_b200.h"
#include "../../mcl_3dl_b200/csrc/pf_funcs.cuh"

using namespace mcl3dl;

static_assert(sizeof(PfState) == sizeof(mcl3dl_state), "PfState is mcl3dl_state");

// mcl3dl_particles_redraw_odom_noise's call `call` on states[0..n), in place
extern "C" void hostsim_pf_redraw(PfState* states, size_t n, uint64_t seed, uint32_t call, double lin_lin, double lin_ang,
                                  double ang_lin, double ang_ang)
{
  OdomNoiseSigma sg;
  sg.ll = lin_lin;
  sg.la = lin_ang;
  sg.aa = ang_ang;
  sg.al = ang_lin;
  for (size_t i = 0; i < n; ++i) pf_redraw_odom_noise(states[i], seed, static_cast<uint32_t>(i), call, sg);
}

// mcl3dl_particles_noise's call `call` on states[0..n), in place; org [n][6] receives the draws
extern "C" void hostsim_pf_noise(PfState* states, size_t n, uint64_t seed, uint32_t call, const float sigma_pos[3],
                                 const float sigma_rpy[3], float* org)
{
  const float sigma[6] = {sigma_pos[0], sigma_pos[1], sigma_pos[2], sigma_rpy[0], sigma_rpy[1], sigma_rpy[2]};
  for (size_t i = 0; i < n; ++i)
  {
    if (org)
      pf_noise6_event(seed, static_cast<uint32_t>(i), call, kPfEventNoise, sigma, org + 6 * i);
    states[i] = pf_expansion_noise(states[i], seed, static_cast<uint32_t>(i), call, sigma);
  }
}

// six draws of (index, call, event) as pf_noise6_event lays them out
extern "C" void hostsim_pf_noise6_event(uint64_t seed, uint32_t index, uint32_t call, uint32_t event, const float sigma[6],
                                        float org[6])
{
  pf_noise6_event(seed, index, call, event, sigma, org);
}

// pf_imu_likelihood of states[0..n) and the host constants of pf_imu_setup (acc_norm, nd_a, nd_sq2)
extern "C" void hostsim_pf_imu(const PfState* states, size_t n, const float acc[3], double acc_var, float* lik, float* consts)
{
  const ImuDev m = pf_imu_setup(acc, static_cast<float>(acc_var));
  for (size_t i = 0; i < n; ++i) lik[i] = pf_imu_likelihood(states[i], m);
  if (consts)
  {
    consts[0] = m.acc_norm;
    consts[1] = m.nd_a;
    consts[2] = m.nd_sq2;
  }
}

extern "C" void hostsim_philox(uint32_t ctr[4], uint32_t k0, uint32_t k1) { philox4x32_10(ctr, k0, k1); }
