// pf_hostsim.cpp — TEST INFRASTRUCTURE ONLY.
//
// Host drivers for mcl_3dl_b200/csrc/pf_funcs.cuh (scope row f3 groundwork: motion prediction, systematic resampling,
// State6DOF noise as per-thread device functions), compiled for the host through cuda_shim.h like hostsim.cpp.
// tests/test_hostsim.py compares them with the oracle pieces that are pinned bit for bit to the reference build.
#include "cuda_shim.h"

#include <random>
#include <vector>

#include "../../include/mcl3dl_b200.h"
#include "../../mcl_3dl_b200/csrc/pf_funcs.cuh"

using namespace mcl3dl;

static_assert(sizeof(PfState) == 17 * sizeof(float), "PfState must match the oracle's mcl3dl_cpu_motion_state");

// MotionPredictionModelDifferentialDrive::setOdoms + predict over n states (in place)
extern "C" int hostsim_pf_predict(const mcl3dl_pose* odom_prev, const mcl3dl_pose* odom_cur, float time_diff, float tc_lin,
                                  float tc_ang, PfState* states, size_t n)
{
  const float pp[3] = {odom_prev->px, odom_prev->py, odom_prev->pz}, pq[4] = {odom_prev->qx, odom_prev->qy, odom_prev->qz, odom_prev->qw};
  const float cp[3] = {odom_cur->px, odom_cur->py, odom_cur->pz}, cq[4] = {odom_cur->qx, odom_cur->qy, odom_cur->qz, odom_cur->qw};
  const MotionDev m = pf_set_odoms(pp, pq, cp, cq, time_diff, tc_lin, tc_ang);
  for (size_t i = 0; i < n; ++i) pf_predict(states[i], m);
  return 0;
}

namespace
{
// the sequential prefix sum of pf.h:189-194 and pstep of :197
float prefix(const float* probs, size_t n, std::vector<float>& accum)
{
  accum.resize(n);
  float a = 0;
  for (size_t i = 0; i < n; ++i)
  {
    a = __fadd_rn(a, probs[i]);
    accum[i] = a;
  }
  return a / static_cast<float>(n);
}
}  // namespace

// pf::ParticleFilter<State6DOF>(n, seed)::resample(State6DOF(sigma_pos, sigma_rpy)) with the device functions doing the
// pick and the noise application, and libstdc++'s engine drawing initial_p and the normals in the REFERENCE'S order (six
// per duplicate, in output order, a fresh std::normal_distribution per draw; sigma == 0 draws nothing).  Must equal the
// oracle / the reference build bit for bit as long as no two particles share an accumulated probability.
extern "C" int hostsim_pf_resample_ref_rng(const float* probs, const PfState* states, size_t n, unsigned int seed,
                                           const float sigma_pos[3], const float sigma_rpy[3], PfState* out, float* out_probs,
                                           uint32_t* src_out, uint8_t* dup_out)
{
  std::default_random_engine engine(seed);
  std::vector<float> accum;
  const float pstep = prefix(probs, n, accum);
  const float initial_p = std::uniform_real_distribution<float>(0.0, pstep)(engine);
  const float sigma[6] = {sigma_pos[0], sigma_pos[1], sigma_pos[2], sigma_rpy[0], sigma_rpy[1], sigma_rpy[2]};
  for (size_t i = 0; i < n; ++i)
  {
    bool dup = false;
    const uint32_t src = pf_pick(accum.data(), static_cast<uint32_t>(n), pstep, initial_p, static_cast<uint32_t>(i), dup);
    if (dup)
    {
      float org[6];
      for (int k = 0; k < 6; ++k) org[k] = sigma[k] == 0 ? 0.0f : std::normal_distribution<float>(0.0f, sigma[k])(engine);
      out[i] = pf_add_noise(states[src], org);
    }
    else
    {
      out[i] = states[src];
    }
    out_probs[i] = static_cast<float>(1.0 / n);
    if (src_out) src_out[i] = src;
    if (dup_out) dup_out[i] = dup ? 1 : 0;
  }
  return 0;
}

// The device's own semantics: initial_p = initial_frac * pstep handed in by the host (drawn with the node's engine),
// Philox noise keyed by (seed, output index, call).  Deterministic; compared statistically and against known answers.
extern "C" int hostsim_pf_resample_philox(const float* probs, const PfState* states, size_t n, float initial_frac, uint64_t seed,
                                          uint32_t call, const float sigma_pos[3], const float sigma_rpy[3], PfState* out,
                                          float* out_probs, uint32_t* src_out, uint8_t* dup_out, float* noise_out /* n x 6 */)
{
  std::vector<float> accum;
  const float pstep = prefix(probs, n, accum);
  const float initial_p = __fmul_rn(initial_frac, pstep);
  const float sigma[6] = {sigma_pos[0], sigma_pos[1], sigma_pos[2], sigma_rpy[0], sigma_rpy[1], sigma_rpy[2]};
  for (size_t i = 0; i < n; ++i)
  {
    bool dup = false;
    const uint32_t src = pf_pick(accum.data(), static_cast<uint32_t>(n), pstep, initial_p, static_cast<uint32_t>(i), dup);
    float org[6] = {0, 0, 0, 0, 0, 0};
    if (dup)
    {
      pf_noise6(seed, static_cast<uint32_t>(i), call, sigma, org);
      out[i] = pf_add_noise(states[src], org);
    }
    else
    {
      out[i] = states[src];
    }
    out_probs[i] = static_cast<float>(1.0 / n);
    if (src_out) src_out[i] = src;
    if (dup_out) dup_out[i] = dup ? 1 : 0;
    if (noise_out)
      for (int k = 0; k < 6; ++k) noise_out[6 * i + k] = org[k];
  }
  return 0;
}

extern "C" void hostsim_philox(uint32_t ctr[4], uint32_t k0, uint32_t k1) { philox4x32_10(ctr, k0, k1); }

extern "C" void hostsim_noise6(uint64_t seed, uint32_t index, uint32_t call, const float sigma[6], float org[6])
{
  pf_noise6(seed, index, call, sigma, org);
}

namespace
{
// mcl3dl_particles_estimate's BiasDev for `prev` (nullptr: the constant bias 1)
BiasDev bias_of(const mcl3dl_pose* prev, float bias_var_dist, float bias_var_ang)
{
  BiasDev b{};
  if (prev)
  {
    b.enabled = 1;
    b.prev_pos[0] = prev->px;
    b.prev_pos[1] = prev->py;
    b.prev_pos[2] = prev->pz;
    const float d = prev->qx * prev->qx + prev->qy * prev->qy + prev->qz * prev->qz + prev->qw * prev->qw;
    const float id = static_cast<float>(1.0 / d);
    b.prev_inv = Q4{-prev->qx * id, -prev->qy * id, -prev->qz * id, prev->qw * id};
    const double sl = bias_var_dist, sa = bias_var_ang;
    b.lin_a = static_cast<float>(1.0 / std::sqrt(2.0 * M_PI * sl * sl));
    b.lin_sq2 = static_cast<float>(sl * sl * 2.0);
    b.ang_a = static_cast<float>(1.0 / std::sqrt(2.0 * M_PI * sa * sa));
    b.ang_sq2 = static_cast<float>(sa * sa * 2.0);
  }
  return b;
}
}  // namespace

// The float terms pf_est_pass1_kernel adds in double, per particle, in its column order: terms[20 i + k] = w, w * pos(3),
// w * front(3), w * up(3), p, p * pos(3), p * front(3), p * up(3), with w = fmul(p, pf_bias).  bias[i] = pf_bias.
extern "C" int hostsim_pf_est_terms(const float* probs, const PfState* states, size_t n, const mcl3dl_pose* prev, float bias_var_dist,
                                    float bias_var_ang, float* bias, float* terms)
{
  const BiasDev b = bias_of(prev, bias_var_dist, bias_var_ang);
  for (size_t i = 0; i < n; ++i)
  {
    const float p = probs[i];
    bias[i] = pf_bias(states[i], b);
    const float w = __fmul_rn(p, bias[i]);
    float t[9];
    pf_mean_terms(states[i], t);
    float* o = terms + 20 * i;
    o[0] = w;
    o[10] = p;
    for (int k = 0; k < 9; ++k)
    {
      o[1 + k] = __fmul_rn(t[k], w);
      o[11 + k] = __fmul_rn(t[k], p);
    }
  }
  return 0;
}

// pf_est_finish1_kernel's derivations from the twenty column sums v: the biased mean (pos, rot) and the centre of the
// covariance (e_pos, e_rpy)
extern "C" void hostsim_pf_est_finish(const double* v, float* mean_pos, float* mean_rot, float* e_pos, float* e_rpy)
{
  for (int a = 0; a < 3; ++a)
  {
    mean_pos[a] = static_cast<float>(v[1 + a] / v[0]);
    e_pos[a] = static_cast<float>(v[11 + a] / v[10]);
  }
  pf_quat_from_front_up(v + 4, v + 7, mean_rot);
  float qu[4];
  pf_quat_from_front_up(v + 14, v + 17, qu);
  pf_rpy(qu, e_rpy);
}

// The float terms pf_est_pass2_kernel adds in double for the centre (e_pos, e_rpy): terms[22 i] = p, then the 21
// upper-triangle products fmul(fmul(fmul(1, d_j), d_k), p); d[6 i + j] = pf_cov_diff
extern "C" int hostsim_pf_cov_terms(const float* probs, const PfState* states, size_t n, const float* e_pos, const float* e_rpy,
                                    float* d, float* terms)
{
  for (size_t i = 0; i < n; ++i)
  {
    float* di = d + 6 * i;
    pf_cov_diff(states[i], e_pos, e_rpy, di);
    float* o = terms + 22 * i;
    o[0] = probs[i];
    int t = 1;
    for (int j = 0; j < 6; ++j)
      for (int k = j; k < 6; ++k) o[t++] = __fmul_rn(__fmul_rn(__fmul_rn(1.0f, di[j]), di[k]), probs[i]);
  }
  return 0;
}

// The pose estimate (pf_kernels.cuh: pf_est_pass1/finish1/pass2/finish2) with the device's per-particle functions and
// double sums in particle order (the kernels fold the same double terms with a fixed tree: equal to ~1e-16 relative).
// out: mean_b pos[3] rot[4] | max_index | weight_sum_biased | cov[36]  (45 floats; max_index stored as float bits)
extern "C" int hostsim_pf_estimate(const float* probs, const PfState* states, size_t n, const mcl3dl_pose* prev, float bias_var_dist,
                                   float bias_var_ang, float* mean_pos, float* mean_rot, uint32_t* max_index, float* wsum, float* cov)
{
  const BiasDev b = bias_of(prev, bias_var_dist, bias_var_ang);
  double v[20] = {0};
  float best = -1.0f;
  uint32_t best_i = 0;
  for (size_t i = 0; i < n; ++i)
  {
    const float p = probs[i], w = p * pf_bias(states[i], b);
    float t[9];
    pf_mean_terms(states[i], t);
    v[0] += w;
    v[10] += p;
    for (int k = 0; k < 9; ++k)
    {
      v[1 + k] += static_cast<double>(t[k] * w);
      v[11 + k] += static_cast<double>(t[k] * p);
    }
    if (p > best)
    {
      best = p;
      best_i = static_cast<uint32_t>(i);
    }
  }
  float e_pos[3], e_rpy[3], qu[4];
  for (int a = 0; a < 3; ++a)
  {
    mean_pos[a] = static_cast<float>(v[1 + a] / v[0]);
    e_pos[a] = static_cast<float>(v[11 + a] / v[10]);
  }
  pf_quat_from_front_up(v + 4, v + 7, mean_rot);
  pf_quat_from_front_up(v + 14, v + 17, qu);
  pf_rpy(qu, e_rpy);
  *max_index = best_i;
  *wsum = static_cast<float>(v[0]);
  double c[22] = {0};
  for (size_t i = 0; i < n; ++i)
  {
    float d[6];
    pf_cov_diff(states[i], e_pos, e_rpy, d);
    c[0] += probs[i];
    int t = 1;
    for (int j = 0; j < 6; ++j)
      for (int k = j; k < 6; ++k) c[t++] += static_cast<double>(1.0f * d[j] * d[k] * probs[i]);
  }
  int t = 1;
  for (int j = 0; j < 6; ++j)
    for (int k = j; k < 6; ++k)
    {
      cov[j * 6 + k] = cov[k * 6 + j] = static_cast<float>(c[t] / c[0]);
      ++t;
    }
  return 0;
}
