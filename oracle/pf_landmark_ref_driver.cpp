// pf_landmark_ref_driver.cpp — TEST INFRASTRUCTURE ONLY ("reference" checker of oracle/pf_landmark_api.h).
//
// The reference's own code, unchanged:
//   - the landmark update: cbLandmark's measure_func (src/mcl_3dl.cpp:913-928) inside pf::ParticleFilter::measure, with
//     the reference's State6DOF::operator-, Quat::inv and Quat::getRPY.  NormalLikelihoodNd itself needs Eigen, which
//     this build does not have, so its operator() (nd.h:76-79) is evaluated from the given a_ and sigma_inv_ in the
//     order include/mcl3dl_b200.h fixes;
//   - the reset: the node's integ_reset_func lambda (src/mcl_3dl.cpp:190-195,653-658) through pf::ParticleFilter::predict;
//   - the poses: publishParticles' loop body (src/mcl_3dl.cpp:1111-1121), getParticle + Quat::normalize on the copy.
#include <ros/ros.h>

#include <vector>

#include <mcl_3dl/pf.h>
#include <mcl_3dl/state_6dof.h>

#include "pf_landmark_api.h"

namespace
{
using mcl_3dl::Quat;
using mcl_3dl::State6DOF;
using mcl_3dl::Vec3;
using Filter6 = mcl_3dl::pf::ParticleFilter<State6DOF, float, mcl_3dl::ParticleWeightedMeanQuat, std::default_random_engine>;

State6DOF toState6(const mcl3dl_state& st)
{
  State6DOF s(Vec3(st.pos[0], st.pos[1], st.pos[2]), Quat(st.rot[0], st.rot[1], st.rot[2], st.rot[3]));
  s.noise_ll_ = st.noise_ll;
  s.noise_la_ = st.noise_la;
  s.noise_al_ = st.noise_al;
  s.noise_aa_ = st.noise_aa;
  s.odom_err_integ_lin_ = Vec3(st.odom_err_integ_lin[0], st.odom_err_integ_lin[1], st.odom_err_integ_lin[2]);
  s.odom_err_integ_ang_ = Vec3(st.odom_err_integ_ang[0], st.odom_err_integ_ang[1], st.odom_err_integ_ang[2]);
  return s;
}

mcl3dl_state fromState6(const State6DOF& s)
{
  mcl3dl_state o;
  o.pos[0] = s.pos_.x_;
  o.pos[1] = s.pos_.y_;
  o.pos[2] = s.pos_.z_;
  o.rot[0] = s.rot_.x_;
  o.rot[1] = s.rot_.y_;
  o.rot[2] = s.rot_.z_;
  o.rot[3] = s.rot_.w_;
  o.noise_ll = s.noise_ll_;
  o.noise_la = s.noise_la_;
  o.noise_al = s.noise_al_;
  o.noise_aa = s.noise_aa_;
  for (int k = 0; k < 3; ++k)
  {
    o.odom_err_integ_lin[k] = s.odom_err_integ_lin_[k];
    o.odom_err_integ_ang[k] = s.odom_err_integ_ang_[k];
  }
  return o;
}

void load(Filter6& pf, const mcl3dl_state* states, const float* probs)
{
  size_t i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i)
  {
    it->state_ = toState6(states[i]);
    it->probability_ = probs ? probs[i] : 1.0f;
  }
}
}  // namespace

extern "C" {

const char* mcl3dl_cpu_pf_landmark_kind(void) { return "reference"; }

int mcl3dl_cpu_pf_landmark(const mcl3dl_state* states, float* probs, size_t n, const float measured_in[7], float nd_a,
                           const float sigma_inv[36], float* lik, int* kept, float* sum_out, float* entropy)
{
  if ((n && (!states || !probs)) || !measured_in || !sigma_inv || !kept || !sum_out || !entropy)
    return MCL3DL_ERR_INVALID_ARG;
  Filter6 pf(static_cast<int>(n), 1);
  load(pf, states, probs);
  const State6DOF measured(Vec3(measured_in[0], measured_in[1], measured_in[2]),
                           Quat(measured_in[3], measured_in[4], measured_in[5], measured_in[6]));
  // NormalLikelihoodNd<float, 6>::operator(): a_ * exp(float(-0.5 x^T sigma_inv_ x)), the product in the documented order
  const auto nd = [nd_a, sigma_inv](const float x[6]) -> float
  {
    float h[6];
    for (int k = 0; k < 6; ++k) h[k] = -0.5f * x[k];
    float q = 0;
    for (int j = 0; j < 6; ++j)
    {
      float r = h[0] * sigma_inv[j];
      for (int k = 1; k < 6; ++k) r = r + h[k] * sigma_inv[k * 6 + j];
      q = j == 0 ? r * x[0] : q + r * x[j];
    }
    return nd_a * std::exp(static_cast<float>(q));
  };
  size_t i = 0;
  float sum = 0;
  const auto measure_func = [&](const State6DOF& s) -> float
  {
    State6DOF diff = s - measured;
    const Vec3 rot_rpy = diff.rot_.getRPY();
    const float diff_vec[6] = {diff.pos_.x_, diff.pos_.y_, diff.pos_.z_, rot_rpy.x_, rot_rpy.y_, rot_rpy.z_};
    const float l = nd(diff_vec);
    if (lik)
      lik[i] = l;
    sum += probs[i] * l;  // the same float products and running sum pf.h:258-259 forms
    ++i;
    return l;
  };
  pf.measure(measure_func);
  *sum_out = sum;
  *kept = sum > 0.0 ? 1 : 0;
  *entropy = *kept ? pf.getEntropy() : 0.0f;
  i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i) probs[i] = it->probability_;
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_reset_odom_err(mcl3dl_state* states, size_t n)
{
  if (n == 0)
    return MCL3DL_OK;
  if (!states)
    return MCL3DL_ERR_INVALID_ARG;
  Filter6 pf(static_cast<int>(n), 1);
  load(pf, states, nullptr);
  const auto integ_reset_func = [](State6DOF& s)
  {
    s.odom_err_integ_lin_ = Vec3();
    s.odom_err_integ_ang_ = Vec3();
  };
  pf.predict(integ_reset_func);
  size_t i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i) states[i] = fromState6(it->state_);
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_poses(const mcl3dl_state* states, size_t n, mcl3dl_pose* out)
{
  if (n == 0)
    return MCL3DL_OK;
  if (!states || !out)
    return MCL3DL_ERR_INVALID_ARG;
  Filter6 pf(static_cast<int>(n), 1);
  load(pf, states, nullptr);
  for (size_t i = 0; i < pf.getParticleSize(); i++)
  {
    auto p = pf.getParticle(i);
    p.rot_.normalize();
    out[i] = mcl3dl_pose{p.pos_.x_, p.pos_.y_, p.pos_.z_, 0.0f, p.rot_.x_, p.rot_.y_, p.rot_.z_, p.rot_.w_};
  }
  return MCL3DL_OK;
}

}  // extern "C"
