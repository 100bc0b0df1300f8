// pf_events_ref_driver.cpp — TEST INFRASTRUCTURE ONLY ("reference" checker of oracle/pf_events_api.h).
//
// The reference's own code, unchanged, on given draws:
//   - the redraw: the node's update_noise_func lambda (src/mcl_3dl.cpp:817-825) through pf::ParticleFilter::predict,
//     with its std::normal_distribution replaced by a replay of the given draws;
//   - expansion resetting: pf::ParticleFilter::addNoiseUsingNoiseGenerator (public, templated on the generator) fed by a
//     generator that replays the given six draws per particle into State6DOF::generateNoise and operator+;
//   - the IMU update: ImuMeasurementModelGravity::setAccMeasure + measure inside pf::ParticleFilter::measure.
#include <ros/ros.h>

#include <cstring>
#include <vector>

#include <mcl_3dl/imu_measurement_models/imu_measurement_model_gravity.h>
#include <mcl_3dl/pf.h>
#include <mcl_3dl/state_6dof.h>

#include "pf_events_api.h"

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

// A noise generator for generateNoise that returns the given draws, six per call, in order (mean 0, dimension 6)
class ReplayNoise : public mcl_3dl::NoiseGeneratorBase<float>
{
public:
  explicit ReplayNoise(const float* org) : org_(org)
  {
    mean_.assign(6, 0.0f);
  }
  template <typename RANDOM_ENGINE>
  std::vector<float> operator()(RANDOM_ENGINE&) const
  {
    std::vector<float> v(org_ + 6 * k_, org_ + 6 * k_ + 6);
    ++k_;
    return v;
  }

private:
  const float* org_;
  mutable size_t k_ = 0;
};
}  // namespace

extern "C" {

const char* mcl3dl_cpu_pf_events_kind(void) { return "reference"; }

int mcl3dl_cpu_pf_redraw(mcl3dl_state* states, size_t n, const float* z, double lin_lin, double lin_ang, double ang_lin,
                         double ang_ang)
{
  if (n == 0)
    return MCL3DL_OK;
  if (!states || !z)
    return MCL3DL_ERR_INVALID_ARG;
  Filter6 pf(static_cast<int>(n), 1);
  load(pf, states, nullptr);
  // the node's lambda with params_.odom_err_* and noise(engine_) replayed from z
  struct
  {
    double odom_err_lin_lin_, odom_err_lin_ang_, odom_err_ang_ang_, odom_err_ang_lin_;
  } params_{lin_lin, lin_ang, ang_ang, ang_lin};
  size_t k = 0;
  const auto noise = [&k, z]() -> float { return z[k++]; };
  const auto update_noise_func = [&params_, &noise](State6DOF& s)
  {
    s.noise_ll_ = noise() * params_.odom_err_lin_lin_;
    s.noise_la_ = noise() * params_.odom_err_lin_ang_;
    s.noise_aa_ = noise() * params_.odom_err_ang_ang_;
    s.noise_al_ = noise() * params_.odom_err_ang_lin_;
  };
  pf.predict(update_noise_func);
  size_t i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i) states[i] = fromState6(it->state_);
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_noise(mcl3dl_state* states, size_t n, const float* org)
{
  if (n == 0)
    return MCL3DL_OK;
  if (!states || !org)
    return MCL3DL_ERR_INVALID_ARG;
  Filter6 pf(static_cast<int>(n), 1);
  load(pf, states, nullptr);
  pf.addNoiseUsingNoiseGenerator(ReplayNoise(org));
  size_t i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i) states[i] = fromState6(it->state_);
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_imu(const mcl3dl_state* states, float* probs, size_t n, const float acc[3], double acc_var, float* lik,
                      int* kept, float* sum_out, float* entropy)
{
  if ((n && (!states || !probs)) || !acc || !kept || !sum_out || !entropy)
    return MCL3DL_ERR_INVALID_ARG;
  Filter6 pf(static_cast<int>(n), 1);
  load(pf, states, probs);
  mcl_3dl::ImuMeasurementModelGravity model(static_cast<float>(acc_var));
  model.setAccMeasure(Vec3(acc[0], acc[1], acc[2]));
  size_t i = 0;
  float sum = 0;
  const auto imu_measure_func = [&](const State6DOF& s) -> float
  {
    const float l = model.measure(s);
    if (lik)
      lik[i] = l;
    sum += probs[i] * l;  // the same float products and running sum pf.h:258-259 forms
    ++i;
    return l;
  };
  pf.measure(imu_measure_func);
  *sum_out = sum;
  *kept = sum > 0.0 ? 1 : 0;
  *entropy = *kept ? pf.getEntropy() : 0.0f;
  i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i) probs[i] = it->probability_;
  return MCL3DL_OK;
}

}  // extern "C"
