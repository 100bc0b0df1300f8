// pf_init_ref_driver.cpp — TEST INFRASTRUCTURE ONLY ("reference" checker of oracle/pf_init_api.h).
//
// The reference's own code, unchanged: pf::ParticleFilter::initUsingNoiseGenerator, State6DOF::generateNoise,
// NoiseGeneratorBase<float>::setMean (Quat::getRPY), Quat(Vec3 rpy) and MultivariateNoiseGenerator<float> (its
// constructor, setCovariance and the members operator() evaluates).  The draws are replayed: std::normal_distribution's
// stream is the documented departure, so
//   - the diagonal tier is a NoiseGeneratorBase<float> subclass with the reference's mean (setMean) that applies
//     DiagonalNoiseGenerator::operator()'s rule (diagonal_noise_generator.h:63-78) to given standard normals:
//     sigma == 0 ? mean : z * sigma + mean (libstdc++'s normal_distribution<float>: z * stddev + mean);
//   - the multivariate tier is a MultivariateNoiseGenerator<float> subclass whose operator() evaluates the reference's
//     own mean_vec_ + norm_transform_ * random on given z.
// MultivariateNoiseGenerator needs Eigen: it is compiled against oracle/shim_mv (repo-written, not Eigen).
#include <ros/ros.h>

#include <array>
#include <vector>

#include <mcl_3dl/noise_generator_base.h>
#include <mcl_3dl/noise_generators/multivariate_noise_generator.h>
#include <mcl_3dl/pf.h>
#include <mcl_3dl/state_6dof.h>

#include "pf_init_api.h"

namespace
{
using mcl_3dl::Quat;
using mcl_3dl::State6DOF;
using mcl_3dl::Vec3;
using Filter6 = mcl_3dl::pf::ParticleFilter<State6DOF, float, mcl_3dl::ParticleWeightedMeanQuat, std::default_random_engine>;

State6DOF meanState(const float p[7])
{
  return State6DOF(Vec3(p[0], p[1], p[2]), Quat(p[3], p[4], p[5], p[6]));
}

class ReplayDiagonal : public mcl_3dl::NoiseGeneratorBase<float>
{
public:
  ReplayDiagonal(const State6DOF& mean, const float sigma[6], const float* z) : sigma_(sigma), z_(z)
  {
    setMean(mean);
  }
  template <typename RANDOM_ENGINE>
  std::vector<float> operator()(RANDOM_ENGINE&) const
  {
    std::vector<float> noise(6);
    for (size_t i = 0; i < 6; i++)
    {
      if (sigma_[i] == 0)
      {
        noise[i] = mean_[i];
        continue;
      }
      noise[i] = z_[6 * k_ + i] * sigma_[i] + mean_[i];
    }
    ++k_;
    return noise;
  }

private:
  const float* sigma_;
  const float* z_;
  mutable size_t k_ = 0;
};

class ReplayMultivariate : public mcl_3dl::MultivariateNoiseGenerator<float>
{
public:
  using Base = mcl_3dl::MultivariateNoiseGenerator<float>;
  // the reference's constructor on a covariance; norm_transform_ is then the given T when there is one
  ReplayMultivariate(const State6DOF& mean, const std::array<double, 36>& cov, const float* T, const float* z)
    : Base(mean, cov), z_(z)
  {
    if (T)
      for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) norm_transform_(r, c) = T[r * 6 + c];
  }
  template <typename RANDOM_ENGINE>
  std::vector<float> operator()(RANDOM_ENGINE&) const
  {
    Vector random(6);
    for (size_t j = 0; j < 6; ++j) random[j] = z_[6 * k_ + j];
    ++k_;
    const Vector sample_noise = mean_vec_ + norm_transform_ * random;
    return std::vector<float>(sample_noise.data(), sample_noise.data() + 6);
  }
  void transform(float T[36]) const
  {
    for (int r = 0; r < 6; ++r)
      for (int c = 0; c < 6; ++c) T[r * 6 + c] = norm_transform_(r, c);
  }

private:
  const float* z_;
  mutable size_t k_ = 0;
};

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
}  // namespace

extern "C" {

const char* mcl3dl_cpu_pf_init_kind(void) { return "reference"; }

int mcl3dl_cpu_pf_init_mean(const float pose7[7], float mean6[6])
{
  if (!pose7 || !mean6)
    return MCL3DL_ERR_INVALID_ARG;
  mcl_3dl::NoiseGeneratorBase<float> base;
  base.setMean(meanState(pose7));
  for (int k = 0; k < 6; ++k) mean6[k] = base.getMean()[k];
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_init(size_t n, int multivariate, const float pose7[7], const float sigma6[6], const float T[36],
                       const float* z, mcl3dl_state* states, float* probs)
{
  if (!pose7 || n == 0 || !z || !states || !probs || (multivariate ? !T : !sigma6))
    return MCL3DL_ERR_INVALID_ARG;
  Filter6 pf(static_cast<int>(n), 1);
  if (multivariate)
    pf.initUsingNoiseGenerator(ReplayMultivariate(meanState(pose7), std::array<double, 36>{}, T, z));
  else
    pf.initUsingNoiseGenerator(ReplayDiagonal(meanState(pose7), sigma6, z));
  size_t i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i)
  {
    states[i] = fromState6(it->state_);
    probs[i] = it->probability_;
  }
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_init_transform(const double covariance[36], float T[36])
{
  if (!covariance || !T)
    return MCL3DL_ERR_INVALID_ARG;
  std::array<double, 36> cov;
  for (int k = 0; k < 36; ++k) cov[k] = covariance[k];
  const float pose7[7] = {0, 0, 0, 0, 0, 0, 1};
  ReplayMultivariate(meanState(pose7), cov, nullptr, nullptr).transform(T);
  return MCL3DL_OK;
}

}  // extern "C"
