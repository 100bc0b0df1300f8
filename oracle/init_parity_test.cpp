// init_parity_test.cpp — TEST INFRASTRUCTURE ONLY.
//
// The node's initial seeds on the RESIDENT particle set through the host C++ adapter (ParticleFilterB200) against the
// reference's own particle filter in one process:
//   the configured start (MCL3dlNode::configure, src/mcl_3dl.cpp:1276: pf_->init(initial_pose, initial_pose_std);
//   initResident, placed after the batcher exists) ->
//   cbPosition (:155-198: initUsingNoiseGenerator(MultivariateNoiseGenerator<float>(mean, covariance)), the integral
//   reset and the published poses; initUsingCovarianceResident, resetOdomErrIntegResident, posesResident) ->
//   a predict / measure (cbLandmark's pf_->measure) / resample cycle on the seeded set ->
//   a seed after the set was resized (the count is particles_.size()) and a covariance the adapter refuses.
// The reference filter gets the device's draws recomputed on the host from include/mcl3dl_b200.h's layout (Philox,
// Box-Muller with glibc's logf / cosf / sinf) through replay generators: the diagonal rule on given normals, and the
// reference's own MultivariateNoiseGenerator<float> whose operator() evaluates mean_vec_ + norm_transform_ * z.  The
// device's logf / cosf / sinf are a few ulp from glibc's, so states agree within a bar; probabilities are exact.
// MultivariateNoiseGenerator and NormalLikelihoodNd are compiled against oracle/shim_mv (repo-written, not Eigen) on both
// sides, so the adapter hands the device exactly the mean_vec_ and norm_transform_ the reference filter uses.
//
//   init_parity_test [n_particles]
//
// Built where a checkout of the reference exists (make -C oracle -f pf_init.mk init-parity); tests/test_gpu_pf_init.py
// runs it on an H100.
#include <array>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>

#include <mcl_3dl/motion_prediction_models/motion_prediction_model_differential_drive.h>
#include <mcl_3dl/nd.h>
#include <mcl_3dl/noise_generator_base.h>
#include <mcl_3dl/noise_generators/multivariate_noise_generator.h>
#include <mcl_3dl/pf.h>
#include <mcl_3dl/state_6dof.h>

#include "../mcl_3dl_b200/host/lidar_measurement_model_b200.h"

using namespace mcl_3dl;
using PF = mcl_3dl_b200::ParticleFilter;
using PFB = mcl_3dl_b200::ParticleFilterB200;

namespace
{
int g_fail = 0;
#define EXPECT(cond, ...)                         \
  do                                              \
  {                                               \
    if (!(cond))                                  \
    {                                             \
      ++g_fail;                                   \
      if (g_fail < 20)                            \
      {                                           \
        std::fprintf(stderr, "FAIL %s: ", #cond); \
        std::fprintf(stderr, __VA_ARGS__);        \
        std::fprintf(stderr, "\n");               \
      }                                           \
    }                                             \
  } while (0)

// ---- the draws, from include/mcl3dl_b200.h's layout (plain host arithmetic; glibc's logf / cosf / sinf)
void philox(uint32_t c[4], uint64_t seed)
{
  uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
  for (int r = 0; r < 10; ++r)
  {
    const uint64_t p0 = uint64_t(0xD2511F53u) * c[0], p1 = uint64_t(0xCD9E8D57u) * c[2];
    const uint32_t n0 = static_cast<uint32_t>(p1 >> 32) ^ c[1] ^ k0, n1 = static_cast<uint32_t>(p1);
    const uint32_t n2 = static_cast<uint32_t>(p0 >> 32) ^ c[3] ^ k1, n3 = static_cast<uint32_t>(p0);
    c[0] = n0;
    c[1] = n1;
    c[2] = n2;
    c[3] = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
}
float uniform(uint32_t w) { return static_cast<float>((w >> 8) + 1) * 5.9604644775390625e-08f; }
void boxMuller(uint32_t u, uint32_t v, float* z)
{
  const float rad = std::sqrt(-2.0f * std::log(uniform(u)));
  const float phi = 6.283185307179586f * uniform(v);
  z[0] = rad * std::cos(phi);
  z[1] = rad * std::sin(phi);
}
// event 3: the six standard normals of particle i of init call `call`, for n particles
std::vector<float> initDraws(uint64_t seed, uint32_t call, size_t n)
{
  std::vector<float> z(6 * n);
  for (uint32_t i = 0; i < n; ++i)
  {
    uint32_t a[4] = {i, call, 0u, 3u}, b[4] = {i, call, 1u, 3u};
    philox(a, seed);
    philox(b, seed);
    boxMuller(a[0], a[1], &z[6 * i]);
    boxMuller(a[2], a[3], &z[6 * i + 2]);
    boxMuller(b[0], b[1], &z[6 * i + 4]);
  }
  return z;
}

// DiagonalNoiseGenerator's rule (diagonal_noise_generator.h:63-78) on given standard normals
class ReplayDiagonal : public NoiseGeneratorBase<float>
{
public:
  ReplayDiagonal(const State6DOF& mean, const State6DOF& sigma, const std::vector<float>& z) : z_(z)
  {
    setMean(mean);
    const DiagonalNoiseGenerator<float> gen(mean, sigma);
    struct Access : DiagonalNoiseGenerator<float>
    {
      static const std::vector<float>& sigma(const DiagonalNoiseGenerator<float>& g) { return g.*(&Access::sigma_); }
    };
    sigma_ = Access::sigma(gen);
  }
  template <typename RANDOM_ENGINE>
  std::vector<float> operator()(RANDOM_ENGINE&) const
  {
    std::vector<float> noise(6);
    for (size_t i = 0; i < 6; i++)
      noise[i] = sigma_[i] == 0 ? mean_[i] : z_[6 * k_ + i] * sigma_[i] + mean_[i];
    ++k_;
    return noise;
  }

private:
  std::vector<float> sigma_;
  const std::vector<float>& z_;
  mutable size_t k_ = 0;
};

// the node's MultivariateNoiseGenerator<float>(mean, covariance), its operator() on given standard normals
class ReplayMultivariate : public MultivariateNoiseGenerator<float>
{
public:
  ReplayMultivariate(const State6DOF& mean, const std::array<double, 36>& cov, const std::vector<float>& z)
    : MultivariateNoiseGenerator<float>(mean, cov), z_(z)
  {
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

private:
  const std::vector<float>& z_;
  mutable size_t k_ = 0;
};

// states within a bar (the device's logf / cosf / sinf), probabilities exact
void compare(const char* what, PF& ref, PFB& gpu, double bar)
{
  EXPECT(ref.getParticleSize() == gpu.getParticleSize(), "%s: %zu vs %zu particles", what, ref.getParticleSize(),
         gpu.getParticleSize());
  double worst = 0;
  size_t bad = 0;
  auto ig = gpu.begin();
  for (auto ir = ref.begin(); ir != ref.end() && ig != gpu.end(); ++ir, ++ig)
  {
    const mcl3dl_state a = PFB::toState(ir->state_), b = PFB::toState(ig->state_);
    const float* fa = &a.pos[0];
    const float* fb = &b.pos[0];
    for (size_t k = 0; k < sizeof(a) / 4; ++k)
    {
      const double d = std::fabs(static_cast<double>(fa[k]) - fb[k]) / std::max(1.0, std::fabs(static_cast<double>(fa[k])));
      worst = std::max(worst, d);
      bad += !(d <= bar);
    }
    bad += ir->probability_ != ig->probability_;
  }
  EXPECT(bad == 0, "%s: %zu differences (worst %.3g)", what, bad, worst);
  std::printf("%s: %zu particles, worst relative difference %.3g\n", what, ref.getParticleSize(), worst);
}

void adopt(PF& ref, PFB& gpu)
{
  auto ir = ref.begin();
  for (auto ig = gpu.begin(); ig != gpu.end(); ++ig, ++ir) *ir = *ig;
}
}  // namespace

int main(int argc, char** argv)
{
  const int n_particles = argc > 1 ? std::atoi(argv[1]) : 500;
  constexpr double kBar = 4e-5;   // a few ulp of logf / cosf / sinf through z * sigma (or T z) + mean and setRPY
  auto lik_params = std::make_shared<LidarMeasurementModelLikelihoodParameters>();
  auto beam_params = std::make_shared<LidarMeasurementModelBeamParameters>();
  const float dist_weight[4] = {1.f, 1.f, 5.f, 0.f};
  const uint64_t seed = 0x1a4d0000c0ffeeull;

  PF pf_ref(n_particles, 7);
  PFB pf_gpu(n_particles, 7);
  auto batcher = std::make_shared<mcl_3dl_b200::MeasurementBatcher>(&pf_gpu, std::vector<int>{0}, lik_params, beam_params,
                                                                   dist_weight);

  // ---- configure (:1276): pf_->init(initial_pose, initial_pose_std), a zero sigma included
  const State6DOF initial_pose(Vec3(2.f, 1.f, 0.3f), Quat(Vec3(0.05f, -0.02f, 0.4f)));
  const State6DOF initial_pose_std(Vec3(0.5f, 0.5f, 0.0f), Vec3(0.0f, 0.0f, 0.2f));
  pf_gpu.initResident(*batcher, initial_pose, initial_pose_std, seed);
  {
    const std::vector<float> z = initDraws(seed, 1, n_particles);
    pf_ref.initUsingNoiseGenerator(ReplayDiagonal(initial_pose, initial_pose_std, z));
  }
  pf_gpu.downloadResident(*batcher);
  compare("configured start", pf_ref, pf_gpu, kBar);

  // ---- cbPosition (:184-197), after the quaternion check and the tf transform, which stay node code
  std::array<double, 36> covariance{};
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c)
      covariance[r * 6 + c] = r == c ? (r < 3 ? 0.2 : 0.05) : (c < r ? 0.01 * std::sin(1.0 + r + 2 * c) : 7.0);  // upper ignored
  const State6DOF mean(Vec3(-1.f, 3.f, 0.1f), Quat(0.f, 0.f, std::sin(1.2f), std::cos(1.2f)));
  EXPECT(pf_gpu.initUsingCovarianceResident(*batcher, mean, covariance, seed + 1), "initUsingCovarianceResident refused");
  {
    const std::vector<float> z = initDraws(seed + 1, 2, n_particles);
    pf_ref.initUsingNoiseGenerator(ReplayMultivariate(mean, covariance, z));
  }
  const auto integ_reset_func = [](State6DOF& s)
  {
    s.odom_err_integ_lin_ = Vec3();
    s.odom_err_integ_ang_ = Vec3();
  };
  pf_ref.predict(integ_reset_func);
  pf_gpu.resetOdomErrIntegResident(*batcher);
  std::vector<mcl3dl_pose> poses;
  pf_gpu.posesResident(*batcher, poses);  // publishParticles()
  {
    size_t bad = 0;
    for (size_t i = 0; i < pf_ref.getParticleSize() && i < poses.size(); i++)
    {
      auto p = pf_ref.getParticle(i);
      p.rot_.normalize();
      const float want[8] = {p.pos_.x_, p.pos_.y_, p.pos_.z_, 0.0f, p.rot_.x_, p.rot_.y_, p.rot_.z_, p.rot_.w_};
      const float* got = &poses[i].px;
      for (int k = 0; k < 8; ++k) bad += !(std::fabs(want[k] - got[k]) <= kBar * std::max(1.0f, std::fabs(want[k])));
    }
    EXPECT(poses.size() == pf_ref.getParticleSize() && bad == 0, "cbPosition poses: %zu differences", bad);
  }
  pf_gpu.downloadResident(*batcher);
  compare("cbPosition", pf_ref, pf_gpu, kBar);

  // ---- a predict / measure / resample cycle on the seeded set
  adopt(pf_ref, pf_gpu);  // from here on both start from the device's bytes
  MotionPredictionModelDifferentialDrive motion(10.0f, 10.0f);
  const State6DOF odom_prev(Vec3(0.f, 0.f, 0.f), Quat(0.f, 0.f, 0.f, 1.f));
  const State6DOF odom_cur(Vec3(0.1f, 0.02f, 0.f), Quat(Vec3(0.f, 0.f, 1.f), 0.03f));
  motion.setOdoms(odom_prev, odom_cur, 0.1f);
  pf_ref.predict([&motion](State6DOF& s) { motion.predict(s); });
  pf_gpu.predictResident(*batcher, odom_prev, odom_cur, 0.1f, 10.0f, 10.0f);
  pf_gpu.downloadResident(*batcher);
  compare("predict after cbPosition", pf_ref, pf_gpu, kBar);
  adopt(pf_ref, pf_gpu);
  std::array<double, 36> lcov{};
  for (int k = 0; k < 6; ++k) lcov[k * 7] = k < 3 ? 0.5 : 0.3;
  const State6DOF measured(Vec3(-0.9f, 3.1f, 0.1f), Quat(Vec3(0.f, 0.f, 1.f), 1.2f * 2.f));
  {
    NormalLikelihoodNd<float, 6> nd(Eigen::Matrix<double, 6, 6>(lcov.data()).cast<float>());
    pf_ref.measure([&measured, &nd](const State6DOF& s) -> float
                   {
                     State6DOF diff = s - measured;
                     const Vec3 rot_rpy = diff.rot_.getRPY();
                     const float x[6] = {diff.pos_.x_, diff.pos_.y_, diff.pos_.z_, rot_rpy.x_, rot_rpy.y_, rot_rpy.z_};
                     return nd(Eigen::Matrix<float, 6, 1>(x));
                   });
  }
  const auto lm = pf_gpu.landmarkMeasureResident(*batcher, measured, lcov);
  EXPECT(lm.kept, "measure after cbPosition not kept");
  pf_gpu.downloadResident(*batcher);
  {
    size_t bad = 0;
    auto ig = pf_gpu.begin();
    for (auto ir = pf_ref.begin(); ir != pf_ref.end(); ++ir, ++ig)
      bad += !(std::fabs(ir->probability_ - ig->probability_) <= 2e-4 * ir->probability_ + 1e-30);
    EXPECT(bad == 0, "measure after cbPosition: %zu posteriors differ", bad);
  }
  pf_gpu.resampleResident(*batcher, Vec3(0.05f, 0.05f, 0.05f), Vec3(0.05f, 0.05f, 0.05f), seed + 2);
  pf_gpu.downloadResident(*batcher);
  {
    size_t bad = 0;
    for (auto ig = pf_gpu.begin(); ig != pf_gpu.end(); ++ig)
      bad += ig->probability_ != static_cast<float>(1.0 / pf_gpu.getParticleSize()) || !std::isfinite(ig->state_.pos_.x_);
    EXPECT(bad == 0, "resample after cbPosition: %zu bad particles", bad);
  }

  // ---- a seed after the set was enlarged (global localisation / resize): the count is particles_.size()
  pf_gpu.resizeResident(*batcher, 2 * n_particles);
  EXPECT(pf_gpu.initUsingCovarianceResident(*batcher, mean, covariance, seed + 3), "seed of the enlarged set refused");
  pf_gpu.downloadResident(*batcher);
  EXPECT(pf_gpu.getParticleSize() == static_cast<size_t>(2 * n_particles), "enlarged seed: %zu particles",
         pf_gpu.getParticleSize());
  {
    PF big(2 * n_particles, 7);
    const std::vector<float> z = initDraws(seed + 3, 3, 2 * n_particles);
    big.initUsingNoiseGenerator(ReplayMultivariate(mean, covariance, z));
    compare("cbPosition on the enlarged set", big, pf_gpu, kBar);
  }

  // ---- a covariance with a negative eigenvalue: refused, the set as it was
  std::array<double, 36> bad_cov{};
  for (int k = 0; k < 6; ++k) bad_cov[k * 7] = k == 4 ? -0.1 : 0.1;
  std::vector<mcl3dl_state> before(pf_gpu.getParticleSize()), after(pf_gpu.getParticleSize());
  {
    size_t i = 0;
    for (auto ig = pf_gpu.begin(); ig != pf_gpu.end(); ++ig) before[i++] = PFB::toState(ig->state_);
  }
  EXPECT(!pf_gpu.initUsingCovarianceResident(*batcher, mean, bad_cov, seed + 4), "a negative eigenvalue was accepted");
  pf_gpu.downloadResident(*batcher);
  {
    size_t i = 0;
    for (auto ig = pf_gpu.begin(); ig != pf_gpu.end(); ++ig) after[i++] = PFB::toState(ig->state_);
  }
  EXPECT(std::memcmp(before.data(), after.data(), before.size() * sizeof(mcl3dl_state)) == 0, "a refused seed changed the set");

  if (g_fail)
  {
    std::fprintf(stderr, "INIT PARITY FAILED (%d)\n", g_fail);
    return 1;
  }
  std::printf("INIT PARITY OK (%d particles)\n", n_particles);
  return 0;
}
