// landmark_parity_test.cpp — TEST INFRASTRUCTURE ONLY.
//
// The node's landmark sequence on the RESIDENT particle set through the host C++ adapter (ParticleFilterB200) against
// the reference's own particle filter in one process, per cycle:
//   predict (src/mcl_3dl.cpp:227-232) -> cbLandmark (:899-940): pf_->measure with the node's lambda and the reference's
//   own NormalLikelihoodNd<float, 6> (landmarkMeasureResident), then pf_->resample (resampleResident) -> a pose-jump
//   reset (:653-658; resetOdomErrIntegResident) -> the published poses (publishParticles, :1101-1125; posesResident).
// NormalLikelihoodNd is compiled against oracle/shim_nd (a repo-written stand-in, not Eigen) on both sides, so the
// adapter hands the device exactly the a_ and sigma_inv_ the reference filter uses.  Resampling's noise is the
// documented departure that cannot be replayed per output, so after resampling the reference filter takes the device's
// set; the reset and the poses are then compared bit for bit, the landmark posteriors within a bar (the device's
// atan2f / asinf / expf and double sums).
//
//   landmark_parity_test [n_particles] [cycles]
//
// Built where a checkout of the reference exists (make -C oracle -f pf_landmark.mk landmark-parity);
// tests/test_gpu_pf_landmark.py runs it on an H100.
#include <array>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <random>
#include <vector>

#include <mcl_3dl/motion_prediction_models/motion_prediction_model_differential_drive.h>
#include <mcl_3dl/nd.h>
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

// the reference filter takes the device's set (after resampling)
void adopt(PF& ref, PFB& gpu)
{
  auto ir = ref.begin();
  for (auto ig = gpu.begin(); ig != gpu.end(); ++ig, ++ir) *ir = *ig;
}
}  // namespace

int main(int argc, char** argv)
{
  const int n_particles = argc > 1 ? std::atoi(argv[1]) : 300;
  const int cycles = argc > 2 ? std::atoi(argv[2]) : 3;
  std::mt19937 rng(42);
  std::normal_distribution<float> n01(0.f, 1.f);

  auto lik_params = std::make_shared<LidarMeasurementModelLikelihoodParameters>();
  auto beam_params = std::make_shared<LidarMeasurementModelBeamParameters>();
  const float dist_weight[4] = {1.f, 1.f, 5.f, 0.f};
  const uint64_t seed = 0x1a4d0000beefull;

  PF pf_ref(n_particles, 7);
  PFB pf_gpu(n_particles, 7);
  const State6DOF mean(Vec3(2.f, 1.f, 0.3f), Quat(Vec3(0, 0, 1), 0.4f));
  const State6DOF sigma(Vec3(0.3f, 0.3f, 0.05f), Vec3(0.05f, 0.05f, 0.2f));
  pf_ref.init(mean, sigma);
  pf_gpu.init(mean, sigma);
  auto batcher = std::make_shared<mcl_3dl_b200::MeasurementBatcher>(&pf_gpu, std::vector<int>{0}, lik_params, beam_params,
                                                                   dist_weight);
  MotionPredictionModelDifferentialDrive motion(10.0f, 10.0f);
  pf_gpu.uploadResident(*batcher);
  State6DOF odom_prev(Vec3(0.f, 0.f, 0.f), Quat(0.f, 0.f, 0.f, 1.f));
  for (int cycle = 0; cycle < cycles; ++cycle)
  {
    State6DOF odom_cur(odom_prev.pos_ + Vec3(0.05f, 0.01f * cycle, 0.f), Quat(Vec3(0.f, 0.f, 1.f), 0.02f * (cycle + 1)) * odom_prev.rot_);
    motion.setOdoms(odom_prev, odom_cur, 0.1f);
    pf_ref.predict([&motion](State6DOF& s) { motion.predict(s); });
    pf_gpu.predictResident(*batcher, odom_prev, odom_cur, 0.1f, 10.0f, 10.0f);
    odom_prev = odom_cur;
    pf_gpu.downloadResident(*batcher);
    adopt(pf_ref, pf_gpu);  // predict's own parity is tests/test_gpu_pf_exact.py's; start the landmark from equal sets

    // ---- cbLandmark: a detector's pose with an anisotropic, correlated (and, on odd cycles, non-symmetric) covariance
    std::array<double, 36> cov{};
    for (int r = 0; r < 6; ++r)
      for (int c = 0; c < 6; ++c)
        cov[r * 6 + c] = (r == c ? (r < 3 ? 0.09 : 0.04) : 0.004 * std::sin(1.0 + r + 2 * c)) + (cycle % 2 && c > r ? 0.002 : 0.0);
    const Vec3 mpos = mean.pos_ + Vec3(0.1f * n01(rng), 0.1f * n01(rng), 0.02f * n01(rng));
    const Quat mrot = Quat(Vec3(0.f, 0.f, 1.f), 0.4f + 0.05f * n01(rng)) * 1.02f;  // as received: not normalised
    {
      // the node's code (src/mcl_3dl.cpp:901-929), the message's covariance as its array
      NormalLikelihoodNd<float, 6> nd(Eigen::Matrix<double, 6, 6>(cov.data()).cast<float>());
      const State6DOF measured(mpos, mrot);
      const auto measure_func = [&measured, &nd](const State6DOF& s) -> float
      {
        State6DOF diff = s - measured;
        const Vec3 rot_rpy = diff.rot_.getRPY();
        const float x[6] = {diff.pos_.x_, diff.pos_.y_, diff.pos_.z_, rot_rpy.x_, rot_rpy.y_, rot_rpy.z_};
        const Eigen::Matrix<float, 6, 1> diff_vec(x);
        const auto n = nd(diff_vec);
        return n;
      };
      pf_ref.measure(measure_func);
    }
    const auto lm = pf_gpu.landmarkMeasureResident(*batcher, State6DOF(mpos, mrot), cov);
    EXPECT(lm.kept, "landmark update kept (cycle %d)", cycle);
    EXPECT(lm.match_ratio_min == 0.0f && lm.match_ratio_max == 0.0f, "landmark match ratios %g/%g", lm.match_ratio_min,
           lm.match_ratio_max);
    EXPECT(std::fabs(pf_gpu.getEntropy() - pf_ref.getEntropy()) <= 2e-4 * std::fabs(pf_ref.getEntropy()) + 1e-6,
           "landmark entropy %g vs %g (cycle %d)", pf_gpu.getEntropy(), pf_ref.getEntropy(), cycle);
    pf_gpu.downloadResident(*batcher);
    {
      double worst = 0;
      size_t changed = 0;
      auto ig = pf_gpu.begin();
      for (auto ir = pf_ref.begin(); ir != pf_ref.end(); ++ir, ++ig)
      {
        const double rel = std::fabs(ir->probability_ - ig->probability_) / std::max(1e-30, static_cast<double>(ir->probability_));
        if (ir->probability_ > 1e-30f)
          worst = std::max(worst, rel);
        EXPECT(rel <= 2e-4 || std::fabs(ir->probability_ - ig->probability_) <= 1e-30, "landmark posterior %g vs %g (cycle %d)",
               ir->probability_, ig->probability_, cycle);
        const mcl3dl_state a = PFB::toState(ir->state_), b = PFB::toState(ig->state_);
        changed += std::memcmp(&a, &b, sizeof(a)) != 0;
      }
      EXPECT(changed == 0, "landmark update changed %zu states (cycle %d)", changed, cycle);
      std::printf("cycle %d: landmark posterior worst %.3g, entropy %g vs %g\n", cycle, worst, pf_gpu.getEntropy(),
                  pf_ref.getEntropy());
    }

    // ---- cbLandmark's resample; the reference filter takes the device's set (noise stream: the documented departure)
    pf_gpu.resampleResident(*batcher, Vec3(0.05f, 0.05f, 0.05f), Vec3(0.05f, 0.05f, 0.05f), seed + cycle);
    pf_gpu.downloadResident(*batcher);
    adopt(pf_ref, pf_gpu);

    // ---- the pose-jump branch's reset
    const auto integ_reset_func = [](State6DOF& s)
    {
      s.odom_err_integ_lin_ = Vec3();
      s.odom_err_integ_ang_ = Vec3();
    };
    pf_ref.predict(integ_reset_func);
    pf_gpu.resetOdomErrIntegResident(*batcher);
    pf_gpu.downloadResident(*batcher);
    {
      size_t bad = 0;
      auto ig = pf_gpu.begin();
      for (auto ir = pf_ref.begin(); ir != pf_ref.end(); ++ir, ++ig)
      {
        const mcl3dl_state a = PFB::toState(ir->state_), b = PFB::toState(ig->state_);
        bad += std::memcmp(&a, &b, sizeof(a)) != 0 || ir->probability_ != ig->probability_;
      }
      EXPECT(bad == 0, "reset: %zu differences (cycle %d)", bad, cycle);
    }

    // ---- publishParticles: the node's loop on the reference filter vs posesResident
    std::vector<mcl3dl_pose> poses;
    pf_gpu.posesResident(*batcher, poses);
    EXPECT(poses.size() == pf_ref.getParticleSize(), "poses %zu vs %zu", poses.size(), pf_ref.getParticleSize());
    size_t bad = 0;
    for (size_t i = 0; i < pf_ref.getParticleSize() && i < poses.size(); i++)
    {
      auto p = pf_ref.getParticle(i);
      p.rot_.normalize();
      const mcl3dl_pose want{p.pos_.x_, p.pos_.y_, p.pos_.z_, 0.0f, p.rot_.x_, p.rot_.y_, p.rot_.z_, p.rot_.w_};
      bad += std::memcmp(&want, &poses[i], sizeof(want)) != 0;
    }
    EXPECT(bad == 0, "published poses: %zu differences (cycle %d)", bad, cycle);
    std::printf("cycle %d: reset and %zu published poses compared\n", cycle, poses.size());
  }
  if (g_fail)
  {
    std::fprintf(stderr, "LANDMARK PARITY FAILED (%d)\n", g_fail);
    return 1;
  }
  std::printf("LANDMARK PARITY OK (%d cycles)\n", cycles);
  return 0;
}
