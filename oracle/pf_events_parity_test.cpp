// pf_events_parity_test.cpp — TEST INFRASTRUCTURE ONLY.
//
// The node's loop on the RESIDENT particle set through the host C++ adapter (ParticleFilterB200) against the
// reference's own particle filter in one process, with the three per-particle events that run between and after the
// clouds:
//   predict (src/mcl_3dl.cpp:227-232) -> IMU gravity update between clouds (cbImu, :1003-1008; imuMeasureResident)
//   -> the LIDAR update (:398-426) -> resample (:809-815) -> the odometry-noise redraw (:817-825; redrawOdomNoiseResident)
//   -> expansion resetting when match_ratio_max < match_ratio_thresh (:853-864; noiseResident).
// The reference filter gets the device's draws, recomputed here on the host from the counter layout that
// include/mcl3dl_b200.h documents (Philox-4x32-10, Box-Muller): the redraw runs the node's lambda through pf_->predict
// with its std::normal_distribution replayed from those draws, expansion resetting runs
// pf::ParticleFilter::addNoiseUsingNoiseGenerator (what pf_->noise calls) with a generator that replays them, and the IMU
// update is ImuMeasurementModelGravity inside pf_->measure.  Resampling's noise is the one documented departure that
// cannot be replayed per output, so after resampling the reference filter takes the device's set; the device set itself
// stays resident for the whole run.  The device evaluates logf / sinf / cosf / acosf / expf with its own code, so states
// and posteriors are compared within bars (tests/test_gpu_pf_events.py derives them), not bit for bit.
//
//   pf_events_parity_test [n_particles] [match_ratio_thresh] [cycles]
//
// Built where a checkout of the reference exists (make -C oracle -f pf_events.mk pf-events-parity);
// tests/test_gpu_pf_events.py runs it on an H100.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <random>
#include <string>
#include <vector>

#include <mcl_3dl/chunked_kdtree.h>
#include <mcl_3dl/imu_measurement_models/imu_measurement_model_gravity.h>
#include <mcl_3dl/lidar_measurement_models/lidar_measurement_model_beam.h>
#include <mcl_3dl/lidar_measurement_models/lidar_measurement_model_likelihood.h>
#include <mcl_3dl/motion_prediction_models/motion_prediction_model_differential_drive.h>
#include <mcl_3dl/nd.h>
#include <mcl_3dl/noise_generator_base.h>
#include <mcl_3dl/pf.h>
#include <mcl_3dl/point_cloud_random_sampler.h>
#include <mcl_3dl/state_6dof.h>

#include "../mcl_3dl_b200/host/lidar_measurement_model_b200.h"

using namespace mcl_3dl;
using PointType = LidarMeasurementModelBase::PointType;
using Cloud = pcl::PointCloud<PointType>;
using PF = mcl_3dl_b200::ParticleFilter;
using PFB = mcl_3dl_b200::ParticleFilterB200;

namespace
{
class HeadSampler : public PointCloudRandomSampler<PointType>
{
public:
  Cloud::Ptr sample(const Cloud::ConstPtr& pc, const size_t num) const final
  {
    Cloud::Ptr out(new Cloud);
    out->header = pc->header;
    for (size_t i = 0; i < pc->points.size() && i < num; ++i) out->push_back(pc->points[i]);
    return out;
  }
};

class XyzRep : public pcl::PointRepresentation<PointType>
{
public:
  XyzRep()
  {
    nr_dimensions_ = 3;
    trivial_ = true;
  }
  void copyToFloatArray(const PointType& p, float* out) const override
  {
    out[0] = p.x;
    out[1] = p.y;
    out[2] = p.z;
  }
};

PointType pt(float x, float y, float z, uint32_t label = 0)
{
  PointType p;
  p.x = x;
  p.y = y;
  p.z = z;
  p.label = label;
  return p;
}

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
// event 1: z0..z3 of particle i, call `call`
void redrawDraws(uint64_t seed, uint32_t i, uint32_t call, float* z)
{
  uint32_t c[4] = {i, call, 0u, 1u};
  philox(c, seed);
  boxMuller(c[0], c[1], z);
  boxMuller(c[2], c[3], z + 2);
}
// event 2: the six draws (x y z roll pitch yaw) times sigma, 0 where sigma is 0
void expansionDraws(uint64_t seed, uint32_t i, uint32_t call, const float sigma[6], float* org)
{
  uint32_t a[4] = {i, call, 0u, 2u}, b[4] = {i, call, 1u, 2u};
  philox(a, seed);
  philox(b, seed);
  float z[6];
  boxMuller(a[0], a[1], z);
  boxMuller(a[2], a[3], z + 2);
  boxMuller(b[0], b[1], z + 4);
  for (int k = 0; k < 6; ++k) org[k] = sigma[k] == 0 ? 0.0f : z[k] * sigma[k];
}

// generateNoise's generator, replaying six given draws per particle in particle order
class ReplayNoise : public NoiseGeneratorBase<float>
{
public:
  explicit ReplayNoise(const std::vector<float>& org) : org_(org)
  {
    mean_.assign(6, 0.0f);
  }
  template <typename RANDOM_ENGINE>
  std::vector<float> operator()(RANDOM_ENGINE&) const
  {
    std::vector<float> v(org_.begin() + 6 * k_, org_.begin() + 6 * k_ + 6);
    ++k_;
    return v;
  }

private:
  const std::vector<float>& org_;
  mutable size_t k_ = 0;
};

constexpr double kOrgRel = 7.0 / 8388608.0;   // ORG_REL of tests/test_gpu_pf_exact.py: logf, cosf / sinf, two products
constexpr double kRotRel = 60.0 / 8388608.0;  // its RESAMPLE_ROT_BAR, which also bounds the un-normalised noise rotation

double ulpOf(float v) { return std::nextafter(std::fabs(v), INFINITY) - std::fabs(v); }

// the reference filter takes the device's set (after resampling, and to drop ulp-level drift at the end of a cycle)
void adopt(PF& ref, PFB& gpu)
{
  auto ir = ref.begin();
  for (auto ig = gpu.begin(); ig != gpu.end(); ++ig, ++ir) *ir = *ig;
}
}  // namespace

int main(int argc, char** argv)
{
  const int n_particles = argc > 1 ? std::atoi(argv[1]) : 300;
  const double match_ratio_thresh = argc > 2 ? std::atof(argv[2]) : 0.0;
  const int cycles = argc > 3 ? std::atoi(argv[3]) : 4;
  std::mt19937 rng(42);
  std::normal_distribution<float> n01(0.f, 1.f);

  // ---- map: 12 x 12 m floor, two walls, a box side (the scene of adapter_parity_test.cpp)
  Cloud::Ptr map(new Cloud);
  for (float x = 0.05f; x < 12.f; x += 0.1f)
    for (float y = 0.05f; y < 12.f; y += 0.1f)
      map->push_back(pt(x + 0.02f * n01(rng), y + 0.02f * n01(rng), 0.03f + 0.01f * n01(rng)));
  for (float y = 0.05f; y < 12.f; y += 0.1f)
    for (float z = 0.05f; z < 3.f; z += 0.1f)
    {
      map->push_back(pt(0.03f + 0.01f * n01(rng), y, z));
      map->push_back(pt(11.97f + 0.01f * n01(rng), y, z));
    }
  for (float x = 4.f; x < 6.f; x += 0.1f)
    for (float z = 0.05f; z < 2.f; z += 0.1f)
      map->push_back(pt(x, 7.03f + 0.01f * n01(rng), z));
  map->header.stamp = 1234;
  const float dist_weight[4] = {1.f, 1.f, 5.f, 0.f};
  auto rep = std::make_shared<XyzRep>();
  rep->setRescaleValues(dist_weight);
  ChunkedKdtree<PointType>::Ptr kdtree(new ChunkedKdtree<PointType>(20.0, 0.4));
  kdtree->setPointRepresentation(rep);
  kdtree->setInputCloud(map);

  auto lik_params = std::make_shared<LidarMeasurementModelLikelihoodParameters>();
  lik_params->num_points_default_ = 96;
  auto beam_params = std::make_shared<LidarMeasurementModelBeamParameters>();
  beam_params->num_points_default_ = 12;
  beam_params->use_raycast_using_dda_ = true;

  const Vec3 truth_pos(6.f, 4.f, 0.5f);
  const Quat truth_rot(Vec3(0, 0, 1), 0.3f);
  Cloud::Ptr scan(new Cloud);
  std::uniform_int_distribution<size_t> pick(0, map->size() - 1);
  while (scan->size() < 400)
  {
    const PointType& mp = map->points[pick(rng)];
    const Vec3 local = truth_rot.inv() * (Vec3(mp.x, mp.y, mp.z) - truth_pos);
    scan->push_back(pt(local.x_ + 0.02f * n01(rng), local.y_ + 0.02f * n01(rng), local.z_ + 0.02f * n01(rng), scan->size() % 2));
  }
  const std::vector<Vec3> origins = {Vec3(0.f, 0.f, 0.3f), Vec3(0.2f, -0.1f, 0.25f)};
  const HeadSampler sampler;

  // ---- the node's parameters (src/parameters.cpp defaults, except match_ratio_thresh from the command line)
  const double odom_err_lin_lin = 0.10, odom_err_lin_ang = 0.05, odom_err_ang_lin = 0.05, odom_err_ang_ang = 0.05;
  const Vec3 expansion_pos(0.2f, 0.2f, 0.2f), expansion_rpy(0.05f, 0.05f, 0.05f);
  const double acc_var = M_PI / 4.0;
  const float odom_err_integ_lin_sigma = 100.0f;
  const uint64_t seed = 0x5eed0000cafeull;

  PF pf_ref(n_particles, 7);
  PFB pf_gpu(n_particles, 7);
  const State6DOF mean(truth_pos, truth_rot);
  const State6DOF sigma(Vec3(0.2f, 0.2f, 0.05f), Vec3(0.02f, 0.02f, 0.1f));
  pf_ref.init(mean, sigma);
  pf_gpu.init(mean, sigma);
  auto batcher = std::make_shared<mcl_3dl_b200::MeasurementBatcher>(&pf_gpu, std::vector<int>{0}, lik_params, beam_params,
                                                                   dist_weight);
  std::map<std::string, LidarMeasurementModelBase::Ptr> lm;
  lm["likelihood"] = std::make_shared<LidarMeasurementModelLikelihood>(lik_params);
  lm["beam"] = std::make_shared<LidarMeasurementModelBeam>(beam_params);
  ImuMeasurementModelGravity imu_model(acc_var);  // the node's model, constructed once (src/mcl_3dl.cpp:1310)
  MotionPredictionModelDifferentialDrive motion(10.0f, 10.0f);
  NormalLikelihood<float> odom_nd(odom_err_integ_lin_sigma);

  pf_gpu.uploadResident(*batcher);  // after init(): from here on the device set stays resident
  State6DOF odom_prev(Vec3(0.f, 0.f, 0.f), Quat(0.f, 0.f, 0.f, 1.f));
  uint32_t redraw_calls = 0, noise_calls = 0;
  int resets = 0;
  for (int cycle = 0; cycle < cycles; ++cycle)
  {
    // predict: pos and rot per particle
    State6DOF odom_cur(odom_prev.pos_ + Vec3(0.05f, 0.01f * cycle, 0.f), Quat(Vec3(0.f, 0.f, 1.f), 0.02f * (cycle + 1)) * odom_prev.rot_);
    motion.setOdoms(odom_prev, odom_cur, 0.1f);
    pf_ref.predict([&motion](State6DOF& s) { motion.predict(s); });
    pf_gpu.predictResident(*batcher, odom_prev, odom_cur, 0.1f, 10.0f, 10.0f);
    odom_prev = odom_cur;

    // IMU gravity update between clouds: a tilted, normalised measurement as cbImu makes it
    const Vec3 acc = Vec3(0.03f * (cycle - 1), -0.02f, 1.0f).normalized();
    imu_model.setAccMeasure(acc);
    pf_ref.measure([&imu_model](const State6DOF& s) -> float { return imu_model.measure(s); });
    const float ref_imu_entropy = pf_ref.getEntropy();
    const auto imu = pf_gpu.imuMeasureResident(*batcher, acc, acc_var);
    EXPECT(imu.kept, "IMU update kept (cycle %d)", cycle);
    EXPECT(imu.match_ratio_min == 0.0f && imu.match_ratio_max == 0.0f, "IMU match ratios %g/%g", imu.match_ratio_min,
           imu.match_ratio_max);
    EXPECT(std::fabs(pf_gpu.getEntropy() - ref_imu_entropy) <= 2e-4 * std::fabs(ref_imu_entropy) + 1e-6,
           "IMU entropy %g vs %g (cycle %d)", pf_gpu.getEntropy(), ref_imu_entropy, cycle);
    pf_gpu.downloadResident(*batcher);
    {
      double worst_p = 0, worst_s = 0;
      auto ig = pf_gpu.begin();
      for (auto ir = pf_ref.begin(); ir != pf_ref.end(); ++ir, ++ig)
      {
        const double rel = std::fabs(ir->probability_ - ig->probability_) / std::max(1e-12, static_cast<double>(ir->probability_));
        worst_p = std::max(worst_p, rel);
        EXPECT(rel <= 2e-4, "IMU posterior %g vs %g (cycle %d)", ir->probability_, ig->probability_, cycle);
        const double ds = std::fabs(ir->state_.pos_.x_ - ig->state_.pos_.x_) + std::fabs(ir->state_.pos_.y_ - ig->state_.pos_.y_) +
                          std::fabs(ir->state_.rot_.z_ - ig->state_.rot_.z_) + std::fabs(ir->state_.rot_.w_ - ig->state_.rot_.w_);
        worst_s = std::max(worst_s, ds);
        EXPECT(ds <= 1e-4, "predicted state differs by %g (cycle %d)", ds, cycle);
      }
      std::printf("cycle %d: predict worst %.3g, IMU posterior worst %.3g, entropy %g vs %g\n", cycle, worst_s, worst_p,
                  pf_gpu.getEntropy(), ref_imu_entropy);
    }

    // the LIDAR update (the node's lambda with the odometry-error term); its match_ratio_max decides the reset
    std::map<std::string, Cloud::Ptr> pc_locals;
    for (const auto& m : lm)
    {
      m.second->setGlobalLocalizationStatus(n_particles, pf_ref.getParticleSize());
      pc_locals[m.first] = m.second->filter(scan, sampler);
    }
    float match_ratio_min = 1.0, match_ratio_max = 0.0;
    pf_ref.measure([&](const State6DOF& s) -> float
    {
      float likelihood = 1;
      std::map<std::string, float> qualities;
      for (const auto& m : lm)
      {
        const LidarMeasurementResult result = m.second->measure(kdtree, pc_locals[m.first], origins, s);
        likelihood *= result.likelihood;
        qualities[m.first] = result.quality;
      }
      if (match_ratio_min > qualities["likelihood"]) match_ratio_min = qualities["likelihood"];
      if (match_ratio_max < qualities["likelihood"]) match_ratio_max = qualities["likelihood"];
      return likelihood * odom_nd(s.odom_err_integ_lin_.norm());
    });
    const auto res = pf_gpu.measureResident(*batcher, kdtree, pc_locals["likelihood"], pc_locals["beam"], origins,
                                            odom_err_integ_lin_sigma);
    EXPECT(res.kept, "LIDAR update kept (cycle %d)", cycle);
    EXPECT(res.match_ratio_min == match_ratio_min && res.match_ratio_max == match_ratio_max, "match ratio %g/%g vs %g/%g",
           res.match_ratio_min, res.match_ratio_max, match_ratio_min, match_ratio_max);
    EXPECT(std::fabs(pf_gpu.getEntropy() - pf_ref.getEntropy()) <= 2e-4 * std::fabs(pf_ref.getEntropy()) + 1e-6,
           "LIDAR entropy %g vs %g", pf_gpu.getEntropy(), pf_ref.getEntropy());

    // resample on the device; the reference filter takes the device's set (noise stream: the documented departure)
    pf_gpu.resampleResident(*batcher, Vec3(0.05f, 0.05f, 0.05f), Vec3(0.05f, 0.05f, 0.05f), seed + cycle);
    pf_gpu.downloadResident(*batcher);
    adopt(pf_ref, pf_gpu);

    // the odometry-noise redraw: the node's lambda through pf_->predict, its normal draws replayed
    ++redraw_calls;
    std::vector<float> z(4 * static_cast<size_t>(n_particles));
    for (int i = 0; i < n_particles; ++i) redrawDraws(seed, static_cast<uint32_t>(i), redraw_calls, &z[4 * i]);
    {
      size_t k = 0;
      const auto noise = [&z, &k]() -> float { return z[k++]; };
      const auto update_noise_func = [&](State6DOF& s)
      {
        s.noise_ll_ = noise() * odom_err_lin_lin;
        s.noise_la_ = noise() * odom_err_lin_ang;
        s.noise_aa_ = noise() * odom_err_ang_ang;
        s.noise_al_ = noise() * odom_err_ang_lin;
      };
      pf_ref.predict(update_noise_func);
    }
    pf_gpu.redrawOdomNoiseResident(*batcher, odom_err_lin_lin, odom_err_lin_ang, odom_err_ang_lin, odom_err_ang_ang, seed);
    pf_gpu.downloadResident(*batcher);
    {
      size_t bad = 0;
      auto ig = pf_gpu.begin();
      for (auto ir = pf_ref.begin(); ir != pf_ref.end(); ++ir, ++ig)
      {
        const float r[4] = {ir->state_.noise_ll_, ir->state_.noise_la_, ir->state_.noise_al_, ir->state_.noise_aa_};
        const float g[4] = {ig->state_.noise_ll_, ig->state_.noise_la_, ig->state_.noise_al_, ig->state_.noise_aa_};
        for (int f = 0; f < 4; ++f)
          if (!(std::fabs(r[f] - g[f]) <= kOrgRel * std::fabs(r[f]) + ulpOf(r[f])))
            ++bad;
        const mcl3dl_state a = PFB::toState(ir->state_), b = PFB::toState(ig->state_);
        if (std::memcmp(a.pos, b.pos, sizeof(a.pos)) || std::memcmp(a.rot, b.rot, sizeof(a.rot)) ||
            std::memcmp(&ir->probability_, &ig->probability_, 4))
          ++bad;
      }
      EXPECT(bad == 0, "redraw: %zu differences (cycle %d)", bad, cycle);
      std::printf("cycle %d: redraw call %u, %zu differ\n", cycle, redraw_calls, bad);
    }

    // expansion resetting on both, from the same (exactly equal) match_ratio_max
    if (match_ratio_max < match_ratio_thresh)
    {
      ++resets;
      ++noise_calls;
      const float sg[6] = {expansion_pos.x_, expansion_pos.y_, expansion_pos.z_, expansion_rpy.x_, expansion_rpy.y_, expansion_rpy.z_};
      std::vector<float> org(6 * static_cast<size_t>(n_particles));
      for (int i = 0; i < n_particles; ++i) expansionDraws(seed, static_cast<uint32_t>(i), noise_calls, sg, &org[6 * i]);
      pf_ref.addNoiseUsingNoiseGenerator(ReplayNoise(org));   // pf_->noise(State6DOF(expansion_pos, expansion_rpy))
      pf_gpu.noiseResident(*batcher, expansion_pos, expansion_rpy, seed);
      pf_gpu.downloadResident(*batcher);
      size_t bad = 0;
      double max_norm_dev = 0;
      auto ig = pf_gpu.begin();
      for (auto ir = pf_ref.begin(); ir != pf_ref.end(); ++ir, ++ig)
      {
        const mcl3dl_state a = PFB::toState(ir->state_), b = PFB::toState(ig->state_);
        const float* o = &org[6 * (ir - pf_ref.begin())];
        for (int k = 0; k < 3; ++k)
        {
          if (!(std::fabs(a.pos[k] - b.pos[k]) <= ulpOf(a.pos[k]) + kOrgRel * std::fabs(o[k])) ||
              !(std::fabs(a.odom_err_integ_lin[k] - b.odom_err_integ_lin[k]) <= ulpOf(a.odom_err_integ_lin[k]) + kOrgRel * std::fabs(o[k])) ||
              !(std::fabs(a.odom_err_integ_ang[k] - b.odom_err_integ_ang[k]) <= ulpOf(a.odom_err_integ_ang[k]) + kOrgRel * std::fabs(o[k + 3])))
            ++bad;
        }
        const double rn = std::sqrt(double(a.rot[0]) * a.rot[0] + double(a.rot[1]) * a.rot[1] + double(a.rot[2]) * a.rot[2] +
                                    double(a.rot[3]) * a.rot[3]);
        max_norm_dev = std::max(max_norm_dev, std::fabs(rn - 1.0));
        for (int k = 0; k < 4; ++k)
          if (!(std::fabs(a.rot[k] - b.rot[k]) <= kRotRel * rn + ulpOf(a.rot[k])))
            ++bad;
        if (b.noise_ll != 0 || b.noise_la != 0 || b.noise_al != 0 || b.noise_aa != 0 ||
            std::memcmp(&ir->probability_, &ig->probability_, 4))
          ++bad;
      }
      EXPECT(bad == 0, "expansion reset: %zu differences (cycle %d)", bad, cycle);
      std::printf("cycle %d: expansion reset (match ratio max %g < %g), %zu differ, max | |rot| - 1 | %.3g\n", cycle,
                  match_ratio_max, match_ratio_thresh, bad, max_norm_dev);
    }
    adopt(pf_ref, pf_gpu);
  }
  std::printf("expansion resets: %d\n", resets);
  if (g_fail)
  {
    std::fprintf(stderr, "PF EVENTS PARITY FAILED (%d)\n", g_fail);
    return 1;
  }
  std::printf("PF EVENTS PARITY OK (%d cycles)\n", cycles);
  return 0;
}
