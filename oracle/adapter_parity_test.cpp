// adapter_parity_test.cpp — TEST INFRASTRUCTURE ONLY.
//
// Drives the host C++ adapter (mcl_3dl_b200/host/lidar_measurement_model_b200.h) exactly the way
// MCL3dlNode::measure does (src/mcl_3dl.cpp:376-426) and compares it, particle by particle, with the
// reference's own LidarMeasurementModelLikelihood / LidarMeasurementModelBeam running on the CPU in
// the same process.  Built only where a checkout of the reference exists (make -C oracle adapter
// REFERENCE=<path>), against oracle/shim/; the binary lands in oracle/_ref/, where tests/test_gpu_adapter.py runs it.
#include <cmath>
#include <cstdio>
#include <map>
#include <memory>
#include <random>
#include <string>
#include <vector>

#include <mcl_3dl/chunked_kdtree.h>
#include <mcl_3dl/lidar_measurement_models/lidar_measurement_model_beam.h>
#include <mcl_3dl/lidar_measurement_models/lidar_measurement_model_likelihood.h>
#include <mcl_3dl/motion_prediction_models/motion_prediction_model_differential_drive.h>
#include <mcl_3dl/nd.h>
#include <mcl_3dl/pf.h>
#include <mcl_3dl/point_cloud_random_sampler.h>
#include <mcl_3dl/state_6dof.h>

#include "../mcl_3dl_b200/host/lidar_measurement_model_b200.h"

using namespace mcl_3dl;
using PointType = LidarMeasurementModelBase::PointType;
using Cloud = pcl::PointCloud<PointType>;
using PF = mcl_3dl_b200::ParticleFilter;

namespace
{
// same idea as DummySampler in test/src/test_beam_likelihood.cpp:47-76, but keeps at most `num` points
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
#define EXPECT(cond, ...)                      \
  do                                           \
  {                                            \
    if (!(cond))                               \
    {                                          \
      ++g_fail;                                \
      if (g_fail < 20)                         \
      {                                        \
        std::fprintf(stderr, "FAIL %s: ", #cond); \
        std::fprintf(stderr, __VA_ARGS__);     \
        std::fprintf(stderr, "\n");            \
      }                                        \
    }                                          \
  } while (0)

struct Models
{
  std::map<std::string, LidarMeasurementModelBase::Ptr> lm;
};

// MCL3dlNode::measure's body from filter to pf_->measure (src/mcl_3dl.cpp:376-426), for one model set.
void runCycle(Models& m, PF& pf, ChunkedKdtree<PointType>::Ptr& kdtree, const Cloud::ConstPtr& pc_local_full,
              const PointCloudRandomSampler<PointType>& sampler, const std::vector<Vec3>& origins, size_t num_particles,
              std::vector<float>* per_particle, float* ratio_min, float* ratio_max)
{
  std::map<std::string, Cloud::Ptr> pc_locals;
  for (const auto& lm : m.lm)
  {
    lm.second->setGlobalLocalizationStatus(num_particles, pf.getParticleSize());
    pc_locals[lm.first] = lm.second->filter(pc_local_full, sampler);
  }
  float match_ratio_min = 1.0, match_ratio_max = 0.0;
  const auto measure_func = [&](const State6DOF& s) -> float
  {
    float likelihood = 1;
    std::map<std::string, float> qualities;
    for (const auto& lm : m.lm)
    {
      const LidarMeasurementResult result = lm.second->measure(kdtree, pc_locals[lm.first], origins, s);
      likelihood *= result.likelihood;
      qualities[lm.first] = result.quality;
    }
    if (match_ratio_min > qualities["likelihood"]) match_ratio_min = qualities["likelihood"];
    if (match_ratio_max < qualities["likelihood"]) match_ratio_max = qualities["likelihood"];
    per_particle->push_back(likelihood);
    return likelihood;
  };
  pf.measure(measure_func);
  *ratio_min = match_ratio_min;
  *ratio_max = match_ratio_max;
}
}  // namespace

int main(int argc, char** argv)
{
  const int n_particles = argc > 1 ? std::atoi(argv[1]) : 300;
  const bool use_dda = !(argc > 2 && std::string(argv[2]) == "kd");  // "kd": the node's default RaycastUsingKDTree
  std::mt19937 rng(42);
  std::normal_distribution<float> n01(0.f, 1.f);
  std::uniform_real_distribution<float> u01(0.f, 1.f);

  // ---- map: 12 x 12 m floor, two walls, one labelled wall (label 2), ~0.1 m spacing
  Cloud::Ptr map(new Cloud);
  for (float x = 0.05f; x < 12.f; x += 0.1f)
    for (float y = 0.05f; y < 12.f; y += 0.1f)
      map->push_back(pt(x + 0.02f * n01(rng), y + 0.02f * n01(rng), 0.03f + 0.01f * n01(rng)));
  for (float y = 0.05f; y < 12.f; y += 0.1f)
    for (float z = 0.05f; z < 3.f; z += 0.1f)
    {
      map->push_back(pt(0.03f + 0.01f * n01(rng), y, z));
      map->push_back(pt(11.97f + 0.01f * n01(rng), y, z, 2));
    }
  for (float x = 4.f; x < 6.f; x += 0.1f)
    for (float z = 0.05f; z < 2.f; z += 0.1f)
      map->push_back(pt(x, 7.03f + 0.01f * n01(rng), z));
  map->header.stamp = 1234;

  // ---- node configure(): kd-tree with the (1,1,5) rescale (src/mcl_3dl.cpp:1270,1326-1329)
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
  beam_params->use_raycast_using_dda_ = use_dda;
  beam_params->filter_label_max_ = 1;

  // ---- scan in the base frame: points of the map seen from (6, 4, 0.5) yaw 0.3, + noise; labels = sensor id
  const Vec3 truth_pos(6.f, 4.f, 0.5f);
  const Quat truth_rot(Vec3(0, 0, 1), 0.3f);
  Cloud::Ptr scan(new Cloud);
  std::uniform_int_distribution<size_t> pick(0, map->size() - 1);
  while (scan->size() < 400)
  {
    const PointType& mp = map->points[pick(rng)];
    const Vec3 local = truth_rot.inv() * (Vec3(mp.x, mp.y, mp.z) - truth_pos);
    scan->push_back(pt(local.x_ + 0.02f * n01(rng), local.y_ + 0.02f * n01(rng), local.z_ + 0.02f * n01(rng),
                       scan->size() % 2));
  }
  const std::vector<Vec3> origins = {Vec3(0.f, 0.f, 0.3f), Vec3(0.2f, -0.1f, 0.25f)};
  const HeadSampler sampler;

  // ---- two identical particle filters (same seed): one per model set
  PF pf_ref(n_particles, 7), pf_gpu(n_particles, 7);
  const State6DOF mean(truth_pos, truth_rot);
  const State6DOF sigma(Vec3(0.2f, 0.2f, 0.05f), Vec3(0.02f, 0.02f, 0.1f));
  pf_ref.init(mean, sigma);
  pf_gpu.init(mean, sigma);

  Models ref, gpu;
  ref.lm["likelihood"] = std::make_shared<LidarMeasurementModelLikelihood>(lik_params);
  ref.lm["beam"] = std::make_shared<LidarMeasurementModelBeam>(beam_params);
  auto batcher = std::make_shared<mcl_3dl_b200::MeasurementBatcher>(&pf_gpu, std::vector<int>{0}, lik_params, beam_params,
                                                                   dist_weight);
  gpu.lm["likelihood"] = std::make_shared<mcl_3dl_b200::LidarMeasurementModelLikelihoodB200>(lik_params, batcher);
  gpu.lm["beam"] = std::make_shared<mcl_3dl_b200::LidarMeasurementModelBeamB200>(beam_params, batcher);
  // the node's marker path must keep working (src/mcl_3dl.cpp:471)
  EXPECT(std::dynamic_pointer_cast<LidarMeasurementModelBeam>(gpu.lm["beam"]) != nullptr, "dynamic_pointer_cast");

  for (int cycle = 0; cycle < 3; ++cycle)
  {
    std::vector<float> a, b;
    float amin, amax, bmin, bmax;
    // cycle 2 emulates global localisation: more particles than num_particles shrink the scan (likelihood.cpp:63-77)
    const size_t nominal = cycle == 2 ? n_particles / 4 : n_particles;
    runCycle(ref, pf_ref, kdtree, scan, sampler, origins, nominal, &a, &amin, &amax);
    runCycle(gpu, pf_gpu, kdtree, scan, sampler, origins, nominal, &b, &bmin, &bmax);
    EXPECT(a.size() == b.size() && a.size() == static_cast<size_t>(n_particles), "sizes %zu %zu", a.size(), b.size());
    double worst = 0;
    for (size_t i = 0; i < a.size() && i < b.size(); ++i)
    {
      const double rel = std::fabs(a[i] - b[i]) / std::max(1e-6, static_cast<double>(std::fabs(a[i])));
      worst = std::max(worst, rel);
      EXPECT(rel <= 1e-4, "cycle %d particle %zu: ref %.9g gpu %.9g", cycle, i, a[i], b[i]);
    }
    EXPECT(amin == bmin && amax == bmax, "match ratio min/max %g/%g vs %g/%g", amin, amax, bmin, bmax);
    // posterior weights and entropy after pf.measure (pf.h:252-279)
    auto ir = pf_ref.begin();
    auto ig = pf_gpu.begin();
    for (; ir != pf_ref.end(); ++ir, ++ig)
      EXPECT(std::fabs(ir->probability_ - ig->probability_) <= 1e-4 * std::fabs(ir->probability_) + 1e-9,
             "posterior %g vs %g", ir->probability_, ig->probability_);
    EXPECT(std::fabs(pf_ref.getEntropy() - pf_gpu.getEntropy()) <= 1e-4 * std::fabs(pf_ref.getEntropy()) + 1e-6,
           "entropy %g vs %g", pf_ref.getEntropy(), pf_gpu.getEntropy());
    std::printf("cycle %d: %zu particles, worst relative diff %.3g, match ratio [%g, %g], entropy %g\n", cycle, a.size(),
                worst, amin, amax, pf_ref.getEntropy());
    // resample both filters identically (same engine seed and same weights up to 1e-4 can still diverge;
    // so copy the reference filter's particles into the GPU one to keep the comparison per-particle)
    pf_ref.resample(State6DOF(Vec3(0.05f, 0.05f, 0.01f), Vec3(0.005f, 0.005f, 0.02f)));
    ir = pf_ref.begin();
    ig = pf_gpu.begin();
    for (; ir != pf_ref.end(); ++ir, ++ig) *ig = *ir;
  }
  // scope row f2: the fused pf update behind ParticleFilterB200::measureBatched vs pf.measure(lambda with the
  // odometry-error term) of the reference (src/mcl_3dl.cpp:402-426)
  {
    mcl_3dl_b200::ParticleFilterB200 pf_fused(n_particles, 7);
    pf_fused.init(mean, sigma);
    auto ir = pf_ref.begin();
    auto ig = pf_fused.begin();
    std::uniform_real_distribution<float> uw(0.2f, 1.0f);
    for (; ir != pf_ref.end(); ++ir, ++ig)
    {
      *ig = *ir;
      ig->probability_ = ir->probability_ = uw(rng);
      ig->state_.odom_err_integ_lin_ = ir->state_.odom_err_integ_lin_ = Vec3(0.02f * n01(rng), 0.02f * n01(rng), 0.f);
    }
    const float sigma_odom = 0.05f;
    const auto odom_term = [sigma_odom](const State6DOF& s) -> float
    {
      // NormalLikelihood<float>(sigma)(x), include/mcl_3dl/nd.h:45-53
      const float a = 1.0 / std::sqrt(2.0 * M_PI * sigma_odom * sigma_odom);
      const float sq2 = sigma_odom * sigma_odom * 2.0;
      const float x = s.odom_err_integ_lin_.norm();
      return a * expf(-x * x / sq2);
    };
    std::map<std::string, Cloud::Ptr> pc_locals;
    for (const auto& lm : ref.lm)
    {
      lm.second->setGlobalLocalizationStatus(n_particles, pf_ref.getParticleSize());
      pc_locals[lm.first] = lm.second->filter(scan, sampler);
    }
    float rmin = 1.0, rmax = 0.0;
    pf_ref.measure([&](const State6DOF& s) -> float
    {
      float likelihood = 1;
      std::map<std::string, float> qualities;
      for (const auto& lm : ref.lm)
      {
        const LidarMeasurementResult result = lm.second->measure(kdtree, pc_locals[lm.first], origins, s);
        likelihood *= result.likelihood;
        qualities[lm.first] = result.quality;
      }
      if (rmin > qualities["likelihood"]) rmin = qualities["likelihood"];
      if (rmax < qualities["likelihood"]) rmax = qualities["likelihood"];
      return likelihood * odom_term(s);
    });
    auto batcher2 = std::make_shared<mcl_3dl_b200::MeasurementBatcher>(&pf_fused, std::vector<int>{0}, lik_params, beam_params,
                                                                      dist_weight);
    const auto res = pf_fused.measureBatched(*batcher2, kdtree, pc_locals["likelihood"], pc_locals["beam"], origins, odom_term);
    EXPECT(res.kept, "fused update kept");
    EXPECT(res.match_ratio_min == rmin && res.match_ratio_max == rmax, "fused match ratio %g/%g vs %g/%g", res.match_ratio_min,
           res.match_ratio_max, rmin, rmax);
    ir = pf_ref.begin();
    ig = pf_fused.begin();
    double worst = 0;
    for (; ir != pf_ref.end(); ++ir, ++ig)
    {
      const double rel = std::fabs(ir->probability_ - ig->probability_) / std::max(1e-12, static_cast<double>(ir->probability_));
      worst = std::max(worst, rel);
      EXPECT(rel <= 1e-4, "fused posterior %g vs %g", ir->probability_, ig->probability_);
    }
    EXPECT(std::fabs(pf_ref.getEntropy() - pf_fused.getEntropy()) <= 1e-4 * std::fabs(pf_ref.getEntropy()) + 1e-6,
           "fused entropy %g vs %g", pf_ref.getEntropy(), pf_fused.getEntropy());
    std::printf("fused update: worst relative posterior diff %.3g, entropy %g vs %g\n", worst, pf_ref.getEntropy(),
                pf_fused.getEntropy());
  }
  // scope row f3: three cycles on the RESIDENT particle set (predict / measure / estimate / resample on the device)
  // against the reference filter doing the same on the host.  Resampling draws different noise (documented departure),
  // so after every cycle the device set is re-uploaded from the reference filter; what is compared per cycle is
  // predict (states), the posterior + entropy + match ratios, and the pose estimate.
  {
    mcl_3dl_b200::ParticleFilterB200 pf_res(n_particles, 7);
    pf_res.init(mean, sigma);
    auto batcher3 = std::make_shared<mcl_3dl_b200::MeasurementBatcher>(&pf_res, std::vector<int>{0}, lik_params, beam_params,
                                                                      dist_weight);
    MotionPredictionModelDifferentialDrive motion(10.0f, 10.0f);
    const float sigma_odom = 0.05f;
    NormalLikelihood<float> odom_nd(sigma_odom);
    State6DOF odom_prev(Vec3(0.f, 0.f, 0.f), Quat(0.f, 0.f, 0.f, 1.f));
    for (int cycle = 0; cycle < 3; ++cycle)
    {
      auto ir = pf_ref.begin();
      auto ig = pf_res.begin();
      for (; ir != pf_ref.end(); ++ir, ++ig)
      {
        ir->state_.noise_ll_ = 0.01f * n01(rng);
        ir->state_.noise_la_ = 0.01f * n01(rng);
        ir->state_.noise_al_ = 0.01f * n01(rng);
        ir->state_.noise_aa_ = 0.01f * n01(rng);
        *ig = *ir;
      }
      pf_res.uploadResident(*batcher3);
      // predict
      State6DOF odom_cur(odom_prev.pos_ + Vec3(0.05f, 0.01f * cycle, 0.f), Quat(Vec3(0.f, 0.f, 1.f), 0.02f * (cycle + 1)) * odom_prev.rot_);
      motion.setOdoms(odom_prev, odom_cur, 0.1f);
      pf_ref.predict([&motion](State6DOF& s) { motion.predict(s); });  // src/mcl_3dl.cpp:227-232
      pf_res.predictResident(*batcher3, odom_prev, odom_cur, 0.1f, 10.0f, 10.0f);
      odom_prev = odom_cur;
      // measure (the node's lambda with the odometry-error term)
      std::map<std::string, Cloud::Ptr> pc_locals;
      for (const auto& lm : ref.lm)
      {
        lm.second->setGlobalLocalizationStatus(n_particles, pf_ref.getParticleSize());
        pc_locals[lm.first] = lm.second->filter(scan, sampler);
      }
      float rmin = 1.0, rmax = 0.0;
      pf_ref.measure([&](const State6DOF& s) -> float
      {
        float likelihood = 1;
        std::map<std::string, float> qualities;
        for (const auto& lm : ref.lm)
        {
          const LidarMeasurementResult result = lm.second->measure(kdtree, pc_locals[lm.first], origins, s);
          likelihood *= result.likelihood;
          qualities[lm.first] = result.quality;
        }
        if (rmin > qualities["likelihood"]) rmin = qualities["likelihood"];
        if (rmax < qualities["likelihood"]) rmax = qualities["likelihood"];
        return likelihood * odom_nd(s.odom_err_integ_lin_.norm());
      });
      const auto res = pf_res.measureResident(*batcher3, kdtree, pc_locals["likelihood"], pc_locals["beam"], origins, sigma_odom);
      EXPECT(res.kept, "resident update kept (cycle %d)", cycle);
      EXPECT(res.match_ratio_min == rmin && res.match_ratio_max == rmax, "resident match ratio %g/%g vs %g/%g", res.match_ratio_min,
             res.match_ratio_max, rmin, rmax);
      // estimate: bias + expectationBiased + max + covariance on the device vs the reference filter
      const State6DOF state_prev = pf_ref.expectation(1.0);
      NormalLikelihood<float> nl_lin(0.2f), nl_ang(0.3f);
      pf_ref.bias([&](const State6DOF& s, float& p_bias) -> void
      {
        const float lin_diff = (s.pos_ - state_prev.pos_).norm();
        Vec3 axis;
        float ang_diff;
        (s.rot_ * state_prev.rot_.inv()).getAxisAng(axis, ang_diff);
        p_bias = nl_lin(lin_diff) * nl_ang(ang_diff) + 1e-6;
      });
      const State6DOF e_ref = pf_ref.expectationBiased();
      const std::vector<State6DOF> cov_ref = pf_ref.covariance(1.0, 1.0);
      const mcl3dl_estimate est = pf_res.estimateResident(*batcher3, &state_prev, 0.2f, 0.3f);
      EXPECT(std::fabs(est.mean_biased.px - e_ref.pos_.x_) < 1e-4 && std::fabs(est.mean_biased.py - e_ref.pos_.y_) < 1e-4 &&
                 std::fabs(est.mean_biased.pz - e_ref.pos_.z_) < 1e-4,
             "resident mean pos (%g %g %g) vs (%g %g %g)", est.mean_biased.px, est.mean_biased.py, est.mean_biased.pz, e_ref.pos_.x_,
             e_ref.pos_.y_, e_ref.pos_.z_);
      EXPECT(std::fabs(est.mean_biased.qz - e_ref.rot_.z_) < 5e-5 && std::fabs(est.mean_biased.qw - e_ref.rot_.w_) < 5e-5,
             "resident mean rot z w (%g %g) vs (%g %g)", est.mean_biased.qz, est.mean_biased.qw, e_ref.rot_.z_, e_ref.rot_.w_);
      for (int j = 0; j < 6; ++j)
        EXPECT(std::fabs(est.cov[j * 6 + j] - cov_ref[j][j]) <= 5e-3 * std::fabs(cov_ref[j][j]) + 1e-8, "resident cov[%d][%d] %g vs %g",
               j, j, est.cov[j * 6 + j], cov_ref[j][j]);
      // states after predict and posterior after measure, per particle
      pf_res.downloadResident(*batcher3);
      ir = pf_ref.begin();
      ig = pf_res.begin();
      double worst_p = 0, worst_s = 0;
      for (; ir != pf_ref.end(); ++ir, ++ig)
      {
        const double rel = std::fabs(ir->probability_ - ig->probability_) / std::max(1e-12, static_cast<double>(ir->probability_));
        worst_p = std::max(worst_p, rel);
        EXPECT(rel <= 2e-4, "resident posterior %g vs %g", ir->probability_, ig->probability_);
        const double ds = std::fabs(ir->state_.pos_.x_ - ig->state_.pos_.x_) + std::fabs(ir->state_.pos_.y_ - ig->state_.pos_.y_) +
                          std::fabs(ir->state_.rot_.z_ - ig->state_.rot_.z_) + std::fabs(ir->state_.rot_.w_ - ig->state_.rot_.w_);
        worst_s = std::max(worst_s, ds);
        EXPECT(ds <= 1e-4, "resident predicted state differs by %g", ds);
      }
      EXPECT(std::fabs(pf_ref.getEntropy() - pf_res.getEntropy()) <= 2e-4 * std::fabs(pf_ref.getEntropy()) + 1e-6,
             "resident entropy %g vs %g", pf_ref.getEntropy(), pf_res.getEntropy());
      std::printf("resident cycle %d: worst posterior diff %.3g, worst state diff %.3g, mean (%g %g), cov xx %g vs %g\n", cycle,
                  worst_p, worst_s, est.mean_biased.px, est.mean_biased.py, est.cov[0], cov_ref[0][0]);
      // resample: on the device (exercised, checked for sanity) and on the reference filter (kept as the next cycle's input)
      pf_res.resampleResident(*batcher3, Vec3(0.05f, 0.05f, 0.01f), Vec3(0.005f, 0.005f, 0.02f), 100 + cycle);
      pf_res.downloadResident(*batcher3);
      float psum = 0;
      for (auto it = pf_res.begin(); it != pf_res.end(); ++it) psum += it->probability_;
      EXPECT(std::fabs(psum - 1.0f) < 1e-3, "resident resample: probabilities sum to %g", psum);
      pf_ref.resample(State6DOF(Vec3(0.05f, 0.05f, 0.01f), Vec3(0.005f, 0.005f, 0.02f)));
    }
  }
  // a state that is not a particle (mean pose): served by a one-particle engine call
  {
    const State6DOF e = pf_ref.expectation(1.0);
    ref.lm["likelihood"]->setGlobalLocalizationStatus(n_particles, n_particles);
    gpu.lm["likelihood"]->setGlobalLocalizationStatus(n_particles, n_particles);
    Cloud::Ptr pcl = ref.lm["likelihood"]->filter(scan, sampler);
    Cloud::Ptr pcg = gpu.lm["likelihood"]->filter(scan, sampler);
    const LidarMeasurementResult r1 = ref.lm["likelihood"]->measure(kdtree, pcl, origins, e);
    const LidarMeasurementResult r2 = gpu.lm["likelihood"]->measure(kdtree, pcg, origins, e);
    EXPECT(std::fabs(r1.likelihood - r2.likelihood) <= 1e-4 * std::fabs(r1.likelihood) && r1.quality == r2.quality,
           "mean pose: %g/%g vs %g/%g", r1.likelihood, r1.quality, r2.likelihood, r2.quality);
  }
  if (g_fail)
  {
    std::fprintf(stderr, "ADAPTER PARITY FAILED (%d)\n", g_fail);
    return 1;
  }
  std::printf("ADAPTER PARITY OK\n");
  return 0;
}
