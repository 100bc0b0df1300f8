// map_update_parity_test.cpp — TEST INFRASTRUCTURE ONLY.
//
// The node's map update against the reference models: measurement cycles as MCL3dlNode::measure runs them
// (src/mcl_3dl.cpp:376-426), then cbMapUpdateTimer's own update code (src/mcl_3dl.cpp:1350-1378) with pc_map2_ aliasing
// pc_map_ as loadMapCloud leaves it, kdtree_->setInputCloud(pc_map2_), and more cycles.  The host C++ adapter
// (mcl_3dl_b200/host/lidar_measurement_model_b200.h) must agree with the reference's LidarMeasurementModelLikelihood /
// LidarMeasurementModelBeam at every cycle, and must have taken every update as an append (mcl3dl_map_append), never as a
// restage.  Built where a checkout of the reference exists (make -C oracle -f map_update.mk map-update-parity); the
// binary lands in oracle/_ref/, where tests/test_gpu_map_update_parity.py runs it on an H100.
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
#include <mcl_3dl/pf.h>
#include <mcl_3dl/point_cloud_random_sampler.h>
#include <mcl_3dl/state_6dof.h>

#include "../mcl_3dl_b200/host/lidar_measurement_model_b200.h"

using namespace mcl_3dl;
using PointType = LidarMeasurementModelBase::PointType;
using Cloud = pcl::PointCloud<PointType>;
using PF = mcl_3dl_b200::ParticleFilter;

namespace pcl
{
// pcl::PointCloud::operator+ (a copy of the left cloud with the right one's points appended), which the node's update
// uses and the shim leaves out
template <typename PointT>
PointCloud<PointT> operator+(const PointCloud<PointT>& a, const PointCloud<PointT>& b)
{
  PointCloud<PointT> out(a);
  out += b;
  return out;
}
}  // namespace pcl

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

// An obstacle box at 0.3 m spacing (a patch after cbMapcloudUpdate's VoxelGrid at update_downsample).
Cloud::Ptr boxPatch(float x0, float y0, float size, uint32_t label)
{
  Cloud::Ptr p(new Cloud);
  for (float a = 0.f; a <= size + 1e-4f; a += 0.3f)
    for (float b = 0.f; b <= size + 1e-4f; b += 0.3f)
    {
      p->push_back(pt(x0 + a, y0, b, label));
      p->push_back(pt(x0 + a, y0 + size, b, label));
      p->push_back(pt(x0, y0 + a, b, label));
      p->push_back(pt(x0 + size, y0 + a, b, label));
      p->push_back(pt(x0 + a, y0 + b, size, label));
    }
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

using Models = std::map<std::string, LidarMeasurementModelBase::Ptr>;

// MCL3dlNode::measure from filter to pf_->measure (src/mcl_3dl.cpp:376-426) for one model set: per-particle likelihoods
// and the match ratio range
void runCycle(Models& m, PF& pf, ChunkedKdtree<PointType>::Ptr& kdtree, const Cloud::ConstPtr& scan,
              const PointCloudRandomSampler<PointType>& sampler, const std::vector<Vec3>& origins, std::vector<float>& out,
              float& ratio_min, float& ratio_max)
{
  std::map<std::string, Cloud::Ptr> pc_locals;
  for (const auto& lm : m)
  {
    lm.second->setGlobalLocalizationStatus(pf.getParticleSize(), pf.getParticleSize());
    pc_locals[lm.first] = lm.second->filter(scan, sampler);
  }
  ratio_min = 1.0f;
  ratio_max = 0.0f;
  pf.measure([&](const State6DOF& s) -> float {
    float likelihood = 1;
    std::map<std::string, float> qualities;
    for (const auto& lm : m)
    {
      const LidarMeasurementResult r = lm.second->measure(kdtree, pc_locals[lm.first], origins, s);
      likelihood *= r.likelihood;
      qualities[lm.first] = r.quality;
    }
    ratio_min = std::min(ratio_min, qualities["likelihood"]);
    ratio_max = std::max(ratio_max, qualities["likelihood"]);
    out.push_back(likelihood);
    return likelihood;
  });
}
}  // namespace

int main(int argc, char** argv)
{
  const int n_particles = argc > 1 ? std::atoi(argv[1]) : 300;
  const bool use_dda = !(argc > 2 && std::string(argv[2]) == "kd");
  std::mt19937 rng(17);
  std::normal_distribution<float> n01(0.f, 1.f);

  // ---- loadMapCloud: pc_map_ (a 12 x 12 m floor and two walls, one labelled), pc_map2_ reset, no update pending
  Cloud::Ptr pc_map_(new Cloud), pc_map2_, pc_update_;
  for (float x = 0.05f; x < 12.f; x += 0.1f)
    for (float y = 0.05f; y < 12.f; y += 0.1f)
      pc_map_->push_back(pt(x + 0.02f * n01(rng), y + 0.02f * n01(rng), 0.03f + 0.01f * n01(rng)));
  for (float y = 0.05f; y < 12.f; y += 0.1f)
    for (float z = 0.05f; z < 3.f; z += 0.1f)
    {
      pc_map_->push_back(pt(0.03f + 0.01f * n01(rng), y, z));
      pc_map_->push_back(pt(11.97f + 0.01f * n01(rng), y, z, 2));
    }
  pc_map_->header.stamp = 1000;

  const float dist_weight[4] = {1.f, 1.f, 5.f, 0.f};
  auto rep = std::make_shared<XyzRep>();
  rep->setRescaleValues(dist_weight);
  ChunkedKdtree<PointType>::Ptr kdtree_(new ChunkedKdtree<PointType>(20.0, 0.4));
  kdtree_->setPointRepresentation(rep);
  uint64_t now = 2000;  // ros::Time::now() of the update stamps
  // cbMapUpdateTimer, src/mcl_3dl.cpp:1350-1378 (the publishing left out)
  const auto cbMapUpdateTimer = [&]() {
    if (pc_update_)
    {
      if (!pc_map2_)
        pc_map2_.reset(new Cloud);
      *pc_map2_ = *pc_map_ + *pc_update_;
      pc_update_.reset();
      pc_map2_->header.stamp = ++now;
    }
    else
    {
      if (pc_map2_)
        return;
      pc_map2_ = pc_map_;
    }
    kdtree_->setInputCloud(pc_map2_);
  };
  cbMapUpdateTimer();

  auto lik_params = std::make_shared<LidarMeasurementModelLikelihoodParameters>();
  lik_params->num_points_default_ = 96;
  auto beam_params = std::make_shared<LidarMeasurementModelBeamParameters>();
  beam_params->num_points_default_ = 12;
  beam_params->use_raycast_using_dda_ = use_dda;
  beam_params->filter_label_max_ = 1;

  // ---- the scan: points of the final map (patches included) seen from (6, 4, 0.5) yaw 0.3, + noise
  const std::vector<Cloud::Ptr> patches = {boxPatch(7.0f, 5.0f, 1.2f, 0), boxPatch(4.0f, 2.5f, 0.9f, 3),
                                           boxPatch(5.5f, 6.5f, 1.5f, 0)};
  Cloud all(*pc_map_);
  for (const auto& p : patches) all += *p;
  const Vec3 truth_pos(6.f, 4.f, 0.5f);
  const Quat truth_rot(Vec3(0, 0, 1), 0.3f);
  Cloud::Ptr scan(new Cloud);
  std::uniform_int_distribution<size_t> pick(0, all.size() - 1);
  while (scan->size() < 400)
  {
    const PointType& mp = all.points[pick(rng)];
    const Vec3 local = truth_rot.inv() * (Vec3(mp.x, mp.y, mp.z) - truth_pos);
    if (local.x_ * local.x_ + local.y_ * local.y_ > 36.f)
      continue;
    scan->push_back(pt(local.x_ + 0.02f * n01(rng), local.y_ + 0.02f * n01(rng), local.z_ + 0.02f * n01(rng),
                       scan->size() % 2));
  }
  const std::vector<Vec3> origins = {Vec3(0.f, 0.f, 0.3f), Vec3(0.2f, -0.1f, 0.25f)};
  const HeadSampler sampler;

  PF pf_ref(n_particles, 7), pf_gpu(n_particles, 7);
  const State6DOF mean(truth_pos, truth_rot);
  const State6DOF sigma(Vec3(0.3f, 0.3f, 0.05f), Vec3(0.02f, 0.02f, 0.1f));
  pf_ref.init(mean, sigma);
  pf_gpu.init(mean, sigma);
  Models ref, gpu;
  ref["likelihood"] = std::make_shared<LidarMeasurementModelLikelihood>(lik_params);
  ref["beam"] = std::make_shared<LidarMeasurementModelBeam>(beam_params);
  auto batcher = std::make_shared<mcl_3dl_b200::MeasurementBatcher>(&pf_gpu, std::vector<int>{0}, lik_params, beam_params,
                                                                   dist_weight);
  gpu["likelihood"] = std::make_shared<mcl_3dl_b200::LidarMeasurementModelLikelihoodB200>(lik_params, batcher);
  gpu["beam"] = std::make_shared<mcl_3dl_b200::LidarMeasurementModelBeamB200>(beam_params, batcher);

  int cycle = 0;
  const auto cycles = [&](int n) {
    for (int k = 0; k < n; ++k, ++cycle)
    {
      std::vector<float> a, b;
      float amin, amax, bmin, bmax;
      runCycle(ref, pf_ref, kdtree_, scan, sampler, origins, a, amin, amax);
      runCycle(gpu, pf_gpu, kdtree_, scan, sampler, origins, b, bmin, bmax);
      EXPECT(a.size() == b.size() && a.size() == static_cast<size_t>(n_particles), "sizes %zu %zu", a.size(), b.size());
      double worst = 0;
      for (size_t i = 0; i < a.size() && i < b.size(); ++i)
      {
        const double rel = std::fabs(a[i] - b[i]) / std::max(1e-6, static_cast<double>(std::fabs(a[i])));
        worst = std::max(worst, rel);
        EXPECT(rel <= 1e-4, "cycle %d particle %zu: ref %.9g gpu %.9g", cycle, i, a[i], b[i]);
      }
      EXPECT(amin == bmin && amax == bmax, "cycle %d match ratio %g/%g vs %g/%g", cycle, amin, amax, bmin, bmax);
      std::printf("cycle %d: map %zu points, worst relative diff %.3g, match ratio [%g, %g]\n", cycle,
                  kdtree_->getInputCloud()->size(), worst, amin, amax);
      // the same particles for the next cycle: resample the reference filter and copy it
      pf_ref.resample(State6DOF(Vec3(0.05f, 0.05f, 0.01f), Vec3(0.005f, 0.005f, 0.02f)));
      auto ir = pf_ref.begin();
      auto ig = pf_gpu.begin();
      for (; ir != pf_ref.end(); ++ir, ++ig) *ig = *ir;
    }
  };

  cycles(2);
  for (const auto& p : patches)
  {
    pc_update_.reset(new Cloud(*p));  // cbMapcloudUpdate
    cbMapUpdateTimer();
    EXPECT(pc_map2_ == pc_map_, "pc_map2_ aliases pc_map_");
    cycles(2);
  }
  cbMapUpdateTimer();  // no update pending: nothing changes
  cycles(1);
  EXPECT(pc_map_->size() == all.size(), "map %zu points, want %zu", pc_map_->size(), all.size());
  EXPECT(batcher->mapAppends() == patches.size() && batcher->mapRestages() == 1, "appends %zu, restages %zu",
         batcher->mapAppends(), batcher->mapRestages());
  std::printf("map updates: %zu appended, %zu staged whole\n", batcher->mapAppends(), batcher->mapRestages());
  if (g_fail)
  {
    std::fprintf(stderr, "MAP UPDATE PARITY FAILED (%d)\n", g_fail);
    return 1;
  }
  std::printf("MAP UPDATE PARITY OK\n");
  return 0;
}
