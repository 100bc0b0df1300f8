// normal_sampler_ref_driver.cpp — TEST INFRASTRUCTURE ONLY ("reference" checker of oracle/normal_sampler_api.h).
//
// The reference's own PointCloudSamplerWithNormal<PointXYZIL> (setParticleStatistics + sample), unchanged, with
// std::default_random_engine(seed).  It compiles against oracle/shim_ns first (NormalEstimation, a double
// SelfAdjointEigenSolver and ros::WallTime, repo-written stand-ins that call oracle/normal_eigen.h), then oracle/shim.
#include <ros/ros.h>

#include <algorithm>
#include <memory>
#include <vector>

#include <mcl_3dl/point_cloud_random_samplers/point_cloud_sampler_with_normal.h>
#include <mcl_3dl/point_types.h>
#include <mcl_3dl/state_6dof.h>

#include "normal_sampler_api.h"

extern "C" {
const char* mcl3dl_cpu_ns_kind(void) { return "reference"; }

int mcl3dl_cpu_ns_sample(const mcl3dl_point* pts, size_t n, const float cov[9], const float mean_rot[4], const double params[4],
                         size_t num, uint32_t seed, mcl3dl_point* out, size_t* n_out, double consts[4])
{
  auto prm = std::make_shared<mcl_3dl::PointCloudSamplerWithNormalParameters>();
  prm->perform_weighting_ratio_ = params[0];
  prm->max_weight_ratio_ = params[1];
  prm->max_weight_ = params[2];
  prm->normal_search_range_ = params[3];
  mcl_3dl::PointCloudSamplerWithNormal<mcl_3dl::PointXYZIL> sampler(prm, seed);
  mcl_3dl::State6DOF mean;
  mean.rot_ = mcl_3dl::Quat(mean_rot[0], mean_rot[1], mean_rot[2], mean_rot[3]);
  std::vector<mcl_3dl::State6DOF> covariances(6);
  for (size_t i = 0; i < 3; ++i)
    for (size_t j = 0; j < 3; ++j) covariances[i][j] = cov[i * 3 + j];
  sampler.setParticleStatistics(mean, covariances);
  pcl::PointCloud<mcl_3dl::PointXYZIL>::Ptr pc(new pcl::PointCloud<mcl_3dl::PointXYZIL>);
  for (size_t i = 0; i < n; ++i)
  {
    mcl_3dl::PointXYZIL p;
    p.x = pts[i].x;
    p.y = pts[i].y;
    p.z = pts[i].z;
    p.label = pts[i].label;
    pc->push_back(p);
  }
  const auto s = sampler.sample(pc, num);
  for (size_t j = 0; j < s->size(); ++j)
    out[j] = mcl3dl_point{s->points[j].x, s->points[j].y, s->points[j].z, s->points[j].label};
  *n_out = s->size();
  if (consts)
    std::fill(consts, consts + 4, 0.0);
  return 0;
}
}
