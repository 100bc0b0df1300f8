// global_localization_parity_test.cpp — TEST INFRASTRUCTURE ONLY.
//
// The node's global localisation through the host C++ adapter against the reference's own particle filter, in one
// process: the global_localization service body (src/mcl_3dl.cpp:1039-1099, restated here afresh on the reference's
// pf::ParticleFilter, Quat, Vec3 and State6DOF and the shim KdTreeFLANN) vs ParticleFilterB200::globalLocalizationResident
// + downloadResident, then the node's shrink rule (src/mcl_3dl.cpp:875-888) step by step, pf_->resizeParticle vs
// resizeResident.  Every particle must be identical bit for bit.  PCL is absent, so the VoxelGrid of the restated body is
// tests/hostsim/scan_hostsim.cpp's, which is bit-exact with the device.  Built where a checkout of the reference exists
// (make -C oracle -f gl.mk gl-parity); tests/test_gpu_global_localization.py runs it on an H100.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <random>
#include <string>
#include <vector>

#include "../tests/hostsim/scan_hostsim.cpp"

#include <mcl_3dl/chunked_kdtree.h>
#include <mcl_3dl/lidar_measurement_models/lidar_measurement_model_likelihood.h>
#include <mcl_3dl/pf.h>
#include <mcl_3dl/state_6dof.h>
#include <pcl/kdtree/kdtree_flann.h>

#include "../mcl_3dl_b200/host/lidar_measurement_model_b200.h"

using mcl_3dl::ChunkedKdtree;
using mcl_3dl::Quat;
using mcl_3dl::State6DOF;
using mcl_3dl::Vec3;
using PointType = mcl_3dl::LidarMeasurementModelBase::PointType;
using Cloud = pcl::PointCloud<PointType>;
using PFB = mcl_3dl_b200::ParticleFilterB200;
using PFRef = mcl_3dl::pf::ParticleFilter<State6DOF, float, mcl_3dl::ParticleWeightedMeanQuat, std::default_random_engine>;

namespace
{
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

PointType pt(float x, float y, float z)
{
  PointType p;
  p.x = x;
  p.y = y;
  p.z = z;
  p.label = 0;
  return p;
}

int g_fail = 0;

template <typename A, typename B>
void compareSets(A& ref, B& gpu, const char* what)
{
  if (ref.getParticleSize() != gpu.getParticleSize())
  {
    ++g_fail;
    std::fprintf(stderr, "FAIL %s: %zu vs %zu particles\n", what, ref.getParticleSize(), gpu.getParticleSize());
    return;
  }
  size_t bad = 0;
  auto ig = gpu.begin();
  for (auto ir = ref.begin(); ir != ref.end(); ++ir, ++ig)
  {
    const mcl3dl_state a = PFB::toState(ir->state_), b = PFB::toState(ig->state_);
    if (std::memcmp(&a, &b, sizeof(a)) != 0 || std::memcmp(&ir->probability_, &ig->probability_, 4) != 0)
    {
      if (bad < 5)
        std::fprintf(stderr, "FAIL %s particle %zu: pos %.9g %.9g %.9g / %.9g %.9g %.9g, prob %.9g / %.9g\n", what,
                     static_cast<size_t>(ir - ref.begin()), a.pos[0], a.pos[1], a.pos[2], b.pos[0], b.pos[1], b.pos[2],
                     ir->probability_, ig->probability_);
      ++bad;
    }
  }
  if (bad)
    ++g_fail;
  std::printf("%s: %zu particles, %zu differ\n", what, ref.getParticleSize(), bad);
}
}  // namespace

int main(int argc, char** argv)
{
  const int num_particles = argc > 1 ? std::atoi(argv[1]) : 512;
  const double grid = 0.3;
  const int div_yaw = argc > 2 ? std::atoi(argv[2]) : 12;
  std::mt19937 rng(23);
  std::normal_distribution<float> n01(0.f, 1.f);

  // ---- the map: a 10 x 10 m floor, a ceiling at 3 m, two walls and a box
  Cloud::Ptr pc_map_(new Cloud);
  for (float x = 0.05f; x < 10.f; x += 0.1f)
    for (float y = 0.05f; y < 10.f; y += 0.1f)
    {
      pc_map_->push_back(pt(x, y, 0.03f + 0.01f * n01(rng)));
      pc_map_->push_back(pt(x, y, 2.97f + 0.01f * n01(rng)));
    }
  for (float a = 0.05f; a < 10.f; a += 0.1f)
    for (float z = 0.05f; z < 3.f; z += 0.1f)
    {
      pc_map_->push_back(pt(0.03f, a, z));
      pc_map_->push_back(pt(a, 9.97f, z));
    }
  for (float a = 0.f; a <= 1.2f; a += 0.1f)
    for (float b = 0.f; b <= 1.2f; b += 0.1f)
      pc_map_->push_back(pt(4.f + a, 4.f + b, 1.2f));
  pc_map_->header.stamp = 1000;

  const float dist_weight[4] = {1.f, 1.f, 5.f, 0.f};
  auto rep = std::make_shared<XyzRep>();
  rep->setRescaleValues(dist_weight);
  ChunkedKdtree<PointType>::Ptr kdtree_(new ChunkedKdtree<PointType>(20.0, 0.4));
  kdtree_->setPointRepresentation(rep);
  kdtree_->setInputCloud(pc_map_);
  const Quat imu_quat_(0.01f, -0.02f, 0.003f, 0.9997f);

  auto lik_params = std::make_shared<mcl_3dl::LidarMeasurementModelLikelihoodParameters>();
  auto beam_params = std::make_shared<mcl_3dl::LidarMeasurementModelBeamParameters>();
  PFB pf_gpu(num_particles, 7);
  auto batcher = std::make_shared<mcl_3dl_b200::MeasurementBatcher>(&pf_gpu, std::vector<int>{0}, lik_params, beam_params,
                                                                   dist_weight);

  // ---- the service body on the reference filter, VoxelGrid from the device restatement
  PFRef pf_ref(num_particles, 7);
  {
    std::vector<mcl3dl_point> in, ds(pc_map_->size());
    for (const auto& p : pc_map_->points) in.push_back(mcl3dl_point{p.x, p.y, p.z, p.label});
    const float leaf[3] = {static_cast<float>(grid), static_cast<float>(grid), static_cast<float>(grid)};
    long m = hostsim_scan_voxel_grid(in.data(), in.size(), leaf, ds.data());
    if (m < 0)
    {
      ds = in;
      m = static_cast<long>(in.size());
    }
    Cloud::Ptr points(new Cloud);
    for (long i = 0; i < m; ++i) points->push_back(pt(ds[i].x, ds[i].y, ds[i].z));
    pcl::KdTreeFLANN<PointType> kdtree;
    kdtree.setPointRepresentation(rep);
    kdtree.setInputCloud(points);
    Cloud seeds;
    std::vector<int> id(1);
    std::vector<float> sqdist(1);
    for (const auto& p : points->points)
    {
      PointType above = p;
      above.z += 0.01 + grid;
      if (!kdtree.radiusSearch(above, grid, id, sqdist, 1))
        seeds.push_back(p);
    }
    pf_ref.resizeParticle(seeds.size() * div_yaw);
    const float prob = 1.0 / static_cast<float>(seeds.size());
    size_t i = 0;
    for (auto it = pf_ref.begin(); it != pf_ref.end(); ++it, ++i)
    {
      const PointType& s = seeds.points[i / div_yaw];
      const int c = static_cast<int>(i % div_yaw);
      it->probability_ = prob;
      it->probability_bias_ = 1.0;
      it->state_ = State6DOF(Vec3(s.x, s.y, s.z), (Quat(Vec3(0.0, 0.0, 2.0 * M_PI * c / div_yaw)) * imu_quat_).normalized());
    }
    std::printf("reference: %ld downsampled, %zu seeds\n", m, seeds.size());
  }

  // ---- the same through the adapter
  mcl3dl_global_localization_params gp{};
  gp.grid = grid;
  gp.div_yaw = div_yaw;
  gp.imu_quat[0] = imu_quat_.x_;
  gp.imu_quat[1] = imu_quat_.y_;
  gp.imu_quat[2] = imu_quat_.z_;
  gp.imu_quat[3] = imu_quat_.w_;
  for (int k = 0; k < 3; ++k) gp.dist_weight[k] = dist_weight[k];
  const mcl3dl_global_localization_info info = pf_gpu.globalLocalizationResident(*batcher, kdtree_, gp);
  std::printf("device: %llu downsampled, %llu seeds, %llu particles, %.3f ms\n",
              static_cast<unsigned long long>(info.n_downsampled), static_cast<unsigned long long>(info.n_seeds),
              static_cast<unsigned long long>(info.n_particles), info.build_ms);
  pf_gpu.downloadResident(*batcher);
  compareSets(pf_ref, pf_gpu, "seed");

  // ---- the node's shrink after each update: non-uniform posteriors (the same on both), then resizeParticle
  std::uniform_real_distribution<float> u(0.05f, 1.f);
  int step = 0;
  while (static_cast<int>(pf_ref.getParticleSize()) > num_particles)
  {
    auto ig = pf_gpu.begin();
    for (auto ir = pf_ref.begin(); ir != pf_ref.end(); ++ir, ++ig)
      ig->probability_ = ir->probability_ = u(rng) / pf_ref.getParticleSize();
    pf_gpu.uploadResident(*batcher);
    const int reduced = pf_ref.getParticleSize() * 0.75;
    const int next = reduced > num_particles ? reduced : num_particles;
    pf_ref.resizeParticle(next);
    pf_gpu.resizeResident(*batcher, next);
    pf_gpu.downloadResident(*batcher);
    const std::string what = "shrink " + std::to_string(++step);
    compareSets(pf_ref, pf_gpu, what.c_str());
  }
  if (step == 0)
  {
    ++g_fail;
    std::fprintf(stderr, "FAIL: no shrink step ran\n");
  }
  if (g_fail)
  {
    std::fprintf(stderr, "GLOBAL LOCALIZATION PARITY FAILED (%d)\n", g_fail);
    return 1;
  }
  std::printf("GLOBAL LOCALIZATION PARITY OK (%d shrink steps)\n", step);
  return 0;
}
