// match_parity_test.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs the node's matched / unmatched loop (src/mcl_3dl.cpp:770-788) with the reference's own State6DOF::transform and
// ChunkedKdtree::radiusSearch, and the host C++ adapter's MeasurementBatcher::matchOutput (mcl3dl_match_output on the
// device) in the same process, and compares the two clouds bit for bit.  Built only where a checkout of the reference
// exists (make -C oracle adapter), against oracle/shim/; tests/test_gpu_match_output.py runs it on an H100.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>
#include <memory>
#include <random>
#include <vector>

#include <mcl_3dl/chunked_kdtree.h>
#include <mcl_3dl/state_6dof.h>

#include "../mcl_3dl_b200/host/lidar_measurement_model_b200.h"

using namespace mcl_3dl;
using PointType = LidarMeasurementModelBase::PointType;
using Cloud = pcl::PointCloud<PointType>;
using CloudXYZ = pcl::PointCloud<pcl::PointXYZ>;

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

PointType pt(float x, float y, float z, uint32_t label = 0)
{
  PointType p;
  p.x = x;
  p.y = y;
  p.z = z;
  p.label = label;
  return p;
}

// src/mcl_3dl.cpp:770-788 as the node runs it
void nodeLoop(ChunkedKdtree<PointType>::Ptr& kdtree, const State6DOF& e, const Cloud::ConstPtr& pc_local_full,
              double match_output_dist, double unmatch_output_dist, CloudXYZ& pc_match, CloudXYZ& pc_unmatch)
{
  Cloud::Ptr pc_local(new Cloud);
  *pc_local = *pc_local_full;
  e.transform(*pc_local);
  std::vector<int> id(1);
  std::vector<float> sqdist(1);
  const double match_dist_sq = match_output_dist * match_output_dist;
  for (const auto& p : pc_local->points)
  {
    if (!kdtree->radiusSearch(p, unmatch_output_dist, id, sqdist, 1))
      pc_unmatch.points.emplace_back(p.x, p.y, p.z);
    else if (sqdist[0] < match_dist_sq)
      pc_match.points.emplace_back(p.x, p.y, p.z);
  }
}

// bit for bit, except that a NaN equals any NaN: the device and x86 write different NaN payloads
bool sameFloat(float a, float b)
{
  return (std::isnan(a) && std::isnan(b)) || std::memcmp(&a, &b, 4) == 0;
}
bool same(const CloudXYZ& a, const CloudXYZ& b)
{
  if (a.points.size() != b.points.size())
    return false;
  for (size_t i = 0; i < a.points.size(); ++i)
    if (!sameFloat(a.points[i].x, b.points[i].x) || !sameFloat(a.points[i].y, b.points[i].y) ||
        !sameFloat(a.points[i].z, b.points[i].z))
      return false;
  return true;
}
}  // namespace

int main()
{
  std::mt19937 rng(42);
  std::normal_distribution<float> n01(0.f, 1.f);
  std::uniform_real_distribution<float> u01(0.f, 1.f);

  // ---- map: 12 x 12 m floor, two walls and a partition, ~0.1 m spacing, off the 1 m lattice
  Cloud::Ptr map(new Cloud);
  for (float x = 0.05f; x < 12.f; x += 0.1f)
    for (float y = 0.05f; y < 12.f; y += 0.1f)
      map->push_back(pt(x + 0.02f * n01(rng), y + 0.02f * n01(rng), 0.43f + 0.01f * n01(rng)));
  for (float y = 0.05f; y < 12.f; y += 0.1f)
    for (float z = 0.45f; z < 3.4f; z += 0.1f)
    {
      map->push_back(pt(0.37f + 0.01f * n01(rng), y, z));
      map->push_back(pt(11.61f + 0.01f * n01(rng), y, z, 2));
    }
  for (float x = 4.f; x < 6.f; x += 0.1f)
    for (float z = 0.45f; z < 2.4f; z += 0.1f)
      map->push_back(pt(x, 7.71f + 0.01f * n01(rng), z));
  map->header.stamp = 1234;

  // ---- scan in the base frame: map points seen from (6, 4, 0.9) yaw 0.3 with wide noise, points far above the map
  // and non-finite points
  const Vec3 truth_pos(6.f, 4.f, 0.9f);
  const Quat truth_rot(Vec3(0, 0, 1), 0.3f);
  Cloud::Ptr scan(new Cloud);
  std::uniform_int_distribution<size_t> pick(0, map->size() - 1);
  while (scan->size() < 4000)
  {
    const PointType& mp = map->points[pick(rng)];
    const Vec3 local = truth_rot.inv() * (Vec3(mp.x, mp.y, mp.z) - truth_pos);
    scan->push_back(pt(local.x_ + 0.15f * n01(rng), local.y_ + 0.15f * n01(rng), local.z_ + 0.15f * n01(rng),
                       scan->size() % 3));
  }
  for (int i = 0; i < 100; ++i)
    scan->push_back(pt(16.f * u01(rng) - 8.f, 16.f * u01(rng) - 8.f, 5.f + 4.f * u01(rng)));
  scan->push_back(pt(std::numeric_limits<float>::quiet_NaN(), 0.f, 0.f));
  scan->push_back(pt(0.f, std::numeric_limits<float>::infinity(), 0.f));
  // State6DOF::transform normalises the rotation (state_6dof.h:217): leave a little drift in it
  const State6DOF e(truth_pos + Vec3(0.03f, -0.02f, 0.01f), Quat(truth_rot.x_ * 1.0003f, truth_rot.y_, truth_rot.z_ * 1.0003f,
                                                                   truth_rot.w_ * 1.0003f));

  auto lik_params = std::make_shared<LidarMeasurementModelLikelihoodParameters>();
  auto beam_params = std::make_shared<LidarMeasurementModelBeamParameters>();
  struct Config
  {
    float chunk_length, max_search_radius;
    float w[4];
  };
  const Config configs[] = {{20.f, 0.2f, {1.f, 1.f, 1.f, 0.f}}, {1.5f, 0.2f, {1.f, 1.f, 1.f, 0.f}}, {1.f, 0.2f, {1.f, 1.f, 5.f, 0.f}}};
  int fail = 0;
  for (const Config& c : configs)
  {
    auto rep = std::make_shared<XyzRep>();
    rep->setRescaleValues(c.w);
    ChunkedKdtree<PointType>::Ptr kdtree(new ChunkedKdtree<PointType>(c.chunk_length, c.max_search_radius));
    kdtree->setPointRepresentation(rep);
    kdtree->setInputCloud(map);
    mcl_3dl_b200::MeasurementBatcher batcher(nullptr, std::vector<int>{0}, lik_params, beam_params, c.w);
    CloudXYZ ref_m, ref_u, gpu_m, gpu_u;
    nodeLoop(kdtree, e, scan, 0.1, 0.5, ref_m, ref_u);
    batcher.matchOutput(kdtree, e, scan, 0.1, 0.5, c.chunk_length, c.max_search_radius, gpu_m, gpu_u);
    const bool ok = same(ref_m, gpu_m) && same(ref_u, gpu_u) && !ref_m.points.empty() && !ref_u.points.empty() &&
                    ref_m.points.size() + ref_u.points.size() < scan->size();
    std::printf("chunk %.2f, weights (%g, %g, %g): matched %zu / %zu, unmatched %zu / %zu of %zu%s\n", c.chunk_length, c.w[0],
                c.w[1], c.w[2], gpu_m.points.size(), ref_m.points.size(), gpu_u.points.size(), ref_u.points.size(),
                scan->size(), ok ? "" : "  MISMATCH");
    fail += ok ? 0 : 1;
  }
  if (fail)
  {
    std::printf("MATCH OUTPUT PARITY FAILED (%d configurations)\n", fail);
    return 1;
  }
  std::printf("MATCH OUTPUT PARITY OK\n");
  return 0;
}
