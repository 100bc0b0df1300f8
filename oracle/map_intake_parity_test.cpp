// map_intake_parity_test.cpp — TEST INFRASTRUCTURE ONLY.
//
// The node's map callbacks (src/mcl_3dl.cpp:127-153 cbMapcloud / cbMapcloudUpdate, :189 cbPosition's reset,
// :1150-1192 loadMapCloud / cbLoadPCD, :1350-1378 cbMapUpdateTimer) run two ways side by side, in one process with the
// reference's own model sources (make -C oracle -f map_intake.mk map-intake-parity; tests/test_gpu_map_intake.py runs it
// on an H100):
//   host:    fromROSMsg restated (fields by name and type, absent or wrongly typed intensity / label -> 0), the VoxelGrid
//            of tests/hostsim/scan_hostsim.cpp (hostsim_scan_voxel_grid) with the intensity centroid restated beside it,
//            the node's pc_map_ / pc_map2_ / pc_update_ logic, and MeasurementBatcher::setMapCloud(pc_map2_);
//   intake:  MeasurementBatcher::loadMapMessage / loadMapCloud / setMapUpdate / commitMapUpdate / clearMapUpdate, the
//            published map from mapCloud.
// Neither node fills its index.  At every timer tick the published maps must be equal byte for byte (x / y / z /
// intensity / label), and pf_->measure(lambda) through the plugin classes, a resident cycle, the estimate, the matched /
// unmatched clouds and the ray markers must be equal, for both casters.  The sequence: xyzil, xyz, xyzi and xyzl maps
// and patches, organised and padded layouts, a wrongly typed intensity field, two patches before one tick, a patch
// cleared by cbPosition, cbLoadPCD from a host PointXYZIL cloud, a reload with a patch pending, and a patch that grows
// the map's box.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <numeric>
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
#include "../tests/hostsim/scan_hostsim.cpp"

using namespace mcl_3dl;
using PointType = LidarMeasurementModelBase::PointType;
using Cloud = pcl::PointCloud<PointType>;
using CloudXYZ = pcl::PointCloud<pcl::PointXYZ>;
using PF = mcl_3dl_b200::ParticleFilterB200;

namespace pcl
{
// pcl::PointCloud::operator+, which the node's map update uses and the shim leaves out
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

bool sameBits(float a, float b) { return std::memcmp(&a, &b, 4) == 0; }
bool sameVec(const Vec3& a, const Vec3& b) { return sameBits(a.x_, b.x_) && sameBits(a.y_, b.y_) && sameBits(a.z_, b.z_); }
bool sameVecNan(const Vec3& a, const Vec3& b)
{
  const auto one = [](float x, float y) { return (std::isnan(x) && std::isnan(y)) || sameBits(x, y); };
  return one(a.x_, b.x_) && one(a.y_, b.y_) && one(a.z_, b.z_);
}
bool sameFloats(const std::vector<float>& a, const std::vector<float>& b)
{
  return a.size() == b.size() && (a.empty() || std::memcmp(a.data(), b.data(), a.size() * 4) == 0);
}
bool sameXyz(const CloudXYZ& a, const CloudXYZ& b)
{
  if (a.points.size() != b.points.size())
    return false;
  for (size_t i = 0; i < a.points.size(); ++i)
    if (!sameBits(a.points[i].x, b.points[i].x) || !sameBits(a.points[i].y, b.points[i].y) || !sameBits(a.points[i].z, b.points[i].z))
      return false;
  return true;
}
bool sameMaps(const Cloud& a, const Cloud& b)
{
  if (a.points.size() != b.points.size())
    return false;
  for (size_t i = 0; i < a.points.size(); ++i)
  {
    const PointType &p = a.points[i], &q = b.points[i];
    if (!sameBits(p.x, q.x) || !sameBits(p.y, q.y) || !sameBits(p.z, q.z) || !sameBits(p.intensity, q.intensity) || p.label != q.label)
      return false;
  }
  return true;
}
std::vector<float> probabilities(PF& pf)
{
  std::vector<float> p;
  for (auto it = pf.begin(); it != pf.end(); ++it) p.push_back(it->probability_);
  return p;
}

PointType pt(float x, float y, float z, uint32_t label, float intensity)
{
  PointType p;
  p.x = x;
  p.y = y;
  p.z = z;
  p.label = label;
  p.intensity = intensity;
  return p;
}

// ---- messages
struct Layout
{
  uint32_t point_step, ox, oy, oz;
  int32_t io, lo;          // -1: no such field
  uint8_t itype, ltype;    // the fields' datatypes (a wrong type is not read by fromROSMsg)
  uint32_t height, row_pad;
};
const Layout XYZIL{32, 0, 4, 8, 16, 20, sensor_msgs::PointField::FLOAT32, sensor_msgs::PointField::UINT32, 1, 0};
const Layout XYZ_ORG{16, 4, 8, 12, -1, -1, 0, 0, 4, 6};
const Layout XYZI_PAD{20, 8, 12, 16, 4, -1, sensor_msgs::PointField::FLOAT32, 0, 1, 3};
const Layout XYZL_ORG{24, 0, 4, 8, -1, 12, 0, sensor_msgs::PointField::UINT32, 2, 5};
const Layout XYZ_BAD_I{24, 0, 4, 8, 12, 20, sensor_msgs::PointField::FLOAT64, sensor_msgs::PointField::UINT32, 3, 0};

sensor_msgs::PointField field(const char* name, uint32_t offset, uint8_t type)
{
  sensor_msgs::PointField f;
  f.name = name;
  f.offset = offset;
  f.datatype = type;
  f.count = 1;
  return f;
}

sensor_msgs::PointCloud2 makeMsg(const Cloud& pts, const Layout& l, uint64_t stamp)
{
  sensor_msgs::PointCloud2 m;
  m.header.stamp = stamp;
  m.height = l.height;
  m.width = static_cast<uint32_t>(pts.size() / l.height);
  m.point_step = l.point_step;
  m.row_step = m.width * l.point_step + l.row_pad;
  m.fields = {field("x", l.ox, sensor_msgs::PointField::FLOAT32), field("y", l.oy, sensor_msgs::PointField::FLOAT32),
              field("z", l.oz, sensor_msgs::PointField::FLOAT32)};
  if (l.io >= 0)
    m.fields.push_back(field("intensity", l.io, l.itype));
  if (l.lo >= 0)
    m.fields.push_back(field("label", l.lo, l.ltype));
  m.data.assign(static_cast<size_t>(m.height) * m.row_step, 0xA5);
  m.is_dense = 1;
  for (uint32_t r = 0; r < m.height; ++r)
    for (uint32_t c = 0; c < m.width; ++c)
    {
      const PointType& p = pts.points[r * m.width + c];
      uint8_t* d = m.data.data() + static_cast<size_t>(r) * m.row_step + static_cast<size_t>(c) * m.point_step;
      std::memcpy(d + l.ox, &p.x, 4);
      std::memcpy(d + l.oy, &p.y, 4);
      std::memcpy(d + l.oz, &p.z, 4);
      if (l.io >= 0)
        std::memcpy(d + l.io, &p.intensity, 4);
      if (l.lo >= 0)
        std::memcpy(d + l.lo, &p.label, 4);
    }
  return m;
}

// mcl_3dl::fromROSMsg into PointXYZIL, restated: x / y / z FLOAT32 or failure; intensity FLOAT32 / label UINT32 by name
// and type, otherwise the PointXYZIL() default 0
bool fromMsg(const sensor_msgs::PointCloud2& m, Cloud& out)
{
  const auto find = [&](const char* name, uint8_t type) -> int64_t {
    for (const auto& f : m.fields)
      if (f.name == name && f.datatype == type)
        return f.offset;
    return -1;
  };
  const int64_t ox = find("x", sensor_msgs::PointField::FLOAT32), oy = find("y", sensor_msgs::PointField::FLOAT32),
                oz = find("z", sensor_msgs::PointField::FLOAT32);
  if (ox < 0 || oy < 0 || oz < 0 || m.width * m.height == 0)
    return false;
  const int64_t oi = find("intensity", sensor_msgs::PointField::FLOAT32), ol = find("label", sensor_msgs::PointField::UINT32);
  out.points.clear();
  for (uint32_t r = 0; r < m.height; ++r)
    for (uint32_t c = 0; c < m.width; ++c)
    {
      const uint8_t* d = m.data.data() + static_cast<size_t>(r) * m.row_step + static_cast<size_t>(c) * m.point_step;
      PointType p;
      std::memcpy(&p.x, d + ox, 4);
      std::memcpy(&p.y, d + oy, 4);
      std::memcpy(&p.z, d + oz, 4);
      if (oi >= 0)
        std::memcpy(&p.intensity, d + oi, 4);
      if (ol >= 0)
        std::memcpy(&p.label, d + ol, 4);
      out.points.push_back(p);
    }
  out.width = static_cast<uint32_t>(out.points.size());
  out.height = 1;
  out.header.stamp = m.header.stamp;
  return true;
}

// pcl::VoxelGrid over PointXYZIL: hostsim_scan_voxel_grid for x / y / z / label, the intensity centroid restated beside
// it (the voxel's intensities summed in input order over float(cnt), voxels in ascending key order)
Cloud::Ptr voxelGrid(const Cloud& in, const float leaf[3])
{
  const size_t n = in.points.size();
  std::vector<mcl3dl_point> pts(n), ds(std::max<size_t>(n, 1));
  for (size_t i = 0; i < n; ++i) pts[i] = mcl3dl_point{in.points[i].x, in.points[i].y, in.points[i].z, in.points[i].label};
  const long m = hostsim_scan_voxel_grid(pts.data(), n, leaf, ds.data());
  Cloud::Ptr out(new Cloud);
  out->header = in.header;
  if (m < 0)  // unfiltered (the maps here are finite)
  {
    *out = in;
    return out;
  }
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (const auto& p : pts)
  {
    const float v[3] = {p.x, p.y, p.z};
    for (int k = 0; k < 3; ++k)
    {
      mn[k] = std::min(mn[k], v[k]);
      mx[k] = std::max(mx[k], v[k]);
    }
  }
  float inv[3];
  int min_b[3], eb = 0;
  uint32_t div_b[3], cells = 0;
  hostsim_scan_lattice(leaf, mn, mx, inv, min_b, div_b, &cells, &eb);
  std::vector<uint64_t> key(n);
  for (size_t i = 0; i < n; ++i)
  {
    const float v[3] = {pts[i].x, pts[i].y, pts[i].z};
    int64_t ijk[3];
    for (int k = 0; k < 3; ++k)
    {
      volatile float prod = v[k] * inv[k];
      ijk[k] = static_cast<int64_t>(std::floor(prod)) - min_b[k];
    }
    key[i] = ijk[0] + ijk[1] * div_b[0] + ijk[2] * static_cast<uint64_t>(div_b[0]) * div_b[1];
  }
  std::vector<size_t> order(n);
  std::iota(order.begin(), order.end(), size_t(0));
  std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return key[a] < key[b]; });
  long v = 0;
  for (size_t i = 0; i < n;)
  {
    size_t cnt = 1;
    while (i + cnt < n && key[order[i + cnt]] == key[order[i]]) ++cnt;
    float s = 0.0f;
    for (size_t j = 0; j < cnt; ++j)
    {
      volatile float t = s + in.points[order[i + j]].intensity;
      s = t;
    }
    const mcl3dl_point& q = ds[v];
    out->push_back(pt(q.x, q.y, q.z, q.label, s / static_cast<float>(cnt)));
    ++v;
    i += cnt;
  }
  EXPECT(v == m, "host VoxelGrid: %ld voxels against %ld", v, m);
  return out;
}

// ---- the two nodes
const float MAP_LEAF[3] = {0.2f, 0.2f, 0.2f};
const float UPDATE_LEAF[3] = {0.15f, 0.15f, 0.15f};

struct HostNode  // the node's own map code, restated, with setMapCloud in place of kdtree_->setInputCloud
{
  std::shared_ptr<mcl_3dl_b200::MeasurementBatcher> batcher;
  Cloud::Ptr pc_map_, pc_map2_, pc_update_;
  bool has_map_ = false;
  void cbMapcloud(const sensor_msgs::PointCloud2& msg)
  {
    Cloud::Ptr tmp(new Cloud);
    if (!fromMsg(msg, *tmp))
    {
      has_map_ = false;
      return;
    }
    loadMapCloud(tmp);
  }
  void cbLoadPCD(const Cloud::Ptr& cloud) { loadMapCloud(cloud); }
  void loadMapCloud(const Cloud::Ptr& cloud)
  {
    pc_map_ = voxelGrid(*cloud, MAP_LEAF);
    pc_map2_.reset();
    pc_update_.reset();
    has_map_ = true;
    timer(cloud->header.stamp);
  }
  void cbMapcloudUpdate(const sensor_msgs::PointCloud2& msg)
  {
    Cloud::Ptr tmp(new Cloud);
    if (!fromMsg(msg, *tmp))
      return;
    pc_update_ = voxelGrid(*tmp, UPDATE_LEAF);
  }
  void cbPosition() { pc_update_.reset(); }
  void timer(uint64_t now)
  {
    if (!has_map_)
      return;
    if (pc_update_)
    {
      if (!pc_map2_)
        pc_map2_.reset(new Cloud);
      *pc_map2_ = *pc_map_ + *pc_update_;
      pc_update_.reset();
      pc_map2_->header.stamp = now;
    }
    else
    {
      if (pc_map2_)
        return;
      pc_map2_ = pc_map_;
    }
    batcher->setMapCloud(pc_map2_);
  }
  Cloud published() const { return *pc_map2_; }
};

struct IntakeNode
{
  std::shared_ptr<mcl_3dl_b200::MeasurementBatcher> batcher;
  void cbMapcloud(const sensor_msgs::PointCloud2& msg) { EXPECT(batcher->loadMapMessage(msg, MAP_LEAF, msg.header.stamp), "load"); }
  void cbLoadPCD(const Cloud::Ptr& cloud) { EXPECT(batcher->loadMapCloud(*cloud, MAP_LEAF, cloud->header.stamp), "load PCD"); }
  void cbMapcloudUpdate(const sensor_msgs::PointCloud2& msg) { EXPECT(batcher->setMapUpdate(msg, UPDATE_LEAF), "patch"); }
  void cbPosition() { batcher->clearMapUpdate(); }
  void timer(uint64_t now) { EXPECT(batcher->commitMapUpdate(now), "commit"); }
  Cloud published() const
  {
    Cloud c;
    batcher->mapCloud(c);
    return c;
  }
};

// a dense raw map: floor and walls at 0.07 m with jitter, intensities and labels
Cloud::Ptr rawMap(std::mt19937& rng, size_t multiple_of)
{
  std::normal_distribution<float> n01(0.f, 1.f);
  std::uniform_real_distribution<float> u(0.f, 100.f);
  Cloud::Ptr map(new Cloud);
  for (float x = 0.03f; x < 12.f; x += 0.07f)
    for (float y = 0.03f; y < 12.f; y += 0.07f) map->push_back(pt(x + 0.01f * n01(rng), y + 0.01f * n01(rng), 0.02f * n01(rng), 0, u(rng)));
  for (float y = 0.03f; y < 12.f; y += 0.07f)
    for (float z = 0.03f; z < 3.f; z += 0.07f)
    {
      map->push_back(pt(0.02f * n01(rng), y, z, 1, u(rng)));
      map->push_back(pt(12.f + 0.02f * n01(rng), y, z, 2, u(rng)));
    }
  while (map->points.size() % multiple_of) map->points.pop_back();
  map->width = static_cast<uint32_t>(map->points.size());
  map->height = 1;
  return map;
}

Cloud::Ptr rawBox(std::mt19937& rng, float x0, float y0, float size, uint32_t label)
{
  std::uniform_real_distribution<float> u(0.f, 50.f);
  Cloud::Ptr p(new Cloud);
  for (float a = 0.f; a <= size; a += 0.06f)
    for (float b = 0.f; b <= size; b += 0.06f)
    {
      p->push_back(pt(x0 + a, y0, b, label, u(rng)));
      p->push_back(pt(x0 + a, y0 + size, b, label, u(rng)));
      p->push_back(pt(x0, y0 + a, b, label, u(rng)));
      p->push_back(pt(x0 + size, y0 + a, b, label, u(rng)));
    }
  while (p->points.size() % 12) p->points.pop_back();  // every layout's height divides it
  return p;
}

Cloud::Ptr makeScan(std::mt19937& rng, const Vec3& truth_pos, const Quat& truth_rot, size_t n_origins)
{
  std::uniform_real_distribution<float> u(0.f, 1.f);
  Cloud::Ptr scan(new Cloud);
  for (int i = 0; i < 500; ++i)
  {
    Vec3 w;
    const int face = i % 3;
    if (face == 0)
      w = Vec3(12.f * u(rng), 12.f * u(rng), 0.f);
    else
      w = Vec3(face == 1 ? 0.f : 12.f, 12.f * u(rng), 3.f * u(rng));
    const Vec3 l = truth_rot.inv() * (w - truth_pos);
    PointType p = pt(l.x_, l.y_, l.z_, static_cast<uint32_t>(i % n_origins), 0.f);
    scan->push_back(p);
  }
  return scan;
}

using Models = std::map<std::string, LidarMeasurementModelBase::Ptr>;

void runCycle(Models& m, PF& pf, ChunkedKdtree<PointType>::Ptr& kdtree, const Cloud::ConstPtr& scan,
              const PointCloudRandomSampler<PointType>& sampler, const std::vector<Vec3>& origins, std::vector<float>& out)
{
  std::map<std::string, Cloud::Ptr> pc_locals;
  for (const auto& lm : m)
  {
    lm.second->setGlobalLocalizationStatus(pf.getParticleSize(), pf.getParticleSize());
    pc_locals[lm.first] = lm.second->filter(scan, sampler);
  }
  pf.measure([&](const State6DOF& s) -> float {
    float likelihood = 1;
    for (const auto& lm : m) likelihood *= lm.second->measure(kdtree, pc_locals[lm.first], origins, s).likelihood;
    out.push_back(likelihood);
    return likelihood;
  });
}

void run(bool dda)
{
  const float w[4] = {1.f, 1.f, 5.f, 0.f};
  auto lik_params = std::make_shared<LidarMeasurementModelLikelihoodParameters>();
  lik_params->num_points_default_ = 96;
  auto beam_params = std::make_shared<LidarMeasurementModelBeamParameters>();
  beam_params->num_points_default_ = 24;
  beam_params->use_raycast_using_dda_ = dda;
  auto rep = std::make_shared<XyzRep>();
  rep->setRescaleValues(w);
  ChunkedKdtree<PointType>::Ptr kd_a(new ChunkedKdtree<PointType>(20.0, 0.4)), kd_b(new ChunkedKdtree<PointType>(20.0, 0.4));
  kd_a->setPointRepresentation(rep);
  kd_b->setPointRepresentation(rep);
  PF pf_a(200, 7), pf_b(200, 7);
  const Vec3 truth_pos(6.f, 4.f, 0.5f);
  const Quat truth_rot(Vec3(0, 0, 1), 0.3f);
  const State6DOF truth(truth_pos, truth_rot);
  const State6DOF sigma(Vec3(0.3f, 0.3f, 0.05f), Vec3(0.02f, 0.02f, 0.1f));
  const std::vector<Vec3> origins = {Vec3(0.f, 0.f, 0.3f), Vec3(0.2f, -0.1f, 0.25f)};
  HostNode a;
  IntakeNode b;
  a.batcher = std::make_shared<mcl_3dl_b200::MeasurementBatcher>(&pf_a, std::vector<int>{0}, lik_params, beam_params, w);
  b.batcher = std::make_shared<mcl_3dl_b200::MeasurementBatcher>(&pf_b, std::vector<int>{0}, lik_params, beam_params, w);
  Models ma, mb;
  ma["likelihood"] = std::make_shared<mcl_3dl_b200::LidarMeasurementModelLikelihoodB200>(lik_params, a.batcher);
  ma["beam"] = std::make_shared<mcl_3dl_b200::LidarMeasurementModelBeamB200>(beam_params, a.batcher);
  mb["likelihood"] = std::make_shared<mcl_3dl_b200::LidarMeasurementModelLikelihoodB200>(lik_params, b.batcher);
  mb["beam"] = std::make_shared<mcl_3dl_b200::LidarMeasurementModelBeamB200>(beam_params, b.batcher);
  const HeadSampler sampler;
  std::mt19937 rng(dda ? 5 : 6);
  Cloud::Ptr scan = makeScan(rng, truth_pos, truth_rot, origins.size());
  const char* caster = dda ? "dda" : "kd";
  int tick = 0;

  const auto check = [&](const char* what) {
    ++tick;
    const Cloud pa = a.published(), pb = b.published();
    EXPECT(!pa.points.empty() && sameMaps(pa, pb), "%s tick %d (%s): published maps (%zu / %zu points)", caster, tick, what,
           pa.points.size(), pb.points.size());
    pf_a.init(truth, sigma);
    pf_b.init(truth, sigma);
    std::vector<float> la, lb;
    runCycle(ma, pf_a, kd_a, scan, sampler, origins, la);
    runCycle(mb, pf_b, kd_b, scan, sampler, origins, lb);
    EXPECT(la.size() == 200 && sameFloats(la, lb), "%s tick %d (%s): per-particle likelihoods", caster, tick, what);
    EXPECT(sameFloats(probabilities(pf_a), probabilities(pf_b)), "%s tick %d (%s): posteriors", caster, tick, what);
    std::map<std::string, Cloud::Ptr> pc_a, pc_b;
    for (const auto& lm : ma) pc_a[lm.first] = lm.second->filter(scan, sampler);
    for (const auto& lm : mb) pc_b[lm.first] = lm.second->filter(scan, sampler);
    pf_a.uploadResident(*a.batcher);
    pf_b.uploadResident(*b.batcher);
    const auto ra = pf_a.measureResident(*a.batcher, kd_a, pc_a["likelihood"], pc_a["beam"], origins, 0.0f);
    const auto rb = pf_b.measureResident(*b.batcher, kd_b, pc_b["likelihood"], pc_b["beam"], origins, 0.0f);
    EXPECT(ra.match_ratio_min == rb.match_ratio_min && ra.match_ratio_max == rb.match_ratio_max && ra.kept == rb.kept,
           "%s tick %d (%s): resident summary", caster, tick, what);
    const mcl3dl_estimate ea = pf_a.estimateResident(*a.batcher, nullptr, 1.0f, 1.0f);
    const mcl3dl_estimate eb = pf_b.estimateResident(*b.batcher, nullptr, 1.0f, 1.0f);
    EXPECT(std::memcmp(&ea, &eb, sizeof(ea)) == 0, "%s tick %d (%s): estimate", caster, tick, what);
    pf_a.downloadResident(*a.batcher);
    pf_b.downloadResident(*b.batcher);
    EXPECT(sameFloats(probabilities(pf_a), probabilities(pf_b)), "%s tick %d (%s): resident posteriors", caster, tick, what);
    State6DOF e(Vec3(ea.mean_biased.px, ea.mean_biased.py, ea.mean_biased.pz),
                Quat(ea.mean_biased.qx, ea.mean_biased.qy, ea.mean_biased.qz, ea.mean_biased.qw));
    e.rot_.normalize();
    CloudXYZ m_a, u_a, m_b, u_b;
    a.batcher->matchOutput(kd_a, e, scan, 0.1, 0.5, 20.f, 0.4f, m_a, u_a);
    b.batcher->matchOutput(kd_b, e, scan, 0.1, 0.5, 20.f, 0.4f, m_b, u_b);
    EXPECT(m_a.size() > 0 && sameXyz(m_a, m_b) && sameXyz(u_a, u_b), "%s tick %d (%s): matched / unmatched", caster, tick, what);
    std::vector<mcl_3dl_b200::MeasurementBatcher::BeamRay> ba, bb;
    a.batcher->castBeams(e, pc_a["beam"], origins, ba);
    b.batcher->castBeams(e, pc_b["beam"], origins, bb);
    bool same = ba.size() == bb.size() && !ba.empty();
    for (size_t i = 0; same && i < ba.size(); ++i)
      same = sameVec(ba[i].begin, bb[i].begin) && sameVec(ba[i].end, bb[i].end) && sameVecNan(ba[i].pos, bb[i].pos) &&
             ba[i].status == bb[i].status;
    EXPECT(same, "%s tick %d (%s): ray markers", caster, tick, what);
    std::printf("%s tick %d (%s): map %zu points, %zu matched / %zu unmatched, %zu rays\n", caster, tick, what, pa.points.size(),
                m_a.size(), u_a.size(), ba.size());
  };
  const auto both = [&](auto f) {
    f(a);
    f(b);
  };
  uint64_t now = 1000;
  // 1. an xyzil map (the node's own type), then patches: xyz (organised, padded) replaced before the tick by xyzi
  //    (padded, intensity first)
  Cloud::Ptr raw = rawMap(rng, 1);
  const sensor_msgs::PointCloud2 map1 = makeMsg(*raw, XYZIL, now);
  both([&](auto& n) { n.cbMapcloud(map1); });
  check("xyzil map");
  const sensor_msgs::PointCloud2 p1 = makeMsg(*rawBox(rng, 3.f, 3.f, 1.0f, 3), XYZ_ORG, 0);
  const sensor_msgs::PointCloud2 p2 = makeMsg(*rawBox(rng, 7.f, 5.f, 1.2f, 4), XYZI_PAD, 0);
  both([&](auto& n) { n.cbMapcloudUpdate(p1); });
  both([&](auto& n) { n.cbMapcloudUpdate(p2); });
  ++now;
  both([&](auto& n) { n.timer(now); });
  check("second patch replaced the first");
  // 2. an xyzl patch cleared by cbPosition: the tick changes nothing
  const sensor_msgs::PointCloud2 p3 = makeMsg(*rawBox(rng, 2.f, 8.f, 0.8f, 5), XYZL_ORG, 0);
  both([&](auto& n) { n.cbMapcloudUpdate(p3); });
  both([&](auto& n) { n.cbPosition(); });
  ++now;
  both([&](auto& n) { n.timer(now); });
  check("patch cleared");
  // 3. a patch with a FLOAT64 "intensity" (not read: 0), organised
  const sensor_msgs::PointCloud2 p4 = makeMsg(*rawBox(rng, 8.f, 8.f, 0.9f, 6), XYZ_BAD_I, 0);
  both([&](auto& n) { n.cbMapcloudUpdate(p4); });
  ++now;
  both([&](auto& n) { n.timer(now); });
  check("wrongly typed intensity");
  // 4. a patch that grows the map's box
  const sensor_msgs::PointCloud2 p5 = makeMsg(*rawBox(rng, 12.5f, 4.f, 1.0f, 7), XYZIL, 0);
  both([&](auto& n) { n.cbMapcloudUpdate(p5); });
  ++now;
  both([&](auto& n) { n.timer(now); });
  check("patch grows the box");
  // 5. a reload with a patch pending (the patch is dropped): cbLoadPCD from a host PointXYZIL cloud
  both([&](auto& n) { n.cbMapcloudUpdate(p2); });
  Cloud::Ptr pcd = rawMap(rng, 1);
  pcd->header.stamp = ++now;
  both([&](auto& n) { n.cbLoadPCD(pcd); });
  ++now;
  both([&](auto& n) { n.timer(now); });
  check("cbLoadPCD with a patch pending");
  // 6. maps without intensity / label: xyz organised and padded, then xyzi, then xyzl
  Cloud::Ptr raw2 = rawMap(rng, 12);
  for (const Layout* l : {&XYZ_ORG, &XYZI_PAD, &XYZL_ORG})
  {
    const sensor_msgs::PointCloud2 m = makeMsg(*raw2, *l, ++now);
    both([&](auto& n) { n.cbMapcloud(m); });
    check(l == &XYZ_ORG ? "xyz map" : l == &XYZI_PAD ? "xyzi map" : "xyzl map");
  }
  EXPECT(!kd_a->getInputCloud() && !kd_b->getInputCloud(), "%s: an index was filled", caster);
  EXPECT(b.batcher->mapIntakeLoads() == 5 && b.batcher->mapIntakeCommits() == 3, "%s: intake loads %zu, commits %zu", caster,
         b.batcher->mapIntakeLoads(), b.batcher->mapIntakeCommits());
  std::printf("%s: %d ticks, intake %zu loads / %zu commits, host path %zu appends / %zu restages\n", caster, tick,
              b.batcher->mapIntakeLoads(), b.batcher->mapIntakeCommits(), a.batcher->mapAppends(), a.batcher->mapRestages());
}
}  // namespace

int main()
{
  run(true);
  run(false);
  if (g_fail)
  {
    std::fprintf(stderr, "MAP INTAKE PARITY FAILED (%d)\n", g_fail);
    return 1;
  }
  std::printf("map intake parity ok\n");
  return 0;
}
