// beam_cast_parity_test.cpp — TEST INFRASTRUCTURE ONLY.
//
// Two legs, in one process with the reference's own sources (built where a checkout of the reference exists, make -C
// oracle -f beam_cast.mk beam-cast-parity; tests/test_gpu_beam_cast.py runs it on an H100):
//  (a) markers: the node's ray-marker loop (src/mcl_3dl.cpp:468-478) on the reference's LidarMeasurementModelBeam over a
//      filled ChunkedKdtree, against MeasurementBatcher::castBeams (mcl3dl_beam_cast): status, pos, end and point.pos_
//      bit for bit, for both casters, with and without the label filter, in and out of short-only mode, for host scans
//      and for the scan mcl3dl_scan_prepare left on the device;
//  (b) a node without its CPU map index: a batcher fed by setMapCloud with a ChunkedKdtree that is never filled runs the
//      same sequence as a batcher whose index is filled (pf_->measure(lambda) through the plugin classes, a resident
//      cycle, the estimate, matchOutput, castBeams, globalLocalizationResident and a resize, a map update on the same
//      cloud object, then a new cloud); every output and the counts of appends and restages must be equal byte for byte.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>
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
using CloudXYZ = pcl::PointCloud<pcl::PointXYZ>;
using PF = mcl_3dl_b200::ParticleFilterB200;
using BeamStatus = LidarMeasurementModelBeam::BeamStatus;

namespace pcl
{
// pcl::PointCloud::operator+ (a copy of the left cloud with the right one's points appended), which the node's map
// update uses and the shim leaves out
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

bool sameBits(float a, float b)
{
  return std::memcmp(&a, &b, 4) == 0;
}
bool sameVec(const Vec3& a, const Vec3& b)
{
  return sameBits(a.x_, b.x_) && sameBits(a.y_, b.y_) && sameBits(a.z_, b.z_);
}
// bit for bit, except that a NaN equals any NaN: the device and x86 write different NaN payloads
bool sameVecNan(const Vec3& a, const Vec3& b)
{
  const auto one = [](float x, float y) { return (std::isnan(x) && std::isnan(y)) || sameBits(x, y); };
  return one(a.x_, b.x_) && one(a.y_, b.y_) && one(a.z_, b.z_);
}

struct NodeRay
{
  Vec3 pos, end, point_pos;
  BeamStatus status;
};

// src/mcl_3dl.cpp:468-478 as the node runs it, e already normalised (:462)
std::vector<NodeRay> nodeMarkerLoop(ChunkedKdtree<PointType>::Ptr& kdtree_, const State6DOF& e, const Cloud::ConstPtr& pc_beam,
                                    const std::vector<Vec3>& origins, const std::shared_ptr<LidarMeasurementModelBeam>& beam_model)
{
  std::vector<NodeRay> out;
  pcl::PointCloud<PointType>::Ptr pc_particle_beam(new pcl::PointCloud<PointType>);
  *pc_particle_beam = *pc_beam;
  e.transform(*pc_particle_beam);
  for (const auto& p : pc_particle_beam->points)
  {
    const int beam_header_id = p.label;
    const Vec3 pos = e.pos_ + e.rot_ * origins[beam_header_id];
    const Vec3 end(p.x, p.y, p.z);
    mcl_3dl::Raycast<PointType>::CastResult point;
    const LidarMeasurementModelBeam::BeamStatus beam_status = beam_model->getBeamStatus(kdtree_, pos, end, point);
    out.push_back(NodeRay{pos, end, point.pos_, beam_status});
  }
  return out;
}

// the marker loop's values against castBeams; returns the number of non-LONG rays
size_t compareMarkers(const char* tag, const std::vector<NodeRay>& want, const std::vector<mcl_3dl_b200::MeasurementBatcher::BeamRay>& got)
{
  EXPECT(want.size() == got.size(), "%s: %zu rays vs %zu", tag, want.size(), got.size());
  size_t n_hit = 0;
  for (size_t i = 0; i < want.size() && i < got.size(); ++i)
  {
    const NodeRay& w = want[i];
    const auto& g = got[i];
    EXPECT(w.status == g.status, "%s ray %zu: status %d vs %d", tag, i, static_cast<int>(w.status), static_cast<int>(g.status));
    EXPECT(sameVec(w.pos, g.begin), "%s ray %zu: begin", tag, i);
    EXPECT(sameVec(w.end, g.end), "%s ray %zu: end", tag, i);
    if (w.status != BeamStatus::LONG)
    {
      ++n_hit;
      EXPECT(sameVec(w.point_pos, g.pos), "%s ray %zu: point.pos_ (%.9g %.9g %.9g) vs (%.9g %.9g %.9g)", tag, i, w.point_pos.x_,
             w.point_pos.y_, w.point_pos.z_, g.pos.x_, g.pos.y_, g.pos.z_);
    }
    else
    {
      EXPECT(std::isnan(g.pos.x_) && std::isnan(g.pos.y_) && std::isnan(g.pos.z_), "%s ray %zu: LONG without NaN", tag, i);
    }
  }
  return n_hit;
}

Cloud::Ptr makeMap(std::mt19937& rng)
{
  std::normal_distribution<float> n01(0.f, 1.f);
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
  // a pillar with label 2 in front of the x = 12 wall: filtered when filter_label_max < 2
  for (float z = 0.05f; z < 2.f; z += 0.1f)
    for (float a = 0.f; a < 0.4f; a += 0.1f)
    {
      map->push_back(pt(9.0f + a, 4.0f, z, 2));
      map->push_back(pt(9.0f, 4.0f + a, z, 2));
    }
  map->header.stamp = 1000;
  return map;
}

// An obstacle box at 0.3 m spacing (a patch after cbMapcloudUpdate's VoxelGrid)
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
    }
  return p;
}

// points of `all` seen from (truth_pos, truth_rot) with noise, labels cycling over the origins; some far beyond the map
Cloud::Ptr makeScan(std::mt19937& rng, const Cloud& all, const Vec3& truth_pos, const Quat& truth_rot, size_t n, size_t n_origins)
{
  std::normal_distribution<float> n01(0.f, 1.f);
  std::uniform_int_distribution<size_t> pick(0, all.size() - 1);
  Cloud::Ptr scan(new Cloud);
  while (scan->size() < n)
  {
    const PointType& mp = all.points[pick(rng)];
    const Vec3 local = truth_rot.inv() * (Vec3(mp.x, mp.y, mp.z) - truth_pos);
    if (local.x_ * local.x_ + local.y_ * local.y_ > 49.f)
      continue;
    scan->push_back(pt(local.x_ + 0.05f * n01(rng), local.y_ + 0.05f * n01(rng), local.z_ + 0.05f * n01(rng),
                       static_cast<uint32_t>(scan->size() % n_origins)));
  }
  for (int i = 0; i < 8; ++i)
    scan->push_back(pt(20.f + i, -15.f + 2.f * i, 3.f, static_cast<uint32_t>(i % n_origins)));
  return scan;
}

using Models = std::map<std::string, LidarMeasurementModelBase::Ptr>;

// MCL3dlNode::measure from filter to pf_->measure (src/mcl_3dl.cpp:376-426): per-particle likelihoods and the match
// ratio range
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

template <typename T>
bool sameBytes(const T& a, const T& b)
{
  return std::memcmp(&a, &b, sizeof(T)) == 0;
}
bool sameFloats(const std::vector<float>& a, const std::vector<float>& b)
{
  return a.size() == b.size() && (a.empty() || std::memcmp(a.data(), b.data(), a.size() * 4) == 0);
}
std::vector<float> probabilities(PF& pf)
{
  std::vector<float> p;
  for (auto it = pf.begin(); it != pf.end(); ++it) p.push_back(it->probability_);
  return p;
}
bool sameClouds(const CloudXYZ& a, const CloudXYZ& b)
{
  if (a.points.size() != b.points.size())
    return false;
  for (size_t i = 0; i < a.points.size(); ++i)
    if (!sameBits(a.points[i].x, b.points[i].x) || !sameBits(a.points[i].y, b.points[i].y) || !sameBits(a.points[i].z, b.points[i].z))
      return false;
  return true;
}

// ---- leg (a)
void markers(const Cloud::Ptr& map, const Cloud::Ptr& scan, const State6DOF& e, const std::vector<Vec3>& origins)
{
  struct Config
  {
    bool dda;
    uint32_t filter_label_max;
    bool short_only;
  };
  const Config configs[] = {{true, 0xFFFFFFFFu, true}, {true, 1u, false}, {false, 0xFFFFFFFFu, true}, {false, 1u, false}};
  const float w[4] = {1.f, 1.f, 5.f, 0.f};
  for (const Config& c : configs)
  {
    auto lik_params = std::make_shared<LidarMeasurementModelLikelihoodParameters>();
    auto beam_params = std::make_shared<LidarMeasurementModelBeamParameters>();
    beam_params->use_raycast_using_dda_ = c.dda;
    beam_params->filter_label_max_ = c.filter_label_max;
    beam_params->add_penalty_short_only_mode_ = c.short_only;
    auto rep = std::make_shared<XyzRep>();
    rep->setRescaleValues(w);
    ChunkedKdtree<PointType>::Ptr kdtree_(new ChunkedKdtree<PointType>(20.0, 0.4));
    kdtree_->setPointRepresentation(rep);
    kdtree_->setInputCloud(map);
    auto beam_model = std::make_shared<LidarMeasurementModelBeam>(beam_params);
    mcl_3dl_b200::MeasurementBatcher batcher(nullptr, std::vector<int>{0}, lik_params, beam_params, w);
    batcher.setMapCloud(map);
    char tag[96];
    std::snprintf(tag, sizeof(tag), "%s filter %u short_only %d", c.dda ? "dda" : "kd", c.filter_label_max, c.short_only);
    // host scan
    std::vector<mcl_3dl_b200::MeasurementBatcher::BeamRay> got;
    batcher.castBeams(e, scan, origins, got);
    const size_t n_host = compareMarkers(tag, nodeMarkerLoop(kdtree_, e, scan, origins, beam_model), got);
    // the prepared scan: mcl3dl_scan_prepare's sampled beam scan, read back for the reference loop
    mcl3dl_scan_params sp{};
    sp.downsample[0] = sp.downsample[1] = sp.downsample[2] = 0.1f;
    sp.lik_clip_near = sp.beam_clip_near = 0.5f;
    sp.lik_clip_far = sp.beam_clip_far = 10.f;
    sp.lik_clip_z_min = sp.beam_clip_z_min = -2.f;
    sp.lik_clip_z_max = sp.beam_clip_z_max = 2.f;
    sp.lik_num_points = 16;
    sp.beam_num_points = 300;
    sp.seed = 5;
    std::vector<mcl3dl_point> raw;
    for (const auto& p : scan->points) raw.push_back(mcl3dl_point{p.x, p.y, p.z, p.label});
    mcl3dl_scan_info info;
    batcher.checked(mcl3dl_scan_prepare(batcher.engine(), raw.data(), raw.size(), &sp, &info), "mcl3dl_scan_prepare");
    std::vector<mcl3dl_point> sampled(info.n_beam);
    size_t n_s = 0;
    batcher.checked(mcl3dl_scan_get(batcher.engine(), 4, sampled.data(), sampled.size(), &n_s), "mcl3dl_scan_get");
    Cloud::Ptr pc_beam(new Cloud);
    for (const auto& p : sampled) pc_beam->push_back(pt(p.x, p.y, p.z, p.label));
    batcher.castBeams(e, nullptr, origins, got);
    const std::string ptag = std::string(tag) + " prepared";
    const size_t n_prep = compareMarkers(ptag.c_str(), nodeMarkerLoop(kdtree_, e, pc_beam, origins, beam_model), got);
    EXPECT(n_s > 100 && n_host > 20 && n_prep > 20, "%s: vacuous (%zu prepared rays, %zu / %zu decided)", tag, n_s, n_host, n_prep);
    std::printf("markers %s: %zu host rays (%zu decided), %zu prepared rays (%zu decided)\n", tag, scan->size(), n_host, n_s, n_prep);
  }
}

// ---- leg (b)
void withoutIndex(bool dda, const Cloud::Ptr& pc_map_, const Cloud::Ptr& scan, const State6DOF& truth, const std::vector<Vec3>& origins)
{
  const float w[4] = {1.f, 1.f, 5.f, 0.f};
  auto lik_params = std::make_shared<LidarMeasurementModelLikelihoodParameters>();
  lik_params->num_points_default_ = 96;
  auto beam_params = std::make_shared<LidarMeasurementModelBeamParameters>();
  beam_params->num_points_default_ = 24;
  beam_params->use_raycast_using_dda_ = dda;
  beam_params->filter_label_max_ = 1;
  auto rep = std::make_shared<XyzRep>();
  rep->setRescaleValues(w);
  // node A fills its index (kdtree_->setInputCloud, src/mcl_3dl.cpp:1369); node B constructs it only (:1327-1329) and
  // hands its maps to setMapCloud
  ChunkedKdtree<PointType>::Ptr kdtree_a(new ChunkedKdtree<PointType>(20.0, 0.4)), kdtree_b(new ChunkedKdtree<PointType>(20.0, 0.4));
  kdtree_a->setPointRepresentation(rep);
  kdtree_b->setPointRepresentation(rep);
  PF pf_a(200, 7), pf_b(200, 7);
  const State6DOF sigma(Vec3(0.3f, 0.3f, 0.05f), Vec3(0.02f, 0.02f, 0.1f));
  pf_a.init(truth, sigma);
  pf_b.init(truth, sigma);
  auto batcher_a = std::make_shared<mcl_3dl_b200::MeasurementBatcher>(&pf_a, std::vector<int>{0}, lik_params, beam_params, w);
  auto batcher_b = std::make_shared<mcl_3dl_b200::MeasurementBatcher>(&pf_b, std::vector<int>{0}, lik_params, beam_params, w);
  Models ma, mb;
  ma["likelihood"] = std::make_shared<mcl_3dl_b200::LidarMeasurementModelLikelihoodB200>(lik_params, batcher_a);
  ma["beam"] = std::make_shared<mcl_3dl_b200::LidarMeasurementModelBeamB200>(beam_params, batcher_a);
  mb["likelihood"] = std::make_shared<mcl_3dl_b200::LidarMeasurementModelLikelihoodB200>(lik_params, batcher_b);
  mb["beam"] = std::make_shared<mcl_3dl_b200::LidarMeasurementModelBeamB200>(beam_params, batcher_b);
  const HeadSampler sampler;
  const char* caster = dda ? "dda" : "kd";

  const auto setMap = [&](const Cloud::Ptr& map) {
    kdtree_a->setInputCloud(map);
    batcher_b->setMapCloud(map);
  };
  int round = 0;
  const auto sequence = [&]() {
    ++round;
    // pf_->measure(lambda) through the plugin classes
    std::vector<float> la, lb;
    float amin, amax, bmin, bmax;
    runCycle(ma, pf_a, kdtree_a, scan, sampler, origins, la, amin, amax);
    runCycle(mb, pf_b, kdtree_b, scan, sampler, origins, lb, bmin, bmax);
    EXPECT(la.size() == 200 && sameFloats(la, lb), "%s round %d: per-particle likelihoods", caster, round);
    EXPECT(amin == bmin && amax == bmax, "%s round %d: match ratios", caster, round);
    EXPECT(sameFloats(probabilities(pf_a), probabilities(pf_b)), "%s round %d: posteriors", caster, round);
    // a resident cycle and the estimate
    std::map<std::string, Cloud::Ptr> pc_a, pc_b;
    for (const auto& lm : ma) pc_a[lm.first] = lm.second->filter(scan, sampler);
    for (const auto& lm : mb) pc_b[lm.first] = lm.second->filter(scan, sampler);
    pf_a.uploadResident(*batcher_a);
    pf_b.uploadResident(*batcher_b);
    const auto ra = pf_a.measureResident(*batcher_a, kdtree_a, pc_a["likelihood"], pc_a["beam"], origins, 0.0f);
    const auto rb = pf_b.measureResident(*batcher_b, kdtree_b, pc_b["likelihood"], pc_b["beam"], origins, 0.0f);
    EXPECT(ra.match_ratio_min == rb.match_ratio_min && ra.match_ratio_max == rb.match_ratio_max && ra.kept == rb.kept,
           "%s round %d: resident summary", caster, round);
    const mcl3dl_estimate ea = pf_a.estimateResident(*batcher_a, nullptr, 1.0f, 1.0f);
    const mcl3dl_estimate eb = pf_b.estimateResident(*batcher_b, nullptr, 1.0f, 1.0f);
    EXPECT(sameBytes(ea, eb), "%s round %d: estimate", caster, round);
    pf_a.downloadResident(*batcher_a);
    pf_b.downloadResident(*batcher_b);
    EXPECT(sameFloats(probabilities(pf_a), probabilities(pf_b)), "%s round %d: resident posteriors", caster, round);
    // the estimate e as the node normalises it (:462): matched / unmatched clouds and the ray markers
    State6DOF e(Vec3(ea.mean_biased.px, ea.mean_biased.py, ea.mean_biased.pz),
                Quat(ea.mean_biased.qx, ea.mean_biased.qy, ea.mean_biased.qz, ea.mean_biased.qw));
    e.rot_.normalize();
    CloudXYZ m_a, u_a, m_b, u_b;
    batcher_a->matchOutput(kdtree_a, e, scan, 0.1, 0.5, 20.f, 0.4f, m_a, u_a);
    batcher_b->matchOutput(kdtree_b, e, scan, 0.1, 0.5, 20.f, 0.4f, m_b, u_b);
    EXPECT(m_a.size() + u_a.size() > 0 && sameClouds(m_a, m_b) && sameClouds(u_a, u_b), "%s round %d: matched / unmatched",
           caster, round);
    std::vector<mcl_3dl_b200::MeasurementBatcher::BeamRay> ba, bb;
    batcher_a->castBeams(e, pc_a["beam"], origins, ba);
    batcher_b->castBeams(e, pc_b["beam"], origins, bb);
    bool same = ba.size() == bb.size() && !ba.empty();
    for (size_t i = 0; same && i < ba.size(); ++i)
      same = sameVec(ba[i].begin, bb[i].begin) && sameVec(ba[i].end, bb[i].end) && sameVecNan(ba[i].pos, bb[i].pos) &&
             ba[i].status == bb[i].status;
    EXPECT(same, "%s round %d: ray markers", caster, round);
    std::printf("%s round %d: map %zu points, match ratio [%g, %g], %zu matched / %zu unmatched, %zu rays\n", caster, round,
                kdtree_a->getInputCloud()->size(), amin, amax, m_a.size(), u_a.size(),
                ba.size());
  };

  setMap(pc_map_);
  sequence();
  // global localisation over the staged map, then a resize
  mcl3dl_global_localization_params gp{};
  gp.grid = 0.6;
  gp.div_yaw = 8;
  gp.imu_quat[3] = 1.f;
  for (int k = 0; k < 3; ++k) gp.dist_weight[k] = w[k];
  const mcl3dl_global_localization_info ga = pf_a.globalLocalizationResident(*batcher_a, kdtree_a, gp);
  const mcl3dl_global_localization_info gb = pf_b.globalLocalizationResident(*batcher_b, kdtree_b, gp);
  EXPECT(ga.n_particles > 200 && ga.n_particles == gb.n_particles && ga.n_seeds == gb.n_seeds &&
             sameBits(ga.probability, gb.probability),
         "%s: global localisation %zu vs %zu particles", caster, static_cast<size_t>(ga.n_particles), static_cast<size_t>(gb.n_particles));
  pf_a.resizeResident(*batcher_a, 200);
  pf_b.resizeResident(*batcher_b, 200);
  pf_a.downloadResident(*batcher_a);
  pf_b.downloadResident(*batcher_b);
  bool same_states = true;
  for (auto ia = pf_a.begin(), ib = pf_b.begin(); ia != pf_a.end(); ++ia, ++ib)
    same_states = same_states && sameVec(ia->state_.pos_, ib->state_.pos_) && ia->probability_ == ib->probability_;
  EXPECT(same_states, "%s: particles after global localisation and resize", caster);
  // the particles for the next rounds: back around the truth, the same in both filters
  pf_a.init(truth, sigma);
  pf_b.init(truth, sigma);
  sequence();
  // cbMapUpdateTimer on the same cloud object (pc_map2_ aliases pc_map_): an append
  *pc_map_ = *pc_map_ + *boxPatch(7.0f, 5.0f, 1.2f, 0);
  pc_map_->header.stamp = 2001;
  setMap(pc_map_);
  EXPECT(batcher_b->mapAppends() == 1, "%s: setMapCloud appended (%zu)", caster, batcher_b->mapAppends());
  sequence();
  // a new cloud object: staged whole
  Cloud::Ptr pc_new(new Cloud(*pc_map_));
  *pc_new += *boxPatch(4.0f, 2.5f, 0.9f, 3);
  pc_new->header.stamp = 3000;
  setMap(pc_new);
  sequence();
  EXPECT(batcher_a->mapAppends() == batcher_b->mapAppends() && batcher_a->mapRestages() == batcher_b->mapRestages() &&
             batcher_b->mapAppends() == 1 && batcher_b->mapRestages() == 2,
         "%s: appends %zu / %zu, restages %zu / %zu", caster, batcher_a->mapAppends(), batcher_b->mapAppends(),
         batcher_a->mapRestages(), batcher_b->mapRestages());
  EXPECT(!kdtree_b->getInputCloud(), "%s: node B's index was filled", caster);
  std::printf("%s without the index: %d rounds, %zu appends, %zu restages\n", caster, round, batcher_b->mapAppends(),
              batcher_b->mapRestages());
}
}  // namespace

int main()
{
  std::mt19937 rng(23);
  Cloud::Ptr map = makeMap(rng);
  const Vec3 truth_pos(6.f, 4.f, 0.5f);
  const Quat truth_rot(Vec3(0, 0, 1), 0.3f);
  const std::vector<Vec3> origins = {Vec3(0.f, 0.f, 0.3f), Vec3(0.2f, -0.1f, 0.25f), Vec3(-0.1f, 0.1f, 0.4f)};
  Cloud::Ptr scan = makeScan(rng, *map, truth_pos, truth_rot, 600, origins.size());
  // the pose estimate after e.rot_.normalize() (:462), a little off the truth
  State6DOF e(truth_pos + Vec3(0.03f, -0.02f, 0.01f), Quat(truth_rot.x_ * 1.0003f, truth_rot.y_, truth_rot.z_ * 1.0003f,
                                                            truth_rot.w_ * 1.0003f));
  e.rot_.normalize();
  markers(map, scan, e, origins);
  for (const bool dda : {true, false})
  {
    std::mt19937 r2(31);
    withoutIndex(dda, makeMap(r2), scan, State6DOF(truth_pos, truth_rot), origins);
  }
  if (g_fail)
  {
    std::fprintf(stderr, "BEAM CAST PARITY FAILED (%d)\n", g_fail);
    return 1;
  }
  std::printf("BEAM CAST PARITY OK\n");
  return 0;
}
