// ref_driver.cpp — TEST INFRASTRUCTURE ONLY.
//
// Thin C-ABI driver around the REFERENCE's own, unmodified hot-path sources.  It is compiled
// (oracle/Makefile, target _ref) together with
//     $(REFERENCE)/src/lidar_measurement_model_likelihood.cpp
//     $(REFERENCE)/src/lidar_measurement_model_beam.cpp
// and the reference headers they include, where they lie, against the stand-in headers in
// oracle/shim/ (PCL, Eigen, ROS are not installed here).  Output: oracle/_ref/libmcl3dl_ref.so,
// git-ignored.  No reference source is copied into this repository.
//
// What it is for: pinning oracle/mcl3dl_oracle.cpp (the repo-owned restatement) to the behaviour
// of the real reference code, generating tests/golden/*.json, and serving as the
// cpu_baseline {"kind": "reference"} arm of bench.py.
#include <cmath>
#include <cstring>
#include <memory>
#include <thread>
#include <vector>

#include <mcl_3dl/chunked_kdtree.h>
#include <mcl_3dl/lidar_measurement_models/lidar_measurement_model_beam.h>
#include <mcl_3dl/lidar_measurement_models/lidar_measurement_model_likelihood.h>
#include <mcl_3dl/motion_prediction_models/motion_prediction_model_differential_drive.h>
#include <mcl_3dl/parameters.h>
#include <mcl_3dl/nd.h>
#include <mcl_3dl/pf.h>
#include <mcl_3dl/point_types.h>
#include <mcl_3dl/quat.h>
#include <mcl_3dl/raycasts/raycast_using_dda.h>
#include <mcl_3dl/raycasts/raycast_using_kdtree.h>
#include <mcl_3dl/state_6dof.h>
#include <mcl_3dl/vec3.h>

#include "oracle_api.h"

using mcl_3dl::ChunkedKdtree;
using mcl_3dl::LidarMeasurementModelBeam;
using mcl_3dl::LidarMeasurementModelLikelihood;
using mcl_3dl::Quat;
using mcl_3dl::State6DOF;
using mcl_3dl::Vec3;
using PointType = mcl_3dl::LidarMeasurementModelBase::PointType;
using Cloud = pcl::PointCloud<PointType>;

namespace
{
// Same shape as MCL3dlNode::MyPointRepresentation (src/mcl_3dl.cpp:109-126), which is a private
// nested class of the node and therefore cannot be named from here.
class XyzRepresentation : public pcl::PointRepresentation<PointType>
{
public:
  XyzRepresentation()
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

Cloud::Ptr toCloud(const mcl3dl_point* pts, size_t n)
{
  Cloud::Ptr pc(new Cloud);
  pc->points.resize(n);
  for (size_t i = 0; i < n; ++i)
  {
    PointType p;
    p.x = pts[i].x;
    p.y = pts[i].y;
    p.z = pts[i].z;
    p.label = pts[i].label;
    pc->points[i] = p;
  }
  pc->width = 1;
  pc->height = static_cast<uint32_t>(n);
  return pc;
}
}  // namespace

struct mcl3dl_cpu
{
  Cloud::Ptr map;
  ChunkedKdtree<PointType>::Ptr kdtree;
  std::shared_ptr<XyzRepresentation> rep;
  std::shared_ptr<mcl_3dl::LidarMeasurementModelLikelihoodParameters> lik_params;
  std::shared_ptr<mcl_3dl::LidarMeasurementModelBeamParameters> beam_params;
  std::shared_ptr<LidarMeasurementModelLikelihood> lik;
  std::vector<std::shared_ptr<LidarMeasurementModelBeam>> beams;  // one per thread (mutable raycaster)
  float dist_weight[4];
  bool tally = true;  // also drive getBeamStatus per ray to fill n_short/n_hit/n_long
};

extern "C" {

const char* mcl3dl_cpu_kind(void)
{
  return "reference";
}

mcl3dl_cpu* mcl3dl_cpu_create(const mcl3dl_point* pts, size_t n, const mcl3dl_lik_params* lik,
                              const mcl3dl_cpu_beam_raw* beam, float chunk_length, float max_search_radius)
{
  auto* h = new mcl3dl_cpu;
  h->map = toCloud(pts, n);
  h->map->header.stamp = 1;
  h->lik_params = std::make_shared<mcl_3dl::LidarMeasurementModelLikelihoodParameters>();
  h->dist_weight[0] = h->dist_weight[1] = h->dist_weight[2] = 1.0f;
  h->dist_weight[3] = 0.0f;
  bool rescale = false;
  if (lik)
  {
    h->lik_params->match_weight_ = lik->match_weight;
    h->lik_params->match_dist_min_ = lik->match_dist_min;
    h->lik_params->match_dist_flat_ = lik->match_dist_flat;
    for (int k = 0; k < 3; ++k)
    {
      h->dist_weight[k] = lik->dist_weight[k];
      if (lik->dist_weight[k] != 1.0f)
        rescale = true;
    }
  }
  h->beam_params = std::make_shared<mcl_3dl::LidarMeasurementModelBeamParameters>();
  if (beam)
  {
    h->beam_params->map_grid_x_ = beam->map_grid_x;
    h->beam_params->map_grid_y_ = beam->map_grid_y;
    h->beam_params->map_grid_z_ = beam->map_grid_z;
    h->beam_params->num_points_default_ = beam->num_points_default;
    h->beam_params->beam_likelihood_min_ = beam->beam_likelihood_min;
    h->beam_params->ang_total_ref_ = beam->ang_total_ref;
    h->beam_params->filter_label_max_ = beam->filter_label_max;
    h->beam_params->hit_range_ = beam->hit_range;
    h->beam_params->add_penalty_short_only_mode_ = beam->add_penalty_short_only_mode != 0;
    h->beam_params->use_raycast_using_dda_ = beam->use_raycast_using_dda != 0;
    h->beam_params->ray_angle_half_ = beam->ray_angle_half;
    h->beam_params->dda_grid_size_ = beam->dda_grid_size;
  }
  else
  {
    h->beam_params->use_raycast_using_dda_ = true;
  }
  h->lik = std::make_shared<LidarMeasurementModelLikelihood>(h->lik_params);
  h->beams.push_back(std::make_shared<LidarMeasurementModelBeam>(h->beam_params));

  // configure() order of the node: src/mcl_3dl.cpp:1270,1326-1329 then setInputCloud :1369
  h->kdtree.reset(new ChunkedKdtree<PointType>(chunk_length, max_search_radius));
  if (rescale)
  {
    h->rep = std::make_shared<XyzRepresentation>();
    h->rep->setRescaleValues(h->dist_weight);
    h->kdtree->setPointRepresentation(h->rep);
  }
  h->kdtree->setInputCloud(h->map);
  return h;
}

void mcl3dl_cpu_destroy(mcl3dl_cpu* h)
{
  delete h;
}

static void measureRange(mcl3dl_cpu* h, LidarMeasurementModelBeam& beam, const mcl3dl_pose* poses, size_t b,
                         size_t e, const Cloud::ConstPtr& pc_lik, const Cloud::ConstPtr& pc_beam,
                         const std::vector<Vec3>& origins, mcl3dl_result* out, uint8_t* status)
{
  for (size_t i = b; i < e; ++i)
  {
    const State6DOF s(Vec3(poses[i].px, poses[i].py, poses[i].pz),
                      Quat(poses[i].qx, poses[i].qy, poses[i].qz, poses[i].qw));
    mcl3dl_result r;
    std::memset(&r, 0, sizeof(r));
    if (out)
    {
      // map-key order of the node's loop: "beam" then "likelihood" (src/mcl_3dl.cpp:409-415)
      const mcl_3dl::LidarMeasurementResult rb = beam.measure(h->kdtree, pc_beam, origins, s);
      r.score_beam = rb.likelihood;
      const mcl_3dl::LidarMeasurementResult rl = h->lik->measure(h->kdtree, pc_lik, origins, s);
      r.score_like = rl.likelihood;
      const size_t nl = pc_lik ? pc_lik->size() : 0;
      r.match_cnt = static_cast<uint32_t>(std::lround(rl.quality * static_cast<float>(nl)));
    }
    // Status tallies: measure() only returns the product, so the per-ray loop of
    // lidar_measurement_model_beam.cpp:138-150 is driven here through the public getBeamStatus().
    if ((h->tally || status) && pc_beam && pc_beam->size())
    {
      Cloud pc_particle = *pc_beam;
      s.transform(pc_particle);
      size_t j = 0;
      for (auto& p : pc_particle.points)
      {
        mcl_3dl::Raycast<PointType>::CastResult point;
        const auto st = beam.getBeamStatus(h->kdtree, s.pos_ + s.rot_ * origins[p.label], Vec3(p.x, p.y, p.z), point);
        const int code = st == LidarMeasurementModelBeam::BeamStatus::SHORT ? 0 :
                         st == LidarMeasurementModelBeam::BeamStatus::HIT   ? 1 :
                         st == LidarMeasurementModelBeam::BeamStatus::LONG  ? 2 : 3;
        if (code == 0) r.n_short++;
        if (code == 1) r.n_hit++;
        if (code == 2) r.n_long++;
        if (status) status[i * pc_beam->size() + j] = static_cast<uint8_t>(code);
        ++j;
      }
    }
    if (out) out[i] = r;
  }
}

static int runMeasure(mcl3dl_cpu* h, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* lik_pts, size_t n_lik,
                      const mcl3dl_point* beam_pts, size_t n_beam, const float* origins_xyz, size_t n_origins,
                      mcl3dl_result* out, uint8_t* status, int n_threads)
{
  if (!h) return MCL3DL_ERR_INVALID_ARG;
  for (size_t j = 0; j < n_beam; ++j)
    if (beam_pts[j].label >= n_origins) return MCL3DL_ERR_INVALID_ARG;
  Cloud::ConstPtr pc_lik = toCloud(lik_pts, n_lik);
  Cloud::ConstPtr pc_beam = toCloud(beam_pts, n_beam);
  std::vector<Vec3> origins;
  for (size_t k = 0; k < n_origins; ++k)
    origins.emplace_back(origins_xyz[3 * k], origins_xyz[3 * k + 1], origins_xyz[3 * k + 2]);
  if (n_threads < 1) n_threads = 1;
  while (static_cast<int>(h->beams.size()) < n_threads)
    h->beams.push_back(std::make_shared<LidarMeasurementModelBeam>(h->beam_params));
  if (n_threads == 1)
  {
    measureRange(h, *h->beams[0], poses, 0, P, pc_lik, pc_beam, origins, out, status);
    return MCL3DL_OK;
  }
  std::vector<std::thread> th;
  for (int t = 0; t < n_threads; ++t)
  {
    const size_t b = P * t / n_threads, e = P * (t + 1) / n_threads;
    th.emplace_back([=]() { measureRange(h, *h->beams[t], poses, b, e, pc_lik, pc_beam, origins, out, status); });
  }
  for (auto& t : th) t.join();
  return MCL3DL_OK;
}

int mcl3dl_cpu_measure(mcl3dl_cpu* h, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* lik_pts, size_t n_lik,
                       const mcl3dl_point* beam_pts, size_t n_beam, const float* origins_xyz, size_t n_origins,
                       mcl3dl_result* out, int n_threads)
{
  return runMeasure(h, poses, P, lik_pts, n_lik, beam_pts, n_beam, origins_xyz, n_origins, out, nullptr, n_threads);
}

int mcl3dl_cpu_beam_status(mcl3dl_cpu* h, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* beam_pts,
                           size_t n_beam, const float* origins_xyz, size_t n_origins, uint8_t* status)
{
  return runMeasure(h, poses, P, nullptr, 0, beam_pts, n_beam, origins_xyz, n_origins, nullptr, status, 1);
}

int mcl3dl_cpu_set_tally(mcl3dl_cpu* h, int enable)
{
  h->tally = enable != 0;
  return MCL3DL_OK;
}

int mcl3dl_cpu_beam_params(mcl3dl_cpu* h, mcl3dl_beam_params* out)
{
  // The derived members are private in the reference class; expose what is observable and
  // recompute the rest with the same expressions the constructor path evaluates
  // (lidar_measurement_model_beam.cpp:60-66) — used only to cross-check the other two derivations.
  const auto& p = *h->beam_params;
  out->map_grid_size[0] = p.map_grid_x_;
  out->map_grid_size[1] = p.map_grid_y_;
  out->map_grid_size[2] = p.map_grid_z_;
  out->dda_grid_size = p.dda_grid_size_;
  out->ray_angle_half = p.ray_angle_half_;
  out->hit_tolerance = p.hit_range_;
  const float hit_range_sq = std::pow(p.hit_range_, 2);
  out->hit_range_sq = hit_range_sq;
  out->sin_total_ref = h->beams[0]->getSinTotalRef();
  const float bl = std::pow(p.beam_likelihood_min_, 1.0 / static_cast<float>(p.num_points_default_));
  out->beam_likelihood = bl;
  out->beam_likelihood_min = p.beam_likelihood_min_;
  out->filter_label_max = h->beams[0]->getFilterLabelMax();
  out->add_penalty_short_only_mode = p.add_penalty_short_only_mode_ ? 1 : 0;
  out->use_raycast_using_dda = p.use_raycast_using_dda_ ? 1 : 0;
  out->_reserved = 0;
  return MCL3DL_OK;
}

int mcl3dl_cpu_radius_search(mcl3dl_cpu* h, const float q[3], float radius, float* d2)
{
  PointType p;
  p.x = q[0];
  p.y = q[1];
  p.z = q[2];
  std::vector<int> id(1);
  std::vector<float> sqdist(1);
  try
  {
    if (!h->kdtree->radiusSearch(p, radius, id, sqdist, 1))
      return -1;
  }
  catch (const std::runtime_error&)
  {
    return -2;
  }
  if (d2) *d2 = sqdist[0];
  return id[0];
}

int mcl3dl_cpu_dda_walk(const mcl3dl_point* pts, size_t n, const double c[6], const float begin[3],
                        const float end[3], int stop_at_collision, float* centres, uint8_t* collision,
                        int max_out, int* collided_id)
{
  // Same fixture shape as test/src/test_raycast_dda.cpp: PointXYZ cloud, ChunkedKdtree(10.0, 1.0).
  pcl::PointCloud<pcl::PointXYZ> pc;
  for (size_t i = 0; i < n; ++i)
    pc.push_back(pcl::PointXYZ(pts[i].x, pts[i].y, pts[i].z));
  pc.header.stamp = 1;
  mcl_3dl::ChunkedKdtree<pcl::PointXYZ>::Ptr kdtree(new mcl_3dl::ChunkedKdtree<pcl::PointXYZ>(10.0, 1.0));
  const pcl::PointCloud<pcl::PointXYZ>::ConstPtr shared = pc.makeShared();
  kdtree->setInputCloud(shared);
  mcl_3dl::RaycastUsingDDA<pcl::PointXYZ> raycaster(c[0], c[1], c[2], c[3], c[4], c[5]);
  raycaster.setRay(kdtree, Vec3(begin[0], begin[1], begin[2]), Vec3(end[0], end[1], end[2]));
  mcl_3dl::Raycast<pcl::PointXYZ>::CastResult r;
  int k = 0;
  if (collided_id) *collided_id = -1;
  while (raycaster.getNextCastResult(r))
  {
    if (k < max_out)
    {
      centres[3 * k + 0] = r.pos_.x_;
      centres[3 * k + 1] = r.pos_.y_;
      centres[3 * k + 2] = r.pos_.z_;
      collision[k] = r.collision_ ? 1 : 0;
    }
    ++k;
    if (r.collision_)
    {
      if (collided_id && *collided_id < 0)
        *collided_id = static_cast<int>(r.point_ - &shared->points[0]);
      if (stop_at_collision) break;
    }
  }
  return k;
}

int mcl3dl_cpu_kd_walk(const mcl3dl_point* pts, size_t n, const float c[4], const float begin[3], const float end[3],
                       int stop_at_collision, float* positions, uint8_t* collision, float* sin_angle, int max_out,
                       int* collided_id)
{
  pcl::PointCloud<pcl::PointXYZ> pc;
  for (size_t i = 0; i < n; ++i)
    pc.push_back(pcl::PointXYZ(pts[i].x, pts[i].y, pts[i].z));
  mcl_3dl::ChunkedKdtree<pcl::PointXYZ>::Ptr kdtree(new mcl_3dl::ChunkedKdtree<pcl::PointXYZ>(10.0, 1.0));
  const pcl::PointCloud<pcl::PointXYZ>::ConstPtr shared = pc.makeShared();
  kdtree->setInputCloud(shared);
  mcl_3dl::RaycastUsingKDTree<pcl::PointXYZ> raycaster(c[0], c[1], c[2], c[3]);
  raycaster.setRay(kdtree, Vec3(begin[0], begin[1], begin[2]), Vec3(end[0], end[1], end[2]));
  mcl_3dl::Raycast<pcl::PointXYZ>::CastResult r;
  int k = 0;
  if (collided_id) *collided_id = -1;
  while (raycaster.getNextCastResult(r))
  {
    if (k < max_out)
    {
      positions[3 * k + 0] = r.pos_.x_;
      positions[3 * k + 1] = r.pos_.y_;
      positions[3 * k + 2] = r.pos_.z_;
      collision[k] = r.collision_ ? 1 : 0;
      sin_angle[k] = r.sin_angle_;
    }
    ++k;
    if (r.collision_)
    {
      if (collided_id && *collided_id < 0) *collided_id = static_cast<int>(r.point_ - &shared->points[0]);
      if (stop_at_collision) break;
    }
  }
  return k;
}

void mcl3dl_cpu_quat_rotate(const float q[4], const float v[3], float out[3])
{
  const Vec3 r = Quat(q[0], q[1], q[2], q[3]) * Vec3(v[0], v[1], v[2]);
  out[0] = r.x_;
  out[1] = r.y_;
  out[2] = r.z_;
}

void mcl3dl_cpu_transform_point(const mcl3dl_pose* pose, const float v[3], float out[3])
{
  const State6DOF s(Vec3(pose->px, pose->py, pose->pz), Quat(pose->qx, pose->qy, pose->qz, pose->qw));
  pcl::PointCloud<pcl::PointXYZ> pc;
  pc.push_back(pcl::PointXYZ(v[0], v[1], v[2]));
  s.transform(pc);
  out[0] = pc.points[0].x;
  out[1] = pc.points[0].y;
  out[2] = pc.points[0].z;
}

int mcl3dl_cpu_pf_update(float* prob, const float* lik, size_t n, float* entropy)
{
  // Drives the reference's own pf::ParticleFilter<State6DOF>::measure (pf.h:252-279).
  mcl_3dl::pf::ParticleFilter<State6DOF, float, mcl_3dl::ParticleWeightedMeanQuat> pf(static_cast<int>(n));
  size_t i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i)
  {
    it->probability_ = prob[i];
    it->state_.pos_.x_ = static_cast<float>(i);  // tag so the likelihood lambda can find its index
  }
  // replay of the sum the reference forms (pf.h:255-260) to report whether the update was kept
  float sum = 0;
  for (size_t k = 0; k < n; ++k)
  {
    const float w = prob[k] * lik[k];
    sum += w;
  }
  pf.measure([&](const State6DOF& s) -> float { return lik[static_cast<size_t>(s.pos_.x_)]; });
  i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i)
    prob[i] = it->probability_;
  if (entropy) *entropy = pf.getEntropy();
  return sum > 0.0 ? 1 : 0;
}

namespace
{
// pass-through sampler that reports how many points it was asked for (DummySampler of test_beam_likelihood.cpp:47-76)
class RecordingSampler : public mcl_3dl::PointCloudRandomSampler<PointType>
{
public:
  mutable size_t asked = 0;
  Cloud::Ptr sample(const Cloud::ConstPtr& pc, const size_t num) const final
  {
    asked = num;
    Cloud::Ptr out(new Cloud);
    *out = *pc;
    return out;
  }
};
}  // namespace

int mcl3dl_cpu_filter_clip(const mcl3dl_point* pts, size_t n, float clip_near, float clip_far, float clip_z_min,
                           float clip_z_max, uint8_t* keep)
{
  auto params = std::make_shared<mcl_3dl::LidarMeasurementModelLikelihoodParameters>();
  params->clip_near_ = clip_near;
  params->clip_far_ = clip_far;
  params->clip_z_min_ = clip_z_min;
  params->clip_z_max_ = clip_z_max;
  LidarMeasurementModelLikelihood model(params);
  Cloud::Ptr pc = toCloud(pts, n);
  for (size_t i = 0; i < n; ++i) pc->points[i].intensity = static_cast<float>(i);  // tag to recover the survivors
  RecordingSampler sampler;
  const Cloud::Ptr out = model.filter(pc, sampler);
  std::memset(keep, 0, n);
  for (const auto& p : out->points) keep[static_cast<size_t>(p.intensity)] = 1;
  return MCL3DL_OK;
}

size_t mcl3dl_cpu_global_localization_points(size_t num_points_default, size_t num_points_global, size_t num_particles,
                                             size_t current_num_particles)
{
  auto params = std::make_shared<mcl_3dl::LidarMeasurementModelLikelihoodParameters>();
  params->num_points_default_ = num_points_default;
  params->num_points_global_ = num_points_global;
  LidarMeasurementModelLikelihood model(params);
  model.setGlobalLocalizationStatus(num_particles, current_num_particles);
  Cloud::Ptr pc(new Cloud);
  pc->push_back(PointType());
  pc->points[0].x = 1.0f;
  RecordingSampler sampler;
  model.filter(pc, sampler);
  return sampler.asked;
}

int mcl3dl_cpu_motion_predict(const mcl3dl_pose* a, const mcl3dl_pose* b, float time_diff, float tc_lin, float tc_ang,
                              mcl3dl_cpu_motion_state* st, size_t n)
{
  mcl_3dl::MotionPredictionModelDifferentialDrive model(tc_lin, tc_ang);
  const State6DOF prev(Vec3(a->px, a->py, a->pz), Quat(a->qx, a->qy, a->qz, a->qw));
  const State6DOF cur(Vec3(b->px, b->py, b->pz), Quat(b->qx, b->qy, b->qz, b->qw));
  model.setOdoms(prev, cur, time_diff);
  for (size_t i = 0; i < n; ++i)
  {
    State6DOF s(Vec3(st[i].pos[0], st[i].pos[1], st[i].pos[2]), Quat(st[i].rot[0], st[i].rot[1], st[i].rot[2], st[i].rot[3]));
    s.noise_ll_ = st[i].noise_ll;
    s.noise_la_ = st[i].noise_la;
    s.noise_al_ = st[i].noise_al;
    s.noise_aa_ = st[i].noise_aa;
    s.odom_err_integ_lin_ = Vec3(st[i].odom_err_integ_lin[0], st[i].odom_err_integ_lin[1], st[i].odom_err_integ_lin[2]);
    s.odom_err_integ_ang_ = Vec3(st[i].odom_err_integ_ang[0], st[i].odom_err_integ_ang[1], st[i].odom_err_integ_ang[2]);
    model.predict(s);
    st[i].pos[0] = s.pos_.x_;
    st[i].pos[1] = s.pos_.y_;
    st[i].pos[2] = s.pos_.z_;
    st[i].rot[0] = s.rot_.x_;
    st[i].rot[1] = s.rot_.y_;
    st[i].rot[2] = s.rot_.z_;
    st[i].rot[3] = s.rot_.w_;
    for (int k = 0; k < 3; ++k)
    {
      st[i].odom_err_integ_lin[k] = s.odom_err_integ_lin_[k];
      st[i].odom_err_integ_ang[k] = s.odom_err_integ_ang_[k];
    }
  }
  return MCL3DL_OK;
}

namespace
{
// the 1-D state of test/src/test_pf.cpp:38-76
class State1D : public mcl_3dl::pf::ParticleBase<float>
{
public:
  float x;
  float& operator[](const size_t) override { return x; }
  const float& operator[](const size_t) const { return x; }
  size_t size() const override { return 1; }
  explicit State1D(const float v) : x(v) {}
  State1D() : x(0) {}
  void normalize() override {}
};
}  // namespace

int mcl3dl_cpu_pf_resample_1d(const float* probs, const float* states, size_t n, unsigned int seed, float sigma,
                              float* out_states, float* out_probs)
{
  mcl_3dl::pf::ParticleFilter<State1D, float> pf(static_cast<int>(n), seed);
  size_t i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i)
  {
    it->state_.x = states[i];
    it->probability_ = probs[i];
  }
  pf.resample(State1D(sigma));
  i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i)
  {
    out_states[i] = it->state_.x;
    out_probs[i] = it->probability_;
  }
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_resample_6dof(const float* probs, const mcl3dl_cpu_motion_state* st, size_t n, unsigned int seed,
                                const float sp[3], const float sr[3], mcl3dl_cpu_motion_state* out, float* out_probs)
{
  mcl_3dl::pf::ParticleFilter<State6DOF, float, mcl_3dl::ParticleWeightedMeanQuat, std::default_random_engine> pf(
      static_cast<int>(n), seed);
  size_t i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i)
  {
    State6DOF s(Vec3(st[i].pos[0], st[i].pos[1], st[i].pos[2]), Quat(st[i].rot[0], st[i].rot[1], st[i].rot[2], st[i].rot[3]));
    s.noise_ll_ = st[i].noise_ll;
    s.noise_la_ = st[i].noise_la;
    s.noise_al_ = st[i].noise_al;
    s.noise_aa_ = st[i].noise_aa;
    s.odom_err_integ_lin_ = Vec3(st[i].odom_err_integ_lin[0], st[i].odom_err_integ_lin[1], st[i].odom_err_integ_lin[2]);
    s.odom_err_integ_ang_ = Vec3(st[i].odom_err_integ_ang[0], st[i].odom_err_integ_ang[1], st[i].odom_err_integ_ang[2]);
    it->state_ = s;
    it->probability_ = probs[i];
  }
  pf.resample(State6DOF(Vec3(sp[0], sp[1], sp[2]), Vec3(sr[0], sr[1], sr[2])));
  i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i)
  {
    const State6DOF& s = it->state_;
    out[i].pos[0] = s.pos_.x_;
    out[i].pos[1] = s.pos_.y_;
    out[i].pos[2] = s.pos_.z_;
    out[i].rot[0] = s.rot_.x_;
    out[i].rot[1] = s.rot_.y_;
    out[i].rot[2] = s.rot_.z_;
    out[i].rot[3] = s.rot_.w_;
    out[i].noise_ll = s.noise_ll_;
    out[i].noise_la = s.noise_la_;
    out[i].noise_al = s.noise_al_;
    out[i].noise_aa = s.noise_aa_;
    for (int k = 0; k < 3; ++k)
    {
      out[i].odom_err_integ_lin[k] = s.odom_err_integ_lin_[k];
      out[i].odom_err_integ_ang[k] = s.odom_err_integ_ang_[k];
    }
    out_probs[i] = it->probability_;
  }
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_estimate(const float* probs, const mcl3dl_cpu_motion_state* st, size_t n, const mcl3dl_pose* prev,
                           float bias_var_dist, float bias_var_ang, mcl3dl_pose* mean_biased, uint32_t* max_index, float cov[36])
{
  mcl_3dl::pf::ParticleFilter<State6DOF, float, mcl_3dl::ParticleWeightedMeanQuat, std::default_random_engine> pf(
      static_cast<int>(n), 1);
  size_t i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i)
  {
    it->state_ = State6DOF(Vec3(st[i].pos[0], st[i].pos[1], st[i].pos[2]), Quat(st[i].rot[0], st[i].rot[1], st[i].rot[2], st[i].rot[3]));
    it->probability_ = probs[i];
  }
  if (prev)
  {
    // src/mcl_3dl.cpp:436-449
    const State6DOF state_prev(Vec3(prev->px, prev->py, prev->pz), Quat(prev->qx, prev->qy, prev->qz, prev->qw));
    mcl_3dl::NormalLikelihood<float> nl_lin(bias_var_dist);
    mcl_3dl::NormalLikelihood<float> nl_ang(bias_var_ang);
    const auto bias_func = [&state_prev, &nl_lin, &nl_ang](const State6DOF& s, float& p_bias) -> void
    {
      const float lin_diff = (s.pos_ - state_prev.pos_).norm();
      Vec3 axis;
      float ang_diff;
      (s.rot_ * state_prev.rot_.inv()).getAxisAng(axis, ang_diff);
      p_bias = nl_lin(lin_diff) * nl_ang(ang_diff) + 1e-6;
    };
    pf.bias(bias_func);
  }
  else
  {
    const auto bias_func = [](const State6DOF& s, float& p_bias) -> void
    {
      p_bias = 1.0;
    };
    pf.bias(bias_func);
  }
  const State6DOF e = pf.expectationBiased();
  mean_biased->px = e.pos_.x_;
  mean_biased->py = e.pos_.y_;
  mean_biased->pz = e.pos_.z_;
  mean_biased->_pad = 0.0f;
  mean_biased->qx = e.rot_.x_;
  mean_biased->qy = e.rot_.y_;
  mean_biased->qz = e.rot_.z_;
  mean_biased->qw = e.rot_.w_;
  // pf.max() returns the state; recover its index (first maximum, pf.h:361-374)
  uint32_t best = 0;
  float bp = probs[0];
  for (size_t k = 0; k < n; ++k)
    if (bp < probs[k])
    {
      bp = probs[k];
      best = static_cast<uint32_t>(k);
    }
  const State6DOF m = pf.max();
  if (!(m.pos_ == State6DOF(Vec3(st[best].pos[0], st[best].pos[1], st[best].pos[2]), Quat()).pos_))
    return MCL3DL_ERR_INVALID_ARG;
  *max_index = best;
  const std::vector<State6DOF> c = pf.covariance(1.0, 1.0);
  for (int j = 0; j < 6; ++j)
    for (int k = 0; k < 6; ++k) cov[j * 6 + k] = c[j][k];
  return MCL3DL_OK;
}

}  // extern "C"
