// lidar_measurement_model_b200.h — host C++ adapter: the reference's own plugin classes with
// measure() re-routed to the CUDA engine (H100) through the C ABI (include/mcl3dl_b200.h).
//
// Drop-in rule: the ROS node keeps calling exactly what it calls today
//   setGlobalLocalizationStatus / filter      once per model per update  (src/mcl_3dl.cpp:378-383)
//   measure(kdtree, pc, origins, state)       once per particle per model, from inside
//                                             pf_->measure(lambda)        (:402-426, pf.h:252-260)
// and gets the same LidarMeasurementResult values.  The classes below DERIVE from the reference's
// LidarMeasurementModelLikelihood / LidarMeasurementModelBeam, so everything except measure()
// (refreshParameters, filter, setGlobalLocalizationStatus, getMaxSearchRange, getBeamStatus for the
// rviz markers, and the node's dynamic_pointer_cast<LidarMeasurementModelBeam> at :471) is literally
// the reference's code.  Only measure() changes: the first call of an update cycle batches ALL
// particles of the attached pf::ParticleFilter into one mcl3dl_measure() call; later calls return
// the cached record of the matching particle.
//
// This header needs the reference's headers (it lives in the node's build, see INTEGRATION.md); in
// this repository it is compiled only by oracle/adapter_parity_test.cpp against oracle/shim/.
#ifndef MCL_3DL_B200_LIDAR_MEASUREMENT_MODEL_B200_H
#define MCL_3DL_B200_LIDAR_MEASUREMENT_MODEL_B200_H

#include <algorithm>
#include <cstring>
#include <memory>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

#include <mcl_3dl/chunked_kdtree.h>
#include <mcl_3dl/lidar_measurement_model_base.h>
#include <mcl_3dl/lidar_measurement_models/lidar_measurement_model_beam.h>
#include <mcl_3dl/lidar_measurement_models/lidar_measurement_model_likelihood.h>
#include <mcl_3dl/parameters.h>
#include <mcl_3dl/pf.h>
#include <mcl_3dl/state_6dof.h>

#include "mcl3dl_b200.h"

namespace mcl_3dl_b200
{
using mcl_3dl::ChunkedKdtree;
using mcl_3dl::LidarMeasurementResult;
using mcl_3dl::State6DOF;
using mcl_3dl::Vec3;
using PointType = mcl_3dl::LidarMeasurementModelBase::PointType;
using Cloud = pcl::PointCloud<PointType>;
// the filter type the node instantiates (src/mcl_3dl.cpp:107)
using ParticleFilter =
    mcl_3dl::pf::ParticleFilter<State6DOF, float, mcl_3dl::ParticleWeightedMeanQuat, std::default_random_engine>;

// State shared by the two model adapters of one node: the engine handle, the particle filter whose
// particles are batched, the clouds of the current cycle and the cached per-particle records.
// A growable array in page-locked memory of the engine (mcl3dl_host_alloc): mcl3dl_measure transfers pose and record
// arrays that live there in place, without a staging copy on either side of the call.
template <typename T>
class PinnedArray
{
public:
  PinnedArray() = default;
  PinnedArray(const PinnedArray&) = delete;
  PinnedArray& operator=(const PinnedArray&) = delete;
  ~PinnedArray()
  {
    release();
  }
  void bind(mcl3dl_engine* engine)
  {
    engine_ = engine;
  }
  // Must run before mcl3dl_destroy of the bound engine.
  void release()
  {
    if (data_)
      mcl3dl_host_free(engine_, data_);
    data_ = nullptr;
    size_ = cap_ = 0;
  }
  // Contents are unspecified after a resize that grows the block (every user refills the array).
  void resize(size_t n)
  {
    if (n > cap_)
    {
      const size_t cap = std::max(n, cap_ * 2);
      void* p = nullptr;
      const int rc = mcl3dl_host_alloc(engine_, cap * sizeof(T), &p);
      if (rc != MCL3DL_OK)
        throw std::runtime_error(std::string("mcl3dl_host_alloc: ") + mcl3dl_strerror(rc));
      if (data_)
        mcl3dl_host_free(engine_, data_);
      data_ = static_cast<T*>(p);
      cap_ = cap;
    }
    size_ = n;
  }
  size_t size() const
  {
    return size_;
  }
  T* data()
  {
    return data_;
  }
  T& operator[](size_t i)
  {
    return data_[i];
  }
  const T& operator[](size_t i) const
  {
    return data_[i];
  }

private:
  mcl3dl_engine* engine_ = nullptr;
  T* data_ = nullptr;
  size_t size_ = 0, cap_ = 0;
};

class MeasurementBatcher
{
public:
  using Ptr = std::shared_ptr<MeasurementBatcher>;

  MeasurementBatcher(ParticleFilter* pf, const std::vector<int>& devices,
                     const std::shared_ptr<mcl_3dl::LidarMeasurementModelLikelihoodParameters>& lik_params,
                     const std::shared_ptr<mcl_3dl::LidarMeasurementModelBeamParameters>& beam_params,
                     const float* dist_weight_xyz)
    : pf_(pf), lik_params_(lik_params), beam_params_(beam_params), engine_(nullptr)
  {
    for (int k = 0; k < 3; ++k) dist_weight_[k] = dist_weight_xyz ? dist_weight_xyz[k] : 1.0f;
    const int rc = mcl3dl_create(&engine_, devices.empty() ? nullptr : devices.data(),
                                 devices.empty() ? 1 : static_cast<int>(devices.size()));
    if (rc != MCL3DL_OK)  // no CPU fallback: the node must not start without its device
      throw std::runtime_error(std::string("mcl3dl_create: ") + mcl3dl_strerror(rc));
    poses_.bind(engine_);
    results_.bind(engine_);
  }
  ~MeasurementBatcher()
  {
    poses_.release();
    results_.release();
    mcl3dl_destroy(engine_);
  }
  MeasurementBatcher(const MeasurementBatcher&) = delete;
  MeasurementBatcher& operator=(const MeasurementBatcher&) = delete;

  // filter() of either model ran: a new update cycle is being prepared.
  void noteFiltered(bool is_beam, const Cloud::ConstPtr& pc)
  {
    (is_beam ? beam_cloud_ : lik_cloud_) = pc;
    valid_ = false;
  }

  // The record of state `s`; batches on the first call of a cycle.
  const mcl3dl_result& lookup(ChunkedKdtree<PointType>::Ptr& kdtree, bool is_beam, const Cloud::ConstPtr& pc,
                              const std::vector<Vec3>& origins, const State6DOF& s)
  {
    const Cloud::ConstPtr& expected = is_beam ? beam_cloud_ : lik_cloud_;
    if (pc != expected)
    {
      // measure() was handed a cloud that did not come from this model's last filter(): honour it
      (is_beam ? beam_cloud_ : lik_cloud_) = pc;
      valid_ = false;
    }
    if (!valid_ || !sameOrigins(origins))
      runBatch(kdtree, origins);
    // pf::ParticleFilter::measure walks particles_ in index order (pf.h:256); each model is called once
    // per particle, so a per-model cursor finds the record in O(1).
    size_t& cur = is_beam ? cursor_beam_ : cursor_lik_;
    for (size_t tries = 0; tries < 2; ++tries)
    {
      if (cur < poses_.size() && samePose(poses_[cur], s))
        return results_[cur++];
      cur = 0;
      for (; cur < poses_.size(); ++cur)
        if (samePose(poses_[cur], s))
          return results_[cur++];
    }
    // a state that is not one of the filter's particles (e.g. the mean pose): one-particle call
    single_pose_ = toPose(s);
    callEngine(&single_pose_, 1, origins, &single_result_);
    return single_result_;
  }
  // Scope row f2: the whole pf_->measure(measure_func) of src/mcl_3dl.cpp:402-426 in one engine call.
  // prior[i] = particle i's probability_, extra[i] = the host-owned factor of the lambda (the odometry-error
  // pdf, :422-424); posterior receives the normalised weights (or the prior when nothing survives).
  void measureUpdate(ChunkedKdtree<PointType>::Ptr& kdtree, const Cloud::ConstPtr& pc_lik, const Cloud::ConstPtr& pc_beam,
                     const std::vector<Vec3>& origins, const std::vector<float>& prior, const std::vector<float>& extra,
                     std::vector<float>& posterior, mcl3dl_update_summary* summary)
  {
    lik_cloud_ = pc_lik;
    beam_cloud_ = pc_beam;
    valid_ = false;
    stageMap(kdtree);
    if (!staged_map_)
      stageMap(kdtree);
    pack(lik_cloud_, lik_pts_);
    pack(beam_cloud_, beam_pts_);
    packPoses();
    posterior.assign(poses_.size(), 0.0f);
    std::vector<float> o(origins.size() * 3);
    for (size_t k = 0; k < origins.size(); ++k)
    {
      o[3 * k] = origins[k].x_;
      o[3 * k + 1] = origins[k].y_;
      o[3 * k + 2] = origins[k].z_;
    }
    check(mcl3dl_measure_update(engine_, poses_.data(), poses_.size(), lik_pts_.data(), lik_pts_.size(), beam_pts_.data(),
                                beam_pts_.size(), o.data(), origins.size(), prior.data(),
                                extra.empty() ? nullptr : extra.data(), posterior.data(), nullptr, summary),
          "mcl3dl_measure_update");
  }
  // Scope row f3: the same update on the engine's RESIDENT particle set (nothing per particle crosses the bus).
  void measureResident(ChunkedKdtree<PointType>::Ptr& kdtree, const Cloud::ConstPtr& pc_lik, const Cloud::ConstPtr& pc_beam,
                       const std::vector<Vec3>& origins, float odom_err_integ_lin_sigma, mcl3dl_update_summary* summary)
  {
    lik_cloud_ = pc_lik;
    beam_cloud_ = pc_beam;
    valid_ = false;
    stageMap(kdtree);
    if (!staged_map_)
      stageMap(kdtree);
    pack(lik_cloud_, lik_pts_);
    pack(beam_cloud_, beam_pts_);
    std::vector<float> o(origins.size() * 3);
    for (size_t k = 0; k < origins.size(); ++k)
    {
      o[3 * k] = origins[k].x_;
      o[3 * k + 1] = origins[k].y_;
      o[3 * k + 2] = origins[k].z_;
    }
    check(mcl3dl_particles_measure_update(engine_, lik_pts_.data(), lik_pts_.size(), beam_pts_.data(), beam_pts_.size(), o.data(),
                                          origins.size(), odom_err_integ_lin_sigma, summary),
          "mcl3dl_particles_measure_update");
  }
  void checked(int rc, const char* what) const { check(rc, what); }
  size_t likPoints() const { return lik_cloud_ ? lik_cloud_->size() : 0; }
  mcl3dl_engine* engine() { return engine_; }

private:
  static mcl3dl_pose toPose(const State6DOF& s)
  {
    mcl3dl_pose p;
    p.px = s.pos_.x_;
    p.py = s.pos_.y_;
    p.pz = s.pos_.z_;
    p._pad = 0.0f;
    p.qx = s.rot_.x_;
    p.qy = s.rot_.y_;
    p.qz = s.rot_.z_;
    p.qw = s.rot_.w_;
    return p;
  }
  static bool samePose(const mcl3dl_pose& p, const State6DOF& s)
  {
    const mcl3dl_pose q = toPose(s);
    return std::memcmp(&p, &q, sizeof(p)) == 0;  // bitwise, as the records are per exact state
  }
  bool sameOrigins(const std::vector<Vec3>& o) const
  {
    if (o.size() * 3 != origins_.size())
      return false;
    for (size_t k = 0; k < o.size(); ++k)
      if (o[k].x_ != origins_[3 * k] || o[k].y_ != origins_[3 * k + 1] || o[k].z_ != origins_[3 * k + 2])
        return false;
    return true;
  }
  static void pack(const Cloud::ConstPtr& pc, std::vector<mcl3dl_point>& out)
  {
    out.clear();
    if (!pc)
      return;
    out.reserve(pc->size());
    for (const auto& p : pc->points)  // PointXYZIL (32 B) -> 16 B, point_types.h:40-55
      out.push_back(mcl3dl_point{p.x, p.y, p.z, p.label});
  }
  void check(int rc, const char* what) const
  {
    if (rc != MCL3DL_OK)
      throw std::runtime_error(std::string(what) + ": " + mcl3dl_strerror(rc) + " " + mcl3dl_last_error_detail(engine_));
  }
  void stageMap(ChunkedKdtree<PointType>::Ptr& kdtree)
  {
    const Cloud::ConstPtr& map = kdtree->getInputCloud();
    if (!map || map->empty())
      throw std::runtime_error("mcl_3dl_b200: measure() without a map cloud");
    // same trigger as RaycastUsingDDA::updatePointCloud (raycast_using_dda.h:162-171): cloud + header.stamp
    if (map.get() == staged_map_ && map->header.stamp == staged_stamp_ && map->size() == staged_size_)
    {
      refreshScalars();
      return;
    }
    std::vector<mcl3dl_point> pts;
    pack(map, pts);
    deriveParams();
    check(mcl3dl_set_map(engine_, pts.data(), pts.size(), ++stamp_counter_, &lik_c_, &beam_c_), "mcl3dl_set_map");
    staged_map_ = map.get();
    staged_stamp_ = map->header.stamp;
    staged_size_ = map->size();
  }
  void deriveParams()
  {
    lik_c_.match_weight = lik_params_->match_weight_;
    lik_c_.match_dist_min = lik_params_->match_dist_min_;
    lik_c_.match_dist_flat = lik_params_->match_dist_flat_;
    for (int k = 0; k < 3; ++k) lik_c_.dist_weight[k] = dist_weight_[k];
    const auto& b = *beam_params_;
    mcl3dl_beam_params_from_reference(&beam_c_, b.map_grid_x_, b.map_grid_y_, b.map_grid_z_, b.num_points_default_,
                                      b.beam_likelihood_min_, b.ang_total_ref_, b.filter_label_max_, b.hit_range_,
                                      b.add_penalty_short_only_mode_ ? 1 : 0, b.use_raycast_using_dda_ ? 1 : 0, b.ray_angle_half_,
                                      b.dda_grid_size_);
  }
  void refreshScalars()
  {
    // parameters are shared_ptr'd with the node and may be edited between updates (refreshParameters())
    const mcl3dl_lik_params l0 = lik_c_;
    const mcl3dl_beam_params b0 = beam_c_;
    deriveParams();
    if (std::memcmp(&l0, &lik_c_, sizeof(l0)) == 0 && std::memcmp(&b0, &beam_c_, sizeof(b0)) == 0)
      return;
    if (mcl3dl_set_params(engine_, &lik_c_, &beam_c_) != MCL3DL_OK)
      staged_map_ = nullptr;  // a grid-shaping parameter changed: restage on the next call
  }
  void callEngine(const mcl3dl_pose* poses, size_t n, const std::vector<Vec3>& origins, mcl3dl_result* out)
  {
    std::vector<float> o(origins.size() * 3);
    for (size_t k = 0; k < origins.size(); ++k)
    {
      o[3 * k] = origins[k].x_;
      o[3 * k + 1] = origins[k].y_;
      o[3 * k + 2] = origins[k].z_;
    }
    check(mcl3dl_measure(engine_, poses, n, lik_pts_.data(), lik_pts_.size(), beam_pts_.data(), beam_pts_.size(),
                         o.data(), origins.size(), out),
          "mcl3dl_measure");
  }
  // State6DOF -> mcl3dl_pose for every particle, straight into the page-locked array the engine copies from
  void packPoses()
  {
    poses_.resize(pf_->getParticleSize());
    size_t i = 0;
    for (auto it = pf_->begin(); it != pf_->end(); ++it) poses_[i++] = toPose(it->state_);
  }
  void runBatch(ChunkedKdtree<PointType>::Ptr& kdtree, const std::vector<Vec3>& origins)
  {
    stageMap(kdtree);
    if (!staged_map_)
      stageMap(kdtree);
    pack(lik_cloud_, lik_pts_);
    pack(beam_cloud_, beam_pts_);
    packPoses();
    results_.resize(poses_.size());
    callEngine(poses_.data(), poses_.size(), origins, results_.data());
    origins_.resize(origins.size() * 3);
    for (size_t k = 0; k < origins.size(); ++k)
    {
      origins_[3 * k] = origins[k].x_;
      origins_[3 * k + 1] = origins[k].y_;
      origins_[3 * k + 2] = origins[k].z_;
    }
    cursor_lik_ = cursor_beam_ = 0;
    valid_ = true;
  }

  ParticleFilter* pf_;
  std::shared_ptr<mcl_3dl::LidarMeasurementModelLikelihoodParameters> lik_params_;
  std::shared_ptr<mcl_3dl::LidarMeasurementModelBeamParameters> beam_params_;
  float dist_weight_[3];
  mcl3dl_engine* engine_;
  mcl3dl_lik_params lik_c_;
  mcl3dl_beam_params beam_c_;
  const Cloud* staged_map_ = nullptr;
  decltype(pcl::PCLHeader().stamp) staged_stamp_ = 0;
  size_t staged_size_ = 0;
  uint64_t stamp_counter_ = 0;
  Cloud::ConstPtr lik_cloud_, beam_cloud_;
  std::vector<mcl3dl_point> lik_pts_, beam_pts_;
  PinnedArray<mcl3dl_pose> poses_;
  PinnedArray<mcl3dl_result> results_;
  std::vector<float> origins_;
  size_t cursor_lik_ = 0, cursor_beam_ = 0;
  bool valid_ = false;
  mcl3dl_pose single_pose_;
  mcl3dl_result single_result_;
};

// LidarMeasurementModelLikelihood with measure() served by the engine
// (replaces src/lidar_measurement_model_likelihood.cpp:105-139).
class LidarMeasurementModelLikelihoodB200 : public mcl_3dl::LidarMeasurementModelLikelihood
{
public:
  LidarMeasurementModelLikelihoodB200(const std::shared_ptr<mcl_3dl::LidarMeasurementModelLikelihoodParameters>& params,
                                      const MeasurementBatcher::Ptr& batcher)
    : mcl_3dl::LidarMeasurementModelLikelihood(params), batcher_(batcher)
  {
  }
  Cloud::Ptr filter(const Cloud::ConstPtr& pc, const mcl_3dl::PointCloudRandomSampler<PointType>& sampler) const override
  {
    Cloud::Ptr out = mcl_3dl::LidarMeasurementModelLikelihood::filter(pc, sampler);  // reference code, unchanged
    batcher_->noteFiltered(false, out);
    return out;
  }
  LidarMeasurementResult measure(ChunkedKdtree<PointType>::Ptr& kdtree, const Cloud::ConstPtr& pc,
                                 const std::vector<Vec3>& origins, const State6DOF& s) const override
  {
    if (!pc || pc->size() == 0)  // likelihood.cpp:111-114
      return LidarMeasurementResult(1, 0);
    const mcl3dl_result& r = batcher_->lookup(kdtree, false, pc, origins, s);
    const float match_ratio = static_cast<float>(r.match_cnt) / pc->points.size();  // :136
    return LidarMeasurementResult(r.score_like, match_ratio);
  }

private:
  MeasurementBatcher::Ptr batcher_;
};

// LidarMeasurementModelBeam with measure() served by the engine
// (replaces src/lidar_measurement_model_beam.cpp:124-155 with either raycaster: RaycastUsingKDTree, the
// node's default, or RaycastUsingDDA when beam/use_raycast_using_dda is set).
class LidarMeasurementModelBeamB200 : public mcl_3dl::LidarMeasurementModelBeam
{
public:
  LidarMeasurementModelBeamB200(const std::shared_ptr<mcl_3dl::LidarMeasurementModelBeamParameters>& params,
                                const MeasurementBatcher::Ptr& batcher)
    : mcl_3dl::LidarMeasurementModelBeam(params), batcher_(batcher)
  {
  }
  Cloud::Ptr filter(const Cloud::ConstPtr& pc, const mcl_3dl::PointCloudRandomSampler<PointType>& sampler) const override
  {
    Cloud::Ptr out = mcl_3dl::LidarMeasurementModelBeam::filter(pc, sampler);
    batcher_->noteFiltered(true, out);
    return out;
  }
  LidarMeasurementResult measure(ChunkedKdtree<PointType>::Ptr& kdtree, const Cloud::ConstPtr& pc,
                                 const std::vector<Vec3>& origins, const State6DOF& s) const override
  {
    if (!pc || pc->size() == 0)  // beam.cpp:130-133
      return LidarMeasurementResult(1, 0);
    const mcl3dl_result& r = batcher_->lookup(kdtree, true, pc, origins, s);
    return LidarMeasurementResult(r.score_beam, 1.0);  // :154
  }

private:
  MeasurementBatcher::Ptr batcher_;
};

// Optional deeper integration (scope row f2).  The node's particle filter with one extra method that replaces
//   pf_->measure(measure_func);                                   (src/mcl_3dl.cpp:426)
// by a single fused engine call: measurement of every particle, multiplication into probability_, normalisation,
// entropy and the match-ratio extremes the lambda tracks (:416-419).  Construct the node's pf_ as this class
// (:1272-1275) and call measureBatched() instead of measure(); everything else of pf::ParticleFilter is inherited.
class ParticleFilterB200 : public ParticleFilter
{
public:
  using ParticleFilter::ParticleFilter;

  struct UpdateResult
  {
    float match_ratio_min, match_ratio_max;
    bool kept;  // false: every weight was zero and the particles were left untouched (pf.h:274-278)
  };

  // extra(const State6DOF&) -> float: the part of the lambda the host owns (odom_error_lin_nd(...), :422-424)
  template <typename EXTRA>
  UpdateResult measureBatched(MeasurementBatcher& batcher, ChunkedKdtree<PointType>::Ptr& kdtree,
                              const Cloud::ConstPtr& pc_likelihood, const Cloud::ConstPtr& pc_beam,
                              const std::vector<Vec3>& origins, EXTRA extra)
  {
    std::vector<float> prior, factor, posterior;
    prior.reserve(particles_.size());
    factor.reserve(particles_.size());
    for (const auto& p : particles_)
    {
      prior.push_back(p.probability_);
      factor.push_back(extra(p.state_));
    }
    mcl3dl_update_summary s;
    batcher.measureUpdate(kdtree, pc_likelihood, pc_beam, origins, prior, factor, posterior, &s);
    if (s.kept)
    {
      for (size_t i = 0; i < particles_.size(); ++i) particles_[i].probability_ = posterior[i];
      entropy_ = s.entropy;
    }
    return UpdateResult{s.match_ratio_min, s.match_ratio_max, s.kept != 0};
  }

  // ---- Scope row f3: the particle set kept RESIDENT on the device between updates.  The node's cycle
  //   pf_->predict(model) / pf_->measure(lambda) / pf_->bias + expectationBiased + max + covariance / pf_->resample(sigma)
  // (src/mcl_3dl.cpp:227-232,402-452,704-724,809-815) becomes predictResident / measureResident / estimateResident /
  // resampleResident; only scans, odometry and summaries cross the bus.  uploadResident() after init() / resizeParticle() /
  // any host-side edit of particles_, downloadResident() whenever host code needs the particles (markers, expansion
  // resetting).  Documented departures (include/mcl3dl_b200.h): counter-based noise instead of the std engine's stream,
  // ties of the accumulated probability go to the lowest index, sums in double.
  static mcl3dl_state toState(const State6DOF& s)
  {
    mcl3dl_state o;
    o.pos[0] = s.pos_.x_;
    o.pos[1] = s.pos_.y_;
    o.pos[2] = s.pos_.z_;
    o.rot[0] = s.rot_.x_;
    o.rot[1] = s.rot_.y_;
    o.rot[2] = s.rot_.z_;
    o.rot[3] = s.rot_.w_;
    o.noise_ll = s.noise_ll_;
    o.noise_la = s.noise_la_;
    o.noise_al = s.noise_al_;
    o.noise_aa = s.noise_aa_;
    for (int k = 0; k < 3; ++k)
    {
      o.odom_err_integ_lin[k] = s.odom_err_integ_lin_[k];
      o.odom_err_integ_ang[k] = s.odom_err_integ_ang_[k];
    }
    return o;
  }
  static void fromState(const mcl3dl_state& o, State6DOF& s)
  {
    s.pos_ = Vec3(o.pos[0], o.pos[1], o.pos[2]);
    s.rot_ = mcl_3dl::Quat(o.rot[0], o.rot[1], o.rot[2], o.rot[3]);
    s.noise_ll_ = o.noise_ll;
    s.noise_la_ = o.noise_la;
    s.noise_al_ = o.noise_al;
    s.noise_aa_ = o.noise_aa;
    s.odom_err_integ_lin_ = Vec3(o.odom_err_integ_lin[0], o.odom_err_integ_lin[1], o.odom_err_integ_lin[2]);
    s.odom_err_integ_ang_ = Vec3(o.odom_err_integ_ang[0], o.odom_err_integ_ang[1], o.odom_err_integ_ang[2]);
  }
  void uploadResident(MeasurementBatcher& batcher)
  {
    std::vector<mcl3dl_state> st;
    std::vector<float> prob;
    st.reserve(particles_.size());
    prob.reserve(particles_.size());
    for (const auto& p : particles_)
    {
      st.push_back(toState(p.state_));
      prob.push_back(p.probability_);
    }
    batcher.checked(mcl3dl_particles_set(batcher.engine(), st.data(), prob.data(), st.size()), "mcl3dl_particles_set");
  }
  void downloadResident(MeasurementBatcher& batcher)
  {
    std::vector<mcl3dl_state> st(particles_.size());
    std::vector<float> prob(particles_.size());
    batcher.checked(mcl3dl_particles_get(batcher.engine(), st.data(), prob.data(), st.size()), "mcl3dl_particles_get");
    for (size_t i = 0; i < particles_.size(); ++i)
    {
      fromState(st[i], particles_[i].state_);
      particles_[i].probability_ = prob[i];
    }
  }
  // pf_->predict(motion_prediction_model) after model->setOdoms(odom_prev, odom_current, dt) (src/mcl_3dl.cpp:227-232)
  void predictResident(MeasurementBatcher& batcher, const State6DOF& odom_prev, const State6DOF& odom_current, float time_diff,
                       float odom_err_integ_lin_tc, float odom_err_integ_ang_tc)
  {
    const mcl3dl_pose a{odom_prev.pos_.x_, odom_prev.pos_.y_, odom_prev.pos_.z_, 0.0f, odom_prev.rot_.x_, odom_prev.rot_.y_,
                        odom_prev.rot_.z_, odom_prev.rot_.w_};
    const mcl3dl_pose b{odom_current.pos_.x_, odom_current.pos_.y_, odom_current.pos_.z_, 0.0f, odom_current.rot_.x_,
                        odom_current.rot_.y_, odom_current.rot_.z_, odom_current.rot_.w_};
    batcher.checked(mcl3dl_particles_predict(batcher.engine(), &a, &b, time_diff, odom_err_integ_lin_tc, odom_err_integ_ang_tc),
                    "mcl3dl_particles_predict");
  }
  // pf_->measure(measure_func) with the node's lambda, odometry-error term included (src/mcl_3dl.cpp:398-426)
  UpdateResult measureResident(MeasurementBatcher& batcher, ChunkedKdtree<PointType>::Ptr& kdtree, const Cloud::ConstPtr& pc_likelihood,
                               const Cloud::ConstPtr& pc_beam, const std::vector<Vec3>& origins, float odom_err_integ_lin_sigma)
  {
    mcl3dl_update_summary s;
    batcher.measureResident(kdtree, pc_likelihood, pc_beam, origins, odom_err_integ_lin_sigma, &s);
    if (s.kept)
      entropy_ = s.entropy;
    return UpdateResult{s.match_ratio_min, s.match_ratio_max, s.kept != 0};
  }
  // pf_->bias(...) + expectationBiased() + max() + covariance(1.0, .) (src/mcl_3dl.cpp:428-452,704-724)
  mcl3dl_estimate estimateResident(MeasurementBatcher& batcher, const State6DOF* state_prev, float bias_var_dist, float bias_var_ang)
  {
    mcl3dl_estimate e;
    mcl3dl_pose prev;
    if (state_prev)
      prev = mcl3dl_pose{state_prev->pos_.x_, state_prev->pos_.y_, state_prev->pos_.z_, 0.0f, state_prev->rot_.x_,
                         state_prev->rot_.y_, state_prev->rot_.z_, state_prev->rot_.w_};
    batcher.checked(mcl3dl_particles_estimate(batcher.engine(), state_prev ? &prev : nullptr, bias_var_dist, bias_var_ang, &e),
                    "mcl3dl_particles_estimate");
    return e;
  }
  // pf_->resample(State6DOF(sigma_pos, sigma_rpy)) (src/mcl_3dl.cpp:809-815); the host draws the start of the systematic scan
  // with the filter's own engine, exactly where pf.h:200 draws it
  void resampleResident(MeasurementBatcher& batcher, const Vec3& sigma_pos, const Vec3& sigma_rpy, uint64_t seed)
  {
    std::uniform_real_distribution<float> ud(0.0f, 1.0f);
    float frac = ud(engine_);
    if (!(frac < 1.0f))
      frac = 0.0f;
    const float sp[3] = {sigma_pos.x_, sigma_pos.y_, sigma_pos.z_}, sr[3] = {sigma_rpy.x_, sigma_rpy.y_, sigma_rpy.z_};
    batcher.checked(mcl3dl_particles_resample(batcher.engine(), sp, sr, frac, seed), "mcl3dl_particles_resample");
  }
};

}  // namespace mcl_3dl_b200
#endif  // MCL_3DL_B200_LIDAR_MEASUREMENT_MODEL_B200_H
