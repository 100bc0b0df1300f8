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
#include <cstddef>
#include <cmath>
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
#include <mcl_3dl/nd.h>
#include <mcl_3dl/parameters.h>
#include <mcl_3dl/pf.h>
#include <mcl_3dl/state_6dof.h>
#include <sensor_msgs/PointCloud2.h>

#include "mcl3dl_b200.h"

namespace mcl_3dl
{
// include/mcl_3dl/noise_generators/multivariate_noise_generator.h (Eigen's eigensolver): a caller of
// initUsingCovarianceResident includes it; nothing else here needs it
template <typename FLT_TYPE>
class MultivariateNoiseGenerator;
}  // namespace mcl_3dl

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
  // the global_localization service on the device over the index's cloud, staged first if it is not (or is stale)
  void globalLocalization(ChunkedKdtree<PointType>::Ptr& kdtree, const mcl3dl_global_localization_params& params,
                          mcl3dl_global_localization_info* info)
  {
    stageMap(kdtree);
    check(mcl3dl_global_localization(engine_, nullptr, 0, &params, info), "mcl3dl_global_localization");
  }
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
  // The node's matched / unmatched output (src/mcl_3dl.cpp:761-805) in one engine call: pc_local_full transformed by
  // the pose estimate e, split by the map index's radius search (mcl3dl_match_output); pc_local_full == nullptr takes
  // the downsampled cloud of the last mcl3dl_scan_prepare.  The clouds are filled as the node fills them.
  void matchOutput(ChunkedKdtree<PointType>::Ptr& kdtree, const State6DOF& e, const Cloud::ConstPtr& pc_local_full,
                   double match_dist, double unmatch_dist, float chunk_length, float max_search_radius,
                   pcl::PointCloud<pcl::PointXYZ>& matched, pcl::PointCloud<pcl::PointXYZ>& unmatched)
  {
    stageMap(kdtree);
    std::vector<mcl3dl_point> in;
    size_t cap = 0;
    if (pc_local_full)
    {
      pack(pc_local_full, in);
      cap = in.size();
    }
    else
    {
      check(mcl3dl_scan_get(engine_, 0, nullptr, 0, &cap), "mcl3dl_scan_get");
    }
    std::vector<mcl3dl_point> m(cap), u(cap);
    const mcl3dl_pose pose = toPose(e);
    const mcl3dl_match_params mp{match_dist, unmatch_dist, chunk_length, max_search_radius};
    size_t n_m = 0, n_u = 0;
    check(mcl3dl_match_output(engine_, &pose, pc_local_full ? in.data() : nullptr, in.size(), &mp, m.data(), &n_m, u.data(),
                              &n_u),
          "mcl3dl_match_output");
    matched.points.clear();
    unmatched.points.clear();
    for (size_t i = 0; i < n_m; ++i) matched.points.emplace_back(m[i].x, m[i].y, m[i].z);
    for (size_t i = 0; i < n_u; ++i) unmatched.points.emplace_back(u[i].x, u[i].y, u[i].z);
  }
  // The node's PointCloudSamplerWithNormal (use_random_sampler_with_normal) on the clipped clouds of the last
  // mcl3dl_scan_prepare, replacing its sampled scans (mcl3dl_scan_sample_with_normal).  The statistics are built exactly
  // as setParticleStatistics builds them (point_cloud_sampler_with_normal.h:75-89): std::abs of the 3 x 3 position block
  // of covariances, SelfAdjointEigenSolver of that double matrix, its eigenvalues and column 2, and mean.rot_ raw.
  // Matrix / Solver are Eigen::MatrixXd and Eigen::SelfAdjointEigenSolver<Eigen::MatrixXd> (template parameters, so
  // only a caller compiles the Eigen code); mean and covariances are pf_->expectation() and pf_->covariance(...), or for
  // the resident set the mean rotation and covariance of mcl3dl_particles_estimate(NULL).
  template <typename Matrix, typename Solver>
  void sampleWithNormalPrepared(const State6DOF& mean, const std::vector<State6DOF>& covariances,
                                const mcl_3dl::PointCloudSamplerWithNormalParameters& params, uint32_t lik_num, uint32_t beam_num,
                                uint64_t seed, mcl3dl_normal_sampler_info* info)
  {
    Matrix pos_cov(3, 3);
    for (size_t i = 0; i < 3; ++i)
      for (size_t j = 0; j < 3; ++j) pos_cov(i, j) = std::abs(covariances[i][j]);
    const Solver solver(pos_cov);
    mcl3dl_normal_sampler_params p{};
    p.perform_weighting_ratio = params.perform_weighting_ratio_;
    p.max_weight_ratio = params.max_weight_ratio_;
    p.max_weight = params.max_weight_;
    p.normal_search_range = params.normal_search_range_;
    for (int k = 0; k < 3; ++k)
    {
      p.eigen_values[k] = solver.eigenvalues()[k];
      p.eigen_vector[k] = solver.eigenvectors()(k, 2);
    }
    p.mean_rot[0] = mean.rot_.x_;
    p.mean_rot[1] = mean.rot_.y_;
    p.mean_rot[2] = mean.rot_.z_;
    p.mean_rot[3] = mean.rot_.w_;
    p.lik_num_points = lik_num;
    p.beam_num_points = beam_num;
    p.seed = seed;
    check(mcl3dl_scan_sample_with_normal(engine_, &p, info), "mcl3dl_scan_sample_with_normal");
  }
  // The map source of a node that does not fill its CPU map index (INTEGRATION.md, "the node without its CPU map index"):
  // cbMapUpdateTimer hands pc_map2_ here in place of kdtree_->setInputCloud(pc_map2_), and the map is staged at once, by
  // the rule of every entry point: the same cloud grown with a new stamp and its staged points unchanged in front is
  // appended (mcl3dl_map_append), anything else is staged whole.  The entry points that take the index read this cloud
  // while the index has none.
  void setMapCloud(const Cloud::ConstPtr& map)
  {
    intake_map_ = false;  // supersedes an intake map
    map_cloud_ = map;
    stageCloud(map);
    if (!staged_map_)
      stageCloud(map);
  }
  // One ray of the node's rviz markers (src/mcl_3dl.cpp:472-523): what the marker loop takes from its getBeamStatus call.
  struct BeamRay
  {
    Vec3 begin;  // pos, e.pos_ + e.rot_ * origins[label]
    Vec3 end;    // end, the scan point transformed by e
    Vec3 pos;    // point.pos_, the deciding cast step's position (NaN for LONG, where the node does not read it)
    mcl_3dl::LidarMeasurementModelBeam::BeamStatus status;
  };
  // The marker loop's casts from the pose estimate e (after e.rot_.normalize()) on the device (mcl3dl_beam_cast) over the
  // staged map; pc_beam == nullptr takes the sampled beam scan of the last mcl3dl_scan_prepare.
  void castBeams(const State6DOF& e, const Cloud::ConstPtr& pc_beam, const std::vector<Vec3>& origins, std::vector<BeamRay>& out)
  {
    using BeamStatus = mcl_3dl::LidarMeasurementModelBeam::BeamStatus;
    static_assert(static_cast<int>(BeamStatus::SHORT) == 0 && static_cast<int>(BeamStatus::HIT) == 1 &&
                      static_cast<int>(BeamStatus::LONG) == 2 && static_cast<int>(BeamStatus::TOTAL_REFLECTION) == 3,
                  "mcl3dl_beam_ray::status codes follow the order of LidarMeasurementModelBeam::BeamStatus");
    std::vector<mcl3dl_point> in;
    size_t cap = 0;
    if (pc_beam)
    {
      pack(pc_beam, in);
      cap = in.size();
    }
    else
    {
      check(mcl3dl_scan_get(engine_, 4, nullptr, 0, &cap), "mcl3dl_scan_get");
    }
    std::vector<float> o(origins.size() * 3);
    for (size_t k = 0; k < origins.size(); ++k)
    {
      o[3 * k] = origins[k].x_;
      o[3 * k + 1] = origins[k].y_;
      o[3 * k + 2] = origins[k].z_;
    }
    std::vector<mcl3dl_beam_ray> rays(cap);
    const mcl3dl_pose pose = toPose(e);
    const mcl3dl_point none{};  // an empty host scan still needs a pointer: NULL selects the prepared scan
    size_t n = 0;
    check(mcl3dl_beam_cast(engine_, &pose, pc_beam ? (in.empty() ? &none : in.data()) : nullptr, in.size(), o.data(), origins.size(),
                           rays.data(), rays.size(), &n),
          "mcl3dl_beam_cast");
    out.clear();
    out.reserve(n);
    for (size_t i = 0; i < n; ++i)
    {
      const mcl3dl_beam_ray& r = rays[i];
      out.push_back(BeamRay{Vec3(r.begin[0], r.begin[1], r.begin[2]), Vec3(r.end[0], r.end[1], r.end[2]),
                            Vec3(r.pos[0], r.pos[1], r.pos[2]), static_cast<BeamStatus>(r.status)});
    }
  }
  // The node's cloud accumulation on the device (mcl3dl_scan_accumulate; INTEGRATION.md, "cloud accumulation").
  // accumCloud (src/mcl_3dl.cpp:274-302) after its tf lookup: false exactly where mcl_3dl::fromROSMsg fails (no x / y / z
  // field, an empty cloud) and, beyond it, where x / y / z are not FLOAT32, the cloud is big-endian or its layout does
  // not hold the points; the accumulation is then unchanged.  odom_from_sensor: the looked-up transform (translation,
  // raw rotation x y z w).
  bool accumulateCloud(const sensor_msgs::PointCloud2& msg, const mcl3dl_transform& odom_from_sensor)
  {
    mcl3dl_cloud_view v{};
    if (!cloudView(msg, v))
      return false;
    check(mcl3dl_scan_accumulate(engine_, &v, &odom_from_sensor, &accumulated_clouds_), "mcl3dl_scan_accumulate");
    return true;
  }
  // accumClear (:266-272)
  void clearAccumulated()
  {
    check(mcl3dl_scan_accumulate_clear(engine_), "mcl3dl_scan_accumulate_clear");
    accumulated_clouds_ = 0;
  }
  // measure()'s transform into base_link and the VoxelGrid / clip / sample after it (:319-383), leaving the prepared
  // scans on the device for measureResidentPrepared-style calls (mcl3dl_particles_measure_update_prepared), matchOutput
  // and castBeams with nullptr clouds.  Throws on an empty accumulation (the node checks pc_accum_header_ first).
  void prepareAccumulated(const mcl3dl_transform& base_from_odom, const mcl3dl_scan_params& params, mcl3dl_scan_info* info)
  {
    check(mcl3dl_scan_prepare_accumulated(engine_, &base_from_odom, &params, info), "mcl3dl_scan_prepare_accumulated");
  }
  // ---- The map intake on the device (mcl3dl_map_load / mcl3dl_map_update_*; INTEGRATION.md, "the map intake").
  // Staging rules: after an intake load the entry points that take the index use the engine's map while the index and
  // setMapCloud have none; a later setMapCloud, or an index that holds a cloud, supersedes it (staged whole).  The node
  // then keeps no host copy of the map: mapCloud reads it back for updated_map.
  // cbMapcloud -> loadMapCloud (src/mcl_3dl.cpp:127-140, 1150-1170): fromROSMsg and the VoxelGrid at map_downsample on
  // the device, staged as the map; a pending patch is dropped.  False, with nothing changed, where accumulateCloud is
  // false (fromROSMsg's failures and its documented departures), for an intensity / label field of the right type that
  // does not fit in point_step, and for a map that keeps no finite point.  An intensity (label) field that is not
  // FLOAT32 (UINT32) is not read: fromROSMsg leaves 0 there.  stamp: the map's header.stamp, as mapCloud reports it.
  bool loadMapMessage(const sensor_msgs::PointCloud2& msg, const float leaf[3], uint64_t stamp)
  {
    mcl3dl_map_cloud m{};
    return mapView(msg, m) && loadMap(m, leaf, stamp);
  }
  // cbLoadPCD (:1172-1192) after loadPCDFile: the PointXYZIL array itself as the view.  False for an empty cloud and as
  // loadMapMessage.
  bool loadMapCloud(const Cloud& cloud, const float leaf[3], uint64_t stamp)
  {
    if (cloud.points.empty())
      return false;
    mcl3dl_map_cloud m{};
    m.view.data = cloud.points.data();
    m.view.width = static_cast<uint32_t>(cloud.points.size());
    m.view.height = 1;
    m.view.point_step = sizeof(PointType);
    m.view.row_step = m.view.width * m.view.point_step;
    m.view.offset[0] = offsetof(PointType, x);
    m.view.offset[1] = offsetof(PointType, y);
    m.view.offset[2] = offsetof(PointType, z);
    m.view.is_dense = cloud.is_dense ? 1 : 0;
    m.intensity_offset = offsetof(PointType, intensity);
    m.label_offset = offsetof(PointType, label);
    return loadMap(m, leaf, stamp);
  }
  // cbMapcloudUpdate (:141-153): the patch's fromROSMsg and VoxelGrid at update_downsample into the engine's pending
  // patch (it replaces one).  False, with nothing changed, as loadMapMessage (an empty patch after the VoxelGrid is valid).
  bool setMapUpdate(const sensor_msgs::PointCloud2& msg, const float leaf[3])
  {
    mcl3dl_map_cloud m{};
    if (!mapView(msg, m))
      return false;
    check(mcl3dl_map_update_set(engine_, &m, leaf, nullptr), "mcl3dl_map_update_set");
    return true;
  }
  // cbMapUpdateTimer (:1350-1378): the pending patch appended to the intake map on the device (mcl3dl_map_update_commit);
  // no pending patch changes nothing.  False, with the patch kept, when the engine's map is not an intake map (no load
  // yet, or setMapCloud / the index superseded it).  stamp: the new header.stamp of the published map.
  bool commitMapUpdate(uint64_t stamp)
  {
    if (!intake_map_)
      return false;
    mcl3dl_map_append_info info{};
    check(mcl3dl_map_update_commit(engine_, ++stamp_counter_, &info), "mcl3dl_map_update_commit");
    if (info.n_appended > 0)
    {
      ++map_intake_commits_;
      map_stamp_ = stamp;
    }
    return true;
  }
  // cbPosition's pc_update_.reset() (:189)
  void clearMapUpdate() { check(mcl3dl_map_update_clear(engine_), "mcl3dl_map_update_clear"); }
  // The staged map with x / y / z / intensity / label (updated_map, :1371-1373); header.stamp: the load's or the last
  // commit's.  Intensities of maps staged from host clouds are 0.
  void mapCloud(Cloud& out)
  {
    size_t n = 0;
    check(mcl3dl_map_get(engine_, nullptr, nullptr, 0, &n), "mcl3dl_map_get");
    std::vector<mcl3dl_point> pts(n);
    std::vector<float> inten(n);
    check(mcl3dl_map_get(engine_, pts.data(), inten.data(), n, &n), "mcl3dl_map_get");
    out.points.resize(n);
    for (size_t i = 0; i < n; ++i)
    {
      PointType& p = out.points[i];
      p.x = pts[i].x;
      p.y = pts[i].y;
      p.z = pts[i].z;
      p.intensity = inten[i];
      p.label = pts[i].label;
    }
    out.width = static_cast<uint32_t>(n);
    out.height = 1;
    out.is_dense = true;
    out.header.stamp = intake_map_ ? map_stamp_ : staged_stamp_;
  }
  // Intake loads, and commits that appended points, since construction
  size_t mapIntakeLoads() const { return map_intake_loads_; }
  size_t mapIntakeCommits() const { return map_intake_commits_; }
  // clouds accumulated since the last clear (the node's pc_accum_header_.size())
  uint32_t accumulatedClouds() const { return accumulated_clouds_; }
  void checked(int rc, const char* what) const { check(rc, what); }
  size_t likPoints() const { return lik_cloud_ ? lik_cloud_->size() : 0; }
  // How each new map reached the engine: appended (mcl3dl_map_append) or staged whole (mcl3dl_set_map).
  size_t mapAppends() const { return map_appends_; }
  size_t mapRestages() const { return map_restages_; }
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
  // The map of an entry point that takes the index: the index's cloud, or while it has none the intake map, or else the
  // last setMapCloud's.
  void stageMap(ChunkedKdtree<PointType>::Ptr& kdtree)
  {
    if (!kdtree->getInputCloud() && intake_map_)
    {
      // no host cloud to restage from: a grid-shaping parameter change needs a new load
      const mcl3dl_lik_params l0 = lik_c_;
      const mcl3dl_beam_params b0 = beam_c_;
      deriveParams();
      if (std::memcmp(&l0, &lik_c_, sizeof(l0)) != 0 || std::memcmp(&b0, &beam_c_, sizeof(b0)) != 0)
        check(mcl3dl_set_params(engine_, &lik_c_, &beam_c_), "mcl3dl_set_params (the intake map needs a new load)");
      staged_map_ = &intake_marker_;
      return;
    }
    intake_map_ = false;
    stageCloud(kdtree->getInputCloud() ? kdtree->getInputCloud() : map_cloud_);
  }
  // Field lookup and layout checks of a PointCloud2 (accumulateCloud, loadMapMessage, setMapUpdate): false where
  // mcl_3dl::fromROSMsg fails (no x / y / z field, an empty cloud) and where x / y / z are not FLOAT32, the cloud is
  // big-endian or its layout does not hold its points.
  static bool cloudView(const sensor_msgs::PointCloud2& msg, mcl3dl_cloud_view& v)
  {
    const char* names[3] = {"x", "y", "z"};
    for (int k = 0; k < 3; ++k)
    {
      const sensor_msgs::PointField* f = findField(msg, names[k]);
      if (!f || f->datatype != sensor_msgs::PointField::FLOAT32)
        return false;
      v.offset[k] = f->offset;
    }
    const uint64_t n = static_cast<uint64_t>(msg.width) * msg.height;
    if (msg.is_bigendian || n == 0)
      return false;
    const uint64_t span = static_cast<uint64_t>(msg.height - 1) * msg.row_step + static_cast<uint64_t>(msg.width) * msg.point_step;
    if (static_cast<uint64_t>(msg.row_step) < static_cast<uint64_t>(msg.width) * msg.point_step || span > msg.data.size())
      return false;
    for (int k = 0; k < 3; ++k)
      if (static_cast<uint64_t>(v.offset[k]) + 4 > msg.point_step)
        return false;
    v.data = msg.data.data();
    v.width = msg.width;
    v.height = msg.height;
    v.point_step = msg.point_step;
    v.row_step = msg.row_step;
    v.is_dense = msg.is_dense ? 1 : 0;
    return true;
  }
  static const sensor_msgs::PointField* findField(const sensor_msgs::PointCloud2& msg, const char* name)
  {
    for (const auto& fl : msg.fields)
      if (fl.name == name)
        return &fl;
    return nullptr;
  }
  // cloudView, plus the intensity (FLOAT32) and label (UINT32) offsets where a field of that name and type exists
  static bool mapView(const sensor_msgs::PointCloud2& msg, mcl3dl_map_cloud& m)
  {
    if (!cloudView(msg, m.view))
      return false;
    const auto offset = [&](const char* name, uint8_t type, int32_t& out) {
      const sensor_msgs::PointField* f = findField(msg, name);
      out = (f && f->datatype == type) ? static_cast<int32_t>(f->offset) : -1;
      return out < 0 || static_cast<uint64_t>(f->offset) + 4 <= msg.point_step;
    };
    return offset("intensity", sensor_msgs::PointField::FLOAT32, m.intensity_offset) &&
           offset("label", sensor_msgs::PointField::UINT32, m.label_offset);
  }
  bool loadMap(const mcl3dl_map_cloud& m, const float leaf[3], uint64_t stamp)
  {
    deriveParams();
    const int rc = mcl3dl_map_load(engine_, &m, leaf, ++stamp_counter_, &lik_c_, &beam_c_, nullptr);
    if (rc == MCL3DL_ERR_INVALID_ARG && m.view.data)
      return false;  // no finite point (the view itself was checked above): the previous map stays
    check(rc, "mcl3dl_map_load");
    staged_map_ = &intake_marker_;
    staged_pts_.clear();
    staged_size_ = 0;
    map_cloud_.reset();
    intake_map_ = true;
    map_stamp_ = stamp;
    ++map_intake_loads_;
    return true;
  }
  void stageCloud(const Cloud::ConstPtr& map)
  {
    if (!map || map->empty())
      throw std::runtime_error("mcl_3dl_b200: measure() without a map cloud");
    // same trigger as RaycastUsingDDA::updatePointCloud (raycast_using_dda.h:162-171): cloud + header.stamp
    if (map.get() == staged_map_ && map->header.stamp == staged_stamp_ && map->size() == staged_size_)
    {
      refreshScalars();
      return;
    }
    // The node's map update (cbMapUpdateTimer, src/mcl_3dl.cpp:1350-1378) appends to the cloud the index already holds:
    // the same object, grown, with a new stamp and the staged points unchanged in front.  Only the tail goes to the
    // engine then.
    if (map.get() == staged_map_ && map->header.stamp != staged_stamp_ && map->size() > staged_size_ && extendsStaged(*map))
    {
      refreshScalars();
      if (staged_map_)  // (null: a grid-shaping parameter changed, restage below)
      {
        std::vector<mcl3dl_point> tail;
        tail.reserve(map->size() - staged_size_);
        for (size_t i = staged_size_; i < map->size(); ++i)
        {
          const auto& p = map->points[i];
          tail.push_back(mcl3dl_point{p.x, p.y, p.z, p.label});
        }
        staged_map_ = nullptr;  // until the engine holds the grown map (a failed append restages on the next call)
        check(mcl3dl_map_append(engine_, tail.data(), tail.size(), ++stamp_counter_, nullptr), "mcl3dl_map_append");
        staged_map_ = map.get();
        staged_pts_.insert(staged_pts_.end(), tail.begin(), tail.end());
        staged_stamp_ = map->header.stamp;
        staged_size_ = map->size();
        ++map_appends_;
        return;
      }
    }
    staged_map_ = nullptr;  // until the engine holds the new map
    pack(map, staged_pts_);
    deriveParams();
    check(mcl3dl_set_map(engine_, staged_pts_.data(), staged_pts_.size(), ++stamp_counter_, &lik_c_, &beam_c_),
          "mcl3dl_set_map");
    staged_map_ = map.get();
    staged_stamp_ = map->header.stamp;
    staged_size_ = map->size();
    ++map_restages_;
  }
  // The first staged_size_ points of `map` pack to the staged points.
  bool extendsStaged(const Cloud& map) const
  {
    for (size_t i = 0; i < staged_size_; ++i)
    {
      const auto& p = map.points[i];
      const mcl3dl_point q{p.x, p.y, p.z, p.label};
      if (std::memcmp(&q, &staged_pts_[i], sizeof(q)) != 0)
        return false;
    }
    return true;
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
  std::vector<mcl3dl_point> staged_pts_;  // the staged map as packed: recognises an append to it
  Cloud::ConstPtr map_cloud_;              // the last setMapCloud's cloud
  uint64_t stamp_counter_ = 0;
  size_t map_appends_ = 0, map_restages_ = 0;
  bool intake_map_ = false;     // the engine's map came from loadMapMessage / loadMapCloud (and commitMapUpdate)
  const Cloud intake_marker_{};  // staged_map_ while the intake map is staged: no host cloud is that object
  uint64_t map_stamp_ = 0;      // the intake map's header.stamp
  size_t map_intake_loads_ = 0, map_intake_commits_ = 0;
  uint32_t accumulated_clouds_ = 0;
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
  // resampleResident; only scans, odometry and summaries cross the bus.  redrawOdomNoiseResident, noiseResident and
  // imuMeasureResident replace the odometry-noise redraw, expansion resetting and cbImu's gravity update;
  // landmarkMeasureResident, resetOdomErrIntegResident and posesResident replace cbLandmark's measure, the pose-jump reset
  // and what publishParticles reads; initResident and initUsingCovarianceResident replace pf_->init and cbPosition's
  // initUsingNoiseGenerator.  uploadResident() after any host-side edit of particles_ (globalLocalizationResident /
  // resizeResident replace the service body and resizeParticle), downloadResident() whenever host code needs the whole
  // particles.
  // Documented departures (include/mcl3dl_b200.h): counter-based noise instead of the std engine's stream,
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
  // The odometry-noise redraw after resampling, pf_->predict(update_noise_func) (src/mcl_3dl.cpp:817-825), with the node's
  // params_.odom_err_lin_lin_, _lin_ang_, _ang_lin_, _ang_ang_
  void redrawOdomNoiseResident(MeasurementBatcher& batcher, double lin_lin, double lin_ang, double ang_lin, double ang_ang, uint64_t seed)
  {
    batcher.checked(mcl3dl_particles_redraw_odom_noise(batcher.engine(), lin_lin, lin_ang, ang_lin, ang_ang, seed),
                    "mcl3dl_particles_redraw_odom_noise");
  }
  // Expansion resetting, pf_->noise(State6DOF(sigma_pos, sigma_rpy)) (src/mcl_3dl.cpp:853-864): rotations are left
  // un-normalised and noise_* zeroed, as the reference leaves them
  void noiseResident(MeasurementBatcher& batcher, const Vec3& sigma_pos, const Vec3& sigma_rpy, uint64_t seed)
  {
    const float sp[3] = {sigma_pos.x_, sigma_pos.y_, sigma_pos.z_}, sr[3] = {sigma_rpy.x_, sigma_rpy.y_, sigma_rpy.z_};
    batcher.checked(mcl3dl_particles_noise(batcher.engine(), sp, sr, seed), "mcl3dl_particles_noise");
  }
  // cbImu's imu_measurement_model_->setAccMeasure(acc_measure) + pf_->measure(imu_measure_func) (src/mcl_3dl.cpp:1003-1008)
  // for ImuMeasurementModelGravity(acc_var)
  UpdateResult imuMeasureResident(MeasurementBatcher& batcher, const Vec3& acc_measure, float acc_var)
  {
    mcl3dl_update_summary s;
    const float acc[3] = {acc_measure.x_, acc_measure.y_, acc_measure.z_};
    batcher.checked(mcl3dl_particles_imu_update(batcher.engine(), acc, acc_var, &s), "mcl3dl_particles_imu_update");
    if (s.kept)
      entropy_ = s.entropy;
    return UpdateResult{s.match_ratio_min, s.match_ratio_max, s.kept != 0};
  }
  // cbLandmark's NormalLikelihoodNd<float, 6> (src/mcl_3dl.cpp:901-905), built by the reference's own class from the
  // message's 36 doubles exactly as the node builds it (Eigen maps them column-major, so a non-symmetric covariance
  // enters transposed), read out through a derived type: a_ and sigma_inv_ (row-major).  The class templates are
  // parameters so that only a caller compiles the Eigen code.
  template <typename Nd = mcl_3dl::NormalLikelihoodNd<float, 6>, typename Matrix6d = Eigen::Matrix<double, 6, 6>>
  static void landmarkNd(const double* covariance, mcl3dl_landmark_params& p)
  {
    struct Access : Nd
    {
      explicit Access(const typename Nd::Matrix& sigma) : Nd(sigma) {}
      void read(mcl3dl_landmark_params& p) const
      {
        p.nd_a = this->a_;
        for (int r = 0; r < 6; ++r)
          for (int c = 0; c < 6; ++c) p.sigma_inv[r * 6 + c] = this->sigma_inv_(r, c);
      }
    };
    Access(Matrix6d(covariance).template cast<float>()).read(p);
  }
  // cbLandmark's pf_->measure (src/mcl_3dl.cpp:899-931) on the resident set: measured as the node builds it from the
  // message, covariance = msg->pose.covariance (36 doubles, e.g. its boost::array).  The states do not change.
  template <typename Covariance>
  UpdateResult landmarkMeasureResident(MeasurementBatcher& batcher, const State6DOF& measured, const Covariance& covariance)
  {
    mcl3dl_landmark_params p;
    p.measured = mcl3dl_pose{measured.pos_.x_, measured.pos_.y_, measured.pos_.z_, 0.0f,
                             measured.rot_.x_, measured.rot_.y_, measured.rot_.z_, measured.rot_.w_};
    landmarkNd(covariance.data(), p);
    mcl3dl_update_summary s;
    batcher.checked(mcl3dl_particles_landmark_update(batcher.engine(), &p, &s), "mcl3dl_particles_landmark_update");
    if (s.kept)
      entropy_ = s.entropy;
    return UpdateResult{s.match_ratio_min, s.match_ratio_max, s.kept != 0};
  }
  // The node's integ_reset_func through pf_->predict (the pose-jump branch, src/mcl_3dl.cpp:653-658, and cbPosition)
  void resetOdomErrIntegResident(MeasurementBatcher& batcher)
  {
    batcher.checked(mcl3dl_particles_reset_odom_err_integ(batcher.engine()), "mcl3dl_particles_reset_odom_err_integ");
  }
  // What publishParticles (src/mcl_3dl.cpp:1101-1125) publishes: position + normalised rotation per resident particle
  void posesResident(MeasurementBatcher& batcher, std::vector<mcl3dl_pose>& poses)
  {
    poses.resize(particles_.size());
    batcher.checked(mcl3dl_particles_get_poses(batcher.engine(), poses.data(), poses.size()), "mcl3dl_particles_get_poses");
  }
  // pf_->init(mean, sigma) (pf.h:169-172; the configured start, src/mcl_3dl.cpp:1276) on the device: the reference's own
  // DiagonalNoiseGenerator<float>(mean, sigma) gives getMean() (setMean's getRPY) and sigma_, read through a derived
  // type; particles_.size() particles are seeded.  particles_ is stale until downloadResident().
  template <typename Gen = mcl_3dl::DiagonalNoiseGenerator<float>>
  void initResident(MeasurementBatcher& batcher, const State6DOF& mean, const State6DOF& sigma, uint64_t seed)
  {
    struct Access : Gen
    {
      Access(const State6DOF& m, const State6DOF& s) : Gen(m, s) {}
      void read(mcl3dl_init_params& p) const
      {
        for (int k = 0; k < 6; ++k)
        {
          p.mean[k] = this->getMean()[k];
          p.sigma[k] = this->sigma_[k];
        }
      }
    };
    mcl3dl_init_params p{};
    p.multivariate = 0;
    Access(mean, sigma).read(p);
    batcher.checked(mcl3dl_particles_init(batcher.engine(), particles_.size(), &p, seed), "mcl3dl_particles_init");
  }
  // cbPosition's pf_->initUsingNoiseGenerator(MultivariateNoiseGenerator<float>(mean, msg->pose.covariance))
  // (src/mcl_3dl.cpp:189-190) on the device: the reference's own generator (its eigendecomposition on the host) gives
  // mean_vec_ and norm_transform_, read through a derived type.  covariance = the message's 36 doubles, read row-major as
  // the generator reads them.  Returns false, the resident set as it was, when norm_transform_ is not finite (a
  // covariance with a negative eigenvalue).  The class template is a parameter, so only a caller compiles the Eigen
  // code; it includes <mcl_3dl/noise_generators/multivariate_noise_generator.h>.
  template <typename Covariance, typename Gen = mcl_3dl::MultivariateNoiseGenerator<float>>
  bool initUsingCovarianceResident(MeasurementBatcher& batcher, const State6DOF& mean, const Covariance& covariance, uint64_t seed)
  {
    struct Access : Gen
    {
      Access(const State6DOF& m, const Covariance& c) : Gen(m, c) {}
      bool read(mcl3dl_init_params& p) const
      {
        bool finite = true;
        for (int r = 0; r < 6; ++r)
        {
          p.mean[r] = this->mean_vec_[r];
          for (int c = 0; c < 6; ++c)
          {
            p.norm_transform[r * 6 + c] = this->norm_transform_(r, c);
            finite = finite && std::isfinite(p.norm_transform[r * 6 + c]);
          }
        }
        return finite;
      }
    };
    mcl3dl_init_params p{};
    p.multivariate = 1;
    if (!Access(mean, covariance).read(p))
      return false;
    batcher.checked(mcl3dl_particles_init(batcher.engine(), particles_.size(), &p, seed), "mcl3dl_particles_init");
    return true;
  }
  // The global_localization service body (src/mcl_3dl.cpp:1039-1099) on the device over the map index's cloud (pc_map_,
  // staged here if it is not yet): VoxelGrid, free-space filter and the div_yaw particles per seed replace the resident
  // set.  particles_ is resized to the new count, its contents stale until downloadResident(), so getParticleSize() and
  // setGlobalLocalizationStatus() keep working.  With no seed nothing changes (the reference would resize to 0).
  mcl3dl_global_localization_info globalLocalizationResident(MeasurementBatcher& batcher, ChunkedKdtree<PointType>::Ptr& kdtree,
                                                             const mcl3dl_global_localization_params& params)
  {
    mcl3dl_global_localization_info info;
    batcher.globalLocalization(kdtree, params, &info);
    if (info.n_particles)
      particles_.resize(info.n_particles);
    return info;
  }
  // pf_->resizeParticle(num) (pf.h:399-436) on the resident set, e.g. the node's shrink after an update while the set is
  // larger than num_particles (src/mcl_3dl.cpp:875-888); particles_ is resized as in globalLocalizationResident
  void resizeResident(MeasurementBatcher& batcher, size_t num)
  {
    batcher.checked(mcl3dl_particles_resize(batcher.engine(), num), "mcl3dl_particles_resize");
    particles_.resize(num);
  }
};

}  // namespace mcl_3dl_b200
#endif  // MCL_3DL_B200_LIDAR_MEASUREMENT_MODEL_B200_H
