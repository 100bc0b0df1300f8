// gl_ref_driver.cpp — TEST INFRASTRUCTURE ONLY ("reference" checker of global localisation and of the resize).
//
// ref_driver.cpp (the C-ABI driver around the reference's own sources, compiled here as part of this translation unit)
// plus the node's global_localization service body after its VoxelGrid, written afresh on the reference's own Quat,
// Vec3, State6DOF and pf::ParticleFilter and the shim KdTreeFLANN with the XyzRepresentation rescale, and a driver of
// the reference's own pf::ParticleFilter::resizeParticle.
#include "ref_driver.cpp"

#include <pcl/kdtree/kdtree_flann.h>

#include "gl_api.h"

namespace
{
using Filter6 = mcl_3dl::pf::ParticleFilter<State6DOF, float, mcl_3dl::ParticleWeightedMeanQuat, std::default_random_engine>;

State6DOF toState6(const mcl3dl_state& st)
{
  State6DOF s(Vec3(st.pos[0], st.pos[1], st.pos[2]), Quat(st.rot[0], st.rot[1], st.rot[2], st.rot[3]));
  s.noise_ll_ = st.noise_ll;
  s.noise_la_ = st.noise_la;
  s.noise_al_ = st.noise_al;
  s.noise_aa_ = st.noise_aa;
  s.odom_err_integ_lin_ = Vec3(st.odom_err_integ_lin[0], st.odom_err_integ_lin[1], st.odom_err_integ_lin[2]);
  s.odom_err_integ_ang_ = Vec3(st.odom_err_integ_ang[0], st.odom_err_integ_ang[1], st.odom_err_integ_ang[2]);
  return s;
}

mcl3dl_state fromState6(const State6DOF& s)
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
}  // namespace

extern "C" {

const char* mcl3dl_cpu_gl_kind(void) { return "reference"; }

int mcl3dl_cpu_gl_seed(const mcl3dl_point* ds, size_t n, double grid, int32_t div_yaw, const float imu_quat[4],
                       const float dist_weight[3], mcl3dl_state* states, float* probs, size_t cap, size_t* n_particles)
{
  if ((n && !ds) || !(grid > 0.0) || div_yaw < 1 || !imu_quat || !dist_weight || !n_particles)
    return MCL3DL_ERR_INVALID_ARG;
  Cloud::Ptr points = toCloud(ds, n);
  auto rep = std::make_shared<XyzRepresentation>();
  rep->setRescaleValues(dist_weight);
  pcl::KdTreeFLANN<PointType> kdtree;
  kdtree.setPointRepresentation(rep);
  kdtree.setInputCloud(points);
  // keep the points with nothing just above them: a radius search around the point raised by 0.01 + grid
  Cloud seeds;
  std::vector<int> id(1);
  std::vector<float> sqdist(1);
  for (const PointType& p : points->points)
  {
    PointType raised = p;
    raised.z += 0.01 + grid;
    if (kdtree.radiusSearch(raised, grid, id, sqdist, 1) == 0)
      seeds.points.push_back(p);
  }
  const size_t np = seeds.points.size() * static_cast<size_t>(div_yaw);
  *n_particles = np;
  if (!states && !probs)
    return MCL3DL_OK;
  if (cap < np)
    return MCL3DL_ERR_INVALID_ARG;
  if (np == 0)
    return MCL3DL_OK;
  Filter6 pf(1);
  pf.resizeParticle(np);
  const Quat imu(imu_quat[0], imu_quat[1], imu_quat[2], imu_quat[3]);
  const float prob = 1.0 / static_cast<float>(seeds.points.size());
  size_t i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i)
  {
    const PointType& p = seeds.points[i / div_yaw];
    const int c = static_cast<int>(i % div_yaw);
    it->probability_ = prob;
    it->probability_bias_ = 1.0;
    it->state_ = State6DOF(Vec3(p.x, p.y, p.z), (Quat(Vec3(0.0, 0.0, 2.0 * M_PI * c / div_yaw)) * imu).normalized());
    if (states)
      states[i] = fromState6(it->state_);
    if (probs)
      probs[i] = it->probability_;
  }
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_resize_6dof(const float* probs, const mcl3dl_state* states, size_t n, size_t num, mcl3dl_state* out_states,
                              float* out_probs)
{
  if (!probs || !states || n == 0 || num == 0 || !out_states || !out_probs)
    return MCL3DL_ERR_INVALID_ARG;
  Filter6 pf(static_cast<int>(n));
  size_t i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i)
  {
    it->state_ = toState6(states[i]);
    it->probability_ = probs[i];
  }
  pf.resizeParticle(num);
  i = 0;
  for (auto it = pf.begin(); it != pf.end(); ++it, ++i)
  {
    out_states[i] = fromState6(it->state_);
    out_probs[i] = it->probability_;
  }
  return MCL3DL_OK;
}

}  // extern "C"
