// beam_cast_ref_driver.cpp — TEST INFRASTRUCTURE ONLY ("reference" checker of the ray markers).
//
// ref_driver.cpp (the C-ABI driver around the reference's own sources, compiled here as part of this translation unit)
// plus the node's marker loop itself: the reference's State6DOF::transform, LidarMeasurementModelBeam::getBeamStatus over
// its ChunkedKdtree and the CastResult it fills.
#include "ref_driver.cpp"

#include "beam_cast_api.h"

extern "C" {

// src/mcl_3dl.cpp:468-478 for one pose e
int mcl3dl_cpu_beam_cast(mcl3dl_cpu* h, const mcl3dl_pose* pose, const mcl3dl_point* pts, size_t n, const float* origins_xyz,
                         size_t n_origins, mcl3dl_beam_ray* out)
{
  if (!h || !pose || (n && (!pts || !out || !origins_xyz)))
    return MCL3DL_ERR_INVALID_ARG;
  for (size_t j = 0; j < n; ++j)
    if (pts[j].label >= n_origins)
      return MCL3DL_ERR_INVALID_ARG;
  std::vector<Vec3> origins;
  for (size_t k = 0; k < n_origins; ++k)
    origins.emplace_back(origins_xyz[3 * k], origins_xyz[3 * k + 1], origins_xyz[3 * k + 2]);
  const State6DOF e(Vec3(pose->px, pose->py, pose->pz), Quat(pose->qx, pose->qy, pose->qz, pose->qw));
  Cloud::Ptr pc_particle_beam = toCloud(pts, n);
  e.transform(*pc_particle_beam);
  LidarMeasurementModelBeam& beam_model = *h->beams[0];
  const float nan = std::numeric_limits<float>::quiet_NaN();
  size_t j = 0;
  for (const auto& p : pc_particle_beam->points)
  {
    const int beam_header_id = p.label;
    const Vec3 pos = e.pos_ + e.rot_ * origins[beam_header_id];
    const Vec3 end(p.x, p.y, p.z);
    mcl_3dl::Raycast<PointType>::CastResult point;
    const LidarMeasurementModelBeam::BeamStatus beam_status = beam_model.getBeamStatus(h->kdtree, pos, end, point);
    const bool lng = beam_status == LidarMeasurementModelBeam::BeamStatus::LONG;
    out[j++] = mcl3dl_beam_ray{{pos.x_, pos.y_, pos.z_},
                               {end.x_, end.y_, end.z_},
                               {lng ? nan : point.pos_.x_, lng ? nan : point.pos_.y_, lng ? nan : point.pos_.z_},
                               static_cast<uint32_t>(beam_status)};
  }
  return MCL3DL_OK;
}

}  // extern "C"
