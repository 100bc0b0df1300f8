// match_ref_driver.cpp — TEST INFRASTRUCTURE ONLY ("reference" checker of the matched / unmatched output).
//
// ref_driver.cpp (the C-ABI driver around the reference's own sources, compiled here as part of this translation unit)
// plus the node's matched / unmatched loop itself, run on the reference's State6DOF and ChunkedKdtree.
#include "ref_driver.cpp"

#include "match_api.h"

extern "C" {

// src/mcl_3dl.cpp:770-788: State6DOF::transform of a copy of the cloud, then
// kdtree_->radiusSearch(p, unmatch_output_dist, id, sqdist, 1) per point.  cls: 1 matched, 2 unmatched, 0 neither.
int mcl3dl_cpu_match_output(mcl3dl_cpu* h, const mcl3dl_pose* pose, const mcl3dl_point* pts, size_t n, double match_dist,
                            double unmatch_dist, uint8_t* cls)
{
  if (!h || !pose || (n && (!pts || !cls)))
    return MCL3DL_ERR_INVALID_ARG;
  const State6DOF e(Vec3(pose->px, pose->py, pose->pz), Quat(pose->qx, pose->qy, pose->qz, pose->qw));
  Cloud::Ptr pc_local = toCloud(pts, n);
  e.transform(*pc_local);
  std::vector<int> id(1);
  std::vector<float> sqdist(1);
  const double match_dist_sq = match_dist * match_dist;
  try
  {
    for (size_t i = 0; i < n; ++i)
    {
      const PointType& p = pc_local->points[i];
      if (!h->kdtree->radiusSearch(p, unmatch_dist, id, sqdist, 1))
        cls[i] = 2;
      else if (sqdist[0] < match_dist_sq)
        cls[i] = 1;
      else
        cls[i] = 0;
    }
  }
  catch (const std::runtime_error&)
  {
    return MCL3DL_ERR_INVALID_ARG;
  }
  return MCL3DL_OK;
}

}  // extern "C"
