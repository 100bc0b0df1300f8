// beam_cast_oracle.cpp — TEST INFRASTRUCTURE ONLY ("port" checker of the ray markers).
//
// The repo-owned restatement (mcl3dl_oracle.cpp, compiled here as part of this translation unit so that its casters are
// at hand) plus the node's marker loop over them, reporting the position of the cast step that decided each ray:
// ddaCentre of the deciding cell, or the marching position kdStep reports.
#include "mcl3dl_oracle.cpp"

#include "beam_cast_api.h"

namespace
{
// beamStatus / beamStatusKd with the deciding step's CastResult::pos_ in *at
int castDda(const DdaGrid& g, const mcl3dl_beam_params& bp, const F3& lidar_pos, const F3& scan_pos, F3* at)
{
  DdaRay r;
  ddaSetRay(g, r, lidar_pos, scan_pos);
  int hit;
  while (ddaStep(g, r, &hit))
  {
    if (hit < 0)
      continue;
    const int st = classifyCollision(g.pts[hit], 1.0f, bp, scan_pos);
    if (st >= 0)
    {
      *at = ddaCentre(g, r.cur);
      return st;
    }
  }
  return ST_LONG;
}

int castKd(const KdCaster& c, const NnIndex& nn, const mcl3dl_point* map, const mcl3dl_beam_params& bp, const F3& lidar_pos,
           const F3& scan_pos, F3* at)
{
  KdRay r;
  kdSetRay(c, r, lidar_pos, scan_pos);
  int hit;
  float sin_ang;
  F3 step;
  while (kdStep(c, nn, r, &hit, &sin_ang, &step))
  {
    if (hit < 0)
      continue;
    const int st = classifyCollision(map[hit], sin_ang, bp, scan_pos);
    if (st >= 0)
    {
      *at = step;
      return st;
    }
  }
  return ST_LONG;
}
}  // namespace

extern "C" {

int mcl3dl_cpu_beam_cast(mcl3dl_cpu* h, const mcl3dl_pose* pose, const mcl3dl_point* pts, size_t n, const float* origins_xyz,
                         size_t n_origins, mcl3dl_beam_ray* out)
{
  if (!h || !pose || (n && (!pts || !out || !origins_xyz)))
    return MCL3DL_ERR_INVALID_ARG;
  for (size_t j = 0; j < n; ++j)
    if (pts[j].label >= n_origins)
      return MCL3DL_ERR_INVALID_ARG;
  const F3 pos{pose->px, pose->py, pose->pz};
  const Q4 rot{pose->qx, pose->qy, pose->qz, pose->qw};
  const Q4 rn = qnormalized(rot);
  const float nan = std::numeric_limits<float>::quiet_NaN();
  for (size_t j = 0; j < n; ++j)
  {
    const F3 end = transformPoint(rn, pos, F3{pts[j].x, pts[j].y, pts[j].z});
    const float* o = origins_xyz + 3 * pts[j].label;
    const F3 begin = add(pos, qrot(rot, F3{o[0], o[1], o[2]}));  // RAW rot_ (mcl_3dl.cpp:475)
    F3 at{nan, nan, nan};
    int st = ST_LONG;
    if (!h->raw.use_raycast_using_dda)
      st = castKd(h->kd, h->nn, h->map.data(), h->beam, begin, end, &at);
    else if (h->dda_ok)
      st = castDda(h->dda, h->beam, begin, end, &at);
    if (st == ST_LONG)
      at = F3{nan, nan, nan};
    out[j] = mcl3dl_beam_ray{{begin.x, begin.y, begin.z}, {end.x, end.y, end.z}, {at.x, at.y, at.z}, static_cast<uint32_t>(st)};
  }
  return MCL3DL_OK;
}

}  // extern "C"
