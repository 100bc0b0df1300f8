// beam_cast_hostsim.cpp — TEST INFRASTRUCTURE ONLY.
//
// Host driver for the ray markers of mcl3dl_beam_cast: the per-thread body of beam_cast_kernel (load_pose, qnormalized,
// transform_point, ray_origin, cast_ray_at / cast_ray_kd_at from mcl_3dl_b200/csrc/device_funcs.cuh) compiled for the
// host through cuda_shim.h, over the grids hostsim.cpp builds the way engine.cu does.  tests/test_beam_cast_on_host.py
// compares it with the CPU checkers of oracle/beam_cast_api.h.
#include "hostsim.cpp"

// One record per ray, the layout of mcl3dl_beam_ray.  Returns -1 on a label >= n_origins (the kernel's error flag).
extern "C" int hostsim_beam_cast(const mcl3dl_point* map, size_t n, const mcl3dl_lik_params* lp, const mcl3dl_beam_params* bp,
                                 const mcl3dl_pose* pose, const mcl3dl_point* pts, size_t n_pts, const float* origins_xyz,
                                 size_t n_origins, mcl3dl_beam_ray* out, int near_k, int near_kd_k, int use_field)
{
  if (!bp || (!bp->use_raycast_using_dda && !lp))
    return -1;
  for (size_t j = 0; j < n_pts; ++j)
    if (pts[j].label >= n_origins)
      return -1;
  HostMap m;
  build(m, map, n, lp, bp, 1.0f, near_k, near_kd_k, use_field);
  F3 pos;
  Q4 q;
  load_pose(pose, pos, q);
  const Q4 rn = qnormalized(q);
  for (size_t j = 0; j < n_pts; ++j)
  {
    const F3 end = transform_point(rn, pos, F3{pts[j].x, pts[j].y, pts[j].z});
    const F3 begin = ray_origin(pos, q, origins_xyz, pts[j].label);
    F3 at;
    const int st = bp->use_raycast_using_dda ? cast_ray_at(m.dda, begin, end, &at) : cast_ray_kd_at(m.kd, m.nn, m.dda, begin, end, &at);
    const float nan = std::numeric_limits<float>::quiet_NaN();
    out[j] = mcl3dl_beam_ray{{begin.x, begin.y, begin.z},
                             {end.x, end.y, end.z},
                             {st == ST_LONG ? nan : at.x, st == ST_LONG ? nan : at.y, st == ST_LONG ? nan : at.z},
                             static_cast<uint32_t>(st)};
  }
  return 0;
}
