// match_hostsim.cpp — TEST INFRASTRUCTURE ONLY.
//
// Host driver for mcl_3dl_b200/csrc/match_funcs.cuh (the matched / unmatched output of mcl3dl_match_output), compiled
// for the host through cuda_shim.h over the likelihood grid that hostsim.cpp builds the way engine.cu does.  The loop
// below stands in for match_classify_kernel; tests/test_match_output_cpu.py compares it with the CPU checkers.
#include "hostsim.cpp"

#include "../../mcl_3dl_b200/csrc/match_funcs.cuh"

// cls[i]: MATCH_MATCHED 1, MATCH_UNMATCHED 2, MATCH_NEITHER 0; tf: the transformed points (label passed through)
extern "C" int hostsim_match_output(const mcl3dl_point* map, size_t n, const mcl3dl_lik_params* lp, const mcl3dl_pose* pose,
                                    const mcl3dl_point* pts, size_t n_pts, double match_dist, double unmatch_dist,
                                    float chunk_length, float max_search_radius, uint8_t* cls, mcl3dl_point* tf)
{
  HostMap hm;
  build(hm, map, n, lp, nullptr, 1.0f, 0, 0, 0);
  const float r = static_cast<float>(unmatch_dist);
  MatchDev m{};
  m.raw_pts = hm.raw_pts.data();
  m.r2 = static_cast<float>(static_cast<double>(r) * static_cast<double>(r));
  m.rpad = r * 1.0001f + 1e-6f;
  m.match_sq = match_dist * match_dist;
  m.chunk_length = chunk_length;
  m.pos_to_chunk = static_cast<float>(1.0 / static_cast<double>(chunk_length));
  m.max_search_radius = max_search_radius;
  const Q4 rn = qnormalized(Q4{pose->qx, pose->qy, pose->qz, pose->qw});
  for (size_t i = 0; i < n_pts; ++i)
  {
    const F3 t = transform_point(rn, F3{pose->px, pose->py, pose->pz}, F3{pts[i].x, pts[i].y, pts[i].z});
    cls[i] = static_cast<uint8_t>(match_classify(hm.nn, m, t));
    tf[i] = mcl3dl_point{t.x, t.y, t.z, pts[i].label};
  }
  return 0;
}
