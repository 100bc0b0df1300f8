// match_oracle.cpp — TEST INFRASTRUCTURE ONLY ("port" checker of the matched / unmatched output).
//
// The repo-owned restatement (mcl3dl_oracle.cpp, compiled here as part of this translation unit so that its map index
// is at hand) plus the node's matched / unmatched loop over NnIndex::search, whose chunk visibility is pinned to the
// reference by tests/golden/chunked_radius_search_*.npz.
#include "mcl3dl_oracle.cpp"

#include "match_api.h"

extern "C" {

// src/mcl_3dl.cpp:770-788: cls 1 matched, 2 unmatched, 0 neither.  A non-finite transformed point is unmatched, which
// is what the reference gets on x86 (floor(NaN) converts to INT_MIN, no chunk has that id, radiusSearch returns 0).
int mcl3dl_cpu_match_output(mcl3dl_cpu* h, const mcl3dl_pose* pose, const mcl3dl_point* pts, size_t n, double match_dist,
                            double unmatch_dist, uint8_t* cls)
{
  if (!h || !pose || (n && (!pts || !cls)))
    return MCL3DL_ERR_INVALID_ARG;
  const float r = static_cast<float>(unmatch_dist);  // radiusSearch(const float radius)
  if (r > h->nn.chunk_length)                         // chunked_kdtree.h:224-225 (throws there)
    return MCL3DL_ERR_INVALID_ARG;
  const Q4 rn = qnormalized(Q4{pose->qx, pose->qy, pose->qz, pose->qw});
  const F3 pos{pose->px, pose->py, pose->pz};
  const double match_dist_sq = match_dist * match_dist;
  for (size_t i = 0; i < n; ++i)
  {
    const F3 t = transformPoint(rn, pos, F3{pts[i].x, pts[i].y, pts[i].z});
    if (!std::isfinite(t.x) || !std::isfinite(t.y) || !std::isfinite(t.z))
    {
      cls[i] = 2;
      continue;
    }
    float d2 = 0.0f;
    if (h->nn.search(t, r, &d2) < 0)
      cls[i] = 2;
    else
      cls[i] = d2 < match_dist_sq ? 1 : 0;
  }
  return MCL3DL_OK;
}

}  // extern "C"
