/*
 * match_api.h — the CPU checkers of the matched / unmatched output.  TEST INFRASTRUCTURE ONLY.
 *
 *   oracle/libmcl3dl_match_oracle.so    "port"      : oracle/mcl3dl_oracle.cpp + oracle/match_oracle.cpp
 *   oracle/_ref/libmcl3dl_match_ref.so  "reference" : oracle/ref_driver.cpp + oracle/match_ref_driver.cpp, with the
 *                                                     reference's own sources as for libmcl3dl_ref.so
 *
 * Each library exports everything of oracle_api.h plus the function below (oracle/match.mk builds them).  Nothing in
 * the product path (mcl_3dl_b200/) may include, link or load this.
 */
#ifndef MCL3DL_MATCH_API_H
#define MCL3DL_MATCH_API_H

#include "oracle_api.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The node's matched / unmatched output loop (src/mcl_3dl.cpp:770-788) over this checker's map index: every point is
 * transformed by `pose` (State6DOF::transform) and searched with radiusSearch(p, unmatch_dist, id, sqdist, 1).
 * cls[i]: 1 matched (sqdist < match_dist^2 in double), 2 unmatched (no point within the radius), 0 neither.
 * INVALID_ARG where the reference throws (float(unmatch_dist) > chunk_length). */
int mcl3dl_cpu_match_output(mcl3dl_cpu*, const mcl3dl_pose* pose, const mcl3dl_point* pts, size_t n, double match_dist,
                            double unmatch_dist, uint8_t* cls);

#ifdef __cplusplus
}
#endif
#endif
