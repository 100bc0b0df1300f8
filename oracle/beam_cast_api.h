/*
 * beam_cast_api.h — the CPU checkers of the ray markers (mcl3dl_beam_cast).  TEST INFRASTRUCTURE ONLY.
 *
 *   oracle/libmcl3dl_beam_cast_oracle.so    "port"      : oracle/mcl3dl_oracle.cpp + oracle/beam_cast_oracle.cpp
 *   oracle/_ref/libmcl3dl_beam_cast_ref.so  "reference" : oracle/ref_driver.cpp + oracle/beam_cast_ref_driver.cpp, with the
 *                                                         reference's own sources as for libmcl3dl_ref.so
 *
 * Each library exports everything of oracle_api.h plus the function below (oracle/beam_cast.mk builds them).  Nothing in
 * the product path (mcl_3dl_b200/) may include, link or load this.
 */
#ifndef MCL3DL_BEAM_CAST_API_H
#define MCL3DL_BEAM_CAST_API_H

#include "oracle_api.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The node's ray-marker loop (src/mcl_3dl.cpp:468-478) from one pose over this checker's map and beam model: the scan
 * transformed by the pose (State6DOF::transform), begin = pos_ + rot_ * origins[label], getBeamStatus(kdtree, begin,
 * end, point).  One mcl3dl_beam_ray per point, in scan order; pos = point.pos_ for every status but LONG, NaN for LONG.
 * INVALID_ARG for a label >= n_origins. */
int mcl3dl_cpu_beam_cast(mcl3dl_cpu*, const mcl3dl_pose* pose, const mcl3dl_point* pts, size_t n, const float* origins_xyz,
                         size_t n_origins, mcl3dl_beam_ray* out);

#ifdef __cplusplus
}
#endif
#endif
