/*
 * gl_api.h — the CPU checkers of global localisation and of resizing the particle set.  TEST INFRASTRUCTURE ONLY.
 *
 *   oracle/libmcl3dl_gl_oracle.so    "port"      : oracle/gl_oracle.cpp (the repo's restatement)
 *   oracle/_ref/libmcl3dl_gl_ref.so  "reference" : oracle/gl_ref_driver.cpp on the reference's own ParticleFilter, Quat,
 *                                                  Vec3 and State6DOF and the shim KdTreeFLANN
 *
 * oracle/gl.mk builds them.  PCL is absent, so neither runs a VoxelGrid: both take the downsampled cloud, which the
 * tests compute with tests/hostsim/scan_hostsim.cpp's hostsim_scan_voxel_grid (bit-exact with the device).  Nothing in
 * the product path (mcl_3dl_b200/) may include, link or load this.
 */
#ifndef MCL3DL_GL_API_H
#define MCL3DL_GL_API_H

#include <stddef.h>
#include <stdint.h>

#include "../include/mcl3dl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

const char* mcl3dl_cpu_gl_kind(void);

/* The node's global_localization service (src/mcl_3dl.cpp:1039-1099) after its VoxelGrid: the free-space filter of the
 * downsampled cloud ds[0..n) (radiusSearch of p raised by 0.01 + grid, radius grid, with the node's point representation
 * rescaled by dist_weight) and the particles of the survivors, div_yaw headings each.  *n_particles = survivors * div_yaw;
 * states / probs (either may be NULL) receive them when cap >= *n_particles (INVALID_ARG otherwise). */
int mcl3dl_cpu_gl_seed(const mcl3dl_point* ds, size_t n, double grid, int32_t div_yaw, const float imu_quat[4],
                       const float dist_weight[3], mcl3dl_state* states, float* probs, size_t cap, size_t* n_particles);

/* pf::ParticleFilter<State6DOF>::resizeParticle(num) (pf.h:399-436) of the set (probs, states)[0..n); out_* hold num. */
int mcl3dl_cpu_pf_resize_6dof(const float* probs, const mcl3dl_state* states, size_t n, size_t num, mcl3dl_state* out_states,
                              float* out_probs);

#ifdef __cplusplus
}
#endif
#endif
