/*
 * pf_landmark_api.h — the CPU checkers of the node's landmark update, odometry-error reset and published particle
 * poses on the resident set.  TEST INFRASTRUCTURE ONLY.
 *
 *   oracle/libmcl3dl_pf_landmark_oracle.so    "port"      : oracle/pf_landmark_oracle.cpp (the repo's restatement)
 *   oracle/_ref/libmcl3dl_pf_landmark_ref.so  "reference" : oracle/pf_landmark_ref_driver.cpp on the reference's own
 *                                                           pf::ParticleFilter, State6DOF::operator-, Quat::inv,
 *                                                           Quat::getRPY and Quat::normalize
 *
 * oracle/pf_landmark.mk builds them.  Eigen is not available to either: both take NormalLikelihoodNd<float, 6>'s a_ and
 * sigma_inv_ as given and evaluate -0.5 x^T S x in the order include/mcl3dl_b200.h fixes for
 * mcl3dl_particles_landmark_update.  Nothing in the product path (mcl_3dl_b200/) may include, link or load this.
 */
#ifndef MCL3DL_PF_LANDMARK_API_H
#define MCL3DL_PF_LANDMARK_API_H

#include <stddef.h>
#include <stdint.h>

#include "../include/mcl3dl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

const char* mcl3dl_cpu_pf_landmark_kind(void);

/* cbLandmark's pf_->measure (src/mcl_3dl.cpp:899-931, pf.h:252-279) on (states, probs)[0..n): measured = x y z, qx qy qz
 * qw (RAW), nd_a / sigma_inv (row-major) = NormalLikelihoodNd's a_ / sigma_inv_.  probs becomes the posterior (or stays
 * the prior when the float sum is not > 0); lik (may be NULL) receives each particle's likelihood, *kept whether the
 * update was applied, *sum the reference's float sum, *entropy its entropy_ (0 when not kept). */
int mcl3dl_cpu_pf_landmark(const mcl3dl_state* states, float* probs, size_t n, const float measured[7], float nd_a,
                           const float sigma_inv[36], float* lik, int* kept, float* sum, float* entropy);

/* The node's integ_reset_func through pf_->predict (src/mcl_3dl.cpp:190-195,653-658) on states[0..n), in place. */
int mcl3dl_cpu_pf_reset_odom_err(mcl3dl_state* states, size_t n);

/* publishParticles' poses (src/mcl_3dl.cpp:1101-1125): out[i] = position + rot_.normalized(), _pad = 0. */
int mcl3dl_cpu_pf_poses(const mcl3dl_state* states, size_t n, mcl3dl_pose* out);

#ifdef __cplusplus
}
#endif
#endif
