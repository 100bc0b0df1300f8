/*
 * pf_events_api.h — the CPU checkers of the node's per-particle events on the resident set: the odometry-noise redraw,
 * expansion resetting's noise and the IMU gravity update.  TEST INFRASTRUCTURE ONLY.
 *
 *   oracle/libmcl3dl_pf_events_oracle.so    "port"      : oracle/pf_events_oracle.cpp (the repo's restatement)
 *   oracle/_ref/libmcl3dl_pf_events_ref.so  "reference" : oracle/pf_events_ref_driver.cpp on the reference's own
 *                                                         pf::ParticleFilter, State6DOF, Quat, Vec3, NormalLikelihood and
 *                                                         ImuMeasurementModelGravity
 *
 * oracle/pf_events.mk builds them.  Both take the normal draws explicitly (the device draws them with Philox, the
 * reference with std::default_random_engine), so given the same draws they must agree bit for bit.  Nothing in the
 * product path (mcl_3dl_b200/) may include, link or load this.
 */
#ifndef MCL3DL_PF_EVENTS_API_H
#define MCL3DL_PF_EVENTS_API_H

#include <stddef.h>
#include <stdint.h>

#include "../include/mcl3dl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

const char* mcl3dl_cpu_pf_events_kind(void);

/* The node's update_noise_func (src/mcl_3dl.cpp:817-825) through pf_->predict on states[0..n), in place; z holds the
 * four standard-normal draws of each particle in draw order (ll, la, aa, al). */
int mcl3dl_cpu_pf_redraw(mcl3dl_state* states, size_t n, const float* z, double lin_lin, double lin_ang, double ang_lin,
                         double ang_ang);

/* pf_->noise(...) = addNoiseUsingNoiseGenerator (pf.h:226-237) on states[0..n), in place; org holds the six draws of
 * each particle (x y z roll pitch yaw, already times sigma, zero where sigma is zero). */
int mcl3dl_cpu_pf_noise(mcl3dl_state* states, size_t n, const float* org);

/* ImuMeasurementModelGravity(float(acc_var)).setAccMeasure(acc) + pf_->measure (pf.h:252-279) on (states, probs)[0..n):
 * probs becomes the posterior (or stays the prior when the float sum is not > 0); lik (may be NULL) receives each
 * particle's likelihood, *kept whether the update was applied, *sum the reference's float sum, *entropy its entropy_
 * (0 when not kept). */
int mcl3dl_cpu_pf_imu(const mcl3dl_state* states, float* probs, size_t n, const float acc[3], double acc_var, float* lik,
                      int* kept, float* sum, float* entropy);

#ifdef __cplusplus
}
#endif
#endif
