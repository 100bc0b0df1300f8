/*
 * pf_init_api.h — the CPU checkers of the resident set's initial seed (pf::ParticleFilter::initUsingNoiseGenerator with
 * the configured start's DiagonalNoiseGenerator and cbPosition's MultivariateNoiseGenerator).  TEST INFRASTRUCTURE ONLY.
 *
 *   oracle/libmcl3dl_pf_init_oracle.so    "port"      : oracle/pf_init_oracle.cpp (the repo's restatement)
 *   oracle/_ref/libmcl3dl_pf_init_ref.so  "reference" : oracle/pf_init_ref_driver.cpp on the reference's own
 *                                                       pf::ParticleFilter::initUsingNoiseGenerator,
 *                                                       State6DOF::generateNoise, NoiseGeneratorBase::setMean,
 *                                                       Quat::getRPY, Quat(rpy) and MultivariateNoiseGenerator
 *
 * oracle/pf_init.mk builds them.  Both take the six standard normals of every particle as given (the device's
 * counter-based draws are the documented departure from std::default_random_engine).  Eigen is not available: the
 * reference tier compiles MultivariateNoiseGenerator against oracle/shim_mv, a repo-written stand-in whose eigensolver is
 * not Eigen's bits.  Nothing in the product path (mcl_3dl_b200/) may include, link or load this.
 */
#ifndef MCL3DL_PF_INIT_API_H
#define MCL3DL_PF_INIT_API_H

#include <stddef.h>
#include <stdint.h>

#include "../include/mcl3dl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

const char* mcl3dl_cpu_pf_init_kind(void);

/* NoiseGeneratorBase::setMean(State6DOF(pos, rot)) (state_6dof.h:277-295): mean6 = x y z, rot.getRPY().
 * pose7 = x y z qx qy qz qw. */
int mcl3dl_cpu_pf_init_mean(const float pose7[7], float mean6[6]);

/* pf_->initUsingNoiseGenerator (pf.h:174-181) on n particles whose generator draws the standard normals z[i * 6 + k]:
 *   multivariate = 0: DiagonalNoiseGenerator<float>(State6DOF(pose7), sigma) with sigma6 = x y z, then rpy_ (setSigma);
 *   multivariate = 1: MultivariateNoiseGenerator<float> with mean_vec_ from pose7 and norm_transform_ = T (row-major).
 * states / probs [n] receive the seeded particles. */
int mcl3dl_cpu_pf_init(size_t n, int multivariate, const float pose7[7], const float sigma6[6], const float T[36],
                       const float* z, mcl3dl_state* states, float* probs);

/* MultivariateNoiseGenerator<float>::setCovariance (multivariate_noise_generator.h:58-74): T = norm_transform_ (row-major)
 * of the 36 doubles read row-major.  Reference tier only (oracle/shim_mv's eigensolver); the port returns INVALID_ARG. */
int mcl3dl_cpu_pf_init_transform(const double covariance[36], float T[36]);

#ifdef __cplusplus
}
#endif
#endif
