// normal_sampler_api.h — TEST INFRASTRUCTURE ONLY: the C interface of the normal-weighted sampler checkers
// (oracle/normal_sampler.mk, bound by oracle/normal_sampler_checker.py).
//   port      (libmcl3dl_normal_oracle.so):     a repo-written restatement of PointCloudSamplerWithNormal
//   reference (_ref/libmcl3dl_normal_ref.so):   the reference's own PointCloudSamplerWithNormal<PointXYZIL>, compiled
//                                               against shim_ns/ (NormalEstimation, a double SelfAdjointEigenSolver and
//                                               ros::WallTime stand-ins that call normal_eigen.h)
#ifndef ORACLE_NORMAL_SAMPLER_API_H
#define ORACLE_NORMAL_SAMPLER_API_H
#include <stddef.h>
#include <stdint.h>

#include "../include/mcl3dl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif
const char* mcl3dl_cpu_ns_kind(void);
/* setParticleStatistics(mean, covariances) + sample(pc, num) of a sampler seeded with `seed`
 * (std::default_random_engine(seed)).  cov: the 3 x 3 position block of the covariances as the State6DOF rows hold it
 * (float, row-major, signed); params: perform_weighting_ratio, max_weight_ratio, max_weight, normal_search_range.
 * out: the sample's points in output order (capacity >= min(num, n)); *n_out its size.  consts (may be NULL): max_weight
 * as sample() computes it, fpc_local[3] (port only; the reference tier leaves them 0). */
int mcl3dl_cpu_ns_sample(const mcl3dl_point* pts, size_t n, const float cov[9], const float mean_rot[4], const double params[4],
                         size_t num, uint32_t seed, mcl3dl_point* out, size_t* n_out, double consts[4]);
/* port only: the pieces of sample() alone */
void mcl3dl_cpu_ns_consts(const float cov[9], const float mean_rot[4], const double params[4], double consts[4]);
void mcl3dl_cpu_ns_normals(const mcl3dl_point* pts, size_t n, double r, float* normals, uint32_t* counts);
void mcl3dl_cpu_ns_weights(const float* normals, size_t n, const float fpc[3], double max_weight, double* w);
void mcl3dl_cpu_ns_select(const double* w, size_t n, size_t num, uint32_t seed, uint64_t* out);
void mcl3dl_cpu_ns_eigen(const float cov[9], double vals[3], double vecs[9]);
#ifdef __cplusplus
}
#endif
#endif
