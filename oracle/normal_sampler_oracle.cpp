// normal_sampler_oracle.cpp — TEST INFRASTRUCTURE ONLY ("port" checker of oracle/normal_sampler_api.h).
//
// PointCloudSamplerWithNormal (setParticleStatistics + sample) restated: |position covariance| -> normal_eigen.h's
// eigendecomposition; the max_weight ladder and fpc_local in the reference's operation order (float Quat arithmetic);
// brute-force normals (normal_eigen.h); per-point weights with std::acos; a sequential double cumulative sum; and the
// reference's selection loop: uniform_real_distribution<double>(0, total) from std::default_random_engine(seed),
// lower_bound, an unordered_set until num distinct indices, output in the set's iteration order.  Also the pieces alone,
// for the tests: the brute-force normals, the weights and the selection over given weights.
#include <algorithm>
#include <cmath>
#include <random>
#include <unordered_set>
#include <vector>

#include "normal_eigen.h"
#include "normal_sampler_api.h"

namespace
{
struct Q
{
  float x, y, z, w;
};
Q qmul(const Q& a, const Q& b)
{
  return Q{a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
           a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}

// sample()'s weight of one normal (point_cloud_sampler_with_normal.h:142-156)
double weight(const float* nrm, const float f[3], double max_weight)
{
  if (std::isnan(nrm[0]) || std::isnan(nrm[1]) || std::isnan(nrm[2]))
    return 1.0;
  double a = std::abs(nrm[0] * f[0] + nrm[1] * f[1] + nrm[2] * f[2]);
  if (a > 1.0)
    a = 1.0;
  const double angle = std::acos(a);
  return 1.0 + (max_weight - 1.0) * ((M_PI / 2 - angle) / (M_PI / 2));
}

// the selection loop over cumulative weights (:159-172); returns the indices in unordered_set iteration order
std::vector<size_t> select(const std::vector<double>& cum, size_t num, uint32_t seed)
{
  std::default_random_engine engine(seed);
  std::uniform_real_distribution<double> ud(0, cum.back());
  std::unordered_set<size_t> ids;
  while (true)
  {
    const double u = ud(engine);
    ids.insert(std::lower_bound(cum.begin(), cum.end(), u) - cum.begin());
    if (ids.size() >= num)
      break;
  }
  return std::vector<size_t>(ids.begin(), ids.end());
}
}  // namespace

extern "C" {
const char* mcl3dl_cpu_ns_kind(void) { return "port"; }

void mcl3dl_cpu_ns_normals(const mcl3dl_point* pts, size_t n, double r, float* normals, uint32_t* counts)
{
  oracle_ns::normals(&pts[0].x, 4, n, r, normals, counts);
}

void mcl3dl_cpu_ns_weights(const float* normals, size_t n, const float fpc[3], double max_weight, double* w)
{
  for (size_t i = 0; i < n; ++i) w[i] = weight(normals + 3 * i, fpc, max_weight);
}

// the selection loop over the sequential double sum of given weights -> indices (out: capacity num)
void mcl3dl_cpu_ns_select(const double* w, size_t n, size_t num, uint32_t seed, uint64_t* out)
{
  std::vector<double> cum(n);
  for (size_t i = 0; i < n; ++i) cum[i] = w[i] + (i == 0 ? 0.0 : cum[i - 1]);
  const std::vector<size_t> ids = select(cum, num, seed);
  for (size_t j = 0; j < ids.size(); ++j) out[j] = ids[j];
}

// setParticleStatistics' eigendecomposition of |cov| (float entries, as State6DOF holds them) -> vals[3], vecs[9]
void mcl3dl_cpu_ns_eigen(const float cov[9], double vals[3], double vecs[9])
{
  double a[9];
  for (int k = 0; k < 9; ++k) a[k] = std::abs(cov[k]);
  oracle_ns::sym3_eigen(a, vals, vecs);
}

// sample()'s max_weight (before any non-finite rule) and fpc_local, from setParticleStatistics' |cov| eigendecomposition
void mcl3dl_cpu_ns_consts(const float cov[9], const float mean_rot[4], const double params[4], double consts[4])
{
  double vals[3], vecs[9];
  mcl3dl_cpu_ns_eigen(cov, vals, vecs);
  const double ratio = std::sqrt(vals[2] / vals[1]);
  double max_weight = 1.0;
  if (ratio < params[0])
    max_weight = 1.0;
  else if (ratio > params[1])
    max_weight = params[2];
  else
    max_weight = 1.0 + (params[2] - 1.0) * ((ratio - params[0]) / (params[1] - params[0]));
  const Q r{mean_rot[0], mean_rot[1], mean_rot[2], mean_rot[3]};
  const float dot = r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w;
  const float s = static_cast<float>(1.0 / dot);
  const Q iv{-r.x * s, -r.y * s, -r.z * s, r.w * s};
  const Q o = qmul(qmul(iv, Q{static_cast<float>(vecs[2]), static_cast<float>(vecs[5]), static_cast<float>(vecs[8]), 0.0f}),
                   Q{-iv.x, -iv.y, -iv.z, iv.w});
  consts[0] = max_weight;
  consts[1] = o.x;
  consts[2] = o.y;
  consts[3] = o.z;
}

int mcl3dl_cpu_ns_sample(const mcl3dl_point* pts, size_t n, const float cov[9], const float mean_rot[4], const double params[4],
                         size_t num, uint32_t seed, mcl3dl_point* out, size_t* n_out, double consts[4])
{
  *n_out = 0;
  if (n == 0 || num == 0)
    return 0;
  if (n <= num)
  {
    std::copy(pts, pts + n, out);
    *n_out = n;
    return 0;
  }
  double c[4];
  mcl3dl_cpu_ns_consts(cov, mean_rot, params, c);
  const double max_weight = c[0];
  const float fpc[3] = {static_cast<float>(c[1]), static_cast<float>(c[2]), static_cast<float>(c[3])};
  if (consts)
    std::copy(c, c + 4, consts);
  std::vector<float> nrm(3 * n);
  oracle_ns::normals(&pts[0].x, 4, n, params[3], nrm.data(), nullptr);
  std::vector<double> cum(n);
  for (size_t i = 0; i < n; ++i) cum[i] = weight(nrm.data() + 3 * i, fpc, max_weight) + (i == 0 ? 0.0 : cum[i - 1]);
  const std::vector<size_t> ids = select(cum, num, seed);
  for (size_t j = 0; j < ids.size(); ++j) out[j] = pts[ids[j]];
  *n_out = ids.size();
  return 0;
}
}
