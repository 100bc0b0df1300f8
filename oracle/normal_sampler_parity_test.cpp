// normal_sampler_parity_test.cpp — TEST INFRASTRUCTURE ONLY.
//
// The normal-weighted sampler through the host C++ adapter (MeasurementBatcher::sampleWithNormalPrepared), with the
// statistics the node hands setParticleStatistics built by the reference's own particle filter: pf_->expectation() and
// pf_->covariance(1.0, 1.0) over a particle set seeded by the reference's initUsingNoiseGenerator.  Per case:
//   - info.max_weight, info.fpc_local and info.weight_shift equal the port's (oracle/normal_sampler_oracle.cpp:
//     |position block| -> normal_eigen.h's eigendecomposition -> the ladder and mean_rot.inv() * column 2 in the
//     reference's operation order).  The position covariance has negative off-diagonal entries and the mean rotation
//     is not the identity, so a missing abs, another eigenvalue order or column, or another x y z w order shows;
//   - per clipped point of both models, the device's neighbour counts equal the port's brute-force ones and its
//     fixed-point weights are within one unit of the port's std::acos weights of the same normals;
//   - both sampled scans equal the draw rule of include/mcl3dl_b200.h (Philox at (t, stream, 0x6e6f726d, t >> 32), the
//     first i with cum_i > r, first draws in draw order) recomputed here over the device's weights_q.
// Eigen is oracle/shim_ns's stand-in (its SelfAdjointEigenSolver calls the port's routine), so both sides use the same
// eigendecomposition.
//
//   normal_sampler_parity_test [n_particles]
//
// Built where a checkout of the reference exists (make -C oracle -f normal_sampler.mk normal-parity);
// tests/test_gpu_normal_sampler.py runs it on an H100.
#include <Eigen/Core>
#include <Eigen/Eigenvalues>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <random>
#include <vector>

#include <mcl_3dl/noise_generator_base.h>
#include <mcl_3dl/parameters.h>
#include <mcl_3dl/pf.h>
#include <mcl_3dl/state_6dof.h>

#include "../mcl_3dl_b200/host/lidar_measurement_model_b200.h"
#include "normal_sampler_api.h"

using namespace mcl_3dl;
using PF = mcl_3dl_b200::ParticleFilter;

namespace
{
int g_fail = 0;
#define EXPECT(cond, ...)                         \
  do                                              \
  {                                               \
    if (!(cond))                                  \
    {                                             \
      ++g_fail;                                   \
      if (g_fail < 20)                            \
      {                                           \
        std::fprintf(stderr, "FAIL %s: ", #cond); \
        std::fprintf(stderr, __VA_ARGS__);        \
        std::fprintf(stderr, "\n");               \
      }                                           \
    }                                             \
  } while (0)

// pos = mean + T z (T lower-triangular, row-major), rpy = mean + sigma_rpy z: a correlated position spread
class CorrelatedNoise : public NoiseGeneratorBase<float>
{
public:
  CorrelatedNoise(const float mean[6], const float t[9], float sigma_rpy) : sigma_rpy_(sigma_rpy)
  {
    mean_.assign(mean, mean + 6);
    std::memcpy(t_, t, sizeof(t_));
  }
  template <typename RANDOM_ENGINE>
  std::vector<float> operator()(RANDOM_ENGINE& engine) const
  {
    std::normal_distribution<float> nd(0.0f, 1.0f);
    float z[6];
    for (float& v : z) v = nd(engine);
    std::vector<float> o(6);
    for (int i = 0; i < 3; ++i) o[i] = mean_[i] + t_[i * 3] * z[0] + t_[i * 3 + 1] * z[1] + t_[i * 3 + 2] * z[2];
    for (int i = 3; i < 6; ++i) o[i] = mean_[i] + sigma_rpy_ * z[i];
    return o;
  }

private:
  float t_[9];
  float sigma_rpy_;
};

// ---- the draw rule, from include/mcl3dl_b200.h's layout (plain host arithmetic)
void philox(uint32_t c[4], uint64_t seed)
{
  uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
  for (int r = 0; r < 10; ++r)
  {
    const uint64_t p0 = uint64_t(0xD2511F53u) * c[0], p1 = uint64_t(0xCD9E8D57u) * c[2];
    const uint32_t n0 = static_cast<uint32_t>(p1 >> 32) ^ c[1] ^ k0, n1 = static_cast<uint32_t>(p1);
    const uint32_t n2 = static_cast<uint32_t>(p0 >> 32) ^ c[3] ^ k1, n3 = static_cast<uint32_t>(p0);
    c[0] = n0;
    c[1] = n1;
    c[2] = n2;
    c[3] = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
}
std::vector<uint32_t> drawRule(const std::vector<uint64_t>& q, uint32_t num, uint64_t seed, uint32_t stream)
{
  const size_t n = q.size();
  std::vector<uint32_t> out;
  if (n == 0 || num == 0)
    return out;
  if (n <= num)
  {
    for (uint32_t i = 0; i < n; ++i) out.push_back(i);
    return out;
  }
  std::vector<uint64_t> cum(n);
  uint64_t acc = 0;
  for (size_t i = 0; i < n; ++i) cum[i] = acc += q[i];
  std::vector<bool> seen(n, false);
  for (uint64_t t = 0; out.size() < num && t < (uint64_t(1) << 32); ++t)
  {
    uint32_t c[4] = {static_cast<uint32_t>(t), stream, 0x6e6f726du, static_cast<uint32_t>(t >> 32)};
    philox(c, seed);
    const uint64_t u = static_cast<uint64_t>(c[0]) | (static_cast<uint64_t>(c[1]) << 32);
    const uint64_t r = static_cast<uint64_t>((static_cast<unsigned __int128>(u) * acc) >> 64);
    const uint32_t i = static_cast<uint32_t>(std::upper_bound(cum.begin(), cum.end(), r) - cum.begin());
    if (!seen[i])
    {
      seen[i] = true;
      out.push_back(i);
    }
  }
  return out;
}

// the scan: a floor, two walls and a tilted slab in the models' clip windows
std::vector<mcl3dl_point> scene(uint32_t seed)
{
  std::mt19937 rng(seed);
  std::uniform_real_distribution<float> u(-1.0f, 1.0f);
  std::vector<mcl3dl_point> pts;
  for (int i = 0; i < 6000; ++i) pts.push_back(mcl3dl_point{6.0f * u(rng), 6.0f * u(rng), -0.6f, 0u});
  for (int i = 0; i < 2500; ++i) pts.push_back(mcl3dl_point{6.0f * u(rng), 3.0f, 0.45f + 1.05f * u(rng), 1u});
  for (int i = 0; i < 2500; ++i) pts.push_back(mcl3dl_point{-2.5f, 6.0f * u(rng), 0.45f + 1.05f * u(rng), 2u});
  for (int i = 0; i < 2000; ++i)
  {
    const float a = 1.5f * u(rng), b = 1.5f * u(rng);
    pts.push_back(mcl3dl_point{1.5f + a, -2.0f + b, 0.3f * a + 0.2f * b, 3u});
  }
  return pts;
}

void runCase(const char* name, mcl_3dl_b200::MeasurementBatcher& batcher, int n_particles, const float mean6[6], const float t[9],
             const PointCloudSamplerWithNormalParameters& prm, uint64_t seed)
{
  PF pf_ref(n_particles, 11);
  pf_ref.initUsingNoiseGenerator(CorrelatedNoise(mean6, t, 0.05f));
  const State6DOF mean = pf_ref.expectation();
  const std::vector<State6DOF> covariances = pf_ref.covariance(1.0, 1.0);

  const std::vector<mcl3dl_point> raw = scene(static_cast<uint32_t>(seed));
  mcl3dl_scan_params sp{};
  for (float& d : sp.downsample) d = 0.1f;
  sp.lik_clip_near = 0.5f;
  sp.lik_clip_far = 10.0f;
  sp.lik_clip_z_min = -2.0f;
  sp.lik_clip_z_max = 2.0f;
  sp.beam_clip_near = 0.5f;
  sp.beam_clip_far = 4.0f;
  sp.beam_clip_z_min = -2.0f;
  sp.beam_clip_z_max = 2.0f;
  sp.lik_num_points = 96;
  sp.beam_num_points = 3;
  sp.seed = seed;
  mcl3dl_scan_info si{};
  batcher.checked(mcl3dl_scan_prepare(batcher.engine(), raw.data(), raw.size(), &sp, &si), "mcl3dl_scan_prepare");

  mcl3dl_normal_sampler_info info{};
  using M = Eigen::Matrix<double, Eigen::Dynamic, Eigen::Dynamic>;
  batcher.sampleWithNormalPrepared<M, Eigen::SelfAdjointEigenSolver<M>>(mean, covariances, prm, sp.lik_num_points,
                                                                        sp.beam_num_points, seed, &info);

  // the statistics, as the port computes them from the same filter outputs
  float cov9[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) cov9[i * 3 + j] = covariances[i][j];
  const float rot[4] = {mean.rot_.x_, mean.rot_.y_, mean.rot_.z_, mean.rot_.w_};
  const double params[4] = {prm.perform_weighting_ratio_, prm.max_weight_ratio_, prm.max_weight_, prm.normal_search_range_};
  double c[4];
  mcl3dl_cpu_ns_consts(cov9, rot, params, c);
  const double max_weight = std::isfinite(c[0]) ? c[0] : 1.0;
  const float fpc[3] = {static_cast<float>(c[1]), static_cast<float>(c[2]), static_cast<float>(c[3])};
  EXPECT(info.max_weight == max_weight, "%s: max_weight %.17g vs port %.17g", name, info.max_weight, max_weight);
  EXPECT(std::memcmp(info.fpc_local, fpc, sizeof(fpc)) == 0, "%s: fpc_local (%.9g %.9g %.9g) vs port (%.9g %.9g %.9g)", name,
         info.fpc_local[0], info.fpc_local[1], info.fpc_local[2], fpc[0], fpc[1], fpc[2]);
  int e = 0;
  const double fr = std::frexp(max_weight > 1.0 ? max_weight : 1.0, &e);
  EXPECT(info.weight_shift == 32 - (fr == 0.5 ? e - 1 : e), "%s: weight_shift %d", name, info.weight_shift);

  const uint32_t nums[2] = {sp.lik_num_points, sp.beam_num_points};
  const uint32_t n_sample[2] = {info.n_lik, info.n_beam};
  for (int k = 0; k < 2; ++k)
  {
    size_t n = 0;
    batcher.checked(mcl3dl_scan_get(batcher.engine(), 1 + k, nullptr, 0, &n), "mcl3dl_scan_get");
    std::vector<mcl3dl_point> clipped(n), sample(std::max<size_t>(n, 1));
    if (n)
      batcher.checked(mcl3dl_scan_get(batcher.engine(), 1 + k, clipped.data(), n, &n), "mcl3dl_scan_get");
    std::vector<float> nrm(3 * n);
    std::vector<uint32_t> cnt(n), p_cnt(n);
    std::vector<uint64_t> q(n);
    size_t n_q = 0;
    batcher.checked(mcl3dl_scan_normals(batcher.engine(), k, nrm.data(), cnt.data(), q.data(), n, &n_q), "mcl3dl_scan_normals");
    EXPECT(n_q == n, "%s model %d: %zu normals for %zu clipped points", name, k, n_q, n);
    std::vector<float> p_nrm(3 * n);
    std::vector<double> w(n);
    if (n)
    {
      mcl3dl_cpu_ns_normals(clipped.data(), n, prm.normal_search_range_, p_nrm.data(), p_cnt.data());
      mcl3dl_cpu_ns_weights(nrm.data(), n, fpc, max_weight, w.data());
    }
    size_t bad_cnt = 0, bad_q = 0;
    for (size_t i = 0; i < n; ++i)
    {
      bad_cnt += cnt[i] != p_cnt[i];
      const double want = std::max(1.0, std::rint(std::ldexp(w[i], info.weight_shift)));
      bad_q += std::fabs(want - static_cast<double>(q[i])) > 1.0;
    }
    EXPECT(bad_cnt == 0, "%s model %d: %zu neighbour counts differ from the brute-force ones", name, k, bad_cnt);
    EXPECT(bad_q == 0, "%s model %d: %zu weights more than one unit from the port's", name, k, bad_q);

    const std::vector<uint32_t> idx = drawRule(q, nums[k], seed, static_cast<uint32_t>(k));
    size_t n_s = 0;
    batcher.checked(mcl3dl_scan_get(batcher.engine(), 3 + k, sample.data(), sample.size(), &n_s), "mcl3dl_scan_get");
    EXPECT(n_s == idx.size() && n_s == n_sample[k], "%s model %d: sample of %zu, draw rule %zu, info %u", name, k, n_s, idx.size(),
           n_sample[k]);
    size_t bad_s = 0;
    for (size_t j = 0; j < std::min(n_s, idx.size()); ++j)
      bad_s += std::memcmp(&sample[j], &clipped[idx[j]], sizeof(mcl3dl_point)) != 0;
    EXPECT(bad_s == 0, "%s model %d: %zu sampled points differ from the draw rule", name, k, bad_s);
    std::printf("%s model %d: %zu clipped, %u finite normals, %zu sampled, %u rounds, %llu draws\n", name, k, n,
                info.n_normal[k], n_s, info.rounds[k], static_cast<unsigned long long>(info.draws[k]));
  }
  std::printf("%s: max_weight %.6f, fpc_local (%.6f %.6f %.6f), F %d\n", name, info.max_weight, info.fpc_local[0],
              info.fpc_local[1], info.fpc_local[2], info.weight_shift);
}
}  // namespace

int main(int argc, char** argv)
{
  const int n_particles = argc > 1 ? std::atoi(argv[1]) : 1000;
  auto lik_params = std::make_shared<LidarMeasurementModelLikelihoodParameters>();
  auto beam_params = std::make_shared<LidarMeasurementModelBeamParameters>();
  const float dist_weight[4] = {1.f, 1.f, 5.f, 0.f};
  PF pf_dummy(1, 1);
  mcl_3dl_b200::MeasurementBatcher batcher(&pf_dummy, std::vector<int>{0}, lik_params, beam_params, dist_weight);
  const PointCloudSamplerWithNormalParameters defaults;  // the node's: 2, 5, 5, 0.4

  // an elongated spread along x - y (negative xy covariance) under a rotated mean: the strong branch
  const float mean_a[6] = {1.0f, -0.5f, 0.2f, 0.15f, -0.1f, 0.7f};
  const float t_a[9] = {0.8f, 0.0f, 0.0f, -0.75f, 0.08f, 0.0f, 0.02f, -0.03f, 0.05f};
  runCase("elongated", batcher, n_particles, mean_a, t_a, defaults, 0x5eed0001ull);
  // a milder spread along y - z: the interpolated branch
  const float mean_b[6] = {-0.3f, 0.4f, 0.0f, -0.2f, 0.3f, -2.5f};
  const float t_b[9] = {0.12f, 0.0f, 0.0f, 0.05f, 0.25f, 0.0f, -0.02f, -0.2f, 0.1f};
  runCase("interpolated", batcher, n_particles, mean_b, t_b, defaults, 0x5eed0002ull);
  // an isotropic spread: max_weight 1, with other parameters
  PointCloudSamplerWithNormalParameters other;
  other.perform_weighting_ratio_ = 1.5;
  other.max_weight_ratio_ = 3.0;
  other.max_weight_ = 9.0;
  other.normal_search_range_ = 0.3;
  const float mean_c[6] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 1.2f};
  const float t_c[9] = {0.3f, 0.0f, 0.0f, 0.0f, 0.3f, 0.0f, 0.0f, 0.0f, 0.3f};
  runCase("isotropic", batcher, n_particles, mean_c, t_c, other, 0x5eed0003ull);

  if (g_fail)
  {
    std::printf("normal sampler parity FAILED (%d)\n", g_fail);
    return 1;
  }
  std::printf("NORMAL SAMPLER PARITY OK\n");
  return 0;
}
