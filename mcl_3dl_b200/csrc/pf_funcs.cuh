// pf_funcs.cuh — per-particle pieces of scope row f3 (SURVEY.md §8f): motion prediction, systematic resampling, the
// State6DOF noise, the initial seed and the terms of the pose estimate, as per-thread device functions called by the kernels of
// pf_kernels.cuh (the resident particle set, mcl3dl_particles_*).  They are also compiled for the host by tests/hostsim
// and checked there against the oracle pieces that are pinned bit for bit to the reference build (tests/test_hostsim.py).
//
// Float rules as in device_math.cuh: explicit round-to-nearest operations in the reference's operand order.
// sinf / cosf / logf are the device's own (a few ulp from glibc's): on the GPU predict() and the noise quaternion are
// equal to the reference to rounding, not bit for bit; everything else (the resampling pick in particular) is exact.
#pragma once
#ifndef MCL3DL_HOSTSIM
#include <cuda_runtime.h>
#endif
#include <math.h>
#include <stdint.h>

#include "device_math.cuh"

namespace mcl3dl
{
// The State6DOF fields that predict() and resample() read and write (include/mcl_3dl/state_6dof.h:55-63), in the
// layout of the oracle's mcl3dl_cpu_motion_state: 17 floats.
struct PfState
{
  float pos[3];
  float rot[4];  // x y z w
  float noise_ll, noise_la, noise_al, noise_aa;
  float lin[3];  // odom_err_integ_lin_
  float ang[3];  // odom_err_integ_ang_
};

// What MotionPredictionModelDifferentialDrive::setOdoms leaves behind
// (motion_prediction_models/motion_prediction_model_differential_drive.h:46-54) plus the two decay factors of :65-66.
struct MotionDev
{
  F3 rel_t;          // relative_translation_
  Q4 rel_q;          // relative_quat_
  float rel_ang;     // relative_angle_
  float rel_t_norm;  // relative_translation_norm_
  float k_lin;       // float(1.0 - time_diff / odom_err_integ_lin_tc)
  float k_ang;       // float(1.0 - time_diff / odom_err_integ_ang_tc)
};

__device__ __forceinline__ float qdot4(const Q4& a, const Q4& b)
{
  return fadd(fadd(fadd(fmul(a.x, b.x), fmul(a.y, b.y)), fmul(a.z, b.z)), fmul(a.w, b.w));  // quat.h:96-99
}
// Quat::operator/(float) == operator*(float(1.0 / s)), quat.h:148-151
__device__ __forceinline__ Q4 qdiv(const Q4& q, float s)
{
  const float inv = __double2float_rn(ddiv(1.0, static_cast<double>(s)));
  Q4 r;
  r.x = fmul(q.x, inv);
  r.y = fmul(q.y, inv);
  r.z = fmul(q.z, inv);
  r.w = fmul(q.w, inv);
  return r;
}
__device__ __forceinline__ Q4 qnormalize4(const Q4& q) { return qdiv(q, __fsqrt_rn(qdot4(q, q))); }  // quat.h:179-182

// Quat(Vec3(0, 0, 1), ang): setAxisAng on the unit z axis + normalize (quat.h:210-221,179-182)
__device__ __forceinline__ Q4 quat_about_z(float ang)
{
  const float half = fdiv(ang, 2.0f);
  Q4 q;
  q.x = fmul(0.0f, sinf(half));
  q.y = fmul(0.0f, sinf(half));
  q.z = fmul(1.0f, sinf(half));
  q.w = cosf(half);
  return qnormalize4(q);
}

// MotionPredictionModelDifferentialDrive::predict, :56-67, for one particle
__device__ __forceinline__ void pf_predict(PfState& s, const MotionDev& m)
{
  // diff = relative_translation_ * (1.0 + noise_ll_) + Vec3(noise_al_ * relative_angle_, 0, 0); the double factor is
  // narrowed to float by Vec3::operator*(float) (vec3.h:119)
  const float f = __double2float_rn(dadd(1.0, static_cast<double>(s.noise_ll)));
  F3 diff;
  diff.x = fadd(fmul(m.rel_t.x, f), fmul(s.noise_al, m.rel_ang));
  diff.y = fadd(fmul(m.rel_t.y, f), 0.0f);
  diff.z = fadd(fmul(m.rel_t.z, f), 0.0f);
  float lin[3] = {fadd(s.lin[0], fsub(diff.x, m.rel_t.x)), fadd(s.lin[1], fsub(diff.y, m.rel_t.y)),
                  fadd(s.lin[2], fsub(diff.z, m.rel_t.z))};
  Q4 rot;
  rot.x = s.rot[0];
  rot.y = s.rot[1];
  rot.z = s.rot[2];
  rot.w = s.rot[3];
  const F3 step = qrot(rot, diff);  // pos_ += rot_ * diff (raw rot_, two Hamilton products)
  s.pos[0] = fadd(s.pos[0], step.x);
  s.pos[1] = fadd(s.pos[1], step.y);
  s.pos[2] = fadd(s.pos[2], step.z);
  const float yaw_diff = fadd(fmul(s.noise_la, m.rel_t_norm), fmul(s.noise_aa, m.rel_ang));
  rot = qnormalize4(qmul(qmul(quat_about_z(yaw_diff), rot), m.rel_q));
  s.rot[0] = rot.x;
  s.rot[1] = rot.y;
  s.rot[2] = rot.z;
  s.rot[3] = rot.w;
  s.lin[0] = fmul(lin[0], m.k_lin);
  s.lin[1] = fmul(lin[1], m.k_lin);
  s.lin[2] = fmul(lin[2], m.k_lin);
  s.ang[0] = fmul(fadd(s.ang[0], 0.0f), m.k_ang);
  s.ang[1] = fmul(fadd(s.ang[1], 0.0f), m.k_ang);
  s.ang[2] = fmul(fadd(s.ang[2], yaw_diff), m.k_ang);
}

// Host side, once per odometry step: MotionPredictionModelDifferentialDrive::setOdoms (:46-54) and the decay factors.
// prev / cur = position + rotation (x y z w) of the two odometry states.  Plain host arithmetic (x86-64 without FMA
// contraction rounds every operation like the reference's own build); kept free of the __device__ helpers above so
// that the file also compiles in nvcc's host pass.
inline MotionDev pf_set_odoms(const float prev_pos[3], const float prev_rot[4], const float cur_pos[3], const float cur_rot[4],
                              float time_diff, float tc_lin, float tc_ang)
{
  struct H
  {
    // Quat::operator*(Quat), quat.h:131-138
    static Q4 mul(const Q4& a, const Q4& b)
    {
      Q4 r;
      r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
      r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
      r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
      r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
      return r;
    }
  };
  const Q4 pr{prev_rot[0], prev_rot[1], prev_rot[2], prev_rot[3]}, cr{cur_rot[0], cur_rot[1], cur_rot[2], cur_rot[3]};
  // Quat::inv() = conj() / dot(*this) (quat.h:187-190); operator/(s) multiplies by float(1.0 / s) (:148-151)
  const float d = pr.x * pr.x + pr.y * pr.y + pr.z * pr.z + pr.w * pr.w;
  const float id = static_cast<float>(1.0 / d);
  const Q4 inv{-pr.x * id, -pr.y * id, -pr.z * id, pr.w * id};
  MotionDev m;
  // Quat * Vec3 = (q * (v, 0) * conj(q)).xyz (quat.h:139-143)
  const Q4 v{cur_pos[0] - prev_pos[0], cur_pos[1] - prev_pos[1], cur_pos[2] - prev_pos[2], 0.0f};
  const Q4 rv = H::mul(H::mul(inv, v), Q4{-inv.x, -inv.y, -inv.z, inv.w});
  m.rel_t = F3{rv.x, rv.y, rv.z};
  m.rel_q = H::mul(inv, cr);
  // Quat::getAxisAng (quat.h:222-235): only the angle is used afterwards
  if (fabs(static_cast<double>(m.rel_q.w)) >= 1.0 - 0.000001)
    m.rel_ang = 0.0f;
  else
  {
    m.rel_ang = static_cast<float>(acos(static_cast<double>(m.rel_q.w)) * 2.0);
    if (static_cast<double>(m.rel_ang) > M_PI)
      m.rel_ang = static_cast<float>(static_cast<double>(m.rel_ang) - 2.0 * M_PI);
  }
  m.rel_t_norm = sqrtf(m.rel_t.x * m.rel_t.x + m.rel_t.y * m.rel_t.y + m.rel_t.z * m.rel_t.z);
  m.k_lin = static_cast<float>(1.0 - static_cast<double>(time_diff / tc_lin));
  m.k_ang = static_cast<float>(1.0 - static_cast<double>(time_diff / tc_ang));
  return m;
}

// ---- systematic resampling, pf::ParticleFilter::resampleUsingNoiseGenerator (include/mcl_3dl/pf.h:186-225)
//
// accum[0..n) is the SEQUENTIAL float prefix sum of the probabilities (:189-194; a parallel scan rounds differently and
// would pick other particles at the boundaries, so the kernel has to accumulate in order).  Output particle i looks at
// pscan = pstep * i + initial_p and takes the first particle whose accum is not below it (std::lower_bound over the
// copy sorted by accum, :196,206; accum is non-decreasing, so the sort only permutes exact ties, i.e. zero-probability
// particles — those ties are resolved by index here, by std::sort's whim in the reference).
__device__ __forceinline__ uint32_t pf_lower_bound(const float* __restrict__ accum, uint32_t n, float pscan)
{
  uint32_t lo = 0, hi = n;  // first index with !(accum[idx] < pscan)
  while (lo < hi)
  {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(accum + mid) < pscan)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}

__device__ __forceinline__ float pf_pscan(float pstep, float initial_p, uint32_t i)
{
  return fadd(fmul(pstep, static_cast<float>(i)), initial_p);  // :205 (size_t -> float conversion, then float ops)
}

// Source particle of output i and whether the reference adds noise to it (:207-222):
//   it == end            -> the state of it_prev (the last particle any earlier output found), no noise;
//   it == it_prev        -> a duplicate: state + noise (output 0 compares with begin(), so it counts as a duplicate
//                           whenever it picks particle 0);
//   otherwise            -> a plain copy.
__device__ __forceinline__ uint32_t pf_pick(const float* __restrict__ accum, uint32_t n, float pstep, float initial_p,
                                            uint32_t i, bool& duplicate)
{
  const uint32_t it = pf_lower_bound(accum, n, pf_pscan(pstep, initial_p, i));
  if (it < n)
  {
    const uint32_t prev = i == 0 ? 0u : pf_lower_bound(accum, n, pf_pscan(pstep, initial_p, i - 1));
    duplicate = it == prev;  // (prev < n here: the picks never decrease)
    return it;
  }
  // past the end (rounding of pstep * i): the last output j < i that still found a particle decides
  duplicate = false;
  uint32_t lo = 0, hi = i;  // first j whose pick is past the end
  while (lo < hi)
  {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (pf_lower_bound(accum, n, pf_pscan(pstep, initial_p, mid)) < n)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo == 0 ? 0u : pf_lower_bound(accum, n, pf_pscan(pstep, initial_p, lo - 1));
}

// Quat(Vec3(rpy)) = Quat::setRPY (quat.h:202-215), rpy = (roll, pitch, yaw); not normalised
__device__ __forceinline__ Q4 quat_rpy(const float rpy[3])
{
  const float t2 = cosf(fdiv(rpy[0], 2.0f)), t3 = sinf(fdiv(rpy[0], 2.0f));
  const float t4 = cosf(fdiv(rpy[1], 2.0f)), t5 = sinf(fdiv(rpy[1], 2.0f));
  const float t0 = cosf(fdiv(rpy[2], 2.0f)), t1 = sinf(fdiv(rpy[2], 2.0f));
  Q4 q;
  q.x = fsub(fmul(fmul(t0, t3), t4), fmul(fmul(t1, t2), t5));
  q.y = fadd(fmul(fmul(t0, t2), t5), fmul(fmul(t1, t3), t4));
  q.z = fsub(fmul(fmul(t1, t2), t4), fmul(fmul(t0, t3), t5));
  q.w = fadd(fmul(fmul(t0, t2), t4), fmul(fmul(t1, t3), t5));
  return q;
}

// state + generateNoise(org[0..6)): State6DOF::generateNoise / operator+ (state_6dof.h:226-261), Quat::setRPY
// (quat.h:196-209).  org = the six draws (x y z roll pitch yaw); the noise mean is zero (DiagonalNoiseGenerator(State6DOF(),
// sigma)).  The result is a fresh State6DOF: noise_* = 0, and rot = nrot * rot as it comes, not normalised — what
// pf::ParticleFilter::addNoiseUsingNoiseGenerator leaves (pf.h:226-237).
__device__ __forceinline__ PfState pf_add_noise_raw(const PfState& s, const float org[6])
{
  const Q4 nrot = quat_rpy(org + 3);
  PfState r;
  r.noise_ll = r.noise_la = r.noise_al = r.noise_aa = 0.0f;
  for (int k = 0; k < 3; ++k)
  {
    r.pos[k] = fadd(s.pos[k], org[k]);
    r.lin[k] = fadd(s.lin[k], org[k]);                      // noise[i + 7] = org[i] (:238)
    r.ang[k] = fadd(s.ang[k], fsub(org[k + 3], 0.0f));      // noise[i + 10] = org[i + 3] - mean[i + 3] (:244)
  }
  Q4 rot;
  rot.x = s.rot[0];
  rot.y = s.rot[1];
  rot.z = s.rot[2];
  rot.w = s.rot[3];
  rot = qmul(nrot, rot);  // ret.rot_ = a.rot_ * rot_ with a = the noise (:259)
  r.rot[0] = rot.x;
  r.rot[1] = rot.y;
  r.rot[2] = rot.z;
  r.rot[3] = rot.w;
  return r;
}

// state + noise followed by normalize() (state_6dof.h:154-157), as resampling treats a duplicate (pf.h:216-217)
__device__ __forceinline__ PfState pf_add_noise(const PfState& s, const float org[6])
{
  PfState r = pf_add_noise_raw(s, org);
  Q4 rot;
  rot.x = r.rot[0];
  rot.y = r.rot[1];
  rot.z = r.rot[2];
  rot.w = r.rot[3];
  rot = qnormalize4(rot);
  r.rot[0] = rot.x;
  r.rot[1] = rot.y;
  r.rot[2] = rot.z;
  r.rot[3] = rot.w;
  return r;
}

// ---- counter-based random numbers for the device (documented departure from std::default_random_engine, whose
// stream a parallel kernel cannot reproduce: the reference draws six normals per DUPLICATE, in output order).
// Philox-4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11), key = seed, counter =
// (output index, call counter, stream).
__device__ __forceinline__ uint32_t mulhi32(uint32_t a, uint32_t b)
{
  return static_cast<uint32_t>((static_cast<uint64_t>(a) * static_cast<uint64_t>(b)) >> 32);
}

__device__ __forceinline__ void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1)
{
  for (int round = 0; round < 10; ++round)
  {
    const uint32_t hi0 = mulhi32(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    const uint32_t hi1 = mulhi32(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
    c[0] = n0;
    c[1] = n1;
    c[2] = n2;
    c[3] = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
}

// uniform in (0, 1]: never 0, so the logarithm below is finite
__device__ __forceinline__ float u01(uint32_t x) { return fmul(fadd(static_cast<float>(x >> 8), 1.0f), 5.9604644775390625e-08f); }

// The counter's fourth word names the event, so that the events of one seed draw from disjoint streams:
//   (index, call, block, kPfEventResample): resampling's duplicate noise, blocks 0 and 1 (pf_noise6);
//   (index, call, 0, kPfEventRedraw):       the odometry-noise redraw, one block = two Box-Muller pairs;
//   (index, call, block, kPfEventNoise):    expansion resetting's noise, blocks 0 and 1, laid out as pf_noise6;
//   (index, call, block, kPfEventInit):     the initial seed's six standard normals, blocks 0 and 1, the same layout.
// `call` is the entry point's own call count (1 on the first call of an engine).
constexpr uint32_t kPfEventResample = 0, kPfEventRedraw = 1, kPfEventNoise = 2, kPfEventInit = 3;

// The six standard normals of particle `index` of call `call` of `event`: the pairs (w0, w1), (w2, w3) of block 0 and
// (w0, w1) of block 1 give rad = sqrtf(-2 logf(u)) and phi = 2 pi v, and pair p's normals are z_2p = rad * cosf(phi)
// and z_2p+1 = rad * sinf(phi).  pair(p, rad, phi) forms them, so that a draw whose sigma is 0 needs no sine or cosine.
template <typename Pair>
__device__ __forceinline__ void pf_normal6_event(uint64_t seed, uint32_t index, uint32_t call, uint32_t event, Pair pair)
{
  uint32_t a[4] = {index, call, 0u, event}, b[4] = {index, call, 1u, event};
  const uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
  philox4x32_10(a, k0, k1);
  philox4x32_10(b, k0, k1);
  const uint32_t w[6] = {a[0], a[1], a[2], a[3], b[0], b[1]};
  for (int p = 0; p < 3; ++p)
  {
    const float rad = __fsqrt_rn(fmul(-2.0f, logf(u01(w[2 * p]))));
    const float phi = fmul(6.283185307179586f, u01(w[2 * p + 1]));
    pair(p, rad, phi);
  }
}

// six N(0, sigma_k) draws for particle `index` of call `call` of `event` (Box-Muller on three pairs)
__device__ __forceinline__ void pf_noise6_event(uint64_t seed, uint32_t index, uint32_t call, uint32_t event, const float sigma[6],
                                                float org[6])
{
  pf_normal6_event(seed, index, call, event, [&](int pair, float rad, float phi) {
    org[2 * pair] = sigma[2 * pair] == 0.0f ? 0.0f : fmul(fmul(rad, cosf(phi)), sigma[2 * pair]);
    org[2 * pair + 1] = sigma[2 * pair + 1] == 0.0f ? 0.0f : fmul(fmul(rad, sinf(phi)), sigma[2 * pair + 1]);
  });
}

// resampling's draws for output particle `index` of resampling call `call`
__device__ __forceinline__ void pf_noise6(uint64_t seed, uint32_t index, uint32_t call, const float sigma[6], float org[6])
{
  pf_noise6_event(seed, index, call, kPfEventResample, sigma, org);
}

// The node's update_noise_func (src/mcl_3dl.cpp:817-825) for particle `index` of redraw call `call`: four standard
// normals z0..z3 (Box-Muller on the two pairs of one Philox block), noise_x = float(double(z_k) * sigma_x) in the node's
// draw order ll, la, aa, al (the reference multiplies its float draw by the double parameter).  Nothing else changes.
struct OdomNoiseSigma
{
  double ll, la, aa, al;  // Parameters::odom_err_lin_lin_, _lin_ang_, _ang_ang_, _ang_lin_
};

__device__ __forceinline__ void pf_redraw_odom_noise(PfState& s, uint64_t seed, uint32_t index, uint32_t call, const OdomNoiseSigma& sg)
{
  uint32_t c[4] = {index, call, 0u, kPfEventRedraw};
  philox4x32_10(c, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  float z[4];
  for (int pair = 0; pair < 2; ++pair)
  {
    const float rad = __fsqrt_rn(fmul(-2.0f, logf(u01(c[2 * pair]))));
    const float phi = fmul(6.283185307179586f, u01(c[2 * pair + 1]));
    z[2 * pair] = fmul(rad, cosf(phi));
    z[2 * pair + 1] = fmul(rad, sinf(phi));
  }
  s.noise_ll = __double2float_rn(dmul(static_cast<double>(z[0]), sg.ll));
  s.noise_la = __double2float_rn(dmul(static_cast<double>(z[1]), sg.la));
  s.noise_aa = __double2float_rn(dmul(static_cast<double>(z[2]), sg.aa));
  s.noise_al = __double2float_rn(dmul(static_cast<double>(z[3]), sg.al));
}

// pf_->noise(State6DOF(sigma_pos, sigma_rpy)) for particle `index` of call `call` (pf.h:226-237): state + noise, the
// rotation NOT normalised and noise_* = 0, as the reference leaves them
__device__ __forceinline__ PfState pf_expansion_noise(const PfState& s, uint64_t seed, uint32_t index, uint32_t call, const float sigma[6])
{
  float org[6];
  pf_noise6_event(seed, index, call, kPfEventNoise, sigma, org);
  return pf_add_noise_raw(s, org);
}

// ---- the initial seed: pf::ParticleFilter::initUsingNoiseGenerator (pf.h:169-181) with the configured start's
// DiagonalNoiseGenerator or cbPosition's MultivariateNoiseGenerator.  mean = NoiseGeneratorBase::getMean() (x y z roll
// pitch yaw, setMean's getRPY on the host); sigma = DiagonalNoiseGenerator::sigma_; T = norm_transform_ (row-major).
struct InitDev
{
  int multivariate;  // 0: diagonal, 1: multivariate
  float mean[6];
  float sigma[6];
  float T[36];
};

// State6DOF::generateNoise (state_6dof.h:226-248) for particle `index` of init call `call`, from six standard normals z:
//   diagonal:     org_k = sigma_k == 0 ? mean_k : z_k * sigma_k + mean_k (libstdc++'s normal_distribution<float>);
//   multivariate: org_i = mean_i + t_i, t_i = sum over k ascending of T(i, k) z_k from its first product.
// pos = org[0..2], odom_err_integ_lin = org[0..2] (the mean included, as the reference leaves it), odom_err_integ_ang =
// org[3..5] - mean[3..5], rot = Quat(Vec3(org[3..5])) not normalised, noise_* = 0.
__device__ __forceinline__ PfState pf_init_state(uint64_t seed, uint32_t index, uint32_t call, const InitDev& g)
{
  float z[6], org[6];
  pf_normal6_event(seed, index, call, kPfEventInit, [&](int pair, float rad, float phi) {
    z[2 * pair] = fmul(rad, cosf(phi));
    z[2 * pair + 1] = fmul(rad, sinf(phi));
  });
  if (g.multivariate)
  {
#pragma unroll
    for (int i = 0; i < 6; ++i)
    {
      float t = fmul(g.T[i * 6], z[0]);
#pragma unroll
      for (int k = 1; k < 6; ++k) t = fadd(t, fmul(g.T[i * 6 + k], z[k]));
      org[i] = fadd(g.mean[i], t);
    }
  }
  else
  {
#pragma unroll
    for (int k = 0; k < 6; ++k) org[k] = g.sigma[k] == 0.0f ? g.mean[k] : fadd(fmul(z[k], g.sigma[k]), g.mean[k]);
  }
  PfState r;
  r.noise_ll = r.noise_la = r.noise_al = r.noise_aa = 0.0f;
  for (int k = 0; k < 3; ++k)
  {
    r.pos[k] = org[k];
    r.lin[k] = org[k];
    r.ang[k] = fsub(org[k + 3], g.mean[k + 3]);
  }
  const Q4 rot = quat_rpy(org + 3);
  r.rot[0] = rot.x;
  r.rot[1] = rot.y;
  r.rot[2] = rot.z;
  r.rot[3] = rot.w;
  return r;
}

// ---- IMU gravity update: ImuMeasurementModelGravity::setAccMeasure + measure (imu_measurement_model_gravity.h:45-55)
struct ImuDev
{
  F3 acc;          // acc_measure_
  float acc_norm;  // acc_measure_norm_ = Vec3::norm (vec3.h:153-156)
  float nd_a;      // NormalLikelihood<float>(float(acc_var)): a_ = float(1.0 / sqrt(2 pi s s)) (nd.h:45-49)
  float nd_sq2;    //   sq2_ = float(float(s * s) * 2.0)
};

// Host side, once per call, in the reference's operation order (plain host arithmetic, as pf_set_odoms)
inline ImuDev pf_imu_setup(const float acc[3], float sigma)
{
  ImuDev m;
  m.acc = F3{acc[0], acc[1], acc[2]};
  m.acc_norm = sqrtf(acc[0] * acc[0] + acc[1] * acc[1] + acc[2] * acc[2]);
  m.nd_a = static_cast<float>(1.0 / sqrt(2.0 * M_PI * sigma * sigma));
  m.nd_sq2 = static_cast<float>(sigma * sigma * 2.0);
  return m;
}

// The likelihood of one particle: acc_estim = rot.inv() * (0, 0, 1) with the RAW rot (Quat::inv = conj * float(1.0 / dot),
// quat.h:187-190, and the two-Hamilton-product rotation), diff = acosf(dot / (|acc_measure| * |acc_estim|)),
// nd(diff) = a * expf(-diff * diff / sq2).  An acosf argument that rounds above 1 gives NaN, as in the reference.
__device__ __forceinline__ float pf_imu_likelihood(const PfState& s, const ImuDev& m)
{
  Q4 r;
  r.x = s.rot[0];
  r.y = s.rot[1];
  r.z = s.rot[2];
  r.w = s.rot[3];
  Q4 cj;
  cj.x = -r.x;
  cj.y = -r.y;
  cj.z = -r.z;
  cj.w = r.w;
  const Q4 inv = qdiv(cj, qdot4(r, r));
  F3 ez;
  ez.x = 0.0f;
  ez.y = 0.0f;
  ez.z = 1.0f;
  const F3 e = qrot(inv, ez);
  const float diff = acosf(fdiv(dot3(e, m.acc), fmul(m.acc_norm, __fsqrt_rn(dot3(e, e)))));
  return fmul(m.nd_a, expf(fdiv(fmul(-diff, diff), m.nd_sq2)));
}

// ---- pose estimate (src/mcl_3dl.cpp:428-452,704-724): per-particle terms
// The bias of pf_->bias(bias_func), mcl_3dl.cpp:436-449: NormalLikelihood(bias_var_dist)(|pos - prev.pos|) *
// NormalLikelihood(bias_var_ang)(angle of rot * prev.rot.inv()) + 1e-6; nd.h:45-53 (a, sq2 as floats).
struct BiasDev
{
  float prev_pos[3];
  Q4 prev_inv;  // state_prev_.rot_.inv(), computed once on the host
  float lin_a, lin_sq2, ang_a, ang_sq2;
  int enabled;  // 0: the constant bias 1 of the global-localisation branch (mcl_3dl.cpp:428-434)
};

__device__ __forceinline__ float pf_bias(const PfState& s, const BiasDev& b)
{
  if (!b.enabled)
    return 1.0f;
  F3 d;
  d.x = fsub(s.pos[0], b.prev_pos[0]);
  d.y = fsub(s.pos[1], b.prev_pos[1]);
  d.z = fsub(s.pos[2], b.prev_pos[2]);
  const float lin_diff = __fsqrt_rn(dot3(d, d));
  Q4 r;
  r.x = s.rot[0];
  r.y = s.rot[1];
  r.z = s.rot[2];
  r.w = s.rot[3];
  const Q4 q = qmul(r, b.prev_inv);
  // Quat::getAxisAng, quat.h:226-239 (only the angle)
  float ang = 0.0f;
  if (!(fabs(static_cast<double>(q.w)) >= 1.0 - 0.000001))
  {
    ang = __double2float_rn(dmul(static_cast<double>(acosf(q.w)), 2.0));
    if (static_cast<double>(ang) > M_PI)
      ang = __double2float_rn(dsub(static_cast<double>(ang), 2.0 * M_PI));
  }
  const float nl = fmul(b.lin_a, expf(fdiv(fmul(-lin_diff, lin_diff), b.lin_sq2)));
  const float na = fmul(b.ang_a, expf(fdiv(fmul(-ang, ang), b.ang_sq2)));
  return __double2float_rn(dadd(static_cast<double>(fmul(nl, na)), 1e-6));
}

// Quat::getRPY, quat.h:191-201: double expressions narrowed to float, float atan2 / asin
__device__ __forceinline__ void pf_rpy(const float rot[4], float rpy[3])
{
  const float x = rot[0], y = rot[1], z = rot[2], w = rot[3];
  const float ysq = fmul(y, y);
  const float t0 = __double2float_rn(dadd(dmul(-2.0, static_cast<double>(fadd(ysq, fmul(z, z)))), 1.0));
  const float t1 = __double2float_rn(dmul(2.0, static_cast<double>(fadd(fmul(x, y), fmul(w, z)))));
  const double t2d = dmul(-2.0, static_cast<double>(fsub(fmul(x, z), fmul(w, y))));
  const float t2 = __double2float_rn(fmax(-1.0, fmin(1.0, t2d)));
  const float t3 = __double2float_rn(dmul(2.0, static_cast<double>(fadd(fmul(y, z), fmul(w, x)))));
  const float t4 = __double2float_rn(dadd(dmul(-2.0, static_cast<double>(fadd(fmul(x, x), ysq))), 1.0));
  rpy[0] = atan2f(t3, t4);
  rpy[1] = asinf(t2);
  rpy[2] = atan2f(t1, t0);
}

// ---- the landmark update of cbLandmark (src/mcl_3dl.cpp:899-940): NormalLikelihoodNd<float, 6> (nd.h:61-83) of the
// pose difference.  nd_a and sigma_inv are the reference's a_ and sigma_inv_, computed once per message on the host.
struct LandmarkDev
{
  float pos[3];          // measured.pos_
  Q4 rot;                // measured.rot_, RAW (as the message carries it)
  float nd_a;            // a_
  float sigma_inv[36];   // sigma_inv_, row-major: [r * 6 + c] = sigma_inv_(r, c)
};

// -0.5 x^T S x in the order include/mcl3dl_b200.h fixes, all in float: h_k = -0.5 x_k, r_j = sum over k ascending of
// h_k S(k, j), q = sum over j ascending of r_j x_j (each sum starts from its first product)
__device__ __forceinline__ float pf_nd6_exponent(const float x[6], const float S[36])
{
  float h[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) h[k] = fmul(-0.5f, x[k]);
  float q = 0.0f;
#pragma unroll
  for (int j = 0; j < 6; ++j)
  {
    float r = fmul(h[0], S[j]);
#pragma unroll
    for (int k = 1; k < 6; ++k) r = fadd(r, fmul(h[k], S[k * 6 + j]));
    q = j == 0 ? fmul(r, x[0]) : fadd(q, fmul(r, x[j]));
  }
  return q;
}

// x of one particle (cbLandmark's measure_func, src/mcl_3dl.cpp:913-926): diff = s - measured (State6DOF::operator-,
// state_6dof.h:262-274: pos_ - measured.pos_ per axis, rot_ = measured.rot_.inv() * rot_ with both rotations RAW and
// Quat::inv = conj * float(1.0 / dot)), x = (diff.pos_, diff.rot_.getRPY())
__device__ __forceinline__ void pf_landmark_x(const PfState& s, const LandmarkDev& m, float x[6])
{
  Q4 cj;
  cj.x = -m.rot.x;
  cj.y = -m.rot.y;
  cj.z = -m.rot.z;
  cj.w = m.rot.w;
  Q4 r;
  r.x = s.rot[0];
  r.y = s.rot[1];
  r.z = s.rot[2];
  r.w = s.rot[3];
  const Q4 d = qmul(qdiv(cj, qdot4(m.rot, m.rot)), r);
  const float drot[4] = {d.x, d.y, d.z, d.w};
  for (int k = 0; k < 3; ++k) x[k] = fsub(s.pos[k], m.pos[k]);
  pf_rpy(drot, x + 3);
}

// The likelihood of one particle: a * expf(-0.5 x^T S x) (nd.h:76-79)
__device__ __forceinline__ float pf_landmark_likelihood(const PfState& s, const LandmarkDev& m)
{
  float x[6];
  pf_landmark_x(s, m, x);
  return fmul(m.nd_a, expf(pf_nd6_exponent(x, m.sigma_inv)));
}

// The node's integ_reset_func through pf_->predict (src/mcl_3dl.cpp:190-195,653-658): odom_err_integ_lin_ = Vec3(),
// odom_err_integ_ang_ = Vec3()
__device__ __forceinline__ void pf_reset_odom_err_integ(PfState& s)
{
#pragma unroll
  for (int k = 0; k < 3; ++k)
  {
    s.lin[k] = 0.0f;
    s.ang[k] = 0.0f;
  }
}

// What publishParticles (src/mcl_3dl.cpp:1101-1125) publishes for one particle: the position and rot_.normalized()
// (quat.h:175-177, q * float(1.0 / double(sqrtf(dot)))); _pad = 0
__device__ __forceinline__ void pf_published_pose(const PfState& s, float out[8])
{
  Q4 r;
  r.x = s.rot[0];
  r.y = s.rot[1];
  r.z = s.rot[2];
  r.w = s.rot[3];
  r = qnormalize4(r);
  out[0] = s.pos[0];
  out[1] = s.pos[1];
  out[2] = s.pos[2];
  out[3] = 0.0f;
  out[4] = r.x;
  out[5] = r.y;
  out[6] = r.z;
  out[7] = r.w;
}

// the terms ParticleWeightedMeanQuat::add accumulates (state_6dof.h:327-341): pos, rot * (1,0,0), rot * (0,0,1) (RAW rot)
__device__ __forceinline__ void pf_mean_terms(const PfState& s, float out[9])
{
  Q4 r;
  r.x = s.rot[0];
  r.y = s.rot[1];
  r.z = s.rot[2];
  r.w = s.rot[3];
  F3 ex, ez;
  ex.x = 1.0f;
  ex.y = 0.0f;
  ex.z = 0.0f;
  ez.x = 0.0f;
  ez.y = 0.0f;
  ez.z = 1.0f;
  const F3 front = qrot(r, ex), up = qrot(r, ez);
  out[0] = s.pos[0];
  out[1] = s.pos[1];
  out[2] = s.pos[2];
  out[3] = front.x;
  out[4] = front.y;
  out[5] = front.z;
  out[6] = up.x;
  out[7] = up.y;
  out[8] = up.z;
}

// Quat(forward, up_raw), quat.h:59-75, from double sums (the filter's sums are float; the device sums in double)
__device__ __forceinline__ void pf_quat_from_front_up(const double f[3], const double u[3], float q[4])
{
  auto unit = [](double v[3]) {
    const double n = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    v[0] /= n;
    v[1] /= n;
    v[2] /= n;
  };
  double xv[3] = {f[0], f[1], f[2]};
  unit(xv);
  double yv[3] = {u[1] * xv[2] - u[2] * xv[1], u[2] * xv[0] - u[0] * xv[2], u[0] * xv[1] - u[1] * xv[0]};
  unit(yv);
  double zv[3] = {xv[1] * yv[2] - xv[2] * yv[1], xv[2] * yv[0] - xv[0] * yv[2], xv[0] * yv[1] - xv[1] * yv[0]};
  unit(zv);
  q[3] = static_cast<float>(sqrt(fmax(0.0, 1.0 + xv[0] + yv[1] + zv[2])) / 2.0);
  q[0] = static_cast<float>(sqrt(fmax(0.0, 1.0 + xv[0] - yv[1] - zv[2])) / 2.0);
  q[1] = static_cast<float>(sqrt(fmax(0.0, 1.0 - xv[0] + yv[1] - zv[2])) / 2.0);
  q[2] = static_cast<float>(sqrt(fmax(0.0, 1.0 - xv[0] - yv[1] + zv[2])) / 2.0);
  if (zv[1] - yv[2] > 0) q[0] = -q[0];
  if (xv[2] - zv[0] > 0) q[1] = -q[1];
  if (yv[0] - xv[1] > 0) q[2] = -q[2];
}

// State6DOF::covElement's differences against the expectation (state_6dof.h:162-184): position, then RPY wrapped to +-pi
__device__ __forceinline__ void pf_cov_diff(const PfState& s, const float e_pos[3], const float e_rpy[3], float d[6])
{
  float rpy[3];
  pf_rpy(s.rot, rpy);
  for (int a = 0; a < 3; ++a)
  {
    d[a] = fsub(s.pos[a], e_pos[a]);
    float diff = fsub(rpy[a], e_rpy[a]);
    while (static_cast<double>(diff) > M_PI) diff = __double2float_rn(dsub(static_cast<double>(diff), 2 * M_PI));
    while (static_cast<double>(diff) < -M_PI) diff = __double2float_rn(dadd(static_cast<double>(diff), 2 * M_PI));
    d[3 + a] = diff;
  }
}

}  // namespace mcl3dl
