// pf_landmark_oracle.cpp — TEST INFRASTRUCTURE ONLY ("port" checker of oracle/pf_landmark_api.h).
//
// Plain C++ restatements of three events of the node:
//   cbLandmark's measure (src/mcl_3dl.cpp:899-931) with State6DOF::operator- (state_6dof.h:262-274), Quat::inv and
//   Quat::getRPY (quat.h:187-201) inside pf::ParticleFilter::measure (pf.h:252-279); the quadratic form in the order
//   include/mcl3dl_b200.h fixes;
//   the odometry-error reset (src/mcl_3dl.cpp:190-195,653-658);
//   publishParticles' normalised poses (src/mcl_3dl.cpp:1101-1125, Quat::normalized, quat.h:175-177).
// Every expression keeps the reference's types and operand order; the Makefile compiles without FMA contraction.
#include <algorithm>
#include <cmath>
#include <vector>

#include "pf_landmark_api.h"

namespace
{
struct Q
{
  float x, y, z, w;
};

// Quat::operator*(Quat), quat.h:131-138
Q mul(const Q& a, const Q& b)
{
  return Q{a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
           a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}

// Quat::operator/(float) = operator*(float(1.0 / s))
Q div(const Q& q, float s)
{
  const float f = 1.0 / s;
  return Q{q.x * f, q.y * f, q.z * f, q.w * f};
}

float dot(const Q& q) { return q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w; }
}  // namespace

extern "C" {

const char* mcl3dl_cpu_pf_landmark_kind(void) { return "port"; }

int mcl3dl_cpu_pf_landmark(const mcl3dl_state* states, float* probs, size_t n, const float measured[7], float nd_a,
                           const float sigma_inv[36], float* lik, int* kept, float* sum_out, float* entropy)
{
  if ((n && (!states || !probs)) || !measured || !sigma_inv || !kept || !sum_out || !entropy)
    return MCL3DL_ERR_INVALID_ARG;
  const Q m{measured[3], measured[4], measured[5], measured[6]};
  std::vector<float> post(probs, probs + n);
  float sum = 0;
  for (size_t i = 0; i < n; ++i)
  {
    const mcl3dl_state& s = states[i];
    // diff = s - measured: the position per axis, rot = measured.rot_.inv() * rot_ (inv = conj() / dot)
    const Q d = mul(div(Q{-m.x, -m.y, -m.z, m.w}, dot(m)), Q{s.rot[0], s.rot[1], s.rot[2], s.rot[3]});
    // Quat::getRPY: double expressions narrowed to float, float atan2 / asin
    const float ysq = d.y * d.y;
    const float t0 = -2.0 * (ysq + d.z * d.z) + 1.0;
    const float t1 = +2.0 * (d.x * d.y + d.w * d.z);
    const float t2 = std::max(-1.0, std::min(1.0, -2.0 * (d.x * d.z - d.w * d.y)));
    const float t3 = +2.0 * (d.y * d.z + d.w * d.x);
    const float t4 = -2.0 * (d.x * d.x + ysq) + 1.0;
    const float x[6] = {s.pos[0] - measured[0], s.pos[1] - measured[1], s.pos[2] - measured[2],
                        std::atan2(t3, t4), std::asin(t2), std::atan2(t1, t0)};
    // -0.5 x^T S x: h = -0.5 x, r_j = sum_k h_k S(k, j), q = sum_j r_j x_j, left to right in float
    float h[6];
    for (int k = 0; k < 6; ++k) h[k] = -0.5f * x[k];
    float q = 0;
    for (int j = 0; j < 6; ++j)
    {
      float r = h[0] * sigma_inv[j];
      for (int k = 1; k < 6; ++k) r = r + h[k] * sigma_inv[k * 6 + j];
      q = j == 0 ? r * x[0] : q + r * x[j];
    }
    const float l = nd_a * std::exp(q);
    if (lik)
      lik[i] = l;
    post[i] *= l;
    sum += post[i];
  }
  *sum_out = sum;
  *kept = sum > 0.0 ? 1 : 0;
  *entropy = 0;
  if (!*kept)
    return MCL3DL_OK;
  float ent = 0;
  for (size_t i = 0; i < n; ++i)
  {
    probs[i] = post[i] / sum;
    if (probs[i] > 0)
      ent += probs[i] * std::log(probs[i]);
  }
  *entropy = ent * -1;
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_reset_odom_err(mcl3dl_state* states, size_t n)
{
  if (n && !states)
    return MCL3DL_ERR_INVALID_ARG;
  for (size_t i = 0; i < n; ++i)
    for (int k = 0; k < 3; ++k)
    {
      states[i].odom_err_integ_lin[k] = 0.0f;
      states[i].odom_err_integ_ang[k] = 0.0f;
    }
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_poses(const mcl3dl_state* states, size_t n, mcl3dl_pose* out)
{
  if (n && (!states || !out))
    return MCL3DL_ERR_INVALID_ARG;
  for (size_t i = 0; i < n; ++i)
  {
    const mcl3dl_state& s = states[i];
    const Q r{s.rot[0], s.rot[1], s.rot[2], s.rot[3]};
    const Q q = div(r, std::sqrt(dot(r)));  // normalized() = *this / norm(), norm = sqrtf(dot)
    out[i] = mcl3dl_pose{s.pos[0], s.pos[1], s.pos[2], 0.0f, q.x, q.y, q.z, q.w};
  }
  return MCL3DL_OK;
}

}  // extern "C"
