// pf_events_oracle.cpp — TEST INFRASTRUCTURE ONLY ("port" checker of oracle/pf_events_api.h).
//
// Plain C++ restatements of three per-particle events of the node, given the normal draws:
//   the odometry-noise redraw (src/mcl_3dl.cpp:817-825), pf::ParticleFilter::addNoiseUsingNoiseGenerator with
//   State6DOF::generateNoise / operator+ (pf.h:226-237, state_6dof.h:226-261) and the IMU gravity update
//   (imu_measurement_model_gravity.h:45-55 inside pf.h:252-279).
// Every expression keeps the reference's types and operand order; the Makefile compiles without FMA contraction.
#include <cmath>
#include <vector>

#include "pf_events_api.h"

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
}  // namespace

extern "C" {

const char* mcl3dl_cpu_pf_events_kind(void) { return "port"; }

int mcl3dl_cpu_pf_redraw(mcl3dl_state* states, size_t n, const float* z, double lin_lin, double lin_ang, double ang_lin,
                         double ang_ang)
{
  if ((n && (!states || !z)))
    return MCL3DL_ERR_INVALID_ARG;
  for (size_t i = 0; i < n; ++i)
  {
    // float draw * double parameter, assigned to the float field
    states[i].noise_ll = static_cast<float>(z[4 * i + 0] * lin_lin);
    states[i].noise_la = static_cast<float>(z[4 * i + 1] * lin_ang);
    states[i].noise_aa = static_cast<float>(z[4 * i + 2] * ang_ang);
    states[i].noise_al = static_cast<float>(z[4 * i + 3] * ang_lin);
  }
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_noise(mcl3dl_state* states, size_t n, const float* org)
{
  if ((n && (!states || !org)))
    return MCL3DL_ERR_INVALID_ARG;
  for (size_t i = 0; i < n; ++i)
  {
    const float* o = org + 6 * i;
    mcl3dl_state& s = states[i];
    // Quat::setRPY, quat.h:202-215
    const float t2 = std::cos(o[3] / 2), t3 = std::sin(o[3] / 2);
    const float t4 = std::cos(o[4] / 2), t5 = std::sin(o[4] / 2);
    const float t0 = std::cos(o[5] / 2), t1 = std::sin(o[5] / 2);
    const Q nrot{t0 * t3 * t4 - t1 * t2 * t5, t0 * t2 * t5 + t1 * t3 * t4, t1 * t2 * t4 - t0 * t3 * t5, t0 * t2 * t4 + t1 * t3 * t5};
    // operator+: a fresh State6DOF (noise_* = 0), fields 0-2 and 7-12 summed, rot = noise.rot * rot; no normalize()
    for (int k = 0; k < 3; ++k)
    {
      s.pos[k] = s.pos[k] + o[k];
      s.odom_err_integ_lin[k] = s.odom_err_integ_lin[k] + o[k];
      s.odom_err_integ_ang[k] = s.odom_err_integ_ang[k] + (o[k + 3] - 0.0f);
    }
    const Q r = mul(nrot, Q{s.rot[0], s.rot[1], s.rot[2], s.rot[3]});
    s.rot[0] = r.x;
    s.rot[1] = r.y;
    s.rot[2] = r.z;
    s.rot[3] = r.w;
    s.noise_ll = s.noise_la = s.noise_al = s.noise_aa = 0.0f;
  }
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_imu(const mcl3dl_state* states, float* probs, size_t n, const float acc[3], double acc_var, float* lik,
                      int* kept, float* sum_out, float* entropy)
{
  if ((n && (!states || !probs)) || !acc || !kept || !sum_out || !entropy)
    return MCL3DL_ERR_INVALID_ARG;
  const float sigma = static_cast<float>(acc_var);
  const float a = 1.0 / std::sqrt(2.0 * M_PI * sigma * sigma);  // NormalLikelihood, nd.h:45-49
  const float sq2 = sigma * sigma * 2.0;
  const float acc_norm = std::sqrt(acc[0] * acc[0] + acc[1] * acc[1] + acc[2] * acc[2]);
  std::vector<float> post(probs, probs + n);
  float sum = 0;
  for (size_t i = 0; i < n; ++i)
  {
    const Q r{states[i].rot[0], states[i].rot[1], states[i].rot[2], states[i].rot[3]};
    // Quat::inv = conj() / dot(*this) = conj() * float(1.0 / dot)
    const float d = r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w;
    const float id = 1.0 / d;
    const Q inv{-r.x * id, -r.y * id, -r.z * id, r.w * id};
    // inv * Vec3(0, 0, 1) = inv * (0, 0, 1, 0) * conj(inv)
    const Q e = mul(mul(inv, Q{0.0f, 0.0f, 1.0f, 0.0f}), Q{-inv.x, -inv.y, -inv.z, inv.w});
    const float dot = e.x * acc[0] + e.y * acc[1] + e.z * acc[2];
    const float en = std::sqrt(e.x * e.x + e.y * e.y + e.z * e.z);
    const float diff = acosf(dot / (acc_norm * en));
    const float l = a * expf(-diff * diff / sq2);
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

}  // extern "C"
