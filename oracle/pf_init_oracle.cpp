// pf_init_oracle.cpp — TEST INFRASTRUCTURE ONLY ("port" checker of oracle/pf_init_api.h).
//
// A plain C++ restatement of the initial seed (include/mcl3dl_b200.h: mcl3dl_particles_init): setMean's getRPY, the two
// generators' rules on given standard normals and State6DOF::generateNoise.  Built with -ffp-contract=off, so every
// float operation rounds as written.
#include <cmath>

#include "pf_init_api.h"

namespace
{
// Quat::getRPY (quat.h:191-201): double expressions narrowed to float, float atan2 / asin
void rpyOf(float x, float y, float z, float w, float rpy[3])
{
  const float ysq = y * y;
  const float t0 = static_cast<float>(-2.0 * static_cast<double>(ysq + z * z) + 1.0);
  const float t1 = static_cast<float>(2.0 * static_cast<double>(x * y + w * z));
  double t2d = -2.0 * static_cast<double>(x * z - w * y);
  t2d = t2d > 1.0 ? 1.0 : t2d;
  t2d = t2d < -1.0 ? -1.0 : t2d;
  const float t2 = static_cast<float>(t2d);
  const float t3 = static_cast<float>(2.0 * static_cast<double>(y * z + w * x));
  const float t4 = static_cast<float>(-2.0 * static_cast<double>(x * x + ysq) + 1.0);
  rpy[0] = std::atan2(t3, t4);
  rpy[1] = std::asin(t2);
  rpy[2] = std::atan2(t1, t0);
}
}  // namespace

extern "C" {

const char* mcl3dl_cpu_pf_init_kind(void) { return "port"; }

int mcl3dl_cpu_pf_init_mean(const float pose7[7], float mean6[6])
{
  if (!pose7 || !mean6)
    return MCL3DL_ERR_INVALID_ARG;
  for (int k = 0; k < 3; ++k) mean6[k] = pose7[k];
  rpyOf(pose7[3], pose7[4], pose7[5], pose7[6], mean6 + 3);
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_init(size_t n, int multivariate, const float pose7[7], const float sigma6[6], const float T[36],
                       const float* z, mcl3dl_state* states, float* probs)
{
  if (!pose7 || (n && (!z || !states || !probs)) || (multivariate ? !T : !sigma6))
    return MCL3DL_ERR_INVALID_ARG;
  float mean[6];
  mcl3dl_cpu_pf_init_mean(pose7, mean);
  for (size_t i = 0; i < n; ++i)
  {
    const float* zi = z + 6 * i;
    float org[6];
    for (int r = 0; r < 6; ++r)
    {
      if (multivariate)
      {
        float t = T[r * 6] * zi[0];
        for (int k = 1; k < 6; ++k) t = t + T[r * 6 + k] * zi[k];
        org[r] = mean[r] + t;
      }
      else
        org[r] = sigma6[r] == 0 ? mean[r] : zi[r] * sigma6[r] + mean[r];
    }
    mcl3dl_state& s = states[i];
    s.noise_ll = s.noise_la = s.noise_al = s.noise_aa = 0.0f;
    for (int k = 0; k < 3; ++k)
    {
      s.pos[k] = org[k];
      s.odom_err_integ_lin[k] = org[k];
      s.odom_err_integ_ang[k] = org[k + 3] - mean[k + 3];
    }
    // Quat::setRPY (quat.h:202-215)
    const float t2 = std::cos(org[3] / 2), t3 = std::sin(org[3] / 2);
    const float t4 = std::cos(org[4] / 2), t5 = std::sin(org[4] / 2);
    const float t0 = std::cos(org[5] / 2), t1 = std::sin(org[5] / 2);
    s.rot[0] = t0 * t3 * t4 - t1 * t2 * t5;
    s.rot[1] = t0 * t2 * t5 + t1 * t3 * t4;
    s.rot[2] = t1 * t2 * t4 - t0 * t3 * t5;
    s.rot[3] = t0 * t2 * t4 + t1 * t3 * t5;
    probs[i] = static_cast<float>(1.0 / static_cast<double>(n));
  }
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_init_transform(const double*, float*) { return MCL3DL_ERR_INVALID_ARG; }

}  // extern "C"
