// gl_oracle.cpp — TEST INFRASTRUCTURE ONLY ("port" checker of global localisation and of the particle set's resize).
//
// The repo-owned restatement, written from the reference's documented behaviour and independent of the device code:
// a hash grid instead of the device's CSR window, std::lower_bound over the prefix sums instead of the device's search.
// Plain C++ arithmetic, compiled without FMA contraction, so every float operation rounds as in the reference build.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <unordered_map>
#include <vector>

#include "gl_api.h"

namespace
{
struct Quat
{
  float x, y, z, w;
};

// Quat::operator*(Quat), left to right as written there
Quat mul(const Quat& a, const Quat& b)
{
  return Quat{a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
              a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}

// Quat(Vec3(roll, pitch, yaw)) = setRPY, float cos / sin of the half angles
Quat from_rpy(float roll, float pitch, float yaw)
{
  const float cr = std::cos(roll / 2), sr = std::sin(roll / 2);
  const float cp = std::cos(pitch / 2), sp = std::sin(pitch / 2);
  const float cy = std::cos(yaw / 2), sy = std::sin(yaw / 2);
  return Quat{cy * sr * cp - sy * cr * sp, cy * cr * sp + sy * sr * cp, sy * cr * cp - cy * sr * sp, cy * cr * cp + sy * sr * sp};
}

// normalized(): multiply by float(1.0 / sqrtf(dot))
Quat normalized(const Quat& q)
{
  const float n = std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  const float s = static_cast<float>(1.0 / n);
  return Quat{q.x * s, q.y * s, q.z * s, q.w * s};
}

int64_t cell_key(int x, int y, int z)
{
  return (static_cast<int64_t>(x) + (1 << 20)) | ((static_cast<int64_t>(y) + (1 << 20)) << 21) | ((static_cast<int64_t>(z) + (1 << 20)) << 42);
}
}  // namespace

extern "C" {

const char* mcl3dl_cpu_gl_kind(void) { return "port"; }

int mcl3dl_cpu_gl_seed(const mcl3dl_point* ds, size_t n, double grid, int32_t div_yaw, const float imu_quat[4],
                       const float dist_weight[3], mcl3dl_state* states, float* probs, size_t cap, size_t* n_particles)
{
  if ((n && !ds) || !(grid > 0.0) || div_yaw < 1 || !imu_quat || !dist_weight || !n_particles)
    return MCL3DL_ERR_INVALID_ARG;
  // the rescaled cloud, bucketed by cells of edge 2 * grid (a point within grid of a query lies in its 27 cells)
  std::vector<float> v(n * 3);
  const double edge = 2.0 * grid;
  std::unordered_map<int64_t, std::vector<uint32_t>> cells;
  for (size_t i = 0; i < n; ++i)
  {
    v[i * 3 + 0] = ds[i].x * dist_weight[0];
    v[i * 3 + 1] = ds[i].y * dist_weight[1];
    v[i * 3 + 2] = ds[i].z * dist_weight[2];
    if (!std::isfinite(v[i * 3]) || !std::isfinite(v[i * 3 + 1]) || !std::isfinite(v[i * 3 + 2]))
      continue;  // no distance to it is below anything
    cells[cell_key(static_cast<int>(std::floor(v[i * 3] / edge)), static_cast<int>(std::floor(v[i * 3 + 1] / edge)),
                   static_cast<int>(std::floor(v[i * 3 + 2] / edge)))]
        .push_back(static_cast<uint32_t>(i));
  }
  const float r2 = static_cast<float>(grid * grid);
  std::vector<uint32_t> seeds;
  for (size_t i = 0; i < n; ++i)
  {
    float z = ds[i].z;
    z += 0.01 + grid;  // p2.z += 0.01 + grid: double addition, stored back in the float
    const float q[3] = {ds[i].x * dist_weight[0], ds[i].y * dist_weight[1], z * dist_weight[2]};
    bool found = false;
    if (std::isfinite(q[0]) && std::isfinite(q[1]) && std::isfinite(q[2]))
    {
      const int c[3] = {static_cast<int>(std::floor(q[0] / edge)), static_cast<int>(std::floor(q[1] / edge)),
                        static_cast<int>(std::floor(q[2] / edge))};
      for (int dz = -1; dz <= 1 && !found; ++dz)
        for (int dy = -1; dy <= 1 && !found; ++dy)
          for (int dx = -1; dx <= 1 && !found; ++dx)
          {
            const auto it = cells.find(cell_key(c[0] + dx, c[1] + dy, c[2] + dz));
            if (it == cells.end())
              continue;
            for (const uint32_t j : it->second)
            {
              float d = 0.0f;  // flann::L2_Simple: sequential sum of squared differences
              for (int k = 0; k < 3; ++k)
              {
                const float e = q[k] - v[j * 3 + k];
                d += e * e;
              }
              if (d < r2)
              {
                found = true;
                break;
              }
            }
          }
    }
    if (!found)
      seeds.push_back(static_cast<uint32_t>(i));
  }
  const size_t np = seeds.size() * static_cast<size_t>(div_yaw);
  *n_particles = np;
  if (!states && !probs)
    return MCL3DL_OK;
  if (cap < np)
    return MCL3DL_ERR_INVALID_ARG;
  const Quat imu{imu_quat[0], imu_quat[1], imu_quat[2], imu_quat[3]};
  std::vector<Quat> yaw(static_cast<size_t>(div_yaw));
  for (int32_t c = 0; c < div_yaw; ++c)
    yaw[c] = normalized(mul(from_rpy(0.0f, 0.0f, static_cast<float>(2.0 * M_PI * c / div_yaw)), imu));
  const float prob = static_cast<float>(1.0 / static_cast<float>(seeds.size()));
  for (size_t i = 0; i < np; ++i)
  {
    if (states)
    {
      const mcl3dl_point& p = ds[seeds[i / div_yaw]];
      const Quat& r = yaw[i % div_yaw];
      mcl3dl_state s;
      std::memset(&s, 0, sizeof(s));
      s.pos[0] = p.x;
      s.pos[1] = p.y;
      s.pos[2] = p.z;
      s.rot[0] = r.x;
      s.rot[1] = r.y;
      s.rot[2] = r.z;
      s.rot[3] = r.w;
      states[i] = s;
    }
    if (probs)
      probs[i] = prob;
  }
  return MCL3DL_OK;
}

int mcl3dl_cpu_pf_resize_6dof(const float* probs, const mcl3dl_state* states, size_t n, size_t num, mcl3dl_state* out_states,
                              float* out_probs)
{
  if (!probs || !states || n == 0 || num == 0 || !out_states || !out_probs)
    return MCL3DL_ERR_INVALID_ARG;
  std::vector<float> accum(n);
  float a = 0.0f;
  for (size_t i = 0; i < n; ++i)
  {
    a += probs[i];
    accum[i] = a;
  }
  const float pstep = a / num;  // float / size_t: num converted to float
  const float prob = static_cast<float>(1.0 / num);
  float pscan = 0.0f;
  size_t prev = 0;  // the last pick that was not past the end (particle 0 before any)
  for (size_t i = 0; i < num; ++i)
  {
    pscan += pstep;
    const size_t it = static_cast<size_t>(std::lower_bound(accum.begin(), accum.end(), pscan) - accum.begin());
    const size_t src = it < n ? it : prev;
    if (it < n)
      prev = it;
    out_states[i] = states[src];
    out_probs[i] = prob;
  }
  return MCL3DL_OK;
}

}  // extern "C"
