// window_hostsim.cpp — TEST INFRASTRUCTURE ONLY.
//
// Host driver for mcl_3dl_b200/csrc/window_funcs.cuh (the map window's arithmetic), compiled for the host through
// cuda_shim.h.  hostsim_win_need restates window_need_kernel serially; tests/test_map_window_on_host.py compares the
// required box, the growth, the clamp and the containment test with a Python restatement, and checks with the kernels'
// own float transform (device_math.cuh) that every query +/- its radius lies inside the required box.
#include "cuda_shim.h"

#include "../../include/mcl3dl_b200.h"
#include "../../mcl_3dl_b200/csrc/device_math.cuh"
#include "../../mcl_3dl_b200/csrc/window_funcs.cuh"

using namespace mcl3dl;

namespace
{
uint32_t ord(float f)
{
  uint32_t b;
  std::memcpy(&b, &f, 4);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
uint32_t bits(float f)
{
  uint32_t b;
  std::memcpy(&b, &f, 4);
  return b;
}
}  // namespace

// window_need_kernel, one item at a time (double arithmetic rounded up as the kernel's __double2float_ru / __dsqrt_ru)
extern "C" void hostsim_win_need(const mcl3dl_pose* poses, size_t P, const mcl3dl_point* pts, size_t n, const float* org, size_t norg,
                                 uint32_t out[8])
{
  uint32_t w[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (size_t i = 0; i < P; ++i)
  {
    const mcl3dl_pose& p = poses[i];
    const float c[7] = {p.px, p.py, p.pz, p.qx, p.qy, p.qz, p.qw};
    bool fin = true;
    for (float v : c) fin = fin && std::isfinite(v);
    if (!fin)
      continue;
    for (int k = 0; k < 3; ++k)
    {
      w[k] = std::max(w[k], ~ord(c[k]));
      w[3 + k] = std::max(w[3 + k], ord(c[k]));
    }
    const double q2 = static_cast<double>(p.qx) * p.qx + static_cast<double>(p.qy) * p.qy + static_cast<double>(p.qz) * p.qz +
                      static_cast<double>(p.qw) * p.qw;
    float s = static_cast<float>(std::max(q2, 1.0));
    if (static_cast<double>(s) < std::max(q2, 1.0))
      s = std::nextafter(s, INFINITY);
    w[7] = std::max(w[7], bits(s));
  }
  auto norm = [&](float x, float y, float z) {
    if (!std::isfinite(x) || !std::isfinite(y) || !std::isfinite(z))
      return;
    const double n2 = static_cast<double>(x) * x + static_cast<double>(y) * y + static_cast<double>(z) * z;
    double r = std::sqrt(n2);
    if (r * r < n2)
      r = std::nextafter(r, INFINITY);
    r *= 1.0 + 0x1p-40;
    float f = static_cast<float>(r);
    if (static_cast<double>(f) < r)
      f = std::nextafter(f, INFINITY);
    w[6] = std::max(w[6], bits(f));
  };
  for (size_t i = 0; i < n; ++i) norm(pts[i].x, pts[i].y, pts[i].z);
  for (size_t i = 0; i < norg; ++i) norm(org[3 * i], org[3 * i + 1], org[3 * i + 2]);
  std::memcpy(out, w, sizeof(w));
}

// win_required; returns 0 when the box is not finite
extern "C" int hostsim_win_required(const uint32_t need[8], float r_scaled, float grid_min, float hit_tolerance, const float w[3],
                                    float box[6])
{
  WinNeed n;
  std::memcpy(&n, need, sizeof(n));
  WinBox b;
  if (!win_required(n, WinSearch{r_scaled, grid_min, hit_tolerance}, w, b))
    return 0;
  std::memcpy(box, &b, sizeof(b));
  return 1;
}

extern "C" double hostsim_win_reach(const uint32_t need[8])
{
  WinNeed n;
  std::memcpy(&n, need, sizeof(n));
  return win_reach(n);
}

// win_choose; returns 0 when the required box alone exceeds the cap
extern "C" int hostsim_win_choose(const float req[6], double reach, const float w[3], float cell, uint64_t cap, float out[6])
{
  WinBox r, o;
  std::memcpy(&r, req, sizeof(r));
  if (!win_choose(r, reach, w, cell, cap, o))
    return 0;
  std::memcpy(out, &o, sizeof(o));
  return 1;
}

// win_box_lattice: cells (0 when refused), dims and origin
extern "C" uint64_t hostsim_win_lattice(const float box[6], const float w[3], float cell, int32_t dims[3], float org[3])
{
  WinBox b;
  std::memcpy(&b, box, sizeof(b));
  size_t cells = 0;
  int d[3];
  if (!win_box_lattice(b, w, cell, d, org, cells))
    return 0;
  for (int k = 0; k < 3; ++k) dims[k] = d[k];
  return cells;
}

extern "C" int hostsim_win_contains(const float outer[6], const float inner[6])
{
  WinBox a, b;
  std::memcpy(&a, outer, sizeof(a));
  std::memcpy(&b, inner, sizeof(b));
  return win_contains(a, b) ? 1 : 0;
}

// The kernels' transforms of scan point p by pose q: the likelihood / match transform (normalised rotation) and the beam
// origin (raw rotation), out[0..2] and out[3..5]
extern "C" void hostsim_win_transform(const mcl3dl_pose* pose, const float p[3], float out[6])
{
  const Q4 q{pose->qx, pose->qy, pose->qz, pose->qw};
  const F3 t = transform_point(qnormalized(q), F3{pose->px, pose->py, pose->pz}, F3{p[0], p[1], p[2]});
  const F3 r = qrot(q, F3{p[0], p[1], p[2]});
  out[0] = t.x;
  out[1] = t.y;
  out[2] = t.z;
  out[3] = __fadd_rn(pose->px, r.x);
  out[4] = __fadd_rn(pose->py, r.y);
  out[5] = __fadd_rn(pose->pz, r.z);
}
