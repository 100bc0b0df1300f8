// window_funcs.cuh — the arithmetic of the map window: the box of raw map space that holds every search of one call, the
// window a rebuild stages around it, and the lattice rule both are measured with.  Also compiled for the host by
// tests/hostsim (window_hostsim.cpp) and checked there against a Python restatement (tests/test_map_window_on_host.py).
//
// A map whose whole likelihood lattice is refused (2^31 cells or more, or above MCL3DL_MAP_MAX_CELLS) is staged
// windowed: its points stay on the device and the search structures are built over the points inside a window, a box
// around the particles.  Every search returns the exact nearest neighbour within its radius (lowest index on ties), so
// restricting the map to a box that holds each query +/- its radius changes no record.
//
// Every map-reading call reduces its inputs on the device (window_need_kernel) to a WinNeed: the box of the finite
// particle positions, the largest |q|^2 of a finite particle's quaternion (qrot with a raw quaternion scales by |q|^2,
// with a normalised one by ~1) and the largest norm of a finite scan point or origin.  The host turns it into the
// required box (win_required): the particle box grown by the scan reach, the searches' radius per axis in raw
// coordinates, the KD march's overshoot and a relative pad for the float transform R p + t.
#pragma once
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define MCL3DL_WIN_HD __host__ __device__
#else
#define MCL3DL_WIN_HD
#endif

namespace mcl3dl
{
// The reduction's 32 bytes.  A zeroed block is the identity: the minimum is kept complemented, the maximum in f2ord's
// encoding (never 0 for a float), the norm and the scale as the bits of non-negative floats.
struct WinNeed
{
  uint32_t pmin_c[3];  // ~f2ord(min particle position); all zero: no finite particle
  uint32_t pmax[3];    // f2ord(max particle position)
  uint32_t reach;      // bits of the largest norm of a finite scan point or origin
  uint32_t scale;      // bits of max(1, largest |q|^2) over the finite particles (rounded up)
};

// What one call searches: the largest padded radius in the rescaled space (likelihood rpad, the KD caster's r2_pad, the
// match output's rpad) and, for the KD caster, its marching step and hit tolerance (0 without a march).
struct WinSearch
{
  float r_scaled;
  float grid_min;
  float hit_tolerance;
};

struct WinBox
{
  float lo[3], hi[3];
};

inline float win_ord2f(uint32_t o)
{
  const uint32_t b = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
  float f;
  std::memcpy(&f, &b, 4);
  return f;
}

inline float win_bits2f(uint32_t b)
{
  float f;
  std::memcpy(&f, &b, 4);
  return f;
}

// Lattice of a likelihood-style search grid with edge `cell` over the rescaled box [sc_min, sc_max]: origin half a cell
// below the minimum, one spare cell above.  false: 2^31 cells or more (or a box that is not finite).
inline bool win_lattice(float cell, const float sc_min[3], const float sc_max[3], int dims[3], float org[3], size_t& cells)
{
  int64_t total = 1;
  for (int k = 0; k < 3; ++k)
  {
    if (!std::isfinite(sc_min[k]) || !std::isfinite(sc_max[k]) || !(sc_max[k] >= sc_min[k]))
      return false;
    org[k] = sc_min[k] - 0.5f * cell;
    const double d = std::floor((static_cast<double>(sc_max[k]) - org[k]) / cell) + 2.0;
    if (!(d < 2147483648.0))
      return false;
    dims[k] = static_cast<int>(d);
    total *= dims[k];
    if (total >= (int64_t(1) << 31))
      return false;
  }
  cells = static_cast<size_t>(total);
  return true;
}

// The lattice of a raw box: its corners rescaled with the float multiply of the grids (monotonic for w > 0)
inline bool win_box_lattice(const WinBox& b, const float w[3], float cell, int dims[3], float org[3], size_t& cells)
{
  float sc_min[3], sc_max[3];
  for (int k = 0; k < 3; ++k)
  {
    sc_min[k] = b.lo[k] * w[k];
    sc_max[k] = b.hi[k] * w[k];
  }
  return win_lattice(cell, sc_min, sc_max, dims, org, cells);
}

// A search of radius r in the rescaled space, along axis k in raw coordinates: r / w, rounded up
inline double win_raw_radius(float r_scaled, float w)
{
  return static_cast<double>(r_scaled) / static_cast<double>(w) * (1.0 + 0x1p-20);
}

inline bool win_has_particles(const WinNeed& n)
{
  return n.pmax[0] != 0u;
}

// The scan reach of a call: the largest distance of a transformed scan point or origin from its particle
inline double win_reach(const WinNeed& n)
{
  return static_cast<double>(win_bits2f(n.reach)) * static_cast<double>(win_bits2f(n.scale)) * (1.0 + 0x1p-20);
}

// The required box: every query of the call +/- its radius.  A KD march runs from the ray's begin up to hit_tolerance
// past its end, and the second search sits two steps behind the marching position, so up to one step before the begin;
// the float accumulation of the march drifts by at most an ulp of the coordinates per step.  The pad covers the
// rounding of R p + t and of the rescaling.  false: the box is not finite.
inline bool win_required(const WinNeed& n, const WinSearch& s, const float w[3], WinBox& out)
{
  double pmin[3], pmax[3];
  for (int k = 0; k < 3; ++k)
  {
    pmin[k] = win_ord2f(~n.pmin_c[k]);
    pmax[k] = win_ord2f(n.pmax[k]);
  }
  const double reach = win_reach(n);
  double extra = 0.0, steps = 0.0;
  if (s.grid_min > 0.0f)
  {
    extra = std::max(static_cast<double>(s.hit_tolerance), static_cast<double>(s.grid_min)) * (1.0 + 0x1p-10);
    steps = std::ceil((2.0 * reach + s.hit_tolerance) / s.grid_min) + 2.0;
  }
  for (int k = 0; k < 3; ++k)
  {
    const double r = win_raw_radius(s.r_scaled, w[k]);
    const double mag = std::max(std::fabs(pmin[k]), std::fabs(pmax[k])) + reach + extra + r;
    const double half = reach + extra + r + mag * (0x1p-16 + steps * 0x1p-21);
    const double lo = pmin[k] - half, hi = pmax[k] + half;
    if (!std::isfinite(lo) || !std::isfinite(hi) || std::fabs(lo) > 1e30 || std::fabs(hi) > 1e30)
      return false;
    // outward to float
    float flo = static_cast<float>(lo), fhi = static_cast<float>(hi);
    if (static_cast<double>(flo) > lo)
      flo = std::nextafter(flo, -INFINITY);
    if (static_cast<double>(fhi) < hi)
      fhi = std::nextafter(fhi, INFINITY);
    out.lo[k] = flo;
    out.hi[k] = fhi;
  }
  return true;
}

inline bool win_contains(const WinBox& outer, const WinBox& inner)
{
  for (int k = 0; k < 3; ++k)
    if (!(outer.lo[k] <= inner.lo[k] && inner.hi[k] <= outer.hi[k]))
      return false;
  return true;
}

MCL3DL_WIN_HD inline bool win_point_inside(const WinBox& b, float x, float y, float z)
{
  return x >= b.lo[0] && x <= b.hi[0] && y >= b.lo[1] && y <= b.hi[1] && z >= b.lo[2] && z <= b.hi[2];
}

// The box `req` grown by `grow` on each side (outward in float)
inline WinBox win_grown(const WinBox& req, double grow)
{
  WinBox b;
  for (int k = 0; k < 3; ++k)
  {
    float lo = static_cast<float>(static_cast<double>(req.lo[k]) - grow);
    float hi = static_cast<float>(static_cast<double>(req.hi[k]) + grow);
    b.lo[k] = std::min(lo, req.lo[k]);
    b.hi[k] = std::max(hi, req.hi[k]);
  }
  return b;
}

// The window of a rebuild: the required box grown by the scan reach on each side, so the particles can travel one sensor
// range before the next rebuild; when that lattice exceeds `cap` cells the growth is halved (down to none) until it fits.
// false: the required box alone exceeds the cap.
inline bool win_choose(const WinBox& req, double reach, const float w[3], float cell, size_t cap, WinBox& out)
{
  int dims[3];
  float org[3];
  size_t cells = 0;
  double g = reach;
  for (int i = 0; i < 8; ++i, g *= 0.5)
  {
    const WinBox b = win_grown(req, g);
    if (win_box_lattice(b, w, cell, dims, org, cells) && cells <= cap)
    {
      out = b;
      return true;
    }
  }
  if (win_box_lattice(req, w, cell, dims, org, cells) && cells <= cap)
  {
    out = req;
    return true;
  }
  return false;
}

}  // namespace mcl3dl
