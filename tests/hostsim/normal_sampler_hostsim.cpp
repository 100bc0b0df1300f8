// normal_sampler_hostsim.cpp — TEST INFRASTRUCTURE ONLY.
//
// Host drivers for the normal-weighted sampler's pieces of mcl_3dl_b200/csrc/scan_funcs.cuh (ns_*), compiled for the host
// through cuda_shim.h.  The serial loops below stand in for the kernels of scan_kernels.cuh (the stable key sort, the
// per-point normal and weight, the draws); tests/test_normal_sampler_on_host.py holds them to the port checker and
// tests/test_gpu_normal_sampler.py holds the device to them bit for bit.
#include "cuda_shim.h"

#include <algorithm>
#include <numeric>
#include <vector>

#include "../../include/mcl3dl_b200.h"
#include "../../mcl_3dl_b200/csrc/scan_funcs.cuh"

using namespace mcl3dl;

// ns_host_consts: max_weight, fpc_local and F
extern "C" void hostsim_ns_consts(const mcl3dl_normal_sampler_params* p, double* max_weight, float fpc_local[3], int* shift)
{
  ns_host_consts(*p, max_weight, fpc_local, shift);
}

// ns_lattice: 1 = a grid with this edge and lattice, 0 = TOO_LARGE
extern "C" int hostsim_ns_lattice(double r, const float mn[3], const float mx[3], float* edge, float inv_leaf[3], int min_b[3],
                                  uint32_t div_b[3], uint32_t* cells)
{
  VoxelGridDev g{};
  int end_bit = 0;
  if (!ns_lattice(r, mn, mx, g, end_bit, *edge))
    return 0;
  for (int k = 0; k < 3; ++k)
  {
    inv_leaf[k] = g.inv_leaf[k];
    min_b[k] = g.min_b[k];
    div_b[k] = g.div_b[k];
  }
  *cells = g.cells;
  return 1;
}

// One clipped cloud as mcl3dl_scan_sample_with_normal treats it: the finite points' bounding box, ns_lattice, the stable
// key sort, then per point ns_point_normal, ns_weight and ns_weight_q.  Returns 0, or -5 (TOO_LARGE).
extern "C" int hostsim_ns_normals(const mcl3dl_point* pts, size_t n, double r, const float fpc[3], double max_weight, double scale,
                                  float* normals, uint32_t* n_nb, uint64_t* q)
{
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (size_t i = 0; i < n; ++i)
  {
    if (!point_finite(pts[i]))
      continue;
    const float v[3] = {pts[i].x, pts[i].y, pts[i].z};
    for (int k = 0; k < 3; ++k)
    {
      mn[k] = std::min(mn[k], v[k]);
      mx[k] = std::max(mx[k], v[k]);
    }
  }
  NsGridDev ng{};
  ng.r2 = static_cast<float>(r * r);
  int end_bit = 1;
  float edge = 0.0f;
  if (n && mn[0] <= mx[0] && !ns_lattice(r, mn, mx, ng.g, end_bit, edge))
    return MCL3DL_ERR_TOO_LARGE;
  std::vector<uint32_t> key(n), order(n), skeys(n);
  std::vector<mcl3dl_point> spts(n);
  for (size_t i = 0; i < n; ++i) key[i] = voxel_key(ng.g, pts[i]);
  std::iota(order.begin(), order.end(), 0u);
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
  for (size_t s = 0; s < n; ++s)
  {
    skeys[s] = key[order[s]];
    spts[s] = pts[order[s]];
  }
  for (size_t i = 0; i < n; ++i)
  {
    float nrm[3];
    n_nb[i] = ns_point_normal(ng, skeys.data(), spts.data(), static_cast<uint32_t>(n), pts[i], nrm);
    normals[3 * i + 0] = nrm[0];
    normals[3 * i + 1] = nrm[1];
    normals[3 * i + 2] = nrm[2];
    q[i] = ns_weight_q(ns_weight(nrm, fpc, max_weight), scale);
  }
  return 0;
}

// ns_weight of given normals (no rounding to q)
extern "C" void hostsim_ns_weights(const float* normals, size_t n, const float fpc[3], double max_weight, double* w)
{
  for (size_t i = 0; i < n; ++i) w[i] = ns_weight(normals + 3 * i, fpc, max_weight);
}

// ns_acos01 of given arguments
extern "C" void hostsim_ns_acos(const double* a, size_t n, double* out)
{
  for (size_t i = 0; i < n; ++i) out[i] = ns_acos01(a[i]);
}

// the indices of draws t0 .. t0 + cnt - 1 of stream over the inclusive sum cum[0..n)
extern "C" void hostsim_ns_draws(const uint64_t* cum, uint32_t n, uint64_t seed, uint32_t stream, uint64_t t0, uint32_t cnt, uint32_t* idx)
{
  for (uint32_t k = 0; k < cnt; ++k) idx[k] = ns_draw_index(cum, n, ns_draw_value(seed, stream, t0 + k, cum[n - 1]));
}
