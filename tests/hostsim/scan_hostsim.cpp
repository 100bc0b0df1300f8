// scan_hostsim.cpp — TEST INFRASTRUCTURE ONLY.
//
// Host drivers for mcl_3dl_b200/csrc/scan_funcs.cuh (scan preprocessing: VoxelGrid lattice and key, the voxel's centroid
// and label vote, the clip, the sampler's index), compiled for the host through cuda_shim.h.  The serial loops below
// stand in for the kernels' sorts, scans and compactions of scan_kernels.cuh; tests/test_gpu_scan_exact.py compares
// them with its numpy restatement, so that a device mismatch can only come from the kernels or their plumbing.
#include "cuda_shim.h"

#include <algorithm>
#include <numeric>
#include <vector>

#include "../../include/mcl3dl_b200.h"
#include "../../mcl_3dl_b200/csrc/scan_funcs.cuh"

using namespace mcl3dl;

// scan_voxel_lattice: 1 = downsample with this lattice, 0 = the cloud passes unfiltered
extern "C" int hostsim_scan_lattice(const float leaf[3], const float mn[3], const float mx[3], float inv_leaf[3], int min_b[3],
                                    uint32_t div_b[3], uint32_t* cells, int* end_bit)
{
  VoxelGridDev g{};
  int eb = 0;
  if (!scan_voxel_lattice(leaf, mn, mx, g, eb))
    return 0;
  for (int k = 0; k < 3; ++k)
  {
    inv_leaf[k] = g.inv_leaf[k];
    min_b[k] = g.min_b[k];
    div_b[k] = g.div_b[k];
  }
  *cells = g.cells;
  *end_bit = eb;
  return 1;
}

// The VoxelGrid stage of mcl3dl_scan_prepare: the finite points' bounding box, the lattice, stable sort by voxel key,
// sort of the (voxel, label) keys, one scan_voxel_point per voxel.  Returns the number of output points, or -1 when the
// cloud passes unfiltered.
extern "C" long hostsim_scan_voxel_grid(const mcl3dl_point* pts, size_t n, const float leaf[3], mcl3dl_point* out)
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
  if (!(mn[0] <= mx[0]))
    return 0;
  VoxelGridDev g{};
  int end_bit = 0;
  if (!scan_voxel_lattice(leaf, mn, mx, g, end_bit))
    return -1;
  std::vector<uint32_t> key(n), order(n);
  std::vector<uint64_t> key_label(n);
  for (size_t i = 0; i < n; ++i)
  {
    key[i] = voxel_key(g, pts[i]);
    key_label[i] = voxel_key_label(key[i], pts[i].label);
  }
  std::iota(order.begin(), order.end(), 0u);
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
  std::sort(key_label.begin(), key_label.end());
  long m = 0;
  for (size_t i = 0; i < n;)
  {
    const uint32_t k = key[order[i]];
    size_t cnt = 1;
    while (i + cnt < n && key[order[i + cnt]] == k) ++cnt;
    if (k != g.cells)
      out[m++] = scan_voxel_point(pts, order.data() + i, key_label.data() + i, static_cast<uint32_t>(cnt));
    i += cnt;
  }
  return m;
}

// one voxel's point straight from its parts (order / key_label as scan_voxel_point takes them)
extern "C" void hostsim_scan_voxel_point(const mcl3dl_point* pts, const uint32_t* order, const uint64_t* key_label, uint32_t cnt,
                                         mcl3dl_point* out)
{
  *out = scan_voxel_point(pts, order, key_label, cnt);
}

// the models' filter() with scan_clip_window / clip_removes: keep[i] = 1 where the point stays
extern "C" void hostsim_scan_clip(const mcl3dl_point* pts, size_t n, float near, float far, float z_min, float z_max, uint8_t* keep)
{
  const ClipDev c = scan_clip_window(near, far, z_min, z_max);
  for (size_t i = 0; i < n; ++i) keep[i] = clip_removes(c, pts[i]) ? 0 : 1;
}

// the sampler's indices of draws 0..num-1 over n clipped points
extern "C" void hostsim_scan_sample(uint64_t seed, uint32_t stream, uint32_t num, uint32_t n, uint32_t* idx)
{
  for (uint32_t t = 0; t < num; ++t) idx[t] = scan_sample_index(seed, stream, t, n);
}
