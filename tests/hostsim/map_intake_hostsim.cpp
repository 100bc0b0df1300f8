// map_intake_hostsim.cpp — TEST INFRASTRUCTURE ONLY.
//
// Host drivers for the map intake's per-point pieces in mcl_3dl_b200/csrc/accum_funcs.cuh (map_read: fromROSMsg into
// PointXYZIL; map_voxel_intensity: a voxel's intensity) with scan_funcs.cuh's VoxelGrid pieces, compiled for the host
// through cuda_shim.h.  The serial loops below stand in for map_read_kernel, voxel_grid()'s sorts and scans,
// map_intensity_kernel and the finite compaction of scan_kernels.cuh; tests/test_map_intake_on_host.py holds them bit for
// bit to tests/map_intake_restate.py.
#include "cuda_shim.h"

#include <algorithm>
#include <numeric>
#include <vector>

#include "../../include/mcl3dl_b200.h"
#include "../../mcl_3dl_b200/csrc/accum_funcs.cuh"

using namespace mcl3dl;

// map_read_kernel's body, point after point
extern "C" void hostsim_map_read(const unsigned char* data, uint32_t width, uint32_t height, uint32_t row_step, uint32_t point_step,
                                 const uint32_t off[3], int32_t io, int32_t lo, mcl3dl_point* out, float* inten)
{
  const uint32_t n = width * height;
  for (uint32_t i = 0; i < n; ++i)
    out[i] = map_read(data, i / width, i % width, row_step, point_step, off[0], off[1], off[2], io, lo, inten[i]);
}

// The intake after the conversion: VoxelGrid with the intensity centroid (leaf all > 0 and PCL's rule passes), else the
// finite points in order.  Returns the output count; *downsampled as mcl3dl_map_intake_info reports it.
extern "C" long hostsim_map_intake(const mcl3dl_point* pts, const float* inten, size_t n, const float leaf[3], mcl3dl_point* out,
                                   float* out_int, int* downsampled)
{
  *downsampled = 0;
  if (leaf[0] > 0.0f && leaf[1] > 0.0f && leaf[2] > 0.0f)
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
    {
      *downsampled = 1;
      return 0;
    }
    VoxelGridDev g{};
    int end_bit = 0;
    if (scan_voxel_lattice(leaf, mn, mx, g, end_bit))
    {
      *downsampled = 1;
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
        if (point_finite(pts[order[i]]))
        {
          out[m] = scan_voxel_point(pts, order.data() + i, key_label.data() + i, static_cast<uint32_t>(cnt));
          out_int[m++] = map_voxel_intensity(inten, order.data() + i, static_cast<uint32_t>(cnt));
        }
        i += cnt;
      }
      return m;
    }
  }
  long m = 0;
  for (size_t i = 0; i < n; ++i)
    if (point_finite(pts[i]))
    {
      out[m] = pts[i];
      out_int[m++] = inten[i];
    }
  return m;
}
