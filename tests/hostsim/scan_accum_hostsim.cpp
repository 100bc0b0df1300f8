// scan_accum_hostsim.cpp — TEST INFRASTRUCTURE ONLY.
//
// Host drivers for mcl_3dl_b200/csrc/accum_funcs.cuh (cloud accumulation: the strided FLOAT32 read of a PointCloud2, the
// transform built from a double translation and a raw double quaternion, the second transform's not-dense rule),
// compiled for the host through cuda_shim.h.  The loops below are the bodies of accum_cloud_kernel and
// accum_transform_kernel (scan_kernels.cuh) run one point after another; tests/test_scan_accum_on_host.py holds them bit
// for bit to its numpy float32 restatement.
#include "cuda_shim.h"

#include "../../include/mcl3dl_b200.h"
#include "../../mcl_3dl_b200/csrc/accum_funcs.cuh"

using namespace mcl3dl;

extern "C" void hostsim_accum_xform(const double t[3], const double q[4], float r[9], float tt[3])
{
  const AccumXform m = accum_xform(t[0], t[1], t[2], q[0], q[1], q[2], q[3]);
  for (int k = 0; k < 9; ++k) r[k] = m.r[k];
  for (int k = 0; k < 3; ++k) tt[k] = m.t[k];
}

// the raw x / y / z of every point, row-major
extern "C" void hostsim_accum_read(const unsigned char* data, uint32_t width, uint32_t height, uint32_t row_step, uint32_t point_step,
                                   const uint32_t off[3], float* xyz)
{
  const uint32_t n = width * height;
  for (uint32_t i = 0; i < n; ++i)
  {
    const F3 p = accum_read(data, i / width, i % width, row_step, point_step, off[0], off[1], off[2]);
    xyz[3 * i] = p.x;
    xyz[3 * i + 1] = p.y;
    xyz[3 * i + 2] = p.z;
  }
}

// accum_cloud_kernel's body
extern "C" void hostsim_accum_cloud(const unsigned char* data, uint32_t width, uint32_t height, uint32_t row_step, uint32_t point_step,
                                    const uint32_t off[3], const double t[3], const double q[4], uint32_t label, mcl3dl_point* out)
{
  const uint32_t n = width * height;
  for (uint32_t i = 0; i < n; ++i)
  {
    const AccumXform m = accum_xform(t[0], t[1], t[2], q[0], q[1], q[2], q[3]);
    const F3 p = accum_apply(m, accum_read(data, i / width, i % width, row_step, point_step, off[0], off[1], off[2]));
    out[i] = mcl3dl_point{p.x, p.y, p.z, label};
  }
}

// accum_transform_kernel's body
extern "C" void hostsim_accum_second(const mcl3dl_point* in, size_t n, const double t[3], const double q[4], int dense, mcl3dl_point* out)
{
  for (size_t i = 0; i < n; ++i)
  {
    const AccumXform m = accum_xform(t[0], t[1], t[2], q[0], q[1], q[2], q[3]);
    const F3 p = accum_second(m, dense != 0, F3{in[i].x, in[i].y, in[i].z});
    out[i] = mcl3dl_point{p.x, p.y, p.z, in[i].label};
  }
}
