// accum_funcs.cuh — per-point pieces of the node's cloud accumulation (src/mcl_3dl.cpp:274-342; mcl3dl_scan_accumulate,
// mcl3dl_scan_prepare_accumulated): the strided read of a PointCloud2's FLOAT32 x / y / z, the rigid transform built from
// a double translation and a raw double quaternion, and the second transform's rule for clouds that are not dense.
// Every operation is rounded on its own (device_math.cuh), so that tests/hostsim/scan_accum_hostsim.cpp can compile these
// very functions for the host and hold them bit for bit to a numpy float32 restatement.
//
// The arithmetic restates Eigen's and PCL's (third-party, absent from the reference tree; "parity unpinned", see
// include/mcl3dl_b200.h):
//   R = Eigen::Quaternion<float>(float(w), float(x), float(y), float(z)).toRotationMatrix(), no normalisation:
//       tx = 2x, ty = 2y, tz = 2z, twx = tx w, twy = ty w, twz = tz w, txx = tx x, txy = ty x, txz = tz x, tyy = ty y,
//       tyz = tz y, tzz = tz z; R00 = 1 - (tyy + tzz), R01 = txy - twz, R02 = txz + twy, R10 = txy + twz,
//       R11 = 1 - (txx + tzz), R12 = tyz - twx, R20 = txz - twy, R21 = tyz + twx, R22 = 1 - (txx + tyy);
//   t = float(translation);
//   out_i = ((R_i0 x + R_i1 y) + R_i2 z) + t_i.
#pragma once
#include <stdint.h>

#include "device_math.cuh"
#include "scan_funcs.cuh"

namespace mcl3dl
{
struct AccumXform
{
  float r[9];  // row-major
  float t[3];
};

// tf2::doTransform (sensor -> odom) and measure()'s Eigen::Affine3f (odom -> base_link): the same construction
__device__ __forceinline__ AccumXform accum_xform(double tx_, double ty_, double tz_, double qx_, double qy_, double qz_, double qw_)
{
  const float x = __double2float_rn(qx_), y = __double2float_rn(qy_), z = __double2float_rn(qz_), w = __double2float_rn(qw_);
  const float tx = fmul(2.0f, x), ty = fmul(2.0f, y), tz = fmul(2.0f, z);
  const float twx = fmul(tx, w), twy = fmul(ty, w), twz = fmul(tz, w);
  const float txx = fmul(tx, x), txy = fmul(ty, x), txz = fmul(tz, x);
  const float tyy = fmul(ty, y), tyz = fmul(tz, y), tzz = fmul(tz, z);
  AccumXform m;
  m.r[0] = fsub(1.0f, fadd(tyy, tzz));
  m.r[1] = fsub(txy, twz);
  m.r[2] = fadd(txz, twy);
  m.r[3] = fadd(txy, twz);
  m.r[4] = fsub(1.0f, fadd(txx, tzz));
  m.r[5] = fsub(tyz, twx);
  m.r[6] = fsub(txz, twy);
  m.r[7] = fadd(tyz, twx);
  m.r[8] = fsub(1.0f, fadd(txx, tyy));
  m.t[0] = __double2float_rn(tx_);
  m.t[1] = __double2float_rn(ty_);
  m.t[2] = __double2float_rn(tz_);
  return m;
}

__device__ __forceinline__ F3 accum_apply(const AccumXform& m, const F3& p)
{
  F3 o;
  o.x = fadd(fadd(fadd(fmul(m.r[0], p.x), fmul(m.r[1], p.y)), fmul(m.r[2], p.z)), m.t[0]);
  o.y = fadd(fadd(fadd(fmul(m.r[3], p.x), fmul(m.r[4], p.y)), fmul(m.r[5], p.z)), m.t[1]);
  o.z = fadd(fadd(fadd(fmul(m.r[6], p.x), fmul(m.r[7], p.y)), fmul(m.r[8], p.z)), m.t[2]);
  return o;
}

// pcl::transformPointCloud: a cloud that is not dense keeps a point with any non-finite coordinate as it is
__device__ __forceinline__ F3 accum_second(const AccumXform& m, bool dense, const F3& p)
{
  return (dense || (scan_finite(p.x) && scan_finite(p.y) && scan_finite(p.z))) ? accum_apply(m, p) : p;
}

// one little-endian FLOAT32 at any byte address
__device__ __forceinline__ float accum_load_f32(const unsigned char* p)
{
  if ((reinterpret_cast<uintptr_t>(p) & 3u) == 0)
    return __uint_as_float(*reinterpret_cast<const uint32_t*>(p));
  const uint32_t b = static_cast<uint32_t>(p[0]) | (static_cast<uint32_t>(p[1]) << 8) | (static_cast<uint32_t>(p[2]) << 16) |
                     (static_cast<uint32_t>(p[3]) << 24);
  return __uint_as_float(b);
}

// the first byte of point (r, c) of a PointCloud2: data + r row_step + c point_step
__device__ __forceinline__ const unsigned char* cloud_point_at(const unsigned char* data, uint32_t r, uint32_t c, uint32_t row_step,
                                                               uint32_t point_step)
{
  return data + static_cast<uint64_t>(r) * row_step + static_cast<uint64_t>(c) * point_step;
}

// point (r, c) of a PointCloud2: data + r row_step + c point_step + offset[i]
__device__ __forceinline__ F3 accum_read(const unsigned char* data, uint32_t r, uint32_t c, uint32_t row_step, uint32_t point_step,
                                         uint32_t ox, uint32_t oy, uint32_t oz)
{
  const unsigned char* p = cloud_point_at(data, r, c, row_step, point_step);
  F3 o;
  o.x = accum_load_f32(p + ox);
  o.y = accum_load_f32(p + oy);
  o.z = accum_load_f32(p + oz);
  return o;
}

// ---- map intake (mcl3dl_map_load / mcl3dl_map_update_set): fromROSMsg into PointXYZIL, no transform
// point (r, c) of a map cloud: x / y / z bits as they are; label from the UINT32 field at lo, intensity from the FLOAT32
// field at io, each 0 when its offset is negative (the PointXYZIL() defaults fromROSMsg leaves for a missing field)
__device__ __forceinline__ mcl3dl_point map_read(const unsigned char* data, uint32_t r, uint32_t c, uint32_t row_step, uint32_t point_step,
                                                 uint32_t ox, uint32_t oy, uint32_t oz, int32_t io, int32_t lo, float& intensity)
{
  const unsigned char* p = cloud_point_at(data, r, c, row_step, point_step);
  mcl3dl_point o;
  o.x = accum_load_f32(p + ox);
  o.y = accum_load_f32(p + oy);
  o.z = accum_load_f32(p + oz);
  o.label = lo >= 0 ? __float_as_uint(accum_load_f32(p + lo)) : 0u;
  intensity = io >= 0 ? accum_load_f32(p + io) : 0.0f;
  return o;
}

// the intensity of one voxel: the float sum of in[order[0..cnt)] in input order over float(cnt), as x / y / z in
// scan_voxel_point
__device__ __forceinline__ float map_voxel_intensity(const float* __restrict__ in, const uint32_t* __restrict__ order, uint32_t cnt)
{
  float s = 0.0f;
  for (uint32_t j = 0; j < cnt; ++j) s = fadd(s, in[order[j]]);
  return fdiv(s, static_cast<float>(cnt));
}

}  // namespace mcl3dl
