// device_math.cuh — float/double arithmetic of the mcl_3dl hot path, operation for operation.
//
// The beam model's HIT/SHORT/LONG tallies must be bit-exact with the reference CPU build, and the
// voxel a ray visits depends on the last bit of the transformed endpoint.  Every expression here is
// therefore written with explicit round-to-nearest intrinsics (no FMA contraction, IEEE division and
// square root) in the operand order of the reference source it cites.  The translation unit is also
// compiled with -fmad=false as a second line of defence.
#pragma once
#ifndef MCL3DL_HOSTSIM  // tests/hostsim compiles this header for the host with its own intrinsic shims
#include <cuda_runtime.h>
#endif
#include <stdint.h>

namespace mcl3dl
{
struct F3
{
  float x, y, z;
};
struct Q4
{
  float x, y, z, w;
};

__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

// float -> unsigned int that orders like the float (for atomicMin / atomicMax bounding boxes)
__device__ __forceinline__ uint32_t f2ord(float f)
{
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// Vec3::dot, include/mcl_3dl/vec3.h:140-143: (x*x' + y*y') + z*z'
__device__ __forceinline__ float dot3(const F3& a, const F3& b)
{
  return fadd(fadd(fmul(a.x, b.x), fmul(a.y, b.y)), fmul(a.z, b.z));
}

// Quat::operator*(Quat), include/mcl_3dl/quat.h:131-138: ((w*qx + x*qw) + y*qz) - z*qy, ...
__device__ __forceinline__ Q4 qmul(const Q4& a, const Q4& b)
{
  Q4 r;
  r.x = fsub(fadd(fadd(fmul(a.w, b.x), fmul(a.x, b.w)), fmul(a.y, b.z)), fmul(a.z, b.y));
  r.y = fsub(fadd(fadd(fmul(a.w, b.y), fmul(a.y, b.w)), fmul(a.z, b.x)), fmul(a.x, b.z));
  r.z = fsub(fadd(fadd(fmul(a.w, b.z), fmul(a.z, b.w)), fmul(a.x, b.y)), fmul(a.y, b.x));
  r.w = fsub(fsub(fsub(fmul(a.w, b.w), fmul(a.x, b.x)), fmul(a.y, b.y)), fmul(a.z, b.z));
  return r;
}

// Quat::operator*(Vec3), quat.h:139-143: q * (v, 0) * conj(q), two full Hamilton products
__device__ __forceinline__ F3 qrot(const Q4& q, const F3& v)
{
  Q4 pv;
  pv.x = v.x;
  pv.y = v.y;
  pv.z = v.z;
  pv.w = 0.0f;
  Q4 c;
  c.x = -q.x;
  c.y = -q.y;
  c.z = -q.z;
  c.w = q.w;
  const Q4 r = qmul(qmul(q, pv), c);
  F3 o;
  o.x = r.x;
  o.y = r.y;
  o.z = r.z;
  return o;
}

// Quat::normalized, quat.h:175-178 -> operator/(s) (:148-151) == operator*(float(1.0 / s))
__device__ __forceinline__ Q4 qnormalized(const Q4& q)
{
  const float n2 = fadd(fadd(fadd(fmul(q.x, q.x), fmul(q.y, q.y)), fmul(q.z, q.z)), fmul(q.w, q.w));
  const float n = __fsqrt_rn(n2);
  const float inv = __double2float_rn(ddiv(1.0, static_cast<double>(n)));
  Q4 r;
  r.x = fmul(q.x, inv);
  r.y = fmul(q.y, inv);
  r.z = fmul(q.z, inv);
  r.w = fmul(q.w, inv);
  return r;
}

// State6DOF::transform, include/mcl_3dl/state_6dof.h:214-225: r * p + pos_
__device__ __forceinline__ F3 transform_point(const Q4& rn, const F3& pos, const F3& p)
{
  const F3 r = qrot(rn, p);
  F3 t;
  t.x = fadd(r.x, pos.x);
  t.y = fadd(r.y, pos.y);
  t.z = fadd(r.z, pos.z);
  return t;
}

}  // namespace mcl3dl
