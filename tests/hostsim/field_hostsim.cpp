// field_hostsim.cpp — TEST INFRASTRUCTURE ONLY.
//
// The per-eval device functions of field mode (mcl_3dl_b200/csrc/device_funcs.cuh: field_dist, lik_term, and the
// transform of device_math.cuh), compiled for the host through cuda_shim.h, plus near_layout, the rule that lays out
// the NN field's lattice and with it the field-mode lattice.  tests/test_field_on_host.py holds them to the numpy
// restatement of tests/field_restate.py; tests/test_gpu_field_exact.py takes the per-point terms of whole scans from
// here.
#include "cuda_shim.h"

#include "../../include/mcl3dl_b200.h"
#include "../../mcl_3dl_b200/csrc/device_funcs.cuh"

using namespace mcl3dl;

namespace
{
FieldDev field(const float4* cells, const int32_t dims[3], const float org[3], float inv_e, float clamp)
{
  FieldDev f{};
  f.cells = cells;
  f.nx = dims[0];
  f.ny = dims[1];
  f.nz = dims[2];
  f.ox = org[0];
  f.oy = org[1];
  f.oz = org[2];
  f.inv_e = inv_e;
  f.clamp = clamp;
  return f;
}
}  // namespace

// field_dist at q[n][3] (rescaled space) over cells [nz][ny][nx][2] (dims: cells per axis)
extern "C" void hostsim_field_dist(const float4* cells, const int32_t dims[3], const float org[3], float inv_e, float clamp,
                                   const float* q, size_t n, float* out)
{
  const FieldDev f = field(cells, dims, org, inv_e, clamp);
  for (size_t i = 0; i < n; ++i) out[i] = field_dist(f, q[3 * i], q[3 * i + 1], q[3 * i + 2]);
}

// lik_kernel_field's test of one interpolated distance: d < match_dist_min && lik_term(d); the contribution or 0
extern "C" void hostsim_field_term(const float* d, size_t n, float R, float flat, float w, float* term, uint8_t* counted)
{
  LikDev lp{};
  lp.match_dist_min = R;
  lp.match_dist_flat = flat;
  lp.match_weight = w;
  for (size_t i = 0; i < n; ++i)
  {
    float t = 0.0f;
    counted[i] = d[i] < lp.match_dist_min && lik_term(d[i], lp, t);
    term[i] = counted[i] ? t : 0.0f;
  }
}

// The per-point terms of a field-mode update: T[p][j] and M[p][j] of particle p at scan point j, as lik_kernel_field
// computes one eval (normalised rotation, transform, dist_weight, field_dist, lik_term).
extern "C" void hostsim_field_terms(const mcl3dl_pose* poses, size_t P, const float4* scan, size_t N, const float4* cells,
                                    const int32_t dims[3], const float org[3], float inv_e, float clamp, const float dw[3],
                                    float R, float flat, float w, float* T, uint8_t* M)
{
  const FieldDev f = field(cells, dims, org, inv_e, clamp);
  LikDev lp{};
  lp.match_dist_min = R;
  lp.match_dist_flat = flat;
  lp.match_weight = w;
  for (size_t p = 0; p < P; ++p)
  {
    F3 pos;
    Q4 q;
    pos.x = poses[p].px;
    pos.y = poses[p].py;
    pos.z = poses[p].pz;
    q.x = poses[p].qx;
    q.y = poses[p].qy;
    q.z = poses[p].qz;
    q.w = poses[p].qw;
    const Q4 rn = qnormalized(q);
    for (size_t j = 0; j < N; ++j)
    {
      F3 v;
      v.x = scan[j].x;
      v.y = scan[j].y;
      v.z = scan[j].z;
      const F3 t = transform_point(rn, pos, v);
      const float d = field_dist(f, fmul(t.x, dw[0]), fmul(t.y, dw[1]), fmul(t.z, dw[2]));
      float c = 0.0f;
      const bool m = d < lp.match_dist_min && lik_term(d, lp, c);
      T[p * N + j] = m ? c : 0.0f;
      M[p * N + j] = m;
    }
  }
}

// near_layout(r, k, sc_min, sc_max, max_bytes): ok, dims[3], origin[3], inv_cell
extern "C" int hostsim_near_layout(float r, int k, const float sc_min[3], const float sc_max[3], size_t max_bytes,
                                   int32_t dims[3], float org[3], float* inv_cell)
{
  NearBitsDev f{};
  if (!near_layout(f, r, k, sc_min, sc_max, max_bytes))
    return 0;
  dims[0] = f.nx;
  dims[1] = f.ny;
  dims[2] = f.nz;
  org[0] = f.ox;
  org[1] = f.oy;
  org[2] = f.oz;
  *inv_cell = f.inv_cell;
  return 1;
}
