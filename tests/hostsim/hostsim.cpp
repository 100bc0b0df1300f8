// hostsim.cpp — TEST INFRASTRUCTURE ONLY.
//
// Compiles the product's per-thread device functions (mcl_3dl_b200/csrc/device_math.cuh, device_funcs.cuh) for the
// HOST through cuda_shim.h and drives them over host-built copies of the device grids, one (particle, point) at a
// time.  tests/test_hostsim.py compares the result with the oracle: a way to check edits to cast_ray / cast_ray_kd /
// nn_dist2 / nn_search_arg / the NN field (nnf_select, nnf_dist2, nnf_search_arg) / the transform / the near-field
// screens without a GPU.  TMA staging, shuffles and the CTA reductions are only covered by the GPU suite.
// The grid construction below restates what engine.cu's build kernels do (same cell functions, same stable order).
#include "cuda_shim.h"
#ifndef MCL3DL_NEAR_BITS
#define MCL3DL_NEAR_BITS 1  // the host build always carries the near-field screens; near_k = 0 switches them off at run time
#endif

#include <algorithm>
#include <numeric>
#include <vector>

#include "../../include/mcl3dl_b200.h"
#include "../../mcl_3dl_b200/csrc/device_funcs.cuh"

using namespace mcl3dl;

namespace
{
struct HostMap
{
  std::vector<uint32_t> nn_cell_start, dda_cell_start, occ;
  std::vector<float4> nn_pts, dda_pts, raw_pts;
  std::vector<uint32_t> near_lik, near_kd;
  std::vector<uint2> nnf_dir;
  std::vector<float4> nnf_cand;
  std::vector<uint4> nnf_wide;
  uint64_t nnf_voxels = 0, nnf_overflow = 0, nnf_wide_cells = 0;
  NnGridDev nn{};
  DdaGridDev dda{};
  KdRayDev kd{};
  LikDev lik{};
};

// engine.cu: build_near_field (same layout function, same marking function)
void build_near(std::vector<uint32_t>& bits, NearBitsDev& out, const mcl3dl_point* pts, size_t n, float wx, float wy, float wz,
                float r, int k, const float sc_min[3], const float sc_max[3])
{
  out = NearBitsDev{};
  NearBitsDev f{};
  if (k <= 0 || !near_layout(f, r, k, sc_min, sc_max, size_t(64) << 20))
    return;
  bits.assign(static_cast<size_t>(f.pitch) * f.ny * f.nz, 0u);
  for (size_t i = 0; i < n; ++i)
    near_mark_point(f, bits.data(), k, __fmul_rn(pts[i].x, wx), __fmul_rn(pts[i].y, wy), __fmul_rn(pts[i].z, wz));
  f.bits = bits.data();
  out = f;
}

void build(HostMap& m, const mcl3dl_point* pts, size_t n, const mcl3dl_lik_params* lp, const mcl3dl_beam_params* bp,
           float cell_factor, int near_k, int near_kd_k, int use_field)
{
  const float wx = lp ? lp->dist_weight[0] : 1.0f, wy = lp ? lp->dist_weight[1] : 1.0f, wz = lp ? lp->dist_weight[2] : 1.0f;
  float raw_min[3], raw_max[3], sc_min[3], sc_max[3];
  for (int k = 0; k < 3; ++k)
  {
    raw_min[k] = sc_min[k] = std::numeric_limits<float>::infinity();
    raw_max[k] = sc_max[k] = -std::numeric_limits<float>::infinity();
  }
  m.raw_pts.resize(n);
  for (size_t i = 0; i < n; ++i)
  {
    const float v[3] = {pts[i].x, pts[i].y, pts[i].z};
    const float s[3] = {__fmul_rn(pts[i].x, wx), __fmul_rn(pts[i].y, wy), __fmul_rn(pts[i].z, wz)};
    for (int k = 0; k < 3; ++k)
    {
      raw_min[k] = std::min(raw_min[k], v[k]);
      raw_max[k] = std::max(raw_max[k], v[k]);
      sc_min[k] = std::min(sc_min[k], s[k]);
      sc_max[k] = std::max(sc_max[k], s[k]);
    }
    m.raw_pts[i] = make_float4(pts[i].x, pts[i].y, pts[i].z, __uint_as_float(pts[i].label));
  }
  if (lp)
  {
    const float R = lp->match_dist_min;
    m.lik.match_dist_min = R;
    m.lik.match_dist_flat = lp->match_dist_flat;
    m.lik.match_weight = lp->match_weight;
    m.lik.r2 = static_cast<float>(static_cast<double>(R) * static_cast<double>(R));
    m.lik.rpad = R * 1.0001f + 1e-6f;
    NnGridDev g{};
    const float cell = std::max(R * cell_factor, m.lik.rpad * 1.01f);
    g.inv_cell = 1.0f / cell;
    g.wx = wx;
    g.wy = wy;
    g.wz = wz;
    int dims[3];
    float org[3];
    for (int k = 0; k < 3; ++k)
    {
      org[k] = sc_min[k] - 0.5f * cell;
      dims[k] = static_cast<int>(std::floor((static_cast<double>(sc_max[k]) - org[k]) / cell)) + 2;
    }
    g.nx = dims[0];
    g.ny = dims[1];
    g.nz = dims[2];
    g.ox = org[0];
    g.oy = org[1];
    g.oz = org[2];
    const size_t cells = static_cast<size_t>(g.nx) * g.ny * g.nz;
    std::vector<uint32_t> key(n);
    for (size_t i = 0; i < n; ++i)
    {
      int cx = __float2int_rd(__fmul_rn(__fsub_rn(__fmul_rn(pts[i].x, wx), g.ox), g.inv_cell));
      int cy = __float2int_rd(__fmul_rn(__fsub_rn(__fmul_rn(pts[i].y, wy), g.oy), g.inv_cell));
      int cz = __float2int_rd(__fmul_rn(__fsub_rn(__fmul_rn(pts[i].z, wz), g.oz), g.inv_cell));
      cx = min(max(cx, 0), g.nx - 1);
      cy = min(max(cy, 0), g.ny - 1);
      cz = min(max(cz, 0), g.nz - 1);
      key[i] = static_cast<uint32_t>((cz * g.ny + cy) * g.nx + cx);
    }
    std::vector<uint32_t> order(n);
    std::iota(order.begin(), order.end(), 0u);
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
    m.nn_cell_start.assign(cells + 1, 0);
    for (size_t i = 0; i < n; ++i) m.nn_cell_start[key[i] + 1]++;
    for (size_t c = 0; c < cells; ++c) m.nn_cell_start[c + 1] += m.nn_cell_start[c];
    m.nn_pts.resize(n);
    for (size_t k = 0; k < n; ++k)
    {
      const mcl3dl_point& p = pts[order[k]];
      m.nn_pts[k] = make_float4(__fmul_rn(p.x, wx), __fmul_rn(p.y, wy), __fmul_rn(p.z, wz), __uint_as_float(order[k]));
    }
    g.cell_start = m.nn_cell_start.data();
    g.pts = m.nn_pts.data();
    build_near(m.near_lik, g.near, pts, n, wx, wy, wz, m.lik.rpad, near_k, sc_min, sc_max);
    g.field = NnFieldDev{};
    if (use_field)
    {
      // engine.cu: build_nn_field (same layout, same marking, same per-voxel selection function, same packing)
      float radius = m.lik.rpad;
      if (bp && !bp->use_raycast_using_dda)
      {
        const float gx = static_cast<float>(bp->map_grid_size[0]), gy = static_cast<float>(bp->map_grid_size[1]),
                    gz = static_cast<float>(bp->map_grid_size[2]);
        const float r1 = static_cast<float>(std::sqrt(2.0) * std::max(gx, std::max(gy, gz)) / 2.0);
        radius = std::max(radius, r1 * 1.0001f + 1e-6f);
      }
      NearBitsDev lay{};
      std::vector<uint32_t> bits;
      if (near_layout(lay, radius, 2, sc_min, sc_max, size_t(1) << 40))
      {
        bits.assign(static_cast<size_t>(lay.pitch) * lay.ny * lay.nz, 0u);
        for (size_t i = 0; i < n; ++i)
          near_mark_point(lay, bits.data(), 2, __fmul_rn(pts[i].x, wx), __fmul_rn(pts[i].y, wy), __fmul_rn(pts[i].z, wz));
        NnFieldDev f{};
        f.nx = lay.nx;
        f.ny = lay.ny;
        f.nz = lay.nz;
        f.cnx = (lay.nx + 1) / 2;
        f.cny = (lay.ny + 1) / 2;
        f.cnz = (lay.nz + 1) / 2;
        f.ox = lay.ox;
        f.oy = lay.oy;
        f.oz = lay.oz;
        f.inv_e = lay.inv_cell;
        f.e = 1.0f / lay.inv_cell;
        f.radius = radius;
        float ext = 0.0f;
        for (int k = 0; k < 3; ++k) ext = std::max(ext, std::max(std::fabs(sc_min[k]), std::fabs(sc_max[k])) + 4.0f * f.e);
        f.pad = 0.01f * f.e + 16.0f * std::numeric_limits<float>::epsilon() * ext;
        const size_t n_cells = static_cast<size_t>(f.cnx) * f.cny * f.cnz;
        m.nnf_dir.assign(n_cells, make_uint2(0u, 0u));
        m.nnf_cand.clear();
        m.nnf_wide.clear();
        for (size_t cell = 0; cell < n_cells; ++cell)
        {
          const int cx = static_cast<int>(cell % f.cnx), cy = static_cast<int>((cell / f.cnx) % f.cny),
                    cz = static_cast<int>(cell / (static_cast<size_t>(f.cnx) * f.cny));
          uint32_t nib = 0, lo = 0, hi = 0;
          bool ovf = false, big = false;
          std::vector<float4> mine;
          for (int sub = 0; sub < 8; ++sub)
          {
            const int vx = 2 * cx + (sub & 1), vy = 2 * cy + ((sub >> 1) & 1), vz = 2 * cz + (sub >> 2);
            if (vx >= f.nx || vy >= f.ny || vz >= f.nz)
              continue;
            if (!((bits[(static_cast<size_t>(vz) * f.ny + vy) * lay.pitch + (vx >> 5)] >> (vx & 31)) & 1u))
              continue;
            uint32_t pos[kNnfMaxSurv];
            const int cnt = nnf_select(g, f, vx, vy, vz, pos);
            if (cnt > kNnfMaxSurv)
            {
              ovf = true;
              continue;
            }
            big |= cnt > kNnfMaxCand;
            nib |= (static_cast<uint32_t>(cnt) & 15u) << (4 * sub);
            (sub < 4 ? lo : hi) |= static_cast<uint32_t>(cnt) << (8 * (sub & 3));
            for (int i = 0; i < cnt; ++i) mine.push_back(g.pts[pos[i]]);
            m.nnf_voxels += cnt > 0;
          }
          if (ovf)
          {
            m.nnf_dir[cell] = make_uint2(0xffffffffu, 0xffffffffu);
            ++m.nnf_overflow;
          }
          else if (big)
          {
            // wide cell: byte counts in the side table (engine.cu: nnf_count_kernel / nnf_base_kernel)
            m.nnf_dir[cell] = make_uint2(0x80000000u | static_cast<uint32_t>(m.nnf_wide.size()), 0xfffffffeu);
            m.nnf_wide.push_back(make_uint4(static_cast<uint32_t>(m.nnf_cand.size()), lo, hi, 0u));
            ++m.nnf_wide_cells;
            m.nnf_cand.insert(m.nnf_cand.end(), mine.begin(), mine.end());
          }
          else
          {
            m.nnf_dir[cell] = make_uint2(static_cast<uint32_t>(m.nnf_cand.size()), nib);
            m.nnf_cand.insert(m.nnf_cand.end(), mine.begin(), mine.end());
          }
        }
        if (m.nnf_cand.empty())
          m.nnf_cand.push_back(make_float4(0, 0, 0, 0));
        if (m.nnf_wide.empty())
          m.nnf_wide.push_back(make_uint4(0, 0, 0, 0));
        f.dir = m.nnf_dir.data();
        f.wide = m.nnf_wide.data();
        f.cand = m.nnf_cand.data();
        g.field = f;
      }
    }
    m.nn = g;
  }
  if (bp)
  {
    DdaGridDev g{};
    g.grid = bp->dda_grid_size;
    g.ray_angle_half = bp->ray_angle_half;
    g.min_dist_thr_sq = bp->map_grid_size[0] * bp->map_grid_size[0] + bp->map_grid_size[1] * bp->map_grid_size[1] +
                        bp->map_grid_size[1] * bp->map_grid_size[1];
    g.hit_tolerance = static_cast<float>(bp->hit_tolerance);
    g.hit_range_sq = bp->hit_range_sq;
    g.sin_total_ref = bp->sin_total_ref;
    g.beam_likelihood = bp->beam_likelihood;
    g.beam_likelihood_min = bp->beam_likelihood_min;
    g.filter_label_max = bp->filter_label_max;
    g.short_only = bp->add_penalty_short_only_mode ? 1 : 0;
    g.min_x = raw_min[0];
    g.min_y = raw_min[1];
    g.min_z = raw_min[2];
    g.max_x = raw_max[0];
    g.max_y = raw_max[1];
    g.max_z = raw_max[2];
    if (bp->use_raycast_using_dda)
    {
      int dims[3];
      for (int k = 0; k < 3; ++k)
        dims[k] = static_cast<int>(static_cast<size_t>(static_cast<double>(raw_max[k] - raw_min[k]) / g.grid) + 1);
      g.nx = dims[0];
      g.ny = dims[1];
      g.nz = dims[2];
      const size_t cells = static_cast<size_t>(g.nx) * g.ny * g.nz;
      std::vector<uint32_t> key(n);
      m.occ.assign((cells + 31) / 32 + 1, 0u);
      for (size_t i = 0; i < n; ++i)
      {
        const int cx = dda_to_index(pts[i].x, g.min_x, g.grid), cy = dda_to_index(pts[i].y, g.min_y, g.grid),
                  cz = dda_to_index(pts[i].z, g.min_z, g.grid);
        key[i] = static_cast<uint32_t>(cx + cy * g.nx + cz * (g.nx * g.ny));
        m.occ[key[i] >> 5] |= 1u << (key[i] & 31);
      }
      std::vector<uint32_t> order(n);
      std::iota(order.begin(), order.end(), 0u);
      std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
      m.dda_cell_start.assign(cells + 2, 0);
      for (size_t i = 0; i < n; ++i) m.dda_cell_start[key[i] + 1]++;
      for (size_t c = 0; c < cells; ++c) m.dda_cell_start[c + 1] += m.dda_cell_start[c];
      m.dda_pts.resize(n);
      for (size_t k = 0; k < n; ++k) m.dda_pts[k] = m.raw_pts[order[k]];
      g.occ = m.occ.data();
      g.cell_start = m.dda_cell_start.data();
      g.pts = m.dda_pts.data();
    }
    else
    {
      const float gx = static_cast<float>(bp->map_grid_size[0]), gy = static_cast<float>(bp->map_grid_size[1]),
                  gz = static_cast<float>(bp->map_grid_size[2]);
      const float gmin = std::min(gx, std::min(gy, gz)), gmax = std::max(gx, std::max(gy, gz));
      KdRayDev k{};
      k.raw_pts = m.raw_pts.data();
      k.grid_min = gmin;
      k.hit_tolerance = static_cast<float>(bp->hit_tolerance);
      k.r1 = static_cast<float>(std::sqrt(2.0) * gmax / 2.0);
      k.r2 = static_cast<float>(gmin * 2 + std::sqrt(2.0) * gmax / 2.0);
      k.r1_sq = static_cast<float>(static_cast<double>(k.r1) * static_cast<double>(k.r1));
      k.r2_sq = static_cast<float>(static_cast<double>(k.r2) * static_cast<double>(k.r2));
      k.r1_pad = k.r1 * 1.0001f + 1e-6f;
      k.r2_pad = k.r2 * 1.0001f + 1e-6f;
      k.sin_den = gmin * 2.0;
      build_near(m.near_kd, k.near, pts, n, wx, wy, wz, k.r1_pad, near_kd_k, sc_min, sc_max);
      m.kd = k;
    }
    m.dda = g;
  }
}
}  // namespace

// near_k / near_kd_k: dilation of the near-field screens (0 = unscreened searches, i.e. MCL3DL_NEAR_K=0 on the device)
extern "C" int hostsim_measure_nf(const mcl3dl_point* map, size_t n, const mcl3dl_lik_params* lp, const mcl3dl_beam_params* bp,
                                  float cell_factor, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* lik_pts,
                                  size_t n_lik, const mcl3dl_point* beam_pts, size_t n_beam, const float* origins_xyz,
                                  size_t n_origins, mcl3dl_result* out, uint8_t* status, int near_k, int near_kd_k,
                                  uint64_t* work /* [5]: nn rows, nn pts, steps, occupied, tested; may be NULL */,
                                  int use_field /* 1: stage the NN field; the likelihood evals and the KD caster's
                                                   marching search go through it (nnf_dist2 / nnf_search_arg) */)
{
  if ((n_lik && !lp) || (n_beam && !bp) || (bp && !bp->use_raycast_using_dda && !lp))
    return -1;
  for (size_t j = 0; j < n_beam; ++j)
    if (beam_pts[j].label >= n_origins)
      return -1;
  HostMap m;
  build(m, map, n, lp, bp, cell_factor, near_k, near_kd_k, use_field);
  uint64_t wk[5] = {0, 0, 0, 0, 0};
  for (size_t p = 0; p < P; ++p)
  {
    F3 pos;
    Q4 q;
    load_pose(poses + p, pos, q);
    const Q4 rn = qnormalized(q);
    mcl3dl_result r;
    std::memset(&r, 0, sizeof(r));
    // beam: the per-ray body of beam_kernel_pl / beam_kernel_dq
    uint32_t a = 0, b = 0, c = 0, s0 = 0, s1 = 0, s2 = 0;
    for (size_t j = 0; j < n_beam; ++j)
    {
      F3 v;
      v.x = beam_pts[j].x;
      v.y = beam_pts[j].y;
      v.z = beam_pts[j].z;
      const F3 end = transform_point(rn, pos, v);
      const F3 begin = ray_origin(pos, q, origins_xyz, beam_pts[j].label);
      const int st = bp->use_raycast_using_dda ? cast_ray(m.dda, begin, end, s0, s1, s2) :
                                                 cast_ray_kd(m.kd, m.nn, m.dda, begin, end, s0, s1, s2);
      a += st == ST_SHORT;
      b += st == ST_HIT;
      c += st == ST_LONG;
      if (status) status[p * n_beam + j] = static_cast<uint8_t>(st);
    }
    wk[2] += s0;
    wk[3] += s1;
    wk[4] += s2;
    r.score_beam = beam_score(a, c, static_cast<int>(n_beam), m.dda);
    r.n_short = a;
    r.n_hit = b;
    r.n_long = c;
    // likelihood: the per-eval body of the likelihood kernels, summed in scan order
    if (n_lik == 0)
    {
      r.score_like = 1.0f;
    }
    else
    {
      float sl = 0.0f;
      uint32_t cnt = 0, rows = 0, npts = 0;
      for (size_t j = 0; j < n_lik; ++j)
      {
        F3 v;
        v.x = lik_pts[j].x;
        v.y = lik_pts[j].y;
        v.z = lik_pts[j].z;
        const F3 t = transform_point(rn, pos, v);
        const float sx = fmul(t.x, m.nn.wx), sy = fmul(t.y, m.nn.wy), sz = fmul(t.z, m.nn.wz);
        const float d2 = m.nn.field.dir ? nnf_dist2(m.nn, m.lik, sx, sy, sz, rows, npts) : nn_dist2(m.nn, m.lik, sx, sy, sz, rows, npts);
        float term;
        if (d2 < m.lik.r2 && lik_term(__fsqrt_rn(d2), m.lik, term))
        {
          sl = fadd(sl, term);
          cnt++;
        }
      }
      r.score_like = sl;
      r.match_cnt = cnt;
      wk[0] += rows;
      wk[1] += npts;
    }
    if (out) out[p] = r;
  }
  if (work)
  {
    for (int i = 0; i < 5; ++i) work[i] = wk[i];
    work[5] = m.nnf_cand.size();
    work[6] = m.nnf_voxels;
    work[7] = m.nnf_overflow;
    work[8] = m.nnf_wide_cells;
  }
  return 0;
}

extern "C" int hostsim_measure(const mcl3dl_point* map, size_t n, const mcl3dl_lik_params* lp, const mcl3dl_beam_params* bp,
                               float cell_factor, const mcl3dl_pose* poses, size_t P, const mcl3dl_point* lik_pts,
                               size_t n_lik, const mcl3dl_point* beam_pts, size_t n_beam, const float* origins_xyz,
                               size_t n_origins, mcl3dl_result* out, uint8_t* status)
{
  return hostsim_measure_nf(map, n, lp, bp, cell_factor, poses, P, lik_pts, n_lik, beam_pts, n_beam, origins_xyz, n_origins, out,
                            status, 2, 1, nullptr, 1);
}

// The near field on its own: build it for radius r / dilation k over `map` (rescaled by w) and evaluate near_maybe for
// `nq` rescaled query points.  layout_out = {nx, ny, nz, pitch}, cell_out = fine cell edge actually used (0 if the field
// could not be laid out, in which case every answer is 1 = "maybe near").
extern "C" int hostsim_near_query(const mcl3dl_point* map, size_t n, const float w[3], float r, int k, size_t max_bytes,
                                  const float* queries_xyz, size_t nq, uint8_t* maybe_out, int32_t layout_out[4],
                                  float* cell_out)
{
  float sc_min[3], sc_max[3];
  for (int a = 0; a < 3; ++a)
  {
    sc_min[a] = std::numeric_limits<float>::infinity();
    sc_max[a] = -std::numeric_limits<float>::infinity();
  }
  for (size_t i = 0; i < n; ++i)
  {
    const float s[3] = {__fmul_rn(map[i].x, w[0]), __fmul_rn(map[i].y, w[1]), __fmul_rn(map[i].z, w[2])};
    for (int a = 0; a < 3; ++a)
    {
      sc_min[a] = std::min(sc_min[a], s[a]);
      sc_max[a] = std::max(sc_max[a], s[a]);
    }
  }
  NearBitsDev f{};
  std::vector<uint32_t> bits;
  if (k > 0 && near_layout(f, r, k, sc_min, sc_max, max_bytes))
  {
    bits.assign(static_cast<size_t>(f.pitch) * f.ny * f.nz, 0u);
    for (size_t i = 0; i < n; ++i)
      near_mark_point(f, bits.data(), k, __fmul_rn(map[i].x, w[0]), __fmul_rn(map[i].y, w[1]), __fmul_rn(map[i].z, w[2]));
    f.bits = bits.data();
  }
  layout_out[0] = f.nx;
  layout_out[1] = f.ny;
  layout_out[2] = f.nz;
  layout_out[3] = f.pitch;
  *cell_out = f.bits ? 1.0f / f.inv_cell : 0.0f;
  for (size_t q = 0; q < nq; ++q)
    maybe_out[q] = near_maybe(f, queries_xyz[3 * q], queries_xyz[3 * q + 1], queries_xyz[3 * q + 2]) ? 1 : 0;
  return 0;
}



// Field mode: field_dist (device_funcs.cuh) over a host copy of the per-cell corner layout built from a node volume
// (x fastest, dims = nodes per axis), exactly as engine.cu's field_expand_kernel lays it out.
extern "C" int hostsim_field_dist(const float* nodes, const int32_t dims[3], const float origin[3], float edge, float clamp,
                                  const float* queries_xyz, size_t nq, float* out)
{
  const int nx = dims[0] - 1, ny = dims[1] - 1, nz = dims[2] - 1;
  if (nx < 1 || ny < 1 || nz < 1)
    return -1;
  std::vector<float4> cells(static_cast<size_t>(nx) * ny * nz * 2);
  auto node = [&](int a, int b, int c) { return nodes[(static_cast<size_t>(c) * dims[1] + b) * dims[0] + a]; };
  for (int k = 0; k < nz; ++k)
    for (int j = 0; j < ny; ++j)
      for (int i = 0; i < nx; ++i)
      {
        const size_t t = (static_cast<size_t>(k) * ny + j) * nx + i;
        cells[2 * t] = make_float4(node(i, j, k), node(i + 1, j, k), node(i, j + 1, k), node(i + 1, j + 1, k));
        cells[2 * t + 1] = make_float4(node(i, j, k + 1), node(i + 1, j, k + 1), node(i, j + 1, k + 1), node(i + 1, j + 1, k + 1));
      }
  FieldDev f{};
  f.cells = cells.data();
  f.nx = nx;
  f.ny = ny;
  f.nz = nz;
  f.ox = origin[0];
  f.oy = origin[1];
  f.oz = origin[2];
  f.inv_e = 1.0f / edge;
  f.clamp = clamp;
  for (size_t q = 0; q < nq; ++q) out[q] = field_dist(f, queries_xyz[3 * q], queries_xyz[3 * q + 1], queries_xyz[3 * q + 2]);
  return 0;
}

// nnf_slot alone (device_funcs.cuh): the (count, first candidate) of voxel `sub` of one directory entry; wide entries
// read `wide` (one uint4).  Returns the count (-1: overflow cell).
extern "C" int hostsim_nnf_slot(uint32_t dir_x, uint32_t dir_y, const uint32_t wide[4], int sub, uint32_t* start)
{
  NnFieldDev f{};
  const uint4 w = make_uint4(wide[0], wide[1], wide[2], wide[3]);
  // a wide entry indexes the side table: give it a table whose entry (dir_x & 0x7fffffff) is `w`
  std::vector<uint4> table((dir_x & 0x80000000u) && dir_x != 0xffffffffu ? (dir_x & 0x7fffffffu) + 1 : 1, make_uint4(0, 0, 0, 0));
  table.back() = w;
  f.wide = table.data();
  uint32_t s = 0;
  const int c = nnf_slot(f, make_uint2(dir_x, dir_y), sub, s);
  *start = s;
  return c;
}
