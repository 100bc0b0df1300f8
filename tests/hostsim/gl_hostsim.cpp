// gl_hostsim.cpp — TEST INFRASTRUCTURE ONLY.
//
// Host driver for mcl_3dl_b200/csrc/gl_funcs.cuh (global localisation and the resident set's resize), compiled for the
// host through cuda_shim.h.  The serial loops below stand in for the kernels of gl_kernels.cuh and the CSR grid that
// engine.cu's build_nn_csr sorts on the device (same lattice rule, same cell function, input order inside a cell);
// tests/test_global_localization_on_host.py compares them with both CPU checkers.  scan_hostsim.cpp comes along for
// the VoxelGrid (hostsim_scan_voxel_grid).
#include "scan_hostsim.cpp"

#include "../../mcl_3dl_b200/csrc/gl_funcs.cuh"

// The service body after the VoxelGrid: free-space filter of ds[0..n) and the particles of the survivors.  Returns the
// number of particles (states / probs need room for n * div_yaw), -1 for a lattice of 2^31 cells or more.
extern "C" long hostsim_gl_seed(const mcl3dl_point* ds, size_t n, double grid, int32_t div_yaw, const float imu[4], const float w[3],
                                mcl3dl_state* states, float* probs, uint64_t* n_seeds)
{
  *n_seeds = 0;
  if (n == 0)
    return 0;
  const float g32 = static_cast<float>(grid);
  GlDev m{};
  m.z_off = 0.01 + grid;
  m.r2 = static_cast<float>(grid * grid);
  m.rpad = g32 * 1.0001f + 1e-6f;
  NnGridDev g{};
  g.wx = w[0];
  g.wy = w[1];
  g.wz = w[2];
  // engine.cu: bbox_kernel's rescaled box (fminf / fmaxf skip NaN), nn_lattice, build_nn_csr
  float sc_min[3] = {INFINITY, INFINITY, INFINITY}, sc_max[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (size_t i = 0; i < n; ++i)
  {
    const float v[3] = {ds[i].x * w[0], ds[i].y * w[1], ds[i].z * w[2]};
    for (int k = 0; k < 3; ++k)
    {
      sc_min[k] = std::fmin(sc_min[k], v[k]);
      sc_max[k] = std::fmax(sc_max[k], v[k]);
    }
  }
  const float cell = m.rpad * 1.01f;
  g.inv_cell = 1.0f / cell;
  int64_t total = 1;
  int dims[3];
  float org[3];
  for (int k = 0; k < 3; ++k)
  {
    if (!std::isfinite(sc_min[k]) || !std::isfinite(sc_max[k]))
      return -1;
    org[k] = sc_min[k] - 0.5f * cell;
    dims[k] = static_cast<int>(std::floor((static_cast<double>(sc_max[k]) - org[k]) / cell)) + 2;
    total *= dims[k];
  }
  if (total >= (int64_t(1) << 31))
    return -1;
  g.nx = dims[0];
  g.ny = dims[1];
  g.nz = dims[2];
  g.ox = org[0];
  g.oy = org[1];
  g.oz = org[2];
  std::vector<uint32_t> key(n), order(n), cell_start(static_cast<size_t>(total) + 1, 0);
  for (size_t i = 0; i < n; ++i)
  {
    int cx = __float2int_rd(__fmul_rn(__fsub_rn(__fmul_rn(ds[i].x, g.wx), g.ox), g.inv_cell));
    int cy = __float2int_rd(__fmul_rn(__fsub_rn(__fmul_rn(ds[i].y, g.wy), g.oy), g.inv_cell));
    int cz = __float2int_rd(__fmul_rn(__fsub_rn(__fmul_rn(ds[i].z, g.wz), g.oz), g.inv_cell));
    cx = min(max(cx, 0), g.nx - 1);
    cy = min(max(cy, 0), g.ny - 1);
    cz = min(max(cz, 0), g.nz - 1);
    key[i] = static_cast<uint32_t>((cz * g.ny + cy) * g.nx + cx);
    cell_start[key[i] + 1]++;
  }
  for (size_t c = 1; c < cell_start.size(); ++c) cell_start[c] += cell_start[c - 1];
  std::iota(order.begin(), order.end(), 0u);
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
  std::vector<float4> pts(n);
  for (size_t k = 0; k < n; ++k)
  {
    const mcl3dl_point& p = ds[order[k]];
    pts[k] = make_float4(p.x * g.wx, p.y * g.wy, p.z * g.wz, __uint_as_float(order[k]));
  }
  g.cell_start = cell_start.data();
  g.pts = pts.data();
  std::vector<mcl3dl_point> seeds;
  for (size_t i = 0; i < n; ++i)
    if (!gl_has_neighbour(g, m, gl_query(g, m, ds[i])))
      seeds.push_back(ds[i]);
  *n_seeds = seeds.size();
  if (seeds.empty())
    return 0;
  std::vector<Q4> yaw(static_cast<size_t>(div_yaw));
  gl_yaw_quats(div_yaw, imu, yaw.data());
  const float prob = gl_probability(seeds.size());
  const size_t np = seeds.size() * static_cast<size_t>(div_yaw);
  for (size_t i = 0; i < np; ++i)
  {
    const PfState s = gl_particle(seeds.data(), yaw.data(), static_cast<uint32_t>(div_yaw), static_cast<uint32_t>(i));
    std::memcpy(states + i, &s, sizeof(s));
    probs[i] = prob;
  }
  return static_cast<long>(np);
}

// the yaw table alone
extern "C" void hostsim_gl_yaw(int32_t div_yaw, const float imu[4], float* out /* 4 * div_yaw */)
{
  gl_yaw_quats(div_yaw, imu, reinterpret_cast<Q4*>(out));
}

extern "C" float hostsim_gl_probability(uint64_t n_seeds) { return gl_probability(n_seeds); }

// mcl3dl_particles_resize: pf_accum_kernel's sequential sum, gl_pscan_kernel's chain, gl_resize_pick per output
extern "C" void hostsim_gl_resize(const float* probs, const mcl3dl_state* states, size_t n, size_t num, mcl3dl_state* out_states,
                                  float* out_probs)
{
  std::vector<float> accum(n), pscan(num);
  float a = 0.0f;
  for (size_t i = 0; i < n; ++i) accum[i] = a = __fadd_rn(a, probs[i]);
  const float pstep = __fdiv_rn(accum[n - 1], static_cast<float>(num));
  a = 0.0f;
  for (size_t i = 0; i < num; ++i) pscan[i] = a = __fadd_rn(a, pstep);
  for (size_t i = 0; i < num; ++i)
  {
    out_states[i] = states[gl_resize_pick(accum.data(), static_cast<uint32_t>(n), pscan.data(), static_cast<uint32_t>(i))];
    out_probs[i] = gl_resize_probability(static_cast<uint32_t>(num));
  }
}
