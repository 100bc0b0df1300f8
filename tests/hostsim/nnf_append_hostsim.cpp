// nnf_append_hostsim.cpp — TEST INFRASTRUCTURE ONLY.
//
// The NN field after an append (engine.cu: update_nn_field), on the host.  The field of map A comes from hostsim.cpp's
// host build (the build kernels restated).  The append marks directory cells with the device's own marking function
// (device_funcs.cuh: nnf_mark_append, compiled verbatim through cuda_shim.h) and re-selects only the marked cells over
// the CSR grid of A + P, with the per-cell rules of nnf_count_kernel (bits, nnf_select, plain / wide / overflow).  Every
// directory cell is then decoded (kind, per-voxel counts, candidate bytes in order) and compared with a fresh host build
// of A + P.  tests/test_nnf_append_on_host.py drives it.
#include "hostsim.cpp"

#include <cstring>

namespace
{
struct CellList
{
  int kind = 0;  // 0 plain, 1 wide, 2 overflow
  int counts[8] = {};
  std::vector<float4> cand;
  bool operator==(const CellList& o) const
  {
    return kind == o.kind && std::memcmp(counts, o.counts, sizeof(counts)) == 0 && cand.size() == o.cand.size() &&
           (cand.empty() || std::memcmp(cand.data(), o.cand.data(), cand.size() * sizeof(float4)) == 0);
  }
};

CellList decode(const NnFieldDev& f, size_t cell)
{
  CellList r;
  const uint2 d = f.dir[cell];
  if (d.x == 0xffffffffu)
  {
    r.kind = 2;
    return r;
  }
  r.kind = (d.x & 0x80000000u) ? 1 : 0;
  for (int sub = 0; sub < 8; ++sub)
  {
    uint32_t start = 0;
    r.counts[sub] = nnf_slot(f, d, sub, start);
    for (int i = 0; i < r.counts[sub]; ++i) r.cand.push_back(f.cand[start + i]);
  }
  return r;
}

// nnf_count_kernel + nnf_fill_kernel for one directory cell of the field's lattice over grid g
CellList select_cell(const NnGridDev& g, const NnFieldDev& f, const std::vector<uint32_t>& bits, int pitch, size_t cell)
{
  CellList r;
  const int cx = static_cast<int>(cell % f.cnx), cy = static_cast<int>((cell / f.cnx) % f.cny),
            cz = static_cast<int>(cell / (static_cast<size_t>(f.cnx) * f.cny));
  bool ovf = false, big = false;
  for (int sub = 0; sub < 8; ++sub)
  {
    const int vx = 2 * cx + (sub & 1), vy = 2 * cy + ((sub >> 1) & 1), vz = 2 * cz + (sub >> 2);
    if (vx >= f.nx || vy >= f.ny || vz >= f.nz || !((bits[(static_cast<size_t>(vz) * f.ny + vy) * pitch + (vx >> 5)] >> (vx & 31)) & 1u))
      continue;
    uint32_t pos[kNnfMaxSurv];
    const int cnt = nnf_select(g, f, vx, vy, vz, pos);
    if (cnt > kNnfMaxSurv)
    {
      ovf = true;
      continue;
    }
    big |= cnt > kNnfMaxCand;
    r.counts[sub] = cnt;
    for (int i = 0; i < cnt; ++i) r.cand.push_back(g.pts[pos[i]]);
  }
  if (ovf)
  {
    CellList o;
    o.kind = 2;
    return o;
  }
  r.kind = big ? 1 : 0;
  return r;
}

void boxes(const mcl3dl_point* p, size_t n, const float w[3], float out[12])
{
  for (int k = 0; k < 3; ++k)
  {
    out[k] = out[6 + k] = std::numeric_limits<float>::infinity();
    out[3 + k] = out[9 + k] = -std::numeric_limits<float>::infinity();
  }
  for (size_t i = 0; i < n; ++i)
  {
    const float v[3] = {p[i].x, p[i].y, p[i].z};
    for (int k = 0; k < 3; ++k)
    {
      out[k] = std::min(out[k], v[k]);
      out[3 + k] = std::max(out[3 + k], v[k]);
      out[6 + k] = std::min(out[6 + k], __fmul_rn(v[k], w[k]));
      out[9 + k] = std::max(out[9 + k], __fmul_rn(v[k], w[k]));
    }
  }
}
}  // namespace

// out: [0] directory cells, [1] marked, [2] cells where the appended field differs from the fresh build of A + P,
// [3] cells whose lists A + P changed against A, [4] of those, cells left unmarked, [5] 1 = both bounding boxes unchanged
// (the incremental path applies; 0: the engine rebuilds, nothing else is computed), [6] wide / [7] overflow cells of the
// fresh build of A + P.
extern "C" int hostsim_nnf_append(const mcl3dl_point* a, size_t na, const mcl3dl_point* p, size_t np,
                                  const mcl3dl_lik_params* lp, uint64_t out[8])
{
  std::memset(out, 0, 8 * sizeof(uint64_t));
  std::vector<mcl3dl_point> ap(a, a + na);
  ap.insert(ap.end(), p, p + np);
  float box_a[12], box_ap[12];
  boxes(a, na, lp->dist_weight, box_a);
  boxes(ap.data(), ap.size(), lp->dist_weight, box_ap);
  out[5] = std::memcmp(box_a, box_ap, sizeof(box_a)) == 0;
  if (!out[5])
    return 0;
  HostMap ma, mf;
  build(ma, a, na, lp, nullptr, 1.0f, 2, 1, 1);
  build(mf, ap.data(), ap.size(), lp, nullptr, 1.0f, 2, 1, 1);
  const NnFieldDev& fa = ma.nn.field;
  const NnFieldDev& ff = mf.nn.field;
  if (!fa.dir || !ff.dir || fa.cnx != ff.cnx || fa.cny != ff.cny || fa.cnz != ff.cnz || fa.pad != ff.pad)
    return -1;
  const size_t n_cells = static_cast<size_t>(fa.cnx) * fa.cny * fa.cnz;
  out[0] = n_cells;
  // the mark pass over the appended points, on the grid of A + P (its lattice is A's)
  std::vector<uint8_t> marked(n_cells, 0);
  for (size_t i = 0; i < np; ++i)
    nnf_mark_append(mf.nn, fa, p[i].x, p[i].y, p[i].z, [&](size_t cell) { marked[cell] = 1; });
  // the field's own k = 2 near field of A + P (update_nn_field rebuilds it the same way)
  NearBitsDev lay{};
  float sc_min[3], sc_max[3];
  for (int k = 0; k < 3; ++k)
  {
    sc_min[k] = box_ap[6 + k];
    sc_max[k] = box_ap[9 + k];
  }
  if (!near_layout(lay, fa.radius, 2, sc_min, sc_max, size_t(1) << 40))
    return -1;
  std::vector<uint32_t> bits(static_cast<size_t>(lay.pitch) * lay.ny * lay.nz, 0u);
  for (const auto& q : ap)
    near_mark_point(lay, bits.data(), 2, __fmul_rn(q.x, lp->dist_weight[0]), __fmul_rn(q.y, lp->dist_weight[1]),
                    __fmul_rn(q.z, lp->dist_weight[2]));
  for (size_t cell = 0; cell < n_cells; ++cell)
  {
    out[1] += marked[cell];
    const CellList fresh = decode(ff, cell);
    const CellList before = decode(fa, cell);
    const CellList after = marked[cell] ? select_cell(mf.nn, fa, bits, lay.pitch, cell) : before;
    out[2] += !(after == fresh);
    const bool changed = !(before == fresh);
    out[3] += changed;
    out[4] += changed && !marked[cell];
    out[6] += fresh.kind == 1;
    out[7] += fresh.kind == 2;
  }
  return 0;
}
