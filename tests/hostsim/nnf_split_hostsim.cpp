// The NN-field lookup in three steps (device_funcs.cuh: nnf_address, nnf_entry, nnf_slot), as the likelihood kernels'
// phase A runs it (kernels.cuh: nf_phase_a, with the directory index cut to 32 bits), against nnf_lookup, over a
// directory given by the caller.  TEST INFRASTRUCTURE ONLY (tests/test_nnf_split_on_host.py).
#include "cuda_shim.h"

#include "../../include/mcl3dl_b200.h"
#include "../../mcl_3dl_b200/csrc/device_funcs.cuh"

using namespace mcl3dl;

// dims = fine voxels per axis; dir: (cnx * cny * cnz) entries as {x, y} pairs; wide: side-table entries as 4 words.
// Writes per query the count and first candidate of nnf_lookup and of the three steps, and whether the address step
// found the query inside the lattice.
extern "C" int hostsim_nnf_split(const int32_t dims[3], const float origin[3], float inv_e, const uint32_t* dir,
                                 const uint32_t* wide, const float* queries_xyz, size_t nq, int32_t* lookup_count,
                                 uint32_t* lookup_start, int32_t* split_count, uint32_t* split_start, uint8_t* inside)
{
  NnFieldDev f{};
  f.dir = reinterpret_cast<const uint2*>(dir);
  f.wide = reinterpret_cast<const uint4*>(wide);
  f.nx = dims[0];
  f.ny = dims[1];
  f.nz = dims[2];
  f.cnx = (f.nx + 1) / 2;
  f.cny = (f.ny + 1) / 2;
  f.cnz = (f.nz + 1) / 2;
  f.ox = origin[0];
  f.oy = origin[1];
  f.oz = origin[2];
  f.inv_e = inv_e;
  f.e = 1.0f / inv_e;
  for (size_t q = 0; q < nq; ++q)
  {
    const float x = queries_xyz[3 * q], y = queries_xyz[3 * q + 1], z = queries_xyz[3 * q + 2];
    uint32_t s = 0;
    lookup_count[q] = nnf_lookup(f, x, y, z, s);
    lookup_start[q] = s;
    size_t cell;
    int sub;
    const bool in = nnf_address(f, x, y, z, cell, sub);
    s = 0;
    split_count[q] = nnf_slot(f, nnf_entry(f, in, static_cast<uint32_t>(cell)), sub, s);
    split_start[q] = s;
    inside[q] = in ? 1 : 0;
  }
  return 0;
}
