// Host model of the owner table of lik_kernel_nf's candidate scan (kernels.cuh: nf_warp_scan, phase B), lane by lane,
// built from the device helpers in device_funcs.cuh, and the candidate scan run on it.  TEST INFRASTRUCTURE ONLY
// (tests/test_nf_owner_table.py).
#include "cuda_shim.h"

#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/mcl3dl_b200.h"
#include "../../mcl_3dl_b200/csrc/device_funcs.cuh"

using namespace mcl3dl;

namespace
{
int log2_units(int U) { return U == 1 ? 0 : U == 2 ? 1 : U == 4 ? 2 : 3; }

// the shuffle scan of the lanes' candidate totals: lanes in order, a lane's evals u = 0 .. U - 1
int flatten(int U, const int* count, std::vector<int>& base)
{
  base.assign(32 * U, 0);
  int W = 0;
  for (int lane = 0; lane < 32; ++lane)
    for (int u = 0; u < U; ++u)
    {
      base[u * 32 + lane] = W;
      W += std::max(count[u * 32 + lane], 0);
    }
  return W;
}

// The owner table of the pass [lo, hi) as nf_warp_scan builds it, in own[0 .. round_up(hi - lo, 16)): clear, every
// lane's marks, then rounds of 32 lanes x 16 bytes; the warp's shuffle max-scan of the lanes' largest marks is the
// running maximum over the lanes in order.
void owner_table(int U, const int* count, const std::vector<int>& base, int lo, int hi, uint8_t* own)
{
  const int n = hi - lo, n16 = (n + 15) / 16;
  std::fill(own, own + 16 * n16, uint8_t(0));
  for (int lane = 0; lane < 32; ++lane)
    for (int u = 0; u < U; ++u)
    {
      const int m = nnf_owner_mark(lo, hi, base[u * 32 + lane], count[u * 32 + lane]);
      if (m >= 0)
        own[m] = static_cast<uint8_t>(lane * U + u);
    }
  uint32_t carry = 0;
  for (int r0 = 0; r0 < n16; r0 += 32)
  {
    uint4 r[32];
    uint32_t incl[32];
    for (int lane = 0; lane < 32; ++lane)
    {
      const int i = r0 + lane;
      r[lane] = make_uint4(0u, 0u, 0u, 0u);
      if (i < n16)
        std::memcpy(&r[lane], own + 16 * i, 16);
      incl[lane] = std::max(nnf_owner_run_max(r[lane]), carry);
      if (lane > 0)
        incl[lane] = std::max(incl[lane], incl[lane - 1]);
    }
    for (int lane = 0; lane < 32; ++lane)
    {
      const int i = r0 + lane;
      uint32_t run = (lane == 0 ? carry : incl[lane - 1]) * 0x00010001u;
      uint32_t* w = &r[lane].x;
      for (int k = 0; k < 4; ++k) w[k] = nnf_owner_evals(nnf_owner_scan_word(w[k], run), log2_units(U));
      if (i < n16)
        std::memcpy(own + 16 * i, &r[lane], 16);
    }
    carry = incl[31];
  }
}

// the owner table as the kernel filled it before (device_funcs.cuh: nnf_fill_owner)
void owner_table_serial(int U, const int* count, const std::vector<int>& base, int lo, int hi, uint8_t* own)
{
  for (int e = 0; e < 32 * U; ++e) nnf_fill_owner(own, lo, hi, base[e], std::max(count[e], 0), e);
}
}  // namespace

// The candidate scan of tests/hostsim/nf_scan_hostsim.cpp on the table above.  One warp trip of U evals per lane (eval e = u * 32 + lane): count[e] candidates from first[e] (count < 0: overflow
// cell, no candidates here), query q[e].  Slots are processed in passes of `pass_slots`, and within a pass in the order
// `perm` (a permutation of 0 .. pass_slots - 1; slots beyond a short pass are skipped) - any order the lanes' rounds and
// atomics may take.  best[e]: the bits the kernel's atomicMin leaves (r2 to start with).  Returns W.
extern "C" int hostsim_nf_owner_warp_scan(int U, const int* count, const uint32_t* first, const float* q, const float4* cand,
                                    float r2, int pass_slots, const int* perm, float* best)
{
  const int E = 32 * U;
  std::vector<int> base;
  const int W = flatten(U, count, base);
  std::vector<uint32_t> off(E), bits(E);
  for (int e = 0; e < E; ++e)
  {
    off[e] = first[e] - static_cast<uint32_t>(base[e]);
    bits[e] = __float_as_uint(r2);
  }
  std::vector<uint8_t> own((pass_slots + 15) / 16 * 16);
  for (int lo = 0; lo < W; lo += pass_slots)
  {
    const int hi = std::min(W, lo + pass_slots);
    owner_table(U, count, base, lo, hi, own.data());
    for (int i = 0; i < pass_slots; ++i)
    {
      const int k = lo + perm[i];
      if (k >= hi)
        continue;
      const int e = own[k - lo];
      const float4 m = cand[off[e] + static_cast<uint32_t>(k)];
      bits[e] = std::min(bits[e], __float_as_uint(nnf_cand_d2(q[3 * e], q[3 * e + 1], q[3 * e + 2], m)));
    }
  }
  for (int e = 0; e < E; ++e) best[e] = __uint_as_float(bits[e]);
  return W;
}

// The owner tables of every pass of one warp trip, as nf_warp_scan builds them (table) and as the serial fill named the
// owners (serial), pass p at [p * pass_slots, p * pass_slots + pass_slots) of each; bytes beyond a short last pass are
// left alone.  Returns W, or -1 when the output holds fewer than the passes need (max_passes).
extern "C" int hostsim_nf_owner_tables(int U, const int* count, int pass_slots, int max_passes, uint8_t* table,
                                       uint8_t* serial)
{
  std::vector<int> base;
  const int W = flatten(U, count, base);
  if ((W + pass_slots - 1) / pass_slots > max_passes)
    return -1;
  std::vector<uint8_t> own((pass_slots + 15) / 16 * 16);
  for (int lo = 0, p = 0; lo < W; lo += pass_slots, ++p)
  {
    const int hi = std::min(W, lo + pass_slots);
    owner_table(U, count, base, lo, hi, own.data());
    std::copy(own.begin(), own.begin() + (hi - lo), table + static_cast<size_t>(p) * pass_slots);
    owner_table_serial(U, count, base, lo, hi, serial + static_cast<size_t>(p) * pass_slots);
  }
  return W;
}

// nnf_owner_scan_word over n words in slot order from the running maximum `run0` (0 .. 255), without the ordinal to
// eval step: out[i] = the scanned bytes of words[i]
extern "C" void hostsim_nf_owner_scan_words(const uint32_t* words, int n, uint32_t run0, uint32_t* out)
{
  uint32_t run = run0 * 0x00010001u;
  for (int i = 0; i < n; ++i) out[i] = nnf_owner_scan_word(words[i], run);
}
