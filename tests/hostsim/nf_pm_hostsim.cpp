// Host model of lik_kernel_nf_pm's point-major mapping and cross-CTA fold (kernels.cuh), warp by warp and lane by lane,
// built from nf_pm_shape / nf_fx_term / nf_pm_word / nf_pm_done of device_funcs.cuh.  TEST INFRASTRUCTURE ONLY
// (tests/test_nf_point_major.py).
#include "cuda_shim.h"

#include <vector>

#include "../../include/mcl3dl_b200.h"
#include "../../mcl_3dl_b200/csrc/device_funcs.cuh"

using namespace mcl3dl;

// shape[6] = {slice, n_slices, fx_shift, arr_bits, cnt_bits, ok} of nf_pm_shape
extern "C" void hostsim_nf_pm_shape(int N, int blocks, int slots, int unit, float match_dist_min, float match_weight,
                                    int* shape)
{
  const NfPmShape s = nf_pm_shape(N, blocks, slots, unit, match_dist_min, match_weight);
  shape[0] = s.slice;
  shape[1] = s.n_slices;
  shape[2] = s.fx_shift;
  shape[3] = s.arr_bits;
  shape[4] = s.cnt_bits;
  shape[5] = s.ok;
}

// One kernel launch over P particles and N points with the shape of nf_pm_shape(N, blocks, slots, unit, r, w).
// contrib[p * N + j]: the float contribution of eval (p, j), NaN when the eval does not count.  The grid's CTAs
// (blocks x n_slices, 256 particles each) run in the order `cta_order`, one after the other: the integer atomics make
// any interleaving equal to some such order.  Writes score / cnt of the particles whose record was stored (written[p] =
// number of stores) and returns the number of accumulators left non-zero.
extern "C" int hostsim_nf_pm_run(int P, int N, int slots, int unit, float r, float w, const float* contrib,
                                 const int* cta_order, float* score, uint32_t* cnt, int* written)
{
  const int groups = (P + 31) / 32, blocks = (groups + 7) / 8;
  const NfPmShape sh = nf_pm_shape(N, blocks, slots, unit, r, w);
  std::vector<unsigned long long> acc(P, 0);
  for (int i = 0; i < blocks * sh.n_slices; ++i)
  {
    const int cta = cta_order[i];
    for (int wp = 0; wp < 8; ++wp)
    {
      const int group = (cta / sh.n_slices) * 8 + wp;
      if (group * 32 >= P)
        continue;
      const int s0 = (cta % sh.n_slices) * sh.slice, s1 = std::min(N, s0 + sh.slice);
      for (int lane = 0; lane < 32; ++lane)
      {
        const int p = group * 32 + lane;
        if (p >= P)
          continue;
        long long sum = 0;
        uint32_t c = 0;
        for (int j0 = s0; j0 < s1; j0 += unit)  // the lane's warp trips, u = 0 .. unit - 1
          for (int j = j0; j < std::min(s1, j0 + unit); ++j)
          {
            const float v = contrib[static_cast<size_t>(p) * N + j];
            if (v == v)
            {
              sum += nf_fx_term(v, sh.fx_shift);
              c++;
            }
          }
        const unsigned long long wd = nf_pm_word(sum, c, sh);
        const unsigned long long v = acc[p] + wd;  // atomicAdd(acc + p, wd) + wd
        acc[p] = v;
        uint32_t n;
        float s;
        if (nf_pm_done(v, sh, n, s))
        {
          acc[p] = 0;
          score[p] = (N == 0) ? 1.0f : s;
          cnt[p] = n;
          written[p]++;
        }
      }
    }
  }
  int dirty = 0;
  for (int p = 0; p < P; ++p) dirty += acc[p] != 0;
  return dirty;
}
