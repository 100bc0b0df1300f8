// Host-side count for profiles/lik_pm_anatomy.py: the candidate count that nnf_lookup gives every (particle, scan point)
// eval of the likelihood model, through the NN field that tests/hostsim/hostsim.cpp builds the way the engine does.
#include "../tests/hostsim/hostsim.cpp"

// count[p * n_lik + j]: candidates of particle p's eval of scan point j (-1: overflow cell).  Returns -1 without a field.
extern "C" int lik_pm_counts(const mcl3dl_point* map, size_t n, const mcl3dl_lik_params* lp, const mcl3dl_pose* poses,
                             size_t P, const mcl3dl_point* lik_pts, size_t n_lik, int32_t* count)
{
  HostMap m;
  build(m, map, n, lp, nullptr, 1.0f, 2, 1, 1);
  if (!m.nn.field.dir)
    return -1;
  for (size_t p = 0; p < P; ++p)
  {
    F3 pos;
    Q4 q;
    load_pose(poses + p, pos, q);
    const Q4 rn = qnormalized(q);
    for (size_t j = 0; j < n_lik; ++j)
    {
      F3 v;
      v.x = lik_pts[j].x;
      v.y = lik_pts[j].y;
      v.z = lik_pts[j].z;
      const F3 t = transform_point(rn, pos, v);
      uint32_t s = 0;
      count[p * n_lik + j] = nnf_lookup(m.nn.field, fmul(t.x, m.nn.wx), fmul(t.y, m.nn.wy), fmul(t.z, m.nn.wz), s);
    }
  }
  return 0;
}
