// normal_eigen.h — TEST INFRASTRUCTURE ONLY: the normal-weighted sampler checkers' shared numerics, repo-written.
//   oracle_sym3_eigen: a symmetric 3 x 3 double eigendecomposition (cyclic Jacobi to convergence, eigenvalues ascending,
//                      eigenvectors as unit columns).  The port's setParticleStatistics and the reference tier's
//                      SelfAdjointEigenSolver stand-in (shim_ns/Eigen/Eigenvalues) both call it, so the two agree bit
//                      for bit; it is not Eigen.
//   oracle_normals:    pcl::NormalEstimation restated by brute force: every finite point within radius r of a finite
//                      query (flann::L2_Simple d2 < float(r * r), the query included, ascending index), count / sum d /
//                      sum d d^T in double relative to the query, C = S / n - m m^T, the eigenvector of the smallest
//                      eigenvalue as float; fewer than 3 neighbours or a non-finite query: NaN.  The port and the
//                      reference tier's pcl::NormalEstimation stand-in (shim_ns/pcl/features/normal_3d.h) call it.
#ifndef ORACLE_NORMAL_EIGEN_H
#define ORACLE_NORMAL_EIGEN_H
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <limits>

namespace oracle_ns
{
// a: row-major symmetric (both triangles read as given: a[r * 3 + c] for c <= r); vals ascending, vecs row-major with
// the eigenvectors as columns
inline void sym3_eigen(const double in[9], double vals[3], double vecs[9])
{
  double a[3][3], v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c <= r; ++c) a[r][c] = a[c][r] = in[r * 3 + c];
  for (int sweep = 0; sweep < 64; ++sweep)
  {
    if (a[0][1] == 0.0 && a[0][2] == 0.0 && a[1][2] == 0.0)
      break;
    for (int p = 0; p < 3; ++p)
      for (int q = p + 1; q < 3; ++q)
      {
        if (a[p][q] == 0.0)
          continue;
        const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
        double t = 1.0 / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        if (theta < 0.0)
          t = -t;
        const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
        const double app = a[p][p] - t * a[p][q], aqq = a[q][q] + t * a[p][q];
        const int r = 3 - p - q;
        const double arp = a[r][p], arq = a[r][q];
        a[p][p] = app;
        a[q][q] = aqq;
        a[p][q] = a[q][p] = 0.0;
        a[r][p] = a[p][r] = c * arp - s * arq;
        a[r][q] = a[q][r] = s * arp + c * arq;
        for (int k = 0; k < 3; ++k)
        {
          const double vp = v[k][p], vq = v[k][q];
          v[k][p] = c * vp - s * vq;
          v[k][q] = s * vp + c * vq;
        }
      }
  }
  int order[3] = {0, 1, 2};
  std::stable_sort(order, order + 3, [&](int x, int y) { return a[x][x] < a[y][y]; });
  for (int j = 0; j < 3; ++j)
  {
    const int src = order[j];
    vals[j] = a[src][src];
    const double len = std::sqrt(v[0][src] * v[0][src] + v[1][src] * v[1][src] + v[2][src] * v[2][src]);
    for (int r = 0; r < 3; ++r) vecs[r * 3 + j] = v[r][src] / len;
  }
}

inline bool finite3(const float* p) { return std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]); }

// xyz: point i at xyz + i * stride (floats); normals [n * 3]; counts [n] (may be null)
inline void normals(const float* xyz, size_t stride, size_t n, double r, float* out, uint32_t* counts)
{
  const float r2 = static_cast<float>(r * r);
  const float nan = std::numeric_limits<float>::quiet_NaN();
  for (size_t i = 0; i < n; ++i)
  {
    const float* q = xyz + i * stride;
    out[3 * i] = out[3 * i + 1] = out[3 * i + 2] = nan;
    uint32_t cnt = 0;
    if (finite3(q))
    {
      double s[3] = {0, 0, 0}, ss[6] = {0, 0, 0, 0, 0, 0};
      for (size_t j = 0; j < n; ++j)
      {
        const float* p = xyz + j * stride;
        if (!finite3(p))
          continue;
        const float dx = q[0] - p[0], dy = q[1] - p[1], dz = q[2] - p[2];
        const float d2 = dx * dx + dy * dy + dz * dz;
        if (!(d2 < r2))
          continue;
        ++cnt;
        const double e[3] = {static_cast<double>(p[0]) - q[0], static_cast<double>(p[1]) - q[1], static_cast<double>(p[2]) - q[2]};
        for (int k = 0; k < 3; ++k) s[k] += e[k];
        ss[0] += e[0] * e[0];
        ss[1] += e[1] * e[1];
        ss[2] += e[2] * e[2];
        ss[3] += e[0] * e[1];
        ss[4] += e[0] * e[2];
        ss[5] += e[1] * e[2];
      }
      if (cnt >= 3)
      {
        const double fn = cnt, m[3] = {s[0] / fn, s[1] / fn, s[2] / fn};
        const double c9[9] = {ss[0] / fn - m[0] * m[0], ss[3] / fn - m[0] * m[1], ss[4] / fn - m[0] * m[2],
                              ss[3] / fn - m[0] * m[1], ss[1] / fn - m[1] * m[1], ss[5] / fn - m[1] * m[2],
                              ss[4] / fn - m[0] * m[2], ss[5] / fn - m[1] * m[2], ss[2] / fn - m[2] * m[2]};
        double vals[3], vecs[9];
        sym3_eigen(c9, vals, vecs);
        for (int k = 0; k < 3; ++k) out[3 * i + k] = static_cast<float>(vecs[k * 3 + 0]);
      }
    }
    if (counts)
      counts[i] = cnt;
  }
}
}  // namespace oracle_ns
#endif
