// accum_host_standin.cpp — a STAND-IN for the host work the node does per update before mcl3dl_scan_prepare when it
// builds the cloud itself (src/mcl_3dl.cpp:274-342), for profiles/scan_accum_timing.py.  PCL and tf2 are not part of
// this project's build, so their steps are restated here, each as one pass of the same shape:
//   per cloud: tf2::doTransform (copy the PointCloud2, transform x / y / z of every point in the copy),
//              mcl_3dl::fromROSMsg (PointCloud2 -> pcl::PointCloud<PointXYZ> -> copyPointCloud into 32-byte PointXYZIL),
//              the label loop, pc_local_accum_ += (append);
//   measure(): pcl::transformPointCloud of the accumulation in place, then the adapter's pack into 16-byte
//              mcl3dl_point for the upload.
// The real libraries may be faster or slower than these loops; the figure says what order of work moves off the
// node's thread, not what PCL costs.
//
//   g++ -O2 -std=c++17 accum_host_standin.cpp -o standin && ./standin <clouds> <points per cloud> <point_step> <reps>
// prints: median_ms min_ms max_ms
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace
{
struct XYZ
{
  float x, y, z, pad;
};
struct XYZIL  // mcl_3dl::PointXYZIL, 32 B
{
  float x, y, z, pad;
  float intensity;
  uint32_t label;
  float pad2[2];
};
struct Pt16
{
  float x, y, z;
  uint32_t label;
};
struct Xf
{
  float r[9], t[3];
};

Xf make_xf(const double t[3], const double q[4])
{
  const float x = static_cast<float>(q[0]), y = static_cast<float>(q[1]), z = static_cast<float>(q[2]), w = static_cast<float>(q[3]);
  const float tx = 2 * x, ty = 2 * y, tz = 2 * z, twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x,
              tyy = ty * y, tyz = tz * y, tzz = tz * z;
  return Xf{{1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1 - (txx + tyy)},
            {static_cast<float>(t[0]), static_cast<float>(t[1]), static_cast<float>(t[2])}};
}

inline void apply(const Xf& m, float& x, float& y, float& z)
{
  const float a = ((m.r[0] * x + m.r[1] * y) + m.r[2] * z) + m.t[0];
  const float b = ((m.r[3] * x + m.r[4] * y) + m.r[5] * z) + m.t[1];
  const float c = ((m.r[6] * x + m.r[7] * y) + m.r[8] * z) + m.t[2];
  x = a;
  y = b;
  z = c;
}
}  // namespace

int main(int argc, char** argv)
{
  if (argc < 5)
    return 2;
  const int clouds = std::atoi(argv[1]);
  const size_t n = std::strtoull(argv[2], nullptr, 10);
  const uint32_t ps = static_cast<uint32_t>(std::atoi(argv[3]));
  const int reps = std::atoi(argv[4]);
  std::vector<std::vector<unsigned char>> msgs(clouds, std::vector<unsigned char>(n * ps));
  uint32_t seed = 1;
  for (auto& m : msgs)
    for (size_t i = 0; i < n; ++i)
      for (int k = 0; k < 3; ++k)
      {
        seed = seed * 1664525u + 1013904223u;
        const float v = (static_cast<float>(seed >> 8) / 16777216.0f - 0.5f) * 40.0f;
        std::memcpy(m.data() + i * ps + 4 * k, &v, 4);
      }
  const double t[3] = {0.3, -0.2, 0.1}, q[4] = {0.01, 0.02, 0.3, 0.95};
  std::vector<double> ms;
  double sink = 0;
  for (int rep = 0; rep < reps + 3; ++rep)
  {
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<XYZIL> accum;
    for (int k = 0; k < clouds; ++k)
    {
      std::vector<unsigned char> bl(msgs[k]);  // doTransform: the output message is a copy
      const Xf m = make_xf(t, q);
      for (size_t i = 0; i < n; ++i)
      {
        float p[3];
        std::memcpy(p, bl.data() + i * ps, 12);
        apply(m, p[0], p[1], p[2]);
        std::memcpy(bl.data() + i * ps, p, 12);
      }
      std::vector<XYZ> raw(n);  // pcl::fromROSMsg
      for (size_t i = 0; i < n; ++i)
      {
        std::memcpy(&raw[i], bl.data() + i * ps, 12);
        raw[i].pad = 1.0f;
      }
      std::vector<XYZIL> tmp(n);  // copyPointCloud
      for (size_t i = 0; i < n; ++i)
      {
        tmp[i] = XYZIL{};
        tmp[i].x = raw[i].x;
        tmp[i].y = raw[i].y;
        tmp[i].z = raw[i].z;
      }
      for (auto& p : tmp) p.label = static_cast<uint32_t>(k);
      accum.insert(accum.end(), tmp.begin(), tmp.end());  // pc_local_accum_ += *pc_tmp
    }
    const Xf m2 = make_xf(t, q);  // measure(): transformPointCloud in place (dense)
    for (auto& p : accum) apply(m2, p.x, p.y, p.z);
    std::vector<Pt16> packed;  // the adapter's pack for the upload
    packed.reserve(accum.size());
    for (const auto& p : accum) packed.push_back(Pt16{p.x, p.y, p.z, p.label});
    const auto t1 = std::chrono::steady_clock::now();
    sink += packed[packed.size() / 2].x;
    if (rep >= 3)
      ms.push_back(std::chrono::duration<double, std::milli>(t1 - t0).count());
  }
  std::sort(ms.begin(), ms.end());
  std::printf("%.3f %.3f %.3f\n", ms[ms.size() / 2], ms.front(), ms.back());
  std::fprintf(stderr, "%g\n", sink);
  return 0;
}
