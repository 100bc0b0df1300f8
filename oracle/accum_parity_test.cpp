// accum_parity_test.cpp — TEST INFRASTRUCTURE ONLY.
//
// The node's cloud accumulation through the C++ adapter against the node's host path, both driven by the reference's
// own CloudAccumulationLogic (src/cloud_accum.cpp, compiled where it lies against oracle/shim/; make -C oracle -f
// accum.mk accum-parity; tests/test_gpu_scan_accum.py runs it on an H100).  Each push of a message sequence goes to one
// logic object whose callbacks feed both paths:
//   host:    accumCloud restated (src/mcl_3dl.cpp:274-302: the sensor -> odom transform of every point, fromROSMsg's
//            rejections, label = header count, append), measure()'s transform into base_link with pcl::transformPointCloud's
//            not-dense rule (:319-342), then mcl3dl_scan_prepare on that host cloud (its own engine);
//   adapter: MeasurementBatcher::accumulateCloud / clearAccumulated / prepareAccumulated.
// At every accumulate both must accept or both reject; at every process() the five prepared stages (scan_get 0..4) must
// be equal byte for byte and the adapter's cloud count must equal the node's header count.  The sequences: accum_cloud
// 1 and 3, two frame_ids interleaved, the total_accum_cloud_max overflow, and clouds that fail to accumulate (empty, no
// z field) and so clear and reset the logic.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <functional>
#include <limits>
#include <map>
#include <memory>
#include <random>
#include <string>
#include <vector>

#include <mcl_3dl/cloud_accum.h>

#include "../mcl_3dl_b200/host/lidar_measurement_model_b200.h"

using namespace mcl_3dl;

namespace
{
int g_fail = 0;

// Eigen::Quaternion<float>(w, x, y, z).toRotationMatrix(), t = float(translation); ((r0 x + r1 y) + r2 z) + t
struct Xf
{
  float r[9], t[3];
};
Xf makeXf(const mcl3dl_transform& tf)
{
  const float x = static_cast<float>(tf.rotation[0]), y = static_cast<float>(tf.rotation[1]), z = static_cast<float>(tf.rotation[2]),
              w = static_cast<float>(tf.rotation[3]);
  const float tx = 2.0f * x, ty = 2.0f * y, tz = 2.0f * z;
  const float twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
  Xf m{{1.0f - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1.0f - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1.0f - (txx + tyy)},
       {static_cast<float>(tf.translation[0]), static_cast<float>(tf.translation[1]), static_cast<float>(tf.translation[2])}};
  return m;
}
void apply(const Xf& m, float& x, float& y, float& z)
{
  const float a = ((m.r[0] * x + m.r[1] * y) + m.r[2] * z) + m.t[0];
  const float b = ((m.r[3] * x + m.r[4] * y) + m.r[5] * z) + m.t[1];
  const float c = ((m.r[6] * x + m.r[7] * y) + m.r[8] * z) + m.t[2];
  x = a;
  y = b;
  z = c;
}

// the tf lookups of the two paths: sensor -> odom per frame_id, odom -> base_link per measure()
mcl3dl_transform odomFrom(const std::string& frame)
{
  if (frame == "lidar_a")
    return mcl3dl_transform{{0.3, -0.1, 0.4}, {0.01, -0.02, 0.2, 0.98}};
  return mcl3dl_transform{{-0.2, 0.25, 0.35}, {0.0, 0.03, -0.6, 0.8}};
}
mcl3dl_transform baseFromOdom(int k)
{
  const double yaw = 0.05 * k;
  return mcl3dl_transform{{0.05 * k, -0.02, 0.0}, {0.0, 0.0, std::sin(yaw / 2), std::cos(yaw / 2)}};
}

sensor_msgs::PointField field(const char* name, uint32_t offset)
{
  sensor_msgs::PointField f;
  f.name = name;
  f.offset = offset;
  f.datatype = sensor_msgs::PointField::FLOAT32;
  f.count = 1;
  return f;
}

// A cloud of n points (width x height) around the sensor, in one of three layouts; `nan_every` > 0 puts NaN / inf points
// in (and marks the cloud not dense).
sensor_msgs::PointCloud2::ConstPtr makeCloud(std::mt19937& rng, const std::string& frame, uint32_t width, uint32_t height, int layout,
                                            int nan_every = 0, bool with_z = true)
{
  auto msg = std::make_shared<sensor_msgs::PointCloud2>();
  msg->header.frame_id = frame;
  msg->width = width;
  msg->height = height;
  uint32_t off[3];
  if (layout == 0)
  {
    msg->point_step = 16;  // x y z intensity
    off[0] = 0, off[1] = 4, off[2] = 8;
    msg->fields = {field("x", 0), field("y", 4), field("z", 8), field("intensity", 12)};
  }
  else if (layout == 1)
  {
    msg->point_step = 32;  // intensity, ring, then z y x
    off[0] = 24, off[1] = 20, off[2] = 16;
    msg->fields = {field("intensity", 0), field("z", 16), field("y", 20), field("x", 24)};
  }
  else
  {
    msg->point_step = 48;
    off[0] = 4, off[1] = 12, off[2] = 40;
    msg->fields = {field("x", 4), field("y", 12), field("label", 20), field("z", 40)};
  }
  if (!with_z)
    msg->fields.erase(std::remove_if(msg->fields.begin(), msg->fields.end(), [](const sensor_msgs::PointField& f) { return f.name == "z"; }),
                      msg->fields.end());
  msg->row_step = width * msg->point_step + 8 * (layout == 1);  // padded rows for one layout
  msg->data.assign(static_cast<size_t>(msg->row_step) * height, 0xA5);
  msg->is_dense = nan_every == 0;
  std::normal_distribution<float> nd(0.0f, 2.5f);
  uint32_t i = 0;
  for (uint32_t r = 0; r < height; ++r)
    for (uint32_t c = 0; c < width; ++c, ++i)
    {
      float p[3] = {nd(rng), nd(rng), 0.3f * nd(rng)};
      if (nan_every && i % nan_every == 0)
        p[i % 3] = (i / nan_every) % 2 ? std::numeric_limits<float>::quiet_NaN() : std::numeric_limits<float>::infinity();
      for (int k = 0; k < 3; ++k)
        std::memcpy(msg->data.data() + static_cast<size_t>(r) * msg->row_step + static_cast<size_t>(c) * msg->point_step + off[k], &p[k], 4);
    }
  return msg;
}

// The node's host path (restated) and the adapter, fed by the same logic object.
class Pair
{
public:
  Pair()
    : batcher_(nullptr, std::vector<int>{0}, std::make_shared<LidarMeasurementModelLikelihoodParameters>(),
               std::make_shared<LidarMeasurementModelBeamParameters>(), nullptr)
  {
    if (mcl3dl_create(&host_engine_, nullptr, 1) != MCL3DL_OK)
    {
      std::fprintf(stderr, "mcl3dl_create failed\n");
      std::exit(2);
    }
    clear();
  }
  ~Pair() { mcl3dl_destroy(host_engine_); }

  // accumCloud
  bool accumulate(const sensor_msgs::PointCloud2::ConstPtr& msg)
  {
    const bool a = hostAccumulate(*msg);
    const bool b = batcher_.accumulateCloud(*msg, odomFrom(msg->header.frame_id));
    if (a != b)
    {
      std::fprintf(stderr, "[%s] accumulate: host %d adapter %d\n", tag_.c_str(), a, b);
      ++g_fail;
    }
    ++accumulates_;
    return a;
  }
  // accumClear
  void clear()
  {
    accum_.clear();
    dense_ = true;
    headers_.clear();
    batcher_.clearAccumulated();
    ++clears_;
  }
  // measure()
  void process()
  {
    ++processes_;
    if (headers_.empty())
    {
      std::fprintf(stderr, "[%s] process() without a cloud\n", tag_.c_str());
      ++g_fail;
      return;
    }
    if (batcher_.accumulatedClouds() != headers_.size())
    {
      std::fprintf(stderr, "[%s] process %d: adapter %u clouds, node %zu headers\n", tag_.c_str(), processes_,
                   batcher_.accumulatedClouds(), headers_.size());
      ++g_fail;
    }
    const mcl3dl_transform base = baseFromOdom(processes_);
    mcl3dl_scan_params sp{};
    sp.downsample[0] = 0.1f;
    sp.downsample[1] = 0.1f;
    sp.downsample[2] = 0.05f;
    sp.lik_clip_near = 0.5f, sp.lik_clip_far = 10.0f, sp.lik_clip_z_min = -2.0f, sp.lik_clip_z_max = 2.0f;
    sp.beam_clip_near = 0.5f, sp.beam_clip_far = 4.0f, sp.beam_clip_z_min = -2.0f, sp.beam_clip_z_max = 2.0f;
    sp.lik_num_points = 96;
    sp.beam_num_points = 3;
    sp.seed = 1000 + processes_;
    // host: pcl::transformPointCloud of the accumulation (in place, as the node does), then scan_prepare
    std::vector<mcl3dl_point> cloud = accum_;
    const Xf m = makeXf(base);
    for (auto& p : cloud)
      if (dense_ || (std::isfinite(p.x) && std::isfinite(p.y) && std::isfinite(p.z)))
        apply(m, p.x, p.y, p.z);
    mcl3dl_scan_info hi{}, ai{};
    check(mcl3dl_scan_prepare(host_engine_, cloud.data(), cloud.size(), &sp, &hi), "mcl3dl_scan_prepare");
    batcher_.prepareAccumulated(base, sp, &ai);
    if (std::memcmp(&hi, &ai, sizeof(hi)) != 0)
    {
      std::fprintf(stderr, "[%s] process %d: info differs (raw %u / %u, downsampled %u / %u)\n", tag_.c_str(), processes_, hi.n_raw,
                   ai.n_raw, hi.n_downsampled, ai.n_downsampled);
      ++g_fail;
    }
    for (int w = 0; w < 5; ++w)
    {
      const std::vector<mcl3dl_point> a = stage(host_engine_, w), b = stage(batcher_.engine(), w);
      if (a.size() != b.size() || (!a.empty() && std::memcmp(a.data(), b.data(), a.size() * sizeof(mcl3dl_point)) != 0))
      {
        std::fprintf(stderr, "[%s] process %d: stage %d differs (%zu / %zu points)\n", tag_.c_str(), processes_, w, a.size(), b.size());
        ++g_fail;
      }
    }
    if (hi.n_raw != accum_.size() || hi.n_downsampled == 0)
    {
      std::fprintf(stderr, "[%s] process %d: %u raw points, %u downsampled\n", tag_.c_str(), processes_, hi.n_raw, hi.n_downsampled);
      ++g_fail;
    }
    clouds_per_process_.push_back(headers_.size());
  }

  void push(CloudAccumulationLogicBase& logic, const sensor_msgs::PointCloud2::ConstPtr& msg)
  {
    logic.push(msg->header.frame_id, msg, std::bind(&Pair::process, this), std::bind(&Pair::accumulate, this, std::placeholders::_1),
               std::bind(&Pair::clear, this));
  }
  void setTag(const std::string& t) { tag_ = t; }
  const std::vector<size_t>& cloudsPerProcess() const { return clouds_per_process_; }
  void resetCounts()
  {
    clouds_per_process_.clear();
    accumulates_ = clears_ = 0;
  }
  int clears() const { return clears_; }

private:
  // accumCloud restated: fromROSMsg's rejections (no x / y / z field, an empty cloud), the transform of every point,
  // label = the header count, append
  bool hostAccumulate(const sensor_msgs::PointCloud2& msg)
  {
    uint32_t off[3];
    const char* names[3] = {"x", "y", "z"};
    for (int k = 0; k < 3; ++k)
    {
      bool found = false;
      for (const auto& f : msg.fields)
        if (f.name == names[k])
        {
          off[k] = f.offset;
          found = true;
        }
      if (!found)
        return false;
    }
    if (msg.width * msg.height == 0)
      return false;
    const Xf m = makeXf(odomFrom(msg.header.frame_id));
    for (uint32_t r = 0; r < msg.height; ++r)
      for (uint32_t c = 0; c < msg.width; ++c)
      {
        float p[3];
        for (int k = 0; k < 3; ++k)
          std::memcpy(&p[k], msg.data.data() + static_cast<size_t>(r) * msg.row_step + static_cast<size_t>(c) * msg.point_step + off[k], 4);
        apply(m, p[0], p[1], p[2]);
        accum_.push_back(mcl3dl_point{p[0], p[1], p[2], static_cast<uint32_t>(headers_.size())});
      }
    dense_ = dense_ && msg.is_dense;
    headers_.push_back(msg.header);
    return true;
  }
  static std::vector<mcl3dl_point> stage(mcl3dl_engine* eng, int which)
  {
    size_t n = 0;
    check(mcl3dl_scan_get(eng, which, nullptr, 0, &n), "mcl3dl_scan_get");
    std::vector<mcl3dl_point> out(n);
    if (n)
      check(mcl3dl_scan_get(eng, which, out.data(), n, &n), "mcl3dl_scan_get");
    return out;
  }
  static void check(int rc, const char* what)
  {
    if (rc != MCL3DL_OK)
    {
      std::fprintf(stderr, "%s: %s\n", what, mcl3dl_strerror(rc));
      std::exit(2);
    }
  }

  mcl_3dl_b200::MeasurementBatcher batcher_;
  mcl3dl_engine* host_engine_ = nullptr;
  std::vector<mcl3dl_point> accum_;
  bool dense_ = true;
  std::vector<std_msgs::Header> headers_;
  std::vector<size_t> clouds_per_process_;
  int processes_ = 0, accumulates_ = 0, clears_ = 0;
  std::string tag_;
};

void expect(const char* tag, const std::vector<size_t>& got, const std::vector<size_t>& want)
{
  if (got != want)
  {
    std::fprintf(stderr, "[%s] clouds per process:", tag);
    for (size_t v : got) std::fprintf(stderr, " %zu", v);
    std::fprintf(stderr, " (want");
    for (size_t v : want) std::fprintf(stderr, " %zu", v);
    std::fprintf(stderr, ")\n");
    ++g_fail;
  }
}
}  // namespace

int main()
{
  std::mt19937 rng(5);
  Pair pair;
  // accum_cloud 1: every cloud after the first processes the one before (src/cloud_accum.cpp:91-118)
  {
    pair.setTag("accum 1");
    pair.resetCounts();
    CloudAccumulationLogic logic(1, 10);
    for (int i = 0; i < 4; ++i) pair.push(logic, makeCloud(rng, "lidar_a", 3000, 1, i % 3));
    expect("accum 1", pair.cloudsPerProcess(), {1, 1, 1});
    logic.reset();
    pair.clear();
  }
  // accum_cloud 3, two frame_ids interleaved: the front key's clouds are counted, the others ride along
  {
    pair.setTag("accum 3 interleaved");
    pair.resetCounts();
    CloudAccumulationLogic logic(3, 10);
    const char* frames[] = {"lidar_a", "lidar_b"};
    for (int i = 0; i < 13; ++i)
      pair.push(logic, makeCloud(rng, frames[i % 2], 1200 + 100 * (i % 3), i % 4 == 3 ? 2 : 1, i % 3, i == 5 ? 37 : 0));
    expect("accum 3 interleaved", pair.cloudsPerProcess(), {6, 6});
    logic.reset();
    pair.clear();
  }
  // total_accum_cloud_max: only the second frame keeps arriving, so the front key's count never fills and the limit
  // forces the process (:108-114); the next accumulation starts with that frame in front
  {
    pair.setTag("overflow");
    pair.resetCounts();
    CloudAccumulationLogic logic(3, 4);
    pair.push(logic, makeCloud(rng, "lidar_a", 2000, 1, 0));
    for (int i = 0; i < 8; ++i) pair.push(logic, makeCloud(rng, "lidar_b", 1500, 1, (i + 1) % 3));
    expect("overflow", pair.cloudsPerProcess(), {4, 3});  // the limit, then accum_cloud of the new front
    logic.reset();
    pair.clear();
  }
  // clouds that fail to accumulate (empty; no z field): the logic clears and resets (:69-73, :83-87), both paths agree
  {
    pair.setTag("failures");
    pair.resetCounts();
    CloudAccumulationLogic logic(3, 10);
    pair.push(logic, makeCloud(rng, "lidar_a", 2000, 1, 0));
    pair.push(logic, makeCloud(rng, "lidar_a", 2000, 1, 1));
    const int clears_before = pair.clears();
    pair.push(logic, makeCloud(rng, "lidar_a", 0, 1, 2));  // empty: "Given PointCloud2 is empty"
    if (pair.clears() != clears_before + 1)
    {
      std::fprintf(stderr, "[failures] the empty cloud did not clear\n");
      ++g_fail;
    }
    for (int i = 0; i < 4; ++i) pair.push(logic, makeCloud(rng, "lidar_a", 1800, 1, i % 3));
    pair.push(logic, makeCloud(rng, "lidar_a", 1800, 1, 0, 0, false));  // no z field
    for (int i = 0; i < 5; ++i) pair.push(logic, makeCloud(rng, "lidar_a", 1700, 2, i % 3, i == 2 ? 11 : 0));
    expect("failures", pair.cloudsPerProcess(), {3, 3});
    logic.reset();
    pair.clear();
  }
  if (g_fail)
  {
    std::fprintf(stderr, "ACCUM PARITY FAILED (%d)\n", g_fail);
    return 1;
  }
  std::printf("accum parity ok\n");
  return 0;
}
