// TEST INFRASTRUCTURE ONLY (oracle/_ref: the normal-weighted sampler's reference tier): oracle/shim's ROS stand-in plus
// ros::WallTime, which PointCloudSamplerWithNormal::sample reads for its debug log.
#ifndef ORACLE_SHIM_NS_ROS_H
#define ORACLE_SHIM_NS_ROS_H
#include <chrono>

#include "../../shim/ros/ros.h"

namespace ros
{
class WallDuration
{
public:
  explicit WallDuration(double s) : sec_(s) {}
  double toSec() const { return sec_; }

private:
  double sec_;
};
class WallTime
{
public:
  static WallTime now()
  {
    WallTime t;
    t.sec_ = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
    return t;
  }
  WallDuration operator-(const WallTime& o) const { return WallDuration(sec_ - o.sec_); }

private:
  double sec_ = 0.0;
};
}  // namespace ros
#endif
