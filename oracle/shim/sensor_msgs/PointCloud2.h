// TEST INFRASTRUCTURE ONLY (oracle/_ref build): stand-in for sensor_msgs/PointCloud2 (and the std_msgs/Header it
// carries) with the members the node's cloud path and the C++ adapter's accumulateCloud read: header, width, height,
// fields {name, offset, datatype, count}, is_bigendian, point_step, row_step, data, is_dense, and ConstPtr.
#ifndef ORACLE_SHIM_SENSOR_MSGS_POINTCLOUD2_H
#define ORACLE_SHIM_SENSOR_MSGS_POINTCLOUD2_H
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

namespace std_msgs
{
struct Header
{
  uint32_t seq = 0;
  uint64_t stamp = 0;  // ros::Time in ROS; nanoseconds here
  std::string frame_id;
};
}  // namespace std_msgs

namespace sensor_msgs
{
struct PointField
{
  enum : uint8_t
  {
    INT8 = 1,
    UINT8 = 2,
    INT16 = 3,
    UINT16 = 4,
    INT32 = 5,
    UINT32 = 6,
    FLOAT32 = 7,
    FLOAT64 = 8
  };
  std::string name;
  uint32_t offset = 0;
  uint8_t datatype = 0;
  uint32_t count = 0;
};

struct PointCloud2
{
  using Ptr = std::shared_ptr<PointCloud2>;
  using ConstPtr = std::shared_ptr<const PointCloud2>;
  std_msgs::Header header;
  uint32_t height = 0, width = 0;
  std::vector<PointField> fields;
  uint8_t is_bigendian = 0;
  uint32_t point_step = 0, row_step = 0;
  std::vector<uint8_t> data;
  uint8_t is_dense = 0;
};
}  // namespace sensor_msgs
#endif
