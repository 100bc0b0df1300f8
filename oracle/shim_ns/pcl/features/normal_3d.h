// TEST INFRASTRUCTURE ONLY (oracle/_ref: the normal-weighted sampler's reference tier): NOT PCL.  pcl::Normal,
// pcl::search::KdTree (a tag: the estimation below searches by brute force) and pcl::NormalEstimation whose compute()
// calls oracle/normal_eigen.h's normals, the port's own normal code, at the radius set by setRadiusSearch.
#ifndef ORACLE_SHIM_NS_PCL_NORMAL_3D_H
#define ORACLE_SHIM_NS_PCL_NORMAL_3D_H
#include <memory>
#include <vector>

#include <pcl/point_cloud.h>
#include <pcl/point_types.h>

#include "../../../normal_eigen.h"

namespace pcl
{
struct Normal
{
  float normal_x, normal_y, normal_z, curvature;
};
namespace search
{
template <typename PointT>
class KdTree
{
public:
  using Ptr = std::shared_ptr<KdTree<PointT>>;
};
}  // namespace search

template <typename PointInT, typename PointOutT>
class NormalEstimation
{
public:
  void setInputCloud(const typename PointCloud<PointInT>::ConstPtr& cloud) { cloud_ = cloud; }
  void setSearchMethod(const typename search::KdTree<PointInT>::Ptr&) {}
  void setRadiusSearch(double r) { r_ = r; }
  void compute(PointCloud<PointOutT>& out) const
  {
    const size_t n = cloud_->size();
    std::vector<float> xyz(3 * n), nrm(3 * n);
    for (size_t i = 0; i < n; ++i)
    {
      xyz[3 * i] = cloud_->points[i].x;
      xyz[3 * i + 1] = cloud_->points[i].y;
      xyz[3 * i + 2] = cloud_->points[i].z;
    }
    oracle_ns::normals(xyz.data(), 3, n, r_, nrm.data(), nullptr);
    out.points.resize(n);
    for (size_t i = 0; i < n; ++i) out.points[i] = PointOutT{nrm[3 * i], nrm[3 * i + 1], nrm[3 * i + 2], 0.0f};
    out.width = static_cast<uint32_t>(n);
    out.height = 1;
  }

private:
  typename PointCloud<PointInT>::ConstPtr cloud_;
  double r_ = 0.0;
};
}  // namespace pcl
#endif
