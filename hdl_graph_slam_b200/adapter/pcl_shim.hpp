// pcl_shim.hpp — TEST-ONLY stand-in for the handful of PCL / Eigen declarations b200_registration.hpp and b200_backend.hpp touch, so
// the adapters can be syntax-checked in an image without PCL (tests/test_adapter_syntax.py).  Signatures follow PCL 1.10
// (the distro package of ROS noetic, /root/reference/docker/noetic/Dockerfile:6).  Nothing here is shipped or linked.
#pragma once
#include <cstdint>
#include <limits>
#include <memory>
#include <string>
#include <vector>

namespace Eigen {
struct Matrix4f {
  float m[16];
  float* data() { return m; }
  const float* data() const { return m; }
  static Matrix4f Identity() {
    Matrix4f I{};
    for (int i = 0; i < 4; i++) I.m[i * 5] = 1.f;
    return I;
  }
};
}  // namespace Eigen

namespace pcl {
struct alignas(16) PointXYZI {
  float x, y, z, _pad;
  float intensity;
  float _pad2[3];
};
static_assert(sizeof(PointXYZI) == 32, "pcl::PointXYZI is a 32-byte record");

// pcl::PCLHeader: stamp in microseconds, as pcl_conversions::toPCL writes it
struct PCLHeader {
  uint32_t seq = 0;
  uint64_t stamp = 0;
  std::string frame_id;
};

template <typename PointT>
struct PointCloud {
  PCLHeader header;
  std::vector<PointT> points;
  uint32_t width = 0, height = 0;
  bool is_dense = true;
  size_t size() const { return points.size(); }
  using Ptr = std::shared_ptr<PointCloud<PointT>>;
  using ConstPtr = std::shared_ptr<const PointCloud<PointT>>;
};

namespace search {
template <typename PointT>
class Search {
public:
  using Ptr = std::shared_ptr<Search<PointT>>;
  using PointCloudConstPtr = typename PointCloud<PointT>::ConstPtr;
  using IndicesConstPtr = std::shared_ptr<const std::vector<int>>;
  explicit Search(const std::string& name = "", bool sorted = false) : name_(name), sorted_(sorted) {}
  virtual ~Search() {}
  virtual void setInputCloud(const PointCloudConstPtr&, const IndicesConstPtr& = IndicesConstPtr()) {}
  virtual int nearestKSearch(const PointT&, int, std::vector<int>&, std::vector<float>&) const = 0;
  virtual int radiusSearch(const PointT&, double, std::vector<int>&, std::vector<float>&, unsigned int = 0) const = 0;

protected:
  std::string name_;
  bool sorted_;
};
}  // namespace search

template <typename PointT>
void transformPointCloud(const PointCloud<PointT>& in, PointCloud<PointT>& out, const Eigen::Matrix4f& T);

template <typename PointSource, typename PointTarget, typename Scalar = float>
class Registration {
public:
  using Matrix4 = Eigen::Matrix4f;
  using PointCloudSource = PointCloud<PointSource>;
  using PointCloudSourceConstPtr = typename PointCloudSource::ConstPtr;
  using PointCloudTarget = PointCloud<PointTarget>;
  using PointCloudTargetConstPtr = typename PointCloudTarget::ConstPtr;
  using KdTreePtr = typename search::Search<PointTarget>::Ptr;
  using Ptr = std::shared_ptr<Registration<PointSource, PointTarget, Scalar>>;
  virtual ~Registration() {}
  virtual void setInputSource(const PointCloudSourceConstPtr& cloud) { input_ = cloud; }
  virtual void setInputTarget(const PointCloudTargetConstPtr& cloud) { target_ = cloud; target_cloud_updated_ = true; }
  void setSearchMethodTarget(const KdTreePtr& tree, bool force_no_recompute = false) { tree_ = tree; force_no_recompute_ = force_no_recompute; }
  KdTreePtr getSearchMethodTarget() const { return tree_; }
  bool hasConverged() const { return converged_; }
  Matrix4 getFinalTransformation() { return final_transformation_; }
  // pcl::Registration::getFitnessScore(max_range) as documented: the source transformed by the final transformation, one
  // nearestKSearch(p, 1) per point in order, the mean of the squared distances that are <= max_range, DBL_MAX when there is none.
  // NOT virtual, as in PCL: both reference callers reach it through the base pointer.
  double getFitnessScore(double max_range = std::numeric_limits<double>::max()) {
    double fitness_score = 0.0;
    PointCloudSource input_transformed;
    transformPointCloud(*input_, input_transformed, final_transformation_);
    std::vector<int> nn_indices(1);
    std::vector<float> nn_dists(1);
    int nr = 0;
    for (size_t i = 0; i < input_transformed.points.size(); ++i) {
      tree_->nearestKSearch(input_transformed.points[i], 1, nn_indices, nn_dists);
      if (nn_dists[0] <= max_range) {
        fitness_score += nn_dists[0];
        nr++;
      }
    }
    return nr > 0 ? fitness_score / nr : std::numeric_limits<double>::max();
  }
  void align(PointCloudSource& output, const Matrix4& guess) {
    output.points = input_->points;
    converged_ = false;
    computeTransformation(output, guess);
  }

protected:
  virtual void computeTransformation(PointCloudSource& output, const Matrix4& guess) = 0;
  std::string reg_name_;
  KdTreePtr tree_;
  PointCloudSourceConstPtr input_;
  PointCloudTargetConstPtr target_;
  int nr_iterations_ = 0, max_iterations_ = 10;
  Matrix4 final_transformation_ = Matrix4::Identity(), transformation_ = Matrix4::Identity(), previous_transformation_ = Matrix4::Identity();
  double transformation_epsilon_ = 0, corr_dist_threshold_ = 0;
  bool converged_ = false, target_cloud_updated_ = true, force_no_recompute_ = false;
};
// stand-in for pcl::transformPointCloud (pcl/common/transforms.h); column-major 4x4 like Eigen
template <typename PointT>
inline void transformPointCloud(const PointCloud<PointT>& in, PointCloud<PointT>& out, const Eigen::Matrix4f& T) {
  out.points = in.points;
  for (auto& p : out.points) {
    const float x = p.x, y = p.y, z = p.z;
    p.x = T.m[0] * x + T.m[4] * y + T.m[8] * z + T.m[12];
    p.y = T.m[1] * x + T.m[5] * y + T.m[9] * z + T.m[13];
    p.z = T.m[2] * x + T.m[6] * y + T.m[10] * z + T.m[14];
  }
}
}  // namespace pcl
