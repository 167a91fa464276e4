// b200_registration.hpp — the pcl::Registration adapter a maintainer of koide3/hdl_graph_slam adds to use libb200reg.so.
//
// It derives from pcl::Registration<PointT, PointT>, so the object returned by select_registration_method()
// (/root/reference/src/hdl_graph_slam/registrations.cpp:22-124) keeps its type and every caller stays untouched:
//   ScanMatchingOdometryNodelet  apps/scan_matching_odometry_nodelet.cpp:172,177,210,214,220,246,307,316
//   LoopDetector                 include/hdl_graph_slam/loop_detector.hpp:122,136,143,146,147,153
// Compiled only where PCL/Eigen exist (not in this repository's image; tests/test_adapter_syntax.py checks it against
// adapter/pcl_shim.hpp, a 1-to-1 stand-in for the few PCL/Eigen declarations used here).  See INTEGRATION.md.
#pragma once
#include <b200reg.h>
#include <limits>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

namespace hdl_graph_slam {

template <typename PointT>
class B200Registration : public pcl::Registration<PointT, PointT> {
public:
  using Base = pcl::Registration<PointT, PointT>;
  using PointCloudSource = typename Base::PointCloudSource;
  using PointCloudSourceConstPtr = typename Base::PointCloudSourceConstPtr;
  using PointCloudTargetConstPtr = typename Base::PointCloudTargetConstPtr;
  using Matrix4 = typename Base::Matrix4;
  using Ptr = std::shared_ptr<B200Registration<PointT>>;

  // NN-search stub installed as the base class' target search with force_no_recompute = true, so that the non-virtual
  // pcl::Registration::align() -> initCompute() does not rebuild a FLANN kd-tree over every new target (SURVEY.md §8b
  // "hidden base-class cost").  nearestKSearch(pt, 1, ...) — the only call the reference makes on it
  // (scan_matching_odometry_nodelet.cpp:316) — forwards to the device grid.
  class DeviceSearch : public pcl::search::Search<PointT> {
  public:
    explicit DeviceSearch(B200Registration* owner) : pcl::search::Search<PointT>("b200"), owner_(owner) {}
    void setInputCloud(const typename pcl::search::Search<PointT>::PointCloudConstPtr&, const typename pcl::search::Search<PointT>::IndicesConstPtr& = typename pcl::search::Search<PointT>::IndicesConstPtr()) override {}
    int nearestKSearch(const PointT& p, int k, std::vector<int>& idx, std::vector<float>& d2) const override {
      idx.assign(1, -1);
      d2.assign(1, std::numeric_limits<float>::max());
      if (k < 1) return 0;
      int32_t i = -1;
      float d = 0.f;
      if (!owner_->cachedNearest(p, &i, &d)) {  // not the sequential sweep of getFitnessScore / the inlier loop: exact single query
        if (b2r_target_nearest(owner_->h_, &p, 1, sizeof(PointT), &i, &d) != B2R_OK) return 0;
      }
      if (i < 0) return 0;
      idx[0] = i;
      d2[0] = d;
      return 1;
    }
    int radiusSearch(const PointT&, double, std::vector<int>& idx, std::vector<float>& d2, unsigned int = 0) const override {
      idx.clear();
      d2.clear();
      return 0;  // not used by hdl_graph_slam on the registration's search object
    }

  private:
    B200Registration* owner_;
  };

  // pcl::Registration::getFitnessScore (non-virtual, called through the base pointer at loop_detector.hpp:146 and
  // scan_matching_odometry_nodelet.cpp:307) and the inlier loop (:314-316) sweep the transformed source cloud point by point
  // through tree_->nearestKSearch.  Answering 65 536 single queries with 65 536 kernel launches would throw the speed-up
  // away, so the first query after an align() transforms the source with PCL's OWN pcl::transformPointCloud (bit-identical
  // coordinates to the ones the base class will ask about), resolves all of them in ONE b2r_target_nearest call and serves
  // the sweep from that cache; a query that is not the next cached point falls back to an exact single query.
  bool cachedNearest(const PointT& p, int32_t* idx, float* d2) {
    if (!this->input_ || this->input_->points.empty()) return false;
    if (!cache_valid_) {
      pcl::transformPointCloud(*this->input_, cache_cloud_, this->final_transformation_);
      const size_t n = cache_cloud_.points.size();
      cache_idx_.resize(n);
      cache_d2_.resize(n);
      if (b2r_target_nearest(h_, cache_cloud_.points.data(), n, sizeof(PointT), cache_idx_.data(), cache_d2_.data()) != B2R_OK) return false;
      cache_valid_ = true;
      cache_cursor_ = 0;
    }
    const size_t n = cache_cloud_.points.size();
    // the consumers sweep the cloud in order: try the cursor, then the start (second consumer), then a short window ahead of the
    // cursor (a consumer that skipped points); a miss moves the cursor on, so one odd point cannot turn the rest of the sweep
    // into single-query launches
    const size_t tries[2] = {cache_cursor_, 0};
    for (size_t c : tries) {
      if (c < n && same_point(cache_cloud_.points[c], p)) { *idx = cache_idx_[c]; *d2 = cache_d2_[c]; cache_cursor_ = c + 1; return true; }
    }
    for (size_t c = cache_cursor_ + 1; c < n && c < cache_cursor_ + 64; c++) {
      if (same_point(cache_cloud_.points[c], p)) { *idx = cache_idx_[c]; *d2 = cache_d2_[c]; cache_cursor_ = c + 1; return true; }
    }
    if (cache_cursor_ < n) cache_cursor_++;
    return false;
  }
  static bool same_point(const PointT& q, const PointT& p) { return q.x == p.x && q.y == p.y && q.z == p.z; }

  explicit B200Registration(const b2r_config& cfg) {
    if (b2r_create(&cfg, &h_) != B2R_OK) throw std::runtime_error(std::string("b200reg: ") + b2r_last_error());
    this->reg_name_ = cfg.method == B2R_METHOD_GICP ? "B200_GICP"
                      : cfg.method == B2R_METHOD_NDT_PCL ? "B200_NDT_PCL"
                      : cfg.method == B2R_METHOD_VGICP ? "B200_VGICP"
                      : cfg.method == B2R_METHOD_GICP_PCL ? "B200_GICP_PCL"
                      : cfg.method == B2R_METHOD_ICP_PCL ? "B200_ICP"
                      : cfg.method == B2R_METHOD_VGICP_CUDA ? "B200_VGICP_CUDA"
                      : cfg.method == B2R_METHOD_GICP_OMP ? "B200_GICP_OMP"
                      : cfg.method == B2R_METHOD_NDT_KDTREE ? "B200_NDT_KDTREE" : "B200_NDT";
    this->max_iterations_ = cfg.max_iterations;
    this->transformation_epsilon_ = cfg.transformation_epsilon;
    this->corr_dist_threshold_ = cfg.max_correspondence_distance;
    this->setSearchMethodTarget(typename pcl::search::Search<PointT>::Ptr(new DeviceSearch(this)), /*force_no_recompute=*/true);
  }
  ~B200Registration() override { b2r_destroy(h_); }

  void setInputSource(const PointCloudSourceConstPtr& cloud) override {
    if (cloud == this->input_ && !source_promoted_) return;  // same early-out as fast_gicp
    Base::setInputSource(cloud);
    cache_valid_ = false;
    source_promoted_ = false;
    b2r_set_source(h_, cloud->points.data(), cloud->points.size(), sizeof(PointT));
  }

  void setInputTarget(const PointCloudTargetConstPtr& cloud) override {
    if (cloud == this->target_) return;
    const bool promote = (cloud == this->input_);  // keyframe switch: the last source becomes the target (:245-246)
    Base::setInputTarget(cloud);
    cache_valid_ = false;
    // the engine has no source after a promotion (b200reg.h): the same cloud set as the source again is uploaded, not skipped
    if (promote) source_promoted_ = b2r_promote_source_to_target(h_) == B2R_OK;
    else b2r_set_target(h_, cloud->points.data(), cloud->points.size(), sizeof(PointT));
  }

  // getFitnessScore is NOT virtual in pcl::Registration, but both reference callers invoke it through the base pointer;
  // the base implementation keeps working because it only needs tree_->nearestKSearch (DeviceSearch above).  Callers that
  // hold the concrete type get the single-kernel version:
  double getFitnessScoreDevice(double max_range = std::numeric_limits<double>::max()) {
    double score = std::numeric_limits<double>::max();
    b2r_fitness(h_, nullptr, max_range, 0.25f, &score, nullptr, nullptr);
    return score;
  }

  b2r_handle* handle() { return h_; }

protected:
  // pcl::Registration::align() copies the source into `output`, then calls this (SURVEY.md A.1)
  void computeTransformation(PointCloudSource& output, const Matrix4& guess) override {
    b2r_result r;
    cache_valid_ = false;
    const int rc = b2r_align(h_, guess.data(), &r);  // Eigen::Matrix4f is column-major, like the ABI
    this->converged_ = (rc == B2R_OK) && r.converged;
    this->nr_iterations_ = r.iterations;
    for (int i = 0; i < 16; i++) this->final_transformation_.data()[i] = r.T[i];
    this->transformation_ = this->final_transformation_;
    // `output` feeds the inlier loop of the status publisher (scan_matching_odometry_nodelet.cpp:314-316), which looks every
    // one of its points up through tree_->nearestKSearch.  It is produced by PCL's OWN pcl::transformPointCloud — the very call
    // that seeds the nearest-neighbour cache (cachedNearest) — so the two clouds are bit-identical by construction, whatever
    // association / SIMD path the installed PCL uses for the 4x4 product, and the sweep is served from the cache.
    if (rc == B2R_OK && this->input_ && !this->input_->points.empty()) pcl::transformPointCloud(*this->input_, output, this->final_transformation_);
  }

private:
  b2r_handle* h_ = nullptr;
  // nearest-neighbour cache of the transformed source (see cachedNearest)
  bool source_promoted_ = false;
  bool cache_valid_ = false;
  size_t cache_cursor_ = 0;
  PointCloudSource cache_cloud_;
  std::vector<int32_t> cache_idx_;
  std::vector<float> cache_d2_;
};

// The branch added to select_registration_method() (registrations.cpp:27-124), mirroring the USE_VGICP_CUDA pattern
// of registrations.cpp:16-18,37-47 / CMakeLists.txt:56-60:
//
//   #ifdef USE_B200REG
//     else if(registration_method == "B200_GICP" || registration_method == "B200_NDT") {
//       b2r_config cfg;
//       b2r_config_default(&cfg, registration_method == "B200_GICP" ? B2R_METHOD_GICP : B2R_METHOD_NDT);
//       cfg.transformation_epsilon = pnh.param<double>("reg_transformation_epsilon", 0.01);
//       cfg.max_iterations = pnh.param<int>("reg_maximum_iterations", 64);
//       cfg.max_correspondence_distance = pnh.param<double>("reg_max_correspondence_distance", 2.5);
//       cfg.k_correspondences = pnh.param<int>("reg_correspondence_randomness", 20);
//       cfg.ndt_resolution = pnh.param<double>("reg_resolution", 0.5);
//       cfg.ndt_search_method = pnh.param<std::string>("reg_nn_search_method", "DIRECT7") == "DIRECT1" ? 1 : 7;
//       cfg.device_id = pnh.param<int>("reg_device_id", 0);
//       return pcl::Registration<PointT, PointT>::Ptr(new B200Registration<PointT>(cfg));
//     }
//     else if(registration_method == "B200_NDT_PCL") {  // in place of the NDT branch (registrations.cpp:93-100)
//       b2r_config cfg;
//       b2r_config_default(&cfg, B2R_METHOD_NDT_PCL);  // pcl::NormalDistributionsTransform: step size 0.1, outlier ratio 0.55
//       cfg.transformation_epsilon = pnh.param<double>("reg_transformation_epsilon", 0.01);
//       cfg.max_iterations = pnh.param<int>("reg_maximum_iterations", 64);
//       cfg.ndt_resolution = pnh.param<double>("reg_resolution", 0.5);
//       cfg.device_id = pnh.param<int>("reg_device_id", 0);
//       return pcl::Registration<PointT, PointT>::Ptr(new B200Registration<PointT>(cfg));
//     }
//     else if(registration_method == "B200_VGICP") {  // in place of the FAST_VGICP branch (registrations.cpp:48-56)
//       b2r_config cfg;
//       b2r_config_default(&cfg, B2R_METHOD_VGICP);  // fast_gicp::FastVGICP: DIRECT1, voxel mode ADDITIVE
//       cfg.ndt_resolution = pnh.param<double>("reg_resolution", 1.0);
//       cfg.transformation_epsilon = pnh.param<double>("reg_transformation_epsilon", 0.01);
//       cfg.max_iterations = pnh.param<int>("reg_maximum_iterations", 64);
//       cfg.k_correspondences = pnh.param<int>("reg_correspondence_randomness", 20);
//       cfg.device_id = pnh.param<int>("reg_device_id", 0);
//       return pcl::Registration<PointT, PointT>::Ptr(new B200Registration<PointT>(cfg));
//     }
//     else if(registration_method == "B200_GICP_PCL") {  // in place of the GICP branch (registrations.cpp:66-76)
//       b2r_config cfg;
//       b2r_config_default(&cfg, B2R_METHOD_GICP_PCL);  // pcl::GeneralizedIterativeClosestPoint: BFGS, rotation epsilon 2e-3
//       cfg.transformation_epsilon = pnh.param<double>("reg_transformation_epsilon", 0.01);
//       cfg.max_iterations = pnh.param<int>("reg_maximum_iterations", 64);
//       cfg.max_correspondence_distance = pnh.param<double>("reg_max_correspondence_distance", 2.5);
//       cfg.k_correspondences = pnh.param<int>("reg_correspondence_randomness", 20);
//       cfg.max_optimizer_iterations = pnh.param<int>("reg_max_optimizer_iterations", 20);
//       cfg.device_id = pnh.param<int>("reg_device_id", 0);
//       return pcl::Registration<PointT, PointT>::Ptr(new B200Registration<PointT>(cfg));
//     }
//     else if(registration_method == "B200_ICP") {  // in place of the ICP branch (registrations.cpp:57-65)
//       b2r_config cfg;
//       b2r_config_default(&cfg, B2R_METHOD_ICP_PCL);  // pcl::IterativeClosestPoint: Umeyama SVD step, the loop on the device
//       cfg.transformation_epsilon = pnh.param<double>("reg_transformation_epsilon", 0.01);
//       cfg.max_iterations = pnh.param<int>("reg_maximum_iterations", 64);
//       cfg.max_correspondence_distance = pnh.param<double>("reg_max_correspondence_distance", 2.5);
//       cfg.use_reciprocal_correspondences = pnh.param<bool>("reg_use_reciprocal_correspondences", false) ? 1 : 0;
//       cfg.device_id = pnh.param<int>("reg_device_id", 0);
//       return pcl::Registration<PointT, PointT>::Ptr(new B200Registration<PointT>(cfg));
//     }
//     else if(registration_method == "B200_VGICP_CUDA") {  // in place of the FAST_VGICP_CUDA branch (registrations.cpp:37-47)
//       b2r_config cfg;
//       b2r_config_default(&cfg, B2R_METHOD_VGICP_CUDA);  // fast_gicp::FastVGICPCuda: k-NN exact, PLANE, DIRECT1, float32 terms
//       cfg.ndt_resolution = pnh.param<double>("reg_resolution", 1.0);
//       cfg.transformation_epsilon = pnh.param<double>("reg_transformation_epsilon", 0.01);
//       cfg.max_iterations = pnh.param<int>("reg_maximum_iterations", 64);
//       cfg.k_correspondences = pnh.param<int>("reg_correspondence_randomness", 20);
//       cfg.device_id = pnh.param<int>("reg_device_id", 0);
//       return pcl::Registration<PointT, PointT>::Ptr(new B200Registration<PointT>(cfg));
//     }
//     else if(registration_method == "B200_NDT_KDTREE") {  // in place of NDT_OMP with reg_nn_search_method = KDTREE (:112-113)
//       b2r_config cfg;
//       b2r_config_default(&cfg, B2R_METHOD_NDT_KDTREE);  // pclomp::NormalDistributionsTransform: radius search over the centroids
//       cfg.transformation_epsilon = pnh.param<double>("reg_transformation_epsilon", 0.01);
//       cfg.max_iterations = pnh.param<int>("reg_maximum_iterations", 64);
//       cfg.ndt_resolution = pnh.param<double>("reg_resolution", 0.5);
//       cfg.device_id = pnh.param<int>("reg_device_id", 0);
//       return pcl::Registration<PointT, PointT>::Ptr(new B200Registration<PointT>(cfg));
//     }
//     else if(registration_method == "B200_GICP_OMP") {  // in place of the GICP_OMP branch (registrations.cpp:76-86)
//       b2r_config cfg;
//       b2r_config_default(&cfg, B2R_METHOD_GICP_OMP);  // pclomp::GeneralizedIterativeClosestPoint: cost poses applyState(guess, x)
//       cfg.transformation_epsilon = pnh.param<double>("reg_transformation_epsilon", 0.01);
//       cfg.max_iterations = pnh.param<int>("reg_maximum_iterations", 64);
//       cfg.max_correspondence_distance = pnh.param<double>("reg_max_correspondence_distance", 2.5);
//       cfg.k_correspondences = pnh.param<int>("reg_correspondence_randomness", 20);
//       cfg.max_optimizer_iterations = pnh.param<int>("reg_max_optimizer_iterations", 20);
//       cfg.device_id = pnh.param<int>("reg_device_id", 0);
//       return pcl::Registration<PointT, PointT>::Ptr(new B200Registration<PointT>(cfg));
//     }
//   #endif

}  // namespace hdl_graph_slam
