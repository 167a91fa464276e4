// b200_backend.hpp — drop-in replacements for the three back-end classes of koide3/hdl_graph_slam that do point-cloud work, all three
// served by ONE device keyframe cache (a b2r_batch of libb200reg.so):
//   LoopDetector                 include/hdl_graph_slam/loop_detector.hpp:31-171        -> B200LoopDetector
//   InformationMatrixCalculator  src/hdl_graph_slam/information_matrix_calculator.cpp     -> B200InformationMatrixCalculator
//   MapCloudGenerator            src/hdl_graph_slam/map_cloud_generator.cpp              -> B200MapCloudGenerator
// Each keyframe cloud (KeyFrame::cloud, keyframe.hpp:42, shared by its KeyFrameSnapshot, :69) is uploaded and preprocessed once, at its
// first use, and then serves loop matching, every information matrix and every map.  Include it after the reference's
// loop_detector.hpp (it uses hdl_graph_slam::Loop, KeyFrame, KeyFrameSnapshot and GraphSLAM from there).  INTEGRATION.md §4 shows the
// nodelet patch.  Compiled only where ROS, PCL, Eigen and g2o exist; tests/test_backend_syntax.py checks it against the test-only
// stand-ins adapter/pcl_shim.hpp and adapter/backend_shim.hpp.
#pragma once
#include <b200reg.h>
#include "b200_select.hpp"
#include <algorithm>
#include <deque>
#include <iostream>
#include <limits>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

namespace hdl_graph_slam {

// The device keyframe cache the three classes below share.  It owns one b2r_batch, configured as select_registration_method(pnh)
// would configure the loop detector's registration (loop_detector.hpp:47), and maps every keyframe cloud object to its cloud id.  It
// holds no graph state: poses and accumulated distances are read from the keyframes at every call.
class B200KeyframeCache {
public:
  using PointT = pcl::PointXYZI;
  using CloudConstPtr = pcl::PointCloud<PointT>::ConstPtr;

  // pnh: the back end's private namespace, the one LoopDetector(pnh) reads.  A registration_method the engine does not re-create
  // (B2R_EUNSUPPORTED) throws here with the engine's message, so the caller can keep the reference classes.
  explicit B200KeyframeCache(ros::NodeHandle& pnh) {
    b2r_handle* h = b200_select::select_registration_method(pnh);
    b2r_config cfg;
    const int rc = b2r_get_config(h, &cfg);
    b2r_destroy(h);
    check(rc);
    check(b2r_batch_create(&cfg, &batch_));
  }
  ~B200KeyframeCache() { b2r_batch_destroy(batch_); }
  B200KeyframeCache(const B200KeyframeCache&) = delete;
  B200KeyframeCache& operator=(const B200KeyframeCache&) = delete;

  // Every use of batch() and id() happens under this lock: the map timer runs outside the nodelet's main_thread_mutex
  // (hdl_graph_slam_nodelet.cpp:139-140), and a b2r_batch takes one thread at a time.
  std::unique_lock<std::mutex> lock() { return std::unique_lock<std::mutex>(mutex_); }

  // The cloud id of `cloud`; its first use uploads it (b2r_batch_add_cloud, PointXYZI records).  The cache keeps the pointer, so the
  // address of a cached cloud is never reused by another one.  Caller holds lock().
  int32_t id(const CloudConstPtr& cloud) {
    auto it = ids_.find(cloud.get());
    if (it != ids_.end()) return it->second.id;
    int32_t cid = -1;
    check(b2r_batch_add_cloud(batch_, cloud->points.data(), cloud->points.size(), sizeof(PointT), &cid));
    ids_.emplace(cloud.get(), Entry{cloud, cid});
    return cid;
  }

  b2r_batch* batch() { return batch_; }

  static void check(int rc) {
    if (rc < 0) throw std::runtime_error(std::string("b200reg: ") + b2r_last_error());
  }

private:
  struct Entry {
    CloudConstPtr cloud;
    int32_t id;
  };
  std::mutex mutex_;
  b2r_batch* batch_ = nullptr;
  std::unordered_map<const void*, Entry> ids_;
};

// LoopDetector (loop_detector.hpp:31-171) with every candidate of every new keyframe matched in one batch call:
// b2r_loop_detect_plan -> b2r_batch_loop_detect -> b2r_loop_detect_replay registers the loops of the reference's sequential walk.
class B200LoopDetector {
public:
  using PointT = pcl::PointXYZI;

  B200LoopDetector(ros::NodeHandle& pnh, std::shared_ptr<B200KeyframeCache> cache) : cache_(std::move(cache)) {
    b2r_loop_params_default(&params_);
    params_.distance_thresh = pnh.param<double>("distance_thresh", 5.0);
    params_.accum_distance_thresh = pnh.param<double>("accum_distance_thresh", 8.0);
    params_.min_edge_interval = pnh.param<double>("min_edge_interval", 5.0);
    params_.fitness_score_max_range = pnh.param<double>("fitness_score_max_range", std::numeric_limits<double>::max());
    params_.fitness_score_thresh = pnh.param<double>("fitness_score_thresh", 0.5);
  }

  std::vector<Loop::Ptr> detect(const std::vector<KeyFrame::Ptr>& keyframes, const std::deque<KeyFrame::Ptr>& new_keyframes, GraphSLAM&) {
    std::vector<Loop::Ptr> detected_loops;
    const size_t n_new = new_keyframes.size();
    if (n_new == 0) return detected_loops;
    std::vector<b2r_keyframe_state> ks(keyframes.size()), ns(n_new);
    for (size_t i = 0; i < keyframes.size(); i++) state(*keyframes[i], &ks[i]);
    for (size_t g = 0; g < n_new; g++) state(*new_keyframes[g], &ns[g]);
    const size_t cap = std::max<size_t>(keyframes.size() * n_new, 1);
    std::vector<int32_t> cand(cap);
    std::vector<float> guesses(16 * cap);
    std::vector<int64_t> first(n_new + 1);
    size_t n_pairs = 0;
    const double planned_last_edge = last_edge_accum_distance;
    B200KeyframeCache::check(b2r_loop_detect_plan(&params_, ks.data(), ks.size(), ns.data(), n_new, planned_last_edge, cand.data(), guesses.data(),
                                                  cap, first.data(), &n_pairs));
    std::vector<b2r_result> results(n_pairs);
    std::vector<int32_t> best(n_new, -1), accepted(n_new, -1);
    if (n_pairs) {
      std::vector<b2r_pair> pairs(n_pairs);
      auto lock = cache_->lock();
      for (size_t g = 0; g < n_new; g++) {
        if (first[g] == first[g + 1]) continue;
        const int32_t target = cache_->id(new_keyframes[g]->cloud);
        for (int64_t j = first[g]; j < first[g + 1]; j++) {
          pairs[j].source = cache_->id(keyframes[cand[j]]->cloud);
          pairs[j].target = target;
          std::copy(guesses.begin() + 16 * j, guesses.begin() + 16 * (j + 1), pairs[j].guess);
        }
      }
      B200KeyframeCache::check(b2r_batch_loop_detect(cache_->batch(), pairs.data(), n_pairs, first.data(), n_new, params_.fitness_score_max_range,
                                                     params_.fitness_score_thresh, results.data(), best.data()));
    }
    B200KeyframeCache::check(b2r_loop_detect_replay(&params_, ns.data(), n_new, first.data(), best.data(), planned_last_edge,
                                                    &last_edge_accum_distance, accepted.data()));
    for (size_t g = 0; g < n_new; g++) {
      if (accepted[g] < 0) continue;
      const int64_t j = first[g] + accepted[g];
      Eigen::Matrix4f relative_pose;
      std::copy(results[j].T, results[j].T + 16, relative_pose.data());  // both column-major
      detected_loops.push_back(std::make_shared<Loop>(new_keyframes[g], keyframes[cand[j]], relative_pose));
    }
    return detected_loops;
  }

  double get_distance_thresh() const { return params_.distance_thresh; }
  // the accumulated distance of the new keyframe that ended the last registered loop (loop_detector.hpp:166)
  double get_last_edge_accum_distance() const { return last_edge_accum_distance; }

private:
  static void state(const KeyFrame& k, b2r_keyframe_state* s) {
    s->accum_distance = k.accum_distance;
    const auto& m = k.node->estimate().matrix();
    std::copy(m.data(), m.data() + 16, s->estimate);
  }

  std::shared_ptr<B200KeyframeCache> cache_;
  b2r_loop_params params_;
  double last_edge_accum_distance = 0.0;
};

// InformationMatrixCalculator (information_matrix_calculator.cpp:10-47) with calc_fitness_score on the cached keyframe clouds.
class B200InformationMatrixCalculator {
public:
  using PointT = pcl::PointXYZI;

  B200InformationMatrixCalculator(ros::NodeHandle& nh, std::shared_ptr<B200KeyframeCache> cache) : cache_(std::move(cache)) {
    b2r_information_params_default(&params_);
    params_.use_const_inf_matrix = nh.param<bool>("use_const_inf_matrix", false) ? 1 : 0;
    params_.const_stddev_x = nh.param<double>("const_stddev_x", 0.5);
    params_.const_stddev_q = nh.param<double>("const_stddev_q", 0.1);
    params_.var_gain_a = nh.param<double>("var_gain_a", 20.0);
    params_.min_stddev_x = nh.param<double>("min_stddev_x", 0.1);
    params_.max_stddev_x = nh.param<double>("max_stddev_x", 5.0);
    params_.min_stddev_q = nh.param<double>("min_stddev_q", 0.05);
    params_.max_stddev_q = nh.param<double>("max_stddev_q", 0.2);
    params_.fitness_score_thresh = nh.param<double>("fitness_score_thresh", 0.5);  // :21 (the header's load() says 2.5)
  }

  Eigen::MatrixXd calc_information_matrix(const pcl::PointCloud<PointT>::ConstPtr& cloud1, const pcl::PointCloud<PointT>::ConstPtr& cloud2,
                                          const Eigen::Isometry3d& relpose) const {
    double fitness_score = 0.0;
    if (!params_.use_const_inf_matrix) {  // :26-31 needs no score
      b2r_pair pair;
      const auto& m = relpose.matrix();
      for (int i = 0; i < 16; i++) pair.guess[i] = static_cast<float>(m.data()[i]);  // relpose.cast<float>() (:58)
      auto lock = cache_->lock();
      pair.target = cache_->id(cloud1);  // the kd-tree's cloud (:50-51)
      pair.source = cache_->id(cloud2);  // the transformed cloud
      B200KeyframeCache::check(b2r_batch_calc_fitness_score(cache_->batch(), &pair, 1, std::numeric_limits<double>::max(), &fitness_score));
    }
    double d[6];
    B200KeyframeCache::check(b2r_information_from_fitness(&params_, fitness_score, d));
    Eigen::MatrixXd inf = Eigen::MatrixXd::Identity(6, 6);
    for (int i = 0; i < 6; i++) inf(i, i) = d[i];
    return inf;
  }

private:
  std::shared_ptr<B200KeyframeCache> cache_;
  b2r_information_params params_;
};

// MapCloudGenerator::generate (map_cloud_generator.cpp:13-51) over the cached keyframe clouds.  At resolution > 0 the points are the
// centres of PCL's occupied octree voxels in ascending key order (not the octree's traversal order), x y z 1 with intensity 0; at
// resolution <= 0 every keyframe's points transformed by its pose, intensity kept.
class B200MapCloudGenerator {
public:
  using PointT = pcl::PointXYZI;

  explicit B200MapCloudGenerator(std::shared_ptr<B200KeyframeCache> cache) : cache_(std::move(cache)) {}

  pcl::PointCloud<PointT>::Ptr generate(const std::vector<KeyFrameSnapshot::Ptr>& keyframes, double resolution) const {
    if (keyframes.empty()) {
      std::cerr << "warning: keyframes empty!!" << std::endl;
      return nullptr;
    }
    std::vector<int32_t> ids(keyframes.size());
    std::vector<float> poses(16 * keyframes.size());
    size_t total = 0;
    for (size_t k = 0; k < keyframes.size(); k++) {
      const auto& m = keyframes[k]->pose.matrix();
      for (int i = 0; i < 16; i++) poses[16 * k + i] = static_cast<float>(m.data()[i]);  // pose.matrix().cast<float>() (:24)
      total += keyframes[k]->cloud->points.size();
    }
    pcl::PointCloud<PointT>::Ptr cloud(new pcl::PointCloud<PointT>());
    cloud->points.resize(total);
    size_t n = 0;
    {
      auto lock = cache_->lock();
      for (size_t k = 0; k < keyframes.size(); k++) ids[k] = cache_->id(keyframes[k]->cloud);
      B200KeyframeCache::check(b2r_batch_map_cloud_generate(cache_->batch(), ids.data(), poses.data(), ids.size(), resolution, sizeof(PointT),
                                                            cloud->points.data(), total, nullptr, &n));
    }
    cloud->points.resize(n);
    cloud->width = n;  // :32-34, :46-48
    cloud->height = 1;
    cloud->is_dense = false;
    return cloud;
  }

private:
  std::shared_ptr<B200KeyframeCache> cache_;
};

}  // namespace hdl_graph_slam
