// backend_harness.cpp — runs adapter/b200_backend.hpp (against the test-only adapter/pcl_shim.hpp and adapter/backend_shim.hpp) the way
// hdl_graph_slam_nodelet drives LoopDetector, InformationMatrixCalculator and MapCloudGenerator, for tests/test_backend_adapter_gpu.py.
//
//   backend_harness <dir> serial|concurrent
// <dir>/in.bin : the rosparams, the clouds and a list of operations (see main); every number little-endian, int32 or float64
// <dir>/out.bin: one length-prefixed block per operation that answers (DETECT, INFO, MAP), then, in serial mode, the session totals
//
// serial: the operations in order, then the whole list once more on the same keyframe cache with a fresh loop detector and fresh
// keyframe objects (same clouds): its answers must equal the first pass's, and only the first pass may upload the clouds.
// concurrent: every MAP runs on a second thread while the operations after it (detect, information matrices) go on, as the map timer
// of the nodelet does; the answers must be the serial ones.
#include "backend_shim.hpp"
#include "b200_backend.hpp"
#include <cstdio>
#include <cstring>
#include <thread>

using namespace hdl_graph_slam;
using PointT = pcl::PointXYZI;
using Cloud = pcl::PointCloud<PointT>;
using Block = std::vector<char>;

enum Op { KEYFRAME = 1, ESTIMATE = 2, DETECT = 3, INFO = 4, MAP = 5 };

struct Reader {
  FILE* f;
  bool ok = true;
  template <typename T>
  T get() {
    T v{};
    ok = ok && std::fread(&v, sizeof(T), 1, f) == 1;
    return v;
  }
  std::string str() {
    std::string s(get<int32_t>(), '\0');
    if (!s.empty()) ok = ok && std::fread(&s[0], 1, s.size(), f) == s.size();
    return s;
  }
  Eigen::Isometry3d iso() {
    Eigen::Isometry3d T;
    for (int i = 0; i < 16; i++) T.matrix().m[i] = get<double>();
    return T;
  }
};

template <typename T>
static void put(Block& b, T v) {
  const char* p = reinterpret_cast<const char*>(&v);
  b.insert(b.end(), p, p + sizeof(T));
}

struct Operation {
  int code = 0;
  int32_t a = 0, b = 0, c = 0;  // KEYFRAME: cloud; ESTIMATE: keyframe; INFO: calculator, cloud1, cloud2
  double accum = 0.0, resolution = 0.0;
  Eigen::Isometry3d T;                                    // KEYFRAME / ESTIMATE: estimate; INFO: relpose
  std::vector<std::pair<int32_t, Eigen::Isometry3d>> snaps;  // MAP: keyframe index, pose
};

static void put_info(Block& out, const Eigen::MatrixXd& inf) {
  put<int32_t>(out, inf.rows());
  put<int32_t>(out, inf.cols());
  for (double v : inf.v) put(out, v);
}

// one pass over the operations on `cache`; blocks[i] receives the answer of operation i
static void run(const std::vector<Operation>& ops, const std::vector<Cloud::ConstPtr>& clouds, ros::NodeHandle& pnh, ros::NodeHandle& pnh_const,
                const std::shared_ptr<B200KeyframeCache>& cache, bool concurrent, std::vector<Block>& blocks) {
  B200LoopDetector loop_detector(pnh, cache);
  const B200InformationMatrixCalculator inf_calc[2] = {B200InformationMatrixCalculator(pnh, cache), B200InformationMatrixCalculator(pnh_const, cache)};
  const B200MapCloudGenerator map_cloud_generator(cache);
  GraphSLAM graph;
  std::vector<std::unique_ptr<g2o::VertexSE3>> nodes;
  std::vector<KeyFrame::Ptr> keyframes;   // every keyframe ever created, in creation order (the indices the test uses)
  std::vector<KeyFrame::Ptr> registered;  // hdl_graph_slam_nodelet's `keyframes`
  std::deque<KeyFrame::Ptr> new_keyframes;
  std::thread map_thread;
  blocks.assign(ops.size(), Block());
  for (size_t i = 0; i < ops.size(); i++) {
    const Operation& op = ops[i];
    Block& out = blocks[i];
    if (op.code == KEYFRAME) {
      nodes.emplace_back(new g2o::VertexSE3());
      nodes.back()->setEstimate(op.T);
      auto kf = std::make_shared<KeyFrame>();
      kf->accum_distance = op.accum;
      kf->cloud = clouds[op.a];
      kf->node = nodes.back().get();
      keyframes.push_back(kf);
      new_keyframes.push_back(kf);
    } else if (op.code == ESTIMATE) {
      keyframes[op.a]->node->setEstimate(op.T);
    } else if (op.code == DETECT) {  // hdl_graph_slam_nodelet.cpp:549-577: detect, one edge per loop, the new keyframes join the graph
      auto index = [&](const KeyFrame::Ptr& k) { return (int32_t)(std::find(keyframes.begin(), keyframes.end(), k) - keyframes.begin()); };
      const auto loops = loop_detector.detect(registered, new_keyframes, graph);
      put<int32_t>(out, (int32_t)loops.size());
      for (const auto& loop : loops) {
        put(out, index(loop->key1));
        put(out, index(loop->key2));
        for (int k = 0; k < 16; k++) put(out, loop->relative_pose.m[k]);
        Eigen::Isometry3d relpose;  // relative_pose.cast<double>() (:569)
        for (int k = 0; k < 16; k++) relpose.matrix().m[k] = (double)loop->relative_pose.m[k];
        put_info(out, inf_calc[0].calc_information_matrix(loop->key1->cloud, loop->key2->cloud, relpose));
      }
      put(out, loop_detector.get_last_edge_accum_distance());
      registered.insert(registered.end(), new_keyframes.begin(), new_keyframes.end());
      new_keyframes.clear();
    } else if (op.code == INFO) {
      put_info(out, inf_calc[op.a].calc_information_matrix(clouds[op.b], clouds[op.c], op.T));
    } else if (op.code == MAP) {  // the snapshots are taken here (:520-526); generate may then run on the timer's own thread
      std::vector<KeyFrameSnapshot::Ptr> snapshots;
      for (const auto& s : op.snaps) snapshots.push_back(std::make_shared<KeyFrameSnapshot>(s.second, keyframes[s.first]->cloud));
      auto job = [&map_cloud_generator, snapshots, &out, resolution = op.resolution]() {
        const Cloud::Ptr map = map_cloud_generator.generate(snapshots, resolution);
        if (!map) {
          put<int64_t>(out, -1);
          return;
        }
        put<int64_t>(out, (int64_t)map->points.size());
        put<int64_t>(out, map->width);
        put<int64_t>(out, map->height);
        put<int64_t>(out, map->is_dense);
        const char* p = reinterpret_cast<const char*>(map->points.data());
        out.insert(out.end(), p, p + map->points.size() * sizeof(PointT));
      };
      if (map_thread.joinable()) map_thread.join();
      if (concurrent) map_thread = std::thread(job);
      else job();
    }
  }
  if (map_thread.joinable()) map_thread.join();
}

static uint64_t h2d_bytes(B200KeyframeCache& cache) {
  b2r_handle* eng = nullptr;
  b2r_stats s;
  B200KeyframeCache::check(b2r_batch_get_engine(cache.batch(), &eng));
  B200KeyframeCache::check(b2r_get_stats(eng, &s, 0));
  return s.h2d_bytes;
}

static int session(int argc, char** argv);

int main(int argc, char** argv) {
  try {
    return session(argc, argv);
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 5;
  }
}

static int session(int argc, char** argv) {
  if (argc != 3) return 2;
  const std::string dir = argv[1];
  const bool concurrent = std::strcmp(argv[2], "concurrent") == 0;
  FILE* f = std::fopen((dir + "/in.bin").c_str(), "rb");
  if (!f) return 3;
  Reader r{f};
  ros::NodeHandle pnh, pnh_const;
  for (int i = 0, n = r.get<int32_t>(); i < n; i++) {
    const std::string k = r.str(), v = r.str();
    pnh.setParam(k, v);
    pnh_const.setParam(k, v);
  }
  pnh_const.setParam("use_const_inf_matrix", "true");
  std::vector<Cloud::ConstPtr> clouds;
  for (int i = 0, n = r.get<int32_t>(); i < n && r.ok; i++) {
    auto c = std::make_shared<Cloud>();
    c->points.resize(r.get<int32_t>());
    if (!c->points.empty()) r.ok = r.ok && std::fread(c->points.data(), sizeof(PointT), c->points.size(), f) == c->points.size();
    clouds.push_back(c);
  }
  std::vector<Operation> ops(r.get<int32_t>());
  for (Operation& op : ops) {
    op.code = r.get<int32_t>();
    if (op.code == KEYFRAME) { op.a = r.get<int32_t>(); op.accum = r.get<double>(); op.T = r.iso(); }
    else if (op.code == ESTIMATE) { op.a = r.get<int32_t>(); op.T = r.iso(); }
    else if (op.code == INFO) { op.a = r.get<int32_t>(); op.b = r.get<int32_t>(); op.c = r.get<int32_t>(); op.T = r.iso(); }
    else if (op.code == MAP) {
      op.resolution = r.get<double>();
      for (int k = 0, n = r.get<int32_t>(); k < n; k++) {
        const int32_t idx = r.get<int32_t>();
        op.snaps.emplace_back(idx, r.iso());
      }
    } else if (op.code != DETECT) return 3;
  }
  std::fclose(f);
  if (!r.ok) return 3;

  auto cache = std::make_shared<B200KeyframeCache>(pnh);
  std::vector<Block> blocks, again;
  run(ops, clouds, pnh, pnh_const, cache, concurrent, blocks);
  Block totals;
  if (!concurrent) {
    const uint64_t h2d_first = h2d_bytes(*cache);
    const int n_first = b2r_batch_cloud_count(cache->batch());
    run(ops, clouds, pnh, pnh_const, cache, false, again);
    put<uint64_t>(totals, h2d_first);
    put<uint64_t>(totals, h2d_bytes(*cache) - h2d_first);
    put<int64_t>(totals, n_first);
    put<int64_t>(totals, b2r_batch_cloud_count(cache->batch()));
    put<int64_t>(totals, again == blocks ? 1 : 0);
  }
  f = std::fopen((dir + "/out.bin").c_str(), "wb");
  if (!f) return 4;
  blocks.push_back(totals);
  for (const Block& b : blocks) {
    const int64_t n = (int64_t)b.size();
    std::fwrite(&n, sizeof n, 1, f);
    if (n) std::fwrite(b.data(), 1, b.size(), f);
  }
  std::fclose(f);
  return 0;
}
