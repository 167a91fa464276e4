// adapter_harness.cpp — runs adapter/b200_registration.hpp (against the test-only adapter/pcl_shim.hpp) the way hdl_graph_slam's two
// callers drive the pcl::Registration handle, for tests/test_adapter_gpu.py.
//
//   adapter_harness <method 0|1|2> <dir>
// <dir>/in.bin : int32 n_frames, then per frame int32 n, int32 switch_keyframe_after, n PointXYZI records (32 bytes)
// <dir>/out.bin: what every call returned, as doubles (see `put` below), read back by the test.
// Walk (apps/scan_matching_odometry_nodelet.cpp:165-262, :298-321): frame 0 setInputTarget; then per frame setInputSource -> align(prev_trans)
// -> hasConverged / getFinalTransformation -> getFitnessScore() through the BASE pointer -> the inlier loop over `aligned` through
// getSearchMethodTarget()->nearestKSearch -> (switch) setInputTarget(filtered).  After the walk: the awkward sweeps on the last frame.
#include "pcl_shim.hpp"
#include "b200_registration.hpp"
#include <cstdio>
#include <cstring>

using PointT = pcl::PointXYZI;
using Cloud = pcl::PointCloud<PointT>;

static std::vector<double> g_out;
static void put(double v) { g_out.push_back(v); }

struct Counters { double launches, h2d; };  // nearest-neighbour kernel launches, bytes uploaded
static Counters counters(b2r_handle* h) {
  b2r_stats s;
  b2r_get_stats(h, &s, 0);
  // the nearest-neighbour queries are launches of the "misc" class; the lazy build of a target's search structure behind the first
  // query (an NDT target has none until then) is of another class and is not a query
  double l = 0;
  for (int i = 0; i < s.n_classes; i++)
    if (std::strcmp(b2r_kernel_class_name(i), "misc") == 0) l += (double)s.launches[i];
  return {l, (double)s.h2d_bytes};
}

// one query through the search object: index, squared distance, and how many kernels it cost
static void query(b2r_handle* h, const pcl::search::Search<PointT>::Ptr& tree, const PointT& p) {
  std::vector<int> idx;
  std::vector<float> d2;
  const Counters a = counters(h);
  const int found = tree->nearestKSearch(p, 1, idx, d2);
  put(found);
  put(idx[0]);
  put(d2[0]);
  put(counters(h).launches - a.launches);
}

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  const std::string dir = argv[2];
  FILE* f = std::fopen((dir + "/in.bin").c_str(), "rb");
  if (!f) return 3;
  int32_t nf = 0;
  if (std::fread(&nf, 4, 1, f) != 1) return 3;
  std::vector<Cloud::Ptr> frames;
  std::vector<int> sw;
  for (int k = 0; k < nf; k++) {
    int32_t hdr[2];
    if (std::fread(hdr, 4, 2, f) != 2) return 3;
    auto c = std::make_shared<Cloud>();
    c->points.resize(hdr[0]);
    if (hdr[0] && std::fread(c->points.data(), sizeof(PointT), hdr[0], f) != (size_t)hdr[0]) return 3;
    frames.push_back(c);
    sw.push_back(hdr[1]);
  }
  std::fclose(f);

  b2r_config cfg;
  b2r_config_default(&cfg, std::atoi(argv[1]));
  cfg.ndt_resolution = 1.0;
  auto* concrete = new hdl_graph_slam::B200Registration<PointT>(cfg);
  pcl::Registration<PointT, PointT>::Ptr reg(concrete);  // the factory's return type
  b2r_handle* h = concrete->handle();

  Eigen::Matrix4f prev = Eigen::Matrix4f::Identity();
  reg->setInputTarget(frames[0]);  // :172
  Cloud aligned;
  for (int k = 1; k < nf; k++) {
    reg->setInputSource(frames[k]);  // :177
    reg->align(aligned, prev);       // :210
    const Counters c0 = counters(h);
    put(reg->hasConverged());
    const Eigen::Matrix4f T = reg->getFinalTransformation();
    for (int i = 0; i < 16; i++) put(T.m[i]);
    put(reg->getFitnessScore());  // :307, the base class' sweep
    int inliers = 0;              // :311-320
    std::vector<int> ki;
    std::vector<float> kd;
    for (size_t i = 0; i < aligned.points.size(); i++) {
      reg->getSearchMethodTarget()->nearestKSearch(aligned.points[i], 1, ki, kd);
      if (kd[0] < 0.5 * 0.5) inliers++;
    }
    put(inliers);
    put(counters(h).launches - c0.launches);  // kernels behind both sweeps together
    put((double)aligned.points.size());
    for (const PointT& p : aligned.points) { put(p.x); put(p.y); put(p.z); }
    if (reg->hasConverged()) prev = T;
    if (sw[k]) {  // :245-246
      reg->setInputTarget(frames[k]);
      prev = Eigen::Matrix4f::Identity();
    }
  }

  // ---- the awkward consumers, on the last frame's `aligned` (the walk must not end with a keyframe switch)
  auto tree = reg->getSearchMethodTarget();
  const size_t n = aligned.points.size();
  // a consumer restarting at 0 after the two full sweeps, then skipping: inside the look-ahead window, to its last slot, beyond it, back
  const size_t order[] = {0, 1, 2, 10, 11, 11 + 64, 11 + 64 + 1, 400, 401, 50, 49, 401, 402, n - 1, 0};
  put((double)(sizeof(order) / sizeof(order[0])));
  for (size_t i : order) { put((double)i); query(h, tree, aligned.points[i]); }
  // a sweep in steps of 64: every query lands on the last slot of the window behind the cursor
  { std::vector<int> ki; std::vector<float> kd; tree->nearestKSearch(aligned.points[0], 1, ki, kd); }
  int extra = 0, cnt = 0;
  for (size_t i = 64; i < n && cnt < 20; i += 64, cnt++) {
    const Counters a = counters(h);
    std::vector<int> ki;
    std::vector<float> kd;
    tree->nearestKSearch(aligned.points[i], 1, ki, kd);
    extra += (int)(counters(h).launches - a.launches);
  }
  put(cnt);
  put(extra);
  // a point that is not in the cloud, then the sweep goes on
  PointT odd = aligned.points[5];
  odd.x += 0.123f;
  put(odd.x); put(odd.y); put(odd.z);
  query(h, tree, odd);
  query(h, tree, aligned.points[6]);
  // the pointer early-outs: nothing is uploaded
  Counters a = counters(h);
  reg->setInputSource(frames[nf - 1]);
  const double up_src = counters(h).h2d - a.h2d;
  a = counters(h);
  reg->setInputTarget(frames[nf - 1 - 1]);  // NOT the current target unless the test made it so: see in.bin
  const double up_tgt_other = counters(h).h2d - a.h2d;
  a = counters(h);
  reg->setInputTarget(frames[nf - 1 - 1]);
  const double up_tgt_same = counters(h).h2d - a.h2d;
  put(up_src); put(up_tgt_other); put(up_tgt_same);
  // align twice on the same source: the cache of the first align must not serve the second
  Eigen::Matrix4f far = Eigen::Matrix4f::Identity();
  far.m[12] = 0.7f;
  reg->align(aligned, far);
  a = counters(h);
  put(reg->hasConverged());
  { const Eigen::Matrix4f T = reg->getFinalTransformation(); for (int i = 0; i < 16; i++) put(T.m[i]); }
  put(reg->getFitnessScore());
  put(counters(h).launches - a.launches);
  put((double)aligned.points.size());
  for (const PointT& p : aligned.points) { put(p.x); put(p.y); put(p.z); }
  // and a third align straight after that sweep, nothing set in between: only computeTransformation can invalidate the cache
  Eigen::Matrix4f other = Eigen::Matrix4f::Identity();
  other.m[13] = -0.5f;
  reg->align(aligned, other);
  a = counters(h);
  put(reg->hasConverged());
  { const Eigen::Matrix4f T = reg->getFinalTransformation(); for (int i = 0; i < 16; i++) put(T.m[i]); }
  put(reg->getFitnessScore());
  put(counters(h).launches - a.launches);
  // keyframe switch to the current source, then the SAME cloud as the next source: it has to be uploaded again and aligns onto itself
  reg->setInputTarget(frames[nf - 1]);
  a = counters(h);
  reg->setInputSource(frames[nf - 1]);
  put(counters(h).h2d - a.h2d);
  reg->align(aligned, Eigen::Matrix4f::Identity());
  put(reg->hasConverged());
  put(reg->getFitnessScore());
  // an empty source: align fails quietly, the sweeps have nothing to do
  auto empty = std::make_shared<Cloud>();
  reg->setInputSource(empty);
  reg->align(aligned, Eigen::Matrix4f::Identity());
  put(reg->hasConverged());
  put((double)aligned.points.size());
  put(reg->getFitnessScore() == std::numeric_limits<double>::max());

  f = std::fopen((dir + "/out.bin").c_str(), "wb");
  if (!f) return 4;
  std::fwrite(g_out.data(), sizeof(double), g_out.size(), f);
  std::fclose(f);
  return 0;
}
