// odometry_harness.cpp — runs adapter/b200_odometry.hpp (against the test-only adapter/pcl_shim.hpp, backend_shim.hpp and
// frontend_shim.hpp) the way ScanMatchingOdometryNodelet drives it, for tests/test_odometry_adapter_gpu.py and
// tools/odometry_adapter_time.py.
//
//   odometry_harness <in.bin> <out.bin> serial|concurrent [times.bin]
// in.bin: a list of jobs.  A job is one B200ScanMatchingOdometry (kind 1) or B200Prefilter (kind 2) built from its rosparams, then a
// list of calls on it: the input (a pcl cloud or a PointCloud2, with its stamp as sec / nsec) and, for the odometry, msf_delta,
// want_status and want_aligned.  Every number little-endian; strings are an int32 length and the bytes.
// out.bin: one length-prefixed block per job, the answers of its calls in order (see run_job).
// serial: the jobs one after the other.  concurrent: every job on its own thread at once; the blocks must be the serial ones.
// times.bin: per call, the wall clock of the matching / filter call in nanoseconds (int64), jobs in order.
#include "frontend_shim.hpp"
#include "b200_odometry.hpp"
#include <chrono>
#include <cstdio>
#include <cstring>
#include <thread>

using namespace hdl_graph_slam;
using PointT = pcl::PointXYZI;
using Cloud = pcl::PointCloud<PointT>;
using Block = std::vector<char>;

enum JobKind { ODOMETRY = 1, PREFILTER = 2 };
enum Status { OK = 0, INVALID_ARGUMENT = 1, RUNTIME_ERROR = 2 };

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
  void bytes(void* p, size_t n) {
    if (n) ok = ok && std::fread(p, 1, n, f) == n;
  }
};

template <typename T>
static void put(Block& b, T v) {
  const char* p = reinterpret_cast<const char*>(&v);
  b.insert(b.end(), p, p + sizeof(T));
}
static void put_str(Block& b, const std::string& s) {
  put<int32_t>(b, (int32_t)s.size());
  b.insert(b.end(), s.begin(), s.end());
}
static void put_mat(Block& b, const Eigen::Matrix4f& m) {
  for (int i = 0; i < 16; i++) put<float>(b, m.data()[i]);
}
// present, header (seq, stamp, frame_id), width, height, is_dense, size, records
static void put_cloud(Block& b, const Cloud* c) {
  put<int32_t>(b, c ? 1 : 0);
  if (!c) return;
  put<uint32_t>(b, c->header.seq);
  put<uint64_t>(b, c->header.stamp);
  put_str(b, c->header.frame_id);
  put<uint32_t>(b, c->width);
  put<uint32_t>(b, c->height);
  put<int32_t>(b, c->is_dense ? 1 : 0);
  put<int64_t>(b, (int64_t)c->points.size());
  const char* p = reinterpret_cast<const char*>(c->points.data());
  b.insert(b.end(), p, p + c->points.size() * sizeof(PointT));
}

struct Call {
  int32_t input = 0;  // 0: pcl cloud, 1: PointCloud2
  ros::Time stamp;
  Cloud::Ptr cloud;
  sensor_msgs::PointCloud2 msg;
  int32_t has_msf = 0, want_status = 0, want_aligned = 0;
  Eigen::Matrix4f msf;
};

struct Job {
  int32_t kind = 0;
  std::vector<std::pair<std::string, std::string>> params;
  std::vector<Call> calls;
};

static Call read_call(Reader& r, int32_t kind) {
  Call c;
  c.input = r.get<int32_t>();
  const uint32_t seq = r.get<uint32_t>();
  c.stamp.sec = r.get<uint32_t>();
  c.stamp.nsec = r.get<uint32_t>();
  const std::string frame_id = r.str();
  if (c.input == 0) {
    c.cloud.reset(new Cloud());
    c.cloud->header.seq = seq;
    c.cloud->header.stamp = c.stamp.toNSec() / 1000ull;  // as pcl_conversions::toPCL
    c.cloud->header.frame_id = frame_id;
    c.cloud->width = r.get<uint32_t>();
    c.cloud->height = r.get<uint32_t>();
    c.cloud->is_dense = r.get<int32_t>() != 0;
    c.cloud->points.resize(r.get<int64_t>());
    r.bytes(c.cloud->points.data(), c.cloud->points.size() * sizeof(PointT));
  } else {
    c.msg.header.seq = seq;
    c.msg.header.stamp = c.stamp;
    c.msg.header.frame_id = frame_id;
    c.msg.width = r.get<uint32_t>();
    c.msg.height = r.get<uint32_t>();
    c.msg.point_step = r.get<uint32_t>();
    c.msg.row_step = r.get<uint32_t>();
    c.msg.is_bigendian = (uint8_t)r.get<int32_t>();
    c.msg.is_dense = (uint8_t)r.get<int32_t>();
    for (int32_t i = 0, n = r.get<int32_t>(); i < n && r.ok; i++) {
      sensor_msgs::PointField f;
      f.name = r.str();
      f.offset = r.get<uint32_t>();
      f.datatype = (uint8_t)r.get<int32_t>();
      f.count = r.get<uint32_t>();
      c.msg.fields.push_back(f);
    }
    c.msg.data.resize(r.get<int64_t>());
    r.bytes(c.msg.data.data(), c.msg.data.size());
  }
  if (kind == ODOMETRY) {
    c.has_msf = r.get<int32_t>();
    for (int i = 0; i < 16; i++) c.msf.m[i] = r.get<float>();  // column-major
    c.want_status = r.get<int32_t>();
    c.want_aligned = r.get<int32_t>();
  }
  return c;
}

// per odometry call: OK, the returned pose, converged, final_transformation, matching_error, inlier_fraction, keyframe_updated,
// frame_rejected, keyframe_pose, aligned (put_cloud); per prefilter call: OK and the filtered cloud.  An exception: its status and text.
static void run_job(const Job& job, Block& out, std::vector<int64_t>& times) {
  ros::NodeHandle pnh;
  for (const auto& kv : job.params) pnh.setParam(kv.first, kv.second);
  std::unique_ptr<B200ScanMatchingOdometry> odom;
  std::unique_ptr<B200Prefilter> prefilter;
  if (job.kind == ODOMETRY) odom.reset(new B200ScanMatchingOdometry(pnh));
  else prefilter.reset(new B200Prefilter(pnh));
  for (const Call& c : job.calls) {
    Block b;
    try {
      const auto t0 = std::chrono::steady_clock::now();
      if (odom) {
        const Eigen::Matrix4f* msf = c.has_msf ? &c.msf : nullptr;
        const Eigen::Matrix4f pose = c.input == 0 ? odom->matching(c.stamp, Cloud::ConstPtr(c.cloud), msf, c.want_status != 0, c.want_aligned != 0)
                                                  : odom->matching(c.msg, msf, c.want_status != 0, c.want_aligned != 0);
        times.push_back(std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count());
        put<int32_t>(b, OK);
        put_mat(b, pose);
        put<int32_t>(b, odom->converged() ? 1 : 0);
        put_mat(b, odom->final_transformation());
        put<double>(b, odom->matching_error());
        put<float>(b, odom->inlier_fraction());
        put<int32_t>(b, odom->keyframe_updated() ? 1 : 0);
        put<int32_t>(b, odom->frame_rejected() ? 1 : 0);
        put_mat(b, odom->keyframe_pose());
        put_cloud(b, odom->aligned().get());
      } else {
        Cloud::ConstPtr res = prefilter->filter(Cloud::ConstPtr(c.cloud), nullptr, nullptr);
        times.push_back(std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count());
        put<int32_t>(b, OK);
        put_cloud(b, res.get());
      }
    } catch (const std::invalid_argument& e) {
      b.clear();
      put<int32_t>(b, INVALID_ARGUMENT);
      put_str(b, e.what());
    } catch (const std::runtime_error& e) {
      b.clear();
      put<int32_t>(b, RUNTIME_ERROR);
      put_str(b, e.what());
    }
    put<int64_t>(out, (int64_t)b.size());
    out.insert(out.end(), b.begin(), b.end());
  }
}

int main(int argc, char** argv) {
  if (argc != 4 && argc != 5) {
    std::fprintf(stderr, "usage: odometry_harness in.bin out.bin serial|concurrent [times.bin]\n");
    return 2;
  }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  Reader r{f};
  std::vector<Job> jobs(r.get<int32_t>());
  for (Job& j : jobs) {
    j.kind = r.get<int32_t>();
    for (int32_t i = 0, n = r.get<int32_t>(); i < n && r.ok; i++) {
      std::string k = r.str();
      j.params.emplace_back(k, r.str());
    }
    for (int32_t i = 0, n = r.get<int32_t>(); i < n && r.ok; i++) j.calls.push_back(read_call(r, j.kind));
  }
  std::fclose(f);
  if (!r.ok) {
    std::fprintf(stderr, "short input\n");
    return 2;
  }
  std::vector<Block> blocks(jobs.size());
  std::vector<std::vector<int64_t>> times(jobs.size());
  try {
    if (std::strcmp(argv[3], "concurrent") == 0) {
      std::vector<std::thread> threads;
      for (size_t i = 0; i < jobs.size(); i++) threads.emplace_back(run_job, std::cref(jobs[i]), std::ref(blocks[i]), std::ref(times[i]));
      for (auto& t : threads) t.join();
    } else {
      for (size_t i = 0; i < jobs.size(); i++) run_job(jobs[i], blocks[i], times[i]);
    }
  } catch (const std::exception& e) {
    std::fprintf(stderr, "constructor: %s\n", e.what());
    return 3;
  }
  FILE* o = std::fopen(argv[2], "wb");
  if (!o) return 2;
  for (const Block& b : blocks) {
    const int64_t n = (int64_t)b.size();
    std::fwrite(&n, sizeof n, 1, o);
    std::fwrite(b.data(), 1, b.size(), o);
  }
  std::fclose(o);
  if (argc == 5) {
    FILE* t = std::fopen(argv[4], "wb");
    if (!t) return 2;
    for (const auto& v : times) std::fwrite(v.data(), sizeof(int64_t), v.size(), t);
    std::fclose(t);
  }
  return 0;
}
