// frontend_harness.cpp — runs adapter/b200_frontend.hpp (against the test-only adapter/pcl_shim.hpp, backend_shim.hpp and
// frontend_shim.hpp) the way PrefilteringNodelet and FloorDetectionNodelet drive it, for tests/test_frontend_adapter_gpu.py.
//
//   frontend_harness <in.bin> <out.bin> serial|concurrent
// in.bin: a list of jobs.  A job is one B200Prefilter or B200FloorDetector built from its rosparams, then a list of calls on it, each
// with the rosparams to set before it (scan_period between two calls), its input (a pcl cloud or a PointCloud2) and its arguments.
// Every number little-endian; strings are an int32 length and the bytes.
// out.bin: one length-prefixed block per job, the answers of its calls in order (see put_cloud and main).
// serial: the jobs one after the other.  concurrent: every job on its own thread at once; the blocks must be the serial ones.
#include "frontend_shim.hpp"
#include "b200_frontend.hpp"
#include <cstdio>
#include <cstring>
#include <thread>

using namespace hdl_graph_slam;
using PointT = pcl::PointXYZI;
using Cloud = pcl::PointCloud<PointT>;
using Block = std::vector<char>;

enum JobKind { PREFILTER = 1, FLOOR = 2 };
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
  std::vector<std::pair<std::string, std::string>> set;
  int32_t input = 0;  // 0: pcl cloud, 1: PointCloud2
  Cloud::Ptr cloud;
  sensor_msgs::PointCloud2 msg;
  int32_t has_imu = 0, has_tf = 0, want_filtered = 0, want_inliers = 0;
  Eigen::Vector3f imu;
  Eigen::Matrix4f tf;
};

struct Job {
  int32_t kind = 0;
  std::vector<std::pair<std::string, std::string>> params;
  std::vector<Call> calls;
};

static Call read_call(Reader& r, int32_t kind) {
  Call c;
  for (int32_t i = 0, n = r.get<int32_t>(); i < n && r.ok; i++) {
    std::string k = r.str();
    c.set.emplace_back(k, r.str());
  }
  c.input = r.get<int32_t>();
  const uint32_t seq = r.get<uint32_t>();
  const uint64_t stamp_us = r.get<uint64_t>();
  const std::string frame_id = r.str();
  if (c.input == 0) {
    c.cloud.reset(new Cloud());
    c.cloud->header.seq = seq;
    c.cloud->header.stamp = stamp_us;
    c.cloud->header.frame_id = frame_id;
    c.cloud->width = r.get<uint32_t>();
    c.cloud->height = r.get<uint32_t>();
    c.cloud->is_dense = r.get<int32_t>() != 0;
    c.cloud->points.resize(r.get<int64_t>());
    r.bytes(c.cloud->points.data(), c.cloud->points.size() * sizeof(PointT));
  } else {
    c.msg.header.seq = seq;
    c.msg.header.stamp.sec = (uint32_t)(stamp_us / 1000000ull);
    c.msg.header.stamp.nsec = (uint32_t)(stamp_us % 1000000ull) * 1000u;
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
  if (kind == PREFILTER) {
    c.has_imu = r.get<int32_t>();
    for (int i = 0; i < 3; i++) c.imu[i] = r.get<float>();
    c.has_tf = r.get<int32_t>();
    for (int i = 0; i < 16; i++) c.tf.m[i] = r.get<float>();
  } else {
    c.want_filtered = r.get<int32_t>();
    c.want_inliers = r.get<int32_t>();
  }
  return c;
}

static void run_job(const Job& job, Block& out) {
  ros::NodeHandle pnh;
  for (const auto& kv : job.params) pnh.setParam(kv.first, kv.second);
  std::unique_ptr<B200Prefilter> prefilter;
  std::unique_ptr<B200FloorDetector> floor;
  if (job.kind == PREFILTER) prefilter.reset(new B200Prefilter(pnh));
  else floor.reset(new B200FloorDetector(pnh));
  for (const Call& c : job.calls) {
    for (const auto& kv : c.set) pnh.setParam(kv.first, kv.second);  // the nodelet's copy of the handle sees it
    Block b;
    try {
      if (prefilter) {
        const Eigen::Vector3f* w = c.has_imu ? &c.imu : nullptr;
        const Eigen::Matrix4f* T = c.has_tf ? &c.tf : nullptr;
        Cloud::ConstPtr res = c.input == 0 ? prefilter->filter(Cloud::ConstPtr(c.cloud), w, T) : prefilter->filter(c.msg, w, T);
        put<int32_t>(b, OK);
        put_cloud(b, res.get());
      } else {
        boost::optional<Eigen::Vector4f> coeffs =
            c.input == 0 ? floor->detect(c.cloud, c.want_filtered != 0, c.want_inliers != 0) : floor->detect(c.msg, c.want_filtered != 0, c.want_inliers != 0);
        put<int32_t>(b, OK);
        put<int32_t>(b, coeffs ? 1 : 0);
        for (int i = 0; i < 4; i++) put<float>(b, coeffs ? (*coeffs)[i] : 0.f);
        const b2r_floor_result& r = floor->last_result();
        const char* p = reinterpret_cast<const char*>(&r);
        b.insert(b.end(), p, p + sizeof(r));
        put_cloud(b, floor->filtered().get());
        put_cloud(b, floor->inliers().get());
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
  if (argc != 4) {
    std::fprintf(stderr, "usage: frontend_harness in.bin out.bin serial|concurrent\n");
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
  try {
    if (std::strcmp(argv[3], "concurrent") == 0) {
      std::vector<std::thread> threads;
      for (size_t i = 0; i < jobs.size(); i++) threads.emplace_back(run_job, std::cref(jobs[i]), std::ref(blocks[i]));
      for (auto& t : threads) t.join();
    } else {
      for (size_t i = 0; i < jobs.size(); i++) run_job(jobs[i], blocks[i]);
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
  return 0;
}
