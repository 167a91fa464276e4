// select_harness.cpp — builds the two drop-ins that configure a registration handle from a nodelet's reg_* rosparams
// (adapter/b200_select.hpp), B200KeyframeCache (b200_backend.hpp) and B200ScanMatchingOdometry (b200_odometry.hpp), against the
// test-only stand-ins, and reports the configuration each one's engine handle ended up with, for tests/test_odometry_methods_gpu.py.
//
//   select_harness <in.bin> <out.bin>
// in.bin : the rosparams: an int32 count, then per parameter the key and the value, each an int32 length and the bytes
// out.bin: per drop-in (the cache, then the odometry): int32 0 and the b2r_config of its handle (b2r_get_config), or int32 1 and the
//          std::runtime_error text its constructor threw (an int32 length and the bytes)
#include "frontend_shim.hpp"
#include "b200_backend.hpp"
#include "b200_odometry.hpp"
#include <cstdio>
#include <string>
#include <vector>

using namespace hdl_graph_slam;

// Test-only access to the odometry's private handle, so the header keeps no accessor for it: an explicit instantiation may name a
// private member, and the friend function it defines hands the member pointer out.
struct OdometryHandle {
  using type = b2r_handle* B200ScanMatchingOdometry::*;
  friend type member(OdometryHandle);
};
template <typename Tag, typename Tag::type M>
struct Expose {
  friend typename Tag::type member(Tag) { return M; }
};
template struct Expose<OdometryHandle, &B200ScanMatchingOdometry::h_>;

static std::string read_str(FILE* f, bool& ok) {
  int32_t n = 0;
  ok = ok && std::fread(&n, sizeof n, 1, f) == 1 && n >= 0;
  std::string s(ok ? n : 0, '\0');
  if (ok && n) ok = std::fread(&s[0], 1, s.size(), f) == s.size();
  return s;
}

static void put_config(std::vector<char>& out, const b2r_config& cfg) {
  const int32_t ok = 0;
  out.insert(out.end(), reinterpret_cast<const char*>(&ok), reinterpret_cast<const char*>(&ok) + sizeof ok);
  out.insert(out.end(), reinterpret_cast<const char*>(&cfg), reinterpret_cast<const char*>(&cfg) + sizeof cfg);
}

static void put_error(std::vector<char>& out, const std::string& what) {
  const int32_t status = 1, n = (int32_t)what.size();
  out.insert(out.end(), reinterpret_cast<const char*>(&status), reinterpret_cast<const char*>(&status) + sizeof status);
  out.insert(out.end(), reinterpret_cast<const char*>(&n), reinterpret_cast<const char*>(&n) + sizeof n);
  out.insert(out.end(), what.begin(), what.end());
}

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  bool ok = true;
  int32_t n = 0;
  ok = std::fread(&n, sizeof n, 1, f) == 1;
  ros::NodeHandle pnh;
  for (int32_t i = 0; i < n && ok; i++) {
    const std::string k = read_str(f, ok), v = read_str(f, ok);
    pnh.setParam(k, v);
  }
  std::fclose(f);
  if (!ok) return 2;
  std::vector<char> out;
  try {
    B200KeyframeCache cache(pnh);
    b2r_handle* eng = nullptr;
    b2r_config cfg;
    B200KeyframeCache::check(b2r_batch_get_engine(cache.batch(), &eng));
    B200KeyframeCache::check(b2r_get_config(eng, &cfg));
    put_config(out, cfg);
  } catch (const std::runtime_error& e) {
    put_error(out, e.what());
  }
  try {
    B200ScanMatchingOdometry odom(pnh);
    b2r_config cfg;
    b200_select::check(b2r_get_config(odom.*member(OdometryHandle()), &cfg));
    put_config(out, cfg);
  } catch (const std::runtime_error& e) {
    put_error(out, e.what());
  }
  FILE* o = std::fopen(argv[2], "wb");
  if (!o) return 2;
  std::fwrite(out.data(), 1, out.size(), o);
  std::fclose(o);
  return 0;
}
