// ingest.cuh — wire / disk formats at the seam ("next" row, SURVEY.md §8f-4): sensor_msgs/PointCloud2 blobs and binary PCD bodies are
// uploaded AS THEY ARE and unpacked into PointXYZI records on the device, instead of the host-side pcl::fromROSMsg /
// pcl::io::loadPCDFile conversions at /root/reference/apps/scan_matching_odometry_nodelet.cpp:118-119,
// apps/hdl_graph_slam_nodelet.cpp:153-154 and src/hdl_graph_slam/keyframe.cpp:57,141.
//   k_unpack_points   <- pcl::fromROSMsg / the PCD reader's field mapping for PointXYZI: x, y, z (FLOAT32) and intensity picked from
//                        arbitrary byte offsets of a point_step-long record.  As in PCL, a field is mapped only when its datatype
//                        and count match the point type's, so intensity is read only when it is FLOAT32; any other intensity
//                        field is left unmapped and the point keeps intensity 0.  is_bigendian byte-swaps (PCL copies native bytes).
//   k_unpack_points_rows <- the same for organized messages with padded rows (row_step > width * point_step).
#pragma once
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "engine.cuh"

namespace b2r {

struct UnpackArgs {
  const unsigned char* data;
  long long n;
  unsigned int point_step, off_x, off_y, off_z, off_i, bigendian;  // off_i = 0xffffffff: no FLOAT32 intensity
  float* out;  // 8 floats per point: x y z 1 | intensity 0 0 0  (pcl::PointXYZI)
};

__device__ __forceinline__ unsigned int load_u32(const unsigned char* p, bool swap) {
  unsigned int v = (unsigned int)p[0] | ((unsigned int)p[1] << 8) | ((unsigned int)p[2] << 16) | ((unsigned int)p[3] << 24);  // unaligned-safe
  return swap ? __byte_perm(v, 0, 0x0123) : v;
}

__global__ void k_unpack_points(const __grid_constant__ UnpackArgs A) {
  const bool swap = A.bigendian != 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < A.n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned char* r = A.data + (size_t)i * A.point_step;
    float* o = A.out + (size_t)i * 8;
    o[0] = __uint_as_float(load_u32(r + A.off_x, swap));
    o[1] = __uint_as_float(load_u32(r + A.off_y, swap));
    o[2] = __uint_as_float(load_u32(r + A.off_z, swap));
    o[3] = 1.0f;
    o[4] = A.off_i != 0xffffffffu ? __uint_as_float(load_u32(r + A.off_i, swap)) : 0.f;
    o[5] = 0.f; o[6] = 0.f; o[7] = 0.f;
  }
}

// k_unpack_points_rows <- the same mapping for an organized message whose rows are padded (row_step > width * point_step), which
// fromROSMsg accepts: record i sits at (i / width) * row_step + (i % width) * point_step.  Kept apart from k_unpack_points so the
// contiguous path's code stays as it is.
struct UnpackRowsArgs {
  const unsigned char* data;
  long long n;
  unsigned int width, row_step;
  unsigned int point_step, off_x, off_y, off_z, off_i, bigendian;
  float* out;
};

__global__ void k_unpack_points_rows(const __grid_constant__ UnpackRowsArgs A) {
  const bool swap = A.bigendian != 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < A.n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned char* r = A.data + (size_t)(i / A.width) * A.row_step + (size_t)(i % A.width) * A.point_step;
    float* o = A.out + (size_t)i * 8;
    o[0] = __uint_as_float(load_u32(r + A.off_x, swap));
    o[1] = __uint_as_float(load_u32(r + A.off_y, swap));
    o[2] = __uint_as_float(load_u32(r + A.off_z, swap));
    o[3] = 1.0f;
    o[4] = A.off_i != 0xffffffffu ? __uint_as_float(load_u32(r + A.off_i, swap)) : 0.f;
    o[5] = 0.f; o[6] = 0.f; o[7] = 0.f;
  }
}

// ---- binary PCD header (the files KeyFrame::save writes with pcl::io::savePCDFileBinary, keyframe.cpp:57)
struct PcdHeader {
  std::vector<std::string> fields;
  std::vector<int> size, count;
  std::vector<char> type;
  size_t points = 0, width = 0, height = 1, data_offset = 0;
  std::string data;  // "binary", "ascii", "binary_compressed"
};

inline bool pcd_parse_header(FILE* f, PcdHeader& H) {
  char line[4096];
  long pos = 0;
  bool have_points = false;
  while (fgets(line, sizeof(line), f)) {
    pos = ftell(f);
    std::string s(line);
    while (!s.empty() && (s.back() == '\n' || s.back() == '\r' || s.back() == ' ')) s.pop_back();
    if (s.empty() || s[0] == '#') continue;
    std::vector<std::string> tok;
    size_t a = 0;
    while (a < s.size()) {
      while (a < s.size() && (s[a] == ' ' || s[a] == '\t')) a++;
      size_t b = a;
      while (b < s.size() && s[b] != ' ' && s[b] != '\t') b++;
      if (b > a) tok.push_back(s.substr(a, b - a));
      a = b;
    }
    if (tok.empty()) continue;
    const std::string& k = tok[0];
    if (k == "FIELDS" || k == "COLUMNS") H.fields.assign(tok.begin() + 1, tok.end());
    else if (k == "SIZE") { H.size.clear(); for (size_t i = 1; i < tok.size(); i++) H.size.push_back(atoi(tok[i].c_str())); }
    else if (k == "TYPE") { H.type.clear(); for (size_t i = 1; i < tok.size(); i++) H.type.push_back(tok[i][0]); }
    else if (k == "COUNT") { H.count.clear(); for (size_t i = 1; i < tok.size(); i++) H.count.push_back(atoi(tok[i].c_str())); }
    else if (k == "WIDTH" && tok.size() > 1) H.width = strtoull(tok[1].c_str(), nullptr, 10);
    else if (k == "HEIGHT" && tok.size() > 1) H.height = strtoull(tok[1].c_str(), nullptr, 10);
    else if (k == "POINTS" && tok.size() > 1) { H.points = strtoull(tok[1].c_str(), nullptr, 10); have_points = true; }
    else if (k == "DATA" && tok.size() > 1) { H.data = tok[1]; H.data_offset = (size_t)pos; break; }
  }
  if (!have_points) H.points = H.width * H.height;
  if (H.count.empty()) H.count.assign(H.fields.size(), 1);
  return !H.data.empty() && !H.fields.empty() && H.size.size() == H.fields.size() && H.type.size() == H.fields.size() && H.count.size() == H.fields.size();
}

}  // namespace b2r
