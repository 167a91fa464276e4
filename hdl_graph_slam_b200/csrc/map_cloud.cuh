// map_cloud.cuh — MapCloudGenerator::generate on the device ("next" row, SURVEY.md §8f-3).
//
// Reference: /root/reference/src/hdl_graph_slam/map_cloud_generator.cpp:13-51 (called from apps/hdl_graph_slam_nodelet.cpp:528,989):
//   for every keyframe snapshot: dst = pose.cast<float>() * src (Vector4f, w = 1), intensity copied, all keyframes concatenated;
//   resolution <= 0: that cloud is the result; otherwise pcl::octree::OctreePointCloud(resolution).addPointsFromInputCloud() and
//   getOccupiedVoxelCenters().
// The octree's bounding box (its float64 min corner defines the voxel lattice) is grown in insertion order; that sequential process
// is replayed exactly on the device (k_oct_first_violator / k_oct_grow: only the few dozen points that ever violate the box
// matter).  Then: one transform kernel over all keyframes, 3 x 21-bit voxel keys (point - min) / resolution in float64, a radix
// sort of the keys (cub::DeviceRadixSort — 10^7..10^8 keys, far beyond the cluster sort's reach), unique, centres
// (key + 0.5) resolution + min.  The result is the same SET of centres as PCL's; PCL emits them in octree traversal order, here
// they come out in ascending (z, y, x) key order — the consumers (rviz, save_map) do not depend on the order.
// b2r_batch_map_cloud_generate builds the same concatenated cloud from a batch's cached keyframes (k_map_gather) instead of
// uploading them; everything after the transform is shared.
#pragma once
#include <cub/device/device_radix_sort.cuh>
#include "engine.cuh"

namespace b2r {

struct MapKf {            // one keyframe snapshot on the device
  const float* pts;       // records (device)
  long long first;        // index of its first point in the concatenated cloud
  int n;
  int pad;
  float T[12];            // rows 0..2 of pose.cast<float>()
};

// pcl::octree::OctreePointCloud's bounding box (float64 min / max / resolution, as PCL keeps them) and its growth state
struct MapGeom {
  double mn[3], mx[3];
  double r;
  int depth;
  int defined;
  int done;
  int overflow;           // depth beyond 21 bits per axis
};

// dst = pose * src (Eigen Matrix4f * Vector4f, column accumulation ((m0 x + m1 y) + m2 z) + m3, w = 1), other fields copied
__global__ void k_map_transform(const MapKf* __restrict__ kfs, int n_kf, int stride_f, long long total, float* __restrict__ out) {
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long long)gridDim.x * blockDim.x) {
    int lo = 0, hi = n_kf - 1;  // keyframe of point g: last one with first <= g
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (kfs[mid].first <= g) lo = mid; else hi = mid - 1; }
    const MapKf& K = kfs[lo];
    const float* p = K.pts + (size_t)(g - K.first) * stride_f;
    float* o = out + (size_t)g * stride_f;
    const float x = p[0], y = p[1], z = p[2];
    for (int k = 3; k < stride_f; k++) o[k] = p[k];
    o[0] = xform_row(K.T[0], K.T[1], K.T[2], K.T[3], x, y, z);
    o[1] = xform_row(K.T[4], K.T[5], K.T[6], K.T[7], x, y, z);
    o[2] = xform_row(K.T[8], K.T[9], K.T[10], K.T[11], x, y, z);
    if (stride_f >= 4) o[3] = 1.0f;
  }
}

// one keyframe of a b2r_batch's cache, read through its search structure (bvh_build.cuh): the raw records of a device-added
// cloud belong to the caller and are gone once the structure is built, the BVH-sorted copy is the engine's own
struct MapCachedKf {
  const float4* sorted;   // (x, y, z, bits(original index)), ascending (Hilbert key, original index)
  const int* pos_of;      // original index -> sorted position; -1 = a non-finite point, dropped from the structure
  long long first;        // index of its first point in the concatenated cloud
  float T[12];            // rows 0..2 of pose.cast<float>()
};

// dst[first + i] = pose * src[i] for point i of every keyframe, in the original point order (the box replay below depends on it),
// packed as float4 (only x, y, z are read downstream).  A point the structure dropped comes out as NaN: pose * (a non-finite
// point) is non-finite on every axis, so the octree skips either one alike.
__global__ void k_map_gather(const MapCachedKf* __restrict__ kfs, int n_kf, long long total, float4* __restrict__ out) {
  const float qnan = __int_as_float(0x7fc00000);
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long long)gridDim.x * blockDim.x) {
    int lo = 0, hi = n_kf - 1;  // keyframe of point g: last one with first <= g
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (kfs[mid].first <= g) lo = mid; else hi = mid - 1; }
    const MapCachedKf& K = kfs[lo];
    const int s = K.pos_of[g - K.first];
    float4 o = make_float4(qnan, qnan, qnan, qnan);
    if (s >= 0) {
      const float4 p = K.sorted[s];
      o.x = xform_row(K.T[0], K.T[1], K.T[2], K.T[3], p.x, p.y, p.z);
      o.y = xform_row(K.T[4], K.T[5], K.T[6], K.T[7], p.x, p.y, p.z);
      o.z = xform_row(K.T[8], K.T[9], K.T[10], K.T[11], p.x, p.y, p.z);
      o.w = 1.0f;
    }
    out[g] = o;
  }
}

// The box is grown exactly as addPointsFromInputCloud grows it (adoptBoundingBoxToPoint, UPSTREAM-RECALL of PCL 1.10): points are
// inserted in index order; the first finite point defines min/max = p -+ resolution/2; a point outside [min, max) doubles the box
// (depth + 1) towards itself until it fits.  Only the violators matter, so the sequential process is replayed as: find the FIRST
// point (lowest index) outside the current box (parallel, atomicMin), grow the box for it (one thread), repeat until nothing
// violates.
__global__ void k_oct_init(MapGeom* g, double r, unsigned long long* first_idx) {
  MapGeom G;
  for (int d = 0; d < 3; d++) { G.mn[d] = 0; G.mx[d] = 0; }
  G.r = r; G.depth = 0; G.defined = 0; G.done = 0; G.overflow = 0;
  *g = G;
  *first_idx = 0xffffffffffffffffull;
}

__global__ void k_oct_first_violator(const float* __restrict__ cloud, int stride_f, long long total, const MapGeom* __restrict__ gp, unsigned long long* first_idx) {
  const MapGeom G = *gp;
  if (G.done) return;
  unsigned long long fi = 0xffffffffffffffffull;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long long)gridDim.x * blockDim.x) {
    const float* p = cloud + (size_t)g * stride_f;
    const float x = p[0], y = p[1], z = p[2];
    if (!finite3(x, y, z)) continue;
    const bool out = !G.defined || (double)x < G.mn[0] || (double)y < G.mn[1] || (double)z < G.mn[2] || (double)x >= G.mx[0] || (double)y >= G.mx[1] || (double)z >= G.mx[2];
    if (out) { fi = (unsigned long long)g; break; }  // this thread's indices ascend: its first violator is its lowest
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const unsigned long long t = __shfl_xor_sync(0xffffffffu, fi, o); fi = t < fi ? t : fi; }
  if ((threadIdx.x & 31) == 0 && fi != 0xffffffffffffffffull) atomicMin(first_idx, fi);
}

__global__ void k_oct_grow(const float* __restrict__ cloud, int stride_f, MapGeom* gp, unsigned long long* first_idx) {
  MapGeom G = *gp;
  if (G.done) return;
  const unsigned long long idx = *first_idx;
  *first_idx = 0xffffffffffffffffull;
  if (idx == 0xffffffffffffffffull) { G.done = 1; *gp = G; return; }
  const float* p = cloud + (size_t)idx * stride_f;
  const double q[3] = {(double)p[0], (double)p[1], (double)p[2]};
  const double eps = (double)1.1920928955078125e-07f;  // std::numeric_limits<float>::epsilon()
  for (int guard = 0; guard < 64; guard++) {
    bool lower[3], upper[3], any = false;
    for (int d = 0; d < 3; d++) { lower[d] = q[d] < G.mn[d]; upper[d] = q[d] >= G.mx[d]; any |= lower[d] | upper[d]; }
    if (G.defined && !any) break;
    if (G.defined) {
      double side = (double)(1 << G.depth) * G.r;
      for (int d = 0; d < 3; d++) if (!upper[d]) G.mn[d] -= side;
      G.depth++;
      side = (double)(1 << G.depth) * G.r - eps;
      for (int d = 0; d < 3; d++) G.mx[d] = G.mn[d] + side;
      if (G.depth > 21) { G.overflow = 1; G.done = 1; break; }
    } else {
      for (int d = 0; d < 3; d++) { G.mn[d] = q[d] - G.r / 2; G.mx[d] = q[d] + G.r / 2; }
      G.defined = 1;
    }
  }
  *gp = G;
}

__global__ void k_map_keys(const float* __restrict__ cloud, int stride_f, long long total, const MapGeom* __restrict__ gp, unsigned long long* keys) {
  const MapGeom G = *gp;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long long)gridDim.x * blockDim.x) {
    const float* p = cloud + (size_t)g * stride_f;
    const float x = p[0], y = p[1], z = p[2];
    unsigned long long key = 0xffffffffffffffffull;  // non-finite points are not inserted (OctreePointCloud::addPointsFromInputCloud)
    if (finite3(x, y, z) && G.defined && !G.overflow) {
      // genOctreeKeyforPoint: key = static_cast<unsigned int>((point - min) / resolution), float64 (the subtraction explicitly rounded)
      const unsigned long long kx = (unsigned long long)(dsub((double)x, G.mn[0]) / G.r);
      const unsigned long long ky = (unsigned long long)(dsub((double)y, G.mn[1]) / G.r);
      const unsigned long long kz = (unsigned long long)(dsub((double)z, G.mn[2]) / G.r);
      key = (kz << 42) | (ky << 21) | kx;
    }
    keys[g] = key;
  }
}

// sorted keys -> one PointXYZI-shaped record per distinct key: the voxel centre (genLeafNodeCenterFromOctreeKey), data[3] = 1,
// intensity 0; `count` is bumped with one atomic per block (the slot of a head = number of heads before it)
__global__ void k_map_heads(const unsigned long long* __restrict__ keys, long long total, int* flags) {
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[g];
    flags[g] = (k != 0xffffffffffffffffull && (g == 0 || keys[g - 1] != k)) ? 1 : 0;
  }
}
__global__ void k_map_centers(const unsigned long long* __restrict__ keys, const int* __restrict__ flags, const int* __restrict__ slots, long long total,
                              const MapGeom* __restrict__ gp, int stride_f, float* __restrict__ out, int* n_out) {
  const MapGeom G = *gp;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long long)gridDim.x * blockDim.x) {
    if (g == total - 1) *n_out = slots[g] + flags[g];
    if (!flags[g]) continue;
    const unsigned long long k = keys[g];
    const unsigned long long kx = k & 0x1fffffull, ky = (k >> 21) & 0x1fffffull, kz = k >> 42;
    float* o = out + (size_t)slots[g] * stride_f;
    // genLeafNodeCenterFromOctreeKey: (key + 0.5f) * resolution + min, float64, narrowed to float.  Multiply and add are rounded
    // separately (dmul / dadd): a contracted DFMA rounds once and can move the centre by one float64 ulp, which the narrowing to
    // float may keep
    o[0] = (float)dadd(dmul(dadd((double)kx, 0.5), G.r), G.mn[0]);
    o[1] = (float)dadd(dmul(dadd((double)ky, 0.5), G.r), G.mn[1]);
    o[2] = (float)dadd(dmul(dadd((double)kz, 0.5), G.r), G.mn[2]);
    if (stride_f >= 4) o[3] = 1.0f;
    for (int q = 4; q < stride_f; q++) o[q] = 0.f;
  }
}

}  // namespace b2r
