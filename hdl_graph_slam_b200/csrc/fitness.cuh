// fitness.cuh — nearest-neighbour fitness score, inlier count, exact 1-NN queries and the `aligned` output cloud.
//
// k_fitness      <- pcl::Registration::getFitnessScore(max_range) (called at apps/scan_matching_odometry_nodelet.cpp:307,
//                   include/hdl_graph_slam/loop_detector.hpp:146; in-tree twin src/hdl_graph_slam/information_matrix_calculator.cpp:49-80)
//                   fused with the inlier loop of apps/scan_matching_odometry_nodelet.cpp:309-320
// k_fitness_batch <- the same score for every pair of a batch call, in one launch (loop_detector.hpp:146)
// k_nearest      <- getSearchMethodTarget()->nearestKSearch(pt, 1, ...) (apps/scan_matching_odometry_nodelet.cpp:316)
// k_transform    <- the `aligned` cloud written by align() (pcl::transformPointCloud with final_transformation_)
#pragma once
#include "common.cuh"
#include "bvh.cuh"
#include "gicp.cuh"
#include "pair_engine.cuh"  // PairReport

namespace b2r {

struct FitArgs {
  Bvh src;                // queries = the source's sorted points (a warp = one leaf = spatial neighbours)
  Bvh tgt;
  float Tf[12];
  double max_range;       // compared with the SQUARED distance (reference semantics)
  float inlier_thresh_sq;
  double* partials;       // [blocks][3]
  double* out;            // [3] = sum d2, count, inliers
  unsigned int* counter;
};

// one block's share of a fitness launch: its kLinThreads source points at the pose Tf (row-major 3x4), each point's nearest target
// point, and the block's sums (sum d2, count, inliers) reduced into acc
__device__ __forceinline__ void fitness_block(const FitArgs& A, const float* Tf, double* acc, double* red) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  acc[0] = acc[1] = acc[2] = 0.0;
  float4 p = make_float4(0.f, 0.f, 0.f, bits_idx(kPadIdx));
  if (s < A.src.nleaf * kLeaf) p = A.src.sp[s];
  float qx = 0.f, qy = 0.f, qz = 0.f;
  Nn1 v;
  v.reset(INFINITY);
  bool active = false;
  if (idx_bits(p.w) != kPadIdx) {
    qx = xform_row(Tf[0], Tf[1], Tf[2], Tf[3], p.x, p.y, p.z);
    qy = xform_row(Tf[4], Tf[5], Tf[6], Tf[7], p.x, p.y, p.z);
    qz = xform_row(Tf[8], Tf[9], Tf[10], Tf[11], p.x, p.y, p.z);
    active = finite3(qx, qy, qz);
  }
  bvh_group_search(A.tgt, qx, qy, qz, active, v, -1);
  if (active && v.best_pos >= 0) {
    if ((double)v.best_d2() <= A.max_range) { acc[0] = (double)v.best_d2(); acc[1] = 1.0; }
    if (v.best_d2() < A.inlier_thresh_sq) acc[2] = 1.0;
  }
  block_reduce<3>(acc, red);
}

__global__ void __launch_bounds__(kLinThreads, 4) k_fitness(const __grid_constant__ FitArgs A) {
  __shared__ double red[3 * 32];
  double acc[3];
  fitness_block(A, A.Tf, acc, red);
  finish_partials<3>(acc, A.partials, A.out, A.counter);
}

// getFitnessScore of many pairs at their final poses in ONE launch (blockIdx.y = pair): per pair exactly k_fitness's work, grid
// (nblk blocks of kLinThreads) and fixed-order reduction, so every score is bitwise b2r_fitness's.  The pose is read from the pair's
// report on the device (the float T the single handle stores as its final transformation); k_fitness_batch_store writes the score back.
struct FitItem {
  FitArgs A;                 // Tf unused: the pose comes from `rep`
  PairReport* rep;
  unsigned int nblk;         // = k_fitness's gridDim.x for this source
  unsigned int pad;
};
__global__ void __launch_bounds__(kLinThreads, 4) k_fitness_batch(const FitItem* __restrict__ items) {
  __shared__ double red[3 * 32];
  const FitItem& it = items[blockIdx.y];
  const unsigned int nblk = it.nblk;
  if (blockIdx.x >= nblk) return;  // before the reduction's block count: only the pair's own nblk blocks take part
  float Tf[12];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 4; c++) Tf[r * 4 + c] = it.rep->r.T[c * 4 + r];
  double acc[3];
  fitness_block(it.A, Tf, acc, red);
  finish_partials<3>(acc, it.A.partials, it.A.out, it.A.counter, nullptr, 0, nullptr, nblk);
}

// score = sum / count, DBL_MAX without a neighbour in range (as b2r_fitness computes it on the host, one IEEE division)
__global__ void k_fitness_batch_store(const FitItem* __restrict__ items, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* o = items[i].A.out;
  items[i].rep->r.fitness = o[1] > 0.0 ? o[0] / o[1] : DBL_MAX;
}

// queries in caller order (no spatial coherence guaranteed: still exact, only less efficient)
__global__ void __launch_bounds__(256, 2) k_nearest(const float* __restrict__ q_raw, int stride_f, int n, const __grid_constant__ Bvh tgt,
                                                    int* idx_out, float* d2_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float qx = 0.f, qy = 0.f, qz = 0.f;
  Nn1 v;
  v.reset(INFINITY);
  bool active = false;
  if (i < n) {
    const float* p = q_raw + (size_t)i * stride_f;
    qx = p[0]; qy = p[1]; qz = p[2];
    active = finite3(qx, qy, qz);
  }
  bvh_group_search(tgt, qx, qy, qz, active, v, -1);
  if (i < n) {
    idx_out[i] = v.best_pos >= 0 ? v.best_idx() : -1;
    d2_out[i] = v.best_d2();
  }
}

struct XfArg { float Tf[12]; };
__global__ void k_transform(const float* __restrict__ raw, int stride_f, int n, XfArg X, float4* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = raw + (size_t)i * stride_f;
  const float x = p[0], y = p[1], z = p[2];
  out[i] = make_float4(xform_row(X.Tf[0], X.Tf[1], X.Tf[2], X.Tf[3], x, y, z), xform_row(X.Tf[4], X.Tf[5], X.Tf[6], X.Tf[7], x, y, z),
                       xform_row(X.Tf[8], X.Tf[9], X.Tf[10], X.Tf[11], x, y, z), 1.0f);
}

// the `aligned_points` cloud of ScanMatchingOdometryNodelet::matching (:254-259), pcl::transformPointCloud(*cloud, *aligned, odom) of the
// frame's raw records: the record copied, then xyz as k_transform and 1.0f at float 3.  is_dense == 0: a record with a non-finite x,
// y or z stays as copied (PCL 1.10's non-dense branch, UPSTREAM-RECALL)
__global__ void k_transform_aligned_records(const float* __restrict__ in, int stride_f, int n, XfArg X, int is_dense, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = in + (size_t)i * stride_f;
  float* o = out + (size_t)i * stride_f;
  for (int k = 0; k < stride_f; k++) o[k] = p[k];
  const float x = p[0], y = p[1], z = p[2];
  if (!is_dense && !finite3(x, y, z)) return;
  o[0] = xform_row(X.Tf[0], X.Tf[1], X.Tf[2], X.Tf[3], x, y, z);
  o[1] = xform_row(X.Tf[4], X.Tf[5], X.Tf[6], X.Tf[7], x, y, z);
  o[2] = xform_row(X.Tf[8], X.Tf[9], X.Tf[10], X.Tf[11], x, y, z);
  if (stride_f > 3) o[3] = 1.0f;
}

}  // namespace b2r
