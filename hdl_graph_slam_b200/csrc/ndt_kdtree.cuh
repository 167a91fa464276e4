// ndt_kdtree.cuh — NDT_OMP with reg_nn_search_method = KDTREE (B2R_METHOD_NDT_KDTREE, opted into as `B200_NDT_KDTREE`).
//
// pclomp::NormalDistributionsTransform in KDTREE mode calls target_cells_.radiusSearch(x_trans_pt, resolution_) in both
// computeDerivatives and computeHessian.  ndt_omp's VoxelGridCovariance is a copy of PCL's, so that neighbourhood is pcl NDT's
// (ndt_pcl.cuh: the centroid cloud of k_pcl_centroids / k_pcl_buckets and the exact radius search pcl_collect) and the arithmetic
// is ndt_omp's (ndt.cuh).  Semantics pinned by tests/ndt_kdtree_ref.cpp (see its header):
//   k_ndt_kdtree_derivatives  <- computeDerivatives: ndt_pcl_derivatives_body with ndt_omp's float32 term (ndt_omp_term), read
//                                from the NdtCell at the neighbour's sorted position
//   k_ndt_kdtree_hessian      <- computeHessian / updateHessian: ndt_hessian_body's per-point setup and float64 term (ndt_hess_term)
//                                over the same radius neighbours, reading NdtVoxel; block_reduce / finish_partials
// A returned leaf is not checked for nr_points >= 6 (an invalidated leaf that has a centroid takes part with the inverse it holds),
// and no cell index is formed (DIRECT7's drop of points beyond 1e9 cells does not apply).
#pragma once

namespace b2r {

// ndt_omp's term rule for ndt_pcl_derivatives_body: the float32 point derivatives and the float32 term of DIRECT1 / DIRECT7
struct NdtKdtreeTermRule {
  template <bool HESS>
  using Point = NdtOmpPoint;
  template <bool HESS>
  static __device__ __forceinline__ void point(const NdtArgs& A, float x, float y, float z, NdtOmpPoint& pd) {
    ndt_omp_point<HESS>(A, x, y, z, pd);
  }
  template <bool HESS>
  static __device__ __forceinline__ void term(const NdtArgs& A, unsigned int s, float xt, float yt, float zt, const NdtOmpPoint& pd, double* acc,
                                              double* low) {
    ndt_omp_term<HESS>(A.d1, (float)A.d2, A.cells + s, xt, yt, zt, pd, acc, low);
  }
};

template <bool HESS>
__global__ void __launch_bounds__(kNdtThreads) k_ndt_kdtree_derivatives(const __grid_constant__ NdtPclArgs P) {
  ndt_pcl_derivatives_body<NdtKdtreeTermRule, HESS>(P);
}

// many pairs: blockIdx.y = the pair's record, each pair with its own tickets, rows and counters (as k_ndt_derivatives_batch)
template <bool HESS>
__global__ void __launch_bounds__(kNdtThreads) k_ndt_kdtree_derivatives_batch(const NdtPclArgs* __restrict__ recs) {
  ndt_pcl_derivatives_body<NdtKdtreeTermRule, HESS>(recs[blockIdx.y]);
}

// float64 Hessian-only pass over the radius neighbours (ascending (d2, leaf), as the derivative pass visits them); one thread per
// point, nrow = the source's 128-point blocks
__device__ __forceinline__ void ndt_kdtree_hessian_body(const NdtPclArgs& P, unsigned int nrow) {
  const NdtArgs& A = P.A;
  __shared__ double red[36 * 32];
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  double acc[36];
#pragma unroll
  for (int k = 0; k < 36; k++) acc[k] = 0.0;
  float4 pt = make_float4(0.f, 0.f, 0.f, bits_idx(kPadIdx));
  if (s < A.n_sorted) pt = A.src[s];
  if (idx_bits(pt.w) != kPadIdx) {
    const VoxGeom V = *A.geom;
    const float xf = pt.x, yf = pt.y, zf = pt.z;
    const float xt = xform_row(A.Tf[0], A.Tf[1], A.Tf[2], A.Tf[3], xf, yf, zf);
    const float yt = xform_row(A.Tf[4], A.Tf[5], A.Tf[6], A.Tf[7], xf, yf, zf);
    const float zt = xform_row(A.Tf[8], A.Tf[9], A.Tf[10], A.Tf[11], xf, yf, zf);
    if (!V.empty && V.ok && finite3(xt, yt, zt)) {
      double J[3][6] = {{1, 0, 0, 0, 0, 0}, {0, 1, 0, 0, 0, 0}, {0, 0, 1, 0, 0, 0}};
      double va[3], vb[3], vc[3], vd[3], ve[3], vf[3];
      ndt_hess_point(A, xf, yf, zf, J, va, vb, vc, vd, ve, vf);
      unsigned long long buf[kPclNb];
      long long after = -1;
      for (;;) {
        const int total = pcl_collect(P, V, xt, yt, zt, after, buf);
        const int m = min(total, kPclNb);
        for (int t = 0; t < m; t++) ndt_hess_term(A, A.vox + (unsigned int)buf[t], xt, yt, zt, J, va, vb, vc, vd, ve, vf, acc);
        if (total <= kPclNb) break;
        after = (long long)buf[kPclNb - 1];
      }
    }
  }
  block_reduce<36>(acc, red);
  finish_partials<36>(acc, A.partials, A.out, A.counter, A.flag, A.seq, nullptr, nrow, A.round, A.round_n);
}

__global__ void __launch_bounds__(kNdtThreads) k_ndt_kdtree_hessian(const __grid_constant__ NdtPclArgs P) { ndt_kdtree_hessian_body(P, gridDim.x); }

// many pairs: blockIdx.y = the pair's record, grid.x covers the largest source; block b of a pair is block b of its own pass
__global__ void __launch_bounds__(kNdtThreads) k_ndt_kdtree_hessian_batch(const NdtPclArgs* __restrict__ recs) {
  const NdtPclArgs& P = recs[blockIdx.y];
  const unsigned int nb = (unsigned int)P.A.n_sorted / kNdtThreads;
  if (blockIdx.x >= nb) return;  // block-uniform
  ndt_kdtree_hessian_body(P, nb);
}

// ------------------------------------------------------------------------------------------------ host side
// blocks of k_ndt_kdtree_derivatives the device holds at once, asked once per process (B2R_NDT_WAVES scales it, as for the others)
inline unsigned ndt_kdtree_resident_blocks(bool hess) {
  static unsigned cached[2] = {0, 0};
  unsigned& c = cached[hess ? 1 : 0];
  if (c == 0) {
    int dev = 0, sms = 132, per = 4;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (hess) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, k_ndt_kdtree_derivatives<true>, kNdtThreads, 0);
    else cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, k_ndt_kdtree_derivatives<false>, kNdtThreads, 0);
    if (const char* e = getenv("B2R_NDT_WAVES")) { const double w = atof(e); if (w > 0) per = std::max(1, (int)(per * w)); }
    c = (unsigned)std::max(1, sms * std::max(per, 1));
  }
  return c;
}

// the targets that carry the searchable centroid cloud (ndt_pcl_build): pcl NDT's, and NDT_OMP's KDTREE one
inline bool ndt_radius_family(int method) { return method == B2R_METHOD_NDT_PCL || method == B2R_METHOD_NDT_KDTREE; }

}  // namespace b2r
