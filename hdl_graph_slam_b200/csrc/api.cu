// api.cu — C ABI of libb200reg.so (see include/b200reg.h) and the host-side drivers above the kernels.
//
// Host mirrors of the reference interface for this path (same names / argument meaning / failure behaviour):
//   b2r_select_registration_method  <- select_registration_method            src/hdl_graph_slam/registrations.cpp:22-124
//   b2r_set_target / b2r_set_source <- pcl::Registration::setInputTarget/Source   (call sites in b200reg.h)
//   b2r_align                       <- pcl::Registration::align -> computeTransformation (fast_gicp LsqRegistration LM loop,
//                                      ndt_omp Newton + More-Thuente loop; SURVEY.md A.2, A.4)
//   b2r_fitness                     <- getFitnessScore
//   b2r_odometry_matching           <- ScanMatchingOdometryNodelet::matching  apps/scan_matching_odometry_nodelet.cpp:165-262
//   b2r_loop_matching               <- LoopDetector::matching                include/hdl_graph_slam/loop_detector.hpp:117-171
// There is deliberately NO CPU fallback in this file: every compute step is a CUDA kernel launch.
#include <cuda_runtime.h>
#include <cmath>
#include <cfloat>
#include <cstdlib>
#include <string>
#include <vector>
#include <algorithm>
#include <cub/device/device_radix_sort.cuh>
#include "engine.cuh"
#include "gicp.cuh"
#include "pair_engine.cuh"
#include "bvh_build.cuh"
#include "fitness.cuh"
#include "ndt.cuh"
#include "voxelgrid.cuh"
#include "prefilter.cuh"
#include "map_cloud.cuh"
#include "ingest.cuh"
#include "loop_gate.cuh"

#ifndef B2R_PREFETCH_KNN_BLOCKS_DEFAULT
#define B2R_PREFETCH_KNN_BLOCKS_DEFAULT 0  // 0 = no cap on the prefetch stream's k-NN kernel
#endif

namespace b2r {
thread_local std::string g_last_error;
}
using namespace b2r;

struct b2r_handle {
  b2r_config cfg;
  cudaStream_t st = nullptr;
  Cloud aux;                        // scratch cloud of the prefilter entry points (never a registration input)
  Cloud clouds[3];
  int src = 0, tgt = 1, nxt = 2;   // nxt: cloud being prefetched for the next set_source (software pipelining)
  cudaStream_t st2 = nullptr;       // prefetch stream (upload + BVH + covariances of the next source overlap the current align)
  cudaEvent_t ev_prefetch = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;  // first LM round beside the source's k-NN covariance kernel (run_single_pair)
  bool prefetched = false;
  unsigned long long prefetch_stamp = 0;   // content stamp of the prefetched host cloud (content_stamp)
  cudaEvent_t upload_ev = nullptr;         // end of the last DMA out of a caller-owned pinned buffer
  bool upload_pending = false;
  // per-align workspaces (sized by the source)
  DevBuf<int> corr[2], cpos[2];     // double-buffered: a speculative linearisation writes the other set
  DevBuf<float> d2;
  DevBuf<double> mahal[2], partials;
  int cur = 0;                      // buffer set holding the correspondences of the last ACCEPTED linearisation
  // device-resident LM (pair_engine.cuh): the handle's single pair record and its host-mapped mailbox
  PairDev* d_pair = nullptr;
  PairReport* h_rep = nullptr; PairReport* h_rep_dev = nullptr;          // report record (128 B, checksummed message)
  unsigned long long* h_pflag = nullptr; unsigned long long* h_pflag_dev = nullptr;  // [0] publication flag, [1] progress word
  double* h_tap = nullptr; double* h_tap_dev = nullptr;                  // parity taps: 29 reduced values
  int last_rounds = 0;              // rounds the previous align needed: that many (+1) are enqueued up front by the next one
  struct b2r_batch* loop_batch = nullptr;  // b2r_loop_matching runs the candidates of a keyframe as one batch (created on first use)
  double* d_out = nullptr;          // 64 doubles
  unsigned int* d_counter = nullptr;
  double* h_out = nullptr;          // pinned + mapped, 64 doubles + flags: reduction kernels write results here directly
  double* h_out_dev = nullptr;      // device alias
  unsigned long long* h_flag = nullptr; unsigned long long* h_flag_dev = nullptr; unsigned long long seq = 0;
  // staging for pageable uploads
  void* staging[3] = {nullptr, nullptr, nullptr};
  size_t staging_cap[3] = {0, 0, 0};
  cudaEvent_t staging_ev[3] = {nullptr, nullptr, nullptr};
  // misc device scratch (queries / outputs)
  DevBuf<float> tmp_f;
  DevBuf<int> tmp_i;
  DevBuf<float4> tmp_f4;
  // device-resident prefilter chain: ping-pong record buffers, keep flags, compaction scratch
  DevBuf<float> pf_buf[2];
  DevBuf<unsigned char> pf_flags;
  DevBuf<int> pf_blocks;
  DevBuf<char> ingest_blob;         // PointCloud2 / PCD bodies as uploaded, and their PointXYZI unpacking
  DevBuf<float> ingest_out;
  void* ingest_pinned = nullptr; size_t ingest_pinned_cap = 0;
  DevBuf<char> map_kf;              // MapCloudGenerator: keyframe descriptors, voxel keys
  DevBuf<unsigned long long> map_keys[2];
  MapGeom* map_geom = nullptr;
  int* map_h = nullptr;
  SorStats* pf_stats = nullptr;
  int* pf_total = nullptr;
  int* pf_h_total = nullptr; int* pf_h_total_dev = nullptr;
  BuildCtx bc[2];                   // per-stream build scratch (main stream, prefetch stream)
  bool knn_smem_attr = false, stat_smem_attr = false;
  int n_sm = 132;
  // last result
  float final_T[16];                // row-major
  bool has_final = false;
  bool corr_valid = false;
  NdtWork ndt_work;
  VoxelWork vg_work;
  Telemetry tel;
};

static Cloud& SRC(b2r_handle* h) { return h->clouds[h->src]; }
static Cloud& TGT(b2r_handle* h) { return h->clouds[h->tgt]; }

extern "C" const char* b2r_last_error(void) { return g_last_error.c_str(); }
extern "C" const char* b2r_version(void) { return "b200reg 0.1 (sm_90a)"; }

extern "C" int b2r_config_default(b2r_config* c, int method) {
  if (!c) return fail(B2R_EINVAL, "cfg is NULL");
  std::memset(c, 0, sizeof(*c));
  c->method = method;
  c->device_id = 0;
  c->max_iterations = 64;             // registrations.cpp:32,110
  c->k_correspondences = 20;          // :34
  c->transformation_epsilon = 0.01;   // :31,109
  c->rotation_epsilon = 2e-3;         // fast_gicp default
  c->max_correspondence_distance = 2.5;  // :33
  c->ndt_resolution = 0.5;            // :93
  c->ndt_step_size = 0.1;             // ndt_omp default (never overridden by the factory)
  c->ndt_outlier_ratio = 0.55;
  c->ndt_search_method = 7;           // :103 DIRECT7
  c->ndt_mt_interval_flag = 0;
  c->ndt_fixed_iterations = 0;
  c->grid_cell_min = 0.5f;
  if (method != B2R_METHOD_GICP && method != B2R_METHOD_NDT) return fail(B2R_EINVAL, "unknown method");
  return B2R_OK;
}

static const char* find_param(const char* const* keys, const char* const* values, int n, const char* key) {
  for (int i = 0; i < n; i++)
    if (keys[i] && std::strcmp(keys[i], key) == 0) return values[i];
  return nullptr;
}

extern "C" int b2r_select_registration_method(const char* const* keys, const char* const* values, int n, int device_id,
                                              b2r_handle** out) {
  if (!out) return fail(B2R_EINVAL, "out is NULL");
  *out = nullptr;
  const char* m = find_param(keys, values, n, "registration_method");
  std::string method = m ? m : "NDT_OMP";  // registrations.cpp:26
  auto dparam = [&](const char* k, double def) { const char* v = find_param(keys, values, n, k); return v ? std::atof(v) : def; };
  auto iparam = [&](const char* k, int def) { const char* v = find_param(keys, values, n, k); return v ? std::atoi(v) : def; };
  b2r_config c;
  if (method == "FAST_GICP" || method == "B200_GICP") {
    b2r_config_default(&c, B2R_METHOD_GICP);
    c.transformation_epsilon = dparam("reg_transformation_epsilon", 0.01);
    c.max_iterations = iparam("reg_maximum_iterations", 64);
    c.max_correspondence_distance = dparam("reg_max_correspondence_distance", 2.5);
    c.k_correspondences = iparam("reg_correspondence_randomness", 20);
  } else if (method == "NDT_OMP" || method == "B200_NDT") {
    b2r_config_default(&c, B2R_METHOD_NDT);
    c.ndt_resolution = dparam("reg_resolution", 0.5);
    c.transformation_epsilon = dparam("reg_transformation_epsilon", 0.01);
    c.max_iterations = iparam("reg_maximum_iterations", 64);
    const char* s = find_param(keys, values, n, "reg_nn_search_method");
    std::string sm = s ? s : "DIRECT7";
    if (sm == "KDTREE") return fail(B2R_EUNSUPPORTED, "reg_nn_search_method=KDTREE is not re-created (DIRECT1/DIRECT7 only)");
    c.ndt_search_method = (sm == "DIRECT1") ? 1 : 7;  // registrations.cpp:112-118: anything else -> DIRECT7
  } else {
    return fail(B2R_EUNSUPPORTED, "registration_method '" + method + "' is not re-created by b200reg; keep the reference branch");
  }
  c.device_id = device_id;
  return b2r_create(&c, out);
}


// may this device run the 16-CTA cluster kernels?  (cluster size 16 is "non-portable": opted into per kernel and probed with the
// occupancy query; B2R_NO_CLUSTER16 forces the portable shapes)
static bool cluster16_allowed();

extern "C" int b2r_create(const b2r_config* cfg, b2r_handle** out) {
  if (!cfg || !out) return fail(B2R_EINVAL, "NULL argument");
  *out = nullptr;
  if (cfg->method != B2R_METHOD_GICP && cfg->method != B2R_METHOD_NDT) return fail(B2R_EINVAL, "unknown method");
  if (cfg->k_correspondences < 1 || cfg->k_correspondences > 64) return fail(B2R_EINVAL, "k_correspondences must be in [1,64]");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev <= 0) return fail(B2R_ENODEVICE, std::string("no CUDA device: ") + cudaGetErrorString(e));
  if (cfg->device_id < 0 || cfg->device_id >= ndev) return fail(B2R_EINVAL, "device_id out of range");
  B2R_CUDA(cudaSetDevice(cfg->device_id));
  b2r_handle* h = new b2r_handle();
  h->cfg = *cfg;
  if (!(h->cfg.grid_cell_min > 0.f)) h->cfg.grid_cell_min = 0.5f;
  {  // round the cell size to a power of two
    int ex;
    float m = std::frexp(h->cfg.grid_cell_min, &ex);
    h->cfg.grid_cell_min = std::ldexp(1.0f, m > 0.5f ? ex : ex - 1);
  }
  auto bail = [&](int code) { b2r_destroy(h); return code; };
  cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, cfg->device_id);
  if (h->n_sm <= 0) h->n_sm = 132;
  {  // the align path (latency-critical chain of small kernels) outranks the prefetch path (throughput work for the NEXT frame)
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    if (getenv("B2R_NO_PRIORITY")) lo = hi = 0;
    if (getenv("B2R_PREFETCH_PRIORITY")) { const int t = lo; lo = hi; hi = t; }  // diagnostic: the prefetch path outranks the align chain
    if (cudaStreamCreateWithPriority(&h->st, cudaStreamNonBlocking, hi) != cudaSuccess) return bail(fail(B2R_ECUDA, "cudaStreamCreate failed"));
    if (cudaStreamCreateWithPriority(&h->st2, cudaStreamNonBlocking, lo) != cudaSuccess) return bail(fail(B2R_ECUDA, "cudaStreamCreate failed"));
  }
  if (cudaEventCreateWithFlags(&h->ev_prefetch, cudaEventDisableTiming) != cudaSuccess) return bail(fail(B2R_ECUDA, "cudaEventCreate failed"));
  if (cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming) != cudaSuccess)
    return bail(fail(B2R_ECUDA, "cudaEventCreate failed"));
  if (cudaEventCreateWithFlags(&h->upload_ev, cudaEventDisableTiming) != cudaSuccess) return bail(fail(B2R_ECUDA, "cudaEventCreate failed"));
  for (int i = 0; i < 3; i++) {
    if (cudaEventCreateWithFlags(&h->staging_ev[i], cudaEventDisableTiming) != cudaSuccess) return bail(fail(B2R_ECUDA, "cudaEventCreate failed"));
  }
  for (int i = 0; i < 2; i++)
    if (cudaMalloc(&h->bc[i].mm, 8 * sizeof(int)) != cudaSuccess) return bail(fail(B2R_ECUDA, "device allocation failed"));
  if (cudaMalloc(&h->d_out, 64 * sizeof(double)) != cudaSuccess ||
      cudaMalloc(&h->d_counter, 4 * sizeof(unsigned int)) != cudaSuccess || cudaHostAlloc(&h->h_out, 72 * sizeof(double), cudaHostAllocMapped) != cudaSuccess ||
      cudaHostGetDevicePointer((void**)&h->h_out_dev, h->h_out, 0) != cudaSuccess)
    return bail(fail(B2R_ECUDA, "device allocation failed"));
  h->h_flag = reinterpret_cast<unsigned long long*>(h->h_out + 64);
  h->h_flag_dev = reinterpret_cast<unsigned long long*>(h->h_out_dev + 64);
  h->h_flag[0] = h->h_flag[1] = h->h_flag[2] = 0;
  {  // mailbox of the device-resident LM: [0,128) report, [128,144) flag + progress, [256,512) tap values
    char* mb = nullptr; char* mb_dev = nullptr;
    if (cudaMalloc(&h->d_pair, sizeof(PairDev)) != cudaSuccess || cudaHostAlloc(&mb, 512, cudaHostAllocMapped) != cudaSuccess ||
        cudaHostGetDevicePointer((void**)&mb_dev, mb, 0) != cudaSuccess)
      return bail(fail(B2R_ECUDA, "device allocation failed"));
    std::memset(mb, 0, 512);
    h->h_rep = reinterpret_cast<PairReport*>(mb); h->h_rep_dev = reinterpret_cast<PairReport*>(mb_dev);
    h->h_pflag = reinterpret_cast<unsigned long long*>(mb + 128); h->h_pflag_dev = reinterpret_cast<unsigned long long*>(mb_dev + 128);
    h->h_tap = reinterpret_cast<double*>(mb + 256); h->h_tap_dev = reinterpret_cast<double*>(mb_dev + 256);
  }
  cudaMemsetAsync(h->d_counter, 0, 4 * sizeof(unsigned int), h->st);
  if (cudaStreamSynchronize(h->st) != cudaSuccess) return bail(fail(B2R_ECUDA, "initialisation failed"));
  for (int i = 0; i < 16; i++) h->final_T[i] = (i % 5 == 0) ? 1.f : 0.f;
  h->ndt_work.bc = &h->bc[0];
  h->ndt_work.tel = &h->tel;
  h->vg_work.tel = &h->tel;
  h->vg_work.wide_clusters = cluster16_allowed();
  *out = h;
  return B2R_OK;
}

extern "C" void b2r_batch_destroy(struct b2r_batch* b);
extern "C" void b2r_destroy(b2r_handle* h) {
  if (!h) return;
  if (h->loop_batch) { b2r_batch_destroy(h->loop_batch); h->loop_batch = nullptr; }
  cudaSetDevice(h->cfg.device_id);
  if (h->st) cudaStreamSynchronize(h->st);
  if (h->st2) cudaStreamSynchronize(h->st2);
  h->aux.raw.release(); h->aux.sorted.release(); h->aux.leaf_lo.release(); h->aux.leaf_hi.release(); h->aux.sup_lo.release(); h->aux.sup_hi.release(); h->aux.pos_of.release(); h->aux.cov.release();
  for (int i = 0; i < 3; i++) {
    Cloud& c = h->clouds[i];
    c.raw.release(); c.sorted.release(); c.leaf_lo.release(); c.leaf_hi.release(); c.sup_lo.release(); c.sup_hi.release(); c.pos_of.release(); c.cov.release();
    ndt_free_map(c.ndt);
    if (h->staging[i]) cudaFreeHost(h->staging[i]);
    if (h->staging_ev[i]) cudaEventDestroy(h->staging_ev[i]);
  }
  for (int i = 0; i < 2; i++) { h->corr[i].release(); h->cpos[i].release(); h->mahal[i].release(); }
  h->d2.release(); h->partials.release();
  h->tmp_f.release(); h->tmp_i.release(); h->tmp_f4.release(); h->bc[0].release(); h->bc[1].release();
  h->pf_buf[0].release(); h->pf_buf[1].release(); h->pf_flags.release(); h->pf_blocks.release();
  h->ingest_blob.release(); h->ingest_out.release();
  if (h->ingest_pinned) cudaFreeHost(h->ingest_pinned);
  h->map_kf.release(); h->map_keys[0].release(); h->map_keys[1].release();
  if (h->map_geom) cudaFree(h->map_geom);
  if (h->map_h) cudaFreeHost(h->map_h);
  if (h->pf_stats) cudaFree(h->pf_stats);
  if (h->pf_total) cudaFree(h->pf_total);
  if (h->pf_h_total) cudaFreeHost(h->pf_h_total);
  h->ndt_work.release();
  h->vg_work.release();
  h->tel.release();
  if (h->d_out) cudaFree(h->d_out);
  if (h->d_counter) cudaFree(h->d_counter);
  if (h->h_out) cudaFreeHost(h->h_out);
  if (h->h_rep) cudaFreeHost(h->h_rep);
  if (h->d_pair) cudaFree(h->d_pair);
  if (h->st) cudaStreamDestroy(h->st);
  if (h->st2) cudaStreamDestroy(h->st2);
  if (h->ev_prefetch) cudaEventDestroy(h->ev_prefetch);
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  if (h->ev_join) cudaEventDestroy(h->ev_join);
  if (h->upload_ev) cudaEventDestroy(h->upload_ev);
  delete h;
}

extern "C" int b2r_get_config(const b2r_handle* h, b2r_config* out) {
  if (!h || !out) return fail(B2R_EINVAL, "NULL argument");
  *out = h->cfg;
  return B2R_OK;
}

// ------------------------------------------------------------------------------------------------ upload + preprocessing
static bool is_pinned_host(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost;
}

static int upload(b2r_handle* h, int which, const void* pts, size_t n, size_t stride_bytes, bool device_ptr, cudaStream_t st) {
  if (stride_bytes < 12 || (stride_bytes & 3)) return fail(B2R_EINVAL, "stride_bytes must be a multiple of 4 and >= 12");
  if (n > 0 && !pts) return fail(B2R_EINVAL, "points is NULL");
  if (n > (size_t)0x3fffffff) return fail(B2R_EINVAL, "too many points");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  Cloud& c = h->clouds[which];
  c.n = n;
  c.stride_f = (int)(stride_bytes / 4);
  c.host_ptr = pts;  // identity of the caller's buffer (host or device): used to recognise a prefetched cloud
  c.invalidate();
  const size_t bytes = n * stride_bytes;
  if (device_ptr && h->cfg.method == B2R_METHOD_NDT) {
    // an NDT cloud's voxel map is built lazily, when the cloud has become the TARGET (possibly many calls later): the engine
    // keeps its own copy (device-to-device, ~1 us per MB) so the caller's buffer is free once the call that first uses it returns
    B2R_CUDA(c.raw.reserve(n * c.stride_f + 4));
    c.raw_view = c.raw.p;
    if (bytes > 0) B2R_CUDA(cudaMemcpyAsync(c.raw.p, pts, bytes, cudaMemcpyDeviceToDevice, st));
  } else if (device_ptr) {
    c.raw_view = (const float*)pts;  // GICP: read while the structures are built, i.e. until the align / matching call that first uses the cloud returns
  } else {
    B2R_CUDA(c.raw.reserve(n * c.stride_f + 4));
    c.raw_view = c.raw.p;
    if (bytes > 0) {
      if (is_pinned_host(pts)) {
        // DMA straight from the caller's pinned buffer; `upload_ev` marks the end of that copy so that a synchronous entry point
        // (b2r_set_source / b2r_set_target) can hand the buffer back to the caller on return, as b200reg.h promises
        B2R_CUDA(cudaMemcpyAsync(c.raw.p, pts, bytes, cudaMemcpyHostToDevice, st));
        B2R_CUDA(cudaEventRecord(h->upload_ev, st));
        h->upload_pending = true;
        h->tel.h2d += bytes;
      } else {
        int sidx = which;
        if (h->staging_cap[sidx] < bytes) {
          if (h->staging[sidx]) { cudaEventSynchronize(h->staging_ev[sidx]); cudaFreeHost(h->staging[sidx]); h->staging[sidx] = nullptr; }
          size_t want = bytes + bytes / 4 + 4096;
          B2R_CUDA(cudaMallocHost(&h->staging[sidx], want));
          h->staging_cap[sidx] = want;
        } else {
          B2R_CUDA(cudaEventSynchronize(h->staging_ev[sidx]));
        }
        std::memcpy(h->staging[sidx], pts, bytes);
        B2R_CUDA(cudaMemcpyAsync(c.raw.p, h->staging[sidx], bytes, cudaMemcpyHostToDevice, st));
        h->tel.h2d += bytes;
        B2R_CUDA(cudaEventRecord(h->staging_ev[sidx], st));
      }
    }
  }
  return B2R_OK;
}

// ---- cluster build (bvh_build.cuh): one launch builds the whole structure of one cloud — or of a set of clouds
static int bvh_alloc(Cloud& c) {
  const size_t n = c.n;
  c.nsup = (int)((n + 1023) / 1024);
  const size_t padded = (size_t)c.nsup * 1024;
  B2R_CUDA(c.sorted.reserve(padded + 32));
  B2R_CUDA(c.pos_of.reserve(n + 1));
  B2R_CUDA(c.leaf_lo.reserve((size_t)c.nsup * kSuper + 1));
  B2R_CUDA(c.leaf_hi.reserve((size_t)c.nsup * kSuper + 1));
  B2R_CUDA(c.sup_lo.reserve(c.nsup + 1));
  B2R_CUDA(c.sup_hi.reserve(c.nsup + 1));
  return B2R_OK;
}
static BuildItem build_item(const Cloud& c) {
  BuildItem it;
  it.raw = c.raw_view; it.sorted = c.sorted.p; it.pos_of = c.pos_of.p; it.leaf_lo = c.leaf_lo.p; it.leaf_hi = c.leaf_hi.p;
  it.sup_lo = c.sup_lo.p; it.sup_hi = c.sup_hi.p; it.stride_f = c.stride_f; it.n = (int)c.n;
  return it;
}
static bool use_cluster_build() {
  static const bool on = !getenv("B2R_CUB_SORT");
  return on;
}
template <int CL, int PER, bool SINGLE>
static cudaError_t launch_cluster_build_t(const BuildItem* d_items, const BuildItem& single, unsigned n_clouds, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k_bvh_build_cluster<CL, PER, SINGLE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BuildGeom<PER>::kSmem);
    if (e != cudaSuccess) return e;
    if (CL > 8) {
      e = cudaFuncSetAttribute(k_bvh_build_cluster<CL, PER, SINGLE>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
      if (e != cudaSuccess) return e;
    }
    attr_set = true;
  }
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3(n_clouds * CL); lc.blockDim = dim3(kBuildThreads); lc.dynamicSmemBytes = BuildGeom<PER>::kSmem; lc.stream = st;
  cudaLaunchAttribute la[1];
  la[0].id = cudaLaunchAttributeClusterDimension;
  la[0].val.clusterDim.x = CL; la[0].val.clusterDim.y = 1; la[0].val.clusterDim.z = 1;
  lc.attrs = la; lc.numAttrs = 1;
  return cudaLaunchKernelEx(&lc, k_bvh_build_cluster<CL, PER, SINGLE>, d_items, single);
}
template <bool SINGLE>
static cudaError_t launch_cluster_build_s(int shape_index, const BuildItem* d_items, const BuildItem& single, unsigned n_clouds, cudaStream_t st) {
  switch (shape_index) {  // build_shape_index(): (cluster size, pairs per thread)
    case 0: return launch_cluster_build_t<1, 1, SINGLE>(d_items, single, n_clouds, st);
    case 1: return launch_cluster_build_t<2, 1, SINGLE>(d_items, single, n_clouds, st);
    case 2: return launch_cluster_build_t<4, 1, SINGLE>(d_items, single, n_clouds, st);
    case 3: return launch_cluster_build_t<8, 1, SINGLE>(d_items, single, n_clouds, st);
    case 4: return launch_cluster_build_t<8, 2, SINGLE>(d_items, single, n_clouds, st);
    case 5: return launch_cluster_build_t<8, 4, SINGLE>(d_items, single, n_clouds, st);
    case 6: return launch_cluster_build_t<8, 8, SINGLE>(d_items, single, n_clouds, st);
    case 7: return launch_cluster_build_t<8, 16, SINGLE>(d_items, single, n_clouds, st);
    default: return launch_cluster_build_t<16, 8, SINGLE>(d_items, single, n_clouds, st);
  }
}
static bool cluster16_allowed() {
  static int ok = -1;
  if (ok < 0) {
    ok = 0;
    if (!getenv("B2R_NO_CLUSTER16")) {
      auto* fn = k_bvh_build_cluster<16, 8, true>;
      if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BuildGeom<8>::kSmem) == cudaSuccess &&
          cudaFuncSetAttribute(fn, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess) {
        cudaLaunchConfig_t lc = {};
        lc.gridDim = dim3(16); lc.blockDim = dim3(kBuildThreads); lc.dynamicSmemBytes = BuildGeom<8>::kSmem;
        cudaLaunchAttribute la[1];
        la[0].id = cudaLaunchAttributeClusterDimension;
        la[0].val.clusterDim.x = 16; la[0].val.clusterDim.y = 1; la[0].val.clusterDim.z = 1;
        lc.attrs = la; lc.numAttrs = 1;
        int n = 0;
        if (cudaOccupancyMaxActiveClusters(&n, fn, &lc) == cudaSuccess && n > 0) ok = 1;
      }
      (void)cudaGetLastError();
    }
  }
  return ok == 1;
}
// one launch builds `n_clouds` clouds of the same shape: the descriptor list d_items, or (d_items == nullptr) the one cloud `single`
static cudaError_t launch_cluster_build(int shape_index, const BuildItem* d_items, const BuildItem& single, unsigned n_clouds, cudaStream_t st) {
  return d_items ? launch_cluster_build_s<false>(shape_index, d_items, single, n_clouds, st) : launch_cluster_build_s<true>(shape_index, d_items, single, n_clouds, st);
}

// builds the implicit BVH of a cloud on stream `st` with build scratch `B` (one scratch per stream)
static int build_bvh(b2r_handle* h, Cloud& c, BuildCtx& B, cudaStream_t st) {
  if (c.bvh_ready) return B2R_OK;
  const size_t n = c.n;
  const int N = (int)n;
  int arc = bvh_alloc(c);
  if (arc) return arc;
  if (n == 0) { c.bvh_ready = true; return B2R_OK; }
  const BuildShape shape = build_shape_for(n, cluster16_allowed());
  if (shape.cl && use_cluster_build()) {  // the whole build as ONE kernel on a cluster (the cloud lives in distributed shared memory)
    TEL_BEGIN(&h->tel, st);
    B2R_CUDA(launch_cluster_build(build_shape_index(shape), nullptr, build_item(c), 1, st));
    TEL_END(&h->tel, KC_GRID, 1, st);
    c.bvh_ready = true;
    return B2R_OK;
  }
  // clouds beyond 131 072 points: bounding box, keys, toolkit radix sort, leaves
  B2R_CUDA(B.keys_a.reserve(n)); B2R_CUDA(B.keys_b.reserve(n)); B2R_CUDA(B.vals_a.reserve(n)); B2R_CUDA(B.vals_b.reserve(n));
  size_t tmp_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, B.keys_a.p, B.keys_b.p, B.vals_a.p, B.vals_b.p, N, 0, 30, st);
  B2R_CUDA(B.sort_tmp.reserve(tmp_bytes + 256));
  TEL_BEGIN(&h->tel, st);
  const unsigned nb = (unsigned)((n + 255) / 256);
  k_grid_reset<<<1, 32, 0, st>>>(B.mm);
  k_bbox<<<nb > 1184 ? 1184 : nb, 256, 0, st>>>(c.raw_view, c.stride_f, N, B.mm);
  k_fill_i32<<<nb, 256, 0, st>>>(c.pos_of.p, N, -1);
  k_morton_keys<<<nb, 256, 0, st>>>(c.raw_view, c.stride_f, N, B.mm, B.keys_a.p, B.vals_a.p);
  size_t tb = B.sort_tmp.cap;
  // stable LSD sort: ties keep ascending index.  Keys are 30-bit Hilbert indices, or 0xffffffff for dropped points: the two top
  // bits are constant among valid keys, so sorting bits [0,30) orders them; dropped points are recognised by their key afterwards
  cub::DeviceRadixSort::SortPairs(B.sort_tmp.p, tb, B.keys_a.p, B.keys_b.p, B.vals_a.p, B.vals_b.p, N, 0, 32, st);
  k_bvh_leaves<<<c.nsup, 1024, 0, st>>>(c.raw_view, c.stride_f, N, B.keys_b.p, B.vals_b.p, c.sorted.p, c.pos_of.p, c.leaf_lo.p, c.leaf_hi.p,
                                        c.sup_lo.p, c.sup_hi.p);
  TEL_END(&h->tel, KC_GRID, 10, st);
  B2R_CUDA(cudaGetLastError());
  c.bvh_ready = true;
  return B2R_OK;
}

static int ensure_grid(b2r_handle* h, Cloud& c, int ctx = 0) { return build_bvh(h, c, h->bc[ctx], ctx ? h->st2 : h->st); }

static int build_cov(b2r_handle* h, Cloud& c, BuildCtx& B, cudaStream_t st) {
  int rc = build_bvh(h, c, B, st);
  if (rc) return rc;
  if (c.cov_ready) return B2R_OK;
  const size_t padded = (size_t)c.nsup * 1024;
  B2R_CUDA(c.cov.reserve(padded * 6 + 6));
  if (c.n > 0) {
    const int k = h->cfg.k_correspondences;
    const size_t smem = (size_t)k * kKnnThreads * sizeof(unsigned long long);
    long long* prof = nullptr;
#ifdef B2R_KNN_PROFILE
    static long long* d_prof = nullptr;
    if (!d_prof) cudaMalloc(&d_prof, (size_t)(1 << 16) * 8 * sizeof(long long));
    cudaMemsetAsync(d_prof, 0, (size_t)c.nsup * kSuper * 8 * sizeof(long long), st);
    prof = d_prof;
#endif
    TEL_BEGIN(&h->tel, st);
    if (k == kKnnRegK) {  // the reference's default reg_correspondence_randomness: lists live in registers
      // On the PREFETCH stream the kernel works for the NEXT frame while the align chain of the current one runs beside it.  All of its
      // 512 blocks become resident at once (104 registers x 128 threads x ~3.9 blocks per SM on 132 SMs = 80 % of the register file) and
      // stay for the kernel's whole run — stream priorities only order PENDING blocks, so the chain's search kernels then run in what is left of each SM.
      // Capping the prefetch kernel's residency with unused dynamic shared memory keeps most of every SM for the chain.
      static const int cap = [] { const char* e = getenv("B2R_PREFETCH_KNN_BLOCKS"); return e ? atoi(e) : B2R_PREFETCH_KNN_BLOCKS_DEFAULT; }();
      size_t pad_smem = 0;
      if (cap > 0 && cap < B2R_KNN_MINBLOCKS && st == h->st2) {
        pad_smem = ((size_t)227 * 1024 / (size_t)cap - (size_t)kKnnRegK * kKnnThreads * sizeof(int) - 2048) & ~(size_t)255;
        static bool attr_set = false;
        if (!attr_set) {
          B2R_CUDA(cudaFuncSetAttribute(k_knn_cov_reg<kKnnRegK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024 - kKnnRegK * kKnnThreads * (int)sizeof(int) - 2048)));
          attr_set = true;
        }
      }
      k_knn_cov_reg<kKnnRegK><<<(unsigned)(padded / kKnnThreads), kKnnThreads, pad_smem, st>>>(c.bvh(), c.raw_view, c.stride_f, c.cov.p, prof);
    } else {
      if (smem > 48 * 1024 && !h->knn_smem_attr) {
        B2R_CUDA(cudaFuncSetAttribute(k_knn_cov, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * kKnnThreads * 8));
        h->knn_smem_attr = true;
      }
      k_knn_cov<<<(unsigned)(padded / kKnnThreads), kKnnThreads, smem, st>>>(c.bvh(), k, c.raw_view, c.stride_f, c.cov.p, prof);
    }
    TEL_END(&h->tel, KC_KNN_COV, 1, st);
#ifdef B2R_KNN_PROFILE
    {
      cudaStreamSynchronize(st);
      const size_t nl = (size_t)c.nsup * kSuper;
      std::vector<long long> hp(nl * 8);
      std::vector<float4> lo(nl), hi(nl);
      cudaMemcpy(hp.data(), d_prof, nl * 8 * sizeof(long long), cudaMemcpyDeviceToHost);
      cudaMemcpy(lo.data(), c.leaf_lo.p, nl * sizeof(float4), cudaMemcpyDeviceToHost);
      cudaMemcpy(hi.data(), c.leaf_hi.p, nl * sizeof(float4), cudaMemcpyDeviceToHost);
      if (FILE* f = fopen("gpurun_out/knn_prof.bin", "wb")) {
        fwrite(hp.data(), sizeof(long long), nl * 8, f);
        fclose(f);
      }
      if (FILE* f = fopen("gpurun_out/knn_prof_box.bin", "wb")) {
        fwrite(lo.data(), sizeof(float4), nl, f);
        fwrite(hi.data(), sizeof(float4), nl, f);
        fclose(f);
      }
    }
#endif
    B2R_CUDA(cudaGetLastError());
  }
  c.cov_ready = true;
  return B2R_OK;
}

static int ensure_cov(b2r_handle* h, Cloud& c, int ctx = 0) { return build_cov(h, c, h->bc[ctx], ctx ? h->st2 : h->st); }

static int preprocess(b2r_handle* h, int which, bool is_target) {
  Cloud& c = h->clouds[which];
  if (h->cfg.method == B2R_METHOD_GICP) {
    // a target gets its covariances now; a SOURCE only its search structure: its k-NN covariance kernel is launched by the align,
    // beside the first correspondence search, which does not read it (run_single_pair) — unless the cloud arrives through the
    // prefetch path, where both have been built ahead on the second stream
    static const bool overlap = !getenv("B2R_NO_COV_OVERLAP");
    return (is_target || !overlap) ? ensure_cov(h, c) : ensure_grid(h, c);
  }
  // NDT: the target needs the voxel Gaussians; the source is put in Hilbert order (the BVH build's sorted array) so that the
  // 128 points of a derivative block are spatial neighbours and share their voxel cells
  if (is_target) return ndt_ensure_map(h->cfg, c, h->ndt_work, h->st);
  return ensure_grid(h, c);
}

// cheap identity of a host cloud's CONTENT: FNV-1a over 64 records spread evenly over the buffer (plus n and stride)
static unsigned long long content_stamp(const void* pts, size_t n, size_t stride) {
  unsigned long long x = 1469598103934665603ull ^ (unsigned long long)n * 1099511628211ull ^ (unsigned long long)stride;
  if (!pts || n == 0) return x;
  const unsigned char* b = (const unsigned char*)pts;
  const size_t step = n > 64 ? n / 64 : 1;
  for (size_t i = 0; i < n; i += step) {
    const unsigned char* r = b + i * stride;
    for (int k = 0; k < 12; k++) { x ^= r[k]; x *= 1099511628211ull; }
  }
  const unsigned char* last = b + (n - 1) * stride;
  for (int k = 0; k < 12; k++) { x ^= last[k]; x *= 1099511628211ull; }
  return x;
}

static int set_cloud(b2r_handle* h, bool is_target, const void* pts, size_t n, size_t stride, bool dev) {
  if (!h) return fail(B2R_EINVAL, "handle is NULL");
  if (!is_target && h->prefetched) {
    Cloud& nx = h->clouds[h->nxt];
    h->prefetched = false;
    // adopt the prefetched cloud only if it is still THE cloud: same buffer, same shape and the same content stamp (a caller that
    // recycles one staging buffer and has rewritten it since the prefetch gets a fresh upload instead of the previous scan)
    if (nx.host_ptr == pts && nx.n == n && (size_t)nx.stride_f * 4 == stride && (dev || content_stamp(pts, n, stride) == h->prefetch_stamp)) {
      B2R_CUDA(cudaSetDevice(h->cfg.device_id));
      std::swap(h->src, h->nxt);
      B2R_CUDA(cudaStreamWaitEvent(h->st, h->ev_prefetch, 0));
      h->corr_valid = false;
      return B2R_OK;
    }
  }
  int which = is_target ? h->tgt : h->src;
  h->upload_pending = false;
  int rc = upload(h, which, pts, n, stride, dev, h->st);
  if (rc) return rc;
  h->corr_valid = false;
  rc = preprocess(h, which, is_target);  // the structure builds are enqueued behind the copy before the host waits for it
  if (h->upload_pending) {
    // the caller keeps ownership of its (pinned) buffer: the copy out of it has finished when this call returns
    B2R_CUDA(cudaEventSynchronize(h->upload_ev));
    h->upload_pending = false;
  }
  return rc;
}

static int prefetch_source(b2r_handle* h, const void* pts, size_t n, size_t stride, bool dev) {
  if (!h) return fail(B2R_EINVAL, "handle is NULL");
  if (!dev && pts) h->prefetch_stamp = content_stamp(pts, n, stride);
  // the buffers of the `nxt` slot may still be read by kernels enqueued on the main stream (it was the source of an earlier
  // align that has completed: b2r_align synchronises), so they are free to be overwritten here
  int rc = upload(h, h->nxt, pts, n, stride, dev, h->st2);
  if (rc) return rc;
  if (h->cfg.method == B2R_METHOD_GICP) {
    rc = ensure_cov(h, h->clouds[h->nxt], 1);
    if (rc) return rc;
  }
  B2R_CUDA(cudaEventRecord(h->ev_prefetch, h->st2));
  h->prefetched = true;
  return B2R_OK;
}

extern "C" int b2r_prefetch_source(b2r_handle* h, const void* p, size_t n, size_t s) { return prefetch_source(h, p, n, s, false); }
extern "C" int b2r_prefetch_source_device(b2r_handle* h, const void* p, size_t n, size_t s) { return prefetch_source(h, p, n, s, true); }

extern "C" int b2r_set_target(b2r_handle* h, const void* p, size_t n, size_t s) { return set_cloud(h, true, p, n, s, false); }
extern "C" int b2r_set_source(b2r_handle* h, const void* p, size_t n, size_t s) { return set_cloud(h, false, p, n, s, false); }
extern "C" int b2r_set_target_device(b2r_handle* h, const void* p, size_t n, size_t s) { return set_cloud(h, true, p, n, s, true); }
extern "C" int b2r_set_source_device(b2r_handle* h, const void* p, size_t n, size_t s) { return set_cloud(h, false, p, n, s, true); }

extern "C" int b2r_synchronize(b2r_handle* h) {
  if (!h) return fail(B2R_EINVAL, "handle is NULL");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  B2R_CUDA(cudaStreamSynchronize(h->st));
  B2R_CUDA(cudaStreamSynchronize(h->st2));
  return B2R_OK;
}

extern "C" int b2r_get_stream(b2r_handle* h, void** stream) {
  if (!h || !stream) return fail(B2R_EINVAL, "NULL argument");
  *stream = (void*)h->st;
  return B2R_OK;
}

extern "C" int b2r_set_profiling(b2r_handle* h, int on) {
  if (!h) return fail(B2R_EINVAL, "handle is NULL");
  h->tel.on = on != 0;
  return B2R_OK;
}

extern "C" const char* b2r_kernel_class_name(int cls) { return kernel_class_name(cls); }

extern "C" int b2r_get_stats(b2r_handle* h, b2r_stats* out, int reset) {
  if (!h || !out) return fail(B2R_EINVAL, "NULL argument");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  B2R_CUDA(cudaStreamSynchronize(h->st));
  B2R_CUDA(cudaStreamSynchronize(h->st2));
  h->tel.resolve();
  std::memset(out, 0, sizeof(*out));
  out->h2d_bytes = h->tel.h2d;
  out->d2h_bytes = h->tel.d2h;
  out->n_classes = KC_COUNT;
  for (int i = 0; i < KC_COUNT; i++) { out->launches[i] = h->tel.launches[i]; out->calls[i] = h->tel.calls[i]; out->ms[i] = h->tel.ms[i]; }
  if (reset) h->tel.reset();
  return B2R_OK;
}

extern "C" int b2r_promote_source_to_target(b2r_handle* h) {
  if (!h) return fail(B2R_EINVAL, "handle is NULL");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  std::swap(h->src, h->tgt);
  h->corr_valid = false;
  // the old target becomes a stale source: callers always set a new source before the next align
  return preprocess(h, h->tgt, true);
}

// ------------------------------------------------------------------------------------------------ GICP align (LM, A.4)
static void colmajor_f_to_row_d(const float* g, double* x) {
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) x[r * 4 + c] = (double)g[c * 4 + r];
}

static int ensure_align_ws(b2r_handle* h, size_t n_in) {
  const size_t n = ((n_in + 1023) / 1024) * 1024;
  for (int i = 0; i < 2; i++) {
    B2R_CUDA(h->corr[i].reserve(n + 1));
    B2R_CUDA(h->cpos[i].reserve(n + 1));
    B2R_CUDA(h->mahal[i].reserve(n * 6 + 6));
  }
  B2R_CUDA(h->d2.reserve(n + 1));
  size_t nb = (n + kAccThreads - 1) / kAccThreads + 1;
  B2R_CUDA(h->partials.reserve((nb + 32) * kAcc + 64));  // [kAcc][blocks rounded up to 32]
  return B2R_OK;
}

static LmCfg make_lm_cfg(const b2r_config& cfg, bool want_fitness, double fit_max_range) {
  LmCfg c;
  c.max_iterations = cfg.max_iterations;
  c.rot_eps = cfg.rotation_epsilon;
  c.trans_eps = cfg.transformation_epsilon;
  const double thr = cfg.max_correspondence_distance;
  c.thr2 = thr * thr;
  float lim = (float)c.thr2;
  if ((double)lim < c.thr2) lim = std::nextafterf(lim, INFINITY);
  c.lim = lim;
  c.want_fitness = want_fitness ? 1 : 0;
  c.fit_max_range = fit_max_range;
  // the fitness search must reach every neighbour with d2 <= max_range: its limit is the next float ABOVE max_range
  float fl = (fit_max_range >= (double)FLT_MAX) ? INFINITY : (float)fit_max_range;
  if (fl < INFINITY) { if ((double)fl < fit_max_range) fl = std::nextafterf(fl, INFINITY); fl = std::nextafterf(fl, INFINITY); }
  c.fit_lim = fl;
  static const bool index_seed = !getenv("B2R_NO_INDEX_SEED");
  c.index_seed = index_seed ? 1 : 0;
  return c;
}

// PairDev of one (source, target) with the handle-independent parts filled in
static void fill_pair_geometry(PairDev& P, const Cloud& s, const Cloud& t) {
  std::memset(&P, 0, sizeof(P));
  P.src = s.bvh(); P.scov = s.cov.p;
  P.tgt = t.bvh(); P.tcov = t.cov.p;
  P.tgt_pos_of = t.pos_of.p; P.tgt_n = (int)t.n;
  P.nblk_acc = (int)((size_t)s.nsup * 1024 / kAccThreads);
}
static void fill_pair_start(PairDev& P, const double* x_row12, int mode) {
  for (int i = 0; i < 12; i++) { P.xe[i] = x_row12[i]; P.x0[i] = x_row12[i]; }
  P.mode = mode;
  P.lambda = -1.0; P.nu = 2.0;
}

template <int C>
static cudaError_t launch_search(PairDev* d_pairs, const int* d_active, unsigned n_slots, unsigned max_sorted, const LmCfg& cfg, cudaStream_t st, bool pdl) {
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3((unsigned)((size_t)max_sorted * C / kLinThreads), n_slots);
  lc.blockDim = dim3(kLinThreads); lc.dynamicSmemBytes = 0; lc.stream = st;
  cudaLaunchAttribute la[1];
  la[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  la[0].val.programmaticStreamSerializationAllowed = 1;
  lc.attrs = la; lc.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&lc, k_pair_search<C>, d_pairs, d_active, cfg);
}

// one round (update_correspondences + linearize/compute_error + LM step) over n_slots pair slots
static int launch_round(PairDev* d_pairs, const int* d_active, unsigned n_slots, unsigned max_sorted, int copies, const LmCfg& cfg, cudaStream_t st,
                        Telemetry* tel, bool search = true) {
  static const bool pdl = !getenv("B2R_NO_PDL");
  if (search) {
    TEL_BEGIN(tel, st);
    cudaError_t e = copies == 1 ? launch_search<1>(d_pairs, d_active, n_slots, max_sorted, cfg, st, pdl)
                  : copies == 2 ? launch_search<2>(d_pairs, d_active, n_slots, max_sorted, cfg, st, pdl)
                                : launch_search<4>(d_pairs, d_active, n_slots, max_sorted, cfg, st, pdl);
    B2R_CUDA(e);
    TEL_END(tel, KC_GICP_CORR, 1, st);
  }
  {
    TEL_BEGIN(tel, st);
    cudaLaunchConfig_t lc = {};
    lc.gridDim = dim3((unsigned)(max_sorted / kAccThreads), n_slots); lc.blockDim = dim3(kAccThreads); lc.dynamicSmemBytes = 0; lc.stream = st;
    cudaLaunchAttribute la[1];
    la[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    la[0].val.programmaticStreamSerializationAllowed = 1;
    lc.attrs = la; lc.numAttrs = pdl ? 1 : 0;
    B2R_CUDA(cudaLaunchKernelEx(&lc, k_pair_accumulate, d_pairs, d_active, cfg));
    lc.gridDim = dim3(n_slots); lc.blockDim = dim3(kLmThreads);
    B2R_CUDA(cudaLaunchKernelEx(&lc, k_pair_lm, d_pairs, d_active, cfg));
    TEL_END(tel, KC_GICP_LIN, 2, st);
  }
  return B2R_OK;
}

__global__ void k_pair_init(const __grid_constant__ PairDev init, PairDev* dst) {
  // the whole record travels as a kernel parameter: no DMA, no staging buffer (single-pair path)
  const unsigned long long* s = reinterpret_cast<const unsigned long long*>(&init);
  unsigned long long* d = reinterpret_cast<unsigned long long*>(dst);
  for (int i = threadIdx.x; i < (int)(sizeof(PairDev) / 8); i += blockDim.x) d[i] = s[i];
}
static_assert(sizeof(PairDev) % 8 == 0, "PairDev is copied in 64-bit words");

// the acceptance test of a report message: flag == seq and word 15 == seq ^ mix(words 0..14)
static bool report_consistent(const volatile unsigned long long* flag, unsigned long long seq, const volatile unsigned long long* w) {
  if (*flag != seq) return false;
  unsigned long long x = seq;
  for (int i = 0; i < 15; i++) x ^= msg_mix(w[i], i);
  return x == w[15];
}

// Run the handle's single pair from `mode` at pose x (row-major 3x4 in x[0..11]) until its report lands in mapped memory.
// Rounds are enqueued ahead of the device (no host wait per iteration); a finished pair's remaining rounds exit at once.
static int run_single_pair(b2r_handle* h, const double* x, int mode, int tap, const LmCfg& cfg, int first_batch, bool cov_beside_first_search = false) {
  Cloud& s = SRC(h);
  Cloud& t = TGT(h);
  PairDev P;
  fill_pair_geometry(P, s, t);
  fill_pair_start(P, x, mode);
  for (int i = 0; i < 2; i++) { P.corr[i] = h->corr[i].p; P.cpos[i] = h->cpos[i].p; P.mahal[i] = h->mahal[i].p; }
  P.d2 = h->d2.p; P.partials = h->partials.p;
  P.report = h->h_rep_dev; P.flag = h->h_pflag_dev; P.progress = h->h_pflag_dev + 1; P.tap_out = h->h_tap_dev;
  P.seq = ++h->seq;
  P.tap = tap;
  P.cur = (mode == PM_FIRST) ? 0 : h->cur;
  const unsigned long long seq = P.seq;
  const unsigned max_sorted = (unsigned)((size_t)s.nsup * 1024);
  static const int copies = [] { const char* e = getenv("B2R_NN_COPIES"); int c = e ? atoi(e) : 4; return (c == 1 || c == 2) ? c : 4; }();
  int enq = 0;
  if (cov_beside_first_search) {
    // The source's covariances do not exist yet (strict call-by-call chain: no prefetch).  The first round's correspondence search
    // reads only the source's sorted points and the target's structure, so it runs on the SECOND (low-priority) stream while the
    // k-NN covariance kernel runs on the main one: that kernel's grid is under one wave with a long tail of single heavy warps
    // and the search's blocks fill the SMs as its blocks retire.  The accumulate kernel, the first reader of the
    // covariances, waits for both.
    B2R_CUDA(cudaEventRecord(h->ev_fork, h->st));  // behind the structure build and whatever the previous align left on the main stream
    B2R_CUDA(cudaStreamWaitEvent(h->st2, h->ev_fork, 0));
    k_pair_init<<<1, 128, 0, h->st2>>>(P, h->d_pair);
    B2R_CUDA(cudaGetLastError());
    { TEL_BEGIN(&h->tel, h->st2);
      cudaError_t e = copies == 1 ? launch_search<1>(h->d_pair, nullptr, 1, max_sorted, cfg, h->st2, false)
                    : copies == 2 ? launch_search<2>(h->d_pair, nullptr, 1, max_sorted, cfg, h->st2, false)
                                  : launch_search<4>(h->d_pair, nullptr, 1, max_sorted, cfg, h->st2, false);
      B2R_CUDA(e);
      TEL_END(&h->tel, KC_GICP_CORR, 1, h->st2); }
    B2R_CUDA(cudaEventRecord(h->ev_join, h->st2));
    int rc0 = ensure_cov(h, s);  // main stream: the k-NN covariance kernel
    if (rc0) return rc0;
    B2R_CUDA(cudaStreamWaitEvent(h->st, h->ev_join, 0));
    rc0 = launch_round(h->d_pair, nullptr, 1, max_sorted, copies, cfg, h->st, &h->tel, false);  // accumulate + LM step of round 1
    if (rc0) return rc0;
    enq = 1;
    first_batch--;
  } else {
    k_pair_init<<<1, 128, 0, h->st>>>(P, h->d_pair);
    B2R_CUDA(cudaGetLastError());
  }
  auto enqueue = [&](int n) -> int {
    for (int i = 0; i < n; i++) {
      int rc = launch_round(h->d_pair, nullptr, 1, max_sorted, copies, cfg, h->st, &h->tel, true);
      if (rc) return rc;
      enq++;
    }
    return B2R_OK;
  };
  int rc = enqueue(first_batch);
  if (rc) return rc;
  const volatile unsigned long long* flag = h->h_pflag;
  const volatile unsigned long long* prog = h->h_pflag + 1;
  const volatile unsigned long long* w = reinterpret_cast<const volatile unsigned long long*>(h->h_rep);
  static const unsigned long spin_limit = [] { const char* e = getenv("B2R_SPIN_LIMIT"); return e ? strtoul(e, nullptr, 10) : 4000000ul; }();
  unsigned long spins = 0;
  for (;;) {
    if (report_consistent(flag, seq, w)) break;
    const unsigned long long pw = *prog;
    const int done = ((pw >> 16) == (seq & 0xffffffffffffull)) ? (int)(pw & 0xffff) : 0;
    if (enq - done < 1 && !tap) { rc = enqueue(1); if (rc) return rc; }  // the prediction fell short: keep one round ahead of the device
    if ((++spins & 0x3fff) == 0) {
      cudaError_t e = cudaStreamQuery(h->st);
      if (e != cudaSuccess && e != cudaErrorNotReady) return fail(B2R_ECUDA, std::string("stream error: ") + cudaGetErrorString(e));
      if (e == cudaSuccess && !report_consistent(flag, seq, w)) {  // everything enqueued has run and the pair is not finished
        if (tap) return fail(B2R_ECUDA, "tap round finished without signalling its result");
        rc = enqueue(2);
        if (rc) return rc;
      }
      if (spins > spin_limit) {  // other streams' work is ahead of ours: stop burning a core and block
        B2R_CUDA(cudaStreamSynchronize(h->st));
        spins = 0;
      }
    }
  }
  h->last_rounds = h->h_rep->rounds;
  h->tel.d2h += sizeof(PairReport);
  return B2R_OK;
}

static void store_result(b2r_handle* h, const float* T_row, bool converged, int iterations, b2r_result* out) {
  for (int i = 0; i < 16; i++) h->final_T[i] = T_row[i];
  h->has_final = true;
  if (out) {
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++) out->T[c * 4 + r] = T_row[r * 4 + c];
    out->fitness = NAN;
    out->converged = converged ? 1 : 0;
    out->iterations = iterations;
  }
}

static int gicp_align(b2r_handle* h, const float* guess, b2r_result* out) {
  Cloud& s = SRC(h);
  Cloud& t = TGT(h);
  double x0[16];
  colmajor_f_to_row_d(guess, x0);
  x0[12] = x0[13] = x0[14] = 0; x0[15] = 1;
  float Tg[16];
  for (int i = 0; i < 16; i++) Tg[i] = (float)x0[i];
  if (s.n == 0 || t.n == 0) {  // pcl::Registration::initCompute fails silently: converged_ = false
    store_result(h, Tg, false, 0, out);
    return B2R_OK;
  }
  static const bool overlap = !getenv("B2R_NO_COV_OVERLAP");
  const bool cov_beside = overlap && !s.cov_ready;  // see run_single_pair
  int rc = cov_beside ? ensure_grid(h, s) : ensure_cov(h, s);
  if (rc) return rc;
  if (cov_beside) B2R_CUDA(s.cov.reserve((size_t)s.nsup * 1024 * 6 + 6));  // the pair record takes the buffer's address before the kernel that fills it is launched
  rc = ensure_cov(h, t);
  if (rc) return rc;
  rc = ensure_align_ws(h, s.n);
  if (rc) return rc;
  // fast_gicp's LM loop (LsqRegistration::computeTransformation / step_lm, SURVEY A.4) runs ON THE DEVICE (pair_engine.cuh):
  // one search + one accumulate launch per LM trial, the accumulate kernel's last block takes the LM step.  The trial cost
  // compute_error(xi) of iteration i and the linearisation linearize(xi) of iteration i+1 walk the same points at the same pose,
  // so they are one pass that writes the NEW correspondences into the other buffer set, adopted only if rho >= 0.
  const LmCfg cfg = make_lm_cfg(h->cfg, false, DBL_MAX);
  // enqueue as many rounds as the previous align needed (consecutive frames need the same number almost always): a finished
  // pair's surplus rounds exit at once, a shortfall is topped up while the device works
  const int predicted = h->last_rounds > 0 ? h->last_rounds : 5;
  rc = run_single_pair(h, x0, PM_FIRST, 0, cfg, predicted < 2 ? 2 : predicted, cov_beside);
  if (rc) return rc;
  const PairReport& rep = *h->h_rep;
  h->cur = rep.cur;
  h->corr_valid = true;
  float Tf[16];
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) Tf[r * 4 + c] = rep.r.T[c * 4 + r];
  store_result(h, Tf, rep.r.converged != 0, rep.r.iterations, out);
  return B2R_OK;
}

extern "C" int b2r_align(b2r_handle* h, const float guess[16], b2r_result* out) {
  if (!h || !guess) return fail(B2R_EINVAL, "NULL argument");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  int rc;
  if (h->cfg.method == B2R_METHOD_GICP) rc = gicp_align(h, guess, out);
  else {
    float Tfinal[16];
    bool conv = false;
    int iters = 0;
    rc = ensure_grid(h, SRC(h));  // Hilbert-ordered source points for the derivative passes
    if (rc == B2R_OK) rc = ndt_align(h->cfg, SRC(h), TGT(h), h->ndt_work, h->st, guess, Tfinal, &conv, &iters);
    if (rc == B2R_OK) store_result(h, Tfinal, conv, iters, out);
  }
  if (rc != B2R_OK && out) {
    for (int i = 0; i < 16; i++) out->T[i] = guess[i];
    out->fitness = NAN; out->converged = 0; out->iterations = 0;
  }
  return rc;
}

// ------------------------------------------------------------------------------------------------ outputs
extern "C" int b2r_get_aligned(b2r_handle* h, void* out_points, size_t n, size_t stride_bytes) {
  if (!h || (!out_points && n)) return fail(B2R_EINVAL, "NULL argument");
  if (stride_bytes < 12 || (stride_bytes & 3)) return fail(B2R_EINVAL, "bad stride");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  Cloud& s = SRC(h);
  if (n != s.n) return fail(B2R_EINVAL, "n does not match the source cloud");
  if (n == 0) return B2R_OK;
  B2R_CUDA(h->tmp_f4.reserve(n));
  XfArg X;
  for (int i = 0; i < 12; i++) X.Tf[i] = h->final_T[i];
  { TEL_BEGIN(&h->tel, h->st);
    k_transform<<<(unsigned)((n + 255) / 256), 256, 0, h->st>>>(s.raw_view, s.stride_f, (int)n, X, h->tmp_f4.p);
    TEL_END(&h->tel, KC_MISC, 1, h->st); }
  h->tel.d2h += n * sizeof(float4);
  B2R_CUDA(cudaGetLastError());
  std::vector<float4> host(n);
  B2R_CUDA(cudaMemcpyAsync(host.data(), h->tmp_f4.p, n * sizeof(float4), cudaMemcpyDeviceToHost, h->st));
  B2R_CUDA(cudaStreamSynchronize(h->st));
  char* o = (char*)out_points;
  for (size_t i = 0; i < n; i++) {
    float* p = (float*)(o + i * stride_bytes);
    p[0] = host[i].x; p[1] = host[i].y; p[2] = host[i].z;
    if (stride_bytes >= 16) p[3] = 1.0f;
  }
  return B2R_OK;
}

static int fitness_impl(b2r_handle* h, const float* T_row, double max_range, float inl, double* score, uint32_t* n_used, uint32_t* n_inl) {
  Cloud& s = SRC(h);
  Cloud& t = TGT(h);
  if (s.n == 0 || t.n == 0) {
    if (score) *score = DBL_MAX;
    if (n_used) *n_used = 0;
    if (n_inl) *n_inl = 0;
    return B2R_OK;
  }
  int rc = ensure_grid(h, t);
  if (rc) return rc;
  rc = ensure_grid(h, s);
  if (rc) return rc;
  size_t nb = (size_t)s.nsup * 1024 / kLinThreads;
  B2R_CUDA(h->partials.reserve(nb * kAcc + kAcc));
  FitArgs A;
  A.src = s.bvh(); A.tgt = t.bvh();
  for (int i = 0; i < 12; i++) A.Tf[i] = T_row[i];
  A.max_range = max_range; A.inlier_thresh_sq = inl;
  A.partials = h->partials.p; A.out = h->d_out + 40; A.counter = h->d_counter + 2;
  { TEL_BEGIN(&h->tel, h->st);
    k_fitness<<<(unsigned)nb, kLinThreads, 0, h->st>>>(A);
    TEL_END(&h->tel, KC_FITNESS, 1, h->st); }
  h->tel.d2h += 3 * sizeof(double);
  B2R_CUDA(cudaGetLastError());
  B2R_CUDA(cudaMemcpyAsync(h->h_out + 40, h->d_out + 40, 3 * sizeof(double), cudaMemcpyDeviceToHost, h->st));
  B2R_CUDA(cudaStreamSynchronize(h->st));
  double sum = h->h_out[40], nr = h->h_out[41], ni = h->h_out[42];
  if (score) *score = nr > 0 ? sum / nr : DBL_MAX;
  if (n_used) *n_used = (uint32_t)nr;
  if (n_inl) *n_inl = (uint32_t)ni;
  return B2R_OK;
}

extern "C" int b2r_fitness(b2r_handle* h, const float* T, double max_range, float inlier_thresh_sq, double* score, uint32_t* n_used,
                           uint32_t* n_inliers) {
  if (!h) return fail(B2R_EINVAL, "handle is NULL");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  float Tr[16];
  if (T) {
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++) Tr[r * 4 + c] = T[c * 4 + r];
  } else {
    std::memcpy(Tr, h->final_T, sizeof(Tr));
  }
  return fitness_impl(h, Tr, max_range, inlier_thresh_sq, score, n_used, n_inliers);
}

extern "C" int b2r_target_nearest(b2r_handle* h, const void* queries, size_t n, size_t stride_bytes, int32_t* idx_out, float* d2_out) {
  if (!h || (n && (!queries || !idx_out || !d2_out))) return fail(B2R_EINVAL, "NULL argument");
  if (stride_bytes < 12 || (stride_bytes & 3)) return fail(B2R_EINVAL, "bad stride");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  Cloud& t = TGT(h);
  if (n == 0) return B2R_OK;
  int rc = ensure_grid(h, t);
  if (rc) return rc;
  const int sf = (int)(stride_bytes / 4);
  B2R_CUDA(h->tmp_f.reserve(n * sf + n));
  B2R_CUDA(h->tmp_i.reserve(n));
  B2R_CUDA(cudaMemcpyAsync(h->tmp_f.p, queries, n * stride_bytes, cudaMemcpyHostToDevice, h->st));
  float* d2d = h->tmp_f.p + n * sf;
  { TEL_BEGIN(&h->tel, h->st);
    k_nearest<<<(unsigned)((n + 255) / 256), 256, 0, h->st>>>(h->tmp_f.p, sf, (int)n, t.bvh(), h->tmp_i.p, d2d);
    TEL_END(&h->tel, KC_MISC, 1, h->st); }
  h->tel.h2d += n * stride_bytes;
  h->tel.d2h += n * 8;
  B2R_CUDA(cudaGetLastError());
  B2R_CUDA(cudaMemcpyAsync(idx_out, h->tmp_i.p, n * sizeof(int), cudaMemcpyDeviceToHost, h->st));
  B2R_CUDA(cudaMemcpyAsync(d2_out, d2d, n * sizeof(float), cudaMemcpyDeviceToHost, h->st));
  B2R_CUDA(cudaStreamSynchronize(h->st));
  return B2R_OK;
}

extern "C" int b2r_get_correspondences(b2r_handle* h, int32_t* out, size_t n) {
  if (!h || !out) return fail(B2R_EINVAL, "NULL argument");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  if (!h->corr_valid) return fail(B2R_ESTATE, "no linearisation has run since the clouds were set");
  if (n != SRC(h).n) return fail(B2R_EINVAL, "n does not match the source cloud");
  B2R_CUDA(cudaMemcpyAsync(out, h->corr[h->cur].p, n * sizeof(int), cudaMemcpyDeviceToHost, h->st));
  B2R_CUDA(cudaStreamSynchronize(h->st));
  return B2R_OK;
}

extern "C" int b2r_get_covariances(b2r_handle* h, int which, double* out, size_t n) {
  if (!h || !out) return fail(B2R_EINVAL, "NULL argument");
  if (h->cfg.method != B2R_METHOD_GICP) return fail(B2R_ESTATE, "covariances exist only for the GICP engine");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  Cloud& c = which ? TGT(h) : SRC(h);
  if (n != c.n) return fail(B2R_EINVAL, "n does not match the cloud");
  int rc = ensure_cov(h, c);
  if (rc) return rc;
  const size_t padded = (size_t)c.nsup * 1024;
  std::vector<double> cov(padded * 6 + 6);
  std::vector<int> pos(n);
  B2R_CUDA(cudaMemcpyAsync(cov.data(), c.cov.p, padded * 6 * sizeof(double), cudaMemcpyDeviceToHost, h->st));
  B2R_CUDA(cudaMemcpyAsync(pos.data(), c.pos_of.p, n * sizeof(int), cudaMemcpyDeviceToHost, h->st));
  B2R_CUDA(cudaStreamSynchronize(h->st));
  for (size_t i = 0; i < n; i++) {
    double* o = out + i * 9;
    if (pos[i] < 0) { for (int k = 0; k < 9; k++) o[k] = NAN; continue; }
    const double* s = &cov[(size_t)pos[i] * 6];
    o[0] = s[0]; o[1] = s[1]; o[2] = s[2]; o[3] = s[1]; o[4] = s[3]; o[5] = s[4]; o[6] = s[2]; o[7] = s[4]; o[8] = s[5];
  }
  return B2R_OK;
}

extern "C" int b2r_gicp_linearize_at(b2r_handle* h, const double T[16], double* H, double* b, double* err) {
  if (!h || !T || !H || !b || !err) return fail(B2R_EINVAL, "NULL argument");
  if (h->cfg.method != B2R_METHOD_GICP) return fail(B2R_ESTATE, "GICP engine required");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  Cloud& s = SRC(h);
  Cloud& t = TGT(h);
  if (s.n == 0 || t.n == 0) return fail(B2R_ESTATE, "source/target not set");
  int rc = ensure_cov(h, s);
  if (!rc) rc = ensure_cov(h, t);
  if (!rc) rc = ensure_align_ws(h, s.n);
  if (rc) return rc;
  double x[16];
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) x[r * 4 + c] = T[c * 4 + r];
  const LmCfg cfg = make_lm_cfg(h->cfg, false, DBL_MAX);
  rc = run_single_pair(h, x, PM_FIRST, 1, cfg, 1);  // one update_correspondences + linearize round, reduced values tapped
  if (rc) return rc;
  B2R_CUDA(cudaStreamSynchronize(h->st));  // the tap words carry no checksum: wait for the stream
  h->cur = 0;
  h->corr_valid = true;
  int k = 0;
  for (int r = 0; r < 6; r++)
    for (int c = r; c < 6; c++) { H[r * 6 + c] = H[c * 6 + r] = h->h_tap[k++]; }
  for (int i = 0; i < 6; i++) b[i] = h->h_tap[21 + i];
  *err = h->h_tap[27];
  return B2R_OK;
}

extern "C" int b2r_gicp_error_at(b2r_handle* h, const double T[16], double* err) {
  if (!h || !T || !err) return fail(B2R_EINVAL, "NULL argument");
  if (!h->corr_valid) return fail(B2R_ESTATE, "no linearisation has run");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  double x[16];
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) x[r * 4 + c] = T[c * 4 + r];
  const LmCfg cfg = make_lm_cfg(h->cfg, false, DBL_MAX);
  int rc = run_single_pair(h, x, PM_ERR, 1, cfg, 1);  // compute_error with the correspondences of the last linearisation
  if (rc) return rc;
  B2R_CUDA(cudaStreamSynchronize(h->st));
  *err = h->h_tap[28];
  return B2R_OK;
}

extern "C" int b2r_ndt_get_voxels(b2r_handle* h, size_t capacity, size_t* n_voxels, int64_t* keys, int32_t* npts, double* mean,
                                  double* icov, int32_t min_b[3], int32_t div_b[3]) {
  if (!h || !n_voxels) return fail(B2R_EINVAL, "NULL argument");
  if (h->cfg.method != B2R_METHOD_NDT) return fail(B2R_ESTATE, "NDT engine required");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  int rc = ndt_ensure_map(h->cfg, TGT(h), h->ndt_work, h->st);
  if (rc) return rc;
  return ndt_dump(TGT(h), h->ndt_work, h->st, capacity, n_voxels, keys, npts, mean, icov, min_b, div_b);
}

extern "C" int b2r_ndt_derivatives_at(b2r_handle* h, const double p[6], double* score, double* g, double* H, uint64_t* n_pairs) {
  if (!h || !p || !score || !g || !H) return fail(B2R_EINVAL, "NULL argument");
  if (h->cfg.method != B2R_METHOD_NDT) return fail(B2R_ESTATE, "NDT engine required");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  if (SRC(h).n == 0 || TGT(h).n == 0) return fail(B2R_ESTATE, "source/target not set");
  int rc = ndt_ensure_map(h->cfg, TGT(h), h->ndt_work, h->st);
  if (rc) return rc;
  rc = ensure_grid(h, SRC(h));
  if (rc) return rc;
  return ndt_derivatives_at(h->cfg, SRC(h), TGT(h), h->ndt_work, h->st, p, score, g, H, n_pairs);
}

extern "C" int b2r_voxelgrid(b2r_handle* h, const void* in, size_t n, size_t stride_bytes, float leaf, void* out, size_t* n_out,
                             int32_t* out_keys, int32_t* out_counts) {
  if (!h || !n_out || (n && (!in || !out))) return fail(B2R_EINVAL, "NULL argument");
  if (stride_bytes < 12 || (stride_bytes & 3)) return fail(B2R_EINVAL, "bad stride");
  if (!(leaf > 0.f)) return fail(B2R_EINVAL, "leaf must be positive");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  return voxelgrid_filter(h->vg_work, h->st, in, n, stride_bytes, leaf, out, n_out, out_keys, out_counts);
}

extern "C" int b2r_voxelgrid_device(b2r_handle* h, const void* d_in, size_t n, size_t stride_bytes, float leaf, const void** d_out, size_t* n_out) {
  if (!h || !n_out || !d_out || (n && !d_in)) return fail(B2R_EINVAL, "NULL argument");
  if (stride_bytes < 12 || (stride_bytes & 3)) return fail(B2R_EINVAL, "bad stride");
  if (!(leaf > 0.f)) return fail(B2R_EINVAL, "leaf must be positive");
  if (n > (size_t)0x3fffffff) return fail(B2R_EINVAL, "too many points");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  *d_out = nullptr; *n_out = 0;
  if (n == 0) return B2R_OK;
  size_t m = 0;
  int overflow = 0;
  int rc = voxelgrid_device(h->vg_work, h->st, (const float*)d_in, n, stride_bytes, leaf, &m, &overflow);
  if (rc) return rc;
  h->tel.d2h += 8;
  if (overflow) { *d_out = d_in; *n_out = n; return 1; }  // PCL: "Leaf size is too small": the input passes through
  *d_out = h->vg_work.out.p;
  *n_out = m;
  return B2R_OK;
}

// ------------------------------------------------------------------------------------------------ prefilter chain (next rows)
// Every stage is device -> device: records in an engine buffer, keep flags and the order-preserving compaction on the GPU; only
// the 4-byte count of a stage comes back (host-mapped word) because the next stage's launch geometry needs it.
static int pf_reserve(b2r_handle* h, size_t n, int sf) {
  B2R_CUDA(h->pf_buf[0].reserve(n * sf + 8));
  B2R_CUDA(h->pf_buf[1].reserve(n * sf + 8));
  B2R_CUDA(h->pf_flags.reserve(n + 8));
  B2R_CUDA(h->pf_blocks.reserve((n + kCompactBlock - 1) / kCompactBlock + 8));
  B2R_CUDA(h->tmp_f.reserve(n + 8));
  if (!h->pf_stats) {
    B2R_CUDA(cudaMalloc(&h->pf_stats, sizeof(SorStats)));
    B2R_CUDA(cudaMalloc(&h->pf_total, 4 * sizeof(int)));
    B2R_CUDA(cudaHostAlloc(&h->pf_h_total, 4 * sizeof(int), cudaHostAllocMapped));
    B2R_CUDA(cudaHostGetDevicePointer((void**)&h->pf_h_total_dev, h->pf_h_total, 0));
  }
  return B2R_OK;
}

// records d_in[0..n) with flags (already on the device) -> d_out, *m = kept count
static int pf_compact(b2r_handle* h, const float* d_in, size_t n, int sf, float* d_out, size_t* m) {
  const unsigned nb = (unsigned)((n + kCompactBlock - 1) / kCompactBlock);
  unsigned char* flags = h->pf_flags.p;
  { TEL_BEGIN(&h->tel, h->st);
    k_compact_count<<<nb, kCompactBlock, 0, h->st>>>(flags, (int)n, h->pf_blocks.p);
    k_compact_scan<<<1, 1024, 0, h->st>>>(h->pf_blocks.p, (int)nb, h->pf_total, h->pf_h_total_dev);
    k_compact_scatter<<<nb, kCompactBlock, 0, h->st>>>(d_in, sf, flags, (int)n, h->pf_blocks.p, d_out);
    TEL_END(&h->tel, KC_MISC, 3, h->st); }
  B2R_CUDA(cudaGetLastError());
  B2R_CUDA(cudaStreamSynchronize(h->st));
  h->tel.d2h += 4;
  *m = (size_t)h->pf_h_total[0];
  return B2R_OK;
}

// PrefilteringNodelet::distance_filter (apps/prefiltering_nodelet.cpp:164-180)
static int pf_distance(b2r_handle* h, const float* d_in, size_t n, int sf, double near_t, double far_t, float* d_out, size_t* m) {
  { TEL_BEGIN(&h->tel, h->st);
    k_distance_flags<<<(unsigned)((n + 255) / 256), 256, 0, h->st>>>(d_in, sf, (int)n, near_t, far_t, h->pf_flags.p);
    TEL_END(&h->tel, KC_MISC, 1, h->st); }
  return pf_compact(h, d_in, n, sf, d_out, m);
}

// per-point neighbour statistic of the cloud against itself (k-th squared distance, or mean distance to the k-1 nearest others)
static int pf_knn_stat(b2r_handle* h, const float* d_in, size_t n, int sf, int k, int mode) {
  if (k < 1 || k > 64) return fail(B2R_EINVAL, "neighbour count must be in [1,64]");
  Cloud& c = h->aux;
  c.n = n; c.stride_f = sf; c.invalidate();
  c.raw_view = d_in;
  int rc = ensure_grid(h, c);
  if (rc) return rc;
  k_fill_i32<<<(unsigned)((n + 255) / 256), 256, 0, h->st>>>(reinterpret_cast<int*>(h->tmp_f.p), (int)n, 0x7fc00000);  // NaN = non-finite point
  const size_t smem = (size_t)k * kKnnThreads * sizeof(unsigned long long);
  if (smem > 48 * 1024 && !h->stat_smem_attr) {
    B2R_CUDA(cudaFuncSetAttribute(k_knn_stat, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * kKnnThreads * 8));
    h->stat_smem_attr = true;
  }
  const size_t padded = (size_t)c.nsup * 1024;
  { TEL_BEGIN(&h->tel, h->st);
    k_knn_stat<<<(unsigned)(padded / kKnnThreads), kKnnThreads, smem, h->st>>>(c.bvh(), k, mode, h->tmp_f.p);
    TEL_END(&h->tel, KC_MISC, 1, h->st); }
  B2R_CUDA(cudaGetLastError());
  return B2R_OK;
}

// pcl::RadiusOutlierRemoval (apps/prefiltering_nodelet.cpp:83-90,151-162)
static int pf_radius(b2r_handle* h, const float* d_in, size_t n, int sf, double radius, int min_neighbors, float* d_out, size_t* m) {
  int rc = pf_knn_stat(h, d_in, n, sf, min_neighbors + 1, 0);
  if (rc) return rc;
  k_radius_flags<<<(unsigned)((n + 255) / 256), 256, 0, h->st>>>(h->tmp_f.p, (int)n, radius * radius, h->pf_flags.p);
  return pf_compact(h, d_in, n, sf, d_out, m);
}

// pcl::StatisticalOutlierRemoval (apps/prefiltering_nodelet.cpp:73-81,151-162)
static int pf_statistical(b2r_handle* h, const float* d_in, size_t n, int sf, int mean_k, double stddev_mul, float* d_out, size_t* m) {
  int rc = pf_knn_stat(h, d_in, n, sf, mean_k + 1, 1);
  if (rc) return rc;
  k_sor_stats<<<1, 1024, 0, h->st>>>(h->tmp_f.p, (int)n, stddev_mul, h->pf_stats);
  k_sor_flags<<<(unsigned)((n + 255) / 256), 256, 0, h->st>>>(h->tmp_f.p, (int)n, h->pf_stats, h->pf_flags.p);
  return pf_compact(h, d_in, n, sf, d_out, m);
}

static int pf_check(b2r_handle* h, const void* in, size_t n, size_t stride_bytes, const void* out, const size_t* n_out) {
  if (!h || !n_out || (n && (!in || !out))) return fail(B2R_EINVAL, "NULL argument");
  if (stride_bytes < 12 || (stride_bytes & 3)) return fail(B2R_EINVAL, "bad stride");
  if (n > (size_t)0x3fffffff) return fail(B2R_EINVAL, "too many points");
  return B2R_OK;
}
// host records -> pf_buf[0]
static int pf_upload(b2r_handle* h, const void* in, size_t n, size_t stride_bytes) {
  int rc = pf_reserve(h, n, (int)(stride_bytes / 4));
  if (rc) return rc;
  B2R_CUDA(cudaMemcpyAsync(h->pf_buf[0].p, in, n * stride_bytes, cudaMemcpyHostToDevice, h->st));
  h->tel.h2d += n * stride_bytes;
  return B2R_OK;
}
static int pf_download(b2r_handle* h, const float* d, size_t m, size_t stride_bytes, void* out) {
  if (m) {
    B2R_CUDA(cudaMemcpyAsync(out, d, m * stride_bytes, cudaMemcpyDeviceToHost, h->st));
    B2R_CUDA(cudaStreamSynchronize(h->st));
    h->tel.d2h += m * stride_bytes;
  }
  return B2R_OK;
}

extern "C" int b2r_distance_filter(b2r_handle* h, const void* in, size_t n, size_t stride_bytes, double near_thresh, double far_thresh, void* out,
                                   size_t* n_out) {
  int rc = pf_check(h, in, n, stride_bytes, out, n_out);
  if (rc) return rc;
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  *n_out = 0;
  if (n == 0) return B2R_OK;
  rc = pf_upload(h, in, n, stride_bytes);
  if (!rc) rc = pf_distance(h, h->pf_buf[0].p, n, (int)(stride_bytes / 4), near_thresh, far_thresh, h->pf_buf[1].p, n_out);
  if (!rc) rc = pf_download(h, h->pf_buf[1].p, *n_out, stride_bytes, out);
  return rc;
}

extern "C" int b2r_radius_outlier_removal(b2r_handle* h, const void* in, size_t n, size_t stride_bytes, double radius, int min_neighbors, void* out,
                                          size_t* n_out) {
  int rc = pf_check(h, in, n, stride_bytes, out, n_out);
  if (rc) return rc;
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  *n_out = 0;
  if (n == 0) return B2R_OK;
  rc = pf_upload(h, in, n, stride_bytes);
  if (!rc) rc = pf_radius(h, h->pf_buf[0].p, n, (int)(stride_bytes / 4), radius, min_neighbors, h->pf_buf[1].p, n_out);
  if (!rc) rc = pf_download(h, h->pf_buf[1].p, *n_out, stride_bytes, out);
  return rc;
}

extern "C" int b2r_statistical_outlier_removal(b2r_handle* h, const void* in, size_t n, size_t stride_bytes, int mean_k, double stddev_mul, void* out,
                                               size_t* n_out) {
  int rc = pf_check(h, in, n, stride_bytes, out, n_out);
  if (rc) return rc;
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  *n_out = 0;
  if (n == 0) return B2R_OK;
  rc = pf_upload(h, in, n, stride_bytes);
  if (!rc) rc = pf_statistical(h, h->pf_buf[0].p, n, (int)(stride_bytes / 4), mean_k, stddev_mul, h->pf_buf[1].p, n_out);
  if (!rc) rc = pf_download(h, h->pf_buf[1].p, *n_out, stride_bytes, out);
  return rc;
}

extern "C" int b2r_deskew(b2r_handle* h, const void* in, size_t n, size_t stride_bytes, double scan_period, const float angular_velocity[3], void* out) {
  size_t dummy = 0;
  int rc = pf_check(h, in, n, stride_bytes, out, &dummy);
  if (rc) return rc;
  if (!angular_velocity) return fail(B2R_EINVAL, "NULL argument");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  if (n == 0) return B2R_OK;
  rc = pf_upload(h, in, n, stride_bytes);
  if (rc) return rc;
  // ang_v *= -1 (prefiltering_nodelet.cpp:217)
  k_deskew<<<(unsigned)((n + 255) / 256), 256, 0, h->st>>>(h->pf_buf[0].p, (int)(stride_bytes / 4), (int)n, scan_period, -angular_velocity[0], -angular_velocity[1],
                                                          -angular_velocity[2], h->pf_buf[1].p);
  B2R_CUDA(cudaGetLastError());
  return pf_download(h, h->pf_buf[1].p, n, stride_bytes, out);
}

extern "C" int b2r_prefilter_params_default(b2r_prefilter_params* p) {
  if (!p) return fail(B2R_EINVAL, "NULL argument");
  std::memset(p, 0, sizeof(*p));
  p->deskewing = 0; p->scan_period = 0.1;                              // prefiltering_nodelet.cpp:36,234
  p->use_distance_filter = 1; p->distance_near_thresh = 1.0; p->distance_far_thresh = 100.0;  // :96-98
  p->downsample_method = B2R_DOWNSAMPLE_VOXELGRID; p->downsample_resolution = 0.1f;            // :51-52
  p->outlier_removal_method = B2R_OUTLIER_STATISTICAL;                  // :71
  p->statistical_mean_k = 20; p->statistical_stddev = 1.0;              // :73-74
  p->radius_radius = 0.8; p->radius_min_neighbors = 2;                  // :83-84
  return B2R_OK;
}

// PrefilteringNodelet::cloud_callback (apps/prefiltering_nodelet.cpp:106-136): deskewing -> [base_link transform] -> distance_filter ->
// downsample -> outlier_removal, the cloud never leaving HBM between the stages
extern "C" int b2r_prefilter(b2r_handle* h, const void* points, size_t n, size_t stride_bytes, int device_input, const b2r_prefilter_params* p,
                             void* out_host, const void** d_out, size_t* n_out) {
  if (!h || !p || !n_out || (n && !points)) return fail(B2R_EINVAL, "NULL argument");
  if (stride_bytes < 12 || (stride_bytes & 3)) return fail(B2R_EINVAL, "bad stride");
  if (n > (size_t)0x3fffffff) return fail(B2R_EINVAL, "too many points");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  *n_out = 0;
  if (d_out) *d_out = nullptr;
  if (n == 0) return B2R_OK;  // cloud_callback returns on an empty cloud (:108-110)
  const int sf = (int)(stride_bytes / 4);
  int rc = pf_reserve(h, n, sf);
  if (rc) return rc;
  const float* cur = nullptr;
  int nxt = 0;  // index of the free ping-pong buffer
  if (device_input) cur = (const float*)points;
  else {
    B2R_CUDA(cudaMemcpyAsync(h->pf_buf[0].p, points, n * stride_bytes, cudaMemcpyHostToDevice, h->st));
    h->tel.h2d += n * stride_bytes;
    cur = h->pf_buf[0].p; nxt = 1;
  }
  size_t m = n;
  auto advance = [&]() { cur = h->pf_buf[nxt].p; nxt ^= 1; };
  const unsigned nb256 = (unsigned)((n + 255) / 256);
  if (p->deskewing) {  // :182-243
    k_deskew<<<nb256, 256, 0, h->st>>>(cur, sf, (int)m, p->scan_period, -p->angular_velocity[0], -p->angular_velocity[1], -p->angular_velocity[2], h->pf_buf[nxt].p);
    advance();
  }
  if (p->use_base_link_transform) {  // :114-129
    XfArgPF X;
    for (int r = 0; r < 3; r++) for (int c = 0; c < 4; c++) X.Tf[r * 4 + c] = p->base_link_transform[c * 4 + r];
    k_transform_records<<<nb256, 256, 0, h->st>>>(cur, sf, (int)m, X, h->pf_buf[nxt].p);
    advance();
  }
  if (p->use_distance_filter) {  // :131
    rc = pf_distance(h, cur, m, sf, p->distance_near_thresh, p->distance_far_thresh, h->pf_buf[nxt].p, &m);
    if (rc) return rc;
    advance();
  }
  if (p->downsample_method == B2R_DOWNSAMPLE_VOXELGRID && m) {  // :132
    size_t mv = 0;
    int overflow = 0;
    rc = voxelgrid_device(h->vg_work, h->st, cur, m, stride_bytes, p->downsample_resolution, &mv, &overflow);
    if (rc) return rc;
    if (!overflow) { cur = h->vg_work.out.p; m = mv; }  // (the voxel grid writes its own buffer: the ping-pong pair stays free)
  }
  if (p->outlier_removal_method == B2R_OUTLIER_STATISTICAL && m) {  // :133
    rc = pf_statistical(h, cur, m, sf, p->statistical_mean_k, p->statistical_stddev, h->pf_buf[nxt].p, &m);
    if (rc) return rc;
    advance();
  } else if (p->outlier_removal_method == B2R_OUTLIER_RADIUS && m) {
    rc = pf_radius(h, cur, m, sf, p->radius_radius, p->radius_min_neighbors, h->pf_buf[nxt].p, &m);
    if (rc) return rc;
    advance();
  }
  B2R_CUDA(cudaGetLastError());
  *n_out = m;
  if (d_out) *d_out = cur;
  if (out_host) return pf_download(h, cur, m, stride_bytes, out_host);
  B2R_CUDA(cudaStreamSynchronize(h->st));
  return B2R_OK;
}

// ------------------------------------------------------------------------------------------------ wire / disk ingest ("next" row f-4)
static int ingest_device(b2r_handle* h, const unsigned char* d_blob, size_t n, const b2r_point_layout& L, const void** d_out) {
  B2R_CUDA(h->ingest_out.reserve(n * 8 + 8));
  UnpackArgs A;
  A.data = d_blob; A.n = (long long)n; A.point_step = L.point_step; A.off_x = L.off_x; A.off_y = L.off_y; A.off_z = L.off_z;
  A.off_i = L.off_intensity; A.type_i = L.intensity_datatype; A.bigendian = L.is_bigendian; A.out = h->ingest_out.p;
  { TEL_BEGIN(&h->tel, h->st);
    k_unpack_points<<<(unsigned)std::min<size_t>((n + 255) / 256, (size_t)h->n_sm * 16), 256, 0, h->st>>>(A);
    TEL_END(&h->tel, KC_MISC, 1, h->st); }
  B2R_CUDA(cudaGetLastError());
  *d_out = h->ingest_out.p;
  return B2R_OK;
}
static int layout_check(const b2r_point_layout* L) {
  if (!L) return fail(B2R_EINVAL, "NULL layout");
  if (L->point_step < 12) return fail(B2R_EINVAL, "point_step too small");
  const unsigned int need[3] = {L->off_x, L->off_y, L->off_z};
  for (unsigned int o : need) if (o + 4 > L->point_step) return fail(B2R_EINVAL, "field offset beyond point_step");
  if (L->off_intensity != 0xffffffffu) {
    const unsigned int t = L->intensity_datatype;
    const unsigned int sz = (t == 1 || t == 2) ? 1 : (t == 3 || t == 4) ? 2 : (t == 8) ? 8 : 4;
    if (t < 1 || t > 8) return fail(B2R_EINVAL, "unknown PointField datatype");
    if (L->off_intensity + sz > L->point_step) return fail(B2R_EINVAL, "intensity offset beyond point_step");
  }
  return B2R_OK;
}

extern "C" int b2r_ingest_pointcloud2(b2r_handle* h, const void* data, size_t n_points, const b2r_point_layout* layout, const void** d_points) {
  if (!h || !d_points || (n_points && !data)) return fail(B2R_EINVAL, "NULL argument");
  int rc = layout_check(layout);
  if (rc) return rc;
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  *d_points = nullptr;
  if (n_points == 0) return B2R_OK;
  if (n_points > (size_t)0x3fffffff) return fail(B2R_EINVAL, "too many points");
  const size_t bytes = n_points * layout->point_step;
  B2R_CUDA(h->ingest_blob.reserve(bytes + 16));
  B2R_CUDA(cudaMemcpyAsync(h->ingest_blob.p, data, bytes, cudaMemcpyHostToDevice, h->st));  // the message's data[] goes up unconverted
  h->tel.h2d += bytes;
  return ingest_device(h, reinterpret_cast<const unsigned char*>(h->ingest_blob.p), n_points, *layout, d_points);
}

extern "C" int b2r_pcd_read_header(const char* path, b2r_point_layout* layout, size_t* n_points, size_t* data_offset) {
  if (!path || !layout || !n_points) return fail(B2R_EINVAL, "NULL argument");
  FILE* f = fopen(path, "rb");
  if (!f) return fail(B2R_EINVAL, std::string("cannot open ") + path);
  PcdHeader H;
  const bool ok = pcd_parse_header(f, H);
  fclose(f);
  if (!ok) return fail(B2R_EINVAL, "not a PCD header");
  if (H.data != "binary") return fail(B2R_EUNSUPPORTED, "only DATA binary is read directly (KeyFrame::save writes savePCDFileBinary)");
  std::memset(layout, 0, sizeof(*layout));
  layout->off_intensity = 0xffffffffu; layout->intensity_datatype = 7;
  unsigned int off = 0, found = 0;
  for (size_t i = 0; i < H.fields.size(); i++) {
    const unsigned int sz = (unsigned int)(H.size[i] * H.count[i]);
    const bool f32 = H.type[i] == 'F' && H.size[i] == 4;
    if (H.fields[i] == "x" && f32) { layout->off_x = off; found |= 1; }
    else if (H.fields[i] == "y" && f32) { layout->off_y = off; found |= 2; }
    else if (H.fields[i] == "z" && f32) { layout->off_z = off; found |= 4; }
    else if (H.fields[i] == "intensity") {
      layout->off_intensity = off;
      const char t = H.type[i];
      layout->intensity_datatype = (t == 'F') ? (H.size[i] == 8 ? 8 : 7) : (t == 'U') ? (H.size[i] == 1 ? 2 : H.size[i] == 2 ? 4 : 6) : (H.size[i] == 1 ? 1 : H.size[i] == 2 ? 3 : 5);
    }
    off += sz;
  }
  if (found != 7) return fail(B2R_EINVAL, "PCD has no float32 x / y / z fields");
  layout->point_step = off;
  *n_points = H.points;
  if (data_offset) *data_offset = H.data_offset;
  return B2R_OK;
}

extern "C" int b2r_ingest_pcd(b2r_handle* h, const char* path, const void** d_points, size_t* n_points) {
  if (!h || !d_points || !n_points) return fail(B2R_EINVAL, "NULL argument");
  b2r_point_layout L;
  size_t n = 0, off = 0;
  int rc = b2r_pcd_read_header(path, &L, &n, &off);
  if (rc) return rc;
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  *d_points = nullptr; *n_points = 0;
  if (n == 0) return B2R_OK;
  const size_t bytes = n * L.point_step;
  if (h->ingest_pinned_cap < bytes) {  // the file body is read straight into pinned memory: no intermediate PointCloud, no repack
    if (h->ingest_pinned) cudaFreeHost(h->ingest_pinned);
    h->ingest_pinned = nullptr; h->ingest_pinned_cap = 0;
    B2R_CUDA(cudaMallocHost(&h->ingest_pinned, bytes + bytes / 4 + 4096));
    h->ingest_pinned_cap = bytes + bytes / 4 + 4096;
  } else {
    B2R_CUDA(cudaStreamSynchronize(h->st));  // a previous upload from this buffer may still be in flight
  }
  FILE* f = fopen(path, "rb");
  if (!f) return fail(B2R_EINVAL, std::string("cannot open ") + path);
  bool ok = fseek(f, (long)off, SEEK_SET) == 0 && fread(h->ingest_pinned, 1, bytes, f) == bytes;
  fclose(f);
  if (!ok) return fail(B2R_EINVAL, "PCD body shorter than its header says");
  B2R_CUDA(h->ingest_blob.reserve(bytes + 16));
  B2R_CUDA(cudaMemcpyAsync(h->ingest_blob.p, h->ingest_pinned, bytes, cudaMemcpyHostToDevice, h->st));
  h->tel.h2d += bytes;
  rc = ingest_device(h, reinterpret_cast<const unsigned char*>(h->ingest_blob.p), n, L, d_points);
  if (rc) return rc;
  *n_points = n;
  return B2R_OK;
}

// ------------------------------------------------------------------------------------------------ map cloud ("next" row f-3)
extern "C" int b2r_map_cloud_generate(b2r_handle* h, const b2r_keyframe_snapshot* keyframes, size_t n_keyframes, size_t stride_bytes, double resolution,
                                      void* out, size_t out_capacity, size_t* n_out) {
  if (!h || !n_out) return fail(B2R_EINVAL, "NULL argument");
  *n_out = 0;
  if (n_keyframes == 0) return 1;  // "warning: keyframes empty!!" -> nullptr (map_cloud_generator.cpp:14-17)
  if (!keyframes || !out) return fail(B2R_EINVAL, "NULL argument");
  if (stride_bytes < 12 || (stride_bytes & 3)) return fail(B2R_EINVAL, "bad stride");
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  const int sf = (int)(stride_bytes / 4);
  size_t total = 0;
  for (size_t k = 0; k < n_keyframes; k++) {
    if (keyframes[k].n && !keyframes[k].points) return fail(B2R_EINVAL, "keyframe cloud is NULL");
    total += keyframes[k].n;
  }
  if (total >= (size_t)0x7fffffff) return fail(B2R_EINVAL, "map cloud too large (>= 2^31 points)");
  if (total == 0) return B2R_OK;
  cudaStream_t st = h->st;
  // upload: all keyframe clouds back to back + their descriptors
  DevBuf<float>& src = h->pf_buf[0];
  DevBuf<float>& cloud = h->pf_buf[1];
  B2R_CUDA(src.reserve(total * sf + 8));
  B2R_CUDA(cloud.reserve(total * sf + 8));
  std::vector<MapKf> kf(n_keyframes);
  size_t first = 0;
  for (size_t k = 0; k < n_keyframes; k++) {
    kf[k].pts = src.p + first * sf; kf[k].first = (long long)first; kf[k].n = (int)keyframes[k].n; kf[k].pad = 0;
    for (int r = 0; r < 3; r++) for (int c = 0; c < 4; c++) kf[k].T[r * 4 + c] = keyframes[k].pose[c * 4 + r];
    if (keyframes[k].n) B2R_CUDA(cudaMemcpyAsync(src.p + first * sf, keyframes[k].points, keyframes[k].n * stride_bytes, cudaMemcpyHostToDevice, st));
    first += keyframes[k].n;
  }
  h->tel.h2d += total * stride_bytes;
  // empty keyframes must not shadow their successors in the binary search: drop them from the descriptor list
  std::vector<MapKf> kf2;
  for (auto& k : kf) if (k.n > 0) kf2.push_back(k);
  B2R_CUDA(h->map_kf.reserve(kf2.size() * sizeof(MapKf) + 64));
  B2R_CUDA(cudaMemcpyAsync(h->map_kf.p, kf2.data(), kf2.size() * sizeof(MapKf), cudaMemcpyHostToDevice, st));
  B2R_CUDA(cudaStreamSynchronize(st));  // kf2 is pageable host memory on the stack of this call
  const long long T = (long long)total;
  unsigned nb = (unsigned)std::min<size_t>((total + 255) / 256, (size_t)h->n_sm * 16);
  { TEL_BEGIN(&h->tel, st);
    k_map_transform<<<nb, 256, 0, st>>>(reinterpret_cast<const MapKf*>(h->map_kf.p), (int)kf2.size(), sf, T, cloud.p);
    TEL_END(&h->tel, KC_MISC, 1, st); }
  if (!(resolution > 0.0)) {  // "To get unfiltered point cloud with intensity" (:39-40)
    if (out_capacity < total) return fail(B2R_EINVAL, "output capacity too small");
    B2R_CUDA(cudaMemcpyAsync(out, cloud.p, total * stride_bytes, cudaMemcpyDeviceToHost, st));
    B2R_CUDA(cudaStreamSynchronize(st));
    h->tel.d2h += total * stride_bytes;
    *n_out = total;
    return B2R_OK;
  }
  // voxel keys -> sort -> unique -> centres
  B2R_CUDA(h->map_keys[0].reserve(total + 8));
  B2R_CUDA(h->map_keys[1].reserve(total + 8));
  B2R_CUDA(h->tmp_i.reserve(2 * total + 16));
  int* flags = h->tmp_i.p;
  int* slots = h->tmp_i.p + total + 8;
  size_t tmp_sort = 0, tmp_scan = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, tmp_sort, h->map_keys[0].p, h->map_keys[1].p, (int)total, 0, 64, st);
  cub::DeviceScan::ExclusiveSum(nullptr, tmp_scan, flags, slots, (int)total, st);
  B2R_CUDA(h->bc[0].sort_tmp.reserve(std::max(tmp_sort, tmp_scan) + 256));
  if (!h->map_geom) {
    B2R_CUDA(cudaMalloc(&h->map_geom, sizeof(MapGeom) + 64));
    B2R_CUDA(cudaMallocHost(&h->map_h, 64));
  }
  unsigned long long* first_idx = reinterpret_cast<unsigned long long*>(reinterpret_cast<char*>(h->map_geom) + sizeof(MapGeom));
  int* n_dev = reinterpret_cast<int*>(first_idx + 1);
  { TEL_BEGIN(&h->tel, st);
    // replay of the octree's bounding-box growth: each round finds the first point outside the box and grows the box for it; the
    // box settles after ~log2(extent / resolution) rounds, further rounds exit at once (G.done)
    k_oct_init<<<1, 1, 0, st>>>(h->map_geom, resolution, first_idx);
    for (int round = 0; round < 48; round++) {
      k_oct_first_violator<<<nb, 256, 0, st>>>(cloud.p, sf, T, h->map_geom, first_idx);
      k_oct_grow<<<1, 1, 0, st>>>(cloud.p, sf, h->map_geom, first_idx);
    }
    k_map_keys<<<nb, 256, 0, st>>>(cloud.p, sf, T, h->map_geom, h->map_keys[0].p);
    size_t tb = h->bc[0].sort_tmp.cap;
    cub::DeviceRadixSort::SortKeys(h->bc[0].sort_tmp.p, tb, h->map_keys[0].p, h->map_keys[1].p, (int)total, 0, 64, st);
    k_map_heads<<<nb, 256, 0, st>>>(h->map_keys[1].p, T, flags);
    tb = h->bc[0].sort_tmp.cap;
    cub::DeviceScan::ExclusiveSum(h->bc[0].sort_tmp.p, tb, flags, slots, (int)total, st);
    k_map_centers<<<nb, 256, 0, st>>>(h->map_keys[1].p, flags, slots, T, h->map_geom, sf, src.p, n_dev);
    TEL_END(&h->tel, KC_MISC, 106, st); }
  B2R_CUDA(cudaGetLastError());
  B2R_CUDA(cudaMemcpyAsync(h->map_h, n_dev, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2R_CUDA(cudaStreamSynchronize(st));
  const size_t m = (size_t)h->map_h[0];
  if (out_capacity < m) return fail(B2R_EINVAL, "output capacity too small");
  if (m) {
    B2R_CUDA(cudaMemcpyAsync(out, src.p, m * stride_bytes, cudaMemcpyDeviceToHost, st));
    B2R_CUDA(cudaStreamSynchronize(st));
    h->tel.d2h += m * stride_bytes;
  }
  *n_out = m;
  return B2R_OK;
}

// ------------------------------------------------------------------------------------------------ odometry mirror
struct b2r_odometry {
  b2r_handle* reg;
  b2r_odometry_params p;
  bool has_keyframe = false;
  double prev_time = 0, keyframe_stamp = 0;
  bool prev_time_zero = true;
  float prev_trans[16];     // row-major
  float keyframe_pose[16];  // row-major
  // announced next cloud (b2r_odometry_prefetch): prefetched right after the current source has been adopted
  const void* next_ptr = nullptr;
  size_t next_n = 0, next_stride = 0;
  bool next_device = false, next_pending = false;
};

static void mat4_identity(float* m) { for (int i = 0; i < 16; i++) m[i] = (i % 5 == 0) ? 1.f : 0.f; }
static void mat4_mul(const float* a, const float* b, float* o) {
  float t[16];
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) {
      float s = a[r * 4 + 0] * b[0 * 4 + c];
      s += a[r * 4 + 1] * b[1 * 4 + c];
      s += a[r * 4 + 2] * b[2 * 4 + c];
      s += a[r * 4 + 3] * b[3 * 4 + c];
      t[r * 4 + c] = s;
    }
  std::memcpy(o, t, sizeof(t));
}
static void mat4_inv_rigid_general(const float* m, float* o) {
  // general affine inverse of [A t; 0 1] with A 3x3 (Eigen Matrix4f::inverse() on a rigid transform)
  double A[9] = {m[0], m[1], m[2], m[4], m[5], m[6], m[8], m[9], m[10]}, Ai[9];
  inv3(A, Ai);
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) o[r * 4 + c] = (float)Ai[r * 3 + c];
    o[r * 4 + 3] = (float)(-(Ai[r * 3 + 0] * m[3] + Ai[r * 3 + 1] * m[7] + Ai[r * 3 + 2] * m[11]));
  }
  o[12] = o[13] = o[14] = 0.f; o[15] = 1.f;
}
// w of Eigen::Quaternionf(R) (rotation matrix -> quaternion, Eigen's branchy algorithm)
static float quat_w_from_R(const float* m) {
  float t = m[0] + m[5] + m[10];
  if (t > 0.f) {
    t = std::sqrt(t + 1.0f);
    return 0.5f * t;
  }
  int i = 0;
  if (m[5] > m[0]) i = 1;
  if (m[10] > m[i * 4 + i]) i = 2;
  int j = (i + 1) % 3, k = (j + 1) % 3;
  t = std::sqrt(m[i * 4 + i] - m[j * 4 + j] - m[k * 4 + k] + 1.0f);
  t = 0.5f / t;
  return (m[k * 4 + j] - m[j * 4 + k]) * t;
}
static void row_to_col(const float* r, float* c) {
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) c[j * 4 + i] = r[i * 4 + j];
}

extern "C" int b2r_odometry_create(b2r_handle* reg, const b2r_odometry_params* p, b2r_odometry** out) {
  if (!reg || !out) return fail(B2R_EINVAL, "NULL argument");
  b2r_odometry* o = new b2r_odometry();
  o->reg = reg;
  if (p) o->p = *p;
  else {
    o->p.keyframe_delta_trans = 0.25; o->p.keyframe_delta_angle = 0.15; o->p.keyframe_delta_time = 1.0;
    o->p.transform_thresholding = 0; o->p.max_acceptable_trans = 1.0; o->p.max_acceptable_angle = 1.0; o->p.publish_status = 0;
  }
  mat4_identity(o->prev_trans);
  mat4_identity(o->keyframe_pose);
  *out = o;
  return B2R_OK;
}
extern "C" void b2r_odometry_destroy(b2r_odometry* o) { delete o; }

static int odometry_matching_impl(b2r_odometry* o, double stamp, const void* cloud, size_t n, size_t stride_bytes, const float* msf_delta,
                                  b2r_odometry_status* out, bool device);
extern "C" int b2r_odometry_prefetch(b2r_odometry* o, const void* cloud, size_t n, size_t stride_bytes, int device) {
  if (!o) return fail(B2R_EINVAL, "NULL argument");
  o->next_ptr = cloud; o->next_n = n; o->next_stride = stride_bytes; o->next_device = device != 0; o->next_pending = true;
  return B2R_OK;
}
static int odometry_issue_prefetch(b2r_odometry* o) {
  if (!o->next_pending) return B2R_OK;
  o->next_pending = false;
  return o->next_device ? b2r_prefetch_source_device(o->reg, o->next_ptr, o->next_n, o->next_stride)
                        : b2r_prefetch_source(o->reg, o->next_ptr, o->next_n, o->next_stride);
}

extern "C" int b2r_odometry_matching(b2r_odometry* o, double stamp, const void* cloud, size_t n, size_t stride_bytes,
                                     const float* msf_delta, b2r_odometry_status* out) {
  return odometry_matching_impl(o, stamp, cloud, n, stride_bytes, msf_delta, out, false);
}
extern "C" int b2r_odometry_matching_device(b2r_odometry* o, double stamp, const void* d_cloud, size_t n, size_t stride_bytes,
                                            const float* msf_delta, b2r_odometry_status* out) {
  return odometry_matching_impl(o, stamp, d_cloud, n, stride_bytes, msf_delta, out, true);
}
static int odometry_matching_impl(b2r_odometry* o, double stamp, const void* cloud, size_t n, size_t stride_bytes, const float* msf_delta,
                                  b2r_odometry_status* out, bool device) {
  if (!o || !out) return fail(B2R_EINVAL, "NULL argument");
  std::memset(out, 0, sizeof(*out));
  out->matching_error = NAN;
  out->inlier_fraction = NAN;
  b2r_handle* reg = o->reg;
  float I[16];
  mat4_identity(I);
  if (!o->has_keyframe) {  // :166-174
    o->prev_time_zero = true;
    mat4_identity(o->prev_trans);
    mat4_identity(o->keyframe_pose);
    o->keyframe_stamp = stamp;
    int rc = device ? b2r_set_target_device(reg, cloud, n, stride_bytes) : b2r_set_target(reg, cloud, n, stride_bytes);
    if (rc) return rc;
    rc = odometry_issue_prefetch(o);
    if (rc) return rc;
    o->has_keyframe = true;
    row_to_col(I, out->odom);
    row_to_col(I, out->trans);
    out->keyframe_updated = 1;
    return B2R_OK;
  }
  int rc = device ? b2r_set_source_device(reg, cloud, n, stride_bytes) : b2r_set_source(reg, cloud, n, stride_bytes);  // :177
  if (rc) return rc;
  rc = odometry_issue_prefetch(o);  // the NEXT frame's upload / BVH / covariances overlap this frame's align on a second stream
  if (rc) return rc;
  float guess_row[16], delta_row[16];
  if (msf_delta) { for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) delta_row[r * 4 + c] = msf_delta[c * 4 + r]; }
  else mat4_identity(delta_row);
  mat4_mul(o->prev_trans, delta_row, guess_row);  // :210 prev_trans * msf_delta.matrix()
  float guess_col[16];
  row_to_col(guess_row, guess_col);
  b2r_result res;
  rc = b2r_align(reg, guess_col, &res);
  if (rc) return rc;
  out->converged = res.converged;
  out->iterations = res.iterations;
  std::memcpy(out->trans, res.T, sizeof(res.T));
  if (o->p.publish_status) {  // :298-335
    double score;
    uint32_t used, inl;
    rc = b2r_fitness(reg, nullptr, DBL_MAX, 0.5f * 0.5f, &score, &used, &inl);
    if (rc) return rc;
    out->matching_error = score;
    out->inlier_fraction = n ? (float)inl / (float)n : 0.f;
  }
  float odom_row[16];
  if (!res.converged) {  // :214-218
    mat4_mul(o->keyframe_pose, o->prev_trans, odom_row);
    row_to_col(odom_row, out->odom);
    out->frame_rejected = 1;
    return B2R_OK;
  }
  float trans[16];
  for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) trans[r * 4 + c] = res.T[c * 4 + r];
  mat4_mul(o->keyframe_pose, trans, odom_row);
  if (o->p.transform_thresholding) {  // :223-233
    float inv[16], delta[16];
    mat4_inv_rigid_general(o->prev_trans, inv);
    mat4_mul(inv, trans, delta);
    double dx = std::sqrt((double)delta[3] * delta[3] + (double)delta[7] * delta[7] + (double)delta[11] * delta[11]);
    double da = std::acos((double)quat_w_from_R(delta));
    if (dx > o->p.max_acceptable_trans || da > o->p.max_acceptable_angle) {
      mat4_mul(o->keyframe_pose, o->prev_trans, odom_row);
      row_to_col(odom_row, out->odom);
      out->frame_rejected = 1;
      return B2R_OK;
    }
  }
  o->prev_time = stamp;
  o->prev_time_zero = false;
  std::memcpy(o->prev_trans, trans, sizeof(trans));
  float tn = std::sqrt(trans[3] * trans[3] + trans[7] * trans[7] + trans[11] * trans[11]);
  double delta_trans = tn;
  double delta_angle = std::acos((double)quat_w_from_R(trans));
  double delta_time = stamp - o->keyframe_stamp;
  if (delta_trans > o->p.keyframe_delta_trans || delta_angle > o->p.keyframe_delta_angle || delta_time > o->p.keyframe_delta_time) {  // :241-252
    rc = b2r_promote_source_to_target(reg);  // keyframe = filtered; registration->setInputTarget(keyframe)
    if (rc) return rc;
    std::memcpy(o->keyframe_pose, odom_row, sizeof(odom_row));
    o->keyframe_stamp = stamp;
    o->prev_time = stamp;
    mat4_identity(o->prev_trans);
    out->keyframe_updated = 1;
  }
  row_to_col(odom_row, out->odom);
  return B2R_OK;
}

// ------------------------------------------------------------------------------------------------ batched path + loop-closure mirror
#include "batch.cuh"

extern "C" int b2r_loop_matching(b2r_handle* h, const void* new_keyframe, size_t n_new, size_t stride_bytes, const void* const* candidates,
                                 const size_t* n_candidates_pts, size_t n_candidates, const float* guesses, double fitness_score_max_range,
                                 double fitness_score_thresh, b2r_result* results, int32_t* best) {
  if (!h || !best) return fail(B2R_EINVAL, "NULL argument");
  *best = -1;
  if (n_candidates == 0) return B2R_OK;  // loop_detector.hpp:118-120
  if (!candidates || !n_candidates_pts || !guesses) return fail(B2R_EINVAL, "NULL argument");
  if (h->cfg.method != B2R_METHOD_GICP) {  // NDT handle: the reference's sequential loop, one align + getFitnessScore per candidate
    int rc = b2r_set_target(h, new_keyframe, n_new, stride_bytes);  // :122
    if (rc) return rc;
    std::vector<b2r_result> rs(n_candidates);
    for (size_t i = 0; i < n_candidates; i++) {  // :135-154
      rc = b2r_set_source(h, candidates[i], n_candidates_pts[i], stride_bytes);
      if (rc) return rc;
      rc = b2r_align(h, guesses + i * 16, &rs[i]);
      if (rc) return rc;
      double score;
      rc = b2r_fitness(h, nullptr, fitness_score_max_range, 0.25f, &score, nullptr, nullptr);
      if (rc) return rc;
      rs[i].fitness = score;
      if (results) results[i] = rs[i];
    }
    return b2r_loop_argmin(rs.data(), n_candidates, fitness_score_thresh, best);
  }
  // GICP: the candidate loop is ONE batched registration — all candidates of the new keyframe share the target (:122) and only
  // couple through the argmin (:147), so every LM iteration of every candidate is one pair of launches (pair_engine.cuh)
  if (!h->loop_batch) {
    int rc = b2r_batch_create(&h->cfg, &h->loop_batch);
    if (rc) return rc;
  }
  b2r_batch* b = h->loop_batch;
  std::vector<int32_t> ids(n_candidates + 1, -1);
  auto cleanup = [&]() { for (int32_t id : ids) if (id >= 0) b2r_batch_remove_cloud(b, id); };
  int rc = b2r_batch_add_cloud(b, new_keyframe, n_new, stride_bytes, &ids[0]);
  for (size_t i = 0; i < n_candidates && !rc; i++) rc = b2r_batch_add_cloud(b, candidates[i], n_candidates_pts[i], stride_bytes, &ids[i + 1]);
  std::vector<b2r_pair> pairs(n_candidates);
  std::vector<b2r_result> rs(n_candidates);
  if (!rc) {
    for (size_t i = 0; i < n_candidates; i++) {
      pairs[i].source = ids[i + 1];
      pairs[i].target = ids[0];
      std::memcpy(pairs[i].guess, guesses + i * 16, 16 * sizeof(float));
    }
    rc = b2r_batch_align(b, pairs.data(), n_candidates, 1, fitness_score_max_range, rs.data());
  }
  if (rc) { const std::string msg = g_last_error; cleanup(); g_last_error = msg; return rc; }
  cleanup();
  if (results) for (size_t i = 0; i < n_candidates; i++) results[i] = rs[i];
  return b2r_loop_argmin(rs.data(), n_candidates, fitness_score_thresh, best);
}
