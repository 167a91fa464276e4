// engine.cuh — handle state of libb200reg: per-cloud device buffers, workspaces, stream.
#pragma once
#include <cuda_runtime.h>
#include <memory>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>
#include <cstring>
#include <cstdio>
#include <cstdlib>
#include "../../include/b200reg.h"
#include "common.cuh"
#include "grid.cuh"
#include "bvh.cuh"

namespace b2r {

extern thread_local std::string g_last_error;
inline int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}
#define B2R_CUDA(expr)                                                                                   \
  do {                                                                                                   \
    cudaError_t _e = (expr);                                                                             \
    if (_e != cudaSuccess) {                                                                             \
      return b2r::fail(B2R_ECUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));                   \
    }                                                                                                    \
  } while (0)

// ---- ownership: every device, pinned and mapped buffer, stream and event of the engine is owned by one of the types below and
// freed by its destructor.  A destructor frees on the CURRENT device: each destroy entry point sets its object's device first.
struct DeviceMem {
  static cudaError_t alloc(void** p, void**, size_t bytes) { return cudaMalloc(p, bytes); }
  static void free(void* p) { cudaFree(p); }
};
struct PinnedMem {
  static cudaError_t alloc(void** p, void**, size_t bytes) { return cudaMallocHost(p, bytes); }
  static void free(void* p) { cudaFreeHost(p); }
};
struct MappedMem {  // pinned host memory that kernels read and write in place, at the device alias `d`
  static cudaError_t alloc(void** p, void** d, size_t bytes) {
    cudaError_t e = cudaHostAlloc(p, bytes, cudaHostAllocMapped);
    return e == cudaSuccess ? cudaHostGetDevicePointer(d, *p, 0) : e;
  }
  static void free(void* p) { cudaFreeHost(p); }
};

template <class T, class Mem>
struct Buf {
  T* p = nullptr;
  T* d = nullptr;  // MappedMem: the device's address of p
  size_t cap = 0;
  Buf() = default;
  Buf(const Buf&) = delete;
  Buf& operator=(const Buf&) = delete;
  Buf(Buf&& o) noexcept : p(o.p), d(o.d), cap(o.cap) { o.p = o.d = nullptr; o.cap = 0; }
  Buf& operator=(Buf&& o) noexcept { std::swap(p, o.p); std::swap(d, o.d); std::swap(cap, o.cap); return *this; }
  ~Buf() { if (p) Mem::free(p); }
  // exactly n elements, unless it holds n already (the old contents are not kept)
  cudaError_t alloc(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) Mem::free(p);
    p = d = nullptr;
    cudaError_t e = Mem::alloc((void**)&p, (void**)&d, n * sizeof(T));
    cap = (e == cudaSuccess) ? n : 0;
    return e;
  }
  // growable workspace: n elements and an eighth (+64) more, so that a slowly growing input does not reallocate on every call
  cudaError_t reserve(size_t n) { return n <= cap ? cudaSuccess : alloc(n + n / 8 + 64); }
};
template <class T> using DevBuf = Buf<T, DeviceMem>;
template <class T> using PinnedBuf = Buf<T, PinnedMem>;
template <class T> using MappedBuf = Buf<T, MappedMem>;
static_assert(!std::is_copy_constructible<DevBuf<char>>::value, "DevBuf owns its memory");

struct Event {
  cudaEvent_t e = nullptr;
  Event() = default;
  Event(const Event&) = delete;
  Event& operator=(const Event&) = delete;
  ~Event() { if (e) cudaEventDestroy(e); }
  cudaError_t create() { return cudaEventCreateWithFlags(&e, cudaEventDisableTiming); }
  operator cudaEvent_t() const { return e; }
};
struct Stream {
  cudaStream_t s = nullptr;
  Stream() = default;
  Stream(const Stream&) = delete;
  Stream& operator=(const Stream&) = delete;
  ~Stream() { if (s) cudaStreamDestroy(s); }
  // priority 0 is the default priority, the one cudaStreamCreateWithFlags gives
  cudaError_t create(unsigned flags, int priority = 0) { return cudaStreamCreateWithPriority(&s, flags, priority); }
  operator cudaStream_t() const { return s; }
};

// ---- telemetry: copy byte counters, launch counters and (optional) CUDA-event timing per kernel class
enum KernelClass { KC_GRID = 0, KC_KNN_COV, KC_GICP_CORR, KC_GICP_LIN, KC_GICP_ERR, KC_FITNESS, KC_NDT_BUILD, KC_NDT_DERIV, KC_NDT_HESS, KC_VOXELGRID, KC_MISC, KC_VGICP_MAP, KC_VGICP_ROUND, KC_GICP_PCL_CORR, KC_GICP_PCL_COST, KC_ICP_PCL, KC_COUNT };
inline const char* kernel_class_name(int c) {
  static const char* n[KC_COUNT] = {"bvh_build", "knn_covariance", "gicp_correspondences", "gicp_linearize", "gicp_error", "nn_fitness", "ndt_voxel_build",
                                    "ndt_derivatives", "ndt_hessian", "voxelgrid_downsample", "misc", "vgicp_voxel_map", "vgicp_round",
                                    "gicp_pcl_correspondences", "gicp_pcl_cost", "icp_pcl_round"};
  return (c >= 0 && c < KC_COUNT) ? n[c] : "?";
}
struct Telemetry {
  unsigned long long h2d = 0, d2h = 0;
  unsigned long long launches[KC_COUNT] = {0}, calls[KC_COUNT] = {0};
  double ms[KC_COUNT] = {0};
  bool on = false;
  struct Span { cudaEvent_t a, b; int cls; };
  std::vector<Span> spans;
  std::vector<cudaEvent_t> pool;
  Telemetry() = default;
  Telemetry(const Telemetry&) = delete;
  Telemetry& operator=(const Telemetry&) = delete;
  ~Telemetry() {
    resolve();
    for (auto e : pool) cudaEventDestroy(e);
  }
  cudaEvent_t get() {
    if (!pool.empty()) { cudaEvent_t e = pool.back(); pool.pop_back(); return e; }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
  }
  cudaEvent_t begin(cudaStream_t st) {
    if (!on) return nullptr;
    cudaEvent_t a = get();
    cudaEventRecord(a, st);
    return a;
  }
  void end(cudaEvent_t a, int cls, int nlaunch, cudaStream_t st) {
    launches[cls] += nlaunch;
    calls[cls] += 1;
    if (!on || !a) return;
    cudaEvent_t b = get();
    cudaEventRecord(b, st);
    spans.push_back({a, b, cls});
  }
  void resolve() {  // caller has synchronised the stream
    for (auto& sp : spans) {
      float t = 0.f;
      if (cudaEventElapsedTime(&t, sp.a, sp.b) == cudaSuccess) ms[sp.cls] += (double)t;
      pool.push_back(sp.a);
      pool.push_back(sp.b);
    }
    spans.clear();
  }
  void reset() {
    h2d = d2h = 0;
    for (int i = 0; i < KC_COUNT; i++) { launches[i] = calls[i] = 0; ms[i] = 0; }
  }
};
#define TEL_BEGIN(tel, st) cudaEvent_t _tel_ev = (tel) ? (tel)->begin(st) : nullptr
#define TEL_END(tel, cls, n, st) do { if (tel) (tel)->end(_tel_ev, cls, n, st); } while (0)

// Wait for the result message of a reduction kernel (finish_partials) in host-mapped memory: `nv` result words at out[0..nv),
// one more word at out[nv] (the optional `extra`, included only if has_extra), the checksum seq ^ xor(mix(word_i, i)) at out[nv+1], and
// `flag` = seq.  The device publishes them without system-scope fences, so the words may land in any order: the message is
// accepted only when it is self-consistent.  Falls back to querying / synchronising the stream so that a failed launch or a
// device fault still surfaces as an error (after a synchronise every store has landed).
// the acceptance test of a result message: flag == seq and checksum word == seq ^ xor(msg_mix(word_i, i)) over the result words [and the extra word]
inline bool result_message_consistent(const volatile unsigned long long* flag, unsigned long long seq, const volatile unsigned long long* w, int nv,
                                      bool has_extra) {
  if (*flag != seq) return false;
  unsigned long long x = seq;
  for (int i = 0; i < nv; i++) x ^= msg_mix(w[i], i);
  if (has_extra) x ^= msg_mix(w[nv], nv);
  return x == w[nv + 1];
}

inline int wait_host_result(const unsigned long long* flag, unsigned long long seq, const double* out, int nv, bool has_extra, cudaStream_t st) {
  const volatile unsigned long long* f = flag;
  const volatile unsigned long long* w = reinterpret_cast<const volatile unsigned long long*>(out);
  auto consistent = [&]() { return result_message_consistent(f, seq, w, nv, has_extra); };
  static const unsigned long spin_limit = [] { const char* e = getenv("B2R_SPIN_LIMIT"); return e ? strtoul(e, nullptr, 10) : 200000ul; }();
  for (unsigned long spins = 1; spins < spin_limit; spins++) {  // ~100-200 us of spinning covers a single in-flight kernel
    if (consistent()) return B2R_OK;
    if ((spins & 0x3fff) == 0) {
      cudaError_t e = cudaStreamQuery(st);
      if (e == cudaSuccess) break;
      if (e != cudaErrorNotReady) return fail(B2R_ECUDA, std::string("stream error: ") + cudaGetErrorString(e));
    }
  }
  // long wait (other streams' work is ahead of ours on the device): stop burning a core and block
  cudaError_t e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(B2R_ECUDA, std::string("stream error: ") + cudaGetErrorString(e));
  if (consistent()) return B2R_OK;
  return fail(B2R_ECUDA, "reduction kernel finished without signalling its result");
}

struct NdtVoxelMap;  // ndt.cuh: complete wherever a Cloud is destroyed
struct VgicpMap;    // vgicp.cuh: likewise

// One point cloud resident on the device with everything derived from it.
struct Cloud {
  size_t n = 0;
  int stride_f = 4;
  const void* host_ptr = nullptr;  // identity of the host buffer last uploaded
  DevBuf<float> raw;               // uploaded records
  const float* raw_view = nullptr; // == raw.p, or a caller-owned device pointer (set_*_device)
  // implicit BVH (bvh.cuh)
  DevBuf<float4> sorted, leaf_lo, leaf_hi, sup_lo, sup_hi;
  DevBuf<int> pos_of;
  int nsup = 0;
  bool bvh_ready = false;
  // GICP
  DevBuf<double> cov;              // sorted order, 6 per point
  bool cov_ready = false;
  // NDT (target only)
  std::unique_ptr<NdtVoxelMap> ndt;
  bool ndt_ready = false;
  // VGICP (target only): Gaussian voxel map built from the BVH arrays and the covariances
  std::unique_ptr<VgicpMap> vgicp;
  bool vgicp_ready = false;
  void invalidate() { bvh_ready = cov_ready = ndt_ready = vgicp_ready = false; }
  Bvh bvh() const {
    Bvh b;
    b.sp = sorted.p; b.leaf_lo = leaf_lo.p; b.leaf_hi = leaf_hi.p; b.sup_lo = sup_lo.p; b.sup_hi = sup_hi.p;
    b.nsup = nsup; b.nleaf = nsup * kSuper; b.n = (int)n;
    return b;
  }
};

// per-stream build scratch (BVH builds, NDT voxel-map builds): keys / values / radix-sort space, min-max cell
struct BuildCtx {
  DevBuf<unsigned int> keys_a, keys_b;
  DevBuf<int> vals_a, vals_b;
  DevBuf<char> sort_tmp;
  DevBuf<int> mm;  // 8 ints
};
static_assert(!std::is_copy_constructible<Cloud>::value && !std::is_copy_constructible<BuildCtx>::value, "a Cloud / BuildCtx owns its buffers");

}  // namespace b2r
