// tests/device_numerics_harness.cu — the engine's shared __host__ __device__ numerics run on the device and on the host from one
// source, so tests/test_device_numerics*.py can hold the two builds against each other and against exact references.
//
// Built twice (tests/device_numerics_build.py):
//   device build (DN_DEVICE): the library's own NVCC_FLAGS, so every contraction decision is the product's; dn_run launches one
//     thread per input, a bounded chunk of inputs at a time, and dn_libm_sweep holds the device's exp / cos / sin against the host's
//     glibc and the device build of atan2_rn against its host build (host side in OpenMP), one chunk in memory at a time.
//   host build: nvcc host code with -ffp-contract=off, as the other harnesses are; dn_run loops over the inputs (OpenMP).
// Both builds export dn_info / dn_run / dn_lm_replay with the same records.  A record is a fixed number of 32-bit words per function;
// float64 fields take two words and start on an even word.  __device__-only functions (vcuda_eigen3, raw_moment_cov_f32) run their
// host restatement of tests/vgicp_cuda_ref.cpp in the host build.  Test infrastructure, never shipped.
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>
#include <omp.h>
#include "../hdl_graph_slam_b200/csrc/floor.cuh"
#include "../hdl_graph_slam_b200/csrc/pair_engine.cuh"
namespace b2r { thread_local std::string g_last_error; }
#ifndef DN_DEVICE
#include "vgicp_cuda_ref.cpp"
#endif
#ifdef DN_ORACLE
#include "../oracle/oracle.h"
#endif

namespace dn {

typedef uint32_t W;
B2R_HD float F(const W* p, int i) { return b2r::bits_idx((int)p[i]); }
B2R_HD void setF(W* p, int i, float v) { p[i] = (W)b2r::idx_bits(v); }
B2R_HD const double* D(const W* p) { return reinterpret_cast<const double*>(p); }
B2R_HD double* D(W* p) { return reinterpret_cast<double*>(p); }

// the transcendental calls inside bit-exact contracts, as the engine writes them
B2R_HD float lm_exp(float x) { return (float)exp((double)x); }                        // ndt.cuh (NDT_OMP term)
B2R_HD float lm_cos(float t) { return (float)cos((double)t); }                        // linalg.cuh pcl_compute_roots
B2R_HD float lm_sin(float t) { return (float)sin((double)t); }
B2R_HD float lm_atan2(float a, float b) { return (float)b2r::atan2_rn((double)a, (double)b); }  // atan2_rn.cuh, shared

struct RansacPts {
  const W* p;
  B2R_HD float3 operator()(int i) const { return make_float3(F(p, 3 * i), F(p, 3 * i + 1), F(p, 3 * i + 2)); }
};

template <int FN> struct Fn;
#define DN_FN(id, inw, outw)                                            \
  template <> struct Fn<id> {                                           \
    static constexpr int in = inw, out = outw;                          \
    static B2R_HD void run(const W* I, W* O);                           \
  };                                                                    \
  B2R_HD void Fn<id>::run(const W* I, W* O)

// ---- class A: host and device must agree bit for bit
DN_FN(0, 2, 1) { setF(O, 0, b2r::fmul(F(I, 0), F(I, 1))); }
DN_FN(1, 2, 1) { setF(O, 0, b2r::fadd(F(I, 0), F(I, 1))); }
DN_FN(2, 2, 1) { setF(O, 0, b2r::fsub(F(I, 0), F(I, 1))); }
DN_FN(3, 2, 1) { setF(O, 0, b2r::fdiv_rn(F(I, 0), F(I, 1))); }
DN_FN(4, 2, 1) { setF(O, 0, b2r::fsqrt_rn(F(I, 0))); }
DN_FN(5, 6, 1) { setF(O, 0, b2r::dist2_f32(F(I, 0), F(I, 1), F(I, 2), F(I, 3), F(I, 4), F(I, 5))); }
DN_FN(6, 7, 1) { setF(O, 0, b2r::xform_row(F(I, 0), F(I, 1), F(I, 2), F(I, 3), F(I, 4), F(I, 5), F(I, 6))); }
DN_FN(7, 2, 3) {
  const unsigned long long k = b2r::nn_key(F(I, 0), (int)I[1]);
  O[0] = (W)k; O[1] = (W)(k >> 32); setF(O, 2, b2r::nn_key_d2(k));
}
DN_FN(8, 3, 1) { O[0] = b2r::hilbert30(I[0], I[1], I[2]); }
DN_FN(9, 18, 24) { b2r::sym_eigen3(D(I), D(O), D(O) + 3); }
DN_FN(10, 18, 20) { D(O)[9] = b2r::inv3_rn(D(I), D(O)); }
DN_FN(11, 36, 18) { b2r::mul3_rn(D(I), D(I) + 9, D(O)); }
// (cnt, S[3], S2[9]) -> (returned count, mean[3], icov[9])
DN_FN(12, 26, 26) { D(O)[0] = (double)b2r::ndt_voxel_gaussian((int)D(I)[0], D(I) + 1, D(I) + 4, D(O) + 1, D(O) + 4); }
DN_FN(13, 9, 21) {
  float A[9], U[9], d[3], V[9];
  for (int i = 0; i < 9; i++) A[i] = F(I, i);
  b2r::icp_jacobi_svd3(A, U, d, V);
  for (int i = 0; i < 9; i++) { setF(O, i, U[i]); setF(O, 12 + i, V[i]); }
  for (int i = 0; i < 3; i++) setF(O, 9 + i, d[i]);
}
DN_FN(14, 9, 1) {
  float A[9];
  for (int i = 0; i < 9; i++) A[i] = F(I, i);
  setF(O, 0, b2r::icp_det3f(A));
}
DN_FN(15, 15, 16) {
  float A[15], Rt[16];
  for (int i = 0; i < 15; i++) A[i] = F(I, i);
  b2r::icp_umeyama(A, A + 9, A + 12, Rt);
  for (int i = 0; i < 16; i++) setF(O, i, Rt[i]);
}
// (T[16] as float64, iterations, max_iterations, rot_thr, trans_thr, mse, prev_mse) -> (converged, prev_mse after the call)
DN_FN(16, 44, 4) {
  const double* x = D(I);
  float T[16];
  for (int i = 0; i < 16; i++) T[i] = (float)x[i];
  double prev = x[21];
  D(O)[0] = b2r::icp_has_converged(T, (int)x[16], (int)x[17], x[18], x[19], x[20], &prev) ? 1.0 : 0.0;
  D(O)[1] = prev;
}
DN_FN(17, 2, 3) {
  float r[3];
  b2r::pcl_compute_roots2(F(I, 0), F(I, 1), r);
  for (int i = 0; i < 3; i++) setF(O, i, r[i]);
}
DN_FN(18, 9, 3) {
  float A[9], r[3];
  for (int i = 0; i < 9; i++) A[i] = F(I, i);
  b2r::pcl_compute_roots(A, r);
  for (int i = 0; i < 3; i++) setF(O, i, r[i]);
}
DN_FN(19, 9, 3) {
  float A[9], v[3];
  for (int i = 0; i < 9; i++) A[i] = F(I, i);
  b2r::pcl_eigen33(A, v);
  for (int i = 0; i < 3; i++) setF(O, i, v[i]);
}
// (seed, skip) -> the 8 words after `skip` draws of the generator
DN_FN(20, 2, 8) {
  b2r::Mt19937 g;
  g.seed(I[0]);
  for (W i = 0; i < I[1]; i++) g.next();
  for (int i = 0; i < 8; i++) O[i] = g.next();
}
// (seed, n <= 16, 16 points xyz) -> the first 4 hypotheses of a model over the n points (idx[3], c[4], ok per hypothesis)
DN_FN(21, 50, 32) {
  b2r::Mt19937 g;
  g.seed(I[0]);
  const int n = (int)I[1];
  int shuffled[16];
  for (int i = 0; i < 16; i++) shuffled[i] = i;
  const RansacPts pt{I + 2};
  for (int t = 0; t < 4; t++) {
    b2r::FloorHyp h;
    b2r::ransac_draw(g, shuffled, n, pt, h);
    W* o = O + 8 * t;
    for (int i = 0; i < 3; i++) o[i] = h.ok ? (W)h.idx[i] : 0u;
    for (int i = 0; i < 4; i++) setF(o, 3 + i, h.ok ? h.c[i] : 0.0f);
    o[7] = (W)h.ok;
  }
}
DN_FN(22, 7, 1) {
  float c[4] = {F(I, 0), F(I, 1), F(I, 2), F(I, 3)};
  O[0] = b2r::ransac_inlier(c, F(I, 4), F(I, 5), F(I, 6)) ? 1u : 0u;
}
DN_FN(23, 32, 16) {
  float A[32], o[16];
  for (int i = 0; i < 32; i++) A[i] = F(I, i);
  b2r::gicp_pcl_mul4f(A, A + 16, o);
  for (int i = 0; i < 16; i++) setF(O, i, o[i]);
}
DN_FN(24, 9, 12) {
  float A[9], w[3], V[9];
  for (int i = 0; i < 9; i++) A[i] = F(I, i);
#if defined(__CUDA_ARCH__)
  b2r::vcuda_eigen3(A, w, V);
#elif !defined(DN_DEVICE)
  eigen3f(A, w, V);
#else
  for (int i = 0; i < 9; i++) V[i] = w[i % 3] = NAN;  // the device build runs records on the device only
#endif
  for (int i = 0; i < 3; i++) setF(O, i, w[i]);
  for (int i = 0; i < 9; i++) setF(O, 3 + i, V[i]);
}
// (kk <= 20, 20 points xyz) -> the float32 raw-moment covariance of the first kk points in list order
DN_FN(25, 61, 9) {
  const int kk = (int)I[0];
  float C[9];
#ifdef __CUDA_ARCH__
  const RansacPts pt{I + 1};
  b2r::raw_moment_cov_f32(kk, pt, C);
#else
  // vgicp_cuda_ref.cpp covariances_f, statement for statement
  float m[3] = {0.f, 0.f, 0.f}, s[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int j = 0; j < kk; j++) {
    const float p[3] = {F(I, 1 + 3 * j), F(I, 2 + 3 * j), F(I, 3 + 3 * j)};
    for (int a = 0; a < 3; a++) m[a] = m[a] + p[a];
    for (int a = 0; a < 3; a++)
      for (int b = a; b < 3; b++) s[a * 3 + b] = s[a * 3 + b] + p[a] * p[b];
  }
  const float kf = (float)kk;
  for (int a = 0; a < 3; a++) m[a] = m[a] / kf;
  for (int a = 0; a < 3; a++)
    for (int b = a; b < 3; b++) C[a * 3 + b] = C[b * 3 + a] = s[a * 3 + b] / kf - m[a] * m[b];
#endif
  for (int i = 0; i < 9; i++) setF(O, i, C[i]);
}

// ---- class B: plain operators (the device may fuse them); tests bound their error instead
// (A[36], b[6]) -> (ok, x[6])
DN_FN(40, 84, 14) {
  double x[6] = {0, 0, 0, 0, 0, 0};
  const bool ok = b2r::ldlt6_solve(D(I), D(I) + 36, x);
  D(O)[0] = ok ? 1.0 : 0.0;
  for (int i = 0; i < 6; i++) D(O)[1 + i] = x[i];
}
DN_FN(41, 12, 32) { b2r::se3_exp(D(I), D(O)); }
DN_FN(42, 64, 32) { b2r::mul_iso(D(I), D(I) + 16, D(O)); }
DN_FN(43, 18, 20) { D(O)[9] = b2r::inv3(D(I), D(O)); }
DN_FN(44, 36, 18) { b2r::mul3(D(I), D(I) + 9, D(O)); }
DN_FN(45, 18, 6) { b2r::sym_min_eigvec3(D(I), D(O)); }
// (a00 a01 a02 a11 a12 a22 lam) -> v
DN_FN(46, 14, 6) { const double* a = D(I); b2r::sym_cross_eigvec3(a[0], a[1], a[2], a[3], a[4], a[5], a[6], D(O)); }
// (D[16], rot_eps, trans_eps) -> converged
DN_FN(47, 36, 2) { D(O)[0] = b2r::gicp_is_converged(D(I), D(I)[16], D(I)[17]) ? 1.0 : 0.0; }

// ---- the transcendental calls of bit-exact contracts: exp, cos, sin from the device's libm against the host's glibc; atan2 the
// shared atan2_rn on both
DN_FN(60, 2, 1) { setF(O, 0, lm_exp(F(I, 0))); }
DN_FN(61, 2, 1) { setF(O, 0, lm_cos(F(I, 0))); }
DN_FN(62, 2, 1) { setF(O, 0, lm_sin(F(I, 0))); }
DN_FN(63, 2, 1) { setF(O, 0, lm_atan2(F(I, 0), F(I, 1))); }
// the shared float64 atan2 itself: (y, x) -> atan2_rn(y, x)
DN_FN(64, 4, 2) { D(O)[0] = b2r::atan2_rn(D(I)[0], D(I)[1]); }

#define DN_ALL(X)                                                                                                      \
  X(0) X(1) X(2) X(3) X(4) X(5) X(6) X(7) X(8) X(9) X(10) X(11) X(12) X(13) X(14) X(15) X(16) X(17) X(18) X(19) X(20) \
  X(21) X(22) X(23) X(24) X(25) X(40) X(41) X(42) X(43) X(44) X(45) X(46) X(47) X(60) X(61) X(62) X(63) X(64)

#ifdef DN_DEVICE
template <int FN>
__global__ void k_dn(const W* __restrict__ in, W* __restrict__ out, long long n) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) Fn<FN>::run(in + i * Fn<FN>::in, out + i * Fn<FN>::out);
}

constexpr long long kChunk = 1 << 20;  // inputs per launch: device buffers stay under 2 * 84 * 4 MiB

template <int FN>
int run_dev(const W* in, long long n, W* out) {
  W *din = nullptr, *dout = nullptr;
  const long long c = n < kChunk ? n : kChunk;
  int rc = 0;
  if (cudaMalloc(&din, c * Fn<FN>::in * 4) != cudaSuccess || cudaMalloc(&dout, c * Fn<FN>::out * 4) != cudaSuccess) rc = -2;
  for (long long s = 0; rc == 0 && s < n; s += c) {
    const long long m = (n - s) < c ? (n - s) : c;
    if (cudaMemcpy(din, in + s * Fn<FN>::in, m * Fn<FN>::in * 4, cudaMemcpyHostToDevice) != cudaSuccess) { rc = -3; break; }
    k_dn<FN><<<(unsigned)((m + 127) / 128), 128>>>(din, dout, m);
    if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) { rc = -4; break; }
    if (cudaMemcpy(out + s * Fn<FN>::out, dout, m * Fn<FN>::out * 4, cudaMemcpyDeviceToHost) != cudaSuccess) { rc = -5; break; }
  }
  cudaFree(din);
  cudaFree(dout);
  return rc;
}
#else
template <int FN>
int run_dev(const W* in, long long n, W* out) {
#pragma omp parallel for schedule(static)
  for (long long i = 0; i < n; i++) Fn<FN>::run(in + i * Fn<FN>::in, out + i * Fn<FN>::out);
  return 0;
}
#endif

// ---- LM replay: the 29 sums of a recorded round sequence fed to lm_advance; the state after every round
constexpr int kLmOut = 22;  // mode, li, it, delta_conv, converged, lm_failed, cur, wc, lambda, nu, x0[12]
B2R_HD void lm_replay(const double* R, int rounds, const double* x0, const double* cfgd, int max_it, double* out) {
  b2r::LmCfg cfg;
  cfg.max_iterations = max_it; cfg.rot_eps = cfgd[0]; cfg.trans_eps = cfgd[1];
  cfg.thr2 = 0; cfg.lim = 0; cfg.want_fitness = 0; cfg.fit_max_range = 0; cfg.fit_lim = 0; cfg.index_seed = 0;
  b2r::PairDev P;
  memset(&P, 0, sizeof(P));
  b2r::PairReport rep;
  P.report = &rep;
  for (int i = 0; i < 12; i++) { P.xe[i] = x0[i]; P.x0[i] = x0[i]; }
  P.mode = b2r::PM_FIRST; P.lambda = -1.0; P.nu = 2.0;
  for (int k = 0; k < rounds; k++) {
    double* o = out + (size_t)k * kLmOut;
    if (P.mode == b2r::PM_DONE) { o[0] = -1.0; continue; }
    b2r::lm_advance(P, R + (size_t)k * b2r::kAcc, cfg);
    o[0] = P.mode; o[1] = P.li; o[2] = P.it; o[3] = P.delta_conv; o[4] = P.converged; o[5] = P.lm_failed; o[6] = P.cur; o[7] = P.wc;
    o[8] = P.lambda; o[9] = P.nu;
    for (int i = 0; i < 12; i++) o[10 + i] = P.x0[i];
  }
}

#ifdef DN_DEVICE
__global__ void k_lm_replay(const double* R, int rounds, const double* x0, const double* cfgd, int max_it, double* out) {
  lm_replay(R, rounds, x0, cfgd, max_it, out);
}
#endif

}  // namespace dn

extern "C" {

int dn_info(int fn, int* in_words, int* out_words) {
  switch (fn) {
#define DN_INFO(id) case id: *in_words = dn::Fn<id>::in; *out_words = dn::Fn<id>::out; return 0;
    DN_ALL(DN_INFO)
#undef DN_INFO
  }
  return -1;
}

int dn_is_device() {
#ifdef DN_DEVICE
  return 1;
#else
  return 0;
#endif
}

// n records of function fn: in -> out (dn_info gives the record sizes in 32-bit words)
int dn_run(int fn, const uint32_t* in, long long n, uint32_t* out) {
  switch (fn) {
#define DN_RUN(id) case id: return dn::run_dev<id>(in, n, out);
    DN_ALL(DN_RUN)
#undef DN_RUN
  }
  return -1;
}

// replay `rounds` rounds of 29 sums (R row-major) from pose x0 (rows 0..2 of the 4x4) with cfgd = (rot_eps, trans_eps); out gets
// kLmOut doubles per round (mode -1 once the state machine has finished)
int dn_lm_replay(const double* R, int rounds, const double* x0, const double* cfgd, int max_it, double* out) {
#ifdef DN_DEVICE
  double *dR = nullptr, *dx = nullptr, *dc = nullptr, *dout = nullptr;
  int rc = 0;
  const size_t nr = (size_t)rounds * b2r::kAcc, no = (size_t)rounds * dn::kLmOut;
  if (cudaMalloc(&dR, nr * 8 + 8) || cudaMalloc(&dx, 12 * 8) || cudaMalloc(&dc, 2 * 8) || cudaMalloc(&dout, no * 8 + 8)) rc = -2;
  if (!rc && (cudaMemcpy(dR, R, nr * 8, cudaMemcpyHostToDevice) || cudaMemcpy(dx, x0, 12 * 8, cudaMemcpyHostToDevice) ||
              cudaMemcpy(dc, cfgd, 2 * 8, cudaMemcpyHostToDevice)))
    rc = -3;
  if (!rc) {
    dn::k_lm_replay<<<1, 1>>>(dR, rounds, dx, dc, max_it, dout);
    if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) rc = -4;
  }
  if (!rc && cudaMemcpy(out, dout, no * 8, cudaMemcpyDeviceToHost)) rc = -5;
  cudaFree(dR); cudaFree(dx); cudaFree(dc); cudaFree(dout);
  return rc;
#else
  dn::lm_replay(R, rounds, x0, cfgd, max_it, out);
  return 0;
#endif
}

#ifdef DN_DEVICE
// splitmix64 of the input's index: the atan2 sweep's pairs, drawn identically on host and device without a transfer
B2R_HD unsigned long long dn_mix(unsigned long long z) {
  z += 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}
// pair i of the atan2 sweep: a >= 0 and b of either sign, both finite, magnitudes 2^-64 .. 2^64 (each float exponent equally likely)
B2R_HD void dn_atan2_pair(unsigned long long seed, unsigned long long i, float* a, float* b) {
  const unsigned long long h = dn_mix(seed ^ dn_mix(i));
  const unsigned ea = 63u + (unsigned)((h >> 0) % 129u), eb = 63u + (unsigned)((h >> 8) % 129u);
  *a = b2r::bits_idx((int)((ea << 23) | (unsigned)((h >> 16) & 0x7fffffu)));
  *b = b2r::bits_idx((int)(((unsigned)(h >> 63) << 31) | (eb << 23) | (unsigned)((h >> 39) & 0x7fffffu)));
}
// input i of sweep fn: 60..62 the float with bits first + i (62, 61 also its negation in the odd slots), 63 a random pair
B2R_HD void dn_sweep_input(int fn, unsigned long long first, unsigned long long i, float* x, float* y) {
  *y = 0.0f;
  if (fn == 63) { dn_atan2_pair(first, i, x, y); return; }
  if (fn == 60) { *x = b2r::bits_idx((int)(unsigned)(first + i)); return; }
  const unsigned bits = (unsigned)(first + (i >> 1));
  *x = b2r::bits_idx((int)(bits | ((unsigned)(i & 1) << 31)));
}
B2R_HD float dn_sweep_eval(int fn, float x, float y) {
  return fn == 60 ? dn::lm_exp(x) : fn == 61 ? dn::lm_cos(x) : fn == 62 ? dn::lm_sin(x) : dn::lm_atan2(x, y);
}
__global__ void k_sweep(int fn, unsigned long long first, unsigned long long base, long long n, float* out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float x, y;
  dn_sweep_input(fn, first, base + i, &x, &y);
  out[i] = dn_sweep_eval(fn, x, y);
}

// Sweep fn (60 exp, 61 cos, 62 sin, 63 atan2) over `count` inputs (see dn_sweep_input; `first` is the first bit pattern, or the
// seed of the atan2 pairs): the device's result against the host's (glibc for exp / cos / sin, atan2_rn's host build for atan2).  Returns the number of results whose bits differ (two
// NaNs agree); the first `keep` mismatches go to bad (x, y, device, host as float bits).  Negative on a CUDA error.
long long dn_libm_sweep(int fn, unsigned long long first, long long count, int keep, uint32_t* bad) {
  const long long chunk = 1ll << 26;
  float* dout = nullptr;
  std::vector<float> hout((size_t)(count < chunk ? count : chunk));
  if (cudaMalloc(&dout, hout.size() * 4) != cudaSuccess) return -2;
  long long mism = 0;
  for (long long s = 0; s < count; s += chunk) {
    const long long m = (count - s) < chunk ? (count - s) : chunk;
    k_sweep<<<(unsigned)((m + 255) / 256), 256>>>(fn, first, (unsigned long long)s, m, dout);
    if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess ||
        cudaMemcpy(hout.data(), dout, m * 4, cudaMemcpyDeviceToHost) != cudaSuccess) {
      cudaFree(dout);
      return -4;
    }
    long long local = 0;
#pragma omp parallel for schedule(static) reduction(+ : local)
    for (long long i = 0; i < m; i++) {
      float x, y;
      dn_sweep_input(fn, first, (unsigned long long)(s + i), &x, &y);
      const float h = dn_sweep_eval(fn, x, y), d = hout[i];
      const bool same = (h != h && d != d) || b2r::idx_bits(h) == b2r::idx_bits(d);
      if (!same) {
        local++;
#pragma omp critical
        {
          for (int k = 0; k < keep; k++)  // free slots hold 0xffffffff; which mismatches fill them is not fixed
            if (bad[4 * k] == 0xffffffffu) {
              bad[4 * k] = (uint32_t)b2r::idx_bits(x); bad[4 * k + 1] = (uint32_t)b2r::idx_bits(y);
              bad[4 * k + 2] = (uint32_t)b2r::idx_bits(d); bad[4 * k + 3] = (uint32_t)b2r::idx_bits(h);
              break;
            }
        }
      }
    }
    mism += local;
  }
  cudaFree(dout);
  return mism;
}
#endif

#ifdef DN_ORACLE
// The oracle-emulated LM rounds of tests/lm_harness.cu (orc_gicp_linearize / orc_gicp_error as the two kernels of a round, the
// host build of lm_advance deciding), recording every round's 29 sums into R (at most max_rounds).  Returns the round count.
int dn_lm_record(const float* src, size_t n, const float* tgt, size_t m, size_t stride, int max_it, double trans_eps, double dist,
                 const float* guess, double* R, int max_rounds) {
  orc_gicp_config oc;
  oc.max_iterations = max_it; oc.transformation_epsilon = trans_eps; oc.rotation_epsilon = 2e-3; oc.max_corr_dist = dist;
  oc.k_correspondences = 20; oc.num_threads = 0;
  std::vector<double> scov(n * 9), tcov(m * 9);
  orc_gicp_covariances(src, n, stride, 20, scov.data(), 0);
  orc_gicp_covariances(tgt, m, stride, 20, tcov.data(), 0);
  b2r::LmCfg cfg;
  cfg.max_iterations = max_it; cfg.rot_eps = oc.rotation_epsilon; cfg.trans_eps = trans_eps;
  cfg.thr2 = dist * dist; cfg.lim = (float)cfg.thr2; cfg.want_fitness = 0; cfg.fit_max_range = 0; cfg.fit_lim = 0; cfg.index_seed = 0;
  b2r::PairDev P;
  std::memset(&P, 0, sizeof(P));
  b2r::PairReport rep;
  P.report = &rep;
  for (int i = 0; i < 12; i++) { P.xe[i] = (double)guess[i]; P.x0[i] = (double)guess[i]; }
  P.mode = b2r::PM_FIRST; P.lambda = -1.0; P.nu = 2.0;
  std::vector<int32_t> corr[2] = {std::vector<int32_t>(n), std::vector<int32_t>(n)};
  std::vector<double> mahal[2] = {std::vector<double>(n * 9), std::vector<double>(n * 9)};
  std::vector<float> d2(n);
  int rounds = 0;
  while (P.mode != b2r::PM_DONE && rounds < max_rounds) {
    double T[16];
    for (int i = 0; i < 12; i++) T[i] = P.xe[i];
    T[12] = T[13] = T[14] = 0; T[15] = 1;
    double* r = R + (size_t)rounds * b2r::kAcc;
    for (int i = 0; i < b2r::kAcc; i++) r[i] = 0;
    const int mode = P.mode, cur = P.cur, wset = (mode == b2r::PM_FIRST) ? cur : (cur ^ 1);
    if (mode == b2r::PM_FUSED || mode == b2r::PM_ERR) r[28] = orc_gicp_error(src, n, stride, tgt, stride, corr[cur].data(), mahal[cur].data(), T, 0);
    if (mode == b2r::PM_FIRST || mode == b2r::PM_FUSED) {
      double H[36], b[6];
      r[27] = orc_gicp_linearize(src, n, stride, scov.data(), tgt, m, stride, tcov.data(), T, dist, corr[wset].data(), d2.data(),
                                 mahal[wset].data(), H, b, 0);
      int k = 0;
      for (int rr = 0; rr < 6; rr++)
        for (int cc = rr; cc < 6; cc++) r[k++] = H[rr * 6 + cc];
      for (int i = 0; i < 6; i++) r[21 + i] = b[i];
    }
    b2r::lm_advance(P, r, cfg);
    rounds++;
  }
  return rounds;
}
#endif

}  // extern "C"
