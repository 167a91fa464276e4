// common.cuh — shared definitions of the scan-matching engine (libb200reg).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#define B2R_HD __host__ __device__ __forceinline__

namespace b2r {

// float <-> order-preserving int (for atomicMin/atomicMax on floats)
B2R_HD int f2ord(float f) {
  int i;
#ifdef __CUDA_ARCH__
  i = __float_as_int(f);
#else
  union { float f; int i; } u; u.f = f; i = u.i;
#endif
  return i >= 0 ? i : i ^ 0x7fffffff;
}
B2R_HD float ord2f(int i) {
  i = i >= 0 ? i : i ^ 0x7fffffff;
#ifdef __CUDA_ARCH__
  return __int_as_float(i);
#else
  union { float f; int i; } u; u.i = i; return u.f;
#endif
}

// Non-contracted float32 arithmetic: the reference is built without FMA (CMakeLists.txt:10-11) and the parity
// contract pins d2 = ((dx*dx + dy*dy) + dz*dz) and x' = ((m0*x + m1*y) + m2*z) + m3 exactly.
B2R_HD float fmul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  volatile float r = a * b; return r;
#endif
}
B2R_HD float fadd(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  volatile float r = a + b; return r;
#endif
}
B2R_HD float fsub(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  volatile float r = a - b; return r;
#endif
}
B2R_HD float dist2_f32(float qx, float qy, float qz, float px, float py, float pz) {
  float dx = fsub(qx, px), dy = fsub(qy, py), dz = fsub(qz, pz);
  return fadd(fadd(fmul(dx, dx), fmul(dy, dy)), fmul(dz, dz));
}
// x' = ((m0*x + m1*y) + m2*z) + m3   (Eigen 4x4 * 4-vector column accumulation / pcl::transformPoint, no FMA)
B2R_HD float xform_row(float m0, float m1, float m2, float m3, float x, float y, float z) {
  return fadd(fadd(fadd(fmul(m0, x), fmul(m1, y)), fmul(m2, z)), m3);
}

B2R_HD int idx_bits(float w) {
#ifdef __CUDA_ARCH__
  return __float_as_int(w);
#else
  union { float f; int i; } u; u.f = w; return u.i;
#endif
}
B2R_HD float bits_idx(int i) {
#ifdef __CUDA_ARCH__
  return __int_as_float(i);
#else
  union { float f; int i; } u; u.i = i; return u.f;
#endif
}

B2R_HD bool finite3(float x, float y, float z) {
  return (x - x == 0.f) && (y - y == 0.f) && (z - z == 0.f);
}

B2R_HD int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// Position-dependent checksum term of the fence-free result messages (engine.cuh, pair_engine.cuh): word i enters rotated by
// (7 i + 1) bits, so two stale words cannot cancel each other (an xor of plain words ignores position).
B2R_HD unsigned long long msg_mix(unsigned long long w, int i) {
  const int r = (7 * i + 1) & 63;
  return (w << r) | (w >> ((64 - r) & 63));
}

}  // namespace b2r
