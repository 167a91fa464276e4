// atan2_rn.cuh — one float64 atan2 for host and device.  The float32 contracts that evaluate atan2 (pcl::eigen33's computeRoots,
// linalg.cuh) compare the device with a host reference bit for bit, and CUDA's atan2 and glibc's are different routines that round
// some float32 results differently.  This one is written only in correctly rounded float64 operations (no contraction on any
// target), so every build computes the same bits; its error is below 1 ulp of float64 (the argument reduction and polynomial of
// the classic fdlibm atan).  Self-contained, so plain C++ references (tests/floor_ref.cpp) include it too.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define B2R_FP_HD __host__ __device__ __forceinline__
#else
#define B2R_FP_HD inline
#endif

namespace b2r {
namespace fp {
B2R_FP_HD double mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  volatile double r = a * b; return r;
#endif
}
B2R_FP_HD double add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  volatile double r = a + b; return r;
#endif
}
B2R_FP_HD double sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  volatile double r = a - b; return r;
#endif
}
B2R_FP_HD double div(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  volatile double r = a / b; return r;
#endif
}

// atan(t) for t >= 0: reduced against atan(0.5), atan(1), atan(1.5) or pi/2 (each as a hi + lo pair), then an odd polynomial
B2R_FP_HD double atan_pos(double t) {
  const double hi[4] = {4.63647609000806093515e-01, 7.85398163397448278999e-01, 9.82793723247329054082e-01, 1.57079632679489655800e+00};
  const double lo[4] = {2.26987774529616870924e-17, 3.06161699786838301793e-17, 1.39033110312309984516e-17, 6.12323399573676603587e-17};
  int id;
  double x = t;
  if (t < 0.4375) {
    id = -1;
  } else if (t < 0.6875) {
    id = 0; x = div(sub(mul(2.0, t), 1.0), add(2.0, t));
  } else if (t < 1.1875) {
    id = 1; x = div(sub(t, 1.0), add(t, 1.0));
  } else if (t < 2.4375) {
    id = 2; x = div(sub(t, 1.5), add(1.0, mul(1.5, t)));
  } else {
    id = 3; x = div(-1.0, t);
  }
  const double z = mul(x, x), w = mul(z, z);
  const double s1 = mul(z, add(3.33333333333329318027e-01, mul(w, add(1.42857142725034663711e-01, mul(w, add(9.09088713343650656196e-02,
                    mul(w, add(6.66107313738753120669e-02, mul(w, add(4.97687799461593236017e-02, mul(w, 1.62858201153657823623e-02)))))))))));
  const double s2 = mul(w, add(-1.99999999998764832476e-01, mul(w, add(-1.11111104054623557880e-01, mul(w, add(-7.69187620504482999495e-02,
                    mul(w, add(-5.83357013379057348645e-02, mul(w, -3.65315727442169155270e-02)))))))));
  if (id < 0) return sub(x, mul(x, add(s1, s2)));
  return sub(hi[id], sub(sub(mul(x, add(s1, s2)), lo[id]), x));
}
}  // namespace fp

// atan2(y, x) with C99's special cases (signed zeros, infinities; NaN in -> NaN out)
B2R_FP_HD double atan2_rn(double y, double x) {
  const double pi = 3.1415926535897931160e+00, pi_lo = 1.2246467991473531772e-16, pi_2 = 1.5707963267948965580e+00;
  if (x != x || y != y) return fp::add(x, y);
  const bool yneg = signbit(y), xneg = signbit(x);
  const double ay = fabs(y), ax = fabs(x);
  double z;
  if (ay == 0.0) {
    z = xneg ? pi : 0.0;
  } else if (ax == 0.0) {
    z = pi_2;
  } else if (ax == INFINITY) {
    z = (ay == INFINITY) ? (xneg ? 2.35619449019234492885e+00 : 7.85398163397448309616e-01) : (xneg ? pi : 0.0);
  } else if (ay == INFINITY) {
    z = pi_2;
  } else {
    z = fp::atan_pos(fp::div(ay, ax));
    if (xneg) z = fp::sub(pi, fp::sub(z, pi_lo));
  }
  return yneg ? -z : z;
}

}  // namespace b2r
