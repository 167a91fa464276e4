// linalg.cuh — small fixed-size float64 linear algebra for the engine (device + host).  Written from scratch:
// Eigen is what the upstream CPU packages use, it does not exist here, and nothing of it is needed on a GPU.
#pragma once
#include "common.cuh"

namespace b2r {

// Symmetric 3x3 stored as 6 doubles: xx, xy, xz, yy, yz, zz
struct Sym3 {
  double xx, xy, xz, yy, yz, zz;
};

// Cyclic Jacobi eigen-decomposition of a symmetric 3x3 (A row-major full).  w ascending, V columns = eigenvectors.
B2R_HD void sym_eigen3(const double* Ain, double* w, double* V) {
  double A[9];
#pragma unroll
  for (int i = 0; i < 9; i++) A[i] = Ain[i];
  V[0] = 1; V[1] = 0; V[2] = 0; V[3] = 0; V[4] = 1; V[5] = 0; V[6] = 0; V[7] = 0; V[8] = 1;
  for (int sweep = 0; sweep < 32; sweep++) {
    double off = A[1] * A[1] + A[2] * A[2] + A[5] * A[5];
    if (off == 0.0) break;
#pragma unroll
    for (int pq = 0; pq < 3; pq++) {
      const int p = (pq == 2) ? 1 : 0;
      const int q = (pq == 0) ? 1 : 2;
      double apq = A[p * 3 + q];
      if (apq == 0.0) continue;
      double app = A[p * 3 + p], aqq = A[q * 3 + q];
      double theta = (aqq - app) / (2.0 * apq);
      double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
      double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
      for (int k = 0; k < 3; k++) {
        double akp = A[k * 3 + p], akq = A[k * 3 + q];
        A[k * 3 + p] = c * akp - s * akq;
        A[k * 3 + q] = s * akp + c * akq;
      }
#pragma unroll
      for (int k = 0; k < 3; k++) {
        double apk = A[p * 3 + k], aqk = A[q * 3 + k];
        A[p * 3 + k] = c * apk - s * aqk;
        A[q * 3 + k] = s * apk + c * aqk;
      }
#pragma unroll
      for (int k = 0; k < 3; k++) {
        double vkp = V[k * 3 + p], vkq = V[k * 3 + q];
        V[k * 3 + p] = c * vkp - s * vkq;
        V[k * 3 + q] = s * vkp + c * vkq;
      }
    }
  }
  w[0] = A[0]; w[1] = A[4]; w[2] = A[8];
  // sort ascending (3-element network), permuting columns
#define B2R_SWAPCOL(a, b)                                  \
  if (w[b] < w[a]) {                                       \
    double tw = w[a]; w[a] = w[b]; w[b] = tw;              \
    for (int k = 0; k < 3; k++) { double tv = V[k * 3 + a]; V[k * 3 + a] = V[k * 3 + b]; V[k * 3 + b] = tv; } \
  }
  B2R_SWAPCOL(0, 1)
  B2R_SWAPCOL(1, 2)
  B2R_SWAPCOL(0, 1)
#undef B2R_SWAPCOL
}

// Unit eigenvector of the SMALLEST eigenvalue of a symmetric 3x3 (A row-major), float64, non-iterative and robust
// (after Eberly, "A Robust Eigensolver for 3x3 Symmetric Matrices"): the trigonometric closed form is accurate only for the
// root that is well separated — the smallest when det(B) <= 0, the largest otherwise.  In the first case the wanted vector is
// the best-conditioned cross product of two rows of (A - lambda0 I).  In the second case the largest eigenvector is deflated
// and the remaining 2x2 problem in its orthogonal complement is solved by one exact Jacobi rotation.
// ~250 flops against ~6 sweeps of 3x3 Jacobi (the iterative solver was a large share of k_knn_cov's instructions).
B2R_HD void sym_cross_eigvec3(double a00, double a01, double a02, double a11, double a12, double a22, double lam, double* v) {
  const double m00 = a00 - lam, m11 = a11 - lam, m22 = a22 - lam;
  const double x0 = a01 * a12 - a02 * m11, y0 = a02 * a01 - m00 * a12, z0 = m00 * m11 - a01 * a01;  // r0 x r1
  const double x1 = a01 * m22 - a02 * a12, y1 = a02 * a02 - m00 * m22, z1 = m00 * a12 - a01 * a02;  // r0 x r2
  const double x2 = m11 * m22 - a12 * a12, y2 = a12 * a02 - a01 * m22, z2 = a01 * a12 - m11 * a02;  // r1 x r2
  const double n0 = x0 * x0 + y0 * y0 + z0 * z0, n1 = x1 * x1 + y1 * y1 + z1 * z1, n2 = x2 * x2 + y2 * y2 + z2 * z2;
  double x = x0, y = y0, z = z0, n = n0;
  if (n1 > n) { x = x1; y = y1; z = z1; n = n1; }
  if (n2 > n) { x = x2; y = y2; z = z2; n = n2; }
  if (!(n > 0.0)) { v[0] = 0.0; v[1] = 0.0; v[2] = 1.0; return; }
  const double inv = 1.0 / sqrt(n);
  v[0] = x * inv; v[1] = y * inv; v[2] = z * inv;
}

B2R_HD void sym_min_eigvec3(const double* A, double* v) {
  const double a00 = A[0], a01 = A[1], a02 = A[2], a11 = A[4], a12 = A[5], a22 = A[8];
  const double q = (a00 + a11 + a22) / 3.0;
  const double b00 = a00 - q, b11 = a11 - q, b22 = a22 - q;
  const double p2 = b00 * b00 + b11 * b11 + b22 * b22 + 2.0 * (a01 * a01 + a02 * a02 + a12 * a12);
  if (!(p2 > 0.0)) { v[0] = 0.0; v[1] = 0.0; v[2] = 1.0; return; }  // A == q*I: every direction is an eigenvector
  const double p = sqrt(p2 / 6.0);
  const double ip = 1.0 / p;
  const double c00 = b00 * ip, c11 = b11 * ip, c22 = b22 * ip, c01 = a01 * ip, c02 = a02 * ip, c12 = a12 * ip;
  double r = 0.5 * (c00 * (c11 * c22 - c12 * c12) - c01 * (c01 * c22 - c12 * c02) + c02 * (c01 * c12 - c11 * c02));
  r = r < -1.0 ? -1.0 : (r > 1.0 ? 1.0 : r);
  const double phi = acos(r) / 3.0;
  if (r <= 0.0) {  // the smallest eigenvalue is the separated one
    sym_cross_eigvec3(a00, a01, a02, a11, a12, a22, q + 2.0 * p * cos(phi + 2.0943951023931953), v);
    return;
  }
  // the largest eigenvalue is the separated one: deflate it
  double e[3];
  sym_cross_eigvec3(a00, a01, a02, a11, a12, a22, q + 2.0 * p * cos(phi), e);
  // orthonormal basis (U, V) of the plane orthogonal to e
  double ux, uy, uz;
  if (fabs(e[0]) <= fabs(e[1]) && fabs(e[0]) <= fabs(e[2])) { ux = 0.0; uy = -e[2]; uz = e[1]; }
  else if (fabs(e[1]) <= fabs(e[2])) { ux = e[2]; uy = 0.0; uz = -e[0]; }
  else { ux = -e[1]; uy = e[0]; uz = 0.0; }
  const double iu = 1.0 / sqrt(ux * ux + uy * uy + uz * uz);
  ux *= iu; uy *= iu; uz *= iu;
  const double vx = e[1] * uz - e[2] * uy, vy = e[2] * ux - e[0] * uz, vz = e[0] * uy - e[1] * ux;
  // 2x2 restriction  [[a, b], [b, d]] = [U V]^T A [U V]
  const double Aux = a00 * ux + a01 * uy + a02 * uz, Auy = a01 * ux + a11 * uy + a12 * uz, Auz = a02 * ux + a12 * uy + a22 * uz;
  const double Avx = a00 * vx + a01 * vy + a02 * vz, Avy = a01 * vx + a11 * vy + a12 * vz, Avz = a02 * vx + a12 * vy + a22 * vz;
  const double a = ux * Aux + uy * Auy + uz * Auz, b = ux * Avx + uy * Avy + uz * Avz, d = vx * Avx + vy * Avy + vz * Avz;
  double cu, cv;  // coefficients of the smaller eigenvector in (U, V)
  if (b == 0.0) {
    if (a <= d) { cu = 1.0; cv = 0.0; } else { cu = 0.0; cv = 1.0; }
  } else {
    const double theta = (d - a) / (2.0 * b);
    const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
    const double c = 1.0 / sqrt(t * t + 1.0), sn = t * c;
    // eigenpairs: (a - t b, (c, -sn)) and (d + t b, (sn, c))
    if (a - t * b <= d + t * b) { cu = c; cv = -sn; } else { cu = sn; cv = c; }
  }
  double x = cu * ux + cv * vx, y = cu * uy + cv * vy, z = cu * uz + cv * vz;
  const double inv = 1.0 / sqrt(x * x + y * y + z * z);
  v[0] = x * inv; v[1] = y * inv; v[2] = z * inv;
}

// general 3x3 inverse by cofactors; returns determinant
B2R_HD double inv3(const double* m, double* o) {
  double c00 = m[4] * m[8] - m[5] * m[7];
  double c01 = m[5] * m[6] - m[3] * m[8];
  double c02 = m[3] * m[7] - m[4] * m[6];
  double det = m[0] * c00 + m[1] * c01 + m[2] * c02;
  double id = 1.0 / det;
  o[0] = c00 * id;
  o[1] = (m[2] * m[7] - m[1] * m[8]) * id;
  o[2] = (m[1] * m[5] - m[2] * m[4]) * id;
  o[3] = c01 * id;
  o[4] = (m[0] * m[8] - m[2] * m[6]) * id;
  o[5] = (m[2] * m[3] - m[0] * m[5]) * id;
  o[6] = c02 * id;
  o[7] = (m[1] * m[6] - m[0] * m[7]) * id;
  o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
  return det;
}

B2R_HD void mul3(const double* a, const double* b, double* o) {
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) o[i * 3 + j] = a[i * 3 + 0] * b[0 * 3 + j] + a[i * 3 + 1] * b[1 * 3 + j] + a[i * 3 + 2] * b[2 * 3 + j];
}

// ---- 6x6 host/device helpers used by the LM / Newton drivers -----------------------------------------------------
// LDL^T solve (fast_gicp: Eigen::LDLT(H + lambda I).solve(-b); SURVEY A.4).  Returns false on a zero/NaN pivot.
B2R_HD bool ldlt6_solve(const double* A, const double* b, double* x) {
  // every loop has a compile-time trip count and is fully unrolled: on the device L, D, y live in registers (the LM step runs in
  // ONE thread at the tail of k_pair_accumulate — dynamically indexed local arrays tripled its latency)
  double L[36], D[6];  // only the strict lower triangle of L is ever read
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 6; j++) {
    double d = A[j * 6 + j];
#pragma unroll
    for (int k = 0; k < j; k++) d -= L[j * 6 + k] * L[j * 6 + k] * D[k];
    D[j] = d;
    if (d == 0.0 || d != d) ok = false;
#pragma unroll
    for (int i = j + 1; i < 6; i++) {
      double s = A[i * 6 + j];
#pragma unroll
      for (int k = 0; k < j; k++) s -= L[i * 6 + k] * L[j * 6 + k] * D[k];
      L[i * 6 + j] = s / d;
    }
  }
  if (!ok) return false;  // a zero / NaN pivot: the caller treats the step as not solvable (values computed past it are discarded)
  double y[6];
#pragma unroll
  for (int i = 0; i < 6; i++) {
    double s = b[i];
#pragma unroll
    for (int k = 0; k < i; k++) s -= L[i * 6 + k] * y[k];
    y[i] = s;
  }
#pragma unroll
  for (int i = 0; i < 6; i++) y[i] /= D[i];
#pragma unroll
  for (int i = 5; i >= 0; i--) {
    double s = y[i];
#pragma unroll
    for (int k = i + 1; k < 6; k++) s -= L[k * 6 + i] * x[k];
    x[i] = s;
  }
  return true;
}

// se3_exp of fast_gicp so3.hpp (SURVEY A.4): a = (omega, v) -> 4x4 row-major isometry
B2R_HD void se3_exp(const double* a, double* D) {
  const double ox = a[0], oy = a[1], oz = a[2];
  double theta_sq = ox * ox + oy * oy + oz * oz;
  double theta = sqrt(theta_sq);
  double imag, real;
  if (theta_sq < 1e-10) {
    double theta_quad = theta_sq * theta_sq;
    imag = 0.5 - 1.0 / 48.0 * theta_sq + 1.0 / 3840.0 * theta_quad;
    real = 1.0 - 1.0 / 8.0 * theta_sq + 1.0 / 384.0 * theta_quad;
  } else {
    double th = sqrt(theta_sq);
    double half = 0.5 * th;
    imag = sin(half) / th;
    real = cos(half);
  }
  double qw = real, qx = imag * ox, qy = imag * oy, qz = imag * oz;
  double tx = 2 * qx, ty = 2 * qy, tz = 2 * qz;
  double twx = tx * qw, twy = ty * qw, twz = tz * qw;
  double txx = tx * qx, txy = ty * qx, txz = tz * qx;
  double tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
  double R[9] = {1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1 - (txx + tyy)};
  double Om[9] = {0, -oz, oy, oz, 0, -ox, -oy, ox, 0};
  double Om2[9];
  mul3(Om, Om, Om2);
  double V[9];
  if (theta < 1e-10) {
#pragma unroll
    for (int i = 0; i < 9; i++) V[i] = R[i];
  } else {
    double c1 = (1.0 - cos(theta)) / theta_sq;
    double c2 = (theta - sin(theta)) / (theta_sq * theta);
#pragma unroll
    for (int i = 0; i < 9; i++) V[i] = ((i % 4 == 0) ? 1.0 : 0.0) + c1 * Om[i] + c2 * Om2[i];
  }
#pragma unroll
  for (int i = 0; i < 16; i++) D[i] = 0;
#pragma unroll
  for (int r = 0; r < 3; r++) {
#pragma unroll
    for (int c = 0; c < 3; c++) D[r * 4 + c] = R[r * 3 + c];
    D[r * 4 + 3] = V[r * 3 + 0] * a[3] + V[r * 3 + 1] * a[4] + V[r * 3 + 2] * a[5];
  }
  D[15] = 1.0;
}

// Isometry product O = A * B (affine 3x4 part; last row 0 0 0 1)
B2R_HD void mul_iso(const double* A, const double* B, double* O) {
  double T[16];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 4; c++) {
      double s = A[r * 4 + 0] * B[0 * 4 + c] + A[r * 4 + 1] * B[1 * 4 + c] + A[r * 4 + 2] * B[2 * 4 + c];
      if (c == 3) s += A[r * 4 + 3];
      T[r * 4 + c] = s;
    }
  T[12] = T[13] = T[14] = 0;
  T[15] = 1;
#pragma unroll
  for (int i = 0; i < 16; i++) O[i] = T[i];
}

B2R_HD bool gicp_is_converged(const double* D, double rot_eps, double trans_eps) {
  double mr = 0, mt = 0;
#pragma unroll
  for (int r = 0; r < 3; r++) {
#pragma unroll
    for (int c = 0; c < 3; c++) {
      double v = 1.0 / rot_eps * fabs(D[r * 4 + c] - (r == c ? 1.0 : 0.0));
      mr = v > mr ? v : mr;
    }
    double v = 1.0 / trans_eps * fabs(D[r * 4 + 3]);
    mt = v > mt ? v : mt;
  }
  return (mr > mt ? mr : mt) < 1;
}

}  // namespace b2r
