// linalg.cuh — small fixed-size float64 linear algebra for the engine (device + host).  Written from scratch:
// Eigen is what the upstream CPU packages use, it does not exist here, and nothing of it is needed on a GPU.
#pragma once
#include "common.cuh"
#include "atan2_rn.cuh"

namespace b2r {

// Symmetric 3x3 stored as 6 doubles: xx, xy, xz, yy, yz, zz
struct Sym3 {
  double xx, xy, xz, yy, yz, zz;
};

// Cyclic Jacobi eigen-decomposition of a symmetric 3x3 (A row-major full).  w ascending, V columns = eigenvectors.
// The NDT voxel finalisation decides validity on the sign of the smallest eigenvalue, which for an exactly planar or linear
// voxel is rounding noise around 0; so this solver reproduces the oracle's orc::sym_eigen<3> bit for bit: the same sweep cap
// (64), the same unfused operation order (dmul / dadd / dsub: no FMA contraction on the device) and the same selection sort
// (it places tied eigenvalues' columns differently from a sorting network).
B2R_HD void sym_eigen3(const double* Ain, double* w, double* V) {
  double A[9];
#pragma unroll
  for (int i = 0; i < 9; i++) A[i] = Ain[i];
  V[0] = 1; V[1] = 0; V[2] = 0; V[3] = 0; V[4] = 1; V[5] = 0; V[6] = 0; V[7] = 0; V[8] = 1;
  for (int sweep = 0; sweep < 64; sweep++) {
    const double off = dadd(dadd(dmul(A[1], A[1]), dmul(A[2], A[2])), dmul(A[5], A[5]));
    if (off == 0.0) break;
#pragma unroll
    for (int pq = 0; pq < 3; pq++) {
      const int p = (pq == 2) ? 1 : 0;
      const int q = (pq == 0) ? 1 : 2;
      double apq = A[p * 3 + q];
      if (apq == 0.0) continue;
      double app = A[p * 3 + p], aqq = A[q * 3 + q];
      double theta = dsub(aqq, app) / dmul(2.0, apq);
      double t = (theta >= 0 ? 1.0 : -1.0) / dadd(fabs(theta), sqrt(dadd(dmul(theta, theta), 1.0)));
      double c = 1.0 / sqrt(dadd(dmul(t, t), 1.0)), s = dmul(t, c);
#pragma unroll
      for (int k = 0; k < 3; k++) {
        double akp = A[k * 3 + p], akq = A[k * 3 + q];
        A[k * 3 + p] = dsub(dmul(c, akp), dmul(s, akq));
        A[k * 3 + q] = dadd(dmul(s, akp), dmul(c, akq));
      }
#pragma unroll
      for (int k = 0; k < 3; k++) {
        double apk = A[p * 3 + k], aqk = A[q * 3 + k];
        A[p * 3 + k] = dsub(dmul(c, apk), dmul(s, aqk));
        A[q * 3 + k] = dadd(dmul(s, apk), dmul(c, aqk));
      }
#pragma unroll
      for (int k = 0; k < 3; k++) {
        double vkp = V[k * 3 + p], vkq = V[k * 3 + q];
        V[k * 3 + p] = dsub(dmul(c, vkp), dmul(s, vkq));
        V[k * 3 + q] = dadd(dmul(s, vkp), dmul(c, vkq));
      }
    }
  }
  w[0] = A[0]; w[1] = A[4]; w[2] = A[8];
  // selection sort ascending (first minimum wins), permuting columns; written with constant indices so w / V stay in registers
#define B2R_SWAPCOL(a, b)                                  \
  {                                                        \
    double tw = w[a]; w[a] = w[b]; w[b] = tw;              \
    for (int k = 0; k < 3; k++) { double tv = V[k * 3 + a]; V[k * 3 + a] = V[k * 3 + b]; V[k * 3 + b] = tv; } \
  }
  if (w[1] < w[0]) {
    if (w[2] < w[1]) B2R_SWAPCOL(0, 2) else B2R_SWAPCOL(0, 1)
  } else if (w[2] < w[0]) {
    B2R_SWAPCOL(0, 2)
  }
  if (w[2] < w[1]) B2R_SWAPCOL(1, 2)
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

// An exactly diagonal A (an axis-aligned line or a single point) has tied eigenvalues, so "the smallest eigenvector" is not
// unique there; it returns the axis upstream's JacobiSVD leaves in U's last column.  JacobiSVD does no rotation on a diagonal
// matrix; its step-4 sort walks i = 0, 1, swapping column i with the FIRST maximum of the remaining |a_jj| only when that is not
// at i, and stops at a zero maximum.  After i = 0 (first maximum p) the remaining columns are (u, w) = (1, 2), (0, 2) or (1, 0);
// i = 1 swaps them only if |a_ww| > |a_uu|.  So the zero matrix and multiples of I give e_z, diag(0, 0, a) gives e_x.
B2R_HD void sym_min_eigvec3(const double* A, double* v) {
  const double a00 = A[0], a01 = A[1], a02 = A[2], a11 = A[4], a12 = A[5], a22 = A[8];
  if (a01 == 0.0 && a02 == 0.0 && a12 == 0.0) {
    const double s0 = fabs(a00), s1 = fabs(a11), s2 = fabs(a22);
    int u = 1, w = 2;
    double su = s1, sw = s2;
    if (!(s0 >= s1 && s0 >= s2)) {
      if (s1 >= s2) { u = 0; su = s0; } else { w = 0; sw = s0; }
    }
    const int axis = sw > su ? u : w;
    v[0] = axis == 0 ? 1.0 : 0.0; v[1] = axis == 1 ? 1.0 : 0.0; v[2] = axis == 2 ? 1.0 : 0.0;
    return;
  }
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

// inv3 / mul3 in the same formulas, unfused (the NDT voxel finalisation; inv3 / mul3 above stay as they are on the GICP path)
B2R_HD double inv3_rn(const double* m, double* o) {
  const double c00 = dsub(dmul(m[4], m[8]), dmul(m[5], m[7]));
  const double c01 = dsub(dmul(m[5], m[6]), dmul(m[3], m[8]));
  const double c02 = dsub(dmul(m[3], m[7]), dmul(m[4], m[6]));
  const double det = dadd(dadd(dmul(m[0], c00), dmul(m[1], c01)), dmul(m[2], c02));
  const double id = 1.0 / det;
  o[0] = dmul(c00, id);
  o[1] = dmul(dsub(dmul(m[2], m[7]), dmul(m[1], m[8])), id);
  o[2] = dmul(dsub(dmul(m[1], m[5]), dmul(m[2], m[4])), id);
  o[3] = dmul(c01, id);
  o[4] = dmul(dsub(dmul(m[0], m[8]), dmul(m[2], m[6])), id);
  o[5] = dmul(dsub(dmul(m[2], m[3]), dmul(m[0], m[5])), id);
  o[6] = dmul(c02, id);
  o[7] = dmul(dsub(dmul(m[1], m[6]), dmul(m[0], m[7])), id);
  o[8] = dmul(dsub(dmul(m[0], m[4]), dmul(m[1], m[3])), id);
  return det;
}

B2R_HD void mul3_rn(const double* a, const double* b, double* o) {
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++)
      o[i * 3 + j] = dadd(dadd(dmul(a[i * 3 + 0], b[0 * 3 + j]), dmul(a[i * 3 + 1], b[1 * 3 + j])), dmul(a[i * 3 + 2], b[2 * 3 + j]));
}

// ndt_omp VoxelGridCovariance::applyFilter, the finalisation of one voxel from its float64 moments (cnt points, sums S, second
// moments S2 row-major): mean, and for cnt >= 6 the covariance with PCL's (n-1)/n factor, its eigenvalues clamped to 1 % of the
// largest, and the inverse.  Returns the voxel's point count, or -1 when the voxel is invalidated (a negative or zero
// eigenvalue, or a non-finite inverse).  Every operation is unfused and in the oracle's order, so host and device agree bitwise.
B2R_HD int ndt_voxel_gaussian(int cnt, const double* S, const double* S2, double* mean, double* icov) {
  const double nn = (double)cnt;
  mean[0] = S[0] / nn; mean[1] = S[1] / nn; mean[2] = S[2] / nn;
#pragma unroll
  for (int k = 0; k < 9; k++) icov[k] = 0.0;
  if (cnt < 6) return cnt;
  double cov[9];
  const double f = dsub(nn, 1.0) / nn;
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int bb = 0; bb < 3; bb++) {
      // cov = (S2 - 2*(sum*mean^T))/n + mean*mean^T ; cov *= (n-1)/n
      const double t = dsub(S2[a * 3 + bb], dmul(2.0, dmul(S[a], mean[bb]))) / nn;
      cov[a * 3 + bb] = dmul(dadd(t, dmul(mean[a], mean[bb])), f);
    }
  double w[3], V[9];
  sym_eigen3(cov, w, V);
  if (w[0] < 0 || w[1] < 0 || w[2] <= 0) return -1;
  const double minv = dmul(0.01, w[2]);
  if (w[0] < minv) {
    w[0] = minv;
    if (w[1] < minv) w[1] = minv;
    double Vi[9], VD[9];
    inv3_rn(V, Vi);
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
      for (int bb = 0; bb < 3; bb++) VD[a * 3 + bb] = dmul(V[a * 3 + bb], w[bb]);
    mul3_rn(VD, Vi, cov);
  }
  inv3_rn(cov, icov);
  bool bad = false;
#pragma unroll
  for (int a = 0; a < 9; a++) bad |= !(fabs(icov[a]) < INFINITY);  // +-inf or NaN
  return bad ? -1 : cnt;
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

// ---- pcl::IterativeClosestPoint (B2R_METHOD_ICP_PCL): Eigen 3.3.7's JacobiSVD<Matrix3f>, pcl::umeyama and DefaultConvergenceCriteria
// in float32 / float64 exactly as upstream types them, every operation unfused (tests/icp_pcl_ref.cpp states each choice; the host
// build in tests/icp_pcl_harness.cu must agree with it bit for bit)
B2R_HD float fdiv_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  volatile float r = a / b; return r;
#endif
}
B2R_HD float fsqrt_rn(float a) {
#ifdef __CUDA_ARCH__
  return __fsqrt_rn(a);
#else
  return sqrtf(a);
#endif
}
// apply_rotation_in_the_plane over rows p, q (stride 1) or columns p, q (stride 3) of a row-major 3x3: x' = c x + s y, y' = -s x + c y
B2R_HD void icp_rotate(float* M, int p, int q, int along, int step, float c, float s) {
  if (c == 1.0f && s == 0.0f) return;
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const float xi = M[p * along + k * step], yi = M[q * along + k * step];
    M[p * along + k * step] = fadd(fmul(c, xi), fmul(s, yi));
    M[q * along + k * step] = fadd(fmul(-s, xi), fmul(c, yi));
  }
}
// JacobiSVD<Matrix3f>(A, ComputeFullU | ComputeFullV): A, U, V row-major; d descending (two-sided Jacobi sweeps of real_2x2_jacobi_svd,
// then |diagonal| with the sign moved into U, times the scale, then the selection sort of step 4)
B2R_HD void icp_jacobi_svd3(const float* A, float* U, float* d, float* V) {
  const float kMin = 1.17549435e-38f, kPrec = 2.0f * 1.1920929e-07f;
  float scale = 0.0f;
#pragma unroll
  for (int i = 0; i < 9; i++) scale = fabsf(A[i]) > scale ? fabsf(A[i]) : scale;
  if (scale == 0.0f) scale = 1.0f;
  float W[9];
#pragma unroll
  for (int i = 0; i < 9; i++) { W[i] = fdiv_rn(A[i], scale); U[i] = (i % 4 == 0) ? 1.0f : 0.0f; V[i] = U[i]; }
  float maxd = 0.0f;
#pragma unroll
  for (int i = 0; i < 3; i++) maxd = fabsf(W[i * 4]) > maxd ? fabsf(W[i * 4]) : maxd;
  bool finished = false;
  while (!finished) {
    finished = true;
    for (int p = 1; p < 3; p++)
      for (int q = 0; q < p; q++) {
        const float pm = fmul(kPrec, maxd);
        const float thr = kMin > pm ? kMin : pm;
        if (fabsf(W[p * 3 + q]) > thr || fabsf(W[q * 3 + p]) > thr) {
          finished = false;
          // real_2x2_jacobi_svd
          float m00 = W[p * 4], m01 = W[p * 3 + q], m10 = W[q * 3 + p], m11 = W[q * 4];
          const float t = fadd(m00, m11), dd = fsub(m10, m01);
          float c1 = 1.0f, s1 = 0.0f;
          if (!(fabsf(dd) < kMin)) {
            const float u = fdiv_rn(t, dd);
            const float tmp = fsqrt_rn(fadd(1.0f, fmul(u, u)));
            s1 = fdiv_rn(1.0f, tmp);
            c1 = fdiv_rn(u, tmp);
          }
          if (!(c1 == 1.0f && s1 == 0.0f)) {
            const float a0 = m00, a1 = m01, b0 = m10, b1 = m11;
            m00 = fadd(fmul(c1, a0), fmul(s1, b0)); m01 = fadd(fmul(c1, a1), fmul(s1, b1));
            m10 = fadd(fmul(-s1, a0), fmul(c1, b0)); m11 = fadd(fmul(-s1, a1), fmul(c1, b1));
          }
          (void)m10;
          // j_right.makeJacobi(m, 0, 1)
          float cr = 1.0f, sr = 0.0f;
          const float deno = fmul(2.0f, fabsf(m01));
          if (!(deno < kMin)) {
            const float tau = fdiv_rn(fsub(m00, m11), deno);
            const float w = fsqrt_rn(fadd(fmul(tau, tau), 1.0f));
            const float tt = tau > 0.0f ? fdiv_rn(1.0f, fadd(tau, w)) : fdiv_rn(1.0f, fsub(tau, w));
            const float sign_t = tt > 0.0f ? 1.0f : -1.0f;
            const float n = fdiv_rn(1.0f, fsqrt_rn(fadd(fmul(tt, tt), 1.0f)));
            sr = fmul(fmul(fmul(-sign_t, fdiv_rn(m01, fabsf(m01))), fabsf(tt)), n);
            cr = n;
          }
          // j_left = rot1 * j_right.transpose()
          const float cl = fsub(fmul(c1, cr), fmul(s1, -sr)), sl = fadd(fmul(c1, -sr), fmul(s1, cr));
          icp_rotate(W, p, q, 3, 1, cl, sl);   // W.applyOnTheLeft(p, q, j_left)
          icp_rotate(U, p, q, 1, 3, cl, sl);   // U.applyOnTheRight(p, q, j_left.transpose())
          icp_rotate(W, p, q, 1, 3, cr, -sr);  // W.applyOnTheRight(p, q, j_right)
          icp_rotate(V, p, q, 1, 3, cr, -sr);  // V.applyOnTheRight(p, q, j_right)
          const float ap = fabsf(W[p * 4]), aq = fabsf(W[q * 4]);
          const float mpq = ap < aq ? aq : ap;
          maxd = maxd < mpq ? mpq : maxd;
        }
      }
  }
#pragma unroll
  for (int i = 0; i < 3; i++) {
    const float a = W[i * 4];
    d[i] = fabsf(a);
    if (a < 0.0f)
      for (int k = 0; k < 3; k++) U[k * 3 + i] = -U[k * 3 + i];
  }
#pragma unroll
  for (int i = 0; i < 3; i++) d[i] = fmul(d[i], scale);
  for (int i = 0; i < 3; i++) {
    int pos = i;
    float mx = d[i];
    for (int j = i + 1; j < 3; j++)
      if (d[j] > mx) { mx = d[j]; pos = j; }
    if (mx == 0.0f) break;
    if (pos != i) {
      float t = d[i]; d[i] = d[pos]; d[pos] = t;
      for (int k = 0; k < 3; k++) {
        t = U[k * 3 + i]; U[k * 3 + i] = U[k * 3 + pos]; U[k * 3 + pos] = t;
        t = V[k * 3 + i]; V[k * 3 + i] = V[k * 3 + pos]; V[k * 3 + pos] = t;
      }
    }
  }
}
// Eigen's 3x3 determinant: (m00 (m11 m22 - m12 m21) - m01 (m10 m22 - m12 m20)) + m02 (m10 m21 - m11 m20), float32
B2R_HD float icp_det3f(const float* m) {
  const float h0 = fmul(m[0], fsub(fmul(m[4], m[8]), fmul(m[5], m[7])));
  const float h1 = fmul(m[1], fsub(fmul(m[3], m[8]), fmul(m[5], m[6])));
  const float h2 = fmul(m[2], fsub(fmul(m[3], m[7]), fmul(m[4], m[6])));
  return fadd(fsub(h0, h1), h2);
}
// a 3-term coefficient of a small fixed-size Eigen product: x0 + (x1 + x2) (redux_novec_unroller splits 3 as 1 + 2)
B2R_HD float icp_dot3f(float a0, float b0, float a1, float b1, float a2, float b2) { return fadd(fmul(a0, b0), fadd(fmul(a1, b1), fmul(a2, b2))); }
// pcl::umeyama(src, dst, false) from sigma = (1/n) dst_demean src_demean^T and the means (PCL's copy with the rank-deficient branch):
// Rt row-major 4x4 float
B2R_HD void icp_umeyama(const float* sigma, const float* src_mean, const float* dst_mean, float* Rt) {
  float U[9], d[3], V[9];
  icp_jacobi_svd3(sigma, U, d, V);
  float S[3] = {1.0f, 1.0f, icp_det3f(sigma) < 0.0f ? -1.0f : 1.0f};
  int rank = 0;
  for (int i = 0; i < 3; i++)
    if (!(fabsf(d[i]) <= fmul(fabsf(d[0]), 1e-5f))) rank++;  // !isMuchSmallerThan(d_i, d_0), float dummy_precision
  if (rank == 2) S[2] = fmul(icp_det3f(U), icp_det3f(V)) > 0.0f ? 1.0f : -1.0f;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      Rt[i * 4 + j] = icp_dot3f(fmul(U[i * 3], S[0]), V[j * 3], fmul(U[i * 3 + 1], S[1]), V[j * 3 + 1], fmul(U[i * 3 + 2], S[2]), V[j * 3 + 2]);
  for (int i = 0; i < 3; i++)
    Rt[i * 4 + 3] = fsub(dst_mean[i], icp_dot3f(Rt[i * 4], src_mean[0], Rt[i * 4 + 1], src_mean[1], Rt[i * 4 + 2], src_mean[2]));
  Rt[12] = Rt[13] = Rt[14] = 0.0f; Rt[15] = 1.0f;
}
// DefaultConvergenceCriteria::hasConverged after ++nr_iterations_ (failure_after_max_iter_ false, max_iterations_similar_transforms_ 0,
// mse_threshold_relative_ = euclidean_fitness_epsilon_ = -DBL_MAX, which never fires): T = transformation_ row-major 4x4, mse = this
// iteration's correspondence MSE, *prev_mse updated as upstream does.  rot_thr = 1 - transformation_epsilon, trans_thr = transformation_epsilon
B2R_HD bool icp_has_converged(const float* T, int iterations, int max_iterations, double rot_thr, double trans_thr, double mse, double* prev_mse) {
  if (iterations >= max_iterations) return true;
  const double cos_angle = 0.5 * (double)fsub(fadd(fadd(T[0], T[5]), T[10]), 1.0f);
  const double tsq = (double)fadd(fadd(fmul(T[3], T[3]), fmul(T[7], T[7])), fmul(T[11], T[11]));
  if (cos_angle >= rot_thr && tsq <= trans_thr) return true;
  if (fabs(mse - *prev_mse) < 1e-12) return true;
  *prev_mse = mse;
  return false;
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

// ---- pcl::eigen33 (PCL 1.10 common/impl/eigen.hpp), the smallest-eigenvalue form NormalEstimation::solvePlaneParameters calls, in
// float32 as upstream types it for a Matrix3f: scale by the largest |entry| (1 when it is <= FLT_MIN), computeRoots (closed form,
// roots sorted ascending; the quadratic computeRoots2 when |c0| < FLT_EPSILON or the smallest root is <= 0), subtract the smallest
// root from the diagonal, and return the row cross product with the largest squared norm over its square root.  Every float32
// operation is correctly rounded and unfused in the order upstream writes it.  atan2f / cosf / sinf are evaluated as
// (float)f((double)x) on host and device alike (glibc's float routines cannot be reproduced on the device); atan2 is atan2_rn.cuh's,
// because CUDA's and glibc's float64 atan2 round some float32 results differently (cos and sin agree on every |t| <= 1.1).  Squared norms associate
// x x + (y y + z z): Eigen 3.3 reduces a fixed-size 3-vector with redux_novec_unroller, which splits at Length / 2 = 1.  A, v row-major / xyz; a NaN entry gives a NaN vector.
B2R_HD void pcl_compute_roots2(float b, float c, float* r) {
  r[0] = 0.0f;
  float d = (float)dsub((double)fmul(b, b), dmul(4.0, (double)c));  // Scalar(b * b - 4.0 * c): b * b in float32, the rest in float64
  if (d < 0.0f) d = 0.0f;
  const float sd = fsqrt_rn(d);
  r[2] = fmul(0.5f, fadd(b, sd));
  r[1] = fmul(0.5f, fsub(b, sd));
}
B2R_HD void pcl_compute_roots(const float* m, float* r) {
  const float m00 = m[0], m01 = m[1], m02 = m[2], m11 = m[4], m12 = m[5], m22 = m[8];
  const float c0 = fsub(fsub(fsub(fadd(fmul(fmul(m00, m11), m22), fmul(fmul(fmul(2.0f, m01), m02), m12)), fmul(fmul(m00, m12), m12)),
                             fmul(fmul(m11, m02), m02)), fmul(fmul(m22, m01), m01));
  const float c1 = fsub(fadd(fsub(fadd(fsub(fmul(m00, m11), fmul(m01, m01)), fmul(m00, m22)), fmul(m02, m02)), fmul(m11, m22)), fmul(m12, m12));
  const float c2 = fadd(fadd(m00, m11), m22);
  if (fabsf(c0) < 1.1920929e-07f) {  // Eigen::NumTraits<float>::epsilon()
    pcl_compute_roots2(c2, c1, r);
    return;
  }
  const float s_inv3 = (float)(1.0 / 3.0);
  const float s_sqrt3 = fsqrt_rn(3.0f);
  const float c2_over_3 = fmul(c2, s_inv3);
  float a_over_3 = fmul(fsub(c1, fmul(c2, c2_over_3)), s_inv3);
  if (a_over_3 > 0.0f) a_over_3 = 0.0f;
  const float half_b = fmul(0.5f, fadd(c0, fmul(c2_over_3, fsub(fmul(fmul(2.0f, c2_over_3), c2_over_3), c1))));
  float q = fadd(fmul(half_b, half_b), fmul(fmul(a_over_3, a_over_3), a_over_3));
  if (q > 0.0f) q = 0.0f;
  const float rho = fsqrt_rn(-a_over_3);
  const float theta = fmul((float)atan2_rn((double)fsqrt_rn(-q), (double)half_b), s_inv3);
  const float cos_theta = (float)cos((double)theta), sin_theta = (float)sin((double)theta);
  r[0] = fadd(c2_over_3, fmul(fmul(2.0f, rho), cos_theta));
  r[1] = fsub(c2_over_3, fmul(rho, fadd(cos_theta, fmul(s_sqrt3, sin_theta))));
  r[2] = fsub(c2_over_3, fmul(rho, fsub(cos_theta, fmul(s_sqrt3, sin_theta))));
  float t;
  if (r[0] >= r[1]) { t = r[0]; r[0] = r[1]; r[1] = t; }
  if (r[1] >= r[2]) {
    t = r[1]; r[1] = r[2]; r[2] = t;
    if (r[0] >= r[1]) { t = r[0]; r[0] = r[1]; r[1] = t; }
  }
  if (r[0] <= 0.0f) pcl_compute_roots2(c2, c1, r);
}
B2R_HD void pcl_eigen33(const float* A, float* v) {
  float scale = fabsf(A[0]);
  for (int i = 1; i < 9; i++) scale = fabsf(A[i]) > scale ? fabsf(A[i]) : scale;
  if (scale <= 1.17549435e-38f) scale = 1.0f;  // std::numeric_limits<float>::min()
  float S[9];
  for (int i = 0; i < 9; i++) S[i] = fdiv_rn(A[i], scale);
  float r[3];
  pcl_compute_roots(S, r);
  S[0] = fsub(S[0], r[0]); S[4] = fsub(S[4], r[0]); S[8] = fsub(S[8], r[0]);
  float V[3][3];  // row0 x row1, row0 x row2, row1 x row2
  const int ra[3] = {0, 0, 1}, rb[3] = {1, 2, 2};
  float len[3];
  for (int k = 0; k < 3; k++) {
    const float* a = S + ra[k] * 3;
    const float* b = S + rb[k] * 3;
    V[k][0] = fsub(fmul(a[1], b[2]), fmul(a[2], b[1]));
    V[k][1] = fsub(fmul(a[2], b[0]), fmul(a[0], b[2]));
    V[k][2] = fsub(fmul(a[0], b[1]), fmul(a[1], b[0]));
    len[k] = fadd(fmul(V[k][0], V[k][0]), fadd(fmul(V[k][1], V[k][1]), fmul(V[k][2], V[k][2])));
  }
  const int k = (len[0] >= len[1] && len[0] >= len[2]) ? 0 : (len[1] >= len[0] && len[1] >= len[2]) ? 1 : 2;
  const float sl = fsqrt_rn(len[k]);
  v[0] = fdiv_rn(V[k][0], sl); v[1] = fdiv_rn(V[k][1], sl); v[2] = fdiv_rn(V[k][2], sl);
}

}  // namespace b2r
