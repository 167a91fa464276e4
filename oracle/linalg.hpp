// oracle/linalg.hpp — TEST INFRASTRUCTURE ONLY (CPU oracle).  Never linked into the product path.
//
// Tiny fixed-size linear algebra needed by the oracle because Eigen is absent in this image.
// Each routine restates the *mathematical* contract of the Eigen routine the upstream packages call
// (SelfAdjointEigenSolver<Matrix3d>, JacobiSVD<Matrix3d/6d>, LDLT<6x6>, Matrix3d/4d::inverse()).
// Eigen's exact rounding sequence cannot be reproduced without Eigen; parity tolerances (DESIGN.md)
// account for that.  "parity unpinned": the reference ships no golden vectors (SURVEY.md §0.2).
#pragma once
#include <cmath>
#include <cstring>
#include <algorithm>

namespace orc {

// ---------------------------------------------------------------- cyclic Jacobi eigen-solver (symmetric, n<=6)
// A: n*n row-major symmetric.  On return w[i] ascending, V column i = eigenvector i (row-major n*n).
// stop_converged: also stop once the off-diagonal mass is below 1e-34 of the diagonal's (off-diagonal entries ~1e-17 relative,
// i.e. below double precision: further sweeps only move rounding noise).  Used by the 6x6 solve, which otherwise spends all 64
// sweeps waiting for the off-diagonal to underflow to an exact zero; the 3x3 users keep the run-to-exact-zero rule.
template <int N>
inline void sym_eigen(const double* A_in, double* w, double* V, bool stop_converged = false) {
  double A[N * N];
  std::memcpy(A, A_in, sizeof(A));
  for (int i = 0; i < N; i++)
    for (int j = 0; j < N; j++) V[i * N + j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 64; sweep++) {
    double off = 0.0;
    for (int p = 0; p < N; p++)
      for (int q = p + 1; q < N; q++) off += A[p * N + q] * A[p * N + q];
    if (off == 0.0) break;
    if (stop_converged) {
      double dg = 0.0;
      for (int p = 0; p < N; p++) dg += A[p * N + p] * A[p * N + p];
      if (off <= 1e-34 * dg) break;
    }
    for (int p = 0; p < N; p++) {
      for (int q = p + 1; q < N; q++) {
        double apq = A[p * N + q];
        if (apq == 0.0) continue;
        double app = A[p * N + p], aqq = A[q * N + q];
        double theta = (aqq - app) / (2.0 * apq);
        double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < N; k++) {  // columns p,q of A
          double akp = A[k * N + p], akq = A[k * N + q];
          A[k * N + p] = c * akp - s * akq;
          A[k * N + q] = s * akp + c * akq;
        }
        for (int k = 0; k < N; k++) {  // rows p,q of A
          double apk = A[p * N + k], aqk = A[q * N + k];
          A[p * N + k] = c * apk - s * aqk;
          A[q * N + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < N; k++) {
          double vkp = V[k * N + p], vkq = V[k * N + q];
          V[k * N + p] = c * vkp - s * vkq;
          V[k * N + q] = s * vkp + c * vkq;
        }
      }
    }
  }
  for (int i = 0; i < N; i++) w[i] = A[i * N + i];
  // selection sort ascending, permuting columns of V
  for (int i = 0; i < N; i++) {
    int m = i;
    for (int j = i + 1; j < N; j++)
      if (w[j] < w[m]) m = j;
    if (m != i) {
      std::swap(w[i], w[m]);
      for (int k = 0; k < N; k++) std::swap(V[k * N + i], V[k * N + m]);
    }
  }
}

// The PLANE normal of an exactly diagonal 3x3 C (row-major), where tied eigenvalues leave the smallest eigenvector undefined:
// the column JacobiSVD<Matrix3d> puts last in U.  On a diagonal matrix JacobiSVD does no rotation, moves negative signs into U
// and then runs its step-4 sort: for each i, the FIRST maximum of the remaining |values| is swapped into place only when it is
// not already at i, and the sort stops once that maximum is 0.  UPSTREAM-RECALL.  V gets column 0 = the normal (the eigenvector
// that PLANE scales by epsilon) and columns 1, 2 = the other two axes, in the layout sym_eigen<3> returns.
inline void diagonal_normal(const double* C, double* V) {
  double s[3] = {std::fabs(C[0]), std::fabs(C[4]), std::fabs(C[8])};
  int col[3] = {0, 1, 2};
  for (int i = 0; i < 3; i++) {
    int pos = i;
    for (int j = i + 1; j < 3; j++)
      if (s[j] > s[pos]) pos = j;
    if (s[pos] == 0.0) break;
    if (pos != i) { std::swap(s[i], s[pos]); std::swap(col[i], col[pos]); }
  }
  for (int a = 0; a < 9; a++) V[a] = 0.0;
  V[col[2] * 3 + 0] = 1.0; V[col[0] * 3 + 1] = 1.0; V[col[1] * 3 + 2] = 1.0;
}

// 3x3 inverse by cofactors (what Eigen's fixed-size inverse() does). returns false if det == 0.
inline bool inv3(const double* m, double* o) {
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
  return det != 0.0;
}

inline void mul3(const double* a, const double* b, double* o) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) o[i * 3 + j] = a[i * 3 + 0] * b[0 * 3 + j] + a[i * 3 + 1] * b[1 * 3 + j] + a[i * 3 + 2] * b[2 * 3 + j];
}
inline void mul3_abt(const double* a, const double* b, double* o) {  // a * b^T
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) o[i * 3 + j] = a[i * 3 + 0] * b[j * 3 + 0] + a[i * 3 + 1] * b[j * 3 + 1] + a[i * 3 + 2] * b[j * 3 + 2];
}

// LDL^T solve of a symmetric 6x6 system (Eigen::LDLT contract; H + lambda*I is SPD on the GICP path).
inline bool ldlt6_solve(const double* A, const double* b, double* x) {
  double L[36] = {0}, D[6];
  for (int j = 0; j < 6; j++) {
    double d = A[j * 6 + j];
    for (int k = 0; k < j; k++) d -= L[j * 6 + k] * L[j * 6 + k] * D[k];
    D[j] = d;
    if (d == 0.0 || d != d) return false;
    L[j * 6 + j] = 1.0;
    for (int i = j + 1; i < 6; i++) {
      double s = A[i * 6 + j];
      for (int k = 0; k < j; k++) s -= L[i * 6 + k] * L[j * 6 + k] * D[k];
      L[i * 6 + j] = s / d;
    }
  }
  double y[6];
  for (int i = 0; i < 6; i++) {
    double s = b[i];
    for (int k = 0; k < i; k++) s -= L[i * 6 + k] * y[k];
    y[i] = s;
  }
  for (int i = 0; i < 6; i++) y[i] /= D[i];
  for (int i = 5; i >= 0; i--) {
    double s = y[i];
    for (int k = i + 1; k < 6; k++) s -= L[k * 6 + i] * x[k];
    x[i] = s;
  }
  return true;
}

// JacobiSVD<6x6>(H).solve(rhs) for SYMMETRIC H: pseudo-inverse through the eigen-decomposition
// (singular values = |eigenvalues|), with Eigen's default rank threshold diagSize*eps*max_sv.
inline void svd6_solve_sym(const double* H, const double* rhs, double* x) {
  double w[6], V[36];
  sym_eigen<6>(H, w, V, true);
  double smax = 0.0;
  for (int i = 0; i < 6; i++) smax = std::max(smax, std::fabs(w[i]));
  double thr = std::max(smax * 6.0 * 2.220446049250313e-16, 2.2250738585072014e-308);
  for (int i = 0; i < 6; i++) x[i] = 0.0;
  for (int k = 0; k < 6; k++) {
    if (!(std::fabs(w[k]) > thr)) continue;
    double dot = 0.0;
    for (int i = 0; i < 6; i++) dot += V[i * 6 + k] * rhs[i];
    dot /= w[k];
    for (int i = 0; i < 6; i++) x[i] += V[i * 6 + k] * dot;
  }
  bool nan_in = false;
  for (int i = 0; i < 36; i++) nan_in |= (H[i] != H[i]);
  for (int i = 0; i < 6; i++) nan_in |= (rhs[i] != rhs[i]);
  if (nan_in)
    for (int i = 0; i < 6; i++) x[i] = NAN;
}

}  // namespace orc
