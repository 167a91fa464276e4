// tests/diag_normal_harness.cu — CPU check (linalg.cuh compiled as host code) of the PLANE normal on exactly diagonal covariances,
// the axis-aligned lines where tied eigenvalues leave the smallest eigenvector undefined.  Test infrastructure, never shipped.
//   diag_normal_harness table     reads "a b c" lines from stdin; prints per line the normal of diag(a, b, c) from sym_min_eigvec3,
//                                 the solver before the diagonal rule (kept below), the oracle's rule (orc::diagonal_normal) and
//                                 the oracle's ascending Jacobi alone (orc::sym_eigen<3> column 0), 3 numbers each
//   diag_normal_harness random N  N random symmetric matrices that are NOT diagonal (generic, and with one or two of the three
//                                 off-diagonals exactly 0): prints "mismatch=M" where M counts outputs not bit-identical to the old solver
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include "../hdl_graph_slam_b200/csrc/linalg.cuh"
#include "../oracle/linalg.hpp"
using namespace b2r;

// sym_min_eigvec3 as it was before the exactly-diagonal branch (the reference for "every other input gives the same bits")
static void old_sym_min_eigvec3(const double* A, double* v) {
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

static double ur(unsigned long long& s) { s = s * 6364136223846793005ull + 1442695040888963407ull; return (double)(s >> 11) / 9007199254740992.0; }

static void print3(const double* v) { printf(" %.17g %.17g %.17g", v[0], v[1], v[2]); }

int main(int argc, char** argv) {
  if (argc >= 2 && !strcmp(argv[1], "table")) {
    double a, b, c;
    while (scanf("%lf %lf %lf", &a, &b, &c) == 3) {
      const double A[9] = {a, 0.0, 0.0, 0.0, b, 0.0, 0.0, 0.0, c};
      double n[3], o[3], w[3], V[9], D[9];
      sym_min_eigvec3(A, n);
      old_sym_min_eigvec3(A, o);
      orc::diagonal_normal(A, D);
      orc::sym_eigen<3>(A, w, V);
      const double d[3] = {D[0], D[3], D[6]}, j[3] = {V[0], V[3], V[6]};
      print3(n); print3(o); print3(d); print3(j);
      printf("\n");
    }
    return 0;
  }
  if (argc >= 3 && !strcmp(argv[1], "random")) {
    const long N = atol(argv[2]);
    unsigned long long s = 11;
    long mismatch = 0, zeros = 0;
    for (long t = 0; t < N; t++) {
      // spectra from isotropic to linear, rotated; then (for 3 of 5) one or two off-diagonals forced to an exact 0
      const double e2 = pow(10.0, -3 * ur(s)), e1 = e2 * pow(10.0, -6 * ur(s)), e0 = e1 * pow(10.0, -6 * ur(s));
      const double x = ur(s) * 6.28, y = ur(s) * 6.28, z = ur(s) * 6.28;
      const double R[9] = {cos(x) * cos(y), cos(x) * sin(y) * sin(z) - sin(x) * cos(z), cos(x) * sin(y) * cos(z) + sin(x) * sin(z), sin(x) * cos(y),
                           sin(x) * sin(y) * sin(z) + cos(x) * cos(z), sin(x) * sin(y) * cos(z) - cos(x) * sin(z), -sin(y), cos(y) * sin(z), cos(y) * cos(z)};
      const double ev[3] = {e0, e1, e2};
      double A[9];
      for (int i = 0; i < 3; i++)
        for (int jj = 0; jj < 3; jj++) { double v = 0; for (int k = 0; k < 3; k++) v += R[i * 3 + k] * ev[k] * R[jj * 3 + k]; A[i * 3 + jj] = v; }
      const int mode = (int)(t % 5);
      if (mode == 2) A[2] = 0.0;                      // xz = 0
      if (mode == 3) A[1] = 0.0;                      // xy = 0
      if (mode == 4) { A[1] = 0.0; A[5] = 0.0; }      // xy = yz = 0, xz stays
      A[3] = A[1]; A[6] = A[2]; A[7] = A[5];
      if (A[1] == 0.0 && A[2] == 0.0 && A[5] == 0.0) continue;  // diagonal: not this check's input
      zeros += (A[1] == 0.0) + (A[2] == 0.0) + (A[5] == 0.0) > 0;
      double n[3], o[3];
      sym_min_eigvec3(A, n);
      old_sym_min_eigvec3(A, o);
      if (memcmp(n, o, sizeof(n)) != 0) mismatch++;
    }
    printf("mismatch=%ld with_zero_offdiagonal=%ld\n", mismatch, zeros);
    return 0;
  }
  fprintf(stderr, "usage: %s table | random N\n", argv[0]);
  return 2;
}
