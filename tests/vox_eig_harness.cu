// tests/vox_eig_harness.cu — CPU check (linalg.cuh compiled as host code): the NDT voxel finalisation the engine runs in
// k_vox_finalize (ndt_voxel_gaussian: covariance, sym_eigen3, eigenvalue clamp, inverse) against the oracle's
// orc_ndt_voxel_gaussian / orc::sym_eigen<3>, BIT FOR BIT, on voxels where the validity decision is rounding noise: points on
// exact planes (axis-aligned and x - y = c), exact lines (axis-aligned and x = y = z), all-identical points, plus generic and
// nearly planar voxels, with and without a large offset of the scene.  Test infrastructure, never shipped.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include "../hdl_graph_slam_b200/csrc/linalg.cuh"
#include "../oracle/linalg.hpp"
#include "../oracle/oracle.h"

static unsigned long long g_s = 12345;
static double ur() { g_s = g_s * 6364136223846793005ull + 1442695040888963407ull; return (double)(g_s >> 11) / 9007199254740992.0; }
static int ui(int n) { return (int)(ur() * n) % n; }

int main(int argc, char** argv) {
  const int N = argc > 1 ? atoi(argv[1]) : 100000;
  long eig_mismatch = 0, gauss_mismatch = 0, invalid = 0, clamped_one = 0, clamped_two = 0, kinds[8] = {0};
  float P[16][3];
  for (int t = 0; t < N; t++) {
    const int kind = t % 8;
    const int n = 5 + ui(11);  // 5 .. 15 points (5: below min_points_per_voxel)
    const bool shifted = (t / 8) % 2 == 1;
    const double ox = shifted ? 2.0e4 : 0.0, oy = shifted ? -3.0e4 : 0.0, oz = shifted ? 50.0 : 0.0;
    // grid values k / 256 are exact in float32, also after adding the offset, and keep x - y = c exact
    const float c0 = (float)(ui(512) - 256) / 256.0f, c1 = (float)(ui(512) - 256) / 256.0f;
    for (int i = 0; i < n; i++) {
      const float a = (float)ui(1024) / 1024.0f, b = (float)ui(1024) / 1024.0f, r = (float)ur();
      float x, y, z;
      switch (kind) {
        case 0: x = a; y = a - c0; z = r; break;                            // plane x - y = c0
        case 1: x = r; y = r; z = r; break;                                 // line x = y = z
        case 2: x = (float)ur(); y = (float)ur(); z = c0; break;            // plane z = c0
        case 3: x = r; y = c0; z = c1; break;                               // line along x
        case 4: x = a; y = a + c0; z = c1; break;                           // diagonal line in a horizontal plane
        case 5: x = c0; y = c1; z = 0.25f; break;                           // all points identical
        case 6: x = (float)ur(); y = (float)ur(); z = (float)ur(); break;   // generic
        default: x = a; y = b; z = c0 + (float)(1e-6 * ur()); break;       // nearly planar
      }
      P[i][0] = (float)(x + ox); P[i][1] = (float)(y + oy); P[i][2] = (float)(z + oz);
    }
    if (kind == 0 || kind == 4) {  // y from the (shifted) x in one exact float subtraction: the plane / line stays exact
      const float C = kind == 0 ? (float)((ox - oy) + c0) : (float)((oy - ox) + c0);
      for (int i = 0; i < n; i++) P[i][1] = kind == 0 ? P[i][0] - C : P[i][0] + C;
    }
    // float64 moments in ascending point order (k_vox_finalize / orc_ndt_build)
    double S[3] = {0, 0, 0}, S2[9] = {0};
    for (int i = 0; i < n; i++) {
      const double q[3] = {(double)P[i][0], (double)P[i][1], (double)P[i][2]};
      for (int u = 0; u < 3; u++) {
        S[u] += q[u];
        for (int v = 0; v < 3; v++) S2[u * 3 + v] += q[u] * q[v];
      }
    }
    double m0[3], i0[9], m1[3], c1v[9], i1[9];
    const int n0 = b2r::ndt_voxel_gaussian(n, S, S2, m0, i0);
    const int n1 = orc_ndt_voxel_gaussian(n, S, S2, m1, c1v, i1);
    if (n0 != n1 || memcmp(m0, m1, sizeof(m0)) != 0 || memcmp(i0, i1, sizeof(i0)) != 0) {
      if (gauss_mismatch < 5) printf("gauss mismatch t=%d kind=%d n=%d npts %d vs %d\n", t, kind, n, n0, n1);
      gauss_mismatch++;
    }
    if (n1 < 0) invalid++;
    if (n >= 6) {
      // the eigen-solver alone on the covariance both sides start from
      double cov[9];
      const double nn = (double)n, f = (nn - 1.0) / nn;
      for (int u = 0; u < 3; u++)
        for (int v = 0; v < 3; v++) {
          volatile double tt = (S2[u * 3 + v] - 2 * (S[u] * m1[v])) / nn;
          volatile double mm = m1[u] * m1[v];
          volatile double sum = tt + mm;
          cov[u * 3 + v] = sum * f;
        }
      double w0[3], V0[9], w1[3], V1[9];
      b2r::sym_eigen3(cov, w0, V0);
      orc::sym_eigen<3>(cov, w1, V1);
      if (memcmp(w0, w1, sizeof(w0)) != 0 || memcmp(V0, V1, sizeof(V0)) != 0) {
        if (eig_mismatch < 5) printf("eigen mismatch t=%d kind=%d w %.17g %.17g %.17g vs %.17g %.17g %.17g\n", t, kind, w0[0], w0[1], w0[2], w1[0], w1[1], w1[2]);
        eig_mismatch++;
      }
      if (n1 > 0 && w1[0] < 0.01 * w1[2]) (w1[1] < 0.01 * w1[2] ? clamped_two : clamped_one)++;
    }
    kinds[kind]++;
  }
  printf("cases=%d eig_mismatch=%ld gauss_mismatch=%ld invalid=%ld clamped_one=%ld clamped_two=%ld\n", N, eig_mismatch, gauss_mismatch, invalid,
         clamped_one, clamped_two);
  return (eig_mismatch == 0 && gauss_mismatch == 0) ? 0 : 1;
}
