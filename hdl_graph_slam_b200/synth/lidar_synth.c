/* lidar_synth.c — seeded synthetic spinning-LiDAR workload generator (SURVEY.md §8d).
 *
 * Workload tooling shared by tests/ and bench.py (NOT part of the oracle, NOT on the product path): it only
 * manufactures input clouds of the shapes BASELINE.json names (VLP-16 16x4096, HDL-32e 32x4096, KITTI 64x1875).
 *
 * World (closed, every ray returns): ground z=0, outer box |x|,|y| <= 60 m, ceiling z=25 m, 40 axis-aligned boxes and
 * 24 vertical cylinders from scene seed 0x5CE9E, placed clear of the sensor circuit (radius ~40 m).
 * Sensor height 1.8 m; the sensor follows the closed circuit of b2s_pose() (radius 40 +- 2 m, ~1 m per frame).  Range noise N(0, sigma) per ray from a counter-based hash of (seed, ray index), seed =
 * 0xB2000000 + frame index by convention.  Points are emitted in the SENSOR frame, azimuth-major (index = az*rings+ring),
 * as `stride` floats per point (x,y,z,1 | intensity,0,0,0 for stride 8  == the 32-byte pcl::PointXYZI record).
 */
#include <math.h>
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#define N_BOX 40
#define N_CYL 24

typedef struct { double cx, cy, hx, hy, h; } box_t;
typedef struct { double cx, cy, r, h; } cyl_t;
static box_t g_box[N_BOX];
static cyl_t g_cyl[N_CYL];
static int g_scene_ready = 0;

static uint64_t splitmix64(uint64_t* s) {
  uint64_t z = (*s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
static double u01(uint64_t* s) { return (double)(splitmix64(s) >> 11) * (1.0 / 9007199254740992.0); }

static void build_scene(void) {
  if (g_scene_ready) return;
  uint64_t s = 0x5CE9Eull;
  for (int i = 0; i < N_BOX; i++) {
    double ang = u01(&s) * 2.0 * M_PI;
    double rad = (i & 1) ? 6.0 + u01(&s) * 24.0 : 49.0 + u01(&s) * 8.0;
    g_box[i].cx = rad * cos(ang);
    g_box[i].cy = rad * sin(ang);
    g_box[i].hx = 0.8 + u01(&s) * 3.0;
    g_box[i].hy = 0.8 + u01(&s) * 3.0;
    g_box[i].h = 2.0 + u01(&s) * 10.0;
  }
  for (int i = 0; i < N_CYL; i++) {
    double ang = u01(&s) * 2.0 * M_PI;
    double rad = (i & 1) ? 8.0 + u01(&s) * 22.0 : 47.0 + u01(&s) * 9.0;
    g_cyl[i].cx = rad * cos(ang);
    g_cyl[i].cy = rad * sin(ang);
    g_cyl[i].r = 0.3 + u01(&s) * 1.2;
    g_cyl[i].h = 3.0 + u01(&s) * 12.0;
  }
  g_scene_ready = 1;
}

/* first positive hit distance of ray o + t d with the world */
static double cast(const double o[3], const double d[3]) {
  double best = 1e30;
  /* ground and ceiling */
  if (d[2] < 0) { double t = (0.0 - o[2]) / d[2]; if (t > 1e-6 && t < best) best = t; }
  if (d[2] > 0) { double t = (25.0 - o[2]) / d[2]; if (t > 1e-6 && t < best) best = t; }
  /* outer walls */
  for (int a = 0; a < 2; a++) {
    if (d[a] > 0) { double t = (60.0 - o[a]) / d[a]; if (t > 1e-6 && t < best) best = t; }
    if (d[a] < 0) { double t = (-60.0 - o[a]) / d[a]; if (t > 1e-6 && t < best) best = t; }
  }
  for (int i = 0; i < N_BOX; i++) {
    const box_t* b = &g_box[i];
    double lo[3] = {b->cx - b->hx, b->cy - b->hy, 0.0}, hi[3] = {b->cx + b->hx, b->cy + b->hy, b->h};
    double t0 = 1e-6, t1 = best;
    int ok = 1;
    for (int a = 0; a < 3 && ok; a++) {
      if (fabs(d[a]) < 1e-12) { if (o[a] < lo[a] || o[a] > hi[a]) ok = 0; continue; }
      double ta = (lo[a] - o[a]) / d[a], tb = (hi[a] - o[a]) / d[a];
      if (ta > tb) { double t = ta; ta = tb; tb = t; }
      if (ta > t0) t0 = ta;
      if (tb < t1) t1 = tb;
      if (t0 > t1) ok = 0;
    }
    if (ok && t0 < best) best = t0;
  }
  for (int i = 0; i < N_CYL; i++) {
    const cyl_t* c = &g_cyl[i];
    double ox = o[0] - c->cx, oy = o[1] - c->cy;
    double A = d[0] * d[0] + d[1] * d[1];
    if (A < 1e-14) continue;
    double B = ox * d[0] + oy * d[1];
    double C = ox * ox + oy * oy - c->r * c->r;
    double disc = B * B - A * C;
    if (disc < 0) continue;
    double t = (-B - sqrt(disc)) / A;
    if (t > 1e-6 && t < best) {
      double z = o[2] + t * d[2];
      if (z >= 0.0 && z <= c->h) best = t;
    }
  }
  return best;
}

/* trajectory pose of frame k: a CLOSED circuit (period 2*pi/0.025 ~ 251.3 frames per lap, ~1 m per frame) that stays inside the
 * object-free corridor: radius 40 +- 2 m around the origin, heading = path tangent plus a bounded wobble.  Closed form, so any
 * frame index (and any rank offset) is valid and loop-closure pairs one lap apart really overlap. */
void b2s_pose(int k, double step, double* x, double* y, double* yaw) {
  const double th = 0.025 * step * (double)k;
  const double r = 40.0 + 2.0 * sin(3.0 * th);
  *x = r * sin(th);
  *y = -r * cos(th);
  *yaw = th + 0.05 * sin(5.0 * th);
}

/* rings: 16 (VLP-16), 32 (HDL-32e), 64 (KITTI HDL-64E shape); any other count from 2 to 64 spreads the beams evenly.
 * returns number of points = rings*n_az, or 0 (nothing written) for a ring count outside [2, 64] (elev[] holds 64 beams) or
 * n_az < 1. */
size_t b2s_scan(int rings, int n_az, double px, double py, double yaw, double roll, double pitch, uint64_t seed, double sigma,
                float* out, size_t stride) {
  double elev[64];
  if (rings < 2 || rings > 64 || n_az < 1) return 0;
  build_scene();
  if (rings == 16) for (int r = 0; r < 16; r++) elev[r] = (-15.0 + 2.0 * r) * M_PI / 180.0;
  else if (rings == 32) for (int r = 0; r < 32; r++) elev[r] = (10.67 - (41.34 / 31.0) * r) * M_PI / 180.0;
  else for (int r = 0; r < rings; r++) elev[r] = (2.0 - (26.8 / (rings - 1)) * r) * M_PI / 180.0;
  /* sensor->world rotation R = Rz(yaw) Ry(pitch) Rx(roll) */
  double cr = cos(roll), sr = sin(roll), cp = cos(pitch), sp = sin(pitch), cy = cos(yaw), sy = sin(yaw);
  double R[9] = {cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr, sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr, -sp, cp * sr, cp * cr};
  double o[3] = {px, py, 1.8};
  size_t n = (size_t)rings * (size_t)n_az;
#pragma omp parallel for schedule(static)
  for (long idx = 0; idx < (long)n; idx++) {
    int az = (int)(idx / rings), r = (int)(idx % rings);
    double a = 2.0 * M_PI * (double)az / (double)n_az, e = elev[r];
    double ds[3] = {cos(e) * cos(a), cos(e) * sin(a), sin(e)};
    double dw[3];
    for (int i = 0; i < 3; i++) dw[i] = R[i * 3 + 0] * ds[0] + R[i * 3 + 1] * ds[1] + R[i * 3 + 2] * ds[2];
    double t = cast(o, dw);
    uint64_t s = seed * 0xD1342543DE82EF95ull + (uint64_t)idx * 0x9E3779B97F4A7C15ull + 0x1234567ull;
    double u1 = u01(&s), u2 = u01(&s);
    if (u1 < 1e-300) u1 = 1e-300;
    double g = sqrt(-2.0 * log(u1)) * cos(2.0 * M_PI * u2);
    t += sigma * g;
    if (t < 0.3) t = 0.3;
    float* p = out + (size_t)idx * stride;
    p[0] = (float)(t * ds[0]);
    p[1] = (float)(t * ds[1]);
    p[2] = (float)(t * ds[2]);
    if (stride >= 4) p[3] = 1.0f;
    if (stride >= 8) {
      p[4] = (float)(u01(&s) * 255.0); /* intensity */
      p[5] = p[6] = p[7] = 0.0f;
    }
  }
  return n;
}
