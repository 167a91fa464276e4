// approx_voxelgrid_ref.cpp — sequential reference of pcl::ApproximateVoxelGrid<PointXYZI>::applyFilter with setLeafSize(r,r,r) and
// every other setting at its default (/root/reference/apps/prefiltering_nodelet.cpp:61-63; SURVEY.md A.5), the yardstick the
// engine's parallel form (hdl_graph_slam_b200/csrc/approx_voxelgrid.cuh) is compared against.  Test infrastructure only: compiled by
// the tests with -ffp-contract=off, like the oracle, and never linked into the product.
//
// PCL is not under /root/reference, so this restates its walk from the library's documented behaviour (UPSTREAM-RECALL): a
// 512-slot history, one pass over the input in index order with no finiteness check, a slot holding another cell flushed to the
// next output position on a collision, then every non-empty slot flushed in slot order.
#include <climits>
#include <cmath>
#include <cstddef>
#include <cstdint>

namespace {

constexpr int kHistSize = 512;  // histsize_

// static_cast<int>(float) as x86's cvttss2si computes it.  The C++ cast is undefined for NaN, +-inf and values outside int32;
// the instruction gives INT_MIN ("integer indefinite") for all of them, and that result is pinned here explicitly.
int x86_cvtt(float f) { return (f >= -2147483648.0f && f < 2147483648.0f) ? static_cast<int>(f) : INT_MIN; }

struct Slot {
  int ix, iy, iz;
  int count;
  float sum[4];  // x, y, z, intensity
};

void flush(const Slot& h, float* out, size_t stride, int32_t* counts, size_t o) {
  const float c = static_cast<float>(h.count);
  float* r = out + o * stride;
  r[0] = h.sum[0] / c; r[1] = h.sum[1] / c; r[2] = h.sum[2] / c;
  if (stride >= 4) r[3] = 1.0f;
  if (stride >= 5) r[4] = h.sum[3] / c;
  for (size_t j = 5; j < stride; j++) r[j] = 0.0f;
  if (counts) counts[o] = h.count;
}

}  // namespace

// in: n records of `stride` floats (x y z at 0..2, intensity at 4 when stride >= 5); out: up to n records of the same layout;
// counts (may be NULL): points per output.  Returns the output count.
extern "C" size_t ref_approximate_voxelgrid(const float* in, size_t n, size_t stride, float leaf, float* out, int32_t* counts) {
  const float inv = 1.0f / leaf;  // inverse_leaf_size_ = Array3f::Ones() / leaf_size_
  Slot hist[kHistSize];
  for (Slot& h : hist) h.count = 0;
  size_t o = 0;
  for (size_t i = 0; i < n; i++) {
    const float* p = in + i * stride;
    const int ix = x86_cvtt(std::floor(p[0] * inv));
    const int iy = x86_cvtt(std::floor(p[1] * inv));
    const int iz = x86_cvtt(std::floor(p[2] * inv));
    const uint32_t hash = (static_cast<uint32_t>(ix) * 7171u + static_cast<uint32_t>(iy) * 3079u + static_cast<uint32_t>(iz) * 4231u) &
                          static_cast<uint32_t>(kHistSize - 1);
    Slot& h = hist[hash];
    if (h.count != 0 && (h.ix != ix || h.iy != iy || h.iz != iz)) {
      flush(h, out, stride, counts, o++);
      h.count = 0;
    }
    if (h.count == 0) {
      h.ix = ix; h.iy = iy; h.iz = iz;
      h.sum[0] = h.sum[1] = h.sum[2] = h.sum[3] = 0.0f;
    }
    h.sum[0] += p[0]; h.sum[1] += p[1]; h.sum[2] += p[2];
    h.sum[3] += stride >= 5 ? p[4] : 0.0f;
    h.count++;
  }
  for (int s = 0; s < kHistSize; s++)
    if (hist[s].count != 0) flush(hist[s], out, stride, counts, o++);
  return o;
}

// the pinned rule and the plain cast side by side, so a test can check the rule against this host's conversion
extern "C" int ref_x86_cvtt(float f) { return x86_cvtt(f); }
extern "C" int ref_static_cast_int(float f) {
  volatile float v = f;  // keep the conversion a run-time cvttss2si, not a constant the compiler folds
  return static_cast<int>(v);
}
