// tests/ndt_pcl_rounds_harness.cu — the radius search of the pcl NDT pass (csrc/ndt_pcl.cuh: pcl_collect through
// k_ndt_pcl_neighbors) at a radius larger than the leaf, where a query has more than kPclNb = 32 neighbours and the search runs
// its second and later selection rounds (`after`, the replacement of the held maximum, the `total` count).  Through the ABI the
// radius is the leaf size and no query reaches 32 neighbours, so those rounds are only reachable from here.
//
// The target is built through the ABI (b2r_create / b2r_set_target / b2r_ndt_get_centroids on a B2R_METHOD_NDT_PCL handle); the
// harness then launches k_ndt_pcl_neighbors itself with the handle's map and NdtPclArgs::r2 / r_margin set for `radius`.
//   usage: ndt_pcl_rounds_harness target.f32 queries.f32 resolution radius out.bin
//   target.f32: n x 4 float32 (x y z 1); queries.f32: m x 3 float32 (taken untransformed: the identity pose)
//   out.bin: m uint32 counts, then the neighbours' leaf keys as int64, per query in the kernel's order (ascending (d2, leaf))
// stdout: "max_count=<largest count> rounds=<queries with more than 32 neighbours>".
// Test infrastructure: built by tests/test_ndt_pcl_edges_gpu.py with nvcc, never shipped.
#include "../hdl_graph_slam_b200/csrc/api.cu"
#include <cstdio>

static std::vector<float> read_f32(const char* path) {
  std::vector<float> v;
  FILE* f = std::fopen(path, "rb");
  if (!f) return v;
  float x[1024];
  size_t k;
  while ((k = std::fread(x, sizeof(float), 1024, f)) > 0) v.insert(v.end(), x, x + k);
  std::fclose(f);
  return v;
}

#define HCHECK(x)                                                                                  \
  do {                                                                                             \
    const long long rc_ = (long long)(x);                                                          \
    if (rc_ != 0) { std::fprintf(stderr, "%s failed: %lld (%s)\n", #x, rc_, b2r_last_error()); return 1; } \
  } while (0)

int main(int argc, char** argv) {
  if (argc != 6) {
    std::fprintf(stderr, "usage: %s target.f32 queries.f32 resolution radius out.bin\n", argv[0]);
    return 2;
  }
  const std::vector<float> tgt = read_f32(argv[1]), q = read_f32(argv[2]);
  const double res = std::atof(argv[3]), radius = std::atof(argv[4]);
  const size_t nt = tgt.size() / 4;
  const int m = (int)(q.size() / 3);
  if (nt == 0 || m == 0) { std::fprintf(stderr, "empty input\n"); return 2; }
  b2r_config cfg;
  HCHECK(b2r_config_default(&cfg, B2R_METHOD_NDT_PCL));
  cfg.ndt_resolution = res;
  b2r_handle* h = nullptr;
  HCHECK(b2r_create(&cfg, &h));
  HCHECK(b2r_set_target(h, tgt.data(), nt, 4 * sizeof(float)));
  size_t nc = 0;
  HCHECK(b2r_ndt_get_centroids(h, 0, &nc, nullptr, nullptr));  // builds the voxel map, the centroids and their buckets
  NdtVoxelMap& M = *TGT(h).ndt;
  HCHECK(ndt_sync_geom(M, h->ndt_work, h->st));
  NdtArgs A;
  std::memset(&A, 0, sizeof(A));
  A.geom = M.geom.p; A.vox = M.vox.p;
  A.Tf[0] = A.Tf[5] = A.Tf[10] = 1.f;  // identity: ((1 x + 0 y) + 0 z) + 0 == x
  NdtPclArgs P;
  ndt_pcl_fill_args(h->cfg, TGT(h), A, P);
  P.r2 = (float)(radius * radius);  // as ndt_pcl_fill_args derives them from the resolution
  P.r_margin = 1.0001 * radius;
  float* d_q = nullptr;
  unsigned int* d_cnt = nullptr;
  unsigned long long* d_off = nullptr;
  int* d_pos = nullptr;
  HCHECK(cudaMalloc(&d_q, q.size() * sizeof(float)));
  HCHECK(cudaMalloc(&d_cnt, (size_t)m * sizeof(unsigned int)));
  HCHECK(cudaMalloc(&d_off, (size_t)m * sizeof(unsigned long long)));
  HCHECK(cudaMemcpy(d_q, q.data(), q.size() * sizeof(float), cudaMemcpyHostToDevice));
  const unsigned nb = (unsigned)((m + 127) / 128);
  k_ndt_pcl_neighbors<<<nb, 128, 0, h->st>>>(P, d_q, 3, m, d_cnt, nullptr, nullptr);
  HCHECK(cudaGetLastError());
  HCHECK(cudaStreamSynchronize(h->st));
  std::vector<unsigned int> cnt((size_t)m);
  HCHECK(cudaMemcpy(cnt.data(), d_cnt, (size_t)m * sizeof(unsigned int), cudaMemcpyDeviceToHost));
  std::vector<unsigned long long> off((size_t)m + 1, 0);
  unsigned int max_count = 0;
  int rounds = 0;
  for (int i = 0; i < m; i++) {
    off[i + 1] = off[i] + cnt[i];
    max_count = std::max(max_count, cnt[i]);
    rounds += cnt[i] > (unsigned)kPclNb;
  }
  std::vector<int> pos((size_t)off[m] + 1);
  std::vector<unsigned int> vkeys(M.n + 1);
  HCHECK(cudaMalloc(&d_pos, pos.size() * sizeof(int)));
  HCHECK(cudaMemcpy(d_off, off.data(), (size_t)m * sizeof(unsigned long long), cudaMemcpyHostToDevice));
  k_ndt_pcl_neighbors<<<nb, 128, 0, h->st>>>(P, d_q, 3, m, d_cnt, d_off, d_pos);
  HCHECK(cudaGetLastError());
  HCHECK(cudaStreamSynchronize(h->st));
  HCHECK(cudaMemcpy(pos.data(), d_pos, pos.size() * sizeof(int), cudaMemcpyDeviceToHost));
  HCHECK(cudaMemcpy(vkeys.data(), M.keys.p, M.n * sizeof(unsigned int), cudaMemcpyDeviceToHost));
  std::vector<long long> keys((size_t)off[m]);
  for (size_t t = 0; t < keys.size(); t++) keys[t] = (long long)vkeys[pos[t]];
  FILE* f = std::fopen(argv[5], "wb");
  if (!f) { std::fprintf(stderr, "cannot write %s\n", argv[5]); return 1; }
  std::fwrite(cnt.data(), sizeof(unsigned int), cnt.size(), f);
  std::fwrite(keys.data(), sizeof(long long), keys.size(), f);
  std::fclose(f);
  cudaFree(d_q); cudaFree(d_cnt); cudaFree(d_off); cudaFree(d_pos);
  b2r_destroy(h);
  std::printf("max_count=%u rounds=%d\n", max_count, rounds);
  return 0;
}
