// batch.cuh — host side of the batched registration path (included by api.cu after the handle and the build helpers).
//
//   b2r_batch            a keyframe-cloud cache + a pool of pair slots on ONE GPU; many (source, target) pairs per launch
//   b2r_batch_add_cloud  <- KeyFrame::cloud becoming known to the loop detector (keyframe.hpp:40): uploaded ONCE, its search
//                           structure and GICP covariances are built once and reused by every pair that names it (the reference
//                           rebuilds kd-tree + covariances at every setInputSource/Target: loop_detector.hpp:122,136)
//   b2r_batch_align      <- the candidate loop of LoopDetector::matching (loop_detector.hpp:135-154): align + getFitnessScore
//   b2r_batch_loop_detect<- LoopDetector::matching for MANY new keyframes, groups sharded over the ranks of an NCCL communicator,
//                           ONE ncclAllGather of 80-byte b2r_result records, per-group argmin with the reference's tie rule (:147,160)
#pragma once
#include <nccl.h>
#include <chrono>

struct b2r_batch {
  b2r_handle* eng = nullptr;  // engine context of this device: config, main stream, telemetry
  static constexpr int kBuildStreams = 4;
  cudaStream_t bst[kBuildStreams] = {nullptr, nullptr, nullptr, nullptr};
  BuildCtx bctx[kBuildStreams];
  cudaEvent_t bev[kBuildStreams] = {nullptr, nullptr, nullptr, nullptr};
  int next_stream = 0;
  std::vector<Cloud*> clouds;
  std::vector<int> free_ids;
  std::vector<Cloud*> recycled;  // removed clouds keep their device buffers for the next add (no cudaMalloc churn per keyframe)
  // pair slots.  A chunk of pairs can be split over kLanes independent round sequences ("lanes"), each on its own stream, so that a
  // lane's search kernel (instruction-issue bound) runs beside the other lane's accumulate kernel and a lane's thin tail rounds
  // overlap the other's fat ones.  Two lanes did not beat one on 256 pairs x 64k points — the block
  // scheduler drains one kernel's grid before it starts the next stream's, so the overlap is confined to the tails; the default
  // is ONE lane (B2R_BATCH_LANES=2 enables the second).  Lane 0 runs on the engine's main stream.
  static constexpr int kLanes = 2;
  struct Lane {
    cudaStream_t st = nullptr;
    cudaEvent_t ev = nullptr;
    DevBuf<PairDev> d_pairs;
    DevBuf<int> d_active;
    unsigned long long* h_word = nullptr;  // host-mapped: (seq << 32) | pairs still active
    unsigned long long* h_word_dev = nullptr;
    unsigned long long seq = 0;
  };
  Lane lane[kLanes];
  cudaEvent_t fork_ev = nullptr;
  int n_lanes = 1;
  DevBuf<PairReport> d_reports;
  DevBuf<char> ws;
  PairDev* h_pairs = nullptr;       // pinned staging
  PairReport* h_reports = nullptr;  // pinned staging
  size_t h_cap = 0;
  unsigned long long* h_word = nullptr;  // host-mapped: [0..kLanes) = the lanes' words, [kLanes] = sum of the pairs' executed rounds
  unsigned long long* h_word_dev = nullptr;
  size_t max_chunk = 1024;  // pairs in flight per launch sequence (~7.7 MB of workspace per 64k-point pair)
  int copies = 1;           // lanes per query of the batched 1-NN search
  // multi-GPU
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1;
  DevBuf<b2r_result> d_send, d_recv;
  DevBuf<BuildItem> d_build;        // descriptor list of the batched cluster builds
  BuildItem* h_build = nullptr;     // pinned staging
  size_t h_build_cap = 0;
  DevBuf<KnnBatchItem> d_knn;       // descriptor list of one batched k-NN covariance launch
  KnnBatchItem* h_knn = nullptr;    // pinned staging
  size_t h_knn_cap = 0;
  b2r_result* h_gather = nullptr;
  size_t h_gather_cap = 0;
  // telemetry of the last b2r_batch_align
  unsigned long long last_rounds = 0, last_pair_rounds = 0;
};

#define B2R_NCCL(expr)                                                                                     \
  do {                                                                                                     \
    ncclResult_t _r = (expr);                                                                              \
    if (_r != ncclSuccess) return b2r::fail(B2R_ENCCL, std::string(#expr) + ": " + ncclGetErrorString(_r)); \
  } while (0)

static void free_cloud(Cloud* c) {
  if (!c) return;
  c->raw.release(); c->sorted.release(); c->leaf_lo.release(); c->leaf_hi.release(); c->sup_lo.release(); c->sup_hi.release(); c->pos_of.release(); c->cov.release();
  ndt_free_map(c->ndt);
  delete c;
}

extern "C" void b2r_batch_destroy(b2r_batch* b) {
  if (!b) return;
  if (b->eng) cudaSetDevice(b->eng->cfg.device_id);
  if (b->eng && b->eng->st) cudaStreamSynchronize(b->eng->st);
  for (int i = 0; i < b2r_batch::kBuildStreams; i++) {
    if (b->bst[i]) { cudaStreamSynchronize(b->bst[i]); cudaStreamDestroy(b->bst[i]); }
    if (b->bev[i]) cudaEventDestroy(b->bev[i]);
    b->bctx[i].release();
  }
  if (b->comm) ncclCommDestroy(b->comm);
  for (Cloud* c : b->clouds) free_cloud(c);
  for (Cloud* c : b->recycled) free_cloud(c);
  for (int l = 0; l < b2r_batch::kLanes; l++) {
    b2r_batch::Lane& L = b->lane[l];
    if (l > 0 && L.st) { cudaStreamSynchronize(L.st); cudaStreamDestroy(L.st); }
    if (L.ev) cudaEventDestroy(L.ev);
    L.d_pairs.release(); L.d_active.release();
  }
  if (b->fork_ev) cudaEventDestroy(b->fork_ev);
  b->d_reports.release(); b->ws.release(); b->d_send.release(); b->d_recv.release();
  if (b->h_pairs) cudaFreeHost(b->h_pairs);
  if (b->h_reports) cudaFreeHost(b->h_reports);
  if (b->h_word) cudaFreeHost(b->h_word);
  if (b->h_gather) cudaFreeHost(b->h_gather);
  if (b->h_knn) cudaFreeHost(b->h_knn);
  if (b->h_build) cudaFreeHost(b->h_build);
  b->d_knn.release(); b->d_build.release();
  if (b->eng) b2r_destroy(b->eng);
  delete b;
}

extern "C" int b2r_batch_create(const b2r_config* cfg, b2r_batch** out) {
  if (!cfg || !out) return fail(B2R_EINVAL, "NULL argument");
  *out = nullptr;
  if (cfg->method != B2R_METHOD_GICP) return fail(B2R_EUNSUPPORTED, "the batched path re-creates the GICP engine only (the reference's loop closure runs FAST_GICP: hdl_graph_slam.launch:127)");
  b2r_batch* b = new b2r_batch();
  int rc = b2r_create(cfg, &b->eng);
  if (rc) { delete b; return rc; }
  auto bail = [&](int code) { b2r_batch_destroy(b); return code; };
  for (int i = 0; i < b2r_batch::kBuildStreams; i++) {
    if (cudaStreamCreateWithFlags(&b->bst[i], cudaStreamNonBlocking) != cudaSuccess || cudaEventCreateWithFlags(&b->bev[i], cudaEventDisableTiming) != cudaSuccess ||
        cudaMalloc(&b->bctx[i].mm, 8 * sizeof(int)) != cudaSuccess)
      return bail(fail(B2R_ECUDA, "stream / scratch creation failed"));
  }
  if (cudaHostAlloc(&b->h_word, 64, cudaHostAllocMapped) != cudaSuccess || cudaHostGetDevicePointer((void**)&b->h_word_dev, b->h_word, 0) != cudaSuccess)
    return bail(fail(B2R_ECUDA, "host allocation failed"));
  for (int i = 0; i < 8; i++) b->h_word[i] = 0;
  if (cudaEventCreateWithFlags(&b->fork_ev, cudaEventDisableTiming) != cudaSuccess) return bail(fail(B2R_ECUDA, "event creation failed"));
  for (int l = 0; l < b2r_batch::kLanes; l++) {
    b2r_batch::Lane& L = b->lane[l];
    L.h_word = b->h_word + l; L.h_word_dev = b->h_word_dev + l;
    if (l == 0) L.st = b->eng->st;
    else if (cudaStreamCreateWithFlags(&L.st, cudaStreamNonBlocking) != cudaSuccess) return bail(fail(B2R_ECUDA, "stream creation failed"));
    if (cudaEventCreateWithFlags(&L.ev, cudaEventDisableTiming) != cudaSuccess) return bail(fail(B2R_ECUDA, "event creation failed"));
  }
  if (const char* e = getenv("B2R_BATCH_LANES")) { const int c = atoi(e); if (c >= 1 && c <= b2r_batch::kLanes) b->n_lanes = c; }
  if (const char* e = getenv("B2R_BATCH_COPIES")) { const int c = atoi(e); if (c == 1 || c == 2 || c == 4) b->copies = c; }
  if (const char* e = getenv("B2R_BATCH_CHUNK")) { const long c = atol(e); if (c > 0) b->max_chunk = (size_t)c; }
  *out = b;
  return B2R_OK;
}

extern "C" int b2r_batch_get_engine(b2r_batch* b, b2r_handle** out) {
  if (!b || !out) return fail(B2R_EINVAL, "NULL argument");
  *out = b->eng;
  return B2R_OK;
}

static int batch_add(b2r_batch* b, const void* pts, size_t n, size_t stride_bytes, bool device_ptr, int32_t* id_out) {
  if (!b || !id_out) return fail(B2R_EINVAL, "NULL argument");
  if (stride_bytes < 12 || (stride_bytes & 3)) return fail(B2R_EINVAL, "stride_bytes must be a multiple of 4 and >= 12");
  if (n > 0 && !pts) return fail(B2R_EINVAL, "points is NULL");
  if (n > (size_t)0x3fffffff) return fail(B2R_EINVAL, "too many points");
  B2R_CUDA(cudaSetDevice(b->eng->cfg.device_id));
  Cloud* c;
  if (!b->recycled.empty()) { c = b->recycled.back(); b->recycled.pop_back(); c->invalidate(); }
  else c = new Cloud();
  c->n = n;
  c->stride_f = (int)(stride_bytes / 4);
  c->host_ptr = pts;
  const int si = b->next_stream;
  b->next_stream = (b->next_stream + 1) % b2r_batch::kBuildStreams;
  cudaStream_t st = b->bst[si];
  if (device_ptr) {
    c->raw_view = (const float*)pts;
  } else {
    cudaError_t e = c->raw.reserve(n * c->stride_f + 4);
    if (e != cudaSuccess) { free_cloud(c); return fail(B2R_ECUDA, std::string("device allocation failed: ") + cudaGetErrorString(e)); }
    c->raw_view = c->raw.p;
    if (n) {
      // pinned buffers are DMA'd in place (asynchronously: see b200reg.h for the lifetime rule); pageable ones are staged by the driver
      e = cudaMemcpyAsync(c->raw.p, pts, n * stride_bytes, cudaMemcpyHostToDevice, st);
      if (e != cudaSuccess) { free_cloud(c); return fail(B2R_ECUDA, std::string("upload failed: ") + cudaGetErrorString(e)); }
      b->eng->tel.h2d += n * stride_bytes;
    }
  }
  // the upload is all that happens here (4 copy streams); the search structures and k-NN covariances of ALL new clouds are built
  // together at the next align: one cluster-build launch per cluster size and one k-NN launch (batch_build_structures)
  int id;
  if (!b->free_ids.empty()) { id = b->free_ids.back(); b->free_ids.pop_back(); b->clouds[id] = c; }
  else { id = (int)b->clouds.size(); b->clouds.push_back(c); }
  *id_out = id;
  return B2R_OK;
}
extern "C" int b2r_batch_add_cloud(b2r_batch* b, const void* pts, size_t n, size_t stride_bytes, int32_t* id_out) { return batch_add(b, pts, n, stride_bytes, false, id_out); }
extern "C" int b2r_batch_add_cloud_device(b2r_batch* b, const void* d_pts, size_t n, size_t stride_bytes, int32_t* id_out) { return batch_add(b, d_pts, n, stride_bytes, true, id_out); }

static int batch_sync_builds(b2r_batch* b, bool host_wait) {
  for (int i = 0; i < b2r_batch::kBuildStreams; i++) {
    if (host_wait) B2R_CUDA(cudaStreamSynchronize(b->bst[i]));
    else {
      B2R_CUDA(cudaEventRecord(b->bev[i], b->bst[i]));
      B2R_CUDA(cudaStreamWaitEvent(b->eng->st, b->bev[i], 0));
    }
  }
  return B2R_OK;
}

extern "C" int b2r_batch_synchronize(b2r_batch* b) {
  if (!b) return fail(B2R_EINVAL, "NULL argument");
  B2R_CUDA(cudaSetDevice(b->eng->cfg.device_id));
  int rc = batch_sync_builds(b, true);
  if (rc) return rc;
  B2R_CUDA(cudaStreamSynchronize(b->eng->st));
  return B2R_OK;
}

extern "C" int b2r_batch_remove_cloud(b2r_batch* b, int32_t id) {
  if (!b) return fail(B2R_EINVAL, "NULL argument");
  if (id < 0 || (size_t)id >= b->clouds.size() || !b->clouds[id]) return fail(B2R_EINVAL, "unknown cloud id");
  int rc = b2r_batch_synchronize(b);  // nothing in flight may still read it
  if (rc) return rc;
  b->recycled.push_back(b->clouds[id]);
  b->clouds[id] = nullptr;
  b->free_ids.push_back(id);
  return B2R_OK;
}

extern "C" int b2r_batch_cloud_count(const b2r_batch* b) {
  if (!b) return 0;
  return (int)(b->clouds.size() - b->free_ids.size());
}

// Search structure (bvh_build.cuh) + FastGICP::calculate_covariances for every cloud a batch names that does not have them yet:
// one cluster-build launch per cluster size and one k-NN launch for all of them (what setInputSource / setInputTarget make the
// reference pay per call: kd-tree build + covariances, loop_detector.hpp:122,136)
static int batch_build_structures(b2r_batch* b, const b2r_pair* pairs, size_t n_pairs, bool need_cov) {
  b2r_handle* h = b->eng;
  cudaStream_t st = h->st;
  std::vector<Cloud*> todo;
  std::vector<char> queued(b->clouds.size(), 0);
  for (size_t i = 0; i < n_pairs; i++)
    for (int32_t id : {pairs[i].source, pairs[i].target}) {
      Cloud* c = b->clouds[id];
      if (queued[id] || c->n == 0 || (c->bvh_ready && (c->cov_ready || !need_cov))) continue;
      queued[id] = 1;
      todo.push_back(c);
    }
  if (todo.empty()) return B2R_OK;
  {  // ---- structures
    std::vector<Cloud*> by_cl[kBuildShapes];  // one launch per (cluster size, pairs per thread) shape
    size_t total = 0;
    for (Cloud* c : todo) {
      if (c->bvh_ready) continue;
      const BuildShape shape = build_shape_for(c->n, cluster16_allowed());
      if (!shape.cl || !use_cluster_build()) { int rc = build_bvh(h, *c, h->bc[0], st); if (rc) return rc; continue; }
      int rc = bvh_alloc(*c);
      if (rc) return rc;
      by_cl[build_shape_index(shape)].push_back(c);
      total++;
    }
    if (total) {
      B2R_CUDA(b->d_build.reserve(total));
      if (b->h_build_cap < total) {
        if (b->h_build) cudaFreeHost(b->h_build);
        b->h_build = nullptr; b->h_build_cap = 0;
        B2R_CUDA(cudaMallocHost(&b->h_build, (total + 64) * sizeof(BuildItem)));
        b->h_build_cap = total + 64;
      }
      size_t k0 = 0;
      for (int g = 0; g < kBuildShapes; g++)
        for (Cloud* c : by_cl[g]) b->h_build[k0++] = build_item(*c);
      B2R_CUDA(cudaMemcpyAsync(b->d_build.p, b->h_build, total * sizeof(BuildItem), cudaMemcpyHostToDevice, st));
      k0 = 0;
      for (int g = 0; g < kBuildShapes; g++) {
        if (by_cl[g].empty()) continue;
        TEL_BEGIN(&h->tel, st);
        B2R_CUDA(launch_cluster_build(g, b->d_build.p + k0, BuildItem(), (unsigned)by_cl[g].size(), st));
        TEL_END(&h->tel, KC_GRID, 1, st);
        for (Cloud* c : by_cl[g]) c->bvh_ready = true;
        k0 += by_cl[g].size();
      }
    }
  }
  if (!need_cov) return B2R_OK;
  {
    std::vector<Cloud*> need;
    for (Cloud* c : todo) if (!c->cov_ready) need.push_back(c);
    todo.swap(need);
  }
  if (todo.empty()) return B2R_OK;
  const int k = h->cfg.k_correspondences;
  for (Cloud* c : todo) B2R_CUDA(c->cov.reserve((size_t)c->nsup * 1024 * 6 + 6));
  if (k != kKnnRegK) {  // other k: the generic shared-memory-list kernel, one launch per cloud
    for (Cloud* c : todo) { int rc = build_cov(h, *c, h->bc[0], st); if (rc) return rc; }
    return B2R_OK;
  }
  B2R_CUDA(b->d_knn.reserve(todo.size()));
  if (b->h_knn_cap < todo.size()) {
    if (b->h_knn) cudaFreeHost(b->h_knn);
    b->h_knn = nullptr; b->h_knn_cap = 0;
    B2R_CUDA(cudaMallocHost(&b->h_knn, (todo.size() + 64) * sizeof(KnnBatchItem)));
    b->h_knn_cap = todo.size() + 64;
  }
  unsigned max_blocks = 0;
  for (size_t i = 0; i < todo.size(); i++) {
    Cloud* c = todo[i];
    KnnBatchItem& it = b->h_knn[i];
    it.b = c->bvh(); it.raw = c->raw_view; it.cov = c->cov.p; it.stride_f = c->stride_f; it.pad = 0;
    max_blocks = std::max(max_blocks, (unsigned)((size_t)c->nsup * 1024 / kKnnThreads));
  }
  B2R_CUDA(cudaMemcpyAsync(b->d_knn.p, b->h_knn, todo.size() * sizeof(KnnBatchItem), cudaMemcpyHostToDevice, st));
  { TEL_BEGIN(&h->tel, st);
    k_knn_cov_reg_batch<kKnnRegK><<<dim3(max_blocks, (unsigned)todo.size()), kKnnThreads, 0, st>>>(b->d_knn.p);
    TEL_END(&h->tel, KC_KNN_COV, 1, st); }
  B2R_CUDA(cudaGetLastError());
  for (Cloud* c : todo) c->cov_ready = true;
  return B2R_OK;
}

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
static size_t pair_ws_bytes(size_t n_pad, bool fit_only) {
  size_t t = 0;
  t += 2 * align_up(n_pad * sizeof(int), 256);          // cpos
  if (!fit_only) {
    t += 2 * align_up(n_pad * sizeof(int), 256);          // corr
    t += 2 * align_up(n_pad * 6 * sizeof(double), 256);   // mahal
  }
  t += align_up(n_pad * sizeof(float), 256);            // d2
  t += align_up((n_pad / kAccThreads + 32) * kAcc * sizeof(double), 256);  // partials: [kAcc][blocks rounded up to 32]
  return t;
}

static void degenerate_report(PairReport& r, const float* guess_col) {
  std::memset(&r, 0, sizeof(r));
  // pcl::Registration::initCompute fails silently on an empty cloud: converged_ = false, final_transformation_ = guess
  // (fast_gicp never runs); getFitnessScore finds no neighbours: DBL_MAX
  for (int i = 0; i < 16; i++) r.r.T[i] = guess_col[i];
  r.r.T[3] = r.r.T[7] = r.r.T[11] = 0.f; r.r.T[15] = 1.f;
  r.r.fitness = DBL_MAX;
}

static int batch_host_staging(b2r_batch* b, size_t n) {
  if (b->h_cap >= n) return B2R_OK;
  const size_t want = n + n / 4 + 16;
  if (b->h_pairs) cudaFreeHost(b->h_pairs);
  if (b->h_reports) cudaFreeHost(b->h_reports);
  b->h_pairs = nullptr; b->h_reports = nullptr; b->h_cap = 0;
  B2R_CUDA(cudaMallocHost(&b->h_pairs, want * sizeof(PairDev)));
  B2R_CUDA(cudaMallocHost(&b->h_reports, want * sizeof(PairReport)));
  b->h_cap = want;
  return B2R_OK;
}

static int wait_word(const b2r_batch::Lane& L, unsigned long long need_seq, size_t* count) {
  const volatile unsigned long long* w = L.h_word;
  unsigned long spins = 0;
  for (;;) {
    const unsigned long long v = *w;
    if ((v >> 32) >= need_seq) { *count = (size_t)(v & 0xffffffffull); return B2R_OK; }
    if ((++spins & 0xffff) == 0) {
      cudaError_t e = cudaStreamQuery(L.st);
      if (e == cudaSuccess) {  // everything has run: the word must be there now
        const unsigned long long v2 = *w;
        if ((v2 >> 32) >= need_seq) { *count = (size_t)(v2 & 0xffffffffull); return B2R_OK; }
        return fail(B2R_ECUDA, "round finished without publishing its active count");
      }
      if (e != cudaErrorNotReady) return fail(B2R_ECUDA, std::string("stream error: ") + cudaGetErrorString(e));
    }
  }
}

// One chunk: pairs[0..m) -> d_rep[0..m) (device).  Every pair of the chunk is in flight at once, split over the lanes; a lane's
// rounds cover all of its pairs.
static int batch_run_chunk(b2r_batch* b, const b2r_pair* pairs, size_t m, const LmCfg& cfg, PairReport* d_rep, bool fit_only) {
  b2r_handle* h = b->eng;
  cudaStream_t st = h->st;
  // per-launch kernel timing (b2r_set_profiling) wants every kernel alone on the device; tiny chunks are not worth a second stream
  const int n_lanes = (h->tel.on || m < 16) ? 1 : b->n_lanes;
  size_t ws_total = 0;
  for (size_t i = 0; i < m; i++) {
    const Cloud& s = *b->clouds[pairs[i].source];
    const Cloud& t = *b->clouds[pairs[i].target];
    if (s.n == 0 || t.n == 0) continue;
    ws_total += pair_ws_bytes((size_t)s.nsup * 1024, fit_only);
  }
  B2R_CUDA(b->ws.reserve(ws_total + 256));
  char* wp = b->ws.p;
  wp = reinterpret_cast<char*>(align_up(reinterpret_cast<size_t>(wp), 256));
  struct LaneRun { size_t i0 = 0, m = 0, known = 0, max_pad = 0; unsigned long long seq_prev = 0; };
  LaneRun run[b2r_batch::kLanes];
  if (n_lanes > 1) {
    B2R_CUDA(cudaEventRecord(b->fork_ev, st));  // the other lanes start after everything the main stream holds so far (uploads, builds, the previous chunk)
    for (int l = 1; l < n_lanes; l++) B2R_CUDA(cudaStreamWaitEvent(b->lane[l].st, b->fork_ev, 0));
  }
  for (int l = 0; l < n_lanes; l++) {
    b2r_batch::Lane& L = b->lane[l];
    LaneRun& R = run[l];
    R.i0 = m * (size_t)l / (size_t)n_lanes;
    R.m = m * (size_t)(l + 1) / (size_t)n_lanes - R.i0;
    if (R.m == 0) continue;
    B2R_CUDA(L.d_pairs.reserve(R.m));
    B2R_CUDA(L.d_active.reserve(R.m + 1));
    for (size_t i = R.i0; i < R.i0 + R.m; i++) {
      PairDev& P = b->h_pairs[i];
      const Cloud& s = *b->clouds[pairs[i].source];
      const Cloud& t = *b->clouds[pairs[i].target];
      if (s.n == 0 || t.n == 0) {
        std::memset(&P, 0, sizeof(P));
        P.mode = PM_DONE;
        degenerate_report(b->h_reports[i], pairs[i].guess);
        B2R_CUDA(cudaMemcpyAsync(d_rep + i, &b->h_reports[i], sizeof(PairReport), cudaMemcpyHostToDevice, L.st));
        continue;
      }
      fill_pair_geometry(P, s, t);
      double x[16];
      colmajor_f_to_row_d(pairs[i].guess, x);
      // a stand-alone fitness evaluation (calc_fitness_score) is a pair that starts in its fitness round at the given pose
      fill_pair_start(P, x, fit_only ? PM_FIT : PM_FIRST);
      const size_t n_pad = (size_t)s.nsup * 1024;
      for (int k = 0; k < 2; k++) { P.cpos[k] = reinterpret_cast<int*>(wp); wp += align_up(n_pad * sizeof(int), 256); }
      if (!fit_only) {
        for (int k = 0; k < 2; k++) { P.corr[k] = reinterpret_cast<int*>(wp); wp += align_up(n_pad * sizeof(int), 256); }
        for (int k = 0; k < 2; k++) { P.mahal[k] = reinterpret_cast<double*>(wp); wp += align_up(n_pad * 6 * sizeof(double), 256); }
      }
      P.d2 = reinterpret_cast<float*>(wp); wp += align_up(n_pad * sizeof(float), 256);
      P.partials = reinterpret_cast<double*>(wp); wp += align_up((n_pad / kAccThreads + 32) * kAcc * sizeof(double), 256);
      P.report = d_rep + i;
      R.known++;
      if (n_pad > R.max_pad) R.max_pad = n_pad;
    }
    B2R_CUDA(cudaMemcpyAsync(L.d_pairs.p, b->h_pairs + R.i0, R.m * sizeof(PairDev), cudaMemcpyHostToDevice, L.st));
    h->tel.h2d += R.m * sizeof(PairDev);
    k_pair_compact<<<1, 1024, 0, L.st>>>(L.d_pairs.p, (int)R.m, L.d_active.p, L.h_word_dev, ++L.seq);
    B2R_CUDA(cudaGetLastError());
  }
  // rounds: the host enqueues round r+1 while the device runs round r and consumes the active count of round r-1 (lag 1), so
  // grid.y shrinks as pairs converge and the device never waits for the host.  The lanes' rounds are enqueued alternately.
  static const bool pdl = !getenv("B2R_NO_PDL");
  for (;;) {
    bool any = false;
    unsigned long long sq[b2r_batch::kLanes] = {};
    for (int l = 0; l < n_lanes; l++) {
      b2r_batch::Lane& L = b->lane[l];
      LaneRun& R = run[l];
      if (R.known == 0) continue;
      any = true;
      int rc = launch_round(L.d_pairs.p, L.d_active.p, (unsigned)R.known, (unsigned)R.max_pad, b->copies, cfg, L.st, &h->tel, true);
      if (rc) return rc;
      b->last_rounds++;
      sq[l] = ++L.seq;
      cudaLaunchConfig_t lc = {};
      lc.gridDim = dim3(1); lc.blockDim = dim3(1024); lc.dynamicSmemBytes = 0; lc.stream = L.st;
      cudaLaunchAttribute la[1];
      la[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      la[0].val.programmaticStreamSerializationAllowed = 1;
      lc.attrs = la; lc.numAttrs = pdl ? 1 : 0;
      B2R_CUDA(cudaLaunchKernelEx(&lc, k_pair_compact, (const PairDev*)L.d_pairs.p, (int)R.m, L.d_active.p, L.h_word_dev, sq[l]));
    }
    if (!any) break;
    for (int l = 0; l < n_lanes; l++) {
      if (!sq[l]) continue;
      LaneRun& R = run[l];
      if (R.seq_prev) {
        int rc = wait_word(b->lane[l], R.seq_prev, &R.known);
        if (rc) return rc;
      }
      R.seq_prev = sq[l];
    }
  }
  for (int l = 1; l < n_lanes; l++) {  // join: whatever follows on the main stream sees every lane's reports
    B2R_CUDA(cudaEventRecord(b->lane[l].ev, b->lane[l].st));
    B2R_CUDA(cudaStreamWaitEvent(st, b->lane[l].ev, 0));
  }
  return B2R_OK;
}

__global__ void k_pack_results(const PairReport* rep, int n, b2r_result* out, int n_out, unsigned long long* round_sum) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_out) return;
  b2r_result r;
  if (i < n) { r = rep[i].r; atomicAdd(round_sum, (unsigned long long)rep[i].rounds); }
  else { for (int k = 0; k < 16; k++) r.T[k] = 0.f; r.fitness = 0.0; r.converged = 0; r.iterations = 0; }
  out[i] = r;
}

// pairs[0..n) -> d_reports[0..n) on the device (no host copy of the results)
static int batch_run(b2r_batch* b, const b2r_pair* pairs, size_t n_pairs, bool want_fitness, double fit_max_range, bool fit_only = false) {
  b2r_handle* h = b->eng;
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  for (size_t i = 0; i < n_pairs; i++) {
    const b2r_pair& pr = pairs[i];
    if (pr.source < 0 || pr.target < 0 || (size_t)pr.source >= b->clouds.size() || (size_t)pr.target >= b->clouds.size() || !b->clouds[pr.source] ||
        !b->clouds[pr.target])
      return fail(B2R_EINVAL, "pair names an unknown cloud id");
  }
  static const bool dbg = getenv("B2R_DEBUG_TIMING") != nullptr;
  const auto t_a = std::chrono::steady_clock::now();
  int rc = batch_sync_builds(b, false);  // the main stream waits for every outstanding upload / build
  if (rc) return rc;
  rc = batch_build_structures(b, pairs, n_pairs, !fit_only);
  if (rc) return rc;
  const auto t_b = std::chrono::steady_clock::now();
  const size_t chunk = std::min(b->max_chunk, std::max<size_t>(n_pairs, 1));
  rc = batch_host_staging(b, std::max(chunk, n_pairs));
  if (rc) return rc;
  B2R_CUDA(b->d_reports.reserve(n_pairs + 1));
  const LmCfg cfg = make_lm_cfg(h->cfg, want_fitness, fit_max_range);
  b->last_rounds = b->last_pair_rounds = 0;
  for (size_t c0 = 0; c0 < n_pairs; c0 += chunk) {
    const size_t m = std::min(chunk, n_pairs - c0);
    rc = batch_run_chunk(b, pairs + c0, m, cfg, b->d_reports.p + c0, fit_only);
    if (rc) return rc;
  }
  if (dbg) {
    const auto t_c = std::chrono::steady_clock::now();
    fprintf(stderr, "[b2r rank %d] batch_run: build enqueue %.3f ms, rounds (host follows the device) %.3f ms, %llu rounds\n", b->rank,
            std::chrono::duration<double, std::milli>(t_b - t_a).count(), std::chrono::duration<double, std::milli>(t_c - t_b).count(), b->last_rounds);
  }
  return B2R_OK;
}

extern "C" int b2r_batch_align(b2r_batch* b, const b2r_pair* pairs, size_t n_pairs, int want_fitness, double fitness_max_range, b2r_result* out) {
  if (!b || (n_pairs && (!pairs || !out))) return fail(B2R_EINVAL, "NULL argument");
  if (n_pairs == 0) return B2R_OK;
  int rc = batch_run(b, pairs, n_pairs, want_fitness != 0, fitness_max_range);
  if (rc) return rc;
  cudaStream_t st = b->eng->st;
  B2R_CUDA(cudaMemcpyAsync(b->h_reports, b->d_reports.p, n_pairs * sizeof(PairReport), cudaMemcpyDeviceToHost, st));
  B2R_CUDA(cudaStreamSynchronize(st));
  b->eng->tel.d2h += n_pairs * sizeof(PairReport);
  b->last_pair_rounds = 0;
  for (size_t i = 0; i < n_pairs; i++) {
    out[i] = b->h_reports[i].r;
    b->last_pair_rounds += (unsigned long long)b->h_reports[i].rounds;
    if (!want_fitness) out[i].fitness = NAN;
  }
  return B2R_OK;
}

// InformationMatrixCalculator::calc_fitness_score(cloud1, cloud2, relpose, max_range)
// (/root/reference/src/hdl_graph_slam/information_matrix_calculator.cpp:49-80; callers apps/hdl_graph_slam_nodelet.cpp:235,569):
// kd-tree on cloud1, cloud2 transformed by relpose.cast<float>(), mean of the squared NN distances <= max_range, DBL_MAX if none.
// Here for MANY edges at once, on the keyframes' cached search structures (pair.target = cloud1, pair.source = cloud2,
// pair.guess = relpose as float): one search + one reduction launch covers all of them.
extern "C" int b2r_batch_calc_fitness_score(b2r_batch* b, const b2r_pair* pairs, size_t n_pairs, double max_range, double* scores) {
  if (!b || (n_pairs && (!pairs || !scores))) return fail(B2R_EINVAL, "NULL argument");
  if (n_pairs == 0) return B2R_OK;
  int rc = batch_run(b, pairs, n_pairs, true, max_range, true);
  if (rc) return rc;
  cudaStream_t st = b->eng->st;
  B2R_CUDA(cudaMemcpyAsync(b->h_reports, b->d_reports.p, n_pairs * sizeof(PairReport), cudaMemcpyDeviceToHost, st));
  B2R_CUDA(cudaStreamSynchronize(st));
  b->eng->tel.d2h += n_pairs * sizeof(PairReport);
  for (size_t i = 0; i < n_pairs; i++) scores[i] = b->h_reports[i].r.fitness;
  return B2R_OK;
}

// InformationMatrixCalculator::calc_information_matrix's mapping from a fitness score to the edge information
// (information_matrix_calculator.cpp:25-47, weight(): information_matrix_calculator.hpp:39-42): inf = diag(1/w_x x3, 1/w_q x3)
extern "C" int b2r_information_params_default(b2r_information_params* p) {
  if (!p) return fail(B2R_EINVAL, "NULL argument");
  p->use_const_inf_matrix = 0; p->reserved = 0;
  p->const_stddev_x = 0.5; p->const_stddev_q = 0.1; p->var_gain_a = 20.0;
  p->min_stddev_x = 0.1; p->max_stddev_x = 5.0; p->min_stddev_q = 0.05; p->max_stddev_q = 0.2;
  p->fitness_score_thresh = 0.5;
  return B2R_OK;
}

extern "C" int b2r_information_from_fitness(const b2r_information_params* p, double fitness_score, double inf_diag[6]) {
  if (!p || !inf_diag) return fail(B2R_EINVAL, "NULL argument");
  double wx, wq;
  if (p->use_const_inf_matrix) {
    wx = p->const_stddev_x; wq = p->const_stddev_q;  // :26-31 (divides by the stddev itself, as the reference does)
  } else {
    auto weight = [](double a, double max_x, double min_y, double max_y, double x) {
      const double y = (1.0 - std::exp(-a * x)) / (1.0 - std::exp(-a * max_x));
      return min_y + (max_y - min_y) * y;
    };
    // float w_x = weight(...): the reference narrows the weights to float before dividing (:40-41)
    wx = (double)(float)weight(p->var_gain_a, p->fitness_score_thresh, p->min_stddev_x * p->min_stddev_x, p->max_stddev_x * p->max_stddev_x, fitness_score);
    wq = (double)(float)weight(p->var_gain_a, p->fitness_score_thresh, p->min_stddev_q * p->min_stddev_q, p->max_stddev_q * p->max_stddev_q, fitness_score);
  }
  for (int i = 0; i < 3; i++) { inf_diag[i] = 1.0 / wx; inf_diag[3 + i] = 1.0 / wq; }
  return B2R_OK;
}

extern "C" int b2r_batch_last_rounds(const b2r_batch* b, uint64_t* rounds, uint64_t* pair_rounds) {
  if (!b) return fail(B2R_EINVAL, "NULL argument");
  if (rounds) *rounds = b->last_rounds;
  if (pair_rounds) *pair_rounds = b->last_pair_rounds;
  return B2R_OK;
}

// LoopDetector::matching's selection (loop_detector.hpp:135-163) over one group's records: best converged fitness, a LATER
// candidate with an equal score replaces an earlier one (`score > best_score` skips), -1 if the best exceeds the threshold
extern "C" int b2r_loop_argmin(const b2r_result* results, size_t n, double fitness_score_thresh, int32_t* best) {
  if (!best || (n && !results)) return fail(B2R_EINVAL, "NULL argument");
  double best_score = DBL_MAX;
  int best_i = -1;
  for (size_t i = 0; i < n; i++) {
    const double score = results[i].fitness;
    if (!results[i].converged || score > best_score) continue;  // :147 (NaN scores compare false and are taken, as in the reference)
    best_score = score;
    best_i = (int)i;
  }
  if (best_score > fitness_score_thresh) best_i = -1;  // :160-163
  *best = best_i;
  return B2R_OK;
}

// ------------------------------------------------------------------------------------------------ multi-GPU (NCCL)
extern "C" int b2r_nccl_unique_id(void* out, size_t capacity) {
  if (!out || capacity < sizeof(ncclUniqueId)) return fail(B2R_EINVAL, "need a 128-byte buffer");
  ncclUniqueId id;
  B2R_NCCL(ncclGetUniqueId(&id));
  std::memcpy(out, &id, sizeof(id));
  return B2R_OK;
}

extern "C" int b2r_batch_comm_init(b2r_batch* b, const void* unique_id, int rank, int world) {
  if (!b || !unique_id || world < 1 || rank < 0 || rank >= world) return fail(B2R_EINVAL, "bad argument");
  B2R_CUDA(cudaSetDevice(b->eng->cfg.device_id));
  if (b->comm) { ncclCommDestroy(b->comm); b->comm = nullptr; }
  b->rank = rank; b->world = world;
  if (world == 1) return B2R_OK;
  ncclUniqueId id;
  std::memcpy(&id, unique_id, sizeof(id));
  B2R_NCCL(ncclCommInitRank(&b->comm, world, id, rank));
  return B2R_OK;
}

extern "C" int b2r_shard_range(size_t n_groups, int world, int rank, size_t* g0, size_t* g1) {
  if (!g0 || !g1 || world < 1 || rank < 0 || rank >= world) return fail(B2R_EINVAL, "bad argument");
  *g0 = n_groups * (size_t)rank / (size_t)world;   // contiguous blocks: neighbouring groups share candidate keyframes,
  *g1 = n_groups * (size_t)(rank + 1) / (size_t)world;  // so a keyframe's structures are built on one GPU only
  return B2R_OK;
}

extern "C" int b2r_batch_loop_detect(b2r_batch* b, const b2r_pair* pairs, size_t n_pairs, const int64_t* group_first, size_t n_groups,
                                     double fitness_score_max_range, double fitness_score_thresh, b2r_result* all_results, int32_t* best) {
  if (!b || !group_first || (n_pairs && (!pairs || !all_results)) || (n_groups && !best)) return fail(B2R_EINVAL, "NULL argument");
  if (group_first[0] != 0 || (size_t)group_first[n_groups] != n_pairs) return fail(B2R_EINVAL, "group_first must run from 0 to n_pairs");
  B2R_CUDA(cudaSetDevice(b->eng->cfg.device_id));
  cudaStream_t st = b->eng->st;
  // who owns what (every rank computes the whole map)
  size_t my_p0 = 0, my_p1 = 0, M = 0;
  std::vector<size_t> p0(b->world), p1(b->world);
  for (int r = 0; r < b->world; r++) {
    size_t g0, g1;
    b2r_shard_range(n_groups, b->world, r, &g0, &g1);
    p0[r] = (size_t)group_first[g0]; p1[r] = (size_t)group_first[g1];
    M = std::max(M, p1[r] - p0[r]);
  }
  my_p0 = p0[b->rank]; my_p1 = p1[b->rank];
  const size_t mine = my_p1 - my_p0;
  if (M == 0) { for (size_t g = 0; g < n_groups; g++) best[g] = -1; return B2R_OK; }
  static const bool dbg = getenv("B2R_DEBUG_TIMING") != nullptr;
  const auto t_a = std::chrono::steady_clock::now();
  int rc = mine ? batch_run(b, pairs + my_p0, mine, true, fitness_score_max_range) : B2R_OK;
  if (rc) return rc;
  if (dbg) cudaStreamSynchronize(st);
  const auto t_b = std::chrono::steady_clock::now();
  B2R_CUDA(b->d_send.reserve(M));
  B2R_CUDA(b->d_recv.reserve(M * (size_t)b->world));
  if (b->h_gather_cap < M * (size_t)b->world) {
    if (b->h_gather) cudaFreeHost(b->h_gather);
    b->h_gather = nullptr; b->h_gather_cap = 0;
    B2R_CUDA(cudaMallocHost(&b->h_gather, M * (size_t)b->world * sizeof(b2r_result)));
    b->h_gather_cap = M * (size_t)b->world;
  }
  B2R_CUDA(b->d_reports.reserve(1));
  b->h_word[b2r_batch::kLanes] = 0;
  k_pack_results<<<(unsigned)((M + 255) / 256), 256, 0, st>>>(b->d_reports.p, (int)mine, b->d_send.p, (int)M, b->h_word_dev + b2r_batch::kLanes);
  B2R_CUDA(cudaGetLastError());
  const b2r_result* gathered = b->d_send.p;
  if (b->world > 1) {
    if (!b->comm) return fail(B2R_ESTATE, "b2r_batch_comm_init has not been called");
    // the ONE data-plane collective of the batch: fixed 80-byte records, padded to the largest per-rank share
    B2R_NCCL(ncclAllGather(b->d_send.p, b->d_recv.p, M * sizeof(b2r_result), ncclChar, b->comm, st));
    gathered = b->d_recv.p;
  }
  B2R_CUDA(cudaMemcpyAsync(b->h_gather, gathered, M * (size_t)b->world * sizeof(b2r_result), cudaMemcpyDeviceToHost, st));
  B2R_CUDA(cudaStreamSynchronize(st));
  b->eng->tel.d2h += M * (size_t)b->world * sizeof(b2r_result);
  b->last_pair_rounds = b->h_word[b2r_batch::kLanes];  // exact: every pair's own round count (the stream has been synchronised)
  if (dbg) {
    const auto t_c = std::chrono::steady_clock::now();
    fprintf(stderr, "[b2r rank %d] loop_detect: batch_run + sync %.3f ms, pack + all-gather + readback %.3f ms\n", b->rank,
            std::chrono::duration<double, std::milli>(t_b - t_a).count(), std::chrono::duration<double, std::milli>(t_c - t_b).count());
  }
  for (int r = 0; r < b->world; r++)
    for (size_t i = p0[r]; i < p1[r]; i++) all_results[i] = b->h_gather[(size_t)r * M + (i - p0[r])];
  for (size_t g = 0; g < n_groups; g++) {
    rc = b2r_loop_argmin(all_results + group_first[g], (size_t)(group_first[g + 1] - group_first[g]), fitness_score_thresh, &best[g]);
    if (rc) return rc;
  }
  return B2R_OK;
}
