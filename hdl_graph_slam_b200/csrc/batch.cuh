// batch.cuh — host side of the batched registration path (included by api.cu after the handle and the build helpers).
//
//   b2r_batch            a keyframe-cloud cache + a pool of pair slots on ONE GPU; many (source, target) pairs per launch
//   b2r_batch_add_cloud  <- KeyFrame::cloud becoming known to the loop detector (keyframe.hpp:40): uploaded ONCE, its search
//                           structure and GICP covariances are built once and reused by every pair that names it (the reference
//                           rebuilds kd-tree + covariances at every setInputSource/Target: loop_detector.hpp:122,136)
//   b2r_batch_align      <- the candidate loop of LoopDetector::matching (loop_detector.hpp:135-154): align + getFitnessScore
//   b2r_batch_loop_detect<- LoopDetector::matching for MANY new keyframes, groups sharded over the ranks of an NCCL communicator,
//                           ONE ncclAllGather of 80-byte b2r_result records, per-group argmin with the reference's tie rule (:147,160)
// A GICP batch runs the device-resident LM engine (pair_engine.cuh).  An NDT batch (the factory's default NDT_OMP, which the
// loop detector builds its registration with) runs every pair's host Newton / More-Thuente driver (NdtPairState, ndt.cuh) in
// rounds: one batched derivative pass per pass kind covers every pair in flight, the host waits once per round.
#pragma once
#include <nccl.h>
#include <chrono>

struct b2r_batch {
  struct EngineDeleter { void operator()(b2r_handle* h) const { b2r_destroy(h); } };
  // engine context of this device: config, main stream, telemetry.  Declared first: destroyed after everything below
  std::unique_ptr<b2r_handle, EngineDeleter> eng;
  static constexpr int kBuildStreams = 4;
  Stream bst[kBuildStreams];
  BuildCtx bctx[kBuildStreams];
  Event bev[kBuildStreams];
  int next_stream = 0;
  std::vector<std::unique_ptr<Cloud>> clouds;
  std::vector<int> free_ids;
  std::vector<std::unique_ptr<Cloud>> recycled;  // removed clouds keep their device buffers for the next add (no cudaMalloc churn per keyframe)
  // pair slots.  A chunk of pairs can be split over kLanes independent round sequences ("lanes"), each on its own stream, so that a
  // lane's search kernel (instruction-issue bound) runs beside the other lane's accumulate kernel and a lane's thin tail rounds
  // overlap the other's fat ones.  Two lanes did not beat one on 256 pairs x 64k points — the block
  // scheduler drains one kernel's grid before it starts the next stream's, so the overlap is confined to the tails; the default
  // is ONE lane (B2R_BATCH_LANES=2 enables the second).  Lane 0 runs on the engine's main stream.
  static constexpr int kLanes = 2;
  struct Lane {
    cudaStream_t st = nullptr;  // lane 0: the engine's main stream; the others: `own`
    Stream own;
    Event ev;
    DevBuf<PairDev> d_pairs;
    DevBuf<int> d_active;
    DevBuf<VgicpMapDev> d_vmaps;     // VGICP: the voxel map of each pair's target, indexed like d_pairs
    unsigned long long* h_word = nullptr;  // host-mapped: (seq << 32) | pairs still active
    unsigned long long* h_word_dev = nullptr;
    unsigned long long seq = 0;
  };
  Lane lane[kLanes];
  Event fork_ev;
  int n_lanes = 1;
  DevBuf<PairReport> d_reports;
  DevBuf<char> ws;
  PinnedBuf<PairDev> h_pairs;       // staging
  PinnedBuf<PairReport> h_reports;  // staging
  PinnedBuf<VgicpMapDev> h_vmaps;   // staging (VGICP)
  DevBuf<char> fit_ws;              // getFitnessScore after the rounds (batch_fitness): per pair the reduction partials, counter and sums
  DevBuf<FitItem> d_fit;            // getFitnessScore after the rounds: one record per pair of the call
  PinnedBuf<FitItem> h_fit;         // staging (filled once per call, so no chunk overwrites a record still being copied)
  MappedBuf<unsigned long long> h_word;  // [0..kLanes) = the lanes' words, [kLanes] = sum of the pairs' executed rounds
  size_t max_chunk = 1024;  // pairs in flight per launch sequence (~7.7 MB of workspace per 64k-point pair)
  int copies = 1;           // lanes per query of the batched 1-NN search
  // multi-GPU
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1;
  DevBuf<b2r_result> d_send, d_recv;
  DevBuf<BuildItem> d_build;        // descriptor list of the batched cluster builds
  PinnedBuf<BuildItem> h_build;     // staging
  DevBuf<KnnBatchItem> d_knn;       // descriptor list of one batched k-NN covariance launch
  PinnedBuf<KnnBatchItem> h_knn;    // staging
  PinnedBuf<b2r_result> h_gather;
  // host-driven methods (NDT, pcl GICP, pcl ICP: batch_run_*_chunk).  A batch serves one method, so they share the workspace
  DevBuf<char> method_ws;           // per pair in flight: ndt_pair_ws, gicp_pcl_pair_ws or icp_pair_ws
  // the round channel of the NDT and pcl GICP rounds (batch_round_channel)
  MappedBuf<double> h_msg;          // one result message per record of the round, then the round's flag (8 doubles)
  DevBuf<unsigned int> d_round;     // messages of the current round (the last one publishes the flag and re-arms it)
  unsigned long long msg_seq = 0;
  // NDT batch (batch_run_ndt_chunk)
  DevBuf<NdtArgs> d_ndt_args;       // the round's pass records, grouped by pass kind
  PinnedBuf<NdtArgs> h_ndt_args;    // staging
  DevBuf<NdtPclArgs> d_pcl_args;    // the same records with the radius-search inputs (B2R_METHOD_NDT_PCL, _NDT_KDTREE)
  PinnedBuf<NdtPclArgs> h_pcl_args;
  // pcl GICP batch (batch_run_gicp_pcl_chunk)
  DevBuf<GicpPclArgs> d_gp_args;    // the round's pass records: correspondence passes first, then cost passes
  PinnedBuf<GicpPclArgs> h_gp_args; // staging
  // pcl ICP batch (batch_run_icp_chunk)
  DevBuf<IcpPairDev> d_icp;         // the pair records
  PinnedBuf<IcpPairDev> h_icp;      // their host copies
  // telemetry of the last b2r_batch_align
  unsigned long long last_rounds = 0, last_pair_rounds = 0;
  ~b2r_batch() {  // what is not a plain free; the members then go in reverse order, the engine last
    if (!eng) return;
    cudaSetDevice(eng->cfg.device_id);
    cudaStreamSynchronize(eng->st);
    for (const Stream& s : bst) if (s) cudaStreamSynchronize(s);
    for (const Lane& L : lane) if (L.st) cudaStreamSynchronize(L.st);
    if (comm) ncclCommDestroy(comm);  // before the send / receive buffers go
  }
};

#define B2R_NCCL(expr)                                                                                     \
  do {                                                                                                     \
    ncclResult_t _r = (expr);                                                                              \
    if (_r != ncclSuccess) return b2r::fail(B2R_ENCCL, std::string(#expr) + ": " + ncclGetErrorString(_r)); \
  } while (0)

extern "C" void b2r_batch_destroy(b2r_batch* b) { delete b; }

extern "C" int b2r_batch_create(const b2r_config* cfg, b2r_batch** out) {
  if (!cfg || !out) return fail(B2R_EINVAL, "NULL argument");
  *out = nullptr;
  if (!known_method(cfg->method)) return fail(B2R_EINVAL, "unknown method");
  std::unique_ptr<b2r_batch> b(new b2r_batch());
  b2r_handle* eng = nullptr;
  int rc = b2r_create(cfg, &eng);
  if (rc) return rc;
  b->eng.reset(eng);
  for (int i = 0; i < b2r_batch::kBuildStreams; i++) {
    if (b->bst[i].create(cudaStreamNonBlocking) != cudaSuccess || b->bev[i].create() != cudaSuccess || b->bctx[i].mm.alloc(8) != cudaSuccess)
      return fail(B2R_ECUDA, "stream / scratch creation failed");
  }
  if (b->h_word.alloc(8) != cudaSuccess) return fail(B2R_ECUDA, "host allocation failed");
  for (int i = 0; i < 8; i++) b->h_word.p[i] = 0;
  if (b->fork_ev.create() != cudaSuccess) return fail(B2R_ECUDA, "event creation failed");
  if (b->d_round.alloc(1) != cudaSuccess || cudaMemset(b->d_round.p, 0, sizeof(unsigned int)) != cudaSuccess)
    return fail(B2R_ECUDA, "device allocation failed");
  for (int l = 0; l < b2r_batch::kLanes; l++) {
    b2r_batch::Lane& L = b->lane[l];
    L.h_word = b->h_word.p + l; L.h_word_dev = b->h_word.d + l;
    if (l == 0) L.st = b->eng->st;
    else if (L.own.create(cudaStreamNonBlocking) != cudaSuccess) return fail(B2R_ECUDA, "stream creation failed");
    else L.st = L.own;
    if (L.ev.create() != cudaSuccess) return fail(B2R_ECUDA, "event creation failed");
  }
  if (const char* e = getenv("B2R_BATCH_LANES")) { const int c = atoi(e); if (c >= 1 && c <= b2r_batch::kLanes) b->n_lanes = c; }
  if (const char* e = getenv("B2R_BATCH_COPIES")) { const int c = atoi(e); if (c == 1 || c == 2 || c == 4) b->copies = c; }
  if (const char* e = getenv("B2R_BATCH_CHUNK")) { const long c = atol(e); if (c > 0) b->max_chunk = (size_t)c; }
  *out = b.release();
  return B2R_OK;
}

extern "C" int b2r_batch_get_engine(b2r_batch* b, b2r_handle** out) {
  if (!b || !out) return fail(B2R_EINVAL, "NULL argument");
  *out = b->eng.get();
  return B2R_OK;
}

static int batch_add(b2r_batch* b, const void* pts, size_t n, size_t stride_bytes, bool device_ptr, int32_t* id_out) {
  if (!b || !id_out) return fail(B2R_EINVAL, "NULL argument");
  if (stride_bytes < 12 || (stride_bytes & 3)) return fail(B2R_EINVAL, "stride_bytes must be a multiple of 4 and >= 12");
  if (n > 0 && !pts) return fail(B2R_EINVAL, "points is NULL");
  if (n > (size_t)0x3fffffff) return fail(B2R_EINVAL, "too many points");
  B2R_CUDA(cudaSetDevice(b->eng->cfg.device_id));
  std::unique_ptr<Cloud> c;
  if (!b->recycled.empty()) { c = std::move(b->recycled.back()); b->recycled.pop_back(); c->invalidate(); }
  else c.reset(new Cloud());
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
    if (e != cudaSuccess) return fail(B2R_ECUDA, std::string("device allocation failed: ") + cudaGetErrorString(e));
    c->raw_view = c->raw.p;
    if (n) {
      // pinned buffers are DMA'd in place (asynchronously: see b200reg.h for the lifetime rule); pageable ones are staged by the driver
      e = cudaMemcpyAsync(c->raw.p, pts, n * stride_bytes, cudaMemcpyHostToDevice, st);
      if (e != cudaSuccess) return fail(B2R_ECUDA, std::string("upload failed: ") + cudaGetErrorString(e));
      b->eng->tel.h2d += n * stride_bytes;
    }
  }
  // the upload is all that happens here (4 copy streams); the search structures and k-NN covariances of ALL new clouds are built
  // together at the next align: one cluster-build launch per cluster size and one k-NN launch (batch_build_structures)
  int id;
  if (!b->free_ids.empty()) { id = b->free_ids.back(); b->free_ids.pop_back(); b->clouds[id] = std::move(c); }
  else { id = (int)b->clouds.size(); b->clouds.push_back(std::move(c)); }
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
  b->recycled.push_back(std::move(b->clouds[id]));
  b->free_ids.push_back(id);
  return B2R_OK;
}

extern "C" int b2r_batch_cloud_count(const b2r_batch* b) {
  if (!b) return 0;
  return (int)(b->clouds.size() - b->free_ids.size());
}

// Search structure (bvh_build.cuh) + FastGICP::calculate_covariances (need_cov) for every cloud of ids[0..n_ids) (known ids, in
// any order, repeats allowed) that does not have them yet: one cluster-build launch per cluster size and one k-NN launch for all of
// them (what setInputSource / setInputTarget make the reference pay per call: kd-tree build + covariances, loop_detector.hpp:122,136)
static int batch_build_structures(b2r_batch* b, const int32_t* ids, size_t n_ids, bool need_cov) {
  b2r_handle* h = b->eng.get();
  cudaStream_t st = h->st;
  std::vector<Cloud*> todo;
  std::vector<char> queued(b->clouds.size(), 0);
  for (size_t i = 0; i < n_ids; i++) {
    const int32_t id = ids[i];
    Cloud* c = b->clouds[id].get();
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
      if (b->h_build.cap < total) B2R_CUDA(b->h_build.alloc(total + 64));
      size_t k0 = 0;
      for (int g = 0; g < kBuildShapes; g++)
        for (Cloud* c : by_cl[g]) b->h_build.p[k0++] = build_item(*c);
      B2R_CUDA(cudaMemcpyAsync(b->d_build.p, b->h_build.p, total * sizeof(BuildItem), cudaMemcpyHostToDevice, st));
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
  if (b->h_knn.cap < todo.size()) B2R_CUDA(b->h_knn.alloc(todo.size() + 64));
  unsigned max_blocks = 0;
  for (size_t i = 0; i < todo.size(); i++) {
    Cloud* c = todo[i];
    KnnBatchItem& it = b->h_knn.p[i];
    it.b = c->bvh(); it.raw = c->raw_view; it.cov = c->cov.p; it.stride_f = c->stride_f; it.pad = 0;
    max_blocks = std::max(max_blocks, (unsigned)((size_t)c->nsup * 1024 / kKnnThreads));
  }
  B2R_CUDA(cudaMemcpyAsync(b->d_knn.p, b->h_knn.p, todo.size() * sizeof(KnnBatchItem), cudaMemcpyHostToDevice, st));
  { TEL_BEGIN(&h->tel, st);
    if (gicp_pcl_family(h->cfg.method))  // pcl GICP's raw-moment covariances (gicp_pcl.cuh)
      k_pcl_cov_reg_batch<kKnnRegK, PclCov><<<dim3(max_blocks, (unsigned)todo.size()), kKnnThreads, 0, st>>>(b->d_knn.p);
    else if (h->cfg.method == B2R_METHOD_VGICP_CUDA)  // FastVGICPCuda's float32 raw-moment covariances (vgicp_cuda.cuh)
      k_pcl_cov_reg_batch<kKnnRegK, VcudaCov><<<dim3(max_blocks, (unsigned)todo.size()), kKnnThreads, 0, st>>>(b->d_knn.p);
    else
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
  if (b->h_pairs.cap >= n && b->h_reports.cap >= n && b->h_vmaps.cap >= n) return B2R_OK;
  const size_t want = n + n / 4 + 16;
  B2R_CUDA(b->h_pairs.alloc(want));
  B2R_CUDA(b->h_reports.alloc(want));
  B2R_CUDA(b->h_vmaps.alloc(want));
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
  b2r_handle* h = b->eng.get();
  cudaStream_t st = h->st;
  const bool vgicp = vgicp_family(h->cfg.method) && !fit_only;  // a stand-alone fitness evaluation runs the GICP search
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
    if (vgicp) B2R_CUDA(L.d_vmaps.reserve(R.m));
    for (size_t i = R.i0; i < R.i0 + R.m; i++) {
      PairDev& P = b->h_pairs.p[i];
      const Cloud& s = *b->clouds[pairs[i].source];
      const Cloud& t = *b->clouds[pairs[i].target];
      if (s.n == 0 || t.n == 0) {
        std::memset(&P, 0, sizeof(P));
        P.mode = PM_DONE;
        degenerate_report(b->h_reports.p[i], pairs[i].guess);
        B2R_CUDA(cudaMemcpyAsync(d_rep + i, &b->h_reports.p[i], sizeof(PairReport), cudaMemcpyHostToDevice, L.st));
        continue;
      }
      fill_pair_geometry(P, s, t);
      if (vgicp) b->h_vmaps.p[i] = t.vgicp->desc;
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
    B2R_CUDA(cudaMemcpyAsync(L.d_pairs.p, b->h_pairs.p + R.i0, R.m * sizeof(PairDev), cudaMemcpyHostToDevice, L.st));
    h->tel.h2d += R.m * sizeof(PairDev);
    if (vgicp) {
      B2R_CUDA(cudaMemcpyAsync(L.d_vmaps.p, b->h_vmaps.p + R.i0, R.m * sizeof(VgicpMapDev), cudaMemcpyHostToDevice, L.st));
      h->tel.h2d += R.m * sizeof(VgicpMapDev);
    }
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
      int rc = launch_round(L.d_pairs.p, L.d_active.p, (unsigned)R.known, (unsigned)R.max_pad, b->copies, cfg, L.st, &h->tel, true,
                            vgicp ? L.d_vmaps.p : nullptr, h->cfg.method == B2R_METHOD_VGICP_CUDA);
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

// ------------------------------------------------------------------------------------------------ VGICP batch
// The voxel map of every cloud a call aligns to (the first use of a keyframe as a target builds it; it stays with the cloud).
static int batch_vgicp_maps(b2r_batch* b, const b2r_pair* pairs, size_t n_pairs) {
  b2r_handle* h = b->eng.get();
  for (size_t i = 0; i < n_pairs; i++) {
    Cloud& t = *b->clouds[pairs[i].target];
    if (t.n == 0 || t.vgicp_ready) continue;
    int rc = vgicp_map_of(h, t);
    if (rc) return rc;
  }
  return B2R_OK;
}

// getFitnessScore at the final pose of every pair of the call (reports d_rep[0..m) on the device): one k_fitness_batch launch covers
// every pair with the kernel, grid and reduction of b2r_fitness, so each score is bitwise b2r_fitness's; no host round trip.
static int batch_fitness(b2r_batch* b, const b2r_pair* pairs, size_t m, double fit_max_range, PairReport* d_rep) {
  b2r_handle* h = b->eng.get();
  cudaStream_t st = h->st;
  std::vector<size_t> live, off;
  size_t ws = 0;
  unsigned max_nb = 0;
  for (size_t i = 0; i < m; i++) {
    const Cloud& s = *b->clouds[pairs[i].source];
    const Cloud& t = *b->clouds[pairs[i].target];
    if (s.n == 0 || t.n == 0) continue;  // degenerate_report / method_report: DBL_MAX already
    const size_t nb = (size_t)s.nsup * 1024 / kLinThreads;
    live.push_back(i);
    off.push_back(ws);
    ws += align_up(nb * 3 * sizeof(double), 256) + 256;  // partials, then counter [0, 16) and the three sums [64, 88)
    max_nb = std::max(max_nb, (unsigned)nb);
  }
  if (live.empty()) return B2R_OK;
  B2R_CUDA(b->fit_ws.reserve(ws + 256));
  B2R_CUDA(b->d_fit.reserve(live.size()));
  if (b->h_fit.cap < live.size()) B2R_CUDA(b->h_fit.alloc(live.size() + live.size() / 4 + 16));
  char* base = reinterpret_cast<char*>(align_up(reinterpret_cast<size_t>(b->fit_ws.p), 256));
  B2R_CUDA(cudaMemsetAsync(base, 0, ws, st));  // the reduction counters start at zero (and re-arm themselves)
  for (size_t k = 0; k < live.size(); k++) {
    const size_t i = live[k];
    const Cloud& s = *b->clouds[pairs[i].source];
    const Cloud& t = *b->clouds[pairs[i].target];
    const size_t nb = (size_t)s.nsup * 1024 / kLinThreads;
    FitItem& it = b->h_fit.p[k];
    std::memset(&it, 0, sizeof(it));
    it.A.src = s.bvh(); it.A.tgt = t.bvh();
    it.A.max_range = fit_max_range; it.A.inlier_thresh_sq = 0.25f;
    char* p = base + off[k];
    it.A.partials = reinterpret_cast<double*>(p);
    it.A.counter = reinterpret_cast<unsigned int*>(p + align_up(nb * 3 * sizeof(double), 256));
    it.A.out = reinterpret_cast<double*>(p + align_up(nb * 3 * sizeof(double), 256) + 64);
    it.rep = d_rep + i;
    it.nblk = (unsigned)nb;
  }
  B2R_CUDA(cudaMemcpyAsync(b->d_fit.p, b->h_fit.p, live.size() * sizeof(FitItem), cudaMemcpyHostToDevice, st));
  h->tel.h2d += live.size() * sizeof(FitItem);
  for (size_t k0 = 0; k0 < live.size(); k0 += 65535) {  // grid.y limit
    const unsigned ny = (unsigned)std::min<size_t>(65535, live.size() - k0);
    TEL_BEGIN(&h->tel, st);
    k_fitness_batch<<<dim3(max_nb, ny), kLinThreads, 0, st>>>(b->d_fit.p + k0);
    TEL_END(&h->tel, KC_FITNESS, 1, st);
    B2R_CUDA(cudaGetLastError());
  }
  k_fitness_batch_store<<<(unsigned)((live.size() + 255) / 256), 256, 0, st>>>(b->d_fit.p, (int)live.size());
  B2R_CUDA(cudaGetLastError());
  return B2R_OK;
}

// ------------------------------------------------------------------------------------------------ NDT batch
// Voxel maps of the clouds a call names: every align target, and every cloud added from device memory (its records are the
// caller's only until this call returns, so the map is built now even if the cloud is a target only later).
static int batch_ndt_maps(b2r_batch* b, const b2r_pair* pairs, size_t n_pairs, bool fit_only) {
  b2r_handle* h = b->eng.get();
  for (size_t i = 0; i < n_pairs; i++) {
    for (int side = 0; side < 2; side++) {
      Cloud& c = *b->clouds[side ? pairs[i].target : pairs[i].source];
      const bool device_added = c.raw_view != c.raw.p;
      if (c.n == 0 || c.ndt_ready || !(device_added || (side == 1 && !fit_only))) continue;
      int rc = ndt_ensure_map(h->cfg, c, h->ndt_work, h->st);
      if (rc) return rc;
    }
  }
  return B2R_OK;
}

// The report of a pair of a host-driven method: T_row is the registration's pose (row-major), or nullptr for a pair that never
// started, which reports the caller's guess exactly as given.  With want_fitness the score is DBL_MAX until batch_fitness, which
// runs after the rounds, overwrites it for every pair with points on both sides.
static void method_report(PairReport& R, const float* T_row, const float* guess_col, bool converged, int iterations, int rounds,
                          bool want_fitness) {
  std::memset(&R, 0, sizeof(R));
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) R.r.T[c * 4 + r] = T_row ? T_row[r * 4 + c] : guess_col[c * 4 + r];
  R.r.fitness = want_fitness ? DBL_MAX : NAN;
  R.r.converged = converged ? 1 : 0;
  R.r.iterations = iterations;
  R.rounds = rounds;
}

constexpr int kRoundMsg = 48;  // doubles per result message: kNdtAcc sums (or 36 Hessian entries, or kGicpPclSums), pair count, checksum

// The round channel of the NDT and pcl GICP rounds, sized for m messages: the flag behind the last message (host and device address)
static int batch_round_channel(b2r_batch* b, size_t m, unsigned long long** flag, unsigned long long** flag_dev) {
  if (b->h_msg.cap < m * kRoundMsg + 8) {
    B2R_CUDA(b->h_msg.alloc(m * kRoundMsg + 8));
    std::memset(b->h_msg.p, 0, b->h_msg.cap * sizeof(double));
  }
  const size_t flag_at = b->h_msg.cap - 8;  // behind the last message the buffer holds
  *flag = reinterpret_cast<unsigned long long*>(b->h_msg.p + flag_at);
  *flag_dev = reinterpret_cast<unsigned long long*>(b->h_msg.d + flag_at);
  return B2R_OK;
}

// per pair in flight: [chunks + 1][kNdtAcc] chunk rows (also the Hessian pass's [blocks][36]), [groups][kNdtAcc] group rows,
// group counters, then counter / pair count / ticket counter — all zero at the start of a chunk of pairs
struct NdtPairWs { size_t partials, grows, gcount, small, bytes; };
static NdtPairWs ndt_pair_ws(const Cloud& s) {
  const size_t nb = (size_t)s.nsup * 1024 / kNdtThreads, ng = (nb + 31) / 32;
  NdtPairWs w;
  w.partials = 0;
  w.grows = align_up((nb + 1) * kNdtAcc * sizeof(double), 256);
  w.gcount = w.grows + align_up(ng * kNdtAcc * sizeof(double), 256);
  w.small = w.gcount + align_up(ng * sizeof(unsigned int), 256);
  w.bytes = w.small + 256;  // [0,16) counter, [16,24) pair count, [24,32) ticket counter
  return w;
}

// pairs[0..m) of an NDT batch -> rep[0..m) (host).  Every pair runs ndt_align's driver (NdtPairState); a round gathers the pass
// each active pair asks for into at most three launches (derivatives with Hessian, without, float64 Hessian only), waits once for
// the round's flag and hands every pair its result.  A pair reduces through its own rows and counters, exactly as alone.
static int batch_run_ndt_chunk(b2r_batch* b, const b2r_pair* pairs, size_t m, bool want_fitness, PairReport* rep) {
  b2r_handle* h = b->eng.get();
  cudaStream_t st = h->st;
  const b2r_config& cfg = h->cfg;
  // pcl::NormalDistributionsTransform: the Hessian-only pass is the derivative pass with the Hessian (ndt_run_pass).  NDT_OMP's KDTREE
  // runs its own three kernels; both read the radius-search records
  const bool pcl = cfg.method == B2R_METHOD_NDT_PCL;
  const bool kd = cfg.method == B2R_METHOD_NDT_KDTREE;
  const bool radius = pcl || kd;
  auto kind_of_pass = [&](int k) { return (pcl && k == NDT_PASS_HESS) ? (int)NDT_PASS_DERIV_HESS : k; };
  std::vector<NdtPairState> S(m);
  std::vector<size_t> active, off(m, 0);
  size_t ws = 0;
  for (size_t i = 0; i < m; i++) {
    Cloud& s = *b->clouds[pairs[i].source];
    Cloud& t = *b->clouds[pairs[i].target];
    if (s.n == 0 || t.n == 0) continue;  // ndt_align: initCompute fails silently (identity, not converged, no iteration)
    int rc = ndt_sync_geom(*t.ndt, h->ndt_work, st);
    if (rc) return rc;
    if (t.ndt->h_geom.empty) continue;  // no finite target point: as above
    S[i].start(cfg, pairs[i].guess);
    active.push_back(i);
    off[i] = ws;
    ws += ndt_pair_ws(s).bytes;
  }
  B2R_CUDA(b->method_ws.reserve(ws + 256));
  char* base = reinterpret_cast<char*>(align_up(reinterpret_cast<size_t>(b->method_ws.p), 256));
  B2R_CUDA(cudaMemsetAsync(base, 0, ws, st));
  B2R_CUDA(b->d_ndt_args.reserve(m));
  B2R_CUDA(b->h_ndt_args.alloc(m));
  if (radius) { B2R_CUDA(b->d_pcl_args.reserve(m)); B2R_CUDA(b->h_pcl_args.alloc(m)); }
  unsigned long long *flag, *flag_dev;
  int rc = batch_round_channel(b, m, &flag, &flag_dev);
  if (rc) return rc;
  std::vector<unsigned long long> qnext(m, 0);
  std::vector<size_t> order;
  std::vector<int> kind_of;
  while (!active.empty()) {
    order.clear(); kind_of.clear();
    size_t cnt[3] = {0, 0, 0};
    unsigned max_nb[3] = {0, 0, 0};
    for (int k = 0; k < 3; k++)
      for (size_t i : active)
        if (S[i].next() != NDT_PASS_DONE && kind_of_pass(S[i].next()) == k) {
          order.push_back(i); kind_of.push_back(k); cnt[k]++;
          max_nb[k] = std::max(max_nb[k], (unsigned)((size_t)b->clouds[pairs[i].source]->nsup * 1024 / kNdtThreads));
        }
    // blocks per pair of a derivative launch: about four waves of the device, and no more than the largest pair has chunks; a
    // pair's blocks draw its chunks from its own ticket counter, so any count gives the same sums
    unsigned G[3] = {0, 0, 0};
    for (int k = 0; k < 2; k++)
      if (cnt[k]) {
        const unsigned res = pcl ? ndt_pcl_resident_blocks(k == 0) : kd ? ndt_kdtree_resident_blocks(k == 0) : ndt_resident_blocks(k == 0);
        G[k] = std::max(1u, std::min(max_nb[k], (unsigned)((4ull * res + cnt[k] - 1) / cnt[k])));
      }
    G[2] = max_nb[2];
    const unsigned long long seq = ++b->msg_seq;
    for (size_t r = 0; r < order.size(); r++) {
      const size_t i = order[r];
      const int k = kind_of[r];
      Cloud& s = *b->clouds[pairs[i].source];
      Cloud& t = *b->clouds[pairs[i].target];
      NdtArgs& A = b->h_ndt_args.p[r];
      ndt_fill_args(cfg, s, t, S[i].K, S[i].Tfinal, k != NDT_PASS_DERIV, A);
      const NdtPairWs w = ndt_pair_ws(s);
      char* p = base + off[i];
      A.partials = reinterpret_cast<double*>(p + w.partials);
      A.grows = reinterpret_cast<double*>(p + w.grows);
      A.gcount = reinterpret_cast<unsigned int*>(p + w.gcount);
      A.counter = reinterpret_cast<unsigned int*>(p + w.small);
      A.pairs = reinterpret_cast<unsigned long long*>(p + w.small + 16);
      A.queue = reinterpret_cast<unsigned long long*>(p + w.small + 24);
      A.qbase = qnext[i];
      if (k != NDT_PASS_HESS) qnext[i] += (unsigned long long)(s.nsup * 1024 / kNdtThreads) + G[k];  // chunks + one closing draw per block
      A.out = b->h_msg.d + r * kRoundMsg;
      A.flag = flag_dev;
      A.seq = seq;
      A.round = b->d_round.p;
      A.round_n = (unsigned)order.size();
      if (radius) ndt_pcl_fill_args(cfg, t, A, b->h_pcl_args.p[r]);
    }
    if (radius) {
      B2R_CUDA(cudaMemcpyAsync(b->d_pcl_args.p, b->h_pcl_args.p, order.size() * sizeof(NdtPclArgs), cudaMemcpyHostToDevice, st));
      h->tel.h2d += order.size() * sizeof(NdtPclArgs);
    } else {
      B2R_CUDA(cudaMemcpyAsync(b->d_ndt_args.p, b->h_ndt_args.p, order.size() * sizeof(NdtArgs), cudaMemcpyHostToDevice, st));
      h->tel.h2d += order.size() * sizeof(NdtArgs);
    }
    size_t r0 = 0;
    for (int k = 0; k < 3; k++) {
      if (!cnt[k]) continue;
      const dim3 grid(G[k], (unsigned)cnt[k]);
      TEL_BEGIN(&h->tel, st);
      if (pcl && k == NDT_PASS_DERIV_HESS) k_ndt_pcl_derivatives_batch<true><<<grid, kNdtThreads, 0, st>>>(b->d_pcl_args.p + r0);
      else if (pcl) k_ndt_pcl_derivatives_batch<false><<<grid, kNdtThreads, 0, st>>>(b->d_pcl_args.p + r0);
      else if (kd && k == NDT_PASS_DERIV_HESS) k_ndt_kdtree_derivatives_batch<true><<<grid, kNdtThreads, 0, st>>>(b->d_pcl_args.p + r0);
      else if (kd && k == NDT_PASS_DERIV) k_ndt_kdtree_derivatives_batch<false><<<grid, kNdtThreads, 0, st>>>(b->d_pcl_args.p + r0);
      else if (kd) k_ndt_kdtree_hessian_batch<<<grid, kNdtThreads, 0, st>>>(b->d_pcl_args.p + r0);
      else if (k == NDT_PASS_DERIV_HESS) k_ndt_derivatives_batch<true><<<grid, kNdtThreads, 0, st>>>(b->d_ndt_args.p + r0);
      else if (k == NDT_PASS_DERIV) k_ndt_derivatives_batch<false><<<grid, kNdtThreads, 0, st>>>(b->d_ndt_args.p + r0);
      else k_ndt_hessian_batch<<<grid, kNdtThreads, 0, st>>>(b->d_ndt_args.p + r0);
      TEL_END(&h->tel, k == NDT_PASS_HESS ? KC_NDT_HESS : KC_NDT_DERIV, 1, st);
      B2R_CUDA(cudaGetLastError());
      r0 += cnt[k];
    }
    h->tel.d2h += order.size() * kRoundMsg * sizeof(double);
    b->last_rounds++;
    for (size_t r = 0; r < order.size(); r++) {  // the first wait covers the round; the rest only check each message
      const int k = kind_of[r];
      const double* msg = b->h_msg.p + r * kRoundMsg;
      rc = (k == NDT_PASS_HESS) ? wait_host_result(flag, seq, msg, 36, false, st) : wait_host_result(flag, seq, msg, kNdtAcc, true, st);
      if (rc) return rc;
      NdtPass P;
      ndt_read_pass(msg, k != NDT_PASS_DERIV, k == NDT_PASS_HESS, &P);
      S[order[r]].consume(P);
    }
    size_t keep = 0;
    for (size_t i : active)
      if (S[i].next() != NDT_PASS_DONE) active[keep++] = i;
    active.resize(keep);
  }
  for (size_t i = 0; i < m; i++)  // a pair that never started reports NdtPairState's identity
    method_report(rep[i], S[i].Tfinal, nullptr, S[i].converged, S[i].nr_iterations, S[i].passes, want_fitness);
  return B2R_OK;
}

// per pair in flight: correspondences [n_pad] ints, M [n_pad][9], reduction partials [blocks][13], then the counter — zero at the start
struct GicpPclPairWs { size_t corr, M, partials, counter, bytes; };
static GicpPclPairWs gicp_pcl_pair_ws(const Cloud& s) {
  const size_t n = (size_t)s.nsup * 1024, nb = n / kGicpPclThreads;
  GicpPclPairWs w;
  w.corr = 0;
  w.M = align_up(n * sizeof(int), 256);
  w.partials = w.M + align_up(n * 9 * sizeof(double), 256);
  w.counter = w.partials + align_up(nb * kGicpPclSums * sizeof(double), 256);
  w.bytes = w.counter + 256;
  return w;
}

// pairs[0..m) of a pcl GICP batch -> rep[0..m) (host).  Every pair runs the single handle's GicpPclPairState; a round gathers the
// pass each active pair asks for into at most two launches (correspondence passes, cost passes; blockIdx.y = pair), waits once for
// the round's flag and hands every pair its result.  A pair reduces through its own partials and counter, exactly as alone.
static int batch_run_gicp_pcl_chunk(b2r_batch* b, const b2r_pair* pairs, size_t m, bool want_fitness, PairReport* rep) {
  b2r_handle* h = b->eng.get();
  cudaStream_t st = h->st;
  const b2r_config& cfg = h->cfg;
  std::vector<GicpPclPairState> S(m);
  std::vector<char> started(m, 0);
  std::vector<size_t> active, off(m, 0);
  size_t ws = 0;
  for (size_t i = 0; i < m; i++) {
    Cloud& s = *b->clouds[pairs[i].source];
    Cloud& t = *b->clouds[pairs[i].target];
    if (s.n == 0 || t.n == 0) continue;  // initCompute fails: the guess, not converged, no iteration (as gicp_pcl_align)
    float G[16];
    colmajor_to_row_f(pairs[i].guess, G);
    S[i].start(cfg, G);
    started[i] = 1;
    active.push_back(i);
    off[i] = ws;
    ws += gicp_pcl_pair_ws(s).bytes;
  }
  B2R_CUDA(b->method_ws.reserve(ws + 256));
  char* base = reinterpret_cast<char*>(align_up(reinterpret_cast<size_t>(b->method_ws.p), 256));
  B2R_CUDA(cudaMemsetAsync(base, 0, ws, st));
  B2R_CUDA(b->d_gp_args.reserve(m));
  if (b->h_gp_args.cap < m) B2R_CUDA(b->h_gp_args.alloc(m));
  unsigned long long *flag, *flag_dev;
  int rc = batch_round_channel(b, m, &flag, &flag_dev);
  if (rc) return rc;
  std::vector<size_t> order;
  std::vector<int> kind_of;
  while (!active.empty()) {
    order.clear(); kind_of.clear();
    size_t cnt[2] = {0, 0};
    unsigned max_nb[2] = {0, 0};
    for (int k = 0; k < 2; k++)
      for (size_t i : active)
        if ((S[i].next() == GicpPclPairState::CORR) == (k == 0)) {
          order.push_back(i); kind_of.push_back(k); cnt[k]++;
          max_nb[k] = std::max(max_nb[k], (unsigned)((size_t)b->clouds[pairs[i].source]->nsup * 1024 / kGicpPclThreads));
        }
    const unsigned long long seq = ++b->msg_seq;
    for (size_t r = 0; r < order.size(); r++) {
      const size_t i = order[r];
      Cloud& s = *b->clouds[pairs[i].source];
      Cloud& t = *b->clouds[pairs[i].target];
      const GicpPclPairWs w = gicp_pcl_pair_ws(s);
      char* p = base + off[i];
      double R[9];
      S[i].rel_rotation(R);
      GicpPclArgs& A = b->h_gp_args.p[r];
      gicp_pcl_fill_args(cfg, s, t, S[i].guess(), S[i].T(), R, reinterpret_cast<int*>(p + w.corr), reinterpret_cast<double*>(p + w.M), A);
      A.partials = reinterpret_cast<double*>(p + w.partials);
      A.counter = reinterpret_cast<unsigned int*>(p + w.counter);
      A.out = b->h_msg.d + r * kRoundMsg;
      A.flag = flag_dev;
      A.seq = seq;
      A.round = b->d_round.p;
      A.round_n = (unsigned)order.size();
      A.nrow = (unsigned)((size_t)s.nsup * 1024 / kGicpPclThreads);
    }
    B2R_CUDA(cudaMemcpyAsync(b->d_gp_args.p, b->h_gp_args.p, order.size() * sizeof(GicpPclArgs), cudaMemcpyHostToDevice, st));
    h->tel.h2d += order.size() * sizeof(GicpPclArgs);
    if (cnt[0]) {
      TEL_BEGIN(&h->tel, st);
      k_gicp_pcl_corr_batch<<<dim3(max_nb[0], (unsigned)cnt[0]), kGicpPclThreads, 0, st>>>(b->d_gp_args.p);
      TEL_END(&h->tel, KC_GICP_PCL_CORR, 1, st);
      B2R_CUDA(cudaGetLastError());
    }
    if (cnt[1]) {
      TEL_BEGIN(&h->tel, st);
      if (gicp_pcl_base_pose(cfg.method))
        k_gicp_omp_cost_batch<<<dim3(max_nb[1], (unsigned)cnt[1]), kGicpPclThreads, 0, st>>>(b->d_gp_args.p + cnt[0]);
      else
        k_gicp_pcl_cost_batch<<<dim3(max_nb[1], (unsigned)cnt[1]), kGicpPclThreads, 0, st>>>(b->d_gp_args.p + cnt[0]);
      TEL_END(&h->tel, KC_GICP_PCL_COST, 1, st);
      B2R_CUDA(cudaGetLastError());
    }
    h->tel.d2h += order.size() * (kGicpPclSums + 2) * sizeof(double);
    b->last_rounds++;
    for (size_t r = 0; r < order.size(); r++) {  // the first wait covers the round; the rest only check each message
      const double* msg = b->h_msg.p + r * kRoundMsg;
      GicpPclPairState& P = S[order[r]];
      if (kind_of[r] == 0) {
        rc = wait_host_result(flag, seq, msg, 1, false, st);
        if (rc) return rc;
        P.consume_corr((uint64_t)msg[0]);
      } else {
        rc = wait_host_result(flag, seq, msg, kGicpPclSums, false, st);
        if (rc) return rc;
        P.consume_cost(msg);
      }
    }
    size_t keep = 0;
    for (size_t i : active)
      if (S[i].next() != GicpPclPairState::DONE) active[keep++] = i;
    active.resize(keep);
  }
  for (size_t i = 0; i < m; i++) {
    const GicpPclPairState& P = S[i];
    if (started[i]) method_report(rep[i], P.Tfinal, nullptr, P.converged, P.nr_iterations, P.corr_passes + P.cost_passes, want_fitness);
    else method_report(rep[i], nullptr, pairs[i].guess, false, 0, 0, want_fitness);
  }
  return B2R_OK;
}

// pairs[0..m) of a pcl ICP batch -> rep[0..m) (host).  Every pair runs the single handle's device loop; one launch per pass covers
// every pair (blockIdx.y = pair), so a round is 2 launches (4 with the reciprocal check) whatever the number of pairs.
static int batch_run_icp_chunk(b2r_batch* b, const b2r_pair* pairs, size_t m, bool want_fitness, PairReport* rep) {
  b2r_handle* h = b->eng.get();
  cudaStream_t st = h->st;
  std::vector<size_t> active, off(m, 0);
  size_t ws = 0;
  for (size_t i = 0; i < m; i++) {
    Cloud& s = *b->clouds[pairs[i].source];
    Cloud& t = *b->clouds[pairs[i].target];
    if (s.n == 0 || t.n == 0) continue;  // initCompute fails: the guess, not converged, no iteration (as icp_align)
    off[i] = ws;
    ws += icp_pair_ws(s).bytes;
    active.push_back(i);
  }
  B2R_CUDA(b->method_ws.reserve(ws + 256));
  char* base = reinterpret_cast<char*>(align_up(reinterpret_cast<size_t>(b->method_ws.p), 256));
  B2R_CUDA(cudaMemsetAsync(base, 0, ws, st));
  const size_t na = active.size();
  if (na) {
    B2R_CUDA(b->d_icp.reserve(na));
    if (b->h_icp.cap < na) B2R_CUDA(b->h_icp.alloc(na + 16));
    for (size_t k = 0; k < na; k++) {
      const size_t i = active[k];
      icp_fill_pair(h->cfg, *b->clouds[pairs[i].source], *b->clouds[pairs[i].target], pairs[i].guess, base + off[i], b->h_icp.p[k]);
    }
    B2R_CUDA(cudaMemcpyAsync(b->d_icp.p, b->h_icp.p, na * sizeof(IcpPairDev), cudaMemcpyHostToDevice, st));
    h->tel.h2d += na * sizeof(IcpPairDev);
    int rounds = 0;
    int rc = icp_run(b->d_icp.p, b->h_icp.p, (unsigned)na, 8, &h->tel, st, &rounds);
    if (rc) return rc;
    b->last_rounds += (unsigned long long)rounds;
  }
  for (size_t i = 0, k = 0; i < m; i++) {  // active[k]: ascending
    if (k < na && active[k] == i) {
      const IcpPairDev& P = b->h_icp.p[k++];
      method_report(rep[i], P.T, nullptr, P.converged != 0, P.iterations, P.rounds, want_fitness);
    } else {
      method_report(rep[i], nullptr, pairs[i].guess, false, 0, 0, want_fitness);
    }
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
  b2r_handle* h = b->eng.get();
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
  std::vector<int32_t> named(2 * n_pairs);
  for (size_t i = 0; i < n_pairs; i++) { named[2 * i] = pairs[i].source; named[2 * i + 1] = pairs[i].target; }
  const bool ndt = ndt_family(h->cfg.method);
  const bool icp = h->cfg.method == B2R_METHOD_ICP_PCL;  // ICP reads the search structures only
  rc = batch_build_structures(b, named.data(), named.size(), !fit_only && !ndt && !icp);
  if (rc) return rc;
  if (ndt) rc = batch_ndt_maps(b, pairs, n_pairs, fit_only);
  if (rc) return rc;
  const bool vgicp = vgicp_family(h->cfg.method) && !fit_only;
  const bool gpcl = gicp_pcl_family(h->cfg.method);
  // NDT, pcl GICP and ICP aligns run their rounds from the host and leave their reports in h_reports; a stand-alone fitness
  // evaluation is the GICP engine's search on every method
  const bool host_driven = !fit_only && (ndt || gpcl || icp);
  if (vgicp) rc = batch_vgicp_maps(b, pairs, n_pairs);
  if (rc) return rc;
  const auto t_b = std::chrono::steady_clock::now();
  const size_t chunk = std::min(b->max_chunk, std::max<size_t>(n_pairs, 1));
  rc = batch_host_staging(b, std::max(chunk, n_pairs));
  if (rc) return rc;
  B2R_CUDA(b->d_reports.reserve(n_pairs + 1));
  // a VGICP round carries no fitness sums: its scores come from batch_fitness after the rounds
  const LmCfg cfg = make_lm_cfg(h->cfg, want_fitness && !vgicp, fit_max_range);
  b->last_rounds = b->last_pair_rounds = 0;
  for (size_t c0 = 0; c0 < n_pairs; c0 += chunk) {
    const size_t m = std::min(chunk, n_pairs - c0);
    if (!host_driven) rc = batch_run_chunk(b, pairs + c0, m, cfg, b->d_reports.p + c0, fit_only);
    else if (ndt) rc = batch_run_ndt_chunk(b, pairs + c0, m, want_fitness, b->h_reports.p + c0);
    else if (gpcl) rc = batch_run_gicp_pcl_chunk(b, pairs + c0, m, want_fitness, b->h_reports.p + c0);
    else rc = batch_run_icp_chunk(b, pairs + c0, m, want_fitness, b->h_reports.p + c0);
    if (rc) return rc;
  }
  if (host_driven)  // the reports go where the GICP engine leaves them: b2r_batch_loop_detect packs and gathers them on the device
    B2R_CUDA(cudaMemcpyAsync(b->d_reports.p, b->h_reports.p, n_pairs * sizeof(PairReport), cudaMemcpyHostToDevice, h->st));
  if (want_fitness && (vgicp || host_driven)) rc = batch_fitness(b, pairs, n_pairs, fit_max_range, b->d_reports.p);
  if (rc) return rc;
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
  B2R_CUDA(cudaMemcpyAsync(b->h_reports.p, b->d_reports.p, n_pairs * sizeof(PairReport), cudaMemcpyDeviceToHost, st));
  B2R_CUDA(cudaStreamSynchronize(st));
  b->eng->tel.d2h += n_pairs * sizeof(PairReport);
  b->last_pair_rounds = 0;
  for (size_t i = 0; i < n_pairs; i++) {
    out[i] = b->h_reports.p[i].r;
    b->last_pair_rounds += (unsigned long long)b->h_reports.p[i].rounds;
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
  B2R_CUDA(cudaMemcpyAsync(b->h_reports.p, b->d_reports.p, n_pairs * sizeof(PairReport), cudaMemcpyDeviceToHost, st));
  B2R_CUDA(cudaStreamSynchronize(st));
  b->eng->tel.d2h += n_pairs * sizeof(PairReport);
  for (size_t i = 0; i < n_pairs; i++) scores[i] = b->h_reports.p[i].r.fitness;
  return B2R_OK;
}

// MapCloudGenerator::generate (map_cloud_generator.cpp:13-51) over the keyframe clouds the batch already holds: keyframe k = cloud
// ids[k] at poses[16k..16k+16).  resolution > 0 reads every cloud's search structure (built here if missing, as the next align
// would), so no record is uploaded and device-added clouds work after their buffers are gone; resolution <= 0 needs the full records
// and therefore the cache's own upload of each cloud.  The result is b2r_map_cloud_generate's on the same clouds and poses.
extern "C" int b2r_batch_map_cloud_generate(b2r_batch* b, const int32_t* ids, const float* poses, size_t n_keyframes, double resolution,
                                            size_t out_stride_bytes, void* out_host, size_t out_capacity, const void** d_out, size_t* n_out) {
  if (!b || !n_out) return fail(B2R_EINVAL, "NULL argument");
  *n_out = 0;
  if (d_out) *d_out = nullptr;
  if (n_keyframes == 0) return 1;  // "warning: keyframes empty!!" -> nullptr (map_cloud_generator.cpp:14-17)
  if (!ids || !poses) return fail(B2R_EINVAL, "NULL argument");
  if (out_stride_bytes < 12 || (out_stride_bytes & 3)) return fail(B2R_EINVAL, "bad stride");
  const bool voxels = resolution > 0.0;
  size_t total = 0;
  for (size_t k = 0; k < n_keyframes; k++) {
    const int32_t id = ids[k];
    if (id < 0 || (size_t)id >= b->clouds.size() || !b->clouds[id]) return fail(B2R_EINVAL, "unknown cloud id " + std::to_string(id));
    const Cloud& c = *b->clouds[id];
    if (!voxels && (c.raw_view != c.raw.p || !c.raw.p))  // a device-added cloud's records are the caller's, valid only until its build
      return fail(B2R_EINVAL, "cloud id " + std::to_string(id) + " was added from device memory: resolution <= 0 needs records the batch holds");
    if (!voxels && (size_t)c.stride_f * 4 != out_stride_bytes)
      return fail(B2R_EINVAL, "cloud id " + std::to_string(id) + " has " + std::to_string(c.stride_f * 4) + "-byte records, not out_stride_bytes");
    total += c.n;
  }
  if (total >= (size_t)0x7fffffff) return fail(B2R_EINVAL, "map cloud too large (>= 2^31 points)");
  if (total == 0) return B2R_OK;
  if (out_host && !voxels && out_capacity < total) return fail(B2R_EINVAL, "output capacity too small");
  b2r_handle* h = b->eng.get();
  B2R_CUDA(cudaSetDevice(h->cfg.device_id));
  cudaStream_t st = h->st;
  int rc = batch_sync_builds(b, false);  // the uploads of the named clouds
  if (rc) return rc;
  const int sf = (int)(out_stride_bytes / 4);
  DevBuf<float>& out = h->pf_buf[0];
  DevBuf<float>& cloud = h->pf_buf[1];
  B2R_CUDA(out.reserve(total * sf + 8));
  size_t m = 0;
  if (!voxels) {  // "To get unfiltered point cloud with intensity" (:39-40): the transformed records, straight into the output
    std::vector<MapKf> kf;
    size_t first = 0;
    for (size_t k = 0; k < n_keyframes; k++) {
      const Cloud& c = *b->clouds[ids[k]];
      if (c.n) {  // empty keyframes must not shadow their successors in the binary search
        MapKf d;
        d.pts = c.raw.p; d.first = (long long)first; d.n = (int)c.n; d.pad = 0;
        for (int r = 0; r < 3; r++) for (int col = 0; col < 4; col++) d.T[r * 4 + col] = poses[16 * k + col * 4 + r];
        kf.push_back(d);
      }
      first += c.n;
    }
    B2R_CUDA(h->map_kf.reserve(kf.size() * sizeof(MapKf) + 64));
    B2R_CUDA(cudaMemcpyAsync(h->map_kf.p, kf.data(), kf.size() * sizeof(MapKf), cudaMemcpyHostToDevice, st));
    { TEL_BEGIN(&h->tel, st);
      k_map_transform<<<map_blocks(h, total), 256, 0, st>>>(reinterpret_cast<const MapKf*>(h->map_kf.p), (int)kf.size(), sf, (long long)total, out.p);
      TEL_END(&h->tel, KC_MISC, 1, st); }
    B2R_CUDA(cudaGetLastError());
    B2R_CUDA(cudaStreamSynchronize(st));  // kf is pageable host memory of this call
    m = total;
  } else {
    rc = batch_build_structures(b, ids, n_keyframes, false);
    if (rc) return rc;
    std::vector<MapCachedKf> kf;
    size_t first = 0;
    for (size_t k = 0; k < n_keyframes; k++) {
      const Cloud& c = *b->clouds[ids[k]];
      if (c.n) {
        MapCachedKf d;
        d.sorted = c.sorted.p; d.pos_of = c.pos_of.p; d.first = (long long)first;
        for (int r = 0; r < 3; r++) for (int col = 0; col < 4; col++) d.T[r * 4 + col] = poses[16 * k + col * 4 + r];
        kf.push_back(d);
      }
      first += c.n;
    }
    B2R_CUDA(cloud.reserve(total * 4 + 8));
    B2R_CUDA(h->map_kf.reserve(kf.size() * sizeof(MapCachedKf) + 64));
    B2R_CUDA(cudaMemcpyAsync(h->map_kf.p, kf.data(), kf.size() * sizeof(MapCachedKf), cudaMemcpyHostToDevice, st));
    B2R_CUDA(cudaStreamSynchronize(st));  // kf is pageable host memory of this call
    { TEL_BEGIN(&h->tel, st);
      k_map_gather<<<map_blocks(h, total), 256, 0, st>>>(reinterpret_cast<const MapCachedKf*>(h->map_kf.p), (int)kf.size(), (long long)total,
                                                         reinterpret_cast<float4*>(cloud.p));
      TEL_END(&h->tel, KC_MISC, 1, st); }
    B2R_CUDA(cudaGetLastError());
    rc = map_voxel_centres(h, cloud.p, 4, total, resolution, out.p, sf, &m);
    if (rc) return rc;
    if (out_host && out_capacity < m) return fail(B2R_EINVAL, "output capacity too small");
  }
  if (out_host && m) {
    B2R_CUDA(cudaMemcpyAsync(out_host, out.p, m * out_stride_bytes, cudaMemcpyDeviceToHost, st));
    B2R_CUDA(cudaStreamSynchronize(st));
    h->tel.d2h += m * out_stride_bytes;
  }
  if (d_out) *d_out = out.p;
  *n_out = m;
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
  B2R_CUDA(b->h_gather.alloc(M * (size_t)b->world));
  B2R_CUDA(b->d_reports.reserve(1));
  b->h_word.p[b2r_batch::kLanes] = 0;
  k_pack_results<<<(unsigned)((M + 255) / 256), 256, 0, st>>>(b->d_reports.p, (int)mine, b->d_send.p, (int)M, b->h_word.d + b2r_batch::kLanes);
  B2R_CUDA(cudaGetLastError());
  const b2r_result* gathered = b->d_send.p;
  if (b->world > 1) {
    if (!b->comm) return fail(B2R_ESTATE, "b2r_batch_comm_init has not been called");
    // the ONE data-plane collective of the batch: fixed 80-byte records, padded to the largest per-rank share
    B2R_NCCL(ncclAllGather(b->d_send.p, b->d_recv.p, M * sizeof(b2r_result), ncclChar, b->comm, st));
    gathered = b->d_recv.p;
  }
  B2R_CUDA(cudaMemcpyAsync(b->h_gather.p, gathered, M * (size_t)b->world * sizeof(b2r_result), cudaMemcpyDeviceToHost, st));
  B2R_CUDA(cudaStreamSynchronize(st));
  b->eng->tel.d2h += M * (size_t)b->world * sizeof(b2r_result);
  b->last_pair_rounds = b->h_word.p[b2r_batch::kLanes];  // exact: every pair's own round count (the stream has been synchronised)
  if (dbg) {
    const auto t_c = std::chrono::steady_clock::now();
    fprintf(stderr, "[b2r rank %d] loop_detect: batch_run + sync %.3f ms, pack + all-gather + readback %.3f ms\n", b->rank,
            std::chrono::duration<double, std::milli>(t_b - t_a).count(), std::chrono::duration<double, std::milli>(t_c - t_b).count());
  }
  for (int r = 0; r < b->world; r++)
    for (size_t i = p0[r]; i < p1[r]; i++) all_results[i] = b->h_gather.p[(size_t)r * M + (i - p0[r])];
  for (size_t g = 0; g < n_groups; g++) {
    rc = b2r_loop_argmin(all_results + group_first[g], (size_t)(group_first[g + 1] - group_first[g]), fitness_score_thresh, &best[g]);
    if (rc) return rc;
  }
  return B2R_OK;
}
