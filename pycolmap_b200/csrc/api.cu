// api.cu -- C ABI of libb200match.so: context, resident image set, batched pair scheduler.
// Host side of the hot path: replaces FeatureMatcherController / FeatureMatcherWorker /
// FeatureMatcherCache (U:controllers/feature_matching_utils.cc) for the pipelines bound at
// R:pipeline/match_features.h:22-68.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>

#include "internal.h"
#include "match_kernel.cuh"
#include "verify.cuh"

using namespace b2m;

namespace b2m {
thread_local std::string g_noctx_err;
}

namespace {

int fail(b2m_ctx* ctx, int code, const std::string& msg) {
  if (ctx) ctx->err = msg; else g_noctx_err = msg;
  return code;
}

#define CU_TRY(ctx, expr)                                                                       \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess) {                                                                    \
      char _b[512];                                                                             \
      snprintf(_b, sizeof(_b), "[%s:%d] CUDA error: %s (%s)", __FILE__, __LINE__,              \
               cudaGetErrorString(_e), #expr);                                                  \
      return fail(ctx, _e == cudaErrorMemoryAllocation ? B2M_ENOMEM : B2M_ECUDA, _b);            \
    }                                                                                           \
  } while (0)

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

int round_up(int v, int m) { return (v + m - 1) / m * m; }

// Lay out the image table and allocate the padded descriptor array (zero-filled).
int layout_images_impl(b2m_ctx* ctx, ImageSet& S, int n_images, const int32_t* n_feat, bool want_kpts);
int layout_images(b2m_ctx* ctx, ImageSet& S, int n_images, const int32_t* n_feat, bool want_kpts) {
  const int rc = layout_images_impl(ctx, S, n_images, n_feat, want_kpts);
  if (rc != B2M_OK) S.release();  // never leave a half-built set behind: a later match call would run on it
  return rc;
}
int layout_images_impl(b2m_ctx* ctx, ImageSet& S, int n_images, const int32_t* n_feat, bool want_kpts) {
  S.release();
  static std::atomic<uint64_t> g_generation{0};
  S.generation = ++g_generation;
  S.n_images = n_images;
  S.nfeat.assign(n_feat, n_feat + n_images);
  S.row0.resize(n_images);
  int64_t rows = 0;
  S.max_feat = 0;
  for (int i = 0; i < n_images; ++i) {
    if (n_feat[i] < 0) return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: n_feat[i] >= 0");
    S.row0[i] = static_cast<int32_t>(rows);
    rows += round_up(n_feat[i], kRowPad);
    S.max_feat = std::max(S.max_feat, n_feat[i]);
    if (rows > (int64_t(1) << 31) - kRowPad)
      return fail(ctx, B2M_EINVAL, "[api.cu] image set exceeds 2^31 descriptor rows");
  }
  rows = std::max<int64_t>(rows, kRowPad);
  S.max_feat_pad = std::max(round_up(S.max_feat, kRowPad), kRowPad);
  S.total_rows = rows;
  CU_TRY(ctx, cudaMalloc(&S.d_desc, static_cast<size_t>(rows) * 128));
  CU_TRY(ctx, cudaMemsetAsync(S.d_desc, 0, static_cast<size_t>(rows) * 128, ctx->stream));
  if (want_kpts) {
    CU_TRY(ctx, cudaMalloc(&S.d_kpts, static_cast<size_t>(rows) * sizeof(float2)));
    CU_TRY(ctx, cudaMemsetAsync(S.d_kpts, 0, static_cast<size_t>(rows) * sizeof(float2), ctx->stream));
  }
  // one extra, all-zero entry behind the table: image index `n_images` = "no features" (the dummy image
  // launch_k1_filter_skip points dead pairs at)
  CU_TRY(ctx, cudaMalloc(&S.d_row0, sizeof(int32_t) * (n_images + 1)));
  CU_TRY(ctx, cudaMalloc(&S.d_nfeat, sizeof(int32_t) * (n_images + 1)));
  CU_TRY(ctx, cudaMemsetAsync(S.d_row0, 0, sizeof(int32_t) * (n_images + 1), ctx->stream));
  CU_TRY(ctx, cudaMemsetAsync(S.d_nfeat, 0, sizeof(int32_t) * (n_images + 1), ctx->stream));
  if (n_images > 0) {
    CU_TRY(ctx, cudaMemcpyAsync(S.d_row0, S.row0.data(), sizeof(int32_t) * n_images, cudaMemcpyHostToDevice,
                                ctx->stream));
    CU_TRY(ctx, cudaMemcpyAsync(S.d_nfeat, S.nfeat.data(), sizeof(int32_t) * n_images, cudaMemcpyHostToDevice,
                                ctx->stream));
  }
  // One TMA tensor map over the whole set: dim0 = 128 descriptor bytes, dim1 = rows; box 128 x 128,
  // SWIZZLE_128B so that the tile lands in the canonical K-major wgmma layout.
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return fail(ctx, B2M_ECUDA, "[api.cu] cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t gdim[2] = {128, static_cast<cuuint64_t>(rows)};
  cuuint64_t gstride[1] = {128};
  cuuint32_t box[2] = {128, 128};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(&S.tmap, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, S.d_desc, gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char b[128];
    snprintf(b, sizeof(b), "[api.cu] cuTensorMapEncodeTiled failed: CUresult %d", static_cast<int>(r));
    return fail(ctx, B2M_ECUDA, b);
  }
  return B2M_OK;
}

int ensure_workspace(b2m_ctx* ctx, int batch, int32_t mstride) {
  Workspace& W = ctx->ws;
  if (W.batch >= batch && W.mstride >= mstride) return B2M_OK;
  W.release();
  batch = std::max(batch, W.batch);
  mstride = std::max(mstride, W.mstride);
  const size_t arena_matches = static_cast<size_t>(batch) * mstride;
  CU_TRY(ctx, cudaMalloc(&W.d_mbuf, sizeof(int32_t) * 2 * arena_matches));
  CU_TRY(ctx, cudaMalloc(&W.d_aux, sizeof(uint2) * 2 * arena_matches));
  CU_TRY(ctx, cudaMalloc(&W.d_cand_rows, sizeof(int32_t) * 2 * arena_matches));
  CU_TRY(ctx, cudaMalloc(&W.d_cand_sorted, sizeof(int32_t) * 2 * arena_matches));
  CU_TRY(ctx, cudaMalloc(&W.d_cand_cnt, sizeof(int32_t) * 2 * batch));
  CU_TRY(ctx, cudaMalloc(&W.d_pairs_dir1, sizeof(int32_t) * 2 * batch));
  for (int s = 0; s < 2; ++s) {
    CU_TRY(ctx, cudaMalloc(&W.d_arena[s], sizeof(uint2) * arena_matches));
    CU_TRY(ctx, cudaMalloc(&W.d_cursor[s], sizeof(unsigned long long)));
    CU_TRY(ctx, cudaMalloc(&W.d_pair_off[s], sizeof(int64_t) * batch));
    CU_TRY(ctx, cudaMalloc(&W.d_pair_cnt[s], sizeof(int32_t) * batch));
    CU_TRY(ctx, cudaMallocHost(&W.h_arena[s], sizeof(uint2) * arena_matches));
    CU_TRY(ctx, cudaMallocHost(&W.h_cursor[s], sizeof(unsigned long long)));
    CU_TRY(ctx, cudaMallocHost(&W.h_pair_off[s], sizeof(int64_t) * batch));
    CU_TRY(ctx, cudaMallocHost(&W.h_pair_cnt[s], sizeof(int32_t) * batch));
  }
  W.batch = batch;
  W.mstride = mstride;
  return B2M_OK;
}

// Scratch of the gathered column direction, sized like the workspace (worst case: every column of every pair matched).
int ensure_gather(b2m_ctx* ctx) {
  Workspace& W = ctx->ws;
  if (W.d_gath_desc) return B2M_OK;
  const size_t rows = static_cast<size_t>(W.batch) * W.mstride;
  CU_TRY(ctx, cudaMalloc(&W.d_gath_desc, rows * 128));
  CU_TRY(ctx, cudaMalloc(&W.d_colrank, sizeof(int32_t) * rows));
  CU_TRY(ctx, cudaMalloc(&W.d_gath_cols, sizeof(int32_t) * rows));
  CU_TRY(ctx, cudaMalloc(&W.d_gath_cnt, sizeof(int32_t) * W.batch));
  CU_TRY(ctx, cudaMalloc(&W.d_gath_items, sizeof(int32_t) * 2 * (rows / kRowPad + 1)));
  CU_TRY(ctx, cudaMalloc(&W.d_gath_n, sizeof(int32_t)));
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return fail(ctx, B2M_ECUDA, "[api.cu] cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t gdim[2] = {128, static_cast<cuuint64_t>(rows)};
  cuuint64_t gstride[1] = {128};
  cuuint32_t box[2] = {128, 128};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(&W.tmap_gath, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, W.d_gath_desc, gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(ctx, B2M_ECUDA, "[api.cu] cuTensorMapEncodeTiled (gather scratch) failed");
  return B2M_OK;
}

int check_sift(b2m_ctx* ctx, const b2m_sift_opts* o) {
  if (!o) return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: sift options != NULL");
  if (!(o->max_ratio > 0.f)) return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: max_ratio > 0");
  if (!(o->max_distance > 0.f)) return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: max_distance > 0");
  return B2M_OK;
}

// Core scheduler: match (and optionally verify) `n_pairs` pairs of image set S in batches.
// One-deep cache of the big host arrays of a result object.  A pipeline repeats similar calls (blocks of an
// exhaustive run, steps of a bench): handing the previous call's pages to the next one saves mapping, first-touch
// faulting and unmapping ~1 GB per call (measured on 1000 x 8192: 145 ms of a 3.5 s call went into freeing alone).
// Bounded: at most the two largest arrays seen since the last reuse; B2M_HOST_CACHE=0 disables it.
struct HostCache {
  std::mutex mu;
  BigU32 matches, inliers;
};
HostCache& host_cache() {
  static HostCache* c = new HostCache;   // never destroyed: a result object may be freed during process teardown
  return *c;
}
bool host_cache_enabled() {
  static const bool on = [] {
    const char* e = getenv("B2M_HOST_CACHE");
    return !(e && e[0] == '0');
  }();
  return on;
}

int match_pairs_impl(b2m_ctx* ctx, ImageSet& S, const int32_t* pairs, int64_t n_pairs, const b2m_sift_opts* sift,
                     const b2m_tvg_opts* tvg, b2m_results** out) {
  if (!out) return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: out != NULL");
  *out = nullptr;
  // B2M_HOSTPROF=1: wall-clock split of this call on the host (set-up, launch loop, tail) on stderr
  static const bool host_prof = getenv("B2M_HOSTPROF") != nullptr;
  auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  const double hp_t0 = now();
  if (int rc = check_sift(ctx, sift)) return rc;
  if (n_pairs < 0 || (n_pairs > 0 && !pairs)) return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: pairs");
  if (!S.d_desc) return fail(ctx, B2M_ESTATE, "[api.cu] b2m_set_images must be called before matching");
  int32_t max_feat_used = 0;  // over the images the pair list references (the resident set may hold others)
  for (int64_t k = 0; k < 2 * n_pairs; ++k) {
    if (pairs[k] < 0 || pairs[k] >= S.n_images)
      return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: pair image index out of range");
    max_feat_used = std::max(max_feat_used, S.nfeat[pairs[k]]);
  }
  if (tvg && (!S.d_kpts || S.cams.empty()))
    return fail(ctx, B2M_ESTATE, "[api.cu] verification requested but the image set has no keypoints/cameras");
  if (tvg && tvg->multiple_models)
    return fail(ctx, B2M_EINVAL, "[api.cu] multiple_models is available through b2m_estimate_two_view_geometry only "
                                 "(the pair pipeline verifies one geometry per pair)");

  // Upstream's GPU matcher warns and truncates an image to max_num_matches features (WarnIfMaxNumMatchesReachedGPU,
  // U:feature/sift.cc); here the truncation belongs to the upload (the host's UploadImageSet does it, with the same
  // warning): a resident image that is too long AND referenced by this call is a caller error.
  if (max_feat_used > sift->max_num_matches)
    return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: num descriptors <= SiftMatchingOptions.max_num_matches "
                                 "(truncate at upload; images the pair list does not reference are not checked)");

  b2m_results* res = new (std::nothrow) b2m_results();
  if (!res) return fail(ctx, B2M_ENOMEM, "[api.cu] out of host memory");
  res->pairs.assign(pairs, pairs + 2 * n_pairs);
  res->off.assign(n_pairs, 0);
  res->cnt.assign(n_pairs, 0);
  if (tvg) verify_results_init(res, n_pairs);
  if (host_cache_enabled()) {
    HostCache& hc = host_cache();
    std::lock_guard<std::mutex> lk(hc.mu);
    res->matches.swap(hc.matches);
    res->inliers.swap(hc.inliers);
    res->matches.clear();
    res->inliers.clear();
  }
  {  // Size the result arrays like the previous call (a pipeline repeats similar calls): growing a flat
     // vector by doubling re-copies hundreds of MB a few times per call and stalls the launch loop.
    const uint64_t cap = static_cast<uint64_t>(n_pairs) * static_cast<uint64_t>(std::max(S.max_feat, 1));
    try {
      res->matches.reserve(static_cast<size_t>(2 * std::min(ctx->hint_matches + ctx->hint_matches / 16, cap)));
      if (tvg) res->inliers.reserve(static_cast<size_t>(2 * std::min(ctx->hint_inliers + ctx->hint_inliers / 16, cap)));
    } catch (const std::bad_alloc&) {  // only a hint
    }
  }
  auto bail = [&](int rc) {
    delete res;
    return rc;
  };

  // pairs per kernel batch; bounded so that the worst-case scratch of the gathered column direction
  // (batch x mstride descriptors) stays below 6 GB even for 32768-feature images
  // Default: as many pairs as keep batch x (padded rows per image) at what 4096 pairs of 8192-feature images are -- the
  // per-batch chain of small kernels and the RANSAC launch tails are a fixed cost per batch, so smaller images take
  // proportionally more pairs per batch (5000 x 4096: 8192).
  const int64_t rows_pad = round_up(S.max_feat_pad, 512);
  const int64_t want = ctx->pair_batch_auto ? std::min<int64_t>(16384, std::max<int64_t>(1024, (int64_t{4096} * 8192) / rows_pad))
                                            : ctx->pair_batch;
  const int B = static_cast<int>(std::min<int64_t>(want, std::max<int64_t>(64, (int64_t{6} << 30) / (rows_pad * 128))));
  // sized for the pairs of this call, not for a full batch: a context that only ever sees small jobs stays small
  if (int rc = ensure_workspace(ctx, static_cast<int>(std::min<int64_t>(B, std::max<int64_t>(n_pairs, 1))),
                                round_up(S.max_feat_pad, 512)))
    return bail(rc);
  if (tvg)
    if (int rc = verify_prepare(ctx, S, ctx->ws.batch, static_cast<int64_t>(ctx->ws.batch) * ctx->ws.mstride))
      return bail(rc);
  if (ctx->d_pairs_cap < n_pairs) {
    if (ctx->d_pairs) cudaFree(ctx->d_pairs);
    ctx->d_pairs = nullptr;
    ctx->d_pairs_cap = 0;
    cudaError_t e = cudaMalloc(&ctx->d_pairs, sizeof(int32_t) * 2 * std::max<int64_t>(n_pairs, 1));
    if (e != cudaSuccess) return bail(fail(ctx, B2M_ENOMEM, "[api.cu] cudaMalloc(pairs) failed"));
    ctx->d_pairs_cap = n_pairs;
  }
  Workspace& W = ctx->ws;
  cudaStream_t st = ctx->stream;
#define CU_TRY_R(expr)                                                                      \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) {                                                                \
      char _b[512];                                                                         \
      snprintf(_b, sizeof(_b), "[%s:%d] CUDA error: %s (%s)", __FILE__, __LINE__,          \
               cudaGetErrorString(_e), #expr);                                              \
      return bail(fail(ctx, B2M_ECUDA, _b));                                                \
    }                                                                                       \
  } while (0)

  if (n_pairs > 0)
    CU_TRY_R(cudaMemcpyAsync(ctx->d_pairs, pairs, sizeof(int32_t) * 2 * n_pairs, cudaMemcpyHostToDevice, st));
  CU_TRY_R(cudaEventRecord(ctx->ev_t0, st));
  ctx->stats.last_k1_ms = 0.0;
  ctx->stats.last_k1_launches = 0;

  const int max_strips = S.max_feat_pad / 128;
  const int n_dirs = sift->cross_check ? 2 : 1;
  const int64_t n_batches = (n_pairs + B - 1) / B;
  double verify_ms = 0.0;
  bool pipelined = false;  // decided below, before the first batch

  // Drain one finished batch: counts -> host, then offsets + matches on the copy stream.
  auto finish = [&](int64_t b) -> int {
    const int s = static_cast<int>(b & 1);
    const int64_t p0 = b * B;
    const int nb = static_cast<int>(std::min<int64_t>(B, n_pairs - p0));
    CU_TRY(ctx, cudaEventSynchronize(ctx->ev_k[s]));
    const unsigned long long total = *W.h_cursor[s];
    {
      float k1ms = 0.f, vms = 0.f;
      if (pipelined) {
        // overlapped order: K1 = the two GEMM launches; everything else (resolve, gather, compaction, RANSAC,
        // decision) is the remainder of the step, computed at the end.  The GEMM0 events of this slot may already
        // belong to batch b + 2 here: the launch loop reads them before re-recording (gemm0_time).
        if (cudaEventElapsedTime(&k1ms, ctx->ev_g2a[s], ctx->ev_g2b[s]) == cudaSuccess) ctx->stats.last_k1_ms += k1ms;
      } else {
        if (cudaEventElapsedTime(&k1ms, ctx->ev_k1a[s], ctx->ev_k1b[s]) == cudaSuccess) ctx->stats.last_k1_ms += k1ms;
        // compaction + verification kernels of this batch
        if (cudaEventElapsedTime(&vms, ctx->ev_k1b[s], ctx->ev_k[s]) == cudaSuccess) verify_ms += vms;
      }
    }
    CU_TRY(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_k[s], 0));
    CU_TRY(ctx, cudaMemcpyAsync(W.h_pair_off[s], W.d_pair_off[s], sizeof(int64_t) * nb, cudaMemcpyDeviceToHost,
                                ctx->copy_stream));
    CU_TRY(ctx, cudaMemcpyAsync(W.h_pair_cnt[s], W.d_pair_cnt[s], sizeof(int32_t) * nb, cudaMemcpyDeviceToHost,
                                ctx->copy_stream));
    if (total > 0)
      CU_TRY(ctx, cudaMemcpyAsync(W.h_arena[s], W.d_arena[s], sizeof(uint2) * total, cudaMemcpyDeviceToHost,
                                  ctx->copy_stream));
    if (tvg)
      if (int rc = verify_batch_download(ctx, res, s, p0, nb)) return rc;
    CU_TRY(ctx, cudaEventRecord(ctx->ev_data[s], ctx->copy_stream));
    CU_TRY(ctx, cudaEventSynchronize(ctx->ev_data[s]));
    const int64_t base = static_cast<int64_t>(res->matches.size() / 2);
    res->matches.resize(res->matches.size() + 2 * total);
    if (total > 0) memcpy(res->matches.data() + 2 * base, W.h_arena[s], sizeof(uint2) * total);
    for (int k = 0; k < nb; ++k) {
      res->off[p0 + k] = base + W.h_pair_off[s][k];
      res->cnt[p0 + k] = W.h_pair_cnt[s][k];
    }
    if (tvg)
      if (int rc = verify_batch_collect(ctx, res, s, p0, nb, tvg->min_num_inliers)) return rc;
    return B2M_OK;
  };

  struct BatchParams {
    int s = 0, nb = 0;
    int64_t p0 = 0;
    MatchParams mp{};
    CompactParams cp{};
  };
  auto batch_params = [&](int64_t b) {
    BatchParams bp;
    bp.s = static_cast<int>(b & 1);
    bp.p0 = b * B;
    bp.nb = static_cast<int>(std::min<int64_t>(B, n_pairs - bp.p0));
    MatchParams& mp = bp.mp;
    mp.pairs = ctx->d_pairs + 2 * bp.p0;
    mp.img_row0 = S.d_row0;
    mp.img_nfeat = S.d_nfeat;
    mp.mbuf = W.d_mbuf;
    mp.mstride = W.mstride;
    mp.acos_lut = ctx->d_lut;
    mp.max_ratio = sift->max_ratio;
    mp.max_distance = sift->max_distance;
    mp.aux = W.d_aux;
    mp.cand_cnt = W.d_cand_cnt;
    mp.cand_rows = W.d_cand_rows;
    mp.cand_sorted = W.d_cand_sorted;
    CompactParams& cp = bp.cp;
    cp.pairs = mp.pairs;
    cp.img_nfeat = S.d_nfeat;
    cp.mbuf = W.d_mbuf;
    cp.mstride = W.mstride;
    cp.cross_check = sift->cross_check ? 1 : 0;
    cp.arena = W.d_arena[bp.s];
    cp.cursor = W.d_cursor[bp.s];
    cp.pair_off = W.d_pair_off[bp.s];
    cp.pair_cnt = W.d_pair_cnt[bp.s];
    cp.img_row0 = S.d_row0;
    cp.kpts = tvg ? S.d_kpts : nullptr;
    cp.pts = tvg ? static_cast<double4*>(verify_points_arena(ctx, bp.s)) : nullptr;
    cp.enable = nullptr;
    cp.cand_cnt = ctx->exact_k1 ? nullptr : W.d_cand_cnt;   // the filter epilogue's candidate counts (not produced by K1-exact)
    return bp;
  };
  // Column direction of the cross-check: computed for the matched columns only (launch_k1_filter_gather).  The
  // first cross-check batch of a context is computed both ways and the match lists compared on the device; on
  // any difference the context stays on the two-direction launch.
  const bool split_capable = !ctx->exact_k1 && n_dirs == 2;
  auto gather_scratch = [&]() {
    GatherScratch g;
    g.desc = W.d_gath_desc; g.colrank = W.d_colrank; g.cols = W.d_gath_cols; g.cnt = W.d_gath_cnt;
    g.items = W.d_gath_items; g.n_items = W.d_gath_n;
    return g;
  };
  // One-time comparison of the gathered schedule against the two-direction launch on one batch (returns a B2M code;
  // leaves ctx->k1_dir1_mode decided unless the batch had no match at all).  The batch itself is redone afterwards.
  auto k1_selftest = [&](const BatchParams& bp) -> int {
    const int s = bp.s, nb = bp.nb;
    const MatchParams& mp = bp.mp;
    const CompactParams& cp = bp.cp;
    uint2* t_arena = nullptr;
    int64_t* t_off = nullptr;
    int32_t *t_cnt = nullptr, *t_flag = nullptr;
    auto drop = [&]() {
      cudaFree(t_arena); cudaFree(t_off); cudaFree(t_cnt); cudaFree(t_flag);
      t_arena = nullptr; t_off = nullptr; t_cnt = nullptr; t_flag = nullptr;
    };
    const size_t arena_matches = static_cast<size_t>(W.batch) * W.mstride;
    if (ensure_gather(ctx) != B2M_OK || cudaMalloc(&t_arena, sizeof(uint2) * arena_matches) != cudaSuccess ||
        cudaMalloc(&t_off, sizeof(int64_t) * nb) != cudaSuccess || cudaMalloc(&t_cnt, sizeof(int32_t) * nb) != cudaSuccess ||
        cudaMalloc(&t_flag, sizeof(int32_t)) != cudaSuccess) {
      drop();
      cudaGetLastError();
      ctx->k1_dir1_mode = B2M_K1_DIR1_FULL_NOMEM;  // no room for the scratch / comparison: stay on the validated launch
      return B2M_OK;
    }
    CompactParams ct = cp;  // the gathered schedule's match lists go to the temporary arena
    ct.arena = t_arena;
    ct.pair_off = t_off;
    ct.pair_cnt = t_cnt;
    ct.kpts = nullptr;
    ct.pts = nullptr;
    ct.colrank = W.d_colrank;
    cudaError_t e = cudaMemsetAsync(W.d_cursor[s], 0, sizeof(unsigned long long), st);
    if (e == cudaSuccess)
      e = launch_k1_filter_gather(S.tmap, W.tmap_gath, mp, S.d_desc, nb, max_strips, ctx->num_sms, gather_scratch(), st, nullptr);
    if (e == cudaSuccess) e = launch_crosscheck_compact(ct, nb, st);
    if (e != cudaSuccess) {
      // the gathered schedule could not even be launched (a non-sticky launch error): stay on the validated
      // launch instead of failing the call; a sticky error resurfaces at the next CUDA call anyway
      cudaGetLastError();
      drop();
      ctx->k1_dir1_mode = B2M_K1_DIR1_FULL_MISMATCH;
      CU_TRY_R(cudaMemsetAsync(W.d_cursor[s], 0, sizeof(unsigned long long), st));
      return B2M_OK;
    }
    int32_t h_flag = -1;
    unsigned long long h_total = 0;
    e = cudaMemsetAsync(W.d_cursor[s], 0, sizeof(unsigned long long), st);
    if (e == cudaSuccess) e = launch_k1_filter(S.tmap, mp, S.d_desc, nb, max_strips, n_dirs, ctx->num_sms, st, nullptr);
    if (e == cudaSuccess) e = launch_crosscheck_compact(cp, nb, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(t_flag, 0, sizeof(int32_t), st);
    if (e == cudaSuccess)
      e = launch_compare_matches(t_arena, t_off, t_cnt, W.d_arena[s], W.d_pair_off[s], W.d_pair_cnt[s], nb, t_flag, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&h_flag, t_flag, sizeof(int32_t), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess)
      e = cudaMemcpyAsync(&h_total, W.d_cursor[s], sizeof(unsigned long long), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    drop();
    if (e != cudaSuccess) CU_TRY_R(e);
    // a batch without a single match compares nothing: stay untested (and on the two-direction launch)
    if (h_flag != 0) ctx->k1_dir1_mode = B2M_K1_DIR1_FULL_MISMATCH;
    else if (h_total > 0) ctx->k1_dir1_mode = B2M_K1_DIR1_GATHER;
    ctx->stats.kernel_launches += 10;
    CU_TRY_R(cudaMemsetAsync(W.d_cursor[s], 0, sizeof(unsigned long long), st));
    return B2M_OK;
  };
  // RANSAC + decision of a compacted batch (+ guided re-matching), then its match total to the host
  auto verify_stage = [&](const BatchParams& bp) -> int {
    const int s = bp.s, nb = bp.nb;
    if (tvg)
      if (int rc = verify_batch_launch(ctx, S, tvg, sift, s, bp.p0, nb)) return bail(rc);
    if (tvg && sift->guided_matching) {
      // K1g: re-match the verified pairs under their geometry; the result replaces the inlier matches
      GuidedSlot gs;
      if (int rc = verify_guided_slot(ctx, s, &gs)) return bail(rc);
      GuidedParams gp{};
      gp.kind = gs.kind;
      gp.model = gs.model;
      gp.kpts = S.d_kpts;
      const float me = static_cast<float>(tvg->ransac.max_error);
      gp.max_residual = me * me;
      // cross-check: the column direction only for the matched columns (B2M_GUIDED_DIR1=full: both directions in full)
      const char* guided_env = getenv("B2M_GUIDED_DIR1");
      const bool guided_full = guided_env && !strcmp(guided_env, "full");
      const bool guided_gather = n_dirs == 2 && !guided_full && ensure_gather(ctx) == B2M_OK;
      if (guided_gather)
        CU_TRY_R(launch_k1_guided_gather(S.tmap, W.tmap_gath, bp.mp, gp, S.d_desc, nb, max_strips, gather_scratch(), st));
      else
        CU_TRY_R(launch_k1_guided(S.tmap, bp.mp, gp, nb, max_strips, n_dirs, st));
      CU_TRY_R(cudaMemsetAsync(gs.cursor, 0, sizeof(unsigned long long), st));
      CompactParams gc = bp.cp;
      gc.arena = gs.arena;
      gc.cursor = gs.cursor;
      gc.pair_off = gs.off;
      gc.pair_cnt = gs.cnt;
      gc.kpts = nullptr;
      gc.pts = nullptr;
      gc.enable = gs.kind;
      gc.cand_cnt = nullptr;   // the guided kernel writes final matches, no candidate lists
      gc.colrank = guided_gather ? W.d_colrank : nullptr;
      CU_TRY_R(launch_crosscheck_compact(gc, nb, st));
      CU_TRY_R(cudaMemcpyAsync(gs.h_cursor, gs.cursor, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
      ctx->stats.kernel_launches += guided_gather ? 4 : 2;
    }
    CU_TRY_R(cudaMemcpyAsync(W.h_cursor[s], W.d_cursor[s], sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    CU_TRY_R(cudaEventRecord(ctx->ev_k[s], st));
    return B2M_OK;
  };
  auto stopped = [&]() -> int {
    cudaStreamSynchronize(st);
    cudaStreamSynchronize(ctx->aux_stream);
    cudaStreamSynchronize(ctx->copy_stream);
    ctx->stop = 0;
    return bail(fail(ctx, B2M_ESTOPPED, "[api.cu] stopped by b2m_request_stop"));
  };

  const double hp_t1 = now();
  bool pretested = false;
  if (n_batches > 0 && split_capable && ctx->k1_dir1_mode == B2M_K1_DIR1_UNTESTED) {
    if (int rc = k1_selftest(batch_params(0))) return rc;  // `res` was released by the failing step
    pretested = true;
  }
  // Overlapped order (gathered schedule + verification, the exhaustive pipeline's case): the ALU-only middle of K1
  // (exact resolve of the row direction, gather of the matched columns) needs neither tensor cores nor much of an SM,
  // and the RANSAC kernels of the previous batch leave SMs idle in their tail: the two run side by side.
  //   main stream:  GEMM0(b) | RANSAC + decision(b-1) | wait | GEMM1(b) | resolve1(b) | cross-check + compaction(b)
  //   aux stream:            | resolve0(b) + gather(b) |
  // The batch buffers are double-buffered already (slot b & 1); results drain with a lag of two batches.
  const bool no_overlap = getenv("B2M_NO_OVERLAP") != nullptr;
  pipelined = split_capable && tvg && !sift->guided_matching && n_batches >= 2 && !no_overlap &&
              (ctx->k1_dir1_mode == B2M_K1_DIR1_GATHER || ctx->k1_dir1_mode == B2M_K1_DIR1_GATHER_FORCED);
  if (pipelined) {
    if (int rc = ensure_gather(ctx)) return bail(rc);
    const GatherScratch g = gather_scratch();
    BatchParams prev;
    auto gemm0_time = [&](int s) {
      float t = 0.f;
      if (cudaEventSynchronize(ctx->ev_k1b[s]) == cudaSuccess &&
          cudaEventElapsedTime(&t, ctx->ev_k1a[s], ctx->ev_k1b[s]) == cudaSuccess)
        ctx->stats.last_k1_ms += t;
    };
    for (int64_t b = 0; b < n_batches; ++b) {
      if (ctx->stop) return stopped();
      BatchParams bp = batch_params(b);
      const int s = bp.s, nb = bp.nb;
      if (b >= 2) gemm0_time(s);  // GEMM0 of batch b - 2: complete (the host waited for RANSAC(b - 3) an iteration ago)
      CU_TRY_R(cudaMemsetAsync(W.d_cursor[s], 0, sizeof(unsigned long long), st));
      CU_TRY_R(cudaEventRecord(ctx->ev_k1a[s], st));
      CU_TRY_R(launch_k1_gather_phase(0, S.tmap, W.tmap_gath, bp.mp, S.d_desc, nb, max_strips, ctx->num_sms, g, st));
      CU_TRY_R(cudaEventRecord(ctx->ev_k1b[s], st));
      CU_TRY_R(cudaStreamWaitEvent(ctx->aux_stream, ctx->ev_k1b[s], 0));
      CU_TRY_R(launch_k1_gather_phase(1, S.tmap, W.tmap_gath, bp.mp, S.d_desc, nb, max_strips, ctx->num_sms, g, ctx->aux_stream));
      CU_TRY_R(cudaEventRecord(ctx->ev_p1[s], ctx->aux_stream));
      if (b > 0)
        if (int rc = verify_stage(prev)) return rc;
      // Drain batch b - 2 (same slot as b) while GEMM0(b) keeps the GPU busy: its RANSAC ran an iteration ago, so the
      // host does not wait; the slot's match arena / verification outputs are next written by the compaction below.
      if (b >= 2)
        if (int rc = finish(b - 2)) return bail(rc);
      CU_TRY_R(cudaStreamWaitEvent(st, ctx->ev_p1[s], 0));
      CU_TRY_R(cudaEventRecord(ctx->ev_g2a[s], st));
      CU_TRY_R(launch_k1_gather_phase(2, S.tmap, W.tmap_gath, bp.mp, S.d_desc, nb, max_strips, ctx->num_sms, g, st));
      CU_TRY_R(cudaEventRecord(ctx->ev_g2b[s], st));
      CU_TRY_R(launch_k1_gather_phase(3, S.tmap, W.tmap_gath, bp.mp, S.d_desc, nb, max_strips, ctx->num_sms, g, st));
      bp.cp.colrank = W.d_colrank;
      CU_TRY_R(launch_crosscheck_compact(bp.cp, nb, st));
      ctx->stats.kernel_launches += 7;
      ctx->stats.last_k1_launches += 1;
      ctx->stats.k1_dir1_mode = static_cast<uint64_t>(ctx->k1_dir1_mode);
      prev = bp;
    }
    if (int rc = verify_stage(prev)) return rc;
    gemm0_time(static_cast<int>((n_batches - 1) & 1));   // the last two batches' GEMM0 launches
    gemm0_time(static_cast<int>((n_batches - 2) & 1));
  } else {
  for (int64_t b = 0; b < n_batches; ++b) {
    if (ctx->stop) return stopped();
    BatchParams bp = batch_params(b);
    const int s = bp.s, nb = bp.nb;
    MatchParams& mp = bp.mp;
    CompactParams& cp = bp.cp;
    if (b >= 2) CU_TRY_R(cudaStreamWaitEvent(st, ctx->ev_data[s], 0));
    CU_TRY_R(cudaMemsetAsync(W.d_cursor[s], 0, sizeof(unsigned long long), st));
    if (split_capable && ctx->k1_dir1_mode == B2M_K1_DIR1_UNTESTED && !(b == 0 && pretested))
      if (int rc = k1_selftest(bp)) return rc;  // `res` was released by the failing step
    const bool use_gather = split_capable && (ctx->k1_dir1_mode == B2M_K1_DIR1_GATHER || ctx->k1_dir1_mode == B2M_K1_DIR1_GATHER_FORCED);
    const bool use_skip = split_capable && (ctx->k1_dir1_mode == B2M_K1_DIR1_SKIP || ctx->k1_dir1_mode == B2M_K1_DIR1_SKIP_FORCED);
    if (use_gather)
      if (int rc = ensure_gather(ctx)) return bail(rc);
    CU_TRY_R(cudaEventRecord(ctx->ev_k1a[s], st));
    if (ctx->exact_k1) {
      CU_TRY_R(launch_k1_match(S.tmap, mp, nb, max_strips, n_dirs, st));
    } else if (use_gather) {
      CU_TRY_R(launch_k1_filter_gather(S.tmap, W.tmap_gath, mp, S.d_desc, nb, max_strips, ctx->num_sms, gather_scratch(), st,
                                       ctx->ev_k1b[s]));
      cp.colrank = W.d_colrank;
      ctx->stats.kernel_launches += 4;  // second GEMM launch, gather, two resolves instead of one
    } else if (use_skip) {
      CU_TRY_R(launch_k1_filter_skip(S.tmap, mp, S.d_desc, nb, max_strips, ctx->num_sms, W.d_pairs_dir1, S.n_images, st,
                                     ctx->ev_k1b[s]));
      ctx->stats.kernel_launches += 3;  // second GEMM launch, pair selection, resolve
    } else {
      CU_TRY_R(launch_k1_filter(S.tmap, mp, S.d_desc, nb, max_strips, n_dirs, ctx->num_sms, st,
                                ctx->ev_k1b[s]));
      ctx->stats.kernel_launches += 1;
    }
    if (ctx->exact_k1) CU_TRY_R(cudaEventRecord(ctx->ev_k1b[s], st));
    ctx->stats.kernel_launches += 1;
    ctx->stats.last_k1_launches += 1;
    ctx->stats.k1_dir1_mode = static_cast<uint64_t>(ctx->k1_dir1_mode);
    CU_TRY_R(launch_crosscheck_compact(cp, nb, st));
    ctx->stats.kernel_launches += 1;
    if (int rc = verify_stage(bp)) return rc;
    if (b > 0)
      if (int rc = finish(b - 1)) return bail(rc);
  }
  }
  const double hp_t2 = now();
  if (pipelined && n_batches >= 2)
    if (int rc = finish(n_batches - 2)) return bail(rc);
  if (n_batches > 0)
    if (int rc = finish(n_batches - 1)) return bail(rc);
  CU_TRY_R(cudaEventRecord(ctx->ev_t1, st));
  CU_TRY_R(cudaEventSynchronize(ctx->ev_t1));
  float ms = 0.f;
  cudaEventElapsedTime(&ms, ctx->ev_t0, ctx->ev_t1);
  ctx->stats.last_total_ms = ms;
  if (pipelined) verify_ms = std::max(0.0, static_cast<double>(ms) - ctx->stats.last_k1_ms);
  ctx->stats.last_verify_ms = verify_ms;
  ctx->stats.last_match_ms = ms - verify_ms;
#undef CU_TRY_R
  if (host_prof)
    fprintf(stderr, "[b2m hostprof] pairs %lld: set-up %.1f ms, launch loop %.1f ms, last batch + sync %.1f ms, device %.1f ms\n",
            static_cast<long long>(n_pairs), hp_t1 - hp_t0, hp_t2 - hp_t1, now() - hp_t2, ms);
  ctx->hint_matches = res->matches.size() / 2;
  ctx->hint_inliers = res->inliers.size() / 2;
  *out = res;
  return B2M_OK;
}

}  // namespace

b2m_results::~b2m_results() {
  constexpr size_t kWorthIt = size_t{1} << 20;   // elements: below 4 MB the allocator's own free lists do
  if (!host_cache_enabled() || (matches.capacity() < kWorthIt && inliers.capacity() < kWorthIt)) return;
  HostCache& hc = host_cache();
  std::lock_guard<std::mutex> lk(hc.mu);
  if (matches.capacity() > hc.matches.capacity()) matches.swap(hc.matches);
  if (inliers.capacity() > hc.inliers.capacity()) inliers.swap(hc.inliers);
}

namespace b2m {
void ImageSet::release() {
  if (d_desc) cudaFree(d_desc);
  if (d_kpts) cudaFree(d_kpts);
  if (d_row0) cudaFree(d_row0);
  if (d_nfeat) cudaFree(d_nfeat);
  d_desc = nullptr;
  d_kpts = nullptr;
  d_row0 = nullptr;
  d_nfeat = nullptr;
  n_images = 0;
  nfeat.clear();
  row0.clear();
  cams.clear();
  max_feat = max_feat_pad = 0;
  total_rows = 0;
}
void Workspace::release() {
  if (d_mbuf) cudaFree(d_mbuf);
  if (d_aux) cudaFree(d_aux);
  if (d_cand_cnt) cudaFree(d_cand_cnt);
  if (d_cand_rows) cudaFree(d_cand_rows);
  if (d_cand_sorted) cudaFree(d_cand_sorted);
  if (d_pairs_dir1) cudaFree(d_pairs_dir1);
  d_pairs_dir1 = nullptr;
  cudaFree(d_gath_desc); cudaFree(d_colrank); cudaFree(d_gath_cols); cudaFree(d_gath_cnt); cudaFree(d_gath_items);
  cudaFree(d_gath_n);
  d_gath_desc = nullptr; d_colrank = nullptr; d_gath_cols = nullptr; d_gath_cnt = nullptr; d_gath_items = nullptr;
  d_gath_n = nullptr;
  d_cand_sorted = nullptr;
  d_mbuf = nullptr;
  d_aux = nullptr;
  d_cand_cnt = nullptr;
  d_cand_rows = nullptr;
  for (int s = 0; s < 2; ++s) {
    if (d_arena[s]) cudaFree(d_arena[s]);
    if (d_cursor[s]) cudaFree(d_cursor[s]);
    if (d_pair_off[s]) cudaFree(d_pair_off[s]);
    if (d_pair_cnt[s]) cudaFree(d_pair_cnt[s]);
    if (h_arena[s]) cudaFreeHost(h_arena[s]);
    if (h_cursor[s]) cudaFreeHost(h_cursor[s]);
    if (h_pair_off[s]) cudaFreeHost(h_pair_off[s]);
    if (h_pair_cnt[s]) cudaFreeHost(h_pair_cnt[s]);
    d_arena[s] = nullptr;
    d_cursor[s] = nullptr;
    d_pair_off[s] = nullptr;
    d_pair_cnt[s] = nullptr;
    h_arena[s] = nullptr;
    h_cursor[s] = nullptr;
    h_pair_off[s] = nullptr;
    h_pair_cnt[s] = nullptr;
  }
  batch = 0;
  mstride = 0;
}
}  // namespace b2m

extern "C" {

int b2m_abi_version(void) { return B2M_ABI_VERSION; }

int b2m_device_count(void) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  int n = 0;
  for (int d = 0; d < ndev; ++d) {
    int major = 0, minor = 0;
    if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, d) == cudaSuccess &&
        cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, d) == cudaSuccess && major == 9 && minor == 0)
      n = d + 1;
  }
  return n;
}

void b2m_sift_opts_default(b2m_sift_opts* o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->struct_size = sizeof(*o);
  o->max_ratio = 0.8f;
  o->max_distance = 0.7f;
  o->cross_check = 1;
  o->max_num_matches = 32768;
  o->guided_matching = 0;
}
void b2m_ransac_opts_default(b2m_ransac_opts* o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->struct_size = sizeof(*o);
  o->min_num_trials = 100;
  o->max_num_trials = 10000;
  o->max_error = 4.0;
  o->min_inlier_ratio = 0.25;
  o->confidence = 0.999;
  o->dyn_num_trials_multiplier = 3.0;
}
void b2m_tvg_opts_default(b2m_tvg_opts* o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->struct_size = sizeof(*o);
  o->min_num_inliers = 15;
  o->min_E_F_inlier_ratio = 0.95;
  o->max_H_inlier_ratio = 0.8;
  o->watermark_min_inlier_ratio = 0.7;
  o->watermark_border_size = 0.1;
  o->detect_watermark = 1;
  o->multiple_ignore_watermark = 1;
  o->force_H_use = 0;
  o->compute_relative_pose = 0;
  o->multiple_models = 0;
  b2m_ransac_opts_default(&o->ransac);
}

int b2m_create(const b2m_device_cfg* cfg, b2m_ctx** out) {
  if (!out) return fail(nullptr, B2M_EINVAL, "[api.cu] Check Failed: out != NULL");
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(nullptr, B2M_ENODEV,
                "[api.cu] no CUDA device visible: libb200match has no CPU fallback (H100 / sm_90 required)");
  }
  const int dev = cfg ? cfg->device : 0;
  if (dev < 0 || dev >= ndev) return fail(nullptr, B2M_EINVAL, "[api.cu] Check Failed: device ordinal in range");
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return fail(nullptr, B2M_ECUDA, "cudaGetDeviceProperties");
  if (prop.major != 9 || prop.minor != 0) {
    char b[256];
    snprintf(b, sizeof(b), "[api.cu] device %d is sm_%d%d; this library is built for sm_90a only", dev, prop.major,
             prop.minor);
    return fail(nullptr, B2M_ENODEV, b);
  }
  b2m_ctx* ctx = new (std::nothrow) b2m_ctx();
  if (!ctx) return fail(nullptr, B2M_ENOMEM, "out of host memory");
  ctx->device = dev;
  ctx->num_sms = prop.multiProcessorCount;
  ctx->seed = cfg ? cfg->seed : 0;
  if (cfg && cfg->pair_batch > 0) {
    ctx->pair_batch = std::min(cfg->pair_batch, 65535);
    ctx->pair_batch_auto = false;
  }
  ctx->stats.struct_size = sizeof(b2m_stats);
#define CU_TRY_C(expr)                                                            \
  do {                                                                            \
    cudaError_t _e = (expr);                                                      \
    if (_e != cudaSuccess) {                                                      \
      std::string m = std::string("[api.cu] CUDA error in b2m_create: ") + cudaGetErrorString(_e); \
      delete ctx;                                                                 \
      return fail(nullptr, B2M_ECUDA, m);                                         \
    }                                                                             \
  } while (0)
  CU_TRY_C(cudaSetDevice(dev));
  CU_TRY_C(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
  CU_TRY_C(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
  CU_TRY_C(cudaStreamCreateWithFlags(&ctx->aux_stream, cudaStreamNonBlocking));
  for (int s = 0; s < 2; ++s) {
    CU_TRY_C(cudaEventCreate(&ctx->ev_k[s]));
    CU_TRY_C(cudaEventCreateWithFlags(&ctx->ev_data[s], cudaEventDisableTiming));
  }
  for (int s = 0; s < 2; ++s) {
    CU_TRY_C(cudaEventCreate(&ctx->ev_k1a[s]));
    CU_TRY_C(cudaEventCreate(&ctx->ev_k1b[s]));
    CU_TRY_C(cudaEventCreateWithFlags(&ctx->ev_p1[s], cudaEventDisableTiming));
    CU_TRY_C(cudaEventCreate(&ctx->ev_g2a[s]));
    CU_TRY_C(cudaEventCreate(&ctx->ev_g2b[s]));
  }
  CU_TRY_C(cudaEventCreate(&ctx->ev_t0));
  CU_TRY_C(cudaEventCreate(&ctx->ev_t1));
  // acos LUT: the float32 accept test of FindBestMatchesOneWayBruteForce depends only on the
  // integer dot product d in [0, 2^18] (clamped); tabulating it with the HOST libm makes the
  // device decisions identical to a CPU run on the same machine.
  {
    std::vector<float> lut(262145);
    const float kDistNorm = 1.0f / (512.0f * 512.0f);
    for (int d = 0; d <= 262144; ++d) lut[d] = acosf(std::min(kDistNorm * static_cast<float>(d), 1.0f));
    // K1 v2 rejects rows against a lower bound of the second-best dot product, which is exact only
    // if the tabulated acos is non-increasing; otherwise (or on request) use the exact epilogue.
    bool monotone = true;
    for (int d = 1; d <= 262144; ++d) monotone &= (lut[d] <= lut[d - 1]);
    const char* env = getenv("B2M_EXACT_K1");
    ctx->exact_k1 = !monotone || (env && env[0] == '1');
    const char* d1 = getenv("B2M_K1_DIR1");  // full | skip: bypass the one-time comparison (profiling, A/B runs)
    if (d1 && !strcmp(d1, "full")) ctx->k1_dir1_mode = B2M_K1_DIR1_FULL_FORCED;
    if (d1 && !strcmp(d1, "skip")) ctx->k1_dir1_mode = B2M_K1_DIR1_SKIP_FORCED;
    if (d1 && !strcmp(d1, "gather")) ctx->k1_dir1_mode = B2M_K1_DIR1_GATHER_FORCED;
    CU_TRY_C(cudaMalloc(&ctx->d_lut, sizeof(float) * lut.size()));
    CU_TRY_C(cudaMemcpy(ctx->d_lut, lut.data(), sizeof(float) * lut.size(), cudaMemcpyHostToDevice));
  }
#undef CU_TRY_C
  *out = ctx;
  return B2M_OK;
}

void b2m_destroy(b2m_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  comm_release(ctx);
  if (ctx->d_verify_counters) cudaFree(ctx->d_verify_counters);
  ctx->images.release();
  ctx->ws.release();
  verify_release(ctx);
  if (ctx->d_pairs) cudaFree(ctx->d_pairs);
  if (ctx->d_lut) cudaFree(ctx->d_lut);
  for (int s = 0; s < 2; ++s) {
    if (ctx->ev_k[s]) cudaEventDestroy(ctx->ev_k[s]);
    if (ctx->ev_data[s]) cudaEventDestroy(ctx->ev_data[s]);
    if (ctx->ev_k1a[s]) cudaEventDestroy(ctx->ev_k1a[s]);
    if (ctx->ev_k1b[s]) cudaEventDestroy(ctx->ev_k1b[s]);
    if (ctx->ev_p1[s]) cudaEventDestroy(ctx->ev_p1[s]);
    if (ctx->ev_g2a[s]) cudaEventDestroy(ctx->ev_g2a[s]);
    if (ctx->ev_g2b[s]) cudaEventDestroy(ctx->ev_g2b[s]);
  }
  if (ctx->ev_t0) cudaEventDestroy(ctx->ev_t0);
  if (ctx->ev_t1) cudaEventDestroy(ctx->ev_t1);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
  if (ctx->aux_stream) cudaStreamDestroy(ctx->aux_stream);
  delete ctx;
}

const char* b2m_last_error(const b2m_ctx* ctx) { return ctx ? ctx->err.c_str() : g_noctx_err.c_str(); }

int b2m_request_stop(b2m_ctx* ctx) {
  if (!ctx) return B2M_EINVAL;
  ctx->stop = 1;
  return B2M_OK;
}

static int set_images_impl(b2m_ctx* ctx, int32_t n_images, const int32_t* n_feat, const uint8_t* const* desc,
                   const float* const* kpts, const b2m_camera* cams) {
  if (!ctx) return B2M_EINVAL;
  if (n_images < 0 || (n_images > 0 && (!n_feat || !desc)))
    return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: n_images >= 0 && n_feat && desc");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  ImageSet& S = ctx->images;
  if (int rc = layout_images(ctx, S, n_images, n_feat, kpts != nullptr)) return rc;
  for (int i = 0; i < n_images; ++i) {
    if (n_feat[i] == 0) continue;
    if (!desc[i]) return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: desc[i] != NULL");
    CU_TRY(ctx, cudaMemcpyAsync(S.d_desc + static_cast<size_t>(S.row0[i]) * 128, desc[i],
                                static_cast<size_t>(n_feat[i]) * 128, cudaMemcpyHostToDevice, ctx->stream));
    if (kpts) {
      if (!kpts[i]) return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: kpts[i] != NULL");
      CU_TRY(ctx, cudaMemcpyAsync(S.d_kpts + S.row0[i], kpts[i], static_cast<size_t>(n_feat[i]) * sizeof(float2),
                                  cudaMemcpyHostToDevice, ctx->stream));
    }
  }
  if (cams) {
    for (int i = 0; i < n_images; ++i)
      if (const char* why = camera_problem(cams[i])) return fail(ctx, B2M_EINVAL, why);
    S.cams.assign(cams, cams + n_images);
  }
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return B2M_OK;
}

int b2m_set_images(b2m_ctx* ctx, int32_t n_images, const int32_t* n_feat, const uint8_t* const* desc,
                   const float* const* kpts, const b2m_camera* cams) {
  const int rc = set_images_impl(ctx, n_images, n_feat, desc, kpts, cams);
  if (rc != B2M_OK && ctx) ctx->images.release();  // never leave a half-uploaded set behind
  return rc;
}

static int set_images_device_impl(b2m_ctx* ctx, int32_t n_images, const int32_t* n_feat, const void* dev_desc_packed,
                          const void* dev_kpts_packed, const b2m_camera* cams) {
  if (!ctx) return B2M_EINVAL;
  if (n_images < 0 || (n_images > 0 && (!n_feat || !dev_desc_packed)))
    return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: n_images >= 0 && n_feat && dev_desc_packed");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  ImageSet& S = ctx->images;
  if (int rc = layout_images(ctx, S, n_images, n_feat, dev_kpts_packed != nullptr)) return rc;
  int64_t src_row = 0;
  const uint8_t* src = static_cast<const uint8_t*>(dev_desc_packed);
  const float2* ksrc = static_cast<const float2*>(dev_kpts_packed);
  // contiguous runs of images whose counts are multiples of kRowPad are copied in one go
  int i = 0;
  while (i < n_images) {
    int j = i;
    int64_t run = 0;
    while (j < n_images && n_feat[j] % kRowPad == 0) run += n_feat[j++];
    if (j == i) {  // ragged image
      run = n_feat[i];
      j = i + 1;
    }
    if (run > 0) {
      CU_TRY(ctx, cudaMemcpyAsync(S.d_desc + static_cast<size_t>(S.row0[i]) * 128, src + src_row * 128,
                                  static_cast<size_t>(run) * 128, cudaMemcpyDeviceToDevice, ctx->stream));
      if (ksrc)
        CU_TRY(ctx, cudaMemcpyAsync(S.d_kpts + S.row0[i], ksrc + src_row, static_cast<size_t>(run) * sizeof(float2),
                                    cudaMemcpyDeviceToDevice, ctx->stream));
    }
    src_row += run;
    i = j;
  }
  if (cams) {
    for (int i = 0; i < n_images; ++i)
      if (const char* why = camera_problem(cams[i])) return fail(ctx, B2M_EINVAL, why);
    S.cams.assign(cams, cams + n_images);
  }
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return B2M_OK;
}

int b2m_set_images_device(b2m_ctx* ctx, int32_t n_images, const int32_t* n_feat, const void* dev_desc_packed,
                          const void* dev_kpts_packed, const b2m_camera* cams) {
  const int rc = set_images_device_impl(ctx, n_images, n_feat, dev_desc_packed, dev_kpts_packed, cams);
  if (rc != B2M_OK && ctx) ctx->images.release();  // never leave a half-uploaded set behind
  return rc;
}

static int set_images_sharded_impl(b2m_ctx* ctx, int32_t n_images, const int32_t* n_feat, const b2m_camera* cams,
                           const b2m_image_shard* mine) {
  if (!ctx) return B2M_EINVAL;
  if (n_images < 0 || (n_images > 0 && !n_feat) || !mine || mine->struct_size != sizeof(b2m_image_shard))
    return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: n_images >= 0 && n_feat && shard (struct_size)");
  int32_t first = 0, count = 0;
  b2m_comm_image_range(n_images, ctx->comm_size, ctx->comm_rank, &first, &count);
  if (mine->first_image != first || mine->n_local != count)
    return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: the shard is this rank's b2m_comm_image_range");
  if (count > 0 && !mine->desc_packed) return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: desc_packed != NULL");
  if (count > 0 && mine->has_keypoints && !mine->kpts_packed)
    return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: kpts_packed != NULL");
  if (mine->location != B2M_LOC_HOST && mine->location != B2M_LOC_DEVICE)
    return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: location is B2M_LOC_HOST or B2M_LOC_DEVICE");
  if (cams)
    for (int i = 0; i < n_images; ++i)
      if (const char* why = camera_problem(cams[i])) return fail(ctx, B2M_EINVAL, why);
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  ImageSet& S = ctx->images;
  const bool kp = mine->has_keypoints != 0;
  if (int rc = layout_images(ctx, S, n_images, n_feat, kp)) return rc;
  cudaStream_t st = ctx->stream;
  const cudaMemcpyKind kind = mine->location == B2M_LOC_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
  CU_TRY(ctx, cudaEventRecord(ctx->ev_t0, st));
  {  // the local shard -> its rows; runs of images without padding go in one copy
    const uint8_t* src = static_cast<const uint8_t*>(mine->desc_packed);
    const float2* ksrc = static_cast<const float2*>(mine->kpts_packed);
    int64_t src_row = 0;
    int i = first;
    while (i < first + count) {
      int j = i;
      int64_t run = 0;
      while (j < first + count && n_feat[j] % kRowPad == 0) run += n_feat[j++];
      if (j == i) {
        run = n_feat[i];
        j = i + 1;
      }
      if (run > 0) {
        CU_TRY(ctx, cudaMemcpyAsync(S.d_desc + static_cast<size_t>(S.row0[i]) * 128, src + src_row * 128,
                                    static_cast<size_t>(run) * 128, kind, st));
        if (kp)
          CU_TRY(ctx, cudaMemcpyAsync(S.d_kpts + S.row0[i], ksrc + src_row, static_cast<size_t>(run) * sizeof(float2), kind, st));
      }
      src_row += run;
      i = j;
    }
  }
  CU_TRY(ctx, cudaEventRecord(ctx->ev_k1a[0], st));
  uint64_t recv_bytes = 0;
  if (ctx->comm && ctx->comm_size > 1) {
    // ONE all-gather of the descriptor rows (and one of the keypoint rows): rank r owns the padded rows of its images
    const int nr = ctx->comm_size;
    std::vector<size_t> off(nr), len(nr);
    auto row_at = [&](int img) { return img < n_images ? static_cast<int64_t>(S.row0[img]) : S.total_rows; };
    for (int r = 0; r < nr; ++r) {
      int32_t f = 0, c = 0;
      b2m_comm_image_range(n_images, nr, r, &f, &c);
      off[r] = static_cast<size_t>(row_at(f));
      len[r] = static_cast<size_t>(row_at(f + c) - row_at(f));
      if (r != ctx->comm_rank) recv_bytes += len[r] * (128 + (kp ? sizeof(float2) : 0));
    }
    std::vector<size_t> o(nr), l(nr);
    for (int r = 0; r < nr; ++r) { o[r] = off[r] * 128; l[r] = len[r] * 128; }
    if (int rc = comm_allgather_regions(ctx, S.d_desc, o, l, st)) return rc;
    if (kp) {
      for (int r = 0; r < nr; ++r) { o[r] = off[r] * sizeof(float2); l[r] = len[r] * sizeof(float2); }
      if (int rc = comm_allgather_regions(ctx, reinterpret_cast<uint8_t*>(S.d_kpts), o, l, st)) return rc;
    }
  }
  CU_TRY(ctx, cudaEventRecord(ctx->ev_k1b[0], st));
  if (cams) S.cams.assign(cams, cams + n_images);
  CU_TRY(ctx, cudaStreamSynchronize(st));
  float up = 0.f, ag = 0.f;
  cudaEventElapsedTime(&up, ctx->ev_t0, ctx->ev_k1a[0]);
  cudaEventElapsedTime(&ag, ctx->ev_k1a[0], ctx->ev_k1b[0]);
  ctx->stats.last_upload_ms = up;
  ctx->stats.last_allgather_ms = (ctx->comm && ctx->comm_size > 1) ? ag : 0.0;
  ctx->stats.last_allgather_bytes = recv_bytes;
  return B2M_OK;
}

int b2m_set_images_sharded(b2m_ctx* ctx, int32_t n_images, const int32_t* n_feat, const b2m_camera* cams,
                           const b2m_image_shard* mine) {
  const int rc = set_images_sharded_impl(ctx, n_images, n_feat, cams, mine);
  if (rc != B2M_OK && ctx) ctx->images.release();  // never leave a half-uploaded set behind
  return rc;
}

int b2m_match_pairs(b2m_ctx* ctx, const int32_t* pairs, int64_t n_pairs, const b2m_sift_opts* sift,
                    const b2m_tvg_opts* tvg, b2m_results** out) {
  if (!ctx) return B2M_EINVAL;
  cudaSetDevice(ctx->device);
  return match_pairs_impl(ctx, ctx->images, pairs, n_pairs, sift, tvg, out);
}

int b2m_match_verify(b2m_ctx* ctx, const int32_t* pairs, int64_t n_pairs, const b2m_sift_opts* sift,
                     const b2m_tvg_opts* tvg, b2m_results** out) {
  return b2m_match_pairs(ctx, pairs, n_pairs, sift, tvg, out);
}

int b2m_match_pair(b2m_ctx* ctx, const uint8_t* desc1, int32_t n1, const uint8_t* desc2, int32_t n2,
                   const b2m_sift_opts* opts, uint32_t* out_matches, int64_t cap, int64_t* out_n) {
  if (!ctx) return B2M_EINVAL;
  if (!out_n) return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: out_n != NULL");
  *out_n = 0;
  if (n1 < 0 || n2 < 0) return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: n1 >= 0 && n2 >= 0");
  if (int rc = check_sift(ctx, opts)) return rc;
  if (n1 == 0 || n2 == 0) return B2M_OK;
  if (!desc1 || !desc2) return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: descriptors != NULL");
  cudaSetDevice(ctx->device);
  // a private two-image set; the resident set of the context is left untouched
  ImageSet tmp;
  const int32_t nf[2] = {n1, n2};
  std::swap(tmp, ctx->images);
  const uint8_t* d[2] = {desc1, desc2};
  int rc = b2m_set_images(ctx, 2, nf, d, nullptr, nullptr);
  b2m_results* res = nullptr;
  const int32_t pr[2] = {0, 1};
  if (rc == B2M_OK) rc = match_pairs_impl(ctx, ctx->images, pr, 1, opts, nullptr, &res);
  ctx->images.release();
  std::swap(tmp, ctx->images);
  if (rc != B2M_OK) return rc;
  const int64_t n = res->cnt[0];
  if (n > cap || (n > 0 && !out_matches)) {
    delete res;
    return fail(ctx, B2M_EINVAL, "[api.cu] Check Failed: out_matches capacity");
  }
  if (n > 0) memcpy(out_matches, res->matches.data() + 2 * res->off[0], sizeof(uint32_t) * 2 * n);
  *out_n = n;
  delete res;
  return B2M_OK;
}

int64_t b2m_results_num_pairs(const b2m_results* r) { return r ? static_cast<int64_t>(r->cnt.size()) : 0; }
int64_t b2m_results_total_matches(const b2m_results* r) { return r ? static_cast<int64_t>(r->matches.size() / 2) : 0; }

int64_t b2m_results_num_verified(const b2m_results* r) {
  if (!r || !r->verified) return 0;
  int64_t n = 0;
  for (int32_t c : r->config) n += (c != B2M_UNDEFINED);
  return n;
}

int b2m_results_get(const b2m_results* r, int64_t pair, b2m_pair_view* out) {
  if (!r || !out || pair < 0 || pair >= static_cast<int64_t>(r->cnt.size())) return B2M_EINVAL;
  memset(out, 0, sizeof(*out));
  out->struct_size = sizeof(*out);
  out->image1 = r->pairs[2 * pair];
  out->image2 = r->pairs[2 * pair + 1];
  out->n_matches = r->cnt[pair];
  out->matches = r->cnt[pair] ? r->matches.data() + 2 * r->off[pair] : nullptr;
  out->config = B2M_UNDEFINED;
  if (r->verified) {
    out->config = r->config[pair];
    out->n_inliers = r->in_cnt[pair];
    out->inlier_matches = r->in_cnt[pair] ? r->inliers.data() + 2 * r->in_off[pair] : nullptr;
    if (r->model_idx[pair] >= 0) {
      const double* m = r->models.data() + 27 * static_cast<size_t>(r->model_idx[pair]);
      memcpy(out->E, m, sizeof(double) * 9);
      memcpy(out->F, m + 9, sizeof(double) * 9);
      memcpy(out->H, m + 18, sizeof(double) * 9);
    }
  }
  out->qvec[0] = 1.0;
  if (r->verified && !r->pose_valid.empty() && r->pose_valid[pair]) {
    memcpy(out->qvec, r->poses.data() + 8 * pair, sizeof(double) * 4);
    memcpy(out->tvec, r->poses.data() + 8 * pair + 4, sizeof(double) * 3);
    out->tri_angle = r->poses[8 * pair + 7];
    out->pose_valid = 1;
  }
  return B2M_OK;
}

void b2m_results_free(b2m_results* r) { delete r; }

int b2m_get_stats(b2m_ctx* ctx, b2m_stats* out) {
  if (!ctx || !out) return B2M_EINVAL;
  *out = ctx->stats;
  out->struct_size = sizeof(b2m_stats);
  out->comm_size = ctx->comm_size;
  out->comm_rank = ctx->comm_rank;
  if (ctx->d_verify_counters) {  // kernel-side counters of the verifier (models scored, residual evaluations per kind)
    unsigned long long h[6] = {0, 0, 0, 0, 0, 0};
    cudaSetDevice(ctx->device);
    if (cudaMemcpy(h, ctx->d_verify_counters, sizeof(h), cudaMemcpyDeviceToHost) == cudaSuccess)
      for (int k = 0; k < 3; ++k) {
        out->verify_models_scored[k] = h[k];
        out->verify_residuals[k] = h[3 + k];
      }
  }
  return B2M_OK;
}
int b2m_reset_stats(b2m_ctx* ctx) {
  if (!ctx) return B2M_EINVAL;
  memset(&ctx->stats, 0, sizeof(ctx->stats));
  ctx->stats.struct_size = sizeof(b2m_stats);
  if (ctx->d_verify_counters) {
    cudaSetDevice(ctx->device);
    cudaMemset(ctx->d_verify_counters, 0, sizeof(unsigned long long) * 6);
  }
  ctx->stats.k1_dir1_mode = static_cast<uint64_t>(ctx->k1_dir1_mode);  // a property of the context, not a counter
  return B2M_OK;
}

}  // extern "C"
