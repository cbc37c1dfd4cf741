// verify.cu -- K2/K3: batched LO-RANSAC two-view geometric verification (E 5-pt, F 7-pt + 8-pt LO,
// H 4-pt DLT), decision tree, inlier extraction and watermark detection, plus the stand-alone
// estimator entry points of the C ABI.
//
// One CTA per (image pair, model kind).  Inside a CTA a round evaluates up to 128 minimal-sample
// hypotheses at once (thread = hypothesis for the solver, warp = model for the residual scoring
// with coalesced double4 loads and shuffle reductions), the best of the round goes through the
// recursive local optimisation (N-point refits from parallel normal-equation reductions), and the
// dynamic trial bound of U:optim/ransac.h terminates the loop.  Sampling is counter-based
// (seed, image ids, kind, trial) so results do not depend on batching or sharding.
//
// Semantics: U:estimators/two_view_geometry.cc (EstimateTwoViewGeometry, EstimateCalibrated...,
// EstimateUncalibrated..., DetectWatermark, ExtractInlierMatches), U:optim/loransac.h, reached from
// R:pipeline/match_features.h:45-48 (VerifierWorker) and R:estimators/two_view_geometry.h:95-151.
// SURVEY.md section 8 rows V1-V9.  RANSAC parity vs the sequential reference is statistical
// (+-1% inliers), as it is between two runs of the reference itself.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "geom.h"
#include "eig_warp.cuh"
#include "five_point_warp.cuh"
#include "pose.h"
#include "verify.cuh"

namespace b2m {

namespace {

using namespace geom;

constexpr int kRansacThreads = 128;
constexpr int kMaxLocalTrials = 10;

struct DevCamera {
  double fx, fy, cx, cy;
  double mean_f;
  int32_t width, height;
  int32_t has_prior;
  int32_t distorted;  // model has a distortion function: the E kernel reads undistorted points (see b2m_undistort_kernel)
};

// Full model of a camera, read only by the undistortion kernel.
struct DevDistortion {
  int32_t model;
  int32_t pad;
  double p[cam::kMaxParams];
};

struct VerifyParams {
  const int32_t* pairs;       // [nb x 2] image indices
  const int64_t* pair_off;    // [nb] offset into the arenas
  const int32_t* pair_cnt;    // [nb] matches of the pair
  const double4* pts;         // arena: (x1, y1, x2, y2) pixel coordinates of each raw match
  const uint2* matches;       // arena: raw matches
  const DevCamera* cams;      // per image
  uint8_t* mask;              // [3][arena_cap] inlier masks per kind
  int64_t arena_cap;
  double* models;             // [nb][3][9]
  int32_t* sup_cnt;           // [nb][3]
  int32_t* success;           // [nb][3]
  // outputs of the decision kernel
  int32_t* config;            // [nb]
  int32_t* inl_cnt;           // [nb]
  uint2* inliers;             // arena (same offsets as matches)
  // options
  b2m_tvg_opts opt;
  uint64_t seed;
  int32_t single_kind;        // >= 0: only this kind runs (stand-alone estimator API), no camera model
  int32_t force_calibrated;   // stand-alone: -1 use camera flags
  unsigned long long* prof;   // optional [3][8] cycle counters (B2M_PROF=1), else nullptr
  unsigned long long* counters;  // [6] models scored / residual evaluations per kind (b2m_stats), or nullptr
  int32_t lo_eig_thread;      // A/B switch B2M_LO_EIG=thread: serial eigen-solve of the LO refits (default: one warp)
  double* e_scratch;          // E kernel, warp / hybrid minimal solves: [nb][kRansacThreads][kEStride] (models, N, polynomial, Mr)
  // guided matching hand-over (written by the decision kernel when guided_min_inliers >= 0)
  int32_t* guided_kind;       // [nb] -1 / 0 (F) / 1 (H)
  float* guided_model;        // [nb][9]
  int32_t guided_min_inliers; // < 0: guided matching off
};

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

__device__ __forceinline__ double shfl_d(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }
__device__ __forceinline__ double warp_sum_d(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// residual of point i under `model` for problem kind (0 = E on normalised coordinates)
struct PointXform {
  double ax1, bx1, ay1, by1, ax2, bx2, ay2, by2;  // n = a * p + b  (identity for F / H)
};
__device__ __forceinline__ void load_pt(const double4* pts, int64_t i, const PointXform& X, double& x1, double& y1,
                                        double& x2, double& y2) {
  const double4 p = pts[i];
  x1 = X.ax1 * p.x + X.bx1;
  y1 = X.ay1 * p.y + X.by1;
  x2 = X.ax2 * p.z + X.bx2;
  y2 = X.ay2 * p.w + X.by2;
}
template <int KIND>
__device__ __forceinline__ double residual(const double* M, double x1, double y1, double x2, double y2) {
  if (KIND == 2) return homography_sq(M, x1, y1, x2, y2);
  return sampson_sq(M, x1, y1, x2, y2);
}

// Division-free fp32 inlier test used by the hypothesis-scoring loop: r <= thr  <=>  lhs <= thr * rhs
// with r = lhs / rhs.  Returns +1 inlier, 0 outlier, -1 borderline (within 1 % of the threshold, or
// not finite): the caller re-evaluates those in fp64, so decisions equal the fp64 evaluation.
template <int KIND>
__device__ __forceinline__ int inlier_f32(const float* M, float x1, float y1, float x2, float y2, float thr) {
  float lhs, rhs;
  if (KIND == 2) {
    const float u = fmaf(M[0], x1, fmaf(M[1], y1, M[2]));
    const float v = fmaf(M[3], x1, fmaf(M[4], y1, M[5]));
    const float w = fmaf(M[6], x1, fmaf(M[7], y1, M[8]));
    const float ex = fmaf(x2, w, -u), ey = fmaf(y2, w, -v);
    lhs = fmaf(ex, ex, ey * ey);
    rhs = thr * w * w;
  } else {
    const float a0 = fmaf(M[0], x1, fmaf(M[1], y1, M[2]));
    const float a1 = fmaf(M[3], x1, fmaf(M[4], y1, M[5]));
    const float a2 = fmaf(M[6], x1, fmaf(M[7], y1, M[8]));
    const float b0 = fmaf(M[0], x2, fmaf(M[3], y2, M[6]));
    const float b1 = fmaf(M[1], x2, fmaf(M[4], y2, M[7]));
    const float num = fmaf(x2, a0, fmaf(y2, a1, a2));
    lhs = num * num;
    rhs = thr * fmaf(a0, a0, fmaf(a1, a1, fmaf(b0, b0, b1 * b1)));
  }
  // STRICT comparisons: lhs == rhs == 0 (both underflowed) or == inf (both overflowed) is neither clearly in nor
  // clearly out, like any NaN -> borderline -> decided in fp64
  const int in = lhs < 0.99f * rhs ? 1 : 0;
  const int out = lhs > 1.01f * rhs ? 1 : 0;
  return in | ((in | out) ^ 1) << 1;  // bit 0: inlier, bit 1: borderline (neither clearly in nor out)
}

template <int KIND>
struct Traits;
template <>
struct Traits<0> {  // E: 5-point for minimal and local
  static constexpr int kMin = 5, kLocalMin = 5, kMaxModels = 10, kMaxLocalModels = 10;
};
template <>
struct Traits<1> {  // F: 7-point minimal, 8-point local
  static constexpr int kMin = 7, kLocalMin = 8, kMaxModels = 3, kMaxLocalModels = 1;
};
template <>
struct Traits<2> {  // H: 4-point DLT for both
  static constexpr int kMin = 4, kLocalMin = 4, kMaxModels = 1, kMaxLocalModels = 1;
};

constexpr int kChunkModels = 256;  // models scored per pass of the fp32 scoring loop
constexpr int kPtsPerThread = 8;    // points held in registers per thread and pass

struct Shared {
  double chunk_d[kChunkModels][9];  // models of the current chunk (fp64, for borderline rechecks)
  float chunk_f[kChunkModels][12];  // same, fp32, padded to three 16-byte loads
  int chunk_cnt[kChunkModels];      // inlier counts of the chunk's models
  int scan[kRansacThreads];
  double best_model[9];
  double cand_models[10 * 9];
  double red[4][64];     // per-warp partial sums (45 normal-equation entries + 8 moments)
  double sum_arr[kRansacThreads];
  int cnt_arr[kRansacThreads];
  int cand_cnt[10];
  double cand_sum[10];
  int n_cand;
  int best_cnt;
  double best_sum;
  int winner;
  int improved;
  int round_max;         // largest (partial) inlier count among the models of the current round, for the exact pruning
  double norm[6];        // s1, cx1, cy1, s2, cx2, cy2
};

// Score `model` (registers of every lane hold the same 9 values) over all points; warp-cooperative.
template <int KIND>
__device__ __forceinline__ void warp_score(const double* M, const double4* pts, int64_t off, int n,
                                           const PointXform& X, double thr, int lane, int& cnt, double& sum) {
  int c = 0;
  double s = 0.0;
  for (int i = lane; i < n; i += 32) {
    double x1, y1, x2, y2;
    load_pt(pts, off + i, X, x1, y1, x2, y2);
    const double r = residual<KIND>(M, x1, y1, x2, y2);
    if (r <= thr) {
      ++c;
      s += r;
    }
  }
  cnt = __reduce_add_sync(0xffffffffu, c);
  sum = warp_sum_d(s);
}

// Hypothesis scoring of one block of points: every thread keeps PPT matches (fp32) in registers and sweeps the
// chunk's models: division-free fp32 test, fp64 only for the borderline points of a (thread, model).  Inlier counts
// go to sh.chunk_cnt.
template <int KIND, int PPT>
__device__ __forceinline__ void score_block(Shared& sh, const double4* pts, int64_t off, const PointXform& X, int n, int pb,
                                            int n_chunk, double thr, float thr_f, int tid, int need) {
  float px1[PPT], py1[PPT], px2[PPT], py2[PPT];
  int live[PPT];   // 1 for a real match, 0 for a slot past the end: such a slot never counts, whatever the model
                   // (its far-away point is an outlier for every sane model, but lhs and rhs can both overflow)
#pragma unroll
  for (int q = 0; q < PPT; ++q) {
    const int i = pb + q * kRansacThreads + tid;
    double x1 = 0, y1 = 0, x2 = 1e15, y2 = 1e15;
    live[q] = i < n ? 1 : 0;
    if (i < n) load_pt(pts, off + i, X, x1, y1, x2, y2);
    px1[q] = static_cast<float>(x1); py1[q] = static_cast<float>(y1);
    px2[q] = static_cast<float>(x2); py2[q] = static_cast<float>(y2);
  }
  for (int m = 0; m < n_chunk; ++m) {
    // exact pruning: a model that cannot reach `need + (matches not yet scored)` even if every remaining match were
    // an inlier can neither beat the best model so far nor the leader of this round (uniform across the CTA)
    if (sh.chunk_cnt[m] < need) continue;
    float Mf[12];
    const float4* mp = reinterpret_cast<const float4*>(sh.chunk_f[m]);
    const float4 m0 = mp[0], m1 = mp[1], m2 = mp[2];
    Mf[0] = m0.x; Mf[1] = m0.y; Mf[2] = m0.z; Mf[3] = m0.w;
    Mf[4] = m1.x; Mf[5] = m1.y; Mf[6] = m1.z; Mf[7] = m1.w; Mf[8] = m2.x;
    int c = 0, flags = 0;
#pragma unroll
    for (int q = 0; q < PPT; ++q) {
      const int f = inlier_f32<KIND>(Mf, px1[q], py1[q], px2[q], py2[q], thr_f);
      c += f & live[q];
      flags |= f;
    }
    if (flags & 2) {  // rare: a borderline point -> redo this thread's points of this model in fp64
      c = 0;
      for (int q = 0; q < PPT; ++q) {
        const int i = pb + q * kRansacThreads + tid;
        if (i < n) {
          double x1, y1, x2, y2;
          load_pt(pts, off + i, X, x1, y1, x2, y2);
          c += (residual<KIND>(sh.chunk_d[m], x1, y1, x2, y2) <= thr) ? 1 : 0;
        }
      }
    }
    if (c) atomicAdd(&sh.chunk_cnt[m], c);  // most hypotheses have (almost) no inliers: cheaper than a warp reduce
  }
}

#define B2M_TICK(slot)                                   \
  do {                                                   \
    if (P.prof && tid == 0) {                            \
      const long long _n = clock64();                    \
      prof_acc[slot] += _n - prof_t;                     \
      prof_t = _n;                                       \
    }                                                    \
  } while (0)

// MIN_MODE (E only): how the minimal 5-point solves of a round are mapped.  0: one THREAD per hypothesis (geom.h
// minimal_E5); 1: one WARP per hypothesis (five_point_warp.cuh); 2: hybrid -- the elimination (the memory-heavy,
// regular half) one warp per hypothesis, the root refinement + models (latency-bound, irregular) one thread per
// hypothesis.  The local-optimisation solve is always the warp solver.
constexpr int kEStride = 200;  // doubles of scratch per hypothesis: models [0, 90), N [90, 126), polynomial [126, 137), Mr [137, 197)
constexpr int kEN = 90, kEPoly = 126, kEMr = 137;
template <int KIND, int MIN_MODE>
__device__ void ransac_problem(const VerifyParams& P, Shared& sh, int pair, int64_t off, int n,
                               const PointXform& X, double thr, uint64_t key, const b2m_ransac_opts& ro) {
  using T = Traits<KIND>;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double4* pts = P.pts;
  uint8_t* mask = P.mask + static_cast<int64_t>(KIND) * P.arena_cap + off;
  const int out_idx = pair * 3 + KIND;

  if (n < T::kMin) {  // report.success = false, no inliers (U:optim/loransac.h)
    for (int i = tid; i < n; i += kRansacThreads) mask[i] = 0;
    if (tid == 0) {
      P.sup_cnt[out_idx] = 0;
      P.success[out_idx] = 0;
      for (int k = 0; k < 9; ++k) P.models[out_idx * 9 + k] = 0.0;
    }
    return;
  }
  // RANSAC ctor: clip max_num_trials by the bound at min_inlier_ratio
  double max_trials_d = compute_num_trials(floor(ro.min_inlier_ratio * 100000.0), 100000.0, ro.confidence,
                                           ro.dyn_num_trials_multiplier, T::kMin);
  const int max_trials = static_cast<int>(fmin(static_cast<double>(ro.max_num_trials), max_trials_d));
  double dyn_max = max_trials;
  if (tid == 0) {
    sh.best_cnt = 0;
    sh.best_sum = 1e300;
    for (int k = 0; k < 9; ++k) sh.best_model[k] = 0.0;
  }
  __syncthreads();

  int trials = 0;
  unsigned long long n_scored = 0;  // models whose residuals were evaluated over all n matches (thread 0 keeps the tally)
  // models of this thread's hypothesis: registers / local memory for F and H, the CTA's slice of the global scratch
  // for E (written by the warp-cooperative solver)
  constexpr bool kWarpMin = KIND == 0 && MIN_MODE != 0;
  constexpr bool kHybrid = KIND == 0 && MIN_MODE == 2;
  double mdl_local[kWarpMin ? 1 : T::kMaxModels * 9];
  double* const e_models = kWarpMin ? P.e_scratch + (static_cast<size_t>(pair) * kRansacThreads + tid) * kEStride : nullptr;
  double* const mdl = kWarpMin ? e_models : mdl_local;
  long long prof_acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  long long prof_t = clock64();
  while (trials < max_trials) {
    int nb = min(kRansacThreads, max_trials - trials);
    if (trials < ro.min_num_trials) nb = min(nb, ro.min_num_trials - trials);
    // past min_num_trials the sequential reference stops at the FIRST trial >= dyn_max: a round never needs more
    // hypotheses than are missing to that bound (a better model found among them only lowers it)
    else if (dyn_max - trials < nb) nb = max(1, static_cast<int>(ceil(dyn_max - trials)));
    // ---- phase 1: one minimal-sample hypothesis per thread
    int nm = 0;
    if (tid < nb) {
      const uint64_t tkey = splitmix64(key + static_cast<uint64_t>(trials + tid) * 0x100000001B3ull);
      int idx[T::kMin];
      for (int j = 0; j < T::kMin; ++j) {
        int cand = 0;
        for (int attempt = 0; attempt < 64; ++attempt) {
          const uint64_t r = splitmix64(tkey + static_cast<uint64_t>(j * 64 + attempt));
          cand = static_cast<int>(__umul64hi(r, static_cast<uint64_t>(n)));
          bool dup = false;
          for (int q = 0; q < j; ++q) dup |= (idx[q] == cand);
          if (!dup) break;
        }
        idx[j] = cand;
      }
      double x1[T::kMin], y1[T::kMin], x2[T::kMin], y2[T::kMin];
      for (int j = 0; j < T::kMin; ++j) load_pt(pts, off + idx[j], X, x1[j], y1[j], x2[j], y2[j]);
      if (KIND == 0 && !kWarpMin) nm = minimal_E5(x1, y1, x2, y2, mdl);
      if (kWarpMin) {
        // thread = hypothesis only for the (small) 5 x 9 null space; the elimination + root finding that follow
        // run one warp per hypothesis (five_point_warp.cuh)
        double A[45], Nb[36];
        for (int i = 0; i < 5; ++i) epipolar_row(x1[i], y1[i], x2[i], y2[i], A + 9 * i);
        nm = nullspace_gauss<5>(A, Nb) ? 1 : 0;
        if (nm)
          for (int k = 0; k < 36; ++k) e_models[kEN + k] = Nb[k];
      }
      if (KIND == 1) nm = minimal_F7(x1, y1, x2, y2, mdl);
      if (KIND == 2) nm = minimal_H4_closed(x1, y1, x2, y2, mdl);
    }
    if (kWarpMin) {
      sh.scan[tid] = nm;
      __syncthreads();
      fpw::Scratch& WS = reinterpret_cast<fpw::Scratch*>(sh.chunk_d)[warp];   // chunk_d is idle outside the scoring loop
      for (int h = warp; h < nb; h += kRansacThreads / 32) {
        int cnt = 0;
        if (sh.scan[h]) {   // uniform in the warp
          double* hm = P.e_scratch + (static_cast<size_t>(pair) * kRansacThreads + h) * kEStride;
          for (int k = lane; k < 36; k += 32) WS.N[k] = hm[kEN + k];
          __syncwarp();
          if (kHybrid) {
            cnt = fpw::eliminate_warp(WS, lane) ? 1 : 0;
            if (cnt) {
              if (lane < 11) hm[kEPoly + lane] = WS.ladder[0][lane];
              for (int k = lane; k < 60; k += 32) hm[kEMr + k] = (&WS.Mr[0][0])[k];
            }
          } else {
            cnt = fpw::five_point_warp(WS, hm, lane);
          }
        }
        __syncwarp();
        if (lane == 0) sh.scan[h] = cnt;
      }
      __syncthreads();
      nm = tid < nb ? sh.scan[tid] : 0;
      if (kHybrid && nm) nm = fpw::finish_thread(e_models + kEN, e_models + kEPoly, e_models + kEMr, e_models);
      __syncthreads();
    }
    // ---- phase 2: score every model of every hypothesis of this warp (warp = one model at a time)
    B2M_TICK(0);
    //      Models go to shared memory in chunks; every thread keeps kPtsPerThread points in registers
    //      (fp32) and sweeps the chunk's models: division-free fp32 test, fp64 only for borderline
    //      points.  Only inlier COUNTS are formed here; among equal counts the earlier trial wins
    //      (the residual-sum tie-break of U:optim/support_measurement.h applies from the LO stage on).
    int my_cnt = -1, my_m = 0;
    double my_sum = 1e300;
    sh.scan[tid] = nm;
    if (tid == 0) sh.round_max = 0;
    __syncthreads();
    int my_base = 0, total_models = 0;
    for (int t = 0; t < kRansacThreads; ++t) {
      const int v = sh.scan[t];
      if (t < tid) my_base += v;
      total_models += v;
    }
    const float thr_f = static_cast<float>(thr);
    n_scored += total_models;
    for (int chunk0 = 0; chunk0 < total_models; chunk0 += kChunkModels) {
      const int n_chunk = min(kChunkModels, total_models - chunk0);
      for (int m = 0; m < nm; ++m) {
        const int g = my_base + m - chunk0;
        if (g >= 0 && g < kChunkModels) {
#pragma unroll
          for (int k = 0; k < 9; ++k) {
            sh.chunk_d[g][k] = mdl[m * 9 + k];
            sh.chunk_f[g][k] = static_cast<float>(mdl[m * 9 + k]);
          }
        }
      }
      for (int m = tid; m < kChunkModels; m += kRansacThreads) sh.chunk_cnt[m] = 0;
      __syncthreads();
      // Blocks of 512 matches.  Between blocks the inlier counts so far are complete (barrier), so a model whose count
      // plus ALL remaining matches stays below the best of the earlier rounds or below what the leader of this round
      // already has is dropped for the rest of the sweep -- exact: it could not have won, nor tied.
      constexpr int kBlock = 4 * kRansacThreads;
      for (int pb = 0; pb < n; pb += kBlock) {
        const int rem = n - pb;
        int need = 0;
        if (pb > 0) {
          __syncthreads();   // chunk_cnt of the previous blocks is complete
          for (int m = tid; m < n_chunk; m += kRansacThreads) atomicMax(&sh.round_max, sh.chunk_cnt[m]);
          __syncthreads();
          need = max(sh.best_cnt + 1, sh.round_max) - rem;
        }
        // the last block takes as few point slots per thread as cover it (a slot past the end costs a full test)
        if (rem > 3 * kRansacThreads) score_block<KIND, 4>(sh, pts, off, X, n, pb, n_chunk, thr, thr_f, tid, need);
        else if (rem > 2 * kRansacThreads) score_block<KIND, 3>(sh, pts, off, X, n, pb, n_chunk, thr, thr_f, tid, need);
        else if (rem > kRansacThreads) score_block<KIND, 2>(sh, pts, off, X, n, pb, n_chunk, thr, thr_f, tid, need);
        else score_block<KIND, 1>(sh, pts, off, X, n, pb, n_chunk, thr, thr_f, tid, need);
      }
      __syncthreads();
      for (int m = 0; m < nm; ++m) {
        const int g = my_base + m - chunk0;
        if (g >= 0 && g < kChunkModels) {
          const int c = sh.chunk_cnt[g];
          if (c > my_cnt) {
            my_cnt = c;
            my_m = m;
          }
        }
      }
      __syncthreads();
    }
    sh.cnt_arr[tid] = my_cnt;
    sh.sum_arr[tid] = my_sum;
    __syncthreads();
    B2M_TICK(1);
    if (tid == 0) {
      int w = -1, bc = sh.best_cnt;
      double bs = sh.best_sum;
      for (int t = 0; t < nb; ++t) {
        const int c = sh.cnt_arr[t];
        const double s = sh.sum_arr[t];
        if (c > bc || (c == bc && s < bs)) {
          bc = c;
          bs = s;
          w = t;
        }
      }
      sh.winner = w;
      sh.improved = (w >= 0);
      if (w >= 0) {
        sh.best_cnt = bc;
        sh.best_sum = bs;
      }
    }
    __syncthreads();
    if (sh.improved) {
      if (tid == sh.winner)
        for (int k = 0; k < 9; ++k) sh.best_model[k] = mdl[my_m * 9 + k];
      __syncthreads();
      {  // exact fp64 support (count, residual sum) of the new best model
        double M[9];
        for (int k = 0; k < 9; ++k) M[k] = sh.best_model[k];
        int c;
        double s;
        int cl = 0;
        double sl = 0.0;
        for (int i = tid; i < n; i += kRansacThreads) {
          double x1, y1, x2, y2;
          load_pt(pts, off + i, X, x1, y1, x2, y2);
          const double r = residual<KIND>(M, x1, y1, x2, y2);
          if (r <= thr) {
            ++cl;
            sl += r;
          }
        }
        c = __reduce_add_sync(0xffffffffu, cl);
        s = warp_sum_d(sl);
        if (lane == 0) {
          sh.cand_cnt[warp] = c;
          sh.cand_sum[warp] = s;
        }
        __syncthreads();
        if (tid == 0) {
          sh.best_cnt = sh.cand_cnt[0] + sh.cand_cnt[1] + sh.cand_cnt[2] + sh.cand_cnt[3];
          sh.best_sum = sh.cand_sum[0] + sh.cand_sum[1] + sh.cand_sum[2] + sh.cand_sum[3];
        }
        __syncthreads();
      }
      B2M_TICK(2);
      n_scored += 1;  // exact fp64 support of the new best
      // ---- phase 3: recursive local optimisation on the inliers of the current best
      if (sh.best_cnt > T::kMin && sh.best_cnt >= T::kLocalMin) {
        for (int lt = 0; lt < kMaxLocalTrials; ++lt) {
          const int prev_best = sh.best_cnt;
          double M[9];
          for (int k = 0; k < 9; ++k) M[k] = sh.best_model[k];
          double s1 = 1, cx1 = 0, cy1 = 0, s2 = 1, cx2 = 0, cy2 = 0;
          if (KIND != 0) {  // Hartley normalisation of the inlier set: moments first
            double mo[7] = {0, 0, 0, 0, 0, 0, 0};
            for (int i = tid; i < n; i += kRansacThreads) {
              double x1, y1, x2, y2;
              load_pt(pts, off + i, X, x1, y1, x2, y2);
              if (residual<KIND>(M, x1, y1, x2, y2) <= thr) {
                mo[0] += 1.0;
                mo[1] += x1; mo[2] += y1; mo[3] += x1 * x1 + y1 * y1;
                mo[4] += x2; mo[5] += y2; mo[6] += x2 * x2 + y2 * y2;
              }
            }
            for (int k = 0; k < 7; ++k) {
              const double v = warp_sum_d(mo[k]);
              if (lane == 0) sh.red[warp][k] = v;
            }
            __syncthreads();
            if (tid == 0) {
              double t[7];
              for (int k = 0; k < 7; ++k) t[k] = sh.red[0][k] + sh.red[1][k] + sh.red[2][k] + sh.red[3][k];
              norm_from_moments(t[0], t[1], t[2], t[3], &sh.norm[0], &sh.norm[1], &sh.norm[2]);
              norm_from_moments(t[0], t[4], t[5], t[6], &sh.norm[3], &sh.norm[4], &sh.norm[5]);
            }
            __syncthreads();
            s1 = sh.norm[0]; cx1 = sh.norm[1]; cy1 = sh.norm[2];
            s2 = sh.norm[3]; cx2 = sh.norm[4]; cy2 = sh.norm[5];
          }
          double S[45];
#pragma unroll
          for (int k = 0; k < 45; ++k) S[k] = 0.0;
          for (int i = tid; i < n; i += kRansacThreads) {
            double x1, y1, x2, y2;
            load_pt(pts, off + i, X, x1, y1, x2, y2);
            if (residual<KIND>(M, x1, y1, x2, y2) <= thr) {
              double r1[9], r2[9];
              if (KIND == 2) {
                dlt_rows(s1 * (x1 - cx1), s1 * (y1 - cy1), s2 * (x2 - cx2), s2 * (y2 - cy2), r1, r2);
                sym9_add_row(S, r1);
                sym9_add_row(S, r2);
              } else {
                epipolar_row(s1 * (x1 - cx1), s1 * (y1 - cy1), s2 * (x2 - cx2), s2 * (y2 - cy2), r1);
                sym9_add_row(S, r1);
              }
            }
          }
#pragma unroll
          for (int k = 0; k < 45; ++k) {
            const double v = warp_sum_d(S[k]);
            if (lane == 0) sh.red[warp][k] = v;
          }
          __syncthreads();
          B2M_TICK(3);
          if (P.lo_eig_thread) {   // A/B switch B2M_LO_EIG=thread: the serial eigen-solve on thread 0
            if (tid == 0) {
              double St[45];
              for (int k = 0; k < 45; ++k) St[k] = sh.red[0][k] + sh.red[1][k] + sh.red[2][k] + sh.red[3][k];
              int nc = 0;
              if (KIND == 0) {
                // least-squares 4-D null space of the N x 9 system.  The 5-point solver fixes the coefficient of its
                // LAST basis vector to 1, so that one must be the smallest singular vector (for noise-free inliers it
                // IS the essential matrix).  The solver itself runs on warp 0 below.
                double Nr[36];
                smallest_eigvecs_invit<4>(St, Nr);
                fpw::Scratch& WS = reinterpret_cast<fpw::Scratch*>(sh.chunk_d)[0];
                for (int k = 0; k < 4; ++k)
                  for (int e = 0; e < 9; ++e) WS.N[k * 9 + e] = Nr[(3 - k) * 9 + e];
              } else if (KIND == 1) {
                nc = finish_F8(St, s1, cx1, cy1, s2, cx2, cy2, sh.cand_models);
              } else {
                nc = finish_H(St, s1, cx1, cy1, s2, cx2, cy2, sh.cand_models);
              }
              sh.n_cand = nc;
            }
            __syncthreads();
          } else {
            // the smallest eigenvector(s) of the normal matrix on warp 0 (eig_warp.cuh: bit-identical to the serial
            // solver, a fraction of its latency -- the other three warps wait at the barrier either way)
            if (warp == 0) {
              double* St = sh.red[0];   // summed in place: red[0][k] += red[1..3][k]
              for (int k = lane; k < 45; k += 32) St[k] = sh.red[0][k] + sh.red[1][k] + sh.red[2][k] + sh.red[3][k];
              __syncwarp();
              // scratch: the second warp slot of the 5-point scratch area (chunk_d is idle outside the scoring loop)
              eigw::Scratch& ES = *reinterpret_cast<eigw::Scratch*>(reinterpret_cast<fpw::Scratch*>(sh.chunk_d) + 1);
              double* vec = sh.sum_arr;   // [K][9], free between rounds
              eigw::smallest_eigvecs_warp<KIND == 0 ? 4 : 1>(St, vec, ES, lane);
              if (lane == 0) {
                int nc = 0;
                if (KIND == 0) {
                  // least-squares 4-D null space of the N x 9 system.  The 5-point solver fixes the coefficient of
                  // its LAST basis vector to 1, so that one must be the smallest singular vector (for noise-free
                  // inliers it IS the essential matrix).
                  fpw::Scratch& WS = reinterpret_cast<fpw::Scratch*>(sh.chunk_d)[0];
                  for (int k = 0; k < 4; ++k)
                    for (int e = 0; e < 9; ++e) WS.N[k * 9 + e] = vec[(3 - k) * 9 + e];
                } else if (KIND == 1) {
                  double Fn[9];
                  for (int e = 0; e < 9; ++e) Fn[e] = vec[e];
                  enforce_rank2(Fn);
                  denormalize_F(Fn, s1, cx1, cy1, s2, cx2, cy2, sh.cand_models);
                  nc = 1;
                } else {
                  double Hn[9];
                  for (int e = 0; e < 9; ++e) Hn[e] = vec[e];
                  denormalize_H(Hn, s1, cx1, cy1, s2, cx2, cy2, sh.cand_models);
                  nc = 1;
                }
                sh.n_cand = nc;
              }
            }
            __syncthreads();
          }
          if (KIND == 0) {
            if (warp == 0) {
              const int nc = fpw::five_point_warp(reinterpret_cast<fpw::Scratch*>(sh.chunk_d)[0], sh.cand_models, lane);
              if (lane == 0) sh.n_cand = nc;
            }
            __syncthreads();
          }
          B2M_TICK(4);
          const int nc = sh.n_cand;
          n_scored += nc + (KIND != 0 ? 2 : 1);  // LO candidates + the inlier passes (moments, normal equations)
          for (int m = warp; m < nc; m += kRansacThreads / 32) {
            double C[9];
            for (int k = 0; k < 9; ++k) C[k] = sh.cand_models[m * 9 + k];
            int c;
            double s;
            warp_score<KIND>(C, pts, off, n, X, thr, lane, c, s);
            if (lane == 0) {
              sh.cand_cnt[m] = c;
              sh.cand_sum[m] = s;
            }
          }
          __syncthreads();
          if (tid == 0) {
            int w = -1;
            for (int m = 0; m < nc; ++m)
              if (sh.cand_cnt[m] > sh.best_cnt || (sh.cand_cnt[m] == sh.best_cnt && sh.cand_sum[m] < sh.best_sum)) {
                sh.best_cnt = sh.cand_cnt[m];
                sh.best_sum = sh.cand_sum[m];
                w = m;
              }
            if (w >= 0)
              for (int k = 0; k < 9; ++k) sh.best_model[k] = sh.cand_models[w * 9 + k];
          }
          __syncthreads();
          B2M_TICK(5);
          if (sh.best_cnt <= prev_best) break;
        }
      }
      dyn_max = compute_num_trials(sh.best_cnt, n, ro.confidence, ro.dyn_num_trials_multiplier, T::kMin);
    }
    trials += nb;
    __syncthreads();
    if (trials >= dyn_max && trials >= ro.min_num_trials) break;
  }

  // ---- final inlier mask from the best model
  double M[9];
  for (int k = 0; k < 9; ++k) M[k] = sh.best_model[k];
  const bool ok = sh.best_cnt >= T::kMin;
  for (int i = tid; i < n; i += kRansacThreads) {
    double x1, y1, x2, y2;
    load_pt(pts, off + i, X, x1, y1, x2, y2);
    mask[i] = (ok && residual<KIND>(M, x1, y1, x2, y2) <= thr) ? 1 : 0;
  }
  B2M_TICK(6);
  if (P.counters && tid == 0) {
    atomicAdd(P.counters + KIND, n_scored + 1);
    atomicAdd(P.counters + 3 + KIND, (n_scored + 1) * static_cast<unsigned long long>(n));
  }
  if (P.prof && tid == 0)
    for (int k = 0; k < 8; ++k) atomicAdd(P.prof + KIND * 8 + k, static_cast<unsigned long long>(prof_acc[k]));
  if (tid == 0) {
    P.sup_cnt[out_idx] = sh.best_cnt;
    P.success[out_idx] = ok ? 1 : 0;
    for (int k = 0; k < 9; ++k) P.models[out_idx * 9 + k] = M[k];
  }
}

// One instantiation per model kind, so that each gets its own register allocation and occupancy
// (the closed-form H path needs a fraction of the registers / local memory of the 5-point E path).
template <int KIND>
struct KindBlocks;
template <>
struct KindBlocks<0> { static constexpr int v = 3; };
template <>
struct KindBlocks<1> { static constexpr int v = 4; };
template <>
struct KindBlocks<2> { static constexpr int v = 5; };

template <int KIND, int MIN_MODE = 0>
__global__ void __launch_bounds__(kRansacThreads, KindBlocks<KIND>::v) b2m_ransac_kernel(const VerifyParams P) {
  __shared__ Shared sh;
  const int pair = blockIdx.x;
  constexpr int kind = KIND;
  const int n = P.pair_cnt[pair];
  const int64_t off = P.pair_off[pair];
  const int i1 = P.pairs[2 * pair], i2 = P.pairs[2 * pair + 1];
  const int out_idx = pair * 3 + kind;
  const DevCamera c1 = P.cams[i1], c2 = P.cams[i2];
  bool run = true;
  if (P.single_kind < 0) {
    const bool calibrated = c1.has_prior && c2.has_prior;
    if (n < P.opt.min_num_inliers) run = false;             // EstimateTwoViewGeometry: DEGENERATE up front
    if (P.opt.force_H_use && kind != 2) run = false;
    if (kind == 0 && !calibrated) run = false;              // uncalibrated: F and H only
  }
  if (!run) {
    if (threadIdx.x == 0) {
      P.sup_cnt[out_idx] = 0;
      P.success[out_idx] = 0;
      for (int k = 0; k < 9; ++k) P.models[out_idx * 9 + k] = 0.0;
    }
    uint8_t* mask = P.mask + static_cast<int64_t>(kind) * P.arena_cap + off;
    for (int i = threadIdx.x; i < n; i += kRansacThreads) mask[i] = 0;
    return;
  }
  PointXform X = {1, 0, 1, 0, 1, 0, 1, 0};
  double thr = P.opt.ransac.max_error * P.opt.ransac.max_error;
  if (kind == 0 && P.single_kind < 0) {
    // CamFromImg for (SIMPLE_)PINHOLE and the CamFromImgThreshold-averaged error (row V9)
    X.ax1 = 1.0 / c1.fx; X.bx1 = -c1.cx / c1.fx; X.ay1 = 1.0 / c1.fy; X.by1 = -c1.cy / c1.fy;
    X.ax2 = 1.0 / c2.fx; X.bx2 = -c2.cx / c2.fx; X.ay2 = 1.0 / c2.fy; X.by2 = -c2.cy / c2.fy;
    const double e = 0.5 * (P.opt.ransac.max_error / c1.mean_f + P.opt.ransac.max_error / c2.mean_f);
    thr = e * e;
  }
  const uint64_t key = splitmix64(P.seed ^ splitmix64((static_cast<uint64_t>(static_cast<uint32_t>(i1)) << 34) ^
                                                        (static_cast<uint64_t>(static_cast<uint32_t>(i2)) << 2) ^
                                                        static_cast<uint64_t>(kind)));
  ransac_problem<KIND, MIN_MODE>(P, sh, pair, off, n, X, thr, key, P.opt.ransac);
}

// The three model kinds are independent problems: E and F go to two side streams so that their
// (few, long) CTAs fill the tail of the H kernel instead of serialising behind it.
struct RansacStreams {
  cudaStream_t side[2] = {nullptr, nullptr};
  cudaEvent_t fork = nullptr, join[2] = {nullptr, nullptr};
};

// ---- relative pose (TwoViewGeometryOptions.compute_relative_pose; pose.h) --------------------------------
// EstimateTwoViewGeometryPose (U:estimators/two_view_geometry.cc; R:estimators/two_view_geometry.h:153-158) for
// every pair of the batch, one CTA per pair: thread 0 decomposes E (CALIBRATED / UNCALIBRATED) or H (PLANAR /
// PANORAMIC / PLANAR_OR_PANORAMIC) into candidate poses; all threads triangulate the inlier matches under each
// candidate and count the points in front of both cameras (CheckCheirality); the candidate with the most points
// wins (later candidates win ties, as upstream's `>=`); the median triangulation angle of its points becomes
// tri_angle; PLANAR_OR_PANORAMIC is resolved into PANORAMIC (t == 0) or PLANAR.
struct PoseParams {
  const int32_t* pairs;      // [nb x 2] indices into cams (and img_row0)
  const int64_t* pair_off;   // [nb] offset of the pair's inlier list / angle scratch
  const int32_t* inl_cnt;    // [nb]
  int32_t* config;           // [nb] in / out
  const uint2* inliers;      // arena of (idx1, idx2)
  const double* models;      // [nb][3][9]
  const DevCamera* cams;
  const DevDistortion* dist; // per camera, or nullptr when no camera has distortion
  // pixel coordinates of a feature: keypoints by padded row (pair pipeline) ...
  const float2* kpts;
  const int32_t* img_row0;
  // ... or the caller's point arrays (estimator entry points): [n x 2] doubles, per-problem offsets in points
  const double* pts1;
  const double* pts2;
  const int64_t* pts1_off;
  const int64_t* pts2_off;
  double* angles;            // scratch arena, same offsets as the inlier lists
  double* out;               // [nb][8]: qvec (w, x, y, z), tvec, tri_angle
  int32_t* out_valid;        // [nb]
};

__device__ __forceinline__ void pose_norm_point(const PoseParams& P, int pair, int side, int img, uint32_t idx, double* u,
                                                double* v) {
  double x, y;
  if (P.kpts) {
    const float2 k = P.kpts[P.img_row0[img] + idx];
    x = k.x;
    y = k.y;
  } else {
    const double* p = (side == 0 ? P.pts1 : P.pts2) + 2 * ((side == 0 ? P.pts1_off : P.pts2_off)[pair] + idx);
    x = p[0];
    y = p[1];
  }
  const DevCamera c = P.cams[img];
  if (P.dist && c.distorted) {
    cam::cam_from_img(P.dist[img].model, P.dist[img].p, x, y, u, v);
  } else {
    *u = (x - c.cx) / c.fx;
    *v = (y - c.cy) / c.fy;
  }
}

__global__ void __launch_bounds__(256) b2m_pose_kernel(const PoseParams P) {
  const int pair = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __shared__ double sR[4][9], st[4][3], s_med[2];
  __shared__ int s_ncand, s_warp[8], s_best, s_best_cnt;
  const int cfg = P.config[pair];
  const int n = P.inl_cnt[pair];
  const int64_t off = P.pair_off[pair];
  const int i1 = P.pairs[2 * pair], i2 = P.pairs[2 * pair + 1];
  double* out = P.out + 8 * pair;
  if (tid == 0) {
    out[0] = 1.0;
    for (int k = 1; k < 8; ++k) out[k] = 0.0;
    P.out_valid[pair] = 0;
  }
  const bool from_E = cfg == B2M_CALIBRATED || cfg == B2M_UNCALIBRATED;
  const bool from_H = cfg == B2M_PLANAR || cfg == B2M_PANORAMIC || cfg == B2M_PLANAR_OR_PANORAMIC;
  if (!from_E && !from_H) return;  // uniform
  if (tid == 0) {
    if (from_E) {
      double R1[9], R2[9], t[3];
      pose::decompose_E(P.models + 27 * pair, R1, R2, t);
      for (int c = 0; c < 4; ++c) {
        for (int k = 0; k < 9; ++k) sR[c][k] = (c & 1) ? R2[k] : R1[k];
        for (int k = 0; k < 3; ++k) st[c][k] = c < 2 ? t[k] : -t[k];
      }
      s_ncand = 4;
    } else {
      const DevCamera c1 = P.cams[i1], c2 = P.cams[i2];
      const double K1[4] = {c1.fx, c1.fy, c1.cx, c1.cy}, K2[4] = {c2.fx, c2.fy, c2.cx, c2.cy};
      double Rc[36], tc[12], nc[12];
      s_ncand = pose::decompose_H(P.models + 27 * pair + 18, K1, K2, Rc, tc, nc);
      for (int c = 0; c < s_ncand; ++c) {
        for (int k = 0; k < 9; ++k) sR[c][k] = Rc[c * 9 + k];
        for (int k = 0; k < 3; ++k) st[c][k] = tc[c * 3 + k];
      }
    }
    s_best = 0;
    s_best_cnt = -1;
  }
  __syncthreads();
  const int n_cand = s_ncand;
  for (int c = 0; c < n_cand; ++c) {
    double Rm[9], tv[3];
    for (int k = 0; k < 9; ++k) Rm[k] = sR[c][k];
    for (int k = 0; k < 3; ++k) tv[k] = st[c][k];
    const double max_depth = pose::cheirality_max_depth(Rm, tv);
    int cnt = 0;
    for (int k = tid; k < n; k += 256) {
      const uint2 m = P.inliers[off + k];
      double u1, v1, u2, v2, X[3];
      pose_norm_point(P, pair, 0, i1, m.x, &u1, &v1);
      pose_norm_point(P, pair, 1, i2, m.y, &u2, &v2);
      if (pose::triangulate(Rm, tv, u1, v1, u2, v2, X) && pose::in_front_of_both(Rm, tv, X, max_depth)) ++cnt;
    }
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) s_warp[warp] = cnt;
    __syncthreads();
    if (tid == 0) {
      int total = 0;
      for (int w = 0; w < 8; ++w) total += s_warp[w];
      if (c == 0 || total >= s_best_cnt) {  // upstream: points3D_cmb.size() >= points3D.size()
        s_best = c;
        s_best_cnt = total;
      }
    }
    __syncthreads();
  }
  const int best = s_best, n_front = s_best_cnt;
  if (from_E && n_front == 0) return;  // PoseFromEssentialMatrix found no point in front of both cameras: no pose
  double Rm[9], tv[3];
  for (int k = 0; k < 9; ++k) Rm[k] = sR[best][k];
  for (int k = 0; k < 3; ++k) tv[k] = st[best][k];
  // triangulation angles of the chosen candidate's points (-1 marks a point that failed the cheirality test)
  {
    const double c2[3] = {-(Rm[0] * tv[0] + Rm[3] * tv[1] + Rm[6] * tv[2]), -(Rm[1] * tv[0] + Rm[4] * tv[1] + Rm[7] * tv[2]),
                          -(Rm[2] * tv[0] + Rm[5] * tv[1] + Rm[8] * tv[2])};
    const double max_depth = pose::cheirality_max_depth(Rm, tv);
    for (int k = tid; k < n; k += 256) {
      const uint2 m = P.inliers[off + k];
      double u1, v1, u2, v2, X[3], a = -1.0;
      pose_norm_point(P, pair, 0, i1, m.x, &u1, &v1);
      pose_norm_point(P, pair, 1, i2, m.y, &u2, &v2);
      if (pose::triangulate(Rm, tv, u1, v1, u2, v2, X) && pose::in_front_of_both(Rm, tv, X, max_depth))
        a = pose::triangulation_angle(c2, X);
      P.angles[off + k] = a;
    }
  }
  if (tid == 0) {
    s_med[0] = s_med[1] = 0.0;
  }
  __syncthreads();
  // median by rank counting (ties broken by position): elements of rank m - 1 and m of the n_front valid angles
  if (n_front > 0) {
    const int m = n_front / 2;
    for (int k = tid; k < n; k += 256) {
      const double a = P.angles[off + k];
      if (a < 0.0) continue;
      int rank = 0;
      for (int j = 0; j < n; ++j) {
        const double b = P.angles[off + j];
        rank += (b >= 0.0 && (b < a || (b == a && j < k))) ? 1 : 0;
      }
      if (rank == m) s_med[1] = a;
      if (rank == m - 1) s_med[0] = a;
    }
  }
  __syncthreads();
  if (tid == 0) {
    double tri = 0.0;
    if (n_front > 0) tri = (n_front % 2 == 0) ? 0.5 * (s_med[0] + s_med[1]) : s_med[1];
    if (cfg == B2M_PLANAR_OR_PANORAMIC) {
      if (tv[0] == 0.0 && tv[1] == 0.0 && tv[2] == 0.0) {
        P.config[pair] = B2M_PANORAMIC;
        tri = 0.0;
      } else {
        P.config[pair] = B2M_PLANAR;
      }
    }
    pose::rotation_to_quat(Rm, out);
    out[4] = tv[0]; out[5] = tv[1]; out[6] = tv[2];
    out[7] = tri;
    P.out_valid[pair] = 1;
  }
}

// CamFromImg for camera models with distortion (row V9).  The E kernel normalises its input with the
// affine map (p - c) / f, which is CamFromImg only for the pinhole models; for a pair with a distorted
// camera this kernel writes "undistorted pixel" coordinates f * CamFromImg(p) + c into a second arena,
// so that the same affine map yields the normalised coordinates.  F and H keep reading the raw pixel
// coordinates, like upstream.  One CTA per pair; launched only when the image set has such a camera.
__global__ void __launch_bounds__(256) b2m_undistort_kernel(const VerifyParams P, const DevDistortion* __restrict__ dist,
                                                            double4* __restrict__ out) {
  const int pair = blockIdx.x;
  const int n = P.pair_cnt[pair];
  const int64_t off = P.pair_off[pair];
  const int i1 = P.pairs[2 * pair], i2 = P.pairs[2 * pair + 1];
  const DevCamera c1 = P.cams[i1], c2 = P.cams[i2];
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double4 p = P.pts[off + i];
    if (c1.distorted) {
      double u, v;
      cam::cam_from_img(dist[i1].model, dist[i1].p, p.x, p.y, &u, &v);
      p.x = c1.fx * u + c1.cx;
      p.y = c1.fy * v + c1.cy;
    }
    if (c2.distorted) {
      double u, v;
      cam::cam_from_img(dist[i2].model, dist[i2].p, p.z, p.w, &u, &v);
      p.z = c2.fx * u + c2.cx;
      p.w = c2.fy * v + c2.cy;
    }
    out[off + i] = p;
  }
}

// B2M_E5_MINIMAL = thread | warp | hybrid: how the minimal 5-point solves of a RANSAC round are mapped (A/B switch,
// DESIGN.md section 4).
int e5_minimal_mode() {
  static const int v = [] {
    const char* e = getenv("B2M_E5_MINIMAL");
    if (e && !strcmp(e, "warp")) return 1;
    if (e && !strcmp(e, "hybrid")) return 2;
    if (e && !strcmp(e, "thread")) return 0;
    return 2;
  }();
  return v;
}
int lo_eig_thread_mode() {
  const char* e = getenv("B2M_LO_EIG");
  return e && !strcmp(e, "thread") ? 1 : 0;
}
void launch_e_kernel(const VerifyParams& PE, int nb, cudaStream_t st) {
  switch (e5_minimal_mode()) {
    case 1: b2m_ransac_kernel<0, 1><<<nb, kRansacThreads, 0, st>>>(PE); break;
    case 2: b2m_ransac_kernel<0, 2><<<nb, kRansacThreads, 0, st>>>(PE); break;
    default: b2m_ransac_kernel<0, 0><<<nb, kRansacThreads, 0, st>>>(PE); break;
  }
}

// `pts_E` (optional): the arena the E kernel reads instead of P.pts (output of b2m_undistort_kernel).
cudaError_t launch_ransac(const VerifyParams& P_in, int nb, cudaStream_t st, RansacStreams* rs = nullptr,
                          const double4* pts_E = nullptr) {
  const VerifyParams& P = P_in;
  VerifyParams PE = P_in;
  if (pts_E) PE.pts = pts_E;
  if (P.single_kind >= 0 || !rs || !rs->side[0]) {
    if (P.single_kind < 0 || P.single_kind == 0) {
      launch_e_kernel(PE, nb, st);
    }
    if (P.single_kind < 0 || P.single_kind == 1) b2m_ransac_kernel<1><<<nb, kRansacThreads, 0, st>>>(P);
    if (P.single_kind < 0 || P.single_kind == 2) b2m_ransac_kernel<2><<<nb, kRansacThreads, 0, st>>>(P);
    return cudaGetLastError();
  }
  cudaError_t e = cudaEventRecord(rs->fork, st);
  if (e != cudaSuccess) return e;
  cudaStreamWaitEvent(rs->side[0], rs->fork, 0);
  cudaStreamWaitEvent(rs->side[1], rs->fork, 0);
  launch_e_kernel(PE, nb, rs->side[0]);
  b2m_ransac_kernel<1><<<nb, kRansacThreads, 0, rs->side[1]>>>(P);
  b2m_ransac_kernel<2><<<nb, kRansacThreads, 0, st>>>(P);
  cudaEventRecord(rs->join[0], rs->side[0]);
  cudaEventRecord(rs->join[1], rs->side[1]);
  cudaStreamWaitEvent(st, rs->join[0], 0);
  cudaStreamWaitEvent(st, rs->join[1], 0);
  return cudaGetLastError();
}

// Decision tree of EstimateCalibrated/UncalibratedTwoViewGeometry, ExtractInlierMatches (ordered
// compaction) and DetectWatermark.  One CTA per pair.
__global__ void __launch_bounds__(256) b2m_decide_kernel(const VerifyParams P) {
  const int pair = blockIdx.x;
  const int n = P.pair_cnt[pair];
  const int64_t off = P.pair_off[pair];
  const int i1 = P.pairs[2 * pair], i2 = P.pairs[2 * pair + 1];
  const DevCamera c1 = P.cams[i1], c2 = P.cams[i2];
  const b2m_tvg_opts& o = P.opt;
  __shared__ int s_cfg, s_kind, s_num, s_base, s_warp[8], s_border;
  __shared__ double s_tsum[2];
  __shared__ int s_tcnt;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    int cfg = B2M_DEGENERATE, kind = -1, num = 0;
    if (n >= o.min_num_inliers) {
      const bool calibrated = c1.has_prior && c2.has_prior && !o.force_H_use;
      const int nE = P.sup_cnt[pair * 3 + 0], nF = P.sup_cnt[pair * 3 + 1], nH = P.sup_cnt[pair * 3 + 2];
      const bool okE = calibrated && P.success[pair * 3 + 0], okF = P.success[pair * 3 + 1] != 0,
                 okH = P.success[pair * 3 + 2] != 0;
      const int mn = o.min_num_inliers;
      if (o.force_H_use) {
        if (okH && nH >= mn) {
          cfg = B2M_PLANAR_OR_PANORAMIC; kind = 2; num = nH;
        }
      } else if (!calibrated) {
        // EstimateUncalibratedTwoViewGeometry: PLANAR_OR_PANORAMIC vs UNCALIBRATED by nH / nF, but the inlier
        // matches (and the watermark test) ALWAYS come from F's mask, also when F found nothing
        if ((!okF && !okH) || (nF < mn && nH < mn)) {
          cfg = B2M_DEGENERATE;
        } else {
          kind = 1; num = nF;
          cfg = (static_cast<double>(nH) / nF > o.max_H_inlier_ratio) ? B2M_PLANAR_OR_PANORAMIC : B2M_UNCALIBRATED;
        }
      } else if ((!okE && !okF && !okH) || (nE < mn && nF < mn && nH < mn)) {
        cfg = B2M_DEGENERATE;
      } else {
        const double E_F = static_cast<double>(nE) / nF, H_F = static_cast<double>(nH) / nF,
                     H_E = static_cast<double>(nH) / nE;
        if (okE && E_F > o.min_E_F_inlier_ratio && nE >= mn) {
          if (nE >= nF) { kind = 0; num = nE; } else { kind = 1; num = nF; }
          if (H_E > o.max_H_inlier_ratio) {
            cfg = B2M_PLANAR_OR_PANORAMIC;
            if (nH > num) { kind = 2; num = nH; }
          } else {
            cfg = B2M_CALIBRATED;
          }
        } else if (okF && nF >= mn) {
          kind = 1; num = nF;
          if (H_F > o.max_H_inlier_ratio) {
            cfg = B2M_PLANAR_OR_PANORAMIC;
            if (nH > num) { kind = 2; num = nH; }
          } else {
            cfg = B2M_UNCALIBRATED;
          }
        } else if (okH && nH >= mn) {
          kind = 2; num = nH; cfg = B2M_PLANAR_OR_PANORAMIC;
        } else {
          cfg = B2M_DEGENERATE;
        }
      }
    }
    s_cfg = cfg; s_kind = kind; s_num = num; s_base = 0; s_border = 0;
    s_tsum[0] = s_tsum[1] = 0.0; s_tcnt = 0;
  }
  __syncthreads();
  const int kind = s_kind;
  if (kind < 0) {
    if (tid == 0) {
      P.config[pair] = s_cfg;
      P.inl_cnt[pair] = 0;
      if (P.guided_kind) P.guided_kind[pair] = -1;
    }
    return;
  }
  const uint8_t* mask = P.mask + static_cast<int64_t>(kind) * P.arena_cap + off;
  // ordered compaction of the inlier matches + border statistics for the watermark test
  const double d1 = o.watermark_border_size * sqrt(static_cast<double>(c1.width) * c1.width + static_cast<double>(c1.height) * c1.height);
  const double d2 = o.watermark_border_size * sqrt(static_cast<double>(c2.width) * c2.width + static_cast<double>(c2.height) * c2.height);
  int border_local = 0;
  for (int i0 = 0; i0 < n; i0 += 256) {
    const int i = i0 + tid;
    const bool keep = i < n && mask[i] != 0;
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    int base = s_base;
    for (int w = 0; w < warp; ++w) base += s_warp[w];
    if (keep) {
      P.inliers[off + base + __popc(ballot & ((1u << lane) - 1u))] = P.matches[off + i];
      const double4 p = P.pts[off + i];
      const bool b1 = p.x < d1 || p.x > c1.width - d1 || p.y < d1 || p.y > c1.height - d1;
      const bool b2 = p.z < d2 || p.z > c2.width - d2 || p.w < d2 || p.w > c2.height - d2;
      border_local += (b1 && b2) ? 1 : 0;
    }
    __syncthreads();
    if (tid == 0) {
      int t = 0;
      for (int w = 0; w < 8; ++w) t += s_warp[w];
      s_base += t;
    }
    __syncthreads();
  }
  border_local = __reduce_add_sync(0xffffffffu, border_local);
  if (lane == 0) atomicAdd(&s_border, border_local);
  __syncthreads();
  int cfg = s_cfg;
  const int num = s_base;
  // DetectWatermark: enough inliers in the border region of BOTH images, then a pure 2-D
  // translation must explain >= watermark_min_inlier_ratio of all inliers.
  if (o.detect_watermark && num > 0 &&
      static_cast<double>(s_border) / num >= o.watermark_min_inlier_ratio) {
    // LO-RANSAC<Translation, Translation> on ALL inlier points (upstream fits inlier_points1/2 of the whole
    // mask; the border ratio only gates the attempt); with kMinNumSamples = 1 every inlier is a hypothesis:
    // evaluate them all (exhaustive instead of sampled), then refit on the inliers of the best (local
    // optimisation), keeping the better of the two.
    const double thr = o.ransac.max_error * o.ransac.max_error;
    __shared__ int s_best_cnt;
    __shared__ double s_best_t[2];
    __shared__ unsigned long long s_best_key;
    if (tid == 0) {
      s_best_cnt = 0;
      s_best_key = 0ull;
    }
    __syncthreads();
    // hypotheses: border inlier h -> t = p2 - p1; support counted over border inliers
    for (int h0 = 0; h0 < n; h0 += 256) {
      const int h = h0 + tid;
      bool is_h = false;
      double tx = 0, ty = 0;
      if (h < n && mask[h]) {
        const double4 p = P.pts[off + h];
        is_h = true;
        tx = p.z - p.x;
        ty = p.w - p.y;
      }
      if (is_h) {
        int c = 0;
        for (int i = 0; i < n; ++i) {
          if (!mask[i]) continue;
          const double4 q = P.pts[off + i];
          const double ex = q.z - (q.x + tx), ey = q.w - (q.y + ty);
          c += (ex * ex + ey * ey <= thr) ? 1 : 0;
        }
        const unsigned long long key = (static_cast<unsigned long long>(c) << 32) | static_cast<unsigned>(n - h);
        atomicMax(&s_best_key, key);
      }
    }
    __syncthreads();
    if (tid == 0 && s_best_key != 0ull) {
      const int h = n - static_cast<int>(s_best_key & 0xffffffffull);
      const double4 p = P.pts[off + h];
      double tx = p.z - p.x, ty = p.w - p.y;
      int bc = static_cast<int>(s_best_key >> 32);
      for (int it = 0; it < kMaxLocalTrials; ++it) {
        double sx = 0, sy = 0;
        int c = 0;
        for (int i = 0; i < n; ++i) {
          if (!mask[i]) continue;
          const double4 q = P.pts[off + i];
          const double ex = q.z - (q.x + tx), ey = q.w - (q.y + ty);
          if (ex * ex + ey * ey <= thr) {
            sx += q.z - q.x;
            sy += q.w - q.y;
            ++c;
          }
        }
        if (c == 0) break;
        const double ntx = sx / c, nty = sy / c;
        int c2n = 0;
        for (int i = 0; i < n; ++i) {
          if (!mask[i]) continue;
          const double4 q = P.pts[off + i];
          const double ex = q.z - (q.x + ntx), ey = q.w - (q.y + nty);
          c2n += (ex * ex + ey * ey <= thr) ? 1 : 0;
        }
        if (c2n > bc) {
          bc = c2n;
          tx = ntx;
          ty = nty;
        } else {
          break;
        }
      }
      s_best_cnt = bc;
    }
    __syncthreads();
    if (s_best_cnt >= 1 && static_cast<double>(s_best_cnt) / num >= o.watermark_min_inlier_ratio) cfg = B2M_WATERMARK;
  }
  if (tid == 0) {
    P.config[pair] = cfg;
    P.inl_cnt[pair] = num;
    if (P.guided_kind) {
      // MatchGuidedSiftFeatures is run when the verified geometry has >= min_num_inliers inliers
      // (U:controllers/feature_matching_utils.cc); F for CALIBRATED / UNCALIBRATED, H for the planar /
      // panoramic configurations (U:feature/sift.cc MatchGuidedSiftFeaturesCPU)
      int gk = -1;
      if (P.guided_min_inliers >= 0 && num >= P.guided_min_inliers) {
        if (cfg == B2M_CALIBRATED || cfg == B2M_UNCALIBRATED) gk = 0;
        else if (cfg == B2M_PLANAR || cfg == B2M_PANORAMIC || cfg == B2M_PLANAR_OR_PANORAMIC) gk = 1;
      }
      P.guided_kind[pair] = gk;
      if (gk >= 0)
        for (int k = 0; k < 9; ++k)
          P.guided_model[pair * 9 + k] = static_cast<float>(P.models[(pair * 3 + (gk == 0 ? 1 : 2)) * 9 + k]);
    }
  }
}

// ---- host side --------------------------------------------------------------------------------

struct VerifyState {
  int batch = 0;
  int64_t arena_cap = 0;
  double4* d_pts[2] = {nullptr, nullptr};
  uint8_t* d_mask = nullptr;      // [3][arena_cap], shared by both slots (stream-ordered)
  double* d_models[2] = {nullptr, nullptr};
  int32_t* d_sup = nullptr;
  int32_t* d_success = nullptr;
  int32_t* d_config[2] = {nullptr, nullptr};
  int32_t* d_inl_cnt[2] = {nullptr, nullptr};
  uint2* d_inliers[2] = {nullptr, nullptr};
  // guided matching (lazily allocated): hand-over arrays + a second match arena per slot
  int32_t* d_guided_kind = nullptr;
  float* d_guided_model = nullptr;
  uint2* d_garena[2] = {nullptr, nullptr};
  unsigned long long* d_gcursor[2] = {nullptr, nullptr};
  int64_t* d_goff[2] = {nullptr, nullptr};
  int32_t* d_gcnt[2] = {nullptr, nullptr};
  uint2* h_garena[2] = {nullptr, nullptr};
  unsigned long long* h_gcursor[2] = {nullptr, nullptr};
  int64_t* h_goff[2] = {nullptr, nullptr};
  int32_t* h_gcnt[2] = {nullptr, nullptr};
  bool guided_on[2] = {false, false};
  double* h_models[2] = {nullptr, nullptr};
  int32_t* h_config[2] = {nullptr, nullptr};
  int32_t* h_inl_cnt[2] = {nullptr, nullptr};
  uint2* h_inliers[2] = {nullptr, nullptr};
  DevCamera* d_cams = nullptr;
  // relative pose (compute_relative_pose), lazily allocated
  double* d_pose[2] = {nullptr, nullptr};        // [batch][8] qvec, tvec, tri_angle
  int32_t* d_pose_valid[2] = {nullptr, nullptr};
  double* h_pose[2] = {nullptr, nullptr};
  int32_t* h_pose_valid[2] = {nullptr, nullptr};
  double* d_angles = nullptr;                    // [arena_cap] triangulation-angle scratch
  bool pose_on[2] = {false, false};
  double* d_e_scratch = nullptr;                 // E kernel: [batch][128][90] null spaces / models (five_point_warp.cuh)
  DevDistortion* d_dist = nullptr;               // per image, only when any_distorted
  double4* d_pts_undist[2] = {nullptr, nullptr}; // E-kernel input per slot, lazily allocated
  bool any_distorted = false;
  unsigned long long* d_prof = nullptr;
  RansacStreams rs;
  int n_cams = 0;
  uint64_t cams_of = 0;  // ImageSet::generation the cameras were uploaded for
  void release() {
    for (int s = 0; s < 2; ++s) {
      cudaFree(d_pts[s]); cudaFree(d_models[s]); cudaFree(d_config[s]); cudaFree(d_inl_cnt[s]); cudaFree(d_inliers[s]);
      cudaFreeHost(h_models[s]); cudaFreeHost(h_config[s]); cudaFreeHost(h_inl_cnt[s]); cudaFreeHost(h_inliers[s]);
      d_pts[s] = nullptr; d_models[s] = nullptr; d_config[s] = nullptr; d_inl_cnt[s] = nullptr; d_inliers[s] = nullptr;
      h_models[s] = nullptr; h_config[s] = nullptr; h_inl_cnt[s] = nullptr; h_inliers[s] = nullptr;
    }
    cudaFree(d_mask); cudaFree(d_sup); cudaFree(d_success); cudaFree(d_cams);
    for (int s = 0; s < 2; ++s) {
      cudaFree(d_pose[s]); cudaFree(d_pose_valid[s]); cudaFreeHost(h_pose[s]); cudaFreeHost(h_pose_valid[s]);
      d_pose[s] = nullptr; d_pose_valid[s] = nullptr; h_pose[s] = nullptr; h_pose_valid[s] = nullptr;
      pose_on[s] = false;
    }
    cudaFree(d_angles);
    d_angles = nullptr;
    cudaFree(d_e_scratch);
    d_e_scratch = nullptr;
    cudaFree(d_dist); cudaFree(d_pts_undist[0]); cudaFree(d_pts_undist[1]);
    d_dist = nullptr; d_pts_undist[0] = d_pts_undist[1] = nullptr; any_distorted = false;
    cudaFree(d_guided_kind); cudaFree(d_guided_model);
    d_guided_kind = nullptr; d_guided_model = nullptr;
    for (int s = 0; s < 2; ++s) {
      cudaFree(d_garena[s]); cudaFree(d_gcursor[s]); cudaFree(d_goff[s]); cudaFree(d_gcnt[s]);
      cudaFreeHost(h_garena[s]); cudaFreeHost(h_gcursor[s]); cudaFreeHost(h_goff[s]); cudaFreeHost(h_gcnt[s]);
      d_garena[s] = nullptr; d_gcursor[s] = nullptr; d_goff[s] = nullptr; d_gcnt[s] = nullptr;
      h_garena[s] = nullptr; h_gcursor[s] = nullptr; h_goff[s] = nullptr; h_gcnt[s] = nullptr;
      guided_on[s] = false;
    }
    d_mask = nullptr; d_sup = nullptr; d_success = nullptr; d_cams = nullptr;
    batch = 0; arena_cap = 0; n_cams = 0; cams_of = 0;
  }
};

VerifyState* vstate(b2m_ctx* ctx) {
  if (!ctx->verify_state) ctx->verify_state = new VerifyState();
  return static_cast<VerifyState*>(ctx->verify_state);
}

#define V_TRY(ctx, expr)                                                                    \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) {                                                                \
      char _b[512];                                                                         \
      snprintf(_b, sizeof(_b), "[%s:%d] CUDA error: %s (%s)", __FILE__, __LINE__,          \
               cudaGetErrorString(_e), #expr);                                              \
      (ctx)->err = _b;                                                                      \
      return _e == cudaErrorMemoryAllocation ? B2M_ENOMEM : B2M_ECUDA;                      \
    }                                                                                       \
  } while (0)

unsigned long long* verify_counters(b2m_ctx* ctx) {
  if (!ctx->d_verify_counters) {
    if (cudaMalloc(&ctx->d_verify_counters, sizeof(unsigned long long) * 6) != cudaSuccess) {
      cudaGetLastError();
      ctx->d_verify_counters = nullptr;
      return nullptr;
    }
    cudaMemset(ctx->d_verify_counters, 0, sizeof(unsigned long long) * 6);
  }
  return ctx->d_verify_counters;
}

DevCamera to_dev(const b2m_camera& c) {
  DevCamera d{};
  int extra;
  cam::intrinsics(c.model, c.params, &d.fx, &d.fy, &d.cx, &d.cy, &extra);
  d.mean_f = cam::mean_focal_length(c.model, c.params);
  d.width = c.width; d.height = c.height; d.has_prior = c.has_prior_focal_length;
  d.distorted = cam::has_distortion(c.model) ? 1 : 0;
  return d;
}

DevDistortion to_dist(const b2m_camera& c) {
  DevDistortion d{};
  d.model = c.model;
  for (int k = 0; k < cam::kMaxParams; ++k) d.p[k] = c.params[k];
  return d;
}

int ensure_verify_ws(b2m_ctx* ctx, int batch, int64_t arena_cap) {
  VerifyState* V = vstate(ctx);
  if (V->batch >= batch && V->arena_cap >= arena_cap) return B2M_OK;
  DevCamera* keep_cams = V->d_cams;
  const int keep_n = V->n_cams;
  const uint64_t keep_of = V->cams_of;
  DevDistortion* keep_dist = V->d_dist;
  const bool keep_any = V->any_distorted;
  V->d_cams = nullptr;
  V->d_dist = nullptr;
  V->release();
  V->d_cams = keep_cams; V->n_cams = keep_n; V->cams_of = keep_of;
  V->d_dist = keep_dist; V->any_distorted = keep_any;
  for (int s = 0; s < 2; ++s) {
    V_TRY(ctx, cudaMalloc(&V->d_pts[s], sizeof(double4) * arena_cap));
    V_TRY(ctx, cudaMalloc(&V->d_models[s], sizeof(double) * 27 * batch));
    V_TRY(ctx, cudaMalloc(&V->d_config[s], sizeof(int32_t) * batch));
    V_TRY(ctx, cudaMalloc(&V->d_inl_cnt[s], sizeof(int32_t) * batch));
    V_TRY(ctx, cudaMalloc(&V->d_inliers[s], sizeof(uint2) * arena_cap));
    V_TRY(ctx, cudaMallocHost(&V->h_models[s], sizeof(double) * 27 * batch));
    V_TRY(ctx, cudaMallocHost(&V->h_config[s], sizeof(int32_t) * batch));
    V_TRY(ctx, cudaMallocHost(&V->h_inl_cnt[s], sizeof(int32_t) * batch));
    V_TRY(ctx, cudaMallocHost(&V->h_inliers[s], sizeof(uint2) * arena_cap));
  }
  V_TRY(ctx, cudaMalloc(&V->d_mask, 3 * arena_cap));
  V_TRY(ctx, cudaMalloc(&V->d_e_scratch, sizeof(double) * kEStride * kRansacThreads * static_cast<size_t>(batch)));
  V_TRY(ctx, cudaMalloc(&V->d_sup, sizeof(int32_t) * 3 * batch));
  V_TRY(ctx, cudaMalloc(&V->d_success, sizeof(int32_t) * 3 * batch));
  V->batch = batch;
  V->arena_cap = arena_cap;
  return B2M_OK;
}

}  // namespace

void* verify_points_arena(b2m_ctx* ctx, int s) {
  VerifyState* V = vstate(ctx);
  return V->d_pts[s];
}

int verify_prepare(b2m_ctx* ctx, ImageSet& S, int batch, int64_t arena_cap) {
  if (int rc = ensure_verify_ws(ctx, batch, arena_cap)) return rc;
  VerifyState* V = vstate(ctx);
  if (V->cams_of != S.generation || V->n_cams != S.n_images) {
    cudaFree(V->d_cams);
    V->d_cams = nullptr;
    std::vector<DevCamera> dc(S.n_images);
    for (int i = 0; i < S.n_images; ++i) dc[i] = to_dev(S.cams[i]);
    V_TRY(ctx, cudaMalloc(&V->d_cams, sizeof(DevCamera) * std::max(1, S.n_images)));
    V_TRY(ctx, cudaMemcpyAsync(V->d_cams, dc.data(), sizeof(DevCamera) * S.n_images, cudaMemcpyHostToDevice,
                               ctx->stream));
    cudaFree(V->d_dist);
    V->d_dist = nullptr;
    V->any_distorted = false;
    for (const DevCamera& c : dc) V->any_distorted = V->any_distorted || c.distorted;
    std::vector<DevDistortion> dd;
    if (V->any_distorted) {
      dd.resize(S.n_images);
      for (int i = 0; i < S.n_images; ++i) dd[i] = to_dist(S.cams[i]);
      V_TRY(ctx, cudaMalloc(&V->d_dist, sizeof(DevDistortion) * S.n_images));
      V_TRY(ctx, cudaMemcpyAsync(V->d_dist, dd.data(), sizeof(DevDistortion) * S.n_images, cudaMemcpyHostToDevice,
                                 ctx->stream));
    }
    V_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    V->n_cams = S.n_images;
    V->cams_of = S.generation;
  }
  return B2M_OK;
}

int verify_guided_slot(b2m_ctx* ctx, int s, GuidedSlot* out) {
  VerifyState* V = vstate(ctx);
  if (!V->d_guided_kind) {
    V_TRY(ctx, cudaMalloc(&V->d_guided_kind, sizeof(int32_t) * V->batch));
    V_TRY(ctx, cudaMalloc(&V->d_guided_model, sizeof(float) * 9 * V->batch));
    for (int k = 0; k < 2; ++k) {
      V_TRY(ctx, cudaMalloc(&V->d_garena[k], sizeof(uint2) * V->arena_cap));
      V_TRY(ctx, cudaMalloc(&V->d_gcursor[k], sizeof(unsigned long long)));
      V_TRY(ctx, cudaMalloc(&V->d_goff[k], sizeof(int64_t) * V->batch));
      V_TRY(ctx, cudaMalloc(&V->d_gcnt[k], sizeof(int32_t) * V->batch));
      V_TRY(ctx, cudaMallocHost(&V->h_garena[k], sizeof(uint2) * V->arena_cap));
      V_TRY(ctx, cudaMallocHost(&V->h_gcursor[k], sizeof(unsigned long long)));
      V_TRY(ctx, cudaMallocHost(&V->h_goff[k], sizeof(int64_t) * V->batch));
      V_TRY(ctx, cudaMallocHost(&V->h_gcnt[k], sizeof(int32_t) * V->batch));
    }
  }
  out->kind = V->d_guided_kind;
  out->model = V->d_guided_model;
  out->arena = V->d_garena[s];
  out->cursor = V->d_gcursor[s];
  out->off = V->d_goff[s];
  out->cnt = V->d_gcnt[s];
  out->h_cursor = V->h_gcursor[s];
  V->guided_on[s] = true;
  return B2M_OK;
}

void verify_results_init(b2m_results* res, int64_t n_pairs) {
  res->verified = true;
  res->config.assign(n_pairs, B2M_UNDEFINED);
  res->in_off.assign(n_pairs, 0);
  res->in_cnt.assign(n_pairs, 0);
  res->model_idx.assign(n_pairs, -1);
  res->models.clear();
  res->poses.clear();
  res->pose_valid.clear();
}

int verify_batch_launch(b2m_ctx* ctx, ImageSet& S, const b2m_tvg_opts* tvg, const b2m_sift_opts* sift, int s,
                        int64_t p0, int nb) {
  VerifyState* V = vstate(ctx);
  Workspace& W = ctx->ws;
  VerifyParams P{};
  P.pairs = ctx->d_pairs + 2 * p0;
  P.pair_off = W.d_pair_off[s];
  P.pair_cnt = W.d_pair_cnt[s];
  P.pts = V->d_pts[s];
  P.matches = W.d_arena[s];
  P.cams = V->d_cams;
  P.mask = V->d_mask;
  P.arena_cap = V->arena_cap;
  P.models = V->d_models[s];
  P.sup_cnt = V->d_sup;
  P.success = V->d_success;
  P.config = V->d_config[s];
  P.inl_cnt = V->d_inl_cnt[s];
  P.inliers = V->d_inliers[s];
  P.opt = *tvg;
  P.seed = ctx->seed;
  P.single_kind = -1;
  P.force_calibrated = -1;
  V->guided_on[s] = false;
  P.guided_min_inliers = -1;
  if (sift && sift->guided_matching) {
    GuidedSlot gs;
    if (int rc = verify_guided_slot(ctx, s, &gs)) return rc;
    P.guided_kind = gs.kind;
    P.guided_model = gs.model;
    P.guided_min_inliers = tvg->min_num_inliers;
  }
  if (!V->d_prof && getenv("B2M_PROF")) {
    cudaMalloc(&V->d_prof, sizeof(unsigned long long) * 24);
    cudaMemset(V->d_prof, 0, sizeof(unsigned long long) * 24);
  }
  P.prof = V->d_prof;
  P.counters = verify_counters(ctx);
  P.e_scratch = V->d_e_scratch;
  P.lo_eig_thread = lo_eig_thread_mode();
  if (!V->rs.side[0]) {
    V_TRY(ctx, cudaStreamCreateWithFlags(&V->rs.side[0], cudaStreamNonBlocking));
    V_TRY(ctx, cudaStreamCreateWithFlags(&V->rs.side[1], cudaStreamNonBlocking));
    V_TRY(ctx, cudaEventCreateWithFlags(&V->rs.fork, cudaEventDisableTiming));
    V_TRY(ctx, cudaEventCreateWithFlags(&V->rs.join[0], cudaEventDisableTiming));
    V_TRY(ctx, cudaEventCreateWithFlags(&V->rs.join[1], cudaEventDisableTiming));
  }
  const double4* pts_E = nullptr;
  if (V->any_distorted) {  // distortion models: the E kernel reads undistorted points (row V9)
    if (!V->d_pts_undist[s]) V_TRY(ctx, cudaMalloc(&V->d_pts_undist[s], sizeof(double4) * V->arena_cap));
    b2m_undistort_kernel<<<nb, 256, 0, ctx->stream>>>(P, V->d_dist, V->d_pts_undist[s]);
    V_TRY(ctx, cudaGetLastError());
    ctx->stats.kernel_launches += 1;
    pts_E = V->d_pts_undist[s];
  }
  V_TRY(ctx, launch_ransac(P, nb, ctx->stream, &V->rs, pts_E));
  ctx->stats.kernel_launches += 2;
  b2m_decide_kernel<<<nb, 256, 0, ctx->stream>>>(P);
  V_TRY(ctx, cudaGetLastError());
  ctx->stats.kernel_launches += 2;
  V->pose_on[s] = false;
  if (tvg->compute_relative_pose) {  // EstimateTwoViewGeometryPose on the verified pairs of the batch
    if (!V->d_angles) V_TRY(ctx, cudaMalloc(&V->d_angles, sizeof(double) * V->arena_cap));
    if (!V->d_pose[s]) {
      V_TRY(ctx, cudaMalloc(&V->d_pose[s], sizeof(double) * 8 * V->batch));
      V_TRY(ctx, cudaMalloc(&V->d_pose_valid[s], sizeof(int32_t) * V->batch));
      V_TRY(ctx, cudaMallocHost(&V->h_pose[s], sizeof(double) * 8 * V->batch));
      V_TRY(ctx, cudaMallocHost(&V->h_pose_valid[s], sizeof(int32_t) * V->batch));
    }
    PoseParams Q{};
    Q.pairs = P.pairs;
    Q.pair_off = P.pair_off;
    Q.inl_cnt = P.inl_cnt;
    Q.config = P.config;
    Q.inliers = P.inliers;
    Q.models = P.models;
    Q.cams = P.cams;
    Q.dist = V->any_distorted ? V->d_dist : nullptr;
    Q.kpts = S.d_kpts;
    Q.img_row0 = S.d_row0;
    Q.angles = V->d_angles;
    Q.out = V->d_pose[s];
    Q.out_valid = V->d_pose_valid[s];
    b2m_pose_kernel<<<nb, 256, 0, ctx->stream>>>(Q);
    V_TRY(ctx, cudaGetLastError());
    ctx->stats.kernel_launches += 1;
    V->pose_on[s] = true;
  }
  return B2M_OK;
}

int verify_batch_download(b2m_ctx* ctx, b2m_results*, int s, int64_t, int nb) {
  VerifyState* V = vstate(ctx);
  Workspace& W = ctx->ws;
  const unsigned long long total = *W.h_cursor[s];
  V_TRY(ctx, cudaMemcpyAsync(V->h_models[s], V->d_models[s], sizeof(double) * 27 * nb, cudaMemcpyDeviceToHost,
                             ctx->copy_stream));
  V_TRY(ctx, cudaMemcpyAsync(V->h_config[s], V->d_config[s], sizeof(int32_t) * nb, cudaMemcpyDeviceToHost,
                             ctx->copy_stream));
  V_TRY(ctx, cudaMemcpyAsync(V->h_inl_cnt[s], V->d_inl_cnt[s], sizeof(int32_t) * nb, cudaMemcpyDeviceToHost,
                             ctx->copy_stream));
  if (total > 0)
    V_TRY(ctx, cudaMemcpyAsync(V->h_inliers[s], V->d_inliers[s], sizeof(uint2) * total, cudaMemcpyDeviceToHost,
                               ctx->copy_stream));
  if (V->pose_on[s]) {
    V_TRY(ctx, cudaMemcpyAsync(V->h_pose[s], V->d_pose[s], sizeof(double) * 8 * nb, cudaMemcpyDeviceToHost, ctx->copy_stream));
    V_TRY(ctx, cudaMemcpyAsync(V->h_pose_valid[s], V->d_pose_valid[s], sizeof(int32_t) * nb, cudaMemcpyDeviceToHost,
                               ctx->copy_stream));
  }
  if (V->guided_on[s]) {
    const unsigned long long gtotal = *V->h_gcursor[s];
    V_TRY(ctx, cudaMemcpyAsync(V->h_goff[s], V->d_goff[s], sizeof(int64_t) * nb, cudaMemcpyDeviceToHost,
                               ctx->copy_stream));
    V_TRY(ctx, cudaMemcpyAsync(V->h_gcnt[s], V->d_gcnt[s], sizeof(int32_t) * nb, cudaMemcpyDeviceToHost,
                               ctx->copy_stream));
    if (gtotal > 0)
      V_TRY(ctx, cudaMemcpyAsync(V->h_garena[s], V->d_garena[s], sizeof(uint2) * gtotal, cudaMemcpyDeviceToHost,
                                 ctx->copy_stream));
  }
  return B2M_OK;
}

int verify_batch_collect(b2m_ctx* ctx, b2m_results* res, int s, int64_t p0, int nb, int min_num_inliers) {
  VerifyState* V = vstate(ctx);
  Workspace& W = ctx->ws;
  for (int k = 0; k < nb; ++k) {
    const int64_t p = p0 + k;
    int cfg = V->h_config[s][k];
    int ni = V->h_inl_cnt[s][k];
    const uint2* inl_src = V->h_inliers[s] + W.h_pair_off[s][k];
    if (V->guided_on[s] && V->h_gcnt[s][k] >= 0) {
      // guided matching replaced TwoViewGeometry::inlier_matches (U:feature/sift.cc MatchGuidedSiftFeaturesCPU)
      ni = V->h_gcnt[s][k];
      inl_src = V->h_garena[s] + V->h_goff[s][k];
    }
    // FeatureMatcherController::Match write rule (row P3): raw matches below min_num_inliers are
    // stored empty (the verifier never ran: default TwoViewGeometry); geometries with fewer than
    // min_num_inliers inliers are stored as the default TwoViewGeometry (config UNDEFINED).
    if (res->cnt[p] < min_num_inliers) {
      res->cnt[p] = 0;
      cfg = B2M_UNDEFINED;
      ni = 0;
    }
    if (ni < min_num_inliers) {
      cfg = B2M_UNDEFINED;
      ni = 0;
    }
    if (V->pose_on[s]) {
      if (res->poses.empty()) {
        const size_t np = res->config.size();
        res->poses.assign(8 * np, 0.0);
        for (size_t q = 0; q < np; ++q) res->poses[8 * q] = 1.0;
        res->pose_valid.assign(np, 0);
      }
      if (ni > 0 && V->h_pose_valid[s][k]) {
        memcpy(res->poses.data() + 8 * p, V->h_pose[s] + 8 * k, sizeof(double) * 8);
        res->pose_valid[p] = 1;
      }
    }
    res->config[p] = cfg;
    res->in_cnt[p] = ni;
    res->in_off[p] = static_cast<int64_t>(res->inliers.size() / 2);
    if (ni > 0) {
      const uint2* src = inl_src;
      const size_t at = res->inliers.size();
      res->inliers.resize(at + 2 * static_cast<size_t>(ni));
      memcpy(res->inliers.data() + at, src, sizeof(uint2) * ni);
      res->model_idx[p] = static_cast<int32_t>(res->models.size() / 27);
      res->models.insert(res->models.end(), V->h_models[s] + 27 * k, V->h_models[s] + 27 * k + 27);
    }
  }
  return B2M_OK;
}

void verify_release(b2m_ctx* ctx) {
  if (ctx->verify_state) {
    VerifyState* V = static_cast<VerifyState*>(ctx->verify_state);
    if (V->d_prof) {
      unsigned long long h[24];
      cudaMemcpy(h, V->d_prof, sizeof(h), cudaMemcpyDeviceToHost);
      const char* names[8] = {"solve", "score", "exact_support", "lo_accumulate", "lo_solve", "lo_score", "final", "-"};
      for (int k = 0; k < 3; ++k)
        for (int j = 0; j < 7; ++j)
          fprintf(stderr, "[b2m prof] kind %d %-14s %10.3f Mcycles\n", k, names[j], h[k * 8 + j] / 1e6);
      cudaFree(V->d_prof);
      V->d_prof = nullptr;
    }
    V->release();
    delete V;
    ctx->verify_state = nullptr;
  }
}

// ---- stand-alone estimators ------------------------------------------------------------------

namespace {

struct Single {
  double4* d_pts = nullptr;
  uint2* d_matches = nullptr;
  uint2* d_inliers = nullptr;
  uint8_t* d_mask = nullptr;
  DevCamera* d_cams = nullptr;
  int32_t* d_i32 = nullptr;   // pairs[2], cnt[1], sup[3], success[3], config[1], inl_cnt[1]
  int64_t* d_off = nullptr;
  double* d_models = nullptr;
  DevDistortion* d_dist = nullptr;  // only when a camera has distortion
  double4* d_pts_undist = nullptr;
  double* d_e_scratch = nullptr;    // E kernel scratch, [problems][128][90]
  // compute_relative_pose
  double *d_p1 = nullptr, *d_p2 = nullptr, *d_angles = nullptr, *d_pose = nullptr;
  int64_t *d_p1_off = nullptr, *d_p2_off = nullptr;
  int32_t* d_pose_valid = nullptr;
  ~Single() {
    cudaFree(d_pts); cudaFree(d_matches); cudaFree(d_inliers); cudaFree(d_mask); cudaFree(d_cams);
    cudaFree(d_i32); cudaFree(d_off); cudaFree(d_models); cudaFree(d_dist); cudaFree(d_pts_undist); cudaFree(d_e_scratch);
    cudaFree(d_p1); cudaFree(d_p2); cudaFree(d_angles); cudaFree(d_pose); cudaFree(d_p1_off); cudaFree(d_p2_off);
    cudaFree(d_pose_valid);
  }
};

// Stand-alone estimator calls with compute_relative_pose: upload the callers' point arrays (concatenated over the
// `nb` problems, offsets in points) and run the pose kernel after the decision kernel.  `P` is the VerifyParams the
// RANSAC / decision kernels ran with; G.d_dist may be null (no distortion).  Outputs stay in G.d_pose / d_pose_valid.
int launch_pose_standalone(b2m_ctx* ctx, Single& G, const VerifyParams& P, int nb, int64_t cap, const std::vector<double>& p1,
                           const std::vector<double>& p2, const std::vector<int64_t>& off1, const std::vector<int64_t>& off2,
                           const b2m_camera* const* cams, int n_cams, cudaStream_t st) {
  V_TRY(ctx, cudaMalloc(&G.d_p1, sizeof(double) * std::max<size_t>(p1.size(), 2)));
  V_TRY(ctx, cudaMalloc(&G.d_p2, sizeof(double) * std::max<size_t>(p2.size(), 2)));
  V_TRY(ctx, cudaMalloc(&G.d_p1_off, sizeof(int64_t) * nb));
  V_TRY(ctx, cudaMalloc(&G.d_p2_off, sizeof(int64_t) * nb));
  V_TRY(ctx, cudaMalloc(&G.d_angles, sizeof(double) * cap));
  V_TRY(ctx, cudaMalloc(&G.d_pose, sizeof(double) * 8 * nb));
  V_TRY(ctx, cudaMalloc(&G.d_pose_valid, sizeof(int32_t) * nb));
  if (!G.d_dist) {  // undistort_for_E uploads the models only when it had to; the pose kernel needs them as well
    bool any = false;
    for (int i = 0; i < n_cams; ++i) any = any || cam::has_distortion(cams[i]->model);
    if (any) {
      std::vector<DevDistortion> dd(n_cams);
      for (int i = 0; i < n_cams; ++i) dd[i] = to_dist(*cams[i]);
      V_TRY(ctx, cudaMalloc(&G.d_dist, sizeof(DevDistortion) * n_cams));
      V_TRY(ctx, cudaMemcpy(G.d_dist, dd.data(), sizeof(DevDistortion) * n_cams, cudaMemcpyHostToDevice));
    }
  }
  // synchronous copies: the host vectors are the caller's locals
  if (!p1.empty()) V_TRY(ctx, cudaMemcpy(G.d_p1, p1.data(), sizeof(double) * p1.size(), cudaMemcpyHostToDevice));
  if (!p2.empty()) V_TRY(ctx, cudaMemcpy(G.d_p2, p2.data(), sizeof(double) * p2.size(), cudaMemcpyHostToDevice));
  V_TRY(ctx, cudaMemcpy(G.d_p1_off, off1.data(), sizeof(int64_t) * nb, cudaMemcpyHostToDevice));
  V_TRY(ctx, cudaMemcpy(G.d_p2_off, off2.data(), sizeof(int64_t) * nb, cudaMemcpyHostToDevice));
  PoseParams Q{};
  Q.pairs = P.pairs;
  Q.pair_off = P.pair_off;
  Q.inl_cnt = P.inl_cnt;
  Q.config = P.config;
  Q.inliers = P.inliers;
  Q.models = P.models;
  Q.cams = P.cams;
  Q.dist = G.d_dist;
  Q.pts1 = G.d_p1;
  Q.pts2 = G.d_p2;
  Q.pts1_off = G.d_p1_off;
  Q.pts2_off = G.d_p2_off;
  Q.angles = G.d_angles;
  Q.out = G.d_pose;
  Q.out_valid = G.d_pose_valid;
  b2m_pose_kernel<<<nb, 256, 0, st>>>(Q);
  V_TRY(ctx, cudaGetLastError());
  ctx->stats.kernel_launches += 1;
  return B2M_OK;
}

// copy the pose of problem k (device arrays already downloaded into h_pose / h_valid) into a result
void fill_pose(b2m_tvg_result* r, const double* h_pose, const int32_t* h_valid, int k) {
  r->qvec[0] = 1.0;
  if (h_pose && h_valid && h_valid[k] && r->n_inliers > 0) {
    memcpy(r->qvec, h_pose + 8 * k, sizeof(double) * 4);
    memcpy(r->tvec, h_pose + 8 * k + 4, sizeof(double) * 3);
    r->tri_angle = h_pose[8 * k + 7];
    r->pose_valid = 1;
  }
}

// Stand-alone estimator calls: upload the full camera models and undistort the E-kernel input when any
// of the `n_cams` cameras has a distortion function.  Returns the E arena (nullptr: use P.pts) in *pts_E.
int undistort_for_E(b2m_ctx* ctx, Single& G, const VerifyParams& P, const b2m_camera* const* cams, int n_cams, int nb,
                    int64_t cap, cudaStream_t st, const double4** pts_E) {
  *pts_E = nullptr;
  bool any = false;
  for (int i = 0; i < n_cams; ++i) any = any || cam::has_distortion(cams[i]->model);
  if (!any) return B2M_OK;
  std::vector<DevDistortion> dd(n_cams);
  for (int i = 0; i < n_cams; ++i) dd[i] = to_dist(*cams[i]);
  V_TRY(ctx, cudaMalloc(&G.d_dist, sizeof(DevDistortion) * n_cams));
  V_TRY(ctx, cudaMalloc(&G.d_pts_undist, sizeof(double4) * cap));
  // synchronous copy: `dd` is a local that must not be read after this function returns
  V_TRY(ctx, cudaMemcpy(G.d_dist, dd.data(), sizeof(DevDistortion) * n_cams, cudaMemcpyHostToDevice));
  b2m_undistort_kernel<<<nb, 256, 0, st>>>(P, G.d_dist, G.d_pts_undist);
  V_TRY(ctx, cudaGetLastError());
  ctx->stats.kernel_launches += 1;
  *pts_E = G.d_pts_undist;
  return B2M_OK;
}

// `full_cams`: the two cameras with their distortion parameters, or nullptr (single-model API: the
// caller's points are already in the frame the model is estimated in).
int run_single(b2m_ctx* ctx, const std::vector<double4>& pts, const std::vector<uint2>& matches, const DevCamera cams[2],
               const b2m_tvg_opts& opt, int single_kind, Single& G, VerifyParams& P,
               const b2m_camera* const* full_cams = nullptr, const double* raw1 = nullptr, int64_t n1 = 0,
               const double* raw2 = nullptr, int64_t n2 = 0) {
  const int64_t m = static_cast<int64_t>(pts.size());
  const int64_t cap = std::max<int64_t>(m, 1);
  V_TRY(ctx, cudaMalloc(&G.d_pts, sizeof(double4) * cap));
  V_TRY(ctx, cudaMalloc(&G.d_matches, sizeof(uint2) * cap));
  V_TRY(ctx, cudaMalloc(&G.d_inliers, sizeof(uint2) * cap));
  V_TRY(ctx, cudaMalloc(&G.d_mask, 3 * cap));
  V_TRY(ctx, cudaMalloc(&G.d_cams, sizeof(DevCamera) * 2));
  V_TRY(ctx, cudaMalloc(&G.d_i32, sizeof(int32_t) * 16));
  V_TRY(ctx, cudaMalloc(&G.d_off, sizeof(int64_t)));
  V_TRY(ctx, cudaMalloc(&G.d_models, sizeof(double) * 27));
  V_TRY(ctx, cudaMalloc(&G.d_e_scratch, sizeof(double) * kEStride * kRansacThreads));
  const int32_t i32[16] = {0, 1, static_cast<int32_t>(m), 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  const int64_t off0 = 0;
  cudaStream_t st = ctx->stream;
  if (m > 0) {
    V_TRY(ctx, cudaMemcpyAsync(G.d_pts, pts.data(), sizeof(double4) * m, cudaMemcpyHostToDevice, st));
    V_TRY(ctx, cudaMemcpyAsync(G.d_matches, matches.data(), sizeof(uint2) * m, cudaMemcpyHostToDevice, st));
  }
  V_TRY(ctx, cudaMemcpyAsync(G.d_cams, cams, sizeof(DevCamera) * 2, cudaMemcpyHostToDevice, st));
  V_TRY(ctx, cudaMemcpyAsync(G.d_i32, i32, sizeof(i32), cudaMemcpyHostToDevice, st));
  V_TRY(ctx, cudaMemcpyAsync(G.d_off, &off0, sizeof(int64_t), cudaMemcpyHostToDevice, st));
  V_TRY(ctx, cudaMemsetAsync(G.d_models, 0, sizeof(double) * 27, st));
  P = VerifyParams{};
  P.pairs = G.d_i32;
  P.pair_cnt = G.d_i32 + 2;
  P.sup_cnt = G.d_i32 + 3;
  P.success = G.d_i32 + 6;
  P.config = G.d_i32 + 9;
  P.inl_cnt = G.d_i32 + 10;
  P.pair_off = G.d_off;
  P.pts = G.d_pts;
  P.matches = G.d_matches;
  P.cams = G.d_cams;
  P.mask = G.d_mask;
  P.arena_cap = cap;
  P.models = G.d_models;
  P.inliers = G.d_inliers;
  P.opt = opt;
  P.seed = ctx->seed;
  P.single_kind = single_kind;
  P.counters = verify_counters(ctx);
  P.e_scratch = G.d_e_scratch;
  P.lo_eig_thread = lo_eig_thread_mode();
  if (single_kind >= 0) {
    V_TRY(ctx, launch_ransac(P, 1, st));
  } else {
    const double4* pts_E = nullptr;
    if (full_cams)
      if (int rc = undistort_for_E(ctx, G, P, full_cams, 2, 1, cap, st, &pts_E)) return rc;
    V_TRY(ctx, launch_ransac(P, 1, st, nullptr, pts_E));
    ctx->stats.kernel_launches += 2;
    b2m_decide_kernel<<<1, 256, 0, st>>>(P);
    ctx->stats.kernel_launches += 1;
    if (opt.compute_relative_pose && full_cams) {
      V_TRY(ctx, cudaGetLastError());
      const std::vector<double> p1(raw1, raw1 + 2 * n1), p2(raw2, raw2 + 2 * n2);
      const std::vector<int64_t> zero(1, 0);
      if (int rc = launch_pose_standalone(ctx, G, P, 1, cap, p1, p2, zero, zero, full_cams, 2, st)) return rc;
    }
  }
  V_TRY(ctx, cudaGetLastError());
  ctx->stats.kernel_launches += 1;
  return B2M_OK;
}

// Instrumentation: the warp-cooperative 5-point solver on caller-provided null spaces, one warp each.
__global__ void __launch_bounds__(128) b2m_five_point_kernel(const double* __restrict__ nullspaces, int64_t n,
                                                             double* __restrict__ models, int32_t* __restrict__ counts) {
  __shared__ fpw::Scratch ws[4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t h = static_cast<int64_t>(blockIdx.x) * 4 + warp;
  if (h >= n) return;
  for (int k = lane; k < 36; k += 32) ws[warp].N[k] = nullspaces[h * 36 + k];
  __syncwarp();
  const int cnt = fpw::five_point_warp(ws[warp], models + h * 90, lane);
  if (lane == 0) counts[h] = cnt;
}

__global__ void b2m_sampson_kernel(const double* p1, const double* p2, int64_t m, const double* E, double* out) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= m) return;
  double M[9];
  for (int k = 0; k < 9; ++k) M[k] = E[k];
  out[i] = sampson_sq(M, p1[2 * i], p1[2 * i + 1], p2[2 * i], p2[2 * i + 1]);
}

__global__ void b2m_cam_from_img_kernel(const DevDistortion* c, const double* pts, int64_t n, double* out) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  cam::cam_from_img(c->model, c->p, pts[2 * i], pts[2 * i + 1], &out[2 * i], &out[2 * i + 1]);
}

}  // namespace
}  // namespace b2m

using namespace b2m;

extern "C" {

// One EstimateTwoViewGeometry run (multiple_models ignored): the body of b2m_estimate_two_view_geometry.
static int estimate_tvg_once(b2m_ctx* ctx, const b2m_camera* cam1, const double* points1, int64_t n1,
                             const b2m_camera* cam2, const double* points2, int64_t n2, const uint32_t* matches,
                             int64_t m, const b2m_tvg_opts* opts, b2m_tvg_result* out, uint32_t* inlier_matches) {
  if (!ctx) return B2M_EINVAL;
  auto bad = [&](const char* msg) {
    ctx->err = msg;
    return B2M_EINVAL;
  };
  if (!cam1 || !cam2 || !opts || !out) return bad("[verify.cu] Check Failed: cameras, options and out != NULL");
  if (const char* why = camera_problem(*cam1)) return bad(why);
  if (const char* why = camera_problem(*cam2)) return bad(why);
  if (n1 < 0 || n2 < 0 || (n1 > 0 && !points1) || (n2 > 0 && !points2)) return bad("[verify.cu] Check Failed: points");
  if (!matches) {  // identity matching (R:estimators/two_view_geometry.h:136-142)
    if (n1 != n2) return bad("[verify.cu] Check Failed: points1.size() == points2.size()");
    m = n1;
  }
  if (m < 0) return bad("[verify.cu] Check Failed: m >= 0");
  cudaSetDevice(ctx->device);
  std::vector<double4> pts(m);
  std::vector<uint2> mm(m);
  for (int64_t i = 0; i < m; ++i) {
    const uint32_t a = matches ? matches[2 * i] : static_cast<uint32_t>(i);
    const uint32_t b = matches ? matches[2 * i + 1] : static_cast<uint32_t>(i);
    if (a >= n1 || b >= n2) return bad("[verify.cu] Check Failed: match index < number of points");
    pts[i] = make_double4(points1[2 * a], points1[2 * a + 1], points2[2 * b], points2[2 * b + 1]);
    mm[i] = make_uint2(a, b);
  }
  const DevCamera cams[2] = {to_dev(*cam1), to_dev(*cam2)};
  Single G;
  VerifyParams P;
  const b2m_camera* full_cams[2] = {cam1, cam2};
  if (int rc = run_single(ctx, pts, mm, cams, *opts, -1, G, P, full_cams, points1, n1, points2, n2)) return rc;
  int32_t i32[16];
  double models[27];
  double h_pose[8] = {1, 0, 0, 0, 0, 0, 0, 0};
  int32_t h_pose_valid = 0;
  V_TRY(ctx, cudaMemcpyAsync(i32, G.d_i32, sizeof(i32), cudaMemcpyDeviceToHost, ctx->stream));
  V_TRY(ctx, cudaMemcpyAsync(models, G.d_models, sizeof(models), cudaMemcpyDeviceToHost, ctx->stream));
  if (G.d_pose) {
    V_TRY(ctx, cudaMemcpyAsync(h_pose, G.d_pose, sizeof(h_pose), cudaMemcpyDeviceToHost, ctx->stream));
    V_TRY(ctx, cudaMemcpyAsync(&h_pose_valid, G.d_pose_valid, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  }
  V_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  memset(out, 0, sizeof(*out));
  out->struct_size = sizeof(*out);
  out->config = i32[9];
  out->n_inliers = i32[10];
  fill_pose(out, h_pose, &h_pose_valid, 0);
  out->nE = i32[3]; out->nF = i32[4]; out->nH = i32[5];
  memcpy(out->E, models, sizeof(double) * 9);
  memcpy(out->F, models + 9, sizeof(double) * 9);
  memcpy(out->H, models + 18, sizeof(double) * 9);
  if (out->n_inliers > 0 && inlier_matches) {
    V_TRY(ctx, cudaMemcpy(inlier_matches, G.d_inliers, sizeof(uint2) * out->n_inliers, cudaMemcpyDeviceToHost));
  }
  return B2M_OK;
}

// EstimateTwoViewGeometry; with opts->multiple_models the loop of EstimateMultipleTwoViewGeometries
// (U:estimators/two_view_geometry.cc): estimate on the remaining matches, keep the geometry (a WATERMARK one
// only if !multiple_ignore_watermark), remove its inliers from the remaining matches, repeat until the
// estimate is DEGENERATE.  No geometry -> DEGENERATE; one -> that geometry; several -> config MULTIPLE with the
// inlier lists concatenated in the order they were found and default (zero) E / F / H.  Every round is one run
// of the GPU verifier; the loop itself is host control flow, as upstream.
int b2m_estimate_two_view_geometry(b2m_ctx* ctx, const b2m_camera* cam1, const double* points1, int64_t n1,
                                   const b2m_camera* cam2, const double* points2, int64_t n2,
                                   const uint32_t* matches, int64_t m, const b2m_tvg_opts* opts,
                                   b2m_tvg_result* out, uint32_t* inlier_matches) {
  if (!ctx) return B2M_EINVAL;
  if (!opts || !opts->multiple_models)
    return estimate_tvg_once(ctx, cam1, points1, n1, cam2, points2, n2, matches, m, opts, out, inlier_matches);
  if (!out) {
    ctx->err = "[verify.cu] Check Failed: out != NULL";
    return B2M_EINVAL;
  }
  if (!matches) {
    if (n1 != n2) {
      ctx->err = "[verify.cu] Check Failed: points1.size() == points2.size()";
      return B2M_EINVAL;
    }
    m = n1;
  }
  if (m < 0) {
    ctx->err = "[verify.cu] Check Failed: m >= 0";
    return B2M_EINVAL;
  }
  std::vector<uint32_t> remaining(static_cast<size_t>(m) * 2);
  for (int64_t i = 0; i < m; ++i) {
    remaining[2 * i] = matches ? matches[2 * i] : static_cast<uint32_t>(i);
    remaining[2 * i + 1] = matches ? matches[2 * i + 1] : static_cast<uint32_t>(i);
  }
  b2m_tvg_opts once = *opts;
  once.multiple_models = 0;
  std::vector<b2m_tvg_result> found;
  std::vector<std::vector<uint32_t>> found_inl;
  for (;;) {
    b2m_tvg_result g;
    const int64_t rem = static_cast<int64_t>(remaining.size() / 2);
    std::vector<uint32_t> inl(static_cast<size_t>(std::max<int64_t>(rem, 1)) * 2);
    if (int rc = estimate_tvg_once(ctx, cam1, points1, n1, cam2, points2, n2, remaining.data(), rem, &once, &g, inl.data()))
      return rc;
    if (g.config == B2M_DEGENERATE || g.n_inliers <= 0) break;
    inl.resize(static_cast<size_t>(g.n_inliers) * 2);
    // ExtractOutlierMatches: the matches that are not inliers of this geometry stay
    std::vector<uint64_t> keys(static_cast<size_t>(g.n_inliers));
    for (int64_t i = 0; i < g.n_inliers; ++i) keys[i] = (static_cast<uint64_t>(inl[2 * i]) << 32) | inl[2 * i + 1];
    std::sort(keys.begin(), keys.end());
    std::vector<uint32_t> next;
    next.reserve(remaining.size());
    for (int64_t i = 0; i < rem; ++i) {
      const uint64_t k = (static_cast<uint64_t>(remaining[2 * i]) << 32) | remaining[2 * i + 1];
      if (!std::binary_search(keys.begin(), keys.end(), k)) {
        next.push_back(remaining[2 * i]);
        next.push_back(remaining[2 * i + 1]);
      }
    }
    if (!(opts->multiple_ignore_watermark && g.config == B2M_WATERMARK)) {
      found.push_back(g);
      found_inl.push_back(std::move(inl));
    }
    remaining.swap(next);
  }
  memset(out, 0, sizeof(*out));
  out->struct_size = sizeof(*out);
  out->qvec[0] = 1.0;
  if (found.empty()) {
    out->config = B2M_DEGENERATE;
    return B2M_OK;
  }
  if (found.size() == 1) {
    *out = found[0];
  } else {
    out->config = B2M_MULTIPLE;
  }
  int64_t total = 0;
  for (const std::vector<uint32_t>& v : found_inl) {
    if (inlier_matches && !v.empty()) memcpy(inlier_matches + 2 * total, v.data(), v.size() * sizeof(uint32_t));
    total += static_cast<int64_t>(v.size() / 2);
  }
  out->n_inliers = total;
  return B2M_OK;
}

// Batched variant of b2m_estimate_two_view_geometry: the same kernels the pair pipeline uses (one CTA
// per problem and model kind, then one decision CTA per problem), fed from caller-provided point sets.
int b2m_estimate_two_view_geometry_batch(b2m_ctx* ctx, const b2m_tvg_problem* problems, int64_t n_problems,
                                         const b2m_tvg_opts* opts, b2m_tvg_result* out,
                                         uint32_t* const* inlier_matches) {
  if (!ctx) return B2M_EINVAL;
  auto bad = [&](const char* msg) {
    ctx->err = msg;
    return B2M_EINVAL;
  };
  if (n_problems < 0 || (n_problems > 0 && (!problems || !out)) || !opts)
    return bad("[verify.cu] Check Failed: problems, options and out != NULL");
  if (opts->multiple_models)
    return bad("[verify.cu] multiple_models: use b2m_estimate_two_view_geometry (the per-problem loop is sequential)");
  for (int64_t k = 0; k < n_problems; ++k) {
    const b2m_tvg_problem& q = problems[k];
    if (q.n1 < 0 || q.n2 < 0 || (q.n1 > 0 && !q.points1) || (q.n2 > 0 && !q.points2))
      return bad("[verify.cu] Check Failed: points");
    if (!q.matches && q.n1 != q.n2) return bad("[verify.cu] Check Failed: points1.size() == points2.size()");
    if (q.matches && q.m < 0) return bad("[verify.cu] Check Failed: m >= 0");
    if ((q.matches ? q.m : q.n1) > INT32_MAX) return bad("[verify.cu] Check Failed: matches per problem < 2^31");
    if (const char* why = camera_problem(q.cam1)) return bad(why);
    if (const char* why = camera_problem(q.cam2)) return bad(why);
  }
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  constexpr int64_t kChunk = 4096;  // problems per launch: bounds the staging memory, plenty to fill 132 SMs
  for (int64_t k0 = 0; k0 < n_problems; k0 += kChunk) {
    const int nb = static_cast<int>(std::min(kChunk, n_problems - k0));
    std::vector<double4> pts;
    std::vector<uint2> mm;
    std::vector<int64_t> off(nb);
    std::vector<int32_t> cnt(nb), pairs(2 * nb);
    std::vector<DevCamera> cams(2 * nb);
    std::vector<const b2m_camera*> full_cams(2 * nb);
    std::vector<double> raw1, raw2;            // compute_relative_pose: the callers' point arrays, concatenated
    std::vector<int64_t> raw1_off(nb, 0), raw2_off(nb, 0);
    for (int k = 0; k < nb; ++k) {
      const b2m_tvg_problem& q = problems[k0 + k];
      full_cams[2 * k] = &q.cam1;
      full_cams[2 * k + 1] = &q.cam2;
      if (opts->compute_relative_pose) {
        raw1_off[k] = static_cast<int64_t>(raw1.size() / 2);
        raw2_off[k] = static_cast<int64_t>(raw2.size() / 2);
        raw1.insert(raw1.end(), q.points1, q.points1 + 2 * q.n1);
        raw2.insert(raw2.end(), q.points2, q.points2 + 2 * q.n2);
      }
      const int64_t m = q.matches ? q.m : q.n1;
      off[k] = static_cast<int64_t>(pts.size());
      cnt[k] = static_cast<int32_t>(m);
      pairs[2 * k] = 2 * k;
      pairs[2 * k + 1] = 2 * k + 1;
      cams[2 * k] = to_dev(q.cam1);
      cams[2 * k + 1] = to_dev(q.cam2);
      for (int64_t i = 0; i < m; ++i) {
        const uint32_t a = q.matches ? q.matches[2 * i] : static_cast<uint32_t>(i);
        const uint32_t b = q.matches ? q.matches[2 * i + 1] : static_cast<uint32_t>(i);
        if (a >= q.n1 || b >= q.n2) return bad("[verify.cu] Check Failed: match index < number of points");
        pts.push_back(make_double4(q.points1[2 * a], q.points1[2 * a + 1], q.points2[2 * b], q.points2[2 * b + 1]));
        mm.push_back(make_uint2(a, b));
      }
    }
    const int64_t total = static_cast<int64_t>(pts.size());
    const int64_t cap = std::max<int64_t>(total, 1);
    Single G;  // owns the arenas; the per-problem scalars live in one int32 block (see the offsets below)
    int32_t* d_i32 = nullptr;  // pairs[2nb] cnt[nb] sup[3nb] success[3nb] config[nb] inl_cnt[nb]
    V_TRY(ctx, cudaMalloc(&G.d_pts, sizeof(double4) * cap));
    V_TRY(ctx, cudaMalloc(&G.d_matches, sizeof(uint2) * cap));
    V_TRY(ctx, cudaMalloc(&G.d_inliers, sizeof(uint2) * cap));
    V_TRY(ctx, cudaMalloc(&G.d_mask, 3 * cap));
    V_TRY(ctx, cudaMalloc(&G.d_cams, sizeof(DevCamera) * 2 * nb));
    V_TRY(ctx, cudaMalloc(&G.d_i32, sizeof(int32_t) * 11 * nb));
    V_TRY(ctx, cudaMalloc(&G.d_off, sizeof(int64_t) * nb));
    V_TRY(ctx, cudaMalloc(&G.d_models, sizeof(double) * 27 * nb));
    V_TRY(ctx, cudaMalloc(&G.d_e_scratch, sizeof(double) * kEStride * kRansacThreads * static_cast<size_t>(nb)));
    d_i32 = G.d_i32;
    if (total > 0) {
      V_TRY(ctx, cudaMemcpyAsync(G.d_pts, pts.data(), sizeof(double4) * total, cudaMemcpyHostToDevice, st));
      V_TRY(ctx, cudaMemcpyAsync(G.d_matches, mm.data(), sizeof(uint2) * total, cudaMemcpyHostToDevice, st));
    }
    V_TRY(ctx, cudaMemcpyAsync(G.d_cams, cams.data(), sizeof(DevCamera) * 2 * nb, cudaMemcpyHostToDevice, st));
    V_TRY(ctx, cudaMemsetAsync(d_i32, 0, sizeof(int32_t) * 11 * nb, st));
    V_TRY(ctx, cudaMemcpyAsync(d_i32, pairs.data(), sizeof(int32_t) * 2 * nb, cudaMemcpyHostToDevice, st));
    V_TRY(ctx, cudaMemcpyAsync(d_i32 + 2 * nb, cnt.data(), sizeof(int32_t) * nb, cudaMemcpyHostToDevice, st));
    V_TRY(ctx, cudaMemcpyAsync(G.d_off, off.data(), sizeof(int64_t) * nb, cudaMemcpyHostToDevice, st));
    V_TRY(ctx, cudaMemsetAsync(G.d_models, 0, sizeof(double) * 27 * nb, st));
    VerifyParams P = VerifyParams{};
    P.pairs = d_i32;
    P.pair_cnt = d_i32 + 2 * nb;
    P.sup_cnt = d_i32 + 3 * nb;
    P.success = d_i32 + 6 * nb;
    P.config = d_i32 + 9 * nb;
    P.inl_cnt = d_i32 + 10 * nb;
    P.pair_off = G.d_off;
    P.pts = G.d_pts;
    P.matches = G.d_matches;
    P.cams = G.d_cams;
    P.mask = G.d_mask;
    P.arena_cap = cap;
    P.models = G.d_models;
    P.inliers = G.d_inliers;
    P.opt = *opts;
    P.seed = ctx->seed;
    P.single_kind = -1;
    P.counters = verify_counters(ctx);
      P.e_scratch = G.d_e_scratch;
    P.lo_eig_thread = lo_eig_thread_mode();
    const double4* pts_E = nullptr;
    if (int rc = undistort_for_E(ctx, G, P, full_cams.data(), 2 * nb, nb, cap, st, &pts_E)) return rc;
    V_TRY(ctx, launch_ransac(P, nb, st, nullptr, pts_E));
    b2m_decide_kernel<<<nb, 256, 0, st>>>(P);
    V_TRY(ctx, cudaGetLastError());
    ctx->stats.kernel_launches += 4;
    if (opts->compute_relative_pose)
      if (int rc = launch_pose_standalone(ctx, G, P, nb, cap, raw1, raw2, raw1_off, raw2_off, full_cams.data(), 2 * nb, st))
        return rc;
    std::vector<double> h_pose(static_cast<size_t>(8) * nb, 0.0);
    std::vector<int32_t> h_pose_valid(nb, 0);
    if (G.d_pose) {
      V_TRY(ctx, cudaMemcpyAsync(h_pose.data(), G.d_pose, sizeof(double) * 8 * nb, cudaMemcpyDeviceToHost, st));
      V_TRY(ctx, cudaMemcpyAsync(h_pose_valid.data(), G.d_pose_valid, sizeof(int32_t) * nb, cudaMemcpyDeviceToHost, st));
    }
    std::vector<int32_t> h_i32(static_cast<size_t>(11) * nb);
    std::vector<double> h_models(static_cast<size_t>(27) * nb);
    std::vector<uint2> h_inl(static_cast<size_t>(cap));
    V_TRY(ctx, cudaMemcpyAsync(h_i32.data(), d_i32, sizeof(int32_t) * 11 * nb, cudaMemcpyDeviceToHost, st));
    V_TRY(ctx, cudaMemcpyAsync(h_models.data(), G.d_models, sizeof(double) * 27 * nb, cudaMemcpyDeviceToHost, st));
    if (total > 0 && inlier_matches)
      V_TRY(ctx, cudaMemcpyAsync(h_inl.data(), G.d_inliers, sizeof(uint2) * total, cudaMemcpyDeviceToHost, st));
    V_TRY(ctx, cudaStreamSynchronize(st));
    for (int k = 0; k < nb; ++k) {
      b2m_tvg_result& r = out[k0 + k];
      memset(&r, 0, sizeof(r));
      r.struct_size = sizeof(r);
      r.config = h_i32[9 * nb + k];
      r.n_inliers = h_i32[10 * nb + k];
      r.nE = h_i32[3 * nb + 3 * k];
      r.nF = h_i32[3 * nb + 3 * k + 1];
      r.nH = h_i32[3 * nb + 3 * k + 2];
      memcpy(r.E, h_models.data() + 27 * k, sizeof(double) * 9);
      memcpy(r.F, h_models.data() + 27 * k + 9, sizeof(double) * 9);
      memcpy(r.H, h_models.data() + 27 * k + 18, sizeof(double) * 9);
      fill_pose(&r, h_pose.data(), h_pose_valid.data(), k);
      if (r.n_inliers > 0 && inlier_matches && inlier_matches[k0 + k])
        memcpy(inlier_matches[k0 + k], h_inl.data() + off[k], sizeof(uint2) * r.n_inliers);
    }
  }
  return B2M_OK;
}

int b2m_ransac_model(b2m_ctx* ctx, int32_t kind, const double* points1, const double* points2, int64_t m,
                     const b2m_ransac_opts* opts, double* out_model, uint8_t* inlier_mask, int64_t* num_inliers,
                     int32_t* success) {
  if (!ctx) return B2M_EINVAL;
  auto bad = [&](const char* msg) {
    ctx->err = msg;
    return B2M_EINVAL;
  };
  if (kind < 0 || kind > 2) return bad("[verify.cu] Check Failed: kind in {0 (E), 1 (F), 2 (H)}");
  if (!opts || !out_model || !num_inliers || !success) return bad("[verify.cu] Check Failed: outputs != NULL");
  if (m < 0 || (m > 0 && (!points1 || !points2))) return bad("[verify.cu] Check Failed: points");
  cudaSetDevice(ctx->device);
  std::vector<double4> pts(m);
  std::vector<uint2> mm(m);
  for (int64_t i = 0; i < m; ++i) {
    pts[i] = make_double4(points1[2 * i], points1[2 * i + 1], points2[2 * i], points2[2 * i + 1]);
    mm[i] = make_uint2(static_cast<uint32_t>(i), static_cast<uint32_t>(i));
  }
  b2m_tvg_opts t;
  b2m_tvg_opts_default(&t);
  t.ransac = *opts;
  DevCamera cams[2];
  memset(cams, 0, sizeof(cams));
  cams[0].fx = cams[0].fy = cams[0].mean_f = 1.0;
  cams[1] = cams[0];
  Single G;
  VerifyParams P;
  if (int rc = run_single(ctx, pts, mm, cams, t, kind, G, P)) return rc;
  int32_t i32[16];
  double models[27];
  V_TRY(ctx, cudaMemcpyAsync(i32, G.d_i32, sizeof(i32), cudaMemcpyDeviceToHost, ctx->stream));
  V_TRY(ctx, cudaMemcpyAsync(models, G.d_models, sizeof(models), cudaMemcpyDeviceToHost, ctx->stream));
  if (m > 0 && inlier_mask)
    V_TRY(ctx, cudaMemcpyAsync(inlier_mask, G.d_mask + static_cast<int64_t>(kind) * P.arena_cap, m,
                               cudaMemcpyDeviceToHost, ctx->stream));
  V_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  *num_inliers = i32[3 + kind];
  *success = i32[6 + kind];
  memcpy(out_model, models + 9 * kind, sizeof(double) * 9);
  return B2M_OK;
}

// EstimateTwoViewGeometryPose on a caller-provided geometry (R:estimators/two_view_geometry.h:153-158): the pose
// kernel alone.  geometry->config / E / H are inputs; config (PLANAR_OR_PANORAMIC -> PLANAR / PANORAMIC), qvec,
// tvec, tri_angle and pose_valid are outputs.  pose_valid = 0 mirrors upstream's `false` return.
int b2m_estimate_two_view_geometry_pose(b2m_ctx* ctx, const b2m_camera* cam1, const double* points1, int64_t n1,
                                        const b2m_camera* cam2, const double* points2, int64_t n2,
                                        const uint32_t* inlier_matches, int64_t n_inliers, b2m_tvg_result* geometry) {
  if (!ctx) return B2M_EINVAL;
  auto bad = [&](const char* msg) {
    ctx->err = msg;
    return B2M_EINVAL;
  };
  if (!cam1 || !cam2 || !geometry) return bad("[verify.cu] Check Failed: cameras and geometry != NULL");
  if (const char* why = camera_problem(*cam1)) return bad(why);
  if (const char* why = camera_problem(*cam2)) return bad(why);
  if (n1 < 0 || n2 < 0 || (n1 > 0 && !points1) || (n2 > 0 && !points2)) return bad("[verify.cu] Check Failed: points");
  if (n_inliers < 0 || n_inliers > INT32_MAX || (n_inliers > 0 && !inlier_matches))
    return bad("[verify.cu] Check Failed: inlier_matches");
  for (int64_t i = 0; i < n_inliers; ++i)
    if (inlier_matches[2 * i] >= n1 || inlier_matches[2 * i + 1] >= n2)
      return bad("[verify.cu] Check Failed: match index < number of points");
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  Single G;
  const int64_t cap = std::max<int64_t>(n_inliers, 1);
  const DevCamera cams[2] = {to_dev(*cam1), to_dev(*cam2)};
  const int32_t i32[4] = {0, 1, static_cast<int32_t>(n_inliers), geometry->config};  // pairs[2], inl_cnt, config
  const int64_t off0 = 0;
  double models[27];
  memset(models, 0, sizeof(models));
  memcpy(models, geometry->E, sizeof(double) * 9);
  memcpy(models + 18, geometry->H, sizeof(double) * 9);
  V_TRY(ctx, cudaMalloc(&G.d_inliers, sizeof(uint2) * cap));
  V_TRY(ctx, cudaMalloc(&G.d_cams, sizeof(DevCamera) * 2));
  V_TRY(ctx, cudaMalloc(&G.d_i32, sizeof(i32)));
  V_TRY(ctx, cudaMalloc(&G.d_off, sizeof(int64_t)));
  V_TRY(ctx, cudaMalloc(&G.d_models, sizeof(models)));
  if (n_inliers > 0)
    V_TRY(ctx, cudaMemcpy(G.d_inliers, inlier_matches, sizeof(uint2) * n_inliers, cudaMemcpyHostToDevice));
  V_TRY(ctx, cudaMemcpy(G.d_cams, cams, sizeof(cams), cudaMemcpyHostToDevice));
  V_TRY(ctx, cudaMemcpy(G.d_i32, i32, sizeof(i32), cudaMemcpyHostToDevice));
  V_TRY(ctx, cudaMemcpy(G.d_off, &off0, sizeof(int64_t), cudaMemcpyHostToDevice));
  V_TRY(ctx, cudaMemcpy(G.d_models, models, sizeof(models), cudaMemcpyHostToDevice));
  VerifyParams P = VerifyParams{};
  P.pairs = G.d_i32;
  P.inl_cnt = G.d_i32 + 2;
  P.config = G.d_i32 + 3;
  P.pair_off = G.d_off;
  P.inliers = G.d_inliers;
  P.models = G.d_models;
  P.cams = G.d_cams;
  const std::vector<double> p1(points1, points1 + 2 * n1), p2(points2, points2 + 2 * n2);
  const std::vector<int64_t> zero(1, 0);
  const b2m_camera* full_cams[2] = {cam1, cam2};
  if (int rc = launch_pose_standalone(ctx, G, P, 1, cap, p1, p2, zero, zero, full_cams, 2, st)) return rc;
  double h_pose[8];
  int32_t h_valid = 0, h_i32[4];
  V_TRY(ctx, cudaMemcpyAsync(h_pose, G.d_pose, sizeof(h_pose), cudaMemcpyDeviceToHost, st));
  V_TRY(ctx, cudaMemcpyAsync(&h_valid, G.d_pose_valid, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  V_TRY(ctx, cudaMemcpyAsync(h_i32, G.d_i32, sizeof(h_i32), cudaMemcpyDeviceToHost, st));
  V_TRY(ctx, cudaStreamSynchronize(st));
  geometry->qvec[0] = 1.0;
  geometry->qvec[1] = geometry->qvec[2] = geometry->qvec[3] = 0.0;
  geometry->tvec[0] = geometry->tvec[1] = geometry->tvec[2] = 0.0;
  geometry->tri_angle = 0.0;
  geometry->pose_valid = 0;
  if (h_valid) {
    geometry->config = h_i32[3];
    memcpy(geometry->qvec, h_pose, sizeof(double) * 4);
    memcpy(geometry->tvec, h_pose + 4, sizeof(double) * 3);
    geometry->tri_angle = h_pose[7];
    geometry->pose_valid = 1;
  }
  return B2M_OK;
}

int b2m_debug_five_point(b2m_ctx* ctx, const double* nullspaces, int64_t n, double* models, int32_t* n_models) {
  if (!ctx) return B2M_EINVAL;
  if (n < 0 || (n > 0 && (!nullspaces || !models || !n_models))) {
    ctx->err = "[verify.cu] Check Failed: nullspaces, models, n_models != NULL";
    return B2M_EINVAL;
  }
  if (n == 0) return B2M_OK;
  cudaSetDevice(ctx->device);
  double *d_n = nullptr, *d_m = nullptr;
  int32_t* d_c = nullptr;
  auto cleanup = [&]() {
    cudaFree(d_n); cudaFree(d_m); cudaFree(d_c);
  };
  if (cudaMalloc(&d_n, sizeof(double) * 36 * n) != cudaSuccess || cudaMalloc(&d_m, sizeof(double) * 90 * n) != cudaSuccess ||
      cudaMalloc(&d_c, sizeof(int32_t) * n) != cudaSuccess) {
    cleanup();
    ctx->err = "[verify.cu] cudaMalloc failed";
    return B2M_ENOMEM;
  }
  cudaMemcpyAsync(d_n, nullspaces, sizeof(double) * 36 * n, cudaMemcpyHostToDevice, ctx->stream);
  cudaMemsetAsync(d_m, 0, sizeof(double) * 90 * n, ctx->stream);
  b2m_five_point_kernel<<<static_cast<unsigned>((n + 3) / 4), 128, 0, ctx->stream>>>(d_n, n, d_m, d_c);
  ctx->stats.kernel_launches += 1;
  cudaMemcpyAsync(models, d_m, sizeof(double) * 90 * n, cudaMemcpyDeviceToHost, ctx->stream);
  cudaMemcpyAsync(n_models, d_c, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, ctx->stream);
  int rc = B2M_OK;
  if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) {
    ctx->err = std::string("[verify.cu] CUDA error: ") + cudaGetErrorString(cudaGetLastError());
    rc = B2M_ECUDA;
  }
  cleanup();
  return rc;
}

int b2m_cam_from_img(b2m_ctx* ctx, const b2m_camera* camera, const double* points, int64_t n, double* out) {
  if (!ctx) return B2M_EINVAL;
  auto bad = [&](const char* msg) {
    ctx->err = msg;
    return B2M_EINVAL;
  };
  if (!camera || n < 0 || (n > 0 && (!points || !out))) return bad("[verify.cu] Check Failed: camera, points, out != NULL");
  if (const char* why = camera_problem(*camera)) return bad(why);
  if (n == 0) return B2M_OK;
  cudaSetDevice(ctx->device);
  const DevDistortion hd = to_dist(*camera);
  DevDistortion* dc = nullptr;
  double *dp = nullptr, *dout = nullptr;
  auto cleanup = [&]() {
    cudaFree(dc); cudaFree(dp); cudaFree(dout);
  };
  if (cudaMalloc(&dc, sizeof(DevDistortion)) != cudaSuccess || cudaMalloc(&dp, sizeof(double) * 2 * n) != cudaSuccess ||
      cudaMalloc(&dout, sizeof(double) * 2 * n) != cudaSuccess) {
    cleanup();
    ctx->err = "[verify.cu] cudaMalloc failed";
    return B2M_ENOMEM;
  }
  cudaMemcpyAsync(dc, &hd, sizeof(hd), cudaMemcpyHostToDevice, ctx->stream);
  cudaMemcpyAsync(dp, points, sizeof(double) * 2 * n, cudaMemcpyHostToDevice, ctx->stream);
  b2m_cam_from_img_kernel<<<static_cast<unsigned>((n + 127) / 128), 128, 0, ctx->stream>>>(dc, dp, n, dout);
  ctx->stats.kernel_launches += 1;
  cudaMemcpyAsync(out, dout, sizeof(double) * 2 * n, cudaMemcpyDeviceToHost, ctx->stream);
  int rc = B2M_OK;
  if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) {
    ctx->err = std::string("[verify.cu] CUDA error: ") + cudaGetErrorString(cudaGetLastError());
    rc = B2M_ECUDA;
  }
  cleanup();
  return rc;
}

int b2m_squared_sampson_error(b2m_ctx* ctx, const double* points1, const double* points2, int64_t m, const double* E,
                              double* out_residuals) {
  if (!ctx) return B2M_EINVAL;
  if (m < 0 || (m > 0 && (!points1 || !points2 || !out_residuals)) || !E) {
    ctx->err = "[verify.cu] Check Failed: points, E, out != NULL";
    return B2M_EINVAL;
  }
  if (m == 0) return B2M_OK;
  cudaSetDevice(ctx->device);
  double *d1 = nullptr, *d2 = nullptr, *dE = nullptr, *dout = nullptr;
  int rc = B2M_OK;
  auto cleanup = [&]() {
    cudaFree(d1); cudaFree(d2); cudaFree(dE); cudaFree(dout);
  };
  if (cudaMalloc(&d1, sizeof(double) * 2 * m) != cudaSuccess || cudaMalloc(&d2, sizeof(double) * 2 * m) != cudaSuccess ||
      cudaMalloc(&dE, sizeof(double) * 9) != cudaSuccess || cudaMalloc(&dout, sizeof(double) * m) != cudaSuccess) {
    cleanup();
    ctx->err = "[verify.cu] cudaMalloc failed";
    return B2M_ENOMEM;
  }
  cudaMemcpyAsync(d1, points1, sizeof(double) * 2 * m, cudaMemcpyHostToDevice, ctx->stream);
  cudaMemcpyAsync(d2, points2, sizeof(double) * 2 * m, cudaMemcpyHostToDevice, ctx->stream);
  cudaMemcpyAsync(dE, E, sizeof(double) * 9, cudaMemcpyHostToDevice, ctx->stream);
  b2m_sampson_kernel<<<static_cast<unsigned>((m + 255) / 256), 256, 0, ctx->stream>>>(d1, d2, m, dE, dout);
  ctx->stats.kernel_launches += 1;
  cudaMemcpyAsync(out_residuals, dout, sizeof(double) * m, cudaMemcpyDeviceToHost, ctx->stream);
  if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) {
    ctx->err = std::string("[verify.cu] CUDA error: ") + cudaGetErrorString(cudaGetLastError());
    rc = B2M_ECUDA;
  }
  cleanup();
  return rc;
}

}  // extern "C"
