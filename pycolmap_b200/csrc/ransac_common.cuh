// ransac_common.cuh -- the LO-RANSAC round shared by the two-view verifier (verify.cu, K2/K3) and the absolute pose
// estimator (abs_pose.cu, K4).  One CTA of kRansacThreads threads runs one problem.  Each kernel keeps its own outer
// loop (minimal solver, local optimisation, dynamic trial bound, output) and calls these pieces between its steps:
//   round_size      how many trials the next round draws (one per thread at most),
//   draw_sample     a thread's minimal sample, counter-based so that results do not depend on batching or sharding,
//   score_round     every model of the round counted over all points, and the round's winner,
//   exact_support   the fp64 count and residual sum of a model over all points.
// The trial cap and the dynamic bound (ComputeNumTrials, U:optim/ransac.h) are geom::ransac_trial_cap and
// geom::compute_num_trials.
//
// score_round and exact_support see a kernel's points and models through a model policy (EpipolarModel in verify.cu,
// ReprojModel in abs_pose.cu):
//   kD                    doubles per model (at most 12: the fp32 copy is padded to 12 for three 16-byte loads)
//   Pt, load_f32(i, live) point i in fp32 registers; live = false for a slot past the end, which gets a sentinel point
//   test(Mf, pt, thr_f)   the division-free fp32 test of residual <= thr: classify_f32's outcome
//   residual(M, i)        the fp64 residual of point i under M
#pragma once
#include <cstdint>

namespace b2m {

constexpr int kRansacThreads = 128;  // threads of a RANSAC CTA: at most this many trials per round
constexpr int kChunkModels = 256;    // models scored per pass of the fp32 scoring loop

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

// Outcome of `residual <= thr` evaluated as lhs <= rhs = thr * denominator in fp32: bit 0 = clearly an inlier,
// bit 1 = borderline (within 1 % of the threshold, or not finite) -- the caller re-evaluates those in fp64, so a
// decision equals the fp64 one as long as the fp32 rounding of lhs and rhs stays inside the 1 % band (see the
// limits at verify.cu inlier_f32).  STRICT comparisons: lhs == rhs == 0 (both underflowed) or == inf (both overflowed) is
// neither clearly in nor clearly out, like any NaN.
__device__ __forceinline__ int classify_f32(float lhs, float rhs) {
  const int in = lhs < 0.99f * rhs ? 1 : 0;
  const int out = lhs > 1.01f * rhs ? 1 : 0;
  return in | ((in | out) ^ 1) << 1;
}

// Trials of the next round: up to min_num_trials first, then past it the sequential reference stops at the FIRST
// trial >= dyn_max, so a round never needs more hypotheses than are missing to that bound (a better model found among
// them only lowers it).
__device__ __forceinline__ int round_size(int trials, int max_trials, int min_num_trials, double dyn_max) {
  int nb = min(kRansacThreads, max_trials - trials);
  if (trials < min_num_trials) nb = min(nb, min_num_trials - trials);
  else if (dyn_max - trials < nb) nb = max(1, static_cast<int>(ceil(dyn_max - trials)));
  return nb;
}

// K distinct indices in [0, n) for `trial`, from the problem's key (a duplicate is redrawn, up to 64 times).
template <int K>
__device__ __forceinline__ void draw_sample(uint64_t key, int trial, int n, int* idx) {
  const uint64_t tkey = splitmix64(key + static_cast<uint64_t>(trial) * 0x100000001B3ull);
  for (int j = 0; j < K; ++j) {
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
}

// Shared memory of score_round, embedded in each kernel's own.  Outside score_round chunk_d and scan are free:
// exact_support keeps its per-warp partials there, and verify.cu uses chunk_d as solver scratch.
template <int D>
struct RoundShared {
  double chunk_d[kChunkModels][D];  // models of the current chunk (fp64, for borderline rechecks)
  float chunk_f[kChunkModels][12];  // same, fp32, padded to three 16-byte loads
  int chunk_cnt[kChunkModels];      // inlier counts of the chunk's models
  int scan[kRansacThreads];         // models per thread
  int cnt_arr[kRansacThreads];      // each thread's best count
  int round_max;                    // largest (partial) count among the models of the round, for the exact pruning
  int winner;
};

struct RoundResult {
  int winner;    // thread whose model beat the best so far, -1 if none did (uniform)
  int model;     // index of this thread's best model
  int n_models;  // models scored in the round (uniform)
};

// Hypothesis scoring of one block of points: every thread keeps PPT points (fp32) in registers and sweeps the chunk's
// models: division-free fp32 test, fp64 only for the borderline points of a (thread, model).  Inlier counts go to
// rs.chunk_cnt.
template <int PPT, class Model>
__device__ __forceinline__ void score_block(RoundShared<Model::kD>& rs, const Model& model, int n, int pb, int n_chunk,
                                            double thr, float thr_f, int need) {
  const int tid = threadIdx.x;
  typename Model::Pt p[PPT];
  int live[PPT];  // 1 for a real point, 0 for a slot past the end: such a slot never counts and never forces a
                  // recheck, whatever the model (its sentinel point is an outlier for every sane model, but the fp32
                  // operands can both overflow).  score_round gives a block more than (PPT - 1) * kRansacThreads
                  // points, so only the last slot can be past the end.
#pragma unroll
  for (int q = 0; q < PPT; ++q) {
    const int i = pb + q * kRansacThreads + tid;
    live[q] = q < PPT - 1 || i < n ? 1 : 0;
    p[q] = model.load_f32(i, live[q]);
  }
  for (int m = 0; m < n_chunk; ++m) {
    // exact pruning: a model that cannot reach `need + (points not yet scored)` even if every remaining point were
    // an inlier can neither beat the best model so far nor the leader of this round (uniform across the CTA)
    if (rs.chunk_cnt[m] < need) continue;
    float Mf[12];
    const float4* mp = reinterpret_cast<const float4*>(rs.chunk_f[m]);
    const float4 m0 = mp[0], m1 = mp[1], m2 = mp[2];
    Mf[0] = m0.x; Mf[1] = m0.y; Mf[2] = m0.z; Mf[3] = m0.w;
    Mf[4] = m1.x; Mf[5] = m1.y; Mf[6] = m1.z; Mf[7] = m1.w;
    Mf[8] = m2.x; Mf[9] = m2.y; Mf[10] = m2.z; Mf[11] = m2.w;
    int c = 0, flags = 0;
#pragma unroll
    for (int q = 0; q < PPT; ++q) {
      const int f = model.test(Mf, p[q], thr_f);
      c += f & live[q];
      flags |= f & (live[q] << 1);
    }
    if (flags & 2) {  // rare: a borderline point -> redo this thread's points of this model in fp64
      c = 0;
      for (int q = 0; q < PPT; ++q) {
        const int i = pb + q * kRansacThreads + tid;
        if (i < n) c += model.residual(rs.chunk_d[m], i) <= thr ? 1 : 0;
      }
    }
    if (c) atomicAdd(&rs.chunk_cnt[m], c);  // most hypotheses have (almost) no inliers: cheaper than a warp reduce
  }
}

// Scores the round's models over all n points.  Thread t holds nm models of trial (first trial of the round + t) in
// mdl ([nm][kD]); the first nb threads drew a trial.  Models go to shared memory in chunks of kChunkModels and are
// swept in blocks of 4 * kRansacThreads points.  Only inlier COUNTS are formed: the winner is the thread whose best
// model has strictly more inliers than best_cnt and than every other thread, the earlier trial on ties (the
// residual-sum tie-break of U:optim/support_measurement.h applies from the LO stage on).
template <class Model>
__device__ RoundResult score_round(RoundShared<Model::kD>& rs, const Model& model, const double* mdl, int nm, int nb,
                                   int n, double thr, int best_cnt) {
  constexpr int D = Model::kD;
  const int tid = threadIdx.x;
  int my_cnt = -1, my_m = 0;
  rs.scan[tid] = nm;
  if (tid == 0) rs.round_max = 0;
  __syncthreads();
  int my_base = 0, total_models = 0;
  for (int t = 0; t < kRansacThreads; ++t) {
    const int v = rs.scan[t];
    if (t < tid) my_base += v;
    total_models += v;
  }
  const float thr_f = static_cast<float>(thr);
  for (int chunk0 = 0; chunk0 < total_models; chunk0 += kChunkModels) {
    const int n_chunk = min(kChunkModels, total_models - chunk0);
    for (int m = 0; m < nm; ++m) {
      const int g = my_base + m - chunk0;
      if (g >= 0 && g < kChunkModels)
#pragma unroll
        for (int k = 0; k < D; ++k) {
          rs.chunk_d[g][k] = mdl[m * D + k];
          rs.chunk_f[g][k] = static_cast<float>(mdl[m * D + k]);
        }
    }
    for (int m = tid; m < kChunkModels; m += kRansacThreads) rs.chunk_cnt[m] = 0;
    __syncthreads();
    // Between blocks the inlier counts so far are complete (barrier), so a model whose count plus ALL remaining points
    // stays below the best of the earlier rounds or below what the leader of this round already has is dropped for
    // the rest of the sweep -- exact: it could not have won, nor tied.
    constexpr int kBlock = 4 * kRansacThreads;
    for (int pb = 0; pb < n; pb += kBlock) {
      const int rem = n - pb;
      int need = 0;
      if (pb > 0) {
        __syncthreads();  // chunk_cnt of the previous blocks is complete
        for (int m = tid; m < n_chunk; m += kRansacThreads) atomicMax(&rs.round_max, rs.chunk_cnt[m]);
        __syncthreads();
        need = max(best_cnt + 1, rs.round_max) - rem;
      }
      // the last block takes as few point slots per thread as cover it (a slot past the end costs a full test)
      if (rem > 3 * kRansacThreads) score_block<4>(rs, model, n, pb, n_chunk, thr, thr_f, need);
      else if (rem > 2 * kRansacThreads) score_block<3>(rs, model, n, pb, n_chunk, thr, thr_f, need);
      else if (rem > kRansacThreads) score_block<2>(rs, model, n, pb, n_chunk, thr, thr_f, need);
      else score_block<1>(rs, model, n, pb, n_chunk, thr, thr_f, need);
    }
    __syncthreads();
    for (int m = 0; m < nm; ++m) {
      const int g = my_base + m - chunk0;
      if (g >= 0 && g < kChunkModels && rs.chunk_cnt[g] > my_cnt) {
        my_cnt = rs.chunk_cnt[g];
        my_m = m;
      }
    }
    __syncthreads();
  }
  rs.cnt_arr[tid] = my_cnt;
  __syncthreads();
  if (tid == 0) {
    int w = -1, bc = best_cnt;
    for (int t = 0; t < nb; ++t)
      if (rs.cnt_arr[t] > bc) {
        bc = rs.cnt_arr[t];
        w = t;
      }
    rs.winner = w;
  }
  __syncthreads();
  return {rs.winner, my_m, total_models};
}

// Exact fp64 support (count, residual sum) of M over all n points, CTA-wide; every thread gets the totals.
template <class Model>
__device__ void exact_support(RoundShared<Model::kD>& rs, const Model& model, const double* M, int n, double thr,
                              int& cnt, double& sum) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int cl = 0;
  double sl = 0.0;
  for (int i = tid; i < n; i += kRansacThreads) {
    const double r = model.residual(M, i);
    if (r <= thr) {
      ++cl;
      sl += r;
    }
  }
  cl = __reduce_add_sync(0xffffffffu, cl);
  sl = warp_sum_d(sl);
  __syncthreads();
  if (lane == 0) {
    rs.scan[warp] = cl;
    rs.chunk_d[0][warp] = sl;
  }
  __syncthreads();
  cnt = rs.scan[0] + rs.scan[1] + rs.scan[2] + rs.scan[3];
  sum = rs.chunk_d[0][0] + rs.chunk_d[0][1] + rs.chunk_d[0][2] + rs.chunk_d[0][3];
  __syncthreads();
}

}  // namespace b2m
