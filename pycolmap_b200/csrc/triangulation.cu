// triangulation.cu -- batched robust multi-view triangulation behind b2m_estimate_triangulation_batch.
//
// Semantics: U:estimators/triangulation.cc EstimateTriangulation (LORANSAC with TriangulationEstimator for both the
// minimal and the local estimator, InlierSupportMeasurer, CombinationSampler, ANGULAR_ERROR residual), reached from
// R:pycolmap/estimators/triangulation.h:17-77; SURVEY.md section 8(a) rows T1-T5.  The specification is
// oracle/triangulation.py.
//
// Kernel b2m_tri_ransac_kernel: one warp per track, tracks of a chunk visited longest first.
//   - Trials come in rounds of 32: lane t takes trial 32 r + t, unranks it into the t-th lexicographic pair (i, j),
//     i < j (CombinationSampler), solves the 4 x 4 DLT by one-sided Jacobi on A itself (not A^T A, which squares the
//     condition number of far, small-baseline points), and runs the cheirality and angle tests.
//   - Every lane then scores its own hypothesis over the track's observations.  Observations are staged in shared
//     memory in tiles of kTile (normalised ray + projection matrix); a track longer than one tile is scored tile by
//     tile, so shared memory does not bound the track length.
//   - The warp walks the 32 lanes in trial order and applies exactly LORANSAC::Estimate's sequential logic: best
//     support (more inliers, then smaller residual sum), the up-to-10 LO rounds on every new best with more than two
//     inliers (warp-cooperative: residuals one lane per observation, the 10 distinct entries of sum term^T term
//     reduced over the warp, a 4 x 4 symmetric Jacobi eigensolve, cheirality and the any-pair angle test on the
//     compacted inliers, one lane per pair with a ballot), the dynamic trial bound, and the abort test after each
//     model.  Lanes after the aborting trial are discarded, so the decisions are those of the sequential loop.
// fp64 throughout, like upstream.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <vector>

#include "geom.h"
#include "internal.h"
#include "ransac_common.cuh"

namespace b2m {
namespace {

constexpr int kWarps = 4;   // tracks per CTA
constexpr int kTile = 64;   // observations staged per warp
constexpr int kObsStride = 16;  // doubles per staged observation: ray (3), P (12), pad
constexpr double kDblEps = 2.220446049250313e-16;

struct TriParams {
  const double* pts;       // [M x 2] normalised points of the chunk
  const int32_t* img;      // [M] image index per observation
  const int64_t* off;      // [nb + 1] observation offsets of the chunk's tracks
  const int32_t* order;    // [nb] track visiting order (longest first)
  const double* cams;      // [n_images x 12] cam_from_world, row-major 3 x 4
  const double* centers;   // [n_images x 3] projection centres -R^T t
  int32_t nb;
  double max_residual;     // max_error^2
  double min_tri_angle;
  double confidence, multiplier;
  double max_trials;       // min(max_num_trials, trials at min_inlier_ratio); clipped per track at C(n, 2)
  double min_num_trials;
  double* xyz;             // [nb x 3], NaN on failure
  int32_t* num_inliers;    // [nb]
  uint8_t* success;        // [nb]
  uint8_t* mask;           // [M]
  int32_t* scratch;        // [M]: compacted inlier positions of the LO rounds
  unsigned long long* counters;  // [2]: models scored, residual evaluations
};

// normalize((u, v, 1)) like Eigen's normalized(): v / sqrt(squaredNorm)
__device__ __forceinline__ void ray_of(double u, double v, double* r) {
  const double nrm = sqrt(u * u + v * v + 1.0);
  r[0] = u / nrm;
  r[1] = v / nrm;
  r[2] = 1.0 / nrm;
}

// CalculateNormalizedAngularError squared: acos(r . normalize(P X~))^2; NaN (never an inlier) when the cosine rounds
// above 1, like upstream (no clamp).  o: staged observation (ray, P).
__device__ __forceinline__ double ang_residual(const double* o, double x, double y, double z) {
  const double* P = o + 3;
  const double px = P[0] * x + P[1] * y + P[2] * z + P[3];
  const double py = P[4] * x + P[5] * y + P[6] * z + P[7];
  const double pz = P[8] * x + P[9] * y + P[10] * z + P[11];
  const double nrm = sqrt(px * px + py * py + pz * pz);
  const double c = o[0] * (px / nrm) + o[1] * (py / nrm) + o[2] * (pz / nrm);
  const double a = acos(c);
  return a * a;
}

// CalculateTriangulationAngle, clipped: min(theta, pi - theta), 0 when a ray has zero length.
__device__ __forceinline__ double tri_angle(const double* c1, const double* c2, double x, double y, double z) {
  const double bx = c1[0] - c2[0], by = c1[1] - c2[1], bz = c1[2] - c2[2];
  const double b2 = bx * bx + by * by + bz * bz;
  const double ax = x - c1[0], ay = y - c1[1], az = z - c1[2];
  const double dx = x - c2[0], dy = y - c2[1], dz = z - c2[2];
  const double r1 = ax * ax + ay * ay + az * az, r2 = dx * dx + dy * dy + dz * dz;
  const double den = 2.0 * sqrt(r1 * r2);
  if (!(den > 0.0)) return 0.0;
  const double ang = fabs(acos(fmin(fmax((r1 + r2 - b2) / den, -1.0), 1.0)));
  return fmin(ang, 3.141592653589793 - ang);
}

__device__ __forceinline__ double depth_of(const double* P, double x, double y, double z) {
  return P[8] * x + P[9] * y + P[10] * z + P[11];
}

// Stage observations [t0, t0 + cnt) of the track starting at `base` into sm (cnt <= kTile).
__device__ __forceinline__ void stage(const TriParams& p, int64_t base, int t0, int cnt, double* sm, int lane) {
  for (int q = lane; q < cnt; q += 32) {
    const int64_t g = base + t0 + q;
    double* o = sm + q * kObsStride;
    ray_of(p.pts[2 * g], p.pts[2 * g + 1], o);
    const double* P = p.cams + 12 * static_cast<int64_t>(p.img[g]);
#pragma unroll
    for (int e = 0; e < 12; ++e) o[3 + e] = P[e];
  }
}

// Two-view hypothesis (TriangulationEstimator::Estimate with two observations): TriangulatePoint's 4 x 4 DLT,
// smallest right singular vector by one-sided (Hestenes) Jacobi on A, then HasPointPositiveDepth in both views and
// CalculateTriangulationAngle >= min_tri_angle.
__device__ bool two_view(const TriParams& p, int64_t base, int i, int j, double* X) {
  const int64_t gi = base + i, gj = base + j;
  const double* Pi = p.cams + 12 * static_cast<int64_t>(p.img[gi]);
  const double* Pj = p.cams + 12 * static_cast<int64_t>(p.img[gj]);
  const double ui = p.pts[2 * gi], vi = p.pts[2 * gi + 1], uj = p.pts[2 * gj], vj = p.pts[2 * gj + 1];
  double a[4][4], v[4][4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    a[0][c] = ui * Pi[8 + c] - Pi[c];
    a[1][c] = vi * Pi[8 + c] - Pi[4 + c];
    a[2][c] = uj * Pj[8 + c] - Pj[c];
    a[3][c] = vj * Pj[8 + c] - Pj[4 + c];
#pragma unroll
    for (int r = 0; r < 4; ++r) v[r][c] = (r == c) ? 1.0 : 0.0;
  }
  for (int sweep = 0; sweep < 20; ++sweep) {
    bool rotated = false;
#pragma unroll
    for (int pp = 0; pp < 3; ++pp) {
#pragma unroll
      for (int qq = pp + 1; qq < 4; ++qq) {
        double al = 0.0, be = 0.0, ga = 0.0;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          al += a[r][pp] * a[r][pp];
          be += a[r][qq] * a[r][qq];
          ga += a[r][pp] * a[r][qq];
        }
        if (!(fabs(ga) > 1e-15 * sqrt(al * be))) continue;
        rotated = true;
        const double zeta = (be - al) / (2.0 * ga);
        const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const double ap = a[r][pp], aq = a[r][qq];
          a[r][pp] = c * ap - s * aq;
          a[r][qq] = s * ap + c * aq;
          const double vp = v[r][pp], vq = v[r][qq];
          v[r][pp] = c * vp - s * vq;
          v[r][qq] = s * vp + c * vq;
        }
      }
    }
    if (!rotated) break;
  }
  double nmin = 0.0;
  int kmin = 0;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const double nc = a[0][c] * a[0][c] + a[1][c] * a[1][c] + a[2][c] * a[2][c] + a[3][c] * a[3][c];
    if (c == 0 || nc < nmin) {
      nmin = nc;
      kmin = c;
    }
  }
  double h[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    h[r] = v[r][0];
#pragma unroll
    for (int c = 1; c < 4; ++c)
      if (kmin == c) h[r] = v[r][c];
  }
  X[0] = h[0] / h[3];
  X[1] = h[1] / h[3];
  X[2] = h[2] / h[3];
  if (!(depth_of(Pi, X[0], X[1], X[2]) >= kDblEps) || !(depth_of(Pj, X[0], X[1], X[2]) >= kDblEps)) return false;
  const double ang = tri_angle(p.centers + 3 * static_cast<int64_t>(p.img[gi]), p.centers + 3 * static_cast<int64_t>(p.img[gj]),
                               X[0], X[1], X[2]);
  return ang >= p.min_tri_angle;
}

// Lexicographic pair number k of n: (i, j), i < j; row i starts at S(i) = i (2n - i - 1) / 2.
__device__ __forceinline__ void unrank_pair(int64_t k, int64_t n, int* i, int* j) {
  const double b = 2.0 * n - 1.0;
  int64_t r = static_cast<int64_t>(floor((b - sqrt(fmax(b * b - 8.0 * static_cast<double>(k), 0.0))) * 0.5));
  r = r < 0 ? 0 : (r > n - 2 ? n - 2 : r);
  auto S = [n](int64_t q) { return q * (2 * n - q - 1) / 2; };
  while (r > 0 && S(r) > k) --r;
  while (r + 1 < n - 1 && S(r + 1) <= k) ++r;
  *i = static_cast<int>(r);
  *j = static_cast<int>(k - S(r) + r + 1);
}

// Warp-wide sum whose result is the same bits on every lane (lane 0's butterfly result, broadcast).
__device__ __forceinline__ double warp_sum_bcast(double v) { return shfl_d(warp_sum_d(v), 0); }

// Support of model (x, y, z) over the track, one lane per observation: (count, residual sum) on every lane.
__device__ void score_warp(const TriParams& p, int64_t base, int n, bool all_staged, double* sm, int lane, double x,
                           double y, double z, int* cnt_out, double* sum_out) {
  int cnt = 0;
  double sum = 0.0;
  for (int t0 = 0; t0 < n; t0 += kTile) {
    const int m = min(kTile, n - t0);
    if (!all_staged) {
      __syncwarp();
      stage(p, base, t0, m, sm, lane);
      __syncwarp();
    }
    for (int q = lane; q < m; q += 32) {
      const double r = ang_residual(sm + q * kObsStride, x, y, z);
      if (r <= p.max_residual) {
        ++cnt;
        sum += r;
      }
    }
  }
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  *cnt_out = cnt;
  *sum_out = warp_sum_bcast(sum);
}

// One LO refit (TriangulationEstimator::Estimate with more than two observations) on the inliers of (x, y, z):
// TriangulateMultiViewPoint, cheirality in every inlier view, then some inlier pair with angle >= min_tri_angle.
// Returns whether a model was produced (then X holds it, the same bits on every lane).
__device__ bool lo_refit(const TriParams& p, int64_t base, int n, bool all_staged, double* sm, int lane, double x,
                         double y, double z, double* X) {
  double A[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};  // upper triangle of sum term^T term, row-major
  int m = 0;                                      // inliers compacted so far (warp-uniform)
  for (int t0 = 0; t0 < n; t0 += kTile) {
    const int mt = min(kTile, n - t0);
    if (!all_staged) {
      __syncwarp();
      stage(p, base, t0, mt, sm, lane);
      __syncwarp();
    }
    for (int q0 = 0; q0 < mt; q0 += 32) {
      const int q = q0 + lane;
      bool in = false;
      if (q < mt) {
        const double* o = sm + q * kObsStride;
        in = ang_residual(o, x, y, z) <= p.max_residual;
        if (in) {
          // term = P - r (r^T P): 3 x 4
          const double* P = o + 3;
          double rP[4];
#pragma unroll
          for (int c = 0; c < 4; ++c) rP[c] = o[0] * P[c] + o[1] * P[4 + c] + o[2] * P[8 + c];
          double tm[3][4];
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) tm[r][c] = P[4 * r + c] - o[r] * rP[c];
          int e = 0;
#pragma unroll
          for (int c1 = 0; c1 < 4; ++c1)
#pragma unroll
            for (int c2 = c1; c2 < 4; ++c2) A[e++] += tm[0][c1] * tm[0][c2] + tm[1][c1] * tm[1][c2] + tm[2][c1] * tm[2][c2];
        }
      }
      const unsigned bal = __ballot_sync(0xffffffffu, in);
      if (in) p.scratch[base + m + __popc(bal & ((1u << lane) - 1u))] = t0 + q;
      m += __popc(bal);
    }
  }
  double S[16], V[16], w[4];
  {
    double Ar[10];
#pragma unroll
    for (int e = 0; e < 10; ++e) Ar[e] = warp_sum_bcast(A[e]);
    int e = 0;
#pragma unroll
    for (int c1 = 0; c1 < 4; ++c1)
#pragma unroll
      for (int c2 = c1; c2 < 4; ++c2) {
        S[4 * c1 + c2] = Ar[e];
        S[4 * c2 + c1] = Ar[e];
        ++e;
      }
  }
  geom::jacobi_eig_sym<4>(S, V, w);
  int k = 0;
#pragma unroll
  for (int c = 1; c < 4; ++c)
    if (w[c] < w[k]) k = c;
  X[0] = V[0 * 4 + k] / V[3 * 4 + k];
  X[1] = V[1 * 4 + k] / V[3 * 4 + k];
  X[2] = V[2 * 4 + k] / V[3 * 4 + k];
  __syncwarp();  // scratch written by other lanes
  // cheirality in every inlier view
  bool bad = false;
  for (int q = lane; q < m; q += 32) {
    const int64_t g = base + p.scratch[base + q];
    bad |= !(depth_of(p.cams + 12 * static_cast<int64_t>(p.img[g]), X[0], X[1], X[2]) >= kDblEps);
  }
  if (__any_sync(0xffffffffu, bad)) return false;
  // some pair (a, b < a) of inliers with a large enough angle
  const int64_t np = static_cast<int64_t>(m) * (m - 1) / 2;
  for (int64_t q0 = 0; q0 < np; q0 += 32) {
    const int64_t q = q0 + lane;
    bool ok = false;
    if (q < np) {
      // pair number q in the order (1, 0), (2, 0), (2, 1), (3, 0), ...: row a starts at a (a - 1) / 2
      int64_t a = static_cast<int64_t>(floor((1.0 + sqrt(1.0 + 8.0 * static_cast<double>(q))) * 0.5));
      while (a * (a - 1) / 2 > q) --a;
      while ((a + 1) * a / 2 <= q) ++a;
      const int64_t b = q - a * (a - 1) / 2;
      const int32_t ia = p.img[base + p.scratch[base + a]], ib = p.img[base + p.scratch[base + b]];
      ok = tri_angle(p.centers + 3 * static_cast<int64_t>(ia), p.centers + 3 * static_cast<int64_t>(ib), X[0], X[1],
                     X[2]) >= p.min_tri_angle;
    }
    if (__any_sync(0xffffffffu, ok)) return true;
  }
  return false;
}

__global__ void __launch_bounds__(32 * kWarps) b2m_tri_ransac_kernel(const TriParams p) {
  __shared__ __align__(16) double smem[kWarps][kTile * kObsStride];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int slot = blockIdx.x * kWarps + warp;
  if (slot >= p.nb) return;
  double* sm = smem[warp];
  const int track = p.order[slot];
  const int64_t base = p.off[track];
  const int n = static_cast<int>(p.off[track + 1] - base);
  const bool all_staged = n <= kTile;
  if (all_staged) {
    stage(p, base, 0, n, sm, lane);
    __syncwarp();
  }
  const double c2 = 0.5 * static_cast<double>(n) * static_cast<double>(n - 1);
  const int64_t K = static_cast<int64_t>(fmin(p.max_trials, c2));
  double dyn_max = static_cast<double>(K);
  int best_cnt = 0;
  double best_sum = INFINITY;
  bool have = false;
  double bx = 0.0, by = 0.0, bz = 0.0;
  unsigned long long scored = 0;
  bool abort = false;
  for (int64_t r0 = 0; r0 < K && !abort; r0 += 32) {
    const int64_t t = r0 + lane;
    double X[3] = {0.0, 0.0, 0.0};
    bool valid = false;
    if (t < K) {
      int i, j;
      unrank_pair(t, n, &i, &j);
      valid = two_view(p, base, i, j, X);
    }
    // every lane scores its own hypothesis, tile by tile
    int cnt = 0;
    double sum = 0.0;
    for (int t0 = 0; t0 < n; t0 += kTile) {
      const int m = min(kTile, n - t0);
      if (!all_staged) {
        __syncwarp();
        stage(p, base, t0, m, sm, lane);
        __syncwarp();
      }
      if (valid)
        for (int q = 0; q < m; ++q) {
          const double r = ang_residual(sm + q * kObsStride, X[0], X[1], X[2]);
          if (r <= p.max_residual) {
            ++cnt;
            sum += r;
          }
        }
    }
    // the sequential walk over the round, in trial order
    const unsigned vmask = __ballot_sync(0xffffffffu, valid);
    for (int l = 0; l < 32; ++l) {
      const int64_t tl = r0 + l;
      if (tl >= K) break;
      if (!((vmask >> l) & 1u)) continue;  // no model: no abort test either
      const int cl = __shfl_sync(0xffffffffu, cnt, l);
      const double sl = shfl_d(sum, l);
      ++scored;
      if (cl > best_cnt || (cl == best_cnt && sl < best_sum)) {
        best_cnt = cl;
        best_sum = sl;
        bx = shfl_d(X[0], l);
        by = shfl_d(X[1], l);
        bz = shfl_d(X[2], l);
        have = true;
        if (cl > 2) {
          double cx = bx, cy = by, cz = bz;  // model whose inliers seed the next refit
          for (int it = 0; it < 10; ++it) {
            const int prev = best_cnt;
            double L[3];
            if (lo_refit(p, base, n, all_staged, sm, lane, cx, cy, cz, L)) {
              int lc;
              double ls;
              score_warp(p, base, n, all_staged, sm, lane, L[0], L[1], L[2], &lc, &ls);
              ++scored;
              if (lc > best_cnt || (lc == best_cnt && ls < best_sum)) {
                best_cnt = lc;
                best_sum = ls;
                bx = cx = L[0];
                by = cy = L[1];
                bz = cz = L[2];
              }
            }
            if (best_cnt <= prev) break;
          }
          if (!all_staged) __syncwarp();
        }
        dyn_max = geom::compute_num_trials(best_cnt, n, p.confidence, p.multiplier, 2);
      }
      if (static_cast<double>(tl) >= dyn_max && static_cast<double>(tl) >= p.min_num_trials) {
        abort = true;
        break;
      }
    }
  }
  // outputs: inlier mask of the best model (same residual as the scoring), xyz, counts
  const bool ok = have && best_cnt >= 2;
  for (int t0 = 0; t0 < n; t0 += kTile) {
    const int m = min(kTile, n - t0);
    if (!all_staged && ok) {
      __syncwarp();
      stage(p, base, t0, m, sm, lane);
      __syncwarp();
    }
    for (int q = lane; q < m; q += 32)
      p.mask[base + t0 + q] = ok ? (ang_residual(sm + q * kObsStride, bx, by, bz) <= p.max_residual) : 0;
  }
  if (lane == 0) {
    p.success[track] = ok ? 1 : 0;
    p.num_inliers[track] = best_cnt;
    p.xyz[3 * track] = ok ? bx : NAN;
    p.xyz[3 * track + 1] = ok ? by : NAN;
    p.xyz[3 * track + 2] = ok ? bz : NAN;
    if (p.counters) {
      atomicAdd(p.counters, scored);
      atomicAdd(p.counters + 1, scored * static_cast<unsigned long long>(n));
    }
  }
}

// Chunk limits: results do not depend on them (tracks are independent).
constexpr int64_t kChunkTracks = int64_t(1) << 15;
constexpr int64_t kChunkObs = int64_t(1) << 21;

}  // namespace

// Pinned staging and device buffers of one chunk of tracks, replaced together when a call needs more.
struct TriChunkBufs {
  int64_t cap_tracks = 0, cap_obs = 0;
  // pinned host staging
  PinnedArray<double> h_pts;
  PinnedArray<int32_t> h_img;
  PinnedArray<int64_t> h_off;
  PinnedArray<int32_t> h_order;
  PinnedArray<double> h_xyz;
  PinnedArray<int32_t> h_inl;
  PinnedArray<uint8_t> h_succ;
  PinnedArray<uint8_t> h_mask;
  // device
  DeviceArray<double> d_pts, d_xyz;
  DeviceArray<int32_t> d_img, d_order, d_inl, d_scratch;
  DeviceArray<int64_t> d_off;
  DeviceArray<uint8_t> d_succ, d_mask;
};

// The buffers of the triangulation path, kept by the context between calls and grown on demand.
struct TriState {
  TriChunkBufs chunk;
  DeviceArray<double> d_cams, d_centers;  // per image
};

void tri_release(b2m_ctx* ctx) {
  delete static_cast<TriState*>(ctx->tri_state);
  ctx->tri_state = nullptr;
}

namespace {

int ensure_state(b2m_ctx* ctx, int64_t tracks, int64_t obs, int64_t images, TriState** out) {
  if (!ctx->tri_state) ctx->tri_state = new TriState();
  TriState* s = static_cast<TriState*>(ctx->tri_state);
  *out = s;
  if (tracks > s->chunk.cap_tracks || obs > s->chunk.cap_obs) {
    const int rc = alloc_group(s->chunk, [&](TriChunkBufs& b) -> int {
      const int64_t T = std::max<int64_t>(tracks, 1), M = std::max<int64_t>(obs, 1);
      B2M_CUDA_TRY(ctx, b.h_pts.ensure(2 * M));
      B2M_CUDA_TRY(ctx, b.h_img.ensure(M));
      B2M_CUDA_TRY(ctx, b.h_off.ensure(T + 1));
      B2M_CUDA_TRY(ctx, b.h_order.ensure(T));
      B2M_CUDA_TRY(ctx, b.h_xyz.ensure(3 * T));
      B2M_CUDA_TRY(ctx, b.h_inl.ensure(T));
      B2M_CUDA_TRY(ctx, b.h_succ.ensure(T));
      B2M_CUDA_TRY(ctx, b.h_mask.ensure(M));
      B2M_CUDA_TRY(ctx, b.d_pts.ensure(2 * M));
      B2M_CUDA_TRY(ctx, b.d_img.ensure(M));
      B2M_CUDA_TRY(ctx, b.d_off.ensure(T + 1));
      B2M_CUDA_TRY(ctx, b.d_order.ensure(T));
      B2M_CUDA_TRY(ctx, b.d_xyz.ensure(3 * T));
      B2M_CUDA_TRY(ctx, b.d_inl.ensure(T));
      B2M_CUDA_TRY(ctx, b.d_succ.ensure(T));
      B2M_CUDA_TRY(ctx, b.d_mask.ensure(M));
      B2M_CUDA_TRY(ctx, b.d_scratch.ensure(M));
      b.cap_tracks = T;
      b.cap_obs = M;
      return B2M_OK;
    });
    if (rc) return rc;
  }
  if (images > 0) {
    B2M_CUDA_TRY(ctx, s->d_cams.ensure(12 * images));
    B2M_CUDA_TRY(ctx, s->d_centers.ensure(3 * images));
  }
  return B2M_OK;
}

}  // namespace
}  // namespace b2m

using namespace b2m;

extern "C" {

void b2m_tri_opts_default(b2m_tri_opts* o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->struct_size = sizeof(*o);
  o->min_tri_angle = 0.0;
  b2m_ransac_opts_default(&o->ransac);
}

int b2m_estimate_triangulation_batch(b2m_ctx* ctx, int64_t n_tracks, const int64_t* track_offsets,
                                     const double* points_normalized, const int32_t* image_idx, int32_t n_images,
                                     const double* cams_from_world, const b2m_tri_opts* opts, double* xyz,
                                     int32_t* num_inliers, uint8_t* success, uint8_t* inlier_mask) {
  if (!ctx) return B2M_EINVAL;
  if (!opts || n_tracks < 0 || (n_tracks > 0 && (!track_offsets || !xyz || !num_inliers || !success)))
    return fail(ctx, B2M_EINVAL, "[triangulation.cu] Check Failed: track_offsets, options and outputs != NULL");
  if (opts->struct_size != sizeof(b2m_tri_opts) || opts->ransac.struct_size != sizeof(b2m_ransac_opts))
    return fail(ctx, B2M_EINVAL, "[triangulation.cu] Check Failed: b2m_tri_opts.struct_size == sizeof(b2m_tri_opts)");
  // EstimateTriangulationOptions::Check, RANSACOptions::Check (U:estimators/triangulation.h, U:optim/ransac.h)
  const b2m_ransac_opts& ro = opts->ransac;
  if (!(opts->min_tri_angle >= 0.0)) return fail(ctx, B2M_EINVAL, "[triangulation.h] Check Failed: min_tri_angle >= 0");
  if (!(ro.max_error > 0.0)) return fail(ctx, B2M_EINVAL, "[ransac.h] Check Failed: max_error > 0");
  if (!(ro.min_inlier_ratio >= 0.0 && ro.min_inlier_ratio <= 1.0))
    return fail(ctx, B2M_EINVAL, "[ransac.h] Check Failed: min_inlier_ratio in [0, 1]");
  if (!(ro.confidence >= 0.0 && ro.confidence <= 1.0)) return fail(ctx, B2M_EINVAL, "[ransac.h] Check Failed: confidence in [0, 1]");
  if (!(ro.min_num_trials <= ro.max_num_trials)) return fail(ctx, B2M_EINVAL, "[ransac.h] Check Failed: min_num_trials <= max_num_trials");
  if (n_tracks == 0) return B2M_OK;
  if (track_offsets[0] != 0) return fail(ctx, B2M_EINVAL, "[triangulation.cu] Check Failed: track_offsets[0] == 0");
  for (int64_t k = 0; k < n_tracks; ++k)
    if (!(track_offsets[k + 1] - track_offsets[k] >= 2))  // THROW_CHECK_GE(point_data.size(), 2)
      return fail(ctx, B2M_EINVAL, "[triangulation.cc] Check Failed: point_data.size() >= 2 (track " + std::to_string(k) + ")");
  const int64_t M = track_offsets[n_tracks];
  if (!points_normalized || !image_idx || !cams_from_world)
    return fail(ctx, B2M_EINVAL, "[triangulation.cu] Check Failed: points, image indices and cameras != NULL");
  for (int64_t i = 0; i < M; ++i)
    if (image_idx[i] < 0 || image_idx[i] >= n_images)
      return fail(ctx, B2M_EINVAL, "[triangulation.cu] Check Failed: 0 <= image_idx < n_images (observation " + std::to_string(i) + ")");
  for (int64_t k = 0; k < n_tracks; ++k)
    if (track_offsets[k + 1] - track_offsets[k] > INT32_MAX)
      return fail(ctx, B2M_EINVAL, "[triangulation.cu] Check Failed: observations per track < 2^31");

  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  // projection centres -R^T t
  std::vector<double> centers(3 * static_cast<size_t>(n_images));
  for (int32_t i = 0; i < n_images; ++i) {
    const double* P = cams_from_world + 12 * static_cast<size_t>(i);
    for (int a = 0; a < 3; ++a)
      centers[3 * i + a] = -(P[0 * 4 + a] * P[3] + P[1 * 4 + a] * P[7] + P[2 * 4 + a] * P[11]);
  }
  const double max_trials = geom::ransac_trial_cap(ro, 2);  // kMinNumSamples = 2

  // chunks: at most kChunkTracks tracks and kChunkObs observations (a longer single track is its own chunk)
  std::vector<int64_t> starts{0};
  int64_t cap_t = 0, cap_o = 0;
  while (starts.back() < n_tracks) {
    const int64_t k0 = starts.back();
    int64_t k1 = k0 + 1;
    while (k1 < n_tracks && k1 - k0 < kChunkTracks && track_offsets[k1 + 1] - track_offsets[k0] <= kChunkObs) ++k1;
    cap_t = std::max(cap_t, k1 - k0);
    cap_o = std::max(cap_o, track_offsets[k1] - track_offsets[k0]);
    starts.push_back(k1);
  }
  TriState* S = nullptr;
  if (int rc = ensure_state(ctx, cap_t, cap_o, n_images, &S)) return rc;
  B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->d_cams, cams_from_world, sizeof(double) * 12 * n_images, cudaMemcpyHostToDevice, st));
  B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->d_centers, centers.data(), sizeof(double) * 3 * n_images, cudaMemcpyHostToDevice, st));
  std::vector<int32_t> order;
  for (size_t c = 0; c + 1 < starts.size(); ++c) {
    if (ctx->stop) return B2M_ESTOPPED;
    const int64_t k0 = starts[c], k1 = starts[c + 1];
    const int nb = static_cast<int>(k1 - k0);
    const int64_t o0 = track_offsets[k0], mo = track_offsets[k1] - o0;
    memcpy(S->chunk.h_pts, points_normalized + 2 * o0, sizeof(double) * 2 * mo);
    memcpy(S->chunk.h_img, image_idx + o0, sizeof(int32_t) * mo);
    for (int k = 0; k <= nb; ++k) S->chunk.h_off[k] = track_offsets[k0 + k] - o0;
    order.resize(nb);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(),
                     [&](int32_t a, int32_t b) { return S->chunk.h_off[a + 1] - S->chunk.h_off[a] > S->chunk.h_off[b + 1] - S->chunk.h_off[b]; });
    memcpy(S->chunk.h_order, order.data(), sizeof(int32_t) * nb);
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->chunk.d_pts, S->chunk.h_pts, sizeof(double) * 2 * mo, cudaMemcpyHostToDevice, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->chunk.d_img, S->chunk.h_img, sizeof(int32_t) * mo, cudaMemcpyHostToDevice, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->chunk.d_off, S->chunk.h_off, sizeof(int64_t) * (nb + 1), cudaMemcpyHostToDevice, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->chunk.d_order, S->chunk.h_order, sizeof(int32_t) * nb, cudaMemcpyHostToDevice, st));
    TriParams P{};
    P.pts = S->chunk.d_pts; P.img = S->chunk.d_img; P.off = S->chunk.d_off; P.order = S->chunk.d_order;
    P.cams = S->d_cams; P.centers = S->d_centers; P.nb = nb;
    P.max_residual = ro.max_error * ro.max_error;
    P.min_tri_angle = opts->min_tri_angle;
    P.confidence = ro.confidence;
    P.multiplier = ro.dyn_num_trials_multiplier;
    P.max_trials = max_trials;
    P.min_num_trials = static_cast<double>(ro.min_num_trials);
    P.xyz = S->chunk.d_xyz; P.num_inliers = S->chunk.d_inl; P.success = S->chunk.d_succ; P.mask = S->chunk.d_mask; P.scratch = S->chunk.d_scratch;
    P.counters = ctx->d_counters + kTriCounters;
    b2m_tri_ransac_kernel<<<static_cast<unsigned>((nb + kWarps - 1) / kWarps), 32 * kWarps, 0, st>>>(P);
    B2M_CUDA_TRY(ctx, cudaGetLastError());
    ctx->stats.kernel_launches += 1;
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->chunk.h_xyz, S->chunk.d_xyz, sizeof(double) * 3 * nb, cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->chunk.h_inl, S->chunk.d_inl, sizeof(int32_t) * nb, cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->chunk.h_succ, S->chunk.d_succ, nb, cudaMemcpyDeviceToHost, st));
    if (inlier_mask) B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->chunk.h_mask, S->chunk.d_mask, mo, cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
    memcpy(xyz + 3 * k0, S->chunk.h_xyz, sizeof(double) * 3 * nb);
    memcpy(num_inliers + k0, S->chunk.h_inl, sizeof(int32_t) * nb);
    memcpy(success + k0, S->chunk.h_succ, nb);
    if (inlier_mask) memcpy(inlier_mask + o0, S->chunk.h_mask, mo);
  }
  return B2M_OK;
}

}  // extern "C"
