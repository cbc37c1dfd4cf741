// eig_warp.cuh -- the K smallest eigenvectors of the N x N normal matrix of an LO refit, computed by ONE WARP
// (N = 9: the E / F / H refits of the verifier; N = 12: the EPnP refit of the absolute pose estimator).
//
// Same algorithm, same operations in the same order per matrix element as geom.h smallest_eigvecs_invit<K>
// (Cholesky-based inverse subspace iteration), so the result is bit-identical; what changes is who computes what:
// the serial version keeps L[81] in thread-local memory and walks one ~1500-operation dependent chain while the other
// 127 threads of the CTA wait at a barrier (B2M_PROF `lo_solve`: 17 % of the CTA time of the RANSAC kernels).  Here
// the matrix lives in shared memory, lane i owns row i (and column i) of the factor in registers, the column of a
// Cholesky step and the updates of a substitution step run in parallel, and only the inherently serial parts (one
// pivot, one solved component at a time) stay serial.
#pragma once
#include <cstdint>

namespace b2m {
namespace eigw {

template <int N>
struct ScratchN {
  double L[N * N];   // the factor, row-major
  double v[4][N];    // the iterated basis
  double inv;        // 1 / L(j, j) of the current Cholesky step
};
using Scratch = ScratchN<9>;

__device__ __forceinline__ double bcast(double x, int src) {
  const int lo = __shfl_sync(0xffffffffu, __double2loint(x), src);
  const int hi = __shfl_sync(0xffffffffu, __double2hiint(x), src);
  return __hiloint2double(hi, lo);
}

// S45: upper triangle of the symmetric matrix, row-major packed (geom.h sym9_expand for N = 9); out: [K][N], out[0]
// belongs to the smallest eigenvalue.  All 32 lanes of the warp must call; S45 / out may live in shared or global
// memory.  ITERS: subspace iterations (K == 1 stops early once the iterate is stationary).
template <int K, int N = 9, int ITERS = 6>
__device__ __forceinline__ void smallest_eigvecs_warp(const double* S45, double* out, ScratchN<N>& W, int lane) {
  // ---- expand + regularise (lane i: row i)
  if (lane < N) {
    for (int j = 0; j < N; ++j) {
      const int a = lane < j ? lane : j, b = lane < j ? j : lane;      // packed index of (a, b), a <= b
      W.L[lane * N + j] = S45[a * N - a * (a - 1) / 2 + (b - a)];
    }
  }
  __syncwarp();
  double tr = 0.0;
  for (int i = 0; i < N; ++i) tr += W.L[i * N + i];
  const double mu = tr * 1e-14 + 1e-300;
  __syncwarp();
  if (lane < N) W.L[lane * N + lane] += mu;
  __syncwarp();
  // ---- in-place Cholesky, lower triangle: the pivot on lane j, the rest of column j on lanes j + 1 .. N - 1
#pragma unroll 1
  for (int j = 0; j < N; ++j) {
    if (lane == j) {
      double d = W.L[j * N + j];
      for (int k = 0; k < j; ++k) d -= W.L[j * N + k] * W.L[j * N + k];
      if (!(d > mu * 1e-3)) d = mu * 1e-3;
      const double ljj = sqrt(d);
      W.L[j * N + j] = ljj;
      W.inv = 1.0 / ljj;
    }
    __syncwarp();
    if (lane > j && lane < N) {
      double s = W.L[lane * N + j];
      for (int k = 0; k < j; ++k) s -= W.L[lane * N + k] * W.L[j * N + k];
      W.L[lane * N + j] = s * W.inv;
    }
    __syncwarp();
  }
  // ---- row / column of this lane in registers, reciprocal diagonal
  const int li = lane < N ? lane : N - 1;
  double row[N], col[N];
#pragma unroll
  for (int j = 0; j < N; ++j) {
    row[j] = W.L[li * N + j];
    col[j] = W.L[j * N + li];
  }
  const double rd = 1.0 / W.L[li * N + li];   // 1 / L(i, i)
  // deterministic, generic start vectors
  if (lane < N)
    for (int k = 0; k < K; ++k) {
      const int h = (lane * 37 + k * 101 + 11) % 17;
      W.v[k][lane] = (static_cast<double>(h) - 8.0) * 0.1 + (lane == N - 1 - k ? 1.0 : 0.0);
    }
  __syncwarp();
#pragma unroll 1
  for (int it = 0; it < ITERS; ++it) {
    double before[N];
    if (K == 1)
      for (int i = 0; i < N; ++i) before[i] = W.v[0][i];
#pragma unroll 1
    for (int k = 0; k < K; ++k) {
      // L y = v: component j is final once the components before it are; every later row then takes its update
      // (row i subtracts L(i, j) y_j in increasing j, the serial order)
      double s = W.v[k][li];
#pragma unroll
      for (int j = 0; j < N; ++j) {
        const double yj = bcast(s * rd, j);
        if (lane > j) s -= row[j] * yj;
        if (lane == j) s = yj;
      }
      // L^T x = y: x_i = (y_i - sum_{j > i} L(j, i) x_j) / L(i, i) with the sum in increasing j (the serial order), so
      // lane i waits for all later components and then runs its own short chain
      double x[N];
#pragma unroll
      for (int i = N - 1; i >= 0; --i) {
        double t = s;
#pragma unroll
        for (int j = i + 1; j < N; ++j) t -= col[j] * x[j];
        x[i] = bcast(t * rd, i);
      }
      __syncwarp();
      if (lane < N) {
        double mine = 0.0;
#pragma unroll
        for (int i = 0; i < N; ++i) mine = (i == lane) ? x[i] : mine;
        W.v[k][lane] = mine;
      }
      __syncwarp();
    }
    // modified Gram-Schmidt + normalisation: N-term serial sums, computed redundantly by every lane (same bits)
#pragma unroll 1
    for (int k = 0; k < K; ++k) {
      for (int q = 0; q < k; ++q) {
        double dot = 0.0;
        for (int i = 0; i < N; ++i) dot += W.v[q][i] * W.v[k][i];
        __syncwarp();
        if (lane < N) W.v[k][lane] -= dot * W.v[q][lane];
        __syncwarp();
      }
      double nn = 0.0;
      for (int i = 0; i < N; ++i) nn += W.v[k][i] * W.v[k][i];
      const double inv = 1.0 / sqrt(nn > 0.0 ? nn : 1.0);
      __syncwarp();
      if (lane < N) W.v[k][lane] *= inv;
      __syncwarp();
    }
    if (K == 1 && it > 0) {
      double dp = 0.0, dm = 0.0;   // the iterate may flip its sign from step to step
      for (int i = 0; i < N; ++i) {
        const double a = W.v[0][i];
        dp += (a - before[i]) * (a - before[i]);
        dm += (a + before[i]) * (a + before[i]);
      }
      if ((dp < dm ? dp : dm) < 1e-30) break;   // uniform across the warp: every lane computed the same sums
    }
  }
  if (lane < N)
    for (int k = 0; k < K; ++k) out[k * N + lane] = W.v[k][lane];
  __syncwarp();
}

}  // namespace eigw
}  // namespace b2m
