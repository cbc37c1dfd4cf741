// geom.h -- two-view geometry math shared by the K2/K3 verification kernels: symmetric Jacobi
// eigen-solver, real polynomial roots, 5-point essential (Nister elimination), 7-point and
// normalised 8-point fundamental, normalised 4-point / N-point DLT homography, Sampson and
// transfer residuals.  Header-only, fp64, `B2M_HD` = __host__ __device__ so that the same code is
// unit-tested on the CPU (tests/helpers/geom_host.cpp) and runs one-hypothesis-per-thread on sm_90a.
//
// Semantics follow COLMAP 3.9.1 (SURVEY.md section 8 rows V4-V7):
//   U:estimators/essential_matrix.cc   EssentialMatrixFivePointEstimator (>=5 points, <=10 models)
//   U:estimators/fundamental_matrix.cc FundamentalMatrixSevenPointEstimator / EightPointEstimator
//   U:estimators/homography_matrix.cc  HomographyMatrixEstimator (normalised DLT, forward transfer error)
//   U:estimators/utils.cc              CenterAndNormalizeImagePoints, ComputeSquaredSampsonError
// reached from R:estimators/two_view_geometry.h:95-151 and R:estimators/essential_matrix.h:48-52,
// R:estimators/fundamental_matrix.h:26-29, R:estimators/homography_matrix.h:25-27.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/b200match.h"

#ifdef __CUDACC__
#define B2M_HD __host__ __device__
#else
#define B2M_HD
#endif

namespace b2m {
namespace geom {

// ---------------------------------------------------------------------------------------------
// Cyclic Jacobi eigen-decomposition of a symmetric N x N matrix (row-major, destroyed).
// On return w[i] are eigenvalues and column i of V (V[r*N+i]) the matching eigenvector.
// ---------------------------------------------------------------------------------------------
template <int N>
B2M_HD inline void jacobi_eig_sym(double* A, double* V, double* w) {
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) V[i * N + j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off = 0.0, diag = 0.0;
    for (int i = 0; i < N; ++i) {
      diag += A[i * N + i] * A[i * N + i];
      for (int j = i + 1; j < N; ++j) off += A[i * N + j] * A[i * N + j];
    }
    if (off <= 1e-30 * diag || off == 0.0) break;
    for (int p = 0; p < N - 1; ++p) {
      for (int q = p + 1; q < N; ++q) {
        const double apq = A[p * N + q];
        if (apq == 0.0) continue;
        const double app = A[p * N + p], aqq = A[q * N + q];
        const double theta = (aqq - app) / (2.0 * apq);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < N; ++k) {  // A <- A J (columns p, q)
          const double akp = A[k * N + p], akq = A[k * N + q];
          A[k * N + p] = c * akp - s * akq;
          A[k * N + q] = s * akp + c * akq;
        }
        for (int k = 0; k < N; ++k) {  // A <- J^T A (rows p, q)
          const double apk = A[p * N + k], aqk = A[q * N + k];
          A[p * N + k] = c * apk - s * aqk;
          A[q * N + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < N; ++k) {
          const double vkp = V[k * N + p], vkq = V[k * N + q];
          V[k * N + p] = c * vkp - s * vkq;
          V[k * N + q] = s * vkp + c * vkq;
        }
      }
    }
  }
  for (int i = 0; i < N; ++i) w[i] = A[i * N + i];
}

// Indices of the `k` smallest eigenvalues, ascending.
template <int N>
B2M_HD inline void smallest_k(const double* w, int k, int* idx) {
  bool used[N];
  for (int i = 0; i < N; ++i) used[i] = false;
  for (int s = 0; s < k; ++s) {
    int best = -1;
    for (int i = 0; i < N; ++i)
      if (!used[i] && (best < 0 || w[i] < w[best])) best = i;
    used[best] = true;
    idx[s] = best;
  }
}

// ---------------------------------------------------------------------------------------------
// Real roots of c[0] + c[1] x + ... + c[deg] x^deg (deg <= 10).  Roots of p lie between
// consecutive critical points, so solve the derivatives bottom-up and bracket + safeguarded
// Newton in every sign-changing interval.  Returns the number of roots (ascending).
// ---------------------------------------------------------------------------------------------
B2M_HD inline double poly_eval(const double* c, int deg, double x) {
  double r = c[deg];
  for (int i = deg - 1; i >= 0; --i) r = r * x + c[i];
  return r;
}

B2M_HD inline double poly_refine(const double* c, int deg, double lo, double hi, double flo) {
  // f(lo) and f(hi) have opposite signs (flo = f(lo)); bisection-safeguarded Newton.
  double x = 0.5 * (lo + hi);
  for (int it = 0; it < 200; ++it) {
    double f = c[deg], df = 0.0;
    for (int i = deg - 1; i >= 0; --i) {
      df = df * x + f;
      f = f * x + c[i];
    }
    if (f == 0.0) return x;
    if ((f < 0.0) == (flo < 0.0)) lo = x; else hi = x;
    double xn = x - f / df;
    if (!(xn > lo && xn < hi)) xn = 0.5 * (lo + hi);
    if (fabs(xn - x) <= 4e-16 * fabs(xn) || hi - lo <= 4e-16 * fabs(lo + hi)) return xn;
    x = xn;
  }
  return x;
}

B2M_HD inline int poly_real_roots(const double* coef, int deg_in, double* roots) {
  constexpr int MAXD = 10;
  double c[MAXD + 1];
  double mx = 0.0;
  for (int i = 0; i <= deg_in; ++i) {
    c[i] = coef[i];
    if (fabs(c[i]) > mx) mx = fabs(c[i]);
  }
  if (!(mx > 0.0) || !(mx < 1e300)) return 0;
  int deg = deg_in;
  while (deg > 0 && fabs(c[deg]) <= 1e-14 * mx) --deg;
  if (deg == 0) return 0;
  // Fujiwara's bound on |root|: 2 max_k |c[deg-k] / c[deg]|^(1/k).  Within a factor 2 of the largest root modulus,
  // where Cauchy's 1 + max |c[i] / c[deg]| can be off by many orders of magnitude -- and the safeguarded Newton in
  // the two outer intervals converges only linearly (factor 1 - 1/deg per step) while it is that far from the root:
  // with Cauchy's bound the degree-10 polynomial of a random 5-point sample regularly burned ~170 iterations per level.
  double bound = 0.0;
  for (int i = 0; i < deg; ++i) {
    const double v = fabs(c[i] / c[deg]);
    if (v > 0.0) {
      const double t = pow(v, 1.0 / static_cast<double>(deg - i));
      if (t > bound) bound = t;
    }
  }
  bound = 2.0 * bound * (1.0 + 1e-9);
  if (!(bound > 0.0)) bound = 1.0;
  // derivative ladder: d[k] = k-th derivative scaled (coefficients), degree deg-k.  (A one-level-at-a-time variant
  // that rebuilds the coefficients per level from c[] was measured SLOWER inside the E kernel -- B2M_PROF `solve`
  // 206 k -> 348 k Mcycles per two steps -- and was reverted.)
  double d[MAXD][MAXD + 1];  // d[0] = p
  for (int i = 0; i <= deg; ++i) d[0][i] = c[i];
  for (int k = 1; k < deg; ++k)
    for (int i = 0; i <= deg - k; ++i) d[k][i] = d[k - 1][i + 1] * (i + 1);
  double prev[MAXD], cur[MAXD];
  int nprev = 0;
  // start from the linear polynomial d[deg-1]
  {
    const double* q = d[deg - 1];
    prev[0] = -q[0] / q[1];
    nprev = 1;
  }
  for (int k = deg - 2; k >= 0; --k) {
    const int dg = deg - k;
    const double* q = d[k];
    int ncur = 0;
    double lo = -bound, flo = poly_eval(q, dg, lo);
    for (int i = 0; i <= nprev; ++i) {
      const double hi = (i < nprev) ? prev[i] : bound;
      if (!(hi > lo)) continue;
      const double fhi = poly_eval(q, dg, hi);
      if (flo == 0.0) {
        if (ncur == 0 || cur[ncur - 1] != lo) cur[ncur++] = lo;
      } else if (fhi != 0.0 && ((flo < 0.0) != (fhi < 0.0))) {
        cur[ncur++] = poly_refine(q, dg, lo, hi, flo);
      }
      lo = hi;
      flo = fhi;
      if (ncur >= dg) break;
    }
    if (flo == 0.0 && ncur < dg && (ncur == 0 || cur[ncur - 1] != lo)) cur[ncur++] = lo;
    for (int i = 0; i < ncur; ++i) prev[i] = cur[i];
    nprev = ncur;
  }
  for (int i = 0; i < nprev; ++i) roots[i] = prev[i];
  return nprev;
}

// ---------------------------------------------------------------------------------------------
// Residuals
// ---------------------------------------------------------------------------------------------
// ComputeSquaredSampsonError (U:estimators/utils.cc); E row-major.
B2M_HD inline double sampson_sq(const double* E, double x1, double y1, double x2, double y2) {
  const double Ex1_0 = E[0] * x1 + E[1] * y1 + E[2];
  const double Ex1_1 = E[3] * x1 + E[4] * y1 + E[5];
  const double Ex1_2 = E[6] * x1 + E[7] * y1 + E[8];
  const double Etx2_0 = E[0] * x2 + E[3] * y2 + E[6];
  const double Etx2_1 = E[1] * x2 + E[4] * y2 + E[7];
  const double x2tEx1 = x2 * Ex1_0 + y2 * Ex1_1 + Ex1_2;
  return x2tEx1 * x2tEx1 / (Ex1_0 * Ex1_0 + Ex1_1 * Ex1_1 + Etx2_0 * Etx2_0 + Etx2_1 * Etx2_1);
}
// HomographyMatrixEstimator::Residuals: squared forward transfer error.
B2M_HD inline double homography_sq(const double* H, double x1, double y1, double x2, double y2) {
  const double pd_0 = H[0] * x1 + H[1] * y1 + H[2];
  const double pd_1 = H[3] * x1 + H[4] * y1 + H[5];
  const double pd_2 = H[6] * x1 + H[7] * y1 + H[8];
  const double inv = 1.0 / pd_2;
  const double dd_0 = x2 - pd_0 * inv, dd_1 = y2 - pd_1 * inv;
  return dd_0 * dd_0 + dd_1 * dd_1;
}

// ---------------------------------------------------------------------------------------------
// Rows of the linear systems (all accumulate A^T A, upper triangle incl. diagonal, 45 entries,
// index(i,j) = i*9 - i*(i-1)/2 + (j-i) for i <= j).
// ---------------------------------------------------------------------------------------------
B2M_HD inline int sym9_index(int i, int j) { return i * 9 - (i * (i - 1)) / 2 + (j - i); }

B2M_HD inline void sym9_add_row(double* S, const double* r) {
  int k = 0;
  for (int i = 0; i < 9; ++i)
    for (int j = i; j < 9; ++j) S[k++] += r[i] * r[j];
}
B2M_HD inline void sym9_expand(const double* S, double* A) {
  int k = 0;
  for (int i = 0; i < 9; ++i)
    for (int j = i; j < 9; ++j) {
      A[i * 9 + j] = S[k];
      A[j * 9 + i] = S[k];
      ++k;
    }
}
// epipolar constraint row x2^T E x1 = 0 (E row-major)
B2M_HD inline void epipolar_row(double x1, double y1, double x2, double y2, double* r) {
  r[0] = x2 * x1; r[1] = x2 * y1; r[2] = x2;
  r[3] = y2 * x1; r[4] = y2 * y1; r[5] = y2;
  r[6] = x1;      r[7] = y1;      r[8] = 1.0;
}
// the two DLT rows of HomographyMatrixEstimator::Estimate (s = source, d = destination)
B2M_HD inline void dlt_rows(double s0, double s1, double d0, double d1, double* r1, double* r2) {
  r1[0] = -s0; r1[1] = -s1; r1[2] = -1.0; r1[3] = 0; r1[4] = 0; r1[5] = 0; r1[6] = s0 * d0; r1[7] = s1 * d0; r1[8] = d0;
  r2[0] = 0; r2[1] = 0; r2[2] = 0; r2[3] = -s0; r2[4] = -s1; r2[5] = -1.0; r2[6] = s0 * d1; r2[7] = s1 * d1; r2[8] = d1;
}

// CenterAndNormalizeImagePoints from moment sums: n, sum x, sum y, sum (x^2+y^2).
// Returns scale s and centroid (cx, cy): normalised p = s * (p - c); T = [[s,0,-s cx],[0,s,-s cy],[0,0,1]].
B2M_HD inline void norm_from_moments(double n, double sx, double sy, double sq, double* s, double* cx, double* cy) {
  *cx = sx / n;
  *cy = sy / n;
  const double ms = sq / n - ((*cx) * (*cx) + (*cy) * (*cy));  // mean squared distance to the centroid
  const double rms = sqrt(ms > 0.0 ? ms : 0.0);
  *s = sqrt(2.0) / rms;
}

// 3x3 helpers (row-major)
B2M_HD inline void mat3_mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
}

// F_pixel = T2^T F_norm T1 with Ti = [[s,0,-s cx],[0,s,-s cy],[0,0,1]]
B2M_HD inline void denormalize_F(const double* Fn, double s1, double cx1, double cy1, double s2, double cx2,
                                 double cy2, double* F) {
  const double T1[9] = {s1, 0, -s1 * cx1, 0, s1, -s1 * cy1, 0, 0, 1};
  const double T2t[9] = {s2, 0, 0, 0, s2, 0, -s2 * cx2, -s2 * cy2, 1};
  double tmp[9];
  mat3_mul(Fn, T1, tmp);
  mat3_mul(T2t, tmp, F);
}
// H_pixel = T2^-1 H_norm T1
B2M_HD inline void denormalize_H(const double* Hn, double s1, double cx1, double cy1, double s2, double cx2,
                                 double cy2, double* H) {
  const double T1[9] = {s1, 0, -s1 * cx1, 0, s1, -s1 * cy1, 0, 0, 1};
  const double T2i[9] = {1.0 / s2, 0, cx2, 0, 1.0 / s2, cy2, 0, 0, 1};
  double tmp[9];
  mat3_mul(Hn, T1, tmp);
  mat3_mul(T2i, tmp, H);
}

// Zero the smallest singular value of a 3x3 matrix: F <- F (I - v v^T), v = eigenvector of F^T F
// with the smallest eigenvalue.
B2M_HD inline void enforce_rank2(double* F) {
  double G[9], V[9], w[3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) G[i * 3 + j] = F[i] * F[j] + F[3 + i] * F[3 + j] + F[6 + i] * F[6 + j];
  jacobi_eig_sym<3>(G, V, w);
  int m = 0;
  if (w[1] < w[m]) m = 1;
  if (w[2] < w[m]) m = 2;
  const double v[3] = {V[m], V[3 + m], V[6 + m]};
  for (int i = 0; i < 3; ++i) {
    const double fv = F[i * 3] * v[0] + F[i * 3 + 1] * v[1] + F[i * 3 + 2] * v[2];
    for (int j = 0; j < 3; ++j) F[i * 3 + j] -= fv * v[j];
  }
}

// Smallest-eigenvalue eigenvector of the accumulated 9x9 normal matrix -> 3x3 (row-major).
B2M_HD inline void smallest_eigvec9_jacobi(const double* S45, double* out9) {
  double A[81], V[81], w[9];
  sym9_expand(S45, A);
  jacobi_eig_sym<9>(A, V, w);
  int idx[1];
  smallest_k<9>(w, 1, idx);
  for (int i = 0; i < 9; ++i) out9[i] = V[i * 9 + idx[0]];
}
template <int K>
B2M_HD inline void smallest_eigvecs_invit(const double* S45, double* out);
B2M_HD inline void smallest_eigvec9(const double* S45, double* out9) { smallest_eigvecs_invit<1>(S45, out9); }

// K smallest eigenvectors (an orthonormal basis of that invariant subspace) of a symmetric
// positive semi-definite 9x9 matrix by Cholesky-based inverse subspace iteration.  ~50x cheaper than
// the Jacobi sweep and good to full precision whenever the K-th and (K+1)-th eigenvalues are
// separated, which is exactly when the least-squares null space of the LO refits is well defined.
// out: [K][9]; out[0] belongs to the smallest eigenvalue (Rayleigh-ordered).
template <int K>
B2M_HD inline void smallest_eigvecs_invit(const double* S45, double* out) {
  double L[81];
  sym9_expand(S45, L);
  double tr = 0.0;
  for (int i = 0; i < 9; ++i) tr += L[i * 9 + i];
  const double mu = tr * 1e-14 + 1e-300;
  for (int i = 0; i < 9; ++i) L[i * 9 + i] += mu;
  // in-place Cholesky, lower triangle
  for (int j = 0; j < 9; ++j) {
    double d = L[j * 9 + j];
    for (int k = 0; k < j; ++k) d -= L[j * 9 + k] * L[j * 9 + k];
    if (!(d > mu * 1e-3)) d = mu * 1e-3;
    const double ljj = sqrt(d);
    L[j * 9 + j] = ljj;
    const double inv = 1.0 / ljj;
    for (int i = j + 1; i < 9; ++i) {
      double s = L[i * 9 + j];
      for (int k = 0; k < j; ++k) s -= L[i * 9 + k] * L[j * 9 + k];
      L[i * 9 + j] = s * inv;
    }
  }
  // deterministic, generic start vectors
  for (int k = 0; k < K; ++k)
    for (int i = 0; i < 9; ++i) {
      const int h = (i * 37 + k * 101 + 11) % 17;
      out[k * 9 + i] = (static_cast<double>(h) - 8.0) * 0.1 + (i == 8 - k ? 1.0 : 0.0);
    }
  double rdiag[9];  // 1 / L(i, i): 9 divisions instead of 108 per basis vector (fp64 division is the slow op here)
  for (int i = 0; i < 9; ++i) rdiag[i] = 1.0 / L[i * 9 + i];
  for (int it = 0; it < 6; ++it) {
    double before[9];  // K == 1: stop as soon as the iterate is stationary (inverse iteration converges geometrically
                       // with ratio lambda_1 / lambda_2: two or three steps on the near-exact systems of the LO refits)
    if (K == 1)
      for (int i = 0; i < 9; ++i) before[i] = out[i];
    for (int k = 0; k < K; ++k) {
      double* v = out + k * 9;
      for (int i = 0; i < 9; ++i) {  // L y = v
        double s = v[i];
        for (int j = 0; j < i; ++j) s -= L[i * 9 + j] * v[j];
        v[i] = s * rdiag[i];
      }
      for (int i = 8; i >= 0; --i) {  // L^T x = y
        double s = v[i];
        for (int j = i + 1; j < 9; ++j) s -= L[j * 9 + i] * v[j];
        v[i] = s * rdiag[i];
      }
    }
    for (int k = 0; k < K; ++k) {  // modified Gram-Schmidt
      double* v = out + k * 9;
      for (int q = 0; q < k; ++q) {
        const double* u = out + q * 9;
        double dot = 0.0;
        for (int i = 0; i < 9; ++i) dot += u[i] * v[i];
        for (int i = 0; i < 9; ++i) v[i] -= dot * u[i];
      }
      double nn = 0.0;
      for (int i = 0; i < 9; ++i) nn += v[i] * v[i];
      const double inv = 1.0 / sqrt(nn > 0.0 ? nn : 1.0);
      for (int i = 0; i < 9; ++i) v[i] *= inv;
    }
    if (K == 1 && it > 0) {
      double dp = 0.0, dm = 0.0;   // the iterate may flip its sign from step to step
      for (int i = 0; i < 9; ++i) {
        dp += (out[i] - before[i]) * (out[i] - before[i]);
        dm += (out[i] + before[i]) * (out[i] + before[i]);
      }
      if ((dp < dm ? dp : dm) < 1e-30) break;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// 7-point fundamental: two null vectors f1, f2 -> det(l f1 + (1-l) f2) = 0 -> 1 or 3 models.
// ---------------------------------------------------------------------------------------------
B2M_HD inline int seven_point_from_nullspace(const double* f1, const double* f2, double* F_out /* [3][9] */) {
  // entries: a_i + l * b_i with a = f2, b = f1 - f2
  double a[9], b[9];
  for (int i = 0; i < 9; ++i) {
    a[i] = f2[i];
    b[i] = f1[i] - f2[i];
  }
  // det = sum over the 6 permutations of products of three linear polynomials
  double c[4] = {0, 0, 0, 0};
  const int perm[6][3] = {{0, 4, 8}, {1, 5, 6}, {2, 3, 7}, {2, 4, 6}, {1, 3, 8}, {0, 5, 7}};
  for (int p = 0; p < 6; ++p) {
    const int i = perm[p][0], j = perm[p][1], k = perm[p][2];
    const double sg = p < 3 ? 1.0 : -1.0;
    // (a_i + l b_i)(a_j + l b_j)(a_k + l b_k)
    const double q0 = a[i] * a[j], q1 = a[i] * b[j] + b[i] * a[j], q2 = b[i] * b[j];
    c[0] += sg * (q0 * a[k]);
    c[1] += sg * (q0 * b[k] + q1 * a[k]);
    c[2] += sg * (q1 * b[k] + q2 * a[k]);
    c[3] += sg * (q2 * b[k]);
  }
  double roots[3];
  const int n = poly_real_roots(c, 3, roots);
  for (int r = 0; r < n; ++r)
    for (int i = 0; i < 9; ++i) F_out[r * 9 + i] = a[i] + roots[r] * b[i];
  return n;
}

// ---------------------------------------------------------------------------------------------
// 5-point essential from a 4-D null space N[4][9] (E = x N0 + y N1 + z N2 + N3).
// Nister's elimination: 10 cubic constraints -> Gauss-Jordan -> 3x3 polynomial matrix in z ->
// degree-10 polynomial -> real roots -> (x, y).  Returns the number of models (<= 10).
// ---------------------------------------------------------------------------------------------
namespace detail {
// dense polynomial storage in (x,y,z): index a*16 + b*4 + c, exponents < 4
B2M_HD inline void lin_mul_lin(const double* p, const double* q, double* out27) {
  // p, q: coefficients of (x, y, z, 1); out: dense deg<=2, index a*9+b*3+c
  for (int i = 0; i < 27; ++i) out27[i] = 0.0;
  const int ea[4] = {1, 0, 0, 0}, eb[4] = {0, 1, 0, 0}, ec[4] = {0, 0, 1, 0};
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j)
      out27[(ea[i] + ea[j]) * 9 + (eb[i] + eb[j]) * 3 + (ec[i] + ec[j])] += p[i] * q[j];
}
B2M_HD inline void quad_mul_lin_acc(const double* q27, const double* p, double sign, double* out64) {
  const int ea[4] = {1, 0, 0, 0}, eb[4] = {0, 1, 0, 0}, ec[4] = {0, 0, 1, 0};
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b + a < 3; ++b)
      for (int c = 0; c + b + a < 3; ++c) {
        const double v = q27[a * 9 + b * 3 + c];
        if (v == 0.0) continue;
        for (int j = 0; j < 4; ++j) out64[(a + ea[j]) * 16 + (b + eb[j]) * 4 + (c + ec[j])] += sign * v * p[j];
      }
}
// gather the 20 cubic monomials in Nister's order:
// x3 y3 x2y xy2 x2z x2 y2z y2 xyz xy | xz2 xz x yz2 yz y z3 z2 z 1
B2M_HD inline void gather20(const double* d64, double* row) {
#define B2M_M(a, b, c) d64[(a) * 16 + (b) * 4 + (c)]
  row[0] = B2M_M(3, 0, 0); row[1] = B2M_M(0, 3, 0); row[2] = B2M_M(2, 1, 0); row[3] = B2M_M(1, 2, 0);
  row[4] = B2M_M(2, 0, 1); row[5] = B2M_M(2, 0, 0); row[6] = B2M_M(0, 2, 1); row[7] = B2M_M(0, 2, 0);
  row[8] = B2M_M(1, 1, 1); row[9] = B2M_M(1, 1, 0); row[10] = B2M_M(1, 0, 2); row[11] = B2M_M(1, 0, 1);
  row[12] = B2M_M(1, 0, 0); row[13] = B2M_M(0, 1, 2); row[14] = B2M_M(0, 1, 1); row[15] = B2M_M(0, 1, 0);
  row[16] = B2M_M(0, 0, 3); row[17] = B2M_M(0, 0, 2); row[18] = B2M_M(0, 0, 1); row[19] = B2M_M(0, 0, 0);
#undef B2M_M
}
// 1-D polynomial helpers (ascending coefficients)
B2M_HD inline void pmul(const double* a, int da, const double* b, int db, double* out) {
  for (int i = 0; i <= da + db; ++i) out[i] = 0.0;
  for (int i = 0; i <= da; ++i)
    for (int j = 0; j <= db; ++j) out[i + j] += a[i] * b[j];
}
}  // namespace detail

B2M_HD inline int five_point_from_nullspace(const double* N /* [4][9] */, double* E_out /* [10][9] */) {
  using namespace detail;
  // E entry e (0..8) as linear polynomial in (x, y, z, 1)
  double L[9][4];
  for (int e = 0; e < 9; ++e)
    for (int k = 0; k < 4; ++k) L[e][k] = N[k * 9 + e];

  double M[10][20];
  double d64[64];
  double q27[27], r27[27];

  // row 0: det(E)
  for (int i = 0; i < 64; ++i) d64[i] = 0.0;
  {
    const int t[6][3] = {{0, 4, 8}, {1, 5, 6}, {2, 3, 7}, {2, 4, 6}, {1, 3, 8}, {0, 5, 7}};
    for (int p = 0; p < 6; ++p) {
      lin_mul_lin(L[t[p][0]], L[t[p][1]], q27);
      quad_mul_lin_acc(q27, L[t[p][2]], p < 3 ? 1.0 : -1.0, d64);
    }
  }
  gather20(d64, M[0]);

  // EEt (symmetric) as dense quadratics; Lambda = EEt - 0.5 trace(EEt) I
  double EEt[6][27];  // (0,0) (0,1) (0,2) (1,1) (1,2) (2,2)
  {
    int k = 0;
    for (int i = 0; i < 3; ++i)
      for (int j = i; j < 3; ++j) {
        for (int t = 0; t < 27; ++t) EEt[k][t] = 0.0;
        for (int m = 0; m < 3; ++m) {
          lin_mul_lin(L[i * 3 + m], L[j * 3 + m], r27);
          for (int t = 0; t < 27; ++t) EEt[k][t] += r27[t];
        }
        ++k;
      }
  }
  for (int t = 0; t < 27; ++t) {
    const double half_tr = 0.5 * (EEt[0][t] + EEt[3][t] + EEt[5][t]);
    EEt[0][t] -= half_tr;
    EEt[3][t] -= half_tr;
    EEt[5][t] -= half_tr;
  }
  const int sym_idx[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
  // rows 1..9: (Lambda * E)(i, j) = sum_m Lambda(i, m) * E(m, j)
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      for (int t = 0; t < 64; ++t) d64[t] = 0.0;
      for (int m = 0; m < 3; ++m) quad_mul_lin_acc(EEt[sym_idx[i][m]], L[m * 3 + j], 1.0, d64);
      gather20(d64, M[1 + i * 3 + j]);
    }

  // Gauss-Jordan on the first 10 columns with partial pivoting
  for (int col = 0; col < 10; ++col) {
    int piv = col;
    double best = fabs(M[col][col]);
    for (int r = col + 1; r < 10; ++r)
      if (fabs(M[r][col]) > best) {
        best = fabs(M[r][col]);
        piv = r;
      }
    if (!(best > 1e-300)) return 0;
    if (piv != col)
      for (int k = 0; k < 20; ++k) {
        const double tmp = M[col][k];
        M[col][k] = M[piv][k];
        M[piv][k] = tmp;
      }
    const double inv = 1.0 / M[col][col];
    for (int k = col; k < 20; ++k) M[col][k] *= inv;
    for (int r = 0; r < 10; ++r) {
      if (r == col) continue;
      const double f = M[r][col];
      if (f == 0.0) continue;
      for (int k = col; k < 20; ++k) M[r][k] -= f * M[col][k];
    }
  }

  // rows e=4 (x2z), f=5 (x2), g=6 (y2z), h=7 (y2), i=8 (xyz), j=9 (xy); columns 10..19 =
  // [xz2 xz x yz2 yz y z3 z2 z 1].  k = e - z f, l = g - z h, m = i - z j give the 3x3 matrix B(z)
  // with B (x, y, 1)^T = 0; entries: degree 3, 3, 4 polynomials in z (ascending coefficients).
  double Bx[3][4], By[3][4], Bc[3][5];
  for (int r = 0; r < 3; ++r) {
    const double* a = &M[4 + 2 * r][10];
    const double* b = &M[5 + 2 * r][10];
    Bx[r][0] = a[2];         Bx[r][1] = a[1] - b[2]; Bx[r][2] = a[0] - b[1]; Bx[r][3] = -b[0];
    By[r][0] = a[5];         By[r][1] = a[4] - b[5]; By[r][2] = a[3] - b[4]; By[r][3] = -b[3];
    Bc[r][0] = a[9];         Bc[r][1] = a[8] - b[9]; Bc[r][2] = a[7] - b[8]; Bc[r][3] = a[6] - b[7];
    Bc[r][4] = -b[6];
  }
  // det B(z) = Bx0 (By1 Bc2 - Bc1 By2) - By0 (Bx1 Bc2 - Bc1 Bx2) + Bc0 (Bx1 By2 - By1 Bx2)
  double n10[11];
  for (int i = 0; i < 11; ++i) n10[i] = 0.0;
  {
    double t7a[8], t7b[8], t6a[7], t6b[7], prod[11];
    pmul(By[1], 3, Bc[2], 4, t7a);
    pmul(Bc[1], 4, By[2], 3, t7b);
    for (int i = 0; i < 8; ++i) t7a[i] -= t7b[i];
    pmul(Bx[0], 3, t7a, 7, prod);
    for (int i = 0; i < 11; ++i) n10[i] += prod[i];
    pmul(Bx[1], 3, Bc[2], 4, t7a);
    pmul(Bc[1], 4, Bx[2], 3, t7b);
    for (int i = 0; i < 8; ++i) t7a[i] -= t7b[i];
    pmul(By[0], 3, t7a, 7, prod);
    for (int i = 0; i < 11; ++i) n10[i] -= prod[i];
    pmul(Bx[1], 3, By[2], 3, t6a);
    pmul(By[1], 3, Bx[2], 3, t6b);
    for (int i = 0; i < 7; ++i) t6a[i] -= t6b[i];
    pmul(Bc[0], 4, t6a, 6, prod);
    for (int i = 0; i < 11; ++i) n10[i] += prod[i];
  }
  double roots[10];
  const int nr = poly_real_roots(n10, 10, roots);
  int nm = 0;
  for (int r = 0; r < nr; ++r) {
    const double z = roots[r];
    double bx[3], by[3], bc[3];
    for (int k = 0; k < 3; ++k) {
      bx[k] = poly_eval(Bx[k], 3, z);
      by[k] = poly_eval(By[k], 3, z);
      bc[k] = poly_eval(Bc[k], 4, z);
    }
    // (x, y, 1) is the null vector of B(z): cross product of the best-conditioned pair of rows
    double bestw = 0.0, X = 0.0, Y = 0.0;
    for (int a = 0; a < 3; ++a) {
      const int b = (a + 1) % 3;
      const double cxp = by[a] * bc[b] - bc[a] * by[b];
      const double cyp = bc[a] * bx[b] - bx[a] * bc[b];
      const double cw = bx[a] * by[b] - by[a] * bx[b];
      if (fabs(cw) > fabs(bestw)) {
        bestw = cw;
        X = cxp;
        Y = cyp;
      }
    }
    if (!(fabs(bestw) > 0.0)) continue;
    const double x = X / bestw, y = Y / bestw;
    double* E = E_out + nm * 9;
    for (int e = 0; e < 9; ++e) E[e] = x * N[e] + y * N[9 + e] + z * N[18 + e] + N[27 + e];
    ++nm;
  }
  return nm;
}

// ---------------------------------------------------------------------------------------------
// Estimators on small explicit point lists (minimal samples).  Points: x1[i], y1[i], x2[i], y2[i].
// ---------------------------------------------------------------------------------------------
// E: >= 5 normalised correspondences -> <= 10 models.
B2M_HD inline int estimate_E(const double* x1, const double* y1, const double* x2, const double* y2, int n,
                             double* models) {
  double S[45];
  for (int i = 0; i < 45; ++i) S[i] = 0.0;
  double r[9];
  for (int i = 0; i < n; ++i) {
    epipolar_row(x1[i], y1[i], x2[i], y2[i], r);
    sym9_add_row(S, r);
  }
  double A[81], V[81], w[9];
  sym9_expand(S, A);
  jacobi_eig_sym<9>(A, V, w);
  int idx[4];
  smallest_k<9>(w, 4, idx);
  double N[36];
  for (int k = 0; k < 4; ++k)
    for (int e = 0; e < 9; ++e) N[k * 9 + e] = V[e * 9 + idx[3 - k]];  // N3 = smallest
  return five_point_from_nullspace(N, models);
}

B2M_HD inline void moments(const double* x, const double* y, int n, double* s, double* cx, double* cy) {
  double sx = 0, sy = 0, sq = 0;
  for (int i = 0; i < n; ++i) {
    sx += x[i];
    sy += y[i];
    sq += x[i] * x[i] + y[i] * y[i];
  }
  norm_from_moments(n, sx, sy, sq, s, cx, cy);
}

// F from exactly 7 pixel correspondences -> 1 or 3 models.  (Points are Hartley-normalised
// internally for conditioning; the solution set is invariant to that.)
B2M_HD inline int estimate_F7(const double* x1, const double* y1, const double* x2, const double* y2,
                              double* models) {
  double s1, cx1, cy1, s2, cx2, cy2;
  moments(x1, y1, 7, &s1, &cx1, &cy1);
  moments(x2, y2, 7, &s2, &cx2, &cy2);
  double S[45];
  for (int i = 0; i < 45; ++i) S[i] = 0.0;
  double r[9];
  for (int i = 0; i < 7; ++i) {
    epipolar_row(s1 * (x1[i] - cx1), s1 * (y1[i] - cy1), s2 * (x2[i] - cx2), s2 * (y2[i] - cy2), r);
    sym9_add_row(S, r);
  }
  double A[81], V[81], w[9];
  sym9_expand(S, A);
  jacobi_eig_sym<9>(A, V, w);
  int idx[2];
  smallest_k<9>(w, 2, idx);
  double f1[9], f2[9];
  for (int e = 0; e < 9; ++e) {
    f1[e] = V[e * 9 + idx[0]];
    f2[e] = V[e * 9 + idx[1]];
  }
  double Fn[27];
  const int n = seven_point_from_nullspace(f1, f2, Fn);
  for (int k = 0; k < n; ++k) denormalize_F(Fn + 9 * k, s1, cx1, cy1, s2, cx2, cy2, models + 9 * k);
  return n;
}

// F from n >= 8 pixel correspondences (normalised 8-point, rank-2 enforced) -> 1 model.
B2M_HD inline int finish_F8(const double* S45, double s1, double cx1, double cy1, double s2, double cx2,
                            double cy2, double* model) {
  double Fn[9];
  smallest_eigvec9(S45, Fn);
  enforce_rank2(Fn);
  denormalize_F(Fn, s1, cx1, cy1, s2, cx2, cy2, model);
  return 1;
}
// H from n >= 4 pixel correspondences (normalised DLT) -> 1 model.
B2M_HD inline int finish_H(const double* S45, double s1, double cx1, double cy1, double s2, double cx2,
                           double cy2, double* model) {
  double Hn[9];
  smallest_eigvec9(S45, Hn);
  denormalize_H(Hn, s1, cx1, cy1, s2, cx2, cy2, model);
  return 1;
}
B2M_HD inline int estimate_H(const double* x1, const double* y1, const double* x2, const double* y2, int n,
                             double* model) {
  double s1, cx1, cy1, s2, cx2, cy2;
  moments(x1, y1, n, &s1, &cx1, &cy1);
  moments(x2, y2, n, &s2, &cx2, &cy2);
  double S[45];
  for (int i = 0; i < 45; ++i) S[i] = 0.0;
  double r1[9], r2[9];
  for (int i = 0; i < n; ++i) {
    dlt_rows(s1 * (x1[i] - cx1), s1 * (y1[i] - cy1), s2 * (x2[i] - cx2), s2 * (y2[i] - cy2), r1, r2);
    sym9_add_row(S, r1);
    sym9_add_row(S, r2);
  }
  return finish_H(S, s1, cx1, cy1, s2, cx2, cy2, model);
}
B2M_HD inline int estimate_F8(const double* x1, const double* y1, const double* x2, const double* y2, int n,
                              double* model) {
  double s1, cx1, cy1, s2, cx2, cy2;
  moments(x1, y1, n, &s1, &cx1, &cy1);
  moments(x2, y2, n, &s2, &cx2, &cy2);
  double S[45];
  for (int i = 0; i < 45; ++i) S[i] = 0.0;
  double r[9];
  for (int i = 0; i < n; ++i) {
    epipolar_row(s1 * (x1[i] - cx1), s1 * (y1[i] - cy1), s2 * (x2[i] - cx2), s2 * (y2[i] - cy2), r);
    sym9_add_row(S, r);
  }
  return finish_F8(S, s1, cx1, cy1, s2, cx2, cy2, model);
}

// ---------------------------------------------------------------------------------------------
// Null space of an R x 9 matrix (R < 9, full row rank) by Gauss-Jordan elimination with complete
// pivoting.  A is destroyed.  basis: [(9-R)][9], not orthonormal (none of the solvers needs that).
// Much cheaper than an eigen-decomposition for the minimal samples (5x9, 7x9, 8x9).
// ---------------------------------------------------------------------------------------------
template <int R>
B2M_HD inline bool nullspace_gauss(double* A /* [R][9] */, double* basis) {
  int perm[9];
  for (int j = 0; j < 9; ++j) perm[j] = j;
  for (int r = 0; r < R; ++r) {
    int pi = r, pj = r;
    double best = 0.0;
    for (int i = r; i < R; ++i)
      for (int j = r; j < 9; ++j) {
        const double v = fabs(A[i * 9 + j]);
        if (v > best) {
          best = v;
          pi = i;
          pj = j;
        }
      }
    if (!(best > 0.0) || !(best < 1e300)) return false;
    if (pi != r)
      for (int j = 0; j < 9; ++j) {
        const double t = A[r * 9 + j];
        A[r * 9 + j] = A[pi * 9 + j];
        A[pi * 9 + j] = t;
      }
    if (pj != r) {
      for (int i = 0; i < R; ++i) {
        const double t = A[i * 9 + r];
        A[i * 9 + r] = A[i * 9 + pj];
        A[i * 9 + pj] = t;
      }
      const int t = perm[r];
      perm[r] = perm[pj];
      perm[pj] = t;
    }
    const double inv = 1.0 / A[r * 9 + r];
    for (int j = r; j < 9; ++j) A[r * 9 + j] *= inv;
    for (int i = 0; i < R; ++i) {
      if (i == r) continue;
      const double f = A[i * 9 + r];
      if (f == 0.0) continue;
      for (int j = r; j < 9; ++j) A[i * 9 + j] -= f * A[r * 9 + j];
    }
  }
  for (int k = 0; k < 9 - R; ++k) {
    double* v = basis + k * 9;
    for (int j = 0; j < 9; ++j) v[j] = 0.0;
    v[perm[R + k]] = 1.0;
    for (int i = 0; i < R; ++i) v[perm[i]] = -A[i * 9 + R + k];
  }
  return true;
}

// Minimal solvers (exactly 5 / 7 / 4 correspondences), elimination-based null spaces.
B2M_HD inline int minimal_E5(const double* x1, const double* y1, const double* x2, const double* y2, double* models) {
  double A[45], N[36];
  for (int i = 0; i < 5; ++i) epipolar_row(x1[i], y1[i], x2[i], y2[i], A + 9 * i);
  if (!nullspace_gauss<5>(A, N)) return 0;
  return five_point_from_nullspace(N, models);
}
B2M_HD inline int minimal_F7(const double* x1, const double* y1, const double* x2, const double* y2, double* models) {
  double s1, cx1, cy1, s2, cx2, cy2;
  moments(x1, y1, 7, &s1, &cx1, &cy1);
  moments(x2, y2, 7, &s2, &cx2, &cy2);
  double A[63], N[18];
  for (int i = 0; i < 7; ++i)
    epipolar_row(s1 * (x1[i] - cx1), s1 * (y1[i] - cy1), s2 * (x2[i] - cx2), s2 * (y2[i] - cy2), A + 9 * i);
  if (!nullspace_gauss<7>(A, N)) return 0;
  double Fn[27];
  const int n = seven_point_from_nullspace(N, N + 9, Fn);
  for (int k = 0; k < n; ++k) denormalize_F(Fn + 9 * k, s1, cx1, cy1, s2, cx2, cy2, models + 9 * k);
  return n;
}
// Closed-form 4-point homography, registers only (no arrays -> no local memory on the GPU):
// for each image find the projective map taking the canonical frame (e1, e2, e3, e1+e2+e3) to the
// four points, A = [l p0 | m p1 | n p2] with l p0 + m p1 + n p2 = p3 (Cramer), then H = B adj(A).
// Four correspondences in general position determine H uniquely up to scale, so this equals the
// DLT null vector of HomographyMatrixEstimator::Estimate for minimal samples.
B2M_HD inline bool frame_from_4pts(const double* x, const double* y, double* A) {
  // columns p0, p1, p2 (homogeneous, w = 1); solve [p0 p1 p2] (l, m, n)^T = p3
  const double x0 = x[0], y0 = y[0], x1 = x[1], y1 = y[1], x2 = x[2], y2 = y[2], x3 = x[3], y3 = y[3];
  const double det = x0 * (y1 - y2) - x1 * (y0 - y2) + x2 * (y0 - y1);
  const double l = x3 * (y1 - y2) - x1 * (y3 - y2) + x2 * (y3 - y1);
  const double m = x0 * (y3 - y2) - x3 * (y0 - y2) + x2 * (y0 - y3);
  const double n = x0 * (y1 - y3) - x1 * (y0 - y3) + x3 * (y0 - y1);
  if (!(fabs(det) > 0.0)) return false;
  // scale by 1/det is irrelevant (homogeneous); keep l, m, n un-normalised
  A[0] = l * x0; A[1] = m * x1; A[2] = n * x2;
  A[3] = l * y0; A[4] = m * y1; A[5] = n * y2;
  A[6] = l;      A[7] = m;      A[8] = n;
  return true;
}
B2M_HD inline int minimal_H4_closed(const double* x1, const double* y1, const double* x2, const double* y2,
                                    double* H) {
  // translate both point sets to their centroids first (conditioning), undo at the end
  const double c1x = 0.25 * (x1[0] + x1[1] + x1[2] + x1[3]), c1y = 0.25 * (y1[0] + y1[1] + y1[2] + y1[3]);
  const double c2x = 0.25 * (x2[0] + x2[1] + x2[2] + x2[3]), c2y = 0.25 * (y2[0] + y2[1] + y2[2] + y2[3]);
  const double ax[4] = {x1[0] - c1x, x1[1] - c1x, x1[2] - c1x, x1[3] - c1x};
  const double ay[4] = {y1[0] - c1y, y1[1] - c1y, y1[2] - c1y, y1[3] - c1y};
  const double bx[4] = {x2[0] - c2x, x2[1] - c2x, x2[2] - c2x, x2[3] - c2x};
  const double by[4] = {y2[0] - c2y, y2[1] - c2y, y2[2] - c2y, y2[3] - c2y};
  double A[9], B[9];
  if (!frame_from_4pts(ax, ay, A) || !frame_from_4pts(bx, by, B)) return 0;
  // adj(A) (transpose of the cofactor matrix)
  const double J[9] = {A[4] * A[8] - A[5] * A[7], A[2] * A[7] - A[1] * A[8], A[1] * A[5] - A[2] * A[4],
                       A[5] * A[6] - A[3] * A[8], A[0] * A[8] - A[2] * A[6], A[2] * A[3] - A[0] * A[5],
                       A[3] * A[7] - A[4] * A[6], A[1] * A[6] - A[0] * A[7], A[0] * A[4] - A[1] * A[3]};
  double Hc[9];
  mat3_mul(B, J, Hc);
  // H = T2^-1 Hc T1 with T1 = translate(-c1), T2^-1 = translate(+c2)
  double nrm = 0.0;
  for (int i = 0; i < 9; ++i) nrm += Hc[i] * Hc[i];
  if (!(nrm > 0.0) || !(nrm < 1e300)) return 0;
  const double s = 1.0 / sqrt(nrm);
  for (int i = 0; i < 9; ++i) Hc[i] *= s;
  // right-multiply by T1: third column += -(c1x * col0 + c1y * col1)
  for (int r = 0; r < 3; ++r) Hc[r * 3 + 2] -= Hc[r * 3] * c1x + Hc[r * 3 + 1] * c1y;
  // left-multiply by T2^-1: row0 += c2x * row2, row1 += c2y * row2
  for (int c = 0; c < 3; ++c) {
    H[c] = Hc[c] + c2x * Hc[6 + c];
    H[3 + c] = Hc[3 + c] + c2y * Hc[6 + c];
    H[6 + c] = Hc[6 + c];
  }
  return 1;
}

B2M_HD inline int minimal_H4(const double* x1, const double* y1, const double* x2, const double* y2, double* model) {
  double s1, cx1, cy1, s2, cx2, cy2;
  moments(x1, y1, 4, &s1, &cx1, &cy1);
  moments(x2, y2, 4, &s2, &cx2, &cy2);
  double A[72], Hn[9];
  for (int i = 0; i < 4; ++i)
    dlt_rows(s1 * (x1[i] - cx1), s1 * (y1[i] - cy1), s2 * (x2[i] - cx2), s2 * (y2[i] - cy2), A + 18 * i, A + 18 * i + 9);
  if (!nullspace_gauss<8>(A, Hn)) return 0;
  denormalize_H(Hn, s1, cx1, cy1, s2, cx2, cy2, model);
  return 1;
}

// ComputeNumTrials (U:optim/ransac.h)
B2M_HD inline double compute_num_trials(double num_inliers, double num_samples, double confidence,
                                        double multiplier, int k_min) {
  const double ratio = num_inliers / num_samples;
  const double nom = 1.0 - confidence;
  if (nom <= 0.0) return 1e18;
  const double denom = 1.0 - pow(ratio, static_cast<double>(k_min));
  if (denom <= 0.0) return 1.0;
  if (denom == 1.0) return 1e18;
  return ceil(log(nom) / log(denom) * multiplier);
}

// The RANSAC constructor's clip (U:optim/ransac.h): max_num_trials, at most the bound at min_inlier_ratio.
B2M_HD inline double ransac_trial_cap(const b2m_ransac_opts& ro, int min_samples) {
  return fmin(static_cast<double>(ro.max_num_trials),
              compute_num_trials(floor(ro.min_inlier_ratio * 100000.0), 100000.0, ro.confidence,
                                 ro.dyn_num_trials_multiplier, min_samples));
}

}  // namespace geom
}  // namespace b2m
