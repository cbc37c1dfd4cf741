// abs_pose.cu -- batched absolute pose estimation (LO-RANSAC with P3P hypotheses and EPnP local optimisation, optional
// focal-length sampling) and robust pose refinement (Levenberg-Marquardt, Cauchy loss, optional camera parameters and
// covariance) behind b2m_estimate_absolute_pose_batch / b2m_refine_absolute_pose_batch.
//
// Semantics: U:estimators/pose.cc EstimateAbsolutePose / RefineAbsolutePose, U:estimators/absolute_pose.cc
// P3PEstimator / EPNPEstimator, reached from R:pycolmap/estimators/absolute_pose.h:18-166; SURVEY.md section 8(a)
// rows A1-A5.  The specification is oracle/abs_pose.py.
//
// Kernels:
//   b2m_abs_ransac_kernel  one CTA per (problem, focal-length sample).  The CTA undistorts the problem's 2-D points
//                          with the scaled camera, then runs LO-RANSAC: a round is up to 128 P3P hypotheses (thread =
//                          hypothesis, <= 4 models each), scored by the whole CTA with the division-free fp32 test
//                          (u Z - X)^2 + (v Z - Y)^2 <= thr Z^2, Z > 0, borderline points re-decided in fp64, and the
//                          exact pruning (the round of ransac_common.cuh); a new best goes through EPnP refits on its
//                          inliers (moments reduced by the CTA, the 12 x 12 eigenproblem on one warp, the beta solve on
//                          one thread).
//   b2m_abs_select_kernel  one warp per problem: the focal sample with strictly the most inliers (earliest on ties),
//                          its inlier mask, the pose in world coordinates and the camera parameters.
//   b2m_abs_refine_kernel  one warp per problem: LM on 6 + k unknowns (k <= 10 camera parameters), exact Jacobians from
//                          forward-mode dual numbers through camera_models.h, Ceres' loss correction, optional
//                          covariance from the same normal matrix.
// Sampling is keyed by (ctx seed, position of the problem in the call, focal sample, trial).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "eig_warp.cuh"
#include "geom.h"
#include "internal.h"
#include "pose.h"
#include "ransac_common.cuh"

namespace b2m {

// ---- forward-mode dual numbers for the refinement Jacobians ------------------------------------------------
namespace ad {
constexpr int kD = 12;  // d/du, d/dv and up to 10 refined camera parameters
struct Dual {
  double v;
  double d[kD];
  __device__ Dual() {}
  __device__ Dual(double x) : v(x) {
#pragma unroll
    for (int i = 0; i < kD; ++i) d[i] = 0.0;
  }
};
#define B2M_AD_BIN(op, dv_expr)                                                        \
  __device__ inline Dual operator op(const Dual& a, const Dual& b) {                   \
    Dual r;                                                                            \
    r.v = a.v op b.v;                                                                  \
    for (int i = 0; i < kD; ++i) r.d[i] = dv_expr;                                     \
    return r;                                                                          \
  }
B2M_AD_BIN(+, a.d[i] + b.d[i])
B2M_AD_BIN(-, a.d[i] - b.d[i])
B2M_AD_BIN(*, a.d[i] * b.v + a.v * b.d[i])
#undef B2M_AD_BIN
__device__ inline Dual operator/(const Dual& a, const Dual& b) {
  Dual r;
  const double ib = 1.0 / b.v;
  r.v = a.v * ib;
  for (int i = 0; i < kD; ++i) r.d[i] = (a.d[i] - r.v * b.d[i]) * ib;
  return r;
}
__device__ inline Dual operator+(const Dual& a, double b) { return a + Dual(b); }
__device__ inline Dual operator+(double a, const Dual& b) { return Dual(a) + b; }
__device__ inline Dual operator-(const Dual& a, double b) { return a - Dual(b); }
__device__ inline Dual operator-(double a, const Dual& b) { return Dual(a) - b; }
__device__ inline Dual operator*(const Dual& a, double b) {
  Dual r;
  r.v = a.v * b;
  for (int i = 0; i < kD; ++i) r.d[i] = a.d[i] * b;
  return r;
}
__device__ inline Dual operator*(double a, const Dual& b) { return b * a; }
__device__ inline Dual operator/(const Dual& a, double b) { return a * (1.0 / b); }
__device__ inline Dual operator/(double a, const Dual& b) { return Dual(a) / b; }
__device__ inline Dual operator-(const Dual& a) { return a * -1.0; }
__device__ inline Dual& operator*=(Dual& a, const Dual& b) { return a = a * b; }
__device__ inline bool operator>(const Dual& a, double b) { return a.v > b; }
__device__ inline bool operator<(const Dual& a, double b) { return a.v < b; }
__device__ inline Dual chain(const Dual& a, double f, double df) {
  Dual r;
  r.v = f;
  for (int i = 0; i < kD; ++i) r.d[i] = df * a.d[i];
  return r;
}
__device__ inline Dual sqrt(const Dual& a) {
  const double s = ::sqrt(a.v);
  return chain(a, s, s > 0.0 ? 0.5 / s : 0.0);
}
__device__ inline Dual atan(const Dual& a) { return chain(a, ::atan(a.v), 1.0 / (1.0 + a.v * a.v)); }
__device__ inline Dual tan(const Dual& a) {
  const double t = ::tan(a.v);
  return chain(a, t, 1.0 + t * t);
}
__device__ inline Dual sin(const Dual& a) { return chain(a, ::sin(a.v), ::cos(a.v)); }
__device__ inline Dual cos(const Dual& a) { return chain(a, ::cos(a.v), -::sin(a.v)); }
__device__ inline Dual fabs(const Dual& a) { return a.v < 0.0 ? -a : a; }
}  // namespace ad

namespace {

using namespace geom;

constexpr int kMaxLocalTrials = 10;
constexpr int kMaxRefine = 16;   // 6 pose + up to 10 camera parameters
constexpr double kDblEps = 2.220446049250313e-16;
constexpr double kDblMax = 1.7976931348623157e308;

struct DevCam {
  int32_t model;
  int32_t pad;
  double p[cam::kMaxParams];
};

struct RansacParams {
  const double* px;          // [total x 2] pixel coordinates
  const double* p3;          // [total x 3] world points
  const double* centroid;    // [nb x 3] per-problem mean of the world points (the kernel scores centred points)
  const int64_t* off;        // [nb] offset (points) of the problem
  const int32_t* cnt;        // [nb]
  const int64_t* xoff;       // [nb * n_factors] offset of the CTA's normalised points / mask
  const DevCam* cams;        // [nb]
  double2* xn;               // normalised points arena
  uint8_t* mask;             // per-CTA inlier masks (same offsets as xn)
  double* models;            // [nb * n_factors][12] 3 x 4 row-major, centred world frame
  int32_t* sup;              // [nb * n_factors]
  int32_t* success;          // [nb * n_factors]
  const double* factors;     // [n_factors]
  int32_t n_factors;
  int32_t pad;
  b2m_ransac_opts ro;
  uint64_t seed;
  int64_t problem_base;      // position of problem 0 of this launch in the call
  unsigned long long* counters;  // [2]: models scored, residual evaluations (b2m_stats), or nullptr
};

struct Shared {
  RoundShared<12> round;
  double best_model[12];
  double cand[3][12];
  double red[4][40];
  double mtm[78];
  double eigv[4][12];
  eigw::ScratchN<12> es;
  double cw[4][3];
  double ccinv[9];
  double mom[10];            // n, sum P (3), sum P P^T (xx, xy, xz, yy, yz, zz)
  double cand_err[3];
  double best_sum;
  int best_cnt;
  int n_cand;
  int first;
  int lo_ok;
};

__device__ __forceinline__ void load_point(const RansacParams& P, const double2* xn, int64_t off, int i, const double* c,
                                           double& u, double& v, double& X, double& Y, double& Z) {
  const double2 x = xn[i];
  u = x.x;
  v = x.y;
  const double* q = P.p3 + 3 * (off + i);
  X = q[0] - c[0];
  Y = q[1] - c[1];
  Z = q[2] - c[2];
}

// P3PEstimator::Residuals / EPNPEstimator::Residuals: squared reprojection error on the normalised plane
__device__ __forceinline__ double reproj_sq(const double* M, double u, double v, double X, double Y, double Z) {
  const double xc = M[0] * X + M[1] * Y + M[2] * Z + M[3];
  const double yc = M[4] * X + M[5] * Y + M[6] * Z + M[7];
  const double zc = M[8] * X + M[9] * Y + M[10] * Z + M[11];
  if (!(zc > kDblEps)) return kDblMax;
  const double du = xc / zc - u, dv = yc / zc - v;
  return du * du + dv * dv;
}

// division-free fp32 test of reproj_sq <= thr (see classify_f32); the camera-side depth must be clearly positive
__device__ __forceinline__ int inlier_f32(const float* M, float u, float v, float X, float Y, float Z, float thr) {
  const float xc = fmaf(M[0], X, fmaf(M[1], Y, fmaf(M[2], Z, M[3])));
  const float yc = fmaf(M[4], X, fmaf(M[5], Y, fmaf(M[6], Z, M[7])));
  const float zc = fmaf(M[8], X, fmaf(M[9], Y, fmaf(M[10], Z, M[11])));
  const float mag = 1e-3f * (fabsf(xc) + fabsf(yc) + fabsf(zc));
  if (zc < -mag) return 0;      // behind the camera in fp64 as well: outlier
  if (!(zc > mag)) return 2;    // near the camera plane or not finite: fp64 decides
  const float ex = fmaf(u, zc, -xc), ey = fmaf(v, zc, -yc);
  return classify_f32(fmaf(ex, ex, ey * ey), thr * zc * zc);
}

// A problem's correspondences and poses in the shared LO-RANSAC round (ransac_common.cuh).
struct ReprojModel {
  static constexpr int kD = 12;
  struct Pt {
    float u, v, X, Y, Z;
  };
  const RansacParams& P;
  const double2* xn;
  int64_t off;
  const double* c;
  // a slot past the end is a point behind the camera (Z = -1)
  __device__ __forceinline__ Pt load_f32(int i, bool live) const {
    double u = 0, v = 0, X = 0, Y = 0, Z = -1;
    if (live) load_point(P, xn, off, i, c, u, v, X, Y, Z);
    return {static_cast<float>(u), static_cast<float>(v), static_cast<float>(X), static_cast<float>(Y), static_cast<float>(Z)};
  }
  __device__ __forceinline__ int test(const float* M, const Pt& p, float thr) const {
    return inlier_f32(M, p.u, p.v, p.X, p.Y, p.Z, thr);
  }
  __device__ __forceinline__ double residual(const double* M, int i) const {
    double u, v, X, Y, Z;
    load_point(P, xn, off, i, c, u, v, X, Y, Z);
    return reproj_sq(M, u, v, X, Y, Z);
  }
};

__device__ void frame3(const double* a, const double* b, const double* c, double* F /* columns e1 e2 e3 */) {
  double e1[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, d2[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]}, e3[3], e2[3];
  pose::cross3(e1, d2, e3);
  const double n1 = pose::norm3(e1), n3 = pose::norm3(e3);
  for (int k = 0; k < 3; ++k) {
    e1[k] /= n1;
    e3[k] /= n3;
  }
  pose::cross3(e3, e1, e2);
  for (int r = 0; r < 3; ++r) {
    F[r * 3 + 0] = e1[r];
    F[r * 3 + 1] = e2[r];
    F[r * 3 + 2] = e3[r];
  }
}

// P3P (Grunert's quartic; the same real solution set as any P3P formulation, oracle/abs_pose.py P3PEstimator).
// x, y: normalised image points; W: 3 world points (row-major [3][3]).  models: [4][12].
__device__ int p3p(const double* x, const double* y, const double* W, double* models) {
  double f[3][3];
  for (int i = 0; i < 3; ++i) {
    const double n = sqrt(x[i] * x[i] + y[i] * y[i] + 1.0);
    f[i][0] = x[i] / n; f[i][1] = y[i] / n; f[i][2] = 1.0 / n;
  }
  auto d2 = [&](int i, int j) {
    const double a = W[3 * i] - W[3 * j], b = W[3 * i + 1] - W[3 * j + 1], c = W[3 * i + 2] - W[3 * j + 2];
    return a * a + b * b + c * c;
  };
  const double a2 = d2(1, 2), b2 = d2(0, 2), c2 = d2(0, 1);
  if (!(a2 > 0.0 && b2 > 0.0 && c2 > 0.0)) return 0;
  const double ca = f[1][0] * f[2][0] + f[1][1] * f[2][1] + f[1][2] * f[2][2];
  const double cb = f[0][0] * f[2][0] + f[0][1] * f[2][1] + f[0][2] * f[2][2];
  const double cg = f[0][0] * f[1][0] + f[0][1] * f[1][1] + f[0][2] * f[1][2];
  const double p = (a2 - c2) / b2, q = (a2 + c2) / b2;
  double coef[5];
  coef[4] = (p - 1) * (p - 1) - 4 * c2 / b2 * ca * ca;
  coef[3] = 4 * (p * (1 - p) * cb - (1 - q) * ca * cg + 2 * c2 / b2 * ca * ca * cb);
  coef[2] = 2 * (p * p - 1 + 2 * p * p * cb * cb + 2 * (b2 - c2) / b2 * ca * ca - 4 * q * ca * cb * cg +
                 2 * (b2 - a2) / b2 * cg * cg);
  coef[1] = 4 * (-p * (1 + p) * cb + 2 * a2 / b2 * cg * cg * cb - (1 - q) * ca * cg);
  coef[0] = (1 + p) * (1 + p) - 4 * a2 / b2 * cg * cg;
  double roots[4];
  const int nr = poly_real_roots(coef, 4, roots);
  double Fw[9];
  frame3(W, W + 3, W + 6, Fw);
  int nm = 0;
  for (int k = 0; k < nr && nm < 4; ++k) {
    const double v = roots[k];
    const double den = 2 * (cg - v * ca);
    if (den == 0.0) continue;
    const double u = ((p - 1) * v * v - 2 * p * cb * v + 1 + p) / den;
    const double s1sq = c2 / (1 + u * u - 2 * u * cg);
    if (!(s1sq > 0.0 && u > 0.0 && v > 0.0)) continue;
    const double s1 = sqrt(s1sq);
    double Q[9];
    for (int r = 0; r < 3; ++r) {
      Q[r] = s1 * f[0][r];
      Q[3 + r] = u * s1 * f[1][r];
      Q[6 + r] = v * s1 * f[2][r];
    }
    double Fc[9], Rm[9];
    frame3(Q, Q + 3, Q + 6, Fc);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) Rm[i * 3 + j] = Fc[i * 3] * Fw[j * 3] + Fc[i * 3 + 1] * Fw[j * 3 + 1] + Fc[i * 3 + 2] * Fw[j * 3 + 2];
    double* M = models + 12 * nm;
    bool finite = true;
    for (int i = 0; i < 3; ++i) {
      M[4 * i] = Rm[3 * i]; M[4 * i + 1] = Rm[3 * i + 1]; M[4 * i + 2] = Rm[3 * i + 2];
      M[4 * i + 3] = Q[i] - (Rm[3 * i] * W[0] + Rm[3 * i + 1] * W[1] + Rm[3 * i + 2] * W[2]);
      for (int j = 0; j < 4; ++j) finite = finite && isfinite(M[4 * i + j]);
    }
    if (finite) ++nm;
  }
  return nm;
}

// Least squares min |A x - b| (A: m x k row-major, k <= 5) through the normal equations.
__device__ void lstsq_small(const double* A, const double* b, int m, int k, double* x) {
  double N[5][6];
  for (int i = 0; i < k; ++i) {
    for (int j = 0; j < k; ++j) {
      double s = 0.0;
      for (int r = 0; r < m; ++r) s += A[r * k + i] * A[r * k + j];
      N[i][j] = s;
    }
    double s = 0.0;
    for (int r = 0; r < m; ++r) s += A[r * k + i] * b[r];
    N[i][k] = s;
  }
  for (int c = 0; c < k; ++c) {  // Gauss-Jordan with partial pivoting
    int piv = c;
    for (int r = c + 1; r < k; ++r)
      if (fabs(N[r][c]) > fabs(N[piv][c])) piv = r;
    for (int j = 0; j <= k; ++j) {
      const double t = N[c][j];
      N[c][j] = N[piv][j];
      N[piv][j] = t;
    }
    const double d = N[c][c];
    if (d == 0.0) {
      for (int i = 0; i < k; ++i) x[i] = 0.0;
      return;
    }
    for (int r = 0; r < k; ++r) {
      if (r == c) continue;
      const double f = N[r][c] / d;
      for (int j = c; j <= k; ++j) N[r][j] -= f * N[c][j];
    }
  }
  for (int i = 0; i < k; ++i) x[i] = N[i][k] / N[i][i];
}

// The beta solve and pose recovery of EPNPEstimator::ComputePose (oracle/abs_pose.py compute_epnp) from the moments
// of the inlier set: V = the 4 smallest eigenvectors of M^T M, cw = control points, sa = sum alpha, saP = sum alpha P^T
// (4 x 3), sP = sum P, a0 = alpha of the first inlier.  cand: [3][12].
__device__ void epnp_candidates(const double (*V)[12], const double (*cw)[3], double n, const double* sa, const double* saP,
                                const double* sP, const double* a0, double (*cand)[12]) {
  const int pa[6] = {0, 0, 0, 1, 1, 2}, pb[6] = {1, 2, 3, 2, 3, 3};
  double L[6][10], rho[6];
  for (int k = 0; k < 6; ++k) {
    double d[4][3];
    for (int i = 0; i < 4; ++i)
      for (int c = 0; c < 3; ++c) d[i][c] = V[i][3 * pa[k] + c] - V[i][3 * pb[k] + c];
    auto dot = [&](int i, int j) { return d[i][0] * d[j][0] + d[i][1] * d[j][1] + d[i][2] * d[j][2]; };
    const double row[10] = {dot(0, 0), 2 * dot(0, 1), dot(1, 1), 2 * dot(0, 2), 2 * dot(1, 2), dot(2, 2),
                            2 * dot(0, 3), 2 * dot(1, 3), 2 * dot(2, 3), dot(3, 3)};
    for (int j = 0; j < 10; ++j) L[k][j] = row[j];
    double r = 0.0;
    for (int c = 0; c < 3; ++c) r += (cw[pa[k]][c] - cw[pb[k]][c]) * (cw[pa[k]][c] - cw[pb[k]][c]);
    rho[k] = r;
  }
  for (int ap = 0; ap < 3; ++ap) {
    double be[4] = {0, 0, 0, 0};
    if (ap == 0) {
      double A[24], b4[4];
      const int cols[4] = {0, 1, 3, 6};
      for (int k = 0; k < 6; ++k)
        for (int j = 0; j < 4; ++j) A[k * 4 + j] = L[k][cols[j]];
      lstsq_small(A, rho, 6, 4, b4);
      const double s = sqrt(fabs(b4[0])), sg = b4[0] < 0 ? -1.0 : 1.0;
      if (s > 0.0) {
        be[0] = s; be[1] = sg * b4[1] / s; be[2] = sg * b4[2] / s; be[3] = sg * b4[3] / s;
      }
    } else {
      const int k = ap == 1 ? 3 : 5;
      double A[30], bb[5];
      for (int r = 0; r < 6; ++r)
        for (int j = 0; j < k; ++j) A[r * k + j] = L[r][j];
      lstsq_small(A, rho, 6, k, bb);
      if (bb[0] < 0) {
        be[0] = sqrt(-bb[0]);
        be[1] = bb[2] < 0 ? sqrt(-bb[2]) : 0.0;
      } else {
        be[0] = sqrt(bb[0]);
        be[1] = bb[2] > 0 ? sqrt(bb[2]) : 0.0;
      }
      if (bb[1] < 0) be[0] = -be[0];
      if (ap == 2) be[2] = be[0] != 0.0 ? bb[3] / be[0] : 0.0;
    }
    for (int it = 0; it < 5; ++it) {  // Gauss-Newton on the betas
      double A[24], r[6], dx[4];
      for (int i = 0; i < 6; ++i) {
        const double* l = L[i];
        A[i * 4 + 0] = 2 * l[0] * be[0] + l[1] * be[1] + l[3] * be[2] + l[6] * be[3];
        A[i * 4 + 1] = l[1] * be[0] + 2 * l[2] * be[1] + l[4] * be[2] + l[7] * be[3];
        A[i * 4 + 2] = l[3] * be[0] + l[4] * be[1] + 2 * l[5] * be[2] + l[8] * be[3];
        A[i * 4 + 3] = l[6] * be[0] + l[7] * be[1] + l[8] * be[2] + 2 * l[9] * be[3];
        const double bb[10] = {be[0] * be[0], be[0] * be[1], be[1] * be[1], be[0] * be[2], be[1] * be[2],
                               be[2] * be[2], be[0] * be[3], be[1] * be[3], be[2] * be[3], be[3] * be[3]};
        double s = 0.0;
        for (int j = 0; j < 10; ++j) s += l[j] * bb[j];
        r[i] = rho[i] - s;
      }
      lstsq_small(A, r, 6, 4, dx);
      for (int j = 0; j < 4; ++j) be[j] += dx[j];
    }
    // control points in the camera frame, sign from the first inlier, then R, t by the Kabsch / Umeyama fit
    double cc[4][3];
    for (int j = 0; j < 4; ++j)
      for (int c = 0; c < 3; ++c) cc[j][c] = be[0] * V[0][3 * j + c] + be[1] * V[1][3 * j + c] + be[2] * V[2][3 * j + c] +
                                             be[3] * V[3][3 * j + c];
    double z0 = 0.0;
    for (int j = 0; j < 4; ++j) z0 += a0[j] * cc[j][2];
    if (z0 < 0)
      for (int j = 0; j < 4; ++j)
        for (int c = 0; c < 3; ++c) cc[j][c] = -cc[j][c];
    double pc0[3], pw0[3], abt[9];
    for (int c = 0; c < 3; ++c) {
      double s = 0.0;
      for (int j = 0; j < 4; ++j) s += sa[j] * cc[j][c];
      pc0[c] = s / n;
      pw0[c] = sP[c] / n;
    }
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) {
        double s = 0.0;
        for (int j = 0; j < 4; ++j) s += cc[j][a] * saP[j * 3 + b];
        abt[a * 3 + b] = s - n * pc0[a] * pw0[b];
      }
    double U[9], S[3], Vv[9], Rm[9];
    pose::svd3(abt, U, S, Vv);
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) Rm[a * 3 + b] = U[a * 3] * Vv[b * 3] + U[a * 3 + 1] * Vv[b * 3 + 1] + U[a * 3 + 2] * Vv[b * 3 + 2];
    for (int a = 0; a < 3; ++a) {
      cand[ap][4 * a] = Rm[3 * a]; cand[ap][4 * a + 1] = Rm[3 * a + 1]; cand[ap][4 * a + 2] = Rm[3 * a + 2];
      cand[ap][4 * a + 3] = pc0[a] - (Rm[3 * a] * pw0[0] + Rm[3 * a + 1] * pw0[1] + Rm[3 * a + 2] * pw0[2]);
    }
  }
}

// One EPnP refit on the inliers of sh.best_model (EPNPEstimator as the local estimator of LORANSAC).  Returns the
// candidate (the one of the three beta approximations with the least total reprojection error on the inliers) in
// sh.cand[0] and 1, or 0 when EPnP returns no model.
__device__ int epnp_refit(Shared& sh, const RansacParams& P, const double2* xn, int64_t off, const double* c, int n, double thr) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double M[12];
  for (int k = 0; k < 12; ++k) M[k] = sh.best_model[k];
  // pass 1: moments of the inlier world points, first inlier
  double mo[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  int first = INT32_MAX;
  for (int i = tid; i < n; i += kRansacThreads) {
    double u, v, X, Y, Z;
    load_point(P, xn, off, i, c, u, v, X, Y, Z);
    if (reproj_sq(M, u, v, X, Y, Z) <= thr) {
      if (first == INT32_MAX) first = i;
      mo[0] += 1.0; mo[1] += X; mo[2] += Y; mo[3] += Z;
      mo[4] += X * X; mo[5] += X * Y; mo[6] += X * Z; mo[7] += Y * Y; mo[8] += Y * Z; mo[9] += Z * Z;
    }
  }
  first = __reduce_min_sync(0xffffffffu, first);
  for (int k = 0; k < 10; ++k) {
    const double s = warp_sum_d(mo[k]);
    if (lane == 0) sh.red[warp][k] = s;
  }
  if (lane == 0) sh.round.scan[warp] = first;
  __syncthreads();
  if (tid == 0) {
    for (int k = 0; k < 10; ++k) sh.mom[k] = sh.red[0][k] + sh.red[1][k] + sh.red[2][k] + sh.red[3][k];
    sh.first = min(min(sh.round.scan[0], sh.round.scan[1]), min(sh.round.scan[2], sh.round.scan[3]));
    const double nn = sh.mom[0];
    const double c0[3] = {sh.mom[1] / nn, sh.mom[2] / nn, sh.mom[3] / nn};
    double A[9] = {sh.mom[4] - nn * c0[0] * c0[0], sh.mom[5] - nn * c0[0] * c0[1], sh.mom[6] - nn * c0[0] * c0[2], 0, 0, 0, 0, 0, 0};
    A[4] = sh.mom[7] - nn * c0[1] * c0[1];
    A[5] = sh.mom[8] - nn * c0[1] * c0[2];
    A[8] = sh.mom[9] - nn * c0[2] * c0[2];
    A[3] = A[1]; A[6] = A[2]; A[7] = A[5];
    double Vv[9], w[3];
    jacobi_eig_sym<3>(A, Vv, w);
    int o[3] = {0, 1, 2};  // eigenvalues descending (the singular values of PW0^T PW0)
    for (int i = 0; i < 3; ++i)
      for (int j = i + 1; j < 3; ++j)
        if (w[o[j]] > w[o[i]]) {
          const int t = o[i]; o[i] = o[j]; o[j] = t;
        }
    for (int k = 0; k < 3; ++k) sh.cw[0][k] = c0[k];
    for (int i = 0; i < 3; ++i) {
      const double s = sqrt(fmax(w[o[i]], 0.0) / nn);
      for (int k = 0; k < 3; ++k) sh.cw[i + 1][k] = c0[k] + s * Vv[k * 3 + o[i]];
    }
    double C[9];  // columns cw[j] - cw[0]
    for (int r = 0; r < 3; ++r)
      for (int j = 0; j < 3; ++j) C[r * 3 + j] = sh.cw[j + 1][r] - sh.cw[0][r];
    const double det = pose::det3(C);
    const double sc = fmax(fmax(fabs(w[o[0]]), 1e-300) / nn, 1e-300);
    sh.lo_ok = fabs(det) > 1e-10 * sc * sqrt(sc) ? 1 : 0;
    if (sh.lo_ok) {
      const double id = 1.0 / det;
      sh.ccinv[0] = (C[4] * C[8] - C[5] * C[7]) * id;
      sh.ccinv[1] = (C[2] * C[7] - C[1] * C[8]) * id;
      sh.ccinv[2] = (C[1] * C[5] - C[2] * C[4]) * id;
      sh.ccinv[3] = (C[5] * C[6] - C[3] * C[8]) * id;
      sh.ccinv[4] = (C[0] * C[8] - C[2] * C[6]) * id;
      sh.ccinv[5] = (C[2] * C[3] - C[0] * C[5]) * id;
      sh.ccinv[6] = (C[3] * C[7] - C[4] * C[6]) * id;
      sh.ccinv[7] = (C[1] * C[6] - C[0] * C[7]) * id;
      sh.ccinv[8] = (C[0] * C[4] - C[1] * C[3]) * id;
    }
  }
  __syncthreads();
  if (!sh.lo_ok) return 0;
  // pass 2: M^T M = sum_i (alpha_i alpha_i^T) (x) [[1, 0, -u], [0, 1, -v], [-u, -v, u^2 + v^2]]: 4 x 10 sums
  double s40[40];
#pragma unroll
  for (int k = 0; k < 40; ++k) s40[k] = 0.0;
  double Ci[9], c0[3];
  for (int k = 0; k < 9; ++k) Ci[k] = sh.ccinv[k];
  for (int k = 0; k < 3; ++k) c0[k] = sh.cw[0][k];
  for (int i = tid; i < n; i += kRansacThreads) {
    double u, v, X, Y, Z;
    load_point(P, xn, off, i, c, u, v, X, Y, Z);
    if (reproj_sq(M, u, v, X, Y, Z) <= thr) {
      const double d[3] = {X - c0[0], Y - c0[1], Z - c0[2]};
      double al[4];
      al[1] = Ci[0] * d[0] + Ci[1] * d[1] + Ci[2] * d[2];
      al[2] = Ci[3] * d[0] + Ci[4] * d[1] + Ci[5] * d[2];
      al[3] = Ci[6] * d[0] + Ci[7] * d[1] + Ci[8] * d[2];
      al[0] = 1.0 - al[1] - al[2] - al[3];
      const double w2 = u * u + v * v;
      int e = 0;
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = a; b < 4; ++b, ++e) {
          const double aa = al[a] * al[b];
          s40[e] += aa;
          s40[10 + e] += aa * u;
          s40[20 + e] += aa * v;
          s40[30 + e] += aa * w2;
        }
    }
  }
#pragma unroll
  for (int k = 0; k < 40; ++k) {
    const double s = warp_sum_d(s40[k]);
    if (lane == 0) sh.red[warp][k] = s;
  }
  __syncthreads();
  if (tid < 78) {  // packed upper triangle of the 12 x 12 matrix, entry (r, q), r <= q
    int r = 0, rem = tid;
    while (rem >= 12 - r) {
      rem -= 12 - r;
      ++r;
    }
    const int q = r + rem;
    const int a = r / 3, ra = r % 3, b = q / 3, rb = q % 3;
    const int lo = a < b ? a : b, hi = a < b ? b : a;
    const int e = lo * 4 - lo * (lo - 1) / 2 + (hi - lo);
    auto S = [&](int base) { return sh.red[0][base + e] + sh.red[1][base + e] + sh.red[2][base + e] + sh.red[3][base + e]; };
    double val;
    if (ra == 2 && rb == 2) val = S(30);
    else if (ra == 2 || rb == 2) {
      const int other = ra == 2 ? rb : ra;
      val = -S(other == 0 ? 10 : 20);
    } else {
      val = ra == rb ? S(0) : 0.0;
    }
    sh.mtm[tid] = val;
  }
  __syncthreads();
  if (warp == 0) eigw::smallest_eigvecs_warp<4, 12, 12>(sh.mtm, &sh.eigv[0][0], sh.es, lane);
  __syncthreads();
  if (tid == 0) {
    // sums the beta solve needs, all from the moments: sum alpha_j (= sum_k sum alpha_j alpha_k) and sum alpha_j P^T
    double sa[4] = {0, 0, 0, 0}, saP[12], sP[3] = {sh.mom[1], sh.mom[2], sh.mom[3]};
    for (int a = 0; a < 4; ++a)
      for (int b = 0; b < 4; ++b) {
        const int lo = a < b ? a : b, hi = a < b ? b : a;
        const int e = lo * 4 - lo * (lo - 1) / 2 + (hi - lo);
        sa[a] += sh.red[0][e] + sh.red[1][e] + sh.red[2][e] + sh.red[3][e];
      }
    const double nn = sh.mom[0];
    // sum (P - cw0) P^T, then alpha_{1..3} = Ci (P - cw0) and alpha_0 = 1 - the others
    const double SPP[9] = {sh.mom[4], sh.mom[5], sh.mom[6], sh.mom[5], sh.mom[7], sh.mom[8], sh.mom[6], sh.mom[8], sh.mom[9]};
    double D[9];
    for (int r = 0; r < 3; ++r)
      for (int q = 0; q < 3; ++q) D[r * 3 + q] = SPP[r * 3 + q] - sh.cw[0][r] * sP[q];
    for (int j = 1; j < 4; ++j)
      for (int q = 0; q < 3; ++q)
        saP[j * 3 + q] = sh.ccinv[(j - 1) * 3] * D[q] + sh.ccinv[(j - 1) * 3 + 1] * D[3 + q] + sh.ccinv[(j - 1) * 3 + 2] * D[6 + q];
    for (int q = 0; q < 3; ++q) saP[q] = sP[q] - saP[3 + q] - saP[6 + q] - saP[9 + q];
    double u, v, X, Y, Z, a0[4];
    load_point(P, xn, off, sh.first, c, u, v, X, Y, Z);
    const double d[3] = {X - sh.cw[0][0], Y - sh.cw[0][1], Z - sh.cw[0][2]};
    a0[1] = sh.ccinv[0] * d[0] + sh.ccinv[1] * d[1] + sh.ccinv[2] * d[2];
    a0[2] = sh.ccinv[3] * d[0] + sh.ccinv[4] * d[1] + sh.ccinv[5] * d[2];
    a0[3] = sh.ccinv[6] * d[0] + sh.ccinv[7] * d[1] + sh.ccinv[8] * d[2];
    a0[0] = 1.0 - a0[1] - a0[2] - a0[3];
    epnp_candidates(sh.eigv, sh.cw, nn, sa, saP, sP, a0, sh.cand);
  }
  __syncthreads();
  // pass 3: total reprojection error (sum of sqrt) of the three candidates on the inlier set
  double e3[3] = {0, 0, 0};
  for (int i = tid; i < n; i += kRansacThreads) {
    double u, v, X, Y, Z;
    load_point(P, xn, off, i, c, u, v, X, Y, Z);
    if (reproj_sq(M, u, v, X, Y, Z) <= thr)
      for (int k = 0; k < 3; ++k) e3[k] += sqrt(reproj_sq(sh.cand[k], u, v, X, Y, Z));
  }
  for (int k = 0; k < 3; ++k) {
    const double s = warp_sum_d(e3[k]);
    if (lane == 0) sh.red[warp][k] = s;
  }
  __syncthreads();
  if (tid == 0) {
    int w = -1;
    double best = INFINITY;
    for (int k = 0; k < 3; ++k) {
      const double err = sh.red[0][k] + sh.red[1][k] + sh.red[2][k] + sh.red[3][k];
      bool finite = true;
      for (int j = 0; j < 12; ++j) finite = finite && isfinite(sh.cand[k][j]);
      if (finite && err < best) {
        best = err;
        w = k;
      }
    }
    sh.n_cand = w >= 0 ? 1 : 0;
    if (w > 0)
      for (int j = 0; j < 12; ++j) sh.cand[0][j] = sh.cand[w][j];
  }
  __syncthreads();
  return sh.n_cand;
}

__global__ void __launch_bounds__(kRansacThreads, 3) b2m_abs_ransac_kernel(const RansacParams P) {
  __shared__ Shared sh;
  const int tid = threadIdx.x;
  const int cta = blockIdx.x;
  const int prob = cta / P.n_factors, fs = cta % P.n_factors;
  const int n = P.cnt[prob];
  const int64_t off = P.off[prob];
  double2* xn = P.xn + P.xoff[cta];
  uint8_t* mask = P.mask + P.xoff[cta];
  DevCam cm = P.cams[prob];
  const double fac = P.factors[fs];
  cm.p[0] *= fac;
  if (!cam::single_focal(cm.model)) cm.p[1] *= fac;
  for (int i = tid; i < n; i += kRansacThreads) {
    double u, v;
    cam::cam_from_img(cm.model, cm.p, P.px[2 * (off + i)], P.px[2 * (off + i) + 1], &u, &v);
    xn[i] = make_double2(u, v);
  }
  const double e = P.ro.max_error / cam::mean_focal_length(cm.model, cm.p);  // CamFromImgThreshold
  const double thr = e * e;
  const double c[3] = {P.centroid[3 * prob], P.centroid[3 * prob + 1], P.centroid[3 * prob + 2]};
  __syncthreads();
  if (n < 3) {
    for (int i = tid; i < n; i += kRansacThreads) mask[i] = 0;
    if (tid == 0) {
      P.sup[cta] = 0;
      P.success[cta] = 0;
      for (int k = 0; k < 12; ++k) P.models[12 * cta + k] = 0.0;
    }
    return;
  }
  const b2m_ransac_opts& ro = P.ro;
  const uint64_t key = splitmix64(P.seed ^ splitmix64((static_cast<uint64_t>(P.problem_base + prob) << 8) ^
                                                      static_cast<uint64_t>(fs) ^ 0x5A00000000000000ull));
  const int max_trials = static_cast<int>(ransac_trial_cap(ro, 3));
  const ReprojModel model{P, xn, off, c};
  double dyn_max = max_trials;
  if (tid == 0) {
    sh.best_cnt = 0;
    sh.best_sum = 1e300;
    for (int k = 0; k < 12; ++k) sh.best_model[k] = 0.0;
  }
  __syncthreads();
  int trials = 0;
  unsigned long long n_scored = 0;
  double mdl[4 * 12];
  while (trials < max_trials) {
    const int nb = round_size(trials, max_trials, ro.min_num_trials, dyn_max);
    // ---- one P3P hypothesis per thread
    int nm = 0;
    if (tid < nb) {
      int idx[3];
      draw_sample<3>(key, trials + tid, n, idx);
      double x[3], y[3], W[9];
      for (int j = 0; j < 3; ++j) load_point(P, xn, off, idx[j], c, x[j], y[j], W[3 * j], W[3 * j + 1], W[3 * j + 2]);
      nm = p3p(x, y, W, mdl);
    }
    // ---- score every model of the round: chunks in shared memory, fp32 with fp64 rechecks, exact pruning
    const RoundResult round = score_round(sh.round, model, mdl, nm, nb, n, thr, sh.best_cnt);
    n_scored += round.n_models;
    if (round.winner >= 0) {
      if (tid == round.winner)
        for (int k = 0; k < 12; ++k) sh.best_model[k] = mdl[round.model * 12 + k];
      __syncthreads();
      int bc;
      double bs;
      exact_support(sh.round, model, sh.best_model, n, thr, bc, bs);
      if (tid == 0) {
        sh.best_cnt = bc;
        sh.best_sum = bs;
      }
      __syncthreads();
      n_scored += 1;
      // ---- recursive local optimisation: EPnP on the inliers of the current best
      if (sh.best_cnt > 3 && sh.best_cnt >= 4) {
        for (int lt = 0; lt < kMaxLocalTrials; ++lt) {
          const int prev_best = sh.best_cnt;
          const int nc = epnp_refit(sh, P, xn, off, c, n, thr);
          n_scored += 2 + 3 * nc;  // the moment passes and the three candidates on the inliers
          if (!nc) break;
          int cc;
          double cs;
          exact_support(sh.round, model, sh.cand[0], n, thr, cc, cs);
          n_scored += 1;
          if (tid == 0 && (cc > sh.best_cnt || (cc == sh.best_cnt && cs < sh.best_sum))) {
            sh.best_cnt = cc;
            sh.best_sum = cs;
            for (int k = 0; k < 12; ++k) sh.best_model[k] = sh.cand[0][k];
          }
          __syncthreads();
          if (sh.best_cnt <= prev_best) break;
        }
      }
      dyn_max = compute_num_trials(sh.best_cnt, n, ro.confidence, ro.dyn_num_trials_multiplier, 3);
    }
    trials += nb;
    __syncthreads();
    if (trials >= dyn_max && trials >= ro.min_num_trials) break;
  }
  double M[12];
  for (int k = 0; k < 12; ++k) M[k] = sh.best_model[k];
  const bool ok = sh.best_cnt >= 3;
  for (int i = tid; i < n; i += kRansacThreads) {
    double u, v, X, Y, Z;
    load_point(P, xn, off, i, c, u, v, X, Y, Z);
    mask[i] = (ok && reproj_sq(M, u, v, X, Y, Z) <= thr) ? 1 : 0;
  }
  if (P.counters && tid == 0) {
    atomicAdd(P.counters, n_scored + 1);
    atomicAdd(P.counters + 1, (n_scored + 1) * static_cast<unsigned long long>(n));
  }
  if (tid == 0) {
    P.sup[cta] = sh.best_cnt;
    P.success[cta] = ok ? 1 : 0;
    for (int k = 0; k < 12; ++k) P.models[12 * cta + k] = M[k];
  }
}

// ---- focal sample selection -------------------------------------------------------------------------------
struct SelectParams {
  const int64_t* off;
  const int32_t* cnt;
  const int64_t* xoff;
  const uint8_t* cta_mask;
  const double* models;
  const int32_t* sup;
  const int32_t* success;
  const double* centroid;
  const double* factors;
  int32_t n_factors;
  int32_t estimate_focal_length;
  const DevCam* cams;
  uint8_t* mask;             // [total] output inlier masks
  double* pose;              // [nb][7] qvec (w, x, y, z), tvec
  double* params;            // [nb][12]
  int32_t* out_success;      // [nb]
  int32_t* out_inliers;      // [nb]
  int32_t* out_factor;       // [nb]
};

__device__ void rotation_to_quat(const double* R, double* q) {  // (w, x, y, z), Eigen's branch selection
  const double tr = R[0] + R[4] + R[8];
  if (tr > 0.0) {
    double s = sqrt(tr + 1.0);
    q[0] = 0.5 * s;
    s = 0.5 / s;
    q[1] = (R[7] - R[5]) * s; q[2] = (R[2] - R[6]) * s; q[3] = (R[3] - R[1]) * s;
  } else {
    int i = 0;
    if (R[4] > R[0]) i = 1;
    if (R[8] > R[i * 4]) i = 2;
    const int j = (i + 1) % 3, k = (i + 2) % 3;
    double s = sqrt(R[i * 4] - R[j * 4] - R[k * 4] + 1.0);
    q[1 + i] = 0.5 * s;
    s = 0.5 / s;
    q[0] = (R[k * 3 + j] - R[j * 3 + k]) * s;
    q[1 + j] = (R[j * 3 + i] + R[i * 3 + j]) * s;
    q[1 + k] = (R[k * 3 + i] + R[i * 3 + k]) * s;
  }
}

__device__ void quat_to_rotation(const double* q0, double* R) {
  const double nq = sqrt(q0[0] * q0[0] + q0[1] * q0[1] + q0[2] * q0[2] + q0[3] * q0[3]);
  const double w = q0[0] / nq, x = q0[1] / nq, y = q0[2] / nq, z = q0[3] / nq;
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - w * z); R[2] = 2 * (x * z + w * y);
  R[3] = 2 * (x * y + w * z); R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - w * x);
  R[6] = 2 * (x * z - w * y); R[7] = 2 * (y * z + w * x); R[8] = 1 - 2 * (x * x + y * y);
}

__global__ void __launch_bounds__(32) b2m_abs_select_kernel(const SelectParams S) {
  const int prob = blockIdx.x, lane = threadIdx.x;
  const int n = S.cnt[prob];
  const int64_t off = S.off[prob];
  int best = 0, bs = -1;
  for (int f = 0; f < S.n_factors; ++f) {
    const int cta = prob * S.n_factors + f;
    if (S.success[cta] && S.sup[cta] > best) {
      best = S.sup[cta];
      bs = f;
    }
  }
  DevCam cm = S.cams[prob];
  if (bs >= 0 && S.estimate_focal_length) {
    cm.p[0] *= S.factors[bs];
    if (!cam::single_focal(cm.model)) cm.p[1] *= S.factors[bs];
  }
  const uint8_t* src = bs >= 0 ? S.cta_mask + S.xoff[prob * S.n_factors + bs] : nullptr;
  for (int i = lane; i < n; i += 32) S.mask[off + i] = src ? src[i] : 0;
  if (lane != 0) return;
  for (int k = 0; k < cam::kMaxParams; ++k) S.params[12 * prob + k] = cm.p[k];
  double* pz = S.pose + 7 * prob;
  pz[0] = 1.0;
  for (int k = 1; k < 7; ++k) pz[k] = 0.0;
  S.out_inliers[prob] = best;
  S.out_factor[prob] = bs;
  if (bs < 0) {
    S.out_success[prob] = 0;
    return;
  }
  const double* M = S.models + 12 * (prob * S.n_factors + bs);
  const double* c = S.centroid + 3 * prob;
  double R[9], t[3];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) R[i * 3 + j] = M[4 * i + j];
    t[i] = M[4 * i + 3] - (R[i * 3] * c[0] + R[i * 3 + 1] * c[1] + R[i * 3 + 2] * c[2]);  // centred -> world frame
  }
  rotation_to_quat(R, pz);
  for (int k = 0; k < 3; ++k) pz[4 + k] = t[k];
  S.out_success[prob] = !(isnan(t[0]) || isnan(t[1]) || isnan(t[2]));
}

// ---- refinement ---------------------------------------------------------------------------------------------
struct RefineParams {
  const double* px;
  const double* p3;
  const int64_t* off;
  const int32_t* cnt;
  const int32_t* model;      // [nb] camera model ids
  const uint8_t* mask;       // [total]
  double* pose;              // [nb][7] in / out
  double* params;            // [nb][12] in / out
  int32_t* success;          // [nb] in (0: skip) / out
  double* cov;               // [nb][36] or nullptr
  double gradient_tolerance;
  double loss_scale;
  int32_t max_num_iterations;
  int32_t refine_focal;
  int32_t refine_extra;
  int32_t pad;
};

struct RefineShared {
  double J[32][2][kMaxRefine + 1];   // per lane: the two loss-corrected Jacobian rows and residuals
  double A[kMaxRefine * kMaxRefine];
  double g[kMaxRefine];
  double sums[kMaxRefine * (kMaxRefine + 1) / 2 + kMaxRefine];
  double step[kMaxRefine];
  double q[4], t[3], p[cam::kMaxParams];
  double qn[4], tn[3], pn[cam::kMaxParams];
  double cost;
  int ridx[10];
  int flag;
};

// Loss-corrected residuals / Jacobian rows of the inlier observations, reduced to J^T J (packed) and J^T r (sums) and
// the robust cost 1/2 sum rho(|r|^2).  want_j = false: cost only.  Warp-wide; returns the cost on every lane.
__device__ double evaluate(RefineShared& sh, const RefineParams& P, int prob, const double* q, const double* t,
                           const double* p, int np, int k, bool want_j, int lane) {
  const int n = P.cnt[prob];
  const int64_t off = P.off[prob];
  const int model = P.model[prob];
  const double a2 = P.loss_scale * P.loss_scale;
  double R[9];
  quat_to_rotation(q, R);
  const int n_sums = np * (np + 1) / 2 + np;
  double acc[6] = {0, 0, 0, 0, 0, 0};   // this lane's share of sums[] (entries lane, lane + 32, ...)
  double cost = 0.0;
  for (int base = 0; base < n; base += 32) {
    const int i = base + lane;
    bool use = i < n && P.mask[off + i];
    double r0 = 0, r1 = 0, w = 0;
    ad::Dual x, y;
    if (use) {
      const double* X = P.p3 + 3 * (off + i);
      double RX[3];
      for (int a = 0; a < 3; ++a) RX[a] = R[a * 3] * X[0] + R[a * 3 + 1] * X[1] + R[a * 3 + 2] * X[2];
      const double Xc[3] = {RX[0] + t[0], RX[1] + t[1], RX[2] + t[2]};
      const double u = Xc[0] / Xc[2], v = Xc[1] / Xc[2];
      ad::Dual U(u), V(v), Pd[cam::kMaxParams];
      U.d[0] = 1.0;
      V.d[1] = 1.0;
      for (int j = 0; j < cam::kMaxParams; ++j) Pd[j] = ad::Dual(p[j]);
      if (want_j)
        for (int j = 0; j < k; ++j) Pd[sh.ridx[j]].d[2 + j] = 1.0;
      cam::img_from_cam(model, Pd, U, V, &x, &y);
      r0 = x.v - P.px[2 * (off + i)];
      r1 = y.v - P.px[2 * (off + i) + 1];
      const double s = r0 * r0 + r1 * r1;
      cost += 0.5 * a2 * log1p(s / a2);
      w = sqrt(1.0 / (1.0 + s / a2));   // sqrt(rho') of the Cauchy loss (Ceres' corrector, rho'' < 0)
      if (want_j) {
        const double iz = 1.0 / Xc[2];
        const double duv[2][3] = {{iz, 0.0, -u * iz}, {0.0, iz, -v * iz}};
        const double dpx[2][2] = {{x.d[0], x.d[1]}, {y.d[0], y.d[1]}};
        // d Xc / d delta_rot = -2 [R X]_x (Ceres' quaternion manifold: rotation by 2 |delta|)
        const double sk[3][3] = {{0.0, 2 * RX[2], -2 * RX[1]}, {-2 * RX[2], 0.0, 2 * RX[0]}, {2 * RX[1], -2 * RX[0], 0.0}};
        for (int rr = 0; rr < 2; ++rr) {
          double dX[3];
          for (int a = 0; a < 3; ++a) dX[a] = dpx[rr][0] * duv[0][a] + dpx[rr][1] * duv[1][a];
          for (int a = 0; a < 3; ++a) sh.J[lane][rr][a] = w * (dX[0] * sk[0][a] + dX[1] * sk[1][a] + dX[2] * sk[2][a]);
          for (int a = 0; a < 3; ++a) sh.J[lane][rr][3 + a] = w * dX[a];
          const ad::Dual& src = rr == 0 ? x : y;
          for (int j = 0; j < k; ++j) sh.J[lane][rr][6 + j] = w * src.d[2 + j];
        }
        sh.J[lane][0][np] = w * r0;
        sh.J[lane][1][np] = w * r1;
      }
    }
    if (want_j) {
      if (!use)
        for (int rr = 0; rr < 2; ++rr)
          for (int a = 0; a <= np; ++a) sh.J[lane][rr][a] = 0.0;
      __syncwarp();
      const int cnt = min(32, n - base);
      for (int s = 0; s < 6; ++s) {
        const int e = lane + 32 * s;
        if (e >= n_sums) break;
        int a, b;  // entry e: packed (a <= b) of J^T J, then J^T r
        if (e < np * (np + 1) / 2) {
          a = 0;
          int rem = e;
          while (rem >= np - a) {
            rem -= np - a;
            ++a;
          }
          b = a + rem;
        } else {
          a = e - np * (np + 1) / 2;
          b = np;
        }
        double sum = acc[s];
        for (int l = 0; l < cnt; ++l) sum += sh.J[l][0][a] * sh.J[l][0][b] + sh.J[l][1][a] * sh.J[l][1][b];
        acc[s] = sum;
      }
      __syncwarp();
    }
  }
  if (want_j) {
    for (int s = 0; s < 6; ++s) {
      const int e = lane + 32 * s;
      if (e < n_sums) sh.sums[e] = acc[s];
    }
  }
  cost = warp_sum_d(cost);
  __syncwarp();
  return cost;
}

// Cholesky solve of the np x np system A x = b in place (lane 0).  false when A is not positive definite.
__device__ bool chol_solve(double* A, int np, double* b) {
  for (int j = 0; j < np; ++j) {
    double d = A[j * np + j];
    for (int k = 0; k < j; ++k) d -= A[j * np + k] * A[j * np + k];
    if (!(d > 0.0)) return false;
    const double l = sqrt(d);
    A[j * np + j] = l;
    for (int i = j + 1; i < np; ++i) {
      double s = A[i * np + j];
      for (int k = 0; k < j; ++k) s -= A[i * np + k] * A[j * np + k];
      A[i * np + j] = s / l;
    }
  }
  for (int i = 0; i < np; ++i) {
    double s = b[i];
    for (int k = 0; k < i; ++k) s -= A[i * np + k] * b[k];
    b[i] = s / A[i * np + i];
  }
  for (int i = np - 1; i >= 0; --i) {
    double s = b[i];
    for (int k = i + 1; k < np; ++k) s -= A[k * np + i] * b[k];
    b[i] = s / A[i * np + i];
  }
  return true;
}

__device__ void unpack(const RefineShared& sh, int np, double* A, double* g) {
  int e = 0;
  for (int a = 0; a < np; ++a)
    for (int b = a; b < np; ++b, ++e) A[a * np + b] = A[b * np + a] = sh.sums[e];
  for (int a = 0; a < np; ++a) g[a] = sh.sums[e + a];
}

// RefineAbsolutePose as restated in oracle/abs_pose.py refine_absolute_pose (Ceres LM): one warp per problem.
__global__ void __launch_bounds__(32) b2m_abs_refine_kernel(const RefineParams P) {
  __shared__ RefineShared sh;
  const int prob = blockIdx.x, lane = threadIdx.x;
  if (!P.success[prob]) return;
  const int model = P.model[prob];
  if (lane == 0) {
    const double* pz = P.pose + 7 * prob;
    const double nq = sqrt(pz[0] * pz[0] + pz[1] * pz[1] + pz[2] * pz[2] + pz[3] * pz[3]);
    for (int j = 0; j < 4; ++j) sh.q[j] = pz[j] / nq;
    for (int j = 0; j < 3; ++j) sh.t[j] = pz[4 + j];
    for (int j = 0; j < cam::kMaxParams; ++j) sh.p[j] = P.params[12 * prob + j];
    int k = 0;
    const int nfoc = cam::single_focal(model) ? 1 : 2, first_extra = cam::single_focal(model) ? 3 : 4;
    if (P.refine_focal)
      for (int j = 0; j < nfoc; ++j) sh.ridx[k++] = j;
    if (P.refine_extra)
      for (int j = first_extra; j < cam::num_params(model); ++j) sh.ridx[k++] = j;
    sh.flag = k;
  }
  __syncwarp();
  const int k = sh.flag, np = 6 + k;
  double cost = evaluate(sh, P, prob, sh.q, sh.t, sh.p, np, k, true, lane);
  int ok = isfinite(cost) ? 1 : 0;
  double radius = 1e4, decrease = 2.0;
  int it = 0;
  bool any = false;
  for (int i = lane; i < P.cnt[prob]; i += 32) any = any || P.mask[P.off[prob] + i];
  any = __any_sync(0xffffffffu, any);
  while (ok && any) {
    // lane 0 decides; the decision is broadcast through sh.flag (0 continue, 1 stop, 2 trial step)
    if (lane == 0) {
      double A[kMaxRefine * kMaxRefine], g[kMaxRefine], scale[kMaxRefine], x[kMaxRefine];
      unpack(sh, np, A, g);
      double gmax = 0.0;
      for (int a = 0; a < np; ++a) gmax = fmax(gmax, fabs(g[a]));
      sh.flag = 1;
      if (!(gmax <= P.gradient_tolerance) && it < P.max_num_iterations) {
        ++it;
        for (int a = 0; a < np; ++a) scale[a] = 1.0 / (1.0 + sqrt(A[a * np + a]));
        double As[kMaxRefine * kMaxRefine];
        for (int a = 0; a < np; ++a)
          for (int b = 0; b < np; ++b) As[a * np + b] = A[a * np + b] * scale[a] * scale[b];
        double gs[kMaxRefine];
        for (int a = 0; a < np; ++a) gs[a] = g[a] * scale[a];
        for (int a = 0; a < np; ++a) x[a] = -gs[a];
        for (int a = 0; a < np * np; ++a) sh.A[a] = As[a];
        for (int a = 0; a < np; ++a) sh.A[a * np + a] += fmin(fmax(As[a * np + a], 1e-6), 1e32) / radius;
        if (chol_solve(sh.A, np, x)) {
          double gx = 0.0, xAx = 0.0, sn = 0.0;
          for (int a = 0; a < np; ++a) {
            gx += gs[a] * x[a];
            double s = 0.0;
            for (int b = 0; b < np; ++b) s += As[a * np + b] * x[b];
            xAx += x[a] * s;
            sh.step[a] = x[a] * scale[a];
            sn += sh.step[a] * sh.step[a];
          }
          sh.g[0] = -(gx + 0.5 * xAx);   // model cost change
          double xn = 0.0;
          for (int j = 0; j < 4; ++j) xn += sh.q[j] * sh.q[j];
          for (int j = 0; j < 3; ++j) xn += sh.t[j] * sh.t[j];
          for (int j = 0; j < k; ++j) xn += sh.p[sh.ridx[j]] * sh.p[sh.ridx[j]];
          if (sqrt(sn) > 1e-8 * (sqrt(xn) + 1e-8)) {
            // candidate: q <- (cos|d|, sin|d| d / |d|) * q, t += dt, p += dp
            const double* d = sh.step;
            const double nd = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
            double dq[4] = {1.0, 0.0, 0.0, 0.0};
            if (nd > 0.0) {
              dq[0] = cos(nd);
              for (int j = 0; j < 3; ++j) dq[1 + j] = sin(nd) / nd * d[j];
            }
            const double* q = sh.q;
            sh.qn[0] = dq[0] * q[0] - dq[1] * q[1] - dq[2] * q[2] - dq[3] * q[3];
            sh.qn[1] = dq[0] * q[1] + dq[1] * q[0] + dq[2] * q[3] - dq[3] * q[2];
            sh.qn[2] = dq[0] * q[2] - dq[1] * q[3] + dq[2] * q[0] + dq[3] * q[1];
            sh.qn[3] = dq[0] * q[3] + dq[1] * q[2] - dq[2] * q[1] + dq[3] * q[0];
            for (int j = 0; j < 3; ++j) sh.tn[j] = sh.t[j] + d[3 + j];
            for (int j = 0; j < cam::kMaxParams; ++j) sh.pn[j] = sh.p[j];
            for (int j = 0; j < k; ++j) sh.pn[sh.ridx[j]] += d[6 + j];
            sh.flag = 2;
          }
        } else {
          sh.flag = 3;   // not positive definite: shrink the trust region
        }
      }
    }
    __syncwarp();
    const int flag = sh.flag;
    if (flag == 1) break;
    if (flag == 3) {
      radius /= decrease;
      decrease *= 2.0;
      if (radius < 1e-32) break;
      continue;
    }
    const double cn = evaluate(sh, P, prob, sh.qn, sh.tn, sh.pn, np, k, false, lane);
    const double ratio = sh.g[0] > 0.0 ? (cost - cn) / sh.g[0] : -1.0;
    if (isfinite(cn) && ratio > 1e-3) {
      const bool done = fabs(cost - cn) <= 1e-6 * cost;
      __syncwarp();
      if (lane == 0) {
        for (int j = 0; j < 4; ++j) sh.q[j] = sh.qn[j];
        for (int j = 0; j < 3; ++j) sh.t[j] = sh.tn[j];
        for (int j = 0; j < cam::kMaxParams; ++j) sh.p[j] = sh.pn[j];
      }
      __syncwarp();
      cost = cn;
      const double tt = 2.0 * ratio - 1.0;
      radius = fmin(1e16, radius / fmax(1.0 / 3.0, 1.0 - tt * tt * tt));
      decrease = 2.0;
      evaluate(sh, P, prob, sh.q, sh.t, sh.p, np, k, true, lane);
      if (done) break;
    } else {
      radius /= decrease;
      decrease *= 2.0;
      if (radius < 1e-32) break;
    }
  }
  if (P.cov && ok) {
    evaluate(sh, P, prob, sh.q, sh.t, sh.p, np, k, true, lane);
    if (lane == 0) {
      // 6 x 6 block of (J^T J)^-1: solve for the first six unit vectors
      double A[kMaxRefine * kMaxRefine], g[kMaxRefine];
      unpack(sh, np, A, g);
      double* out = P.cov + 36 * prob;
      for (int col = 0; col < 6 && ok; ++col) {
        double e[kMaxRefine];
        for (int a = 0; a < np; ++a) e[a] = a == col ? 1.0 : 0.0;
        for (int a = 0; a < np * np; ++a) sh.A[a] = A[a];
        if (!chol_solve(sh.A, np, e)) ok = 0;
        for (int a = 0; a < 6; ++a) out[a * 6 + col] = e[a];
      }
    }
    ok = __shfl_sync(0xffffffffu, ok, 0);
  }
  if (lane == 0) {
    double* pz = P.pose + 7 * prob;
    for (int j = 0; j < 4; ++j) pz[j] = sh.q[j];
    for (int j = 0; j < 3; ++j) pz[4 + j] = sh.t[j];
    for (int j = 0; j < cam::kMaxParams; ++j) P.params[12 * prob + j] = sh.p[j];
    P.success[prob] = ok;
  }
}

// Packed host copies of a chunk [k0, k0 + nb) of the problems.
struct Packed {
  std::vector<double> px, p3, centroid;
  std::vector<int64_t> off;
  std::vector<int32_t> cnt, model;
  std::vector<DevCam> cams;
  int64_t total = 0;
};

void pack(const b2m_abs_pose_problem* q, int nb, Packed* out) {
  out->off.resize(nb);
  out->cnt.resize(nb);
  out->model.resize(nb);
  out->cams.resize(nb);
  out->centroid.assign(3 * static_cast<size_t>(nb), 0.0);
  int64_t total = 0;
  for (int k = 0; k < nb; ++k) total += q[k].n;
  out->px.resize(2 * static_cast<size_t>(total));
  out->p3.resize(3 * static_cast<size_t>(total));
  int64_t pos = 0;
  for (int k = 0; k < nb; ++k) {
    const int64_t n = q[k].n;
    out->off[k] = pos;
    out->cnt[k] = static_cast<int32_t>(n);
    out->model[k] = q[k].camera.model;
    DevCam d{};
    d.model = q[k].camera.model;
    for (int j = 0; j < cam::kMaxParams; ++j) d.p[j] = q[k].camera.params[j];
    out->cams[k] = d;
    if (n > 0) {
      memcpy(out->px.data() + 2 * pos, q[k].points2D, sizeof(double) * 2 * n);
      memcpy(out->p3.data() + 3 * pos, q[k].points3D, sizeof(double) * 3 * n);
      double s[3] = {0, 0, 0};
      for (int64_t i = 0; i < n; ++i)
        for (int a = 0; a < 3; ++a) s[a] += q[k].points3D[3 * i + a];
      for (int a = 0; a < 3; ++a) out->centroid[3 * k + a] = s[a] / static_cast<double>(n);
    }
    pos += n;
  }
  out->total = total;
}

const char* check_problems(const b2m_abs_pose_problem* problems, int64_t n_problems) {
  for (int64_t k = 0; k < n_problems; ++k) {
    const b2m_abs_pose_problem& q = problems[k];
    if (q.struct_size != sizeof(b2m_abs_pose_problem))
      return "[abs_pose.cu] Check Failed: b2m_abs_pose_problem.struct_size == sizeof(b2m_abs_pose_problem)";
    if (q.n < 0 || (q.n > 0 && (!q.points2D || !q.points3D))) return "[abs_pose.cu] Check Failed: points2D, points3D";
    if (q.n > INT32_MAX) return "[abs_pose.cu] Check Failed: correspondences per problem < 2^31";
    if (const char* why = camera_problem(q.camera)) return why;
  }
  return nullptr;
}

const char* check_refine_opts(const b2m_pose_refine_opts* r) {
  if (r->struct_size != sizeof(b2m_pose_refine_opts))
    return "[abs_pose.cu] Check Failed: b2m_pose_refine_opts.struct_size == sizeof(b2m_pose_refine_opts)";
  if (!(r->gradient_tolerance >= 0.0)) return "[abs_pose.cu] Check Failed: gradient_tolerance >= 0";
  if (r->max_num_iterations < 0) return "[abs_pose.cu] Check Failed: max_num_iterations >= 0";
  if (!(r->loss_function_scale >= 0.0)) return "[abs_pose.cu] Check Failed: loss_function_scale >= 0";
  return nullptr;
}

// d_model and d_cov (left empty unless want_cov) belong to the caller's chunk: the kernel reads them after the return.
int launch_refine(b2m_ctx* ctx, const Packed& H, int nb, const double* d_px, const double* d_p3, const int64_t* d_off,
                  const int32_t* d_cnt, const uint8_t* d_mask, double* d_pose, double* d_params, int32_t* d_success,
                  const b2m_pose_refine_opts* r, int want_cov, DeviceArray<int32_t>& d_model, DeviceArray<double>& d_cov) {
  B2M_CUDA_TRY(ctx, d_model.ensure(nb));
  B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_model, H.model.data(), sizeof(int32_t) * nb, cudaMemcpyHostToDevice, ctx->stream));
  if (want_cov) B2M_CUDA_TRY(ctx, d_cov.ensure(36 * static_cast<size_t>(nb)));
  if (want_cov) B2M_CUDA_TRY(ctx, cudaMemsetAsync(d_cov, 0, sizeof(double) * 36 * nb, ctx->stream));
  RefineParams Q{};
  Q.px = d_px; Q.p3 = d_p3; Q.off = d_off; Q.cnt = d_cnt; Q.model = d_model; Q.mask = d_mask;
  Q.pose = d_pose; Q.params = d_params; Q.success = d_success; Q.cov = d_cov;
  Q.gradient_tolerance = r->gradient_tolerance;
  Q.loss_scale = r->loss_function_scale;
  Q.max_num_iterations = r->max_num_iterations;
  Q.refine_focal = r->refine_focal_length;
  Q.refine_extra = r->refine_extra_params;
  b2m_abs_refine_kernel<<<nb, 32, 0, ctx->stream>>>(Q);
  B2M_CUDA_TRY(ctx, cudaGetLastError());
  ctx->stats.kernel_launches += 1;
  return B2M_OK;
}

void fill_result(b2m_abs_pose_result* r, const double* pose, const double* params, int success, int inliers, int factor,
                 const double* cov, int model) {
  memset(r, 0, sizeof(*r));
  r->struct_size = sizeof(*r);
  r->success = success;
  r->num_inliers = inliers;
  r->focal_sample = factor;
  r->qvec[0] = 1.0;
  if (success) {
    memcpy(r->qvec, pose, sizeof(double) * 4);
    memcpy(r->tvec, pose + 4, sizeof(double) * 3);
    if (cov) memcpy(r->covariance, cov, sizeof(double) * 36);
  }
  const int np = cam::num_params(model);
  for (int j = 0; j < np; ++j) r->params[j] = params[j];
}

}  // namespace
}  // namespace b2m

using namespace b2m;

extern "C" {

void b2m_abs_pose_opts_default(b2m_abs_pose_opts* o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->struct_size = sizeof(*o);
  o->estimate_focal_length = 0;
  o->num_focal_length_samples = 30;
  o->min_focal_length_ratio = 0.2;
  o->max_focal_length_ratio = 5.0;
  b2m_ransac_opts_default(&o->ransac);
}

void b2m_pose_refine_opts_default(b2m_pose_refine_opts* o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->struct_size = sizeof(*o);
  o->gradient_tolerance = 1.0;
  o->max_num_iterations = 100;
  o->loss_function_scale = 1.0;
  o->refine_focal_length = 1;
  o->refine_extra_params = 1;
  o->print_summary = 1;
}

int b2m_estimate_absolute_pose_batch(b2m_ctx* ctx, const b2m_abs_pose_problem* problems, int64_t n_problems,
                                     const b2m_abs_pose_opts* opts, const b2m_pose_refine_opts* refine,
                                     int32_t want_covariance, b2m_abs_pose_result* out, uint8_t* const* inlier_masks) {
  if (!ctx) return B2M_EINVAL;
  if (n_problems < 0 || (n_problems > 0 && (!problems || !out)) || !opts)
    return fail(ctx, B2M_EINVAL, "[abs_pose.cu] Check Failed: problems, options and out != NULL");
  if (opts->struct_size != sizeof(b2m_abs_pose_opts))
    return fail(ctx, B2M_EINVAL, "[abs_pose.cu] Check Failed: b2m_abs_pose_opts.struct_size == sizeof(b2m_abs_pose_opts)");
  // AbsolutePoseEstimationOptions::Check (U:estimators/pose.h)
  if (opts->num_focal_length_samples <= 0) return fail(ctx, B2M_EINVAL, "[pose.h] Check Failed: num_focal_length_samples > 0");
  if (!(opts->min_focal_length_ratio > 0)) return fail(ctx, B2M_EINVAL, "[pose.h] Check Failed: min_focal_length_ratio > 0");
  if (!(opts->max_focal_length_ratio > 0)) return fail(ctx, B2M_EINVAL, "[pose.h] Check Failed: max_focal_length_ratio > 0");
  if (!(opts->min_focal_length_ratio < opts->max_focal_length_ratio))
    return fail(ctx, B2M_EINVAL, "[pose.h] Check Failed: min_focal_length_ratio < max_focal_length_ratio");
  if (!(opts->ransac.max_error > 0)) return fail(ctx, B2M_EINVAL, "[ransac.h] Check Failed: max_error > 0");
  if (refine)
    if (const char* why = check_refine_opts(refine)) return fail(ctx, B2M_EINVAL, why);
  if (const char* why = check_problems(problems, n_problems)) return fail(ctx, B2M_EINVAL, why);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  std::vector<double> factors;
  if (opts->estimate_focal_length) {
    const int ns = opts->num_focal_length_samples;
    for (int i = 0; i <= ns; ++i) {
      const double f = static_cast<double>(i) / ns;
      factors.push_back(opts->min_focal_length_ratio + (opts->max_focal_length_ratio - opts->min_focal_length_ratio) * f * f);
    }
  } else {
    factors.push_back(1.0);
  }
  const int nf = static_cast<int>(factors.size());
  // chunks: at most 4096 problems and ~2^25 (point, focal sample) slots of normalised points per launch
  constexpr int64_t kChunk = 4096, kSlots = int64_t(1) << 25;
  int64_t k0 = 0;
  while (k0 < n_problems) {
    int nb = 0;
    int64_t slots = 0;
    while (k0 + nb < n_problems && nb < kChunk) {
      const int64_t s = problems[k0 + nb].n * nf;
      if (nb > 0 && slots + s > kSlots) break;
      slots += s;
      ++nb;
    }
    Packed H;
    pack(problems + k0, nb, &H);
    std::vector<int64_t> xoff(static_cast<size_t>(nb) * nf);
    int64_t pos = 0;
    for (int k = 0; k < nb; ++k)
      for (int f = 0; f < nf; ++f) {
        xoff[static_cast<size_t>(k) * nf + f] = pos;
        pos += H.cnt[k];
      }
    DeviceArray<double> d_px, d_p3, d_cent, d_models, d_fac, d_pose, d_params, d_cov;
    DeviceArray<int64_t> d_off, d_xoff;
    DeviceArray<int32_t> d_cnt, d_sup, d_succ, d_osucc, d_oinl, d_ofac, d_model;
    DeviceArray<DevCam> d_cams;
    DeviceArray<double2> d_xn;
    DeviceArray<uint8_t> d_cmask, d_mask;
    const size_t nc = static_cast<size_t>(nb) * nf;
    B2M_CUDA_TRY(ctx, d_px.ensure(2 * H.total));
    B2M_CUDA_TRY(ctx, d_p3.ensure(3 * H.total));
    B2M_CUDA_TRY(ctx, d_cent.ensure(3 * static_cast<size_t>(nb)));
    B2M_CUDA_TRY(ctx, d_models.ensure(12 * nc));
    B2M_CUDA_TRY(ctx, d_fac.ensure(nf));
    B2M_CUDA_TRY(ctx, d_pose.ensure(7 * static_cast<size_t>(nb)));
    B2M_CUDA_TRY(ctx, d_params.ensure(12 * static_cast<size_t>(nb)));
    B2M_CUDA_TRY(ctx, d_off.ensure(nb));
    B2M_CUDA_TRY(ctx, d_xoff.ensure(nc));
    B2M_CUDA_TRY(ctx, d_cnt.ensure(nb));
    B2M_CUDA_TRY(ctx, d_sup.ensure(nc));
    B2M_CUDA_TRY(ctx, d_succ.ensure(nc));
    B2M_CUDA_TRY(ctx, d_osucc.ensure(nb));
    B2M_CUDA_TRY(ctx, d_oinl.ensure(nb));
    B2M_CUDA_TRY(ctx, d_ofac.ensure(nb));
    B2M_CUDA_TRY(ctx, d_cams.ensure(nb));
    B2M_CUDA_TRY(ctx, d_xn.ensure(pos));
    B2M_CUDA_TRY(ctx, d_cmask.ensure(pos));
    B2M_CUDA_TRY(ctx, d_mask.ensure(H.total));
    if (H.total > 0) {
      B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_px, H.px.data(), sizeof(double) * 2 * H.total, cudaMemcpyHostToDevice, st));
      B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_p3, H.p3.data(), sizeof(double) * 3 * H.total, cudaMemcpyHostToDevice, st));
    }
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_cent, H.centroid.data(), sizeof(double) * 3 * nb, cudaMemcpyHostToDevice, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_fac, factors.data(), sizeof(double) * nf, cudaMemcpyHostToDevice, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_off, H.off.data(), sizeof(int64_t) * nb, cudaMemcpyHostToDevice, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_xoff, xoff.data(), sizeof(int64_t) * nc, cudaMemcpyHostToDevice, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_cnt, H.cnt.data(), sizeof(int32_t) * nb, cudaMemcpyHostToDevice, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_cams, H.cams.data(), sizeof(DevCam) * nb, cudaMemcpyHostToDevice, st));
    RansacParams P{};
    P.px = d_px; P.p3 = d_p3; P.centroid = d_cent; P.off = d_off; P.cnt = d_cnt; P.xoff = d_xoff; P.cams = d_cams;
    P.xn = d_xn; P.mask = d_cmask; P.models = d_models; P.sup = d_sup; P.success = d_succ;
    P.factors = d_fac; P.n_factors = nf; P.ro = opts->ransac; P.seed = ctx->seed; P.problem_base = k0;
    P.counters = ctx->d_counters + kAbsPoseCounters;
    b2m_abs_ransac_kernel<<<static_cast<unsigned>(nc), kRansacThreads, 0, st>>>(P);
    B2M_CUDA_TRY(ctx, cudaGetLastError());
    SelectParams S{};
    S.off = d_off; S.cnt = d_cnt; S.xoff = d_xoff; S.cta_mask = d_cmask; S.models = d_models; S.sup = d_sup;
    S.success = d_succ; S.centroid = d_cent; S.factors = d_fac; S.n_factors = nf;
    S.estimate_focal_length = opts->estimate_focal_length; S.cams = d_cams; S.mask = d_mask; S.pose = d_pose;
    S.params = d_params; S.out_success = d_osucc; S.out_inliers = d_oinl; S.out_factor = d_ofac;
    b2m_abs_select_kernel<<<nb, 32, 0, st>>>(S);
    B2M_CUDA_TRY(ctx, cudaGetLastError());
    ctx->stats.kernel_launches += 2;
    if (refine)
      if (int rc = launch_refine(ctx, H, nb, d_px, d_p3, d_off, d_cnt, d_mask, d_pose, d_params, d_osucc, refine,
                                 want_covariance, d_model, d_cov))
        return rc;
    std::vector<double> h_pose(7 * static_cast<size_t>(nb)), h_params(12 * static_cast<size_t>(nb)),
        h_cov(d_cov ? 36 * static_cast<size_t>(nb) : 0);
    std::vector<int32_t> h_succ(nb), h_inl(nb), h_fac(nb);
    std::vector<uint8_t> h_mask(static_cast<size_t>(std::max<int64_t>(H.total, 1)));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(h_pose.data(), d_pose, sizeof(double) * 7 * nb, cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(h_params.data(), d_params, sizeof(double) * 12 * nb, cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(h_succ.data(), d_osucc, sizeof(int32_t) * nb, cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(h_inl.data(), d_oinl, sizeof(int32_t) * nb, cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(h_fac.data(), d_ofac, sizeof(int32_t) * nb, cudaMemcpyDeviceToHost, st));
    if (d_cov) B2M_CUDA_TRY(ctx, cudaMemcpyAsync(h_cov.data(), d_cov, sizeof(double) * 36 * nb, cudaMemcpyDeviceToHost, st));
    if (H.total > 0 && inlier_masks)
      B2M_CUDA_TRY(ctx, cudaMemcpyAsync(h_mask.data(), d_mask, H.total, cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
    for (int k = 0; k < nb; ++k) {
      // params: the camera's parameters after estimation (focal scaled when estimating it) and refinement
      fill_result(&out[k0 + k], h_pose.data() + 7 * k, h_params.data() + 12 * k, h_succ[k], h_inl[k], h_fac[k],
                  d_cov ? h_cov.data() + 36 * k : nullptr, H.model[k]);
      if (inlier_masks && inlier_masks[k0 + k] && H.cnt[k] > 0)
        memcpy(inlier_masks[k0 + k], h_mask.data() + H.off[k], H.cnt[k]);
    }
    k0 += nb;
  }
  return B2M_OK;
}

int b2m_refine_absolute_pose_batch(b2m_ctx* ctx, const b2m_abs_pose_problem* problems, int64_t n_problems,
                                   const double* init_poses, const uint8_t* const* inlier_masks,
                                   const b2m_pose_refine_opts* refine, int32_t want_covariance, b2m_abs_pose_result* out) {
  if (!ctx) return B2M_EINVAL;
  if (n_problems < 0 || (n_problems > 0 && (!problems || !out || !init_poses || !inlier_masks)) || !refine)
    return fail(ctx, B2M_EINVAL, "[abs_pose.cu] Check Failed: problems, initial poses, inlier masks, options and out != NULL");
  if (const char* why = check_refine_opts(refine)) return fail(ctx, B2M_EINVAL, why);
  if (const char* why = check_problems(problems, n_problems)) return fail(ctx, B2M_EINVAL, why);
  for (int64_t k = 0; k < n_problems; ++k)
    if (problems[k].n > 0 && !inlier_masks[k]) return fail(ctx, B2M_EINVAL, "[abs_pose.cu] Check Failed: inlier_mask.size() == points2D.size()");
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  constexpr int64_t kChunk = 4096;
  for (int64_t k0 = 0; k0 < n_problems; k0 += kChunk) {
    const int nb = static_cast<int>(std::min(kChunk, n_problems - k0));
    Packed H;
    pack(problems + k0, nb, &H);
    std::vector<uint8_t> mask(static_cast<size_t>(std::max<int64_t>(H.total, 1)), 0);
    std::vector<double> params(12 * static_cast<size_t>(nb), 0.0);
    std::vector<int32_t> succ(nb, 1);
    for (int k = 0; k < nb; ++k) {
      for (int j = 0; j < cam::kMaxParams; ++j) params[12 * k + j] = H.cams[k].p[j];
      for (int64_t i = 0; i < H.cnt[k]; ++i) mask[H.off[k] + i] = inlier_masks[k0 + k][i] ? 1 : 0;
    }
    DeviceArray<double> d_px, d_p3, d_pose, d_params, d_cov;
    DeviceArray<int64_t> d_off;
    DeviceArray<int32_t> d_cnt, d_succ, d_model;
    DeviceArray<uint8_t> d_mask;
    B2M_CUDA_TRY(ctx, d_px.ensure(2 * H.total));
    B2M_CUDA_TRY(ctx, d_p3.ensure(3 * H.total));
    B2M_CUDA_TRY(ctx, d_pose.ensure(7 * static_cast<size_t>(nb)));
    B2M_CUDA_TRY(ctx, d_params.ensure(12 * static_cast<size_t>(nb)));
    B2M_CUDA_TRY(ctx, d_off.ensure(nb));
    B2M_CUDA_TRY(ctx, d_cnt.ensure(nb));
    B2M_CUDA_TRY(ctx, d_succ.ensure(nb));
    B2M_CUDA_TRY(ctx, d_mask.ensure(H.total));
    if (H.total > 0) {
      B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_px, H.px.data(), sizeof(double) * 2 * H.total, cudaMemcpyHostToDevice, st));
      B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_p3, H.p3.data(), sizeof(double) * 3 * H.total, cudaMemcpyHostToDevice, st));
      B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_mask, mask.data(), H.total, cudaMemcpyHostToDevice, st));
    }
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_pose, init_poses + 7 * k0, sizeof(double) * 7 * nb, cudaMemcpyHostToDevice, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_params, params.data(), sizeof(double) * 12 * nb, cudaMemcpyHostToDevice, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_off, H.off.data(), sizeof(int64_t) * nb, cudaMemcpyHostToDevice, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_cnt, H.cnt.data(), sizeof(int32_t) * nb, cudaMemcpyHostToDevice, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_succ, succ.data(), sizeof(int32_t) * nb, cudaMemcpyHostToDevice, st));
    if (int rc = launch_refine(ctx, H, nb, d_px, d_p3, d_off, d_cnt, d_mask, d_pose, d_params, d_succ, refine,
                               want_covariance, d_model, d_cov))
      return rc;
    std::vector<double> h_pose(7 * static_cast<size_t>(nb)), h_cov(d_cov ? 36 * static_cast<size_t>(nb) : 0);
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(h_pose.data(), d_pose, sizeof(double) * 7 * nb, cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(params.data(), d_params, sizeof(double) * 12 * nb, cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(succ.data(), d_succ, sizeof(int32_t) * nb, cudaMemcpyDeviceToHost, st));
    if (d_cov) B2M_CUDA_TRY(ctx, cudaMemcpyAsync(h_cov.data(), d_cov, sizeof(double) * 36 * nb, cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
    for (int k = 0; k < nb; ++k) {
      int inl = 0;
      for (int64_t i = 0; i < H.cnt[k]; ++i) inl += mask[H.off[k] + i];
      fill_result(&out[k0 + k], h_pose.data() + 7 * k, params.data() + 12 * k, succ[k], inl, 0,
                  d_cov ? h_cov.data() + 36 * k : nullptr, H.model[k]);
    }
  }
  return B2M_OK;
}

}  // extern "C"
