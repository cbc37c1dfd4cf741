// fusion_math.h -- the float32 arithmetic of stereo fusion, operation by operation: K9 (csrc/fusion.cu, compiled
// without FMA contraction) and the scalar oracle (oracle/fusion.cpp, -ffp-contract=off) both include it, so that a
// pixel's acceptance, its 3-D point and a cluster's medians round the same way on both sides.  Traversal order and
// the seed schedule are not here: each side restates them (DESIGN.md section 4, K9).
#pragma once
#include <float.h>
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define B2M_FU_HD __host__ __device__ __forceinline__
#else
#define B2M_FU_HD inline
#endif

namespace b2m_fu {

// One image as fusion sees it.  P = K [R | t] with K scaled per axis to the depth-map size, inv_P the top 3 rows of
// [P; 0 0 0 1]^-1, inv_R = R^T: computed in fp64 on the host and rounded to fp32 once.
struct Cam {
  float P[12], iP[12], iR[9];
  float sx, sy;       // bitmap_scale: depth-map size / camera (bitmap) size, per axis
  int32_t W, H;       // depth-map size
  int32_t bw, bh;     // bitmap size
  int64_t px_off;     // offset of the image's pixels in the concatenated maps; -1: no maps (not a seed, not a target)
  int64_t rgb_off;    // offset of the bitmap's RGB bytes
  int32_t ov_off, ov_n;  // the overlap list: ov[ov_off .. ov_off + ov_n)
};

struct Opts {
  int32_t min_num_pixels, max_num_pixels, max_traversal_depth;
  float max_reproj_sq;   // max_reproj_error * max_reproj_error (fp32)
  float max_depth_error;
  float min_cos_normal;  // cos(max_normal_error in radians), fp64 rounded once
  float bbox[6];         // min x, y, z, max x, y, z
};

// out = M x for a 3 x 4 row-major M and the homogeneous point (x, 1)
B2M_FU_HD void affine(const float* M, const float* x, float* out) {
  for (int k = 0; k < 3; ++k) out[k] = ((M[4 * k] * x[0] + M[4 * k + 1] * x[1]) + M[4 * k + 2] * x[2]) + M[4 * k + 3];
}

B2M_FU_HD void rotate(const float* R, const float* n, float* out) {
  for (int k = 0; k < 3; ++k) out[k] = (R[3 * k] * n[0] + R[3 * k + 1] * n[1]) + R[3 * k + 2] * n[2];
}

// xyz = inv_P (col d, row d, d, 1): integer pixel coordinates, no half-pixel offset.
B2M_FU_HD void backproject(const Cam& c, int row, int col, float d, float* xyz) {
  const float h[3] = {static_cast<float>(col) * d, static_cast<float>(row) * d, d};
  affine(c.iP, h, xyz);
}

// The checks of a popped pixel at traversal depth > 0 against the cluster's reference point and normal; nw = the
// pixel's normal in world coordinates.
B2M_FU_HD bool consistent(const Cam& c, const Opts& o, const float* ref_xyz, const float* ref_n, int row, int col, float d,
                          const float* nw) {
  float p[3];
  affine(c.P, ref_xyz, p);
  if (fabsf(p[2] - d) / d > o.max_depth_error) return false;
  const float dc = p[0] / p[2] - static_cast<float>(col);
  const float dr = p[1] / p[2] - static_cast<float>(row);
  if (dc * dc + dr * dr > o.max_reproj_sq) return false;
  return (ref_n[0] * nw[0] + ref_n[1] * nw[1]) + ref_n[2] * nw[2] >= o.min_cos_normal;
}

// The pixel of image c that xyz projects to, rounded half away from zero; false outside the depth map.
B2M_FU_HD bool child_pixel(const Cam& c, const float* xyz, int* row, int* col) {
  float p[3];
  affine(c.P, xyz, p);
  const float fc = roundf(p[0] / p[2]);
  const float fr = roundf(p[1] / p[2]);
  if (!(fc >= 0.f && fc < static_cast<float>(c.W) && fr >= 0.f && fr < static_cast<float>(c.H))) return false;
  *col = static_cast<int>(fc);
  *row = static_cast<int>(fr);
  return true;
}

B2M_FU_HD bool in_box(const Opts& o, const float* x) {
  for (int k = 0; k < 3; ++k)
    if (!(x[k] >= o.bbox[k] && x[k] <= o.bbox[3 + k])) return false;
  return true;
}

// Nearest bitmap pixel of depth-map pixel (row, col): (round(col / sx), round(row / sy)); black outside the bitmap.
B2M_FU_HD void colour(const Cam& c, const uint8_t* rgb, int row, int col, float* out) {
  const float fx = roundf(static_cast<float>(col) / c.sx);
  const float fy = roundf(static_cast<float>(row) / c.sy);
  out[0] = out[1] = out[2] = 0.f;
  if (!(fx >= 0.f && fx < static_cast<float>(c.bw) && fy >= 0.f && fy < static_cast<float>(c.bh))) return;
  const uint8_t* q = rgb + c.rgb_off + 3 * (static_cast<int64_t>(fy) * c.bw + static_cast<int64_t>(fx));
  for (int k = 0; k < 3; ++k) out[k] = static_cast<float>(q[k]);
}

// In-place ascending heap sort (the medians need the order statistics only, so any sort gives the same values).
template <typename T>
B2M_FU_HD void heap_sort(T* v, int n) {
  auto sift = [&](int i, int m) {
    for (;;) {
      int c = 2 * i + 1;
      if (c >= m) return;
      if (c + 1 < m && v[c] < v[c + 1]) ++c;
      if (!(v[i] < v[c])) return;
      const T t = v[i];
      v[i] = v[c];
      v[c] = t;
      i = c;
    }
  };
  for (int i = n / 2 - 1; i >= 0; --i) sift(i, n);
  for (int m = n - 1; m > 0; --m) {
    const T t = v[0];
    v[0] = v[m];
    v[m] = t;
    sift(0, m);
  }
}

// Median of n >= 1 sorted values: the middle one, or the fp32 mean of the two middle ones.
B2M_FU_HD float median_sorted(const float* v, int n) {
  return (n & 1) ? v[n / 2] : (v[n / 2 - 1] + v[n / 2]) * 0.5f;
}

// A cluster's point from its per-channel medians m[9] = (x, y, z, nx, ny, nz, r, g, b): false when the median normal
// has a norm below FLT_EPSILON (no point).
B2M_FU_HD bool finish_point(const float* m, float* xyz, float* nrm, uint8_t* rgb) {
  const float norm = sqrtf((m[3] * m[3] + m[4] * m[4]) + m[5] * m[5]);
  if (!(norm >= FLT_EPSILON)) return false;
  for (int k = 0; k < 3; ++k) {
    xyz[k] = m[k];
    nrm[k] = m[3 + k] / norm;
    rgb[k] = static_cast<uint8_t>(roundf(m[6 + k]));
  }
  return true;
}

}  // namespace b2m_fu
