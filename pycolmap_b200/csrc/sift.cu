// sift.cu -- K6: SIFT feature extraction (replaces SiftCPUFeatureExtractor::Extract, U:feature/sift.cc, which runs
// VLFeat's vl_sift; SURVEY.md rows X1-X8).  The arithmetic restates VLFeat operation for operation, in VLFeat's types
// (this file is compiled without FMA contraction), so that the pyramid, the DoG and the keypoints equal the numpy
// oracle (oracle/sift.py) bit for bit.  The histograms of the orientation and descriptor stages are summed per lane
// and then over the lanes in a fixed order: deterministic, but a different rounding than VLFeat's single running sum.
//
// Per image, per octave: base level (upsample / copy / subsample), incremental separable Gaussian levels with the DoG
// of each level formed in the pass that blurs it, gradients (modulus, angle) of the detection levels, then detection
// in scan order through a three-pass deterministic compaction (count per block, scan, write).  After the last octave
// the keypoint list comes to the host for the max_num_features cut; one warp per kept keypoint computes the
// orientations, one warp per (keypoint, orientation) the descriptor.  No floating-point atomics anywhere.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "internal.h"

namespace b2m {
namespace {

constexpr double kPi = 3.14159265358979323846;
constexpr int kMaxOctaves = 32;
constexpr int kKpCap = 1 << 20;  // keypoints per image before the cut
constexpr int kDetectThreads = 256;
constexpr int kOriWarps = 4;
constexpr int kDescWarps = 2;

struct Kp {
  float x, y, s, sigma;
  int o, ix, iy, is;
};

__constant__ double c_expn[258];  // VLFeat's fast_expn table exp(-k 25 / 256), k = 0 .. 256, and a 0 guard

__device__ __forceinline__ double fast_expn(double x) {
  if (x > 25.0) return 0.0;
  x *= 256 / 25.0;
  const int i = static_cast<int>(floor(x));
  const double r = x - i;
  const double a = c_expn[i], b = c_expn[i + 1];
  return a + r * (b - a);
}

__device__ __forceinline__ float fast_atan2_f(float y, float x) {
  const float c3 = 0.1821F, c1 = 0.9675F;
  const float abs_y = fabsf(y) + 1.19209290E-07F;
  float angle, r;
  if (x >= 0) {
    r = (x - abs_y) / (x + abs_y);
    angle = static_cast<float>(kPi / 4);
  } else {
    r = (x + abs_y) / (abs_y - x);
    angle = static_cast<float>(3 * kPi / 4);
  }
  angle += (c3 * r * r - c1) * r;
  return (y < 0) ? -angle : angle;
}

__device__ __forceinline__ float fast_sqrt_f(float x) {
  if (static_cast<double>(x) < 1e-8) return 0.0f;
  const float xhalf = 0.5f * x;
  float y = __int_as_float(0x5f3759df - (__float_as_int(x) >> 1));
  y = y * (1.5f - xhalf * y * y);
  y = y * (1.5f - xhalf * y * y);
  return x * y;
}

__device__ __forceinline__ float mod_2pi_f(float x) {
  const float tp = static_cast<float>(2 * kPi);
  while (x > tp) x -= tp;
  while (x < 0.0f) x += tp;
  return x;
}

// ---- pyramid ------------------------------------------------------------------------------------------------------
__global__ void b2m_sift_to_float_kernel(const uint8_t* __restrict__ img, int64_t stride, int w, int h, float* out) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(w) * h) return;
  const int y = static_cast<int>(i / w), x = static_cast<int>(i % w);
  out[i] = static_cast<float>(img[y * stride + x]) / 255.0f;
}

// copy_and_upsample_rows applied twice: (h, w) -> (2h, 2w), linear interpolation, the last sample repeated
__global__ void b2m_sift_upsample_kernel(const float* __restrict__ in, int w, int h, float* out) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int W2 = 2 * w;
  if (i >= static_cast<int64_t>(W2) * 2 * h) return;
  const int Y = static_cast<int>(i / W2), X = static_cast<int>(i % W2);
  const int x = X >> 1, y = Y >> 1, x1 = min(x + 1, w - 1), y1 = min(y + 1, h - 1);
  auto row = [&](int yy) {
    const float a = in[static_cast<int64_t>(yy) * w + x];
    return (X & 1) ? (a + in[static_cast<int64_t>(yy) * w + x1]) * 0.5f : a;
  };
  const float a = row(y);
  out[i] = (Y & 1) ? (a + row(y1)) * 0.5f : a;
}

__global__ void b2m_sift_subsample_kernel(const float* __restrict__ in, int w_in, int d, int w, int h, float* out) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(w) * h) return;
  const int y = static_cast<int>(i / w), x = static_cast<int>(i % w);
  out[i] = in[static_cast<int64_t>(y) * d * w_in + static_cast<int64_t>(x) * d];
}

// vl_imconvcol_vf along y: taps g[0 .. 2R] over rows y - R .. y + R, replicated border, one running fp32 sum in tap
// order.  A 32 x 8 CTA owns a tile of 32 columns x kBlurRowsV rows; the tile's rows with their halo (clamped at the
// border) and the taps are staged in shared memory, so every input sample is read from HBM once per tile.
constexpr int kBlurRowsV = 64;
constexpr int kBlurColsH = 128;
constexpr int kMaxBlurR = 150;
__global__ void __launch_bounds__(256) b2m_sift_blur_v_kernel(const float* __restrict__ in, int w, int h,
                                                              const float* __restrict__ g, int R, float* __restrict__ out) {
  extern __shared__ float sm[];
  float* taps = sm;                          // 2R + 1
  float* tile = sm + 2 * R + 1;              // (kBlurRowsV + 2R) x 32
  const int tx = threadIdx.x, ty = threadIdx.y, t = ty * 32 + tx;
  const int x = blockIdx.x * 32 + tx, y0 = blockIdx.y * kBlurRowsV;
  for (int k = t; k <= 2 * R; k += 256) taps[k] = g[k];
  const int rows = kBlurRowsV + 2 * R;
  for (int r = ty; r < rows; r += 8) {
    const int yy = min(max(y0 - R + r, 0), h - 1);
    tile[r * 32 + tx] = x < w ? __ldg(in + static_cast<int64_t>(yy) * w + x) : 0.0f;
  }
  __syncthreads();
  if (x >= w) return;
  for (int r = ty; r < kBlurRowsV && y0 + r < h; r += 8) {
    float acc = 0.0f;
    for (int k = 0; k <= 2 * R; ++k) acc += tile[(r + k) * 32 + tx] * taps[k];
    out[static_cast<int64_t>(y0 + r) * w + x] = acc;
  }
}

// the same along x over a tile of kBlurColsH columns x 8 rows; with `prev`, also the DoG out - prev of the level just
// blurred
__global__ void __launch_bounds__(256) b2m_sift_blur_h_dog_kernel(const float* __restrict__ in, int w, int h,
                                                                  const float* __restrict__ g, int R, float* __restrict__ out,
                                                                  const float* __restrict__ prev, float* __restrict__ dog) {
  extern __shared__ float sm[];
  float* taps = sm;
  const int cols = kBlurColsH + 2 * R;
  float* tile = sm + 2 * R + 1;              // 8 x cols
  const int tx = threadIdx.x, ty = threadIdx.y, t = ty * 32 + tx;
  const int x0 = blockIdx.x * kBlurColsH, y = blockIdx.y * 8 + ty;
  for (int k = t; k <= 2 * R; k += 256) taps[k] = g[k];
  if (y < h) {
    const float* row = in + static_cast<int64_t>(y) * w;
    for (int c = tx; c < cols; c += 32) tile[ty * cols + c] = __ldg(row + min(max(x0 - R + c, 0), w - 1));
  }
  __syncthreads();
  if (y >= h) return;
  for (int c = tx; c < kBlurColsH && x0 + c < w; c += 32) {
    float acc = 0.0f;
    for (int k = 0; k <= 2 * R; ++k) acc += tile[ty * cols + c + k] * taps[k];
    const int64_t i = static_cast<int64_t>(y) * w + x0 + c;
    out[i] = acc;
    if (dog) dog[i] = acc - prev[i];
  }
}

// update_gradient: (modulus, angle in [0, 2 pi]) with one-sided differences at the border
__global__ void b2m_sift_gradient_kernel(const float* __restrict__ L, int w, int h, float2* __restrict__ grad) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(w) * h) return;
  const int y = static_cast<int>(i / w), x = static_cast<int>(i % w);
  const float* p = L + i;
  float gx, gy;
  if (x == 0) gx = p[1] - p[0];
  else if (x == w - 1) gx = p[0] - p[-1];
  else gx = 0.5f * (p[1] - p[-1]);
  if (y == 0) gy = p[w] - p[0];
  else if (y == h - 1) gy = p[0] - p[-w];
  else gy = 0.5f * (p[w] - p[-w]);
  const float mod = fast_sqrt_f(gx * gx + gy * gy);
  const float ang = mod_2pi_f(static_cast<float>(static_cast<double>(fast_atan2_f(gy, gx)) + 2 * kPi));
  grad[i] = make_float2(mod, ang);
}

// ---- detection ----------------------------------------------------------------------------------------------------
struct DetectParams {
  const float* dog;  // levels s = -1 .. S, each w x h
  int w, h, S, o;
  double peak, edge, sigma0;
  int64_t n;         // S * (w - 2) * (h - 2) samples, scan order (s, y, x)
};

__device__ bool detect_one(const DetectParams& P, int64_t idx, Kp* kp) {
  const int iw = P.w - 2, ih = P.h - 2;
  int x = static_cast<int>(idx % iw) + 1;
  int y = static_cast<int>((idx / iw) % ih) + 1;
  const int s = static_cast<int>(idx / (static_cast<int64_t>(iw) * ih));
  const int64_t xo = 1, yo = P.w, so = static_cast<int64_t>(P.w) * P.h;
  const float* pt = P.dog + so * (s + 1) + yo * y + x;
  const float v = *pt;
  const double tp = 0.8 * P.peak;
  bool is_max = static_cast<double>(v) >= tp, is_min = static_cast<double>(v) <= -tp;
  if (!is_max && !is_min) return false;
  for (int ds = -1; ds <= 1; ++ds)
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        if (!ds && !dy && !dx) continue;
        const float n = pt[ds * so + dy * yo + dx * xo];
        is_max = is_max && v > n;
        is_min = is_min && v < n;
      }
  if (!is_max && !is_min) return false;
  // refinement (vl_sift_detect): up to 5 quadratic fits, stepping one pixel while |offset| > 0.6
  double Dx = 0, Dy = 0, Ds = 0, Dxx = 0, Dyy = 0, Dxy = 0, b[3] = {0, 0, 0};
  int dx = 0, dy = 0;
  for (int iter = 0; iter < 5; ++iter) {
    x += dx;
    y += dy;
    const float* q = P.dog + so * (s + 1) + yo * y + x;
#define AT(DX, DY, DS) (q[(DX) * xo + (DY) * yo + (DS) * so])
    Dx = 0.5 * (AT(+1, 0, 0) - AT(-1, 0, 0));
    Dy = 0.5 * (AT(0, +1, 0) - AT(0, -1, 0));
    Ds = 0.5 * (AT(0, 0, +1) - AT(0, 0, -1));
    Dxx = static_cast<double>(AT(+1, 0, 0) + AT(-1, 0, 0)) - 2.0 * AT(0, 0, 0);
    Dyy = static_cast<double>(AT(0, +1, 0) + AT(0, -1, 0)) - 2.0 * AT(0, 0, 0);
    const double Dss = static_cast<double>(AT(0, 0, +1) + AT(0, 0, -1)) - 2.0 * AT(0, 0, 0);
    Dxy = 0.25 * (AT(+1, +1, 0) + AT(-1, -1, 0) - AT(-1, +1, 0) - AT(+1, -1, 0));
    const double Dxs = 0.25 * (AT(+1, 0, +1) + AT(-1, 0, -1) - AT(-1, 0, +1) - AT(+1, 0, -1));
    const double Dys = 0.25 * (AT(0, +1, +1) + AT(0, -1, -1) - AT(0, -1, +1) - AT(0, +1, -1));
    double A[3][3] = {{Dxx, Dxy, Dxs}, {Dxy, Dyy, Dys}, {Dxs, Dys, Dss}};
    b[0] = -Dx;
    b[1] = -Dy;
    b[2] = -Ds;
    for (int j = 0; j < 3; ++j) {
      double maxa = 0, maxabsa = 0;
      int maxi = -1;
      for (int i = j; i < 3; ++i) {
        const double a = A[i][j], absa = fabs(a);
        if (absa > maxabsa) {
          maxa = a;
          maxabsa = absa;
          maxi = i;
        }
      }
      if (maxabsa < 1e-10f) {
        b[0] = b[1] = b[2] = 0;
        break;
      }
      const int i = maxi;
      for (int jj = j; jj < 3; ++jj) {
        const double t = A[i][jj];
        A[i][jj] = A[j][jj];
        A[j][jj] = t;
        A[j][jj] /= maxa;
      }
      const double t = b[j];
      b[j] = b[i];
      b[i] = t;
      b[j] /= maxa;
      for (int ii = j + 1; ii < 3; ++ii) {
        const double xx = A[ii][j];
        for (int jj = j; jj < 3; ++jj) A[ii][jj] -= xx * A[j][jj];
        b[ii] -= xx * b[j];
      }
    }
    for (int i = 2; i > 0; --i) {
      const double xx = b[i];
      for (int ii = i - 1; ii >= 0; --ii) b[ii] -= xx * A[ii][i];
    }
    dx = ((b[0] > 0.6 && x < P.w - 2) ? 1 : 0) + ((b[0] < -0.6 && x > 1) ? -1 : 0);
    dy = ((b[1] > 0.6 && y < P.h - 2) ? 1 : 0) + ((b[1] < -0.6 && y > 1) ? -1 : 0);
    if (dx == 0 && dy == 0) break;
  }
  const float* q = P.dog + so * (s + 1) + yo * y + x;
  const double val = static_cast<double>(q[0]) + 0.5 * (Dx * b[0] + Dy * b[1] + Ds * b[2]);
  const double score = (Dxx + Dyy) * (Dxx + Dyy) / (Dxx * Dyy - Dxy * Dxy);
  const double xn = x + b[0], yn = y + b[1], sn = s + b[2];
  const bool good = fabs(val) > P.peak && score < (P.edge + 1) * (P.edge + 1) / P.edge && score >= 0 &&
                    fabs(b[0]) < 1.5 && fabs(b[1]) < 1.5 && fabs(b[2]) < 1.5 && xn >= 0 && xn <= P.w - 1 && yn >= 0 &&
                    yn <= P.h - 1 && sn >= -1 && sn <= P.S + 1;
  if (!good) return false;
  const double xper = ldexp(1.0, P.o);
  kp->o = P.o;
  kp->ix = x;
  kp->iy = y;
  kp->is = s;
  kp->s = static_cast<float>(sn);
  kp->x = static_cast<float>(xn * xper);
  kp->y = static_cast<float>(yn * xper);
  kp->sigma = static_cast<float>(P.sigma0 * pow(2.0, sn / P.S) * xper);
  return true;
#undef AT
}

__global__ void __launch_bounds__(kDetectThreads) b2m_sift_detect_count_kernel(DetectParams P, int* __restrict__ counts) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(kDetectThreads) + threadIdx.x;
  Kp kp;
  const int c = __syncthreads_count(i < P.n && detect_one(P, i, &kp));
  if (threadIdx.x == 0) counts[blockIdx.x] = c;
}

// exclusive scan of the block counts (one CTA), offset by the keypoints already found; advances *total
__global__ void __launch_bounds__(1024) b2m_sift_scan_kernel(const int* __restrict__ counts, int nb, int* __restrict__ offs,
                                                           int* __restrict__ total) {
  __shared__ int part[1024];
  const int t = threadIdx.x, per = (nb + 1023) / 1024, b0 = min(t * per, nb), b1 = min(b0 + per, nb);
  int sum = 0;
  for (int b = b0; b < b1; ++b) sum += counts[b];
  part[t] = sum;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {
    const int v = t >= d ? part[t - d] : 0;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  const int base = *total;
  int run = base + part[t] - sum;
  for (int b = b0; b < b1; ++b) {
    offs[b] = run;
    run += counts[b];
  }
  __syncthreads();
  if (t == 1023) *total = base + part[1023];
}

__global__ void __launch_bounds__(kDetectThreads) b2m_sift_detect_write_kernel(DetectParams P, const int* __restrict__ offs,
                                                                               Kp* __restrict__ out) {
  __shared__ int warp_base[kDetectThreads / 32];
  const int64_t i = blockIdx.x * static_cast<int64_t>(kDetectThreads) + threadIdx.x;
  Kp kp;
  const bool f = i < P.n && detect_one(P, i, &kp);
  const unsigned m = __ballot_sync(0xffffffffu, f);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) warp_base[wid] = __popc(m);
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int k = 0; k < kDetectThreads / 32; ++k) {
      const int c = warp_base[k];
      warp_base[k] = run;
      run += c;
    }
  }
  __syncthreads();
  if (f) {
    const int pos = offs[blockIdx.x] + warp_base[wid] + __popc(m & ((1u << lane) - 1));
    if (pos < kKpCap) out[pos] = kp;
  }
}

// ---- orientation and descriptor ------------------------------------------------------------------------------------
struct OctTab {
  int o_min, n;
  int w[kMaxOctaves], h[kMaxOctaves];
  int64_t goff[kMaxOctaves];  // float2 offset of the octave's gradient levels (S levels of w x h)
};

// vl_sift_calc_keypoint_orientations with bilinear binning; one warp per keypoint
__global__ void __launch_bounds__(32 * kOriWarps) b2m_sift_orientation_kernel(const Kp* __restrict__ kps, int n, OctTab T,
                                                                            const float2* __restrict__ grad,
                                                                            int* __restrict__ n_ang, double* __restrict__ ang_out) {
  __shared__ double hist[kOriWarps][32][37];
  __shared__ double tot[kOriWarps][36];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int k = blockIdx.x * kOriWarps + wid;
  if (k >= n) return;
  const Kp kp = kps[k];
  const int oi = kp.o - T.o_min, w = T.w[oi], h = T.h[oi];
  const double xper = ldexp(1.0, kp.o);
  const double x = kp.x / xper, y = kp.y / xper, sigma = kp.sigma / xper;
  const int xi = static_cast<int>(x + 0.5), yi = static_cast<int>(y + 0.5);
  const double sigmaw = 1.5 * sigma;
  const int W = static_cast<int>(fmax(floor(3.0 * sigmaw), 1.0));
  if (xi < 0 || xi > w - 1 || yi < 0 || yi > h - 1) {
    if (lane == 0) n_ang[k] = 0;
    return;
  }
  const float2* g = grad + T.goff[oi] + static_cast<int64_t>(kp.is) * w * h;
  double* hl = hist[wid][lane];
  for (int b = 0; b < 36; ++b) hl[b] = 0.0;
  const int ys0 = max(-W, -yi), ys1 = min(W, h - 1 - yi), xs0 = max(-W, -xi), xs1 = min(W, w - 1 - xi);
  const int nx = xs1 - xs0 + 1, npix = nx * (ys1 - ys0 + 1);
  for (int p = lane; p < npix; p += 32) {
    const int ys = ys0 + p / nx, xs = xs0 + p % nx;
    const double dx = static_cast<double>(xi + xs) - x, dy = static_cast<double>(yi + ys) - y;
    const double r2 = dx * dx + dy * dy;
    if (r2 >= W * W + 0.6) continue;
    const double wgt = fast_expn(r2 / (2 * sigmaw * sigmaw));
    const float2 ma = g[static_cast<int64_t>(yi + ys) * w + xi + xs];
    const double mod = ma.x, fbin = 36 * static_cast<double>(ma.y) / (2 * kPi);
    const int bin = static_cast<int>(floor(fbin - 0.5));
    const double rbin = fbin - bin - 0.5;
    hl[(bin + 36) % 36] += (1 - rbin) * mod * wgt;
    hl[(bin + 1) % 36] += rbin * mod * wgt;
  }
  __syncwarp();
  for (int b = lane; b < 36; b += 32) {
    double s = 0.0;
    for (int l = 0; l < 32; ++l) s += hist[wid][l][b];
    tot[wid][b] = s;
  }
  __syncwarp();
  if (lane != 0) return;
  double* H = tot[wid];
  for (int iter = 0; iter < 6; ++iter) {
    double prev = H[35];
    const double first = H[0];
    int i;
    for (i = 0; i < 35; ++i) {
      const double nh = (prev + H[i] + H[i + 1]) / 3.0;
      prev = H[i];
      H[i] = nh;
    }
    H[i] = (prev + H[i] + first) / 3.0;
  }
  double maxh = 0;
  for (int i = 0; i < 36; ++i) maxh = fmax(maxh, H[i]);
  int na = 0;
  for (int i = 0; i < 36 && na < 4; ++i) {
    const double h0 = H[i], hm = H[(i + 35) % 36], hp = H[(i + 1) % 36];
    if (h0 > 0.8 * maxh && h0 > hm && h0 > hp) {
      const double di = -0.5 * (hp - hm) / (hp + hm - 2 * h0);
      ang_out[4 * k + na++] = 2 * kPi * (i + di + 0.5) / 36;
    }
  }
  n_ang[k] = na;
}

struct DescEntry {
  int kp;
  int reserved;
  double angle;
};

// vl_sift_calc_keypoint_descriptor, then COLMAP's normalisation, u8 conversion and the VLFeat -> UBC layout; one warp
// per (keypoint, orientation)
__global__ void __launch_bounds__(32 * kDescWarps) b2m_sift_descriptor_kernel(const Kp* __restrict__ kps,
                                                                            const DescEntry* __restrict__ ent, int n, OctTab T,
                                                                            const float2* __restrict__ grad, int l2,
                                                                            float* __restrict__ kp_out, uint8_t* __restrict__ d_out) {
  __shared__ float hist[kDescWarps][32][129];
  __shared__ float tot[kDescWarps][128];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int e = blockIdx.x * kDescWarps + wid;
  if (e >= n) return;
  const DescEntry E = ent[e];
  const Kp kp = kps[E.kp];
  const double angle0 = E.angle;
  const int oi = kp.o - T.o_min, w = T.w[oi], h = T.h[oi];
  const double xper = ldexp(1.0, kp.o);
  const double x = kp.x / xper, y = kp.y / xper, sigma = kp.sigma / xper;
  const int xi = static_cast<int>(x + 0.5), yi = static_cast<int>(y + 0.5);
  const double st0 = sin(angle0), ct0 = cos(angle0);
  const double SBP = 3.0 * sigma + 2.220446049250313e-16;
  const int W = static_cast<int>(floor(sqrt(2.0) * SBP * 5 / 2.0 + 0.5));
  float* hl = hist[wid][lane];
  for (int b = 0; b < 128; ++b) hl[b] = 0.0f;
  const bool inside = !(xi < 0 || xi >= w || yi < 0 || yi >= h - 1);
  if (inside) {
    const float2* g = grad + T.goff[oi] + static_cast<int64_t>(kp.is) * w * h;
    const int ys0 = max(-W, 1 - yi), ys1 = min(W, h - yi - 2), xs0 = max(-W, 1 - xi), xs1 = min(W, w - xi - 2);
    const int nx = xs1 - xs0 + 1, ny_ = ys1 - ys0 + 1;
    const int npix = (nx > 0 && ny_ > 0) ? nx * ny_ : 0;
    for (int p = lane; p < npix; p += 32) {
      const int dyi = ys0 + p / nx, dxi = xs0 + p % nx;
      const float2 ma = g[static_cast<int64_t>(yi + dyi) * w + xi + dxi];
      const float mod = ma.x;
      const float theta = mod_2pi_f(static_cast<float>(ma.y - angle0));
      const float dx = static_cast<float>(xi + dxi - x), dy = static_cast<float>(yi + dyi - y);
      const float nxf = static_cast<float>((ct0 * dx + st0 * dy) / SBP);
      const float nyf = static_cast<float>((-st0 * dx + ct0 * dy) / SBP);
      const float nt = static_cast<float>(8 * theta / (2 * kPi));
      const float win = static_cast<float>(fast_expn((nxf * nxf + nyf * nyf) / (2.0 * 2.0f * 2.0f)));
      const int binx = static_cast<int>(floorf(static_cast<float>(nxf - 0.5)));
      const int biny = static_cast<int>(floorf(static_cast<float>(nyf - 0.5)));
      const int bint = static_cast<int>(floorf(nt));
      const float rbinx = static_cast<float>(nxf - (binx + 0.5));
      const float rbiny = static_cast<float>(nyf - (biny + 0.5));
      const float rbint = nt - bint;
      for (int dbx = 0; dbx < 2; ++dbx)
        for (int dby = 0; dby < 2; ++dby)
          for (int dbt = 0; dbt < 2; ++dbt)
            if (binx + dbx >= -2 && binx + dbx < 2 && biny + dby >= -2 && biny + dby < 2) {
              const float wt = win * mod * fabsf(1 - dbx - rbinx) * fabsf(1 - dby - rbiny) * fabsf(1 - dbt - rbint);
              hl[(biny + dby + 2) * 32 + (binx + dbx + 2) * 8 + (bint + dbt) % 8] += wt;
            }
    }
  }
  __syncwarp();
  for (int b = lane; b < 128; b += 32) {
    float s = 0.0f;
    for (int l = 0; l < 32; ++l) s += hist[wid][l][b];
    tot[wid][b] = s;
  }
  __syncwarp();
  if (lane != 0) return;
  float* d = tot[wid];
  auto normalize = [&]() {
    float nrm = 0.0f;
    for (int b = 0; b < 128; ++b) nrm += d[b] * d[b];
    nrm = fast_sqrt_f(nrm) + 1.19209290E-07F;
    for (int b = 0; b < 128; ++b) d[b] /= nrm;
  };
  normalize();
  for (int b = 0; b < 128; ++b)
    if (d[b] > 0.2) d[b] = 0.2f;
  normalize();
  if (l2) {
    float s = 0.0f;
    for (int b = 0; b < 128; ++b) s += d[b] * d[b];
    if (s > 0) {
      const float r = sqrtf(s);
      for (int b = 0; b < 128; ++b) d[b] /= r;
    }
  } else {
    float s = 0.0f;
    for (int b = 0; b < 128; ++b) s += fabsf(d[b]);
    for (int b = 0; b < 128; ++b) d[b] = sqrtf(d[b] / s);
  }
  uint8_t* o = d_out + static_cast<int64_t>(e) * 128;
  for (int c = 0; c < 16; ++c)
    for (int q = 0; q < 8; ++q) {
      const float v = fminf(roundf(512.0f * d[8 * c + q]), 255.0f);
      o[8 * c + (q ? 8 - q : 0)] = static_cast<uint8_t>(v);
    }
  // FeatureKeypoint(x + 0.5, y + 0.5, sigma, angle) read back through ComputeScale / ComputeOrientation
  const float af = static_cast<float>(angle0), sc = kp.sigma;
  const float a11 = sc * cosf(af), a21 = sc * sinf(af), a12 = -sc * sinf(af), a22 = sc * cosf(af);
  float* ko = kp_out + static_cast<int64_t>(e) * 4;
  ko[0] = kp.x + 0.5f;
  ko[1] = kp.y + 0.5f;
  ko[2] = (sqrtf(a11 * a11 + a21 * a21) + sqrtf(a12 * a12 + a22 * a22)) / 2.0f;
  ko[3] = atan2f(a21, a11);
}

// ---- host side ---------------------------------------------------------------------------------------------------
// Buffers of the Gaussian pyramid: sized by the largest first octave and the number of levels, replaced together.
struct SiftPyramid {
  int64_t cap_px = 0;
  int cap_levels = 0;
  DeviceArray<uint8_t> d_img;
  DeviceArray<float> d_G, d_D, d_T, d_U;
};

// Fixed-size buffers, allocated (and the exp table uploaded) by the first call.
struct SiftTables {
  DeviceArray<int> d_total, d_nang;
  DeviceArray<double> d_ang;
  DeviceArray<Kp> d_kp;
  DeviceArray<float> d_taps;
};

struct SiftState {
  SiftPyramid px;
  SiftTables tab;
  DeviceArray<float2> d_grad;
  DeviceArray<int> d_counts, d_offs;
  DeviceArray<DescEntry> d_ent;
  DeviceArray<float> d_kout;
  DeviceArray<uint8_t> d_dout;
};

// _vl_sift_smooth's kernel: half-width max(ceil(4 sigma), 1), fp32 taps normalised by their fp32 running sum
std::vector<float> gauss_taps(double sigma) {
  const int R = std::max(static_cast<int>(std::ceil(4.0 * sigma)), 1);
  std::vector<float> g(2 * R + 1);
  float acc = 0;
  for (int j = 0; j < 2 * R + 1; ++j) {
    const float d = static_cast<float>(j - R) / static_cast<float>(sigma);
    g[j] = static_cast<float>(std::exp(-0.5 * (d * d)));
    acc += g[j];
  }
  for (float& v : g) v /= acc;
  return g;
}

// VL_SHIFT_LEFT(width, -o): the size of octave o of a W x H image
void octave_dims(int W, int H, int o, int* w, int* h) {
  *w = o < 0 ? W << -o : W >> o;
  *h = o < 0 ? H << -o : H >> o;
}

// octaves extract_one builds: from o_min, at most num_octaves (and kMaxOctaves), while at least 3 x 3
int num_octaves_built(int W, int H, const b2m_extract_opts& op) {
  int n = 0;
  for (int o = op.first_octave; o < op.first_octave + op.num_octaves && n < kMaxOctaves; ++o, ++n) {
    int w, h;
    octave_dims(W, H, o, &w, &h);
    if (w < 3 || h < 3) break;
  }
  return n;
}

inline unsigned blocks_for(int64_t n, int t) { return static_cast<unsigned>((n + t - 1) / t); }

int extract_one(b2m_ctx* ctx, SiftState* S, const uint8_t* src, int64_t stride, int W, int H, cudaMemcpyKind kind,
                const b2m_extract_opts& op, const std::vector<int>& tap_off, const std::vector<int>& tap_r, b2m_features* F) {
  cudaStream_t st = ctx->stream;
  const int Sr = op.octave_resolution, o_min = op.first_octave;
  const double sigmak = std::pow(2.0, 1.0 / Sr), sigma0 = 1.6 * sigmak;
  auto dims = [&](int o, int* w, int* h) { octave_dims(W, H, o, w, h); };
  int w0, h0;
  dims(o_min, &w0, &h0);
  const int64_t A0 = static_cast<int64_t>(w0) * h0;
  // base level
  B2M_CUDA_TRY(ctx, cudaMemcpy2DAsync(S->px.d_img, W, src, stride, W, H, kind, st));
  float* G = S->px.d_G;
  float* base = G;  // level s = -1
  {
    float* a = o_min < 0 ? S->px.d_T : (o_min > 0 ? S->px.d_U : base);
    b2m_sift_to_float_kernel<<<blocks_for(static_cast<int64_t>(W) * H, 256), 256, 0, st>>>(S->px.d_img, W, W, H, a);
    ctx->stats.kernel_launches += 1;
    if (o_min < 0) {
      int w = W, h = H;
      for (int k = 0; k < -o_min; ++k) {
        float* dst = (k == -o_min - 1) ? base : (a == S->px.d_T ? S->px.d_U : S->px.d_T);
        b2m_sift_upsample_kernel<<<blocks_for(4LL * w * h, 256), 256, 0, st>>>(a, w, h, dst);
        ctx->stats.kernel_launches += 1;
        a = dst;
        w *= 2;
        h *= 2;
      }
    } else if (o_min > 0) {
      b2m_sift_subsample_kernel<<<blocks_for(A0, 256), 256, 0, st>>>(a, W, 1 << o_min, w0, h0, base);
      ctx->stats.kernel_launches += 1;
    }
  }
  B2M_CUDA_TRY(ctx, cudaGetLastError());
  auto blur = [&](const float* in, int w, int h, int f, float* out, const float* prev, float* dog) {
    const int64_t n = static_cast<int64_t>(w) * h;
    const int R = tap_r[f];
    const dim3 bv((w + 31) / 32, (h + kBlurRowsV - 1) / kBlurRowsV), bh((w + kBlurColsH - 1) / kBlurColsH, (h + 7) / 8);
    b2m_sift_blur_v_kernel<<<bv, dim3(32, 8), sizeof(float) * (2 * R + 1 + 32 * (kBlurRowsV + 2 * R)), st>>>(
        in, w, h, S->tab.d_taps + tap_off[f], R, S->px.d_T);
    b2m_sift_blur_h_dog_kernel<<<bh, dim3(32, 8), sizeof(float) * (2 * R + 1 + 8 * (kBlurColsH + 2 * R)), st>>>(
        S->px.d_T, w, h, S->tab.d_taps + tap_off[f], R, out,
                                                                   prev, dog);
    ctx->stats.kernel_launches += 2;
  };
  if (tap_r[0] > 0) blur(base, w0, h0, 0, base, nullptr, nullptr);  // in place: the vertical pass reads `base` first
  OctTab T{};
  T.o_min = o_min;
  int64_t goff = 0;
  B2M_CUDA_TRY(ctx, cudaMemsetAsync(S->tab.d_total, 0, sizeof(int), st));
  const int nlev = Sr + 3;
  const int n_oct = num_octaves_built(W, H, op);
  for (int o = o_min; o < o_min + n_oct; ++o) {
    int w, h;
    dims(o, &w, &h);
    const int64_t A = static_cast<int64_t>(w) * h;
    if (o > o_min) {  // level S - 1 of the previous octave at even indices (no extra smoothing: sa == sb)
      int pw, ph;
      dims(o - 1, &pw, &ph);
      b2m_sift_subsample_kernel<<<blocks_for(A, 256), 256, 0, st>>>(G + static_cast<int64_t>(Sr) * A0, pw, 2, w, h, S->px.d_U);
      B2M_CUDA_TRY(ctx, cudaMemcpyAsync(G, S->px.d_U, sizeof(float) * A, cudaMemcpyDeviceToDevice, st));
      ctx->stats.kernel_launches += 1;
    }
    for (int s = 1; s < nlev; ++s)  // level s - 1 of VLFeat's numbering; DoG s - 2 = G[s] - G[s - 1]
      blur(G + (s - 1) * A0, w, h, s, G + s * A0, G + (s - 1) * A0, S->px.d_D + (s - 1) * A);
    B2M_CUDA_TRY(ctx, cudaGetLastError());
    T.w[o - o_min] = w;
    T.h[o - o_min] = h;
    T.goff[o - o_min] = goff;
    T.n = o - o_min + 1;
    for (int s = 0; s < Sr; ++s)
      b2m_sift_gradient_kernel<<<blocks_for(A, 256), 256, 0, st>>>(G + (s + 1) * A0, w, h, S->d_grad + goff + s * A);
    ctx->stats.kernel_launches += Sr;
    goff += Sr * A;
    DetectParams P;
    P.dog = S->px.d_D;
    P.w = w;
    P.h = h;
    P.S = Sr;
    P.o = o;
    P.peak = op.peak_threshold;
    P.edge = op.edge_threshold;
    P.sigma0 = sigma0;
    P.n = static_cast<int64_t>(Sr) * (w - 2) * (h - 2);
    const unsigned nb = blocks_for(P.n, kDetectThreads);
    b2m_sift_detect_count_kernel<<<nb, kDetectThreads, 0, st>>>(P, S->d_counts);
    b2m_sift_scan_kernel<<<1, 1024, 0, st>>>(S->d_counts, static_cast<int>(nb), S->d_offs, S->tab.d_total);
    b2m_sift_detect_write_kernel<<<nb, kDetectThreads, 0, st>>>(P, S->d_offs, S->tab.d_kp);
    ctx->stats.kernel_launches += 3;
    B2M_CUDA_TRY(ctx, cudaGetLastError());
  }
  int total = 0;
  B2M_CUDA_TRY(ctx, cudaMemcpyAsync(&total, S->tab.d_total, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
  if (total > kKpCap) {
    ctx->err = "[sift.cu] more than 2^20 keypoints in one image before the max_num_features cut";
    return B2M_ENOMEM;
  }
  std::vector<Kp> kp(total);
  if (total) B2M_CUDA_TRY(ctx, cudaMemcpy(kp.data(), S->tab.d_kp, sizeof(Kp) * total, cudaMemcpyDeviceToHost));
  // max_num_features: (octave, level) runs from the coarsest down; the run that passes the limit is kept whole
  std::vector<int> run_start;
  for (int i = 0; i < total; ++i)
    if (i == 0 || kp[i].o != kp[i - 1].o || kp[i].is != kp[i - 1].is) run_start.push_back(i);
  int first = 0;
  {
    int64_t cnt = 0;
    for (int r = static_cast<int>(run_start.size()) - 1; r >= 0; --r) {
      const int end = r + 1 < static_cast<int>(run_start.size()) ? run_start[r + 1] : total;
      cnt += end - run_start[r];
      if (cnt > op.max_num_features) {
        first = run_start[r];
        break;
      }
    }
  }
  const int nk = total - first;
  std::vector<int> nang(nk, 1);
  std::vector<double> ang(4 * static_cast<size_t>(nk), 0.0);
  if (nk && !op.upright) {
    b2m_sift_orientation_kernel<<<blocks_for(nk, kOriWarps), 32 * kOriWarps, 0, st>>>(S->tab.d_kp + first, nk, T, S->d_grad,
                                                                                    S->tab.d_nang, S->tab.d_ang);
    ctx->stats.kernel_launches += 1;
    B2M_CUDA_TRY(ctx, cudaGetLastError());
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(nang.data(), S->tab.d_nang, sizeof(int) * nk, cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(ang.data(), S->tab.d_ang, sizeof(double) * 4 * nk, cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
  }
  std::vector<DescEntry> ent;
  for (int k = 0; k < nk; ++k)
    for (int a = 0; a < std::min(nang[k], op.max_num_orientations); ++a) ent.push_back(DescEntry{first + k, 0, ang[4 * k + a]});
  const int ne = static_cast<int>(ent.size());
  const size_t f0 = F->kpts.size() / 4;
  F->kpts.resize(4 * (f0 + ne));
  F->desc.resize(128 * (f0 + ne));
  if (ne) {
    B2M_CUDA_TRY(ctx, S->d_ent.ensure(ne));
    B2M_CUDA_TRY(ctx, S->d_kout.ensure(4 * static_cast<size_t>(ne)));
    B2M_CUDA_TRY(ctx, S->d_dout.ensure(128 * static_cast<size_t>(ne)));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->d_ent, ent.data(), sizeof(DescEntry) * ne, cudaMemcpyHostToDevice, st));
    b2m_sift_descriptor_kernel<<<blocks_for(ne, kDescWarps), 32 * kDescWarps, 0, st>>>(
        S->tab.d_kp, S->d_ent, ne, T, S->d_grad, op.normalization == B2M_NORMALIZATION_L2, S->d_kout, S->d_dout);
    ctx->stats.kernel_launches += 1;
    B2M_CUDA_TRY(ctx, cudaGetLastError());
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(F->kpts.data() + 4 * f0, S->d_kout, sizeof(float) * 4 * ne, cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(F->desc.data() + 128 * f0, S->d_dout, 128 * static_cast<size_t>(ne), cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
  }
  F->off.push_back(static_cast<int64_t>(f0) + ne);
  ctx->stats.sift_images += 1;
  ctx->stats.sift_keypoints += nk;
  ctx->stats.sift_descriptors += ne;
  return B2M_OK;
}

}  // namespace

void sift_release(b2m_ctx* ctx) {
  delete static_cast<SiftState*>(ctx->sift_state);
  ctx->sift_state = nullptr;
}

int sift_begin(b2m_ctx* ctx, const b2m_extract_opts* opts, const int32_t* widths, const int32_t* heights, int32_t n,
               SiftPlan* plan) {
  if (opts->struct_size != sizeof(b2m_extract_opts))
    return fail(ctx, B2M_EINVAL, "[sift.cu] Check Failed: b2m_extract_opts.struct_size == sizeof(b2m_extract_opts)");
  const b2m_extract_opts& o = *opts;
  // SiftExtractionOptions::Check (U:feature/sift.cc)
  if (!(o.max_image_size > 0)) return fail(ctx, B2M_EINVAL, "[sift.cc] Check Failed: max_image_size > 0");
  if (!(o.max_num_features > 0)) return fail(ctx, B2M_EINVAL, "[sift.cc] Check Failed: max_num_features > 0");
  if (!(o.octave_resolution > 0)) return fail(ctx, B2M_EINVAL, "[sift.cc] Check Failed: octave_resolution > 0");
  if (!(o.peak_threshold > 0.0)) return fail(ctx, B2M_EINVAL, "[sift.cc] Check Failed: peak_threshold > 0");
  if (!(o.edge_threshold > 0.0)) return fail(ctx, B2M_EINVAL, "[sift.cc] Check Failed: edge_threshold > 0");
  if (!(o.max_num_orientations > 0)) return fail(ctx, B2M_EINVAL, "[sift.cc] Check Failed: max_num_orientations > 0");
  if (!(o.num_octaves > 0)) return fail(ctx, B2M_EINVAL, "[sift.cu] Check Failed: num_octaves > 0");
  if (!(o.first_octave >= -3 && o.first_octave <= 16)) return fail(ctx, B2M_EINVAL, "[sift.cu] Check Failed: -3 <= first_octave <= 16");
  if (o.normalization != B2M_NORMALIZATION_L1_ROOT && o.normalization != B2M_NORMALIZATION_L2)
    return fail(ctx, B2M_EINVAL, "[sift.cu] Check Failed: normalization is L1_ROOT or L2");
  if (o.estimate_affine_shape || o.domain_size_pooling)
    return fail(ctx, B2M_EINVAL, "[sift.cu] Check Failed: estimate_affine_shape and domain_size_pooling (the covariant path) are not supported");
  if (o.darkness_adaptivity) return fail(ctx, B2M_EINVAL, "[sift.cu] Check Failed: darkness_adaptivity (SiftGPU only) is not supported");
  plan->opts = o;
  int64_t max_a0 = 0, need_grad = 1;
  int max_w = 0, max_h = 0;
  for (int32_t i = 0; i < n; ++i) {
    const b2m_image im{widths[i], heights[i], widths[i], nullptr};
    if (im.width > o.max_image_size || im.height > o.max_image_size)
      return fail(ctx, B2M_EINVAL, "[sift.h] Check Failed: image " + std::to_string(i) + " within max_image_size");
    const int f = o.first_octave;
    const int64_t a0 = f < 0 ? (static_cast<int64_t>(im.width) << -f) * (static_cast<int64_t>(im.height) << -f)
                             : static_cast<int64_t>(im.width >> f) * (im.height >> f);
    if (a0 > (int64_t(1) << 30)) return fail(ctx, B2M_EINVAL, "[sift.cu] Check Failed: first octave of at most 2^30 pixels");
    max_a0 = std::max(max_a0, a0);
    // gradients of every octave stay resident until the descriptors are done: S levels per octave
    int64_t areas = 0;
    for (int k = 0, no = num_octaves_built(im.width, im.height, o); k < no; ++k) {
      int w, h;
      octave_dims(im.width, im.height, o.first_octave + k, &w, &h);
      areas += static_cast<int64_t>(w) * h;
    }
    need_grad = std::max(need_grad, static_cast<int64_t>(o.octave_resolution) * areas);
    max_w = std::max(max_w, im.width);
    max_h = std::max(max_h, im.height);
  }
  cudaSetDevice(ctx->device);
  if (!ctx->sift_state) ctx->sift_state = new SiftState();
  SiftState* S = static_cast<SiftState*>(ctx->sift_state);
  if (!S->tab.d_taps) {
    const int rc = alloc_group(S->tab, [&](SiftTables& t) -> int {
      double tab[258];
      for (int k = 0; k < 257; ++k) tab[k] = std::exp(-static_cast<double>(k) * (25.0 / 256));
      tab[257] = 0.0;
      B2M_CUDA_TRY(ctx, cudaMemcpyToSymbol(c_expn, tab, sizeof(tab)));
      B2M_CUDA_TRY(ctx, t.d_total.ensure(1));
      B2M_CUDA_TRY(ctx, t.d_nang.ensure(kKpCap));
      B2M_CUDA_TRY(ctx, t.d_ang.ensure(4 * kKpCap));
      B2M_CUDA_TRY(ctx, t.d_kp.ensure(kKpCap));
      B2M_CUDA_TRY(ctx, t.d_taps.ensure(65536));
      return B2M_OK;
    });
    if (rc) return rc;
  }
  const int nlev = o.octave_resolution + 3;
  const int64_t img_px = static_cast<int64_t>(max_w) * max_h;
  const int64_t need_px = std::max(max_a0, img_px);
  if (n > 0 && (need_px > S->px.cap_px || nlev > S->px.cap_levels)) {
    const int rc = alloc_group(S->px, [&](SiftPyramid& p) -> int {
      B2M_CUDA_TRY(ctx, p.d_img.ensure(need_px));
      B2M_CUDA_TRY(ctx, p.d_G.ensure(static_cast<size_t>(nlev) * need_px));
      B2M_CUDA_TRY(ctx, p.d_D.ensure(static_cast<size_t>(nlev - 1) * need_px));
      B2M_CUDA_TRY(ctx, p.d_T.ensure(need_px));
      B2M_CUDA_TRY(ctx, p.d_U.ensure(need_px));
      p.cap_px = need_px;
      p.cap_levels = nlev;
      return B2M_OK;
    });
    if (rc) return rc;
  }
  const int64_t need_blocks = (static_cast<int64_t>(o.octave_resolution) * max_a0 + kDetectThreads - 1) / kDetectThreads + 1;
  if (n > 0) {
    B2M_CUDA_TRY(ctx, S->d_grad.ensure(need_grad));
    B2M_CUDA_TRY(ctx, S->d_counts.ensure(need_blocks));
    B2M_CUDA_TRY(ctx, S->d_offs.ensure(need_blocks));
  }
  // filters: [0] the first level's (0 taps when sa <= sb), [s] level s - 1 of VLFeat's numbering from level s - 2
  const int Sr = o.octave_resolution;
  const double sigmak = std::pow(2.0, 1.0 / Sr), sigma0 = 1.6 * sigmak;
  const double dsigma0 = sigma0 * std::sqrt(1.0 - 1.0 / (sigmak * sigmak));
  std::vector<float> taps;
  std::vector<int>& tap_off = plan->tap_off;
  std::vector<int>& tap_r = plan->tap_r;
  tap_off.assign(nlev, 0);
  tap_r.assign(nlev, 0);
  {
    const double sa = sigma0 * std::pow(sigmak, -1), sb = 0.5 * std::pow(2.0, -o.first_octave);
    tap_off[0] = 0;
    tap_r[0] = 0;
    if (sa > sb) {
      const std::vector<float> g = gauss_taps(std::sqrt(sa * sa - sb * sb) / std::pow(2.0, o.first_octave));
      taps = g;
      tap_r[0] = static_cast<int>(g.size() / 2);
    }
    for (int s = 1; s < nlev; ++s) {
      const std::vector<float> g = gauss_taps(dsigma0 * std::pow(sigmak, s - 1));
      tap_off[s] = static_cast<int>(taps.size());
      tap_r[s] = static_cast<int>(g.size() / 2);
      taps.insert(taps.end(), g.begin(), g.end());
    }
  }
  if (taps.size() > 65536) return fail(ctx, B2M_EINVAL, "[sift.cu] Check Failed: Gaussian filters of at most 65536 taps in all");
  // the blur tiles stage 32 x (64 + 2R) samples in the 48 KB of default shared memory
  if (*std::max_element(tap_r.begin(), tap_r.end()) > kMaxBlurR)
    return fail(ctx, B2M_EINVAL, "[sift.cu] Check Failed: Gaussian half-width <= " + std::to_string(kMaxBlurR) +
               " (octave_resolution and first_octave give a smoothing this wide)");
  B2M_CUDA_TRY(ctx, cudaMemcpy(S->tab.d_taps, taps.data(), sizeof(float) * std::max<size_t>(taps.size(), 1), cudaMemcpyHostToDevice));
  return B2M_OK;
}

int sift_extract(b2m_ctx* ctx, const SiftPlan& plan, const uint8_t* img, int64_t stride, int W, int H, bool on_device,
                 b2m_features* F, const float** d_kout) {
  SiftState* S = static_cast<SiftState*>(ctx->sift_state);
  if (int rc = extract_one(ctx, S, img, stride, W, H, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                           plan.opts, plan.tap_off, plan.tap_r, F))
    return rc;
  if (d_kout) *d_kout = S->d_kout;
  return B2M_OK;
}

}  // namespace b2m

using namespace b2m;

extern "C" {

void b2m_extract_opts_default(b2m_extract_opts* o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->struct_size = sizeof(*o);
  o->max_image_size = 3200;
  o->max_num_features = 8192;
  o->first_octave = -1;
  o->num_octaves = 4;
  o->octave_resolution = 3;
  o->peak_threshold = 0.02 / 3;
  o->edge_threshold = 10.0;
  o->max_num_orientations = 2;
  o->upright = 0;
  o->normalization = B2M_NORMALIZATION_L1_ROOT;
}

int b2m_extract_features_batch(b2m_ctx* ctx, const b2m_image* images, int32_t n, const b2m_extract_opts* opts,
                               b2m_features** out) {
  if (!ctx) return B2M_EINVAL;
  if (!out || !opts || n < 0 || (n > 0 && !images)) return fail(ctx, B2M_EINVAL, "[sift.cu] Check Failed: images, options and out != NULL");
  *out = nullptr;
  if (opts->struct_size != sizeof(b2m_extract_opts))
    return fail(ctx, B2M_EINVAL, "[sift.cu] Check Failed: b2m_extract_opts.struct_size == sizeof(b2m_extract_opts)");
  std::vector<int32_t> widths(n), heights(n);
  for (int32_t i = 0; i < n; ++i) {
    const b2m_image& im = images[i];
    if (!im.data || im.width <= 0 || im.height <= 0 || im.stride < im.width)
      return fail(ctx, B2M_EINVAL, "[sift.cu] Check Failed: image " + std::to_string(i) + " is non-empty with stride >= width");
    widths[i] = im.width;
    heights[i] = im.height;
  }
  SiftPlan plan;
  if (int rc = sift_begin(ctx, opts, widths.data(), heights.data(), n, &plan)) return rc;
  b2m_features* F = new b2m_features();
  F->off.push_back(0);
  for (int32_t i = 0; i < n; ++i) {
    if (ctx->stop) {
      delete F;
      return B2M_ESTOPPED;
    }
    if (int rc = sift_extract(ctx, plan, images[i].data, images[i].stride, images[i].width, images[i].height, false, F, nullptr)) {
      delete F;
      return rc;
    }
  }
  *out = F;
  return B2M_OK;
}

int b2m_features_get(const b2m_features* f, int32_t image, b2m_feature_view* out) {
  if (!f || !out || image < 0 || image + 1 >= static_cast<int64_t>(f->off.size())) return B2M_EINVAL;
  const int64_t a = f->off[image], b = f->off[image + 1];
  out->struct_size = sizeof(*out);
  out->reserved = 0;
  out->n = b - a;
  out->keypoints = f->kpts.data() + 4 * a;
  out->descriptors = f->desc.data() + 128 * a;
  return B2M_OK;
}

void b2m_features_free(b2m_features* f) { delete f; }

}  // extern "C"
