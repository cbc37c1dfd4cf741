// patch_match.cu -- K8: PatchMatch stereo with pixelwise view selection (Schoenberger et al., ECCV 2016; what
// U:mvs/patch_match_cuda.cu computes), over a batch of reference images.
//
// Decomposition (DESIGN.md section 4, K8): one warp per scan line -- a column for the vertical sweeps, a row for the
// horizontal ones -- of every problem of the batch, four warps per CTA.  The line is walked sequentially (the only
// dependency is along the sweep); inside a pixel the 32 lanes share the window samples of each (hypothesis, source)
// evaluation, and lane s keeps the per-source state of source s (its cost, selection probability and draw count).
// Window sums are reduced with a fixed xor-butterfly, so a pixel's arithmetic depends on nothing but its inputs: the
// maps of a problem are the same alone or at any position of any batch.
//
// Random numbers are counter-based (pm_uniform): keyed by (ctx seed, reference image index, pixel, iteration, sweep,
// draw).  Interpolation is explicit fp32 bilinear with zero outside the image (oracle/patch_match.py restates it), and
// the file is compiled without FMA contraction so that the oracle's per-operation float32 rounding is the device's.
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "internal.h"

struct b2m_depth_maps {
  std::vector<int32_t> width, height;
  std::vector<int64_t> off;  // pixel offset of map k
  std::vector<float> depth, normal;
};

namespace b2m {
namespace {

constexpr int kMaxSrc = B2M_PM_MAX_SOURCES;
constexpr int kWarpsPerCta = 4;
constexpr int kInitSweep = 4;   // RNG sweep id of the random start hypotheses
constexpr int kMaxWindowRadius = 32;
// The hidden Markov chain of a source's visibility along a sweep (Schoenberger et al. 2016, section 3.2): it keeps its
// state from one pixel to the next with probability kStay; an occluded source emits an NCC cost with the uniform
// density kUniformProb, a visible one with the likelihood exp(-cost^2 / (2 ncc_sigma^2)).
constexpr float kStay = 0.999f;
constexpr float kUniformProb = 0.5f;

struct PmCam {
  float fx, fy, cx, cy;
  float R[9], t[3];  // cam_from_world
  int W, H;
  int64_t img_off;   // into the image pool
  int64_t dmap_off;  // into the depth-map pool, -1 = none
};

// One problem, with the source poses relative to the reference (src_from_ref) precomputed on the host in fp64.
struct PmProblem {
  int ref, n_src;
  int key;           // the caller's stable id of the reference: the key of its random numbers
  int src[kMaxSrc];
  float Rs[kMaxSrc][9], ts[kMaxSrc][3];
  float dmin, dmax;
  int64_t map_off;   // pixel offset of this problem's maps
  int64_t sel_off;   // offset of its backward messages, n_src per pixel
};

struct PmParams {
  int radius, step, side, n_win;     // side = 2 radius / step + 1 offsets per axis, n_win = side^2
  int num_samples, geom, filter, filter_min_num_consistent;
  float inv_2ss, inv_2sc;            // 1 / (2 sigma_spatial^2), 1 / (2 sigma_color^2)
  float inv_2ncc, min_tri, inv_2inc;
  float geom_reg, geom_max, filter_max_cost, filter_min_tri, filter_geom_max;
};

struct Hyp {
  float d, n0, n1, n2;
};

// ---- counter-based random numbers (splitmix64 finaliser over the key) ----
__device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ float pm_uniform(uint64_t seed, int image, int pixel, int iter, int sweep, int draw) {
  uint64_t h = mix64(seed ^ static_cast<uint32_t>(image));
  h = mix64(h ^ static_cast<uint32_t>(pixel));
  h = mix64(h ^ ((static_cast<uint64_t>(static_cast<uint32_t>(iter)) << 8) | static_cast<uint32_t>(sweep)));
  h = mix64(h ^ static_cast<uint32_t>(draw));
  return static_cast<float>(h >> 40) * (1.0f / 16777216.0f);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float pix(const uint8_t* img, int W, int H, int x, int y) {
  return (x >= 0 && y >= 0 && x < W && y < H) ? static_cast<float>(img[static_cast<int64_t>(y) * W + x]) * (1.0f / 255.0f)
                                              : 0.0f;
}

// Bilinear sample at COLMAP image coordinates (pixel centres at +0.5), zero outside the image.
__device__ __forceinline__ float bilinear(const uint8_t* img, int W, int H, float u, float v) {
  const float x = u - 0.5f, y = v - 0.5f;
  if (!(fabsf(x) < 1e6f) || !(fabsf(y) < 1e6f)) return 0.0f;
  const float fx = floorf(x), fy = floorf(y);
  const int x0 = static_cast<int>(fx), y0 = static_cast<int>(fy);
  const float ax = x - fx, ay = y - fy;
  const float top = (1.0f - ax) * pix(img, W, H, x0, y0) + ax * pix(img, W, H, x0 + 1, y0);
  const float bot = (1.0f - ax) * pix(img, W, H, x0, y0 + 1) + ax * pix(img, W, H, x0 + 1, y0 + 1);
  return (1.0f - ay) * top + ay * bot;
}

__device__ __forceinline__ void ray_of(const PmCam& c, int x, int y, float* r) {
  r[0] = (static_cast<float>(x) + 0.5f - c.cx) / c.fx;
  r[1] = (static_cast<float>(y) + 0.5f - c.cy) / c.fy;
  r[2] = 1.0f;
}

// Weighted window sums of the reference around (x, y): sum w, sum w r, sum w r^2 (all lanes get the totals).
struct RefWin {
  float sw, swr, swrr;
};

__device__ RefWin ref_window(const PmParams& P, const uint8_t* img, int W, int H, int x, int y, int lane) {
  const float c0 = pix(img, W, H, x, y);
  float sw = 0.f, swr = 0.f, swrr = 0.f;
  for (int k = lane; k < P.n_win; k += 32) {
    const int dy = -P.radius + (k / P.side) * P.step, dx = -P.radius + (k % P.side) * P.step;
    const int xx = x + dx, yy = y + dy;
    if (xx < 0 || yy < 0 || xx >= W || yy >= H) continue;
    const float r = pix(img, W, H, xx, yy);
    const float dc = r - c0;
    const float w = expf(-static_cast<float>(dx * dx + dy * dy) * P.inv_2ss - dc * dc * P.inv_2sc);
    sw += w;
    swr += w * r;
    swrr += w * r * r;
  }
  return RefWin{warp_sum(sw), warp_sum(swr), warp_sum(swrr)};
}

// 1 - weighted NCC of hypothesis h at (x, y) against source slot s, clamped to [0, 2].
__device__ float photo_cost(const PmParams& P, const PmCam& rc, const uint8_t* rimg, const PmCam& sc, const uint8_t* simg,
                            const float* Rs, const float* ts, const Hyp& h, int x, int y, const RefWin& rw, int lane,
                            unsigned long long* samples) {
  float ray[3];
  ray_of(rc, x, y, ray);
  const float dn = h.d * (h.n0 * ray[0] + h.n1 * ray[1] + h.n2 * ray[2]);  // n . X0
  // M = Rs + ts n^T / (n . X0): the plane-induced map of normalised reference coordinates to the source camera frame
  float M[9];
  const float n[3] = {h.n0, h.n1, h.n2};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) M[i * 3 + j] = Rs[i * 3 + j] + ts[i] * n[j] / dn;
  const int W = rc.W, H = rc.H;
  const float c0 = pix(rimg, W, H, x, y);
  float sws = 0.f, swss = 0.f, swrs = 0.f;
  int cnt = 0;
  for (int k = lane; k < P.n_win; k += 32) {
    const int dy = -P.radius + (k / P.side) * P.step, dx = -P.radius + (k % P.side) * P.step;
    const int xx = x + dx, yy = y + dy;
    if (xx < 0 || yy < 0 || xx >= W || yy >= H) continue;
    const float r = pix(rimg, W, H, xx, yy);
    const float dc = r - c0;
    const float w = expf(-static_cast<float>(dx * dx + dy * dy) * P.inv_2ss - dc * dc * P.inv_2sc);
    const float q0 = (static_cast<float>(xx) + 0.5f - rc.cx) / rc.fx, q1 = (static_cast<float>(yy) + 0.5f - rc.cy) / rc.fy;
    const float Y0 = M[0] * q0 + M[1] * q1 + M[2], Y1 = M[3] * q0 + M[4] * q1 + M[5], Y2 = M[6] * q0 + M[7] * q1 + M[8];
    float s = 0.f;
    if (Y2 > 0.f) s = bilinear(simg, sc.W, sc.H, sc.fx * (Y0 / Y2) + sc.cx, sc.fy * (Y1 / Y2) + sc.cy);
    sws += w * s;
    swss += w * s * s;
    swrs += w * r * s;
    ++cnt;
  }
  if (samples) *samples += static_cast<unsigned long long>(cnt);
  sws = warp_sum(sws);
  swss = warp_sum(swss);
  swrs = warp_sum(swrs);
  const float inv = 1.0f / rw.sw;
  const float mr = rw.swr * inv, ms = sws * inv;
  const float vr = rw.swrr * inv - mr * mr, vs = swss * inv - ms * ms;
  const float cv = swrs * inv - mr * ms;
  if (!(vr > 1e-5f) || !(vs > 1e-5f) || !(fabsf(dn) > 0.f)) return 2.0f;
  const float ncc = cv / sqrtf(vr * vs);
  return fminf(fmaxf(1.0f - ncc, 0.0f), 2.0f);
}

// Forward-backward reprojection error (pixels) of the hypothesis point through the source's depth map, at most `cap`.
__device__ float geom_error(const PmCam& rc, const PmCam& sc, const float* sdepth, const float* Rs, const float* ts,
                            const Hyp& h, int x, int y, float cap) {
  float ray[3];
  ray_of(rc, x, y, ray);
  const float X[3] = {h.d * ray[0], h.d * ray[1], h.d * ray[2]};
  const float Y[3] = {Rs[0] * X[0] + Rs[1] * X[1] + Rs[2] * X[2] + ts[0], Rs[3] * X[0] + Rs[4] * X[1] + Rs[5] * X[2] + ts[1],
                      Rs[6] * X[0] + Rs[7] * X[1] + Rs[8] * X[2] + ts[2]};
  if (!(Y[2] > 0.f)) return cap;
  const float u = sc.fx * (Y[0] / Y[2]) + sc.cx, v = sc.fy * (Y[1] / Y[2]) + sc.cy;
  if (!(u >= 0.f && v >= 0.f && u < static_cast<float>(sc.W) && v < static_cast<float>(sc.H))) return cap;
  const int su = static_cast<int>(u), sv = static_cast<int>(v);
  const float ds = sdepth[static_cast<int64_t>(sv) * sc.W + su];
  if (!(ds > 0.f)) return cap;
  // back-project the source pixel centre at its depth, map it to the reference (X = Rs^T (Y - ts)) and project
  const float Z[3] = {ds * ((static_cast<float>(su) + 0.5f - sc.cx) / sc.fx) - ts[0],
                      ds * ((static_cast<float>(sv) + 0.5f - sc.cy) / sc.fy) - ts[1], ds - ts[2]};
  const float B[3] = {Rs[0] * Z[0] + Rs[3] * Z[1] + Rs[6] * Z[2], Rs[1] * Z[0] + Rs[4] * Z[1] + Rs[7] * Z[2],
                      Rs[2] * Z[0] + Rs[5] * Z[1] + Rs[8] * Z[2]};
  if (!(B[2] > 0.f)) return cap;
  const float ex = rc.fx * (B[0] / B[2]) + rc.cx - (static_cast<float>(x) + 0.5f);
  const float ey = rc.fy * (B[1] / B[2]) + rc.cy - (static_cast<float>(y) + 0.5f);
  return fminf(sqrtf(ex * ex + ey * ey), cap);
}

// Cosine of the triangulation angle and of the incident angle of source slot s for hypothesis h at (x, y).
__device__ void view_angles(const PmCam& rc, const float* Rs, const float* ts, const Hyp& h, int x, int y, float* cos_tri,
                            float* cos_inc) {
  float ray[3];
  ray_of(rc, x, y, ray);
  const float X[3] = {h.d * ray[0], h.d * ray[1], h.d * ray[2]};
  // source centre in the reference frame: C = -Rs^T ts
  const float C[3] = {-(Rs[0] * ts[0] + Rs[3] * ts[1] + Rs[6] * ts[2]), -(Rs[1] * ts[0] + Rs[4] * ts[1] + Rs[7] * ts[2]),
                      -(Rs[2] * ts[0] + Rs[5] * ts[1] + Rs[8] * ts[2])};
  const float v[3] = {X[0] - C[0], X[1] - C[1], X[2] - C[2]};
  const float nx = sqrtf(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]), nv = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  *cos_tri = (X[0] * v[0] + X[1] * v[1] + X[2] * v[2]) / (nx * nv);
  *cos_inc = -(h.n0 * v[0] + h.n1 * v[1] + h.n2 * v[2]) / nv;
}

__device__ __forceinline__ void face_camera(const float* ray, Hyp* h) {
  if (h->n0 * ray[0] + h->n1 * ray[1] + h->n2 * ray[2] > 0.f) {
    h->n0 = -h->n0;
    h->n1 = -h->n1;
    h->n2 = -h->n2;
  }
}

// A random hypothesis from three draws starting at `draw`: depth uniform in the range, normal uniform on the sphere,
// turned towards the camera.
__device__ Hyp random_hyp(uint64_t seed, int image, int pixel, int iter, int sweep, int draw, float dmin, float dmax,
                          const float* ray) {
  const float u0 = pm_uniform(seed, image, pixel, iter, sweep, draw);
  const float u1 = pm_uniform(seed, image, pixel, iter, sweep, draw + 1);
  const float u2 = pm_uniform(seed, image, pixel, iter, sweep, draw + 2);
  const float z = 2.0f * u1 - 1.0f, phi = 6.2831853f * u2;
  const float rxy = sqrtf(fmaxf(1.0f - z * z, 0.0f));
  Hyp h{dmin + u0 * (dmax - dmin), rxy * cosf(phi), rxy * sinf(phi), z};
  face_camera(ray, &h);
  return h;
}

struct PmArgs {
  const uint8_t* images;
  const float* dmaps;
  const PmCam* cams;
  const PmProblem* probs;
  const int64_t* line_start;  // [n_probs + 1]: lines of this sweep direction per problem, prefix sums
  int n_probs;
  float* depth;
  float* normal;
  float* bmsg;         // [sel_off + pixel * n_src + s]: backward message of source s at the pixel, of the running sweep
  const float* refwin; // [3 * (map_off + pixel)]: the reference's weighted window sums (sw, swr, swrr)
  PmParams P;
  uint64_t seed;
  int iter, sweep;
  float perturb;
  unsigned long long* counter;  // window samples evaluated
};

__device__ __forceinline__ void load_hyp(const PmArgs& a, int64_t p, Hyp* h) {
  h->d = a.depth[p];
  h->n0 = a.normal[3 * p];
  h->n1 = a.normal[3 * p + 1];
  h->n2 = a.normal[3 * p + 2];
}

// Per-source photometric + geometric cost of h for every source (lane s holds source s's), and lane s's angles.
struct SrcEval {
  float cost, cos_tri, cos_inc, geom;
};

__device__ SrcEval eval_all(const PmArgs& a, const PmProblem& pr, const PmCam& rc, const uint8_t* rimg, const Hyp& h, int x,
                            int y, const RefWin& rw, int lane, unsigned long long* samples) {
  SrcEval e{2.0f, 1.0f, 0.0f, 0.0f};
  for (int s = 0; s < pr.n_src; ++s) {
    const PmCam& sc = a.cams[pr.src[s]];
    const float c = photo_cost(a.P, rc, rimg, sc, a.images + sc.img_off, pr.Rs[s], pr.ts[s], h, x, y, rw, lane, samples);
    if (lane == s) e.cost = c;
  }
  if (lane < pr.n_src) {
    view_angles(rc, pr.Rs[lane], pr.ts[lane], h, x, y, &e.cos_tri, &e.cos_inc);
    if (a.P.geom) {
      const PmCam& sc = a.cams[pr.src[lane]];
      e.geom = geom_error(rc, sc, a.dmaps + sc.dmap_off, pr.Rs[lane], pr.ts[lane], h, x, y, a.P.geom_max);
    }
  }
  return e;
}

// Which problem a global line index belongs to.
__device__ __forceinline__ int problem_of(const int64_t* start, int n, int64_t line) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (start[mid] <= line) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(32 * kWarpsPerCta) b2m_pm_init_kernel(PmArgs a, const float* init_depth,
                                                                        const float* init_normal) {
  const int64_t line = static_cast<int64_t>(blockIdx.x) * kWarpsPerCta + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (line >= a.line_start[a.n_probs]) return;
  const int k = problem_of(a.line_start, a.n_probs, line);
  const PmProblem& pr = a.probs[k];
  const PmCam& rc = a.cams[pr.ref];
  const int x = static_cast<int>(line - a.line_start[k]);
  for (int y = lane; y < rc.H; y += 32) {
    const int pixel = y * rc.W + x;
    const int64_t p = pr.map_off + pixel;
    float ray[3];
    ray_of(rc, x, y, ray);
    Hyp h;
    if (init_depth && init_depth[p] > 0.f) {
      h = Hyp{init_depth[p], init_normal[3 * p], init_normal[3 * p + 1], init_normal[3 * p + 2]};
    } else {
      h = random_hyp(a.seed, pr.key, pixel, 0, kInitSweep, 0, pr.dmin, pr.dmax, ray);
    }
    a.depth[p] = h.d;
    a.normal[3 * p] = h.n0;
    a.normal[3 * p + 1] = h.n1;
    a.normal[3 * p + 2] = h.n2;
  }
}

// The reference's weighted window sums of every pixel, once per batch (one warp per column).
__global__ void __launch_bounds__(32 * kWarpsPerCta) b2m_pm_refwin_kernel(PmArgs a, float* refwin) {
  const int64_t line = static_cast<int64_t>(blockIdx.x) * kWarpsPerCta + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (line >= a.line_start[a.n_probs]) return;
  const int k = problem_of(a.line_start, a.n_probs, line);
  const PmProblem& pr = a.probs[k];
  const PmCam& rc = a.cams[pr.ref];
  const uint8_t* rimg = a.images + rc.img_off;
  const int x = static_cast<int>(line - a.line_start[k]);
  for (int y = 0; y < rc.H; ++y) {
    const RefWin rw = ref_window(a.P, rimg, rc.W, rc.H, x, y, lane);
    if (lane == 0) {
      const int64_t p = pr.map_off + y * rc.W + x;
      refwin[3 * p] = rw.sw;
      refwin[3 * p + 1] = rw.swr;
      refwin[3 * p + 2] = rw.swrr;
    }
  }
}

__device__ __forceinline__ RefWin load_refwin(const PmArgs& a, int64_t p) {
  return RefWin{a.refwin[3 * p], a.refwin[3 * p + 1], a.refwin[3 * p + 2]};
}

// P(visible at this pixel | message m of the neighbouring pixel): one step of the chain.
__device__ __forceinline__ float hmm_predict(float m) { return m * kStay + (1.0f - m) * (1.0f - kStay); }
// The message after observing `cost` at this pixel, from the predicted visibility.
__device__ __forceinline__ float hmm_update(const PmParams& P, float pred, float cost) {
  const float z1 = pred * expf(-cost * cost * P.inv_2ncc);
  const float z0 = (1.0f - pred) * kUniformProb;
  return z1 / (z0 + z1);
}
// Posterior visibility from the forward message (this pixel's observation included) and the predicted backward one.
__device__ __forceinline__ float hmm_posterior(float f, float b) {
  const float v = f * b, o = (1.0f - f) * (1.0f - b);
  return v / (v + o);
}

// Writes the predicted backward message of every pixel of the line (lane s: source s), walking it against `forward`,
// from the current hypotheses.
__device__ void backward_messages(const PmArgs& a, const PmProblem& pr, const PmCam& rc, const uint8_t* rimg, int l,
                                  bool vertical, bool forward, int lane, unsigned long long* samples) {
  const int len = vertical ? rc.H : rc.W;
  float b = 0.5f;
  for (int i = len - 1; i >= 0; --i) {
    const int j = forward ? i : len - 1 - i;
    const int x = vertical ? l : j, y = vertical ? j : l;
    const int pixel = y * rc.W + x;
    const int64_t p = pr.map_off + pixel;
    const float pred = hmm_predict(b);
    if (lane < pr.n_src) a.bmsg[pr.sel_off + static_cast<int64_t>(pixel) * pr.n_src + lane] = pred;
    Hyp cur;
    load_hyp(a, p, &cur);
    const SrcEval e = eval_all(a, pr, rc, rimg, cur, x, y, load_refwin(a, p), lane, samples);
    if (lane < pr.n_src) b = hmm_update(a.P, pred, e.cost);
  }
}

// Source selection probability of lane s's source: its posterior visibility times the triangulation-angle and
// incident-angle priors of the current hypothesis.
__device__ __forceinline__ float select_prob(const PmParams& P, const SrcEval& e, float post, int lane, int n_src) {
  if (lane >= n_src) return 0.f;
  const float tri = acosf(fminf(fmaxf(e.cos_tri, -1.f), 1.f));
  const float prior_tri = tri < P.min_tri ? (tri / P.min_tri) * (tri / P.min_tri) : 1.0f;
  const float one_m = 1.0f - e.cos_inc;
  const float prior_inc = e.cos_inc > 0.f ? expf(-one_m * one_m * P.inv_2inc) : 0.f;
  return post * prior_tri * prior_inc;
}

// One sweep over every line of the batch.  First the backward messages of the line, from its current hypotheses; then
// the line in sweep order: the forward message of each source (from the previous pixel's message and the current
// hypothesis's cost), the posterior visibility with the backward message, the draws of the sources from posterior x
// priors, the candidates (current, propagated, random, perturbed) scored as the mean cost over the draws, the best kept.
__global__ void __launch_bounds__(32 * kWarpsPerCta) b2m_pm_sweep_kernel(PmArgs a) {
  const int64_t line = static_cast<int64_t>(blockIdx.x) * kWarpsPerCta + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (line >= a.line_start[a.n_probs]) return;
  const int k = problem_of(a.line_start, a.n_probs, line);
  const PmProblem& pr = a.probs[k];
  const PmCam& rc = a.cams[pr.ref];
  const uint8_t* rimg = a.images + rc.img_off;
  const int l = static_cast<int>(line - a.line_start[k]);
  const bool vertical = a.sweep < 2, forward = (a.sweep & 1) == 0;
  const int len = vertical ? rc.H : rc.W;
  unsigned long long samples = 0;
  backward_messages(a, pr, rc, rimg, l, vertical, forward, lane, &samples);
  __syncwarp();
  float fwd = 0.5f;
  Hyp prev{};
  for (int i = 0; i < len; ++i) {
    const int j = forward ? i : len - 1 - i;
    const int x = vertical ? l : j, y = vertical ? j : l;
    const int pixel = y * rc.W + x;
    const int64_t p = pr.map_off + pixel;
    float ray[3];
    ray_of(rc, x, y, ray);
    Hyp cur;
    load_hyp(a, p, &cur);
    const RefWin rw = load_refwin(a, p);
    const SrcEval e = eval_all(a, pr, rc, rimg, cur, x, y, rw, lane, &samples);
    float post = 0.f;
    if (lane < pr.n_src) {
      fwd = hmm_update(a.P, hmm_predict(fwd), e.cost);
      post = hmm_posterior(fwd, a.bmsg[pr.sel_off + static_cast<int64_t>(pixel) * pr.n_src + lane]);
    }
    // inclusive scan of the selection probabilities over the lanes (= sources)
    const float prob = select_prob(a.P, e, post, lane, pr.n_src);
    float cum = prob;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float v = __shfl_up_sync(0xffffffffu, cum, o);
      if (lane >= o) cum += v;
    }
    const float total = __shfl_sync(0xffffffffu, cum, 31);
    const bool uniform = !(total > 1e-20f);
    int count = 0;
    for (int q = 0; q < a.P.num_samples; ++q) {
      const float u = pm_uniform(a.seed, pr.key, pixel, a.iter, a.sweep, q);
      if (uniform) {
        count += (lane == min(static_cast<int>(u * pr.n_src), pr.n_src - 1)) ? 1 : 0;
      } else {
        const float t = u * total;
        const float lo = cum - prob;
        // the first source whose cumulative probability passes t; the last one catches rounding at the top
        count += (lane < pr.n_src && prob > 0.f && t >= lo && (t < cum || lane == pr.n_src - 1)) ? 1 : 0;
      }
    }
    const float inv_n = 1.0f / static_cast<float>(a.P.num_samples);
    auto total_cost = [&](float c, float g) {
      const float v = lane < pr.n_src ? static_cast<float>(count) * (c + a.P.geom_reg * g) : 0.f;
      return warp_sum(v) * inv_n;
    };
    float best_cost = total_cost(e.cost, e.geom);
    Hyp best = cur;
    const unsigned sel = __ballot_sync(0xffffffffu, count > 0 && lane < pr.n_src);
    Hyp cand[3];
    int n_cand = 0;
    if (i > 0) {  // propagated: the previous pixel's plane, intersected with this pixel's ray
      const float dp = prev.n0 * ray[0] + prev.n1 * ray[1] + prev.n2 * ray[2];
      float pray[3];
      const int px = vertical ? x : (forward ? x - 1 : x + 1), py = vertical ? (forward ? y - 1 : y + 1) : y;
      ray_of(rc, px, py, pray);
      const float num = prev.d * (prev.n0 * pray[0] + prev.n1 * pray[1] + prev.n2 * pray[2]);
      float d = num / dp;
      if (!(d > 0.f) || !isfinite(d)) d = prev.d;
      cand[n_cand++] = Hyp{fminf(fmaxf(d, pr.dmin), pr.dmax), prev.n0, prev.n1, prev.n2};
    }
    const int q0 = a.P.num_samples;
    cand[n_cand++] = random_hyp(a.seed, pr.key, pixel, a.iter, a.sweep, q0, pr.dmin, pr.dmax, ray);
    {  // perturbed current
      const float u0 = pm_uniform(a.seed, pr.key, pixel, a.iter, a.sweep, q0 + 3);
      const float u1 = pm_uniform(a.seed, pr.key, pixel, a.iter, a.sweep, q0 + 4);
      const float u2 = pm_uniform(a.seed, pr.key, pixel, a.iter, a.sweep, q0 + 5);
      const float u3 = pm_uniform(a.seed, pr.key, pixel, a.iter, a.sweep, q0 + 6);
      const float d = cur.d * (1.0f + 0.05f * a.perturb * (2.0f * u0 - 1.0f));
      float m0 = cur.n0 + 0.5f * a.perturb * (2.0f * u1 - 1.0f), m1 = cur.n1 + 0.5f * a.perturb * (2.0f * u2 - 1.0f),
            m2 = cur.n2 + 0.5f * a.perturb * (2.0f * u3 - 1.0f);
      const float inv = 1.0f / sqrtf(m0 * m0 + m1 * m1 + m2 * m2);
      m0 *= inv;
      m1 *= inv;
      m2 *= inv;
      Hyp h{fminf(fmaxf(d, pr.dmin), pr.dmax), m0, m1, m2};
      if (m0 * ray[0] + m1 * ray[1] + m2 * ray[2] > 0.f) {
        h.n0 = cur.n0;
        h.n1 = cur.n1;
        h.n2 = cur.n2;
      }
      cand[n_cand++] = h;
    }
    for (int c = 0; c < n_cand; ++c) {
      float cs = 2.0f, gs = 0.f;
      for (int s = 0; s < pr.n_src; ++s) {
        if (!((sel >> s) & 1u)) continue;
        const PmCam& sc = a.cams[pr.src[s]];
        const float v = photo_cost(a.P, rc, rimg, sc, a.images + sc.img_off, pr.Rs[s], pr.ts[s], cand[c], x, y, rw, lane,
                                   &samples);
        if (lane == s) cs = v;
      }
      if (a.P.geom && lane < pr.n_src && ((sel >> lane) & 1u)) {
        const PmCam& sc = a.cams[pr.src[lane]];
        gs = geom_error(rc, sc, a.dmaps + sc.dmap_off, pr.Rs[lane], pr.ts[lane], cand[c], x, y, a.P.geom_max);
      }
      const float tc = total_cost(cs, gs);
      if (tc < best_cost) {
        best_cost = tc;
        best = cand[c];
      }
    }
    if (lane == 0) {
      a.depth[p] = best.d;
      a.normal[3 * p] = best.n0;
      a.normal[3 * p + 1] = best.n1;
      a.normal[3 * p + 2] = best.n2;
    }
    prev = best;
    __syncwarp();
  }
  for (int o = 16; o > 0; o >>= 1) samples += __shfl_xor_sync(0xffffffffu, samples, o);
  if (lane == 0) atomicAdd(a.counter, samples);
}

// The filter, one warp per column over the final hypotheses: backward and forward messages as in a downward sweep; a
// source is selected at a pixel when its posterior visibility is at least 1/2.  A pixel is kept when at least
// filter_min_num_consistent selected sources pass the NCC, triangulation-angle and (in the geometric pass)
// forward-backward error tests; others get depth 0 and normal 0.
__global__ void __launch_bounds__(32 * kWarpsPerCta) b2m_pm_filter_kernel(PmArgs a) {
  const int64_t line = static_cast<int64_t>(blockIdx.x) * kWarpsPerCta + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (line >= a.line_start[a.n_probs]) return;
  const int k = problem_of(a.line_start, a.n_probs, line);
  const PmProblem& pr = a.probs[k];
  const PmCam& rc = a.cams[pr.ref];
  const uint8_t* rimg = a.images + rc.img_off;
  const int x = static_cast<int>(line - a.line_start[k]);
  unsigned long long samples = 0;
  backward_messages(a, pr, rc, rimg, x, true, true, lane, &samples);
  __syncwarp();
  float fwd = 0.5f;
  for (int y = 0; y < rc.H; ++y) {
    const int pixel = y * rc.W + x;
    const int64_t p = pr.map_off + pixel;
    Hyp cur;
    load_hyp(a, p, &cur);
    const SrcEval e = eval_all(a, pr, rc, rimg, cur, x, y, load_refwin(a, p), lane, &samples);
    float post = 0.f;
    if (lane < pr.n_src) {
      fwd = hmm_update(a.P, hmm_predict(fwd), e.cost);
      post = hmm_posterior(fwd, a.bmsg[pr.sel_off + static_cast<int64_t>(pixel) * pr.n_src + lane]);
    }
    const float tri = acosf(fminf(fmaxf(e.cos_tri, -1.f), 1.f));
    const bool ok = lane < pr.n_src && post >= 0.5f && e.cost <= a.P.filter_max_cost && tri >= a.P.filter_min_tri &&
                    (!a.P.geom || e.geom <= a.P.filter_geom_max);
    const int n_ok = __popc(__ballot_sync(0xffffffffu, ok));
    __syncwarp();
    if (lane == 0 && n_ok < a.P.filter_min_num_consistent) {
      a.depth[p] = 0.f;
      a.normal[3 * p] = a.normal[3 * p + 1] = a.normal[3 * p + 2] = 0.f;
    }
    __syncwarp();
  }
  for (int o = 16; o > 0; o >>= 1) samples += __shfl_xor_sync(0xffffffffu, samples, o);
  if (lane == 0) atomicAdd(a.counter, samples);
}

// b2m_debug_patch_match_cost: one warp per query.
__global__ void __launch_bounds__(32 * kWarpsPerCta) b2m_pm_debug_kernel(PmArgs a, const float* q, int n, float* out) {
  const int i = blockIdx.x * kWarpsPerCta + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  const PmProblem& pr = a.probs[0];
  const PmCam& rc = a.cams[pr.ref];
  const uint8_t* rimg = a.images + rc.img_off;
  const int x = static_cast<int>(q[7 * i]), y = static_cast<int>(q[7 * i + 1]), s = static_cast<int>(q[7 * i + 6]);
  const Hyp h{q[7 * i + 2], q[7 * i + 3], q[7 * i + 4], q[7 * i + 5]};
  const PmCam& sc = a.cams[pr.src[s]];
  const RefWin rw = ref_window(a.P, rimg, rc.W, rc.H, x, y, lane);
  const float c = photo_cost(a.P, rc, rimg, sc, a.images + sc.img_off, pr.Rs[s], pr.ts[s], h, x, y, rw, lane, nullptr);
  if (lane == 0) {
    out[3 * i] = c;
    out[3 * i + 1] = sc.dmap_off >= 0 ? geom_error(rc, sc, a.dmaps + sc.dmap_off, pr.Rs[s], pr.ts[s], h, x, y, a.P.geom_max)
                                      : 0.f;
    float ray[3], nray[3];
    ray_of(rc, x, y, ray);
    ray_of(rc, x, y + 1, nray);
    const float num = h.d * (h.n0 * ray[0] + h.n1 * ray[1] + h.n2 * ray[2]);
    out[3 * i + 2] = num / (h.n0 * nray[0] + h.n1 * nray[1] + h.n2 * nray[2]);
  }
}

// ---- host side ----
struct PmState {
  int n_images = 0;
  std::vector<PmCam> cams;
  std::vector<std::array<double, 16>> cam_params;
  DeviceArray<uint8_t> images;
  DeviceArray<float> dmaps;
  DeviceArray<PmCam> d_cams;
  DeviceArray<PmProblem> d_probs;
  DeviceArray<int64_t> d_lines;  // [2][n + 1]
  DeviceArray<float> depth, normal, init_depth, init_normal, bmsg, refwin;
  DeviceArray<float> d_q, d_out;
};

PmState* pm_state(b2m_ctx* ctx) {
  if (!ctx->pm_state) ctx->pm_state = new PmState();
  return static_cast<PmState*>(ctx->pm_state);
}

int check_opts(b2m_ctx* ctx, const b2m_patch_match_opts* o, PmParams* P) {
  auto bad = [&](const char* what) { return fail(ctx, B2M_EINVAL, std::string("[patch_match.cu] Check Failed: ") + what); };
  if (!o || o->struct_size != sizeof(b2m_patch_match_opts)) return bad("opts != NULL (struct_size)");
  if (!(o->window_radius > 0 && o->window_radius <= kMaxWindowRadius)) return bad("0 < window_radius <= 32");
  if (!(o->window_step > 0 && o->window_step <= 2)) return bad("window_step in {1, 2}");
  if (!(o->num_samples > 0)) return bad("num_samples > 0");
  if (!(o->num_iterations > 0)) return bad("num_iterations > 0");
  if (!(o->sigma_color > 0.f)) return bad("sigma_color > 0");
  if (!(o->ncc_sigma > 0.f)) return bad("ncc_sigma > 0");
  if (!(o->min_triangulation_angle >= 0.f && o->min_triangulation_angle < 180.f)) return bad("min_triangulation_angle");
  if (!(o->incident_angle_sigma > 0.f)) return bad("incident_angle_sigma > 0");
  if (!(o->filter_min_num_consistent >= 0)) return bad("filter_min_num_consistent >= 0");
  const float ss = o->sigma_spatial > 0.f ? o->sigma_spatial : static_cast<float>(o->window_radius);
  const float deg = 3.14159265358979f / 180.0f;
  P->radius = o->window_radius;
  P->step = o->window_step;
  P->side = 2 * o->window_radius / o->window_step + 1;
  P->n_win = P->side * P->side;
  P->num_samples = o->num_samples;
  P->geom = o->geom_consistency ? 1 : 0;
  P->filter = o->filter ? 1 : 0;
  P->filter_min_num_consistent = o->filter_min_num_consistent;
  P->inv_2ss = 1.0f / (2.0f * ss * ss);
  P->inv_2sc = 1.0f / (2.0f * o->sigma_color * o->sigma_color);
  P->inv_2ncc = 1.0f / (2.0f * o->ncc_sigma * o->ncc_sigma);
  P->min_tri = fmaxf(o->min_triangulation_angle * deg, 1e-6f);
  P->inv_2inc = 1.0f / (2.0f * o->incident_angle_sigma * o->incident_angle_sigma);
  P->geom_reg = o->geom_consistency_regularizer;
  P->geom_max = o->geom_consistency_max_cost;
  P->filter_max_cost = 1.0f - o->filter_min_ncc;
  P->filter_min_tri = o->filter_min_triangulation_angle * deg;
  P->filter_geom_max = o->filter_geom_consistency_max_cost;
  return B2M_OK;
}

// The problem as the kernels see it: indices checked, source poses relative to the reference in fp64.
int make_problem(b2m_ctx* ctx, const PmState& S, const b2m_patch_match_problem& q, bool geom, PmProblem* out) {
  auto bad = [&](const std::string& what) { return fail(ctx, B2M_EINVAL, "[patch_match.cu] Check Failed: " + what); };
  if (q.struct_size != sizeof(b2m_patch_match_problem)) return bad("b2m_patch_match_problem.struct_size");
  if (q.ref < 0 || q.ref >= S.n_images) return bad("ref is an index into the image set");
  if (q.n_src < 1 || q.n_src > kMaxSrc || !q.src) return bad("1 <= n_src <= 32");
  if (!(q.depth_min > 0.f && q.depth_max > q.depth_min)) return bad("0 < depth_min < depth_max");
  if (!q.init_normal != !q.init_depth) return bad("init_depth and init_normal come together");
  std::memset(out, 0, sizeof(*out));
  out->ref = q.ref;
  out->key = q.image_id;
  out->n_src = q.n_src;
  out->dmin = q.depth_min;
  out->dmax = q.depth_max;
  const auto& r = S.cam_params[q.ref];
  for (int s = 0; s < q.n_src; ++s) {
    const int j = q.src[s];
    if (j < 0 || j >= S.n_images || j == q.ref) return bad("sources are indices into the image set other than ref");
    for (int t = 0; t < s; ++t)
      if (q.src[t] == j) return bad("sources are distinct");
    if (geom && S.cams[j].dmap_off < 0) return bad("geom_consistency: every source has a depth map");
    out->src[s] = j;
    const auto& c = S.cam_params[j];
    // src_from_ref = src_from_world * ref_from_world^-1: R = Rs Rr^T, t = ts - R tr
    double R[9];
    for (int i = 0; i < 3; ++i)
      for (int k = 0; k < 3; ++k) {
        double v = 0.0;
        for (int m = 0; m < 3; ++m) v += c[4 + i * 3 + m] * r[4 + k * 3 + m];
        R[i * 3 + k] = v;
      }
    for (int i = 0; i < 9; ++i) out->Rs[s][i] = static_cast<float>(R[i]);
    for (int i = 0; i < 3; ++i) {
      double v = c[13 + i];
      for (int k = 0; k < 3; ++k) v -= R[i * 3 + k] * r[13 + k];
      out->ts[s][i] = static_cast<float>(v);
    }
  }
  return B2M_OK;
}

}  // namespace

void pm_release(b2m_ctx* ctx) {
  delete static_cast<PmState*>(ctx->pm_state);
  ctx->pm_state = nullptr;
}

}  // namespace b2m

using namespace b2m;

extern "C" {

void b2m_patch_match_opts_default(b2m_patch_match_opts* o) {
  if (!o) return;
  std::memset(o, 0, sizeof(*o));
  o->struct_size = sizeof(*o);
  o->window_radius = 5;
  o->window_step = 1;
  o->num_samples = 15;
  o->num_iterations = 5;
  o->geom_consistency = 0;
  o->filter = 1;
  o->filter_min_num_consistent = 2;
  o->sigma_spatial = -1.0f;
  o->sigma_color = 0.2f;
  o->ncc_sigma = 0.6f;
  o->min_triangulation_angle = 1.0f;
  o->incident_angle_sigma = 0.9f;
  o->geom_consistency_regularizer = 0.3f;
  o->geom_consistency_max_cost = 3.0f;
  o->filter_min_ncc = 0.1f;
  o->filter_min_triangulation_angle = 3.0f;
  o->filter_geom_consistency_max_cost = 1.0f;
}

int b2m_patch_match_set_images(b2m_ctx* ctx, int32_t n, const b2m_image* images, const double* cameras,
                               const float* const* depth_maps) {
  if (!ctx) return B2M_EINVAL;
  if (n < 1 || !images || !cameras)
    return fail(ctx, B2M_EINVAL, "[patch_match.cu] Check Failed: n >= 1 && images && cameras");
  PmState* S = pm_state(ctx);
  S->n_images = 0;
  std::vector<PmCam> cams(n);
  std::vector<std::array<double, 16>> par(n);
  int64_t img_bytes = 0, map_px = 0;
  for (int i = 0; i < n; ++i) {
    const b2m_image& im = images[i];
    if (im.width < 1 || im.height < 1 || !im.data || im.stride < im.width)
      return fail(ctx, B2M_EINVAL, "[patch_match.cu] Check Failed: image " + std::to_string(i) + " is a non-empty grey image");
    std::copy(cameras + 16 * i, cameras + 16 * i + 16, par[i].begin());
    if (!(par[i][0] > 0.0) || !(par[i][1] > 0.0))
      return fail(ctx, B2M_EINVAL, "[patch_match.cu] Check Failed: camera " + std::to_string(i) + " focal length > 0");
    PmCam& c = cams[i];
    c.fx = static_cast<float>(par[i][0]);
    c.fy = static_cast<float>(par[i][1]);
    c.cx = static_cast<float>(par[i][2]);
    c.cy = static_cast<float>(par[i][3]);
    for (int k = 0; k < 9; ++k) c.R[k] = static_cast<float>(par[i][4 + k]);
    for (int k = 0; k < 3; ++k) c.t[k] = static_cast<float>(par[i][13 + k]);
    c.W = im.width;
    c.H = im.height;
    c.img_off = img_bytes;
    img_bytes += static_cast<int64_t>(im.width) * im.height;
    c.dmap_off = -1;
    if (depth_maps && depth_maps[i]) {
      c.dmap_off = map_px;
      map_px += static_cast<int64_t>(im.width) * im.height;
    }
  }
  size_t free_b = 0, total_b = 0;
  cudaSetDevice(ctx->device);
  cudaMemGetInfo(&free_b, &total_b);
  // ensure() frees a block that is too small before allocating: the blocks held now count as available
  const double need = static_cast<double>(img_bytes) + 4.0 * static_cast<double>(map_px);
  const double avail = static_cast<double>(free_b) + static_cast<double>(S->images.capacity()) +
                       4.0 * static_cast<double>(S->dmaps.capacity());
  if (need > avail) {
    char b[256];
    snprintf(b, sizeof(b), "[patch_match.cu] the workspace's images and depth maps need %.1f MB of device memory, %.1f MB "
             "are available", need / 1e6, avail / 1e6);
    return fail(ctx, B2M_ENOMEM, b);
  }
  B2M_CUDA_TRY(ctx, S->images.ensure(img_bytes));
  B2M_CUDA_TRY(ctx, S->dmaps.ensure(map_px));
  B2M_CUDA_TRY(ctx, S->d_cams.ensure(n));
  for (int i = 0; i < n; ++i) {
    B2M_CUDA_TRY(ctx, cudaMemcpy2DAsync(S->images + cams[i].img_off, cams[i].W, images[i].data, images[i].stride, cams[i].W,
                                        cams[i].H, cudaMemcpyHostToDevice, ctx->stream));
    if (cams[i].dmap_off >= 0)
      B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->dmaps + cams[i].dmap_off, depth_maps[i],
                                        sizeof(float) * cams[i].W * cams[i].H, cudaMemcpyHostToDevice, ctx->stream));
  }
  B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->d_cams, cams.data(), sizeof(PmCam) * n, cudaMemcpyHostToDevice, ctx->stream));
  B2M_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  S->cams = std::move(cams);
  S->cam_params = std::move(par);
  S->n_images = n;
  return B2M_OK;
}

int b2m_patch_match_batch(b2m_ctx* ctx, const b2m_patch_match_problem* problems, int32_t n, const b2m_patch_match_opts* opts,
                          b2m_depth_maps** out) {
  if (!ctx) return B2M_EINVAL;
  if (!out || n < 0 || (n > 0 && !problems))
    return fail(ctx, B2M_EINVAL, "[patch_match.cu] Check Failed: out != NULL && problems");
  *out = nullptr;
  PmParams P;
  if (int rc = check_opts(ctx, opts, &P)) return rc;
  PmState* S = pm_state(ctx);
  if (S->n_images == 0) return fail(ctx, B2M_ESTATE, "[patch_match.cu] b2m_patch_match_set_images must come first");
  std::vector<PmProblem> probs(n);
  std::vector<int64_t> lines(2 * (n + 1), 0);
  int64_t px = 0, sel = 0;
  bool any_init = false;
  for (int k = 0; k < n; ++k) {
    if (int rc = make_problem(ctx, *S, problems[k], P.geom != 0, &probs[k])) return rc;
    const PmCam& rc = S->cams[problems[k].ref];
    probs[k].map_off = px;
    probs[k].sel_off = sel;
    px += static_cast<int64_t>(rc.W) * rc.H;
    sel += static_cast<int64_t>(rc.W) * rc.H * problems[k].n_src;
    lines[k + 1] = lines[k] + rc.W;
    lines[n + 1 + k + 1] = lines[n + 1 + k] + rc.H;
    any_init = any_init || problems[k].init_depth;
  }
  std::unique_ptr<b2m_depth_maps> M(new (std::nothrow) b2m_depth_maps());
  if (!M) return fail(ctx, B2M_ENOMEM, "[patch_match.cu] out of host memory");
  M->off.push_back(0);
  for (int k = 0; k < n; ++k) {
    const PmCam& rc = S->cams[problems[k].ref];
    M->width.push_back(rc.W);
    M->height.push_back(rc.H);
    M->off.push_back(M->off.back() + static_cast<int64_t>(rc.W) * rc.H);
  }
  if (n == 0) {
    *out = M.release();
    return B2M_OK;
  }
  cudaSetDevice(ctx->device);
  {  // depth, normal, window sums (7 floats per pixel), backward messages, start maps (4 floats per pixel)
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    const double need = 4.0 * (7.0 * px + sel + (any_init ? 4.0 * px : 0.0));
    const double avail = static_cast<double>(free_b) +
                         4.0 * (S->depth.capacity() + S->normal.capacity() + S->refwin.capacity() + S->bmsg.capacity() +
                                S->init_depth.capacity() + S->init_normal.capacity());
    if (need > avail) {
      char b[256];
      snprintf(b, sizeof(b), "[patch_match.cu] the batch's maps need %.1f MB of device memory, %.1f MB are available",
               need / 1e6, avail / 1e6);
      return fail(ctx, B2M_ENOMEM, b);
    }
  }
  cudaStream_t st = ctx->stream;
  B2M_CUDA_TRY(ctx, S->d_probs.ensure(n));
  B2M_CUDA_TRY(ctx, S->d_lines.ensure(lines.size()));
  B2M_CUDA_TRY(ctx, S->depth.ensure(px));
  B2M_CUDA_TRY(ctx, S->normal.ensure(3 * px));
  B2M_CUDA_TRY(ctx, S->refwin.ensure(3 * px));
  B2M_CUDA_TRY(ctx, S->bmsg.ensure(sel));
  B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->d_probs, probs.data(), sizeof(PmProblem) * n, cudaMemcpyHostToDevice, st));
  B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->d_lines, lines.data(), sizeof(int64_t) * lines.size(), cudaMemcpyHostToDevice, st));
  if (any_init) {
    B2M_CUDA_TRY(ctx, S->init_depth.ensure(px));
    B2M_CUDA_TRY(ctx, S->init_normal.ensure(3 * px));
    B2M_CUDA_TRY(ctx, cudaMemsetAsync(S->init_depth, 0, sizeof(float) * px, st));
    for (int k = 0; k < n; ++k) {
      if (!problems[k].init_depth) continue;
      const int64_t m = M->off[k + 1] - M->off[k];
      B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->init_depth + probs[k].map_off, problems[k].init_depth, sizeof(float) * m,
                                        cudaMemcpyHostToDevice, st));
      B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->init_normal + 3 * probs[k].map_off, problems[k].init_normal,
                                        sizeof(float) * 3 * m, cudaMemcpyHostToDevice, st));
    }
  }
  PmArgs a{};
  a.images = S->images;
  a.dmaps = S->dmaps;
  a.cams = S->d_cams;
  a.probs = S->d_probs;
  a.n_probs = n;
  a.depth = S->depth;
  a.normal = S->normal;
  a.bmsg = S->bmsg;
  a.refwin = S->refwin;
  a.P = P;
  a.seed = ctx->seed;
  a.counter = ctx->d_counters + kPmCounters;
  const int64_t* d_lines = S->d_lines;
  auto grid = [](int64_t total) { return static_cast<unsigned>((total + kWarpsPerCta - 1) / kWarpsPerCta); };
  a.line_start = d_lines;
  b2m_pm_refwin_kernel<<<grid(lines[n]), 32 * kWarpsPerCta, 0, st>>>(a, S->refwin);
  B2M_CUDA_TRY(ctx, cudaGetLastError());
  b2m_pm_init_kernel<<<grid(lines[n]), 32 * kWarpsPerCta, 0, st>>>(a, any_init ? static_cast<const float*>(S->init_depth) : nullptr,
                                                                  any_init ? static_cast<const float*>(S->init_normal) : nullptr);
  B2M_CUDA_TRY(ctx, cudaGetLastError());
  uint64_t launches = 2;
  for (int it = 0; it < opts->num_iterations; ++it) {
    for (int sw = 0; sw < 4; ++sw) {
      if (ctx->stop) return fail(ctx, B2M_ESTOPPED, "[patch_match.cu] stopped by b2m_request_stop");
      a.iter = it;
      a.sweep = sw;
      a.perturb = std::ldexp(1.0f, -it);
      a.line_start = sw < 2 ? d_lines : d_lines + (n + 1);
      const int64_t total = sw < 2 ? lines[n] : lines[2 * n + 1];
      b2m_pm_sweep_kernel<<<grid(total), 32 * kWarpsPerCta, 0, st>>>(a);
      B2M_CUDA_TRY(ctx, cudaGetLastError());
      ++launches;
    }
    B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));  // lets b2m_request_stop take effect between iterations
  }
  if (P.filter) {
    a.line_start = d_lines;
    b2m_pm_filter_kernel<<<grid(lines[n]), 32 * kWarpsPerCta, 0, st>>>(a);
    B2M_CUDA_TRY(ctx, cudaGetLastError());
    ++launches;
  }
  try {
    M->depth.resize(px);
    M->normal.resize(3 * px);
  } catch (const std::bad_alloc&) {
    return fail(ctx, B2M_ENOMEM, "[patch_match.cu] out of host memory for the maps");
  }
  B2M_CUDA_TRY(ctx, cudaMemcpyAsync(M->depth.data(), S->depth, sizeof(float) * px, cudaMemcpyDeviceToHost, st));
  B2M_CUDA_TRY(ctx, cudaMemcpyAsync(M->normal.data(), S->normal, sizeof(float) * 3 * px, cudaMemcpyDeviceToHost, st));
  B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
  ctx->stats.kernel_launches += launches;
  ctx->stats.pm_problems += n;
  ctx->stats.pm_pixel_updates += static_cast<uint64_t>(px) * 4 * opts->num_iterations;
  *out = M.release();
  return B2M_OK;
}

int b2m_depth_maps_get(const b2m_depth_maps* m, int32_t k, b2m_depth_map_view* out) {
  if (!m || !out || k < 0 || k >= static_cast<int32_t>(m->width.size())) return B2M_EINVAL;
  out->struct_size = sizeof(*out);
  out->width = m->width[k];
  out->height = m->height[k];
  out->reserved = 0;
  out->depth = m->depth.data() + m->off[k];
  out->normal = m->normal.data() + 3 * m->off[k];
  return B2M_OK;
}

void b2m_depth_maps_free(b2m_depth_maps* m) { delete m; }

int b2m_debug_patch_match_cost(b2m_ctx* ctx, const b2m_patch_match_problem* problem, const b2m_patch_match_opts* opts,
                               const float* queries, int32_t n, float* out) {
  if (!ctx) return B2M_EINVAL;
  if (!problem || n < 0 || (n > 0 && (!queries || !out)))
    return fail(ctx, B2M_EINVAL, "[patch_match.cu] Check Failed: problem, queries and out");
  PmParams P;
  if (int rc = check_opts(ctx, opts, &P)) return rc;
  PmState* S = pm_state(ctx);
  if (S->n_images == 0) return fail(ctx, B2M_ESTATE, "[patch_match.cu] b2m_patch_match_set_images must come first");
  PmProblem pr;
  if (int rc = make_problem(ctx, *S, *problem, false, &pr)) return rc;
  const PmCam& rc = S->cams[pr.ref];
  for (int i = 0; i < n; ++i) {
    const int x = static_cast<int>(queries[7 * i]), y = static_cast<int>(queries[7 * i + 1]), s = static_cast<int>(queries[7 * i + 6]);
    if (x < 0 || y < 0 || x >= rc.W || y >= rc.H || s < 0 || s >= pr.n_src || queries[7 * i] != x || queries[7 * i + 1] != y)
      return fail(ctx, B2M_EINVAL, "[patch_match.cu] Check Failed: query pixel in the reference, source slot in range");
  }
  if (n == 0) return B2M_OK;
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  B2M_CUDA_TRY(ctx, S->d_probs.ensure(1));
  B2M_CUDA_TRY(ctx, S->d_q.ensure(7 * static_cast<size_t>(n)));
  B2M_CUDA_TRY(ctx, S->d_out.ensure(3 * static_cast<size_t>(n)));
  B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->d_probs, &pr, sizeof(pr), cudaMemcpyHostToDevice, st));
  B2M_CUDA_TRY(ctx, cudaMemcpyAsync(S->d_q, queries, sizeof(float) * 7 * n, cudaMemcpyHostToDevice, st));
  PmArgs a{};
  a.images = S->images;
  a.dmaps = S->dmaps;
  a.cams = S->d_cams;
  a.probs = S->d_probs;
  a.P = P;
  b2m_pm_debug_kernel<<<(n + kWarpsPerCta - 1) / kWarpsPerCta, 32 * kWarpsPerCta, 0, st>>>(a, S->d_q, n, S->d_out);
  B2M_CUDA_TRY(ctx, cudaGetLastError());
  B2M_CUDA_TRY(ctx, cudaMemcpyAsync(out, S->d_out, sizeof(float) * 3 * n, cudaMemcpyDeviceToHost, st));
  B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
  ctx->stats.kernel_launches += 1;
  return B2M_OK;
}

}  // extern "C"
