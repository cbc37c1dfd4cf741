// Scalar, single-threaded restatement of COLMAP's stereo fusion (U:mvs/fusion.cc, recalled; DESIGN.md section 4, K9)
// and of K9's seed schedule.  TEST INFRASTRUCTURE ONLY, and the CPU arm of tools/bench_stereo_fusion.py.
// The float32 arithmetic is ../pycolmap_b200/csrc/fusion_math.h; compiled with -ffp-contract=off.
//
// Fuse(image, row, col) -- a LIFO stack of (image, row, col, traversal depth) entries, seeded with (image, row, col, 0):
//   pop; skip when the pixel is fused, its depth <= 0, or (traversal depth > 0) it fails the depth, reprojection or
//   normal check against the cluster's reference point; otherwise xyz = inv_P (col d, row d, d, 1), mark it fused,
//   skip it when xyz is outside the bounding box, accumulate it (the first accumulated pixel is the reference), stop
//   at max_num_pixels, and when depth + 1 < max_traversal_depth push every overlapping image (list order) that has
//   maps and into which xyz projects (rounded) inside the map.  With >= min_num_pixels accumulated pixels the cluster
//   emits the per-channel medians, unless the median normal's norm is below FLT_EPSILON.
//
// Orders: 0 = rows (images in index order, pixels row-major: upstream with one thread), 1 = schedule (K9's rounds),
// 2 = replay (an explicit seed list).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../pycolmap_b200/csrc/fusion_math.h"

using b2m_fu::Cam;
using b2m_fu::Opts;

namespace {

struct Scene {
  int n = 0;
  std::vector<Cam> cams;
  std::vector<int32_t> ov;
  std::vector<float> depth, normal;  // concatenated maps of the images with maps
  std::vector<uint8_t> rgb;
  std::vector<uint8_t> fused;        // per map pixel; masked pixels start fused
  Opts o{};
};

struct Result {
  std::vector<float> xyz, nrm;
  std::vector<uint8_t> rgb;
  std::vector<int64_t> vis_off{0};
  std::vector<int32_t> vis, seed, order;
  int64_t stats[5] = {0, 0, 0, 0, 0};  // pops, traversals, rounds, deferred seeds, committed seeds
};

struct Entry {
  int img, row, col, td;
};

// One traversal from (img, row, col); marks what it fuses in S.fused and lists it in *fused (map pixel ids) with the
// accumulated ones in *acc.  Returns the number of pops.
int64_t fuse(Scene& S, int img, int row, int col, std::vector<int64_t>* fused, std::vector<int64_t>* acc,
             std::vector<int32_t>* acc_img) {
  std::vector<Entry> stack{{img, row, col, 0}};
  float ref_xyz[3] = {0, 0, 0}, ref_n[3] = {0, 0, 0};
  int64_t pops = 0;
  while (!stack.empty()) {
    const Entry e = stack.back();
    stack.pop_back();
    ++pops;
    const Cam& c = S.cams[e.img];
    const int64_t id = c.px_off + static_cast<int64_t>(e.row) * c.W + e.col;
    if (S.fused[id]) continue;
    const float d = S.depth[id];
    if (!(d > 0.f)) continue;
    float nw[3];
    b2m_fu::rotate(c.iR, &S.normal[3 * id], nw);
    if (e.td > 0 && !b2m_fu::consistent(c, S.o, ref_xyz, ref_n, e.row, e.col, d, nw)) continue;
    float xyz[3];
    b2m_fu::backproject(c, e.row, e.col, d, xyz);
    S.fused[id] = 1;
    fused->push_back(id);
    if (!b2m_fu::in_box(S.o, xyz)) continue;
    if (acc->empty()) {
      std::memcpy(ref_xyz, xyz, sizeof(xyz));
      std::memcpy(ref_n, nw, sizeof(nw));
    }
    acc->push_back(id);
    acc_img->push_back(e.img);
    if (static_cast<int64_t>(acc->size()) >= S.o.max_num_pixels) break;
    if (e.td + 1 < S.o.max_traversal_depth) {
      for (int k = 0; k < c.ov_n; ++k) {
        const int j = S.ov[c.ov_off + k];
        const Cam& cj = S.cams[j];
        int r, q;
        if (cj.px_off < 0 || !b2m_fu::child_pixel(cj, xyz, &r, &q)) continue;
        stack.push_back({j, r, q, e.td + 1});
      }
    }
  }
  return pops;
}

// The point of a cluster (accumulated ids and their images), appended to R when it has one.
void emit(const Scene& S, const std::vector<int64_t>& acc, const std::vector<int32_t>& acc_img, int img, int row, int col,
          Result* R) {
  const int n = static_cast<int>(acc.size());
  if (n < S.o.min_num_pixels || n == 0) return;
  std::vector<float> ch[9];
  for (auto& v : ch) v.resize(n);
  for (int i = 0; i < n; ++i) {
    const Cam& c = S.cams[acc_img[i]];
    const int64_t local = acc[i] - c.px_off;
    const int row_i = static_cast<int>(local / c.W), col_i = static_cast<int>(local % c.W);
    float xyz[3], nw[3], rgb[3];
    b2m_fu::backproject(c, row_i, col_i, S.depth[acc[i]], xyz);
    b2m_fu::rotate(c.iR, &S.normal[3 * acc[i]], nw);
    b2m_fu::colour(c, S.rgb.data(), row_i, col_i, rgb);
    for (int k = 0; k < 3; ++k) {
      ch[k][i] = xyz[k];
      ch[3 + k][i] = nw[k];
      ch[6 + k][i] = rgb[k];
    }
  }
  float m[9];
  for (int k = 0; k < 9; ++k) {
    std::sort(ch[k].begin(), ch[k].end());
    m[k] = b2m_fu::median_sorted(ch[k].data(), n);
  }
  float xyz[3], nrm[3];
  uint8_t rgb[3];
  if (!b2m_fu::finish_point(m, xyz, nrm, rgb)) return;
  R->xyz.insert(R->xyz.end(), xyz, xyz + 3);
  R->nrm.insert(R->nrm.end(), nrm, nrm + 3);
  R->rgb.insert(R->rgb.end(), rgb, rgb + 3);
  std::vector<int32_t> v(acc_img);
  std::sort(v.begin(), v.end());
  v.erase(std::unique(v.begin(), v.end()), v.end());
  R->vis.insert(R->vis.end(), v.begin(), v.end());
  R->vis_off.push_back(static_cast<int64_t>(R->vis.size()));
  R->seed.insert(R->seed.end(), {img, row, col});
}

// One committed seed: its traversal (already run on S.fused), its order entry and its point.
void commit(Scene& S, int img, int row, int col, int round, Result* R) {
  std::vector<int64_t> fused, acc;
  std::vector<int32_t> acc_img;
  R->stats[0] += fuse(S, img, row, col, &fused, &acc, &acc_img);
  R->stats[1] += 1;
  R->stats[4] += 1;
  R->order.insert(R->order.end(), {img, row, col, round});
  emit(S, acc, acc_img, img, row, col, R);
}

bool live(const Scene& S, int img, int row, int col) {
  const Cam& c = S.cams[img];
  const int64_t id = c.px_off + static_cast<int64_t>(row) * c.W + col;
  return !S.fused[id] && S.depth[id] > 0.f;
}

// K9's schedule: per image with maps (index order), per phase (py, px) of the s x s lattice (row-major), rounds until
// the phase has no live seed.  A round's candidates are the live lattice pixels, keyed by their row-major position; each
// traverses against the round-start mask and claims (minimum key) every pixel it would fuse; a candidate commits when
// none of those pixels carries a smaller key.  The committed candidates then run in key order.
void schedule(Scene& S, int s, Result* R) {
  std::vector<int32_t> claim(S.fused.size(), INT32_MAX);
  int round = 0;
  for (int img = 0; img < S.n; ++img) {
    const Cam& c = S.cams[img];
    if (c.px_off < 0) continue;
    for (int phase = 0; phase < s * s; ++phase) {
      const int py = phase / s, px = phase % s;
      const int lw = (c.W - px + s - 1) / s, lh = (c.H - py + s - 1) / s;
      for (;;) {
        std::vector<int> keys;
        std::vector<std::vector<int64_t>> lists;
        for (int q = 0; q < lh; ++q)
          for (int w = 0; w < lw; ++w) {
            const int row = py + s * q, col = px + s * w;
            if (!live(S, img, row, col)) continue;
            std::vector<int64_t> fused, acc;
            std::vector<int32_t> acc_img;
            R->stats[0] += fuse(S, img, row, col, &fused, &acc, &acc_img);
            R->stats[1] += 1;
            for (int64_t id : fused) S.fused[id] = 0;  // speculative: roll back to the round-start mask
            const int key = q * lw + w;
            for (int64_t id : fused) claim[id] = std::min(claim[id], key);
            keys.push_back(key);
            lists.push_back(std::move(fused));
          }
        if (keys.empty()) break;
        std::vector<int> winners;
        for (size_t k = 0; k < keys.size(); ++k) {
          bool ok = true;
          for (int64_t id : lists[k]) ok = ok && claim[id] >= keys[k];
          if (ok) winners.push_back(keys[k]); else R->stats[3] += 1;
        }
        for (auto& l : lists)
          for (int64_t id : l) claim[id] = INT32_MAX;
        for (int key : winners) commit(S, img, py + s * (key / lw), px + s * (key % lw), round, R);
        ++round;
      }
    }
  }
  R->stats[2] = round;
}

}  // namespace

extern "C" {

// dims [n x 4] (W, H, bitmap W, bitmap H); depth / normal / mask / rgb: n pointers (depth NULL: no maps; mask NULL:
// none; rgb [bh x bw x 3]); cams [n x 35] (P 12, inv_P 12, inv_R 9, sx, sy); ov_off [n + 1], ov; opts [12]
// (min_num_pixels, max_num_pixels, max_traversal_depth, max_reproj_error, max_depth_error, cos of max_normal_error,
// bounding box 6); mode 0 rows / 1 schedule / 2 replay (seeds [n_seeds x 3] (image, row, col)).
void* orc_fu_run(int n, const int32_t* dims, const float* const* depth, const float* const* normal,
                 const uint8_t* const* mask, const uint8_t* const* rgb, const float* cams, const int32_t* ov_off,
                 const int32_t* ov, const double* opts, int mode, int s, const int32_t* seeds, int64_t n_seeds) {
  Scene S;
  S.n = n;
  S.cams.resize(n);
  S.ov.assign(ov, ov + ov_off[n]);
  int64_t px = 0, rgb_px = 0;
  for (int i = 0; i < n; ++i) {
    Cam& c = S.cams[i];
    std::memcpy(c.P, cams + 35 * i, 12 * sizeof(float));
    std::memcpy(c.iP, cams + 35 * i + 12, 12 * sizeof(float));
    std::memcpy(c.iR, cams + 35 * i + 24, 9 * sizeof(float));
    c.sx = cams[35 * i + 33];
    c.sy = cams[35 * i + 34];
    c.W = dims[4 * i];
    c.H = dims[4 * i + 1];
    c.bw = dims[4 * i + 2];
    c.bh = dims[4 * i + 3];
    c.ov_off = ov_off[i];
    c.ov_n = ov_off[i + 1] - ov_off[i];
    c.px_off = depth[i] ? px : -1;
    if (depth[i]) px += static_cast<int64_t>(c.W) * c.H;
    c.rgb_off = 3 * rgb_px;
    rgb_px += static_cast<int64_t>(c.bw) * c.bh;
  }
  S.depth.resize(px);
  S.normal.resize(3 * px);
  S.fused.assign(px, 0);
  S.rgb.resize(3 * rgb_px);
  for (int i = 0; i < n; ++i) {
    const Cam& c = S.cams[i];
    const int64_t m = static_cast<int64_t>(c.W) * c.H;
    if (c.px_off >= 0) {
      std::memcpy(&S.depth[c.px_off], depth[i], m * sizeof(float));
      std::memcpy(&S.normal[3 * c.px_off], normal[i], 3 * m * sizeof(float));
      if (mask[i])
        for (int64_t k = 0; k < m; ++k) S.fused[c.px_off + k] = mask[i][k] == 0;
    }
    if (rgb[i]) std::memcpy(&S.rgb[c.rgb_off], rgb[i], 3 * static_cast<size_t>(c.bw) * c.bh);
  }
  S.o.min_num_pixels = static_cast<int32_t>(opts[0]);
  S.o.max_num_pixels = static_cast<int32_t>(opts[1]);
  S.o.max_traversal_depth = static_cast<int32_t>(opts[2]);
  const float reproj = static_cast<float>(opts[3]);
  S.o.max_reproj_sq = reproj * reproj;
  S.o.max_depth_error = static_cast<float>(opts[4]);
  S.o.min_cos_normal = static_cast<float>(opts[5]);
  for (int k = 0; k < 6; ++k) S.o.bbox[k] = static_cast<float>(opts[6 + k]);

  Result* R = new Result();
  if (mode == 0) {
    for (int img = 0; img < n; ++img) {
      const Cam& c = S.cams[img];
      if (c.px_off < 0) continue;
      for (int row = 0; row < c.H; ++row)
        for (int col = 0; col < c.W; ++col)
          if (live(S, img, row, col)) commit(S, img, row, col, 0, R);
    }
  } else if (mode == 1) {
    schedule(S, s, R);
  } else {
    for (int64_t k = 0; k < n_seeds; ++k) {
      const int img = seeds[3 * k], row = seeds[3 * k + 1], col = seeds[3 * k + 2];
      if (img >= 0 && img < n && S.cams[img].px_off >= 0 && row >= 0 && row < S.cams[img].H && col >= 0 &&
          col < S.cams[img].W && live(S, img, row, col))
        commit(S, img, row, col, 0, R);
    }
  }
  return R;
}

// what: 0 xyz, 1 normals, 2 colours, 3 vis_off, 4 vis, 5 point seeds, 6 order, 7 stats; count in elements.
int64_t orc_fu_count(void* h, int what) {
  const Result* R = static_cast<Result*>(h);
  switch (what) {
    case 0: return static_cast<int64_t>(R->xyz.size());
    case 1: return static_cast<int64_t>(R->nrm.size());
    case 2: return static_cast<int64_t>(R->rgb.size());
    case 3: return static_cast<int64_t>(R->vis_off.size());
    case 4: return static_cast<int64_t>(R->vis.size());
    case 5: return static_cast<int64_t>(R->seed.size());
    case 6: return static_cast<int64_t>(R->order.size());
    default: return 5;
  }
}

void orc_fu_copy(void* h, int what, void* dst) {
  const Result* R = static_cast<Result*>(h);
  switch (what) {
    case 0: std::memcpy(dst, R->xyz.data(), R->xyz.size() * sizeof(float)); break;
    case 1: std::memcpy(dst, R->nrm.data(), R->nrm.size() * sizeof(float)); break;
    case 2: std::memcpy(dst, R->rgb.data(), R->rgb.size()); break;
    case 3: std::memcpy(dst, R->vis_off.data(), R->vis_off.size() * sizeof(int64_t)); break;
    case 4: std::memcpy(dst, R->vis.data(), R->vis.size() * sizeof(int32_t)); break;
    case 5: std::memcpy(dst, R->seed.data(), R->seed.size() * sizeof(int32_t)); break;
    case 6: std::memcpy(dst, R->order.data(), R->order.size() * sizeof(int32_t)); break;
    default: std::memcpy(dst, R->stats, sizeof(R->stats)); break;
  }
}

void orc_fu_free(void* h) { delete static_cast<Result*>(h); }

}  // extern "C"
