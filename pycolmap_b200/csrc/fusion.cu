// fusion.cu -- K9: stereo fusion (what U:mvs/fusion.cc computes) over the depth and normal maps of a workspace.
//
// Seeds depend on each other through the fused mask, so K9 speculates and commits by a fixed rule (DESIGN.md section 4,
// K9).  Images go one at a time in index order; each image's pixels are split into the kLattice x kLattice phases of a
// sub-lattice, and a phase runs in rounds until none of its lattice pixels is live (unfused with depth > 0):
//   speculate -- one thread per live lattice pixel (a candidate, keyed by its row-major lattice position) runs the
//                traversal against the round-start mask and atomicMin's its key into the claim of every pixel it fuses;
//   decide    -- a candidate commits when none of its pixels carries a smaller key (the lowest candidate always does);
//   commit    -- committed candidates mark their pixels fused and emit their points; every candidate resets its claims.
// Committed clusters are pairwise disjoint and each read only pixels no earlier candidate fused, so the result equals
// the sequential traversal over (round, key) -- the order returned to the caller.  It depends on the inputs only.
//
// The traversal keeps no stack of pushed pixels: a child's pixel is a function of its parent's point, so one frame
// (image, point, depth, next child) per level replays the LIFO order.  A candidate's fused pixels live in a bounded
// slot (list + open-addressing set); a cluster that outgrows it is redone exactly by one thread with workspace-sized
// storage (the overflow path).  The float32 arithmetic is fusion_math.h, compiled without FMA contraction.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "fusion_math.h"
#include "internal.h"

using b2m_fu::Cam;
using b2m_fu::Opts;

struct b2m_fused_points {
  std::vector<float> xyz, nrm;
  std::vector<uint8_t> rgb;
  std::vector<int64_t> vis_off{0};
  std::vector<int32_t> vis, seeds, order;
};

namespace b2m {
namespace {

constexpr int kLattice = 16;    // s: the seed sub-lattice spacing (part of the result's definition)
constexpr int kCap = 512;       // fused pixels a candidate's slot holds
constexpr int kHash = 1024;     // its open-addressing set (2 x kCap)
constexpr int kFrames = 128;    // traversal levels a slot holds
constexpr int kThreads = 128;

// kOvf*: candidates of the overflow path, whose slots hold nothing (the slot kernels leave them alone)
enum : int32_t { kNone = 0, kLive = 1, kOverflow = 2, kDeferred = 3, kCommit = 4, kOvfDeferred = 5, kOvfCommit = 6 };

struct Frame {
  float xyz[3];
  int32_t img, td, next;
};

struct Counters {
  unsigned long long live, ovf, deferred, n_rec, n_vis, pops, traversals;
};

struct Rec {
  int32_t key, img, row, col, emitted, nvis;
  int64_t vis_off;
  float xyz[3], nrm[3];
  uint8_t rgb[4];
};

struct FuArgs {
  const Cam* cams;
  const int32_t* ov;
  const float* depth;
  const float* normal;
  const uint8_t* rgb;
  uint8_t* fused;
  int32_t* claim;
  Opts o;
  // slots, [L x kCap] / [L x kHash] / [L x kFrames]
  int64_t* list_id;   // map pixel id << 1 | accumulated
  int32_t* list_img;
  int16_t* list_slot;
  int64_t* hash;      // id + 1, 0 = empty
  Frame* frames;
  int32_t* scratch;
  int32_t* status;    // [L]
  int32_t* n_list;    // [L]
  // overflow path: workspace-sized
  int64_t* big_id;
  int32_t* big_img;
  uint32_t* stamp;    // per map pixel
  uint32_t* stamp_next;
  Frame* big_frames;
  int32_t* big_scratch;
  int64_t big_cap;
  int32_t* ovf_keys;
  // this round
  int32_t img, py, px, lw, L, round;
  Counters* cnt;
  Rec* rec;
  int32_t* vis;
};

// A candidate's slot: own-fused set by hash, list bounded by kCap, frames by kFrames.
struct SlotStore {
  int64_t* id;
  int32_t* img;
  int16_t* hslot;
  int64_t* hash;
  Frame* frames;
  int n = 0;
  __device__ int probe(int64_t key) const {
    unsigned h = static_cast<unsigned>((static_cast<unsigned long long>(key) * 0x9E3779B97F4A7C15ull) >> 54);
    for (;;) {
      const int64_t v = hash[h];
      if (v == 0 || v == key + 1) return static_cast<int>(h);
      h = (h + 1) & (kHash - 1);
    }
  }
  __device__ bool own(int64_t key) const { return hash[probe(key)] == key + 1; }
  __device__ bool add(int64_t key, int32_t im, bool acc) {
    if (n == kCap) return false;
    const int h = probe(key);
    hash[h] = key + 1;
    hslot[n] = static_cast<int16_t>(h);
    id[n] = key << 1 | (acc ? 1 : 0);
    img[n] = im;
    ++n;
    return true;
  }
  __device__ void clear() {
    for (int i = 0; i < n; ++i) hash[hslot[i]] = 0;
  }
  __device__ int frame_cap() const { return kFrames; }
};

// The overflow path's storage: own-fused set by a per-pixel stamp unique to the traversal.
struct BigStore {
  int64_t* id;
  int32_t* img;
  uint32_t* stamp;
  uint32_t mine;
  Frame* frames;
  int64_t cap;
  int fcap;
  int64_t n = 0;
  __device__ bool own(int64_t key) const { return stamp[key] == mine; }
  __device__ bool add(int64_t key, int32_t im, bool acc) {
    if (n == cap) return false;
    stamp[key] = mine;
    id[n] = key << 1 | (acc ? 1 : 0);
    img[n] = im;
    ++n;
    return true;
  }
  __device__ int frame_cap() const { return fcap; }
};

struct Trav {
  int64_t nacc = 0, pops = 0;
  bool overflow = false;
};

// One traversal from (img, row, col) against the mask `a.fused` plus the store's own pixels (oracle/fusion.cpp fuse()).
template <class Store>
__device__ Trav traverse(const FuArgs& a, int img, int row, int col, Store& st) {
  Trav t;
  float ref_xyz[3] = {0.f, 0.f, 0.f}, ref_n[3] = {0.f, 0.f, 0.f};
  int top = -1;
  int pi = img, pr = row, pc = col, ptd = 0;
  bool have = true;
  for (;;) {
    if (have) {
      have = false;
      ++t.pops;
      const Cam& c = a.cams[pi];
      const int64_t id = c.px_off + static_cast<int64_t>(pr) * c.W + pc;
      const float d = a.depth[id];
      if (!a.fused[id] && !st.own(id) && d > 0.f) {
        float nw[3];
        b2m_fu::rotate(c.iR, a.normal + 3 * id, nw);
        if (ptd == 0 || b2m_fu::consistent(c, a.o, ref_xyz, ref_n, pr, pc, d, nw)) {
          float xyz[3];
          b2m_fu::backproject(c, pr, pc, d, xyz);
          const bool acc = b2m_fu::in_box(a.o, xyz);
          if (!st.add(id, pi, acc)) {
            t.overflow = true;
            return t;
          }
          if (acc) {
            if (t.nacc == 0) {
              for (int k = 0; k < 3; ++k) {
                ref_xyz[k] = xyz[k];
                ref_n[k] = nw[k];
              }
            }
            ++t.nacc;
            if (t.nacc >= a.o.max_num_pixels) return t;
            if (ptd + 1 < a.o.max_traversal_depth) {
              if (top + 1 == st.frame_cap()) {
                t.overflow = true;
                return t;
              }
              Frame& f = st.frames[++top];
              for (int k = 0; k < 3; ++k) f.xyz[k] = xyz[k];
              f.img = pi;
              f.td = ptd;
              f.next = c.ov_n - 1;
            }
          }
        }
      }
    }
    if (top < 0) return t;
    Frame& f = st.frames[top];
    if (f.next < 0) {
      --top;
      continue;
    }
    const int j = a.ov[a.cams[f.img].ov_off + f.next];
    --f.next;
    const Cam& cj = a.cams[j];
    int r, q;
    if (cj.px_off < 0 || !b2m_fu::child_pixel(cj, f.xyz, &r, &q)) continue;
    pi = j;
    pr = r;
    pc = q;
    ptd = f.td + 1;
    have = true;
  }
}

// The point of a committed cluster (list id / img of n entries, nacc accumulated) into a record; `scratch` holds n.
__device__ void emit(const FuArgs& a, const int64_t* id, const int32_t* img, int64_t n, int64_t nacc, int32_t* scratch,
                     int key, int row, int col) {
  const unsigned long long r = atomicAdd(&a.cnt->n_rec, 1ull);
  Rec& R = a.rec[r];
  R.key = key;
  R.img = a.img;
  R.row = row;
  R.col = col;
  R.emitted = 0;
  R.nvis = 0;
  R.vis_off = 0;
  if (nacc < a.o.min_num_pixels || nacc == 0) return;
  float* fs = reinterpret_cast<float*>(scratch);
  float m[9];
  for (int ch = 0; ch < 9; ++ch) {
    int64_t k = 0;
    for (int64_t i = 0; i < n; ++i) {
      if (!(id[i] & 1)) continue;
      const int64_t p = id[i] >> 1;
      const Cam& c = a.cams[img[i]];
      const int64_t local = p - c.px_off;
      const int rr = static_cast<int>(local / c.W), cc = static_cast<int>(local % c.W);
      float v[3];
      if (ch < 3) b2m_fu::backproject(c, rr, cc, a.depth[p], v);
      else if (ch < 6) b2m_fu::rotate(c.iR, a.normal + 3 * p, v);
      else b2m_fu::colour(c, a.rgb, rr, cc, v);
      fs[k++] = v[ch % 3];
    }
    b2m_fu::heap_sort(fs, static_cast<int>(k));
    m[ch] = b2m_fu::median_sorted(fs, static_cast<int>(k));
  }
  if (!b2m_fu::finish_point(m, R.xyz, R.nrm, R.rgb)) return;
  R.emitted = 1;
  int64_t k = 0;
  for (int64_t i = 0; i < n; ++i)
    if (id[i] & 1) scratch[k++] = img[i];
  b2m_fu::heap_sort(scratch, static_cast<int>(k));
  int u = 0;
  for (int64_t i = 0; i < k; ++i)
    if (i == 0 || scratch[i] != scratch[i - 1]) scratch[u++] = scratch[i];
  const unsigned long long off = atomicAdd(&a.cnt->n_vis, static_cast<unsigned long long>(u));
  for (int i = 0; i < u; ++i) a.vis[off + i] = scratch[i];
  R.nvis = u;
  R.vis_off = static_cast<int64_t>(off);
}

__device__ SlotStore slot_of(const FuArgs& a, int k) {
  SlotStore s;
  s.id = a.list_id + static_cast<int64_t>(k) * kCap;
  s.img = a.list_img + static_cast<int64_t>(k) * kCap;
  s.hslot = a.list_slot + static_cast<int64_t>(k) * kCap;
  s.hash = a.hash + static_cast<int64_t>(k) * kHash;
  s.frames = a.frames + static_cast<int64_t>(k) * kFrames;
  return s;
}

__device__ void lattice_pixel(const FuArgs& a, int k, int* row, int* col) {
  *row = a.py + kLattice * (k / a.lw);
  *col = a.px + kLattice * (k % a.lw);
}

__global__ void b2m_fu_speculate_kernel(FuArgs a) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.L) return;
  a.status[k] = kNone;
  int row, col;
  lattice_pixel(a, k, &row, &col);
  const Cam& c = a.cams[a.img];
  const int64_t id = c.px_off + static_cast<int64_t>(row) * c.W + col;
  if (a.fused[id] || !(a.depth[id] > 0.f)) return;
  SlotStore s = slot_of(a, k);
  const Trav t = traverse(a, a.img, row, col, s);
  s.clear();
  atomicAdd(&a.cnt->live, 1ull);
  atomicAdd(&a.cnt->traversals, 1ull);
  atomicAdd(&a.cnt->pops, static_cast<unsigned long long>(t.pops));
  if (t.overflow) {
    a.status[k] = kOverflow;
    a.ovf_keys[atomicAdd(&a.cnt->ovf, 1ull)] = k;
    return;
  }
  a.status[k] = kLive;
  a.n_list[k] = s.n;
  a.scratch[static_cast<int64_t>(k) * kCap] = static_cast<int32_t>(t.nacc);  // kept for the commit
  for (int i = 0; i < s.n; ++i) atomicMin(a.claim + (s.id[i] >> 1), k);
}

__global__ void b2m_fu_decide_kernel(FuArgs a) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.L || a.status[k] != kLive) return;
  const int64_t* id = a.list_id + static_cast<int64_t>(k) * kCap;
  bool ok = true;
  for (int i = 0; i < a.n_list[k] && ok; ++i) ok = a.claim[id[i] >> 1] >= k;
  a.status[k] = ok ? kCommit : kDeferred;
  if (!ok) atomicAdd(&a.cnt->deferred, 1ull);
}

__global__ void b2m_fu_commit_kernel(FuArgs a) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.L) return;
  const int32_t st = a.status[k];
  if (st != kCommit && st != kDeferred) return;
  const int64_t* id = a.list_id + static_cast<int64_t>(k) * kCap;
  const int32_t* img = a.list_img + static_cast<int64_t>(k) * kCap;
  const int n = a.n_list[k];
  for (int i = 0; i < n; ++i) a.claim[id[i] >> 1] = INT_MAX;
  if (st != kCommit) return;
  for (int i = 0; i < n; ++i) a.fused[id[i] >> 1] = 1;
  int32_t* scratch = a.scratch + static_cast<int64_t>(k) * kCap;
  const int64_t nacc = scratch[0];
  int row, col;
  lattice_pixel(a, k, &row, &col);
  emit(a, id, img, n, nacc, scratch, k, row, col);
}

// The overflow path: one thread walks the overflowing candidates of the round (ascending key) in one of four steps.
// 0: claim, 1: decide, 2: reset claims (before any pixel of the round is marked), 3: commit.
__global__ void b2m_fu_overflow_kernel(FuArgs a, int n_ovf, int step) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  for (int e = 0; e < n_ovf; ++e) {
    const int k = a.ovf_keys[e];
    if (step == 3 && a.status[k] != kOvfCommit) continue;
    int row, col;
    lattice_pixel(a, k, &row, &col);
    BigStore s;
    s.id = a.big_id;
    s.img = a.big_img;
    s.stamp = a.stamp;
    s.mine = ++*a.stamp_next;
    s.frames = a.big_frames;
    s.cap = a.big_cap;
    s.fcap = a.o.max_traversal_depth;
    const Trav t = traverse(a, a.img, row, col, s);
    a.cnt->traversals += 1;
    a.cnt->pops += static_cast<unsigned long long>(t.pops);
    if (step == 0) {
      for (int64_t i = 0; i < s.n; ++i) atomicMin(a.claim + (s.id[i] >> 1), k);
    } else if (step == 1) {
      bool ok = true;
      for (int64_t i = 0; i < s.n && ok; ++i) ok = a.claim[s.id[i] >> 1] >= k;
      a.status[k] = ok ? kOvfCommit : kOvfDeferred;
      if (!ok) a.cnt->deferred += 1;
    } else if (step == 2) {
      for (int64_t i = 0; i < s.n; ++i) a.claim[s.id[i] >> 1] = INT_MAX;
    } else {
      for (int64_t i = 0; i < s.n; ++i) a.fused[s.id[i] >> 1] = 1;
      emit(a, s.id, s.img, s.n, t.nacc, a.big_scratch, k, row, col);
    }
  }
}

// The bitmap of one image as RGB: `src` holds W x H x channels bytes (1: grey, 3: RGB, 4: RGBA), `stride` per row.
__global__ void b2m_fu_rgb_kernel(const uint8_t* src, int64_t stride, int W, int H, int channels, uint8_t* dst) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<int64_t>(W) * H) return;
  const uint8_t* p = src + (i / W) * stride + (i % W) * channels;
  for (int k = 0; k < 3; ++k) dst[3 * i + k] = channels == 1 ? p[0] : p[k];
}

__global__ void b2m_fu_fill_kernel(int32_t* p, int64_t n, int32_t v) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

__global__ void b2m_fu_mask_kernel(const uint8_t* mask, int64_t n, uint8_t* fused) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) fused[i] = mask[i] == 0;
}

inline unsigned blocks(int64_t n) { return static_cast<unsigned>((n + kThreads - 1) / kThreads); }

// The 4 x 4 top-rows inverse and the other per-image arrays are the caller's (fp64 rounded once): checked only for size.
int check_inputs(b2m_ctx* ctx, const b2m_fusion_image* im, int32_t n, const b2m_fusion_opts* o) {
  auto bad = [&](const std::string& what) { return fail(ctx, B2M_EINVAL, "[fusion.cu] Check Failed: " + what); };
  if (!o || o->struct_size != sizeof(b2m_fusion_opts)) return bad("opts != NULL (struct_size)");
  if (!(o->min_num_pixels >= 0)) return bad("min_num_pixels >= 0");
  if (!(o->min_num_pixels <= o->max_num_pixels)) return bad("min_num_pixels <= max_num_pixels");
  if (!(o->max_traversal_depth > 0)) return bad("max_traversal_depth > 0");
  if (!(o->max_reproj_error >= 0.f)) return bad("max_reproj_error >= 0");
  if (!(o->max_depth_error >= 0.f)) return bad("max_depth_error >= 0");
  if (!(o->max_normal_error >= 0.f)) return bad("max_normal_error >= 0");
  for (int i = 0; i < n; ++i) {
    const b2m_fusion_image& m = im[i];
    const std::string at = "image " + std::to_string(i) + ": ";
    if (m.struct_size != sizeof(b2m_fusion_image)) return bad(at + "b2m_fusion_image.struct_size");
    if (m.depth && (m.width < 1 || m.height < 1 || !m.normal)) return bad(at + "maps of width, height >= 1 with normals");
    if (m.n_overlap < 0 || (m.n_overlap > 0 && !m.overlap)) return bad(at + "n_overlap >= 0 with an overlap list");
    for (int k = 0; k < m.n_overlap; ++k)
      if (m.overlap[k] < 0 || m.overlap[k] >= n) return bad(at + "overlap entries are image indices");
    if (m.depth && !(m.bitmap_scale[0] > 0.f && m.bitmap_scale[1] > 0.f)) return bad(at + "bitmap_scale > 0");
    const b2m_image_source& s = m.color;
    if (s.data && s.kind == B2M_SOURCE_PIXELS &&
        (s.width < 1 || s.height < 1 || !(s.channels == 1 || s.channels == 3 || s.channels == 4) ||
         s.stride < static_cast<int64_t>(s.width) * s.channels))
      return bad(at + "color pixels of 1, 3 or 4 channels with stride >= width x channels");
    if (s.data && s.kind != B2M_SOURCE_PIXELS && s.kind != B2M_SOURCE_JPEG) return bad(at + "color.kind");
  }
  return B2M_OK;
}

}  // namespace
}  // namespace b2m

using namespace b2m;

extern "C" {

void b2m_fusion_opts_default(b2m_fusion_opts* o) {
  if (!o) return;
  std::memset(o, 0, sizeof(*o));
  o->struct_size = sizeof(*o);
  o->min_num_pixels = 5;
  o->max_num_pixels = 10000;
  o->max_traversal_depth = 100;
  o->max_reproj_error = 2.0f;
  o->max_depth_error = 0.01f;
  o->max_normal_error = 10.0f;
  for (int k = 0; k < 3; ++k) {
    o->bounding_box[k] = -FLT_MAX;
    o->bounding_box[3 + k] = FLT_MAX;
  }
}

int b2m_stereo_fusion(b2m_ctx* ctx, const b2m_fusion_image* images, int32_t n, const b2m_fusion_opts* opts,
                      b2m_fused_points** out) {
  if (!ctx) return B2M_EINVAL;
  if (!out || n < 0 || (n > 0 && !images)) return fail(ctx, B2M_EINVAL, "[fusion.cu] Check Failed: out != NULL && images");
  *out = nullptr;
  if (int rc = check_inputs(ctx, images, n, opts)) return rc;
  std::unique_ptr<b2m_fused_points> F(new (std::nothrow) b2m_fused_points());
  if (!F) return fail(ctx, B2M_ENOMEM, "[fusion.cu] out of host memory");
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;

  // ---- layout and residency
  std::vector<Cam> cams(n);
  std::vector<int32_t> ov;
  int64_t px = 0, lmax = 0;
  for (int i = 0; i < n; ++i) {
    const b2m_fusion_image& m = images[i];
    Cam& c = cams[i];
    std::memcpy(c.P, m.P, sizeof(c.P));
    std::memcpy(c.iP, m.inv_P, sizeof(c.iP));
    std::memcpy(c.iR, m.inv_R, sizeof(c.iR));
    c.sx = m.bitmap_scale[0];
    c.sy = m.bitmap_scale[1];
    c.W = m.depth ? m.width : 0;
    c.H = m.depth ? m.height : 0;
    c.px_off = m.depth ? px : -1;
    if (m.depth) {
      px += static_cast<int64_t>(m.width) * m.height;
      lmax = std::max<int64_t>(lmax, static_cast<int64_t>((m.width + kLattice - 1) / kLattice) *
                                         ((m.height + kLattice - 1) / kLattice));
    }
    c.ov_off = static_cast<int32_t>(ov.size());
    c.ov_n = m.n_overlap;
    ov.insert(ov.end(), m.overlap, m.overlap + m.n_overlap);
  }
  // bitmaps: decoded (JPEG) or uploaded (pixels) one at a time, expanded to RGB
  std::vector<DeviceArray<uint8_t>> bitmaps(n);
  DeviceArray<uint8_t> staging;
  int64_t rgb_px = 0;
  uint64_t launches = 0;
  for (int i = 0; i < n; ++i) {
    const b2m_image_source& s = images[i].color;
    cams[i].bw = cams[i].bh = 0;
    cams[i].rgb_off = 3 * rgb_px;
    if (!s.data) continue;
    const uint8_t* src = nullptr;
    int W = 0, H = 0, ch = 0;
    int64_t stride = 0;
    if (s.kind == B2M_SOURCE_JPEG) {
      if (int rc = image_io_decode_jpeg(ctx, s, &src, &W, &H, &ch)) return rc;
      stride = static_cast<int64_t>(W) * ch;
    } else {
      W = s.width;
      H = s.height;
      ch = s.channels;
      stride = static_cast<int64_t>(W) * ch;
      B2M_CUDA_TRY(ctx, staging.ensure(static_cast<size_t>(stride) * H));
      B2M_CUDA_TRY(ctx, cudaMemcpy2DAsync(staging, stride, s.data, s.stride, stride, H, cudaMemcpyHostToDevice, st));
      src = staging;
    }
    B2M_CUDA_TRY(ctx, bitmaps[i].ensure(3 * static_cast<size_t>(W) * H));
    b2m_fu_rgb_kernel<<<blocks(static_cast<int64_t>(W) * H), kThreads, 0, st>>>(src, stride, W, H, ch, bitmaps[i]);
    B2M_CUDA_TRY(ctx, cudaGetLastError());
    B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));  // the staging / decode buffer is reused by the next image
    ++launches;
    cams[i].bw = W;
    cams[i].bh = H;
    rgb_px += static_cast<int64_t>(W) * H;
  }
  staging.reset();
  // depth 4, normal 12, mask 1, claim 4, overflow path 8 + 4 + 4 + 4 bytes per map pixel; RGB 3 per bitmap pixel;
  // per lattice slot kCap x (8 + 4 + 2 + 4) + kHash x 8 + kFrames x 24 + 8 bytes + records and visibility
  const double slot_b = kCap * 18.0 + kHash * 8.0 + kFrames * static_cast<double>(sizeof(Frame)) + 8.0 + sizeof(Rec);
  const double need = 41.0 * px + 3.0 * rgb_px + slot_b * lmax + 4.0 * std::min<double>(lmax * (double)n, (double)px) +
                      static_cast<double>(sizeof(Frame)) * opts->max_traversal_depth;
  {
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    if (need > static_cast<double>(free_b)) {
      char b[256];
      snprintf(b, sizeof(b), "[fusion.cu] the workspace's maps and fusion state need %.1f MB of device memory, %.1f MB "
               "are available", need / 1e6, free_b / 1e6);
      return fail(ctx, B2M_ENOMEM, b);
    }
  }
  DeviceArray<Cam> d_cams;
  DeviceArray<int32_t> d_ov, claim, status, n_list, scratch, big_img, big_scratch, ovf_keys, vis;
  DeviceArray<float> depth, normal;
  DeviceArray<uint8_t> rgb, fused, mask_stage;
  DeviceArray<int64_t> list_id, hash, big_id;
  DeviceArray<int32_t> list_img;
  DeviceArray<int16_t> list_slot;
  DeviceArray<Frame> frames, big_frames;
  DeviceArray<uint32_t> stamp;
  DeviceArray<Counters> cnt;
  DeviceArray<Rec> rec;
  const int64_t L = std::max<int64_t>(lmax, 1);
  const int64_t vis_cap = std::max<int64_t>(1, std::min<int64_t>(L * std::max(n, 1), std::max<int64_t>(px, 1)));
  B2M_CUDA_TRY(ctx, d_cams.ensure(std::max(n, 1)));
  B2M_CUDA_TRY(ctx, d_ov.ensure(ov.size()));
  B2M_CUDA_TRY(ctx, depth.ensure(px));
  B2M_CUDA_TRY(ctx, normal.ensure(3 * px));
  B2M_CUDA_TRY(ctx, fused.ensure(px));
  B2M_CUDA_TRY(ctx, claim.ensure(px));
  B2M_CUDA_TRY(ctx, rgb.ensure(3 * rgb_px));
  B2M_CUDA_TRY(ctx, big_id.ensure(px));
  B2M_CUDA_TRY(ctx, big_img.ensure(px));
  B2M_CUDA_TRY(ctx, big_scratch.ensure(px));
  B2M_CUDA_TRY(ctx, stamp.ensure(px + 1));
  B2M_CUDA_TRY(ctx, big_frames.ensure(opts->max_traversal_depth));
  B2M_CUDA_TRY(ctx, list_id.ensure(L * kCap));
  B2M_CUDA_TRY(ctx, list_img.ensure(L * kCap));
  B2M_CUDA_TRY(ctx, list_slot.ensure(L * kCap));
  B2M_CUDA_TRY(ctx, scratch.ensure(L * kCap));
  B2M_CUDA_TRY(ctx, hash.ensure(L * kHash));
  B2M_CUDA_TRY(ctx, frames.ensure(L * kFrames));
  B2M_CUDA_TRY(ctx, status.ensure(L));
  B2M_CUDA_TRY(ctx, n_list.ensure(L));
  B2M_CUDA_TRY(ctx, ovf_keys.ensure(L));
  B2M_CUDA_TRY(ctx, rec.ensure(L));
  B2M_CUDA_TRY(ctx, vis.ensure(vis_cap));
  B2M_CUDA_TRY(ctx, cnt.ensure(1));
  if (n > 0) B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_cams, cams.data(), sizeof(Cam) * n, cudaMemcpyHostToDevice, st));
  if (!ov.empty()) B2M_CUDA_TRY(ctx, cudaMemcpyAsync(d_ov, ov.data(), sizeof(int32_t) * ov.size(), cudaMemcpyHostToDevice, st));
  B2M_CUDA_TRY(ctx, cudaMemsetAsync(fused, 0, px, st));
  B2M_CUDA_TRY(ctx, cudaMemsetAsync(hash, 0, sizeof(int64_t) * L * kHash, st));
  B2M_CUDA_TRY(ctx, cudaMemsetAsync(stamp, 0, sizeof(uint32_t) * (px + 1), st));
  b2m_fu_fill_kernel<<<blocks(std::max<int64_t>(px, 1)), kThreads, 0, st>>>(claim, px, INT_MAX);
  B2M_CUDA_TRY(ctx, cudaGetLastError());
  ++launches;
  for (int i = 0; i < n; ++i) {
    const b2m_fusion_image& m = images[i];
    if (!m.depth) continue;
    const int64_t np = static_cast<int64_t>(m.width) * m.height;
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(depth + cams[i].px_off, m.depth, 4 * np, cudaMemcpyHostToDevice, st));
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(normal + 3 * cams[i].px_off, m.normal, 12 * np, cudaMemcpyHostToDevice, st));
    if (m.mask) {
      B2M_CUDA_TRY(ctx, mask_stage.ensure(np));
      B2M_CUDA_TRY(ctx, cudaMemcpyAsync(mask_stage, m.mask, np, cudaMemcpyHostToDevice, st));
      b2m_fu_mask_kernel<<<blocks(np), kThreads, 0, st>>>(mask_stage, np, fused + cams[i].px_off);
      B2M_CUDA_TRY(ctx, cudaGetLastError());
      B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
      ++launches;
    }
    if (cams[i].bw > 0)
      B2M_CUDA_TRY(ctx, cudaMemcpyAsync(rgb + cams[i].rgb_off, bitmaps[i], 3 * static_cast<size_t>(cams[i].bw) * cams[i].bh,
                                        cudaMemcpyDeviceToDevice, st));
  }
  B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
  bitmaps.clear();

  FuArgs a{};
  a.cams = d_cams;
  a.ov = d_ov;
  a.depth = depth;
  a.normal = normal;
  a.rgb = rgb;
  a.fused = fused;
  a.claim = claim;
  a.o.min_num_pixels = opts->min_num_pixels;
  a.o.max_num_pixels = opts->max_num_pixels;
  a.o.max_traversal_depth = opts->max_traversal_depth;
  a.o.max_reproj_sq = opts->max_reproj_error * opts->max_reproj_error;
  a.o.max_depth_error = opts->max_depth_error;
  a.o.min_cos_normal = static_cast<float>(std::cos(static_cast<double>(opts->max_normal_error) * 3.14159265358979323846 / 180.0));
  std::memcpy(a.o.bbox, opts->bounding_box, sizeof(a.o.bbox));
  a.list_id = list_id;
  a.list_img = list_img;
  a.list_slot = list_slot;
  a.hash = hash;
  a.frames = frames;
  a.scratch = scratch;
  a.status = status;
  a.n_list = n_list;
  a.big_id = big_id;
  a.big_img = big_img;
  a.stamp = stamp;
  a.stamp_next = stamp + px;
  a.big_frames = big_frames;
  a.big_scratch = big_scratch;
  a.big_cap = px;
  a.ovf_keys = ovf_keys;
  a.cnt = cnt;
  a.rec = rec;
  a.vis = vis;

  Counters total{};
  uint64_t rounds = 0;
  std::vector<Rec> hrec;
  std::vector<int32_t> hvis, hkeys;
  for (int img = 0; img < n; ++img) {
    if (!images[img].depth) continue;
    const int W = images[img].width, H = images[img].height;
    for (int phase = 0; phase < kLattice * kLattice; ++phase) {
      a.img = img;
      a.py = phase / kLattice;
      a.px = phase % kLattice;
      a.lw = (W - a.px + kLattice - 1) / kLattice;
      a.L = a.lw * ((H - a.py + kLattice - 1) / kLattice);
      if (a.L <= 0) continue;
      for (;;) {
        if (ctx->stop) return fail(ctx, B2M_ESTOPPED, "[fusion.cu] stopped by b2m_request_stop");
        Counters c{};
        B2M_CUDA_TRY(ctx, cudaMemsetAsync(cnt, 0, sizeof(Counters), st));
        a.round = static_cast<int32_t>(rounds);
        b2m_fu_speculate_kernel<<<blocks(a.L), kThreads, 0, st>>>(a);
        B2M_CUDA_TRY(ctx, cudaGetLastError());
        B2M_CUDA_TRY(ctx, cudaMemcpyAsync(&c, cnt, sizeof(Counters), cudaMemcpyDeviceToHost, st));
        B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
        ++launches;
        if (c.live == 0) break;
        const int n_ovf = static_cast<int>(c.ovf);
        if (n_ovf > 0) {  // ascending key, so that the overflow path's work does not depend on thread timing
          hkeys.resize(n_ovf);
          B2M_CUDA_TRY(ctx, cudaMemcpy(hkeys.data(), ovf_keys, sizeof(int32_t) * n_ovf, cudaMemcpyDeviceToHost));
          std::sort(hkeys.begin(), hkeys.end());
          B2M_CUDA_TRY(ctx, cudaMemcpy(ovf_keys, hkeys.data(), sizeof(int32_t) * n_ovf, cudaMemcpyHostToDevice));
          b2m_fu_overflow_kernel<<<1, 1, 0, st>>>(a, n_ovf, 0);
          B2M_CUDA_TRY(ctx, cudaGetLastError());
          ++launches;
        }
        b2m_fu_decide_kernel<<<blocks(a.L), kThreads, 0, st>>>(a);
        B2M_CUDA_TRY(ctx, cudaGetLastError());
        ++launches;
        if (n_ovf > 0) {
          for (int step = 1; step <= 2; ++step) {
            b2m_fu_overflow_kernel<<<1, 1, 0, st>>>(a, n_ovf, step);
            B2M_CUDA_TRY(ctx, cudaGetLastError());
            ++launches;
          }
        }
        b2m_fu_commit_kernel<<<blocks(a.L), kThreads, 0, st>>>(a);
        B2M_CUDA_TRY(ctx, cudaGetLastError());
        ++launches;
        if (n_ovf > 0) {
          b2m_fu_overflow_kernel<<<1, 1, 0, st>>>(a, n_ovf, 3);
          B2M_CUDA_TRY(ctx, cudaGetLastError());
          ++launches;
        }
        B2M_CUDA_TRY(ctx, cudaMemcpyAsync(&c, cnt, sizeof(Counters), cudaMemcpyDeviceToHost, st));
        B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
        hrec.resize(c.n_rec);
        hvis.resize(c.n_vis);
        if (c.n_rec) B2M_CUDA_TRY(ctx, cudaMemcpy(hrec.data(), rec, sizeof(Rec) * c.n_rec, cudaMemcpyDeviceToHost));
        if (c.n_vis) B2M_CUDA_TRY(ctx, cudaMemcpy(hvis.data(), vis, sizeof(int32_t) * c.n_vis, cudaMemcpyDeviceToHost));
        std::sort(hrec.begin(), hrec.end(), [](const Rec& x, const Rec& y) { return x.key < y.key; });
        for (const Rec& r : hrec) {
          F->order.insert(F->order.end(), {r.img, r.row, r.col, static_cast<int32_t>(rounds)});
          if (!r.emitted) continue;
          F->xyz.insert(F->xyz.end(), r.xyz, r.xyz + 3);
          F->nrm.insert(F->nrm.end(), r.nrm, r.nrm + 3);
          F->rgb.insert(F->rgb.end(), r.rgb, r.rgb + 3);
          F->vis.insert(F->vis.end(), hvis.begin() + r.vis_off, hvis.begin() + r.vis_off + r.nvis);
          F->vis_off.push_back(static_cast<int64_t>(F->vis.size()));
          F->seeds.insert(F->seeds.end(), {r.img, r.row, r.col});
        }
        total.live += c.live;
        total.deferred += c.deferred;
        total.n_rec += c.n_rec;
        total.pops += c.pops;
        total.traversals += c.traversals;
        ++rounds;
        if (c.deferred == 0) break;  // committed pixels stay fused: without a deferred candidate nothing is live
      }
    }
  }
  ctx->stats.kernel_launches += launches;
  ctx->stats.fusion_seeds += total.n_rec;
  ctx->stats.fusion_traversals += total.traversals;
  ctx->stats.fusion_pops += total.pops;
  ctx->stats.fusion_rounds += rounds;
  ctx->stats.fusion_deferred += total.deferred;
  ctx->stats.fusion_points += F->xyz.size() / 3;
  *out = F.release();
  return B2M_OK;
}

int b2m_fused_points_get(const b2m_fused_points* p, b2m_fused_points_view* out) {
  if (!p || !out) return B2M_EINVAL;
  std::memset(out, 0, sizeof(*out));
  out->struct_size = sizeof(*out);
  out->n_points = static_cast<int64_t>(p->xyz.size() / 3);
  out->xyz = p->xyz.data();
  out->normals = p->nrm.data();
  out->colors = p->rgb.data();
  out->vis_off = p->vis_off.data();
  out->vis = p->vis.data();
  out->seeds = p->seeds.data();
  out->n_order = static_cast<int64_t>(p->order.size() / 4);
  out->order = p->order.data();
  return B2M_OK;
}

void b2m_fused_points_free(b2m_fused_points* p) { delete p; }

}  // extern "C"
