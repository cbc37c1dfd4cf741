// internal.h -- context / image-set / results objects behind the C ABI (include/b200match.h).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "../../include/b200match.h"
#include "camera_models.h"

namespace b2m {

// nullptr when the verifier can take this camera, else the reason (-> B2M_EINVAL message).
inline const char* camera_problem(const b2m_camera& c) {
  if (c.struct_size != sizeof(b2m_camera))
    return "[internal.h] Check Failed: b2m_camera.struct_size == sizeof(b2m_camera) (ABI version 2: 12 parameters)";
  if (cam::num_params(c.model) < 0)
    return "[internal.h] camera model id is not supported (COLMAP 3.9.1 model ids 0-10)";
  double fx, fy, cx, cy;
  int extra;
  cam::intrinsics(c.model, c.params, &fx, &fy, &cx, &cy, &extra);
  if (!(fx > 0.0) || !(fy > 0.0)) return "[internal.h] Check Failed: camera focal length > 0";
  return nullptr;
}

// The descriptor set resident in HBM (replaces upstream's host-side FeatureMatcherCache,
// U:controllers/feature_matching_utils.cc).  Layout: one [total_rows x 128] uint8 array, image i
// occupying rows [row0[i], row0[i] + nfeat[i]) followed by zero rows up to a multiple of kRowPad.
struct ImageSet {
  int n_images = 0;
  std::vector<int32_t> nfeat, row0;
  int32_t max_feat = 0;      // max valid rows
  int32_t max_feat_pad = 0;  // max padded rows
  int64_t total_rows = 0;    // padded rows over all images
  uint8_t* d_desc = nullptr;
  float2* d_kpts = nullptr;  // indexed by padded row, or nullptr
  int32_t* d_row0 = nullptr;
  int32_t* d_nfeat = nullptr;
  std::vector<b2m_camera> cams;
  uint64_t generation = 0;  // bumped by every b2m_set_images*: consumers caching per-set state (device cameras)
                            // key on this, not on d_desc (the allocator may hand the same address out again)
  CUtensorMap tmap{};       // box 128 bytes x 128 rows
  void release();
};

struct Workspace {
  int batch = 0;
  int32_t mstride = 0;
  int32_t* d_mbuf = nullptr;
  uint2* d_aux = nullptr;          // K1 v2: (best, S1) per candidate row
  int32_t* d_cand_cnt = nullptr;   // K1 v2: [batch][2]
  int32_t* d_cand_rows = nullptr;  // K1 v2: [batch][2][mstride]
  int32_t* d_cand_sorted = nullptr;
  int32_t* d_pairs_dir1 = nullptr; // [batch][2] swapped / dummy pairs of launch_k1_filter_skip
  // gathered column direction (launch_k1_filter_gather), allocated on first use
  uint8_t* d_gath_desc = nullptr;  // [batch x mstride x 128]
  int32_t* d_colrank = nullptr;    // [batch][mstride]
  int32_t* d_gath_cols = nullptr;  // [batch][mstride]
  int32_t* d_gath_cnt = nullptr;   // [batch]
  int32_t* d_gath_items = nullptr; // [batch x mstride / 256][2]
  int32_t* d_gath_n = nullptr;     // [1]
  CUtensorMap tmap_gath{};
  uint2* d_arena[2] = {nullptr, nullptr};
  unsigned long long* d_cursor[2] = {nullptr, nullptr};
  int64_t* d_pair_off[2] = {nullptr, nullptr};
  int32_t* d_pair_cnt[2] = {nullptr, nullptr};
  uint2* h_arena[2] = {nullptr, nullptr};
  unsigned long long* h_cursor[2] = {nullptr, nullptr};
  int64_t* h_pair_off[2] = {nullptr, nullptr};
  int32_t* h_pair_cnt[2] = {nullptr, nullptr};
  void release();
};

// message of a failing call that has no context to carry it (b2m_create, b2m_comm_get_unique_id)
extern thread_local std::string g_noctx_err;

}  // namespace b2m

struct b2m_ctx;
namespace b2m {
// comm.cu
void comm_release(b2m_ctx* ctx);
int comm_allgather_regions(b2m_ctx* ctx, uint8_t* base, const std::vector<size_t>& off, const std::vector<size_t>& len,
                           cudaStream_t st);
}  // namespace b2m

struct b2m_ctx {
  int device = 0;
  int num_sms = 132;
  uint64_t seed = 0;
  bool pair_batch_auto = true;  // no explicit b2m_device_cfg.pair_batch: the batch scales with the image size (api.cu)
  int pair_batch = 4096;  // pairs per kernel batch: ~380 verifiable pairs x 3 model kinds per launch keep the RANSAC
                          // kernels at several CTAs per SM
  cudaStream_t stream = nullptr;
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_k[2] = {nullptr, nullptr};
  cudaEvent_t ev_data[2] = {nullptr, nullptr};
  cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;
  cudaEvent_t ev_k1a[2] = {nullptr, nullptr}, ev_k1b[2] = {nullptr, nullptr};
  // overlapped schedule (api.cu): exact resolve + gather of batch b run on `aux_stream` next to the RANSAC kernels of
  // batch b - 1; ev_p1 = that work done, ev_g2a / ev_g2b bracket the gathered GEMM (timing)
  cudaStream_t aux_stream = nullptr;
  cudaEvent_t ev_p1[2] = {nullptr, nullptr}, ev_g2a[2] = {nullptr, nullptr}, ev_g2b[2] = {nullptr, nullptr};
  float* d_lut = nullptr;
  b2m::ImageSet images;
  b2m::Workspace ws;
  int32_t* d_pairs = nullptr;
  int64_t d_pairs_cap = 0;
  std::string err;
  volatile int stop = 0;
  bool exact_k1 = false;  // use the exact top-2 epilogue (K1 v1) instead of filter + resolve (K1 v2)
  int k1_dir1_mode = B2M_K1_DIR1_UNTESTED;  // see b2m_stats.k1_dir1_mode
  uint64_t hint_matches = 0, hint_inliers = 0;  // result sizes of the previous b2m_match_pairs (reserve hints)
  b2m_stats stats{};
  void* verify_state = nullptr;  // b2m::VerifyState (verify.cu)
  // multi-GPU (comm.cu): the NCCL communicator this context joined, or nullptr
  void* comm = nullptr;          // ncclComm_t
  int comm_size = 1, comm_rank = 0;
  unsigned long long* d_verify_counters = nullptr;  // [6]: models scored / residual evaluations per kind (verify.cu)
};

namespace b2m {
// Allocator of the two big result arrays (hundreds of MB per exhaustive call): resize() leaves new elements
// uninitialised -- every element is overwritten by the memcpy that follows -- instead of zero-filling them first.
template <class T>
struct NoInitAlloc : std::allocator<T> {
  template <class U> struct rebind { using other = NoInitAlloc<U>; };
  NoInitAlloc() = default;
  template <class U> NoInitAlloc(const NoInitAlloc<U>&) {}
  template <class U> void construct(U* p) noexcept { ::new (static_cast<void*>(p)) U; }
  template <class U, class... A> void construct(U* p, A&&... a) { ::new (static_cast<void*>(p)) U(std::forward<A>(a)...); }
};
using BigU32 = std::vector<uint32_t, NoInitAlloc<uint32_t>>;
}  // namespace b2m

struct b2m_results {
  ~b2m_results();                // parks the two big arrays in a one-deep process-wide cache (api.cu)
  std::vector<int32_t> pairs;    // [n x 2]
  std::vector<int64_t> off;      // per pair offset (in matches) into `matches`
  std::vector<int32_t> cnt;      // per pair match count
  b2m::BigU32 matches;           // [total x 2]
  // verification outputs (filled when tvg options were given)
  bool verified = false;
  std::vector<int32_t> config;
  std::vector<int64_t> in_off;
  std::vector<int32_t> in_cnt;
  b2m::BigU32 inliers;
  std::vector<int32_t> model_idx; // per pair: index into `models` (x 27), or -1 (no geometry: E = F = H = 0)
  std::vector<double> models;    // 27 doubles (E, F, H) per pair that has a geometry -- ~10 % of an exhaustive run
  std::vector<double> poses;     // per pair 8 doubles: qvec (w, x, y, z), tvec, tri_angle (compute_relative_pose)
  std::vector<int32_t> pose_valid;
};
