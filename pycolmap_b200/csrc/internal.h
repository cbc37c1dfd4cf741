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
#include "cuda_owned.cuh"

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
  DeviceArray<uint8_t> d_desc;
  DeviceArray<float2> d_kpts;  // indexed by padded row, or empty
  DeviceArray<int32_t> d_row0;
  DeviceArray<int32_t> d_nfeat;
  std::vector<b2m_camera> cams;
  uint64_t generation = 0;  // bumped by every b2m_set_images*: consumers caching per-set state (device cameras)
                            // key on this, not on d_desc (the allocator may hand the same address out again)
  CUtensorMap tmap{};       // box 128 bytes x 128 rows
  void release() { *this = ImageSet(); }
};

// Scratch of the gathered column direction (launch_k1_filter_gather), allocated on first use.
struct GatherBufs {
  DeviceArray<uint8_t> desc;    // [batch x mstride x 128]
  DeviceArray<int32_t> colrank; // [batch][mstride]
  DeviceArray<int32_t> cols;    // [batch][mstride]
  DeviceArray<int32_t> cnt;     // [batch]
  DeviceArray<int32_t> items;   // [batch x mstride / 256][2]
  DeviceArray<int32_t> n;       // [1]
  CUtensorMap tmap{};
};

struct Workspace {
  int batch = 0;
  int32_t mstride = 0;
  DeviceArray<int32_t> d_mbuf;
  DeviceArray<uint2> d_aux;           // K1 v2: (best, S1) per candidate row
  DeviceArray<int32_t> d_cand_cnt;    // K1 v2: [batch][2]
  DeviceArray<int32_t> d_cand_rows;   // K1 v2: [batch][2][mstride]
  DeviceArray<int32_t> d_cand_sorted;
  DeviceArray<int32_t> d_pairs_dir1;  // [batch][2] swapped / dummy pairs of launch_k1_filter_skip
  GatherBufs gath;
  DeviceArray<uint2> d_arena[2];
  DeviceArray<unsigned long long> d_cursor[2];
  DeviceArray<int64_t> d_pair_off[2];
  DeviceArray<int32_t> d_pair_cnt[2];
  PinnedArray<uint2> h_arena[2];
  PinnedArray<unsigned long long> h_cursor[2];
  PinnedArray<int64_t> h_pair_off[2];
  PinnedArray<int32_t> h_pair_cnt[2];
};

// message of a failing call that has no context to carry it (b2m_create, b2m_comm_get_unique_id)
extern thread_local std::string g_noctx_err;

// Indices into b2m_ctx::d_counters, the kernel-side counters behind b2m_stats: models scored, then residual evaluations.
constexpr int kVerifyCounters = 0;    // [6]: per model kind E, F, H (verify.cu)
constexpr int kAbsPoseCounters = 6;   // [2] (abs_pose.cu)
constexpr int kTriCounters = 8;       // [2] (triangulation.cu)
constexpr int kPmCounters = 10;       // [1]: window samples evaluated (patch_match.cu)
constexpr int kNumCounters = 11;

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
  b2m::Stream stream;
  b2m::Stream copy_stream;
  b2m::Event ev_k[2];
  b2m::Event ev_data[2];
  b2m::Event ev_t0, ev_t1;
  b2m::Event ev_k1a[2], ev_k1b[2];
  // overlapped schedule (api.cu): exact resolve + gather of batch b run on `aux_stream` next to the RANSAC kernels of
  // batch b - 1; ev_p1 = that work done, ev_g2a / ev_g2b bracket the gathered GEMM (timing)
  b2m::Stream aux_stream;
  b2m::Event ev_p1[2], ev_g2a[2], ev_g2b[2];
  b2m::DeviceArray<float> d_lut;
  b2m::DeviceArray<unsigned long long> d_counters;  // [kNumCounters], zeroed by b2m_create and b2m_reset_stats
  b2m::ImageSet images;
  b2m::Workspace ws;
  b2m::DeviceArray<int32_t> d_pairs;
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
  void* tri_state = nullptr;     // b2m::TriState (triangulation.cu): pinned staging and device buffers
  void* sift_state = nullptr;    // b2m::SiftState (sift.cu): pyramid, gradient and keypoint buffers
  void* image_io_state = nullptr;  // b2m::ImageIoState (image_io.cu): nvJPEG handles, decode and rescale buffers
  void* pm_state = nullptr;        // b2m::PmState (patch_match.cu): the resident images, depth maps and map buffers
  void* undistort_state = nullptr; // b2m::UndistortState (undistort.cu): source, warp and rescale buffers
};

namespace b2m {
// Sets the error message of `ctx` (nullptr: of the calling thread) and returns `code`.
inline int fail(b2m_ctx* ctx, int code, const std::string& msg) {
  if (ctx) ctx->err = msg; else g_noctx_err = msg;
  return code;
}
// triangulation.cu
void tri_release(b2m_ctx* ctx);
// sift.cu
void sift_release(b2m_ctx* ctx);
// One extraction call: the options, checked, and the Gaussian filters sift_begin uploaded for them.
struct SiftPlan {
  b2m_extract_opts opts;
  std::vector<int> tap_off, tap_r;
};
// SiftExtractionOptions::Check and the size checks of n images (widths / heights), then the buffers sized for the
// largest of them and the filter taps uploaded.
int sift_begin(b2m_ctx* ctx, const b2m_extract_opts* opts, const int32_t* widths, const int32_t* heights, int32_t n,
               SiftPlan* plan);
// K6 on one W x H grey image (`stride` bytes per row) in host memory, or in device memory when `on_device`; appends
// its features to F.  *d_kout (when not NULL) = the device copy of its [n x 4] keypoints, valid until the next call.
int sift_extract(b2m_ctx* ctx, const SiftPlan& plan, const uint8_t* img, int64_t stride, int W, int H, bool on_device,
                 b2m_features* F, const float** d_kout);
// image_io.cu
void image_io_release(b2m_ctx* ctx);
// Decodes a B2M_SOURCE_JPEG source with nvJPEG: *pixels = W x H x channels (1 or 3) bytes in device memory, valid until
// the next decode on this context.
int image_io_decode_jpeg(b2m_ctx* ctx, const b2m_image_source& src, const uint8_t** pixels, int* W, int* H,
                         int* channels);
// FreeImage's bilinear Rescale (FILTER_BILINEAR) of a W x H image of `channels` interleaved bytes per pixel into dst
// (w x h x channels) on `st`: fp64 weight tables per axis, two separable passes through an 8-bit intermediate, the
// pass order chosen from the aspect ratio as CResizeEngine::scale does.  Returns once the result is on the device.
struct RescaleBufs {
  DeviceArray<uint8_t> tmp;
  DeviceArray<int> tab_i;
  DeviceArray<double> tab_w;
};
int rescale_bilinear(b2m_ctx* ctx, const uint8_t* src, int W, int H, int channels, int w, int h, RescaleBufs& b,
                     uint8_t* dst, cudaStream_t st);
// nvJPEG's encoder on a W x H RGB interleaved device image, quality 100, 4:2:0: the file's bytes in *out.
int image_io_encode_jpeg(b2m_ctx* ctx, const uint8_t* rgb, int W, int H, cudaStream_t st, std::vector<uint8_t>* out);
// patch_match.cu
void pm_release(b2m_ctx* ctx);
// undistort.cu
void undistort_release(b2m_ctx* ctx);
}  // namespace b2m

struct b2m_features {
  std::vector<int64_t> off;   // [n_images + 1] feature offsets
  std::vector<float> kpts;    // [total x 4] (b2m_extract_features_batch) or [total x 6] (b2m_extract_features_sources)
  std::vector<uint8_t> desc;  // [total x 128]
  // b2m_extract_features_sources only, per image: decoded width / height, status and the reason of a failed decode
  std::vector<int32_t> width, height, status;
  std::vector<std::string> error;
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
