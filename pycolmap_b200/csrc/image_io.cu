// image_io.cu -- K7: what COLMAP's feature extraction does to an image around SIFT (U:controllers/image_reader.cc,
// U:controllers/feature_extraction.cc; SURVEY.md rows U1-U6), on the device:
//   decode      JPEG with nvJPEG (linked statically); host pixels (grey / RGB / RGBA) are uploaded as they are
//   grey        FreeImage's ConvertToGreyscale: (BYTE)(0.2126f r + 0.7152f g + 0.0722f b + 0.5f), alpha ignored
//   downscale   FreeImage's Rescale with FILTER_BILINEAR when max(w, h) > max_image_size: per-axis weight tables
//               (built on the host in fp64, as CWeightsTable does), two separable passes with fp64 accumulation and an
//               8-bit rounded intermediate, the pass order chosen from the aspect ratio as CResizeEngine::scale does
//   SIFT        K6 (sift.cu) started from the device buffer; decode, grey and rescale of the next images run on a
//               decoder thread and a side stream while K6 runs the current one
//   keypoints   FeatureKeypoint(x, y, scale, orientation) -> 6 columns, ScaleKeypoints back to the original size and
//               MaskKeypoints, one thread per keypoint; the kept rows are compacted in the copy to the host
// The file is compiled without FMA contraction: the grey conversion and the rescale sums are rounded per operation, as
// the x86 code of FreeImage rounds them.
#include <cuda_runtime.h>
#include <nvjpeg.h>

#include <algorithm>
#include <cmath>
#include <condition_variable>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "internal.h"

namespace b2m {
namespace {

// ---- kernels --------------------------------------------------------------------------------------------------------
// Rec709 luma of FreeImage's GREY macro; one channel passes through.
__global__ void b2m_grey_kernel(const uint8_t* __restrict__ src, int64_t pitch, int channels, int W, int H,
                                uint8_t* __restrict__ dst) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<int64_t>(W) * H) return;
  const int y = static_cast<int>(i / W), x = static_cast<int>(i % W);
  const uint8_t* p = src + y * pitch + static_cast<int64_t>(x) * channels;
  if (channels == 1) {
    dst[i] = p[0];
    return;
  }
  float v = __fadd_rn(__fmul_rn(0.2126f, static_cast<float>(p[0])), __fmul_rn(0.7152f, static_cast<float>(p[1])));
  v = __fadd_rn(v, __fmul_rn(0.0722f, static_cast<float>(p[2])));
  dst[i] = static_cast<uint8_t>(__fadd_rn(v, 0.5f));
}

// One axis of FreeImage's weight table: destination pixel u reads count[u] source pixels from left[u] with the
// weights w[off[u] ...].
struct Weights {
  const int* left;
  const int* count;
  const int* off;
  const double* w;
};

__device__ __forceinline__ uint8_t round_byte(double v) {
  const int r = static_cast<int>(v + 0.5);
  return static_cast<uint8_t>(r < 0 ? 0 : (r > 255 ? 255 : r));
}

// horizontalFilter: src sw x h -> dst dw x h, `channels` interleaved bytes per pixel, each filtered on its own
__global__ void b2m_rescale_h_kernel(const uint8_t* __restrict__ src, int sw, int h, int channels, Weights t, int dw,
                                     uint8_t* __restrict__ dst) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<int64_t>(dw) * h * channels) return;
  const int64_t px = i / channels;
  const int c = static_cast<int>(i % channels);
  const int y = static_cast<int>(px / dw), x = static_cast<int>(px % dw);
  const uint8_t* row = src + (static_cast<int64_t>(y) * sw + t.left[x]) * channels + c;
  const double* w = t.w + t.off[x];
  double v = 0.0;
  for (int k = 0; k < t.count[x]; ++k)
    v = __dadd_rn(v, __dmul_rn(w[k], static_cast<double>(row[static_cast<int64_t>(k) * channels])));
  dst[i] = round_byte(v);
}

// verticalFilter: src w x sh -> dst w x dh, `channels` interleaved bytes per pixel
__global__ void b2m_rescale_v_kernel(const uint8_t* __restrict__ src, int w, int sh, int channels, Weights t, int dh,
                                     uint8_t* __restrict__ dst) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t rowlen = static_cast<int64_t>(w) * channels;
  if (i >= rowlen * dh) return;
  const int y = static_cast<int>(i / rowlen);
  const int64_t xc = i % rowlen;
  const uint8_t* col = src + static_cast<int64_t>(t.left[y]) * rowlen + xc;
  const double* wt = t.w + t.off[y];
  double v = 0.0;
  for (int k = 0; k < t.count[y]; ++k) v = __dadd_rn(v, __dmul_rn(wt[k], static_cast<double>(col[static_cast<int64_t>(k) * rowlen])));
  dst[i] = round_byte(v);
}

// FeatureKeypoint(x, y, scale, orientation), then FeatureKeypoint::Rescale(sx, sy) when the image was downscaled, then
// the mask test at the integer pixel of the original-image position.  cos / sin in fp64 rounded to fp32: the correctly
// rounded value std::cos(float) gives on the host.
__global__ void b2m_keypoint_finish_kernel(const float* __restrict__ k4, int n, int rescale, float sx, float sy,
                                           const uint8_t* __restrict__ mask, int mw, int mh, int64_t mstride,
                                           float* __restrict__ k6, uint8_t* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float x = k4[4 * i], y = k4[4 * i + 1];
  const float sc = k4[4 * i + 2], ori = k4[4 * i + 3];
  const float c = __fmul_rn(sc, static_cast<float>(cos(static_cast<double>(ori))));
  const float s = __fmul_rn(sc, static_cast<float>(sin(static_cast<double>(ori))));
  float a11 = c, a12 = -s, a21 = s, a22 = c;
  if (rescale) {
    x = __fmul_rn(x, sx);
    y = __fmul_rn(y, sy);
    a11 = __fmul_rn(a11, sx);
    a12 = __fmul_rn(a12, sy);
    a21 = __fmul_rn(a21, sx);
    a22 = __fmul_rn(a22, sy);
  }
  float* o = k6 + 6 * static_cast<int64_t>(i);
  o[0] = x; o[1] = y; o[2] = a11; o[3] = a12; o[4] = a21; o[5] = a22;
  uint8_t k = 1;
  if (mask) {
    const int px = static_cast<int>(x), py = static_cast<int>(y);
    k = (px >= 0 && py >= 0 && px < mw && py < mh && mask[static_cast<int64_t>(py) * mstride + px] != 0) ? 1 : 0;
  }
  keep[i] = k;
}

// ---- host side ------------------------------------------------------------------------------------------------------
// nvJPEG: the hardware backend (the JPEG engines of the GPU; baseline, single-scan files) where it exists and takes the
// file, the GPU hybrid backend (Huffman decoding on the host; also progressive files) otherwise.
struct Nvjpeg {
  nvjpegHandle_t hybrid = nullptr, hw = nullptr;
  nvjpegJpegState_t hybrid_state = nullptr, hw_rgb = nullptr, hw_y = nullptr;
  nvjpegJpegStream_t hw_stream = nullptr;
  nvjpegEncoderState_t enc_state = nullptr;  // K10's JPEG output, on the hybrid handle
  nvjpegEncoderParams_t enc_params = nullptr;
  bool hw_tried = false;
  void drop_hw() {
    if (hw_stream) nvjpegJpegStreamDestroy(hw_stream);
    if (hw_rgb) nvjpegJpegStateDestroy(hw_rgb);
    if (hw_y) nvjpegJpegStateDestroy(hw_y);
    if (hw) nvjpegDestroy(hw);
    hw_stream = nullptr;
    hw_rgb = hw_y = nullptr;
    hw = nullptr;
  }
  ~Nvjpeg() {
    drop_hw();
    if (enc_params) nvjpegEncoderParamsDestroy(enc_params);
    if (enc_state) nvjpegEncoderStateDestroy(enc_state);
    if (hybrid_state) nvjpegJpegStateDestroy(hybrid_state);
    if (hybrid) nvjpegDestroy(hybrid);
  }
};

// The buffers one image goes through between decode and SIFT.
struct Slot {
  DeviceArray<uint8_t> src, grey, small;
  RescaleBufs rs;
};

constexpr int kSlots = 3;  // images decoded ahead of K6, plus the one K6 reads

struct ImageIoState {
  Nvjpeg jpeg;
  Stream side;  // decode, grey and rescale run here, next to K6 on the library stream
  Slot slot[kSlots];
  DeviceArray<uint8_t> d_mask, d_keep;
  DeviceArray<float> d_k6;
};

inline unsigned blocks_for(int64_t n, int t) { return static_cast<unsigned>((n + t - 1) / t); }

// CWeightsTable(CBilinearFilter, dst, src): FreeImage's contributions of one axis, in fp64.
struct AxisTable {
  std::vector<int> left, count, off;
  std::vector<double> w;
};

AxisTable bilinear_table(int dst, int src) {
  AxisTable t;
  const double filter_width = 1.0;  // CBilinearFilter
  const double scale = static_cast<double>(dst) / static_cast<double>(src);
  const double width = scale < 1.0 ? filter_width / scale : filter_width;
  const double fscale = scale < 1.0 ? scale : 1.0;
  const double offset = 0.5 / scale;
  for (int u = 0; u < dst; ++u) {
    const double center = static_cast<double>(u) / scale + offset;
    const int left = std::max(0, static_cast<int>(center - width + 0.5));
    int right = std::min(static_cast<int>(center + width + 0.5), src);
    std::vector<double> w;
    double total = 0.0;
    for (int s = left; s < right; ++s) {
      const double d = std::fabs(fscale * (static_cast<double>(s) + 0.5 - center));
      const double weight = fscale * (d < filter_width ? filter_width - d : 0.0);
      w.push_back(weight);
      total += weight;
    }
    if (total > 0 && total != 1)
      for (double& v : w) v /= total;
    int trailing = right - left - 1;  // discard null weights at the right
    while (trailing >= 0 && w[trailing] == 0) {
      --right;
      --trailing;
      if (right == left) break;
    }
    t.left.push_back(left);
    t.count.push_back(right - left);
    t.off.push_back(static_cast<int>(t.w.size()));
    t.w.insert(t.w.end(), w.begin(), w.begin() + (right - left));
  }
  return t;
}

}  // namespace

int rescale_bilinear(b2m_ctx* ctx, const uint8_t* src, int W, int H, int channels, int w, int h, RescaleBufs& b,
                     uint8_t* dst, cudaStream_t st) {
  const AxisTable tx = bilinear_table(w, W), ty = bilinear_table(h, H);
  // one upload: [left | count | off] of x, then of y; weights of x then of y
  std::vector<int> ti;
  for (const AxisTable* t : {&tx, &ty}) {
    ti.insert(ti.end(), t->left.begin(), t->left.end());
    ti.insert(ti.end(), t->count.begin(), t->count.end());
    ti.insert(ti.end(), t->off.begin(), t->off.end());
  }
  std::vector<double> tw(tx.w);
  tw.insert(tw.end(), ty.w.begin(), ty.w.end());
  B2M_CUDA_TRY(ctx, b.tab_i.ensure(ti.size()));
  B2M_CUDA_TRY(ctx, b.tab_w.ensure(tw.size()));
  B2M_CUDA_TRY(ctx, cudaMemcpyAsync(b.tab_i, ti.data(), sizeof(int) * ti.size(), cudaMemcpyHostToDevice, st));
  B2M_CUDA_TRY(ctx, cudaMemcpyAsync(b.tab_w, tw.data(), sizeof(double) * tw.size(), cudaMemcpyHostToDevice, st));
  const int* di = b.tab_i;
  const Weights wx{di, di + w, di + 2 * w, b.tab_w};
  const int* dy = di + 3 * w;
  const Weights wy{dy, dy + h, dy + 2 * h, b.tab_w + tx.w.size()};
  const int c = channels;
  if (static_cast<int64_t>(w) * H <= static_cast<int64_t>(h) * W) {  // xy filtering: horizontal pass first
    B2M_CUDA_TRY(ctx, b.tmp.ensure(static_cast<size_t>(w) * H * c));
    b2m_rescale_h_kernel<<<blocks_for(static_cast<int64_t>(w) * H * c, 256), 256, 0, st>>>(src, W, H, c, wx, w, b.tmp);
    b2m_rescale_v_kernel<<<blocks_for(static_cast<int64_t>(w) * h * c, 256), 256, 0, st>>>(b.tmp, w, H, c, wy, h, dst);
  } else {  // yx filtering
    B2M_CUDA_TRY(ctx, b.tmp.ensure(static_cast<size_t>(W) * h * c));
    b2m_rescale_v_kernel<<<blocks_for(static_cast<int64_t>(W) * h * c, 256), 256, 0, st>>>(src, W, H, c, wy, h, b.tmp);
    b2m_rescale_h_kernel<<<blocks_for(static_cast<int64_t>(w) * h * c, 256), 256, 0, st>>>(b.tmp, W, h, c, wx, w, dst);
  }
  B2M_CUDA_TRY(ctx, cudaGetLastError());
  // the weight tables are pageable host memory read by the copies above: they live until the stream is done
  B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return B2M_OK;
}

namespace {

ImageIoState* state_of(b2m_ctx* ctx) {
  if (!ctx->image_io_state) ctx->image_io_state = new ImageIoState();
  return static_cast<ImageIoState*>(ctx->image_io_state);
}

// The size SIFT sees: ImageResizerThread's (int)(w * s) x (int)(h * s), s = max_image_size / max(w, h).
void target_size(int W, int H, int max_image_size, int* tw, int* th) {
  *tw = W;
  *th = H;
  if (W > max_image_size || H > max_image_size) {
    const double s = static_cast<double>(max_image_size) / std::max(W, H);
    *tw = static_cast<int>(W * s);
    *th = static_cast<int>(H * s);
  }
}

// What the decoder counted; added to b2m_stats by the calling thread.
struct DecodeCounts {
  uint64_t launches = 0, bytes = 0, images = 0, hardware = 0;
};

// The decoded image of one source, as K6 will read it.
struct Decoded {
  int rc = B2M_OK;      // B2M_EINVAL with `why` for a source that does not decode; other codes fail the call
  std::string why;      // or the error message of a failed call
  const uint8_t* grey = nullptr;
  int W = 0, H = 0, w = 0, h = 0;
};

// JPEG -> RGB interleaved (or the Y plane of a one-component file) in s.src on `st`.  B2M_EINVAL with *why when the
// file does not decode.  Errors of the CUDA runtime go to the calling thread's error (fail with a null context).
int ensure_hybrid(Nvjpeg& J) {
  if (!J.hybrid) {
    if (nvjpegCreateSimple(&J.hybrid) != NVJPEG_STATUS_SUCCESS)
      return fail(nullptr, B2M_ECUDA, "[image_io.cu] nvjpegCreateSimple failed");
    if (nvjpegJpegStateCreate(J.hybrid, &J.hybrid_state) != NVJPEG_STATUS_SUCCESS)
      return fail(nullptr, B2M_ECUDA, "[image_io.cu] nvjpegJpegStateCreate failed");
  }
  return B2M_OK;
}

int decode_jpeg(Nvjpeg& J, Slot& s, cudaStream_t st, const b2m_image_source& src, int* W, int* H, int* channels,
                DecodeCounts* cnt, std::string* why) {
  if (int rc = ensure_hybrid(J)) return rc;
  if (!J.hw_tried) {  // a GPU or driver without JPEG engines refuses the backend: the hybrid one does every file
    J.hw_tried = true;
    const bool ok = nvjpegCreateEx(NVJPEG_BACKEND_HARDWARE, nullptr, nullptr, 0, &J.hw) == NVJPEG_STATUS_SUCCESS &&
                    nvjpegJpegStateCreate(J.hw, &J.hw_rgb) == NVJPEG_STATUS_SUCCESS &&
                    nvjpegJpegStateCreate(J.hw, &J.hw_y) == NVJPEG_STATUS_SUCCESS &&
                    nvjpegDecodeBatchedInitialize(J.hw, J.hw_rgb, 1, 1, NVJPEG_OUTPUT_RGBI) == NVJPEG_STATUS_SUCCESS &&
                    nvjpegDecodeBatchedInitialize(J.hw, J.hw_y, 1, 1, NVJPEG_OUTPUT_Y) == NVJPEG_STATUS_SUCCESS &&
                    nvjpegJpegStreamCreate(J.hw, &J.hw_stream) == NVJPEG_STATUS_SUCCESS;
    if (!ok) J.drop_hw();
  }
  const unsigned char* data = src.data;
  const size_t size = static_cast<size_t>(src.size);
  int ncomp = 0, ws[NVJPEG_MAX_COMPONENT], hs[NVJPEG_MAX_COMPONENT];
  nvjpegChromaSubsampling_t sub;
  if (nvjpegGetImageInfo(J.hybrid, data, size, &ncomp, &sub, ws, hs) != NVJPEG_STATUS_SUCCESS || ws[0] <= 0 ||
      hs[0] <= 0) {
    *why = "not a JPEG stream nvJPEG can read";
    return B2M_EINVAL;
  }
  *W = ws[0];
  *H = hs[0];
  *channels = ncomp == 1 ? 1 : 3;
  const int64_t pitch = static_cast<int64_t>(*W) * *channels;
  B2M_CUDA_TRY(nullptr, s.src.ensure(static_cast<size_t>(pitch) * *H));
  nvjpegImage_t img;
  memset(&img, 0, sizeof(img));
  img.channel[0] = s.src;
  img.pitch[0] = static_cast<size_t>(pitch);
  int unsupported = 1;
  if (J.hw && nvjpegJpegStreamParse(J.hw, data, size, 0, 0, J.hw_stream) == NVJPEG_STATUS_SUCCESS &&
      nvjpegDecodeBatchedSupported(J.hw, J.hw_stream, &unsupported) == NVJPEG_STATUS_SUCCESS && unsupported == 0 &&
      nvjpegDecodeBatched(J.hw, ncomp == 1 ? J.hw_y : J.hw_rgb, &data, &size, &img, st) == NVJPEG_STATUS_SUCCESS) {
    cnt->hardware += 1;
  } else {
    const nvjpegStatus_t rc = nvjpegDecode(J.hybrid, J.hybrid_state, data, size,
                                           ncomp == 1 ? NVJPEG_OUTPUT_Y : NVJPEG_OUTPUT_RGBI, &img, st);
    if (rc != NVJPEG_STATUS_SUCCESS) {
      B2M_CUDA_TRY(nullptr, cudaStreamSynchronize(st));
      *why = "nvJPEG cannot decode it (status " + std::to_string(static_cast<int>(rc)) + ")";
      return B2M_EINVAL;
    }
  }
  cnt->bytes += size;
  return B2M_OK;
}

// Decodes `src` to grey in slot `s` on stream `st` and downscales it to fit max_image_size; returns once the result is
// on the device.  Errors of the CUDA runtime go to the calling thread's error (fail with a null context).
int decode_grey(Nvjpeg& J, Slot& s, cudaStream_t st, const b2m_image_source& src, int max_image_size, Decoded* d,
                DecodeCounts* cnt) {
  int channels = src.channels;
  int& W = d->W;
  int& H = d->H;
  if (src.kind == B2M_SOURCE_JPEG) {
    if (int rc = decode_jpeg(J, s, st, src, &W, &H, &channels, cnt, &d->why)) return rc;
  } else {
    W = src.width;
    H = src.height;
    const int64_t pitch = static_cast<int64_t>(W) * channels;
    B2M_CUDA_TRY(nullptr, s.src.ensure(static_cast<size_t>(pitch) * H));
    B2M_CUDA_TRY(nullptr, cudaMemcpy2DAsync(s.src, pitch, src.data, src.stride, pitch, H, cudaMemcpyHostToDevice, st));
  }
  cnt->images += 1;
  const int64_t n = static_cast<int64_t>(W) * H;
  B2M_CUDA_TRY(nullptr, s.grey.ensure(n));
  b2m_grey_kernel<<<blocks_for(n, 256), 256, 0, st>>>(s.src, static_cast<int64_t>(W) * channels, channels, W, H, s.grey);
  cnt->launches += 1;
  B2M_CUDA_TRY(nullptr, cudaGetLastError());
  int& w = d->w;
  int& h = d->h;
  target_size(W, H, max_image_size, &w, &h);
  d->grey = s.grey;
  if (w <= 0 || h <= 0) {
    d->why = "downscaled to an empty image";
    return B2M_EINVAL;
  }
  if (w != W || h != H) {
    B2M_CUDA_TRY(nullptr, s.small.ensure(static_cast<size_t>(w) * h));
    if (int rc = rescale_bilinear(nullptr, s.grey, W, H, 1, w, h, s.rs, s.small, st)) return rc;
    cnt->launches += 2;
    d->grey = s.small;
  }
  B2M_CUDA_TRY(nullptr, cudaStreamSynchronize(st));
  return B2M_OK;
}

// Runs decode_grey over the sources on its own thread and stream, up to kSlots - 1 images ahead of the consumer:
// while K6 runs image i on the library stream, images i + 1 ... are decoded, converted and downscaled (and the hybrid
// backend's host-side Huffman decoding runs on this thread).
class Decoder {
 public:
  Decoder(b2m_ctx* ctx, ImageIoState* S, const b2m_image_source* src, int n, int max_image_size)
      : S_(S), src_(src), n_(n), max_(max_image_size), out_(n) {
    thread_ = std::thread([this, dev = ctx->device] { run(dev); });
  }
  ~Decoder() {
    {
      std::lock_guard<std::mutex> lk(m_);
      abort_ = true;
    }
    cv_.notify_all();
    thread_.join();
  }
  // Waits for image i; its slot stays untouched until release(i).
  const Decoded& get(int i) {
    std::unique_lock<std::mutex> lk(m_);
    cv_.wait(lk, [&] { return done_ > i; });
    return out_[i];
  }
  void release(int i) {
    {
      std::lock_guard<std::mutex> lk(m_);
      released_ = i + 1;
    }
    cv_.notify_all();
  }
  DecodeCounts counts() {
    std::lock_guard<std::mutex> lk(m_);
    return cnt_;
  }

 private:
  void run(int dev) {
    cudaSetDevice(dev);
    for (int i = 0; i < n_; ++i) {
      {
        std::unique_lock<std::mutex> lk(m_);
        cv_.wait(lk, [&] { return abort_ || i - released_ < kSlots; });
        if (abort_) break;
      }
      Decoded d;
      DecodeCounts c;
      d.rc = S_->side ? decode_grey(S_->jpeg, S_->slot[i % kSlots], S_->side, src_[i], max_, &d, &c)
                      : fail(nullptr, B2M_ECUDA, "[image_io.cu] no side stream");
      if (d.rc != B2M_OK && d.why.empty()) d.why = g_noctx_err;
      {
        std::lock_guard<std::mutex> lk(m_);
        out_[i] = std::move(d);
        cnt_.launches += c.launches;
        cnt_.bytes += c.bytes;
        cnt_.images += c.images;
        cnt_.hardware += c.hardware;
        done_ = i + 1;
      }
      cv_.notify_all();
    }
  }
  ImageIoState* S_;
  const b2m_image_source* src_;
  int n_, max_;
  std::vector<Decoded> out_;
  DecodeCounts cnt_;
  std::mutex m_;
  std::condition_variable cv_;
  int done_ = 0, released_ = 0;
  bool abort_ = false;
  std::thread thread_;
};

int check_source(b2m_ctx* ctx, const b2m_image_source& s, int i) {
  const std::string at = "[image_io.cu] Check Failed: source " + std::to_string(i) + " ";
  if (!s.data) return fail(ctx, B2M_EINVAL, at + "has data");
  if (s.kind == B2M_SOURCE_JPEG) {
    if (s.size <= 0) return fail(ctx, B2M_EINVAL, at + "has size > 0");
  } else if (s.kind == B2M_SOURCE_PIXELS) {
    if (s.channels != 1 && s.channels != 3 && s.channels != 4) return fail(ctx, B2M_EINVAL, at + "has 1, 3 or 4 channels");
    if (s.width <= 0 || s.height <= 0 || s.stride < static_cast<int64_t>(s.width) * s.channels)
      return fail(ctx, B2M_EINVAL, at + "is non-empty with stride >= width x channels");
  } else {
    return fail(ctx, B2M_EINVAL, at + "kind is B2M_SOURCE_JPEG or B2M_SOURCE_PIXELS");
  }
  if (s.mask && (s.mask_width <= 0 || s.mask_height <= 0 || s.mask_stride < s.mask_width))
    return fail(ctx, B2M_EINVAL, at + "mask is non-empty with mask_stride >= mask_width");
  return B2M_OK;
}

}  // namespace

void image_io_release(b2m_ctx* ctx) {
  delete static_cast<ImageIoState*>(ctx->image_io_state);
  ctx->image_io_state = nullptr;
}

}  // namespace b2m

using namespace b2m;

namespace {

void add_counts(b2m_ctx* ctx, const DecodeCounts& c) {
  ctx->stats.kernel_launches += c.launches;
  ctx->stats.sift_decoded_bytes += c.bytes;
  ctx->stats.sift_decode_images += c.images;
  ctx->stats.sift_decode_hardware += c.hardware;
}

int prepare(b2m_ctx* ctx, ImageIoState** S) {
  cudaSetDevice(ctx->device);
  *S = state_of(ctx);
  if (!(*S)->side) B2M_CUDA_TRY(ctx, (*S)->side.create(cudaStreamNonBlocking));
  return B2M_OK;
}

}  // namespace

namespace b2m {
int image_io_decode_jpeg(b2m_ctx* ctx, const b2m_image_source& src, const uint8_t** pixels, int* W, int* H,
                         int* channels) {
  ImageIoState* S = nullptr;
  if (int rc = prepare(ctx, &S)) return rc;
  DecodeCounts c;
  std::string why;
  const int rc = decode_jpeg(S->jpeg, S->slot[0], S->side, src, W, H, channels, &c, &why);
  c.images += rc == B2M_OK;
  add_counts(ctx, c);
  if (rc == B2M_EINVAL && !why.empty()) return fail(ctx, rc, "[image_io.cu] source does not decode: " + why);
  if (rc) return fail(ctx, rc, g_noctx_err);
  B2M_CUDA_TRY(ctx, cudaStreamSynchronize(S->side));
  *pixels = S->slot[0].src;
  return B2M_OK;
}

int image_io_encode_jpeg(b2m_ctx* ctx, const uint8_t* rgb, int W, int H, cudaStream_t st, std::vector<uint8_t>* out) {
  ImageIoState* S = nullptr;
  if (int rc = prepare(ctx, &S)) return rc;
  Nvjpeg& J = S->jpeg;
  if (int rc = ensure_hybrid(J)) return fail(ctx, rc, g_noctx_err);
  auto check = [&](nvjpegStatus_t e, const char* what) {
    return e == NVJPEG_STATUS_SUCCESS ? B2M_OK
                                      : fail(ctx, B2M_ECUDA, std::string("[image_io.cu] ") + what + " failed (status " +
                                                                 std::to_string(static_cast<int>(e)) + ")");
  };
  if (!J.enc_state) {  // FreeImage's JPEG_QUALITYSUPERB with its default 4:2:0 subsampling
    nvjpegEncoderParams_t p = nullptr;
    nvjpegEncoderState_t e = nullptr;
    int rc = check(nvjpegEncoderParamsCreate(J.hybrid, &p, st), "nvjpegEncoderParamsCreate");
    if (!rc) rc = check(nvjpegEncoderParamsSetQuality(p, 100, st), "nvjpegEncoderParamsSetQuality");
    if (!rc) rc = check(nvjpegEncoderParamsSetSamplingFactors(p, NVJPEG_CSS_420, st), "nvjpegEncoderParamsSetSamplingFactors");
    if (!rc) rc = check(nvjpegEncoderStateCreate(J.hybrid, &e, st), "nvjpegEncoderStateCreate");
    if (rc) {  // nothing half-built is kept: the next call starts over
      if (e) nvjpegEncoderStateDestroy(e);
      if (p) nvjpegEncoderParamsDestroy(p);
      return rc;
    }
    J.enc_params = p;
    J.enc_state = e;
  }
  nvjpegImage_t img;
  memset(&img, 0, sizeof(img));
  img.channel[0] = const_cast<uint8_t*>(rgb);
  img.pitch[0] = static_cast<size_t>(W) * 3;
  if (int rc = check(nvjpegEncodeImage(J.hybrid, J.enc_state, J.enc_params, &img, NVJPEG_INPUT_RGBI, W, H, st),
                     "nvjpegEncodeImage"))
    return rc;
  size_t n = 0;
  if (int rc = check(nvjpegEncodeRetrieveBitstream(J.hybrid, J.enc_state, nullptr, &n, st), "nvjpegEncodeRetrieveBitstream"))
    return rc;
  B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
  out->resize(n);
  if (int rc = check(nvjpegEncodeRetrieveBitstream(J.hybrid, J.enc_state, out->data(), &n, st), "nvjpegEncodeRetrieveBitstream"))
    return rc;
  B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
  out->resize(n);
  return B2M_OK;
}
}  // namespace b2m

extern "C" {

int b2m_extract_features_sources(b2m_ctx* ctx, const b2m_image_source* sources, int32_t n, const b2m_extract_opts* opts,
                                 b2m_features** out) {
  if (!ctx) return B2M_EINVAL;
  if (!out || !opts || n < 0 || (n > 0 && !sources))
    return fail(ctx, B2M_EINVAL, "[image_io.cu] Check Failed: sources, options and out != NULL");
  *out = nullptr;
  for (int32_t i = 0; i < n; ++i)
    if (int rc = check_source(ctx, sources[i], i)) return rc;
  ImageIoState* S = nullptr;
  if (int rc = prepare(ctx, &S)) return rc;
  SiftPlan plan;
  if (int rc = sift_begin(ctx, opts, nullptr, nullptr, 0, &plan)) return rc;  // the option checks
  cudaStream_t st = ctx->stream;
  std::unique_ptr<b2m_features> F(new b2m_features());
  F->off.push_back(0);
  b2m_features one;
  std::vector<float> k6;
  std::vector<uint8_t> keep;
  int rc = B2M_OK;
  {
    Decoder dec(ctx, S, sources, n, opts->max_image_size);
    for (int32_t i = 0; i < n && rc == B2M_OK; ++i) {
      if (ctx->stop) {
        ctx->stop = 0;
        rc = fail(ctx, B2M_ESTOPPED, "[image_io.cu] stopped by b2m_request_stop");
        break;
      }
      const b2m_image_source& src = sources[i];
      const Decoded& d = dec.get(i);
      F->width.push_back(d.W);
      F->height.push_back(d.H);
      if (d.rc == B2M_EINVAL) {
        F->status.push_back(B2M_EINVAL);
        F->error.push_back(d.why);
        F->off.push_back(F->off.back());
        dec.release(i);
        continue;
      }
      if (d.rc) {
        rc = fail(ctx, d.rc, d.why);
        break;
      }
      int w = d.w, h = d.h;
      if ((rc = sift_begin(ctx, opts, &w, &h, 1, &plan))) break;
      one.off.assign(1, 0);
      one.kpts.clear();
      one.desc.clear();
      const float* d_k4 = nullptr;
      if ((rc = sift_extract(ctx, plan, d.grey, w, w, h, true, &one, &d_k4))) break;
      dec.release(i);  // sift_extract copied the image and synchronised the library stream
      const int ne = static_cast<int>(one.off.back());
      int kept = 0;
      if (ne) {
        rc = [&]() -> int {
          const bool rescale = w != d.W || h != d.H;
          const float sx = static_cast<float>(d.W) / static_cast<float>(w), sy = static_cast<float>(d.H) / static_cast<float>(h);
          if (src.mask) {
            B2M_CUDA_TRY(ctx, S->d_mask.ensure(static_cast<size_t>(src.mask_width) * src.mask_height));
            B2M_CUDA_TRY(ctx, cudaMemcpy2DAsync(S->d_mask, src.mask_width, src.mask, src.mask_stride, src.mask_width,
                                                src.mask_height, cudaMemcpyHostToDevice, st));
          }
          B2M_CUDA_TRY(ctx, S->d_k6.ensure(6 * static_cast<size_t>(ne)));
          B2M_CUDA_TRY(ctx, S->d_keep.ensure(ne));
          b2m_keypoint_finish_kernel<<<blocks_for(ne, 128), 128, 0, st>>>(
              d_k4, ne, rescale ? 1 : 0, sx, sy, src.mask ? static_cast<const uint8_t*>(S->d_mask) : nullptr,
              src.mask_width, src.mask_height, src.mask_width, S->d_k6, S->d_keep);
          ctx->stats.kernel_launches += 1;
          B2M_CUDA_TRY(ctx, cudaGetLastError());
          k6.resize(6 * static_cast<size_t>(ne));
          keep.resize(ne);
          B2M_CUDA_TRY(ctx, cudaMemcpyAsync(k6.data(), S->d_k6, sizeof(float) * k6.size(), cudaMemcpyDeviceToHost, st));
          B2M_CUDA_TRY(ctx, cudaMemcpyAsync(keep.data(), S->d_keep, ne, cudaMemcpyDeviceToHost, st));
          B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
          return B2M_OK;
        }();
        if (rc) break;
        for (int k = 0; k < ne; ++k) {
          if (!keep[k]) continue;
          F->kpts.insert(F->kpts.end(), k6.begin() + 6 * k, k6.begin() + 6 * (k + 1));
          F->desc.insert(F->desc.end(), one.desc.begin() + 128 * static_cast<size_t>(k),
                         one.desc.begin() + 128 * static_cast<size_t>(k + 1));
          ++kept;
        }
      }
      F->status.push_back(B2M_OK);
      F->error.emplace_back();
      F->off.push_back(F->off.back() + kept);
    }
    add_counts(ctx, dec.counts());
  }  // the decoder thread is joined here, before any return
  if (rc) return rc;
  *out = F.release();
  return B2M_OK;
}

int b2m_source_features_get(const b2m_features* f, int32_t image, b2m_source_view* out) {
  if (!f || !out || image < 0 || image >= static_cast<int64_t>(f->status.size())) return B2M_EINVAL;
  const int64_t a = f->off[image], b = f->off[image + 1];
  out->struct_size = sizeof(*out);
  out->status = f->status[image];
  out->error = f->error[image].c_str();
  out->width = f->width[image];
  out->height = f->height[image];
  out->n = b - a;
  out->keypoints = f->kpts.data() + 6 * a;
  out->descriptors = f->desc.data() + 128 * a;
  return B2M_OK;
}

int b2m_debug_decode_grey(b2m_ctx* ctx, const b2m_image_source* source, int32_t max_image_size, uint8_t* grey,
                          int32_t* width, int32_t* height) {
  if (!ctx) return B2M_EINVAL;
  if (!source || !width || !height || max_image_size <= 0)
    return fail(ctx, B2M_EINVAL, "[image_io.cu] Check Failed: source, width, height != NULL and max_image_size > 0");
  if (int rc = check_source(ctx, *source, 0)) return rc;
  ImageIoState* S = nullptr;
  if (int rc = prepare(ctx, &S)) return rc;
  Decoded d;
  DecodeCounts c;
  const int rc = decode_grey(S->jpeg, S->slot[0], S->side, *source, max_image_size, &d, &c);
  add_counts(ctx, c);
  if (rc == B2M_EINVAL && !d.why.empty()) return fail(ctx, rc, "[image_io.cu] source does not decode: " + d.why);
  if (rc) return fail(ctx, rc, g_noctx_err);
  *width = d.w;
  *height = d.h;
  if (grey) B2M_CUDA_TRY(ctx, cudaMemcpy(grey, d.grey, static_cast<size_t>(d.w) * d.h, cudaMemcpyDeviceToHost));
  return B2M_OK;
}

}  // extern "C"
