// undistort.cu -- K10: what COLMAP's image undistorter does to one image (U:image/undistortion.cc UndistortCamera,
// UndistortImage; U:image/warp.cc WarpImageBetweenCameras; U:sensor/bitmap.cc InterpolateBilinear, Rescale; recalled,
// DESIGN.md section 4 K10), on the device:
//   camera   UndistortCamera on the host (b2m_undistort_camera): a PINHOLE camera whose size and principal point follow
//            the ROI, the border scan of the distorted image and max_image_size
//   decode   JPEG with K7's nvJPEG path; host pixels (grey / RGB / RGBA) uploaded as they are
//   warp     at the source resolution, one thread per target pixel: pinhole CamFromImg of the pixel centre, the
//            distorted camera's ImgFromCam (camera_models.h), then InterpolateBilinear in fp64 on FreeImage's bottom-up
//            rows, rounded to fp32 (BitmapColor<float>) and cast to uint8; RGB out
//   rescale  FreeImage's bilinear Rescale to the undistorted size, per channel (K7's kernels)
//   encode   nvJPEG's encoder (quality 100, 4:2:0), or the RGB pixels back to the host
// The file is compiled without FMA contraction: the coordinate map and the interpolation are rounded per operation, as
// the x86 code upstream runs rounds them and as oracle/undistort.py restates them.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "internal.h"
#include "undistort_camera.h"

struct b2m_undistorted {
  std::vector<int32_t> status, width, height;
  std::vector<std::string> error;
  std::vector<b2m_camera> camera;
  std::vector<std::vector<uint8_t>> data;  // JPEG bytes or width x height x 3 RGB
};

namespace b2m {
namespace {

// The two cameras of one warp: the distorted source and the pinhole target rescaled to the source size.
struct WarpCams {
  int model;
  double p[cam::kMaxParams];
  double q[4];  // fx, fy, cx, cy
};

__global__ void b2m_undistort_warp_kernel(const uint8_t* __restrict__ src, int W, int H, int channels, WarpCams c,
                                          uint8_t* __restrict__ dst) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<int64_t>(W) * H) return;
  const int y = static_cast<int>(i / W), x = static_cast<int>(i % W);
  double u, v, sx, sy;
  cam::cam_from_img(cam::kPinhole, c.q, x + 0.5, y + 0.5, &u, &v);
  cam::img_from_cam(c.model, c.p, u, v, &sx, &sy);
  // Bitmap::InterpolateBilinear(sx - 0.5, sy - 0.5): FreeImage's scan line y0 is image row H - 1 - y0
  const double bx = sx - 0.5, inv_y = static_cast<double>(H - 1) - (sy - 0.5);
  const double fx0 = floor(bx), fy0 = floor(inv_y);
  uint8_t* o = dst + 3 * i;
  if (!(fx0 >= 0.0 && fx0 + 1.0 < W && fy0 >= 0.0 && fy0 + 1.0 < H)) {  // NaN lands here too
    o[0] = o[1] = o[2] = 0;
    return;
  }
  const int x0 = static_cast<int>(fx0), y0 = static_cast<int>(fy0);
  const double dx = bx - x0, dy = inv_y - y0, dx_1 = 1.0 - dx, dy_1 = 1.0 - dy;
  const int64_t stride = static_cast<int64_t>(W) * channels;
  const uint8_t* line0 = src + (H - 1 - y0) * stride;
  const uint8_t* line1 = line0 - stride;
  for (int k = 0; k < 3; ++k) {
    const int ch = channels == 1 ? 0 : k;
    const int64_t a = static_cast<int64_t>(x0) * channels + ch, b = a + channels;
    const double v0 = dx_1 * line0[a] + dx * line0[b];
    const double v1 = dx_1 * line1[a] + dx * line1[b];
    const float f = static_cast<float>(dy_1 * v0 + dy * v1);
    o[k] = static_cast<uint8_t>(fminf(255.0f, fmaxf(0.0f, roundf(f))));
  }
}

struct UndistortState {
  DeviceArray<uint8_t> src, warp, out;
  RescaleBufs rs;
};

UndistortState* state_of(b2m_ctx* ctx) {
  if (!ctx->undistort_state) ctx->undistort_state = new UndistortState();
  return static_cast<UndistortState*>(ctx->undistort_state);
}

inline unsigned blocks_for(int64_t n, int t) { return static_cast<unsigned>((n + t - 1) / t); }

int check_item(b2m_ctx* ctx, const b2m_undistort_item& it, int i) {
  const std::string at = "[undistort.cu] Check Failed: item " + std::to_string(i) + " ";
  if (it.struct_size != sizeof(b2m_undistort_item)) return fail(ctx, B2M_EINVAL, at + "struct_size == sizeof(b2m_undistort_item)");
  if (it.output != B2M_UNDISTORT_JPEG && it.output != B2M_UNDISTORT_PIXELS)
    return fail(ctx, B2M_EINVAL, at + "output is B2M_UNDISTORT_JPEG or B2M_UNDISTORT_PIXELS");
  if (const char* why = camera_problem(it.camera)) return fail(ctx, B2M_EINVAL, at + "camera: " + why);
  if (it.camera.width <= 0 || it.camera.height <= 0) return fail(ctx, B2M_EINVAL, at + "camera has a size");
  const b2m_image_source& s = it.source;
  if (!s.data) return fail(ctx, B2M_EINVAL, at + "source has data");
  if (s.kind == B2M_SOURCE_JPEG) {
    if (s.size <= 0) return fail(ctx, B2M_EINVAL, at + "source has size > 0");
  } else if (s.kind == B2M_SOURCE_PIXELS) {
    if (s.channels != 1 && s.channels != 3 && s.channels != 4)
      return fail(ctx, B2M_EINVAL, at + "source has 1, 3 or 4 channels");
    if (s.width <= 0 || s.height <= 0 || s.stride < static_cast<int64_t>(s.width) * s.channels)
      return fail(ctx, B2M_EINVAL, at + "source is non-empty with stride >= width x channels");
  } else {
    return fail(ctx, B2M_EINVAL, at + "source kind is B2M_SOURCE_JPEG or B2M_SOURCE_PIXELS");
  }
  return B2M_OK;
}

// One image: decode, warp, rescale, then the JPEG file or the RGB pixels in *data.  B2M_EINVAL with *why for an image
// that does not decode or whose size is not its camera's (the call goes on); other codes fail the call.
int undistort_one(b2m_ctx* ctx, UndistortState* S, const b2m_undistort_item& it, const b2m_camera& und, bool jpeg,
                  std::vector<uint8_t>* data, std::string* why) {
  cudaStream_t st = ctx->stream;
  const b2m_image_source& s = it.source;
  const uint8_t* src = nullptr;
  int W = 0, H = 0, channels = 0;
  if (s.kind == B2M_SOURCE_JPEG) {
    const int rc = image_io_decode_jpeg(ctx, s, &src, &W, &H, &channels);
    if (rc == B2M_EINVAL) {
      *why = ctx->err;
      return rc;
    }
    if (rc) return rc;
  } else {
    W = s.width;
    H = s.height;
    channels = s.channels;
    const int64_t pitch = static_cast<int64_t>(W) * channels;
    B2M_CUDA_TRY(ctx, S->src.ensure(static_cast<size_t>(pitch) * H));
    B2M_CUDA_TRY(ctx, cudaMemcpy2DAsync(S->src, pitch, s.data, s.stride, pitch, H, cudaMemcpyHostToDevice, st));
    src = S->src;
  }
  if (W != it.camera.width || H != it.camera.height) {
    *why = "the image is " + std::to_string(W) + " x " + std::to_string(H) + ", its camera " +
           std::to_string(it.camera.width) + " x " + std::to_string(it.camera.height);
    return B2M_EINVAL;
  }
  WarpCams c;
  c.model = it.camera.model;
  std::copy(it.camera.params, it.camera.params + cam::kMaxParams, c.p);
  std::copy(und.params, und.params + 4, c.q);
  if (und.width != W || und.height != H) {  // Camera::Rescale(W, H) of the target
    const double sx = static_cast<double>(W) / static_cast<double>(und.width);
    const double sy = static_cast<double>(H) / static_cast<double>(und.height);
    c.q[2] = sx * c.q[2];
    c.q[3] = sy * c.q[3];
    c.q[0] = sx * c.q[0];
    c.q[1] = sy * c.q[1];
  }
  const int64_t n = static_cast<int64_t>(W) * H;
  B2M_CUDA_TRY(ctx, S->warp.ensure(3 * static_cast<size_t>(n)));
  b2m_undistort_warp_kernel<<<blocks_for(n, 256), 256, 0, st>>>(src, W, H, channels, c, S->warp);
  ctx->stats.kernel_launches += 1;
  B2M_CUDA_TRY(ctx, cudaGetLastError());
  const uint8_t* out = S->warp;
  if (und.width != W || und.height != H) {
    B2M_CUDA_TRY(ctx, S->out.ensure(3 * static_cast<size_t>(und.width) * und.height));
    if (int rc = rescale_bilinear(ctx, S->warp, W, H, 3, und.width, und.height, S->rs, S->out, st)) return rc;
    ctx->stats.kernel_launches += 2;
    out = S->out;
  }
  if (jpeg) {
    if (int rc = image_io_encode_jpeg(ctx, out, und.width, und.height, st, data)) return rc;
  } else {
    data->resize(3 * static_cast<size_t>(und.width) * und.height);
    B2M_CUDA_TRY(ctx, cudaMemcpyAsync(data->data(), out, data->size(), cudaMemcpyDeviceToHost, st));
    B2M_CUDA_TRY(ctx, cudaStreamSynchronize(st));
  }
  return B2M_OK;
}

}  // namespace

void undistort_release(b2m_ctx* ctx) {
  delete static_cast<UndistortState*>(ctx->undistort_state);
  ctx->undistort_state = nullptr;
}

}  // namespace b2m

using namespace b2m;
using namespace b2m::undistort;

extern "C" {

void b2m_undistort_opts_default(b2m_undistort_opts* o) {
  if (!o) return;
  std::memset(o, 0, sizeof(*o));
  o->struct_size = sizeof(*o);
  o->max_image_size = -1;
  o->blank_pixels = 0.0;
  o->min_scale = 0.2;
  o->max_scale = 2.0;
  o->roi_min_x = o->roi_min_y = 0.0;
  o->roi_max_x = o->roi_max_y = 1.0;
}

int b2m_undistort_camera(b2m_ctx* ctx, const b2m_undistort_opts* opts, const b2m_camera* camera, b2m_camera* out) {
  if (!opts || !camera || !out) return fail(ctx, B2M_EINVAL, "[undistort.cu] Check Failed: options, camera and out != NULL");
  if (const char* why = opts_problem(*opts)) return fail(ctx, B2M_EINVAL, std::string("[undistort.cu] Check Failed: ") + why);
  if (const char* why = camera_problem(*camera)) return fail(ctx, B2M_EINVAL, std::string("[undistort.cu] ") + why);
  if (camera->width <= 0 || camera->height <= 0)
    return fail(ctx, B2M_EINVAL, "[undistort.cu] Check Failed: camera width > 0 and height > 0");
  undistort_camera(*opts, *camera, out);
  return B2M_OK;
}

int b2m_undistort_images(b2m_ctx* ctx, const b2m_undistort_item* items, int32_t n, const b2m_undistort_opts* opts,
                         b2m_undistorted** out) {
  if (!ctx) return B2M_EINVAL;
  if (!out || !opts || n < 0 || (n > 0 && !items))
    return fail(ctx, B2M_EINVAL, "[undistort.cu] Check Failed: items, options and out != NULL");
  *out = nullptr;
  if (const char* why = opts_problem(*opts)) return fail(ctx, B2M_EINVAL, std::string("[undistort.cu] Check Failed: ") + why);
  for (int32_t i = 0; i < n; ++i)
    if (int rc = check_item(ctx, items[i], i)) return rc;
  std::unique_ptr<b2m_undistorted> R(new (std::nothrow) b2m_undistorted());
  if (!R) return fail(ctx, B2M_ENOMEM, "[undistort.cu] out of host memory");
  std::vector<b2m_camera> und(n);
  // The images run one after the other through the same buffers: the call needs the largest image's worth.
  double need = 0.0;
  for (int32_t i = 0; i < n; ++i) {
    undistort_camera(*opts, items[i].camera, &und[i]);
    const double src = static_cast<double>(items[i].camera.width) * items[i].camera.height;
    const double dst = static_cast<double>(und[i].width) * und[i].height;
    need = std::max(need, src * 4 + src * 3 + 2 * 3 * std::max(src, dst) + 3 * dst);
  }
  B2M_CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  {
    size_t free_b = 0, total_b = 0;
    B2M_CUDA_TRY(ctx, cudaMemGetInfo(&free_b, &total_b));
    if (need > static_cast<double>(free_b)) {
      char b[256];
      snprintf(b, sizeof(b), "[undistort.cu] the largest image of the call needs %.1f MB of device memory, %.1f MB are "
               "available", need / 1e6, free_b / 1e6);
      return fail(ctx, B2M_ENOMEM, b);
    }
  }
  UndistortState* S = state_of(ctx);
  for (int32_t i = 0; i < n; ++i) {
    if (ctx->stop) {
      ctx->stop = 0;
      return fail(ctx, B2M_ESTOPPED, "[undistort.cu] stopped by b2m_request_stop");
    }
    std::vector<uint8_t> data;
    std::string why;
    const int rc = undistort_one(ctx, S, items[i], und[i], items[i].output == B2M_UNDISTORT_JPEG, &data, &why);
    if (rc != B2M_OK && rc != B2M_EINVAL) return rc;
    R->status.push_back(rc);
    R->error.push_back(why);
    R->width.push_back(und[i].width);
    R->height.push_back(und[i].height);
    R->camera.push_back(und[i]);
    if (rc == B2M_OK) {
      ctx->stats.undistort_images += 1;
      ctx->stats.undistort_pixels += static_cast<uint64_t>(und[i].width) * und[i].height;
      if (items[i].output == B2M_UNDISTORT_JPEG) ctx->stats.undistort_encoded_bytes += data.size();
    }
    R->data.push_back(std::move(data));
  }
  *out = R.release();
  return B2M_OK;
}

int b2m_undistorted_get(const b2m_undistorted* r, int32_t k, b2m_undistorted_view* out) {
  if (!r || !out || k < 0 || k >= static_cast<int64_t>(r->status.size())) return B2M_EINVAL;
  out->struct_size = sizeof(*out);
  out->status = r->status[k];
  out->error = r->error[k].c_str();
  out->width = r->width[k];
  out->height = r->height[k];
  out->camera = r->camera[k];
  out->size = static_cast<int64_t>(r->data[k].size());
  out->data = r->data[k].data();
  return B2M_OK;
}

void b2m_undistorted_free(b2m_undistorted* r) { delete r; }

int b2m_debug_undistort_pixels(b2m_ctx* ctx, const b2m_undistort_item* item, const b2m_undistort_opts* opts, uint8_t* rgb,
                               int32_t* width, int32_t* height) {
  if (!ctx) return B2M_EINVAL;
  if (!item || !width || !height)
    return fail(ctx, B2M_EINVAL, "[undistort.cu] Check Failed: item, width and height != NULL");
  b2m_undistort_item one = *item;
  one.output = B2M_UNDISTORT_PIXELS;
  b2m_undistorted* r = nullptr;
  if (int rc = b2m_undistort_images(ctx, &one, 1, opts, &r)) return rc;
  std::unique_ptr<b2m_undistorted> guard(r);
  if (r->status[0] != B2M_OK) return fail(ctx, r->status[0], "[undistort.cu] source does not undistort: " + r->error[0]);
  *width = r->width[0];
  *height = r->height[0];
  if (rgb) std::memcpy(rgb, r->data[0].data(), r->data[0].size());
  return B2M_OK;
}

}  // extern "C"
