// undistort_camera.h -- UndistortCamera (U:image/undistortion.cc, recalled; DESIGN.md section 4 K10) on the host: the
// PINHOLE camera of an undistorted image.  Shared by b2m_undistort_camera / b2m_undistort_images (undistort.cu) and the
// CPU stand-in of the library the host tests run against, so that both compute the same cameras.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>

#include "../../include/b200match.h"
#include "camera_models.h"

namespace b2m {
namespace undistort {

inline const char* opts_problem(const b2m_undistort_opts& o) {
  if (o.struct_size != sizeof(b2m_undistort_opts)) return "b2m_undistort_opts.struct_size == sizeof(b2m_undistort_opts)";
  if (!(o.blank_pixels >= 0.0)) return "blank_pixels >= 0";
  if (!(o.blank_pixels <= 1.0)) return "blank_pixels <= 1";
  if (!(o.min_scale > 0.0)) return "min_scale > 0";
  if (!(o.min_scale <= o.max_scale)) return "min_scale <= max_scale";
  if (o.max_image_size == 0) return "max_image_size != 0";
  if (!(o.roi_min_x >= 0.0)) return "roi_min_x >= 0";
  if (!(o.roi_min_y >= 0.0)) return "roi_min_y >= 0";
  if (!(o.roi_max_x <= 1.0)) return "roi_max_x <= 1";
  if (!(o.roi_max_y <= 1.0)) return "roi_max_y <= 1";
  if (!(o.roi_min_x < o.roi_max_x)) return "roi_min_x < roi_max_x";
  if (!(o.roi_min_y < o.roi_max_y)) return "roi_min_y < roi_max_y";
  return nullptr;
}

// PINHOLE parameters p = (fx, fy, cx, cy)
inline void pinhole_img_from_cam(const double* p, double u, double v, double* x, double* y) {
  cam::img_from_cam(cam::kPinhole, p, u, v, x, y);
}

// Camera::Rescale(scale) of a PINHOLE camera: the new size is round(scale * size); focal lengths and principal point
// follow the per-axis ratio that rounding gives.
inline void rescale_pinhole(double scale, b2m_camera* c) {
  const double sx = std::round(scale * c->width) / static_cast<double>(c->width);
  const double sy = std::round(scale * c->height) / static_cast<double>(c->height);
  c->width = static_cast<int32_t>(std::round(scale * c->width));
  c->height = static_cast<int32_t>(std::round(scale * c->height));
  c->params[2] = sx * c->params[2];
  c->params[3] = sy * c->params[3];
  c->params[0] = sx * c->params[0];
  c->params[1] = sy * c->params[1];
}

// UndistortCamera (U:image/undistortion.cc), options already checked.
inline void undistort_camera(const b2m_undistort_opts& o, const b2m_camera& d, b2m_camera* out) {
  b2m_camera u;
  std::memset(&u, 0, sizeof(u));
  u.struct_size = sizeof(u);
  u.model = cam::kPinhole;
  u.width = d.width;
  u.height = d.height;
  double fx, fy, cx, cy;
  int extra;
  cam::intrinsics(d.model, d.params, &fx, &fy, &cx, &cy, &extra);
  u.params[0] = fx;
  u.params[1] = fy;
  u.params[2] = cx;
  u.params[3] = cy;
  int64_t roi_min_x = 0, roi_min_y = 0, roi_max_x = d.width, roi_max_y = d.height;
  const bool roi = o.roi_min_x > 0.0 || o.roi_min_y > 0.0 || o.roi_max_x < 1.0 || o.roi_max_y < 1.0;
  if (roi) {
    roi_min_x = static_cast<int64_t>(std::round(o.roi_min_x * static_cast<double>(u.width)));
    roi_min_y = static_cast<int64_t>(std::round(o.roi_min_y * static_cast<double>(u.height)));
    roi_max_x = static_cast<int64_t>(std::round(o.roi_max_x * static_cast<double>(u.width)));
    roi_max_y = static_cast<int64_t>(std::round(o.roi_max_y * static_cast<double>(u.height)));
    roi_min_x = std::min<int64_t>(roi_min_x, u.width - 1);
    roi_min_y = std::min<int64_t>(roi_min_y, u.height - 1);
    roi_max_x = std::max<int64_t>(roi_max_x, roi_min_x + 1);
    roi_max_y = std::max<int64_t>(roi_max_y, roi_min_y + 1);
    u.width = static_cast<int32_t>(roi_max_x - roi_min_x);
    u.height = static_cast<int32_t>(roi_max_y - roi_min_y);
    u.params[2] -= static_cast<double>(roi_min_x);
    u.params[3] -= static_cast<double>(roi_min_y);
  }
  if (roi || cam::has_distortion(d.model)) {
    const double kMax = 1.79769313486231570815e+308;
    double left_min_x = kMax, left_max_x = -kMax, right_min_x = kMax, right_max_x = -kMax;
    double a, b, px, py;
    for (int64_t y = roi_min_y; y < roi_max_y; ++y) {
      cam::cam_from_img(d.model, d.params, 0.5, y + 0.5, &a, &b);
      pinhole_img_from_cam(u.params, a, b, &px, &py);
      left_min_x = std::min(left_min_x, px);
      left_max_x = std::max(left_max_x, px);
      cam::cam_from_img(d.model, d.params, d.width - 0.5, y + 0.5, &a, &b);
      pinhole_img_from_cam(u.params, a, b, &px, &py);
      right_min_x = std::min(right_min_x, px);
      right_max_x = std::max(right_max_x, px);
    }
    double top_min_y = kMax, top_max_y = -kMax, bottom_min_y = kMax, bottom_max_y = -kMax;
    for (int64_t x = roi_min_x; x < roi_max_x; ++x) {
      cam::cam_from_img(d.model, d.params, x + 0.5, 0.5, &a, &b);
      pinhole_img_from_cam(u.params, a, b, &px, &py);
      top_min_y = std::min(top_min_y, py);
      top_max_y = std::max(top_max_y, py);
      cam::cam_from_img(d.model, d.params, x + 0.5, d.height - 0.5, &a, &b);
      pinhole_img_from_cam(u.params, a, b, &px, &py);
      bottom_min_y = std::min(bottom_min_y, py);
      bottom_max_y = std::max(bottom_max_y, py);
    }
    const double ucx = u.params[2], ucy = u.params[3];
    // scale such that the undistorted image holds every pixel of the distorted one ...
    const double min_scale_x = std::min(ucx / (ucx - left_min_x), (u.width - 0.5 - ucx) / (right_max_x - ucx));
    const double min_scale_y = std::min(ucy / (ucy - top_min_y), (u.height - 0.5 - ucy) / (bottom_max_y - ucy));
    // ... or such that it has no blank pixel
    const double max_scale_x = std::max(ucx / (ucx - left_max_x), (u.width - 0.5 - ucx) / (right_min_x - ucx));
    const double max_scale_y = std::max(ucy / (ucy - top_max_y), (u.height - 0.5 - ucy) / (bottom_min_y - ucy));
    double scale_x = 1.0 / (min_scale_x * o.blank_pixels + max_scale_x * (1.0 - o.blank_pixels));
    double scale_y = 1.0 / (min_scale_y * o.blank_pixels + max_scale_y * (1.0 - o.blank_pixels));
    scale_x = std::min(std::max(scale_x, o.min_scale), o.max_scale);
    scale_y = std::min(std::max(scale_y, o.min_scale), o.max_scale);
    const int64_t w0 = u.width, h0 = u.height;
    u.width = static_cast<int32_t>(static_cast<int64_t>(std::max(1.0, scale_x * u.width)));
    u.height = static_cast<int32_t>(static_cast<int64_t>(std::max(1.0, scale_y * u.height)));
    u.params[2] = u.params[2] * static_cast<double>(u.width) / static_cast<double>(w0);
    u.params[3] = u.params[3] * static_cast<double>(u.height) / static_cast<double>(h0);
  }
  if (o.max_image_size > 0) {
    const double s = std::min(o.max_image_size / static_cast<double>(u.width), o.max_image_size / static_cast<double>(u.height));
    if (s < 1.0) rescale_pinhole(s, &u);
  }
  *out = u;
}

}  // namespace undistort
}  // namespace b2m
