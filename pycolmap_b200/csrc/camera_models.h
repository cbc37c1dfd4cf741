// camera_models.h -- CamFromImg for COLMAP's camera models (SURVEY.md row V9), host + device.
//
// Follows the published definitions of U:sensor/models.h (COLMAP 3.9.1), reached in the reference
// through Camera::CamFromImg / CamFromImgThreshold / MeanFocalLength (R:scene/camera.h:20-213,
// R:estimators/essential_matrix.h:31-46): a model is (focal parameters, principal point, a distortion
// function d(u, v) on normalised coordinates); ImgFromCam is  x = f1 * (u + du) + c1,  y = f2 * (v + dv) + c2
// and CamFromImg inverts it -- closed form for the pinhole models, Newton iterations on
// g(u, v) = (u, v) + d(u, v) - (u0, v0) with a central-difference Jacobian for the others (upstream's
// IterativeUndistortion: at most 100 iterations, stop when |step|^2 < 1e-10, relative step 1e-6).
// Model ids and parameter orders are COLMAP's; all eleven models of 3.9.1 are implemented.  Two have their own
// structure: FOV (Devernay-Faugeras) distorts multiplicatively, r_d = atan(2 r tan(w/2)) / w, and is inverted in
// closed form; THIN_PRISM_FISHEYE applies its polynomial + thin-prism terms to the equidistant fisheye
// coordinates theta * (u, v) / r and maps back with tan(theta) / theta after the iterative undistortion.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define B2M_CAM_HD __host__ __device__ __forceinline__
#else
#define B2M_CAM_HD inline
#endif

namespace b2m {
namespace cam {

enum ModelId {
  kSimplePinhole = 0,       // f, cx, cy
  kPinhole = 1,             // fx, fy, cx, cy
  kSimpleRadial = 2,        // f, cx, cy, k
  kRadial = 3,              // f, cx, cy, k1, k2
  kOpenCV = 4,              // fx, fy, cx, cy, k1, k2, p1, p2
  kOpenCVFisheye = 5,       // fx, fy, cx, cy, k1, k2, k3, k4
  kFullOpenCV = 6,          // fx, fy, cx, cy, k1, k2, p1, p2, k3, k4, k5, k6
  kFOV = 7,                 // fx, fy, cx, cy, omega
  kSimpleRadialFisheye = 8, // f, cx, cy, k
  kRadialFisheye = 9,       // f, cx, cy, k1, k2
  kThinPrismFisheye = 10    // fx, fy, cx, cy, k1, k2, p1, p2, k3, k4, sx1, sy1
};

constexpr int kMaxParams = 12;

// number of parameters of a supported model, -1 for an unknown / unsupported id
B2M_CAM_HD int num_params(int model) {
  switch (model) {
    case kSimplePinhole: return 3;
    case kPinhole: return 4;
    case kSimpleRadial: return 4;
    case kRadial: return 5;
    case kOpenCV: return 8;
    case kOpenCVFisheye: return 8;
    case kFullOpenCV: return 12;
    case kFOV: return 5;
    case kSimpleRadialFisheye: return 4;
    case kRadialFisheye: return 5;
    case kThinPrismFisheye: return 12;
    default: return -1;
  }
}

B2M_CAM_HD bool single_focal(int model) {
  return model == kSimplePinhole || model == kSimpleRadial || model == kRadial || model == kSimpleRadialFisheye ||
         model == kRadialFisheye;
}
B2M_CAM_HD bool has_distortion(int model) { return model != kSimplePinhole && model != kPinhole; }

// fx, fy, cx, cy and the index of the first distortion parameter.  The functions that take a scalar type T are
// templates so that the pose refinement can run them on forward-mode dual numbers (abs_pose.cu); with T = double
// they are the plain functions.
template <class T>
B2M_CAM_HD void intrinsics(int model, const T* p, T* fx, T* fy, T* cx, T* cy, int* extra) {
  if (single_focal(model)) {
    *fx = *fy = p[0]; *cx = p[1]; *cy = p[2]; *extra = 3;
  } else {
    *fx = p[0]; *fy = p[1]; *cx = p[2]; *cy = p[3]; *extra = 4;
  }
}

// MeanFocalLength: mean over the model's focal-length parameters
B2M_CAM_HD double mean_focal_length(int model, const double* p) { return single_focal(model) ? p[0] : 0.5 * (p[0] + p[1]); }

// d(u, v) of the model; k = pointer to the first distortion parameter
template <class T>
B2M_CAM_HD void distortion(int model, const T* k, T u, T v, T* du, T* dv) {
  const T u2 = u * u, v2 = v * v, r2 = u2 + v2;
  switch (model) {
    case kSimpleRadial: {
      const T radial = k[0] * r2;
      *du = u * radial; *dv = v * radial;
      return;
    }
    case kRadial: {
      const T radial = k[0] * r2 + k[1] * r2 * r2;
      *du = u * radial; *dv = v * radial;
      return;
    }
    case kOpenCV: {
      const T uv = u * v, radial = k[0] * r2 + k[1] * r2 * r2;
      *du = u * radial + 2.0 * k[2] * uv + k[3] * (r2 + 2.0 * u2);
      *dv = v * radial + 2.0 * k[3] * uv + k[2] * (r2 + 2.0 * v2);
      return;
    }
    case kFullOpenCV: {  // k1, k2, p1, p2, k3, k4, k5, k6
      const T uv = u * v, r4 = r2 * r2, r6 = r4 * r2;
      const T radial = (1.0 + k[0] * r2 + k[1] * r4 + k[4] * r6) / (1.0 + k[5] * r2 + k[6] * r4 + k[7] * r6);
      *du = u * radial + 2.0 * k[2] * uv + k[3] * (r2 + 2.0 * u2) - u;
      *dv = v * radial + 2.0 * k[3] * uv + k[2] * (r2 + 2.0 * v2) - v;
      return;
    }
    case kOpenCVFisheye:
    case kSimpleRadialFisheye:
    case kRadialFisheye: {
      const T r = sqrt(r2);
      if (r > 2.220446049250313e-16) {  // std::numeric_limits<double>::epsilon()
        const T theta = atan(r), t2 = theta * theta, t4 = t2 * t2;
        T poly;
        if (model == kOpenCVFisheye) poly = 1.0 + k[0] * t2 + k[1] * t4 + k[2] * t4 * t2 + k[3] * t4 * t4;
        else if (model == kRadialFisheye) poly = 1.0 + k[0] * t2 + k[1] * t4;
        else poly = 1.0 + k[0] * t2;
        const T thetad = theta * poly;
        *du = u * thetad / r - u;
        *dv = v * thetad / r - v;
      } else {
        *du = T(0.0); *dv = T(0.0);
      }
      return;
    }
    case kThinPrismFisheye: {  // on the equidistant fisheye coordinates: k1, k2, p1, p2, k3, k4, sx1, sy1
      const T uv = u * v, r4 = r2 * r2, r6 = r4 * r2, r8 = r6 * r2;
      const T radial = k[0] * r2 + k[1] * r4 + k[4] * r6 + k[5] * r8;
      *du = u * radial + 2.0 * k[2] * uv + k[3] * (r2 + 2.0 * u2) + k[6] * r2;
      *dv = v * radial + 2.0 * k[3] * uv + k[2] * (r2 + 2.0 * v2) + k[7] * r2;
      return;
    }
    default:
      *du = T(0.0); *dv = T(0.0);
  }
}

// FOV model: distorted = factor * undistorted with factor = atan(2 r tan(w/2)) / (r w) (-> 2 tan(w/2) / w as r -> 0,
// -> 1 as w -> 0), and its closed-form inverse factor = tan(r_d w) / (2 r_d tan(w/2)).
template <class T>
B2M_CAM_HD T fov_distort_factor(T omega, T r2) {
  const T t = tan(0.5 * omega);
  if (fabs(omega) < 1e-8) return T(1.0);
  const T x = 2.0 * sqrt(r2) * t;
  if (fabs(x) < 1e-6) return (2.0 * t / omega) * (1.0 - x * x / 3.0);
  return atan(x) / (sqrt(r2) * omega);
}
B2M_CAM_HD double fov_undistort_factor(double omega, double r2) {
  const double t = tan(0.5 * omega);
  if (fabs(omega) < 1e-8) return 1.0;
  const double y = sqrt(r2) * omega;
  if (fabs(y) < 1e-6) return (omega / (2.0 * t)) * (1.0 + y * y / 3.0);
  return tan(y) / (2.0 * sqrt(r2) * t);
}

// (u, v) -> the point whose distorted image is (u, v): Newton with a central-difference Jacobian
B2M_CAM_HD void iterative_undistortion(int model, const double* k, double* u, double* v) {
  const double kEps = 2.220446049250313e-16, kRelStep = 1e-6, kMaxStepNorm = 1e-10;
  const double u0 = *u, v0 = *v;
  double x = u0, y = v0;
  for (int it = 0; it < 100; ++it) {
    const double hx = fmax(kEps, fabs(kRelStep * x)), hy = fmax(kEps, fabs(kRelStep * y));
    double dx, dy, ax, ay, bx, by, cx, cy, ex, ey;
    distortion(model, k, x, y, &dx, &dy);
    distortion(model, k, x - hx, y, &ax, &ay);
    distortion(model, k, x + hx, y, &bx, &by);
    distortion(model, k, x, y - hy, &cx, &cy);
    distortion(model, k, x, y + hy, &ex, &ey);
    const double j00 = 1.0 + (bx - ax) / (2.0 * hx), j01 = (ex - cx) / (2.0 * hy);
    const double j10 = (by - ay) / (2.0 * hx), j11 = 1.0 + (ey - cy) / (2.0 * hy);
    const double gx = x + dx - u0, gy = y + dy - v0;
    const double det = j00 * j11 - j01 * j10;
    const double sx = (j11 * gx - j01 * gy) / det, sy = (j00 * gy - j10 * gx) / det;
    x -= sx;
    y -= sy;
    if (sx * sx + sy * sy < kMaxStepNorm) break;
  }
  *u = x;
  *v = y;
}

// Camera::CamFromImg: pixel -> normalised camera coordinates
B2M_CAM_HD void cam_from_img(int model, const double* p, double x, double y, double* u, double* v) {
  double fx, fy, cx, cy;
  int extra;
  intrinsics(model, p, &fx, &fy, &cx, &cy, &extra);
  *u = (x - cx) / fx;
  *v = (y - cy) / fy;
  if (model == kFOV) {
    const double f = fov_undistort_factor(p[extra], *u * *u + *v * *v);
    *u *= f;
    *v *= f;
  } else if (has_distortion(model)) {
    iterative_undistortion(model, p + extra, u, v);
    if (model == kThinPrismFisheye) {  // fisheye coordinates (theta direction) -> normalised plane
      const double theta = sqrt(*u * *u + *v * *v), tc = theta * cos(theta);
      if (tc > 2.220446049250313e-16) {
        const double sc = sin(theta) / tc;
        *u *= sc;
        *v *= sc;
      }
    }
  }
}

// Camera::ImgFromCam on normalised coordinates (used by the tests for round trips and to build scenes)
template <class T>
B2M_CAM_HD void img_from_cam(int model, const T* p, T u, T v, T* x, T* y) {
  T fx, fy, cx, cy, du = T(0.0), dv = T(0.0);
  int extra;
  intrinsics(model, p, &fx, &fy, &cx, &cy, &extra);
  if (model == kFOV) {
    const T f = fov_distort_factor(p[extra], u * u + v * v);
    u *= f;
    v *= f;
  } else if (model == kThinPrismFisheye) {
    const T r = sqrt(u * u + v * v);
    if (r > 2.220446049250313e-16) {
      const T theta = atan(r);
      u = theta * u / r;
      v = theta * v / r;
    }
    distortion(model, p + extra, u, v, &du, &dv);
  } else if (has_distortion(model)) {
    distortion(model, p + extra, u, v, &du, &dv);
  }
  *x = fx * (u + du) + cx;
  *y = fy * (v + dv) + cy;
}

}  // namespace cam
}  // namespace b2m
