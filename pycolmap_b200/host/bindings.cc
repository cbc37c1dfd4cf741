// bindings.cc -- pybind11 module `pycolmap_b200._core`: the C++ host side of the drop-in boundary.
//
// Mirrors, name for name and keyword for keyword, the part of the reference's Python surface that
// reaches the matching / verification hot path:
//   match_exhaustive, match_sequential, verify_matches        R:pipeline/match_features.h:22-68, 219-260
//   SiftMatchingOptions, Exhaustive/SequentialMatchingOptions R:pipeline/match_features.h:71-152
//   TwoViewGeometryOptions, TwoViewGeometry(Configuration)    R:estimators/two_view_geometry.h:41-93
//   estimate_(calibrated_)two_view_geometry, squared_sampson_error   R:estimators/two_view_geometry.h:95-175
//   essential / fundamental / homography_matrix_estimation    R:estimators/essential_matrix.h:19-103,
//                                                             fundamental_matrix.h:17-50, homography_matrix.h:17-48
//   RANSACOptions                                             R:optim/bindings.h:7-27
//   absolute_pose_estimation, pose_refinement, AbsolutePose*Options  R:pycolmap/estimators/absolute_pose.h:18-166
//   estimate_triangulation, PointData, EstimateTriangulationOptions  R:pycolmap/estimators/triangulation.h:17-77
//   Device, has_cuda                                          R:utils.h:9-31, R:main.cc:98-106
//   Database (open/close/counters/read_two_view_geometry/image_pair_to_pair_id)  R:scene/database.h:10-47
// Everything below the option structs goes through the C ABI of include/b200match.h; there is no CPU path.
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <dlfcn.h>

#include <array>
#include <cfloat>
#include <atomic>
#include <chrono>
#include <cstring>
#include <filesystem>
#include <fstream>
#include <functional>
#include <future>
#include <thread>

#include "../csrc/camera_models.h"
#include "controllers.h"
#include "dataclass.h"
#include "database.h"
#include "image_reader.h"

namespace py = pybind11;
using namespace b2mh;
using namespace pybind11::literals;

namespace {

enum class Device { AUTO = -1, CPU = 0, CUDA = 1 };  // R:utils.h:9

enum class TwoViewGeometryConfiguration {  // R:estimators/two_view_geometry.h:67-80
  UNDEFINED = 0, DEGENERATE, CALIBRATED, UNCALIBRATED, PLANAR, PANORAMIC, PLANAR_OR_PANORAMIC, WATERMARK, MULTIPLE
};

using ArrD = py::array_t<double, py::array::c_style | py::array::forcecast>;
using ArrU8 = py::array_t<uint8_t, py::array::c_style | py::array::forcecast>;
using ArrF32 = py::array_t<float, py::array::c_style | py::array::forcecast>;
using ArrU32 = py::array_t<uint32_t, py::array::c_style | py::array::forcecast>;
using ArrI32 = py::array_t<int32_t, py::array::c_style | py::array::forcecast>;

py::array_t<double> MatToNumpy(const double* m) {
  py::array_t<double> a(std::vector<py::ssize_t>{3, 3});
  memcpy(a.mutable_data(), m, 72);
  return a;
}

py::array_t<uint32_t> MatchesToNumpy(const uint32_t* m, int64_t n) {
  py::array_t<uint32_t> a(std::vector<py::ssize_t>{static_cast<py::ssize_t>(n), 2});
  if (n > 0) memcpy(a.mutable_data(), m, static_cast<size_t>(n) * 8);
  return a;
}

std::string FsPath(const py::object& p) { return py::module_::import("os").attr("fspath")(p).cast<std::string>(); }

void CheckPoints(const ArrD& p, const char* name) {
  if (p.ndim() != 2 || p.shape(1) != 2)
    throw std::invalid_argument(std::string("[bindings.cc] Check Failed: ") + name + " is an N x 2 array");
}

// A camera is a dict {model, width, height, params, has_prior_focal_length} or any object with those
// attributes (a pycolmap.Camera: `model` may be an enum with a .name, R:scene/camera.h:20-213).
b2m_camera CameraFromPython(const py::object& cam) {
  auto get = [&](const char* key, py::object def) -> py::object {
    if (py::isinstance<py::dict>(cam)) {
      const py::dict d = cam;
      return d.contains(key) ? py::object(d[key]) : def;
    }
    return py::hasattr(cam, key) ? py::object(cam.attr(key)) : def;
  };
  py::object model = get("model", py::none());
  if (model.is_none()) model = get("model_id", py::int_(0));
  if (py::hasattr(model, "name")) model = model.attr("name");
  CameraRow row;
  if (py::isinstance<py::str>(model)) {
    const std::string name = model.cast<std::string>();
    static const char* kNames[] = {"SIMPLE_PINHOLE", "PINHOLE", "SIMPLE_RADIAL", "RADIAL", "OPENCV", "OPENCV_FISHEYE",
                                   "FULL_OPENCV", "FOV", "SIMPLE_RADIAL_FISHEYE", "RADIAL_FISHEYE", "THIN_PRISM_FISHEYE"};
    row.model = -1;
    for (int i = 0; i < 11; ++i)
      if (name == kNames[i]) row.model = i;
    if (row.model < 0) throw std::invalid_argument("[bindings.cc] unknown camera model " + name);
  } else {
    row.model = model.cast<int>();
  }
  row.width = get("width", py::int_(0)).cast<int64_t>();
  row.height = get("height", py::int_(0)).cast<int64_t>();
  row.params = get("params", py::list()).cast<std::vector<double>>();
  row.has_prior_focal_length = py::bool_(get("has_prior_focal_length", py::bool_(false)));
  return ToAbi(row);
}

py::dict CameraToDict(const CameraRow& c) {
  return py::dict("model"_a = c.model, "width"_a = c.width, "height"_a = c.height, "params"_a = c.params,
                  "has_prior_focal_length"_a = c.has_prior_focal_length ? 1 : 0);
}

// ---- TwoViewGeometry (R:estimators/two_view_geometry.h:82-93) --------------------------------------
// Minimal stand-ins for pycolmap.Rotation3d / Rigid3d (R:geometry bindings): x_cam2 = rotation * x_cam1 + translation.
struct Rotation3d {
  std::array<double, 4> wxyz{1.0, 0.0, 0.0, 0.0};
};
struct Rigid3d {
  Rotation3d rotation;
  std::array<double, 3> translation{0.0, 0.0, 0.0};
};

// Rigid3d::ToMatrix(): [R | t], 3 x 4 row-major
std::array<double, 12> RigidToMatrix(const Rigid3d& g) {
  const Mat3 R = QuatToRotation(g.rotation.wxyz);
  std::array<double, 12> p;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) p[i * 4 + j] = R[i * 3 + j];
    p[i * 4 + 3] = g.translation[i];
  }
  return p;
}

struct TwoViewGeometry {
  TwoViewGeometryConfiguration config = TwoViewGeometryConfiguration::UNDEFINED;
  Mat3 E{}, F{}, H{};
  std::vector<uint32_t> inlier_matches;
  double tri_angle = 0.0;
  std::array<double, 4> qvec{1.0, 0.0, 0.0, 0.0};  // cam2_from_cam1 (w, x, y, z); identity unless a pose was recovered
  std::array<double, 3> tvec{0.0, 0.0, 0.0};
  int nE = 0, nF = 0, nH = 0;  // diagnostic inlier counts of the three LO-RANSAC runs

  void Invert() {
    InvertPose(&qvec, &tvec);
    F = Transposed(F);
    E = Transposed(E);
    Mat3 inv;
    bool zero = true;
    for (double v : H) zero = zero && v == 0.0;
    if (!zero && Invert3x3(H, &inv)) H = inv;
    for (size_t i = 0; i + 1 < inlier_matches.size(); i += 2) std::swap(inlier_matches[i], inlier_matches[i + 1]);
  }
};

// ---- PyWait (R:helpers.h:335-347): run `fn` on a worker thread with the GIL released; the calling
// thread polls for signals so that Ctrl-C stops the GPU work between batches and surfaces as
// KeyboardInterrupt.
template <typename Fn>
void RunInterruptible(Fn&& fn) {
  std::exception_ptr error;
  PyObject *et = nullptr, *ev = nullptr, *tb = nullptr;
  bool interrupted = false;
  {
    py::gil_scoped_release release;
    std::atomic<bool> done{false};
    std::thread worker([&] {
      try {
        fn();
      } catch (...) {
        error = std::current_exception();
      }
      done = true;
    });
    while (!done) {
      std::this_thread::sleep_for(std::chrono::milliseconds(20));
      if (interrupted) continue;
      py::gil_scoped_acquire acquire;
      if (PyErr_CheckSignals() != 0) {
        PyErr_Fetch(&et, &ev, &tb);
        interrupted = true;
        Engine::RequestStopAll();
      }
    }
    worker.join();
  }
  if (interrupted) {
    PyErr_Restore(et, ev, tb);
    throw py::error_already_set();
  }
  if (error) std::rethrow_exception(error);
}

std::vector<int> ResolveDevices(Device device, const SiftMatchingOptions& sift) {
  // IsGPU / VerifyGPUParams (R:utils.h:11-31): `auto` is the GPU; this build has nothing else.
  if (device == Device::CPU)
    throw std::invalid_argument("[bindings.cc] pycolmap_b200 has no CPU path: use Device.auto or Device.cuda");
  return ParseGpuIndices(sift.gpu_index);
}

// ---- estimators --------------------------------------------------------------------------------------
// `get_ctx` is called only after every argument check passed (checks come before any GPU work).
TwoViewGeometry EstimateTvg(const std::function<b2m_ctx*()>& get_ctx, const py::object& camera1, const ArrD& points1, const py::object& camera2,
                            const ArrD& points2, const py::object& matches, const TwoViewGeometryOptions& options) {
  CheckPoints(points1, "points1");
  CheckPoints(points2, "points2");
  const b2m_camera c1 = CameraFromPython(camera1), c2 = CameraFromPython(camera2);
  const b2m_tvg_opts opts = ToAbi(options);
  ArrU32 m;
  const uint32_t* mptr = nullptr;
  int64_t n_m = points1.shape(0);
  if (!matches.is_none()) {
    m = ArrU32::ensure(matches);
    if (!m || m.ndim() != 2 || m.shape(1) != 2)
      throw std::invalid_argument("[bindings.cc] Check Failed: matches is an N x 2 uint32 array");
    mptr = m.data();
    n_m = m.shape(0);
  } else if (points1.shape(0) != points2.shape(0)) {
    throw std::invalid_argument("[two_view_geometry.h:137] Check Failed: points1.size() == points2.size()");
  }
  b2m_tvg_result r;
  memset(&r, 0, sizeof(r));
  r.struct_size = sizeof(r);
  std::vector<uint32_t> inl(static_cast<size_t>(std::max<int64_t>(1, n_m)) * 2);
  b2m_ctx* ctx = get_ctx();
  int rc;
  {
    py::gil_scoped_release release;
    rc = b2m_estimate_two_view_geometry(ctx, &c1, points1.data(), points1.shape(0), &c2, points2.data(),
                                        points2.shape(0), mptr, n_m, &opts, &r, inl.data());
  }
  ThrowOnError(ctx, rc);
  TwoViewGeometry g;
  g.config = static_cast<TwoViewGeometryConfiguration>(r.config);
  std::copy(r.E, r.E + 9, g.E.begin());
  std::copy(r.F, r.F + 9, g.F.begin());
  std::copy(r.H, r.H + 9, g.H.begin());
  inl.resize(static_cast<size_t>(r.n_inliers) * 2);
  g.inlier_matches = std::move(inl);
  g.nE = r.nE; g.nF = r.nF; g.nH = r.nH;
  std::copy(r.qvec, r.qvec + 4, g.qvec.begin());
  std::copy(r.tvec, r.tvec + 3, g.tvec.begin());
  g.tri_angle = r.tri_angle;
  return g;
}

// Single-model LO-RANSAC; returns None on failure like the reference (R:estimators/fundamental_matrix.h:31-33).
py::object RansacModel(b2m_ctx* ctx, int kind, const char* key, const ArrD& p1, const ArrD& p2,
                       const RANSACOptions& options) {
  const b2m_ransac_opts o = ToAbi(options);
  const int64_t m = p1.shape(0);
  double model[9] = {0};
  std::vector<uint8_t> mask(static_cast<size_t>(std::max<int64_t>(1, m)));
  int64_t n_inl = 0;
  int32_t ok = 0;
  int rc;
  {
    py::gil_scoped_release release;
    rc = b2m_ransac_model(ctx, kind, p1.data(), p2.data(), m, &o, model, mask.data(), &n_inl, &ok);
  }
  ThrowOnError(ctx, rc);
  if (!ok) return py::none();
  py::array_t<bool> inliers(static_cast<py::ssize_t>(m));
  bool* ip = inliers.mutable_data();
  for (int64_t i = 0; i < m; ++i) ip[i] = mask[i] != 0;
  py::dict out;
  out[key] = MatToNumpy(model);
  out["num_inliers"] = n_inl;
  out["inliers"] = inliers;
  return out;
}

void CheckSameLength(const ArrD& p1, const ArrD& p2, const char* where) {
  CheckPoints(p1, "points1");
  CheckPoints(p2, "points2");
  if (p1.shape(0) != p2.shape(0))
    throw std::invalid_argument(std::string("[") + where + "] Check Failed: points1.size() == points2.size()");
}

// ---- low-level context (what tests and benchmarks drive directly) ------------------------------------
struct CoreResults {
  b2m_results* r = nullptr;
  ~CoreResults() { Free(); }
  void Free() {
    if (r) b2m_results_free(r);
    r = nullptr;
  }
  b2m_pair_view View(int64_t k) const {
    if (!r) throw std::runtime_error("[bindings.cc] results were freed");
    b2m_pair_view v;
    memset(&v, 0, sizeof(v));
    v.struct_size = sizeof(v);
    if (b2m_results_get(r, k, &v) != B2M_OK) throw py::index_error(std::to_string(k));
    return v;
  }
};

struct CoreContext {
  b2m_ctx* ctx = nullptr;
  CoreContext(int device, uint64_t seed, int pair_batch) {
    b2m_device_cfg cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.struct_size = sizeof(cfg);
    cfg.device = device;
    cfg.seed = seed;
    cfg.pair_batch = pair_batch;
    ThrowOnError(nullptr, b2m_create(&cfg, &ctx));
  }
  ~CoreContext() { Close(); }
  void Close() {
    if (ctx) b2m_destroy(ctx);
    ctx = nullptr;
  }
  b2m_ctx* Handle() const {
    if (!ctx) throw std::runtime_error("[bindings.cc] context is closed");
    return ctx;
  }
};

std::vector<b2m_camera> CamerasFromPython(const py::object& cams) {
  std::vector<b2m_camera> out;
  for (const auto& c : cams) out.push_back(CameraFromPython(py::reinterpret_borrow<py::object>(c)));
  return out;
}


// ---- absolute pose (R:pycolmap/estimators/absolute_pose.h:18-166) ------------------------------------------
void CheckAbsPoints(const ArrD& p2, const ArrD& p3) {
  if (p2.ndim() != 2 || p2.shape(1) != 2)
    throw std::invalid_argument("[bindings.cc] Check Failed: points2D is an N x 2 array");
  if (p3.ndim() != 2 || p3.shape(1) != 3)
    throw std::invalid_argument("[bindings.cc] Check Failed: points3D is an N x 3 array");
  if (p2.shape(0) != p3.shape(0))  // THROW_CHECK_EQ(points2D.size(), points3D.size()), R:absolute_pose.h:26
    throw std::invalid_argument("[absolute_pose.h:26] Check Failed: points2D.size() == points3D.size() (" +
                                std::to_string(p2.shape(0)) + " vs. " + std::to_string(p3.shape(0)) + ")");
}

b2m_abs_pose_problem AbsProblem(const b2m_camera& cam, const ArrD& p2, const ArrD& p3) {
  b2m_abs_pose_problem q;
  memset(&q, 0, sizeof(q));
  q.struct_size = sizeof(q);
  q.camera = cam;
  q.points2D = p2.data();
  q.points3D = p3.data();
  q.n = p2.shape(0);
  return q;
}

// The reference takes Camera& and lets the estimator / the solver change its parameters: write them back into the
// caller's object (the "params" key of a dict, else the `params` attribute).
void WriteCameraParams(const py::object& camera, const b2m_abs_pose_result& r, int model) {
  std::vector<double> p(r.params, r.params + b2m::cam::num_params(model));
  if (py::isinstance<py::dict>(camera)) {
    py::dict d = camera;
    d["params"] = p;
  } else {
    py::setattr(camera, "params", py::array_t<double>(static_cast<py::ssize_t>(p.size()), p.data()));
  }
}

py::object PoseToPython(const py::module_& m, const double* q, const double* t) {
  const std::array<double, 4> xyzw{q[1], q[2], q[3], q[0]};
  const std::array<double, 3> tr{t[0], t[1], t[2]};
  return m.attr("Rigid3d")(m.attr("Rotation3d")(xyzw), tr);
}

// The absolute pose entry points (C ABI version 4) are bound at run time, like SQLite (sqlite_dyn.cc) and NCCL
// (csrc/comm.cu): the host module references no version-4 symbol at link time, so it still loads against a
// libb200match.so that predates them (the matching and verification surface keeps working) and reports their
// absence when an absolute pose function is called.  There is no other path to these computations.
struct AbsPoseApi {
  decltype(&b2m_estimate_absolute_pose_batch) estimate = nullptr;
  decltype(&b2m_refine_absolute_pose_batch) refine = nullptr;
};
const AbsPoseApi& AbsPose() {
  static const AbsPoseApi api = [] {
    AbsPoseApi a;
    Dl_info info;   // the libb200match.so this module is linked against, found through one of its symbols
    if (dladdr(reinterpret_cast<void*>(&b2m_abi_version), &info) && info.dli_fname)
      if (void* h = dlopen(info.dli_fname, RTLD_NOW | RTLD_NOLOAD)) {
        a.estimate = reinterpret_cast<decltype(a.estimate)>(dlsym(h, "b2m_estimate_absolute_pose_batch"));
        a.refine = reinterpret_cast<decltype(a.refine)>(dlsym(h, "b2m_refine_absolute_pose_batch"));
      }
    return a;
  }();
  if (!api.estimate || !api.refine)
    throw std::runtime_error("[bindings.cc] libb200match.so does not export the absolute pose entry points "
                             "(C ABI version 4): rebuild it");
  return api;
}

py::array_t<bool> MaskToNumpy(const std::vector<uint8_t>& mask, int64_t n) {
  py::array_t<bool> a(static_cast<py::ssize_t>(n));
  bool* p = a.mutable_data();
  for (int64_t i = 0; i < n; ++i) p[i] = mask[i] != 0;
  return a;
}

// Batched estimation + refinement; results in r, masks in masks.
void EstimateAbsolutePoses(b2m_ctx* ctx, const std::vector<b2m_abs_pose_problem>& q, const AbsolutePoseEstimationOptions& eo,
                           const AbsolutePoseRefinementOptions& ro, bool cov, std::vector<b2m_abs_pose_result>* r,
                           std::vector<std::vector<uint8_t>>* masks) {
  const b2m_abs_pose_opts e = ToAbi(eo);
  const b2m_pose_refine_opts f = ToAbi(ro);
  const AbsPoseApi& api = AbsPose();
  const size_t n = q.size();
  r->assign(n, b2m_abs_pose_result{});
  masks->resize(n);
  std::vector<uint8_t*> mp(n);
  for (size_t k = 0; k < n; ++k) {
    (*masks)[k].assign(static_cast<size_t>(std::max<int64_t>(q[k].n, 1)), 0);
    mp[k] = (*masks)[k].data();
  }
  int rc;
  {
    py::gil_scoped_release release;
    rc = api.estimate(ctx, q.data(), static_cast<int64_t>(n), &e, &f, cov ? 1 : 0, r->data(), mp.data());
  }
  ThrowOnError(ctx, rc);
}

py::object AbsResultToPython(const py::module_& m, const b2m_abs_pose_result& r, const std::vector<uint8_t>& mask, int64_t n,
                             bool cov) {
  if (!r.success) return py::none();
  py::dict d;
  d["cam_from_world"] = PoseToPython(m, r.qvec, r.tvec);
  d["num_inliers"] = r.num_inliers;
  d["inliers"] = MaskToNumpy(mask, n);
  if (cov) {
    py::array_t<double> c(std::vector<py::ssize_t>{6, 6});
    memcpy(c.mutable_data(), r.covariance, sizeof(double) * 36);
    d["covariance"] = c;
  }
  return d;
}

// ---- triangulation (R:pycolmap/estimators/triangulation.h:17-77) -------------------------------------------
// PointData (R:pycolmap/estimators/triangulation.h): the pixel and the camera-normalised observation; only
// point_normalized enters the angular residual.
struct PointData {
  std::array<double, 2> point{0.0, 0.0}, point_normalized{0.0, 0.0};
};

// Bound at run time like the absolute pose entry points: the host references no C ABI version 5 symbol at link time.
using TriEstimateFn = decltype(&b2m_estimate_triangulation_batch);
TriEstimateFn TriEstimate() {
  static const TriEstimateFn fn = []() -> TriEstimateFn {
    Dl_info info;
    if (dladdr(reinterpret_cast<void*>(&b2m_abi_version), &info) && info.dli_fname)
      if (void* h = dlopen(info.dli_fname, RTLD_NOW | RTLD_NOLOAD))
        return reinterpret_cast<TriEstimateFn>(dlsym(h, "b2m_estimate_triangulation_batch"));
    return nullptr;
  }();
  if (!fn)
    throw std::runtime_error("[bindings.cc] libb200match.so does not export the triangulation entry point "
                             "(C ABI version 5): rebuild it");
  return fn;
}

// EstimateTriangulationOptions::Check and RANSACOptions::Check (U:estimators/triangulation.h, U:optim/ransac.h); upstream
// CHECKs abort the process, here they raise ValueError before any GPU work.
void CheckTriOptions(const EstimateTriangulationOptions& o) {
  auto fail = [](const char* what) { throw std::invalid_argument(std::string("[triangulation.h] Check Failed: ") + what); };
  if (!(o.min_tri_angle >= 0.0)) fail("min_tri_angle >= 0");
  if (!(o.ransac.max_error > 0.0)) fail("ransac.max_error > 0");
  if (!(o.ransac.min_inlier_ratio >= 0.0 && o.ransac.min_inlier_ratio <= 1.0)) fail("0 <= ransac.min_inlier_ratio <= 1");
  if (!(o.ransac.confidence >= 0.0 && o.ransac.confidence <= 1.0)) fail("0 <= ransac.confidence <= 1");
  if (!(o.ransac.min_num_trials <= o.ransac.max_num_trials)) fail("ransac.min_num_trials <= ransac.max_num_trials");
}

// cam_from_world of an entry of `images`: an object with a `cam_from_world` attribute (pycolmap's Image; a method
// returning it is called) or a Rigid3d itself.
std::array<double, 12> ImagePoseMatrix(const py::handle& image) {
  py::object g = py::reinterpret_borrow<py::object>(image);
  if (!py::isinstance<Rigid3d>(g) && py::hasattr(g, "cam_from_world")) {
    g = g.attr("cam_from_world");
    if (!py::isinstance<Rigid3d>(g) && PyCallable_Check(g.ptr())) g = g();
  }
  if (!py::isinstance<Rigid3d>(g))
    throw std::invalid_argument("[bindings.cc] Check Failed: each image is a Rigid3d or has a cam_from_world Rigid3d");
  return RigidToMatrix(g.cast<Rigid3d>());
}

struct TriBatchOut {
  std::vector<double> xyz;
  std::vector<int32_t> num_inliers;
  std::vector<uint8_t> success, mask;
};

// One call of the batch entry point; offsets [T + 1], points [M x 2], image indices [M], cams [I x 12].
TriBatchOut EstimateTriangulationsAbi(b2m_ctx* ctx, const std::vector<int64_t>& off, const double* pts, const int32_t* img,
                                      int32_t n_images, const double* cams, const EstimateTriangulationOptions& options) {
  const b2m_tri_opts o = ToAbi(options);
  const TriEstimateFn fn = TriEstimate();
  const int64_t T = static_cast<int64_t>(off.size()) - 1, M = off.back();
  TriBatchOut r;
  r.xyz.assign(3 * static_cast<size_t>(std::max<int64_t>(T, 1)), 0.0);
  r.num_inliers.assign(static_cast<size_t>(std::max<int64_t>(T, 1)), 0);
  r.success.assign(static_cast<size_t>(std::max<int64_t>(T, 1)), 0);
  r.mask.assign(static_cast<size_t>(std::max<int64_t>(M, 1)), 0);
  int rc;
  {
    py::gil_scoped_release release;
    rc = fn(ctx, T, off.data(), pts, img, n_images, cams, &o, r.xyz.data(), r.num_inliers.data(), r.success.data(),
            r.mask.data());
  }
  ThrowOnError(ctx, rc);
  return r;
}

// estimate_triangulations: (M, 2) points, (T,) lengths, (M,) image indices, (I, 3, 4) cams_from_world.
py::dict EstimateTriangulationsPy(const std::function<b2m_ctx*()>& get_ctx, const py::object& points_normalized,
                                  const py::object& track_lengths, const py::object& image_idxs,
                                  const py::object& cams_from_world, const EstimateTriangulationOptions& options) {
  CheckTriOptions(options);
  const ArrD pts = ArrD::ensure(points_normalized);
  if (!pts || pts.ndim() != 2 || pts.shape(1) != 2)
    throw std::invalid_argument("[bindings.cc] Check Failed: points_normalized is an M x 2 float64 array");
  using ArrI64 = py::array_t<int64_t, py::array::c_style | py::array::forcecast>;
  const ArrI64 len = ArrI64::ensure(track_lengths), idx = ArrI64::ensure(image_idxs);
  if (!len || len.ndim() != 1) throw std::invalid_argument("[bindings.cc] Check Failed: track_lengths is a 1-D integer array");
  if (!idx || idx.ndim() != 1) throw std::invalid_argument("[bindings.cc] Check Failed: image_idxs is a 1-D integer array");
  const ArrD cams = ArrD::ensure(cams_from_world);
  if (!cams || cams.ndim() != 3 || cams.shape(1) != 3 || cams.shape(2) != 4)
    throw std::invalid_argument("[bindings.cc] Check Failed: cams_from_world is an I x 3 x 4 float64 array");
  const int64_t T = len.shape(0), M = pts.shape(0), I = cams.shape(0);
  if (I > INT32_MAX) throw std::invalid_argument("[bindings.cc] Check Failed: fewer than 2^31 images");
  std::vector<int64_t> off(static_cast<size_t>(T) + 1, 0);
  for (int64_t k = 0; k < T; ++k) {
    if (len.data()[k] < 2)  // THROW_CHECK_GE(point_data.size(), 2)
      throw std::invalid_argument("[triangulation.cc] Check Failed: track_lengths[" + std::to_string(k) + "] >= 2");
    off[k + 1] = off[k] + len.data()[k];
  }
  if (off[T] != M)
    throw std::invalid_argument("[bindings.cc] Check Failed: sum(track_lengths) == len(points_normalized) (" +
                                std::to_string(off[T]) + " vs. " + std::to_string(M) + ")");
  if (idx.shape(0) != M)
    throw std::invalid_argument("[bindings.cc] Check Failed: len(image_idxs) == len(points_normalized)");
  std::vector<int32_t> img(static_cast<size_t>(std::max<int64_t>(M, 1)));
  for (int64_t i = 0; i < M; ++i) {
    const int64_t v = idx.data()[i];
    if (v < 0 || v >= I)
      throw std::invalid_argument("[bindings.cc] Check Failed: 0 <= image_idxs[" + std::to_string(i) + "] < " + std::to_string(I));
    img[i] = static_cast<int32_t>(v);
  }
  const TriBatchOut r = EstimateTriangulationsAbi(get_ctx(), off, pts.data(), img.data(), static_cast<int32_t>(I), cams.data(),
                                                  options);
  py::array_t<double> xyz(std::vector<py::ssize_t>{static_cast<py::ssize_t>(T), 3});
  py::array_t<bool> success(static_cast<py::ssize_t>(T));
  py::array_t<int64_t> num_inliers(static_cast<py::ssize_t>(T));
  for (int64_t k = 0; k < T; ++k) {
    for (int a = 0; a < 3; ++a) xyz.mutable_data()[3 * k + a] = r.xyz[3 * k + a];
    success.mutable_data()[k] = r.success[k] != 0;
    num_inliers.mutable_data()[k] = r.num_inliers[k];
  }
  py::dict d;
  d["xyz"] = xyz;
  d["success"] = success;
  d["num_inliers"] = num_inliers;
  d["inliers"] = MaskToNumpy(r.mask, M);
  return d;
}

// ---- SIFT extraction (R:pycolmap/feature/sift.h, R:pipeline/extract_features.h:63-139) ------------------------------
// Bound at run time like the triangulation entry point: the host references no C ABI version 6 symbol at link time.
template <typename F>
F SiftSymbol(const char* name) {
  static void* handle = []() -> void* {
    Dl_info info;
    if (dladdr(reinterpret_cast<void*>(&b2m_abi_version), &info) && info.dli_fname)
      return dlopen(info.dli_fname, RTLD_NOW | RTLD_NOLOAD);
    return nullptr;
  }();
  void* p = handle ? dlsym(handle, name) : nullptr;
  if (!p)
    throw std::runtime_error(std::string("[bindings.cc] libb200match.so does not export ") + name +
                             " (C ABI version 6): rebuild it");
  return reinterpret_cast<F>(p);
}

// SiftExtractionOptions::Check (U:feature/sift.cc); the options without a path here are refused, not ignored.
void CheckSiftOptions(const SiftExtractionOptions& o) {
  auto fail = [](const std::string& what) { throw std::invalid_argument("[sift.cc] Check Failed: " + what); };
  if (!(o.max_image_size > 0)) fail("max_image_size > 0");
  if (!(o.max_num_features > 0)) fail("max_num_features > 0");
  if (!(o.octave_resolution > 0)) fail("octave_resolution > 0");
  if (!(o.peak_threshold > 0.0)) fail("peak_threshold > 0");
  if (!(o.edge_threshold > 0.0)) fail("edge_threshold > 0");
  if (!(o.max_num_orientations > 0)) fail("max_num_orientations > 0");
  if (o.domain_size_pooling) {
    if (!(o.dsp_min_scale > 0)) fail("dsp_min_scale > 0");
    if (!(o.dsp_max_scale >= o.dsp_min_scale)) fail("dsp_max_scale >= dsp_min_scale");
    if (!(o.dsp_num_scales > 0)) fail("dsp_num_scales > 0");
  }
  auto unsupported = [](const std::string& what) {
    throw std::invalid_argument("[bindings.cc] Check Failed: " + what + " is not supported (no GPU path)");
  };
  if (!(o.num_octaves > 0)) unsupported("num_octaves <= 0");
  if (!(o.first_octave >= -3 && o.first_octave <= 16)) unsupported("first_octave outside [-3, 16]");
  if (o.estimate_affine_shape) unsupported("estimate_affine_shape");
  if (o.domain_size_pooling) unsupported("domain_size_pooling");
  if (o.darkness_adaptivity) unsupported("darkness_adaptivity");
}

// IsGPU / VerifyGPUParams (R:utils.h:11-31) for one extractor: Device.cpu is refused, gpu_index names one device.
int SiftDevice(Device device, const SiftExtractionOptions& o) {
  if (device == Device::CPU)
    throw std::invalid_argument("[bindings.cc] pycolmap_b200 has no CPU path: use Device.auto or Device.cuda");
  if (o.gpu_index.find(',') != std::string::npos)
    throw std::invalid_argument("[bindings.cc] Check Failed: Sift runs on one GPU: gpu_index is a single index, got \"" +
                                o.gpu_index + "\"");
  int v;
  try {
    v = std::stoi(o.gpu_index);
  } catch (const std::exception&) {
    throw std::invalid_argument("[bindings.cc] Check Failed: gpu_index is an integer, got \"" + o.gpu_index + "\"");
  }
  if (v < -1) throw std::invalid_argument("[bindings.cc] Check Failed: gpu_index >= -1");
  return v < 0 ? 0 : v;
}

struct Sift {
  SiftExtractionOptions options;
  Device device = Device::AUTO;
};

// A 2-D uint8 or float32 array -> a packed uint8 copy; float32 goes through (x * 255) cast to uint8 like
// R:pycolmap/feature/sift.h:82-85, after a range check (upstream's cast is undefined outside [0, 1]).
std::vector<uint8_t> ImageToU8(const py::handle& obj, int max_image_size, int* w, int* h) {
  if (!py::isinstance<py::array>(obj)) throw py::type_error("Sift.extract: image is a 2-D numpy array of uint8 or float32");
  const py::array a = py::reinterpret_borrow<py::array>(obj);
  const bool u8 = a.dtype().is(py::dtype::of<uint8_t>()), f32 = a.dtype().is(py::dtype::of<float>());
  if (!u8 && !f32)
    throw py::type_error("Sift.extract: image dtype must be uint8 or float32, got " + py::str(a.dtype()).cast<std::string>());
  if (a.ndim() != 2) throw std::invalid_argument("[bindings.cc] Check Failed: image.ndim() == 2");
  const int64_t rows = a.shape(0), cols = a.shape(1);
  if (rows == 0 || cols == 0) throw std::invalid_argument("[bindings.cc] Check Failed: image is not empty");
  if (rows > max_image_size)
    throw std::invalid_argument("[sift.h:42] Check Failed: image.rows() <= options_.max_image_size (" + std::to_string(rows) +
                                " vs. " + std::to_string(max_image_size) + ")");
  if (cols > max_image_size)
    throw std::invalid_argument("[sift.h:43] Check Failed: image.cols() <= options_.max_image_size (" + std::to_string(cols) +
                                " vs. " + std::to_string(max_image_size) + ")");
  *w = static_cast<int>(cols);
  *h = static_cast<int>(rows);
  std::vector<uint8_t> out(static_cast<size_t>(rows * cols));
  if (u8) {
    const auto v = py::array_t<uint8_t, py::array::c_style | py::array::forcecast>::ensure(a);
    std::memcpy(out.data(), v.data(), out.size());
  } else {
    const auto v = py::array_t<float, py::array::c_style | py::array::forcecast>::ensure(a);
    const float* p = v.data();
    for (size_t i = 0; i < out.size(); ++i) {
      if (!(p[i] >= 0.0f && p[i] <= 1.0f))
        throw std::invalid_argument("[bindings.cc] Check Failed: float32 image values are finite and in [0, 1]");
      out[i] = static_cast<uint8_t>(p[i] * 255.0f);
    }
  }
  return out;
}

// One ABI call over all images; each result is (keypoints (N, 4) float32, descriptors (N, 128) float32 = u8 / 512).
py::list ExtractBatch(const Sift& s, const py::sequence& images) {
  CheckSiftOptions(s.options);
  const int dev = SiftDevice(s.device, s.options);
  const size_t n = images.size();
  std::vector<std::vector<uint8_t>> px(n);
  std::vector<b2m_image> im(n);
  for (size_t i = 0; i < n; ++i) {
    int w = 0, h = 0;
    px[i] = ImageToU8(images[i], s.options.max_image_size, &w, &h);
    im[i] = b2m_image{w, h, w, px[i].data()};
  }
  const auto extract = SiftSymbol<decltype(&b2m_extract_features_batch)>("b2m_extract_features_batch");
  const auto get = SiftSymbol<decltype(&b2m_features_get)>("b2m_features_get");
  const auto release = SiftSymbol<decltype(&b2m_features_free)>("b2m_features_free");
  b2m_ctx* ctx = Engine::Get(dev);
  const b2m_extract_opts o = ToAbi(s.options);
  b2m_features* f = nullptr;
  int rc;
  {
    py::gil_scoped_release release_gil;
    rc = extract(ctx, im.data(), static_cast<int32_t>(n), &o, &f);
  }
  ThrowOnError(ctx, rc);
  std::unique_ptr<b2m_features, decltype(release)> guard(f, release);
  py::list out;
  for (size_t i = 0; i < n; ++i) {
    b2m_feature_view v;
    std::memset(&v, 0, sizeof(v));
    v.struct_size = sizeof(v);
    ThrowOnError(ctx, get(f, static_cast<int32_t>(i), &v));
    py::array_t<float> kp(std::vector<py::ssize_t>{static_cast<py::ssize_t>(v.n), 4});
    py::array_t<float> desc(std::vector<py::ssize_t>{static_cast<py::ssize_t>(v.n), 128});
    if (v.n) std::memcpy(kp.mutable_data(), v.keypoints, sizeof(float) * 4 * v.n);
    float* d = desc.mutable_data();
    for (int64_t k = 0; k < 128 * v.n; ++k) d[k] = static_cast<float>(v.descriptors[k]) / 512.0f;
    out.append(py::make_tuple(kp, desc));
  }
  return out;
}


// b2m_debug_decode_grey on a JPEG / PNG file's bytes (PNG decoded by the host reader first).
py::array_t<uint8_t> DebugDecodeGrey(b2m_ctx* ctx, const py::bytes& file, int max_image_size) {
  const std::string buf = file;
  const std::vector<uint8_t> bytes(buf.begin(), buf.end());
  ImageHeader h;
  std::string why;
  if (!ReadImageHeader(bytes, &h, &why)) throw std::invalid_argument("[bindings.cc] " + why);
  b2m_image_source s;
  std::memset(&s, 0, sizeof(s));
  Pixels px;
  if (h.format == ImageFormat::PNG) {
    if (!DecodePng(bytes, &px, &why)) throw std::invalid_argument("[bindings.cc] " + why);
    s.kind = B2M_SOURCE_PIXELS;
    s.channels = px.channels;
    s.width = px.width;
    s.height = px.height;
    s.stride = static_cast<int64_t>(px.width) * px.channels;
    s.data = px.data.data();
  } else {
    s.kind = B2M_SOURCE_JPEG;
    s.data = bytes.data();
    s.size = static_cast<int64_t>(bytes.size());
  }
  const auto decode = SiftSymbol<decltype(&b2m_debug_decode_grey)>("b2m_debug_decode_grey");
  int32_t w = 0, hh = 0;
  ThrowOnError(ctx, decode(ctx, &s, max_image_size, nullptr, &w, &hh));
  py::array_t<uint8_t> out(std::vector<py::ssize_t>{hh, w});
  ThrowOnError(ctx, decode(ctx, &s, max_image_size, out.mutable_data(), &w, &hh));
  return out;
}

// ---- feature extraction from image files (R:pycolmap/pipeline/extract_features.h:23-61, images.h:24-94) ------------
// THROW_CHECK_MSG's message (R:log_exceptions.h): "[file:line] Check Failed: <expression> : <message>"
[[noreturn]] void CheckFailed(const char* where, const std::string& expr, const std::string& msg) {
  throw std::invalid_argument(std::string("[") + where + "] Check Failed: " + expr + (msg.empty() ? "" : " : " + msg));
}

bool IsDir(const std::string& p) {
  std::error_code ec;
  return std::filesystem::is_directory(p, ec);
}

bool IsFile(const std::string& p) {
  std::error_code ec;
  return std::filesystem::is_regular_file(p, ec);
}

// Bitmap::Read(path, false) of a mask: grey pixels, or false when the file is not a PNG this reader decodes.
bool ReadMask(const std::string& path, Pixels* grey, std::string* why) {
  Pixels px;
  if (!DecodePng(ReadFileBytes(path), &px, why)) return false;
  grey->width = px.width;
  grey->height = px.height;
  grey->channels = 1;
  grey->data = ToGrey(px);
  return true;
}

// A keypoint passes both masks iff it lies inside both and both are nonzero there: the mask over the common extent.
Pixels MaskAnd(const Pixels& a, const Pixels& b) {
  Pixels m;
  m.width = std::min(a.width, b.width);
  m.height = std::min(a.height, b.height);
  m.channels = 1;
  m.data.resize(static_cast<size_t>(m.width) * m.height);
  for (int y = 0; y < m.height; ++y)
    for (int x = 0; x < m.width; ++x)
      m.data[static_cast<size_t>(y) * m.width + x] =
          a.data[static_cast<size_t>(y) * a.width + x] && b.data[static_cast<size_t>(y) * b.width + x] ? 255 : 0;
  return m;
}

// One image between the reader thread and the device: the file, its decoded PNG pixels, its mask.
struct Loaded {
  ImageReader::Item item;
  Pixels pixels;  // PNG only
  Pixels mask;    // mask_path/<name>.png when it exists
  bool has_mask = false;
};

// Images per device call, and the host bytes (files, PNG pixels, masks) one call may hold: the reader runs one call
// ahead and the writer one call behind, so at most three calls' worth is in memory.
constexpr size_t kExtractBatch = 32;
constexpr size_t kExtractBatchBytes = size_t(256) << 20;

// File reading, PNG decoding and mask reading of images [begin, end) up to the byte budget; touches no database.
std::vector<Loaded> LoadBatch(const ImageReader& reader, const ImageReaderOptions& ro, size_t begin, size_t* end) {
  std::vector<Loaded> out;
  size_t bytes = 0;
  size_t i = begin;
  for (; i < reader.NumImages() && out.size() < kExtractBatch && (out.empty() || bytes < kExtractBatchBytes); ++i) {
    Loaded l;
    reader.Load(i, &l.item);
    try {
      if (l.item.error.empty() && l.item.header.format == ImageFormat::PNG && !DecodePng(l.item.bytes, &l.pixels, &l.item.error))
        l.item.bytes.clear();
      if (l.item.error.empty() && !ro.mask_path.empty()) {
        const std::string mp = (std::filesystem::path(ro.mask_path) / (l.item.name + ".png")).string();
        std::string why;
        if (IsFile(mp)) {
          if (ReadMask(mp, &l.mask, &why)) l.has_mask = true;
          else l.item.error = "mask " + mp + ": " + why;
        }
      }
    } catch (const std::exception& e) {  // out of host memory for one file's pixels: that file is skipped
      l.item.error = std::string("cannot decode it: ") + e.what();
      l.pixels = Pixels();
      l.mask = Pixels();
      l.has_mask = false;
    }
    bytes += l.item.bytes.size() + l.pixels.data.size() + l.mask.data.size();
    out.push_back(std::move(l));
  }
  *end = i;
  return out;
}

// One device call's worth: the loaded images, the sources handed to the device (index into `batch` in `which`) and,
// once the call returned, its features.
struct Call {
  std::vector<Loaded> batch;
  std::vector<b2m_image_source> src;
  std::vector<size_t> which;
  std::vector<Pixels> masks;
  std::shared_ptr<b2m_features> features;
};

// ImageReader::Assign over a loaded batch (cameras go to the database here), and the device sources of the images
// that pass.
void AssignBatch(ImageReader& reader, const Pixels& camera_mask, Call* c) {
  c->masks.resize(c->batch.size());
  for (size_t k = 0; k < c->batch.size(); ++k) {
    Loaded& l = c->batch[k];
    if (reader.Assign(&l.item) != ImageReader::Status::SUCCESS) continue;
    b2m_image_source s;
    std::memset(&s, 0, sizeof(s));
    if (l.item.header.format == ImageFormat::JPEG) {
      s.kind = B2M_SOURCE_JPEG;
      s.data = l.item.bytes.data();
      s.size = static_cast<int64_t>(l.item.bytes.size());
    } else {
      s.kind = B2M_SOURCE_PIXELS;
      s.channels = l.pixels.channels;
      s.width = l.pixels.width;
      s.height = l.pixels.height;
      s.stride = static_cast<int64_t>(l.pixels.width) * l.pixels.channels;
      s.data = l.pixels.data.data();
    }
    const Pixels* m = nullptr;
    if (l.has_mask && !camera_mask.data.empty()) m = &(c->masks[k] = MaskAnd(l.mask, camera_mask));
    else if (l.has_mask) m = &l.mask;
    else if (!camera_mask.data.empty()) m = &camera_mask;
    if (m) {
      s.mask = m->data.data();
      s.mask_width = m->width;
      s.mask_height = m->height;
      s.mask_stride = m->width;
    }
    c->src.push_back(s);
    c->which.push_back(k);
  }
}

// The images, keypoints and descriptors of one call, in one transaction; a source the device could not decode is
// skipped with a warning.
void WriteCall(Database& db, const Call& c, decltype(&b2m_source_features_get) get) {
  DatabaseTransaction txn(&db);
  for (size_t j = 0; j < c.src.size(); ++j) {
    const ImageReader::Item& it = c.batch[c.which[j]].item;
    b2m_source_view v;
    std::memset(&v, 0, sizeof(v));
    if (get(c.features.get(), static_cast<int32_t>(j), &v) != B2M_OK)
      throw std::runtime_error("[bindings.cc] b2m_source_features_get failed for " + it.name);
    if (v.status != B2M_OK) {
      ImageReader::Warn(it.name, v.error && *v.error ? v.error : "does not decode");
      continue;
    }
    if (v.width != it.camera.width || v.height != it.camera.height) {
      ImageReader::Warn(it.name, "decodes to a size other than its header's");
      continue;
    }
    const int64_t id = db.AddImage(it.name, it.camera.camera_id);
    db.WriteKeypoints(id, v.keypoints, v.n, 6);
    db.WriteDescriptors(id, v.descriptors, v.n, 128);
  }
}

// Three stages, as MatchPairsIntoDb has: a reader thread loads call k + 1 (files, PNG, masks), the device runs call k
// (decode, grey, rescale and SIFT; inside it the decoder runs ahead of SIFT), and a writer thread commits call k - 1.
// The database sees one thread at a time: cameras of call k + 1 are assigned after the writer of call k - 1 is done
// and before the writer of call k starts.
void ExtractFeaturesRun(const std::string& database_path, const std::string& image_path,
                        const std::vector<std::string>& image_list, CameraMode mode, const ImageReaderOptions& ro,
                        const SiftExtractionOptions& so, int dev) {
  const auto extract = SiftSymbol<decltype(&b2m_extract_features_sources)>("b2m_extract_features_sources");
  const auto get = SiftSymbol<decltype(&b2m_source_features_get)>("b2m_source_features_get");
  const auto release = SiftSymbol<decltype(&b2m_features_free)>("b2m_features_free");
  Pixels camera_mask;
  if (!ro.camera_mask_path.empty()) {
    std::string why;
    if (!ReadMask(ro.camera_mask_path, &camera_mask, &why)) {  // FeatureExtractorController: go on without the mask
      fprintf(stderr, "E [bindings.cc] Cannot read camera mask file: %s (%s). No mask is going to be used.\n",
              ro.camera_mask_path.c_str(), why.c_str());
      camera_mask = Pixels();
    }
  }
  b2m_ctx* ctx = Engine::Get(dev);
  const b2m_extract_opts opts = ToAbi(so);
  Database db(database_path);
  ImageReader reader(ro, mode, image_path, image_list, &db);
  size_t next = 0;
  auto cur = std::make_unique<Call>();
  cur->batch = LoadBatch(reader, ro, 0, &next);
  AssignBatch(reader, camera_mask, cur.get());
  std::future<void> writer;
  std::future<std::vector<Loaded>> ahead;
  auto drain = [&] {  // leaves no thread behind when an exception unwinds
    if (ahead.valid()) ahead.wait();
    if (writer.valid()) writer.wait();
  };
  try {
    while (!cur->batch.empty()) {
      ahead = std::async(std::launch::async, [&, begin = next] { return LoadBatch(reader, ro, begin, &next); });
      b2m_features* f = nullptr;
      if (!cur->src.empty()) ThrowOnError(ctx, extract(ctx, cur->src.data(), static_cast<int32_t>(cur->src.size()), &opts, &f));
      cur->features.reset(f, release);
      auto following = std::make_unique<Call>();
      following->batch = ahead.get();
      if (writer.valid()) writer.get();
      AssignBatch(reader, camera_mask, following.get());
      writer = std::async(std::launch::async, [&db, get, c = std::shared_ptr<Call>(std::move(cur))] {
        if (c->features) WriteCall(db, *c, get);
      });
      cur = std::move(following);
    }
    if (writer.valid()) writer.get();
  } catch (...) {
    drain();
    throw;
  }
}

// ---- PatchMatch stereo (R:pipeline/mvs.h:92-190; U:mvs/patch_match.h PatchMatchOptions) -----------------------------
// The workspace I/O and the pass controller live in pycolmap_b200/mvs.py; this is the option class and the device call.
struct PatchMatchOptions {
  int max_image_size = -1;
  std::string gpu_index = "-1";
  double depth_min = -1.0;
  double depth_max = -1.0;
  int window_radius = 5;
  int window_step = 1;
  double sigma_spatial = -1.0;
  double sigma_color = 0.2;
  int num_samples = 15;
  double ncc_sigma = 0.6;
  double min_triangulation_angle = 1.0;
  double incident_angle_sigma = 0.9;
  int num_iterations = 5;
  bool geom_consistency = true;
  double geom_consistency_regularizer = 0.3;
  double geom_consistency_max_cost = 3.0;
  bool filter = true;
  double filter_min_ncc = 0.1;
  double filter_min_triangulation_angle = 3.0;
  int filter_min_num_consistent = 2;
  double filter_geom_consistency_max_cost = 1.0;
  double cache_size = 32.0;
  bool allow_missing_files = false;
  bool write_consistency_graph = false;
};

// PatchMatchOptions::Check (U:mvs/patch_match.h), in its order.
void CheckPatchMatchOptions(const PatchMatchOptions& o) {
  auto check = [](bool ok, const char* expr) {
    if (!ok) throw std::invalid_argument(std::string("[patch_match.h] Check Failed: ") + expr);
  };
  if (o.depth_min != -1.0 || o.depth_max != -1.0) {
    check(o.depth_min <= o.depth_max, "depth_min <= depth_max");
    check(o.depth_min >= 0.0, "depth_min >= 0");
  }
  check(o.window_radius <= 32, "window_radius <= kMaxPatchMatchWindowRadius (32)");
  check(o.sigma_color > 0.0, "sigma_color > 0");
  check(o.window_radius > 0, "window_radius > 0");
  check(o.window_step > 0, "window_step > 0");
  check(o.window_step <= 2, "window_step <= 2");
  check(o.num_samples > 0, "num_samples > 0");
  check(o.ncc_sigma > 0.0, "ncc_sigma > 0");
  check(o.min_triangulation_angle >= 0.0, "min_triangulation_angle >= 0");
  check(o.min_triangulation_angle < 180.0, "min_triangulation_angle < 180");
  check(o.incident_angle_sigma > 0.0, "incident_angle_sigma > 0");
  check(o.num_iterations > 0, "num_iterations > 0");
  check(o.geom_consistency_regularizer >= 0.0, "geom_consistency_regularizer >= 0");
  check(o.geom_consistency_max_cost >= 0.0, "geom_consistency_max_cost >= 0");
  check(o.filter_min_ncc >= -1.0, "filter_min_ncc >= -1");
  check(o.filter_min_ncc <= 1.0, "filter_min_ncc <= 1");
  check(o.filter_min_triangulation_angle >= 0.0, "filter_min_triangulation_angle >= 0");
  check(o.filter_min_triangulation_angle <= 180.0, "filter_min_triangulation_angle <= 180");
  check(o.filter_min_num_consistent >= 0, "filter_min_num_consistent >= 0");
  check(o.filter_geom_consistency_max_cost >= 0.0, "filter_geom_consistency_max_cost >= 0");
  check(o.cache_size > 0.0, "cache_size > 0");
}

// One device for PatchMatch, as for extraction: gpu_index is a single ordinal, -1 = device 0.
int PatchMatchDevice(const PatchMatchOptions& o) {
  if (o.gpu_index.find(',') != std::string::npos)
    throw std::invalid_argument("[bindings.cc] Check Failed: patch_match_stereo runs on one GPU: gpu_index is a single "
                                "index, got \"" + o.gpu_index + "\"");
  int v;
  try {
    v = std::stoi(o.gpu_index);
  } catch (const std::exception&) {
    throw std::invalid_argument("[bindings.cc] Check Failed: gpu_index is an integer, got \"" + o.gpu_index + "\"");
  }
  if (v < -1) throw std::invalid_argument("[bindings.cc] Check Failed: gpu_index >= -1");
  return v < 0 ? 0 : v;
}

// The pass a call runs: geometric (geom_consistency) or photometric, filtered or not.
b2m_patch_match_opts ToAbi(const PatchMatchOptions& o, bool geom, bool filter) {
  b2m_patch_match_opts a;  // every field set below: no link-time reference to an ABI 8 symbol
  std::memset(&a, 0, sizeof(a));
  a.struct_size = sizeof(a);
  a.window_radius = o.window_radius;
  a.window_step = o.window_step;
  a.num_samples = o.num_samples;
  a.num_iterations = o.num_iterations;
  a.geom_consistency = geom ? 1 : 0;
  a.filter = filter ? 1 : 0;
  a.filter_min_num_consistent = o.filter_min_num_consistent;
  a.sigma_spatial = static_cast<float>(o.sigma_spatial);
  a.sigma_color = static_cast<float>(o.sigma_color);
  a.ncc_sigma = static_cast<float>(o.ncc_sigma);
  a.min_triangulation_angle = static_cast<float>(o.min_triangulation_angle);
  a.incident_angle_sigma = static_cast<float>(o.incident_angle_sigma);
  a.geom_consistency_regularizer = static_cast<float>(o.geom_consistency_regularizer);
  a.geom_consistency_max_cost = static_cast<float>(o.geom_consistency_max_cost);
  a.filter_min_ncc = static_cast<float>(o.filter_min_ncc);
  a.filter_min_triangulation_angle = static_cast<float>(o.filter_min_triangulation_angle);
  a.filter_geom_consistency_max_cost = static_cast<float>(o.filter_geom_consistency_max_cost);
  return a;
}

// The host copies one device call reads: grey images, cameras [n x 16], optional depth maps, problems.
struct PmInputs {
  std::vector<ArrU8> images;
  std::vector<b2m_image> ims;
  ArrD cameras;
  std::vector<ArrF32> dmaps;
  std::vector<const float*> dmap_ptrs;
  std::vector<std::vector<int32_t>> src;
  std::vector<ArrF32> init;
  std::vector<b2m_patch_match_problem> probs;
};

void LoadPmInputs(const py::list& images, const ArrD& cameras, const py::object& depth_maps, const py::list& problems,
                  PmInputs* in) {
  const size_t n = images.size();
  if (cameras.ndim() != 2 || cameras.shape(0) != static_cast<py::ssize_t>(n) || cameras.shape(1) != 16)
    throw std::invalid_argument("[bindings.cc] Check Failed: cameras is an n x 16 array (fx, fy, cx, cy, R, t)");
  in->cameras = cameras;
  for (size_t i = 0; i < n; ++i) {
    ArrU8 a = ArrU8::ensure(images[i]);
    if (!a || a.ndim() != 2) throw std::invalid_argument("[bindings.cc] Check Failed: images are 2-D uint8 arrays");
    in->ims.push_back(b2m_image{static_cast<int32_t>(a.shape(1)), static_cast<int32_t>(a.shape(0)), a.shape(1), a.data()});
    in->images.push_back(std::move(a));
  }
  if (!depth_maps.is_none()) {
    const py::list dl = depth_maps;
    if (dl.size() != n) throw std::invalid_argument("[bindings.cc] Check Failed: one depth map entry per image");
    for (size_t i = 0; i < n; ++i) {
      if (dl[i].is_none()) {
        in->dmap_ptrs.push_back(nullptr);
        continue;
      }
      ArrF32 d = ArrF32::ensure(dl[i]);
      if (!d || d.ndim() != 2 || d.shape(0) != in->ims[i].height || d.shape(1) != in->ims[i].width)
        throw std::invalid_argument("[bindings.cc] Check Failed: a depth map has its image's size");
      in->dmap_ptrs.push_back(d.data());
      in->dmaps.push_back(std::move(d));
    }
  }
  in->src.resize(problems.size());
  for (size_t k = 0; k < problems.size(); ++k) {
    const py::dict d = problems[k];
    b2m_patch_match_problem p;
    std::memset(&p, 0, sizeof(p));
    p.struct_size = sizeof(p);
    p.ref = d["ref"].cast<int32_t>();
    p.image_id = d.contains("image_id") ? d["image_id"].cast<int32_t>() : p.ref;
    in->src[k] = d["src"].cast<std::vector<int32_t>>();
    p.n_src = static_cast<int32_t>(in->src[k].size());
    p.src = in->src[k].data();
    p.depth_min = d["depth_min"].cast<float>();
    p.depth_max = d["depth_max"].cast<float>();
    if (d.contains("init_depth") && !d["init_depth"].is_none()) {
      if (p.ref < 0 || p.ref >= static_cast<int32_t>(n)) throw std::invalid_argument("[bindings.cc] Check Failed: ref in range");
      ArrF32 dep = ArrF32::ensure(d["init_depth"]), nor = ArrF32::ensure(d["init_normal"]);
      const b2m_image& im = in->ims[p.ref];
      if (!dep || !nor || dep.ndim() != 2 || dep.shape(0) != im.height || dep.shape(1) != im.width || nor.ndim() != 3 ||
          nor.shape(0) != im.height || nor.shape(1) != im.width || nor.shape(2) != 3)
        throw std::invalid_argument("[bindings.cc] Check Failed: init_depth (H, W) and init_normal (H, W, 3) of the reference");
      p.init_depth = dep.data();
      p.init_normal = nor.data();
      in->init.push_back(std::move(dep));
      in->init.push_back(std::move(nor));
    }
    in->probs.push_back(p);
  }
}

// One device call: upload the image set, run the problems, return [(depth (H, W), normal (H, W, 3))].
py::list PatchMatchRun(b2m_ctx* ctx, const py::list& images, const ArrD& cameras, const py::object& depth_maps,
                       const py::list& problems, const PatchMatchOptions& options, bool geom, bool filter) {
  CheckPatchMatchOptions(options);
  PmInputs in;
  LoadPmInputs(images, cameras, depth_maps, problems, &in);
  const auto set = SiftSymbol<decltype(&b2m_patch_match_set_images)>("b2m_patch_match_set_images");
  const auto batch = SiftSymbol<decltype(&b2m_patch_match_batch)>("b2m_patch_match_batch");
  const auto get = SiftSymbol<decltype(&b2m_depth_maps_get)>("b2m_depth_maps_get");
  const auto release = SiftSymbol<decltype(&b2m_depth_maps_free)>("b2m_depth_maps_free");
  const b2m_patch_match_opts o = ToAbi(options, geom, filter);
  b2m_depth_maps* maps = nullptr;
  RunInterruptible([&] {
    ThrowOnError(ctx, set(ctx, static_cast<int32_t>(in.ims.size()), in.ims.data(), in.cameras.data(),
                          in.dmap_ptrs.empty() ? nullptr : in.dmap_ptrs.data()));
    ThrowOnError(ctx, batch(ctx, in.probs.data(), static_cast<int32_t>(in.probs.size()), &o, &maps));
  });
  std::unique_ptr<b2m_depth_maps, decltype(release)> guard(maps, release);
  py::list out;
  for (size_t k = 0; k < in.probs.size(); ++k) {
    b2m_depth_map_view v;
    std::memset(&v, 0, sizeof(v));
    ThrowOnError(ctx, get(maps, static_cast<int32_t>(k), &v));
    py::array_t<float> dep(std::vector<py::ssize_t>{v.height, v.width});
    py::array_t<float> nor(std::vector<py::ssize_t>{v.height, v.width, 3});
    std::memcpy(dep.mutable_data(), v.depth, sizeof(float) * v.width * v.height);
    std::memcpy(nor.mutable_data(), v.normal, sizeof(float) * 3 * v.width * v.height);
    out.append(py::make_tuple(dep, nor));
  }
  return out;
}

// ---- stereo fusion (R:pipeline/mvs.h:43-90, 193-254; U:mvs/fusion.h StereoFusionOptions) ----------------------------
// The workspace I/O lives in pycolmap_b200/mvs.py; this is the option class and the device call.
struct StereoFusionOptions {
  std::string mask_path = "";
  int num_threads = -1;
  int max_image_size = -1;
  int min_num_pixels = 5;
  int max_num_pixels = 10000;
  int max_traversal_depth = 100;
  double max_reproj_error = 2.0;
  double max_depth_error = 0.01;
  double max_normal_error = 10.0;
  int check_num_images = 50;
  bool use_cache = false;
  double cache_size = 32.0;
  std::pair<std::array<float, 3>, std::array<float, 3>> bounding_box{{-FLT_MAX, -FLT_MAX, -FLT_MAX},
                                                                      {FLT_MAX, FLT_MAX, FLT_MAX}};
};

// StereoFusionOptions::Check (U:mvs/fusion.cc), in its order; num_threads, use_cache and cache_size have no effect.
void CheckStereoFusionOptions(const StereoFusionOptions& o) {
  auto check = [](bool ok, const char* expr) {
    if (!ok) throw std::invalid_argument(std::string("[fusion.cc] Check Failed: ") + expr);
  };
  check(o.min_num_pixels >= 0, "min_num_pixels >= 0");
  check(o.min_num_pixels <= o.max_num_pixels, "min_num_pixels <= max_num_pixels");
  check(o.max_traversal_depth > 0, "max_traversal_depth > 0");
  check(o.max_reproj_error >= 0.0, "max_reproj_error >= 0");
  check(o.max_depth_error >= 0.0, "max_depth_error >= 0");
  check(o.max_normal_error >= 0.0, "max_normal_error >= 0");
  check(o.check_num_images > 0, "check_num_images > 0");
  check(o.cache_size > 0.0, "cache_size > 0");
  check(o.num_threads == -1 || o.num_threads > 0, "num_threads == -1 || num_threads > 0");
}

// One device call: images [dict(depth, normal, mask, P, inv_P, inv_R, bitmap_scale, overlap, color)] -> dict.
// color: a JPEG / PNG file's bytes, an (H, W[, C]) uint8 array, or None.
py::dict StereoFusionRun(b2m_ctx* ctx, const py::list& images, const StereoFusionOptions& options) {
  CheckStereoFusionOptions(options);
  const size_t n = images.size();
  std::vector<b2m_fusion_image> im(n);
  std::vector<ArrF32> keep_f;
  std::vector<ArrU8> keep_u;
  std::vector<std::vector<int32_t>> ov(n);
  std::vector<std::vector<uint8_t>> bytes(n);
  std::vector<Pixels> px(n);
  auto f32 = [&](const py::handle& o, size_t count, float* dst, const char* what) {
    ArrF32 a = ArrF32::ensure(o);
    if (!a || static_cast<size_t>(a.size()) != count)
      throw std::invalid_argument(std::string("[bindings.cc] Check Failed: ") + what + " has " + std::to_string(count) + " values");
    std::memcpy(dst, a.data(), sizeof(float) * count);
  };
  for (size_t i = 0; i < n; ++i) {
    const py::dict d = images[i];
    b2m_fusion_image& m = im[i];
    std::memset(&m, 0, sizeof(m));
    m.struct_size = sizeof(m);
    if (d.contains("depth") && !d["depth"].is_none()) {
      ArrF32 dep = ArrF32::ensure(d["depth"]), nor = ArrF32::ensure(d["normal"]);
      if (!dep || dep.ndim() != 2 || !nor || nor.ndim() != 3 || nor.shape(0) != dep.shape(0) || nor.shape(1) != dep.shape(1) ||
          nor.shape(2) != 3)
        throw std::invalid_argument("[bindings.cc] Check Failed: depth (H, W) and normal (H, W, 3) float32 maps");
      m.width = static_cast<int32_t>(dep.shape(1));
      m.height = static_cast<int32_t>(dep.shape(0));
      m.depth = dep.data();
      m.normal = nor.data();
      keep_f.push_back(std::move(dep));
      keep_f.push_back(std::move(nor));
      if (d.contains("mask") && !d["mask"].is_none()) {
        ArrU8 mk = ArrU8::ensure(d["mask"]);
        if (!mk || mk.ndim() != 2 || mk.shape(0) != m.height || mk.shape(1) != m.width)
          throw std::invalid_argument("[bindings.cc] Check Failed: a mask has its depth map's size");
        m.mask = mk.data();
        keep_u.push_back(std::move(mk));
      }
    }
    f32(d["P"], 12, m.P, "P");
    f32(d["inv_P"], 12, m.inv_P, "inv_P");
    f32(d["inv_R"], 9, m.inv_R, "inv_R");
    f32(d["bitmap_scale"], 2, m.bitmap_scale, "bitmap_scale");
    ov[i] = d["overlap"].cast<std::vector<int32_t>>();
    m.overlap = ov[i].data();
    m.n_overlap = static_cast<int32_t>(ov[i].size());
    b2m_image_source& s = m.color;
    const py::object c = d.contains("color") ? py::object(d["color"]) : py::object(py::none());
    if (py::isinstance<py::bytes>(c)) {
      const std::string buf = c.cast<std::string>();
      bytes[i].assign(buf.begin(), buf.end());
      ImageHeader h;
      std::string why;
      if (!ReadImageHeader(bytes[i], &h, &why)) throw std::invalid_argument("[bindings.cc] image " + std::to_string(i) + ": " + why);
      if (h.format == ImageFormat::PNG) {
        if (!DecodePng(bytes[i], &px[i], &why)) throw std::invalid_argument("[bindings.cc] image " + std::to_string(i) + ": " + why);
        s.kind = B2M_SOURCE_PIXELS;
        s.channels = px[i].channels;
        s.width = px[i].width;
        s.height = px[i].height;
        s.stride = static_cast<int64_t>(px[i].width) * px[i].channels;
        s.data = px[i].data.data();
      } else {
        s.kind = B2M_SOURCE_JPEG;
        s.data = bytes[i].data();
        s.size = static_cast<int64_t>(bytes[i].size());
      }
    } else if (!c.is_none()) {
      ArrU8 a = ArrU8::ensure(c);
      if (!a || (a.ndim() != 2 && a.ndim() != 3) || (a.ndim() == 3 && a.shape(2) != 1 && a.shape(2) != 3 && a.shape(2) != 4))
        throw std::invalid_argument("[bindings.cc] Check Failed: a color array is (H, W) or (H, W, 1 | 3 | 4) uint8");
      s.kind = B2M_SOURCE_PIXELS;
      s.channels = a.ndim() == 3 ? static_cast<int32_t>(a.shape(2)) : 1;
      s.width = static_cast<int32_t>(a.shape(1));
      s.height = static_cast<int32_t>(a.shape(0));
      s.stride = static_cast<int64_t>(s.width) * s.channels;
      s.data = a.data();
      keep_u.push_back(std::move(a));
    }
  }
  b2m_fusion_opts o;  // every field set below: no link-time reference to an ABI 9 symbol
  std::memset(&o, 0, sizeof(o));
  o.struct_size = sizeof(o);
  o.min_num_pixels = options.min_num_pixels;
  o.max_num_pixels = options.max_num_pixels;
  o.max_traversal_depth = options.max_traversal_depth;
  o.max_reproj_error = static_cast<float>(options.max_reproj_error);
  o.max_depth_error = static_cast<float>(options.max_depth_error);
  o.max_normal_error = static_cast<float>(options.max_normal_error);
  for (int k = 0; k < 3; ++k) {
    o.bounding_box[k] = options.bounding_box.first[k];
    o.bounding_box[3 + k] = options.bounding_box.second[k];
  }
  const auto fuse = SiftSymbol<decltype(&b2m_stereo_fusion)>("b2m_stereo_fusion");
  const auto get = SiftSymbol<decltype(&b2m_fused_points_get)>("b2m_fused_points_get");
  const auto release = SiftSymbol<decltype(&b2m_fused_points_free)>("b2m_fused_points_free");
  b2m_fused_points* pts = nullptr;
  RunInterruptible([&] { ThrowOnError(ctx, fuse(ctx, im.data(), static_cast<int32_t>(n), &o, &pts)); });
  std::unique_ptr<b2m_fused_points, decltype(release)> guard(pts, release);
  b2m_fused_points_view v;
  std::memset(&v, 0, sizeof(v));
  ThrowOnError(ctx, get(pts, &v));
  const py::ssize_t N = v.n_points, M = v.n_order;
  py::array_t<float> xyz(std::vector<py::ssize_t>{N, 3}), nrm(std::vector<py::ssize_t>{N, 3});
  py::array_t<uint8_t> col(std::vector<py::ssize_t>{N, 3});
  py::array_t<int32_t> seeds(std::vector<py::ssize_t>{N, 3}), order(std::vector<py::ssize_t>{M, 4});
  py::array_t<int64_t> voff(N + 1);
  py::array_t<int32_t> vis(static_cast<py::ssize_t>(N ? v.vis_off[N] : 0));
  if (N) {
    std::memcpy(xyz.mutable_data(), v.xyz, sizeof(float) * 3 * N);
    std::memcpy(nrm.mutable_data(), v.normals, sizeof(float) * 3 * N);
    std::memcpy(col.mutable_data(), v.colors, 3 * N);
    std::memcpy(seeds.mutable_data(), v.seeds, sizeof(int32_t) * 3 * N);
    std::memcpy(vis.mutable_data(), v.vis, sizeof(int32_t) * v.vis_off[N]);
  }
  std::memcpy(voff.mutable_data(), v.vis_off, sizeof(int64_t) * (N + 1));
  if (M) std::memcpy(order.mutable_data(), v.order, sizeof(int32_t) * 4 * M);
  py::dict out;
  out["xyz"] = xyz;
  out["normals"] = nrm;
  out["colors"] = col;
  out["vis_off"] = voff;
  out["vis"] = vis;
  out["seeds"] = seeds;
  out["order"] = order;
  return out;
}

// ---- image undistortion (R:pipeline/images.h:96-261; U:image/undistortion.h UndistortCameraOptions) ----------------
// The workspace I/O lives in pycolmap_b200/mvs.py; this is the option class, the camera and the device call.
struct UndistortCameraOptions {
  double blank_pixels = 0.0;
  double min_scale = 0.2;
  double max_scale = 2.0;
  int max_image_size = -1;
  double roi_min_x = 0.0;
  double roi_min_y = 0.0;
  double roi_max_x = 1.0;
  double roi_max_y = 1.0;
};

enum class CopyType { COPY = 0, SOFT_LINK = 1, HARD_LINK = 2 };  // U:util/misc.h FileCopyType

// UndistortCameraOptions' checks (UndistortCamera's CHECKs, U:image/undistortion.cc), in their order.
void CheckUndistortOptions(const UndistortCameraOptions& o) {
  auto check = [](bool ok, const char* expr) {
    if (!ok) throw std::invalid_argument(std::string("[undistortion.cc] Check Failed: ") + expr);
  };
  check(o.blank_pixels >= 0, "blank_pixels >= 0");
  check(o.blank_pixels <= 1, "blank_pixels <= 1");
  check(o.min_scale > 0.0, "min_scale > 0");
  check(o.min_scale <= o.max_scale, "min_scale <= max_scale");
  check(o.max_image_size != 0, "max_image_size != 0");
  check(o.roi_min_x >= 0.0, "roi_min_x >= 0");
  check(o.roi_min_y >= 0.0, "roi_min_y >= 0");
  check(o.roi_max_x <= 1.0, "roi_max_x <= 1");
  check(o.roi_max_y <= 1.0, "roi_max_y <= 1");
  check(o.roi_min_x < o.roi_max_x, "roi_min_x < roi_max_x");
  check(o.roi_min_y < o.roi_max_y, "roi_min_y < roi_max_y");
}

b2m_undistort_opts ToAbi(const UndistortCameraOptions& o) {
  b2m_undistort_opts a;  // every field set here: no link-time reference to an ABI 10 symbol
  std::memset(&a, 0, sizeof(a));
  a.struct_size = sizeof(a);
  a.max_image_size = o.max_image_size;
  a.blank_pixels = o.blank_pixels;
  a.min_scale = o.min_scale;
  a.max_scale = o.max_scale;
  a.roi_min_x = o.roi_min_x;
  a.roi_min_y = o.roi_min_y;
  a.roi_max_x = o.roi_max_x;
  a.roi_max_y = o.roi_max_y;
  return a;
}

py::dict AbiCameraToDict(const b2m_camera& c) {
  const int n = b2m::cam::num_params(c.model);
  return py::dict("model"_a = c.model, "width"_a = c.width, "height"_a = c.height,
                  "params"_a = std::vector<double>(c.params, c.params + std::max(n, 0)));
}

py::dict UndistortCameraPy(const UndistortCameraOptions& options, const py::object& camera) {
  CheckUndistortOptions(options);
  const b2m_camera c = CameraFromPython(camera);
  const b2m_undistort_opts o = ToAbi(options);
  const auto und = SiftSymbol<decltype(&b2m_undistort_camera)>("b2m_undistort_camera");
  b2m_camera out;
  std::memset(&out, 0, sizeof(out));
  if (und(nullptr, &o, &c, &out) != B2M_OK) throw std::invalid_argument(b2m_last_error(nullptr));
  return AbiCameraToDict(out);
}

// The device source of a JPEG / PNG file's bytes: JPEG goes whole to the device, PNG is decoded here into *px (which
// must outlive the source).  False with *why for a file that is neither, or a PNG this reader does not decode.
bool SourceFromFile(const std::vector<uint8_t>& bytes, Pixels* px, b2m_image_source* s, std::string* why) {
  ImageHeader h;
  if (!ReadImageHeader(bytes, &h, why)) return false;
  if (h.format == ImageFormat::PNG) {
    if (!DecodePng(bytes, px, why)) return false;
    s->kind = B2M_SOURCE_PIXELS;
    s->channels = px->channels;
    s->width = px->width;
    s->height = px->height;
    s->stride = static_cast<int64_t>(px->width) * px->channels;
    s->data = px->data.data();
  } else {
    s->kind = B2M_SOURCE_JPEG;
    s->data = bytes.data();
    s->size = static_cast<int64_t>(bytes.size());
  }
  return true;
}

// One device call over items [(file bytes, camera, "jpeg" | "pixels")]: per item dict(status, error, camera, data), data
// = the JPEG file's bytes or an (H, W, 3) uint8 array.  PNG files are decoded here; a file that is neither JPEG nor a
// PNG this reader decodes gets an error status, like one the device cannot decode.
py::list UndistortRun(b2m_ctx* ctx, const py::list& items, const UndistortCameraOptions& options) {
  CheckUndistortOptions(options);
  const size_t n = items.size();
  std::vector<std::vector<uint8_t>> bytes(n);
  std::vector<Pixels> px(n);
  std::vector<std::string> host_error(n);
  std::vector<b2m_undistort_item> it;
  std::vector<size_t> which;
  for (size_t i = 0; i < n; ++i) {
    const py::tuple t = items[i];
    const std::string buf = t[0].cast<std::string>();
    bytes[i].assign(buf.begin(), buf.end());
    const std::string kind = t[2].cast<std::string>();
    if (kind != "jpeg" && kind != "pixels")
      throw std::invalid_argument("[bindings.cc] Check Failed: output is \"jpeg\" or \"pixels\", got \"" + kind + "\"");
    b2m_undistort_item m;
    std::memset(&m, 0, sizeof(m));
    m.struct_size = sizeof(m);
    m.output = kind == "jpeg" ? B2M_UNDISTORT_JPEG : B2M_UNDISTORT_PIXELS;
    m.camera = CameraFromPython(t[1]);
    if (!SourceFromFile(bytes[i], &px[i], &m.source, &host_error[i])) continue;
    it.push_back(m);
    which.push_back(i);
  }
  const b2m_undistort_opts o = ToAbi(options);
  const auto run = SiftSymbol<decltype(&b2m_undistort_images)>("b2m_undistort_images");
  const auto get = SiftSymbol<decltype(&b2m_undistorted_get)>("b2m_undistorted_get");
  const auto release = SiftSymbol<decltype(&b2m_undistorted_free)>("b2m_undistorted_free");
  b2m_undistorted* r = nullptr;
  RunInterruptible([&] { ThrowOnError(ctx, run(ctx, it.data(), static_cast<int32_t>(it.size()), &o, &r)); });
  std::unique_ptr<b2m_undistorted, decltype(release)> guard(r, release);
  std::vector<py::object> out(n, py::none());
  for (size_t j = 0; j < which.size(); ++j) {
    b2m_undistorted_view v;
    std::memset(&v, 0, sizeof(v));
    ThrowOnError(ctx, get(r, static_cast<int32_t>(j), &v));
    py::object data = py::none();
    if (v.status == B2M_OK) {
      if (it[j].output == B2M_UNDISTORT_JPEG) {
        data = py::bytes(reinterpret_cast<const char*>(v.data), static_cast<size_t>(v.size));
      } else {
        py::array_t<uint8_t> a(std::vector<py::ssize_t>{v.height, v.width, 3});
        std::memcpy(a.mutable_data(), v.data, static_cast<size_t>(v.size));
        data = a;
      }
    }
    out[which[j]] = py::dict("status"_a = v.status, "error"_a = std::string(v.error ? v.error : ""),
                             "camera"_a = AbiCameraToDict(v.camera), "data"_a = data);
  }
  py::list res;
  for (size_t i = 0; i < n; ++i) {
    if (out[i].is_none())
      out[i] = py::dict("status"_a = static_cast<int>(B2M_EINVAL), "error"_a = host_error[i], "camera"_a = py::none(),
                        "data"_a = py::none());
    res.append(out[i]);
  }
  return res;
}

void CheckCameraMode(const ImageReaderOptions& o, const char* where) {
  if (CameraModelId(o.camera_model) < 0)
    throw std::invalid_argument(std::string("[") + where + "] Invalid camera model: " + o.camera_model);
}
}  // namespace

PYBIND11_MODULE(_core, m) {
  m.doc() = "C++ host layer of pycolmap_b200 (pybind11 over the C ABI of libb200match.so)";
  m.attr("has_cuda") = true;  // R:main.cc:98
  m.attr("abi_version") = b2m_abi_version();

  py::register_exception_translator([](std::exception_ptr p) {
    try {
      if (p) std::rethrow_exception(p);
    } catch (const StoppedError&) {
      PyErr_SetString(PyExc_KeyboardInterrupt, "stopped");
    }
  });

  // ---- enums ----
  auto device = py::enum_<Device>(m, "Device").value("auto", Device::AUTO).value("cpu", Device::CPU).value("cuda", Device::CUDA);
  AddStringConstructor(device);
  auto config = py::enum_<TwoViewGeometryConfiguration>(m, "TwoViewGeometryConfiguration")
                    .value("UNDEFINED", TwoViewGeometryConfiguration::UNDEFINED)
                    .value("DEGENERATE", TwoViewGeometryConfiguration::DEGENERATE)
                    .value("CALIBRATED", TwoViewGeometryConfiguration::CALIBRATED)
                    .value("UNCALIBRATED", TwoViewGeometryConfiguration::UNCALIBRATED)
                    .value("PLANAR", TwoViewGeometryConfiguration::PLANAR)
                    .value("PANORAMIC", TwoViewGeometryConfiguration::PANORAMIC)
                    .value("PLANAR_OR_PANORAMIC", TwoViewGeometryConfiguration::PLANAR_OR_PANORAMIC)
                    .value("WATERMARK", TwoViewGeometryConfiguration::WATERMARK)
                    .value("MULTIPLE", TwoViewGeometryConfiguration::MULTIPLE);
  AddStringConstructor(config);

  // ---- option classes ----
  OptionsClass<RANSACOptions>(m, "RANSACOptions")
      .field("max_error", &RANSACOptions::max_error)
      .field("min_inlier_ratio", &RANSACOptions::min_inlier_ratio)
      .field("confidence", &RANSACOptions::confidence)
      .field("dyn_num_trials_multiplier", &RANSACOptions::dyn_num_trials_multiplier)
      .field("min_num_trials", &RANSACOptions::min_num_trials)
      .field("max_num_trials", &RANSACOptions::max_num_trials)
      .Finish();
  OptionsClass<SiftMatchingOptions>(m, "SiftMatchingOptions")
      .field("num_threads", &SiftMatchingOptions::num_threads)
      .field("gpu_index", &SiftMatchingOptions::gpu_index,
             "Index of the GPU used for feature matching. For multi-GPU matching, you should separate multiple "
             "GPU indices by comma, e.g., \"0,1,2,3\".")
      .field("max_ratio", &SiftMatchingOptions::max_ratio, "Maximum distance ratio between first and second best match.")
      .field("max_distance", &SiftMatchingOptions::max_distance, "Maximum distance to best match.")
      .field("cross_check", &SiftMatchingOptions::cross_check, "Whether to enable cross checking in matching.")
      .field("max_num_matches", &SiftMatchingOptions::max_num_matches, "Maximum number of matches.")
      .field("guided_matching", &SiftMatchingOptions::guided_matching,
             "Whether to perform guided matching, if geometric verification succeeds.")
      .Finish();
  OptionsClass<ExhaustiveMatchingOptions>(m, "ExhaustiveMatchingOptions")
      .field("block_size", &ExhaustiveMatchingOptions::block_size)
      .Finish();
  OptionsClass<SequentialMatchingOptions>(m, "SequentialMatchingOptions")
      .field("overlap", &SequentialMatchingOptions::overlap, "Number of overlapping image pairs.")
      .field("quadratic_overlap", &SequentialMatchingOptions::quadratic_overlap,
             "Whether to match images against their quadratic neighbors.")
      .field("loop_detection", &SequentialMatchingOptions::loop_detection,
             "Loop detection is invoked every `loop_detection_period` images.")
      .field("loop_detection_period", &SequentialMatchingOptions::loop_detection_period)
      .field("loop_detection_num_images", &SequentialMatchingOptions::loop_detection_num_images)
      .field("loop_detection_num_nearest_neighbors", &SequentialMatchingOptions::loop_detection_num_nearest_neighbors)
      .field("loop_detection_num_checks", &SequentialMatchingOptions::loop_detection_num_checks)
      .field("loop_detection_num_images_after_verification",
             &SequentialMatchingOptions::loop_detection_num_images_after_verification)
      .field("loop_detection_max_num_features", &SequentialMatchingOptions::loop_detection_max_num_features)
      .field("vocab_tree_path", &SequentialMatchingOptions::vocab_tree_path)
      .Finish();
  OptionsClass<SpatialMatchingOptions>(m, "SpatialMatchingOptions")
      .field("is_gps", &SpatialMatchingOptions::is_gps,
             "Whether the location priors in the database are GPS coordinates in the form of longitude and latitude "
             "coordinates in degrees.")
      .field("ignore_z", &SpatialMatchingOptions::ignore_z, "Whether to ignore the Z-component of the location prior.")
      .field("max_num_neighbors", &SpatialMatchingOptions::max_num_neighbors, "The maximum number of nearest neighbors to match.")
      .field("max_distance", &SpatialMatchingOptions::max_distance,
             "The maximum distance between the query and nearest neighbor [meters].")
      .Finish();
  OptionsClass<TwoViewGeometryOptions>(m, "TwoViewGeometryOptions")
      .field("min_num_inliers", &TwoViewGeometryOptions::min_num_inliers)
      .field("min_E_F_inlier_ratio", &TwoViewGeometryOptions::min_E_F_inlier_ratio)
      .field("max_H_inlier_ratio", &TwoViewGeometryOptions::max_H_inlier_ratio)
      .field("watermark_min_inlier_ratio", &TwoViewGeometryOptions::watermark_min_inlier_ratio)
      .field("watermark_border_size", &TwoViewGeometryOptions::watermark_border_size)
      .field("detect_watermark", &TwoViewGeometryOptions::detect_watermark)
      .field("multiple_ignore_watermark", &TwoViewGeometryOptions::multiple_ignore_watermark)
      .field("force_H_use", &TwoViewGeometryOptions::force_H_use)
      .field("compute_relative_pose", &TwoViewGeometryOptions::compute_relative_pose)
      .field("multiple_models", &TwoViewGeometryOptions::multiple_models)
      .field("ransac", &TwoViewGeometryOptions::ransac)
      .Finish();

  py::class_<Rotation3d>(m, "Rotation3d")
      .def(py::init<>())
      .def(py::init([](const std::array<double, 4>& xyzw) {   // Eigen coefficient order, like the reference
             Rotation3d r;
             r.wxyz = {xyzw[3], xyzw[0], xyzw[1], xyzw[2]};
             return r;
           }),
           "xyzw"_a)
      .def_property_readonly("quat", [](const Rotation3d& r) {   // (x, y, z, w) like the reference's Eigen coefficients
        py::array_t<double> a(4);
        double* p = a.mutable_data();
        p[0] = r.wxyz[1]; p[1] = r.wxyz[2]; p[2] = r.wxyz[3]; p[3] = r.wxyz[0];
        return a;
      })
      .def("matrix", [](const Rotation3d& r) { return MatToNumpy(QuatToRotation(r.wxyz).data()); });
  py::class_<Rigid3d>(m, "Rigid3d")
      .def(py::init<>())
      .def(py::init([](const Rotation3d& rotation, const std::array<double, 3>& translation) {
             return Rigid3d{rotation, translation};
           }),
           "rotation"_a, "translation"_a)
      .def_readonly("rotation", &Rigid3d::rotation)
      .def_property_readonly("translation", [](const Rigid3d& g) {
        py::array_t<double> a(3);
        std::copy(g.translation.begin(), g.translation.end(), a.mutable_data());
        return a;
      })
      .def("matrix", [](const Rigid3d& g) {
        const std::array<double, 12> m = RigidToMatrix(g);
        py::array_t<double> a(std::vector<py::ssize_t>{3, 4});
        std::copy(m.begin(), m.end(), a.mutable_data());
        return a;
      })
      .def("inverse", [](const Rigid3d& g) {
        Rigid3d o = g;
        InvertPose(&o.rotation.wxyz, &o.translation);
        return o;
      });

  // ---- TwoViewGeometry ----
  py::class_<TwoViewGeometry>(m, "TwoViewGeometry")
      .def(py::init<>())
      .def(py::init([](TwoViewGeometryConfiguration config, const py::object& E, const py::object& F,
                       const py::object& H, const py::object& inlier_matches, double tri_angle, const py::object& qvec,
                       const py::object& tvec) {
             TwoViewGeometry g;
             g.config = config;
             auto mat = [](const py::object& o, Mat3* out) {
               if (o.is_none()) return;
               const ArrD a = ArrD::ensure(o);
               if (!a || a.size() != 9) throw std::invalid_argument("[bindings.cc] Check Failed: matrix is 3 x 3");
               std::copy(a.data(), a.data() + 9, out->begin());
             };
             mat(E, &g.E); mat(F, &g.F); mat(H, &g.H);
             if (!inlier_matches.is_none()) {
               const ArrU32 a = ArrU32::ensure(inlier_matches);
               if (!a || a.size() % 2) throw std::invalid_argument("[bindings.cc] Check Failed: matches is N x 2");
               g.inlier_matches.assign(a.data(), a.data() + a.size());
             }
             g.tri_angle = tri_angle;
             auto vec = [](const py::object& o, double* out, py::ssize_t n, const char* what) {
               if (o.is_none()) return;
               const ArrD a = ArrD::ensure(o);
               if (!a || a.size() != n) throw std::invalid_argument(std::string("[bindings.cc] Check Failed: ") + what);
               std::copy(a.data(), a.data() + n, out);
             };
             vec(qvec, g.qvec.data(), 4, "qvec = (w, x, y, z)");
             vec(tvec, g.tvec.data(), 3, "tvec has 3 entries");
             return g;
           }),
           "config"_a = TwoViewGeometryConfiguration::UNDEFINED, "E"_a = py::none(), "F"_a = py::none(),
           "H"_a = py::none(), "inlier_matches"_a = py::none(), "tri_angle"_a = 0.0, "qvec"_a = py::none(),
           "tvec"_a = py::none())
      .def_property_readonly("config", [](const TwoViewGeometry& g) { return g.config; })
      .def_property_readonly("E", [](const TwoViewGeometry& g) { return MatToNumpy(g.E.data()); })
      .def_property_readonly("F", [](const TwoViewGeometry& g) { return MatToNumpy(g.F.data()); })
      .def_property_readonly("H", [](const TwoViewGeometry& g) { return MatToNumpy(g.H.data()); })
      .def_property_readonly("cam2_from_cam1",
                             [](const TwoViewGeometry& g) { return Rigid3d{Rotation3d{g.qvec}, g.tvec}; },
                             "Relative pose (identity unless options.compute_relative_pose recovered one).")
      .def_property_readonly("inlier_matches",
                             [](const TwoViewGeometry& g) {
                               return MatchesToNumpy(g.inlier_matches.data(),
                                                     static_cast<int64_t>(g.inlier_matches.size() / 2));
                             })
      .def_readonly("tri_angle", &TwoViewGeometry::tri_angle)
      .def_property_readonly("num_inliers_EFH", [](const TwoViewGeometry& g) { return py::make_tuple(g.nE, g.nF, g.nH); })
      .def("invert", &TwoViewGeometry::Invert)
      .def("__repr__", [](const TwoViewGeometry& g) {
        return "TwoViewGeometry(config=" + py::str(py::cast(g.config).attr("name")).cast<std::string>() +
               ", num_inliers=" + std::to_string(g.inlier_matches.size() / 2) + ")";
      });

  // ---- pipelines ----
  m.def("match_exhaustive",
        [](const py::object& database_path, SiftMatchingOptions sift_options, ExhaustiveMatchingOptions matching_options,
           TwoViewGeometryOptions verification_options, Device device) {
          const std::string path = FsPath(database_path);
          CheckFileExists(path, "match_features.h:32");  // before the device check, R:match_features.h:32-38
          const std::vector<int> dev = ResolveDevices(device, sift_options);
          RunInterruptible([&] { MatchExhaustive(path, sift_options, matching_options, verification_options, dev); });
        },
        "database_path"_a, "sift_options"_a = SiftMatchingOptions(), "matching_options"_a = ExhaustiveMatchingOptions(),
        "verification_options"_a = TwoViewGeometryOptions(), "device"_a = Device::AUTO,
        "Exhaustive feature matching + geometric verification of every image pair of the database");
  m.def("match_sequential",
        [](const py::object& database_path, SiftMatchingOptions sift_options, SequentialMatchingOptions matching_options,
           TwoViewGeometryOptions verification_options, Device device) {
          const std::string path = FsPath(database_path);
          CheckFileExists(path, "match_features.h:32");  // before the device check, R:match_features.h:32-38
          const std::vector<int> dev = ResolveDevices(device, sift_options);
          RunInterruptible([&] { MatchSequential(path, sift_options, matching_options, verification_options, dev); });
        },
        "database_path"_a, "sift_options"_a = SiftMatchingOptions(), "matching_options"_a = SequentialMatchingOptions(),
        "verification_options"_a = TwoViewGeometryOptions(), "device"_a = Device::AUTO,
        "Sequential feature matching (images ordered by name; overlap / quadratic overlap)");
  m.def("match_spatial",
        [](const py::object& database_path, SiftMatchingOptions sift_options, SpatialMatchingOptions matching_options,
           TwoViewGeometryOptions verification_options, Device device) {
          const std::string path = FsPath(database_path);
          CheckFileExists(path, "match_features.h:32");
          const std::vector<int> dev = ResolveDevices(device, sift_options);
          RunInterruptible([&] { MatchSpatial(path, sift_options, matching_options, verification_options, dev); });
        },
        "database_path"_a, "sift_options"_a = SiftMatchingOptions(), "matching_options"_a = SpatialMatchingOptions(),
        "verification_options"_a = TwoViewGeometryOptions(), "device"_a = Device::AUTO,
        "Spatial feature matching (nearest neighbours by location prior)");
  m.def("match_vocabtree",
        [](const py::object&, const py::args&, const py::kwargs&) {
          throw std::invalid_argument("[bindings.cc] match_vocabtree needs a vocabulary tree index: out of scope (SURVEY.md section 8(f) item 4)");
        },
        "database_path"_a, "Not available: vocabulary-tree retrieval is outside the hot path this library covers.");
  m.def("verify_matches",
        [](const py::object& database_path, const py::object& pairs_path, TwoViewGeometryOptions options) {
          const std::string db = FsPath(database_path), pairs = FsPath(pairs_path);
          RunInterruptible([&] { VerifyMatches(db, pairs, options); });
        },
        "database_path"_a, "pairs_path"_a, "options"_a = TwoViewGeometryOptions(),
        "Run geometric verification of the matches of the listed pairs");

  // ---- estimators ----
  m.def("estimate_two_view_geometry",
        [](const py::object& camera1, const ArrD& points1, const py::object& camera2, const ArrD& points2,
           const py::object& matches, const TwoViewGeometryOptions& options) {
          return EstimateTvg([] { return Engine::Get(0); }, camera1, points1, camera2, points2, matches, options);
        },
        "camera1"_a, "points1"_a, "camera2"_a, "points2"_a, "matches"_a = py::none(),
        "options"_a = TwoViewGeometryOptions());
  m.def("estimate_calibrated_two_view_geometry",
        [](const py::object& camera1, const ArrD& points1, const py::object& camera2, const ArrD& points2,
           const py::object& matches, const TwoViewGeometryOptions& options) {
          // EstimateCalibratedTwoViewGeometry: the E branch runs whatever the prior flags say
          auto forced = [](const py::object& cam) {
            b2m_camera c = CameraFromPython(cam);
            return py::dict("model"_a = c.model, "width"_a = c.width, "height"_a = c.height,
                            "params"_a = std::vector<double>(c.params, c.params + b2m::cam::num_params(c.model)),
                            "has_prior_focal_length"_a = 1);
          };
          return EstimateTvg([] { return Engine::Get(0); }, forced(camera1), points1, forced(camera2), points2, matches, options);
        },
        "camera1"_a, "points1"_a, "camera2"_a, "points2"_a, "matches"_a = py::none(),
        "options"_a = TwoViewGeometryOptions());
  m.def("estimate_two_view_geometries",
        [](const py::list& problems, const TwoViewGeometryOptions& options) {
          // Batched estimate_two_view_geometry (SURVEY.md section 8(f) item 3): every problem is a tuple
          // (camera1, points1, camera2, points2[, matches]); one GPU launch verifies them all.
          const size_t n = problems.size();
          std::vector<ArrD> p1(n), p2(n);
          std::vector<ArrU32> mm(n);
          std::vector<b2m_tvg_problem> q(n);
          std::vector<std::vector<uint32_t>> inl(n);
          std::vector<uint32_t*> inl_ptr(n);
          for (size_t k = 0; k < n; ++k) {
            const py::tuple t = py::tuple(problems[k]);
            if (t.size() != 4 && t.size() != 5)
              throw std::invalid_argument("[bindings.cc] Check Failed: problem = (camera1, points1, camera2, points2[, matches])");
            p1[k] = ArrD::ensure(t[1]);
            p2[k] = ArrD::ensure(t[3]);
            if (!p1[k] || !p2[k]) throw std::invalid_argument("[bindings.cc] Check Failed: points are N x 2 float64 arrays");
            CheckPoints(p1[k], "points1");
            CheckPoints(p2[k], "points2");
            memset(&q[k], 0, sizeof(q[k]));
            q[k].struct_size = sizeof(q[k]);
            q[k].cam1 = CameraFromPython(py::reinterpret_borrow<py::object>(t[0]));
            q[k].cam2 = CameraFromPython(py::reinterpret_borrow<py::object>(t[2]));
            q[k].points1 = p1[k].data();
            q[k].n1 = p1[k].shape(0);
            q[k].points2 = p2[k].data();
            q[k].n2 = p2[k].shape(0);
            int64_t m = q[k].n1;
            if (t.size() == 5 && !t[4].is_none()) {
              mm[k] = ArrU32::ensure(t[4]);
              if (!mm[k] || mm[k].ndim() != 2 || mm[k].shape(1) != 2)
                throw std::invalid_argument("[bindings.cc] Check Failed: matches is an N x 2 uint32 array");
              q[k].matches = mm[k].data();
              q[k].m = m = mm[k].shape(0);
            } else if (q[k].n1 != q[k].n2) {
              throw std::invalid_argument("[two_view_geometry.h:137] Check Failed: points1.size() == points2.size()");
            }
            inl[k].resize(static_cast<size_t>(std::max<int64_t>(1, m)) * 2);
            inl_ptr[k] = inl[k].data();
          }
          const b2m_tvg_opts opts = ToAbi(options);
          std::vector<b2m_tvg_result> r(n);
          b2m_ctx* ctx = Engine::Get(0);
          int rc;
          {
            py::gil_scoped_release release;
            rc = b2m_estimate_two_view_geometry_batch(ctx, q.data(), static_cast<int64_t>(n), &opts, r.data(), inl_ptr.data());
          }
          ThrowOnError(ctx, rc);
          std::vector<TwoViewGeometry> out(n);
          for (size_t k = 0; k < n; ++k) {
            out[k].config = static_cast<TwoViewGeometryConfiguration>(r[k].config);
            std::copy(r[k].E, r[k].E + 9, out[k].E.begin());
            std::copy(r[k].F, r[k].F + 9, out[k].F.begin());
            std::copy(r[k].H, r[k].H + 9, out[k].H.begin());
            inl[k].resize(static_cast<size_t>(r[k].n_inliers) * 2);
            out[k].inlier_matches = std::move(inl[k]);
            out[k].nE = r[k].nE; out[k].nF = r[k].nF; out[k].nH = r[k].nH;
            std::copy(r[k].qvec, r[k].qvec + 4, out[k].qvec.begin());
            std::copy(r[k].tvec, r[k].tvec + 3, out[k].tvec.begin());
            out[k].tri_angle = r[k].tri_angle;
          }
          return out;
        },
        "problems"_a, "options"_a = TwoViewGeometryOptions(),
        "Batched estimate_two_view_geometry: problems = [(camera1, points1, camera2, points2[, matches]), ...]");
  m.def("estimate_two_view_geometry_pose",
        [](const py::object& camera1, const ArrD& points1, const py::object& camera2, const ArrD& points2, TwoViewGeometry& geometry) {
          CheckPoints(points1, "points1");
          CheckPoints(points2, "points2");
          const b2m_camera c1 = CameraFromPython(camera1), c2 = CameraFromPython(camera2);
          b2m_tvg_result g;
          memset(&g, 0, sizeof(g));
          g.struct_size = sizeof(g);
          g.config = static_cast<int>(geometry.config);
          std::copy(geometry.E.begin(), geometry.E.end(), g.E);
          std::copy(geometry.H.begin(), geometry.H.end(), g.H);
          b2m_ctx* ctx = Engine::Get(0);
          ThrowOnError(ctx, b2m_estimate_two_view_geometry_pose(ctx, &c1, points1.data(), points1.shape(0), &c2, points2.data(),
                                                               points2.shape(0), geometry.inlier_matches.data(),
                                                               static_cast<int64_t>(geometry.inlier_matches.size() / 2), &g));
          if (!g.pose_valid) return false;
          geometry.config = static_cast<TwoViewGeometryConfiguration>(g.config);
          std::copy(g.qvec, g.qvec + 4, geometry.qvec.begin());
          std::copy(g.tvec, g.tvec + 3, geometry.tvec.begin());
          geometry.tri_angle = g.tri_angle;
          return true;
        },
        "camera1"_a, "points1"_a, "camera2"_a, "points2"_a, "geometry"_a,
        "Relative pose of an estimated geometry, in place (R:estimators/two_view_geometry.h:153-158).");
  // ---- absolute pose ----
  OptionsClass<AbsolutePoseEstimationOptions>(m, "AbsolutePoseEstimationOptions")
      .field("estimate_focal_length", &AbsolutePoseEstimationOptions::estimate_focal_length)
      .field("num_focal_length_samples", &AbsolutePoseEstimationOptions::num_focal_length_samples)
      .field("min_focal_length_ratio", &AbsolutePoseEstimationOptions::min_focal_length_ratio)
      .field("max_focal_length_ratio", &AbsolutePoseEstimationOptions::max_focal_length_ratio)
      .field("ransac", &AbsolutePoseEstimationOptions::ransac)
      .Finish();
  OptionsClass<AbsolutePoseRefinementOptions>(m, "AbsolutePoseRefinementOptions")
      .field("gradient_tolerance", &AbsolutePoseRefinementOptions::gradient_tolerance)
      .field("max_num_iterations", &AbsolutePoseRefinementOptions::max_num_iterations)
      .field("loss_function_scale", &AbsolutePoseRefinementOptions::loss_function_scale)
      .field("refine_focal_length", &AbsolutePoseRefinementOptions::refine_focal_length)
      .field("refine_extra_params", &AbsolutePoseRefinementOptions::refine_extra_params)
      .field("print_summary", &AbsolutePoseRefinementOptions::print_summary)
      .Finish();
  m.def("absolute_pose_estimation",
        [m](const ArrD& points2D, const ArrD& points3D, const py::object& camera,
            const AbsolutePoseEstimationOptions& estimation_options, const AbsolutePoseRefinementOptions& refinement_options,
            bool return_covariance) {
          CheckAbsPoints(points2D, points3D);
          const b2m_camera c = CameraFromPython(camera);
          std::vector<b2m_abs_pose_problem> q{AbsProblem(c, points2D, points3D)};
          std::vector<b2m_abs_pose_result> r;
          std::vector<std::vector<uint8_t>> masks;
          EstimateAbsolutePoses(Engine::Get(0), q, estimation_options, refinement_options, return_covariance, &r, &masks);
          // the camera changes when the estimator scaled its focal length (EstimateAbsolutePose found inliers) or when
          // RefineAbsolutePose, which runs after every such estimate, refined camera parameters
          const bool estimated = r[0].focal_sample >= 0;
          const bool refines = refinement_options.refine_focal_length || refinement_options.refine_extra_params;
          if (estimated && (estimation_options.estimate_focal_length || refines))
            WriteCameraParams(camera, r[0], c.model);
          return AbsResultToPython(m, r[0], masks[0], q[0].n, return_covariance);
        },
        "points2D"_a, "points3D"_a, "camera"_a, "estimation_options"_a = AbsolutePoseEstimationOptions(),
        "refinement_options"_a = AbsolutePoseRefinementOptions(), "return_covariance"_a = false,
        "Absolute pose estimation with non-linear refinement.");
  m.def("estimate_absolute_poses",
        [m](const py::list& problems, const AbsolutePoseEstimationOptions& estimation_options,
            const AbsolutePoseRefinementOptions& refinement_options, bool return_covariance) {
          // Batched absolute_pose_estimation: problems = [(camera, points2D, points3D), ...], one GPU launch for all.
          // Cameras are not modified; a successful result carries "camera_params" (the parameters after the call).
          const size_t n = problems.size();
          std::vector<ArrD> p2(n), p3(n);
          std::vector<b2m_abs_pose_problem> q(n);
          for (size_t k = 0; k < n; ++k) {
            const py::tuple t = py::tuple(problems[k]);
            if (t.size() != 3) throw std::invalid_argument("[bindings.cc] Check Failed: problem = (camera, points2D, points3D)");
            p2[k] = ArrD::ensure(t[1]);
            p3[k] = ArrD::ensure(t[2]);
            if (!p2[k] || !p3[k]) throw std::invalid_argument("[bindings.cc] Check Failed: points are float64 arrays");
            CheckAbsPoints(p2[k], p3[k]);
            q[k] = AbsProblem(CameraFromPython(py::reinterpret_borrow<py::object>(t[0])), p2[k], p3[k]);
          }
          std::vector<b2m_abs_pose_result> r;
          std::vector<std::vector<uint8_t>> masks;
          EstimateAbsolutePoses(Engine::Get(0), q, estimation_options, refinement_options, return_covariance, &r, &masks);
          py::list out;
          for (size_t k = 0; k < n; ++k) {
            py::object o = AbsResultToPython(m, r[k], masks[k], q[k].n, return_covariance);
            if (!o.is_none()) {
              const int np = b2m::cam::num_params(q[k].camera.model);
              o.attr("__setitem__")("camera_params", py::array_t<double>(np, r[k].params));
            }
            out.append(o);
          }
          return out;
        },
        "problems"_a, "estimation_options"_a = AbsolutePoseEstimationOptions(),
        "refinement_options"_a = AbsolutePoseRefinementOptions(), "return_covariance"_a = false,
        "Batched absolute_pose_estimation: problems = [(camera, points2D, points3D), ...]");
  m.def("pose_refinement",
        [m](const py::object& cam_from_world, const ArrD& points2D, const ArrD& points3D, const py::object& inlier_mask,
            const py::object& camera, const AbsolutePoseRefinementOptions& refinement_options) {
          CheckAbsPoints(points2D, points3D);
          const py::array_t<bool, py::array::c_style | py::array::forcecast> mask =
              py::array_t<bool, py::array::c_style | py::array::forcecast>::ensure(inlier_mask);
          if (!mask || mask.ndim() != 1 || mask.shape(0) != points2D.shape(0))  // R:absolute_pose.h:75
            throw std::invalid_argument("[absolute_pose.h:75] Check Failed: inlier_mask.size() == points2D.size()");
          const b2m_camera c = CameraFromPython(camera);
          const py::array_t<double> quat = py::array_t<double>::ensure(cam_from_world.attr("rotation").attr("quat"));
          const py::array_t<double> tr = py::array_t<double>::ensure(cam_from_world.attr("translation"));
          if (!quat || quat.size() != 4 || !tr || tr.size() != 3)
            throw std::invalid_argument("[bindings.cc] Check Failed: cam_from_world is a Rigid3d");
          const double init[7] = {quat.data()[3], quat.data()[0], quat.data()[1], quat.data()[2], tr.data()[0], tr.data()[1],
                                  tr.data()[2]};
          std::vector<uint8_t> m8(static_cast<size_t>(std::max<py::ssize_t>(mask.shape(0), 1)), 0);
          for (py::ssize_t i = 0; i < mask.shape(0); ++i) m8[i] = mask.data()[i] ? 1 : 0;
          const uint8_t* mp = m8.data();
          const b2m_abs_pose_problem q = AbsProblem(c, points2D, points3D);
          const b2m_pose_refine_opts f = ToAbi(refinement_options);
          b2m_abs_pose_result r;
          const AbsPoseApi& api = AbsPose();
          b2m_ctx* ctx = Engine::Get(0);
          int rc;
          {
            py::gil_scoped_release release;
            rc = api.refine(ctx, &q, 1, init, &mp, &f, 0, &r);
          }
          ThrowOnError(ctx, rc);
          if (refinement_options.refine_focal_length || refinement_options.refine_extra_params) WriteCameraParams(camera, r, c.model);
          if (!r.success) return py::object(py::none());
          py::dict d;
          d["cam_from_world"] = PoseToPython(m, r.qvec, r.tvec);
          return py::object(d);
        },
        "cam_from_world"_a, "points2D"_a, "points3D"_a, "inlier_mask"_a, "camera"_a,
        "refinement_options"_a = AbsolutePoseRefinementOptions(), "Non-linear refinement of absolute pose.");
  // ---- triangulation ----
  py::class_<PointData>(m, "PointData")
      .def(py::init([](const std::array<double, 2>& point, const std::array<double, 2>& point_normalized) {
             return PointData{point, point_normalized};
           }),
           "point"_a, "point_normalized"_a)
      .def_property_readonly("point", [](const PointData& d) { return py::array_t<double>(2, d.point.data()); })
      .def_property_readonly("point_normalized",
                             [](const PointData& d) { return py::array_t<double>(2, d.point_normalized.data()); })
      .def("__repr__", [](const PointData& d) {
        return "PointData(point=[" + std::to_string(d.point[0]) + ", " + std::to_string(d.point[1]) +
               "], point_normalized=[" + std::to_string(d.point_normalized[0]) + ", " +
               std::to_string(d.point_normalized[1]) + "])";
      });
  OptionsClass<EstimateTriangulationOptions>(m, "EstimateTriangulationOptions")
      .field("min_tri_angle", &EstimateTriangulationOptions::min_tri_angle, "Minimum triangulation angle in radians.")
      .field("ransac", &EstimateTriangulationOptions::ransac, "RANSAC options; max_error is an angle in radians.")
      .Finish();
  m.def("estimate_triangulation",
        [](const py::list& point_data, const py::list& images, const py::list& cameras,
           const EstimateTriangulationOptions& opions) {
          const size_t n = images.size();
          if (cameras.size() != n)  // THROW_CHECK_EQ(images.size(), cameras.size()), R:triangulation.h
            throw std::invalid_argument("[triangulation.h] Check Failed: images.size() == cameras.size() (" +
                                        std::to_string(n) + " vs. " + std::to_string(cameras.size()) + ")");
          if (point_data.size() != n)
            throw std::invalid_argument("[triangulation.h] Check Failed: images.size() == point_data.size() (" +
                                        std::to_string(n) + " vs. " + std::to_string(point_data.size()) + ")");
          CheckTriOptions(opions);
          if (n < 2) throw std::invalid_argument("[triangulation.cc] Check Failed: point_data.size() >= 2");
          std::vector<double> pts(2 * n), cams(12 * n);
          std::vector<int32_t> img(n);
          for (size_t i = 0; i < n; ++i) {
            CameraFromPython(py::reinterpret_borrow<py::object>(cameras[i]));  // validates; the angular residual does not use it
            const PointData d = point_data[i].cast<PointData>();
            pts[2 * i] = d.point_normalized[0];
            pts[2 * i + 1] = d.point_normalized[1];
            const std::array<double, 12> P = ImagePoseMatrix(images[i]);
            std::copy(P.begin(), P.end(), cams.begin() + 12 * i);
            img[i] = static_cast<int32_t>(i);
          }
          const std::vector<int64_t> off{0, static_cast<int64_t>(n)};
          const TriBatchOut r =
              EstimateTriangulationsAbi(Engine::Get(0), off, pts.data(), img.data(), static_cast<int32_t>(n), cams.data(), opions);
          if (!r.success[0]) return py::object(py::none());
          py::dict d;
          d["xyz"] = py::array_t<double>(3, r.xyz.data());
          d["inliers"] = MaskToNumpy(r.mask, static_cast<int64_t>(n));
          return py::object(d);
        },
        "point_data"_a, "images"_a, "cameras"_a, "opions"_a = EstimateTriangulationOptions(),
        "Robustly triangulate one track from its observations (the options keyword is spelled `opions`, as in pycolmap).");
  m.def("estimate_triangulations",
        [](const py::object& points_normalized, const py::object& track_lengths, const py::object& image_idxs,
           const py::object& cams_from_world, const EstimateTriangulationOptions& options) {
          return EstimateTriangulationsPy([] { return Engine::Get(0); }, points_normalized, track_lengths, image_idxs,
                                          cams_from_world, options);
        },
        "points_normalized"_a, "track_lengths"_a, "image_idxs"_a, "cams_from_world"_a,
        "options"_a = EstimateTriangulationOptions(),
        "Batched estimate_triangulation over T tracks stored back to back: returns dict(xyz (T, 3), NaN rows on failure; "
        "success (T,); num_inliers (T,); inliers (M,))");
  // ---- SIFT extraction ----
  auto normalization = py::enum_<Normalization>(m, "Normalization")
                           .value("L1_ROOT", Normalization::L1_ROOT,
                                  "L1-normalizes each descriptor followed by element-wise square rooting.")
                           .value("L2", Normalization::L2, "Each vector is L2-normalized.");
  AddStringConstructor(normalization);
  OptionsClass<SiftExtractionOptions>(m, "SiftExtractionOptions")
      .field("num_threads", &SiftExtractionOptions::num_threads, "Number of threads (accepted; extraction runs on the GPU).")
      .field("gpu_index", &SiftExtractionOptions::gpu_index, "Index of the GPU used for feature extraction (one index).")
      .field("max_image_size", &SiftExtractionOptions::max_image_size,
             "Maximum image size; Sift.extract refuses larger images (it does not resize).")
      .field("max_num_features", &SiftExtractionOptions::max_num_features,
             "Maximum number of features to detect, keeping larger-scale features.")
      .field("first_octave", &SiftExtractionOptions::first_octave,
             "First octave in the pyramid, i.e. -1 upsamples the image by one level.")
      .field("num_octaves", &SiftExtractionOptions::num_octaves)
      .field("octave_resolution", &SiftExtractionOptions::octave_resolution, "Number of levels per octave.")
      .field("peak_threshold", &SiftExtractionOptions::peak_threshold, "Peak threshold for detection.")
      .field("edge_threshold", &SiftExtractionOptions::edge_threshold, "Edge threshold for detection.")
      .field("estimate_affine_shape", &SiftExtractionOptions::estimate_affine_shape,
             "Estimate affine shape of SIFT features (not supported: True is refused).")
      .field("max_num_orientations", &SiftExtractionOptions::max_num_orientations,
             "Maximum number of orientations per keypoint.")
      .field("upright", &SiftExtractionOptions::upright, "Fix the orientation to 0 for upright features")
      .field("darkness_adaptivity", &SiftExtractionOptions::darkness_adaptivity,
             "SiftGPU-only upstream (not supported: True is refused).")
      .field("domain_size_pooling", &SiftExtractionOptions::domain_size_pooling,
             "Domain-size pooling (not supported: True is refused).")
      .field("dsp_min_scale", &SiftExtractionOptions::dsp_min_scale)
      .field("dsp_max_scale", &SiftExtractionOptions::dsp_max_scale)
      .field("dsp_num_scales", &SiftExtractionOptions::dsp_num_scales)
      .field("normalization", &SiftExtractionOptions::normalization, "L1_ROOT or L2 descriptor normalization")
      .Finish();
  {
    SiftExtractionOptions pycolmap_defaults;  // R:pycolmap/feature/sift.h:99-102
    pycolmap_defaults.peak_threshold = 0.01;
    pycolmap_defaults.first_octave = 0;
    pycolmap_defaults.max_image_size = 7000;
    py::class_<Sift>(m, "Sift")
        .def(py::init([](const SiftExtractionOptions& options, Device device) {
               CheckSiftOptions(options);
               SiftDevice(device, options);
               return Sift{options, device};
             }),
             "options"_a = pycolmap_defaults, "device"_a = Device::AUTO)
        .def("extract",
             [](const Sift& s, const py::object& image) {
               py::list one;
               one.append(image);
               const py::list r = ExtractBatch(s, one);
               return py::object(r[0]);
             },
             "image"_a,
             "SIFT features of a 2-D uint8 or float32 image: (keypoints (N, 4) [x, y, scale, orientation], "
             "descriptors (N, 128) float32 = uint8 / 512)")
        .def("extract_batch", &ExtractBatch, "images"_a,
             "Sift.extract over a list of images in one GPU call; a list of (keypoints, descriptors)")
        .def_property_readonly("options", [](const Sift& s) { return s.options; })
        .def_property_readonly(
            "device", [](const Sift&) { return Device::CUDA; },
            "The device the extractor runs on, resolved like upstream's Sift::GetDevice (use_gpu ? CUDA : CPU): always "
            "Device.cuda, since Device.auto resolves to the GPU and Device.cpu is refused.");
  }
  // ---- feature extraction from image files ----
  auto camera_mode = py::enum_<CameraMode>(m, "CameraMode")
                         .value("AUTO", CameraMode::AUTO)
                         .value("SINGLE", CameraMode::SINGLE)
                         .value("PER_FOLDER", CameraMode::PER_FOLDER)
                         .value("PER_IMAGE", CameraMode::PER_IMAGE);
  AddStringConstructor(camera_mode);
  OptionsClass<ImageReaderOptions>(m, "ImageReaderOptions")
      .field("camera_model", &ImageReaderOptions::camera_model, "Name of the camera model.")
      .field("mask_path", &ImageReaderOptions::mask_path,
             "Optional root path to folder which contains image masks: the mask of image_path/abc/012.jpg is "
             "mask_path/abc/012.jpg.png.  No features are kept where the mask is black (grey value 0).")
      .field("existing_camera_id", &ImageReaderOptions::existing_camera_id,
             "Use this existing camera for all images (the camera model and parameters are then ignored).")
      .field("camera_params", &ImageReaderOptions::camera_params,
             "Manual specification of camera parameters.  If empty, they come from EXIF (focal length) and the "
             "image size (principal point).")
      .field("default_focal_length_factor", &ImageReaderOptions::default_focal_length_factor,
             "Without manual parameters or an EXIF focal length, the focal length is "
             "default_focal_length_factor * max(width, height).")
      .field("camera_mask_path", &ImageReaderOptions::camera_mask_path,
             "Optional mask for all images: no features are kept where it is black (grey value 0).")
      .Finish();
  {
    SiftExtractionOptions cxx_defaults;  // the C++ constructor's (R:pipeline/extract_features.h:140), not Sift()'s
    m.def("extract_features",
          [](const py::object& database_path, const py::object& image_path, const std::vector<std::string>& image_list,
             CameraMode camera_mode, const std::string& camera_model, ImageReaderOptions reader_options,
             const SiftExtractionOptions& sift_options, Device device) {
            const std::string db = FsPath(database_path), images = FsPath(image_path);
            if (std::filesystem::exists(db)) CheckFailed("extract_features.h:31", "!ExistsFile(database_path)", db + " already exists.");
            if (!(db.size() >= 3 && db.compare(db.size() - 3, 3, ".db") == 0))
              CheckFailed("extract_features.h:33", "HasFileExtension(database_path, \".db\")",
                          "Path " + db + " does not match file extension .db.");
            if (!std::ofstream(db, std::ios::trunc).is_open())
              CheckFailed("extract_features.h:34", "std::ofstream(database_path, std::ios::trunc).is_open()",
                          ": Could not open " + db + ". Is the path a directory or does the parent dir not exist?");
            if (!IsDir(images)) CheckFailed("extract_features.h:35", "ExistsDir(image_path)", "Directory " + images + " does not exist.");
            const int dev = SiftDevice(device, sift_options);
            reader_options.camera_model = camera_model;
            if (CameraModelId(camera_model) < 0)
              CheckFailed("extract_features.h:49", "ExistsCameraModelWithName(reader_options.camera_model)", "");
            if (!VerifyCameraParams(camera_model, reader_options.camera_params))
              throw std::invalid_argument("[extract_features.h:51] Invalid camera parameters.");
            CheckSiftOptions(sift_options);
            RunInterruptible([&] { ExtractFeaturesRun(db, images, image_list, camera_mode, reader_options, sift_options, dev); });
          },
          "database_path"_a, "image_path"_a, "image_list"_a = std::vector<std::string>(), "camera_mode"_a = CameraMode::AUTO,
          "camera_model"_a = "SIMPLE_RADIAL", "reader_options"_a = ImageReaderOptions(), "sift_options"_a = cxx_defaults,
          "device"_a = Device::AUTO,
          "Extract SIFT features of the JPEG / PNG files under image_path and write cameras, images, keypoints and "
          "descriptors to a new database");
  }
  OptionsClass<PatchMatchOptions>(m, "PatchMatchOptions")
      .field("max_image_size", &PatchMatchOptions::max_image_size,
             "Maximum image size in either dimension; larger images are downscaled (-1: no limit).")
      .field("gpu_index", &PatchMatchOptions::gpu_index, "Index of the GPU used for patch match (one index; -1: device 0).")
      .field("depth_min", &PatchMatchOptions::depth_min, "Minimum depth (-1: from the sparse points of each image).")
      .field("depth_max", &PatchMatchOptions::depth_max, "Maximum depth (-1: from the sparse points of each image).")
      .field("window_radius", &PatchMatchOptions::window_radius, "Half window size to compute NCC photo-consistency cost.")
      .field("window_step", &PatchMatchOptions::window_step, "Number of pixels to skip when computing NCC (1 or 2).")
      .field("sigma_spatial", &PatchMatchOptions::sigma_spatial,
             "Spatial sigma for bilaterally weighted NCC (-1: window_radius).")
      .field("sigma_color", &PatchMatchOptions::sigma_color, "Color sigma for bilaterally weighted NCC.")
      .field("num_samples", &PatchMatchOptions::num_samples, "Number of random samples to draw in Monte Carlo sampling.")
      .field("ncc_sigma", &PatchMatchOptions::ncc_sigma, "Spread of the NCC likelihood function.")
      .field("min_triangulation_angle", &PatchMatchOptions::min_triangulation_angle,
             "Minimum triangulation angle in degrees.")
      .field("incident_angle_sigma", &PatchMatchOptions::incident_angle_sigma,
             "Spread of the incident angle likelihood function.")
      .field("num_iterations", &PatchMatchOptions::num_iterations, "Number of coordinate descent iterations.")
      .field("geom_consistency", &PatchMatchOptions::geom_consistency,
             "Whether to add a regularized geometric consistency term to the cost function.")
      .field("geom_consistency_regularizer", &PatchMatchOptions::geom_consistency_regularizer,
             "The relative weight of the geometric consistency term w.r.t. the photo-consistency term.")
      .field("geom_consistency_max_cost", &PatchMatchOptions::geom_consistency_max_cost,
             "Maximum geometric consistency cost in terms of the forward-backward reprojection error in pixels.")
      .field("filter", &PatchMatchOptions::filter, "Whether to enable filtering.")
      .field("filter_min_ncc", &PatchMatchOptions::filter_min_ncc, "Minimum NCC coefficient for pixel to be photo-consistent.")
      .field("filter_min_triangulation_angle", &PatchMatchOptions::filter_min_triangulation_angle,
             "Minimum triangulation angle to be stable.")
      .field("filter_min_num_consistent", &PatchMatchOptions::filter_min_num_consistent,
             "Minimum number of source images have to be consistent for pixel not to be filtered.")
      .field("filter_geom_consistency_max_cost", &PatchMatchOptions::filter_geom_consistency_max_cost,
             "Maximum forward-backward reprojection error for pixel to be geometrically consistent.")
      .field("cache_size", &PatchMatchOptions::cache_size,
             "Cache size in gigabytes for patch match.  Checked and otherwise without effect: every image of the "
             "workspace is decoded once per call and held on the GPU.")
      .field("allow_missing_files", &PatchMatchOptions::allow_missing_files,
             "Whether to tolerate missing images/maps in the problem setup (skipped with a warning).")
      .field("write_consistency_graph", &PatchMatchOptions::write_consistency_graph,
             "Whether to write the consistency graph (not supported: True is refused).")
      .Finish();
  m.def("_check_patch_match_options", [](const PatchMatchOptions& o) {
    CheckPatchMatchOptions(o);
    return PatchMatchDevice(o);
  });
  m.def("_patch_match_run",
        [](const py::list& images, const ArrD& cameras, const py::object& depth_maps, const py::list& problems,
           const PatchMatchOptions& options, bool geom, bool filter) {
          return PatchMatchRun(Engine::Get(PatchMatchDevice(options)), images, cameras, depth_maps, problems, options, geom,
                               filter);
        },
        "images"_a, "cameras"_a, "depth_maps"_a, "problems"_a, "options"_a, "geom"_a, "filter"_a,
        "One PatchMatch device call (pycolmap_b200.mvs): [(depth (H, W), normal (H, W, 3))] per problem");
  m.def("_patch_match_stats",
        [](int device) {
          b2m_ctx* ctx = Engine::Get(device);
          b2m_stats st;
          std::memset(&st, 0, sizeof(st));
          st.struct_size = sizeof(st);
          ThrowOnError(ctx, b2m_get_stats(ctx, &st));
          return py::dict("pm_problems"_a = st.pm_problems, "pm_pixel_updates"_a = st.pm_pixel_updates,
                          "pm_window_samples"_a = st.pm_window_samples, "kernel_launches"_a = st.kernel_launches);
        },
        "device"_a = 0, "The PatchMatch counters of the context patch_match_stereo uses on this device (since it was created)");
  m.def("debug_patch_match_cost",
        [](const py::list& images, const ArrD& cameras, const py::object& depth_maps, const py::dict& problem,
           const ArrF32& queries, const PatchMatchOptions& options) {
          CheckPatchMatchOptions(options);
          PmInputs in;
          py::list one;
          one.append(problem);
          LoadPmInputs(images, cameras, depth_maps, one, &in);
          if (queries.ndim() != 2 || queries.shape(1) != 7)
            throw std::invalid_argument("[bindings.cc] Check Failed: queries is an n x 7 float32 array");
          b2m_ctx* ctx = Engine::Get(PatchMatchDevice(options));
          const auto set = SiftSymbol<decltype(&b2m_patch_match_set_images)>("b2m_patch_match_set_images");
          const auto cost = SiftSymbol<decltype(&b2m_debug_patch_match_cost)>("b2m_debug_patch_match_cost");
          ThrowOnError(ctx, set(ctx, static_cast<int32_t>(in.ims.size()), in.ims.data(), in.cameras.data(),
                                in.dmap_ptrs.empty() ? nullptr : in.dmap_ptrs.data()));
          const b2m_patch_match_opts o = ToAbi(options, false, false);
          py::array_t<float> out(std::vector<py::ssize_t>{queries.shape(0), 3});
          ThrowOnError(ctx, cost(ctx, &in.probs[0], &o, queries.data(), static_cast<int32_t>(queries.shape(0)),
                                 out.mutable_data()));
          return out;
        },
        "images"_a, "cameras"_a, "depth_maps"_a, "problem"_a, "queries"_a, "options"_a,
        "Instrumentation: K8's cost arithmetic, [n x 3] = (photometric cost, geometric cost, depth of the plane at "
        "(x, y + 1)) for queries [n x 7] = (x, y, depth, nx, ny, nz, source slot)");
  OptionsClass<StereoFusionOptions>(m, "StereoFusionOptions")
      .field("mask_path", &StereoFusionOptions::mask_path,
             "Path for PNG masks. Same format expected as ImageReaderOptions.")
      .field("num_threads", &StereoFusionOptions::num_threads, "The number of threads to use during fusion (no effect).")
      .field("max_image_size", &StereoFusionOptions::max_image_size,
             "Maximum image size in either dimension (images larger than it are refused).")
      .field("min_num_pixels", &StereoFusionOptions::min_num_pixels, "Minimum number of fused pixels to produce a point.")
      .field("max_num_pixels", &StereoFusionOptions::max_num_pixels,
             "Maximum number of pixels to fuse into a single point.")
      .field("max_traversal_depth", &StereoFusionOptions::max_traversal_depth,
             "Maximum depth in consistency graph traversal.")
      .field("max_reproj_error", &StereoFusionOptions::max_reproj_error, "Maximum relative difference between measured and projected pixel.")
      .field("max_depth_error", &StereoFusionOptions::max_depth_error, "Maximum relative difference between measured and projected depth.")
      .field("max_normal_error", &StereoFusionOptions::max_normal_error, "Maximum angular difference in degrees of normals of pixels to be fused.")
      .field("check_num_images", &StereoFusionOptions::check_num_images,
             "Number of overlapping images to transitively check for fusing points.")
      .field("use_cache", &StereoFusionOptions::use_cache, "Flag indicating whether to use LRU cache or pre-load all data (no effect).")
      .field("cache_size", &StereoFusionOptions::cache_size, "Maximum cache size in gigabytes (no effect).")
      .field("bounding_box", &StereoFusionOptions::bounding_box, "Bounding box Tuple[min, max]")
      .Finish();
  m.def("_check_stereo_fusion_options", [](const StereoFusionOptions& o) { CheckStereoFusionOptions(o); });
  m.def("_stereo_fusion_run",
        [](const py::list& images, const StereoFusionOptions& options, int device) {
          return StereoFusionRun(Engine::Get(device), images, options);
        },
        "images"_a, "options"_a, "device"_a = 0, "One stereo fusion device call (pycolmap_b200.mvs)");
  m.def("_stereo_fusion_stats",
        [](int device) {
          b2m_stats st;
          std::memset(&st, 0, sizeof(st));
          st.struct_size = sizeof(st);
          b2m_ctx* ctx = Engine::Get(device);
          ThrowOnError(ctx, b2m_get_stats(ctx, &st));
          return py::dict("fusion_seeds"_a = st.fusion_seeds, "fusion_traversals"_a = st.fusion_traversals,
                          "fusion_pops"_a = st.fusion_pops, "fusion_rounds"_a = st.fusion_rounds,
                          "fusion_deferred"_a = st.fusion_deferred, "fusion_points"_a = st.fusion_points,
                          "kernel_launches"_a = st.kernel_launches);
        },
        "device"_a = 0, "The stereo fusion counters of the context stereo_fusion uses on this device (since it was created)");
  OptionsClass<UndistortCameraOptions>(m, "UndistortCameraOptions")
      .field("blank_pixels", &UndistortCameraOptions::blank_pixels,
             "The amount of blank pixels in the undistorted image in the range [0, 1].")
      .field("min_scale", &UndistortCameraOptions::min_scale, "Minimum scale change of camera used to satisfy the blank pixel constraint.")
      .field("max_scale", &UndistortCameraOptions::max_scale, "Maximum scale change of camera used to satisfy the blank pixel constraint.")
      .field("max_image_size", &UndistortCameraOptions::max_image_size,
             "Maximum image size in terms of width or height of the undistorted camera.")
      .field("roi_min_x", &UndistortCameraOptions::roi_min_x, "The 4 factors in the range [0, 1] that define the ROI (region of interest) in original image. The bounding box pixel coordinates are calculated as (roi_min_x * Width, roi_min_y * Height) and (roi_max_x * Width, roi_max_y * Height).")
      .field("roi_min_y", &UndistortCameraOptions::roi_min_y)
      .field("roi_max_x", &UndistortCameraOptions::roi_max_x)
      .field("roi_max_y", &UndistortCameraOptions::roi_max_y)
      .Finish();
  auto copy_type = py::enum_<CopyType>(m, "CopyType")
                       .value("copy", CopyType::COPY)
                       .value("soft-link", CopyType::SOFT_LINK)
                       .value("hard-link", CopyType::HARD_LINK);
  copy_type.def(py::init([](const std::string& name) {
                  if (name == "copy") return CopyType::COPY;
                  if (name == "soft-link") return CopyType::SOFT_LINK;
                  if (name == "hard-link") return CopyType::HARD_LINK;
                  throw std::invalid_argument("Invalid string value " + name + " for enum CopyType");
                }),
                "name"_a);
  py::implicitly_convertible<std::string, CopyType>();
  m.def("_check_undistort_options", [](const UndistortCameraOptions& o) { CheckUndistortOptions(o); });
  m.def("_undistort_camera", &UndistortCameraPy, "options"_a, "camera"_a,
        "UndistortCamera on the host: the PINHOLE camera (dict) of the undistorted image");
  m.def("_undistort_run",
        [](const py::list& items, const UndistortCameraOptions& options, int device) {
          return UndistortRun(Engine::Get(device), items, options);
        },
        "items"_a, "options"_a, "device"_a = 0, "One undistortion device call (pycolmap_b200.mvs)");
  m.def("_undistort_stats",
        [](int device) {
          b2m_stats st;
          std::memset(&st, 0, sizeof(st));
          st.struct_size = sizeof(st);
          b2m_ctx* ctx = Engine::Get(device);
          ThrowOnError(ctx, b2m_get_stats(ctx, &st));
          return py::dict("undistort_images"_a = st.undistort_images, "undistort_pixels"_a = st.undistort_pixels,
                          "undistort_encoded_bytes"_a = st.undistort_encoded_bytes, "kernel_launches"_a = st.kernel_launches);
        },
        "device"_a = 0, "The undistortion counters of the context undistort_images uses on this device");
  m.def("debug_undistort_pixels",
        [](const py::bytes& file, const py::object& camera, const UndistortCameraOptions& options, int device) {
          CheckUndistortOptions(options);
          const std::string buf = file;
          const std::vector<uint8_t> bytes(buf.begin(), buf.end());
          Pixels px;
          std::string why;
          b2m_undistort_item it;
          std::memset(&it, 0, sizeof(it));
          it.struct_size = sizeof(it);
          it.output = B2M_UNDISTORT_PIXELS;
          it.camera = CameraFromPython(camera);
          if (!SourceFromFile(bytes, &px, &it.source, &why)) throw std::invalid_argument("[bindings.cc] " + why);
          const b2m_undistort_opts o = ToAbi(options);
          const auto dbg = SiftSymbol<decltype(&b2m_debug_undistort_pixels)>("b2m_debug_undistort_pixels");
          b2m_ctx* ctx = Engine::Get(device);
          int32_t w = 0, h = 0;
          ThrowOnError(ctx, dbg(ctx, &it, &o, nullptr, &w, &h));
          py::array_t<uint8_t> out(std::vector<py::ssize_t>{h, w, 3});
          ThrowOnError(ctx, dbg(ctx, &it, &o, out.mutable_data(), &w, &h));
          return out;
        },
        "file"_a, "camera"_a, "options"_a, "device"_a = 0,
        "Instrumentation: b2m_debug_undistort_pixels, the RGB image undistort_images encodes for this JPEG / PNG "
        "file's bytes under `camera`");
  m.def("_encode_png",
        [](const py::array_t<uint8_t, py::array::c_style | py::array::forcecast>& a) {
          if (a.ndim() != 2 && a.ndim() != 3) throw std::invalid_argument("[bindings.cc] Check Failed: an (H, W[, C]) image");
          const int c = a.ndim() == 3 ? static_cast<int>(a.shape(2)) : 1;
          std::vector<uint8_t> png;
          {
            py::gil_scoped_release release;
            png = EncodePng(a.data(), static_cast<int>(a.shape(1)), static_cast<int>(a.shape(0)), c);
          }
          return py::bytes(reinterpret_cast<const char*>(png.data()), png.size());
        },
        "image"_a, "An 8-bit PNG file of an (H, W), (H, W, 3) or (H, W, 4) uint8 image");
  m.def("debug_decode_grey",
        [](const py::bytes& file, int max_image_size, int device) { return DebugDecodeGrey(Engine::Get(device), file, max_image_size); },
        "file"_a, "max_image_size"_a = 3200, "device"_a = 0,
        "Instrumentation: the grey image extract_features feeds to SIFT for this JPEG / PNG file's bytes (decoded on "
        "the device, downscaled when larger than max_image_size)");
  m.def("debug_decode_png",
        [](const py::bytes& file) {
          const std::string buf = file;
          Pixels px;
          std::string why;
          if (!DecodePng(std::vector<uint8_t>(buf.begin(), buf.end()), &px, &why)) throw std::invalid_argument("[bindings.cc] " + why);
          py::array_t<uint8_t> out(std::vector<py::ssize_t>{px.height, px.width, px.channels});
          std::memcpy(out.mutable_data(), px.data.data(), px.data.size());
          return out;
        },
        "file"_a,
        "Instrumentation: the pixels extract_features' host PNG decoder gives for a PNG file's bytes, (H, W, C) with C = 1 "
        "(grey, grey + alpha), 3 (RGB, palette) or 4 (RGBA)");
  m.def("import_images",
        [](const py::object& database_path, const py::object& image_path, CameraMode camera_mode,
           const std::vector<std::string>& image_list, const ImageReaderOptions& options) {
          const std::string db_path = FsPath(database_path), images = FsPath(image_path);
          if (!IsFile(db_path)) CheckFailed("images.h:29", "ExistsFile(database_path)", "File " + db_path + " does not exist.");
          if (!IsDir(images)) CheckFailed("images.h:30", "ExistsDir(image_path)", "Directory " + images + " does not exist.");
          CheckCameraMode(options, "images.h:37");
          Database db(db_path);
          ImageReader reader(options, camera_mode, images, image_list, &db);
          for (size_t i = 0; i < reader.NumImages(); ++i) {
            if (PyErr_CheckSignals() != 0) throw py::error_already_set();
            ImageReader::Item item;
            reader.Load(i, &item);
            DatabaseTransaction txn(&db);
            if (reader.Assign(&item) == ImageReader::Status::SUCCESS) db.AddImage(item.name, item.camera.camera_id);
          }
        },
        "database_path"_a, "image_path"_a, "camera_mode"_a = CameraMode::AUTO, "image_list"_a = std::vector<std::string>(),
        "options"_a = ImageReaderOptions(),
        "Write a camera and an image row for every JPEG / PNG file under image_path (images already in the database "
        "are skipped)");
  m.def("infer_camera_from_image",
        [](const py::object& image_path, const ImageReaderOptions& options) {
          const std::string path = FsPath(image_path);
          if (!IsFile(path)) CheckFailed("images.h:67", "ExistsFile(image_path)", "File " + path + " does not exist.");
          ImageHeader h;
          std::string why;
          if (!ReadImageHeader(ReadFileBytes(path), &h, &why))
            throw std::invalid_argument("[images.h:70] Cannot read image file: " + path);
          CheckCameraMode(options, "images.h:76");
          CameraRow c;
          c.model = CameraModelId(options.camera_model);
          c.width = h.width;
          c.height = h.height;
          c.has_prior_focal_length = h.has_focal;
          const double f = h.has_focal ? h.focal : options.default_focal_length_factor * std::max(h.width, h.height);
          c.params = InitialCameraParams(c.model, f, h.width, h.height);
          return CameraToDict(c);
        },
        "image_path"_a, "options"_a = ImageReaderOptions(),
        "The camera ImageReader would create for this image: a dict {model, width, height, params, "
        "has_prior_focal_length}");
  m.def("fundamental_matrix_estimation",
        [](const ArrD& points1, const ArrD& points2, const RANSACOptions& estimation_options) {
          CheckSameLength(points1, points2, "fundamental_matrix.h:22");
          return RansacModel(Engine::Get(0), 1, "F", points1, points2, estimation_options);
        },
        "points2D1"_a, "points2D2"_a, "estimation_options"_a = RANSACOptions());
  m.def("homography_matrix_estimation",
        [](const ArrD& points1, const ArrD& points2, const RANSACOptions& estimation_options) {
          CheckSameLength(points1, points2, "homography_matrix.h:21");
          return RansacModel(Engine::Get(0), 2, "H", points1, points2, estimation_options);
        },
        "points2D1"_a, "points2D2"_a, "estimation_options"_a = RANSACOptions());
  m.def("essential_matrix_estimation",
        [](const ArrD& points1, const ArrD& points2, const py::object& camera1, const py::object& camera2,
           const RANSACOptions& estimation_options) {
          CheckSameLength(points1, points2, "essential_matrix.h:26");
          const b2m_camera c1 = CameraFromPython(camera1), c2 = CameraFromPython(camera2);
          // Camera::CamFromImg on both point lists (R:estimators/essential_matrix.h:31-39; on the GPU, every
          // supported model) and the threshold averaged over both cameras (:42-46).
          b2m_ctx* ctx = Engine::Get(0);
          auto normalise = [ctx](const b2m_camera& c, const ArrD& p) {
            ArrD out(std::vector<py::ssize_t>{p.shape(0), 2});
            ThrowOnError(ctx, b2m_cam_from_img(ctx, &c, p.data(), p.shape(0), out.mutable_data()));
            return out;
          };
          auto mean_f = [](const b2m_camera& c) { return b2m::cam::mean_focal_length(c.model, c.params); };
          RANSACOptions o = estimation_options;
          o.max_error = 0.5 * (o.max_error / mean_f(c1) + o.max_error / mean_f(c2));
          py::object res = RansacModel(ctx, 0, "E", normalise(c1, points1), normalise(c2, points2), o);
          if (res.is_none()) return res;
          // PoseFromEssentialMatrix on the inliers (R:estimators/essential_matrix.h:62-83), on the GPU
          py::dict d = res;
          const py::array_t<bool> mask = py::array_t<bool>::ensure(d["inliers"]);
          std::vector<uint32_t> inl;
          for (py::ssize_t i = 0; i < mask.size(); ++i)
            if (mask.data()[i]) {
              inl.push_back(static_cast<uint32_t>(i));
              inl.push_back(static_cast<uint32_t>(i));
            }
          b2m_tvg_result g;
          memset(&g, 0, sizeof(g));
          g.struct_size = sizeof(g);
          g.config = B2M_CALIBRATED;
          const ArrD E = ArrD::ensure(py::object(d["E"]));
          std::copy(E.data(), E.data() + 9, g.E);
          ThrowOnError(ctx, b2m_estimate_two_view_geometry_pose(ctx, &c1, points1.data(), points1.shape(0), &c2, points2.data(),
                                                               points2.shape(0), inl.data(), static_cast<int64_t>(inl.size() / 2),
                                                               &g));
          Rigid3d pose;
          std::copy(g.qvec, g.qvec + 4, pose.rotation.wxyz.begin());
          std::copy(g.tvec, g.tvec + 3, pose.translation.begin());
          d["cam2_from_cam1"] = pose;
          return res;
        },
        "points2D1"_a, "points2D2"_a, "camera1"_a, "camera2"_a, "estimation_options"_a = RANSACOptions());
  m.def("cam_from_img",
        [](const py::object& camera, const ArrD& points) {
          CheckPoints(points, "points");
          const b2m_camera c = CameraFromPython(camera);
          ArrD out(std::vector<py::ssize_t>{points.shape(0), 2});
          b2m_ctx* ctx = Engine::Get(0);
          ThrowOnError(ctx, b2m_cam_from_img(ctx, &c, points.data(), points.shape(0), out.mutable_data()));
          return out;
        },
        "camera"_a, "points"_a, "Camera.cam_from_img on an N x 2 point list (R:scene/camera.h), every supported model");
  m.def("squared_sampson_error",
        [](const ArrD& points1, const ArrD& points2, const ArrD& E) {
          CheckSameLength(points1, points2, "two_view_geometry.h:165");
          if (E.size() != 9) throw std::invalid_argument("[bindings.cc] Check Failed: E is 3 x 3");
          py::array_t<double> out(points1.shape(0));
          b2m_ctx* ctx = Engine::Get(0);
          ThrowOnError(ctx, b2m_squared_sampson_error(ctx, points1.data(), points2.data(), points1.shape(0), E.data(),
                                                      out.mutable_data()));
          return out;
        },
        "points2D1"_a, "points2D2"_a, "E"_a);

  // ---- pair generators (exposed for tests and tools) ----
  m.def("exhaustive_pair_blocks",
        [](int n_images, int block_size) {
          py::list out;
          for (const PairList& b : ExhaustivePairBlocks(n_images, block_size)) {
            py::array_t<int32_t> a(std::vector<py::ssize_t>{static_cast<py::ssize_t>(b.size() / 2), 2});
            memcpy(a.mutable_data(), b.data(), b.size() * 4);
            out.append(a);
          }
          return out;
        },
        "n_images"_a, "block_size"_a);
  m.def("comm_image_range",
        [](int n_images, int n_ranks, int rank) {
          int32_t first = 0, count = 0;
          b2m_comm_image_range(n_images, n_ranks, rank, &first, &count);
          return py::make_tuple(first, count);
        },
        "n_images"_a, "n_ranks"_a, "rank"_a, "The contiguous image range rank `rank` uploads (b2m_comm_image_range)");
  m.def("last_pipeline_timing", []() {
    const PipelineTiming t = LastPipelineTiming();
    return py::dict("read_s"_a = t.read_s, "upload_s"_a = t.upload_s, "gpu_s"_a = t.gpu_s, "write_s"_a = t.write_s,
                    "write_wait_s"_a = t.write_wait_s, "total_s"_a = t.total_s, "pairs"_a = t.pairs,
                    "sharded_upload"_a = t.sharded_upload);
  }, "Wall-clock breakdown of the last match_* / verify_matches call of this process");
  m.def("parse_gpu_indices", &ParseGpuIndices, "gpu_index"_a);
  m.def("split_pairs_by_cost",
        [](const ArrI32& pairs, const std::vector<int32_t>& n_feat, int parts) {
          if (pairs.size() % 2) throw std::invalid_argument("[bindings.cc] Check Failed: pairs is N x 2 int32");
          for (py::ssize_t i = 0; i < pairs.size(); ++i)
            if (pairs.data()[i] < 0 || pairs.data()[i] >= static_cast<int32_t>(n_feat.size()))
              throw std::invalid_argument("[bindings.cc] Check Failed: pair index < number of images");
          return SplitPairsByCost(PairList(pairs.data(), pairs.data() + pairs.size()), n_feat, parts);
        },
        "pairs"_a, "n_feat"_a, "parts"_a);
  m.def("spatial_pairs",
        [](const ArrD& prior_t, const std::vector<bool>& has_prior, const SpatialMatchingOptions& options) {
          if (prior_t.ndim() != 2 || prior_t.shape(1) != 3 || prior_t.shape(0) != static_cast<py::ssize_t>(has_prior.size()))
            throw std::invalid_argument("[bindings.cc] Check Failed: prior_t is N x 3 with one flag per row");
          std::vector<std::array<double, 3>> t(has_prior.size());
          for (size_t i = 0; i < t.size(); ++i) t[i] = {prior_t.data()[3 * i], prior_t.data()[3 * i + 1], prior_t.data()[3 * i + 2]};
          const PairList p = SpatialPairs(t, has_prior, options);
          py::array_t<int32_t> a(std::vector<py::ssize_t>{static_cast<py::ssize_t>(p.size() / 2), 2});
          if (!p.empty()) memcpy(a.mutable_data(), p.data(), p.size() * 4);
          return a;
        },
        "prior_t"_a, "has_prior"_a, "options"_a = SpatialMatchingOptions());
  m.def("sequential_pairs",
        [](int n_images, int overlap, bool quadratic_overlap) {
          const PairList p = SequentialPairs(n_images, overlap, quadratic_overlap);
          py::array_t<int32_t> a(std::vector<py::ssize_t>{static_cast<py::ssize_t>(p.size() / 2), 2});
          if (!p.empty()) memcpy(a.mutable_data(), p.data(), p.size() * 4);
          return a;
        },
        "n_images"_a, "overlap"_a, "quadratic_overlap"_a);

  // ---- database ----
  m.def("image_pair_to_pair_id", &ImagePairToPairId, "image_id1"_a, "image_id2"_a);
  m.def("pair_id_to_image_pair", [](int64_t pid) {
    int64_t a, b;
    PairIdToImagePair(pid, &a, &b);
    return py::make_tuple(a, b);
  });
  m.def("sqlite_version", []() { return std::string(sq::api().libversion()); });
  py::class_<Database>(m, "Database")
      .def(py::init<>())
      .def(py::init([](const py::object& path) { return std::make_unique<Database>(FsPath(path)); }), "path"_a)
      .def_static("connect", [](const py::object& path) { return std::make_unique<Database>(FsPath(path)); }, "path"_a)
      .def("open", [](Database& db, const py::object& path) { db.Open(FsPath(path)); }, "path"_a)
      .def("close", &Database::Close)
      .def("__enter__", [](py::object self) { return self; })
      .def("__exit__", [](Database& db, const py::args&) { db.Close(); })
      .def_property_readonly("num_cameras", &Database::NumCameras)
      .def_property_readonly("num_images", &Database::NumImages)
      .def_property_readonly("num_keypoints", &Database::NumKeypoints)
      .def_property_readonly("num_descriptors", &Database::NumDescriptors)
      .def_property_readonly("num_matches", &Database::NumMatches)
      .def_property_readonly("num_inlier_matches", &Database::NumInlierMatches)
      .def_property_readonly("num_matched_image_pairs", &Database::NumMatchedImagePairs)
      .def_property_readonly("num_verified_image_pairs", &Database::NumVerifiedImagePairs)
      .def("num_rows", &Database::NumRows, "table"_a)
      .def("add_camera",
           [](Database& db, int model, int64_t width, int64_t height, const std::vector<double>& params,
              bool prior_focal_length) { return db.AddCamera(model, width, height, params, prior_focal_length); },
           "model"_a, "width"_a, "height"_a, "params"_a, "prior_focal_length"_a = false)
      .def("add_image",
           [](Database& db, const std::string& name, int64_t camera_id, const py::object& prior_t) {
             if (prior_t.is_none()) return db.AddImage(name, camera_id);
             const std::vector<double> t = prior_t.cast<std::vector<double>>();
             if (t.size() != 3) throw std::invalid_argument("[bindings.cc] Check Failed: prior_t has 3 entries");
             return db.AddImage(name, camera_id, std::array<double, 3>{t[0], t[1], t[2]});
           },
           "name"_a, "camera_id"_a, "prior_t"_a = py::none())
      .def("write_keypoints",
           [](Database& db, int64_t image_id, const ArrF32& kp) {
             if (kp.ndim() != 2) throw std::invalid_argument("[bindings.cc] Check Failed: keypoints is a 2-D array");
             db.WriteKeypoints(image_id, kp.data(), kp.shape(0), kp.shape(1));
           },
           "image_id"_a, "keypoints"_a)
      .def("write_descriptors",
           [](Database& db, int64_t image_id, const ArrU8& d) {
             if (d.ndim() != 2) throw std::invalid_argument("[bindings.cc] Check Failed: descriptors is a 2-D array");
             db.WriteDescriptors(image_id, d.data(), d.shape(0), d.shape(1));
           },
           "image_id"_a, "descriptors"_a)
      .def("read_all_images",
           [](Database& db) {
             py::list out;
             for (const ImageRow& r : db.ReadAllImages()) out.append(py::make_tuple(r.image_id, r.name, r.camera_id));
             return out;
           })
      .def("read_camera", [](Database& db, int64_t camera_id) { return CameraToDict(db.ReadCamera(camera_id)); },
           "camera_id"_a)
      // the rest of the reference's Database surface (R:scene/database.h:10-47); cameras are dicts, images are
      // (image_id, name, camera_id) tuples here -- pycolmap.Camera / Image belong to the reconstruction object model
      .def("read_all_cameras",
           [](Database& db) {
             py::list out;
             for (const CameraRow& c : db.ReadAllCameras()) {
               py::dict d = CameraToDict(c);
               d["camera_id"] = c.camera_id;
               out.append(d);
             }
             return out;
           })
      .def("read_image",
           [](Database& db, int64_t image_id) -> py::object {
             ImageRow r;
             if (!db.ReadImage(image_id, &r)) throw std::invalid_argument("[bindings.cc] Check Failed: image exists");
             return py::make_tuple(r.image_id, r.name, r.camera_id);
           },
           "image_id"_a)
      .def("read_image_with_name",
           [](Database& db, const std::string& name) -> py::object {
             ImageRow r;
             if (!db.ReadImageWithName(name, &r)) throw std::invalid_argument("[bindings.cc] Check Failed: image exists");
             return py::make_tuple(r.image_id, r.name, r.camera_id);
           },
           "name"_a)
      .def("num_keypoints_for_image", &Database::NumKeypointsForImage, "image_id"_a)
      .def("num_descriptors_for_image", &Database::NumDescriptorsForImage, "image_id"_a)
      .def("image_pair_to_pair_id", [](Database&, int64_t a, int64_t b) { return ImagePairToPairId(a, b); },
           "image_id1"_a, "image_id2"_a)
      .def("pair_id_to_image_pair",
           [](Database&, int64_t pid) {
             int64_t a, b;
             PairIdToImagePair(pid, &a, &b);
             return py::make_tuple(a, b);
           },
           "pair_id"_a)
      .def("write_camera",
           [](Database& db, const py::object& camera) {
             const b2m_camera c = CameraFromPython(camera);   // validates model id and parameter count
             return db.AddCamera(c.model, c.width, c.height,
                                 std::vector<double>(c.params, c.params + b2m::cam::num_params(c.model)),
                                 c.has_prior_focal_length != 0);
           },
           "camera"_a)
      .def("write_image", [](Database& db, const std::string& name, int64_t camera_id) { return db.AddImage(name, camera_id); },
           "name"_a, "camera_id"_a)
      .def("read_keypoints",
           [](Database& db, int64_t image_id) {
             const KeypointsBlob k = db.ReadKeypoints(image_id);
             py::array_t<float> a(std::vector<py::ssize_t>{static_cast<py::ssize_t>(k.rows), static_cast<py::ssize_t>(k.cols)});
             if (!k.data.empty()) memcpy(a.mutable_data(), k.data.data(), k.data.size() * 4);
             return a;
           },
           "image_id"_a)
      .def("read_descriptors",
           [](Database& db, int64_t image_id) {
             const DescriptorsBlob d = db.ReadDescriptors(image_id);
             py::array_t<uint8_t> a(std::vector<py::ssize_t>{static_cast<py::ssize_t>(d.rows), 128});
             if (!d.data.empty()) memcpy(a.mutable_data(), d.data.data(), d.data.size());
             return a;
           },
           "image_id"_a)
      .def("exists_matches", &Database::ExistsMatches, "image_id1"_a, "image_id2"_a)
      .def("exists_inlier_matches", &Database::ExistsInlierMatches, "image_id1"_a, "image_id2"_a)
      .def("read_matches",
           [](Database& db, int64_t id1, int64_t id2) {
             const std::vector<uint32_t> mm = db.ReadMatches(id1, id2);
             return MatchesToNumpy(mm.data(), static_cast<int64_t>(mm.size() / 2));
           },
           "image_id1"_a, "image_id2"_a)
      .def("read_two_view_geometry",
           [](Database& db, int64_t id1, int64_t id2) -> py::object {
             TwoViewGeometryRow row;
             if (!db.ReadTwoViewGeometry(id1, id2, &row)) return py::none();
             TwoViewGeometry g;
             g.config = static_cast<TwoViewGeometryConfiguration>(row.config);
             g.E = row.E; g.F = row.F; g.H = row.H;
             g.qvec = row.qvec; g.tvec = row.tvec;
             g.inlier_matches = std::move(row.inlier_matches);
             return py::cast(std::move(g));
           },
           "image_id1"_a, "image_id2"_a)
      .def("write_matches",
           [](Database& db, int64_t id1, int64_t id2, const ArrU32& mm) {
             if (mm.size() % 2) throw std::invalid_argument("[bindings.cc] Check Failed: matches is N x 2");
             db.WriteMatches(id1, id2, mm.data(), mm.size() / 2);
           },
           "image_id1"_a, "image_id2"_a, "matches"_a)
      .def("write_two_view_geometry",
           [](Database& db, int64_t id1, int64_t id2, const TwoViewGeometry& g) {
             db.WriteTwoViewGeometry(id1, id2, static_cast<int>(g.config), g.inlier_matches.data(),
                                     static_cast<int64_t>(g.inlier_matches.size() / 2), g.F, g.E, g.H, g.qvec, g.tvec);
           },
           "image_id1"_a, "image_id2"_a, "two_view_geometry"_a)
      .def("clear_matches", &Database::ClearMatches)
      .def("clear_two_view_geometries", &Database::ClearTwoViewGeometries)
      .def("begin", &Database::Begin)
      .def("commit", &Database::Commit)
      .def("rollback", &Database::Rollback);

  py::class_<DatabaseTransaction>(m, "DatabaseTransaction")   // R:scene/database.h:45-46: BEGIN now, COMMIT when released
      .def(py::init<Database*>(), "database"_a, py::keep_alive<1, 2>());

  // ---- low-level context ----
  py::class_<CoreResults>(m, "Results")
      .def("__len__", [](const CoreResults& r) { return r.r ? b2m_results_num_pairs(r.r) : 0; })
      .def_property_readonly("total_matches", [](const CoreResults& r) { return r.r ? b2m_results_total_matches(r.r) : 0; })
      .def_property_readonly("num_verified", [](const CoreResults& r) { return r.r ? b2m_results_num_verified(r.r) : 0; })
      .def("matches", [](const CoreResults& r, int64_t k) {
        const b2m_pair_view v = r.View(k);
        return MatchesToNumpy(v.matches, v.n_matches);
      })
      .def("inlier_matches", [](const CoreResults& r, int64_t k) {
        const b2m_pair_view v = r.View(k);
        return MatchesToNumpy(v.inlier_matches, v.n_inliers);
      })
      .def("two_view_geometry", [](const CoreResults& r, int64_t k) {
        const b2m_pair_view v = r.View(k);
        TwoViewGeometry g;
        g.config = static_cast<TwoViewGeometryConfiguration>(v.config);
        std::copy(v.E, v.E + 9, g.E.begin());
        std::copy(v.F, v.F + 9, g.F.begin());
        std::copy(v.H, v.H + 9, g.H.begin());
        g.inlier_matches.assign(v.inlier_matches, v.inlier_matches + 2 * v.n_inliers);
        std::copy(v.qvec, v.qvec + 4, g.qvec.begin());
        std::copy(v.tvec, v.tvec + 3, g.tvec.begin());
        g.tri_angle = v.tri_angle;
        return g;
      })
      .def("image_pair", [](const CoreResults& r, int64_t k) {
        const b2m_pair_view v = r.View(k);
        return py::make_tuple(v.image1, v.image2);
      })
      .def("free", &CoreResults::Free);

  py::class_<CoreContext>(m, "Context")
      .def(py::init<int, uint64_t, int>(), "device"_a = 0, "seed"_a = 0, "pair_batch"_a = 0)
      .def("close", &CoreContext::Close)
      .def("set_images",
           [](CoreContext& c, const py::list& descs, const py::object& kpts, const py::object& cams) {
             const size_t n = descs.size();
             std::vector<ArrU8> d(n);
             std::vector<ArrF32> k(n);
             std::vector<int32_t> n_feat(n);
             std::vector<const uint8_t*> dptr(n);
             std::vector<const float*> kptr(n);
             for (size_t i = 0; i < n; ++i) {
               d[i] = ArrU8::ensure(descs[i]);
               if (!d[i] || d[i].size() % 128)
                 throw std::invalid_argument("[bindings.cc] Check Failed: descriptors are N x 128 uint8");
               n_feat[i] = static_cast<int32_t>(d[i].size() / 128);
               dptr[i] = d[i].data();
             }
             if (!kpts.is_none()) {
               const py::list kl = kpts;
               if (kl.size() != n) throw std::invalid_argument("[bindings.cc] Check Failed: one keypoint array per image");
               for (size_t i = 0; i < n; ++i) {
                 k[i] = ArrF32::ensure(kl[i]);
                 if (!k[i] || k[i].size() != 2 * static_cast<py::ssize_t>(n_feat[i]))
                   throw std::invalid_argument("[bindings.cc] Check Failed: keypoints.rows == descriptors.rows (N x 2 float32)");
                 kptr[i] = k[i].data();
               }
             }
             std::vector<b2m_camera> cc;
             if (!cams.is_none()) {
               cc = CamerasFromPython(cams);
               if (cc.size() != n) throw std::invalid_argument("[bindings.cc] Check Failed: one camera per image");
             }
             b2m_ctx* ctx = c.Handle();
             int rc;
             {
               py::gil_scoped_release release;
               rc = b2m_set_images(ctx, static_cast<int32_t>(n), n_feat.data(), dptr.data(),
                                   kpts.is_none() ? nullptr : kptr.data(), cams.is_none() ? nullptr : cc.data());
             }
             ThrowOnError(ctx, rc);
           },
           "descriptors"_a, "keypoints"_a = py::none(), "cameras"_a = py::none())
      .def("set_images_device",
           [](CoreContext& c, const ArrI32& n_feat, uint64_t dev_desc_ptr, uint64_t dev_kpts_ptr, const py::object& cams) {
             std::vector<b2m_camera> cc;
             if (!cams.is_none()) cc = CamerasFromPython(cams);
             b2m_ctx* ctx = c.Handle();
             ThrowOnError(ctx, b2m_set_images_device(ctx, static_cast<int32_t>(n_feat.size()), n_feat.data(),
                                                     reinterpret_cast<const void*>(dev_desc_ptr),
                                                     reinterpret_cast<const void*>(dev_kpts_ptr),
                                                     cams.is_none() ? nullptr : cc.data()));
           },
           "n_feat"_a, "dev_desc_ptr"_a, "dev_kpts_ptr"_a = 0, "cameras"_a = py::none())
      // ---- multi-GPU (include/b200match.h: b2m_comm_*, b2m_set_images_sharded) ----
      .def_static("comm_unique_id",
                  []() {
                    b2m_comm_id id;
                    ThrowOnError(nullptr, b2m_comm_get_unique_id(&id));
                    return py::bytes(reinterpret_cast<const char*>(id.bytes), B2M_COMM_ID_BYTES);
                  },
                  "Rank 0: a fresh communicator id (128 bytes) to hand to every rank through the launcher's side channel")
      .def("comm_init_rank",
           [](CoreContext& c, int n_ranks, int rank, const py::bytes& id) {
             const std::string raw = id;
             if (raw.size() != B2M_COMM_ID_BYTES) throw std::invalid_argument("[bindings.cc] Check Failed: id has 128 bytes");
             b2m_comm_id cid;
             memcpy(cid.bytes, raw.data(), B2M_COMM_ID_BYTES);
             b2m_ctx* ctx = c.Handle();
             int rc;
             {
               py::gil_scoped_release release;
               rc = b2m_comm_init_rank(ctx, n_ranks, rank, &cid);
             }
             ThrowOnError(ctx, rc);
           },
           "n_ranks"_a, "rank"_a, "id"_a)
      .def("comm_destroy", [](CoreContext& c) { ThrowOnError(c.Handle(), b2m_comm_destroy(c.Handle())); })
      .def("set_images_sharded",
           [](CoreContext& c, const ArrI32& n_feat, int first_image, int n_local, const py::object& desc_local,
              const py::object& kpts_local, const py::object& cams, bool has_keypoints) {
             // desc_local / kpts_local: numpy arrays (host: [rows x 128] uint8, [rows x 2] float32) or device pointers (int)
             b2m_image_shard sh;
             memset(&sh, 0, sizeof(sh));
             sh.struct_size = sizeof(sh);
             sh.first_image = first_image;
             sh.n_local = n_local;
             sh.has_keypoints = has_keypoints ? 1 : 0;
             ArrU8 d;
             ArrF32 k;
             if (py::isinstance<py::int_>(desc_local)) {
               sh.location = B2M_LOC_DEVICE;
               sh.desc_packed = reinterpret_cast<const void*>(desc_local.cast<uint64_t>());
               if (!kpts_local.is_none()) sh.kpts_packed = reinterpret_cast<const void*>(kpts_local.cast<uint64_t>());
             } else {
               sh.location = B2M_LOC_HOST;
               int64_t rows = 0;
               for (int i = first_image; i < first_image + n_local && i < n_feat.size(); ++i) rows += n_feat.data()[i];
               if (!desc_local.is_none()) {
                 d = ArrU8::ensure(desc_local);
                 if (!d || d.size() != rows * 128)
                   throw std::invalid_argument("[bindings.cc] Check Failed: local descriptors are (sum of local n_feat) x 128 uint8");
                 sh.desc_packed = d.data();
               }
               if (!kpts_local.is_none()) {
                 k = ArrF32::ensure(kpts_local);
                 if (!k || k.size() != rows * 2)
                   throw std::invalid_argument("[bindings.cc] Check Failed: local keypoints are (sum of local n_feat) x 2 float32");
                 sh.kpts_packed = k.data();
               }
             }
             std::vector<b2m_camera> cc;
             if (!cams.is_none()) {
               cc = CamerasFromPython(cams);
               if (static_cast<py::ssize_t>(cc.size()) != n_feat.size())
                 throw std::invalid_argument("[bindings.cc] Check Failed: one camera per image (all images, not only the local ones)");
             }
             b2m_ctx* ctx = c.Handle();
             int rc;
             {
               py::gil_scoped_release release;
               rc = b2m_set_images_sharded(ctx, static_cast<int32_t>(n_feat.size()), n_feat.data(),
                                           cams.is_none() ? nullptr : cc.data(), &sh);
             }
             ThrowOnError(ctx, rc);
           },
           "n_feat"_a, "first_image"_a, "n_local"_a, "descriptors_local"_a, "keypoints_local"_a = py::none(),
           "cameras"_a = py::none(), "has_keypoints"_a = false)
      .def("match_pair",
           [](CoreContext& c, const ArrU8& d1, const ArrU8& d2, const SiftMatchingOptions& options) {
             if (d1.size() % 128 || d2.size() % 128)
               throw std::invalid_argument("[bindings.cc] Check Failed: descriptors are N x 128 uint8");
             const int32_t n1 = static_cast<int32_t>(d1.size() / 128), n2 = static_cast<int32_t>(d2.size() / 128);
             std::vector<uint32_t> out(static_cast<size_t>(std::max(1, n1)) * 2);
             int64_t n = 0;
             const b2m_sift_opts o = ToAbi(options);
             b2m_ctx* ctx = c.Handle();
             int rc;
             {
               py::gil_scoped_release release;
               rc = b2m_match_pair(ctx, d1.data(), n1, d2.data(), n2, &o, out.data(), std::max(1, n1), &n);
             }
             ThrowOnError(ctx, rc);
             return MatchesToNumpy(out.data(), n);
           },
           "descriptors1"_a, "descriptors2"_a, "options"_a = SiftMatchingOptions())
      .def("match_pairs",
           [](CoreContext& c, const ArrI32& pairs, const SiftMatchingOptions& sift, const py::object& tvg) {
             if (pairs.size() % 2) throw std::invalid_argument("[bindings.cc] Check Failed: pairs is N x 2 int32");
             const b2m_sift_opts so = ToAbi(sift);
             b2m_tvg_opts to;
             const bool verify = !tvg.is_none();
             if (verify) to = ToAbi(tvg.cast<TwoViewGeometryOptions>());
             auto res = std::make_unique<CoreResults>();
             b2m_ctx* ctx = c.Handle();
             int rc = B2M_OK;
             RunInterruptible([&] {
               rc = b2m_match_pairs(ctx, pairs.data(), pairs.size() / 2, &so, verify ? &to : nullptr, &res->r);
             });
             ThrowOnError(ctx, rc);
             return res;
           },
           "pairs"_a, "sift_options"_a = SiftMatchingOptions(), "verification_options"_a = py::none())
      .def("estimate_two_view_geometry",
           [](CoreContext& c, const py::object& camera1, const ArrD& points1, const py::object& camera2,
              const ArrD& points2, const py::object& matches, const TwoViewGeometryOptions& options) {
             return EstimateTvg([&c] { return c.Handle(); }, camera1, points1, camera2, points2, matches, options);
           },
           "camera1"_a, "points1"_a, "camera2"_a, "points2"_a, "matches"_a = py::none(),
           "options"_a = TwoViewGeometryOptions())
      .def("estimate_triangulations",
           [](CoreContext& c, const py::object& points_normalized, const py::object& track_lengths,
              const py::object& image_idxs, const py::object& cams_from_world, const EstimateTriangulationOptions& options) {
             return EstimateTriangulationsPy([&c] { return c.Handle(); }, points_normalized, track_lengths, image_idxs,
                                             cams_from_world, options);
           },
           "points_normalized"_a, "track_lengths"_a, "image_idxs"_a, "cams_from_world"_a,
           "options"_a = EstimateTriangulationOptions())
      .def("debug_five_point",
           [](CoreContext& c, const ArrD& nullspaces) {
             if (nullspaces.size() % 36) throw std::invalid_argument("[bindings.cc] Check Failed: null spaces are n x 4 x 9");
             const int64_t n = nullspaces.size() / 36;
             ArrD models(std::vector<py::ssize_t>{static_cast<py::ssize_t>(n), 10, 9});
             py::array_t<int32_t> counts(static_cast<py::ssize_t>(n));
             ThrowOnError(c.Handle(), b2m_debug_five_point(c.Handle(), nullspaces.data(), n, models.mutable_data(),
                                                           counts.mutable_data()));
             return py::make_tuple(models, counts);
           },
           "nullspaces"_a, "The device 5-point solver (one warp per 4-D null space): (models [n, 10, 9], counts [n])")
      .def("debug_decode_grey",
           [](CoreContext& c, const py::bytes& file, int max_image_size) { return DebugDecodeGrey(c.Handle(), file, max_image_size); },
           "file"_a, "max_image_size"_a = 3200, "pycolmap_b200.debug_decode_grey on this context")
      .def("stats", [](CoreContext& c) {
        b2m_stats s;
        memset(&s, 0, sizeof(s));
        s.struct_size = sizeof(s);
        ThrowOnError(c.Handle(), b2m_get_stats(c.Handle(), &s));
        return py::dict("kernel_launches"_a = s.kernel_launches, "match_tiles"_a = s.match_tiles,
                        "last_match_ms"_a = s.last_match_ms, "last_verify_ms"_a = s.last_verify_ms,
                        "last_total_ms"_a = s.last_total_ms, "last_k1_ms"_a = s.last_k1_ms,
                        "last_k1_launches"_a = s.last_k1_launches,
                        "k1_dir1_mode"_a = s.k1_dir1_mode, "last_allgather_ms"_a = s.last_allgather_ms,
                        "last_allgather_bytes"_a = s.last_allgather_bytes, "last_upload_ms"_a = s.last_upload_ms,
                        "verify_models_scored"_a = py::make_tuple(s.verify_models_scored[0], s.verify_models_scored[1],
                                                                  s.verify_models_scored[2]),
                        "verify_residuals"_a = py::make_tuple(s.verify_residuals[0], s.verify_residuals[1],
                                                              s.verify_residuals[2]),
                        "comm_size"_a = s.comm_size, "comm_rank"_a = s.comm_rank,
                        "tri_models_scored"_a = s.tri_models_scored, "tri_residuals"_a = s.tri_residuals,
                        "sift_images"_a = s.sift_images, "sift_keypoints"_a = s.sift_keypoints,
                        "sift_descriptors"_a = s.sift_descriptors, "sift_decoded_bytes"_a = s.sift_decoded_bytes,
                        "sift_decode_images"_a = s.sift_decode_images,
                        "sift_decode_hardware"_a = s.sift_decode_hardware, "pm_problems"_a = s.pm_problems,
                        "pm_pixel_updates"_a = s.pm_pixel_updates, "pm_window_samples"_a = s.pm_window_samples);
      })
      .def("reset_stats", [](CoreContext& c) { ThrowOnError(c.Handle(), b2m_reset_stats(c.Handle()));
      });

  // test hook for the PyWait logic: blocks `seconds` on the worker thread like a long GPU call would
  m.def("_sleep_interruptible", [](double seconds) {
    RunInterruptible([seconds] { std::this_thread::sleep_for(std::chrono::duration<double>(seconds)); });
  });

  // destroy the per-device contexts of the pipeline / estimator functions at interpreter exit
  m.add_object("_cleanup", py::capsule([]() { Engine::DestroyAll(); }));
}
