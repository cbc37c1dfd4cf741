#include "controllers.h"

#include "../csrc/camera_models.h"  // header-only; model ids / parameter counts shared with the kernels

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <exception>
#include <fstream>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <set>
#include <sstream>
#include <stdexcept>
#include <thread>
#include <unordered_map>

namespace b2mh {

namespace {
PipelineTiming g_timing;
double Now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
}  // namespace
PipelineTiming LastPipelineTiming() { return g_timing; }

// ---- option conversion ---------------------------------------------------------------------------
b2m_sift_opts ToAbi(const SiftMatchingOptions& o) {
  b2m_sift_opts s;
  b2m_sift_opts_default(&s);
  s.max_ratio = static_cast<float>(o.max_ratio);  // double -> float at use, like upstream
  s.max_distance = static_cast<float>(o.max_distance);
  s.cross_check = o.cross_check ? 1 : 0;
  s.max_num_matches = o.max_num_matches;
  s.guided_matching = o.guided_matching ? 1 : 0;
  return s;
}

b2m_ransac_opts ToAbi(const RANSACOptions& o) {
  b2m_ransac_opts r;
  b2m_ransac_opts_default(&r);
  r.max_error = o.max_error;
  r.min_inlier_ratio = o.min_inlier_ratio;
  r.confidence = o.confidence;
  r.dyn_num_trials_multiplier = o.dyn_num_trials_multiplier;
  r.min_num_trials = o.min_num_trials;
  r.max_num_trials = o.max_num_trials;
  return r;
}

// The absolute pose structs are filled field by field (no b2m_*_opts_default call): the host module binds the absolute
// pose entry points at run time (bindings.cc) and references no symbol of C ABI version 4 at link time.
b2m_abs_pose_opts ToAbi(const AbsolutePoseEstimationOptions& o) {
  b2m_abs_pose_opts r;
  memset(&r, 0, sizeof(r));
  r.struct_size = sizeof(r);
  r.estimate_focal_length = o.estimate_focal_length ? 1 : 0;
  r.num_focal_length_samples = o.num_focal_length_samples;
  r.min_focal_length_ratio = o.min_focal_length_ratio;
  r.max_focal_length_ratio = o.max_focal_length_ratio;
  r.ransac = ToAbi(o.ransac);
  return r;
}

// Filled field by field for the same reason (C ABI version 6).
b2m_extract_opts ToAbi(const SiftExtractionOptions& o) {
  b2m_extract_opts r;
  memset(&r, 0, sizeof(r));
  r.struct_size = sizeof(r);
  r.max_image_size = o.max_image_size;
  r.max_num_features = o.max_num_features;
  r.first_octave = o.first_octave;
  r.num_octaves = o.num_octaves;
  r.octave_resolution = o.octave_resolution;
  r.peak_threshold = o.peak_threshold;
  r.edge_threshold = o.edge_threshold;
  r.max_num_orientations = o.max_num_orientations;
  r.upright = o.upright;
  r.normalization = o.normalization == Normalization::L2 ? B2M_NORMALIZATION_L2 : B2M_NORMALIZATION_L1_ROOT;
  r.estimate_affine_shape = o.estimate_affine_shape;
  r.domain_size_pooling = o.domain_size_pooling;
  r.darkness_adaptivity = o.darkness_adaptivity;
  return r;
}

// Filled field by field for the same reason (C ABI version 5).
b2m_tri_opts ToAbi(const EstimateTriangulationOptions& o) {
  b2m_tri_opts r;
  memset(&r, 0, sizeof(r));
  r.struct_size = sizeof(r);
  r.min_tri_angle = o.min_tri_angle;
  r.ransac = ToAbi(o.ransac);
  return r;
}

b2m_pose_refine_opts ToAbi(const AbsolutePoseRefinementOptions& o) {
  b2m_pose_refine_opts r;
  memset(&r, 0, sizeof(r));
  r.struct_size = sizeof(r);
  r.gradient_tolerance = o.gradient_tolerance;
  r.max_num_iterations = o.max_num_iterations;
  r.loss_function_scale = o.loss_function_scale;
  r.refine_focal_length = o.refine_focal_length ? 1 : 0;
  r.refine_extra_params = o.refine_extra_params ? 1 : 0;
  r.print_summary = o.print_summary ? 1 : 0;
  return r;
}

b2m_tvg_opts ToAbi(const TwoViewGeometryOptions& o) {
  b2m_tvg_opts t;
  b2m_tvg_opts_default(&t);
  t.min_num_inliers = o.min_num_inliers;
  t.min_E_F_inlier_ratio = o.min_E_F_inlier_ratio;
  t.max_H_inlier_ratio = o.max_H_inlier_ratio;
  t.watermark_min_inlier_ratio = o.watermark_min_inlier_ratio;
  t.watermark_border_size = o.watermark_border_size;
  t.detect_watermark = o.detect_watermark;
  t.multiple_ignore_watermark = o.multiple_ignore_watermark;
  t.force_H_use = o.force_H_use;
  t.compute_relative_pose = o.compute_relative_pose;
  t.multiple_models = o.multiple_models;
  t.ransac = ToAbi(o.ransac);
  return t;
}

b2m_camera ToAbi(const CameraRow& c) {
  if (b2m::cam::num_params(c.model) < 0)
    throw std::invalid_argument("[controllers.cc] camera model id " + std::to_string(c.model) +
                                " is not supported by the GPU verifier (COLMAP 3.9.1 model ids 0-10)");
  const size_t need = static_cast<size_t>(b2m::cam::num_params(c.model));
  if (c.params.size() != need)
    throw std::invalid_argument("[controllers.cc] Check Failed: camera has " + std::to_string(need) + " parameters");
  b2m_camera b;
  memset(&b, 0, sizeof(b));
  b.struct_size = sizeof(b);
  b.model = c.model;
  b.width = static_cast<int32_t>(c.width);
  b.height = static_cast<int32_t>(c.height);
  b.has_prior_focal_length = c.has_prior_focal_length ? 1 : 0;
  std::copy(c.params.begin(), c.params.end(), b.params);
  return b;
}

std::vector<int> ParseGpuIndices(const std::string& gpu_index) {
  std::vector<int> out;
  std::stringstream ss(gpu_index);
  std::string item;
  while (std::getline(ss, item, ',')) {
    item.erase(std::remove_if(item.begin(), item.end(), [](unsigned char ch) { return std::isspace(ch); }), item.end());
    if (item.empty()) continue;
    size_t used = 0;
    int v = 0;
    try {
      v = std::stoi(item, &used);
    } catch (const std::exception&) {
      used = 0;
    }
    if (used != item.size() || v < -1)
      throw std::invalid_argument("[controllers.cc] Check Failed: gpu_index is a comma-separated list of integers >= -1");
    if (v == -1) {  // upstream: "-1" = every visible GPU, one matcher each (U:feature/sift.cc CreateSiftFeatureMatcher path)
      const int n = std::max(1, b2m_device_count());
      for (int d = 0; d < n; ++d)
        if (std::find(out.begin(), out.end(), d) == out.end()) out.push_back(d);
      continue;
    }
    if (std::find(out.begin(), out.end(), v) == out.end()) out.push_back(v);
  }
  if (out.empty()) out.push_back(0);
  return out;
}

std::vector<int64_t> SplitPairsByCost(const PairList& pairs, const std::vector<int32_t>& n_feat, int parts) {
  const int64_t n = static_cast<int64_t>(pairs.size() / 2);
  parts = std::max(1, parts);
  std::vector<int64_t> cut(static_cast<size_t>(parts) + 1, n);
  cut[0] = 0;
  if (parts == 1 || n == 0) return cut;
  // cost of a pair = work of its distance matrix (K1 dominates): n_feat[a] * n_feat[b], at least 1
  std::vector<double> prefix(static_cast<size_t>(n) + 1, 0.0);
  for (int64_t k = 0; k < n; ++k) {
    const double c = static_cast<double>(n_feat[pairs[2 * k]]) * static_cast<double>(n_feat[pairs[2 * k + 1]]);
    prefix[k + 1] = prefix[k] + std::max(1.0, c);
  }
  for (int d = 1; d < parts; ++d) {
    const double target = prefix[n] * d / parts;
    cut[d] = std::lower_bound(prefix.begin(), prefix.end(), target) - prefix.begin();
    cut[d] = std::min(n, std::max(cut[d], cut[d - 1]));
  }
  return cut;
}

// ---- pair generators -----------------------------------------------------------------------------
std::vector<PairList> ExhaustivePairBlocks(int n, int bs) {
  if (bs < 1) throw std::invalid_argument("[controllers.cc] Check Failed: block_size >= 1");
  std::vector<PairList> out;
  for (int s1 = 0; s1 < n; s1 += bs) {
    const int e1 = std::min(n, s1 + bs);
    for (int s2 = 0; s2 < n; s2 += bs) {
      const int e2 = std::min(n, s2 + bs);
      PairList block;
      for (int i1 = s1; i1 < e1; ++i1) {
        const int r1 = i1 % bs;
        for (int i2 = s2; i2 < e2; ++i2) {
          const int r2 = i2 % bs;
          // the upstream rule that visits every unordered pair exactly once over the block grid
          if ((i1 > i2 && r1 <= r2) || (i1 < i2 && r1 < r2)) {
            block.push_back(i1);
            block.push_back(i2);
          }
        }
      }
      if (!block.empty()) out.push_back(std::move(block));
    }
  }
  return out;
}

PairList SequentialPairs(int n, int overlap, bool quadratic_overlap) {
  PairList out;
  std::set<std::pair<int, int>> seen;
  auto emit = [&](int64_t i1, int64_t i2) {
    if (i2 < n && seen.insert({static_cast<int>(i1), static_cast<int>(i2)}).second) {
      out.push_back(static_cast<int32_t>(i1));
      out.push_back(static_cast<int32_t>(i2));
    }
  };
  // U:controllers/feature_matching.cc SequentialFeatureMatcher::RunSequentialMatching (COLMAP 3.9.1):
  // image_idx2 = image_idx1 + i for i in [0, overlap) -- i = 0 is the self pair, which the controller drops, so
  // there are overlap - 1 linear neighbours -- and image_idx1 + 2^i inside the same in-range test.
  for (int i1 = 0; i1 < n; ++i1) {
    for (int k = 0; k < overlap; ++k) {
      const int64_t i2 = static_cast<int64_t>(i1) + k;
      if (i2 >= n) break;
      if (i2 != i1) emit(i1, i2);
      if (quadratic_overlap) emit(i1, static_cast<int64_t>(i1) + (k < 40 ? (int64_t{1} << k) : int64_t{1} << 40));
    }
  }
  return out;
}

std::array<double, 3> GpsToEcef(double lat_deg, double lon_deg, double alt) {
  const double a = 6378137.0, f = 1.0 / 298.257223563, b = a * (1.0 - f);   // WGS84
  const double e2 = (a * a - b * b) / (a * a);
  const double kDeg = 3.14159265358979323846 / 180.0;
  const double lat = lat_deg * kDeg, lon = lon_deg * kDeg;
  const double sl = std::sin(lat), cl = std::cos(lat);
  const double N = a / std::sqrt(1.0 - e2 * sl * sl);
  return {(N + alt) * cl * std::cos(lon), (N + alt) * cl * std::sin(lon), ((b * b) / (a * a) * N + alt) * sl};
}

PairList SpatialPairs(const std::vector<std::array<double, 3>>& prior_t, const std::vector<bool>& has_prior,
                      const SpatialMatchingOptions& o) {
  std::vector<int> idx;                       // images with a location prior
  std::vector<std::array<double, 3>> loc;
  for (size_t i = 0; i < prior_t.size(); ++i) {
    if (!has_prior[i]) continue;
    std::array<double, 3> p = prior_t[i];
    if (o.is_gps) p = GpsToEcef(p[0], p[1], o.ignore_z ? 0.0 : p[2]);
    else if (o.ignore_z) p[2] = 0.0;
    idx.push_back(static_cast<int>(i));
    loc.push_back(p);
  }
  PairList out;
  const int n = static_cast<int>(loc.size());
  const int knn = std::min(o.max_num_neighbors, n);
  const double max_d2 = o.max_distance * o.max_distance;
  std::vector<std::pair<double, int>> d(n);
  for (int i = 0; i < n; ++i) {
    for (int j = 0; j < n; ++j) {
      const double dx = loc[i][0] - loc[j][0], dy = loc[i][1] - loc[j][1], dz = loc[i][2] - loc[j][2];
      d[j] = {dx * dx + dy * dy + dz * dz, j};
    }
    std::partial_sort(d.begin(), d.begin() + knn, d.end());   // the knn nearest (the query itself included), by (distance, index)
    for (int k = 0; k < knn; ++k) {
      if (d[k].second == i) continue;
      if (d[k].first > max_d2) break;
      out.push_back(idx[i]);
      out.push_back(idx[d[k].second]);
    }
  }
  return out;
}

// ---- engine --------------------------------------------------------------------------------------
namespace {
std::mutex g_engine_mutex;
constexpr int kMaxDevices = 64;
b2m_ctx* g_ctx[kMaxDevices] = {};  // plain array: RequestStopAll must not take locks
}  // namespace

void ThrowOnError(b2m_ctx* ctx, int rc) {
  if (rc == B2M_OK) return;
  const char* m = b2m_last_error(ctx);
  const std::string msg = m ? m : "";
  switch (rc) {
    case B2M_EINVAL: throw std::invalid_argument(msg);  // -> ValueError, as THROW_CHECK (R:log_exceptions.h:114-147)
    case B2M_ESTOPPED: throw StoppedError();            // -> KeyboardInterrupt (R:helpers.h:306-347)
    case B2M_ENOMEM: throw std::bad_alloc();
    default: throw std::runtime_error("b200match error " + std::to_string(rc) + ": " + msg);
  }
}

std::vector<b2m_ctx*> Engine::GetAll(const std::vector<int>& devices) {
  std::vector<b2m_ctx*> out;
  for (int d : devices) out.push_back(Get(d));
  if (out.empty()) out.push_back(Get(0));
  return out;
}

b2m_ctx* Engine::Get(int device) {
  if (device < 0 || device >= kMaxDevices) throw std::invalid_argument("[controllers.cc] Check Failed: 0 <= gpu index < 64");
  std::lock_guard<std::mutex> lock(g_engine_mutex);
  if (!g_ctx[device]) {
    b2m_device_cfg cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.struct_size = sizeof(cfg);
    cfg.device = device;
    cfg.seed = 0;  // SetPRNGSeed(0) (R:estimators/essential_matrix.h:25)
    b2m_ctx* ctx = nullptr;
    ThrowOnError(nullptr, b2m_create(&cfg, &ctx));
    g_ctx[device] = ctx;
  }
  return g_ctx[device];
}

bool Engine::EnsureLocalComm(const std::vector<b2m_ctx*>& ctxs) {
  static std::vector<b2m_ctx*> current;   // the context list the live communicator spans
  std::lock_guard<std::mutex> lock(g_engine_mutex);
  if (ctxs.size() < 2) return false;
  if (current == ctxs) return true;
  current.clear();
  if (b2m_comm_init_local(ctxs.data(), static_cast<int32_t>(ctxs.size())) != B2M_OK) return false;  // no NCCL: full uploads
  current = ctxs;
  return true;
}

void Engine::RequestStopAll() {
  for (int i = 0; i < kMaxDevices; ++i)
    if (g_ctx[i]) b2m_request_stop(g_ctx[i]);
}

void Engine::DestroyAll() {
  std::lock_guard<std::mutex> lock(g_engine_mutex);
  for (int i = 0; i < kMaxDevices; ++i) {
    if (g_ctx[i]) b2m_destroy(g_ctx[i]);
    g_ctx[i] = nullptr;
  }
}

// ---- pipelines -----------------------------------------------------------------------------------
void CheckFileExists(const std::string& path, const char* where) {
  std::ifstream f(path, std::ios::binary);
  if (!f.good()) throw std::invalid_argument(std::string("[") + where + "] Check Failed: File " + path + " does not exist.");
}

namespace {

struct LoadedSet {
  std::vector<int64_t> ids;
  std::vector<std::string> names;
  std::vector<int64_t> camera_ids;
  std::vector<b2m_camera> cams;
  // filled by UploadImageSet
  std::vector<int32_t> n_feat;
  std::vector<std::vector<float>> xy;   // keypoint positions per image (kept for the multiple_models re-estimation)
  bool uploaded = false;
};

// The image table without the blobs: ids, names, cameras.  verify_matches needs no more than this plus the
// keypoints of the images its pairs name (upstream's FeatureMatcherCache reads descriptors lazily, only for pairs
// that must be matched: a database of learned-feature matches has no descriptor rows at all).
LoadedSet ReadImageTable(Database& db, bool order_by_name) {
  std::vector<ImageRow> images = db.ReadAllImages();
  if (order_by_name)
    std::stable_sort(images.begin(), images.end(), [](const ImageRow& a, const ImageRow& b) { return a.name < b.name; });
  LoadedSet L;
  std::unordered_map<int64_t, b2m_camera> cam_cache;
  for (const ImageRow& im : images) {
    L.ids.push_back(im.image_id);
    L.names.push_back(im.name);
    L.camera_ids.push_back(im.camera_id);
    auto it = cam_cache.find(im.camera_id);
    if (it == cam_cache.end()) it = cam_cache.emplace(im.camera_id, ToAbi(db.ReadCamera(im.camera_id))).first;
    L.cams.push_back(it->second);
  }
  return L;
}

std::vector<float> KeypointPositions(Database& db, int64_t image_id) {
  const KeypointsBlob kp = db.ReadKeypoints(image_id);
  std::vector<float> xy(static_cast<size_t>(kp.rows) * 2);
  for (int64_t r = 0; r < kp.rows; ++r) {
    xy[2 * r] = kp.data[r * kp.cols];
    xy[2 * r + 1] = kp.data[r * kp.cols + 1];
  }
  return xy;
}

// FeatureMatcherCache: every image's descriptors, keypoint positions and camera go to the GPU(s) once.  With
// several contexts that share a communicator (Engine::EnsureLocalComm) every GPU uploads only ITS contiguous share
// of the images over PCIe and ONE all-gather over NVLink makes the set resident everywhere
// (b2m_set_images_sharded); without NCCL every GPU uploads the whole set.
//
// An image with more than `max_num_matches` features is truncated to its first max_num_matches, with the warning
// upstream's GPU matcher prints (WarnIfMaxNumMatchesReachedGPU, U:feature/sift.cc): match indices stay valid
// because the kept features are a prefix.
void UploadImageSet(Database& db, const std::vector<b2m_ctx*>& ctxs, LoadedSet* L, int max_num_matches) {
  const double t_read0 = Now();
  const size_t n = L->ids.size();
  std::vector<DescriptorsBlob> desc(n);
  L->xy.assign(n, {});
  L->n_feat.assign(n, 0);
  for (size_t i = 0; i < n; ++i) {
    desc[i] = db.ReadDescriptors(L->ids[i]);
    L->xy[i] = KeypointPositions(db, L->ids[i]);
    if (static_cast<int64_t>(L->xy[i].size() / 2) != desc[i].rows)
      throw std::invalid_argument("[controllers.cc] Check Failed: keypoints.rows == descriptors.rows");
    if (desc[i].rows > max_num_matches) {
      fprintf(stderr, "W [controllers.cc] Clamping features from %lld to %d - consider increasing the maximum number of matches.\n",
              static_cast<long long>(desc[i].rows), max_num_matches);
      desc[i].rows = max_num_matches;
      desc[i].data.resize(static_cast<size_t>(max_num_matches) * 128);
      L->xy[i].resize(static_cast<size_t>(max_num_matches) * 2);
    }
    L->n_feat[i] = static_cast<int32_t>(desc[i].rows);
  }
  const int32_t n_images = static_cast<int32_t>(n);
  const double t_up0 = Now();
  g_timing.read_s += t_up0 - t_read0;
  std::vector<int> rc(ctxs.size(), B2M_OK);
  const bool sharded = ctxs.size() > 1 && Engine::EnsureLocalComm(ctxs);
  auto upload = [&](size_t d) {
    if (!sharded) {
      std::vector<const uint8_t*> dptr(n);
      std::vector<const float*> kptr(n);
      for (size_t i = 0; i < n; ++i) {
        dptr[i] = desc[i].data.data();
        kptr[i] = L->xy[i].data();
      }
      rc[d] = b2m_set_images(ctxs[d], n_images, L->n_feat.data(), dptr.data(), kptr.data(), L->cams.data());
      return;
    }
    int32_t first = 0, count = 0;
    b2m_comm_image_range(n_images, static_cast<int32_t>(ctxs.size()), static_cast<int32_t>(d), &first, &count);
    std::vector<uint8_t> dpack;
    std::vector<float> kpack;
    for (int32_t i = first; i < first + count; ++i) {
      dpack.insert(dpack.end(), desc[i].data.begin(), desc[i].data.end());
      kpack.insert(kpack.end(), L->xy[i].begin(), L->xy[i].end());
    }
    b2m_image_shard sh;
    memset(&sh, 0, sizeof(sh));
    sh.struct_size = sizeof(sh);
    sh.location = B2M_LOC_HOST;
    sh.first_image = first;
    sh.n_local = count;
    sh.has_keypoints = 1;
    sh.desc_packed = dpack.data();
    sh.kpts_packed = kpack.data();
    rc[d] = b2m_set_images_sharded(ctxs[d], n_images, L->n_feat.data(), L->cams.data(), &sh);
  };
  std::vector<std::thread> workers;
  for (size_t d = 1; d < ctxs.size(); ++d) workers.emplace_back(upload, d);
  upload(0);
  for (std::thread& w : workers) w.join();
  for (size_t d = 0; d < ctxs.size(); ++d) ThrowOnError(ctxs[d], rc[d]);
  L->uploaded = true;
  g_timing.upload_s += Now() - t_up0;
  g_timing.sharded_upload = sharded;
}

Mat3 ToMat3(const double* p) {
  Mat3 m;
  std::copy(p, p + 9, m.begin());
  return m;
}

struct ResultsGuard {
  b2m_results* r = nullptr;
  ~ResultsGuard() {
    if (r) b2m_results_free(r);
  }
};

// Verification of pairs whose raw matches are already in the database (verify_matches; pairs with stored matches
// but no geometry inside the match_* pipelines): keypoints of the named images only, ONE batched GPU call per
// 4096 pairs (b2m_estimate_two_view_geometry_batch), then the controller's write rule (row P3): raw matches below
// min_num_inliers are rewritten empty, geometries below min_num_inliers are stored as the default one.
void VerifyStoredPairs(Database& db, b2m_ctx* ctx, const LoadedSet& L, const std::vector<std::pair<int, int>>& pairs,
                       const b2m_tvg_opts& tvg) {
  constexpr size_t kChunk = 4096;
  std::unordered_map<int, std::vector<double>> pts;   // image index -> keypoint positions as doubles
  auto points_of = [&](int img) -> const std::vector<double>& {
    auto it = pts.find(img);
    if (it == pts.end()) {
      std::vector<float> xy;
      if (L.uploaded) xy = L.xy[img]; else xy = KeypointPositions(db, L.ids[img]);
      it = pts.emplace(img, std::vector<double>(xy.begin(), xy.end())).first;
    }
    return it->second;
  };
  for (size_t c0 = 0; c0 < pairs.size(); c0 += kChunk) {
    const size_t c1 = std::min(pairs.size(), c0 + kChunk);
    std::vector<std::vector<uint32_t>> mm(c1 - c0);
    std::vector<b2m_tvg_problem> prob;
    std::vector<size_t> prob_of;                       // index into the chunk
    pts.clear();
    for (size_t k = c0; k < c1; ++k) {
      mm[k - c0] = db.ReadMatches(L.ids[pairs[k].first], L.ids[pairs[k].second]);
      if (static_cast<int64_t>(mm[k - c0].size() / 2) < tvg.min_num_inliers) continue;
      points_of(pairs[k].first);
      points_of(pairs[k].second);
    }
    for (size_t k = c0; k < c1; ++k) {
      const std::vector<uint32_t>& m = mm[k - c0];
      if (static_cast<int64_t>(m.size() / 2) < tvg.min_num_inliers) continue;
      const std::vector<double>&p1 = pts.at(pairs[k].first), &p2 = pts.at(pairs[k].second);
      b2m_tvg_problem q;
      memset(&q, 0, sizeof(q));
      q.struct_size = sizeof(q);
      q.cam1 = L.cams[pairs[k].first];
      q.cam2 = L.cams[pairs[k].second];
      q.points1 = p1.data(); q.n1 = static_cast<int64_t>(p1.size() / 2);
      q.points2 = p2.data(); q.n2 = static_cast<int64_t>(p2.size() / 2);
      q.matches = m.data();  q.m = static_cast<int64_t>(m.size() / 2);
      prob.push_back(q);
      prob_of.push_back(k - c0);
    }
    std::vector<b2m_tvg_result> res(prob.size());
    std::vector<std::vector<uint32_t>> inl(prob.size());
    std::vector<uint32_t*> inl_ptr(prob.size());
    for (size_t j = 0; j < prob.size(); ++j) {
      inl[j].resize(static_cast<size_t>(std::max<int64_t>(1, prob[j].m)) * 2);
      inl_ptr[j] = inl[j].data();
    }
    if (!prob.empty()) {
      if (tvg.multiple_models) {   // the per-problem loop of EstimateMultipleTwoViewGeometries is sequential
        for (size_t j = 0; j < prob.size(); ++j) {
          memset(&res[j], 0, sizeof(res[j]));
          res[j].struct_size = sizeof(res[j]);
          ThrowOnError(ctx, b2m_estimate_two_view_geometry(ctx, &prob[j].cam1, prob[j].points1, prob[j].n1, &prob[j].cam2,
                                                           prob[j].points2, prob[j].n2, prob[j].matches, prob[j].m, &tvg,
                                                           &res[j], inl_ptr[j]));
        }
      } else {
        ThrowOnError(ctx, b2m_estimate_two_view_geometry_batch(ctx, prob.data(), static_cast<int64_t>(prob.size()), &tvg,
                                                               res.data(), inl_ptr.data()));
      }
    }
    std::vector<int> res_of(c1 - c0, -1);
    for (size_t j = 0; j < prob_of.size(); ++j) res_of[prob_of[j]] = static_cast<int>(j);
    DatabaseTransaction tx(&db);
    for (size_t k = c0; k < c1; ++k) {
      const int64_t id1 = L.ids[pairs[k].first], id2 = L.ids[pairs[k].second];
      const int j = res_of[k - c0];
      if (j < 0) {  // raw matches below min_num_inliers: stored empty, default geometry
        db.WriteMatches(id1, id2, nullptr, 0);
        db.WriteTwoViewGeometry(id1, id2, B2M_UNDEFINED, nullptr, 0, Mat3{}, Mat3{}, Mat3{}, {1.0, 0.0, 0.0, 0.0}, {0.0, 0.0, 0.0});
        continue;
      }
      const b2m_tvg_result& r = res[j];
      if (r.n_inliers < tvg.min_num_inliers) {
        db.WriteTwoViewGeometry(id1, id2, B2M_UNDEFINED, nullptr, 0, Mat3{}, Mat3{}, Mat3{}, {1.0, 0.0, 0.0, 0.0}, {0.0, 0.0, 0.0});
      } else {
        db.WriteTwoViewGeometry(id1, id2, r.config, inl[j].data(), r.n_inliers, ToMat3(r.F), ToMat3(r.E), ToMat3(r.H),
                                {r.qvec[0], r.qvec[1], r.qvec[2], r.qvec[3]}, {r.tvec[0], r.tvec[1], r.tvec[2]});
      }
    }
  }
}

// FeatureMatcherController::Match (row P3): skip self pairs, duplicates and pairs with both results
// stored; match + verify the rest on the GPU(s); write both tables in one transaction per chunk.
// With several contexts the chunk is cut into contiguous cost-balanced slices, one host thread per GPU
// (upstream: one matcher worker per entry of gpu_index); results are written in pair order, so the
// database does not depend on the number of GPUs.
void MatchPairsIntoDb(Database& db, const std::vector<b2m_ctx*>& ctxs, const LoadedSet& L,
                      const std::vector<PairList>& chunks, const b2m_sift_opts& sift, const b2m_tvg_opts& tvg,
                      bool skip_existing) {
  std::unordered_set<int64_t> have_m, have_g;
  if (skip_existing) {
    have_m = db.ExistingPairIds("matches");
    have_g = db.ExistingPairIds("two_view_geometries");
  }
  std::vector<std::pair<int, int>> stored_only;
  std::thread writer;
  std::exception_ptr writer_error;
  auto join_writer = [&]() {
    const double t0 = Now();
    if (writer.joinable()) writer.join();
    g_timing.write_wait_s += Now() - t0;
    if (writer_error) {
      std::exception_ptr e = writer_error;
      writer_error = nullptr;
      std::rethrow_exception(e);
    }
  };
  struct JoinOnExit {   // an exception on the GPU side must not leave a running thread behind (std::terminate)
    std::thread& t;
    ~JoinOnExit() {
      if (t.joinable()) t.join();
    }
  } join_on_exit{writer};
  for (const PairList& chunk : chunks) {
    PairList todo;
    for (size_t k = 0; k + 1 < chunk.size(); k += 2) {
      const int32_t a = chunk[k], b = chunk[k + 1];
      if (a == b) continue;
      const int64_t pid = ImagePairToPairId(L.ids[a], L.ids[b]);
      const bool has_m = have_m.count(pid) != 0, has_g = have_g.count(pid) != 0;
      have_m.insert(pid);
      have_g.insert(pid);
      if (has_m && has_g) continue;
      if (has_m) {  // stored (imported / custom) matches without a geometry: verified as they are, never re-matched
        stored_only.push_back({a, b});
        continue;
      }
      todo.push_back(a);
      todo.push_back(b);
    }
    if (!stored_only.empty()) {
      join_writer();   // one writer at a time on the connection
      VerifyStoredPairs(db, ctxs[0], L, stored_only, tvg);
      stored_only.clear();
    }
    if (todo.empty()) continue;
    const std::vector<int64_t> cut = SplitPairsByCost(todo, L.n_feat, static_cast<int>(ctxs.size()));
    std::vector<ResultsGuard> res(ctxs.size());
    std::vector<int> rc(ctxs.size(), B2M_OK);
    // TwoViewGeometryOptions.multiple_models: the batched verifier finds one geometry per pair; the pairs it
    // verified are then re-estimated through the estimator entry point, which runs upstream's
    // estimate / remove inliers / repeat loop (EstimateMultipleTwoViewGeometries) on the raw matches.
    b2m_tvg_opts tvg_batch = tvg;
    tvg_batch.multiple_models = 0;
    auto run = [&](size_t d) {
      const int64_t n = cut[d + 1] - cut[d];
      if (n > 0) rc[d] = b2m_match_pairs(ctxs[d], todo.data() + 2 * cut[d], n, &sift, &tvg_batch, &res[d].r);
    };
    const double t_gpu0 = Now();
    std::vector<std::thread> workers;
    for (size_t d = 1; d < ctxs.size(); ++d) workers.emplace_back(run, d);
    run(0);
    for (std::thread& w : workers) w.join();
    g_timing.gpu_s += Now() - t_gpu0;
    g_timing.pairs += static_cast<int64_t>(todo.size() / 2);
    for (size_t d = 0; d < ctxs.size(); ++d) {
      if (rc[d] != B2M_OK) join_writer();   // do not leave the writer running behind an exception
      ThrowOnError(ctxs[d], rc[d]);
    }
    // The chunk's results go to the database on a WRITER THREAD, one transaction per chunk, while the GPU(s) work on
    // the next chunk (SURVEY.md section 7 item 7).  multiple_models re-estimates on the GPU while writing: that stays
    // on this thread (one in-flight call per context).
    auto results = std::make_shared<std::vector<ResultsGuard>>(std::move(res));
    auto todo_p = std::make_shared<PairList>(std::move(todo));
    auto write_chunk = [&db, &ctxs, &L, &tvg, results, todo_p, cut]() {
      const double t0 = Now();
      const PairList& todo = *todo_p;
      DatabaseTransaction tx(&db);
      for (size_t d = 0; d < ctxs.size(); ++d) {
        b2m_results* r_d = (*results)[d].r;
        const int64_t n = r_d ? b2m_results_num_pairs(r_d) : 0;
        for (int64_t k = 0; k < n; ++k) {
          b2m_pair_view v;
          memset(&v, 0, sizeof(v));
          v.struct_size = sizeof(v);
          ThrowOnError(ctxs[d], b2m_results_get(r_d, k, &v));
          const int32_t a = todo[2 * (cut[d] + k)], b = todo[2 * (cut[d] + k) + 1];
          const int64_t id1 = L.ids[a], id2 = L.ids[b];
          db.WriteMatches(id1, id2, v.matches, v.n_matches);
          if (tvg.multiple_models && v.config != B2M_UNDEFINED && v.n_matches > 0) {
            auto as_double = [](const std::vector<float>& f) { return std::vector<double>(f.begin(), f.end()); };
            const std::vector<double> p1 = as_double(L.xy[a]), p2 = as_double(L.xy[b]);
            b2m_tvg_result r;
            memset(&r, 0, sizeof(r));
            r.struct_size = sizeof(r);
            std::vector<uint32_t> inl(static_cast<size_t>(v.n_matches) * 2);
            ThrowOnError(ctxs[d], b2m_estimate_two_view_geometry(ctxs[d], &L.cams[a], p1.data(), static_cast<int64_t>(p1.size() / 2),
                                                                 &L.cams[b], p2.data(), static_cast<int64_t>(p2.size() / 2),
                                                                 v.matches, v.n_matches, &tvg, &r, inl.data()));
            const bool keep = r.n_inliers >= tvg.min_num_inliers;   // controller write rule (row P3)
            db.WriteTwoViewGeometry(id1, id2, keep ? r.config : B2M_UNDEFINED, inl.data(), keep ? r.n_inliers : 0,
                                    keep ? ToMat3(r.F) : Mat3{}, keep ? ToMat3(r.E) : Mat3{}, keep ? ToMat3(r.H) : Mat3{},
                                    {r.qvec[0], r.qvec[1], r.qvec[2], r.qvec[3]}, {r.tvec[0], r.tvec[1], r.tvec[2]});
            continue;
          }
          db.WriteTwoViewGeometry(id1, id2, v.config, v.inlier_matches, v.n_inliers, ToMat3(v.F), ToMat3(v.E),
                                  ToMat3(v.H), {v.qvec[0], v.qvec[1], v.qvec[2], v.qvec[3]}, {v.tvec[0], v.tvec[1], v.tvec[2]});
        }
      }
      g_timing.write_s += Now() - t0;
    };
    join_writer();                       // the previous chunk's transaction is committed before the next one opens
    if (tvg.multiple_models) {
      write_chunk();
    } else {
      writer = std::thread([write_chunk, &writer_error]() {
        try {
          write_chunk();
        } catch (...) {
          writer_error = std::current_exception();
        }
      });
    }
  }
  join_writer();
}

// Concatenate block pair lists into chunks of >= `target` pairs: one GPU call + one transaction each.
std::vector<PairList> Chunked(const std::vector<PairList>& blocks, size_t target = 16384) {
  std::vector<PairList> out;
  PairList cur;
  for (const PairList& b : blocks) {
    cur.insert(cur.end(), b.begin(), b.end());
    if (cur.size() / 2 >= target) {
      out.push_back(std::move(cur));
      cur.clear();
    }
  }
  if (!cur.empty()) out.push_back(std::move(cur));
  return out;
}

}  // namespace

void MatchExhaustive(const std::string& database_path, const SiftMatchingOptions& sift,
                     const ExhaustiveMatchingOptions& matching, const TwoViewGeometryOptions& verification,
                     const std::vector<int>& devices) {
  g_timing = PipelineTiming{};
  const double t_total0 = Now();
  struct Total { double t0; ~Total() { g_timing.total_s = Now() - t0; } } total_guard{t_total0};
  CheckFileExists(database_path, "match_features.h:32");
  if (matching.block_size <= 1) throw std::invalid_argument("[controllers.cc] Check Failed: block_size > 1");
  const std::vector<b2m_ctx*> ctxs = Engine::GetAll(devices);
  Database db(database_path);
  LoadedSet L = ReadImageTable(db, /*order_by_name=*/false);
  UploadImageSet(db, ctxs, &L, sift.max_num_matches);
  MatchPairsIntoDb(db, ctxs, L, Chunked(ExhaustivePairBlocks(static_cast<int>(L.ids.size()), matching.block_size)),
                   ToAbi(sift), ToAbi(verification), /*skip_existing=*/true);
}

void MatchSequential(const std::string& database_path, const SiftMatchingOptions& sift,
                     const SequentialMatchingOptions& matching, const TwoViewGeometryOptions& verification,
                     const std::vector<int>& devices) {
  g_timing = PipelineTiming{};
  const double t_total0 = Now();
  struct Total { double t0; ~Total() { g_timing.total_s = Now() - t0; } } total_guard{t_total0};
  CheckFileExists(database_path, "match_features.h:32");
  if (matching.loop_detection)
    throw std::invalid_argument("[controllers.cc] loop_detection needs a vocabulary tree: out of scope (SURVEY.md row B6)");
  if (matching.overlap < 1) throw std::invalid_argument("[controllers.cc] Check Failed: overlap > 0");
  const std::vector<b2m_ctx*> ctxs = Engine::GetAll(devices);
  Database db(database_path);
  LoadedSet L = ReadImageTable(db, /*order_by_name=*/true);
  UploadImageSet(db, ctxs, &L, sift.max_num_matches);
  MatchPairsIntoDb(db, ctxs, L,
                   {SequentialPairs(static_cast<int>(L.ids.size()), matching.overlap, matching.quadratic_overlap)},
                   ToAbi(sift), ToAbi(verification), /*skip_existing=*/true);
}

void MatchSpatial(const std::string& database_path, const SiftMatchingOptions& sift, const SpatialMatchingOptions& matching,
                  const TwoViewGeometryOptions& verification, const std::vector<int>& devices) {
  g_timing = PipelineTiming{};
  const double t_total0 = Now();
  struct Total { double t0; ~Total() { g_timing.total_s = Now() - t0; } } total_guard{t_total0};
  CheckFileExists(database_path, "match_features.h:32");
  if (matching.max_num_neighbors < 1) throw std::invalid_argument("[controllers.cc] Check Failed: max_num_neighbors > 0");
  if (!(matching.max_distance > 0.0)) throw std::invalid_argument("[controllers.cc] Check Failed: max_distance > 0");
  const std::vector<b2m_ctx*> ctxs = Engine::GetAll(devices);
  Database db(database_path);
  LoadedSet L = ReadImageTable(db, /*order_by_name=*/false);
  UploadImageSet(db, ctxs, &L, sift.max_num_matches);
  std::vector<std::array<double, 3>> prior_t;
  std::vector<bool> has_prior;
  db.ReadLocationPriors(&prior_t, &has_prior);   // same order as ReadAllImages (image_id)
  // the controller drops the pairs it has seen already, (a, b) and (b, a) alike: both map to one pair_id
  MatchPairsIntoDb(db, ctxs, L, {SpatialPairs(prior_t, has_prior, matching)}, ToAbi(sift), ToAbi(verification),
                   /*skip_existing=*/true);
}

void VerifyMatches(const std::string& database_path, const std::string& pairs_path,
                   const TwoViewGeometryOptions& options) {
  g_timing = PipelineTiming{};
  const double t_total0 = Now();
  struct Total { double t0; ~Total() { g_timing.total_s = Now() - t0; } } total_guard{t_total0};
  CheckFileExists(database_path, "match_features.h:54");
  CheckFileExists(pairs_path, "match_features.h:55");
  b2m_ctx* ctx = Engine::Get(0);
  Database db(database_path);
  LoadedSet L = ReadImageTable(db, /*order_by_name=*/false);   // no descriptors, no keypoints yet
  std::unordered_map<std::string, int> index_of;
  for (size_t i = 0; i < L.names.size(); ++i) index_of[L.names[i]] = static_cast<int>(i);

  // pair list: `name1 name2` per line; unknown names, self pairs and repeats are skipped like upstream
  std::vector<std::pair<int, int>> todo_verify;
  PairList todo_match;
  std::set<std::pair<int, int>> seen;
  std::ifstream f(pairs_path);
  std::string line;
  while (std::getline(f, line)) {
    std::istringstream ss(line);
    std::string n1, n2;
    if (!(ss >> n1) || n1[0] == '#' || !(ss >> n2)) continue;
    const auto a = index_of.find(n1), b = index_of.find(n2);
    if (a == index_of.end() || b == index_of.end() || a->second == b->second) continue;
    if (!seen.insert({std::min(a->second, b->second), std::max(a->second, b->second)}).second) continue;
    const bool has_m = db.ExistsMatches(L.ids[a->second], L.ids[b->second]);
    const bool has_g = db.ExistsInlierMatches(L.ids[a->second], L.ids[b->second]);
    if (has_m && has_g) continue;
    if (has_m) {
      todo_verify.push_back({a->second, b->second});
    } else {
      todo_match.push_back(a->second);
      todo_match.push_back(b->second);
    }
  }
  const b2m_tvg_opts tvg = ToAbi(options);
  if (!todo_match.empty()) {   // only now are descriptors needed (and keypoints.rows == descriptors.rows enforced)
    UploadImageSet(db, {ctx}, &L, SiftMatchingOptions().max_num_matches);
    MatchPairsIntoDb(db, {ctx}, L, {todo_match}, ToAbi(SiftMatchingOptions()), tvg, /*skip_existing=*/false);
  }
  VerifyStoredPairs(db, ctx, L, todo_verify, tvg);
}

}  // namespace b2mh
