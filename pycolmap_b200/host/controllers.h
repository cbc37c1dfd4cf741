// controllers.h -- host side of the matching / verification pipelines, above the C ABI
// (include/b200match.h).  What the reference's bound functions do around COLMAP's controllers:
//   MatchFeatures<Opts, Factory>        R:pipeline/match_features.h:22-49
//   verify_matches                      R:pipeline/match_features.h:51-68
//   option structs                      R:pipeline/match_features.h:71-152, R:estimators/two_view_geometry.h:41-65,
//                                       R:optim/bindings.h:7-27
// and what the controllers themselves do on the host (pair generation, database I/O, write rules;
// U:controllers/feature_matching.cc, U:controllers/feature_matching_utils.cc; SURVEY.md rows P1-P3).
// All arithmetic happens behind the C ABI on the GPU; nothing here touches a descriptor or a match
// except to move it between SQLite and libb200match.so.
#pragma once
#include <array>
#include <cstdint>
#include <string>
#include <utility>
#include <vector>

#include "../../include/b200match.h"
#include "database.h"

namespace b2mh {

// ---- option structs (field names, defaults = the C++ structs the reference binds) ---------------
struct SiftMatchingOptions {
  int num_threads = -1;
  std::string gpu_index = "-1";
  double max_ratio = 0.8;
  double max_distance = 0.7;
  bool cross_check = true;
  int max_num_matches = 32768;
  bool guided_matching = false;
};

struct ExhaustiveMatchingOptions {
  int block_size = 50;
};

struct SequentialMatchingOptions {
  int overlap = 10;
  bool quadratic_overlap = true;
  bool loop_detection = false;
  int loop_detection_period = 10;
  int loop_detection_num_images = 50;
  int loop_detection_num_nearest_neighbors = 1;
  int loop_detection_num_checks = 256;
  int loop_detection_num_images_after_verification = 0;
  int loop_detection_max_num_features = -1;
  std::string vocab_tree_path;
};

// SpatialMatchingOptions (R:pipeline/match_features.h:154-174; defaults U:controllers/feature_matching.h)
struct SpatialMatchingOptions {
  bool is_gps = true;        // priors are (latitude, longitude, altitude) in degrees / metres
  bool ignore_z = true;
  int max_num_neighbors = 50;
  double max_distance = 100.0;  // metres
};

// Defaults = what `pycolmap.RANSACOptions()` constructs (R:optim/bindings.h:10-18).
struct RANSACOptions {
  double max_error = 4.0;
  double min_inlier_ratio = 0.01;
  double confidence = 0.9999;
  double dyn_num_trials_multiplier = 3.0;
  int min_num_trials = 1000;
  int max_num_trials = 100000;
};

// `ransac` keeps the values the C++ constructor of colmap::TwoViewGeometryOptions sets
// (py::init<>() at R:estimators/two_view_geometry.h:43 runs that constructor).
struct TwoViewGeometryOptions {
  int min_num_inliers = 15;
  double min_E_F_inlier_ratio = 0.95;
  double max_H_inlier_ratio = 0.8;
  double watermark_min_inlier_ratio = 0.7;
  double watermark_border_size = 0.1;
  bool detect_watermark = true;
  bool multiple_ignore_watermark = true;
  bool force_H_use = false;
  bool compute_relative_pose = false;
  bool multiple_models = false;
  RANSACOptions ransac{4.0, 0.25, 0.999, 3.0, 100, 10000};
};

b2m_sift_opts ToAbi(const SiftMatchingOptions& o);
b2m_ransac_opts ToAbi(const RANSACOptions& o);
b2m_tvg_opts ToAbi(const TwoViewGeometryOptions& o);
// Database camera -> ABI camera; throws std::invalid_argument for models the verifier does not take.
b2m_camera ToAbi(const CameraRow& c);
// SiftMatchingOptions.gpu_index: comma-separated CUDA ordinals, "0,1,2,3" = one matcher per listed GPU
// (R:pipeline/match_features.h:76-81).  Duplicates are dropped, order kept.  "-1" (the default) expands to
// every visible sm_90 device like upstream (b2m_device_count; device 0 when the count cannot be had).
std::vector<int> ParseGpuIndices(const std::string& gpu_index);

// ---- pair generators (rows P1, P2) -------------------------------------------------------------
using PairList = std::vector<int32_t>;  // [n x 2] image indices, flattened

// ExhaustiveFeatureMatcher::Run order: block pairs (s1, s2) row-major, inside a block pair i1-major;
// each unordered pair appears exactly once over the whole grid.  One PairList per non-empty block pair.
std::vector<PairList> ExhaustivePairBlocks(int n_images, int block_size);
// SequentialFeatureMatcher::Run: (i1, i1+1+k) and, with quadratic_overlap, (i1, i1+2^k), k < overlap;
// out-of-range dropped, duplicates removed, generation order kept.
PairList SequentialPairs(int n_images, int overlap, bool quadratic_overlap);

// Cut `pairs` into `parts` contiguous slices of about equal cost (cost of a pair = n_feat[a] * n_feat[b],
// the size of its distance matrix).  Returns parts + 1 offsets (in pairs), cut[0] = 0, cut[parts] = n.
std::vector<int64_t> SplitPairsByCost(const PairList& pairs, const std::vector<int32_t>& n_feat, int parts);

// SpatialFeatureMatcher::Run (row f4): every image with a location prior is paired with its nearest neighbours
// among the images with priors -- the k = min(max_num_neighbors, #locations) nearest including itself, skipping
// itself, stopping at max_distance.  GPS priors go through WGS84 ellipsoid -> ECEF first.  Indices are positions
// in the image list; pairs are emitted per query image in order of increasing distance, duplicates across
// queries are left to the controller (which skips pairs it has already seen).
PairList SpatialPairs(const std::vector<std::array<double, 3>>& prior_t, const std::vector<bool>& has_prior,
                      const SpatialMatchingOptions& options);
std::array<double, 3> GpsToEcef(double lat_deg, double lon_deg, double alt);  // WGS84

// ---- engine: one b2m_ctx per process and GPU -----------------------------------------------------
class Engine {
 public:
  // Lazily creates the context; throws std::runtime_error / std::invalid_argument with b2m_last_error().
  static b2m_ctx* Get(int device);
  static std::vector<b2m_ctx*> GetAll(const std::vector<int>& devices);
  // One NCCL communicator over the given contexts (b2m_comm_init_local), created once per context list.  False
  // when NCCL is not available: callers then upload the whole image set to every GPU instead of sharding it.
  static bool EnsureLocalComm(const std::vector<b2m_ctx*>& ctxs);
  static void RequestStopAll();  // async-signal-safe flags only (b2m_request_stop on every live context)
  static void DestroyAll();
};

// Throws the C++ exception that pybind11 maps to the Python type the reference raises for this code.
void ThrowOnError(b2m_ctx* ctx, int rc);

struct StoppedError : std::exception {
  const char* what() const noexcept override { return "stopped"; }
};

// THROW_CHECK_FILE_EXISTS (R:log_exceptions.h:137-141): std::invalid_argument -> ValueError,
// message "[<where>] Check Failed: File <path> does not exist."
void CheckFileExists(const std::string& path, const char* where);

// Wall-clock breakdown of the last pipeline call of this process (DB-inclusive end-to-end, SURVEY.md section 7 item 7):
// reading the database, uploading to the GPU(s), the b2m_match_pairs calls, writing (on the writer thread, overlapped
// with the GPU) and the time the GPU side had to wait for the writer.
struct PipelineTiming {
  double read_s = 0, upload_s = 0, gpu_s = 0, write_s = 0, write_wait_s = 0, total_s = 0;
  int64_t pairs = 0;
  bool sharded_upload = false;
};
PipelineTiming LastPipelineTiming();

// ---- pipelines -----------------------------------------------------------------------------------
void MatchExhaustive(const std::string& database_path, const SiftMatchingOptions& sift,
                     const ExhaustiveMatchingOptions& matching, const TwoViewGeometryOptions& verification,
                     const std::vector<int>& devices);
void MatchSequential(const std::string& database_path, const SiftMatchingOptions& sift,
                     const SequentialMatchingOptions& matching, const TwoViewGeometryOptions& verification,
                     const std::vector<int>& devices);
void MatchSpatial(const std::string& database_path, const SiftMatchingOptions& sift, const SpatialMatchingOptions& matching,
                  const TwoViewGeometryOptions& verification, const std::vector<int>& devices);
void VerifyMatches(const std::string& database_path, const std::string& pairs_path,
                   const TwoViewGeometryOptions& options);

}  // namespace b2mh
