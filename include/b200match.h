/* b200match.h -- C ABI of libb200match.so (H100 / sm_90a exhaustive matcher + two-view verifier).
 *
 * This is the drop-in boundary for the hot path of pycolmap.match_exhaustive /
 * match_sequential / verify_matches / estimate_two_view_geometry.  Every entry point
 * cites the reference interface it replaces.  Citation tags:
 *   R:<path>:<lines>  file under /root/reference (colmap/pycolmap @ b6627db)
 *   U:<path>          upstream COLMAP 3.9.1 (the un-vendored dependency the reference
 *                     forwards into, R:CMakeLists.txt:17, R:pyproject.toml:36)
 *
 * Rules of the ABI: plain C structs, `struct_size` first (forward compatibility), plain
 * pointers + sizes, no exceptions, no STL, no torch / Python types.  All functions return
 * 0 on success or a negative B2M_E* code; the message is in b2m_last_error().  The caller
 * owns every input buffer (the library copies what it keeps); the library owns a
 * b2m_results until b2m_results_free().  One in-flight call per context.
 *
 * There is NO CPU fallback: b2m_create() fails with B2M_ENODEV when no sm_90 device is
 * visible.
 */
#ifndef B200MATCH_H_
#define B200MATCH_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2M_ABI_VERSION 3   /* 2: b2m_camera carries 12 parameters, batch estimator; 3: multi-GPU entry points (NCCL) */

/* error codes */
#define B2M_OK 0
#define B2M_EINVAL (-1)   /* bad argument (reference: THROW_CHECK -> ValueError, R:log_exceptions.h:114-147) */
#define B2M_ENODEV (-2)   /* no CUDA device / not sm_90 (reference: VerifyGPUParams, R:utils.h:22-31) */
#define B2M_ECUDA (-3)    /* CUDA runtime / driver error */
#define B2M_ENOMEM (-4)
#define B2M_ESTOPPED (-5) /* b2m_request_stop() honoured (reference: PyInterrupt, R:helpers.h:306-347) */
#define B2M_ESTATE (-6)   /* call order violated (e.g. match before set_images) */

typedef struct b2m_ctx b2m_ctx;
typedef struct b2m_results b2m_results;

/* ---- context ----------------------------------------------------------------------- */

typedef struct b2m_device_cfg {
  uint32_t struct_size;
  int32_t device;        /* CUDA ordinal; replaces SiftMatchingOptions.gpu_index (R:pipeline/match_features.h:76-81) */
  uint64_t seed;         /* RANSAC seed; replaces SetPRNGSeed(0) (R:estimators/essential_matrix.h:25) */
  int32_t pair_batch;    /* image pairs per kernel batch; 0 = default: 4096 for 8192-feature images, proportionally more for
                          * smaller ones (1024 .. 16384).  Results do not depend on it (RANSAC is keyed by image ids). */
  int32_t reserved;
} b2m_device_cfg;

int b2m_abi_version(void);
/* Number of visible sm_90 devices (what SiftMatchingOptions.gpu_index = "-1" expands to, R:pipeline/match_features.h:76-81);
 * 0 without a driver or a suitable device. */
int b2m_device_count(void);
int b2m_create(const b2m_device_cfg* cfg, b2m_ctx** out);
void b2m_destroy(b2m_ctx* ctx);
/* Message of the last failing call on this context (ctx may be NULL for create failures). */
const char* b2m_last_error(const b2m_ctx* ctx);
/* Async-signal-safe stop flag, checked between batches (R:helpers.h:335-347 PyWait / Thread::Stop). */
int b2m_request_stop(b2m_ctx* ctx);

/* ---- options ------------------------------------------------------------------------ */

/* SiftMatchingOptions (R:pipeline/match_features.h:71-100; defaults U:feature/sift.h). */
typedef struct b2m_sift_opts {
  uint32_t struct_size;
  float max_ratio;        /* 0.8 */
  float max_distance;     /* 0.7 */
  int32_t cross_check;    /* 1 */
  int32_t max_num_matches;/* 32768: upper bound on descriptors per image taken into account */
  int32_t guided_matching;/* 0 */
} b2m_sift_opts;

/* RANSACOptions (R:optim/bindings.h:7-27; U:optim/ransac.h). */
typedef struct b2m_ransac_opts {
  uint32_t struct_size;
  int32_t min_num_trials;           /* 100  */
  int32_t max_num_trials;           /* 10000 */
  int32_t reserved;
  double max_error;                 /* 4.0  */
  double min_inlier_ratio;          /* 0.25 */
  double confidence;                /* 0.999 */
  double dyn_num_trials_multiplier; /* 3.0  */
} b2m_ransac_opts;

/* TwoViewGeometryOptions (R:estimators/two_view_geometry.h:41-65; U:estimators/two_view_geometry.h). */
typedef struct b2m_tvg_opts {
  uint32_t struct_size;
  int32_t min_num_inliers;            /* 15 */
  double min_E_F_inlier_ratio;        /* 0.95 */
  double max_H_inlier_ratio;          /* 0.8 */
  double watermark_min_inlier_ratio;  /* 0.7 */
  double watermark_border_size;       /* 0.1 */
  int32_t detect_watermark;           /* 1 */
  int32_t multiple_ignore_watermark;  /* 1 */
  int32_t force_H_use;                /* 0 */
  int32_t compute_relative_pose;      /* 0; 1: also EstimateTwoViewGeometryPose (qvec, tvec, tri_angle; may turn
                                       * PLANAR_OR_PANORAMIC into PLANAR / PANORAMIC) */
  int32_t multiple_models;            /* 0 */
  int32_t reserved;
  b2m_ransac_opts ransac;
} b2m_tvg_opts;

void b2m_sift_opts_default(b2m_sift_opts* o);
void b2m_ransac_opts_default(b2m_ransac_opts* o);
void b2m_tvg_opts_default(b2m_tvg_opts* o);

/* TwoViewGeometryConfiguration (R:estimators/two_view_geometry.h:67-80). */
enum b2m_tvg_config {
  B2M_UNDEFINED = 0,
  B2M_DEGENERATE = 1,
  B2M_CALIBRATED = 2,
  B2M_UNCALIBRATED = 3,
  B2M_PLANAR = 4,
  B2M_PANORAMIC = 5,
  B2M_PLANAR_OR_PANORAMIC = 6,
  B2M_WATERMARK = 7,
  B2M_MULTIPLE = 8
};

/* Camera (the part of R:scene/camera.h:20-213 the verifier touches: CamFromImg, CamFromImgThreshold,
 * MeanFocalLength, width / height, has_prior_focal_length).  `model` and the parameter order are
 * COLMAP's (U:sensor/models.h): 0 SIMPLE_PINHOLE (f, cx, cy), 1 PINHOLE (fx, fy, cx, cy),
 * 2 SIMPLE_RADIAL (f, cx, cy, k), 3 RADIAL (f, cx, cy, k1, k2), 4 OPENCV (fx, fy, cx, cy, k1, k2, p1, p2),
 * 5 OPENCV_FISHEYE (fx, fy, cx, cy, k1, k2, k3, k4), 6 FULL_OPENCV (fx, fy, cx, cy, k1, k2, p1, p2, k3, k4, k5, k6),
 * 7 FOV (fx, fy, cx, cy, omega), 8 SIMPLE_RADIAL_FISHEYE (f, cx, cy, k), 9 RADIAL_FISHEYE (f, cx, cy, k1, k2),
 * 10 THIN_PRISM_FISHEYE (fx, fy, cx, cy, k1, k2, p1, p2, k3, k4, sx1, sy1).  Other ids are rejected with
 * B2M_EINVAL.  Unused params must be 0. */
#define B2M_CAMERA_MAX_PARAMS 12
typedef struct b2m_camera {
  uint32_t struct_size;
  int32_t model;
  int32_t width, height;
  int32_t has_prior_focal_length;
  int32_t reserved;
  double params[B2M_CAMERA_MAX_PARAMS];
} b2m_camera;

/* ---- single-pair entry points (the unit the reference's workers call) -------------- */

/* Replaces FeatureMatcher::Match(descriptors1, descriptors2, &matches)
 * (U:feature/sift.cc MatchSiftFeaturesCPUBruteForce semantics; called from
 * U:controllers/feature_matching_utils.cc FeatureMatcherWorker::Run; reached from
 * R:pipeline/match_features.h:45-48).
 * desc1/desc2: HOST pointers, [n x 128] uint8 row-major.  out_matches: HOST buffer of
 * capacity `cap` (idx1, idx2) uint32 pairs (PyFeatureMatches layout, R:estimators/two_view_geometry.h:19-38);
 * *out_n receives the number of matches (sorted by idx1 ascending). */
int b2m_match_pair(b2m_ctx* ctx, const uint8_t* desc1, int32_t n1, const uint8_t* desc2, int32_t n2,
                   const b2m_sift_opts* opts, uint32_t* out_matches, int64_t cap, int64_t* out_n);

/* ---- image-set path (exhaustive / sequential / pair-list pipelines) ---------------- */

/* Upload the descriptor set once; it stays resident in HBM (replaces FeatureMatcherCache,
 * U:controllers/feature_matching_utils.cc).  desc[i]: HOST [n_feat[i] x 128] uint8.
 * kpts[i]: HOST [n_feat[i] x 2] float32 (x, y) or kpts == NULL for match-only.
 * cams: one per image, or NULL for match-only. */
int b2m_set_images(b2m_ctx* ctx, int32_t n_images, const int32_t* n_feat, const uint8_t* const* desc,
                   const float* const* kpts, const b2m_camera* cams);

/* Same, but the descriptors already live in device memory as one packed array
 * [sum(n_feat) x 128] (row-major, image after image).  Used by the multi-GPU path after the
 * NCCL all-gather and by benchmarks that keep inputs resident in HBM. */
int b2m_set_images_device(b2m_ctx* ctx, int32_t n_images, const int32_t* n_feat, const void* dev_desc_packed,
                          const void* dev_kpts_packed /* float2 per feature or NULL */, const b2m_camera* cams);

/* Match (and verify when tvg != NULL) a list of image pairs given as indices into the image
 * set.  Replaces FeatureMatcherController::Match (U:controllers/feature_matching_utils.cc)
 * as driven by Exhaustive/Sequential/ImagePairs FeatureMatcher::Run
 * (U:controllers/feature_matching.cc; R:pipeline/match_features.h:22-68).  Blocking. */
int b2m_match_pairs(b2m_ctx* ctx, const int32_t* pairs /* [n_pairs x 2] */, int64_t n_pairs,
                    const b2m_sift_opts* sift, const b2m_tvg_opts* tvg /* NULL = match only */,
                    b2m_results** out);
/* The same entry point under the name SURVEY.md section 8(b) gives it. */
int b2m_match_verify(b2m_ctx* ctx, const int32_t* pairs, int64_t n_pairs, const b2m_sift_opts* sift,
                     const b2m_tvg_opts* tvg, b2m_results** out);

typedef struct b2m_pair_view {
  uint32_t struct_size;
  int32_t image1, image2;
  int32_t config;                /* enum b2m_tvg_config; B2M_UNDEFINED when not verified */
  int64_t n_matches;
  const uint32_t* matches;       /* [n_matches x 2] raw matches (idx1, idx2), idx1 ascending */
  int64_t n_inliers;
  const uint32_t* inlier_matches;/* [n_inliers x 2] */
  double E[9], F[9], H[9];       /* row-major, zero when not estimated */
  /* relative pose, filled when b2m_tvg_opts.compute_relative_pose (TwoViewGeometry::cam2_from_cam1, tri_angle;
   * R:estimators/two_view_geometry.h:82-93): x_cam2 = R(qvec) x_cam1 + tvec, qvec = (w, x, y, z) */
  double qvec[4], tvec[3];
  double tri_angle;              /* median triangulation angle of the inliers, radians */
  int32_t pose_valid;            /* 0: not requested / not recoverable (qvec = identity, tvec = 0) */
  int32_t reserved;
} b2m_pair_view;

int64_t b2m_results_num_pairs(const b2m_results* r);
int64_t b2m_results_total_matches(const b2m_results* r);
/* Number of pairs whose stored geometry is not the default one (config != UNDEFINED), i.e. pairs the
 * controller would write a verified TwoViewGeometry for (U:controllers/feature_matching_utils.cc). */
int64_t b2m_results_num_verified(const b2m_results* r);
int b2m_results_get(const b2m_results* r, int64_t pair, b2m_pair_view* out);
void b2m_results_free(b2m_results* r);

/* ---- multi-GPU: image pairs shard across GPUs, ONE all-gather of the descriptor set ----- */

/* Replaces upstream's "one matcher thread per entry of SiftMatchingOptions.gpu_index, every worker reads every image
 * from the host-side FeatureMatcherCache" (U:controllers/feature_matching_utils.cc; gpu_index list:
 * R:pipeline/match_features.h:76-81).  Here every GPU has one b2m_ctx -- in one process (a host thread per GPU, like
 * upstream) or in one process per GPU (torchrun / MPI) -- uploads only ITS contiguous share of the images and a single
 * NCCL all-gather over NVLink makes the whole set resident everywhere; pairs then shard freely, no further exchange.
 * NCCL (libnccl.so.2) is bound at run time; without it these calls fail with B2M_ENODEV and nothing else changes. */
#define B2M_COMM_ID_BYTES 128
typedef struct b2m_comm_id {
  uint8_t bytes[B2M_COMM_ID_BYTES];   /* ncclUniqueId */
} b2m_comm_id;
/* Rank 0 creates the id; the launcher's side channel (torchrun store, MPI_Bcast, a file) carries it to the other ranks. */
int b2m_comm_get_unique_id(b2m_comm_id* out);
/* Collective over all ranks: joins the communicator of `id` with this context's device as rank `rank` of `n_ranks`. */
int b2m_comm_init_rank(b2m_ctx* ctx, int32_t n_ranks, int32_t rank, const b2m_comm_id* id);
/* Single-process form: contexts on distinct devices of this process, rank = position in `ctxs`. */
int b2m_comm_init_local(b2m_ctx* const* ctxs, int32_t n);
int b2m_comm_destroy(b2m_ctx* ctx);
/* The partition every rank must agree on: rank r owns the contiguous images [first, first + count) with
 * ceil(n_images / n_ranks) images per rank (the last ranks may own fewer, or none). */
void b2m_comm_image_range(int32_t n_images, int32_t n_ranks, int32_t rank, int32_t* first, int32_t* count);

#define B2M_LOC_HOST 0
#define B2M_LOC_DEVICE 1
typedef struct b2m_image_shard {
  uint32_t struct_size;
  int32_t location;          /* B2M_LOC_HOST (pageable or pinned) / B2M_LOC_DEVICE (this context's device) */
  int32_t first_image;       /* must equal b2m_comm_image_range(...) of this rank */
  int32_t n_local;
  int32_t has_keypoints;     /* the same on every rank (a rank without images has no pointer to tell by) */
  int32_t reserved;
  const void* desc_packed;   /* [sum of n_feat over the local images x 128] uint8, image after image */
  const void* kpts_packed;   /* float32 (x, y) per feature, same order, or NULL for match-only */
} b2m_image_shard;
/* b2m_set_images for a context that joined a communicator: lays out the WHOLE set (n_feat and cams describe all
 * images), copies the local shard into place, then one all-gather (ncclAllGather when the per-rank regions are
 * equal, else one grouped ncclBroadcast per owner) fills in the other ranks' images.  Collective: every rank
 * calls it with the same n_images / n_feat.  Without a communicator (or n_ranks == 1) it is b2m_set_images with a
 * packed source.  b2m_stats.last_allgather_* describe the collective. */
int b2m_set_images_sharded(b2m_ctx* ctx, int32_t n_images, const int32_t* n_feat, const b2m_camera* cams,
                           const b2m_image_shard* mine);

/* ---- estimators (callable without an image set) ------------------------------------ */

/* Replaces EstimateTwoViewGeometry / EstimateCalibratedTwoViewGeometry
 * (U:estimators/two_view_geometry.cc; R:estimators/two_view_geometry.h:95-151).
 * points: HOST [n x 2] float64; matches: [m x 2] uint32 or NULL (identity, R:two_view_geometry.h:136-142).
 * inlier_matches: HOST buffer capacity m x 2. */
typedef struct b2m_tvg_result {
  uint32_t struct_size;
  int32_t config;
  int64_t n_inliers;
  double E[9], F[9], H[9];
  int32_t nE, nF, nH;            /* inlier counts of the three LO-RANSAC runs (diagnostic) */
  int32_t pose_valid;            /* see b2m_pair_view */
  double qvec[4], tvec[3];
  double tri_angle;
} b2m_tvg_result;

int b2m_estimate_two_view_geometry(b2m_ctx* ctx, const b2m_camera* cam1, const double* points1, int64_t n1,
                                   const b2m_camera* cam2, const double* points2, int64_t n2,
                                   const uint32_t* matches, int64_t m, const b2m_tvg_opts* opts,
                                   b2m_tvg_result* out, uint32_t* inlier_matches);

/* Batched form of the call above for callers that verify many pairs from their own point sets (e.g. a
 * loop over estimate_two_view_geometry, R:estimators/two_view_geometry.h:95-151): one launch of the
 * pipeline's kernels over all problems (internally in chunks of 4096).  A problem's RANSAC stream is
 * keyed by (ctx seed, position of the problem in the call mod 4096): a given call is reproducible, and
 * problems of one call draw independent samples.
 * out: [n_problems]; inlier_matches: [n_problems] HOST buffers of capacity (m_k x 2) uint32, or NULL /
 * NULL entries to skip the inlier lists. */
typedef struct b2m_tvg_problem {
  uint32_t struct_size;
  int32_t reserved;
  b2m_camera cam1, cam2;
  const double* points1;   /* HOST [n1 x 2] float64 */
  int64_t n1;
  const double* points2;   /* HOST [n2 x 2] float64 */
  int64_t n2;
  const uint32_t* matches; /* HOST [m x 2] uint32, or NULL = identity (then n1 == n2) */
  int64_t m;
} b2m_tvg_problem;

int b2m_estimate_two_view_geometry_batch(b2m_ctx* ctx, const b2m_tvg_problem* problems, int64_t n_problems,
                                         const b2m_tvg_opts* opts, b2m_tvg_result* out,
                                         uint32_t* const* inlier_matches);

/* Replaces EstimateTwoViewGeometryPose (R:estimators/two_view_geometry.h:153-158): relative pose of an existing
 * geometry.  In: geometry->config, E (CALIBRATED / UNCALIBRATED) or H (PLANAR / PANORAMIC / PLANAR_OR_PANORAMIC) and
 * its inlier matches over the given points.  Out: qvec, tvec, tri_angle, pose_valid (0 = upstream's `false`), and
 * config when PLANAR_OR_PANORAMIC is resolved. */
int b2m_estimate_two_view_geometry_pose(b2m_ctx* ctx, const b2m_camera* cam1, const double* points1, int64_t n1,
                                        const b2m_camera* cam2, const double* points2, int64_t n2,
                                        const uint32_t* inlier_matches, int64_t n_inliers, b2m_tvg_result* geometry);

/* Single-model LO-RANSAC.  Replaces essential/fundamental/homography_matrix_estimation
 * (R:estimators/essential_matrix.h:19-103, fundamental_matrix.h:17-50, homography_matrix.h:17-48).
 * kind: 0 = E (points already normalised by the caller), 1 = F, 2 = H.
 * out_model: 9 doubles row-major; inlier_mask: m bytes.  *success = 0 mirrors the `None` return. */
int b2m_ransac_model(b2m_ctx* ctx, int32_t kind, const double* points1, const double* points2, int64_t m,
                     const b2m_ransac_opts* opts, double* out_model, uint8_t* inlier_mask,
                     int64_t* num_inliers, int32_t* success);

/* Replaces Camera::CamFromImg applied to a point list (R:scene/camera.h cam_from_img; the loop at
 * R:estimators/essential_matrix.h:31-39): pixel -> normalised camera coordinates, iterative undistortion
 * for the models with distortion.  points / out: HOST [n x 2] float64. */
int b2m_cam_from_img(b2m_ctx* ctx, const b2m_camera* camera, const double* points, int64_t n, double* out);

/* Replaces ComputeSquaredSampsonError (U:estimators/utils.cc; R:estimators/two_view_geometry.h:161-175). */
int b2m_squared_sampson_error(b2m_ctx* ctx, const double* points1, const double* points2, int64_t m,
                              const double* E, double* out_residuals);

/* ---- instrumentation ---------------------------------------------------------------- */

/* The cross-check consults m21 only at the columns some row matched (m21[m12[i]]): the column-direction GEMM is run
 * for those columns only (their descriptors gathered per pair into a scratch image; pairs without a match cost
 * nothing).  The first cross-check batch of a context is computed both ways -- gathered, and with the full
 * two-direction launch -- and the match lists are compared on the device before the context switches over.
 * Env B2M_K1_DIR1 = full | skip | gather forces a schedule without the comparison (skip = round 1's schedule:
 * full column direction for the pairs with at least one row-direction candidate). */
enum b2m_k1_dir1_mode {
  B2M_K1_DIR1_UNTESTED = 0,      /* no cross-check batch seen yet */
  B2M_K1_DIR1_SKIP = 1,          /* comparison passed: dead pairs skip the column direction */
  B2M_K1_DIR1_FULL_MISMATCH = 2, /* comparison FAILED: both directions for every pair (a bug to report) */
  B2M_K1_DIR1_FULL_FORCED = 3,   /* B2M_K1_DIR1=full */
  B2M_K1_DIR1_SKIP_FORCED = 4,   /* B2M_K1_DIR1=skip */
  B2M_K1_DIR1_FULL_NOMEM = 5,    /* no memory for the comparison buffers */
  B2M_K1_DIR1_GATHER = 6,        /* comparison passed: column direction computed for the MATCHED columns only (gathered) */
  B2M_K1_DIR1_GATHER_FORCED = 7  /* B2M_K1_DIR1=gather */
};

/* The verifier's 5-point essential-matrix solver (one warp per hypothesis, csrc/five_point_warp.cuh) on
 * caller-provided 4-D null spaces: nullspaces [n][4][9], models [n][10][9] (E = x N0 + y N1 + z N2 + N3 for every
 * real solution), n_models [n].  Exists so that tests can hold the device solver against the serial solver of
 * csrc/geom.h compiled for the host (U:estimators/essential_matrix.cc EssentialMatrixFivePointEstimator). */
int b2m_debug_five_point(b2m_ctx* ctx, const double* nullspaces, int64_t n, double* models, int32_t* n_models);

typedef struct b2m_stats {
  uint32_t struct_size;
  uint32_t reserved;
  uint64_t kernel_launches;   /* kernels of this library launched since create / last reset */
  uint64_t match_tiles;       /* 128x256 MMA tiles issued */
  double last_match_ms;       /* device time of the matching stage of the last b2m_match_pairs */
  double last_verify_ms;      /* device time of the verification stage */
  double last_total_ms;       /* device time of the whole call (events on the library stream) */
  double last_k1_ms;          /* sum of K1 (GEMM + fused top-2) kernel durations of the last call */
  uint64_t last_k1_launches;  /* K1 passes (one per pair batch) of the last call */
  uint64_t k1_dir1_mode;      /* enum b2m_k1_dir1_mode: how the column direction of the cross-check is computed */
  double last_allgather_ms;   /* device time of the all-gather of the last b2m_set_images_sharded (0 without a communicator) */
  uint64_t last_allgather_bytes; /* bytes this rank RECEIVED in it (descriptors + keypoints of the other ranks' images) */
  double last_upload_ms;      /* device time of the host -> device (or device -> device) copy of the local shard / set */
  uint64_t verify_models_scored[3];   /* E / F / H: hypotheses + LO candidates scored against all matches since reset */
  uint64_t verify_residuals[3];       /* E / F / H: residual evaluations (models scored x matches of the pair) since reset */
  int32_t comm_size, comm_rank;       /* 1, 0 without a communicator */
} b2m_stats;
int b2m_get_stats(b2m_ctx* ctx, b2m_stats* out);
int b2m_reset_stats(b2m_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* B200MATCH_H_ */
