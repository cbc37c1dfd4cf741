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

#define B2M_ABI_VERSION 10  /* 2: b2m_camera carries 12 parameters, batch estimator; 3: multi-GPU entry points (NCCL);
                             * 4: absolute pose estimation / refinement, b2m_stats.abs_pose_*;
                             * 5: triangulation, b2m_stats.tri_*; 6: SIFT feature extraction, b2m_stats.sift_*;
                             * 7: extraction from encoded / RGB sources, b2m_stats.sift_decode*;
                             * 8: PatchMatch stereo, b2m_stats.pm_*; 9: stereo fusion, b2m_stats.fusion_*;
                             * 10: image undistortion, b2m_stats.undistort_* */

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

/* ---- absolute pose (callable without an image set) ----------------------------------- */

/* AbsolutePoseEstimationOptions (R:pycolmap/estimators/absolute_pose.h:97-114; U:estimators/pose.h).  The defaults of
 * b2m_abs_pose_opts_default are the C++ constructor's; pycolmap's Python-side defaults (estimate_focal_length = 0,
 * ransac = RANSACOptions() with max_error 12) are set by the host module. */
typedef struct b2m_abs_pose_opts {
  uint32_t struct_size;
  int32_t estimate_focal_length;    /* 0 */
  int32_t num_focal_length_samples; /* 30 */
  int32_t reserved;
  double min_focal_length_ratio;    /* 0.2 */
  double max_focal_length_ratio;    /* 5 */
  b2m_ransac_opts ransac;           /* max_error in pixels */
} b2m_abs_pose_opts;

/* AbsolutePoseRefinementOptions (R:pycolmap/estimators/absolute_pose.h:116-131; U:estimators/pose.h). */
typedef struct b2m_pose_refine_opts {
  uint32_t struct_size;
  int32_t max_num_iterations;       /* 100 */
  double gradient_tolerance;        /* 1.0 */
  double loss_function_scale;       /* 1.0 (CauchyLoss) */
  int32_t refine_focal_length;      /* 1 */
  int32_t refine_extra_params;      /* 1 */
  int32_t print_summary;            /* 1; accepted and ignored (no solver log) */
  int32_t reserved;
} b2m_pose_refine_opts;

void b2m_abs_pose_opts_default(b2m_abs_pose_opts* o);
void b2m_pose_refine_opts_default(b2m_pose_refine_opts* o);

/* One 2D-3D correspondence set: points2D[i] (pixels) observes points3D[i] (world). */
typedef struct b2m_abs_pose_problem {
  uint32_t struct_size;
  int32_t reserved;
  b2m_camera camera;
  const double* points2D;  /* HOST [n x 2] float64 */
  const double* points3D;  /* HOST [n x 3] float64 */
  int64_t n;
} b2m_abs_pose_problem;

typedef struct b2m_abs_pose_result {
  uint32_t struct_size;
  int32_t success;          /* 0 mirrors the reference's `None` */
  int64_t num_inliers;
  double qvec[4];           /* cam_from_world rotation (w, x, y, z); identity on failure */
  double tvec[3];           /* x_cam = R(qvec) x_world + tvec */
  double params[B2M_CAMERA_MAX_PARAMS]; /* the camera's parameters after the call: focal scaled by the chosen factor when
                                         * estimate_focal_length, refined ones after refinement; unchanged otherwise */
  double covariance[36];    /* 6 x 6 row-major over (rotation tangent, translation) when requested */
  int32_t focal_sample;     /* index of the chosen focal-length factor, -1 when no sample succeeded */
  int32_t reserved;
} b2m_abs_pose_result;

/* Replaces EstimateAbsolutePose followed by RefineAbsolutePose (U:estimators/pose.cc), what
 * pycolmap.absolute_pose_estimation runs per query (R:pycolmap/estimators/absolute_pose.h:18-63), over a batch of
 * problems: one LO-RANSAC CTA per (problem, focal-length sample), then one warp per problem for the selection and the
 * refinement.  refine == NULL: estimation only.  want_covariance: fill result.covariance (needs refine).
 * inlier_masks: NULL, or [n_problems] HOST buffers of n_k bytes (NULL entries skip a problem).  Problem k is keyed by
 * its position in the call, so problem 0 of any batch equals the single call bit for bit. */
int b2m_estimate_absolute_pose_batch(b2m_ctx* ctx, const b2m_abs_pose_problem* problems, int64_t n_problems,
                                     const b2m_abs_pose_opts* opts, const b2m_pose_refine_opts* refine,
                                     int32_t want_covariance, b2m_abs_pose_result* out, uint8_t* const* inlier_masks);

/* Replaces RefineAbsolutePose on caller-provided poses (pycolmap.pose_refinement,
 * R:pycolmap/estimators/absolute_pose.h:65-94).  init_poses: [n_problems x 7] (qvec w, x, y, z, tvec);
 * inlier_masks: [n_problems] HOST buffers of n_k bytes (nonzero = inlier). */
int b2m_refine_absolute_pose_batch(b2m_ctx* ctx, const b2m_abs_pose_problem* problems, int64_t n_problems,
                                   const double* init_poses, const uint8_t* const* inlier_masks,
                                   const b2m_pose_refine_opts* refine, int32_t want_covariance, b2m_abs_pose_result* out);

/* ---- triangulation (callable without an image set) ----------------------------------- */

/* EstimateTriangulationOptions (R:pycolmap/estimators/triangulation.h:46-77; U:estimators/triangulation.h).  The
 * residual is upstream's default and pycolmap's only one, ANGULAR_ERROR: ransac.max_error is an angle in radians.
 * b2m_tri_opts_default gives the C++ RANSACOptions defaults; the host module sets pycolmap's Python-side ones. */
typedef struct b2m_tri_opts {
  uint32_t struct_size;
  int32_t reserved;
  double min_tri_angle;          /* 0, radians */
  b2m_ransac_opts ransac;        /* max_error in radians (angular residual) */
} b2m_tri_opts;

void b2m_tri_opts_default(b2m_tri_opts* o);

/* Replaces EstimateTriangulation (U:estimators/triangulation.cc; R:pycolmap/estimators/triangulation.h:17-44) over a
 * batch of tracks: LO-RANSAC with the two-view DLT as minimal estimator and TriangulateMultiViewPoint as local one,
 * sample pairs enumerated in lexicographic order (CombinationSampler), so the result is deterministic.
 * Track k owns observations [track_offsets[k], track_offsets[k + 1]) of points_normalized (camera-normalised (u, v))
 * and image_idx (index into cams_from_world, [n_images x 12], each a 3 x 4 row-major cam_from_world); every track needs
 * at least 2 observations (B2M_EINVAL otherwise, as for an out-of-range image index).  The projection centres are
 * -R^T t of the given matrices.  Out: xyz [n_tracks x 3] (NaN on failure), num_inliers [n_tracks] (the best support,
 * also on failure), success [n_tracks], inlier_mask [M] or NULL.  Internally in chunks of up to 32768 tracks; results
 * do not depend on the chunking or the order of the tracks. */
int b2m_estimate_triangulation_batch(b2m_ctx* ctx, int64_t n_tracks, const int64_t* track_offsets /* n_tracks + 1 */,
                                     const double* points_normalized /* [M x 2] */, const int32_t* image_idx /* [M] */,
                                     int32_t n_images, const double* cams_from_world /* [n_images x 12] */,
                                     const b2m_tri_opts* opts, double* xyz /* [n_tracks x 3] */, int32_t* num_inliers,
                                     uint8_t* success, uint8_t* inlier_mask /* [M] or NULL */);

/* ---- SIFT feature extraction (callable without an image set) -------------------------- */

/* SiftExtractionOptions (R:pipeline/extract_features.h:78-139; defaults U:feature/sift.h, the C++ constructor's).
 * pycolmap.Sift() overrides peak_threshold = 0.01, first_octave = 0, max_image_size = 7000 (R:pycolmap/feature/sift.h:
 * 99-102); the host module sets those.  The covariant path (estimate_affine_shape, domain_size_pooling) and SiftGPU's
 * darkness_adaptivity have no implementation here: a nonzero value is B2M_EINVAL. */
#define B2M_NORMALIZATION_L1_ROOT 0
#define B2M_NORMALIZATION_L2 1
typedef struct b2m_extract_opts {
  uint32_t struct_size;
  int32_t max_image_size;        /* 3200: larger images are B2M_EINVAL (pycolmap's Sift.extract does not resize) */
  int32_t max_num_features;      /* 8192 */
  int32_t first_octave;          /* -1 */
  int32_t num_octaves;           /* 4 */
  int32_t octave_resolution;     /* 3 */
  double peak_threshold;         /* 0.02 / 3 */
  double edge_threshold;         /* 10 */
  int32_t max_num_orientations;  /* 2 */
  int32_t upright;               /* 0 */
  int32_t normalization;         /* B2M_NORMALIZATION_L1_ROOT */
  int32_t estimate_affine_shape; /* 0 */
  int32_t domain_size_pooling;   /* 0 */
  int32_t darkness_adaptivity;   /* 0 */
} b2m_extract_opts;

void b2m_extract_opts_default(b2m_extract_opts* o);

/* One grey image: row-major uint8, `stride` bytes between rows (>= width). */
typedef struct b2m_image {
  int32_t width, height;
  int64_t stride;
  const uint8_t* data;
} b2m_image;

typedef struct b2m_features b2m_features;

typedef struct b2m_feature_view {
  uint32_t struct_size;
  int32_t reserved;
  int64_t n;                     /* features of the image */
  const float* keypoints;        /* [n x 4] (x, y, scale, orientation): x, y with pixel centres at +0.5, orientation in
                                  * (-pi, pi] (FeatureKeypoint::ComputeScale / ComputeOrientation) */
  const uint8_t* descriptors;    /* [n x 128] uint8, UBC layout */
} b2m_feature_view;

/* Replaces SiftCPUFeatureExtractor::Extract (U:feature/sift.cc; VLFeat's vl_sift) as pycolmap.Sift.extract calls it
 * (R:pycolmap/feature/sift.h:41-80), over `n` images.  Output order per image: octave ascending, then VLFeat's
 * detection scan order (level, y, x), the orientations of one keypoint consecutive; the max_num_features cut keeps
 * whole (octave, level) runs from the coarsest down, the run that passes the limit included.  Deterministic, and
 * independent of the other images of the call.  *out is owned by the caller until b2m_features_free. */
int b2m_extract_features_batch(b2m_ctx* ctx, const b2m_image* images, int32_t n, const b2m_extract_opts* opts,
                               b2m_features** out);
int b2m_features_get(const b2m_features* f, int32_t image, b2m_feature_view* out);
void b2m_features_free(b2m_features* f);

/* ---- feature extraction from image sources (ABI 7) ----------------------------------------------------------------
 * What COLMAP's feature extraction does to one image between reading the file and writing the database (U:controllers/
 * feature_extraction.cc, U:controllers/image_reader.cc; SURVEY.md rows U1-U6): decode, convert to grey (FreeImage's
 * ConvertToGreyscale, Rec709 weights), downscale when max(w, h) > max_image_size (FreeImage's bilinear Rescale), SIFT,
 * keypoints back to original-image coordinates as FeatureKeypoint's 6 columns, and the mask test.  Decoding uses
 * nvJPEG's hardware backend where the GPU has JPEG engines and the file is baseline, the hybrid backend otherwise; a
 * decoder thread and a side stream decode, convert and downscale the next images while SIFT runs the current one. */
#define B2M_SOURCE_JPEG 0    /* data / size: a whole JPEG file, decoded on the device (nvJPEG) */
#define B2M_SOURCE_PIXELS 1  /* data: width x height pixels of `channels` bytes (1 grey, 3 RGB, 4 RGBA: alpha ignored),
                              * `stride` bytes per row, in host memory */
typedef struct b2m_image_source {
  int32_t kind;                  /* B2M_SOURCE_* */
  int32_t channels;              /* B2M_SOURCE_PIXELS: 1, 3 or 4 */
  int32_t width, height;         /* B2M_SOURCE_PIXELS: the size; JPEG: ignored, read from the stream */
  int64_t stride;                /* B2M_SOURCE_PIXELS: bytes between rows (>= width x channels) */
  const uint8_t* data;
  int64_t size;                  /* B2M_SOURCE_JPEG: bytes */
  const uint8_t* mask;           /* NULL, or a grey mask in original-image coordinates: a keypoint is dropped when its
                                  * integer pixel (int)x, (int)y lies outside the mask or the mask is 0 there
                                  * (MaskKeypoints) */
  int32_t mask_width, mask_height;
  int64_t mask_stride;
} b2m_image_source;

typedef struct b2m_source_view {
  uint32_t struct_size;
  int32_t status;                /* B2M_OK, or B2M_EINVAL when the source could not be decoded (nothing else is set) */
  const char* error;             /* why, when status != B2M_OK */
  int32_t width, height;         /* decoded (original) size */
  int64_t n;                     /* features kept */
  const float* keypoints;        /* [n x 6] (x, y, a11, a12, a21, a22) in original-image coordinates */
  const uint8_t* descriptors;    /* [n x 128] */
} b2m_source_view;

/* Extracts `n` sources in order.  An image whose larger side exceeds opts->max_image_size is downscaled to
 * (int)(w * s) x (int)(h * s), s = max_image_size / max(w, h), before SIFT, and its keypoints scaled back per axis
 * (ScaleKeypoints).  A source that does not decode gets status B2M_EINVAL and the others go on; a bad argument fails
 * the call.  *out is read with b2m_source_features_get and released with b2m_features_free. */
int b2m_extract_features_sources(b2m_ctx* ctx, const b2m_image_source* sources, int32_t n, const b2m_extract_opts* opts,
                                 b2m_features** out);
int b2m_source_features_get(const b2m_features* f, int32_t image, b2m_source_view* out);

/* ---- PatchMatch stereo (ABI 8) -------------------------------------------------------------------------------------
 * What COLMAP's PatchMatch stereo (U:mvs/patch_match_cuda.cu; Schoenberger et al., ECCV 2016) computes for one reference
 * image and its sources: a depth (camera z) and a normal (camera frame, facing the camera) per pixel, chosen by
 * propagation and random search to minimise 1 - bilaterally weighted NCC through the plane-induced homography, averaged
 * over Monte Carlo draws of the sources from their posterior visibility (forward / backward messages of a hidden Markov
 * chain along each sweep) times the triangulation- and incident-angle priors.  K8 (csrc/patch_match.cu); the schedule is spelled out in DESIGN.md section 4
 * and restated by oracle/patch_match.py. */
#define B2M_PM_MAX_SOURCES 32
typedef struct b2m_patch_match_opts {
  uint32_t struct_size;
  int32_t window_radius;                  /* 5 */
  int32_t window_step;                    /* 1 */
  int32_t num_samples;                    /* 15: Monte Carlo draws of sources per pixel and hypothesis */
  int32_t num_iterations;                 /* 5: each of four sweeps (down, up, right, left) */
  int32_t geom_consistency;               /* 0: photometric pass; 1: geometric term through the sources' depth maps */
  int32_t filter;                         /* 1 */
  int32_t filter_min_num_consistent;      /* 2 */
  float sigma_spatial;                    /* -1 = window_radius */
  float sigma_color;                      /* 0.2 (intensities in [0, 1]) */
  float ncc_sigma;                        /* 0.6 */
  float min_triangulation_angle;          /* 1, degrees */
  float incident_angle_sigma;             /* 0.9 */
  float geom_consistency_regularizer;     /* 0.3 */
  float geom_consistency_max_cost;        /* 3, pixels */
  float filter_min_ncc;                   /* 0.1 */
  float filter_min_triangulation_angle;   /* 3, degrees */
  float filter_geom_consistency_max_cost; /* 1, pixels */
} b2m_patch_match_opts;
void b2m_patch_match_opts_default(b2m_patch_match_opts* o);

/* Uploads the images of a workspace once: grey uint8 images and pinhole cameras, cameras[i] = 16 doubles (fx, fy, cx,
 * cy, then cam_from_world as R row-major (9) and t (3)).  They stay resident until the next call or b2m_destroy.
 * depth_maps: NULL, or n entries of NULL / a width x height float32 depth map of that image (the photometric maps the
 * geometric pass reads).  A set that does not fit in device memory is B2M_ENOMEM with its size in the message. */
int b2m_patch_match_set_images(b2m_ctx* ctx, int32_t n, const b2m_image* images, const double* cameras,
                               const float* const* depth_maps);

typedef struct b2m_patch_match_problem {
  uint32_t struct_size;
  int32_t ref;                  /* index into the image set */
  int32_t n_src;                /* 1 .. B2M_PM_MAX_SOURCES */
  int32_t image_id;             /* a stable id of the reference (e.g. its workspace image_id): the key of its random
                                 * numbers, so that its maps do not depend on which image set or batch it runs in */
  const int32_t* src;           /* n_src image indices, distinct and != ref */
  float depth_min, depth_max;   /* 0 < depth_min < depth_max */
  const float* init_depth;      /* NULL, or the ref's width x height start depths (0 = start at random) */
  const float* init_normal;     /* NULL, or width x height x 3 start normals (with init_depth) */
} b2m_patch_match_problem;

typedef struct b2m_depth_maps b2m_depth_maps;
typedef struct b2m_depth_map_view {
  uint32_t struct_size;
  int32_t width, height;
  int32_t reserved;
  const float* depth;           /* [height x width]; 0 where filtered */
  const float* normal;          /* [height x width x 3]; 0 where filtered */
} b2m_depth_map_view;

/* Runs the problems in one batch of launches; with opts->geom_consistency every source of every problem needs a depth
 * map in the image set.  Problem k's maps depend only on (ctx seed, its image_id, its images, cameras and options),
 * never on the index of its images in the set, its position in the batch or the batch's other problems.  Read with b2m_depth_maps_get, release with
 * b2m_depth_maps_free. */
int b2m_patch_match_batch(b2m_ctx* ctx, const b2m_patch_match_problem* problems, int32_t n,
                          const b2m_patch_match_opts* opts, b2m_depth_maps** out);
int b2m_depth_maps_get(const b2m_depth_maps* m, int32_t k, b2m_depth_map_view* out);
void b2m_depth_maps_free(b2m_depth_maps* m);

/* K8's cost arithmetic for given hypotheses of `problem`: queries [n x 7] = (x, y, depth, nx, ny, nz, source slot);
 * out [n x 3] = (photometric cost 1 - NCC in [0, 2], geometric cost min(forward-backward reprojection error,
 * geom_consistency_max_cost) or 0 without source depth maps, depth of the same plane at pixel (x, y + 1)).  Exists so
 * that tests can hold the device arithmetic against oracle/patch_match.py. */
int b2m_debug_patch_match_cost(b2m_ctx* ctx, const b2m_patch_match_problem* problem, const b2m_patch_match_opts* opts,
                               const float* queries, int32_t n, float* out);

/* ---- stereo fusion (ABI 9) ------------------------------------------------------------------------------------------
 * What COLMAP's StereoFusion (U:mvs/fusion.cc, recalled) computes from a workspace's depth and normal maps: from every
 * seed pixel a depth-first traversal through the overlapping images gathers the pixels whose depth, reprojection and
 * normal agree with the seed's point, and a cluster of at least min_num_pixels pixels becomes one point (per-channel
 * medians of position, normal and colour; visibility = the images that contributed).  K9 (csrc/fusion.cu): seeds run in
 * rounds over a 16 x 16 lattice of each image; a round's seeds traverse speculatively and commit by a fixed rule, so that
 * the result equals the sequential traversal over the committed-seed order it reports (DESIGN.md section 4, K9) and is
 * a function of the inputs alone.  oracle/fusion.cpp restates it. */
typedef struct b2m_fusion_image {
  uint32_t struct_size;
  int32_t width, height;           /* depth-map size */
  const float* depth;              /* [height x width], or NULL: the image has no maps (neither a seed nor a target) */
  const float* normal;             /* [height x width x 3] (camera frame), with depth */
  const uint8_t* mask;             /* NULL, or [height x width]: pixels where it is 0 are never fused */
  float P[12];                     /* K [R | t], K scaled per axis by bitmap_scale, row-major 3 x 4 */
  float inv_P[12];                 /* the top 3 rows of [P; 0 0 0 1]^-1 */
  float inv_R[9];                  /* R^T */
  float bitmap_scale[2];           /* depth-map width / camera width, depth-map height / camera height */
  const int32_t* overlap;          /* n_overlap image indices, in the order the traversal pushes them */
  int32_t n_overlap;
  int32_t reserved;
  b2m_image_source color;          /* the image at camera size: JPEG (decoded by nvJPEG) or host pixels of 1, 3 or 4
                                    * channels; data NULL = black (allowed for images without maps) */
} b2m_fusion_image;

typedef struct b2m_fusion_opts {
  uint32_t struct_size;
  int32_t min_num_pixels;          /* 5 */
  int32_t max_num_pixels;          /* 10000 */
  int32_t max_traversal_depth;     /* 100 */
  float max_reproj_error;          /* 2, pixels */
  float max_depth_error;           /* 0.01, relative */
  float max_normal_error;          /* 10, degrees */
  float bounding_box[6];           /* min x, y, z, max x, y, z: -FLT_MAX .. FLT_MAX */
} b2m_fusion_opts;
void b2m_fusion_opts_default(b2m_fusion_opts* o);

typedef struct b2m_fused_points b2m_fused_points;
typedef struct b2m_fused_points_view {
  uint32_t struct_size;
  int32_t reserved;
  int64_t n_points;
  const float* xyz;                /* [n_points x 3] */
  const float* normals;            /* [n_points x 3] */
  const uint8_t* colors;           /* [n_points x 3] */
  const int64_t* vis_off;          /* [n_points + 1]: point k is seen by vis[vis_off[k] .. vis_off[k + 1]) */
  const int32_t* vis;              /* image indices, ascending per point */
  const int32_t* seeds;            /* [n_points x 3]: (image, row, col) of the seed that made the point */
  int64_t n_order;
  const int32_t* order;            /* [n_order x 4]: every committed seed (image, row, col, round), in commit order,
                                    * including those whose cluster made no point */
} b2m_fused_points_view;

/* Fuses n images in one call (nothing stays resident).  A workspace that does not fit in device memory is B2M_ENOMEM
 * with its size in the message; b2m_request_stop is honoured between rounds. */
int b2m_stereo_fusion(b2m_ctx* ctx, const b2m_fusion_image* images, int32_t n, const b2m_fusion_opts* opts,
                      b2m_fused_points** out);
int b2m_fused_points_get(const b2m_fused_points* p, b2m_fused_points_view* out);
void b2m_fused_points_free(b2m_fused_points* p);

/* ---- image undistortion (ABI 10) ------------------------------------------------------------------------------------
 * What COLMAP's image undistorter (U:image/undistortion.cc, U:image/warp.cc, U:sensor/bitmap.cc; recalled, DESIGN.md
 * section 4 K10) does to one image: UndistortCamera gives a PINHOLE camera (ROI, scale from the distorted image's
 * borders, max_image_size), and the image is warped at the source resolution (pinhole CamFromImg of each pixel centre,
 * the distorted ImgFromCam, fp64 bilinear interpolation on FreeImage's bottom-up rows, black outside), then rescaled to
 * the undistorted size with FreeImage's bilinear filter.  K10 (csrc/undistort.cu); oracle/undistort.py restates it. */
typedef struct b2m_undistort_opts {
  uint32_t struct_size;
  int32_t max_image_size;          /* -1: no limit; > 0: the undistorted image is scaled down to fit */
  double blank_pixels;             /* 0: no blank pixel in the output; 1: every input pixel in the output */
  double min_scale;                /* 0.2 */
  double max_scale;                /* 2 */
  double roi_min_x, roi_min_y;     /* 0, 0: the region of interest as fractions of the image size */
  double roi_max_x, roi_max_y;     /* 1, 1 */
} b2m_undistort_opts;
void b2m_undistort_opts_default(b2m_undistort_opts* o);

/* UndistortCamera on the host (no device work; ctx may be NULL, the message then goes to b2m_last_error(NULL)).  Bad
 * options or camera: B2M_EINVAL. */
int b2m_undistort_camera(b2m_ctx* ctx, const b2m_undistort_opts* opts, const b2m_camera* camera, b2m_camera* out);

#define B2M_UNDISTORT_JPEG 0     /* the undistorted image as a JPEG file (nvJPEG, quality 100, 4:2:0) */
#define B2M_UNDISTORT_PIXELS 1   /* the undistorted image as width x height x 3 RGB bytes */
typedef struct b2m_undistort_item {
  uint32_t struct_size;
  int32_t output;                  /* B2M_UNDISTORT_* */
  b2m_camera camera;               /* the distorted camera; the decoded source must be its size */
  b2m_image_source source;         /* JPEG, or host pixels of 1 (grey, replicated), 3 or 4 (alpha dropped) channels;
                                    * the mask fields are ignored */
} b2m_undistort_item;

typedef struct b2m_undistorted b2m_undistorted;
typedef struct b2m_undistorted_view {
  uint32_t struct_size;
  int32_t status;                  /* B2M_OK, or B2M_EINVAL when the source does not decode or is not its camera's size */
  const char* error;               /* why, when status != B2M_OK */
  int32_t width, height;           /* the undistorted size */
  b2m_camera camera;               /* the undistorted (PINHOLE) camera */
  int64_t size;                    /* bytes at data: the JPEG file, or width x height x 3 */
  const uint8_t* data;
} b2m_undistorted_view;

/* Undistorts n items in order, one after the other on the device.  An item whose source does not decode or has not its
 * camera's size gets an error status and the others go on; a bad argument fails the call.  A call whose largest image
 * does not fit in device memory is B2M_ENOMEM with its size in the message.  Read with b2m_undistorted_get, release with
 * b2m_undistorted_free. */
int b2m_undistort_images(b2m_ctx* ctx, const b2m_undistort_item* items, int32_t n, const b2m_undistort_opts* opts,
                         b2m_undistorted** out);
int b2m_undistorted_get(const b2m_undistorted* r, int32_t k, b2m_undistorted_view* out);
void b2m_undistorted_free(b2m_undistorted* r);

/* The RGB image b2m_undistort_images encodes for `item` (whatever its output kind).  With rgb == NULL only *width /
 * *height are set; otherwise rgb holds width x height x 3 bytes.  Exists so that tests can hold K10 against
 * oracle/undistort.py exactly. */
int b2m_debug_undistort_pixels(b2m_ctx* ctx, const b2m_undistort_item* item, const b2m_undistort_opts* opts, uint8_t* rgb,
                               int32_t* width, int32_t* height);

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

/* The grey image b2m_extract_features_sources feeds to SIFT for `source` (decoded, grey, downscaled when it exceeds
 * max_image_size).  With grey == NULL only *width / *height are set; otherwise grey holds width x height bytes.
 * Exists so that tests can hold the device decoder and the rescale against a host decoder / the numpy oracle. */
int b2m_debug_decode_grey(b2m_ctx* ctx, const b2m_image_source* source, int32_t max_image_size, uint8_t* grey,
                          int32_t* width, int32_t* height);

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
  uint64_t abs_pose_models_scored;    /* absolute pose: P3P / EPnP models scored against all correspondences since reset */
  uint64_t abs_pose_residuals;        /* absolute pose: residual evaluations (models scored x correspondences) */
  uint64_t tri_models_scored;         /* triangulation: two-view and LO models scored against all observations */
  uint64_t tri_residuals;             /* triangulation: residual evaluations (models scored x observations of the track) */
  uint64_t sift_images;               /* SIFT extraction: images processed since reset */
  uint64_t sift_keypoints;            /* SIFT extraction: keypoints kept after the max_num_features cut */
  uint64_t sift_descriptors;          /* SIFT extraction: descriptors computed (keypoints x orientations) */
  uint64_t sift_decoded_bytes;        /* extraction from sources: encoded JPEG bytes decoded on the device */
  uint64_t sift_decode_images;        /* extraction from sources: images decoded (JPEG) or uploaded (pixels) */
  uint64_t sift_decode_hardware;      /* of those, JPEG files decoded by nvJPEG's hardware backend (the JPEG engines) */
  uint64_t pm_problems;               /* PatchMatch: reference images processed since reset */
  uint64_t pm_pixel_updates;          /* PatchMatch: pixel x sweep steps */
  uint64_t pm_window_samples;         /* PatchMatch: window samples evaluated (one reference / source pixel pair each) */
  uint64_t fusion_seeds;              /* stereo fusion: committed seeds since reset */
  uint64_t fusion_traversals;         /* stereo fusion: traversals run (speculative and committing) */
  uint64_t fusion_pops;               /* stereo fusion: pixels popped by those traversals */
  uint64_t fusion_rounds;             /* stereo fusion: rounds */
  uint64_t fusion_deferred;           /* stereo fusion: candidates deferred to a later round */
  uint64_t fusion_points;             /* stereo fusion: points emitted */
  uint64_t undistort_images;          /* undistortion: images undistorted since reset */
  uint64_t undistort_pixels;          /* undistortion: output pixels */
  uint64_t undistort_encoded_bytes;   /* undistortion: bytes of the JPEG files written by nvJPEG */
} b2m_stats;
int b2m_get_stats(b2m_ctx* ctx, b2m_stats* out);
int b2m_reset_stats(b2m_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* B200MATCH_H_ */
