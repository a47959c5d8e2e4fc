/*
 * esvo_b200.h -- C ABI of the Hopper-native (sm_90a) ESVO mapping/tracking hot path.
 *
 * The reference (HKUST-Aerial-Robotics/ESVO) has no FFI/plugin layer: its seam is the C++
 * class surface of esvo_time_surface::TimeSurface and esvo_core::core::{EventBM,
 * DepthProblemSolver, DepthFusion, RegProblemSolverLM}.  Every entry point below replaces
 * one of those methods; the citation after "replaces:" is the reference file:line whose
 * behaviour the entry point reproduces.  The C++ shim classes in include/esvo_b200/ keep the
 * reference names and forward to this ABI (see INTEGRATION.md).
 *
 * Conventions
 *   - plain pointers and sizes only; all pointers are HOST pointers owned by the caller unless
 *     the function name ends in _dev;
 *   - 4x4 poses are row-major double[16] (T_world_cam: camera -> world), the matrix form of the
 *     reference's kindr::minimal::QuatTransformation;
 *   - images are row-major (y*W + x); time stamps are int64 nanoseconds (ros::Time.toNSec());
 *   - return value 0 = ok, <0 = esvo_status error code, never abort(); data-dependent
 *     "no result" conditions are reported through counts, like the reference's bool returns;
 *   - one esvo_ctx per event stream / GPU; a ctx is NOT thread-safe (the reference solver
 *     objects are not re-entrant either, SURVEY 8b); distinct ctxs are independent;
 *   - there is NO CPU fallback: esvo_create fails with ESVO_ERR_NO_DEVICE when no CUDA device
 *     is usable.
 *
 * The same declarations, with the prefix esvo_oracle_ instead of esvo_, are exported by the
 * CPU oracle (oracle/), which is test infrastructure only.
 */
#ifndef ESVO_B200_H_
#define ESVO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef ESVO_API
#define ESVO_API __attribute__((visibility("default")))
#endif

typedef enum {
  ESVO_OK = 0,
  ESVO_ERR_INVALID_ARG = -1,
  ESVO_ERR_NO_DEVICE = -2,
  ESVO_ERR_CUDA = -3,
  ESVO_ERR_CAPACITY = -4,
  ESVO_ERR_STATE = -5,      /* call order violated (e.g. bm_match before set_ts_pair) */
  ESVO_ERR_UNSUPPORTED = -6 /* the reference exit(-1)s on these configs, we return instead */
} esvo_status;

enum { ESVO_DIST_PLUMB_BOB = 0, ESVO_DIST_EQUIDISTANT = 1 };
enum { ESVO_LSNORM_L2 = 0, ESVO_LSNORM_TDIST = 1, ESVO_LSNORM_ZNCC = 2 };
enum { ESVO_TRK_LSNORM_L2 = 0, ESVO_TRK_LSNORM_HUBER = 1 };
enum { ESVO_FUSION_CONST_FRAMES = 0, ESVO_FUSION_CONST_POINTS = 1 };
enum { ESVO_TS_BACKWARD = 0, ESVO_TS_FORWARD = 1 };

/* One camera of the rig: the fields of calib/<dataset>/{left,right}.yaml
 * (reference esvo_core/src/container/CameraSystem.cpp:168-216, all row-major). */
typedef struct {
  int32_t width, height;
  int32_t distortion_model; /* ESVO_DIST_* */
  int32_t _pad;
  double K[9];
  double D[4];
  double R[9];  /* rectification_matrix */
  double P[12]; /* projection_matrix    */
} esvo_calib;

/* All yaml keys that reach the hot path (reference esvo_core/cfg/{mapping,tracking}/ *.yaml,
 * esvo_time_surface/cfg/parameters.yaml; defaults = reference tools::param defaults,
 * esvo_Mapping.cpp:36-94, esvo_Tracking.cpp:24-36, TimeSurface.cpp:23-30). */
typedef struct {
  /* --- time surface (esvo_time_surface) --- */
  double decay_ms;                 /* 30 */
  int32_t ignore_polarity;         /* 1 */
  int32_t median_blur_kernel_size; /* 1  -> 3x3 */
  int32_t max_event_queue_len;     /* 20 */
  int32_t time_surface_mode;       /* ESVO_TS_BACKWARD */
  /* --- EventBM --- */
  int32_t patch_size_x, patch_size_y; /* 15, 7 in every shipped cfg */
  int32_t bm_min_disparity, bm_max_disparity; /* yaml values, BEFORE the invDepth clip */
  int32_t bm_step;
  int32_t bm_updown;               /* BM_bUpDownConfiguration */
  int32_t smooth_time_surface;     /* SmoothTimeSurface */
  double bm_zncc_threshold;
  /* --- DepthProblem / solver --- */
  int32_t lsnorm;                  /* ESVO_LSNORM_* */
  int32_t max_iteration;           /* ITERATION_OPTIMIZATION, 10 */
  double td_nu, td_scale;
  /* --- culling / fusion / map --- */
  double invdepth_min_range, invdepth_max_range;
  double residual_vis_threshold, stdvar_vis_threshold;
  double age_vis_threshold;
  int32_t fusion_radius;
  int32_t fusion_strategy;         /* ESVO_FUSION_* */
  int32_t max_num_fusion_frames;
  int32_t max_num_fusion_points;
  /* --- DepthRegularization --- */
  int32_t regularization;
  int32_t reg_radius, reg_min_neighbours, reg_min_close_neighbours;
  /* --- tracking (RegProblemConfig) --- */
  int32_t trk_patch_size_x, trk_patch_size_y; /* 1,1 */
  int32_t trk_kernel_size;         /* 5 */
  int32_t trk_lsnorm;              /* ESVO_TRK_LSNORM_* */
  double trk_huber_threshold;
  int32_t trk_max_registration_points;
  int32_t trk_batch_size;
  int32_t trk_max_iteration;
  int32_t trk_min_num_events;
  /* --- compiled-in thread counts of the reference; only used to reproduce its
   *     thread-major output ORDER (utils.h:35-36), no CPU threads are spawned --- */
  int32_t num_thread_mapping;      /* 4 */
  int32_t _pad;
} esvo_params;

/* POD form of esvo_core::core::EventMatchPair (EventMatchPair.h:16-40). */
typedef struct {
  double x_left_raw[2];
  double x_left[2];
  double x_right[2];
  int64_t t_ns;
  double T_world_virtual[16];
  double inv_depth;
  double cost;
  double disp;
} esvo_seed;

/* POD form of esvo_core::container::DepthPoint (DepthPoint.h:70-88). */
typedef struct {
  int32_t row, col;
  double x[2];
  double inv_depth;
  double scale2;
  double nu;
  double variance;
  double residual;
  int64_t age;
  double p_cam[3];
  double T_world_cam[16];
} esvo_depth_point;

/* RegProblemSolverLM::lmStatics_ (RegProblemSolverLM.h:26-31). */
typedef struct {
  int64_t n_points;
  int64_t nfev;
  int64_t n_iter;
} esvo_lm_stats;

typedef struct esvo_ctx esvo_ctx;

/* Fills *p with the reference's defaults. */
ESVO_API void esvo_default_params(esvo_params* p);

/* replaces: CameraSystem ctor + PerspectiveCamera::preComputeRectifiedCoordinate
 * (CameraSystem.cpp:37-112,150-166), TimeSurface::cameraInfoCallback (TimeSurface.cpp:313-401),
 * esvo_Mapping ctor disparity clip (esvo_Mapping.cpp:110-121).  device = CUDA ordinal. */
ESVO_API esvo_ctx* esvo_create(int device, const esvo_calib* left, const esvo_calib* right,
                               const esvo_params* params, int* status_out);
ESVO_API void esvo_destroy(esvo_ctx* ctx);

/* Optional: override the internally computed rectification tables with tables produced by the
 * integrator's own OpenCV (the reference's tables depend on the OpenCV version, SURVEY A.2).
 * map1/map2: H*W float (initUndistortRectifyMap CV_32FC1); lut_xy: H*W*2 double
 * (precomputed_rectified_points_, x then y per pixel); mask: H*W uint8 {0,255}
 * (UndistortRectify_mask_).  Any pointer may be NULL to keep the current table. */
ESVO_API int esvo_set_rectify_tables(esvo_ctx* ctx, int cam, const float* map1, const float* map2,
                                     const double* lut_xy, const uint8_t* mask);
/* Read back the tables in use (same layouts; NULL pointers are skipped). */
ESVO_API int esvo_get_rectify_tables(esvo_ctx* ctx, int cam, float* map1, float* map2,
                                     double* lut_xy, uint8_t* mask);
/* The same tables WITHOUT a context or a GPU (pure host code, one-time setup): what esvo_create computes for one camera.
 * replaces: cv::initUndistortRectifyMap / cv::undistortPoints (+ fisheye variants) and the validity mask as used by
 * TimeSurface::cameraInfoCallback (TimeSurface.cpp:313-401) and PerspectiveCamera::preComputeRectifiedCoordinate
 * (CameraSystem.cpp:37-112).  Lets an integrator (and tests/test_product_tables_cv2.py) compare them with their OpenCV. */
ESVO_API int esvo_compute_rectify_tables(const esvo_calib* cam, float* map1, float* map2, double* lut_xy, uint8_t* mask);
/* Derived constants: out[0]=baseline, out[1]=min disparity, out[2]=max disparity (after clip),
 * out[3]=td_stdvar. */
ESVO_API int esvo_get_derived(esvo_ctx* ctx, double out[4]);

/* ---------------- time surface ---------------- */
/* replaces: TimeSurface::eventsCallback + EventQueueMat::insertEvent
 * (TimeSurface.cpp:403-425, TimeSurface.h:39-50).  cam: 0 left, 1 right. */
ESVO_API int esvo_ts_push_events(esvo_ctx* ctx, int cam, const uint16_t* x, const uint16_t* y,
                                 const int64_t* t_ns, const uint8_t* pol, size_t n);
/* Out-of-order stamps.  The reference's eventsCallback insertion-sorts every new event into its global deque and then
 * queues events_.back() -- the event with the largest stamp so far -- into the per-pixel queues
 * (esvo_time_surface/src/TimeSurface.cpp:410-422); for time-ordered input that is the new event itself.  With
 * enable = 1 pushes of this camera go through a device prefix scan (running arg-max of the stamps) that reproduces
 * this for arbitrary input order, at the cost of two extra kernels per push.  With enable = 0 (default) input must be
 * time-ordered; a violation is detected on the device and reported by esvo_ts_build as ESVO_ERR_UNSUPPORTED (the
 * flag stays up until esvo_ts_reset).
 * The scan carries events_.back() from push to push, and ordered pushes do not record it.  So enable = 1 is accepted
 * only while the camera holds no events (after esvo_create or esvo_ts_reset); on a camera that already took ordered
 * pushes it returns ESVO_ERR_UNSUPPORTED and changes nothing. */
ESVO_API int esvo_ts_set_unordered_input(esvo_ctx* ctx, int cam, int enable);


/* replaces: TimeSurface::createTimeSurfaceAtTime (TimeSurface.cpp:52-152) incl.
 * EventQueueMat::getMostRecentEventBeforeT (TimeSurface.h:52-75).
 * idx_grid_out (H*W, may be NULL): index, in push order since create/reset, of the event each
 * pixel's value was taken from, -1 if none.  ts_out (H*W, may be NULL): the published mono8 image.
 * How far back t_sync_ns may lie: each camera keeps its newest events resident (4 Mi; when a push would overflow
 * that, all but the newest 1 Mi are folded into one most-recent-event grid, so at least 1 Mi events are always
 * resident).  The folded events' queues are gone, so t_sync_ns must be newer than the newest folded stamp:
 * otherwise esvo_ts_build returns ESVO_ERR_UNSUPPORTED and esvo_last_error names the oldest t_sync_ns it can answer.
 * The reference answers such a time from its 20-deep queues; this library does not guess.  esvo_run_ts_build does
 * not read the device flags back and reports neither this nor an order violation.
 * median_blur_kernel_size > 1 is not implemented: ESVO_ERR_UNSUPPORTED. */
ESVO_API int esvo_ts_build(esvo_ctx* ctx, int cam, int64_t t_sync_ns, int64_t* idx_grid_out,
                           uint8_t* ts_out);
ESVO_API int esvo_ts_reset(esvo_ctx* ctx, int cam);

/* ---------------- mapping ---------------- */
/* replaces: TimeSurfaceObservation ctor (TimeSurfaceObservation.h:59-89) + setTransformation.
 * ts_left/ts_right may be NULL = "use the images produced by the last esvo_ts_build of that
 * camera" (device-resident hand-off, no host round trip). */
ESVO_API int esvo_set_ts_pair(esvo_ctx* ctx, const uint8_t* ts_left, const uint8_t* ts_right,
                              const double T_world_left[16]);
/* replaces: EventBM::createMatchProblem + match_all_HyperThread (EventBM.cpp:56-78,269-315).
 * poses: the StampTransformationMap (sorted by pose_t_ns).  seeds_out in the reference's
 * thread-major order.  *n_seeds: in = capacity, out = count.  n_patch_evals: number of
 * zncc_cost evaluations performed (may be NULL). */
ESVO_API int esvo_bm_match(esvo_ctx* ctx, const uint16_t* ex, const uint16_t* ey,
                           const int64_t* et_ns, size_t n_events, const int64_t* pose_t_ns,
                           const double* poses, size_t n_poses, esvo_seed* seeds_out,
                           size_t* n_seeds, uint64_t* n_patch_evals);
/* replaces: DepthProblemSolver::solve (DepthProblemSolver.cpp:28-214).  *n_out: in = capacity,
 * out = count.  n_patch_evals: number of DepthProblem::operator() evaluations (nfev summed). */
ESVO_API int esvo_depth_solve(esvo_ctx* ctx, const esvo_seed* seeds, size_t n,
                              esvo_depth_point* out, size_t* n_out, uint64_t* n_patch_evals);
/* replaces: DepthProblemSolver::pointCulling (DepthProblemSolver.cpp:217-244); in place. */
ESVO_API int esvo_depth_cull(esvo_ctx* ctx, esvo_depth_point* pts, size_t* n, double std_thr,
                             double cost_thr, double rho_min, double rho_max);
/* replaces: DepthFusion::update (DepthFusion.cpp:71-87) into the ctx's DepthFrame.
 * reset_map != 0 first replaces the DepthFrame by an empty one with pose T_world_frame
 * (esvo_Mapping.cpp:268-272). */
ESVO_API int esvo_fuse(esvo_ctx* ctx, const esvo_depth_point* pts, size_t n,
                       const double T_world_frame[16], int fusion_radius, int reset_map,
                       int* n_fusions);
/* replaces: SmartGrid::clean (SmartGrid.h:222-243). */
ESVO_API int esvo_map_clean(esvo_ctx* ctx, double var_thr, double age_thr, double rho_max,
                            double rho_min);
/* replaces: DepthRegularization::apply (DepthRegularization.cpp:19-110). */
ESVO_API int esvo_map_regularize(esvo_ctx* ctx);
/* DepthMap element list in insertion order (SmartGrid::_elements). *n: in = cap, out = count. */
ESVO_API int esvo_map_download(esvo_ctx* ctx, esvo_depth_point* out, size_t* n);

/* replaces: esvo_Mapping::MappingAtTime (esvo_Mapping.cpp:261-399) -- the whole frame with
 * device-resident hand-off between the stages: BM -> solve -> cull -> window update -> fusion
 * of the whole window (newest first) -> clean -> (regularize).  Results are fetched with
 * esvo_map_download.  counters_out[8] (may be NULL): n_events, n_seeds, n_solved, n_culled,
 * n_fusions, bm_evals, lm_evals, map_size. */
ESVO_API int esvo_mapping_at_time(esvo_ctx* ctx, const uint16_t* ex, const uint16_t* ey,
                                  const int64_t* et_ns, size_t n_events,
                                  const int64_t* pose_t_ns, const double* poses, size_t n_poses,
                                  uint64_t* counters_out);
/* The SGM of esvo_Mapping::InitializationAtTime: cv::StereoSGBM::create(0, numDisparities, blockSize, P1, P2,
 * disp12MaxDiff, preFilterCap, uniquenessRatio)->compute(left, right, disp) in MODE_SGBM with minDisparity 0
 * (esvo_core/src/esvo_Mapping.cpp:101-108 uses (0, 48, 11, 8*11*11, 32*11*11, -1, 0, 11); :444 compute).
 * Bit-exact restatement of OpenCV's integer algorithm on the device (Birchfield-Tomasi cost, 11x11 box aggregation,
 * five 16-bit path costs, uniqueness + left-right check, 3x3 median).  left/right: H*W mono8 host images, or both NULL to
 * use the observation pair currently on the device (esvo_set_ts_pair[_dev]).  disp16_out: H*W CV_16S (disparity * 16,
 * -16 = invalid), host.  Feed it to esvo_init_from_disparity.  numDisparities <= 128. */
ESVO_API int esvo_sgbm_compute(esvo_ctx* ctx, const uint8_t* left, const uint8_t* right, int num_disparities, int block_size,
                               int P1, int P2, int disp12_max_diff, int pre_filter_cap, int uniqueness_ratio, int16_t* disp16_out);

/* esvo_Mapping::InitializationAtTime (esvo_core/src/esvo_Mapping.cpp:433-492) downstream of its SGM call, incl.
 * createEdgeMask (:1000-1044, undistorted events, radius 0) and DepthFusion::naive_propagation
 * (esvo_core/src/core/DepthFusion.cpp:232-327).  `disp16` is the H*W CV_16S map cv::StereoSGBM::compute returns
 * (disparity * 16, negative = invalid) for the current time-surface pair -- the SGM itself stays with the caller
 * (OpenCV, once at start-up).  One DepthPoint (Gaussian, variance 1e-6, age = age_vis_threshold) is created per event
 * whose rectified pixel carries a disparity inside the inverse-depth range, in event order; if there are at least
 * `min_points` (INIT_SGM_DP_NUM_Threshold) of them they become the first vector of the fusion window and are splat
 * (nearest wins) into a fresh map at T_world_left, which esvo_map_download then returns.  *accepted = 0 otherwise. */
ESVO_API int esvo_init_from_disparity(esvo_ctx* ctx, const int16_t* disp16, const uint16_t* ex, const uint16_t* ey,
                                      size_t n_events, const double T_world_left[16], size_t min_points,
                                      size_t* n_points, int* accepted);

/* Copies vector `index` (0 = oldest) of the fusion window dqvDepthPoints_ (esvo_Mapping.h:165) to the host, in its
 * stored order; *n in: capacity, out: count.  ESVO_ERR_INVALID_ARG if there is no such vector. */
ESVO_API int esvo_window_download(esvo_ctx* ctx, int index, esvo_depth_point* out, size_t* n);

/* Drops the fusion window (dqvDepthPoints_) -- the reference does this on reset. */
ESVO_API int esvo_mapping_reset(esvo_ctx* ctx);

/* ---------------- comparison modes of esvo_MVStereo (SURVEY 8f row 4) ---------------- */
/* EventMatcher parameters: EventMatcher ctor / resetParameters (esvo_core/src/core/EventMatcher.cpp:9-49) as esvo_MVStereo
 * fills them from its yaml (esvo_core/src/esvo_MVStereo.cpp:81-91: EM_Time_THRESHOLD, EM_EPIPOLAR_THRESHOLD,
 * EM_TS_NCC_THRESHOLD, patch_size_X/Y) and its thread count NUM_THREAD_MAPPING (:45; output order only). */
typedef struct {
  double time_threshold_s;   /* EM_Time_THRESHOLD   (5e-5; 5e-4 in the shipped yamls) */
  double epipolar_threshold; /* EM_EPIPOLAR_THRESHOLD (0.5; 1.0)                       */
  double ts_ncc_threshold;   /* EM_TS_NCC_THRESHOLD (0.1)                              */
  int32_t patch_size_x, patch_size_y;
  int32_t num_thread;
  int32_t _pad;
} esvo_em_params;

/* replaces: EventMatcher::createMatchProblem + match_all_HyperThread / match / match_an_event
 * (esvo_core/src/core/EventMatcher.cpp:51-58,60-163,185-251) -- the event-to-event matcher of [26] the reference keeps for
 * its MVStereo modes 0 and 2: per left event the time-ordered right events within +-time_threshold/2 of the same polarity
 * (temporal check), within epipolar_threshold rows of the rectified left event and left of it (epipolar check) are
 * triangulated and scored by the ZNCC of the two time-surface patches warped with that depth (warping2,
 * patchInterpolation2, zncc_cost :253-346); the cheapest one below ts_ncc_threshold wins.
 * Left events: the contiguous events of all slices (eventSlicingForEM, esvo_MVStereo.cpp:1008-1040); slice_counts[s] =
 * EventSlice::numEvents_, slice_poses[16 s] = EventSlice::transf_ (T_world_virtual, row-major).  Right events: the
 * candidate vector vEventsPtr_right_, time-ordered.  Uses the observation pair of esvo_set_ts_pair.
 * seeds_out in the reference's thread-major order; *n_seeds: in = capacity, out = count; n_patch_evals = zncc_cost calls. */
ESVO_API int esvo_em_match(esvo_ctx* ctx, const esvo_em_params* prm, const uint16_t* lx, const uint16_t* ly,
                           const int64_t* lt_ns, const uint8_t* lpol, size_t n_left, const int32_t* slice_counts,
                           const double* slice_poses, size_t n_slices, const uint16_t* rx, const uint16_t* ry,
                           const int64_t* rt_ns, const uint8_t* rpol, size_t n_right, esvo_seed* seeds_out,
                           size_t* n_seeds, uint64_t* n_patch_evals);
/* replaces: esvo_MVStereo::vEMP2vDP (esvo_core/src/esvo_MVStereo.cpp:1072-1097): EventMatchPairs -> Gaussian DepthPoints
 * (row/col = floor of the rectified coordinate, variance bounded to 1e-6, residual = cost, age = age_vis_threshold). */
ESVO_API int esvo_seeds_to_points(esvo_ctx* ctx, const esvo_seed* seeds, size_t n, esvo_depth_point* pts_out);
/* replaces: DepthFusion::naive_propagation (esvo_core/src/core/DepthFusion.cpp:232-327) of one DepthPoint vector into the
 * ctx's DepthFrame (nearest wins, no fusion) -- the accumulation step of MVStereo modes 0, 1 and 4
 * (esvo_MVStereo.cpp:280-286,355-361,423-427).  reset_map as in esvo_fuse. */
ESVO_API int esvo_naive_propagate(esvo_ctx* ctx, const esvo_depth_point* pts, size_t n, const double T_world_frame[16],
                                  int reset_map);

/* ---------------- tracking ---------------- */
/* replaces: RegProblemSolverLM::resetRegProblem -> RegProblemLM::setProblem
 * (RegProblemSolverLM.cpp:45-74, RegProblemLM.cpp:24-68).  ref_xyz: the reference point cloud in
 * WORLD coordinates (pcl::PointXYZ floats); it is permuted in place by the reference's
 * rand()-driven partial shuffle, exactly like ref->vPointXYZPtr_.  ts_left: current mono8 TS
 * (NULL = last esvo_ts_build(cam 0)).  Returns 1 when the reference would return false
 * (fewer ref points than BATCH_SIZE). */
ESVO_API int esvo_track_reset(esvo_ctx* ctx, float* ref_xyz, size_t n, const double T_world_ref[16],
                              const double T_world_cur_prior[16], const uint8_t* ts_left);
/* replaces: RegProblemSolverLM::solve_analytical / solve_numerical
 * (RegProblemSolverLM.cpp:76-146,148-217) + RegProblemLM::setPose. */
ESVO_API int esvo_track_solve(esvo_ctx* ctx, int analytical, double T_world_cur_out[16],
                              esvo_lm_stats* stats);
/* Seeds the C library rand() stream used by setProblem's stochastic sampling (the reference
 * never seeds it, i.e. glibc seed 1).  Only meaningful for reproducible tests. */
ESVO_API int esvo_track_srand(esvo_ctx* ctx, unsigned seed);
/* Debug/parity taps: negative TS and its Sobel gradients (TimeSurfaceObservation.h:118-147). */
ESVO_API int esvo_track_get_negative_ts(esvo_ctx* ctx, double* ts_neg, double* d_du, double* d_dv);

/* ---------------- device-resident staging (bench "value" leg, pipelines) ---------------- */
/* Split forms of the host-buffer calls above: stage = H2D only, run = kernels only (async on
 * the ctx stream), fetch = D2H only.  esvo_sync waits for the ctx stream.
 * Event packets: when x, y, t_ns and pol (>= 4096 events) lie next to each other in host memory -- one packet buffer in any
 * order, at most 64 bytes of padding in total -- esvo_stage_ts_events / esvo_ts_push_events move them with ONE copy instead
 * of four (the host-buffer path is host-issue-bound); separate allocations work as before. */
ESVO_API int esvo_stage_ts_events(esvo_ctx* ctx, int cam, const uint16_t* x, const uint16_t* y,
                                  const int64_t* t_ns, const uint8_t* pol, size_t n);
ESVO_API int esvo_run_ts_build(esvo_ctx* ctx, int cam, int64_t t_sync_ns);
ESVO_API int esvo_stage_mapping_inputs(esvo_ctx* ctx, const uint16_t* ex, const uint16_t* ey,
                                       const int64_t* et_ns, size_t n_events,
                                       const int64_t* pose_t_ns, const double* poses,
                                       size_t n_poses);
ESVO_API int esvo_run_mapping(esvo_ctx* ctx);
ESVO_API int esvo_fetch_mapping_counters(esvo_ctx* ctx, uint64_t counters_out[8]);
ESVO_API int esvo_sync(esvo_ctx* ctx);
/* Software pipelining of consecutive mapping frames (1 = strictly sequential, the default; up to 16).
 * With depth S the frames issued through esvo_set_ts_pair_dev / esvo_stage_mapping_inputs(_dev) /
 * esvo_run_mapping rotate over S buffer sets and CUDA streams so that the serial tail of one frame's
 * LM kernel overlaps with the next frames; results are identical to depth 1. */
ESVO_API int esvo_set_pipeline_depth(esvo_ctx* ctx, int depth);
/* Asynchronous result hand-off for pipelined operation.  esvo_results_begin enqueues, right behind the
 * frame just issued with esvo_run_mapping, the compaction of its fused map and the read-back of its
 * counters; esvo_results_end(ticket) waits for that frame only, copies the map out in element-list order
 * (same content as esvo_map_download) and fills counters_out[8] (same layout as esvo_mapping_at_time).
 * Each pipeline slot holds one pending ticket: collect frame j before issuing frame j + depth. */
ESVO_API int esvo_results_begin(esvo_ctx* ctx, int64_t* ticket_out);
ESVO_API int esvo_results_end(esvo_ctx* ctx, int64_t ticket, esvo_depth_point* out, size_t* n,
                              uint64_t* counters_out);
/* Zero-copy form of esvo_results_end: *out points into the slot's pinned host landing buffer, which the gather kernel
 * filled over PCIe (element-list order); it stays valid until that slot's next esvo_results_begin. */
ESVO_API int esvo_results_end_view(esvo_ctx* ctx, int64_t ticket, const esvo_depth_point** out, size_t* n,
                                   uint64_t* counters_out);
/* Device-pointer forms (suffix _dev): the arrays are CUDA device pointers on the ctx's device, i.e.
 * the inputs are already resident in HBM; work is enqueued on the ctx stream, nothing is synchronised.
 * esvo_stage_mapping_inputs_dev uses its arrays IN PLACE (no copy): keep them valid and unchanged until the frame has
 * been collected with esvo_results_end or the ctx synchronised.
 * esvo_set_ts_pair_dev hands the images of the last two esvo_run_ts_build calls to the mapper. */
ESVO_API int esvo_ts_push_events_dev(esvo_ctx* ctx, int cam, const uint16_t* x_dev, const uint16_t* y_dev,
                                     const int64_t* t_ns_dev, const uint8_t* pol_dev, size_t n);
ESVO_API int esvo_stage_mapping_inputs_dev(esvo_ctx* ctx, const uint16_t* ex_dev, const uint16_t* ey_dev,
                                           const int64_t* et_ns_dev, size_t n_events,
                                           const int64_t* pose_t_ns_dev, const double* poses_dev,
                                           size_t n_poses);
ESVO_API int esvo_set_ts_pair_dev(esvo_ctx* ctx, const double T_world_left[16]);

/* Device-resident hand-off of the closed loop: the time-surface history, the published local map and the tracker's
 * reference cloud stay in HBM.  Results are bit for bit those of the host forms on host copies of the same data.
 *
 * replaces: esvo_Mapping::TS_history_ (esvo_Mapping.h, std::map<ros::Time, TimeSurfaceObservation>) as timeSurfaceCallback
 * fills it (esvo_Mapping.cpp:716-762).  A ring of `capacity` stereo pairs on the device, keyed by build stamp.  capacity 0
 * (the default) frees it; any call drops what the history held. */
ESVO_API int esvo_ts_history_reserve_dev(esvo_ctx* ctx, size_t capacity);
/* Stores the images of the last esvo_ts_build / esvo_run_ts_build of both cameras under stamp_ns: the device-to-device copy is
 * ordered behind both builds with CUDA events, no host sync.  Like the map's operator[] followed by erase(begin()) while over
 * capacity: a stored stamp is overwritten, and a full history drops its smallest stamp (or the new pair, if that is smaller).
 * ESVO_ERR_STATE without a reserved history or before both cameras were built. */
ESVO_API int esvo_ts_history_store_dev(esvo_ctx* ctx, int64_t stamp_ns);
/* replaces: the TimeSurfaceObservation dataTransferring takes from TS_history_ (esvo_Mapping.cpp:494-533) handed to the mapper:
 * the same effect as esvo_set_ts_pair with the two images stored under stamp_ns (SmoothTimeSurface included), so that
 * esvo_bm_match / esvo_mapping_at_time / esvo_sgbm_compute(NULL, NULL) run on it.  A stamp that was never stored or has been
 * dropped returns ESVO_ERR_STATE (esvo_last_error says which) and leaves the context as it was. */
ESVO_API int esvo_set_ts_pair_stored_dev(esvo_ctx* ctx, int64_t stamp_ns, const double T_world_left[16]);
/* replaces: publishPointCloud's packing (esvo_Mapping.cpp:909-953; the host form is frontend::packPointCloud over
 * esvo_map_download): every DepthMap element, in element-list order, becomes p_world = R p_cam + t of T_world_result as f32
 * x, y, z, into a device cloud the context keeps as "the cloud published at stamp_ns".  *n_points: the point count (0 for an
 * empty map; the reference then publishes nothing).  Synchronises once, for the count. */
ESVO_API int esvo_map_publish_dev(esvo_ctx* ctx, const double T_world_result[16], int64_t stamp_ns, size_t* n_points);
/* Read-back of the published cloud into a device buffer of *n (in: capacity in points, out: count) x 3 floats, and its stamp
 * (may be NULL); synchronous.  ESVO_ERR_STATE before the first publish, ESVO_ERR_CAPACITY (with *n set) if it does not fit. */
ESVO_API int esvo_map_published_cloud_dev(esvo_ctx* ctx, float* xyz_dev, size_t* n, int64_t* stamp_ns);
/* replaces: esvo_Tracking::refDataTransferring's copy of the reference cloud (esvo_Tracking.cpp:177-211): snapshots the newest
 * cloud published on this context, which must be the one of stamp_ns (ESVO_ERR_STATE otherwise), for esvo_track_reset_dev;
 * later publishes do not change it.  *n_points (may be NULL): its point count. */
ESVO_API int esvo_track_adopt_map_dev(esvo_ctx* ctx, int64_t stamp_ns, size_t* n_points);
/* replaces: RegProblemSolverLM::resetRegProblem -> RegProblemLM::setProblem (RegProblemSolverLM.cpp:45-74,
 * RegProblemLM.cpp:24-68) on the adopted cloud: esvo_track_reset with the reference cloud on the device.  The stochastic
 * sampling permutes an index list of the adopted cloud instead of the cloud, carried from reset to reset until the next
 * adoption, with the same rand() draws (the stream esvo_track_reset and esvo_track_srand use); the result is exactly that of
 * esvo_track_reset on a host copy of the cloud.  ts_left as in esvo_track_reset.  Returns 1 when the cloud has fewer than
 * BATCH_SIZE points; ESVO_ERR_STATE before an adoption. */
ESVO_API int esvo_track_reset_dev(esvo_ctx* ctx, const double T_world_ref[16], const double T_world_cur_prior[16],
                                  const uint8_t* ts_left);
/* Event windows read from the time-surface log: the left events the closed loop's mapper and tracker search were pushed into
 * camera cam's log (esvo_ts_push_events), so the nodes' own event buffers are not needed.  A node's buffer is the logical
 * buffer [front, total) of global push indices: total = events pushed since esvo_create / esvo_ts_reset, front = where the
 * node's deque would begin (the mapper caps it at 3e6 events: max(0, total - 3e6); the tracker at 5e6 and clears it on
 * reset(): max(push index at its last reset, total - 5e6)).  The results equal the host forms on that deque bit for bit.
 * Refusals, with the reason in esvo_last_error: ESVO_ERR_UNSUPPORTED when the answer depends on events folded out of the
 * resident log (the newest 1 Mi at least stay resident; see esvo_ts_build), when the camera takes unordered input or its
 * events were not pushed in time order (the log is in arrival order, the deques are sorted); ESVO_ERR_STATE at pipeline
 * depth > 1; ESVO_ERR_INVALID_ARG for front outside [0, total].
 *
 * replaces: the newest-first walk of esvo_Mapping::dataTransferring (esvo_Mapping.cpp:538-552 SGM, :554-575 BM; host form
 * frontend::selectSGMEvents / selectCloseEvents) and, with denoise != 0, createDenoisingMask + extractDenoisedEvents
 * (:282-296,1046-1072).  The walk starts at lower_bound(t_end_ns) and stops before lower_bound(t_begin_ns) (tools::
 * EventBuffer_lower_bound, utils.h:50-55: toSec() doubles) after at most `budget` events (PROCESS_EVENT_NUM for BM,
 * PROCESS_EVENT_NUM + 1 for SGM); when no event is at or after t_end_ns, the one-past-the-end slot is skipped but keeps its
 * place in the budget.  t_begin_ns is the caller's fromSec(max(0, toSec(t_end) - window)), t_begin_ns <= t_end_ns.  With
 * denoise, the walked events with x < W, y < H draw a 0/255 event map, a 3x3 median (borders replicated) keeps a pixel when at
 * least 5 of its 9 neighbours are on, and the walked events whose mask value at the flat index y * W + x is 255 are kept in walk
 * order; without, every walked event is.  At most max_keep are kept.  Deviation: a flat index >= H * W reads outside the
 * reference's mask (undefined behaviour); such an event is not kept.  The selection stays on the device for the _selected_dev
 * calls below; *n (may be NULL): its size.  Work and memory are linear in min(budget, resident events): a walk over the whole
 * resident log (4 Mi events) is allowed, the closed loop's windows are ~1 000 events.  Synchronises once, for the scalars. */
ESVO_API int esvo_events_window_dev(esvo_ctx* ctx, int cam, int64_t front, int64_t t_begin_ns, int64_t t_end_ns, size_t budget,
                                    int denoise, size_t max_keep, size_t* n);
/* replaces: the two EventBuffer_lower_bound calls of esvo_Tracking::curDataTransferring (esvo_Tracking.cpp:240-263), whose
 * difference + 1 is numEventsSinceLastObs_.  idx_out[i]: lower_bound(t_ns[i]) over [front, total) as a global push index;
 * k <= 64 stamps per call.  Synchronous.  When some bounds lie among events folded out of the resident log, the others are
 * still written, those are -1, and the call returns ESVO_ERR_UNSUPPORTED; on every other refusal idx_out is left untouched. */
ESVO_API int esvo_events_lower_bound_dev(esvo_ctx* ctx, int cam, int64_t front, const int64_t* t_ns, size_t k, int64_t* idx_out);
/* Read-back of the last selection into device buffers of *n (in: capacity, out: count) events, newest first; synchronous.
 * ESVO_ERR_STATE without a selection, ESVO_ERR_CAPACITY (with *n set) if it does not fit. */
ESVO_API int esvo_events_selected_dev(esvo_ctx* ctx, uint16_t* x_dev, uint16_t* y_dev, int64_t* t_ns_dev, size_t* n);
/* replaces: esvo_Mapping::MappingAtTime (esvo_Mapping.cpp:261-399) on the last selection: esvo_mapping_at_time with the selected
 * events, used in place.  Poses and counters as there. */
ESVO_API int esvo_mapping_at_time_selected_dev(esvo_ctx* ctx, const int64_t* pose_t_ns, const double* poses, size_t n_poses,
                                               uint64_t* counters_out);
/* replaces: InitializationAtTime downstream of the SGM (esvo_Mapping.cpp:433-492) on the last selection: esvo_init_from_disparity
 * with the selected events. */
ESVO_API int esvo_init_from_disparity_selected_dev(esvo_ctx* ctx, const int16_t* disp16, const double T_world_left[16],
                                                   size_t min_points, size_t* n_points, int* accepted);
/* Per-stage device timing with CUDA events on the ctx stream.  Stages: 0 time surface, 1 block
 * matching, 2 seed ordering, 3 depth LM, 4 point ordering/culling, 5 fusion+clean+regularise,
 * 6 tracking.  esvo_profile(ctx, stage_mask): bit s switches the timing of stage s on (0 = off, 0xff = all).
 * esvo_profile_read synchronises, returns accumulated ms and launch counts per stage since the last read
 * and clears them. */
/* Raw device counters of the last esvo_fetch_mapping_counters / esvo_mapping_at_time
 * (idx 7 = DepthProblem evaluations actually executed by the LM kernel, which re-uses f(x) inside
 * the forward difference instead of recomputing it like NumericalDiff does). */
ESVO_API uint64_t esvo_debug_counter(esvo_ctx* ctx, int idx);
ESVO_API int esvo_profile(esvo_ctx* ctx, int stage_mask);
ESVO_API int esvo_profile_read(esvo_ctx* ctx, double ms_out[8], uint64_t count_out[8]);
/* CUDA stream of the ctx (cudaStream_t as void*), so callers can record events on it. */
ESVO_API void* esvo_stream(esvo_ctx* ctx);
/* Number of kernel launches issued by this ctx so far. */
ESVO_API uint64_t esvo_launch_count(esvo_ctx* ctx);
ESVO_API const char* esvo_last_error(esvo_ctx* ctx);
ESVO_API const char* esvo_version(void);

#ifdef __cplusplus
}
#endif

#include "esvo_b200_bag.h"   /* the packed event ingest (no oracle counterpart) */
#include "esvo_b200_hotpix.h"   /* hot pixels at the packed ingest (no oracle counterpart) */
#include "esvo_b200_inflate.h"   /* compressed bag chunks inflated on the device (no oracle counterpart) */
#endif /* ESVO_B200_H_ */
