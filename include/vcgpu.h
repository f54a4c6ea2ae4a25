/* vcgpu.h — C-ABI of the H100 calibration-solve library (libvcgpu.so).
 *
 * Drop-in boundary for the path that sits behind `ceres::Solve` in the reference:
 * it replaces ceres::Problem construction + ceres::Solve + Problem::Evaluate as used by
 * ViCalibrator (include/vicalib/vicalibrator.h:152, 548-679, 859-916, 956-971).  Plain
 * pointers and sizes only; every entry point returns 0 on success and a negative code on
 * error (message via vcgpu_last_error); nothing throws or aborts across this boundary.
 *
 * All arithmetic is FP64.  Quaternions are (x, y, z, w); SE3 is [q(4) | t(3)], the storage
 * the reference's parameter blocks use (local-param-se3.h:34, vicalibrator.h:460-461).
 */
#ifndef VCGPU_H_
#define VCGPU_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vcgpu_handle vcgpu_handle;

/* camera model ids; intrinsics are fu, fv, u0, v0, <distortion...> (vicalib-engine.cc:205-250) */
enum {
  VCGPU_CAM_LINEAR = 0, /* K=4  calibu_fu_fv_u0_v0         vicalibrator.h:448 */
  VCGPU_CAM_FOV = 1,    /* K=5  calibu_fu_fv_u0_v0_w       vicalibrator.h:412 */
  VCGPU_CAM_POLY2 = 2,  /* K=6  calibu_fu_fv_u0_v0_k1_k2   vicalibrator.h:419 */
  VCGPU_CAM_POLY3 = 3,  /* K=7  ..._k1_k2_k3               vicalibrator.h:427 */
  VCGPU_CAM_KB4 = 4     /* K=8  calibu_fu_fv_u0_v0_kb4     vicalibrator.h:441 */
};
#define VCGPU_MAX_INTR 10 /* stride of the intrinsics array per camera */

enum {
  VCGPU_OK = 0,
  VCGPU_ERR_INVALID = -1,  /* bad argument / call order (reference: glog CHECK, vicalibrator.h:254,356,396) */
  VCGPU_ERR_CUDA = -2,     /* CUDA runtime failure (no CPU fallback exists) */
  VCGPU_ERR_NUMERIC = -3,  /* normal equations not positive definite even after damping */
  VCGPU_ERR_COMM = -4      /* NCCL failure */
};

typedef struct {
  int device; /* CUDA device ordinal, -1 = current device */
} vcgpu_config;

/* Which parameter blocks are variable — ViCalibrator::SetupProblem's constant masks
 * (vicalibrator.h:572-592, 651-676) and SetOptimizationFlags (vicalibrator.h:252-260). */
typedef struct {
  int inertial;         /* is_inertial_active_ && FLAGS_calibrate_imu: IMU residuals on, cam0 q_ck variable */
  int rotation_only;    /* optimize_rotation_only_: IMU residual rows 0-2,6-8 zeroed, gravity & cam0 p_ck constant */
  int bias_active;      /* is_bias_active_ */
  int scale_active;     /* is_scale_factor_active_ */
  int optimize_ts;      /* optimize_time_offset_ */
  int fix_intrinsics;   /* fix_intrinsics_ (vicalibrator.h:346,591) */
  int visual;           /* is_visual_active_ */
  double visual_mult;   /* residual-block multiplicity of the staged flow (vicalibrator.h:641-656 re-adds blocks) */
  double imu_mult;
} vcgpu_flags;

/* ceres::Solver::Options as ViCalibrator sets them (vicalibrator.h:141-152) */
typedef struct {
  int max_iters;           /* FLAGS_max_iters, default 200 (vicalib-engine.cc:94) */
  double function_tol;     /* 1e-6 (vicalibrator.h:149) */
  double gradient_tol;     /* Ceres default 1e-10 */
  double param_tol;        /* Ceres default 1e-8 */
  double init_radius;      /* Ceres default 1e4 */
  int strategy;            /* 0 = LEVENBERG_MARQUARDT, 1 = DOGLEG (vicalibrator.h:151) */
  int jacobi_scaling;      /* Ceres default on */
  int update_imu_weights;  /* run UpdateImuWeights before the solve and after every iteration (vicalibrator.h:691,955) */
  int update_state_every_iteration; /* copy the state to the host mirrors before each callback (vicalibrator.h:148) */
} vcgpu_options;

/* ceres::IterationSummary fields the reference's callback reads (vicalibrator.h:696-714) */
typedef struct {
  int iteration;
  int step_is_successful;
  double cost;
  double cost_change;
  double gradient_max_norm;
  double gradient_norm;
  double step_norm;
  double relative_decrease;
  double trust_region_radius;
} vcgpu_iteration;

/* return nonzero to stop (ceres::SOLVER_TERMINATE_SUCCESSFULLY, vicalibrator.h:717) */
typedef int (*vcgpu_iter_cb)(const vcgpu_iteration* it, void* user);

enum {
  VCGPU_TERM_NO_CONVERGENCE = 0, /* max iterations */
  VCGPU_TERM_FUNCTION_TOL = 1,
  VCGPU_TERM_GRADIENT_TOL = 2,
  VCGPU_TERM_PARAM_TOL = 3,
  VCGPU_TERM_CALLBACK = 4,       /* callback asked to stop, or gradient norm < 1e-9 rule (vicalibrator.h:713-717) */
  VCGPU_TERM_RADIUS = 5
};

/* ceres::Solver::Summary subset (vicalibrator.h:975-976) */
typedef struct {
  int iterations;
  int successful_steps;
  int termination;
  int num_residuals;
  double initial_cost;
  double final_cost;
  double device_seconds; /* CUDA-event time of the iteration loop */
  int kernel_launches;   /* kernels this library launched during the solve */
} vcgpu_summary;

int vcgpu_create(const vcgpu_config* cfg, vcgpu_handle** out);
int vcgpu_destroy(vcgpu_handle* h);
const char* vcgpu_last_error(const vcgpu_handle* h);

/* ---- problem upload (host buffers are copied; caller keeps ownership) --------------------
 * replaces AddParameterBlock / AddResidualBlock (vicalibrator.h:559-604, 628-632, 645-654) */
int vcgpu_set_cameras(vcgpu_handle* h, int n_cams, const int32_t* model, const double* intr /*n*10*/,
                      const double* q_ck /*n*4*/, const double* p_ck /*n*3*/);
/* time: absolute stamps on the IMU's clock, Unix time included (the reference stamps frames and samples with the host's
 * clock by default).  Every time sum is formed in binary64 in the reference's order (t_i + ts, z0.time + dt / 2,
 * z0.time + dt), and results depend on the stamps only through those roundings: no stamp is rebased or narrowed.  At
 * current Unix times (2^30 s < t < 2^31 s) a sum t + ts resolves 2^-22 s, so a change of ts below ~1.2e-7 s does not
 * move the residual although the Jacobian's ts column is not zero.  That is the reference's behaviour. */
int vcgpu_set_frames(vcgpu_handle* h, int n_frames, const double* T_wp /*n*7*/, const double* v_w /*n*3*/,
                     const double* time /*n*/);
/* any order; the library groups by (camera, frame) internally and keeps the caller's order for outputs */
int vcgpu_set_observations(vcgpu_handle* h, int64_t n_obs, const int32_t* frame_id, const int32_t* cam_id,
                           const double* p_w /*n*3*/, const double* p_c /*n*2*/);
/* strictly increasing timestamps (vicalibrator.h:373-378), absolute like vcgpu_set_frames' (Unix time included) and
 * used as given: the time arithmetic and its rounding are vcgpu_set_frames' */
int vcgpu_set_imu(vcgpu_handle* h, int n, const double* t, const double* w /*n*3*/, const double* a /*n*3*/,
                  double sigma_g, double sigma_a);
int vcgpu_set_imu_params(vcgpu_handle* h, const double g[2], const double b[6], const double sf[6], double ts);
int vcgpu_set_flags(vcgpu_handle* h, const vcgpu_flags* flags);
int vcgpu_set_options(vcgpu_handle* h, const vcgpu_options* opts);
void vcgpu_default_flags(vcgpu_flags* flags);
void vcgpu_default_options(vcgpu_options* opts);

/* host mirrors updated before every callback when update_state_every_iteration is set, and at
 * the end of vcgpu_solve; any pointer may be NULL (vicalibrator.h:148: the GUI thread polls them) */
int vcgpu_register_mirrors(vcgpu_handle* h, double* intr, double* q_ck, double* p_ck, double* T_wp,
                           double* v_w, double* g, double* b, double* sf, double* ts);

/* ---- the hot path ---------------------------------------------------------------------- */
/* ceres::Solve(solver_options_, problem_, &summary)  (vicalibrator.h:956) */
int vcgpu_solve(vcgpu_handle* h, vcgpu_iter_cb cb, void* user, vcgpu_summary* out);
/* vcgpu_solve of n handles in one call, free-running (no callback; the host mirrors are written once, at the end).
 * Every rig runs inside its own thread-block cluster of 1, 2, 4 or 8 CTAs (the fewest whose warps hold the rig's
 * frames), so many small rigs share the GPU instead of taking it in turns; rigs of the same strategy, cluster size
 * and warp count go into ONE kernel launch.  Each handle's own options (strategy, tolerances, max_iters,
 * jacobi_scaling, init_radius) and flags apply to it, each rig stops on its own, and its result equals its
 * vcgpu_solve to rounding and does not depend, bit for bit, on what else is in the batch or in which order.
 * out: n summaries or NULL.  device_seconds is the CUDA-event time of the launch the rig ran in (shared by the rigs
 * of that launch); kernel_launches counts the rig's own start-point launches plus that one.
 * Returns VCGPU_ERR_INVALID before anything is launched, with a message naming the index in vcgpu_last_error of every
 * non-null handle of the batch, for: n <= 0, a null or repeated handle, handles on different devices, and a handle
 * that has inertial terms on, frame shards, a vcgpu_set_profiling bit (1, 4) or L2 flushing set,
 * update_state_every_iteration set, no active observation, or a rig too large for the persistent vision kernel.
 * There is no sequential fallback: call vcgpu_solve on such a handle.  A refused batch leaves its handles as they were.
 * Device memory: nothing beyond what each handle holds for vcgpu_solve, which includes a 32 MiB totals buffer per
 * handle (so n handles hold n x 32 MiB plus their problems), and n x ~1 KB of kernel arguments. */
int vcgpu_solve_batch(vcgpu_handle* const* handles, int n, vcgpu_summary* out /* n, or NULL */);
/* how vcgpu_solve_batch would run this handle: CTAs per cluster (1, 2, 4 or 8), warps per CTA, and how many clusters
 * of that shape the device holds at once (cudaOccupancyMaxActiveClusters; further rigs of a batch queue behind them).
 * Any pointer may be NULL.  VCGPU_ERR_INVALID where the batch would refuse the handle's rig. */
int vcgpu_batch_plan(vcgpu_handle* h, int* cluster_size, int* warps, int* resident_clusters);
/* vcgpu_solve of n handles with inertial terms on, in one call, free-running (no callback; the host mirrors are written
 * once, at the end).  Every rig runs inside its own thread-block cluster of 1, 2, 4 or 8 CTAs of the persistent
 * inertial kernels (the fewest whose two elimination groups per CTA take the rig's level-0 chunks in one round), so
 * many rigs share the GPU instead of taking it in turns.  An iteration is one solve launch and one evaluation launch
 * per cluster size for the whole batch; the host reads every rig's control block between bursts of up to 4
 * iterations.  Each handle's own options (max_iters, tolerances, jacobi_scaling, init_radius, update_imu_weights)
 * and flags apply to it, each rig stops on its own, and its result equals its vcgpu_solve to rounding (the weights
 * update runs in the evaluation launch, as with VCGPU_NO_DEFERRED_WEIGHTS) and does not depend, bit for bit, on what
 * else is in the batch or in which order.  A vcgpu_solve after the batch gives the bits it gives on a fresh handle.
 * out: n summaries or NULL.  device_seconds is the CUDA-event time of the batch's iteration loop (shared by all its
 * rigs); kernel_launches counts the rig's own launches (Jacobi scale, weights updates) plus every batch launch it
 * took part in: the start point's evaluation and two per iteration queued for it, the same count as vcgpu_solve's
 * when every iteration runs.
 * Returns VCGPU_ERR_INVALID before any kernel is launched, with a message naming the index in vcgpu_last_error of
 * every non-null handle of the batch, for: n <= 0, a null or repeated handle, handles on different devices, and a
 * handle without inertial terms (vision rigs: vcgpu_solve_batch), with strategy 1 (inertial DOGLEG runs on the
 * multi-launch engine), frame shards, a vcgpu_set_profiling bit (1, 4, 8) or L2 flushing set, update_state_every_iteration set,
 * or a rig the persistent inertial kernels do not fit (G >= 68 on an H100).  There is no sequential fallback: call
 * vcgpu_solve on such a handle.  A refused batch leaves its handles as they were.
 * Device memory: nothing beyond what each handle holds for vcgpu_solve, and n x ~5 KB of kernel arguments held by
 * handle 0. */
int vcgpu_solve_batch_inertial(vcgpu_handle* const* handles, int n, vcgpu_summary* out /* n, or NULL */);
/* how vcgpu_solve_batch_inertial would run this handle: CTAs per cluster (1, 2, 4 or 8) and how many clusters of that
 * size the device holds at once (the smaller count of the solve and the evaluation kernel; further rigs of a batch
 * queue behind them).  Any pointer may be NULL.  VCGPU_ERR_INVALID where the batch would refuse the handle. */
int vcgpu_batch_plan_inertial(vcgpu_handle* h, int* cluster_size, int* resident_clusters);
/* The staged calibration flow of ViCalibrator::SolveThread (vicalibrator.h:919-1040) for n rigs in one call.  Per rig:
 * vision only -> inertial, rotation only -> translation, gravity and biases -> scale factors -> outlier removal ->
 * finished, a stage advancing only when its solve converges (termination other than VCGPU_TERM_NO_CONVERGENCE).  At
 * every stage entry the handle gets what SetupProblem gives it: its own state uploaded again (vcgpu_set_cameras,
 * vcgpu_set_frames, vcgpu_set_imu_params), the stage's flags and, with block_duplication, the multiplicities of the
 * blocks added so far (visual 1, 2, 3, ...; IMU 1, 1, 2, 3, ... from the first inertial stage on); then, on entering
 * the first stage past rotation-only with gravity not yet initialised, gravity from the mid-frame accelerometer sample.
 * After each solve: the per-camera RMSE sqrt(cost / n) (vcgpu_evaluate), the stage decision and, at its step,
 * vcgpu_remove_outliers with the rig's own RMSE.  Each rig starts at the stage its vcgpu_set_flags describe (inertial,
 * rotation_only, bias_active, scale_active as SetOptimizationFlags sets them; without calibrate_imu every stage is a
 * vision stage) and runs every solve with its own options, strategy included.
 * A round solves every rig still working: the rigs at a vision stage as one vcgpu_solve_batch (LM or DOGLEG), those at
 * an inertial stage as one vcgpu_solve_batch_inertial, which here also takes strategy 1 (DOGLEG inside the inertial
 * cluster kernels); then one vcgpu_evaluate_batch of them all and one vcgpu_remove_outliers_batch of the rigs at that
 * step.  A rig's whole trajectory of stages, solves and results does not depend, bit for bit, on what else is in the
 * batch or in which order.  A rig leaves when it finishes or has had max_solves solves (or has no residual left).
 * out: n summaries or NULL; cam_rmse: NULL, or n pointers (an entry may be NULL) to n_cams RMSEs of the rig's last solve.
 * Returns VCGPU_ERR_INVALID before anything is launched, with a message naming the index in vcgpu_last_error of every
 * non-null handle, for: n <= 0, a null flow, max_solves <= 0, a null or repeated handle, handles on different devices,
 * and a rig that a batch of a kind of stage it can reach would refuse: vcgpu_solve_batch where it starts at a vision
 * stage or calibrate_imu is off, vcgpu_solve_batch_inertial (strategy 1 excepted) where calibrate_imu is on.  A refused
 * call changes no handle's state, flags or options, and a handle solves after it as a fresh one at that state does (a
 * handle checked with its inertial switch flipped is prepared again by its next call). */
typedef struct {
  int calibrate_imu;        /* FLAGS_calibrate_imu: advance through the inertial stages */
  int remove_outliers;      /* FLAGS_remove_outliers */
  double outlier_threshold; /* FLAGS_outlier_threshold */
  int block_duplication;    /* re-add blocks per stage as SetupProblem does (the host mirror's default: on) */
  int gravity_initialized;  /* is_gravity_initialized_ at the start: nonzero keeps the handles' gravity */
  int max_solves;           /* solves per rig at most (the reference repeats a stage that does not converge forever) */
} vcgpu_flow;
enum {  /* vcgpu_flow_summary::stage */
  VCGPU_FLOW_VISION = 0,       /* inertial terms off */
  VCGPU_FLOW_ROTATION = 1,     /* inertial, rotation only */
  VCGPU_FLOW_TRANSLATION = 2,  /* inertial: translation, gravity and biases */
  VCGPU_FLOW_SCALE = 3,        /* inertial: also the scale factors (and the solves after the outlier removal) */
  VCGPU_FLOW_FINISHED = 4      /* the stage machine reached its end */
};
typedef struct {
  int solves, iterations;   /* solves run, and their iterations summed */
  int finished;             /* the stage machine reached its end */
  int stage;                /* VCGPU_FLOW_* at return */
  int64_t outliers_removed; /* observations RemoveOutliers removed */
  double mse;               /* final_cost / num_residuals of the last solve (vicalibrator.h:975) */
  vcgpu_summary last;       /* the last solve's summary */
  vcgpu_flags flags;        /* the handle's flags at return: its last stage's, as SetupProblem set them */
} vcgpu_flow_summary;
int vcgpu_calibrate_batch(vcgpu_handle* const* handles, int n, const vcgpu_flow* flow, vcgpu_flow_summary* out /* n, or NULL */,
                          double* const* cam_rmse /* n pointers to n_cams, or NULL */);
/* run exactly n trust-region iterations with no convergence test and no host round trip per
 * iteration (benchmark entry: LM iterations / second) */
int vcgpu_iterate(vcgpu_handle* h, int n_iterations, vcgpu_summary* out);

/* Problem::Evaluate with residual_blocks = camera `cam` (or all visual blocks if cam < 0),
 * apply_loss_function = false: cost = 1/2 sum |r|^2, residuals in caller observation order
 * (2 per active observation of that camera)  (vicalibrator.h:873-887, 958-966).  Runs as vcgpu_evaluate_batch of this
 * handle alone: the cost of cam < 0 is the sum of the per-camera costs, and the handle keeps that call's device memory.
 * Unlike the batch call it takes frame shards, each evaluating its own observations.  VCGPU_ERR_INVALID: cam >= the
 * number of cameras. */
int vcgpu_evaluate(vcgpu_handle* h, int cam, double* cost, double* residuals_or_null, int64_t* n_blocks);
/* total robustified cost 1/2 sum rho(|r|^2) over all active residual blocks at the current state */
int vcgpu_cost(vcgpu_handle* h, double* cost);
/* RemoveOutliers (vicalibrator.h:859-916): drops observations with |r| > threshold * rmse[cam].  Runs as
 * vcgpu_remove_outliers_batch of this handle alone, and takes frame shards. */
int vcgpu_remove_outliers(vcgpu_handle* h, const double* rmse, double threshold, int64_t* n_removed);
int vcgpu_get_obs_active(vcgpu_handle* h, uint8_t* active /*n_obs, caller order*/);
/* vcgpu_evaluate of every camera of n rigs in one call.  Per rig i: cam_cost[i][c] = 1/2 sum |r|^2 over camera c's
 * active observations (loss-free, as vcgpu_evaluate(h, c)), and cam_blocks[i][c] their count (cam_blocks, or an entry of
 * it, may be NULL); residuals_or_null[i] (the array or an entry may be NULL) gets 2 doubles per active observation in
 * vcgpu_evaluate(h, -1, ...)'s layout, caller order.  The residuals are the bits vcgpu_eval_reproj returns.  One launch covers every rig:
 * tiles of 256 consecutive observations of one camera, one CTA each, a tiling that is a function of the rig alone, so a
 * rig's costs are the same bits whatever else is in the batch and in whatever order.  Per handle, on its own stream,
 * the uploads of vcgpu_evaluate; then the launch and one download of the costs, and one of each rig's residuals.
 * Nothing on the handle changes but what vcgpu_evaluate changes: state, IMU weights and what a later vcgpu_solve or batch
 * solve computes stay as they were.
 * Returns VCGPU_ERR_INVALID before anything is launched and writes nothing, with a message naming the index in
 * vcgpu_last_error of every non-null handle, for: n <= 0, a null or repeated handle, a null cam_cost[i], handles on
 * different devices, and frame shards.
 * Device memory, held by handle 0: 8 bytes per tile and 96 bytes per rig of workspace, and 240 bytes per rig and
 * 24 per tile of kernel arguments; with residuals, per handle 2 n_obs doubles (and n_obs int32 when the caller's order
 * is not sorted by camera and frame). */
int vcgpu_evaluate_batch(vcgpu_handle* const* handles, int n, double* const* cam_cost /* n pointers to n_cams */,
                         int64_t* const* cam_blocks /* n pointers to n_cams, or NULL */,
                         double* const* residuals_or_null /* n pointers to 2 * active observations, or NULL */);
/* vcgpu_remove_outliers of n rigs in one call: rmse[i] holds rig i's n_cams values; an active observation of camera c
 * leaves the problem where |r| > threshold * rmse[i][c], |r| = sqrt(r0 * r0 + r1 * r1) formed without a fused
 * multiply-add.  n_removed: n counts, or NULL.  The residuals are computed as
 * vcgpu_evaluate_batch computes them, in the same launch layout; the marks come back in one download.  A rig that loses
 * nothing is left exactly as it was.  Refusals as vcgpu_evaluate_batch, with a null rmse[i] in place of a null
 * cam_cost[i].  Device memory: vcgpu_evaluate_batch's, and one byte per active observation of every rig, held by
 * handle 0. */
int vcgpu_remove_outliers_batch(vcgpu_handle* const* handles, int n, const double* const* rmse /* n pointers */, double threshold,
                                int64_t* n_removed /* n, or NULL */);
/* UpdateImuWeights (vicalibrator.h:723-799) */
int vcgpu_update_imu_weights(vcgpu_handle* h);
int vcgpu_get_imu_weights(vcgpu_handle* h, double* w_sqrt /*(n_frames-1)*81*/);
int vcgpu_set_imu_weights(vcgpu_handle* h, const double* w_sqrt);

int vcgpu_get_state(vcgpu_handle* h, double* intr, double* q_ck, double* p_ck, double* T_wp, double* v_w,
                    double* g, double* b, double* sf, double* ts);
int vcgpu_num_residuals(vcgpu_handle* h, int* out);
int vcgpu_frame_dim(vcgpu_handle* h, int* out);   /* 6, or 9 with inertial terms */
int vcgpu_num_globals(vcgpu_handle* h, int* out); /* sum_c (6 + K_c) (+15 with inertial terms) */

/* Batched pose initialisation — replaces the per-frame, per-camera `PosePnPRansac(camera, ellipses, target.Circles3D(),
 * ellipse_target_map, 0, 0, &t_cw)` of VicalibTask (src/vicalib-task.cc:322-325; Calibu + OpenCV solvePnP, un-vendored).
 * View v uses camera cam_id[v] (model / intrinsics from vcgpu_set_cameras) and the correspondences
 * [start[v], start[v] + count[v]) of pix (pixels) / pw (target points on the z = 0 plane, vicalib-task.cc:357-358).
 * robust_its > 0: RANSAC over 4-point homographies with inlier tolerance robust_tol (normalised image coordinates);
 * the reference calls it with 0, 0.  Out: T_cw[v] = (qx qy qz qw tx ty tz), p_c = R p_w + t; rmse[v] in normalised
 * coordinates; n_used[v] = points in the final fit (0: fewer than 4 usable points, T_cw[v] = identity).
 * The frame pose the solve is seeded with is T_wp = T_cw^-1 * T_ck (vicalib-task.cc:341-349).
 * Runs as vcgpu_pose_pnp_ransac_batch of this handle alone: the same refusals and memory, which the handle keeps. */
int vcgpu_pose_pnp_ransac(vcgpu_handle* h, int n_views, const int32_t* cam_id, const int64_t* start, const int32_t* count,
                          const double* pix, const double* pw, int robust_its, double robust_tol, double* T_cw /*n_views*7*/,
                          double* rmse_or_null, int32_t* n_used_or_null);
/* one rig's views for vcgpu_pose_pnp_ransac_batch: exactly vcgpu_pose_pnp_ransac's view arguments and outputs */
typedef struct {
  int n_views;
  const int32_t* cam_id;   /* n_views */
  const int64_t* start;    /* n_views */
  const int32_t* count;    /* n_views */
  const double* pix;       /* [..][2] */
  const double* pw;        /* [..][3] */
  double* T_cw;            /* n_views * 7 */
  double* rmse_or_null;    /* n_views, or NULL */
  int32_t* n_used_or_null; /* n_views, or NULL */
} vcgpu_pnp_views;
/* vcgpu_pose_pnp_ransac of n rigs in one call: views[i] are rig i's views, seen by handles[i]'s cameras (those of
 * vcgpu_set_cameras).  Every rig's outputs are the bits vcgpu_pose_pnp_ransac(handles[i], ...) writes for the same views,
 * whatever else is in the batch and in whatever order: a view's RANSAC draws are seeded by its index within its rig.
 * A rig with n_views = 0 is allowed and gets nothing written.  One launch covers every view of every rig, one warp per
 * view; every rig's views and correspondences are packed into one upload and all outputs come back in one download, all
 * on handle 0's stream.  The correspondences of a view are copied per view, so views may share correspondences.
 * Returns VCGPU_ERR_INVALID before anything is uploaded or launched and writes nothing, with a message naming the rig's
 * index (and for a bad view the view's index) in vcgpu_last_error of every non-null handle, for: n <= 0, a null views,
 * a null or repeated handle, handles on different devices, a handle without cameras, n_views < 0, a rig with views and
 * a null cam_id, start, count, pix, pw or T_cw, and a view vcgpu_pose_pnp_ransac refuses (cam_id outside the handle's
 * cameras, start < 0 or count < 0).
 * Memory, held by handle 0 and grown to the largest batch, never freed per call: on the device 672 bytes per rig, 92
 * per view and 57 per correspondence; in page-locked host memory the same without the scratch, 40 bytes per
 * correspondence instead of 57. */
int vcgpu_pose_pnp_ransac_batch(vcgpu_handle* const* handles, int n, const vcgpu_pnp_views* views, int robust_its,
                                double robust_tol);

/* GetSolutionCovariance (vicalibrator.h:802-857; compiled out upstream behind COMPUTE_VICALIB_COVARIANCE): the
 * [globals, globals] block of (J^T J)^-1 at the current state, tangent space, G x G row-major with G = vcgpu_num_globals:
 * per camera (w_ck 3 | p_ck 3 | intrinsics K), then with inertial terms (g 2 | b 6 | sf 6 | ts 1).  Computed on the
 * Jacobi-scaled undamped system (constant globals on a unit diagonal) by one elimination of the frames, as the solve
 * runs it, and one dense inversion of the system that elimination leaves: [globals] (vision) or [globals | top nodes]
 * (inertial), whose globals' block this is; unscaled on the host.  The matrix is exactly symmetric (one triangle is
 * computed and mirrored).  Rows / columns of constant or unused parameter blocks (the blocks of a camera no active
 * observation sees) are exactly 0.0 (ceres::Covariance convention).  Options play no part.  Nothing on the handle
 * changes: state, IMU weights and what a later vcgpu_solve or batch solve computes stay as they were.  Frame shards are
 * accepted: every rank calls with its shard, and each gets the same matrix.
 * VCGPU_ERR_NUMERIC: J^T J is not positive definite at the current state; cov is not written.
 * Device memory, kept on the handle and shared with vcgpu_get_frame_covariance: vision G^2 doubles; inertial N^2,
 * N = G + 9 t, t the nodes of the chain's top level (at most 4; on frame shards, the number of ranks). */
int vcgpu_get_covariance(vcgpu_handle* h, double* cov);
/* vcgpu_get_covariance of n handles in one call; vision and inertial rigs may be mixed.  cov[i] (G_i x G_i row-major,
 * G_i = vcgpu_num_globals) gets what vcgpu_get_covariance(handles[i]) returns at the handle's current state, equal to
 * rounding: the same tangent layout, the same Jacobi-scaled undamped system, rows and columns of constant or unused blocks exactly
 * 0.0; each matrix is exactly symmetric (one triangle is computed and mirrored).  Every rig runs inside its own
 * thread-block cluster, of the size its batch solve takes (a function of the rig alone), so its matrix does not depend,
 * bit for bit, on what else is in the batch or in which order: per handle the start point's evaluation and Jacobi scale
 * on its own stream, then one launch per (kind, cluster size) group in which each cluster eliminates the frames once,
 * factors the reduced system once and solves its G unit right-hand sides, then one copy back per handle.  Options
 * (strategy, tolerances, max_iters) play no part.  Nothing on the handle changes: state, IMU weights and what a later
 * vcgpu_solve or batch solve computes stay as they were.
 * status: n codes or NULL.  VCGPU_ERR_NUMERIC: the system of one or more rigs is not positive definite; their status is
 * VCGPU_ERR_NUMERIC and their cov[i] is not written, every other rig's matrix is written with status VCGPU_OK, and the
 * message names the failing indices.
 * Returns VCGPU_ERR_INVALID before anything is launched and writes nothing, with a message naming the index in
 * vcgpu_last_error of every non-null handle, for: n <= 0, a null or repeated handle, a null cov[i], handles on
 * different devices, frame shards, any vcgpu_set_profiling bit (1, 4, 8) or L2 flushing, and a rig the cluster kernels do not
 * fit (vision: the persistent vision kernel's fit, or no active observation; inertial: G >= 68 on an H100).
 * Device memory: per handle G^2 + 16 doubles (vision rigs also 9 (G^2 + G) of workspace), and a few KB of kernel
 * arguments per rig, held by handle 0. */
int vcgpu_get_covariance_batch(vcgpu_handle* const* handles, int n, double* const* cov /* n pointers */,
                               int* status /* n, or NULL */);
/* Marginal covariance of every frame's tangent (ceres::Covariance::GetCovarianceBlock(t_wp, t_wp), and (v_w, v_w) with
 * the inertial terms on): the [frame f, frame f] blocks of (J^T J)^-1 at the current state, on the system
 * vcgpu_get_covariance inverts (undamped J^T J, constant or unused globals taken out).  cov: n_frames blocks of fd x fd,
 * row-major, in upload order; fd is 6, or 9 with the inertial terms on, and a block's rows follow the frame's rows of
 * vcgpu_normal_equations' B.  Each block is exactly symmetric.  A vision frame no active observation sees gets a block
 * of exactly 0.0, and the other blocks are those of the problem without it; so do the velocity rows and columns of a
 * rotation-only run, which no residual reads.  Computed by a selected inversion of the
 * frame elimination: no dense inverse of J^T J is formed.  Nothing on the handle changes: state, IMU weights and what a
 * later vcgpu_solve computes stay as they were.
 * VCGPU_ERR_NUMERIC: J^T J is not positive definite at the current state; cov is not written.  VCGPU_ERR_INVALID: a
 * null argument, or frame shards (the call is one-GPU only).
 * Device memory, kept on the handle: vision G^2 + 36 n_frames doubles; inertial (G + 9 t)^2 + 81 n_frames + about
 * 8/7 n_frames (162 + 9 G) doubles, t <= 4 the nodes of the chain's top level. */
int vcgpu_get_frame_covariance(vcgpu_handle* h, double* cov /* n_frames * fd * fd */);
/* vcgpu_get_frame_covariance of n independent rigs in one call, one thread-block cluster per rig; vision and inertial
 * rigs may be mixed.  cov[i] receives rig i's blocks exactly as vcgpu_get_frame_covariance lays them out (n_frames_i
 * blocks of fd_i x fd_i; equal to its result to rounding, each block exactly symmetric, the same exact zeros).  Each rig
 * takes the cluster size its batch solve takes, a function of the rig alone, so its blocks are the same bits whatever
 * else is in the batch and in whatever order.  Per handle, on its own stream, the point is evaluated; then one launch
 * runs per group of like rigs; then one copy back per handle.  Nothing on the handle changes: state, IMU weights and what
 * a later vcgpu_solve or batch solve computes stay as they were.
 * status, VCGPU_ERR_NUMERIC and VCGPU_ERR_INVALID: as vcgpu_get_covariance_batch (the same refusals: n <= 0, a null or
 * repeated handle, a null cov[i], handles on different devices, frame shards, any vcgpu_set_profiling bit (1, 4, 8) or L2 flushing,
 * and a rig the cluster kernels do not fit, which includes inertial G >= 68 on an H100).
 * Device memory: per handle the workspace of vcgpu_get_frame_covariance and that of vcgpu_get_covariance_batch, and a few
 * KB of kernel arguments per rig, held by handle 0. */
int vcgpu_get_frame_covariance_batch(vcgpu_handle* const* handles, int n, double* const* cov /* n pointers */,
                                     int* status /* n, or NULL */);
/* The frame blocks of (J^T J)^-1 off its block diagonal (ceres::Covariance::GetCovarianceBlock(t_wp[f], globals) and
 * (t_wp[f], t_wp[f+1]), with v_w the same way when the inertial terms are on), on the system
 * vcgpu_get_frame_covariance inverts, by the same selected inversion of the frame elimination.
 * cov_fg: n_frames blocks of fd x G, row-major: Σ[frame f, globals].  Rows follow the frame's rows of
 *         vcgpu_normal_equations' B; columns follow vcgpu_get_covariance's tangent layout.
 * cov_fn: n_frames - 1 blocks of fd x fd: Σ[frame f, frame f+1], rows frame f, columns frame f+1.
 * Either may be NULL, but not both.  With vcgpu_get_frame_covariance's Σ_ff, the covariance of the relative motion of
 * frames f and f+1 is Σ_ff + Σ_f+1,f+1 - Σ_f,f+1 - Σ_f,f+1^T.  On vision rigs Σ_f,f+1 = X_f Σ_gg X_f+1^T (X_f =
 * B_f^-1 E_f), off the pattern of J^T J but well defined, so both kinds of rig share one layout.
 * Exactly 0.0: the columns of constant or unused globals, every row and column of a vision frame no active observation
 * sees, and the velocity rows and columns of a rotation-only run.  Options play no part.  Nothing on the handle changes:
 * state, IMU weights and what a later vcgpu_solve computes stay as they were.
 * VCGPU_ERR_NUMERIC: J^T J is not positive definite at the current state; nothing is written.  VCGPU_ERR_INVALID: a null
 * handle, both outputs null, or frame shards (the call is one-GPU only).
 * Device memory, kept on the handle: vision G^2 + n_frames (6 G + 36) doubles; inertial (G + 9 t)^2 + n_frames (9 G + 81)
 * + about 8/7 n_frames (162 + 9 G) doubles, t <= 4 the nodes of the chain's top level. */
int vcgpu_get_frame_cross_covariance(vcgpu_handle* h, double* cov_fg /* n_frames * fd * G, or NULL */,
                                     double* cov_fn /* (n_frames - 1) * fd * fd, or NULL */);
/* vcgpu_get_frame_cross_covariance of n independent rigs in one call, one thread-block cluster per rig, as
 * vcgpu_get_frame_covariance_batch runs them; vision and inertial rigs may be mixed.  cov_fg[i] and cov_fn[i] receive rig
 * i's blocks as vcgpu_get_frame_cross_covariance lays them out, equal to its result to rounding and with the same exact
 * zeros; each rig takes the cluster size its batch solve takes, so its blocks are the same bits whatever else is in the
 * batch and in whatever order.  Either array may be NULL (n NULL pointers), and either pointer of a rig may be NULL, but
 * not both of one rig.  Nothing on the handle changes.
 * status, VCGPU_ERR_NUMERIC and VCGPU_ERR_INVALID: as vcgpu_get_frame_covariance_batch, each refusal naming the index,
 * with both pointers of a rig null in place of a null cov[i].
 * Device memory: per handle the workspace of vcgpu_get_frame_cross_covariance and that of vcgpu_get_covariance_batch,
 * and a few KB of kernel arguments per rig, held by handle 0. */
int vcgpu_get_frame_cross_covariance_batch(vcgpu_handle* const* handles, int n, double* const* cov_fg /* n pointers, or NULL */,
                                           double* const* cov_fn /* n pointers, or NULL */, int* status /* n, or NULL */);

/* The pixel uncertainty the calibration leaves at projected points.  Point i: camera c = cam_id[i], pixel z = pix[i],
 * depth d = depth[i] >= 0 (NULL: every d = 0) and a frame:
 *   ray      unproject_c(z), the unit vector whose projection at the current intrinsics is z (ray_or_null).
 *            linear: closed form.  FOV: closed form in the model's own branches (w^2 <= 1e-5; the small-rad branch
 *            where its undistorted radius has r^2 < 1e-5, else r = tan(r_d w) / m, m = 2 tan(w / 2), r_d |w| < pi / 2).
 *            poly2 / poly3: r f(r) = r_d on [0, r_fold), r_fold the first zero of d(r f(r))/dr.  KB4: theta d(theta) =
 *            r_d on [0, theta_max), theta_max = min(pi, the first zero of its derivative); rays beyond 90 degrees point
 *            behind the image plane.  Both by Newton from r_d, at most 50 steps, converged where |r f(r) - r_d| <=
 *            1e-15 r_d or after a step |dr| <= 1e-14 r;
 *            every derivative it divides by must be positive and every iterate must stay inside the domain.
 *   point    d > 0: P_c = d * ray (d is the distance along the ray, not z-depth).  d == 0: the point at infinity.
 *   J        2 x (6 + K): the derivatives of the projection of that fixed point with respect to the camera's globals,
 *            in vcgpu_get_covariance's tangent (w_ck 3 | p_ck 3 | intrinsics K), vcgpu_eval_reproj's columns.
 *            VCGPU_PROJ_CAMERA: the point is fixed in the camera frame; only the intrinsics' columns are nonzero.
 *            VCGPU_PROJ_RIG: it is fixed in the rig (IMU) frame, P_k = R_ck^T (P_c - p_ck); at d == 0 the p_ck columns
 *            are exactly 0.0, the limit as d goes to infinity.
 *   cov      Sigma_z = J Sigma_c J^T as (S_uu, S_uv, S_vv), Sigma_c camera c's (6+K)^2 diagonal block of the globals'
 *            covariance; products in a fixed order, one triangle, so Sigma_z is exactly symmetric.  Like Sigma_c it
 *            assumes unit observation variance: scale it by the residual variance (e.g. 2 cost / (n - G)).  Constant
 *            or unused blocks are exactly 0.0 in Sigma_c and give exact zeros here (fix_intrinsics in CAMERA frame, a
 *            camera no observation sees).
 * A pixel outside its model's domain, or where Newton does not converge, gets NaN in every output. */
enum { VCGPU_PROJ_CAMERA = 0, VCGPU_PROJ_RIG = 1 };
typedef struct {
  int64_t n;               /* points */
  const int32_t* cam_id;   /* n */
  const double* pix;       /* n * 2 */
  const double* depth;     /* n, or NULL: every point at infinity */
  int frame;               /* VCGPU_PROJ_* */
  double* cov;             /* n * 3: S_uu, S_uv, S_vv */
  double* ray_or_null;     /* n * 3 unit rays, or NULL */
} vcgpu_proj_points;
/* globals_cov_or_null: NULL computes the matrix as vcgpu_get_covariance does, keeping that call's device memory; or a
 * G x G matrix in its layout (e.g. from vcgpu_get_covariance_batch), uploaded in place of the elimination.  A given
 * matrix gives the same bits on either path.  Evaluated at the handle's current accepted state; one kernel launch, one
 * thread per point.  Nothing on the handle changes: state, IMU weights, the weight update's stored eigenvectors and what
 * a later vcgpu_solve or batch computes stay as they were.
 * VCGPU_ERR_NUMERIC: as vcgpu_get_covariance (nothing is written).  VCGPU_ERR_INVALID, before anything is launched and
 * naming the point: a null pts or cov, n < 0, null cam_id or pix with n > 0, a cam_id outside the handle's cameras, a
 * negative or non-finite depth, an unknown frame, frame shards (one GPU only).
 * Device memory, held by the handle and grown to the largest call, never freed per call: G^2 doubles, and per point 28
 * bytes of inputs (20 without depths) and 24 bytes of outputs (48 with rays); plus vcgpu_get_covariance's when it computes
 * the matrix. */
int vcgpu_get_projection_covariance(vcgpu_handle* h, const double* globals_cov_or_null /* G x G */,
                                    const vcgpu_proj_points* pts);
/* vcgpu_get_projection_covariance of n rigs in one call: pts[i] are rig i's points.  The matrices are
 * vcgpu_get_covariance_batch's (its cluster kernels), then one point launch covers every rig: tiles of 256 consecutive
 * points of one rig, so a rig's outputs do not depend, bit for bit, on the rest of the batch or its order, and equal its
 * single call to rounding (as the covariance calls do).  A rig with n = 0 gets nothing written.
 * status, VCGPU_ERR_NUMERIC: as vcgpu_get_covariance_batch; a failing rig's outputs are not written, every other rig's are.
 * VCGPU_ERR_INVALID before anything is launched and writes nothing, with a message naming the index in vcgpu_last_error
 * of every non-null handle: n <= 0, a null pts, a rig vcgpu_get_projection_covariance refuses (naming the point), and
 * everything vcgpu_get_covariance_batch refuses.
 * Device memory: vcgpu_get_covariance_batch's, and held by handle 0 per rig G^2 doubles and 152 bytes of kernel
 * arguments, and per point what vcgpu_get_projection_covariance takes. */
int vcgpu_get_projection_covariance_batch(vcgpu_handle* const* handles, int n, const vcgpu_proj_points* pts,
                                          int* status /* n, or NULL */);

/* The information candidate views of the target would add to the globals, to choose the next view to capture.  A
 * candidate is a rig pose T_wp (vcgpu_set_frames' storage, q | t) from which the target's points p_w (world frame, as
 * vcgpu_set_observations' p_w) may be seen.  At the handle's current accepted state, corner j is seen by camera c of
 * candidate i when
 *   domain   KB4: theta < theta_max; every other model: z > 0 in the camera frame; poly2 / poly3: the undistorted
 *            radius is below r_fold; FOV: r_d |w| < pi / 2 past its small-rad branch.  These are the limits
 *            vcgpu_get_projection_covariance documents, from the same device routines;
 *   image    its projection lies in [0, width[c]) x [0, height[c]);
 *   facing   with facing != NULL (the target's front normal n, world frame): (c_w - p_w) . n > 0, c_w the camera centre.
 * A seen corner is an observation at its own projection (residual 0, SoftLOne weight 1) weighted by the flags'
 * visual_mult, as the solve weights a frame.  The view couples only its own pose and the globals; eliminating the pose
 * leaves S = C_v - E_v^T B_v^-1 E_v (G x G), and the posterior of the globals is Sigma' = (Sigma^-1 + S)^-1.  F: the rows
 * of Sigma whose diagonal is not exactly 0.0 (constant globals, a camera no active observation sees).  Corners of a
 * camera no active observation sees count in n_seen but add nothing; constant globals are masked as the solve masks
 * them.  Per candidate i:
 *   n_seen[i][c]  the corners camera c sees;
 *   gain[i]       1/2 log det(Sigma_F Sigma'_F^-1) = 1/2 log det(I + Sigma_F S_F), the entropy in nats the view removes
 *                 from the globals, >= 0 (rounding below 0 is clamped to 0.0);
 *   var[i]        (G, or NULL) diag(Sigma'), exactly 0.0 outside F, bitwise the diagonal of post;
 *   post[i]       (G x G, or NULL) Sigma', one triangle computed and mirrored (exactly symmetric), 0.0 outside F.
 * Pass post as globals_cov_or_null of the next call to plan greedily (score, take the best, score it alone with post,
 * chain), and to vcgpu_get_projection_covariance to map the pixel uncertainty after that view.
 * A candidate that sees no corner of a used camera gets gain 0.0 and var / post copied from Sigma's bits.  One that sees
 * 1 to 3 such corners, or whose B_v fails the frame elimination's positive-definiteness test (a Cholesky pivot that is
 * not positive), gets NaN in gain, var and post: the view does not fix its pose.  n_seen is written either way.
 * Assumptions: a candidate is a free-pose view.  On an inertial rig it gets no IMU interval, so its gain is what its
 * images alone add, a lower bound on what an IMU-tied frame would add.  Like Sigma, the result assumes unit observation
 * variance.
 * Computation (vc_view_info.cuh): Sigma_F is Jacobi-scaled and factored once per rig; one CTA per candidate projects the
 * target, builds the view's blocks with the solve's frame build, forms I + L^T S~ L and factors and inverts it in shared
 * memory.  Nothing on the handle changes: state, IMU weights, the weight update's stored eigenvectors and what a later
 * vcgpu_solve or batch computes stay as they were. */
typedef struct {
  int64_t n_cand;            /* candidates */
  const double* T_wp;        /* n_cand * 7: q (4) | t (3), |q| within 1e-6 of 1 */
  int n_pts;                 /* target points, 1 .. 400 (a candidate's corners of 8 cameras fit the CTA's workspace) */
  const double* p_w;         /* n_pts * 3 */
  const double* facing;      /* 3, or NULL: every side is the front */
  const int32_t* width;      /* n_cams image widths, pixels */
  const int32_t* height;     /* n_cams image heights */
  int32_t* n_seen;           /* n_cand * n_cams */
  double* gain;              /* n_cand */
  double* var_or_null;       /* n_cand * G, or NULL */
  double* post_or_null;      /* n_cand * G * G, or NULL */
} vcgpu_view_candidates;
/* globals_cov_or_null: NULL computes Sigma as vcgpu_get_covariance does; or a G x G matrix in its layout (e.g. a post of
 * an earlier call), uploaded in place of the elimination.  A given matrix gives the same bits on either path.
 * VCGPU_ERR_NUMERIC: Sigma_F is not positive definite (as vcgpu_get_covariance's own); nothing is written.
 * VCGPU_ERR_INVALID, before anything is launched and naming the candidate, point or camera: a null v, n_cand < 0 or
 * above 2^31 - 1 (one CTA per candidate), with
 * candidates a null T_wp, p_w, width, height, n_seen or gain, n_pts <= 0 or above 400, a width or height <= 0, a
 * non-finite p_w, facing or pose entry, a quaternion whose norm is not within 1e-6 of 1, frame shards (one GPU only).
 * n_cand = 0 writes nothing.
 * Device memory, held by the handle and grown to the largest call, never freed per call: G^2 + G_F^2 doubles, 56 bytes
 * per candidate and 24 per point of inputs, per candidate 4 n_cams + 8 bytes of outputs (+ 8 G with var, + 8 G^2 with
 * post); plus vcgpu_get_covariance's when it computes the matrix. */
int vcgpu_get_view_information(vcgpu_handle* h, const double* globals_cov_or_null /* G x G */, const vcgpu_view_candidates* v);
/* vcgpu_get_view_information of n rigs in one call: v[i] are rig i's candidates.  The matrices are
 * vcgpu_get_covariance_batch's (its cluster kernels), then one prior launch and one candidate launch cover every rig, one
 * CTA per candidate, so a rig's outputs do not depend, bit for bit, on the rest of the batch or its order, and equal its
 * single call to rounding.  A rig with n_cand = 0 gets nothing written.
 * status, VCGPU_ERR_NUMERIC: as vcgpu_get_covariance_batch (and a rig whose Sigma_F is not positive definite); a failing
 * rig's outputs are not written, every other rig's are.
 * VCGPU_ERR_INVALID before anything is launched and writes nothing, with a message naming the index in vcgpu_last_error
 * of every non-null handle: n <= 0, a null v, a rig vcgpu_get_view_information refuses, more than 2^31 - 1 candidates
 * in all, and everything
 * vcgpu_get_covariance_batch refuses.
 * Device memory: vcgpu_get_covariance_batch's, and held by handle 0 per rig what vcgpu_get_view_information takes and
 * its kernel arguments. */
int vcgpu_get_view_information_batch(vcgpu_handle* const* handles, int n, const vcgpu_view_candidates* v,
                                     int* status /* n, or NULL */);

/* Regression diagnostics of every reprojection observation: which corners the calibration rests on, which pull it away
 * from the rest of the data, and whether a large residual is a bad detection or a corner the model cannot fit.
 * Observation i has camera c and frame f.  P = (frame f's 6 pose tangents | camera c's 6 + K globals in
 * vcgpu_get_covariance's layout, w_ck 3 | p_ck 3 | intrinsics K), p = 12 + K.  At the handle's current accepted state:
 *   J_i, r_i   the loss-free 2 x p Jacobian and residual of vcgpu_eval_reproj, restricted to P; constant globals'
 *              columns masked as the solve masks them;
 *   w_i        visual_mult * rho'(|r_i|^2), the solve's SoftLOne weight;  J~ = sqrt(w_i) J_i,  r~ = sqrt(w_i) r_i;
 *   Sigma_PP   the P x P block of the inverse vcgpu_get_covariance takes (from Sigma_ff, Sigma_fc and Sigma_cc);
 *   Sigma_F    the globals' covariance on F, the globals whose variance is not exactly 0.0.
 * Per observation, active or removed by vcgpu_remove_outliers, in caller order (as vcgpu_get_obs_active):
 *   h[i]     (H_uu, H_uv, H_vv) of the leverage H_i = J~ Sigma_PP J~^T;
 *   stud[i]  active: r~^T (I - H_i)^-1 r~, the deleted (studentized) residual; removed: r~^T (I + H_i)^-1 r~, the
 *            predictive residual of a point outside the fit;
 *   infl[i]  Dg^T Sigma_F^-1 Dg, Dg = Sigma_gP J~^T (I -+ H_i)^-1 r~ (minus: active, plus: removed): the shift of the
 *            globals that deleting (or re-admitting) the observation causes in the linearised problem at a stationary
 *            point, measured in the calibration's own uncertainty.
 * Like every covariance call these assume unit observation variance: divide stud and infl by sigma^2 (e.g. 2 cost /
 * (n - dim)) before reading either against a chi-square quantile (chi2inv(0.99, 2) = 9.2103 for stud).  h is
 * scale-free.  On a vision rig the sum of tr(H_i) over the active observations is the number of free tangents: 6 per
 * used frame plus |F|.
 * NaN in all three: an observation of a camera no active observation sees, or of a vision frame no active observation
 * sees (its prediction is not determined).  A frame of an inertial rig stays determined by its IMU intervals.  An active
 * observation whose I - H_i is not positive definite as computed ((0,0) entry or determinant not > 0): h is written,
 * stud and infl are NaN.
 * Computation (vc_obs_infl.cuh): Sigma_gg, Sigma_ff and Sigma_fg from one elimination and selected inversion, as
 * vcgpu_get_frame_covariance and vcgpu_get_frame_cross_covariance form them, kept on the device; Sigma_F factored once (as
 * vcgpu_get_view_information's prior); Q_f = Sigma_fF Sigma_F^-1 Sigma_Ff per frame; then one thread per observation
 * in tiles of at most 64 of one (frame, camera), so infl = a^T M_P a with a = J~^T u and M_P = Sigma_PP with Q_f in
 * its pose block.  Nothing on the handle changes: state, IMU weights, the weight update's stored eigenvectors and what a
 * later vcgpu_solve or batch computes stay as they were.
 * VCGPU_ERR_NUMERIC: where vcgpu_get_covariance returns it, or Sigma_F is not positive definite; nothing is written.
 * VCGPU_ERR_INVALID: a null handle or out, all three outputs null, frame shards (one GPU only).  Accepts every rig
 * vcgpu_get_frame_cross_covariance accepts, inertial G >= 68 included.
 * Device memory, held by the handle and grown to the largest call, never freed per call: vcgpu_get_frame_cross_covariance's
 * plus n_frames fd^2 doubles for Sigma_ff; G^2 + G_F^2 + 36 n_frames doubles; per observation 49 bytes of inputs (the
 * observations sorted by (camera, frame), uploaded once and kept until the problem changes) and 24 (h), 8 (stud) and 8
 * (infl) of outputs; 24 bytes per tile and a few hundred per rig of kernel arguments. */
typedef struct {
  double* h;     /* n_obs * 3, or NULL */
  double* stud;  /* n_obs, or NULL */
  double* infl;  /* n_obs, or NULL */
} vcgpu_obs_influence;
int vcgpu_get_observation_influence(vcgpu_handle* h, vcgpu_obs_influence* out);
/* vcgpu_get_observation_influence of n rigs in one call: out[i] receives rig i's values.  Sigma_gg, Sigma_ff and
 * Sigma_fg come from one elimination per rig by the frame cross-covariance batch's cluster kernels in a mode that also
 * writes the diagonal blocks (one cluster per rig, of the size its batch solve takes), and stay on the device; then one
 * launch of each influence kernel covers every rig.  A rig's values are the same bits
 * whatever else is in the batch and in whatever order, and equal its single call to rounding; vision and inertial rigs
 * may be mixed.
 * status, VCGPU_ERR_NUMERIC: as vcgpu_get_frame_cross_covariance_batch (and a rig whose Sigma_F is not positive definite);
 * a failing rig's outputs are not written, every other rig's are.
 * VCGPU_ERR_INVALID before anything is launched and writes nothing, with a message naming the index in vcgpu_last_error
 * of every non-null handle: n <= 0, a null out, a rig vcgpu_get_observation_influence refuses, and everything
 * vcgpu_get_frame_cross_covariance_batch refuses (a rig with no active observation, inertial G >= 68 on an H100).
 * Device memory: per handle what vcgpu_get_observation_influence keeps and vcgpu_get_covariance_batch's workspace; held by
 * handle 0 per rig G^2 + G_F^2 + 36 n_frames doubles, the outputs and the kernel arguments. */
int vcgpu_get_observation_influence_batch(vcgpu_handle* const* handles, int n, const vcgpu_obs_influence* out,
                                          int* status /* n, or NULL */);

/* Regression diagnostics of every IMU interval: which intervals the calibration rests on and which pull the gravity,
 * biases, scale factors or time offset towards themselves.  Interval k = 0 .. n_frames - 2 (the indexing of
 * vcgpu_get_imu_mahalanobis and vcgpu_eval_imu) touches P = (frame k: pose 6, v 3 | frame k+1: pose 6, v 3 | IMU
 * globals g 2, b 6, sf 6, ts 1), p = 33; the frame rows follow vcgpu_normal_equations' B, the IMU globals are
 * vcgpu_get_covariance's columns at the IMU offset.  At the handle's current accepted state, with its current IMU weights:
 *   r_w, J_w   the interval's residual (r^T W)^T and its 9 x 33 tangent Jacobian, loss-free, as vcgpu_eval_imu returns
 *              them (rows 0-2 and 6-8 zero in rotation-only stages); constant IMU globals' columns masked as the solve
 *              masks them;
 *   w          imu_mult * rho'(|r_w|^2), CauchyLoss(100) (rho' = 1 / (1 + s / 1e4)), the solve's weight;
 *              J~ = sqrt(w) J_w,  r~ = sqrt(w) r_w;
 *   Sigma_PP   the 33 x 33 block of the inverse vcgpu_get_covariance takes (from Sigma_kk, Sigma_k+1,k+1, Sigma_k,k+1,
 *              Sigma_kg, Sigma_k+1,g and Sigma_gg);
 *   Sigma_F    the globals' covariance on F, the globals whose variance is not exactly 0.0.
 * Per interval:
 *   h[k]     81 doubles, H_k = J~ Sigma_PP J~^T row-major in the rows of r_w; one triangle formed and mirrored, so it is
 *            exactly symmetric;
 *   stud[k]  r~^T (I - H_k)^-1 r~, the deleted (studentized) residual;
 *   infl[k]  Dg^T Sigma_F^-1 Dg, Dg = Sigma_FP J~^T (I - H_k)^-1 r~: the shift of the globals that deleting the interval
 *            causes in the linearised problem at a stationary point, measured in the calibration's own uncertainty; the
 *            observation call's metric, so intervals and corners can be ranked together.
 * vcgpu_get_imu_mahalanobis measures an interval's residual against the integration covariance, the noise model
 * UpdateImuWeights builds; stud measures it against what the fit leaves when the interval is taken out.  An interval
 * that pulls the fit towards itself keeps a small residual and a small Mahalanobis distance, but not a small stud.
 * Like every covariance call these assume unit observation variance: divide stud and infl by sigma^2 before reading stud
 * against a chi-square quantile with 9 degrees of freedom (chi2inv(0.99, 9) = 21.666), or 3 in rotation-only stages,
 * which keep the attitude rows 3-5 only.  h is scale-free.  On an inertial rig, sum tr(H_obs) over the active observations
 * plus sum tr(H_k) is the number of free tangents: 9 per frame (6 rotation-only) plus |F|.
 * Exact cases: an interval with no measurements gets NaN in all three (the solve gives it a zero residual and Jacobian,
 * and vcgpu_get_imu_mahalanobis returns NaN there).  In rotation-only runs rows and columns 0-2 and 6-8 of H_k are exactly
 * 0.0.  Where I - H_k fails a pivot test of its Cholesky factorisation (a pivot not > 0), h is written, stud and infl are
 * NaN; typically an interval that alone fixes a direction: the last interval of a last frame no active observation sees
 * has H_k = I, and the interval before it three unit leverages (it alone fixes the velocity of the frame between).  Near
 * that boundary the test follows H_k's rounding, which on inertial rigs can reach 1e-4 where H_k cancels large terms.
 * obs_or_null: vcgpu_get_observation_influence's outputs, the same bits, from the same elimination: a caller who screens
 * both kinds of residual pays for one elimination.
 * Computation (vc_imu_infl.cuh): the covariance blocks as vcgpu_get_observation_influence forms them, Sigma_f,f+1 too;
 * the intervals' weighted rows by the solve's IMU evaluation into the call's own buffers; then one CTA per interval:
 * Sigma_PP and J~ in shared memory, H, a 9 x 9 Cholesky of I - H, a = J~^T u, Dg = Sigma_FP a and a triangular solve with
 * the factor of Sigma_F.  Nothing on the handle changes: state, IMU weights, the weight update's stored eigenvectors and
 * what a later vcgpu_solve or batch computes stay as they were.
 * VCGPU_ERR_NUMERIC: where vcgpu_get_covariance returns it, or Sigma_F is not positive definite; nothing is written.
 * VCGPU_ERR_INVALID, before anything is launched and with nothing written: a null handle or imu, all three IMU outputs
 * null, inertial terms off, fewer than two frames, frame shards (one GPU only), or obs_or_null refused as
 * vcgpu_get_observation_influence refuses it.  Accepts inertial G >= 68.
 * Device memory, held by the handle and grown to the largest call, never freed per call: vcgpu_get_observation_influence's
 * (its per-observation part only with obs_or_null); per interval 2456 bytes of weighted rows, and 648 (h), 8 (stud) and
 * 8 (infl) of outputs; a few hundred bytes per rig of kernel arguments. */
typedef struct {
  double* h;     /* (n_frames - 1) * 81, or NULL */
  double* stud;  /* n_frames - 1, or NULL */
  double* infl;  /* n_frames - 1, or NULL */
} vcgpu_imu_influence;
int vcgpu_get_imu_influence(vcgpu_handle* h, vcgpu_imu_influence* imu, vcgpu_obs_influence* obs_or_null);
/* vcgpu_get_imu_influence of n rigs in one call: imu[i] (and obs_or_null[i]) receive rig i's values.  The covariance
 * blocks come from the frame cross-covariance batch's cluster kernels, as vcgpu_get_observation_influence_batch takes
 * them; then one IMU evaluation per rig and one launch of each influence kernel covers every rig.  A rig's values are
 * the same bits whatever else is in the batch and in whatever order, and equal its single call to rounding; obs
 * outputs are the bits vcgpu_get_observation_influence_batch returns.
 * status, VCGPU_ERR_NUMERIC: as vcgpu_get_observation_influence_batch; a failing rig's outputs are not written, every
 * other rig's are.
 * VCGPU_ERR_INVALID before anything is launched and writes nothing, with a message naming the index in vcgpu_last_error
 * of every non-null handle: n <= 0, a null imu, a rig vcgpu_get_imu_influence refuses (a vision rig among them), and
 * everything vcgpu_get_frame_cross_covariance_batch refuses (inertial G >= 68 on an H100).
 * Device memory: per handle vcgpu_get_covariance_batch's workspace and what vcgpu_get_imu_influence keeps; held by
 * handle 0 what vcgpu_get_imu_influence takes for every rig. */
int vcgpu_get_imu_influence_batch(vcgpu_handle* const* handles, int n, const vcgpu_imu_influence* imu,
                                  const vcgpu_obs_influence* obs_or_null /* n, or NULL */, int* status /* n, or NULL */);

/* Each IMU interval's Mahalanobis distance, as UpdateImuWeights computes it and logs it against chi2inv(0.95, 9) =
 * 16.9190 (vicalibrator.h:786-794): per interval k (n_frames - 1 of them),
 *   r = [SE3::log(T_end * T_w,k+1^-1) (upsilon 3, omega 3); v_end - v_w[k+1]]   (the reference's `residuals`)
 *   dist[k] = r^T (Jt C Jt^T)^-1 r
 * where T_end, v_end and C are the interval's integrated end pose, velocity and covariance and Jt the Jacobian of r, the
 * same RK4 covariance chain, Jt and symmetrised P = Jt C Jt^T the weight update forms.  P = V diag(lambda) V^T by the
 * weight update's cyclic Jacobi sweeps, started from the identity; dist[k] = sum_k (V[:,k] . r)^2 / lambda_k, summed in
 * k order.  r_or_null: NULL, or (n_frames - 1) * 9 doubles.  Reading it against 16.919 is an observation: the reference's
 * covariance chain is approximate, and whether the distances follow chi-square with 9 degrees of freedom is not known.
 * NaN: dist[k] and r[k] of an interval with no measurements (the reference skips it and logs nothing); dist[k] where
 * some lambda_k <= 0 (there the weight update leaves the interval's weight as it is).
 * Evaluated at the handle's current accepted state, with its IMU parameters, sigmas and time offset; after a solve that
 * ended on an accepted step, that is the state of the reference's last UpdateImuWeights log.  Runs whenever the inertial
 * terms are on, rotation-only included, though the reference runs no weight update in a rotation-only stage.  Nothing on
 * the handle changes: state, IMU weights, the weight update's stored eigenvectors and what a later vcgpu_solve or batch
 * computes stay as they were.  Runs as vcgpu_get_imu_mahalanobis_batch of this handle alone: the same refusals and memory.
 * VCGPU_ERR_INVALID: a null handle or dist, inertial terms off, fewer than two frames, or frame shards (one GPU only). */
int vcgpu_get_imu_mahalanobis(vcgpu_handle* h, double* dist /* n_frames - 1 */, double* r_or_null /* (n_frames - 1) * 9 */);
/* vcgpu_get_imu_mahalanobis of n rigs in one call: dist[i] and r[i] receive rig i's values, the bits
 * vcgpu_get_imu_mahalanobis(handles[i]) writes whatever else is in the batch and in whatever order (each interval reads
 * only its own rig).  r: NULL, or n pointers of which any may be NULL.  Per handle, on its own stream, the uploads of
 * the handle; then one launch over every interval of every rig (a team of 16 threads per interval) and one download of
 * every output, on handle 0's stream.
 * Returns VCGPU_ERR_INVALID before anything is launched and writes nothing, with a message naming the index in
 * vcgpu_last_error of every non-null handle, for: n <= 0, a null dist, a null or repeated handle, a null dist[i], handles
 * on different devices, and a handle vcgpu_get_imu_mahalanobis refuses.
 * Device memory, held by handle 0 and grown to the largest batch, never freed per call: 80 bytes per interval of
 * outputs and 104 bytes per rig of kernel arguments. */
int vcgpu_get_imu_mahalanobis_batch(vcgpu_handle* const* handles, int n, double* const* dist /* n pointers */,
                                    double* const* r /* n pointers, or NULL; an entry may be NULL */);

/* ViCalibrator::GetIntegrationPoses(k) for every interval k = 0 .. n_frames - 2 (vicalibrator.h:508-533): the poses
 * ImuResidualT::IntegrateResidual's double-precision RK4 (types.h:611-687, IntegrateImu :575-594) passes through from
 * frame k over the measurements GetRange(t_k, t_k+1, ts) returns, with the handle's biases, scale factors, gravity and
 * time offset.  Interval k has as many poses as measurements (none: 0 poses): the frame's own ImuPoseT first (its pose,
 * velocity, w_w = 0 and time t_k), then one per later measurement.  Each pose is 14 doubles:
 *   q (x y z w) | t (3) | v_w (3) | w_w (3) | time
 * Two quirks are the reference's, as it writes them:
 *   - w_w is k.segment<3>(3) of the unnormalised RK4 sum k1 + 2 k2 + 2 k3 + k4: six times the step's mean rate.
 *   - a step of dt == 0 (a sample on an interval end, frame-tied streams) repeats the previous pose unchanged, its time
 *     and w_w included.
 * Times are the measurements' own: sample time + ts in binary64, or the interval end t_k+1 where GetRange interpolates
 * (the time sums of vcgpu_set_frames).
 * start: n_frames entries; start[k] is interval k's first pose, start[n_frames-1] the total.
 * poses: NULL (sizes only) or start[n_frames-1] * 14 doubles, sized from an earlier call at the same state.
 * Evaluated at the handle's current accepted state.  Rotation-only stages are computed too; the reference returns
 * nothing there, a gate its callers apply (ViCalibrator::GetAllIntegrationPoses does).  Nothing on the handle changes:
 * state, IMU weights, the weight update's stored eigenvectors and what a later vcgpu_solve or batch computes stay as
 * they were.  Runs as vcgpu_get_integration_poses_batch of this handle alone: the same refusals and memory.
 * VCGPU_ERR_INVALID: a null handle or start, inertial terms off, fewer than two frames, or frame shards (one GPU only). */
int vcgpu_get_integration_poses(vcgpu_handle* h, int64_t* start, double* poses_or_null);
/* vcgpu_get_integration_poses of n rigs in one call: start[i] and poses[i] receive rig i's values, the bits
 * vcgpu_get_integration_poses(handles[i]) writes whatever else is in the batch and in whatever order (each interval
 * reads only its own rig).  poses: NULL, or n pointers of which any may be NULL (that rig's sizes only).  Per handle, on
 * its own stream, the uploads of the handle; then on handle 0's stream a count pass over every interval of every rig
 * (one thread per interval), a prefix sum per rig and one download of the offsets; then, if some poses[i] is given, the
 * fill pass over those rigs and one download of their poses.
 * Returns VCGPU_ERR_INVALID before anything is launched and writes nothing, with a message naming the index in
 * vcgpu_last_error of every non-null handle, for: n <= 0, a null start, a null or repeated handle, a null start[i],
 * handles on different devices, and a handle vcgpu_get_integration_poses refuses.
 * Device memory, held by handle 0 and grown to the largest batch, never freed per call: 8 bytes per frame of offsets,
 * 112 bytes per returned pose and 96 bytes per rig of kernel arguments. */
int vcgpu_get_integration_poses_batch(vcgpu_handle* const* handles, int n, int64_t* const* start,
                                      double* const* poses /* n pointers, or NULL; an entry may be NULL */);

/* Hand-eye alignment of the gyro stream with the vision poses: the rotation Q from the IMU's axes to the rig's, the time
 * offset ts and the gyro bias b_g, which every inertial solve starts from and the library cannot otherwise produce.  The
 * intended call sits between a vision-only flow and the inertial one (INTEGRATION.md).  At the handle's current accepted
 * state, over interval f = 0 .. n_frames - 2 (frames f, f+1):
 *   a_f        log(R_f^T R_f+1), R_f the rotation of T_wp[f]: the rig's turn in its current axes;
 *   b_f(s, b_g) log(dR_f), dR_f the attitude the solve's RK4 reaches from the identity over GetRange(t_f, t_f+1, s) with
 *              the handle's gyro scale factors sf[0..2] and bias b_g (the accelerometer terms do not reach it);
 *   usable     both frames are seen by an active observation, and [t_f, t_f+1] lies inside [t_first + s, t_last + s]
 *              (t_first, t_last: the first and last IMU sample) for every s tried: [ts_lo, ts_hi], or the handle's ts
 *              without find_time_offset.  n is their number; every sum below is over them.
 *   grid       n_ts candidates s_c = ts_lo + c (ts_hi - ts_lo) / (n_ts - 1), the last exactly ts_hi (one candidate: ts_lo);
 *              M(s) = sum a_f b_f^T, and cost(s) = (sum |a|^2 + sum |b|^2 - 2 lambda_max(N(M))) / n, N Horn's 4 x 4
 *              matrix: the least mean |a_f - Q b_f|^2 over rotations Q, reached at Horn's Q.
 *   start      the candidate of least cost (lowest index among equals), its Horn Q and the handle's b_g.
 *   refinement up to max_iters Gauss-Newton iterations on (dtheta, s, b_g) with residual a_f - Exp(dtheta) Q b_f(s, b_g):
 *              the s and b_g columns by one-direction duals through the interpolation and the RK4 chain (ts flows through
 *              GetRange as in the solve's ts column).  A step is taken only if it lowers the cost, else it is halved, at
 *              most 10 times; s is clamped to [ts_lo, ts_hi]; Q is renormalised after each step.  The fit stops when no
 *              halving lowers the cost.
 *   find_time_offset = 0 (the reference's flag name): no grid, s stays the handle's ts bit for bit, and only Q and b_g are
 *              fitted; ts_lo, ts_hi and n_ts are checked but play no other part, and curve is not written.
 * Outputs (vcgpu_imu_alignment): Q (IMU axes to the current rig axes, x y z w, w >= 0), ts, b_g, rms = sqrt(mean
 * |a_f - Q b_f|^2) at the result in radians, excitation = the ascending eigenvalues of (1/n) sum b_f b_f^T at the result
 * (two near zero: rotation about one axis, which leaves Q unobservable), n_intervals, iterations (steps taken), and, with
 * find_time_offset, curve_or_null[n_ts] = cost(s_c) if the pointer is not NULL.
 * apply = 0: nothing on the handle changes.  apply != 0 and VCGPU_OK: for every camera c and frame f q_ck[c] <- q_ck[c] (x)
 * Q and T_wp[f].q <- T_wp[f].q (x) Q (Hamilton products, not renormalised), ts and b_g take the result; every camera pose
 * T_wk T_ck^-1 is unchanged, and translations, p_ck, velocities, intrinsics, gravity, accelerometer bias and scale factors
 * keep their bits.  The handle is left as vcgpu_set_cameras + vcgpu_set_frames + vcgpu_set_imu_params with those values
 * leave it.
 * The inertial flag is not required: without it the IMU samples of vcgpu_set_imu are uploaded by the call.
 * VCGPU_ERR_NUMERIC, nothing applied: fewer than 3 usable intervals, or a Gauss-Newton normal matrix that fails its
 * Cholesky factorisation.  curve, excitation, n_intervals and iterations are still written, Q, ts, b_g and rms are NaN.
 * VCGPU_ERR_INVALID, before anything is launched and with nothing written: a null handle, opts or out; n_ts < 1 or above
 * 65536; ts_lo > ts_hi or a bound that is not finite; max_iters < 0; fewer than two frames; no IMU samples; frame shards
 * (one GPU only).  Runs as vcgpu_align_imu_batch of this handle alone: the same memory. */
typedef struct {
  double ts_lo, ts_hi;   /* seconds: the candidate time offsets' range, both ends included */
  int n_ts;              /* candidates, 1 .. 65536 */
  int find_time_offset;  /* 0: s stays the handle's ts */
  int max_iters;         /* Gauss-Newton iterations at most, >= 0 */
  int apply;             /* nonzero: the result goes on the handle */
} vcgpu_imu_align_opts;
typedef struct {
  double Q[4];           /* x y z w, w >= 0 */
  double ts;
  double b_g[3];
  double rms;            /* radians */
  double excitation[3];  /* ascending */
  int n_intervals, iterations;
  double* curve_or_null; /* caller's n_ts doubles, or NULL */
} vcgpu_imu_alignment;
int vcgpu_align_imu(vcgpu_handle* h, const vcgpu_imu_align_opts* opts, vcgpu_imu_alignment* out);
/* vcgpu_align_imu of n rigs in one call: opts[i] and out[i] are rig i's.  Per handle, on its own stream, prepare(), the
 * accepted state read back and (inertial terms off) the IMU samples uploaded; then on handle 0's stream one upload of
 * every rig's usable intervals and four launches over every rig: a_f (one thread per interval), the grid (one CTA per
 * rig, candidate and tile of 128 intervals; each thread integrates its interval's attitude and the CTA reduces the 11
 * sums in a fixed order into the tile's partial), the costs (one thread per candidate: the tiles in order, Horn's
 * matrix and its cyclic Jacobi eigen-solve) and the refinement (one CTA per rig: the argmin, Gauss-Newton with fixed-order
 * 7 x 7 reductions and a one-thread Cholesky, the excitation).  Every reduction order is a function of the rig alone, so a
 * rig's outputs are the bits of its own call whatever else is in the batch and in whatever order.
 * status: n codes or NULL.  VCGPU_ERR_NUMERIC: as vcgpu_align_imu for one or more rigs; their status is
 * VCGPU_ERR_NUMERIC and nothing is applied to them, every other rig is written (and applied) with status VCGPU_OK, and
 * the message names the first failing index.
 * VCGPU_ERR_INVALID before anything is launched and writes nothing, with a message naming the index in vcgpu_last_error
 * of every non-null handle: n <= 0, a null opts or out, a null or repeated handle, handles on different devices, a rig
 * vcgpu_align_imu refuses, and more than 2^31 - 1 grid CTAs in all.
 * Device memory, held by handle 0 and grown to the largest batch, never freed per call: per usable interval 48 bytes, per
 * candidate 40 bytes and 88 per tile of 128 intervals (the partials: 401 candidates of 2000 intervals take 0.6 MB), 128
 * bytes per rig of results and the kernel arguments; per handle without inertial terms its IMU samples, 56 bytes each. */
int vcgpu_align_imu_batch(vcgpu_handle* const* handles, int n, const vcgpu_imu_align_opts* opts /* n */,
                          vcgpu_imu_alignment* out /* n */, int* status /* n, or NULL */);

/* ---- inspection hooks used by the parity tests (what AutoDiffCostFunction::Evaluate and the
 * normal-equation build produce inside Ceres) ------------------------------------------------ */
/* loss-free residuals and tangent-space Jacobians per observation, caller order.
 * J: n_obs * 2 * 22, row-major 2 x (6 pose | 3 w_ck | 3 p_ck | K), zero padded to 22 columns. */
int vcgpu_eval_reproj(vcgpu_handle* h, double* r /*n*2*/, double* J_or_null);
/* per IMU interval: r 9, J 9 x 33 = (pose2 6 | pose1 6 | v2 3 | v1 3 | g 2 | b 6 | sf 6 | ts 1) */
int vcgpu_eval_imu(vcgpu_handle* h, double* r /*(n_frames-1)*9*/, double* J_or_null);
/* block normal equations at the current state: B nf*fd*fd, U nf*fd*fd (U[f] = H[f-1,f]),
 * E nf*fd*G, gf nf*fd, C G*G, gc G; any may be NULL */
int vcgpu_normal_equations(vcgpu_handle* h, double* B, double* U, double* E, double* gf, double* C,
                           double* gc, double* cost);
/* one damped solve (H*scale^2 + diag(D2)) x = -g*scale with the device arrow solver */
int vcgpu_solve_arrow(vcgpu_handle* h, const double* scale, const double* D2, double* x);

/* ---- measurement hooks (bench.py) ------------------------------------------------------------
 * profile (bit mask): 1 = bracket every kernel stage of the multi-launch engine with CUDA events on the
 *          launching stream; 4 = multi-launch engine even where the persistent kernel applies; 8 = persistent kernel
 *          records per-phase device clocks (read back through vcgpu_get_stage_times).  Any other bit: VCGPU_ERR_INVALID,
 *          and the handle is left as it was.
 * flush_l2: overwrite a 256 MiB scratch buffer before every iteration and time iterations
 *           individually, so no iteration starts with its inputs resident in the 50 MB L2 */
enum {
  VCGPU_STAGE_DIAG = 0,         /* LM diagonal */
  VCGPU_STAGE_FRAME_SOLVE = 1,  /* per-frame Cholesky + Schur contribution (or IMU chain elimination) */
  VCGPU_STAGE_GLOBAL_SOLVE = 2, /* dense reduced system */
  VCGPU_STAGE_BACKSUB = 3,      /* back-substitution + x (+) delta */
  VCGPU_STAGE_EVAL_REPROJ = 4,  /* unused: the reprojection evaluation is part of VCGPU_STAGE_BUILD */
  VCGPU_STAGE_BUILD = 5,        /* per-frame block normal equations */
  VCGPU_STAGE_REDUCE = 6,       /* global block tree reduction, level 1 */
  VCGPU_STAGE_FINALIZE = 7,     /* level 2 + cost + gradient norms */
  VCGPU_STAGE_IMU_EVAL = 8,     /* IMU residual + Jacobian */
  VCGPU_STAGE_IMU_WEIGHTS = 9,  /* UpdateImuWeights */
  VCGPU_STAGE_GRID_SYNC = 10,   /* persistent vision kernel: the two grid barriers of an iteration */
  VCGPU_STAGE_EVAL_TASKS = 11,  /* persistent inertial kernels: IMU residual/Jacobian + reprojection evaluate/build (one task queue) */
  VCGPU_STAGE_IMU_ACCUM = 12,   /* persistent inertial kernels: J^T J of the IMU factors into the frame blocks */
  VCGPU_STAGE_COUNT = 16
};
/* Measured FP64 throughput of `device` in TFLOP/s (FMA = 2 flop): independent DFMA chains and independent
 * mma.sync.m8n8k4.f64 chains on every SM.  The roofline denominators for the FP64-bound kernels. */
int vcgpu_fp64_peak(int device, double* dfma_tflops, double* dmma_tflops);
int vcgpu_set_profiling(vcgpu_handle* h, int profile, int flush_l2);
int vcgpu_get_stage_times(vcgpu_handle* h, double ms_total[VCGPU_STAGE_COUNT], int64_t launches[VCGPU_STAGE_COUNT]);
/* raw device phase clocks (ns, summed over the iterations since vcgpu_set_profiling) of the persistent inertial kernels:
 * chain_solve_kernel: elimination level l at [l], Schur reduce [10], dense solve [11], back-substitution level at [12 + k],
 * state update + step statistics [22], tail of the deferred UpdateImuWeights [23]; eval_mega_kernel: tasks [32], IMU
 * accumulate [33], reduce [34], decide [35], weights [36] (only when the update is not deferred into the solve launch) */
int vcgpu_get_phase_clocks(vcgpu_handle* h, uint64_t ns[64]);

/* ---- multi-GPU: one process per GPU of one node, frames sharded contiguously.  Two reductions per LM iteration (the
 * reduced system before the dense solve; global blocks + cost / step scalars before the decision), both INSIDE the
 * persistent kernels over NVLink peer memory: vcgpu_comm_init maps a 32 MiB totals buffer of every rank into every rank
 * (CUDA IPC; NCCL is used to pass the handles).  If the mapping is not possible the same reductions run as NCCL
 * all-reduces between kernel launches.  Every rank must issue the same sequence of calls. ---------------------------- */
#define VCGPU_UNIQUE_ID_BYTES 128
int vcgpu_comm_unique_id(uint8_t id[VCGPU_UNIQUE_ID_BYTES]);
int vcgpu_comm_init(vcgpu_handle* h, const uint8_t id[VCGPU_UNIQUE_ID_BYTES], int rank, int nranks);

#ifdef __cplusplus
}
#endif
#endif /* VCGPU_H_ */
