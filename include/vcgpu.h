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
