// Internal declarations shared by the .cu translation units of libvcgpu.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <new>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/vcgpu.h"

namespace vc {

struct MegaArgs;  // vc_mega.cuh
struct ChainSolveArgs;  // vc_imu_mega.cuh
struct EvalMegaArgs;  // vc_imu_eval_mega.cuh
struct CovArgs;  // vc_mega.cuh
struct ChainCovArgs;  // vc_imu_mega.cuh
constexpr int kMaxCams = 8;
constexpr int kCamStateStride = 17;  // q_ck(4) p_ck(3) intr(10)
constexpr int kImuStateSize = 15;    // g2 b6 sf6 ts1
constexpr int kMaxW = 21;            // 6 pose + (6 + K<=8) globals + residual column
constexpr int kCgStride = 120;       // per-group packed global block: sym (6+K)^2 (<=105) + gradient (<=14)
constexpr int kReduceBlocks = 64;
constexpr int kImuProfSlots = 64;   // phase clock slots of the persistent inertial kernels    // level-1 partials of the global-block reduction

constexpr int kFreeCam = 3, kFreeImu = kFreeCam * kMaxCams;  // DevProblem::free_blocks

// one tile of infl_obs_kernel (vc_obs_infl.cuh): sorted observations [start, start + count) of camera cam in frame f
struct InflTile {
  int64_t start;
  int rig, cam, frame, count;
};

struct CamInfo {
  int model, K;
  int goff;         // offset of [w_ck p_ck intr] in the global tangent vector
  int obs_start;    // first sorted observation of this camera
  int n_obs;
  int group_start;  // first (cam, frame) group
  int n_groups;
  int64_t joff;     // offset (doubles) of this camera's Jacobian columns in d_J
};

// device-resident description handed to kernels by value
struct DevProblem {
  int n_cams, n_frames, fd, G, imu_goff;
  int inertial, rotation_only;
  // frame-sharded run: with inertial terms every rank but the last carries the next rank's first frame as
  // a trailing ghost (n_frames counts it, n_own does not); vision-only shards have no ghost
  int rank, nranks, ghost, n_own;
  double visual_mult, imu_mult;
  // which global blocks are free (the global mask, one bit per block): camera c's q_ck, p_ck and intrinsics at bits
  // kFreeCam * c + 0, 1, 2; g, b, sf and ts at kFreeImu + 0 .. 3 (inertial runs only)
  unsigned free_blocks;
  CamInfo cams[kMaxCams];
  // state layout (doubles): T_wp 7*nf | v_w 3*nf | cams 17*nc | imu 15
  int64_t off_v, off_cam, off_imu, state_size;
};

struct Blocks {  // block normal equations (device pointers)
  double *B, *U, *E, *gf, *C, *gc, *cost;
};

// Trust-region state kept ON THE DEVICE so iterations can be enqueued back to back with no host
// round trip: the accept/reject decision (Ceres TrustRegionMinimizer + LevenbergMarquardtStrategy,
// SURVEY App. A.3) is taken by decide_step (vc_kernels.cuh) and every kernel selects its buffers through `cur`.
struct Ctl {
  int cur;           // which double buffer holds the accepted point
  int done;          // 0 = running, else 1 + VCGPU_TERM_*
  int iter;          // iterations executed so far
  int successful;    // accepted steps
  int fixed;         // benchmark mode: never terminate on tolerances
  int max_iters;
  int last_accepted; // summary of the most recent iteration
  int pad_;
  double radius, decrease_factor;
  double cost, x_norm, gmax, gnorm;
  double function_tol, gradient_tol, param_tol;
  double last_cost_change, last_rho, last_step_norm, last_cand_cost;
  double initial_cost;
  // dogleg strategy state (vc_dogleg.cuh)
  double dl_mu, dl_alpha, dl_g2, dl_gn2, dl_b, dl_step_norm, dl_model_change;
  int dl_ok, pad2_;
};

// damping of LevenbergMarquardtStrategy::ComputeStep: D^2 = clamp(diag(J'J), 1e-6, 1e32) / radius,
// on the Jacobi-scaled system
__host__ __device__ inline double lm_damp(double diag, double scale, double radius_inv) {
  const double d = diag * scale * scale;
  return (d < 1e-6 ? 1e-6 : (d > 1e32 ? 1e32 : d)) * radius_inv;
}

}  // namespace vc

// std::vector whose storage is page-locked, so uploads are true asynchronous DMA (no staging copy)
template <class T>
struct PinnedAlloc {
  typedef T value_type;
  PinnedAlloc() {}
  template <class U> PinnedAlloc(const PinnedAlloc<U>&) {}
  T* allocate(size_t n) {
    void* p = nullptr;
    if (cudaMallocHost(&p, n * sizeof(T)) != cudaSuccess) throw std::bad_alloc();
    return static_cast<T*>(p);
  }
  void deallocate(T* p, size_t) { cudaFreeHost(p); }
  template <class U> bool operator==(const PinnedAlloc<U>&) const { return true; }
  template <class U> bool operator!=(const PinnedAlloc<U>&) const { return false; }
};

struct vcgpu_handle {
  std::string err;
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  // UpdateImuWeights of iteration k runs on a side stream next to the arrow solve of iteration k+1 (which only
  // reads blocks built earlier); the IMU evaluation of k+1 joins it
  cudaStream_t stream2 = nullptr;
  cudaEvent_t ev_dec = nullptr, ev_wts = nullptr;
  bool wts_pending = false;
  long launches = 0, collectives = 0;
  std::unordered_map<void*, size_t> capacity;  // bytes held by each dev_alloc()ed pointer slot
  // measurement hooks
  bool profiling = false, flush_l2 = false;
  bool multi_launch = false;  // force the multi-launch engine (A/B against the persistent kernel)
  bool phase_clocks = false;  // persistent kernel: per-phase %globaltimer deltas into the stage times
  cudaEvent_t st_ev[VCGPU_STAGE_COUNT][2] = {};
  bool st_used[VCGPU_STAGE_COUNT] = {};
  double st_ms[VCGPU_STAGE_COUNT] = {};
  int64_t st_n[VCGPU_STAGE_COUNT] = {};
  long st_l0 = 0;
  cudaEvent_t it_ev[2] = {nullptr, nullptr};
  void* d_flush = nullptr;

  // ---- host copies of the problem
  int n_cams = 0, n_frames = 0;
  int64_t n_obs_all = 0;  // as given by the caller
  std::vector<int32_t> h_model;
  std::vector<double> h_intr, h_qck, h_pck, h_T, h_v, h_time;
  std::vector<int32_t, PinnedAlloc<int32_t>> h_obs_frame, h_obs_cam;
  std::vector<double, PinnedAlloc<double>> h_pw, h_pc;          // caller order, AoS [n][3] / [n][2]
  std::vector<int32_t, PinnedAlloc<int32_t>> h_stage_frame;     // (camera, frame)-sorted staging, used only when
  std::vector<double, PinnedAlloc<double>> h_stage_pw, h_stage_pc;  // the caller's order is not already sorted
  std::vector<uint8_t> h_active;
  std::vector<double> h_imu_t, h_imu_w, h_imu_a;
  double sigma_g = 5.3088444e-5, sigma_a = 0.001883649;
  double h_g[2] = {0, 0}, h_b[6] = {0, 0, 0, 0, 0, 0}, h_sf[6] = {1, 1, 1, 1, 1, 1}, h_ts = 0;
  vcgpu_flags flags;
  vcgpu_options opts;
  double* mirror[9] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};

  // ---- derived (rebuilt by prepare())
  bool dirty = true;        // structure changed: re-sort / re-allocate
  bool state_dirty = true;  // host state changed: re-upload
  vc::DevProblem dp;
  int64_t n_obs = 0;               // active observations (sorted order)
  std::vector<int64_t> perm;       // sorted index -> caller index (empty when perm_identity)
  bool perm_identity = false;      // the caller's observations were already sorted by (camera, frame)
  int n_groups = 0;
  int cur = 0;                     // which of the double buffers holds the accepted point
  bool blocks_valid = false;

  // ---- device memory
  double* d_state[2] = {nullptr, nullptr};
  double* d_pw = nullptr;         // [n_obs][3] grid-corner positions, sorted by (camera, frame)
  double* d_pc = nullptr;         // [n_obs][2] detected pixel
  int32_t* d_obs_frame = nullptr;
  int32_t *d_grp_start = nullptr, *d_grp_count = nullptr, *d_group_of = nullptr;
  double* d_mask = nullptr;       // [G] 0/1 per global tangent column
  // [nf] 1 if a residual uses the frame: every frame of an inertial run, else the frames an active observation sees.
  // The others are constant to the solve and left out of x_norm (as Ceres drops parameter blocks no residual uses)
  std::vector<uint8_t> h_frame_used;
  uint8_t* d_frame_used = nullptr;
  double* d_r = nullptr;          // loss-free residuals: vcgpu_eval_reproj [2][n_obs] sorted, the evaluate calls [n_obs][2] caller order
  double* d_J = nullptr;          // vcgpu_eval_reproj, per camera: [2*(12+K)][n_obs_cam] column SoA, loss-free
  int64_t j_doubles = 0;
  double* d_cost_part = nullptr;  // [n_frames] per-frame partial costs of the fused build
  double* d_Cg = nullptr;         // [n_groups][kCgStride]
  double* d_Cpart = nullptr;      // [kReduceBlocks][G*G+G]
  vc::Blocks blk[2];
  double* d_blk_mem[2] = {nullptr, nullptr};
  double* d_scale = nullptr;      // Jacobi scaling [nf*fd+G]
  double* d_X = nullptr;          // [nf][fd][G+1]
  double* d_Spart = nullptr;      // [solve blocks][G*G+G]
  double* d_Ssum = nullptr;       // [G*G+G] summed Schur partials
  int n_solve_blocks = 0;
  double* d_delta = nullptr;      // [nf*fd+G] scaled step
  double* d_red = nullptr;        // step reductions [n_frames+1][4]
  double* d_red_part = nullptr;   // [kReduceBlocks][8] level-1 scalar partials
  unsigned* d_counter = nullptr;  // last-CTA tickets
  // persistent vision kernel (vc_mega.cuh)
  double *d_partS = nullptr, *d_partC = nullptr;  // [grid][G*G+G+8] / [grid][n_cams*kCgStride+8]
  unsigned long long* d_prof = nullptr;
  int dev_sms = 0, dev_smem_optin = 0;
  int mega_grid = 0, mega_warps[2] = {0, 0};  // [strategy]; 0 warps: does not fit / not supported, use the multi-launch engine
  // the batch calls (vc_batch.inl): the kernel arguments of every rig of a batch this handle was handle 0 of, laid out
  // by the call
  unsigned char* d_batch_args = nullptr;
  // vcgpu_evaluate / vcgpu_remove_outliers, or their batch calls with this handle as handle 0: the tiles' partials, the
  // per-camera costs and tickets, and every rig's outlier marks (vc_batch.inl: run_evaluate_batch)
  unsigned char* d_eval = nullptr;
  // vcgpu_evaluate(_batch) with residuals: [n_obs] each sorted observation's place in caller order, when that is not its own
  int32_t* d_rank = nullptr;
  // vcgpu_pose_pnp_ransac, or its batch call with this handle as handle 0: the packed inputs, outputs and scratch
  // (d_pnp), and the packed inputs and outputs in page-locked host memory (h_pnp) (vc_batch.inl: run_pnp_batch)
  unsigned char* d_pnp = nullptr;
  std::vector<unsigned char, PinnedAlloc<unsigned char>> h_pnp;
  // vcgpu_get_imu_mahalanobis(_batch) with this handle as handle 0: every rig's [ni][10] outputs (vc_batch.inl)
  double* d_mahal = nullptr;
  // vcgpu_get_integration_poses(_batch) with this handle as handle 0: every rig's [n_frames] offsets and its poses
  int64_t* d_pstart = nullptr;
  double* d_poses = nullptr;
  // vcgpu_get_projection_covariance(_batch) with this handle as handle 0: every rig's matrix and points, then every
  // rig's outputs (vc_batch.inl: run_proj_cov)
  unsigned char* d_proj = nullptr;
  // vcgpu_get_view_information(_batch) with this handle as handle 0: every rig's inputs, its factored prior and every
  // rig's outputs (vc_batch.inl: run_view_info)
  unsigned char* d_view = nullptr;
  // vcgpu_get_observation_influence(_batch) with this handle as handle 0: the argument tables, every rig's covariance
  // blocks and sorted observations, its factored prior and Q_f, then the flags and every rig's outputs (run_obs_infl)
  unsigned char* d_infl = nullptr;
  // vcgpu_get_observation_influence(_batch): every observation of this handle, removed ones included, sorted by (camera,
  // frame) with its caller index and active flag, and its tiles; valid until prepare() rebuilds the problem
  unsigned char* d_infl_obs = nullptr;
  std::vector<vc::InflTile> infl_tiles;
  bool infl_obs_valid = false;
  // vcgpu_align_imu(_batch) with this handle as handle 0: every rig's usable intervals, a_j, grid partials, curve,
  // candidate rotations and results (vc_batch.inl: run_align_imu_batch)
  double* d_align = nullptr;
  // vcgpu_get_covariance_batch: this handle's [G*G] matrix | [kScCount] flags | vision: [8][G*G+G] CTA partials | [G*G+G] total
  double* d_cov = nullptr;
  // persistent inertial kernels (vc_imu_mega.cuh, vc_imu_eval_mega.cuh)
  bool imu_mega_ok = false;
  int imu_mega_grid = 0;
  unsigned long long* d_prof2 = nullptr;  // [kImuProfSlots] phase clocks: chain_solve [0,32), eval [32,48)
  unsigned long long phase_ns[64] = {};   // accumulated since the last vcgpu_set_profiling (vcgpu_get_phase_clocks)
  int n_step_part = 0;            // entries of d_red written by the last state update
  double* d_dl = nullptr;         // dogleg work vectors [6][nf*fd+G] + matvec partials
  double* d_dl_part = nullptr;    // [kDlBlocks][4]
  double* d_scalars = nullptr;    // device scalars (see vcgpu.cu)
  double* h_scalars = nullptr;    // pinned mirror
  vc::Ctl* d_ctl = nullptr;       // device-resident trust-region state
  vc::Ctl* h_ctl = nullptr;       // pinned mirror
  // IMU
  double* d_imu = nullptr;        // [7][n_imu]: t w3 a3
  int n_imu = 0;
  double* d_wsqrt = nullptr;      // [2][(nf-1)][81]: the weights, then d_wvec
  double* d_wvec = nullptr;       // [(nf-1)][81] eigenvectors of each interval's last weights update (all NaN: none)
  bool wvec_cold = true;          // d_wvec is to be reset (prepare) before the next weights update
  double* d_imu_r = nullptr;      // [(nf-1)][9]
  double* d_imu_J = nullptr;      // [(nf-1)][9*33]
  void* imu = nullptr;            // ImuDevHost (vc_imu_host.inl)
  // multi-GPU (one process per GPU; frames sharded; see vc_engine.inl)
  void* comm = nullptr;           // ncclComm_t
  // totals buffer of the persistent kernel (vc_mega.cuh): one 4 MiB buffer per rank; in a sharded run it is mapped
  // into every rank of the node through CUDA IPC and written with NVLink peer stores from inside the kernel
  double* xchg_local = nullptr;
  double* xchg_peer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  bool xchg_ready = false;
  int rank = 0, nranks = 1;
  double* d_mg = nullptr;         // all-reduce buffer [G*G+G+6+nranks (+ 18*nranks)]
  double* d_sep = nullptr;        // [2][nranks*9]: summed diag(B) and g of the separator frames (sharded inertial runs)
  unsigned long long* d_csync = nullptr;  // persistent inertial solve: two sets of kCsSyncWords counters (ChainSolveArgs::sync)
  unsigned cs_launches = 0;
  bool smem_optin_done = false;   // dynamic shared-memory opt-ins of the multi-launch engine's kernels (per device)
  size_t elim_smem_max = 0, dense_smem_max = 0;  // ... what chain_eliminate_kernel / dense_solve_kernel may then ask for
  size_t selinv_smem_max = 0;     // ... and chain_selinv_kernel
  // vcgpu_get_frame_covariance: the inverse of the dense phase [N*N] | the frame blocks [nf*fd*fd] | inertial: every
  // chain level's SigmaLevel blocks
  double* d_fcov = nullptr;
  double* d_dsys = nullptr;       // persistent sharded inertial solve: the summed dense system in block form
  unsigned xchg_tag_dense = 0, xchg_tag_eval = 0;  // exchange numbers of the persistent inertial kernels (vc_xchg.cuh)
  double* d_dense = nullptr;      // [N*N+N] all-reduced dense system, N = G + 9*nranks
};
