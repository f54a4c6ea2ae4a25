// eval_kernel — the evaluation half of an inertial trust-region iteration in ONE cooperative launch (one CTA of 256
// threads per SM), grid barriers where the multi-launch engine has launch boundaries:
//
//   T  warp tasks from one queue (longest first): IMU residuals + 9x33 Jacobians of three intervals (a team of 10
//      lanes each, vc_imu.cuh) | reprojection evaluate + Gram build of a frame (build_frame_warp, vc_fused.cuh, as
//      lm_mega_kernel's phase B): frame block, E, gradient, per-(frame, camera) packed global block
//   -- grid barrier
//   A  per frame (one warp): J^T J of the two intervals touching the frame into B, U, E, gradient, and
//      the interval's packed 15x15 IMU global block
//   -- grid barrier
//   R1 slice b of the per-group global blocks / cost / gradient-norm / step partials by CTA b (fixed order)
//   -- grid barrier
//   R2 entry e of C | gc summed over the CTAs by one warp of CTA (e mod grid)
//   -- grid barrier
//   D  CTA 0: scalars, accept / reject (decide_step: Ceres' TrustRegionMinimizer + LM radius rules)
//   -- grid barrier
//   W  UpdateImuWeights at the (new) accepted point, a team of 16 lanes per interval (vc_imu_weights.cuh) — only
//      after an accepted step
//
// Replaces, per iteration, the residual / Jacobian evaluation and normal-equation build inside ceres::Solve and the
// iteration callback's UpdateImuWeights (vicalibrator.h:690-721, 956).
#pragma once
#include <cooperative_groups.h>

#include "vc_imu.cuh"
#include "vc_imu_mega.cuh"
#include "vc_imu_weights.cuh"
#include "vc_xchg.cuh"

namespace vc {

enum { kEvProfTasks = 0, kEvProfAccum, kEvProfReduce, kEvProfDecide, kEvProfWeights, kEvProfCount };

struct EvalMegaArgs {
  DevProblem dp;       // n_cams = 0 when the visual terms are off
  Ctl* ctl;
  int which;           // 0: the accepted point, 1: the trial point
  int decide_mode;     // -1 none, 0 initial point, 1 iteration
  int do_weights;      // 1: UpdateImuWeights after the decision
  double* state[2];
  Blocks blk[2];
  const int32_t *grp_start, *grp_count, *group_of;
  const double *pw, *pc, *mask;
  double* Cg;          // [n_groups][kCgStride]
  double* cost_part;   // [n_frames]
  // IMU
  imu::ImuBuf buf;
  const double* ftime;
  double* wsqrt;
  double *imu_r, *imu_J, *imu_cost, *imuCg;
  double sigma_g, sigma_a;
  // reduction
  double* Cpart;       // [grid][G*G+G]
  double* red_part;    // [grid][8]
  const double* step_part;  // [n_step_part][4] or null
  int n_step_part;
  double* scalars;
  unsigned* counter;   // task queue
  // frame-sharded run (x.nranks > 1): global blocks, scalars and the separator frames' diagonal / gradient are summed
  // over the ranks through the in-kernel exchange before the decision
  Xchg x;
  double* sep_out;     // [2][ranks * 9] summed diag(B) | gradient of every rank's first frame
  unsigned long long* prof;  // [kEvProfCount] or null
};

constexpr int kEvThreads = 256;
constexpr int kEvWarps = kEvThreads / 32;

__host__ __device__ inline size_t eval_mega_smem_doubles(int G) {
  const size_t NS = static_cast<size_t>(G) * G + G;
  const size_t build = static_cast<size_t>(kEvWarps) * kWarpDoubles;
  const size_t wts = (kEvThreads / wts::kTeam) * (sizeof(wts::Work) / sizeof(double) + 1);
  size_t m = build > wts ? build : wts;
  if (NS > m) m = NS;
  return m + kMaxCams * (kCamStateStride + 9) + 16;
}

// reprojection blocks of frame f by one warp (build_frame_warp): the packed camera blocks are stored per (frame,
// camera) group, the frame's cost goes to cost_part[f]
__device__ inline void evm_build_frame(const EvalMegaArgs& a, const Blocks& bt, const double* x, int f, double* slab, const double* smCam,
                                       const double* smRc, const unsigned char* tri_lut, int lane) {
  constexpr int FD = 9;
  const int G = a.dp.G, nf = a.dp.n_frames;
  double cost = build_frame_warp<FD, false>(
      a.dp, x + 7 * static_cast<int64_t>(f), smCam, smRc, a.mask, a.pw, a.pc, bt.E + static_cast<int64_t>(f) * FD * G, slab, tri_lut,
      lane, 0.0,
      [&](int c) {
        const int g = a.group_of[c * nf + f];
        return g < 0 ? make_int2(0, 0) : make_int2(a.grp_start[g], a.grp_count[g]);
      },
      [&](int c) { return a.Cg + static_cast<int64_t>(a.group_of[c * nf + f]) * kCgStride; });
  __syncwarp();
  store_frame_block<FD>(slab + kSlabDoubles, slab + kSlabDoubles + 36, bt.B + static_cast<int64_t>(f) * FD * FD,
                        bt.gf + static_cast<int64_t>(f) * FD, lane, 32);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cost += __shfl_xor_sync(0xffffffffu, cost, o);
  if (lane == 0) a.cost_part[f] = cost;
}

// Phase W: the weights of intervals bid * 16 + k (+ nb * 16 ...), a team of 16 lanes each (CTA bid of the nb that
// evaluate the rig).  A function of its own, as the solve kernel's weights queue (chain_weights_queue): inlined, its
// registers join the kernel's and both spill more.
__device__ __noinline__ void eval_weights(const WeightQueueArgs w, const double* xs, double* smem, int bid, int nb) {
  constexpr int kTeams = kEvThreads / wts::kTeam;
  const int tid = threadIdx.x, warp = tid >> 5, team = tid / wts::kTeam, tl = tid & (wts::kTeam - 1);
  wts::Work* work = reinterpret_cast<wts::Work*>(smem);
  for (int base = bid * kTeams; base < w.ni; base += nb * kTeams) {
    if (base + (warp * (32 / wts::kTeam)) >= w.ni) break;  // whole warp past the end
    wts::imu_weights_team(w, xs, base + team, &work[team], tl);
  }
}

// Phase T's IMU task: intervals 3 task + 0..2 by one warp.  A function of its own, as eval_weights: inlined, the
// teams' registers join the kernel's and both spill more.
__device__ __noinline__ void eval_imu_task(const ImuEvalView a, int task, int lane, const double* x) {
  imu_eval_warp(a, task, lane, x);
}

// The evaluation of the rig `a` by the CTAs of `scope` (vc_mega.cuh): the cooperative grid (eval_mega_kernel) or one
// thread-block cluster (eval_mega_batch_kernel; never sharded: the exchange is compiled out for it).  Str: the strategy
// whose decision D takes (decide_step<Str>: a DOGLEG step's model change, mu and radius are the solve launch's, in Ctl).
template <Strategy Str, class Scope>
__device__ __forceinline__ void eval_mega(const EvalMegaArgs& a, Scope scope) {
  extern __shared__ double smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nb = scope.nb(), bid = scope.bid();
  const int G = a.dp.G, NS = G * G + G, nf = a.dp.n_frames, ni = nf - 1, n_cams = a.dp.n_cams;
  __shared__ unsigned char tri_lut[128];
  __shared__ double shr[8][8];
  __shared__ unsigned task_s[kEvWarps];
  __shared__ unsigned long long* xbufs[kMaxRanks];
  if constexpr (Scope::kSharded) xchg_stage(a.x, xbufs);  // (visible after the first barrier below)
  if (a.ctl->done) return;  // uniform over the grid: written before this launch
  const int buf = a.which ? 1 - a.ctl->cur : a.ctl->cur;
  const Blocks& bt = a.blk[buf];
  const double* x = a.state[buf];
  unsigned long long t_prev = 0;
  const bool prof = a.prof != nullptr && bid == 0 && tid == 0;
  if (prof) t_prev = global_ns();
  auto mark = [&](int slot) {
    if (prof) {
      const unsigned long long t = global_ns();
      a.prof[slot] += t - t_prev;
      t_prev = t;
    }
  };
  // tail of the dynamic shared memory: camera states and rotations of the evaluated point
  const size_t head = eval_mega_smem_doubles(G) - (kMaxCams * (kCamStateStride + 9) + 16);
  double* smCam = smem + head;
  double* smRc = smCam + kMaxCams * kCamStateStride;
  fill_tri_lut(tri_lut, tid, kEvThreads);
  if (tid < n_cams) {
    const double* xc = x + a.dp.off_cam + kCamStateStride * tid;
    double R[9];
    qmat(Q4{xc[0], xc[1], xc[2], xc[3]}, R);
    for (int q = 0; q < kCamStateStride; ++q) smCam[kCamStateStride * tid + q] = xc[q];
    for (int q = 0; q < 9; ++q) smRc[9 * tid + q] = R[q];
  }
  __syncthreads();

  // ------------------------------------------------------------ T: task queue — IMU intervals first, then frames
  {
    const ImuEvalView ia{{a.dp.off_v, a.dp.off_imu, a.dp.rotation_only}, a.buf, a.ftime, a.wsqrt, a.mask + a.dp.imu_goff, a.imu_r, a.imu_J, a.imu_cost, ni, 1, a.dp.imu_mult};
    double* slab = smem + static_cast<size_t>(warp) * kWarpDoubles;
    const unsigned n_imu = static_cast<unsigned>((ni + kImuTeams - 1) / kImuTeams);
    const unsigned n_tasks = n_imu + static_cast<unsigned>(nf);
    for (;;) {
      unsigned t = 0;
      if (lane == 0) t = atomicAdd(a.counter, 1u);
      t = __shfl_sync(0xffffffffu, t, 0);
      if (t >= n_tasks) break;
      if (t < n_imu) eval_imu_task(ia, static_cast<int>(t), lane, x);
      else evm_build_frame(a, bt, x, static_cast<int>(t - n_imu), slab, smCam, smRc, tri_lut, lane);
    }
  }
  mark(kEvProfTasks);
  scope.sync();
  // ------------------------------------------------------------ A: IMU blocks of every frame
  {
    const ImuAccView aa{a.dp, a.imu_r, a.imu_J, a.imuCg, ni};
    double (*Jl)[9][34] = reinterpret_cast<double (*)[9][34]>(smem + static_cast<size_t>(warp) * 2 * 9 * 34);
    for (int f = bid * kEvWarps + warp; f < nf; f += nb * kEvWarps) {
      __syncwarp();  // the warp's previous frame is done with the staging area
      imu_accumulate_frame<32>(aa, bt, f, lane, Jl, [] { __syncwarp(); });
    }
  }
  mark(kEvProfAccum);
  scope.sync();
  // ------------------------------------------------------------ R1: slice partials
  RedFinArgs ra;
  ra.ctl = a.ctl; ra.which = a.which; ra.decide_mode = a.decide_mode; ra.multi = 0; ra.level1_only = 1;
  const bool sharded = Scope::kSharded && a.x.nranks > 1;
  // sharded: the separator frames' (first frame, ghost) gradients are normed after they have been summed
  ra.gf_skip_below = sharded ? a.dp.fd : 0;
  ra.gf_skip_from = static_cast<int64_t>(sharded ? a.dp.n_own : nf) * a.dp.fd;
  ra.Cg = a.Cg; ra.imuCg = a.imuCg; ra.ni = ni; ra.imu_goff = a.dp.imu_goff; ra.imu_stride = kImuCgStride;
  ra.Cpart = a.Cpart; ra.red_part = a.red_part;
  ra.cost_part = a.cost_part; ra.n_cost_part = nf;
  ra.imu_cost_part = a.imu_cost; ra.n_imu_cost_part = ni;
  ra.step_part = a.step_part; ra.n_step_part = a.n_step_part; ra.n_frames_fd = nf * a.dp.fd;
  ra.out[0] = a.blk[0]; ra.out[1] = a.blk[1]; ra.scalars = a.scalars; ra.counter = nullptr;
  reduce_level1(ra, a.dp, bt, smem, shr, bid, nb);
  scope.sync();
  // ------------------------------------------------------------ R2: C | gc totals (contiguous in Blocks)
  mega_reduce_stage1(a.Cpart, NS, nb, NS, bt.C, -1, -1, bid, nb);
  mark(kEvProfReduce);
  scope.sync();
  // ------------------------------------------------------------ D: scalars + decision (CTA 0)
  // entries of a rank's slot in the exchange: C | gc (NS), scalars kScCost .. kScGmax (+ 1 pad), own first frame diag 9 | gradient 9,
  // ghost diag 9 | gradient 9
  constexpr int kSepFd = 9;
  const int eSc = NS, eSep = NS + 8;
  if (bid == 0) {
    double w[kScNotPD] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int b = tid; b < nb; b += kEvThreads) {
      for (int q = 0; q < kScGmax; ++q) w[q] += __ldcg(a.red_part + 8 * b + q);
      w[kScGmax] = fmax(w[kScGmax], __ldcg(a.red_part + 8 * b + kScGmax));
    }
    if (!sharded) {
      for (int k = tid; k < G; k += kEvThreads) {
        const double v = __ldcg(bt.gc + k);
        w[kScGnorm2] += v * v;
        w[kScGmax] = fmax(w[kScGmax], fabs(v));
      }
    }
    double t[kScNotPD];
    cta_sum_scalars(w, shr, t);
    if (tid == 0) {
      if (sharded) {  // this rank's share; the totals are formed below
        for (int q = 0; q < kScNotPD; ++q) xchg_put(a.x, xbufs, eSc + q, t[q]);
      } else {
        finish_scalars<Str>(a.ctl, a.scalars, bt.cost, t, a.step_part != nullptr, a.decide_mode);
        *a.counter = 0u;  // the task queue of the next launch
        __threadfence();
      }
    }
  }
  if (sharded) {
    // publish this rank's global blocks and separator entries; one reader per entry sums the ranks (in order)
    const int nsep = (1 + a.dp.ghost) * 2 * kSepFd;
    for (int e = bid * kEvThreads + tid; e < NS + nsep; e += nb * kEvThreads) {
      if (e < NS) {
        xchg_put(a.x, xbufs, e, __ldcg(bt.C + e));  // C | gc are contiguous
      } else {
        const int o = e - NS, t = o / (2 * kSepFd), q = o - t * 2 * kSepFd;
        const int64_t f = t == 0 ? 0 : nf - 1;
        const double v = q < kSepFd ? __ldcg(bt.B + (f * kSepFd + q) * kSepFd + q) : __ldcg(bt.gf + f * kSepFd + (q - kSepFd));
        xchg_put(a.x, xbufs, eSep + o, v);
      }
    }
    const int nslot = a.x.nranks * 2 * kSepFd;
    for (int e = bid * kEvThreads + tid; e < NS + nslot; e += nb * kEvThreads) {
      double v = 0.0;
      if (e < NS) {
        for (int r = 0; r < a.x.nranks; ++r) v += xchg_get(a.x, xbufs, r, e);
        bt.C[e] = v;
      } else {
        const int o = e - NS, k = o / (2 * kSepFd), q = o - k * 2 * kSepFd;  // slot k = rank k's first frame
        if (k > 0) v = xchg_get(a.x, xbufs, k - 1, eSep + 2 * kSepFd + q);          // rank k-1's ghost copy
        v += xchg_get(a.x, xbufs, k, eSep + q);
        a.sep_out[(q < kSepFd ? 0 : a.x.nranks * kSepFd) + k * kSepFd + (q < kSepFd ? q : q - kSepFd)] = v;
      }
    }
    scope.sync();
    if (bid == 0) {
      double* tot = &shr[0][0];  // [ranks][8] the ranks' scalars
      if (tid < a.x.nranks * kScNotPD) tot[(tid / kScNotPD) * 8 + tid % kScNotPD] = xchg_get(a.x, xbufs, tid / kScNotPD, eSc + tid % kScNotPD);
      double gm = 0.0, g2 = 0.0;
      for (int k = tid; k < G; k += kEvThreads) {
        const double v = __ldcg(bt.gc + k);
        g2 += v * v;
        gm = fmax(gm, fabs(v));
      }
      for (int k = tid; k < a.x.nranks * kSepFd; k += kEvThreads) {
        const double v = __ldcg(a.sep_out + a.x.nranks * kSepFd + k);
        g2 += v * v;
        gm = fmax(gm, fabs(v));
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        g2 += __shfl_down_sync(0xffffffffu, g2, o);
        gm = fmax(gm, __shfl_down_sync(0xffffffffu, gm, o));
      }
      __shared__ double gsh[kEvWarps][2];
      if (lane == 0) { gsh[warp][0] = g2; gsh[warp][1] = gm; }
      __syncthreads();
      if (tid == 0) {
        double t[kScNotPD] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        for (int r = 0; r < a.x.nranks; ++r) {
          for (int q = 0; q < kScGmax; ++q) t[q] += tot[r * 8 + q];
          t[kScGmax] = fmax(t[kScGmax], tot[r * 8 + kScGmax]);
        }
        for (int ww = 0; ww < kEvWarps; ++ww) {
          t[kScGnorm2] += gsh[ww][0];
          t[kScGmax] = fmax(t[kScGmax], gsh[ww][1]);
        }
        finish_scalars<Str>(a.ctl, a.scalars, bt.cost, t, a.step_part != nullptr, a.decide_mode);
        *a.counter = 0u;
        __threadfence();
      }
    }
  }
  mark(kEvProfDecide);
  if (!a.do_weights || a.dp.rotation_only) return;  // uniform
  scope.sync();
  // ------------------------------------------------------------ W: UpdateImuWeights at the accepted point
  {
    const volatile Ctl* c = a.ctl;
    if (c->done || !(c->iter == 0 || c->last_accepted)) return;  // uniform: written before the barrier
    WeightQueueArgs wa;
    wa.dp.off_v = a.dp.off_v; wa.dp.off_imu = a.dp.off_imu; wa.buf = a.buf; wa.ftime = a.ftime; wa.wsqrt = a.wsqrt;
    wa.ni = ni; wa.sigma_g = a.sigma_g; wa.sigma_a = a.sigma_a;
    eval_weights(wa, a.state[c->cur], smem, bid, nb);
  }
  mark(kEvProfWeights);
}

// One rig on the whole cooperative grid.
__global__ void __launch_bounds__(kEvThreads, 1) eval_mega_kernel(EvalMegaArgs a) { eval_mega<Strategy::kLM>(a, GridScope()); }

// A batch of rigs, one thread-block cluster each: cluster k evaluates args[k], read where they are (as
// chain_solve_batch_kernel's), and decides as strategy Str
template <Strategy Str>
__global__ void __launch_bounds__(kEvThreads, 1) eval_mega_batch_kernel(const EvalMegaArgs* __restrict__ args) {
  ClusterScope scope;
  eval_mega<Str>(args[blockIdx.x / scope.nb()], scope);
}

}  // namespace vc
