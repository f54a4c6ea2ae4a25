// eval_kernel — the evaluation half of an inertial trust-region iteration in ONE cooperative launch (one CTA of 256
// threads per SM), grid barriers where the multi-launch engine has launch boundaries:
//
//   T  warp tasks from one queue (longest first): IMU residual + 9x33 Jacobian of an interval (lane per tangent
//      direction, vc_imu.cuh) | reprojection evaluate + Gram build of a frame (32 corners per slab through the
//      warp's shared-memory slab and FP64 DMMA, vc_mega.cuh's phase B): frame block, E, gradient, per-(frame,
//      camera) packed global block
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

template <int MODEL>
__device__ __forceinline__ double evm_eval(const double* T, const double* cam, const double* Rc, const double* mask, V3 pw, double pcu,
                                           double pcv, double mult, double* slab, int lane) {
  return eval_obs_to_tile<MODEL, kSlabLd>(T, cam, Rc, mask, pw, pcu, pcv, mult, slab, lane, 32 + lane);
}

// reprojection evaluate + Gram build of frame f by one warp (vc_mega.cuh phase B, with 9 x 9 frame blocks and the
// packed camera blocks written per (frame, camera) group instead of accumulated per warp)
__device__ inline void evm_build_frame(const EvalMegaArgs& a, const Blocks& bt, const double* x, int f, double* slab, const double* smCam,
                                       const double* smRc, const unsigned char* tri_lut, int lane) {
  constexpr int FD = 9;
  const int G = a.dp.G, nf = a.dp.n_frames, n_cams = a.dp.n_cams;
  double* smB = slab + kSlabDoubles;  // [36] | [6]
  double* smg = smB + 36;
  const double* frag = slab + (lane >> 2) * kSlabLd + (lane & 3);
  const double* T = x + 7 * static_cast<int64_t>(f);
  __syncwarp();
  for (int q = lane; q < 42; q += 32) smB[q] = 0.0;
  double* Ef = bt.E + static_cast<int64_t>(f) * FD * G;
  for (int q = lane; q < FD * G; q += 32) Ef[q] = 0.0;
  double cost = 0.0;
  for (int c = 0; c < n_cams; ++c) {
    const int g = a.group_of[c * nf + f];
    if (g < 0) continue;
    const CamInfo& ci = a.dp.cams[c];
    const int K = ci.K, NG = 6 + K, model = ci.model;
    const int start = a.grp_start[g], cnt = a.grp_count[g];
    const double* cam = smCam + kCamStateStride * c;
    const double* Rc = smRc + 9 * c;
    const double* mask = a.mask + ci.goff;
    double acc[3][2];
#pragma unroll
    for (int b = 0; b < 3; ++b) acc[b][0] = acc[b][1] = 0.0;
    // software pipeline: the next slab's observation is loaded while this slab goes through the DMMAs
    double nx[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
    if (lane < cnt) {
      const int64_t i = start + lane;
      nx[0] = a.pw[3 * i]; nx[1] = a.pw[3 * i + 1]; nx[2] = a.pw[3 * i + 2]; nx[3] = a.pc[2 * i]; nx[4] = a.pc[2 * i + 1];
    }
    for (int s0 = 0; s0 < cnt; s0 += 32) {
      const int m = min(32, cnt - s0);
      const int m4 = (m + 3) & ~3;
      const V3 pw{nx[0], nx[1], nx[2]};
      const double pcu = nx[3], pcv = nx[4];
      if (s0 + 32 + lane < cnt) {
        const int64_t i = start + s0 + 32 + lane;
        nx[0] = a.pw[3 * i]; nx[1] = a.pw[3 * i + 1]; nx[2] = a.pw[3 * i + 2]; nx[3] = a.pc[2 * i]; nx[4] = a.pc[2 * i + 1];
      }
      __syncwarp();  // the previous slab's fragment loads are done
      if (lane < m) {
        switch (model) {
          case kLinear: cost += evm_eval<kLinear>(T, cam, Rc, mask, pw, pcu, pcv, a.dp.visual_mult, slab, lane); break;
          case kFov: cost += evm_eval<kFov>(T, cam, Rc, mask, pw, pcu, pcv, a.dp.visual_mult, slab, lane); break;
          case kPoly2: cost += evm_eval<kPoly2>(T, cam, Rc, mask, pw, pcu, pcv, a.dp.visual_mult, slab, lane); break;
          case kPoly3: cost += evm_eval<kPoly3>(T, cam, Rc, mask, pw, pcu, pcv, a.dp.visual_mult, slab, lane); break;
          default: cost += evm_eval<kKb4>(T, cam, Rc, mask, pw, pcu, pcv, a.dp.visual_mult, slab, lane); break;
        }
      } else if (lane < m4) {  // zero the padding rows of both halves
#pragma unroll
        for (int q = 0; q < kFusedCols; ++q) {
          slab[q * kSlabLd + lane] = 0.0;
          slab[q * kSlabLd + 32 + lane] = 0.0;
        }
      }
      __syncwarp();
      // SYRK over k: steps [0, m4/4) cover residual row 0, [m4/4, m4/2) residual row 1
      const int ns = m4 >> 2;
      for (int s = 0; s < 2 * ns; ++s) {
        const int k0 = s < ns ? 4 * s : 32 + 4 * (s - ns);
        const double a0 = frag[k0], a1 = frag[8 * kSlabLd + k0];
        dmma_m8n8k4(acc[0][0], acc[0][1], a0, a0);  // (0,0)
        dmma_m8n8k4(acc[1][0], acc[1][1], a1, a0);  // (1,0)
        dmma_m8n8k4(acc[2][0], acc[2][1], a1, a1);  // (1,1)
      }
    }
    // the three accumulator blocks -> symmetric 16 x 16 Gram matrix (in the slab)
    __syncwarp();
    double* Gm = slab;
    {
      const int rr = lane >> 2, cc = 2 * (lane & 3);
      const double vm = a.dp.visual_mult;
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        const int i = (b == 0 ? 0 : 8) + rr, j = (b == 2 ? 8 : 0) + cc;
        const double v0 = acc[b][0] * vm, v1 = acc[b][1] * vm;
        if (b == 1 || j <= i) { Gm[i * 16 + j] = v0; Gm[j * 16 + i] = v0; }
        if (b == 1 || j + 1 <= i) { Gm[i * 16 + j + 1] = v1; Gm[(j + 1) * 16 + i] = v1; }
      }
    }
    __syncwarp();
    // expand: frame block, frame gradient, E (extrinsic columns through A), the camera's packed global block
    const double* Grf = Gm + (6 + K) * 16;
    const int nsym = NG * (NG + 1) / 2;
    const int n_out = 36 + 6 + 6 * NG + nsym + NG;
    double* Cc = a.Cg + static_cast<int64_t>(g) * kCgStride;
    for (int e = lane; e < n_out; e += 32) {
      int o = e;
      if (o < 36) { smB[o] += Gm[(o / 6) * 16 + (o % 6)]; continue; }
      o -= 36;
      if (o < 6) { smg[o] += Grf[o]; continue; }
      o -= 6;
      if (o < 6 * NG) {
        const int j = o / NG, p = o - j * NG;
        Ef[j * G + ci.goff + p] = p < 6 ? mask[p] * times_A(Gm + j * 16, p, Rc) : Gm[p * 16 + j];
        continue;
      }
      o -= 6 * NG;
      if (o < nsym) {
        const int p = tri_lut[o] >> 4, q = tri_lut[o] & 15;
        double v;
        if (q >= 6) {
          v = Gm[p * 16 + q];                                        // intrinsics x intrinsics
        } else if (p >= 6) {
          v = mask[q] * times_A(Gm + p * 16, q, Rc);                // intrinsics x extrinsics
        } else {                                                     // extrinsics x extrinsics: (A^T Gff A)[p][q]
          if (p < 3) {
            v = -times_A(Gm + (3 + p) * 16, q, Rc);
          } else {
            const double* r = Rc + 3 * (p - 3);
            v = -(r[0] * times_A(Gm, q, Rc) + r[1] * times_A(Gm + 16, q, Rc) + r[2] * times_A(Gm + 32, q, Rc));
          }
          v *= mask[p] * mask[q];
        }
        Cc[o] = v;
        continue;
      }
      o -= nsym;
      Cc[105 + o] = o < 6 ? mask[o] * times_A(Grf, o, Rc) : Grf[o];
    }
  }
  __syncwarp();
  double* Bf = bt.B + static_cast<int64_t>(f) * FD * FD;
  for (int q = lane; q < FD * FD; q += 32) {
    const int i = q / FD, j = q - i * FD;
    Bf[q] = (i < 6 && j < 6) ? smB[i * 6 + j] : 0.0;
  }
  if (lane < FD) bt.gf[static_cast<int64_t>(f) * FD + lane] = lane < 6 ? smg[lane] : 0.0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cost += __shfl_xor_sync(0xffffffffu, cost, o);
  if (lane == 0) a.cost_part[f] = cost;
}

// Phase W: the weights of intervals bid * 16 + k (+ grid * 16 ...), a team of 16 lanes each.  A function of its own, as
// the solve kernel's weights queue (chain_weights_queue): inlined, its registers join the kernel's and both spill more.
__device__ __noinline__ void eval_weights(const WeightQueueArgs w, const double* xs, double* smem) {
  constexpr int kTeams = kEvThreads / wts::kTeam;
  const int tid = threadIdx.x, warp = tid >> 5, team = tid / wts::kTeam, tl = tid & (wts::kTeam - 1);
  wts::Work* work = reinterpret_cast<wts::Work*>(smem);
  for (int base = blockIdx.x * kTeams; base < w.ni; base += gridDim.x * kTeams) {
    if (base + (warp * (32 / wts::kTeam)) >= w.ni) break;  // whole warp past the end
    wts::imu_weights_team(w, xs, base + team, &work[team], tl);
  }
}

__global__ void __launch_bounds__(kEvThreads, 1) eval_mega_kernel(EvalMegaArgs a) {
  extern __shared__ double smem[];
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nb = gridDim.x, bid = blockIdx.x;
  const int G = a.dp.G, NS = G * G + G, nf = a.dp.n_frames, ni = nf - 1, n_cams = a.dp.n_cams;
  __shared__ unsigned char tri_lut[128];
  __shared__ double shr[8][8];
  __shared__ unsigned task_s[kEvWarps];
  __shared__ unsigned long long* xbufs[kMaxRanks];
  xchg_stage(a.x, xbufs);  // (visible after the first barrier below)
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
  for (int e = tid; e < 105; e += kEvThreads) {
    int p = 0;
    while ((p + 1) * (p + 2) / 2 <= e) ++p;
    tri_lut[e] = static_cast<unsigned char>((p << 4) | (e - p * (p + 1) / 2));
  }
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
    const ImuEvalView ia{a.dp, a.buf, a.ftime, a.wsqrt, a.mask + a.dp.imu_goff, a.imu_r, a.imu_J, a.imu_cost, ni, 1, a.dp.imu_mult};
    double* slab = smem + static_cast<size_t>(warp) * kWarpDoubles;
    const unsigned n_tasks = static_cast<unsigned>(ni + nf);
    for (;;) {
      unsigned t = 0;
      if (lane == 0) t = atomicAdd(a.counter, 1u);
      t = __shfl_sync(0xffffffffu, t, 0);
      if (t >= n_tasks) break;
      if (t < static_cast<unsigned>(ni)) imu_eval_interval(ia, static_cast<int>(t), lane, x);
      else evm_build_frame(a, bt, x, static_cast<int>(t) - ni, slab, smCam, smRc, tri_lut, lane);
    }
  }
  mark(kEvProfTasks);
  grid.sync();
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
  grid.sync();
  // ------------------------------------------------------------ R1: slice partials
  RedFinArgs ra;
  ra.ctl = a.ctl; ra.which = a.which; ra.decide_mode = a.decide_mode; ra.multi = 0; ra.level1_only = 1;
  const bool sharded = a.x.nranks > 1;
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
  grid.sync();
  // ------------------------------------------------------------ R2: C | gc totals (contiguous in Blocks)
  mega_reduce_stage1(a.Cpart, NS, nb, NS, bt.C, -1, -1);
  mark(kEvProfReduce);
  grid.sync();
  // ------------------------------------------------------------ D: scalars + decision (CTA 0)
  // entries of a rank's slot in the exchange: C | gc (NS), 7 scalars (+ 1 pad), own first frame diag 9 | gradient 9,
  // ghost diag 9 | gradient 9
  constexpr int kSepFd = 9;
  const int eSc = NS, eSep = NS + 8;
  if (bid == 0) {
    double w[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int b = tid; b < nb; b += kEvThreads) {
      for (int q = 0; q < 6; ++q) w[q] += __ldcg(a.red_part + 8 * b + q);
      w[6] = fmax(w[6], __ldcg(a.red_part + 8 * b + 6));
    }
    if (!sharded) {
      for (int k = tid; k < G; k += kEvThreads) {
        const double v = __ldcg(bt.gc + k);
        w[1] += v * v;
        w[6] = fmax(w[6], fabs(v));
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int q = 0; q < 6; ++q) w[q] += __shfl_down_sync(0xffffffffu, w[q], o);
      w[6] = fmax(w[6], __shfl_down_sync(0xffffffffu, w[6], o));
    }
    __syncthreads();
    if (lane == 0)
      for (int q = 0; q < 7; ++q) shr[warp][q] = w[q];
    __syncthreads();
    if (tid == 0) {
      double t[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      for (int ww = 0; ww < kEvWarps; ++ww) {
        for (int q = 0; q < 6; ++q) t[q] += shr[ww][q];
        t[6] = fmax(t[6], shr[ww][6]);
      }
      if (sharded) {  // this rank's share; the totals are formed below
        for (int q = 0; q < 7; ++q) xchg_put(a.x, xbufs, eSc + q, t[q]);
      } else {
        *bt.cost = t[0];
        a.scalars[kScCost] = t[0];
        a.scalars[kScGmax] = t[6];
        a.scalars[kScGnorm2] = t[1];
        if (a.step_part) {
          a.scalars[kScDotG] = t[2];
          a.scalars[kScDotD] = t[3];
          a.scalars[kScStep2] = t[4];
          a.scalars[kScXnorm2] = t[5];
        }
        if (a.decide_mode >= 0) decide_step(a.ctl, a.scalars, a.decide_mode);
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
    grid.sync();
    if (bid == 0) {
      double* tot = &shr[0][0];  // [ranks][8] the ranks' scalars
      if (tid < a.x.nranks * 7) tot[(tid / 7) * 8 + tid % 7] = xchg_get(a.x, xbufs, tid / 7, eSc + tid % 7);
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
        double t[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        for (int r = 0; r < a.x.nranks; ++r) {
          for (int q = 0; q < 6; ++q) t[q] += tot[r * 8 + q];
          t[6] = fmax(t[6], tot[r * 8 + 6]);
        }
        for (int ww = 0; ww < kEvWarps; ++ww) {
          t[1] += gsh[ww][0];
          t[6] = fmax(t[6], gsh[ww][1]);
        }
        *bt.cost = t[0];
        a.scalars[kScCost] = t[0];
        a.scalars[kScGmax] = t[6];
        a.scalars[kScGnorm2] = t[1];
        if (a.step_part) {
          a.scalars[kScDotG] = t[2];
          a.scalars[kScDotD] = t[3];
          a.scalars[kScStep2] = t[4];
          a.scalars[kScXnorm2] = t[5];
        }
        if (a.decide_mode >= 0) decide_step(a.ctl, a.scalars, a.decide_mode);
        *a.counter = 0u;
        __threadfence();
      }
    }
  }
  mark(kEvProfDecide);
  if (!a.do_weights || a.dp.rotation_only) return;  // uniform
  grid.sync();
  // ------------------------------------------------------------ W: UpdateImuWeights at the accepted point
  {
    const volatile Ctl* c = a.ctl;
    if (c->done || !(c->iter == 0 || c->last_accepted)) return;  // uniform: written before the barrier
    WeightQueueArgs wa;
    wa.dp.off_v = a.dp.off_v; wa.dp.off_imu = a.dp.off_imu; wa.buf = a.buf; wa.ftime = a.ftime; wa.wsqrt = a.wsqrt;
    wa.ni = ni; wa.sigma_g = a.sigma_g; wa.sigma_a = a.sigma_a;
    eval_weights(wa, a.state[c->cur], smem);
  }
  mark(kEvProfWeights);
}

}  // namespace vc
