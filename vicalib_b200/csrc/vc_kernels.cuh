// CUDA kernels of the calibration solve (sm_90a, FP64).
//
// One trust-region iteration, vision terms (the fused evaluate+build kernel is in vc_fused.cuh):
//   frame_solve_kernel    per-frame (damped, Jacobi-scaled) 6x6 Cholesky, X = (B+D)^-1 [E | g],
//                         Schur contribution E^T X; one warp per frame
//   sum_partials_kernel   fixed-order sum of the per-CTA Schur partials           (vc_chain.cuh)
//   global_solve_kernel   dense Cholesky of the reduced (globals) system
//   backsub_update_kernel back-substitution + x (+) delta into the trial state
//   fused_build_kernel    residuals + Jacobians + block normal equations at the trial point
//   reduce_finalize_kernel  global blocks, cost, gradient norms and — in the CTA that arrives last —
//                         decide_step: accept / reject, trust-region radius, termination tests, on the device
// Every kernel picks its double buffer through Ctl::cur, so the host only enqueues.  The single- and
// multi-GPU vision solves run the same phases inside one persistent kernel instead (vc_mega.cuh).
// The reference does all of this inside ceres::Solve (vicalibrator.h:956).
#pragma once
#include "vc_internal.h"
#include "vc_math.cuh"

namespace vc {

__device__ __forceinline__ int pick(const Ctl* c, int which) { return which ? 1 - c->cur : c->cur; }

// scalars of a trust-region step, in one order for the per-CTA partials, the multi-GPU all-reduce buffer, the persistent
// kernels' exchange slots and d_scalars (decide_step reads them there).  The entries before kScGmax are sums, kScGmax
// and kScNotPD are maxima.
enum {
  kScCost = 0,      // robust cost of the evaluated point
  kScGnorm2 = 1,    // gradient squared 2-norm
  kScDotG = 2,      // step . g        (scaled space)
  kScDotD = 3,      // step . D2 step  (scaled space)
  kScStep2 = 4,     // |x_trial - x|^2 (ambient)
  kScXnorm2 = 5,    // |x_trial|^2 (ambient)
  kScGmax = 6,      // gradient max norm
  kScNotPD = 7,     // >0 if a Cholesky pivot failed
  kScCount = 16
};

// v plus the damping D^2 of diagonal entry r of frame f of the Jacobi-scaled system (diag: the frame's B_rr): the
// explicit D2x if one is given, else the LM rule on B_rr or, for a sharded run's first frame, on the diagonal summed over
// the two ranks that hold a piece of it (sepdiag).  The ghost (the next rank's first frame) is damped once, by its owner,
// never here (DESIGN §6).  v = 0 gives the damping itself.  (The add stays inside each case: the compiler fuses it with
// lm_damp's multiply there, which the solves' bits depend on.)
template <int FD>
__device__ __forceinline__ double frame_damp(double v, int f, int r, double diag, double scale, double rinv, const double* D2x,
                                             const double* sepdiag, int rank, bool is_ghost) {
  if (is_ghost) return v;
  if (D2x) return v + D2x[static_cast<int64_t>(f) * FD + r];
  if (sepdiag && f == 0) return v + lm_damp(sepdiag[rank * FD + r], scale, rinv);
  return v + lm_damp(diag, scale, rinv);
}
// ... and to diagonal entry k of the globals (Ckk: C_kk; nfp: frame entries before the globals in D2x)
__device__ __forceinline__ double global_damp(int k, double Ckk, double scale, double rinv, const double* D2x, int64_t nfp) {
  return D2x ? D2x[nfp + k] : lm_damp(Ckk, scale, rinv);
}

// ---------------------------------------------------------------- loss-free reprojection residual
// One observation: the target point pw seen from the frame pose T (T_wk, 7 doubles) through the camera cam (q_ck 4 |
// p_ck 3 | intrinsics), less the detected pixel z.  Also the pose chain's intermediates pk = T_wk^-1 pw and R = R(q_ck),
// and, where not null, the projection's derivatives dzp = dz/dp_c [2][3] and dzi = dz/d intrinsics [2][K].
template <int MODEL>
__device__ __forceinline__ void reproj_residual(const double* T, const double* cam, const double* pw, const double* z, double* r0,
                                                double* r1, V3* pk, double R[9], double* dzp, double* dzi) {
  const Q4 q{T[0], T[1], T[2], T[3]};
  const V3 t{T[4], T[5], T[6]};
  *pk = qrot(qconj(q), V3{pw[0], pw[1], pw[2]} - t);  // T_wk^-1 * p_w
  const Q4 qc{cam[0], cam[1], cam[2], cam[3]};
  qmat(qc, R);
  const V3 pc = mat_mul(R, *pk) + V3{cam[4], cam[5], cam[6]};
  double zp[2];
  Cam<MODEL>::project(pc, cam + 7, zp, dzp, dzi);
  *r0 = zp[0] - z[0];
  *r1 = zp[1] - z[1];
}

// ---------------------------------------------------------------- reprojection residuals and Jacobians (vcgpu_eval_reproj)
struct EvalArgs {
  const double* state[2];
  const Ctl* ctl;          // the evaluated buffer is pick(ctl, 0)
  int64_t cam_off;         // offset of this camera's 17 state doubles
  const int32_t* frame;    // per observation (camera-local arrays from here on)
  const double *pw, *pc;   // AoS [n][3], [n][2]
  const double* mask;      // 6+K column mask (w_ck, p_ck, intr)
  double *r0, *r1;
  double* J;               // column c at J + c*n
  int n;
};

template <int MODEL, bool JAC>
__global__ void __launch_bounds__(256) eval_reproj_kernel(EvalArgs a) {
  constexpr int K = Cam<MODEL>::K, NT = 12 + K;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const double* state = a.state[pick(a.ctl, 0)];
  V3 pk;
  double R[9], dzp[6], dzi[2 * K], r0, r1;
  reproj_residual<MODEL>(state + 7 * static_cast<int64_t>(a.frame[i]), state + a.cam_off, a.pw + 3 * i, a.pc + 2 * i, &r0, &r1, &pk, R,
                         JAC ? dzp : nullptr, JAC ? dzi : nullptr);
  a.r0[i] = r0;
  a.r1[i] = r1;
  if (JAC) {
    const int64_t n = a.n;
#pragma unroll
    for (int row = 0; row < 2; ++row) {
      const double* d = dzp + 3 * row;
      const double m0 = d[0] * R[0] + d[1] * R[3] + d[2] * R[6];
      const double m1 = d[0] * R[1] + d[1] * R[4] + d[2] * R[7];
      const double m2 = d[0] * R[2] + d[1] * R[5] + d[2] * R[8];
      const double w0 = m1 * pk.z - m2 * pk.y;
      const double w1 = m2 * pk.x - m0 * pk.z;
      const double w2 = m0 * pk.y - m1 * pk.x;
      double* Jc = a.J + static_cast<int64_t>(row * NT) * n + i;
      Jc[0 * n] = -m0;
      Jc[1 * n] = -m1;
      Jc[2 * n] = -m2;
      Jc[3 * n] = w0;
      Jc[4 * n] = w1;
      Jc[5 * n] = w2;
      Jc[6 * n] = -w0 * a.mask[0];
      Jc[7 * n] = -w1 * a.mask[1];
      Jc[8 * n] = -w2 * a.mask[2];
      Jc[9 * n] = d[0] * a.mask[3];
      Jc[10 * n] = d[1] * a.mask[4];
      Jc[11 * n] = d[2] * a.mask[5];
#pragma unroll
      for (int k = 0; k < K; ++k) Jc[(12 + k) * n] = dzi[row * K + k] * a.mask[6 + k];
    }
  }
}

// ---------------------------------------------------------------- accept / reject on the device
enum class Strategy { kLM, kDogleg };  // Ceres' LevenbergMarquardtStrategy, DoglegStrategy (vc_dogleg.cuh)

// mode 0: initial point (iteration 0): adopt cost / gradient norms
// mode 1: one iteration of Ceres' TrustRegionMinimizer loop.  The strategy decides what an invalid step does, the
// radius after an accepted or rejected step, where the model change comes from and the reset at the radius floor.
template <Strategy S>
__device__ inline void decide_step(Ctl* c, double* sc, int mode) {
  constexpr bool kDl = S == Strategy::kDogleg;
  if (c->done) return;
  if (mode == 0) {
    c->cost = sc[kScCost];
    c->initial_cost = sc[kScCost];
    c->gmax = sc[kScGmax];
    c->gnorm = sqrt(sc[kScGnorm2]);
    c->last_accepted = 1;
    if (!c->fixed && c->gmax <= c->gradient_tol) c->done = 1 + VCGPU_TERM_GRADIENT_TOL;
    sc[kScNotPD] = 0.0;
    return;
  }
  const int iter = ++c->iter;
  const double cand = sc[kScCost];
  // model_cost_change = -step.g - step.H.step/2; LM: with (H + D2) step = -g; dogleg: from dl_dots_kernel
  const double model_change = kDl ? c->dl_model_change : -0.5 * sc[kScDotG] + 0.5 * sc[kScDotD];
  const bool solved = kDl ? c->dl_ok != 0 : !(sc[kScNotPD] > 0.0);
  const bool invalid = !solved || !(model_change > 0.0) || !isfinite(cand);
  sc[kScNotPD] = 0.0;
  c->last_accepted = 0;
  c->last_cand_cost = cand;
  c->last_rho = 0.0;
  c->last_cost_change = 0.0;
  c->last_step_norm = 0.0;
  if (invalid) {
    if (kDl) {  // DoglegStrategy::StepIsInvalid: more regularisation for the next Gauss-Newton solve
      c->dl_mu *= 10.0;
    } else {    // StepIsInvalid == StepRejected for the LM strategy
      c->radius /= c->decrease_factor;
      c->decrease_factor *= 2.0;
    }
  } else {
    const double step_norm = sqrt(sc[kScStep2]);
    const double cost_change = c->cost - cand;
    c->last_step_norm = step_norm;
    c->last_cost_change = cost_change;
    if (!c->fixed && step_norm <= c->param_tol * (c->x_norm + c->param_tol)) {
      c->done = 1 + VCGPU_TERM_PARAM_TOL;
      return;
    }
    if (!c->fixed && fabs(cost_change) <= c->function_tol * c->cost) {
      c->done = 1 + VCGPU_TERM_FUNCTION_TOL;
      return;
    }
    const double rho = cost_change / model_change;
    c->last_rho = rho;
    if (rho > 1e-3) {
      c->cur = 1 - c->cur;  // the candidate's blocks were built speculatively: accept = flip
      c->cost = cand;
      c->gmax = sc[kScGmax];
      c->gnorm = sqrt(sc[kScGnorm2]);
      c->x_norm = sqrt(sc[kScXnorm2]);
      ++c->successful;
      if (kDl) {  // DoglegStrategy::StepAccepted
        if (rho < 0.25) c->radius *= 0.5;
        if (rho > 0.75) c->radius = fmax(c->radius, 3.0 * c->dl_step_norm);
        c->dl_mu = fmax(1e-8, 2.0 * c->dl_mu / 10.0);
      } else {
        const double t = 2.0 * rho - 1.0;
        c->radius = fmin(1e16, c->radius / fmax(1.0 / 3.0, 1.0 - t * t * t));
        c->decrease_factor = 2.0;
      }
      c->last_accepted = 1;
      if (!c->fixed) {
        if (c->gmax <= c->gradient_tol) c->done = 1 + VCGPU_TERM_GRADIENT_TOL;
        else if (c->gnorm > 0.0 && c->gnorm < 1e-9) c->done = 1 + VCGPU_TERM_CALLBACK;  // vicalibrator.h:713-717
      }
    } else if (kDl) {  // DoglegStrategy::StepRejected
      c->radius *= 0.5;
    } else {
      c->radius /= c->decrease_factor;
      c->decrease_factor *= 2.0;
    }
  }
  if (c->radius < 1e-32) {
    if (c->fixed) {
      c->radius = 1e4;
      if (!kDl) c->decrease_factor = 2.0;
    } else if (!c->done) {
      c->done = 1 + VCGPU_TERM_RADIUS;
    }
  }
  if (!c->done && iter >= c->max_iters) c->done = 1 + VCGPU_TERM_NO_CONVERGENCE;
}

// v[kScCost .. kScGmax] of every thread summed (kScGmax: maximised) over the CTA in a fixed order: a shuffle-down tree
// per warp, one slot per warp (shr), then thread 0 adds the warps up in order into t.  Every thread of the CTA calls it.
__device__ inline void cta_sum_scalars(double v[kScNotPD], double (*shr)[8], double t[kScNotPD]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int q = 0; q < kScGmax; ++q) v[q] += __shfl_down_sync(0xffffffffu, v[q], o);
    v[kScGmax] = fmax(v[kScGmax], __shfl_down_sync(0xffffffffu, v[kScGmax], o));
  }
  __syncthreads();  // shr is free
  if (lane == 0)
    for (int q = 0; q < kScNotPD; ++q) shr[warp][q] = v[q];
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int q = 0; q < kScNotPD; ++q) t[q] = 0.0;
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) {
      for (int q = 0; q < kScGmax; ++q) t[q] += shr[w][q];
      t[kScGmax] = fmax(t[kScGmax], shr[w][kScGmax]);
    }
  }
}

// the evaluated point's totals t[kScCost .. kScXnorm2, kScGmax] -> its cost (unless null) and the scalars sc (the step
// entries only when the point is a trial step), then the decision (decide_mode: -1 none, else decide_step's mode)
template <Strategy S = Strategy::kLM>
__device__ inline void finish_scalars(Ctl* ctl, double* sc, double* cost, const double* t, bool with_step, int decide_mode) {
  if (cost) *cost = t[kScCost];
  sc[kScCost] = t[kScCost];
  sc[kScGnorm2] = t[kScGnorm2];
  sc[kScGmax] = t[kScGmax];
  if (with_step)
    for (int q = kScDotG; q <= kScXnorm2; ++q) sc[q] = t[q];
  if (decide_mode >= 0) decide_step<S>(ctl, sc, decide_mode);
}

// ---------------------------------------------------------------- reduce + finalize + decide in one launch
// Level 1 (every CTA): a slice of the per-group global blocks, cost partials, gradient norms and step
// reductions.  Level 2 (the CTA that arrives last, found with a self-resetting ticket): fixed-order sum
// of the level-1 partials, C / gc / scalars, then the accept-reject decision.  One launch instead of
// three; deterministic because level 2 always sums in block order.
struct RedFinArgs {
  DevProblem dp;        // cameras to reduce (n_cams = 0 when visual terms are off)
  Ctl* ctl;
  int which;
  int decide_mode;      // -1: none (multi-GPU: decide after the all-reduce), 0: initial point, 1: iteration
  int multi;            // 1: frame-sharded run: scalars cover this rank's frames only (gc joins after the all-reduce)
  int level1_only;      // 1: stop after the per-CTA partials (large G: level 2 runs as its own parallel launches)
  int64_t gf_skip_below, gf_skip_from;  // sharded inertial run: separator frames' gradients are normed after the all-reduce
  const double* Cg;
  const double* imuCg;  // [ni][kImuCgStride] or null
  int ni, imu_goff, imu_stride;
  double* Cpart;        // [gridDim][G*G+G]
  double* red_part;     // [gridDim][8]
  const double* cost_part;
  int n_cost_part;
  const double* imu_cost_part;
  int n_imu_cost_part;
  const double* step_part;  // [n_step_part][4] or null
  int n_step_part;
  int n_frames_fd;      // n_frames * fd
  Blocks out[2];
  double* scalars;
  unsigned* counter;
};
// Level 1 of the reduction for slice `bid` of `nb` (256 threads): the slice's share of the per-group global blocks
// -> Cpart[bid], of the cost / gradient-norm / step partials -> red_part[bid].  acc: NS doubles of shared memory.
__device__ __forceinline__ void reduce_level1(const RedFinArgs& a, const DevProblem& dp, const Blocks& out, double* acc, double (*shr)[8],
                                              int bid, int nb) {
  const int G = dp.G, tid = threadIdx.x, NS = G * G + G;
  for (int k = tid; k < NS; k += 256) acc[k] = 0.0;
  __syncthreads();
  for (int c = 0; c < dp.n_cams; ++c) {
    const CamInfo& ci = dp.cams[c];
    const int NG = 6 + ci.K, nsym = NG * (NG + 1) / 2;
    const int lo = static_cast<int>(static_cast<int64_t>(ci.n_groups) * bid / nb);
    const int hi = static_cast<int>(static_cast<int64_t>(ci.n_groups) * (bid + 1) / nb);
    for (int e = tid; e < nsym + NG; e += 256) {
      int src, dst, dst2 = -1;
      if (e < nsym) {
        int i = static_cast<int>((sqrt(8.0 * e + 1.0) - 1.0) * 0.5);
        while ((i + 1) * (i + 2) / 2 <= e) ++i;
        while (i * (i + 1) / 2 > e) --i;
        const int j = e - i * (i + 1) / 2;
        src = e;
        dst = (ci.goff + i) * G + ci.goff + j;
        if (i != j) dst2 = (ci.goff + j) * G + ci.goff + i;
      } else {
        src = 105 + (e - nsym);
        dst = G * G + ci.goff + (e - nsym);
      }
      double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
      const double* p = a.Cg + static_cast<int64_t>(ci.group_start + lo) * kCgStride + src;
      int g = lo;
      for (; g + 3 < hi; g += 4, p += 4 * kCgStride) {
        s0 += p[0]; s1 += p[kCgStride]; s2 += p[2 * kCgStride]; s3 += p[3 * kCgStride];
      }
      for (; g < hi; ++g, p += kCgStride) s0 += *p;
      const double s = (s0 + s1) + (s2 + s3);
      acc[dst] += s;
      if (dst2 >= 0) acc[dst2] += s;
    }
    __syncthreads();
  }
  if (a.imuCg) {
    const int io = a.imu_goff;
    const int lo = static_cast<int>(static_cast<int64_t>(a.ni) * bid / nb);
    const int hi = static_cast<int>(static_cast<int64_t>(a.ni) * (bid + 1) / nb);
    for (int q = tid; q < 135; q += 256) {
      double s0 = 0.0, s1 = 0.0;
      const double* p = a.imuCg + static_cast<int64_t>(lo) * a.imu_stride + q;
      int k = lo;
      for (; k + 1 < hi; k += 2, p += 2 * a.imu_stride) { s0 += p[0]; s1 += p[a.imu_stride]; }
      if (k < hi) s0 += *p;
      const double s = s0 + s1;
      if (q < 120) {
        int i = static_cast<int>((sqrt(8.0 * q + 1.0) - 1.0) * 0.5);
        while ((i + 1) * (i + 2) / 2 <= q) ++i;
        while (i * (i + 1) / 2 > q) --i;
        const int j = q - i * (i + 1) / 2;
        acc[(io + i) * G + io + j] = s;
        if (i != j) acc[(io + j) * G + io + i] = s;
      } else {
        acc[G * G + io + (q - 120)] = s;
      }
    }
    __syncthreads();
  }
  double* cp = a.Cpart + static_cast<int64_t>(bid) * NS;
  for (int k = tid; k < NS; k += 256) cp[k] = acc[k];
  // slice reductions: cost, |gf|^2, step sums (4), |gf|_inf
  double v[kScNotPD] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  {
    const int lo = static_cast<int>(static_cast<int64_t>(a.n_cost_part) * bid / nb), hi = static_cast<int>(static_cast<int64_t>(a.n_cost_part) * (bid + 1) / nb);
    for (int k = lo + tid; k < hi; k += 256) v[kScCost] += a.cost_part[k];
    const int li = static_cast<int>(static_cast<int64_t>(a.n_imu_cost_part) * bid / nb), hi2 = static_cast<int>(static_cast<int64_t>(a.n_imu_cost_part) * (bid + 1) / nb);
    for (int k = li + tid; k < hi2; k += 256) v[kScCost] += a.imu_cost_part[k];
    const int64_t lg = static_cast<int64_t>(a.n_frames_fd) * bid / nb, hg = static_cast<int64_t>(a.n_frames_fd) * (bid + 1) / nb;
    for (int64_t k = lg + tid; k < hg; k += 256) {
      if (k < a.gf_skip_below || k >= a.gf_skip_from) continue;
      const double g = out.gf[k];
      v[kScGmax] = fmax(v[kScGmax], fabs(g));
      v[kScGnorm2] += g * g;
    }
    if (a.step_part) {  // step_part rows: step.g, step.D2.step, |x_new - x|^2, |x_new|^2 (kScDotG ..)
      const int ls = static_cast<int>(static_cast<int64_t>(a.n_step_part) * bid / nb), hs = static_cast<int>(static_cast<int64_t>(a.n_step_part) * (bid + 1) / nb);
      for (int k = ls + tid; k < hs; k += 256)
        for (int q = 0; q < 4; ++q) v[kScDotG + q] += a.step_part[4 * k + q];
    }
  }
  double t[kScNotPD];
  cta_sum_scalars(v, shr, t);
  if (tid == 0)
    for (int q = 0; q < kScNotPD; ++q) a.red_part[8 * bid + q] = t[q];
}

__global__ void __launch_bounds__(256) reduce_finalize_kernel(RedFinArgs a) {
  extern __shared__ double acc[];
  __shared__ double shr[8][8];
  __shared__ double sh4[4][64];
  __shared__ int is_last;
  if (a.ctl->done) return;
  const Blocks& out = a.out[pick(a.ctl, a.which)];
  const int G = a.dp.G, tid = threadIdx.x, NS = G * G + G;
  const int nb = gridDim.x, bid = blockIdx.x;
  reduce_level1(a, a.dp, out, acc, shr, bid, nb);
  if (tid == 0) {
    if (a.level1_only) { is_last = 0; }
    __threadfence();
    if (!a.level1_only) {
      const unsigned ticket = atomicInc(a.counter, static_cast<unsigned>(nb - 1));
      is_last = ticket == static_cast<unsigned>(nb - 1);
    }
  }
  __threadfence();
  __syncthreads();
  if (!is_last) return;
  // ---- level 2 (one CTA)
  __threadfence();
  double gm = 0.0, g2 = 0.0;
  const int el = tid & 63, slice = tid >> 6;
  for (int e0 = 0; e0 < NS; e0 += 64) {
    const int e = e0 + el;
    double s0 = 0.0, s1 = 0.0;
    if (e < NS) {
      int b = slice;
      for (; b + 4 < nb; b += 8) {
        s0 += __ldcg(a.Cpart + static_cast<int64_t>(b) * NS + e);
        s1 += __ldcg(a.Cpart + static_cast<int64_t>(b + 4) * NS + e);
      }
      if (b < nb) s0 += __ldcg(a.Cpart + static_cast<int64_t>(b) * NS + e);
    }
    sh4[slice][el] = s0 + s1;
    __syncthreads();
    if (slice == 0 && e < NS) {
      const double s = (sh4[0][el] + sh4[1][el]) + (sh4[2][el] + sh4[3][el]);
      if (e < G * G) {
        out.C[e] = s;
      } else {
        out.gc[e - G * G] = s;
        gm = fmax(gm, fabs(s));
        g2 += s * s;
      }
    }
    __syncthreads();
  }
  double w[kScNotPD] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (tid < nb)
    for (int q = 0; q < kScNotPD; ++q) w[q] = __ldcg(a.red_part + 8 * tid + q);
  if (!a.multi) {
    w[kScGnorm2] += g2;
    w[kScGmax] = fmax(w[kScGmax], gm);
  }
  double t[kScNotPD];
  cta_sum_scalars(w, shr, t);
  if (tid == 0) finish_scalars(a.ctl, a.scalars, out.cost, t, a.step_part != nullptr, a.decide_mode);
}

// level 2 for large global blocks: C | gc were summed by sum_partials_kernel; this one-CTA launch
// finishes the scalars (fixed order) and decides
__global__ void __launch_bounds__(256) finalize_small_kernel(RedFinArgs a, int nb) {
  __shared__ double shr[8][8];
  if (a.ctl->done) return;
  const Blocks& out = a.out[pick(a.ctl, a.which)];
  const int G = a.dp.G, tid = threadIdx.x;
  double w[kScNotPD] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (tid < nb)
    for (int q = 0; q < kScNotPD; ++q) w[q] = a.red_part[8 * tid + q];
  if (!a.multi)
    for (int k = tid; k < G; k += 256) {
      const double v = out.gc[k];
      w[kScGnorm2] += v * v;
      w[kScGmax] = fmax(w[kScGmax], fabs(v));
    }
  double t[kScNotPD];
  cta_sum_scalars(w, shr, t);
  if (tid == 0) finish_scalars(a.ctl, a.scalars, out.cost, t, a.step_part != nullptr, a.decide_mode);
}

// ---------------------------------------------------------------- multi-GPU: pack / unpack around the all-reduce
// buffer: [C G*G | gc G | scalars kScCost .. kScXnorm2 | per-rank |gf|_inf slots]
// sharded inertial runs append [diag(B) of separator frames P*9 | g of separator frames P*9]
__global__ void mg_pack_kernel(int G, const Ctl* ctl, int which, Blocks b0, Blocks b1, const double* scalars, int rank,
                               int nranks, double* buf, int sep_fd, int n_frames, int ghost) {
  if (ctl->done) return;
  const Blocks& b = pick(ctl, which) ? b1 : b0;
  const int NS = G * G + G, tid = blockIdx.x * blockDim.x + threadIdx.x;
  for (int k = tid; k < NS; k += gridDim.x * blockDim.x) buf[k] = k < G * G ? b.C[k] : b.gc[k - G * G];
  if (sep_fd > 0) {
    double* sd = buf + NS + kScGmax + nranks;
    double* sg = sd + nranks * sep_fd;
    for (int k = tid; k < nranks * sep_fd; k += gridDim.x * blockDim.x) {
      const int slot = k / sep_fd, r = k - slot * sep_fd;
      const int f = slot == rank ? 0 : (ghost && slot == rank + 1 ? n_frames - 1 : -1);
      sd[k] = f >= 0 ? b.B[(static_cast<int64_t>(f) * sep_fd + r) * sep_fd + r] : 0.0;
      sg[k] = f >= 0 ? b.gf[static_cast<int64_t>(f) * sep_fd + r] : 0.0;
    }
  }
  if (tid == 0) {
    for (int q = 0; q < kScGmax; ++q) buf[NS + q] = scalars[q];
    for (int r = 0; r < nranks; ++r) buf[NS + kScGmax + r] = r == rank ? scalars[kScGmax] : 0.0;
  }
}
__global__ void mg_unpack_decide_kernel(int G, Ctl* ctl, int which, Blocks b0, Blocks b1, double* scalars, int nranks,
                                        const double* buf, int decide_mode, int sep_fd, double* sep_out) {
  if (ctl->done) return;
  const Blocks& b = pick(ctl, which) ? b1 : b0;
  const int NS = G * G + G, tid = threadIdx.x;
  __shared__ double shm[256], shs[256];
  double gm = 0.0, g2 = 0.0;
  for (int k = tid; k < NS; k += 256) {
    const double v = buf[k];
    if (k < G * G) {
      b.C[k] = v;
    } else {
      b.gc[k - G * G] = v;
      gm = fmax(gm, fabs(v));
      g2 += v * v;
    }
  }
  if (sep_fd > 0) {  // separator frames: keep the summed diagonal / gradient, norm the gradient once
    const double* sd = buf + NS + kScGmax + nranks;
    for (int k = tid; k < 2 * nranks * sep_fd; k += 256) {
      sep_out[k] = sd[k];
      if (k >= nranks * sep_fd) {
        gm = fmax(gm, fabs(sd[k]));
        g2 += sd[k] * sd[k];
      }
    }
  }
  shm[tid] = gm;
  shs[tid] = g2;
  __syncthreads();
  if (tid == 0) {
    gm = 0.0; g2 = 0.0;
    for (int k = 0; k < 256; ++k) { gm = fmax(gm, shm[k]); g2 += shs[k]; }
    double t[kScNotPD];
    for (int q = 0; q < kScGmax; ++q) t[q] = buf[NS + q];
    for (int r = 0; r < nranks; ++r) gm = fmax(gm, buf[NS + kScGmax + r]);
    t[kScGnorm2] += g2;
    t[kScGmax] = gm;
    finish_scalars(ctl, scalars, b.cost, t, true, decide_mode);
  }
}

// ---------------------------------------------------------------- Jacobi scaling
// scale = 1/(1+sqrt(diag(J'J)))   (Ceres TrustRegionMinimizer, jacobi_scaling, computed once)
__global__ void jacobi_scale_kernel(DevProblem dp, Blocks b0, Blocks b1, const Ctl* ctl, double* out, const double* sepdiag) {
  const Blocks& b = ctl->cur ? b1 : b0;
  const int64_t n = static_cast<int64_t>(dp.n_frames) * dp.fd + dp.G;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t nfp = static_cast<int64_t>(dp.n_frames) * dp.fd;
  double d;
  if (i < nfp) {
    const int64_t f = i / dp.fd;
    const int k = static_cast<int>(i - f * dp.fd);
    d = b.B[(f * dp.fd + k) * dp.fd + k];
    if (sepdiag) {  // separator frames: the diagonal summed over the two ranks that hold a piece of it
      if (f == 0) d = sepdiag[dp.rank * dp.fd + k];
      else if (dp.ghost && f == dp.n_frames - 1) d = sepdiag[(dp.rank + 1) * dp.fd + k];
    }
  } else {
    const int k = static_cast<int>(i - nfp);
    d = b.C[k * dp.G + k];
  }
  out[i] = 1.0 / (1.0 + sqrt(d));
}

// ---------------------------------------------------------------- per-frame solve (no coupling)
struct SolveArgs {
  DevProblem dp;
  Blocks b[2];
  const Ctl* ctl;
  const double* scale;
  const double* D2x;  // explicit damping (inspection hook) or null: lm_damp(diag, scale, 1/radius)
  double* X;          // [nf][fd][G+1]  = (B + D)^-1 [E | g]   (scaled space)
  double* Spart;      // [gridDim][G*G+G]
  double* scalars;
};
constexpr int kSolveThreads = 128;
constexpr int kSolveWarps = kSolveThreads / 32;

// The CTA's E^T X of the frames its first nact warps just staged (scaled [E | g] [FD][G + 1], then X_f [FD][G + 1];
// stages `stride` doubles apart), added to Sacc: the lower triangle of [G][G], then the right-hand side [G].  Thread tid
// of nthreads owns the same entries every time (deterministic).
template <int FD>
__device__ __forceinline__ void schur_accumulate(double* Sacc, const double* stages, int stride, int nact, int G, int tid,
                                                 int nthreads) {
  const int M = G + 1, NS = G * G + G;
  for (int e = tid; e < NS; e += nthreads) {
    const int ra = e < G * G ? e / G : e - G * G;
    const int cb = e < G * G ? e - ra * G : G;
    if (e < G * G && cb > ra) continue;  // lower triangle only
    double sum = 0.0;
    for (int w = 0; w < nact; ++w) {
      const double* Ew = stages + static_cast<size_t>(w) * stride;
      const double* Xv = Ew + FD * M;
#pragma unroll
      for (int q = 0; q < FD; ++q) sum += Ew[q * M + ra] * Xv[q * M + cb];
    }
    Sacc[e] += sum;
  }
}

// Cholesky factor of a frame block held in registers: the lower triangle of L is overwritten by the factor and iL gets
// the reciprocals of its pivots.  A pivot that is not positive is taken as 1; the return value is false then.
template <int FD>
__device__ __forceinline__ bool frame_chol(double (&L)[FD][FD], double (&iL)[FD]) {
  bool ok = true;
#pragma unroll
  for (int j = 0; j < FD; ++j) {
    double d = L[j][j];
#pragma unroll
    for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k];
    if (!(d > 0.0)) { ok = false; d = 1.0; }
    d = sqrt(d);
    L[j][j] = d;
    const double inv = 1.0 / d;
    iL[j] = inv;
#pragma unroll
    for (int i = j + 1; i < FD; ++i) {
      double t = L[i][j];
#pragma unroll
      for (int k = 0; k < j; ++k) t -= L[i][k] * L[j][k];
      L[i][j] = t * inv;
    }
  }
  return ok;
}

// One warp per frame: every lane factors the (damped, scaled) FD x FD block in registers and the
// lanes split the right-hand-side columns [E | g]; the CTA then accumulates E^T X for its four
// frames (schur_accumulate).
template <int FD>
__global__ void __launch_bounds__(kSolveThreads) frame_solve_kernel(SolveArgs a) {
  extern __shared__ double sm[];
  if (a.ctl->done) return;
  const Blocks& b = a.b[a.ctl->cur];
  const double rinv = 1.0 / a.ctl->radius;
  const int G = a.dp.G, M = G + 1, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, NS = G * G + G;
  double* Sacc = sm;                                   // [G*G+G]
  double* Esw = Sacc + NS + warp * (2 * FD * M);       // per warp: Es [FD][M] (col G = scaled g)
  double* Xw = Esw + FD * M;                           // per warp: X  [FD][M]
  const double* sc = a.scale + static_cast<int64_t>(a.dp.n_frames) * FD;
  for (int k = tid; k < NS; k += kSolveThreads) Sacc[k] = 0.0;
  for (int base = blockIdx.x * kSolveWarps; base < a.dp.n_frames; base += gridDim.x * kSolveWarps) {
    const int f = base + warp;
    __syncthreads();
    if (f < a.dp.n_frames) {
      const double* sf = a.scale + static_cast<int64_t>(f) * FD;
      const double* Bf = b.B + static_cast<int64_t>(f) * FD * FD;
      const double* Ef = b.E + static_cast<int64_t>(f) * FD * G;
      double s[FD], L[FD][FD], iL[FD];
#pragma unroll
      for (int i = 0; i < FD; ++i) s[i] = sf[i];
#pragma unroll
      for (int i = 0; i < FD; ++i)
#pragma unroll
        for (int j = 0; j <= i; ++j) {
          const double bij = Bf[i * FD + j];
          double v = bij * s[i] * s[j];
          if (i == j) v += frame_damp<FD>(0.0, f, i, bij, s[i], rinv, a.D2x, nullptr, 0, a.dp.ghost && f == a.dp.n_frames - 1);
          L[i][j] = v;
        }
      const bool ok = frame_chol<FD>(L, iL);
      if (!ok && lane == 0) a.scalars[kScNotPD] = 1.0;
      double* Xf = a.X + static_cast<int64_t>(f) * FD * M;
      for (int c = lane; c < M; c += 32) {
        double x[FD];
        const double scc = c < G ? sc[c] : 1.0;
#pragma unroll
        for (int i = 0; i < FD; ++i) {
          const double r = (c < G ? Ef[i * G + c] : b.gf[static_cast<int64_t>(f) * FD + i]) * s[i] * scc;
          Esw[i * M + c] = r;
          x[i] = r;
        }
#pragma unroll
        for (int i = 0; i < FD; ++i) {
          double t = x[i];
#pragma unroll
          for (int k = 0; k < i; ++k) t -= L[i][k] * x[k];
          x[i] = t * iL[i];
        }
#pragma unroll
        for (int i = FD - 1; i >= 0; --i) {
          double t = x[i];
#pragma unroll
          for (int k = i + 1; k < FD; ++k) t -= L[k][i] * x[k];
          x[i] = t * iL[i];
        }
#pragma unroll
        for (int i = 0; i < FD; ++i) {
          Xw[i * M + c] = x[i];
          Xf[i * M + c] = x[i];
        }
      }
    }
    __syncthreads();
    schur_accumulate<FD>(Sacc, sm + NS, 2 * FD * M, min(kSolveWarps, a.dp.n_frames - base), G, tid, kSolveThreads);
  }
  __syncthreads();
  double* out = a.Spart + static_cast<int64_t>(blockIdx.x) * NS;
  for (int k = tid; k < NS; k += kSolveThreads) out[k] = Sacc[k];
}

// Entry e of the reduced (globals) system [S | rhs] = [S C S + D - sum E^T X | -S g_c + sum E^T x]: c is entry e of
// [C | g_c], p of the summed Schur partials, sc the globals' scale (global_damp's arguments after it).
__device__ __forceinline__ double reduced_system_entry(int e, int G, double c, double p, const double* sc, double rinv,
                                                       const double* D2x, int64_t nfp) {
  if (e >= G * G) return -c * sc[e - G * G] + p;
  const int r = e / G, q = e - r * G;
  double v = c * sc[r] * sc[q] - p;
  if (r == q) v += global_damp(r, c, sc[r], rinv, D2x, nfp);
  return v;
}

// ---------------------------------------------------------------- reduced dense solve
struct GlobalSolveArgs {
  DevProblem dp;
  Blocks b[2];
  const Ctl* ctl;
  const double* scale;
  const double* D2x;
  const double* Ssum;  // [G*G+G] summed Schur partials (lower triangle | right-hand side)
  double* delta;       // scaled step; globals written at delta[nf*fd ...]
  double* scalars;
};
__global__ void __launch_bounds__(256) global_solve_kernel(GlobalSolveArgs a) {
  extern __shared__ double sm[];
  if (a.ctl->done) return;
  const Blocks& b = a.b[a.ctl->cur];
  const double rinv = 1.0 / a.ctl->radius;
  const int G = a.dp.G, tid = threadIdx.x, NS = G * G + G;
  double* S = sm;           // [G*G]
  double* rhs = sm + G * G; // [G]
  __shared__ int bad;
  if (tid == 0) bad = 0;
  const int64_t nfp = static_cast<int64_t>(a.dp.n_frames) * a.dp.fd;
  const double* sc = a.scale + nfp;
  for (int e = tid; e < NS; e += 256)  // (the strict upper triangle of S is never read)
    S[e] = reduced_system_entry(e, G, e < G * G ? b.C[e] : b.gc[e - G * G], a.Ssum[e], sc, rinv, a.D2x, nfp);
  __syncthreads();
  for (int j = 0; j < G; ++j) {
    if (tid == 0) {
      double d = S[j * G + j];
      if (!(d > 0.0)) { bad = 1; d = 1.0; }
      S[j * G + j] = sqrt(d);
    }
    __syncthreads();
    const double dj = S[j * G + j];
    for (int i = j + 1 + tid; i < G; i += 256) S[i * G + j] /= dj;
    __syncthreads();
    const int rem = G - j - 1;
    for (int e = tid; e < rem * rem; e += 256) {
      const int i = j + 1 + e / rem, k = j + 1 + e % rem;
      if (k <= i) S[i * G + k] -= S[i * G + j] * S[k * G + j];
    }
    __syncthreads();
  }
  if (tid < 32) {  // warp-cooperative triangular solves (column oriented), L L^T x = rhs
    const int lane = tid;
    for (int i = 0; i < G; ++i) {
      const double xi = rhs[i] / S[i * G + i];
      __syncwarp();
      if (lane == 0) rhs[i] = xi;
      for (int k = i + 1 + lane; k < G; k += 32) rhs[k] -= S[k * G + i] * xi;
      __syncwarp();
    }
    for (int i = G - 1; i >= 0; --i) {
      const double xi = rhs[i] / S[i * G + i];
      __syncwarp();
      if (lane == 0) rhs[i] = xi;
      for (int k = lane; k < i; k += 32) rhs[k] -= S[i * G + k] * xi;
      __syncwarp();
    }
    if (bad && lane == 0) a.scalars[kScNotPD] = 1.0;
  }
  __syncthreads();
  for (int i = tid; i < G; i += 256) a.delta[nfp + i] = bad ? 0.0 : rhs[i];
}

// ---------------------------------------------------------------- x (+) delta of the globals
// Ceres minimises over the blocks that are neither constant nor unused (Program::RemoveFixedBlocks): it never moves the
// others and leaves them out of x_norm.  So a constant block (DevProblem::free_blocks) is copied, not pushed through
// Plus (so3_plus renormalises, which can change a constant quaternion's last bits), and only free blocks count towards
// |x_new|^2.
__device__ __forceinline__ bool block_free(const DevProblem& dp, int bit) { return (dp.free_blocks >> bit) & 1u; }

// Camera c's state [q_ck p_ck intr]; dg: the scaled global step (null: a zero step), sc: the globals' scaling.
__device__ inline void cam_plus(const DevProblem& dp, int c, const double* x, const double* dg, const double* sc, double* xo) {
  const CamInfo& ci = dp.cams[c];
  const int o = ci.goff;
  if (block_free(dp, kFreeCam * c)) {
    double du[3];
    for (int k = 0; k < 3; ++k) du[k] = dg ? dg[o + k] * sc[o + k] : 0.0;
    so3_plus(x, du, xo);
  } else {
    for (int k = 0; k < 4; ++k) xo[k] = x[k];
  }
  const bool p_free = dg && block_free(dp, kFreeCam * c + 1), intr_free = dg && block_free(dp, kFreeCam * c + 2);
  for (int k = 0; k < 3; ++k) xo[4 + k] = p_free ? x[4 + k] + dg[o + 3 + k] * sc[o + 3 + k] : x[4 + k];
  for (int k = 0; k < 10; ++k) xo[7 + k] = k < ci.K && intr_free ? x[7 + k] + dg[o + 6 + k] * sc[o + 6 + k] : x[7 + k];
}
// adds camera c's |x_new - x|^2 to st[0] and, over its free blocks, |x_new|^2 to st[1]
__device__ inline void cam_stats(const DevProblem& dp, int c, const double* x, const double* xo, double* st) {
  for (int k = 0; k < 7 + dp.cams[c].K; ++k) {
    st[0] += (xo[k] - x[k]) * (xo[k] - x[k]);
    if (block_free(dp, kFreeCam * c + (k < 4 ? 0 : k < 7 ? 1 : 2))) st[1] += xo[k] * xo[k];
  }
}
// the IMU parameters [g2 b6 sf6 ts1] (their tangent columns are the same 15 entries, at dp.imu_goff), with their step
// statistics; all constant in a vision-only run
__device__ inline void imu_plus(const DevProblem& dp, const double* x, const double* dg, const double* sc, double* xo,
                                double* st) {
  for (int k = 0; k < kImuStateSize; ++k) {
    const int q = dp.imu_goff + k;
    const bool free = block_free(dp, kFreeImu + (k < 2 ? 0 : k < 8 ? 1 : k < 14 ? 2 : 3));
    const double dd = free && dg ? dg[q] * sc[q] : 0.0;
    xo[k] = free ? x[k] + dd : x[k];
    st[0] += dd * dd;
    if (free) st[1] += xo[k] * xo[k];
  }
}
// every camera and the IMU parameters into the trial state, with their |x_new - x|^2 and |x_new|^2 added to st[0..1]
__device__ inline void globals_plus(const DevProblem& dp, const double* x_cur, double* x_new, const double* dg, const double* sc,
                                    double* st) {
  for (int c = 0; c < dp.n_cams; ++c) {
    const double* x = x_cur + dp.off_cam + kCamStateStride * c;
    double* xo = x_new + dp.off_cam + kCamStateStride * c;
    cam_plus(dp, c, x, dg, sc, xo);
    cam_stats(dp, c, x, xo, st);
  }
  imu_plus(dp, x_cur + dp.off_imu, dg, sc, x_new + dp.off_imu, st);
}

// Frame f into the trial state (d: its scaled step): se3_plus of the pose (copied when no residual uses the frame), the
// velocity plus its step for FD == 9 (copied for FD == 6), and the frame's share of the step statistics acc: step.g,
// step.D2.step, |x_new - x|^2, |x_new|^2.  The ghost moves with the step too; its damping and norms are counted by its
// owner, and its gradient is this rank's piece of the shared frame's gradient, so step.g counts it.
template <int FD>
__device__ __forceinline__ void frame_plus(const DevProblem& dp, const Blocks& b, const double* scale, double rinv,
                                           const double* D2x, const double* sepdiag, int f, const double* d, bool used,
                                           const double* x_cur, double* x_new, double acc[4]) {
  const bool is_ghost = FD == 9 && dp.ghost && f == dp.n_frames - 1;  // (only inertial runs have a ghost)
  double du[FD];
#pragma unroll
  for (int r = 0; r < FD; ++r) {
    const int64_t k = static_cast<int64_t>(f) * FD + r;
    const double sc = scale[k];
    const double d2 = frame_damp<FD>(0.0, f, r, b.B[k * FD + r], sc, rinv, D2x, sepdiag, dp.rank, is_ghost);
    acc[0] += d[r] * b.gf[k] * sc;
    acc[1] += d[r] * d[r] * d2;
    du[r] = d[r] * sc;
  }
  const bool counted = used && !is_ghost;
  const double* x = x_cur + 7 * static_cast<int64_t>(f);
  double xo[7];
  if (used) {
    se3_plus(x, du, xo);
  } else {
#pragma unroll
    for (int k = 0; k < 7; ++k) xo[k] = x[k];
  }
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    x_new[7 * static_cast<int64_t>(f) + k] = xo[k];
    if (counted) {
      acc[2] += (xo[k] - x[k]) * (xo[k] - x[k]);
      acc[3] += xo[k] * xo[k];
    }
  }
  const double* v = x_cur + dp.off_v + 3 * static_cast<int64_t>(f);
  double* vo = x_new + dp.off_v + 3 * static_cast<int64_t>(f);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double nv = (FD == 9) ? v[k] + du[(FD == 9) ? 6 + k : 0] : v[k];
    vo[k] = nv;
    if (FD == 9 && counted) {
      acc[2] += (nv - v[k]) * (nv - v[k]);
      acc[3] += nv * nv;
    }
  }
}

// ---------------------------------------------------------------- back-substitution + x (+) delta
struct UpdateArgs {
  DevProblem dp;
  Blocks b[2];
  const Ctl* ctl;
  const uint8_t* frame_used;  // [nf] 0: a vision-only frame that no active observation sees (left as it is)
  const double* scale;
  const double* D2x;
  const double* X;    // null: the chain solver already wrote the frame steps into delta
  double* delta;
  double* state[2];
  double* step_part;  // [gridDim+1][4]
  const double* sepdiag;  // sharded inertial run: summed diagonal of the separator frames, else null
};
constexpr int kUpdateWarps = 4;

// One warp: a frame's back-substitution d = -x_f - X_f[:, :G] dg from Xf [FD][G + 1] (column G: x_f = (B_f + D_f)^-1 g_f)
// and the globals' step dg; every lane gets d.
template <int FD>
__device__ __forceinline__ void frame_backsub(const double* Xf, const double* dg, int G, int lane, double* d) {
  const int M = G + 1;
#pragma unroll
  for (int r = 0; r < FD; ++r) {
    double s = 0.0;
    for (int c = lane; c < G; c += 32) s += Xf[r * M + c] * dg[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    d[r] = -Xf[r * M + G] - s;
  }
}

template <int FD>
__global__ void __launch_bounds__(32 * kUpdateWarps) backsub_update_kernel(UpdateArgs a) {
  if (a.ctl->done) return;
  const int cur = a.ctl->cur;
  const Blocks& b = a.b[cur];
  const double* x_cur = a.state[cur];
  double* x_new = a.state[1 - cur];
  const double rinv = 1.0 / a.ctl->radius;
  const int G = a.dp.G, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nf = a.dp.n_frames;
  const int64_t nfp = static_cast<int64_t>(nf) * FD;
  const double* dc = a.delta + nfp;
  __shared__ double part[kUpdateWarps][4];
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  const int f = blockIdx.x * kUpdateWarps + warp;
  if (f < nf) {
    double d[FD];
    if (a.X) {
      frame_backsub<FD>(a.X + static_cast<int64_t>(f) * FD * (G + 1), dc, G, lane, d);
    } else {
#pragma unroll
      for (int r = 0; r < FD; ++r) d[r] = a.delta[static_cast<int64_t>(f) * FD + r];
    }
    if (lane == 0) {
#pragma unroll
      for (int r = 0; r < FD; ++r) a.delta[static_cast<int64_t>(f) * FD + r] = d[r];
      frame_plus<FD>(a.dp, b, a.scale, rinv, a.D2x, a.sepdiag, f, d, a.frame_used[f] != 0, x_cur, x_new, acc);
    }
  }
  if (lane == 0)
    for (int q = 0; q < 4; ++q) part[warp][q] = acc[q];
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int q = 0; q < 4; ++q) {
      double s = 0.0;
      for (int w = 0; w < kUpdateWarps; ++w) s += part[w][q];
      a.step_part[4 * static_cast<int64_t>(blockIdx.x) + q] = s;
    }
  }
  // globals: cameras + IMU parameters (one thread of block 0)
  if (blockIdx.x == 0 && threadIdx.x == 32 * kUpdateWarps - 1) {
    double g4[4] = {0.0, 0.0, 0.0, 0.0};
    const double* sc = a.scale + nfp;
    globals_plus(a.dp, x_cur, x_new, dc, sc, g4 + 2);
    for (int k = 0; k < G; ++k) {
      const double d2 = global_damp(k, b.C[k * G + k], sc[k], rinv, a.D2x, nfp);
      g4[0] += dc[k] * b.gc[k] * sc[k];
      g4[1] += dc[k] * dc[k] * d2;
    }
    for (int q = 0; q < 4; ++q) a.step_part[4 * static_cast<int64_t>(gridDim.x) + q] = g4[q];
  }
}

}  // namespace vc
