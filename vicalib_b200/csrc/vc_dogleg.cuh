// Dogleg trust-region strategy on the device (the reference's setting: solver_options_.trust_region_
// strategy_type = DOGLEG, TRADITIONAL_DOGLEG; vicalibrator.h:151, Ceres DoglegStrategy).
//
// Per iteration, on the Jacobi-scaled block-arrow system  H = S J^T J S,  g = S J^T r  of the accepted point:
//   D      = sqrt(clamp(diag H, 1e-6, 1e32))                (dl_prep_kernel)
//   g~     = g / D,   alpha = |g~|^2 / (u . H u),  u = g~ / D     Cauchy step = -alpha g~   (matvec + dots)
//   gn     = D * [(H + mu D^2)^-1 (-g)]                      Gauss-Newton step (the engine's arrow solve)
//   step~  = gn                                  if |gn| <= radius
//          = -(radius / |g~|) g~                 if alpha |g~| >= radius
//          = the dogleg point on the segment     otherwise                                (dl_combine_kernel)
//   step   = step~ / D,  model change = -step.g - step.H.step / 2                         (matvec + dots)
// then x (+) S step, evaluate there, and dl_decide_kernel applies Ceres' accept / radius / mu rules.
// All state (mu, alpha, norms) lives in Ctl, so iterations are enqueued without a host round trip, like
// the LM engine.  Deterministic: every reduction is two-level with a fixed order.
#pragma once
#include "vc_internal.h"
#include "vc_kernels.cuh"

namespace vc {

constexpr int kDlBlocks = 64;

struct DlVecs {           // all [nf*fd + G]
  double *diag, *grad, *gn, *vec, *Hv, *D2;
};

// ---------------------------------------------------------------- D, g~, u, mu D^2
// D^2 of entry i: clamp(diag H) of the scaled system (diag: the unscaled H_ii, s: its Jacobi scale)
__device__ __forceinline__ double dl_clamp(double diag, double s) {
  const double c = diag * s * s;
  return c < 1e-6 ? 1e-6 : (c > 1e32 ? 1e32 : c);
}
// D and g~ = g / D of entry i of the scaled system (g: the unscaled gradient entry)
__device__ __forceinline__ void dl_scaled(double diag, double g, double s, double* D, double* gt) {
  *D = sqrt(dl_clamp(diag, s));
  *gt = g * s / *D;
}
__global__ void dl_prep_kernel(DevProblem dp, Blocks b0, Blocks b1, const Ctl* ctl, const double* scale, DlVecs v) {
  if (ctl->done) return;
  const Blocks& b = ctl->cur ? b1 : b0;
  const int64_t nfp = static_cast<int64_t>(dp.n_frames) * dp.fd, n = nfp + dp.G;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double d, g;
  if (i < nfp) {
    const int64_t f = i / dp.fd;
    const int k = static_cast<int>(i - f * dp.fd);
    d = b.B[(f * dp.fd + k) * dp.fd + k];
    g = b.gf[i];
  } else {
    const int k = static_cast<int>(i - nfp);
    d = b.C[k * dp.G + k];
    g = b.gc[k];
  }
  const double s = scale[i];
  double D, gt;
  dl_scaled(d, g, s, &D, &gt);
  v.diag[i] = D;
  v.grad[i] = gt;
  v.vec[i] = gt / D;
  v.D2[i] = dl_clamp(d, s) * ctl->dl_mu;
}

// ---------------------------------------------------------------- y = S H S v on the block-arrow system
// One warp per frame: rows of the frame block (plus the tridiagonal IMU coupling U and E w_g); the frames'
// contributions E^T w_f to the globals' rows go to per-CTA partials, summed in order by the second kernel.
constexpr int kMvWarps = 4;
template <int FD>
__global__ void __launch_bounds__(32 * kMvWarps) arrow_matvec_frames_kernel(DevProblem dp, Blocks b0, Blocks b1, const Ctl* ctl,
                                                                            const double* scale, const double* v, double* y,
                                                                            double* zpart) {
  extern __shared__ double zs[];  // [kMvWarps][G]
  if (ctl->done) return;
  const Blocks& b = ctl->cur ? b1 : b0;
  const int G = dp.G, nf = dp.n_frames, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t nfp = static_cast<int64_t>(nf) * FD;
  const int f = blockIdx.x * kMvWarps + warp;
  double* zw = zs + warp * G;
  for (int c = lane; c < G; c += 32) zw[c] = 0.0;
  if (f < nf) {
    const int64_t o = static_cast<int64_t>(f) * FD;
    double w[FD];
#pragma unroll
    for (int r = 0; r < FD; ++r) w[r] = scale[o + r] * v[o + r];
    double acc[FD];
#pragma unroll
    for (int r = 0; r < FD; ++r) {  // E w_g, lanes split the columns
      double s = 0.0;
      for (int c = lane; c < G; c += 32) s += b.E[(o + r) * G + c] * (scale[nfp + c] * v[nfp + c]);
#pragma unroll
      for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
      acc[r] = s;
    }
    if (lane < FD) {
      const int r = lane;
      double s = 0.0;
#pragma unroll
      for (int c = 0; c < FD; ++c) s += b.B[(o + r) * FD + c] * w[c];
      if (FD == 9 && dp.inertial) {
        if (f > 0) {  // U[f] = H[f-1, f]:  y_f += U[f]^T w_{f-1}
          const double* U = b.U + o * FD;
          for (int a = 0; a < FD; ++a) s += U[a * FD + r] * (scale[o - FD + a] * v[o - FD + a]);
        }
        if (f + 1 < nf) {  // y_f += U[f+1] w_{f+1}
          const double* U = b.U + (o + FD) * FD;
          for (int c = 0; c < FD; ++c) s += U[r * FD + c] * (scale[o + FD + c] * v[o + FD + c]);
        }
      }
      double e = 0.0;
#pragma unroll
      for (int q = 0; q < FD; ++q) e = (q == r) ? acc[q] : e;
      y[o + r] = scale[o + r] * (s + e);
    }
    for (int c = lane; c < G; c += 32) {  // E^T w_f
      double s = 0.0;
#pragma unroll
      for (int r = 0; r < FD; ++r) s += b.E[(o + r) * G + c] * w[r];
      zw[c] = s;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < G; c += blockDim.x) {
    double s = 0.0;
    for (int k = 0; k < kMvWarps; ++k) s += zs[k * G + c];
    zpart[static_cast<int64_t>(blockIdx.x) * G + c] = s;
  }
}
// mode 0: one GPU — sum of the per-CTA partials + C w_g.  Frame shards: mode 1 leaves this rank's sum of E^T w_f in
// zsum [G] (all-reduced by the host code), mode 2 finishes y_g from the summed zsum.
__global__ void __launch_bounds__(256) arrow_matvec_globals_kernel(DevProblem dp, Blocks b0, Blocks b1, const Ctl* ctl,
                                                                    const double* scale, const double* v, double* y,
                                                                    const double* zpart, int nparts, int mode, double* zsum) {
  if (ctl->done) return;
  const Blocks& b = ctl->cur ? b1 : b0;
  const int G = dp.G;
  const int64_t nfp = static_cast<int64_t>(dp.n_frames) * dp.fd;
  for (int c = threadIdx.x; c < G; c += blockDim.x) {
    double s = 0.0;
    if (mode != 2) {
      double s0 = 0.0, s1 = 0.0;
      int k = 0;
      for (; k + 1 < nparts; k += 2) { s0 += zpart[static_cast<int64_t>(k) * G + c]; s1 += zpart[static_cast<int64_t>(k + 1) * G + c]; }
      if (k < nparts) s0 += zpart[static_cast<int64_t>(k) * G + c];
      s = s0 + s1;
      if (mode == 1) { zsum[c] = s; continue; }
    } else {
      s = zsum[c];
    }
    for (int q = 0; q < G; ++q) s += b.C[c * G + q] * (scale[nfp + q] * v[nfp + q]);
    y[nfp + c] = scale[nfp + c] * s;
  }
}

// ---------------------------------------------------------------- fixed-order dot products + the scalar steps
// mode 0: alpha = |g~|^2 / (u . H u)
// mode 1: gn = delta * D (stored); |gn|^2, g~ . gn
// mode 2: step . g (scaled gradient = g~ * D) and step . H step  ->  model change
struct DlDotArgs {
  Ctl* ctl;
  DlVecs v;
  const double* delta;   // scaled Gauss-Newton step from the arrow solve
  const double* scalars; // kSc*: not-PD flag of the solve
  double* part;          // [kDlBlocks][4]
  unsigned* counter;
  int64_t n;       // entries of the vectors (mode 1 stores gn for all of them)
  int64_t n_sum;   // entries this rank sums: all of them, or on ranks > 0 of a sharded run only its frames' (the
                   // globals' entries are replicated and counted once, by rank 0)
  int mode;
  double* mg;      // frame shards: the two sums go here ([2], all-reduced by the host code) and dl_dots_finish_kernel
                   // applies them; null: one GPU, applied here
};
__device__ inline void dl_apply_dots(Ctl* c, int mode, double t0, double t1, const double* scalars) {
  if (mode == 0) {
    c->dl_g2 = t0;
    c->dl_alpha = t0 / t1;
  } else if (mode == 1) {
    c->dl_gn2 = t0;
    c->dl_b = t1;
    c->dl_ok = scalars[kScNotPD] > 0.0 ? 0 : 1;
  } else {
    c->dl_model_change = -t0 - 0.5 * t1;
  }
}
__global__ void dl_dots_finish_kernel(Ctl* c, int mode, const double* mg, const double* scalars) {
  if (threadIdx.x == 0 && blockIdx.x == 0 && !c->done) dl_apply_dots(c, mode, mg[0], mg[1], scalars);
}
__global__ void __launch_bounds__(256) dl_dots_kernel(DlDotArgs a) {
  __shared__ double sh[8][3];
  __shared__ int is_last;
  if (a.ctl->done) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nb = gridDim.x, bid = blockIdx.x;
  const int64_t lo = a.n * bid / nb, hi = a.n * (bid + 1) / nb;
  double s[3] = {0.0, 0.0, 0.0};
  for (int64_t i = lo + tid; i < hi; i += 256) {
    const double on = i < a.n_sum ? 1.0 : 0.0;
    if (a.mode == 0) {
      s[0] += on * a.v.grad[i] * a.v.grad[i];
      s[1] += on * a.v.vec[i] * a.v.Hv[i];
    } else if (a.mode == 1) {
      const double gn = a.delta[i] * a.v.diag[i];
      a.v.gn[i] = gn;
      s[0] += on * gn * gn;
      s[1] += on * a.v.grad[i] * gn;
    } else {
      s[0] += on * a.v.vec[i] * (a.v.grad[i] * a.v.diag[i]);
      s[1] += on * a.v.vec[i] * a.v.Hv[i];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
#pragma unroll
    for (int q = 0; q < 2; ++q) s[q] += __shfl_down_sync(0xffffffffu, s[q], o);
  if (lane == 0) { sh[warp][0] = s[0]; sh[warp][1] = s[1]; }
  __syncthreads();
  if (tid == 0) {
    double t0 = 0.0, t1 = 0.0;
    for (int w = 0; w < 8; ++w) { t0 += sh[w][0]; t1 += sh[w][1]; }
    a.part[4 * bid] = t0;
    a.part[4 * bid + 1] = t1;
    __threadfence();
    const unsigned ticket = atomicInc(a.counter, static_cast<unsigned>(nb - 1));
    is_last = ticket == static_cast<unsigned>(nb - 1);
  }
  __syncthreads();
  if (!is_last || tid != 0) return;
  __threadfence();
  double t0 = 0.0, t1 = 0.0;
  for (int k = 0; k < nb; ++k) { t0 += __ldcg(a.part + 4 * k); t1 += __ldcg(a.part + 4 * k + 1); }
  if (a.mg) { a.mg[0] = t0; a.mg[1] = t1; }
  else dl_apply_dots(a.ctl, a.mode, t0, t1, a.scalars);
}

// ---------------------------------------------------------------- the dogleg point (Ceres DoglegStrategy::ComputeTraditionalDoglegStep)
// step~ = cg g~ + cn gn from the step's scalars (radius, alpha, |g~|^2, |gn|^2, b = g~ . gn); returns |step~|.  The one
// definition of the branch rule: dl_combine_kernel and the persistent kernel (vc_mega.cuh) both call it.
__device__ inline double dogleg_point(double radius, double alpha, double g2, double gn2, double b, double* cg, double* cn) {
  const double gn_norm = sqrt(gn2), g_norm = sqrt(g2);
  if (gn_norm <= radius) {
    *cg = 0.0; *cn = 1.0;
    return gn_norm;
  }
  if (g_norm * alpha >= radius) {
    *cg = -(radius / g_norm); *cn = 0.0;
    return radius;
  }
  const double b_dot_a = -alpha * b;
  const double a_sq = (alpha * g_norm) * (alpha * g_norm);
  const double bma_sq = a_sq - 2.0 * b_dot_a + gn_norm * gn_norm;
  const double cc = b_dot_a - a_sq;
  const double d = sqrt(cc * cc + bma_sq * (radius * radius - a_sq));
  const double beta = cc <= 0.0 ? (d - cc) / bma_sq : (radius * radius - a_sq) / (d + cc);
  *cg = -alpha * (1.0 - beta); *cn = beta;
  // |cg g~ + cn gn|^2 from the known inner products
  return sqrt(fmax(0.0, *cg * *cg * g2 + 2.0 * *cg * *cn * b + *cn * *cn * gn2));
}
__global__ void dl_combine_kernel(Ctl* ctl, DlVecs v, double* delta, int64_t n) {
  if (ctl->done) return;
  double cg, cn;
  const double step_norm = dogleg_point(ctl->radius, ctl->dl_alpha, ctl->dl_g2, ctl->dl_gn2, ctl->dl_b, &cg, &cn);
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) {
    const double st = ctl->dl_ok ? (cg * v.grad[i] + cn * v.gn[i]) / v.diag[i] : 0.0;
    v.vec[i] = st;
    delta[i] = st;
  }
  if (i == 0) ctl->dl_step_norm = step_norm;
}

// ---------------------------------------------------------------- accept / reject, radius and mu (Ceres TrustRegionMinimizer + DoglegStrategy)
__global__ void dl_decide_kernel(Ctl* c, double* sc) {
  if (threadIdx.x == 0 && blockIdx.x == 0) decide_step<Strategy::kDogleg>(c, sc, 1);
}

}  // namespace vc
