// Regression diagnostics of every IMU interval (vcgpu_get_imu_influence(_batch)).  Interval k touches
// P = (frame k: pose 6, v 3 | frame k+1: pose 6, v 3 | IMU globals g 2, b 6, sf 6, ts 1), p = 33.  With J~ and r~ the
// interval's 9 x 33 Jacobian and residual as the solve's build weights them (sqrt(imu_mult rho'), CauchyLoss(100);
// imu_eval_kernel with the loss applied, into the call's own buffers), Sigma_PP the P x P block of the covariance and,
// on F (the globals whose variance is not 0.0),
//   H    = J~ Sigma_PP J~^T                       (9 x 9 leverage, one triangle formed and mirrored)
//   u    = (I - H)^-1 r~                           (9 x 9 Cholesky, fixed order)
//   stud = r~ . u
//   infl = Dg^T Sigma_F^-1 Dg = |y|^2,  Dg = Sigma_FP a,  a = J~^T u,  y = L^-1 D^-1 Dg
// with L, D view_prior_kernel's factor of Sigma_F.  One CTA per interval (imu_infl_kernel): Sigma_PP (assembled from
// Sigma_kk, Sigma_k+1,k+1, Sigma_k,k+1, Sigma_kg, Sigma_k+1,g and Sigma_gg's IMU block) and J~ staged in shared memory;
// the triangular solve by one warp.  Every output has one owner and a fixed summation order, so a rig's bits depend on
// nothing else in the launch.
#pragma once
#include "vc_imu.cuh"
#include "vc_obs_infl.cuh"

namespace vc {

constexpr int kImuInflThreads = 128;
constexpr int kImuInflP = 33;  // P's size, the staged matrices' leading dimension

// one rig of a launch: its intervals are CTAs [cta0, cta0 + ni)
struct ImuInflRig {
  imu::ImuBuf buf;            // the interval's has-measurement test, imu_integrate's
  const double* ftime;        // [nf] frame times
  const double* state;        // the accepted state buffer (ts)
  int64_t off_imu;
  const double* r;            // [ni][9]   imu_eval_kernel's, loss applied
  const double* J;            // [ni][297] imu_eval_kernel's, loss applied and masked, vcgpu_eval_imu's column order
  const double* Sff;          // [nf][81]
  const double* Sfn;          // [nf-1][81] Sigma_f,f+1, rows frame f
  const double* Sfg;          // [nf][9][G]
  const double* Sgg;          // [G][G] unscaled (infl_sgg_kernel)
  const int32_t* fidx;        // [GF] global index of each row of F (view_prior_kernel's)
  const double* L;            // [GF][GF] chol of the Jacobi-scaled Sigma_F (view_prior_kernel)
  const double* D;            // [GF] sqrt(diag Sigma_F)
  const int* prior_ok;        // view_prior_kernel's flag
  double *h, *stud, *infl;    // [ni][81], [ni], [ni], each may be null
  double sm;                  // sqrt(imu_mult)
  int64_t cta0;
  int ni, G, GF, io;          // io: the IMU globals' offset in G
};

// entry (i, j) of interval k's Sigma_PP
__device__ __forceinline__ double imu_infl_sigma(const ImuInflRig& a, int k, int i, int j) {
  const int bi = i < 9 ? 0 : i < 18 ? 1 : 2, bj = j < 9 ? 0 : j < 18 ? 1 : 2;
  const int64_t G = a.G;
  if (bi < 2 && bj < 2) {
    if (bi == bj) return a.Sff[static_cast<int64_t>(k + bi) * 81 + (i - 9 * bi) * 9 + (j - 9 * bj)];
    return bi == 0 ? a.Sfn[static_cast<int64_t>(k) * 81 + i * 9 + (j - 9)] : a.Sfn[static_cast<int64_t>(k) * 81 + j * 9 + (i - 9)];
  }
  if (bi < 2) return a.Sfg[(static_cast<int64_t>(k + bi) * 9 + (i - 9 * bi)) * G + a.io + j - 18];
  if (bj < 2) return a.Sfg[(static_cast<int64_t>(k + bj) * 9 + (j - 9 * bj)) * G + a.io + i - 18];
  return a.Sgg[(a.io + i - 18) * G + a.io + j - 18];
}

__global__ void __launch_bounds__(kImuInflThreads) imu_infl_kernel(const ImuInflRig* __restrict__ rigs, int n_rigs) {
  __shared__ double S[kImuInflP * kImuInflP], Jt[9 * kImuInflP], T[kImuInflP * 9], H[81], A[81], rt[9], u[9];
  __shared__ double av[kImuInflP], y[kInflMaxGF];
  __shared__ int pd;
  int lo = 0, hi = n_rigs - 1;  // the last rig whose cta0 <= blockIdx.x
  while (lo < hi) {
    const int mid = (lo + hi + 1) / 2;
    if (rigs[mid].cta0 <= blockIdx.x) lo = mid;
    else hi = mid - 1;
  }
  const ImuInflRig& a = rigs[lo];
  const int k = static_cast<int>(blockIdx.x - a.cta0), tid = threadIdx.x, nt = blockDim.x;
  if (!*a.prior_ok) return;  // the rig's outputs are not returned
  double* ho = a.h ? a.h + static_cast<int64_t>(k) * 81 : nullptr;
  // no measurements: the solve gives the interval a zero residual and Jacobian (imu_integrate's HasElement test)
  const double ts = a.state[a.off_imu + 14], t0 = a.ftime[k];
  if (!(t0 >= a.buf.start_time + ts && t0 <= a.buf.end_time + ts) || a.buf.n == 0) {
    if (ho)
      for (int e = tid; e < 81; e += nt) ho[e] = NAN;
    if (tid == 0) {
      if (a.stud) a.stud[k] = NAN;
      if (a.infl) a.infl[k] = NAN;
    }
    return;
  }
  for (int e = tid; e < kImuInflP * kImuInflP; e += nt) S[e] = imu_infl_sigma(a, k, e / kImuInflP, e % kImuInflP);
  const double* Jk = a.J + static_cast<int64_t>(k) * 297;
  for (int e = tid; e < 9 * kImuInflP; e += nt) {
    const int row = e / kImuInflP, c = e % kImuInflP;
    Jt[e] = a.sm * Jk[row * 33 + imu_local_col(c)];  // into P's order
  }
  if (tid < 9) rt[tid] = a.sm * a.r[static_cast<int64_t>(k) * 9 + tid];
  __syncthreads();
  // T = Sigma_PP J~^T (33 x 9)
  for (int e = tid; e < kImuInflP * 9; e += nt) {
    const int i = e / 9, r = e % 9;
    double s = 0.0;
    for (int j = 0; j < kImuInflP; ++j) s += S[i * kImuInflP + j] * Jt[r * kImuInflP + j];
    T[e] = s;
  }
  __syncthreads();
  // H = J~ T, the lower triangle mirrored
  for (int e = tid; e < 81; e += nt) {
    const int r = e / 9, c = e % 9;
    if (c > r) continue;
    double s = 0.0;
    for (int i = 0; i < kImuInflP; ++i) s += Jt[r * kImuInflP + i] * T[i * 9 + c];
    H[r * 9 + c] = s;
    H[c * 9 + r] = s;
  }
  __syncthreads();
  if (ho)
    for (int e = tid; e < 81; e += nt) ho[e] = H[e];
  // I - H = L L^T in place (lower triangle of A), then u = (L L^T)^-1 r~: one thread
  if (tid == 0) {
    bool ok = true;
    for (int j = 0; j < 9 && ok; ++j) {
      double d = 1.0 - H[j * 9 + j];
      for (int p = 0; p < j; ++p) d -= A[j * 9 + p] * A[j * 9 + p];
      if (!(d > 0.0)) { ok = false; break; }
      const double ljj = sqrt(d);
      A[j * 9 + j] = ljj;
      for (int i = j + 1; i < 9; ++i) {
        double s = -H[i * 9 + j];
        for (int p = 0; p < j; ++p) s -= A[i * 9 + p] * A[j * 9 + p];
        A[i * 9 + j] = s / ljj;
      }
    }
    pd = ok ? 1 : 0;
    if (ok) {
      double z[9];
      for (int i = 0; i < 9; ++i) {
        double s = rt[i];
        for (int p = 0; p < i; ++p) s -= A[i * 9 + p] * z[p];
        z[i] = s / A[i * 9 + i];
      }
      double st = 0.0;
      for (int i = 8; i >= 0; --i) {
        double s = z[i];
        for (int p = i + 1; p < 9; ++p) s -= A[p * 9 + i] * u[p];
        u[i] = s / A[i * 9 + i];
      }
      for (int i = 0; i < 9; ++i) st += rt[i] * u[i];
      if (a.stud) a.stud[k] = st;
    } else if (a.stud) {
      a.stud[k] = NAN;
    }
  }
  __syncthreads();
  if (!pd) {
    if (tid == 0 && a.infl) a.infl[k] = NAN;
    return;
  }
  if (!a.infl) return;
  // a = J~^T u
  if (tid < kImuInflP) {
    double s = 0.0;
    for (int r = 0; r < 9; ++r) s += Jt[r * kImuInflP + tid] * u[r];
    av[tid] = s;
  }
  __syncthreads();
  // D^-1 Dg = D^-1 Sigma_FP a, one row of F per thread
  const int GF = a.GF;
  const int64_t G = a.G;
  for (int i = tid; i < GF; i += nt) {
    const int64_t g = a.fidx[i];
    const double* f0 = a.Sfg + static_cast<int64_t>(k) * 9 * G + g;
    const double* f1 = f0 + 9 * G;
    double s = 0.0;
    for (int c = 0; c < 9; ++c) s += f0[c * G] * av[c];
    for (int c = 0; c < 9; ++c) s += f1[c * G] * av[9 + c];
    for (int c = 0; c < 15; ++c) s += a.Sgg[g * G + a.io + c] * av[18 + c];
    y[i] = s / a.D[i];
  }
  __syncthreads();
  // y = L^-1 y by warp 0, column-oriented in j order; infl = sum_j y_j^2 in j order
  if (tid >= 32) return;
  double infl = 0.0;
  for (int j = 0; j < GF; ++j) {
    const double yj = y[j] / a.L[static_cast<int64_t>(j) * GF + j];
    infl += yj * yj;
    __syncwarp();
    for (int i = j + 1 + tid; i < GF; i += 32) y[i] -= a.L[static_cast<int64_t>(i) * GF + j] * yj;
    __syncwarp();
  }
  if (tid == 0) a.infl[k] = infl;
}

}  // namespace vc
