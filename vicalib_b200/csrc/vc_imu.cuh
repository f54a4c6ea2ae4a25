// IMU residual family on the device and the block-tridiagonal frame chain it induces.
//
//   imu_eval_kernel      three frame intervals per warp, a team of 10 lanes each: a lane carries one attitude-coupled
//                        tangent direction through the RK4 integrator (forward-mode dual numbers) and two (p, v)-only
//                        or end-map-only columns beside it: r (9) and J (9x33)
//                        [SwitchedFullImuCostFunction, ceres-cost-functions.h:379-490]
//   imu_accumulate_kernel adds J^T J of the two intervals touching a frame into the frame blocks
//                        (B, off-diagonal U, E columns of the 15 IMU globals, gradients)
//   chain_*              partitioned elimination of the block-tridiagonal + arrow system
//   imu_weights_kernel   UpdateImuWeights (vicalibrator.h:723-799)
#pragma once
#include <algorithm>
#include <vector>

#include "vc_imu_math.cuh"
#include "vc_internal.h"

namespace vc {

constexpr int kImuCgStride = 136;  // 15*16/2 = 120 packed sym + 15 gradient (+1 pad)

// ---------------------------------------------------------------- IMU evaluate
struct ImuEvalArgs {
  DevProblem dp;
  imu::ImuBuf buf;
  const Ctl* ctl;
  int which;
  const double* states[2];
  const double* ftime;
  const double* wsqrt;  // [ni][81]
  const double* mask;   // 15 IMU global columns
  double *r, *J, *cost;
  int ni, apply_loss;
  double mult;
};

// column `col` (0..5) of LocalParamSe3::ComputeJacobian (local-param-se3.h:61-88), 7 entries
__device__ __forceinline__ void se3_local_column(const double* x, int col, double out[7]) {
  const double q1 = x[0], q2 = x[1], q3 = x[2], q0 = x[3];
#pragma unroll
  for (int i = 0; i < 7; ++i) out[i] = 0.0;
  switch (col) {
    case 0: out[4] = 1.0 - 2.0 * (q2 * q2 + q3 * q3); out[5] = 2.0 * (q1 * q2 + q0 * q3); out[6] = 2.0 * (q1 * q3 - q0 * q2); break;
    case 1: out[4] = 2.0 * (q1 * q2 - q0 * q3); out[5] = 1.0 - 2.0 * (q1 * q1 + q3 * q3); out[6] = 2.0 * (q2 * q3 + q0 * q1); break;
    case 2: out[4] = 2.0 * (q1 * q3 + q0 * q2); out[5] = 2.0 * (q2 * q3 - q0 * q1); out[6] = 1.0 - 2.0 * (q1 * q1 + q2 * q2); break;
    case 3: out[0] = 0.5 * q0; out[1] = 0.5 * q3; out[2] = -0.5 * q2; out[3] = -0.5 * q1; break;
    case 4: out[0] = -0.5 * q3; out[1] = 0.5 * q0; out[2] = 0.5 * q1; out[3] = -0.5 * q2; break;
    case 5: out[0] = 0.5 * q2; out[1] = -0.5 * q1; out[2] = 0.5 * q0; out[3] = -0.5 * q3; break;
  }
}

// the fields of ImuEvalArgs the evaluation reads, by value (the persistent kernel passes them to a __noinline__ task
// function: a reference to its parameter block would force the whole block into local memory)
struct ImuEvalView {
  struct { int64_t off_v, off_imu; int rotation_only; } dp;
  imu::ImuBuf buf;
  const double* ftime;
  const double* wsqrt;
  const double* mask;
  double *r, *J, *cost;
  int ni, apply_loss;
  double mult;
};
// the same fields as ImuAccArgs with the problem description by reference
struct ImuAccView {
  const DevProblem& dp;
  const double *r, *J;
  double* Cg;
  int ni;
};

constexpr int kImuWarps = 4;
// An interval's 33 Jacobian columns by a team of 10 lanes, 3 teams per warp (lanes 30, 31 idle).  p and v never feed
// back into the integrator, so only 10 columns reach the attitude: pose1 rotation 9-11, gyro bias 20-22, gyro scale
// 26-28 and ts 32.  Team lane t carries column imu_col_chain(t) through the RK4 chain as a dual number, and two more
// columns that need only the end map T_end T2^-1 -> log: imu_col_acc(t) (accelerometer bias 23-25 and scale 29-31 on
// lanes 0-5, an AccelTangent of the chain; gravity 18-19 and v1 15-16 on lanes 6-9) and imu_col_end(t) (pose2 0-5,
// pose1 translation 6-8, v1 17).  The v2 columns 12-14 are analytic.
constexpr int kImuTeam = 10, kImuTeams = 3;
__device__ __forceinline__ int imu_col_chain(int t) { return t < 3 ? 9 + t : t < 6 ? 17 + t : t < 9 ? 20 + t : 32; }
__device__ __forceinline__ int imu_col_acc(int t) { return t < 3 ? 23 + t : t < 6 ? 26 + t : t < 8 ? 12 + t : 7 + t; }
__device__ __forceinline__ int imu_col_end(int t) { return t < 9 ? t : 17; }

// residual (9) and tangent Jacobian (9 x 33) of interval k by team lane t (0..9) of its team
// A: ImuEvalArgs or a view with the same fields (the persistent kernel binds `dp` by reference to its own parameter)
template <class A>
__device__ __forceinline__ void imu_eval_team(const A& a, int k, int t, const double* state) {
  using imu::D1;
  const int cc = imu_col_chain(t);
  const double* X2 = state + 7 * static_cast<int64_t>(k + 1);
  const double* X1 = state + 7 * static_cast<int64_t>(k);
  const double* V2 = state + a.dp.off_v + 3 * static_cast<int64_t>(k + 1);
  const double* V1 = state + a.dp.off_v + 3 * static_cast<int64_t>(k);
  const double* P = state + a.dp.off_imu;  // g2 b6 sf6 ts
  double s1[7];
  se3_local_column(X1, t < 3 ? 3 + t : 0, s1);
  D1 x1[7], v1[3], g2[2], b[6], sf[6], ts;
#pragma unroll
  for (int i = 0; i < 7; ++i) x1[i] = D1(X1[i], t < 3 ? s1[i] : 0.0);
#pragma unroll
  for (int i = 0; i < 3; ++i) v1[i] = D1(V1[i], 0.0);
  g2[0] = D1(P[0], 0.0);
  g2[1] = D1(P[1], 0.0);
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    b[i] = D1(P[2 + i], cc == 20 + i ? 1.0 : 0.0);
    sf[i] = D1(P[8 + i], cc == 26 + i ? 1.0 : 0.0);
  }
  ts = D1(P[14], cc == 32 ? 1.0 : 0.0);
  imu::AccelTangent at{t < 6 ? t % 3 : 0, t < 3 ? 1.0 : 0.0, (t >= 3 && t < 6) ? 1.0 : 0.0};
  imu::Pose<D1> y;
  const bool ok = imu::imu_integrate<D1>(a.buf, a.ftime[k], a.ftime[k + 1], x1, v1, g2, b, sf, ts, &y, at);
  const double* W = a.wsqrt + static_cast<int64_t>(k) * 81;
  double* rk = a.r + static_cast<int64_t>(k) * 9;
  double* Jk = a.J + static_cast<int64_t>(k) * 297;
  const bool zero_rows = a.dp.rotation_only && (t < 3 || t >= 6);  // of row t, for the v2 columns
  if (!ok) {  // no measurements: zero residual (ceres-cost-functions.h:452-455)
    if (t == 0) {
      for (int j = 0; j < 9; ++j) rk[j] = 0.0;
      a.cost[k] = 0.0;
    }
    for (int j = 0; j < 9; ++j) {
      Jk[j * 33 + cc] = 0.0;
      Jk[j * 33 + imu_col_acc(t)] = 0.0;
      Jk[j * 33 + imu_col_end(t)] = 0.0;
    }
    if (t < 9) { Jk[t * 33 + 12] = 0.0; Jk[t * 33 + 13] = 0.0; Jk[t * 33 + 14] = 0.0; }
    return;
  }
  D1 x2[7], v2[3];
#pragma unroll
  for (int i = 0; i < 7; ++i) x2[i] = D1(X2[i], 0.0);
#pragma unroll
  for (int i = 0; i < 3; ++i) v2[i] = D1(V2[i], 0.0);
  double sc = 1.0;
  // e = 0: the chain's column; e = 1, 2: end-map-only columns, their (p, v) tangents assembled from the seeds and `at`
#pragma unroll 1
  for (int e = 0; e < 3; ++e) {
    const int c = e == 0 ? cc : e == 1 ? imu_col_acc(t) : imu_col_end(t);
    imu::Pose<D1> ye = y;
    if (e > 0) {
      double s[7];
      se3_local_column(X2, c < 6 ? c : 0, s);
#pragma unroll
      for (int i = 0; i < 7; ++i) x2[i].v = c < 6 ? s[i] : 0.0;
      se3_local_column(X1, (c >= 6 && c < 9) ? c - 6 : 0, s);
      const bool tr = c >= 6 && c < 9, acc = e == 1 && t < 6;
      const imu::Vec<double> dp0{tr ? s[4] : 0.0, tr ? s[5] : 0.0, tr ? s[6] : 0.0};
      const imu::Vec<double> dv0{c == 15 ? 1.0 : 0.0, c == 16 ? 1.0 : 0.0, c == 17 ? 1.0 : 0.0};
      const imu::Vec<D1> gv = imu::gravity_vector<D1>(D1(P[0], c == 18 ? 1.0 : 0.0), D1(P[1], c == 19 ? 1.0 : 0.0));
      const imu::Vec<double> dg{gv.x.v, gv.y.v, gv.z.v};
      const double T = at.dur;
      const imu::Vec<double> dp = dp0 + imu::scale(dv0, T) - imu::scale(dg, 0.5 * T * T) +
                                  (acc ? at.dp : imu::Vec<double>{0.0, 0.0, 0.0});
      const imu::Vec<double> dv = dv0 - imu::scale(dg, T) + (acc ? at.dv : imu::Vec<double>{0.0, 0.0, 0.0});
      ye.p = {D1(y.p.x.a, dp.x), D1(y.p.y.a, dp.y), D1(y.p.z.a, dp.z)};
      ye.q = {D1(y.q.x.a, 0.0), D1(y.q.y.a, 0.0), D1(y.q.z.a, 0.0), D1(y.q.w.a, 0.0)};
      ye.v = {D1(y.v.x.a, dv.x), D1(y.v.y.a, dv.y), D1(y.v.z.a, dv.z)};
    }
    D1 raw[9];
    imu::imu_end_residual<D1>(ye, x2, v2, raw);
    // residuals_vec = (r^T W)^T  (:476-477); rotation-only switch zeroes rows 0-2 and 6-8 (:479-482)
    D1 rw[9];
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < 9; ++j) {
      double va = 0.0, vv = 0.0;
#pragma unroll
      for (int i = 0; i < 9; ++i) {
        va += raw[i].a * W[i * 9 + j];
        vv += raw[i].v * W[i * 9 + j];
      }
      const bool off = a.dp.rotation_only && (j < 3 || j >= 6);
      rw[j] = off ? D1(0.0, 0.0) : D1(va, vv);
      s += rw[j].a * rw[j].a;
    }
    if (e == 0) {  // the residual is the same on every column's pass
      double cost = 0.5 * s;
      if (a.apply_loss) {
        double rho0, rho1;
        cauchy(s, &rho0, &rho1);  // CauchyLoss(100), vicalibrator.h:133
        cost = 0.5 * rho0 * a.mult;
        sc = sqrt(rho1);
      }
      if (t == 0) {
#pragma unroll
        for (int j = 0; j < 9; ++j) rk[j] = rw[j].a * sc;
        a.cost[k] = cost;
      }
    }
    const double m = c >= 18 ? a.mask[c - 18] : 1.0;
#pragma unroll
    for (int j = 0; j < 9; ++j) Jk[j * 33 + c] = rw[j].v * sc * m;
  }
  // d r / d v2 = -W[6+i][:]  (v_end - v2 enters rows 6-8 of the raw residual): row t by team lane t
  if (t < 9) {
#pragma unroll
    for (int i = 0; i < 3; ++i) Jk[t * 33 + 12 + i] = zero_rows ? 0.0 : -W[(6 + i) * 9 + t] * sc;
  }
}

// intervals kImuTeams * task + 0..2 by one warp
template <class A>
__device__ __forceinline__ void imu_eval_warp(const A& a, int task, int lane, const double* state) {
  const int k = task * kImuTeams + lane / kImuTeam;
  if (lane < kImuTeams * kImuTeam && k < a.ni) imu_eval_team(a, k, lane % kImuTeam, state);
}

__global__ void __launch_bounds__(32 * kImuWarps) imu_eval_kernel(ImuEvalArgs a) {
  const int task = blockIdx.x * kImuWarps + (threadIdx.x >> 5);
  if (task * kImuTeams >= a.ni || a.ctl->done) return;
  imu_eval_warp(a, task, threadIdx.x & 31, a.states[a.which ? 1 - a.ctl->cur : a.ctl->cur]);
}

// ---------------------------------------------------------------- IMU -> frame blocks
struct ImuAccArgs {
  DevProblem dp;
  const Ctl* ctl;
  int which;
  const double *r, *J;  // [ni][9], [ni][9*33] (loss-corrected, masked)
  Blocks outs[2];
  double* Cg;  // [ni][kImuCgStride]
  int ni;
};
// local column layout of an interval: frame k (pose1 6, v1 3) = 0..8 | frame k+1 (pose2 6, v2 3) = 9..17 | globals 18..32
__device__ __forceinline__ int imu_local_col(int c) {
  return c < 6 ? 6 + c : c < 9 ? 15 + (c - 6) : c < 15 ? (c - 9) : c < 18 ? 12 + (c - 15) : c;
}
// frame f by a group of NT threads: interval f-1 (f is its second frame) and interval f (f is its first frame).
// Jl: the group's [2][9][34] staging area ([which][row][local col 0..32, 33 = residual]); SYNC: the group's barrier
template <int NT, class A, class SYNC>
__device__ __forceinline__ void imu_accumulate_frame(const A& a, const Blocks& out, int f, int tid, double (*Jl)[9][34],
                                                     SYNC sync) {
  const int G = a.dp.G, nf = a.dp.n_frames, io = a.dp.imu_goff;
  const bool hasP = f > 0, hasN = f < nf - 1;
  double* Bf = out.B + static_cast<int64_t>(f) * 81;
  double* Uf = out.U + static_cast<int64_t>(f) * 81;
  double* Ef = out.E + static_cast<int64_t>(f) * 9 * G;
  double* gf = out.gf + static_cast<int64_t>(f) * 9;
  constexpr int kIn = 2 * 9 * 34, kOut = 81 + 81 + 135 + 9 + 135;
  constexpr int kItIn = (kIn + NT - 1) / NT, kItOut = (kOut + NT - 1) / NT;
  // every global load first (the two intervals' Jacobians and the entries the reprojection build left in B and the
  // gradient), then the arithmetic: a load-use loop would pay one memory round trip per iteration
  double vin[kItIn], old[kItOut];
#pragma unroll
  for (int it = 0; it < kItIn; ++it) {
    const int e = tid + it * NT;
    const int which = e / (9 * 34), row = (e / 34) % 9, c = e % 34;
    const int k = which == 0 ? f - 1 : f;
    vin[it] = 0.0;
    if (e < kIn && k >= 0 && k < a.ni)
      vin[it] = c < 33 ? a.J[static_cast<int64_t>(k) * 297 + row * 33 + imu_local_col(c)] : a.r[static_cast<int64_t>(k) * 9 + row];
  }
#pragma unroll
  for (int it = 0; it < kItOut; ++it) {
    const int e = tid + it * NT;
    old[it] = e < 81 ? Bf[e] : (e >= 297 && e < 306) ? gf[e - 297] : 0.0;
  }
#pragma unroll
  for (int it = 0; it < kItIn; ++it) {
    const int e = tid + it * NT;
    if (e < kIn) Jl[e / (9 * 34)][(e / 34) % 9][e % 34] = vin[it];
  }
  sync();
  const double m = a.dp.imu_mult;
  // B (81) | U (81) | E imu columns (9*15) | g (9) | Cg of interval f (120 + 15)
#pragma unroll
  for (int it = 0; it < kItOut; ++it) {
    const int e = tid + it * NT;
    if (e >= kOut) break;
    if (e < 81) {
      const int i = e / 9, j = e % 9;
      double s = 0.0;
#pragma unroll
      for (int row = 0; row < 9; ++row) {
        if (hasP) s += Jl[0][row][9 + i] * Jl[0][row][9 + j];
        if (hasN) s += Jl[1][row][i] * Jl[1][row][j];
      }
      Bf[e] = old[it] + s * m;
    } else if (e < 162) {
      const int i = (e - 81) / 9, j = (e - 81) % 9;  // U[f] = H[f-1, f] = J1(f-1)^T J2(f-1)
      double s = 0.0;
      if (hasP) {
#pragma unroll
        for (int row = 0; row < 9; ++row) s += Jl[0][row][i] * Jl[0][row][9 + j];
      }
      Uf[e - 81] = s * m;
    } else if (e < 297) {
      const int i = (e - 162) / 15, j = (e - 162) % 15;
      double s = 0.0;
#pragma unroll
      for (int row = 0; row < 9; ++row) {
        if (hasP) s += Jl[0][row][9 + i] * Jl[0][row][18 + j];
        if (hasN) s += Jl[1][row][i] * Jl[1][row][18 + j];
      }
      Ef[i * G + io + j] = s * m;
    } else if (e < 306) {
      const int i = e - 297;
      double s = 0.0;
#pragma unroll
      for (int row = 0; row < 9; ++row) {
        if (hasP) s += Jl[0][row][9 + i] * Jl[0][row][33];
        if (hasN) s += Jl[1][row][i] * Jl[1][row][33];
      }
      gf[i] = old[it] + s * m;
    } else if (hasN) {
      const int q = e - 306;  // packed lower triangle of the 15x15 global block, then gradient
      double s = 0.0;
      if (q < 120) {
        int i = 0;
        while ((i + 1) * (i + 2) / 2 <= q) ++i;
        const int j = q - i * (i + 1) / 2;
#pragma unroll
        for (int row = 0; row < 9; ++row) s += Jl[1][row][18 + i] * Jl[1][row][18 + j];
      } else {
#pragma unroll
        for (int row = 0; row < 9; ++row) s += Jl[1][row][18 + (q - 120)] * Jl[1][row][33];
      }
      a.Cg[static_cast<int64_t>(f) * kImuCgStride + q] = s * m;
    }
  }
}
__global__ void __launch_bounds__(128) imu_accumulate_kernel(ImuAccArgs a) {
  __shared__ double Jl[2][9][34];
  if (a.ctl->done) return;
  imu_accumulate_frame<128>(a, a.outs[a.which ? 1 - a.ctl->cur : a.ctl->cur], blockIdx.x, threadIdx.x, Jl, [] { __syncthreads(); });
}

}  // namespace vc
