// UpdateImuWeights on the device: a team of 16 lanes per frame interval (two teams per warp), small dense
// matrices in shared memory, products shared across the lanes of the team.
//
// Reference being reproduced (formulas AS WRITTEN, approximations included):
//   ViCalibrator::UpdateImuWeights                        vicalibrator.h:723-799
//   ImuResidualT::IntegratePose / GetPoseDerivative / IntegrateImu / IntegrateResidual
//                                                         types.h:330-378, 380-425, 427-595, 611-687
//   dLog_dq, dqExp_dw, dq1q2_dq2, dq1q2_dq1, dqx_dq, dt1t2_dt1, dLog_dSE3
//                                                         vicalibrator-utils.h:106-154,187-202,214-230,234-274,307-434
// Only values that reach an output are computed (SURVEY App. C): per IMU step
//   C <- A C A^T + G R G^T,  A = d y/d y0 (10x10), G = d y/d b (10x6) of the full RK4 step,
// then info = (Jt C Jt^T)^-1 and W = sqrtm(info): with P = Jt C Jt^T = V L V^T (cyclic Jacobi), W = V L^-1/2 V^T —
// the principal root Eigen's MatrixFunctions sqrt returns for the symmetric positive definite info matrix, without
// forming the inverse.
#pragma once
#include "vc_imu_math.cuh"
#include "vc_internal.h"

namespace vc {
namespace wts {

using imu::Meas;
using imu::Pose;
using imu::Quat;
using imu::Vec;

__device__ inline double powi(double x, int y) {  // vicalibrator-utils.h:69-82
  double r = x;
  for (int i = 1; i < y; ++i) r *= x;
  return r;
}

// vicalibrator-utils.h:234-254 (3x4, row-major, ld = 4)
__device__ inline void dqx_dq(Quat<double> q, Vec<double> v, double* o, int ld) {
  const double x = v.x, y = v.y, z = v.z;
  const double s1 = 2 * q.x * y, s2 = 2 * q.y * y, s3 = 2 * q.x * x, s4 = 2 * q.z * x, s5 = 2 * q.y * z, s6 = 2 * q.z * z;
  o[0] = s2 + s6; o[1] = s1 - 4 * q.y * x + 2 * q.w * z; o[2] = 2 * q.x * z - 2 * q.w * y - 4 * q.z * x; o[3] = s5 - 2 * q.z * y;
  o[ld + 0] = 2 * q.y * x - 4 * q.x * y - 2 * q.w * z; o[ld + 1] = s3 + s6; o[ld + 2] = s5 + 2 * q.w * x - 4 * q.z * y; o[ld + 3] = s4 - 2 * q.x * z;
  o[2 * ld + 0] = s4 + 2 * q.w * y - 4 * q.x * z; o[2 * ld + 1] = 2 * q.z * y - 2 * q.w * x - 4 * q.y * z; o[2 * ld + 2] = s2 + s3; o[2 * ld + 3] = s1 - 2 * q.y * x;
}
// vicalibrator-utils.h:214-220 / 224-230 (4x4 with leading dimension ld)
__device__ inline void dq1q2_dq2(Quat<double> q1, double* o, int ld) {
  o[0] = q1.w; o[1] = -q1.z; o[2] = q1.y; o[3] = q1.x;
  o[ld] = q1.z; o[ld + 1] = q1.w; o[ld + 2] = -q1.x; o[ld + 3] = q1.y;
  o[2 * ld] = -q1.y; o[2 * ld + 1] = q1.x; o[2 * ld + 2] = q1.w; o[2 * ld + 3] = q1.z;
  o[3 * ld] = -q1.x; o[3 * ld + 1] = -q1.y; o[3 * ld + 2] = -q1.z; o[3 * ld + 3] = q1.w;
}
__device__ inline void dq1q2_dq1(Quat<double> q2, double* o, int ld) {
  o[0] = q2.w; o[1] = q2.z; o[2] = -q2.y; o[3] = q2.x;
  o[ld] = -q2.z; o[ld + 1] = q2.w; o[ld + 2] = q2.x; o[ld + 3] = q2.y;
  o[2 * ld] = q2.y; o[2 * ld + 1] = -q2.x; o[2 * ld + 2] = q2.w; o[2 * ld + 3] = q2.z;
  o[3 * ld] = -q2.x; o[3 * ld + 1] = -q2.y; o[3 * ld + 2] = -q2.z; o[3 * ld + 3] = q2.w;
}
// vicalibrator-utils.h:187-202 (4x3)
__device__ inline void dqExp_dw(Vec<double> w, double o[12]) {
  const double t = sqrt(w.x * w.x + w.y * w.y + w.z * w.z);
  const double s1 = t / 20 - 1, s2 = powi(t, 2) / 48 - 0.5;
  const double s3 = (s1 * w.y * w.z) / 24, s4 = (s1 * w.x * w.z) / 24, s5 = (s1 * w.x * w.y) / 24, s6 = powi(t, 2);
  o[0] = (s1 * powi(w.x, 2)) / 24 - s6 / 48 + 0.5; o[1] = s5; o[2] = s4;
  o[3] = s5; o[4] = (s1 * powi(w.y, 2)) / 24 - s6 / 48 + 0.5; o[5] = s3;
  o[6] = s4; o[7] = s3; o[8] = (s1 * powi(w.z, 2)) / 24 - s6 / 48 + 0.5;
  o[9] = (s2 * w.x) / 2; o[10] = (s2 * w.y) / 2; o[11] = (s2 * w.z) / 2;
}
// vicalibrator-utils.h:106-154 (3x4)
__device__ inline void dLog_dq(Quat<double> q, double o[12]) {
  const double x = q.x, y = q.y, z = q.z, w = q.w;
  const double vsq = powi(x, 2) + powi(y, 2) + powi(z, 2), vn = sqrt(vsq);
  if (vn < 1e-9) {
    const double s1 = 2 * vsq, s2 = 1.0 / powi(w, 3), s3 = (3 * s1) / powi(w, 4) - 2 / powi(w, 2), s4 = 2 / w;
    o[0] = -4 * s2 * powi(x, 2) + s4 - s1 * s2; o[1] = -4 * x * y * s2; o[2] = -4 * x * z * s2; o[3] = x * s3;
    o[4] = -4 * x * y * s2; o[5] = -4 * s2 * powi(y, 2) + s4 - s1 * s2; o[6] = -4 * y * z * s2; o[7] = y * s3;
    o[8] = -4 * x * z * s2; o[9] = -4 * y * z * s2; o[10] = -4 * s2 * powi(z, 2) + s4 - s1 * s2; o[11] = z * s3;
  } else {
    const double s1 = vsq, s2 = 1 / (s1 / powi(w, 2) + 1), s3 = atan(sqrt(s1) / w), s4 = 1 / pow(s1, 1.5), s5 = 1 / s1,
                 s6 = 1 / w, s7 = (2 * s3) / sqrt(s1);
    const double s8 = 2 * y * z * s2 * s5 * s6 - 2 * y * z * s3 * s4;
    const double s9 = 2 * x * z * s2 * s5 * s6 - 2 * x * z * s3 * s4;
    const double s10 = 2 * x * y * s2 * s5 * s6 - 2 * x * y * s3 * s4;
    o[0] = s7 - 2 * powi(x, 2) * s3 * s4 + 2 * powi(x, 2) * s2 * s5 * s6; o[1] = s10; o[2] = s9; o[3] = -(2 * x * s2) / powi(w, 2);
    o[4] = s10; o[5] = s7 - 2 * powi(y, 2) * s3 * s4 + 2 * powi(y, 2) * s2 * s5 * s6; o[6] = s8; o[7] = -(2 * y * s2) / powi(w, 2);
    o[8] = s9; o[9] = s8; o[10] = s7 - 2 * powi(z, 2) * s3 * s4 + 2 * powi(z, 2) * s2 * s5 * s6; o[11] = -(2 * z * s2) / powi(w, 2);
  }
}

// vicalibrator-utils.h:307-434: dlog (6x7) for t = (q, tr); 7-vector = (translation 3, quaternion 4)
__device__ inline void dLog_dSE3(Quat<double> q, Vec<double> tr, double dlog[42]) {
  double dw_dq[12];
  dLog_dq(q, dw_dq);
  const double x = tr.x, y = tr.y, z = tr.z;
  double theta;
  const Vec<double> w = imu::so3_log<double>(q, &theta);
  const double wx = w.x, wy = w.y, wz = w.z;
  const bool close_to_zero = fabs(theta) < kSophusEps;
  const double O[9] = {0, -wz, wy, wz, 0, -wx, -wy, wx, 0};
  double O2[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0;
      for (int k = 0; k < 3; ++k) s += O[i * 3 + k] * O[k * 3 + j];
      O2[i * 3 + j] = s;
    }
  const double cc = close_to_zero ? 1. / 12. : (1.0 - theta / (2.0 * tan(theta / 2.0))) / (theta * theta);
  for (int i = 0; i < 42; ++i) dlog[i] = 0.0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) dlog[i * 7 + j] = (i == j ? 1.0 : 0.0) - 0.5 * O[i * 3 + j] + cc * O2[i * 3 + j];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j) dlog[(3 + i) * 7 + 3 + j] = dw_dq[i * 4 + j];
  double d[9];
  if (close_to_zero) {
    const double div_12 = 1. / 12, div_6 = 1. / 6.;
    const double wx_x = wx * x, wy_x = wy * x, wz_x = wz * x, wx_y = wx * y, wy_y = wy * y, wz_y = wz * y, wx_z = wx * z,
                 wy_z = wy * z, wz_z = wz * z;
    d[0] = div_12 * (wy_y + wz_z); d[1] = div_12 * wx_y - div_6 * wy_x - 0.5 * z; d[2] = 0.5 * y - div_6 * wz_x + div_12 * wx_z;
    d[3] = 0.5 * z + div_12 * wy_x - div_6 * wx_y; d[4] = div_12 * (wx_x + wz_z); d[5] = div_12 * wy_z - div_6 * wz_y - 0.5 * x;
    d[6] = div_12 * wz_x - div_6 * wx_z - 0.5 * y; d[7] = 0.5 * x + div_12 * wz_y - div_6 * wy_z; d[8] = div_12 * (wx_x * wy_y);
  } else {
    const double s1 = powi(wx, 2) + powi(wy, 2) + powi(wz, 2);
    const double s2 = tan(sqrt(s1) / 2);
    const double s3 = sqrt(s1) / (2 * s2) - 1;
    const double s4 = wz / (2 * sqrt(s1) * s2) - (wz * (powi(s2, 2) + 1)) / (4 * powi(s2, 2));
    const double s5 = wy / (2 * sqrt(s1) * s2) - (wy * (powi(s2, 2) + 1)) / (4 * powi(s2, 2));
    const double s6 = wx / (2 * sqrt(s1) * s2) - (wx * (powi(s2, 2) + 1)) / (4 * powi(s2, 2));
    const double s7 = 1 / s1, s8 = 1 / powi(s1, 2);
    const double s9 = powi(wx, 2) + powi(wy, 2), s10 = powi(wx, 2) + powi(wz, 2), s11 = powi(wy, 2) + powi(wz, 2);
    const double s12 = 2 * s3 * s8 * wx * wy * wz;
    const double s13 = -2 * s3 * s8 * wy * powi(wz, 2) + s4 * s7 * wy * wz + s3 * s7 * wy;
    const double s14 = -2 * s3 * s8 * wx * powi(wz, 2) + s4 * s7 * wx * wz + s3 * s7 * wx;
    const double s15 = -2 * s3 * s8 * wz * powi(wy, 2) + s5 * s7 * wz * wy + s3 * s7 * wz;
    const double s16 = -2 * s3 * s8 * wz * powi(wx, 2) + s6 * s7 * wz * wx + s3 * s7 * wz;
    const double s17 = -2 * s3 * s8 * wx * powi(wy, 2) + s5 * s7 * wx * wy + s3 * s7 * wx;
    const double s18 = -2 * s3 * s8 * wy * powi(wx, 2) + s6 * s7 * wy * wx + s3 * s7 * wy;
    const double s19 = 2 * s3 * s7 * wy, s20 = 2 * s3 * s7 * wx;
    d[0] = x * (s6 * s7 * s11 - 2 * s3 * s8 * s11 * wx) - s18 * y - s16 * z;
    d[1] = x * (s19 + s5 * s7 * s11 - 2 * s3 * s8 * s11 * wy) - s17 * y - z * (s5 * s7 * wx * wz - 2 * s3 * s8 * wx * wy * wz + 0.5);
    d[2] = x * (s4 * s7 * s11 + 2 * s3 * s7 * wz - 2 * s3 * s8 * s11 * wz) - s14 * z + y * (s12 - s4 * s7 * wx * wy + 0.5);
    d[3] = y * (s20 + s6 * s7 * s10 - 2 * s3 * s8 * s10 * wx) - s18 * x + z * (s12 - s6 * s7 * wy * wz + 0.5);
    d[4] = y * (s5 * s7 * s10 - 2 * s3 * s8 * s10 * wy) - s17 * x - s15 * z;
    d[5] = y * (s4 * s7 * s10 + 2 * s3 * s7 * wz - 2 * s3 * s8 * s10 * wz) - s13 * z - x * (s4 * s7 * wx * wy - s12 + 0.5);
    d[6] = z * (s20 + s6 * s7 * s9 - 2 * s3 * s8 * s9 * wx) - s16 * x - y * (s6 * s7 * wy * wz - s12 + 0.5);
    d[7] = z * (s19 + s5 * s7 * s9 - 2 * s3 * s8 * s9 * wy) - s15 * y + x * (s12 - s5 * s7 * wx * wz + 0.5);
    d[8] = z * (s4 * s7 * s9 - 2 * s3 * s8 * s9 * wz) - s14 * x - s13 * y;
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j) {
      double s = 0;
      for (int k = 0; k < 3; ++k) s += d[i * 3 + k] * dw_dq[k * 4 + j];
      dlog[i * 7 + 3 + j] = s;
    }
}

// ---- team layout --------------------------------------------------------------------------------------------
// One interval is worked on by a TEAM of 16 lanes (the RK4 Jacobian [dy/dy0 (10) | dy/db (6)] has 16 columns: one
// per lane); a warp carries two teams.  Every small dense product is spread over the 16 lanes of the team through
// the team's shared-memory workspace; nothing runs on a single lane except the scalar formula tables of dLog_dSE3,
// which lane 0 of the team writes straight into shared memory (no local-memory arrays, no stack frame).
constexpr int kTeam = 16;
struct Work {
  double C[100], A[100], Gm[60], t1[100], t2[100];
  double rot[8];  // (c, s) of the four rotations of a Jacobi round
  int rpq[8];     // their index pairs
};

// out[R x C] = A[R x K] * op(B); transB: B is stored [C x K].  Caller synchronises.
__device__ __forceinline__ void tmm(double* out, const double* A, const double* B, int R, int K, int C, int tl,
                                    bool transB = false) {
  for (int e = tl; e < R * C; e += kTeam) {
    const int r = e / C, c = e - r * C;
    double s = 0.0;
    for (int k = 0; k < K; ++k) s += A[r * K + k] * (transB ? B[c * K + k] : B[k * C + c]);
    out[e] = s;
  }
}

// Jacobian pieces of one RK4 stage (types.h:380-425), computed by every lane (all lanes need all of them)
struct StageJac {
  double R[9];    // dw/dbg = da/dba = R(q)
  double Dw[12];  // dw/dq = dqx_dq(q, zg) + dqx_dq(q, bg)   (unscaled measurements, as the reference)
  double Da[12];  // da/dq = dqx_dq(q, za) + dqx_dq(q, ba)
};
__device__ __forceinline__ void stage_jac(const Pose<double>& y, const Meas<double>& z0, const Meas<double>& z1, Vec<double> bg,
                                          Vec<double> ba, double dt, StageJac* J) {
  const double alpha = (z1.time - (z0.time + dt)) / (z1.time - z0.time);
  const Vec<double> zg = imu::scale(z0.w, alpha) + imu::scale(z1.w, 1.0 - alpha);
  const Vec<double> za = imu::scale(z0.a, alpha) + imu::scale(z1.a, 1.0 - alpha);
  qmat(Q4{y.q.x, y.q.y, y.q.z, y.q.w}, J->R);
  dqx_dq(y.q, zg + bg, J->Dw, 4);
  dqx_dq(y.q, za + ba, J->Da, 4);
}
// column j of the total derivative of this stage's k (9) w.r.t. [y0 (10) | b (6)]:
//   T_j = dk_db[:, j-10] + dk_dy * col_j        (types.h:466-467 and the analogous lines per stage)
__device__ __forceinline__ void stage_T(const double col[10], int j, const StageJac& J, double T[9]) {
  T[0] = col[7]; T[1] = col[8]; T[2] = col[9];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    T[3 + i] = J.Dw[i * 4] * col[3] + J.Dw[i * 4 + 1] * col[4] + J.Dw[i * 4 + 2] * col[5] + J.Dw[i * 4 + 3] * col[6];
    T[6 + i] = J.Da[i * 4] * col[3] + J.Da[i * 4 + 1] * col[4] + J.Da[i * 4 + 2] * col[5] + J.Da[i * 4 + 3] * col[6];
  }
  // bias columns: dk_db = [0; R 0; 0 R]  (types.h:410-411)
  const double sel_g = (j >= 10 && j < 13) ? 1.0 : 0.0, sel_a = j >= 13 ? 1.0 : 0.0;
  const int bc = j >= 13 ? j - 13 : (j >= 10 ? j - 10 : 0);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double rv = bc == 0 ? J.R[i * 3] : (bc == 1 ? J.R[i * 3 + 1] : J.R[i * 3 + 2]);
    T[3 + i] += sel_g * rv;
    T[6 + i] += sel_a * rv;
  }
}
// IntegratePose(y0, k, h) with its Jacobians folded into column j:
//   col_j <- dy_dy[:, j] (direct dependence on y0; zero for the bias columns) + dy_dk * T_j   (types.h:330-378)
__device__ __forceinline__ Pose<double> integrate_push(const Pose<double>& y0, const double k[9], double h, const double T[9], int j,
                                                       double col[10]) {
  const Vec<double> wdt{k[3] * h, k[4] * h, k[5] * h};
  const Quat<double> r = imu::so3_exp<double>(wdt);
  double a[16], e[12];
  dq1q2_dq1(y0.q, a, 4);
  dqExp_dw(wdt, e);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    col[i] = h * T[i] + (j == i ? 1.0 : 0.0);
    col[7 + i] = h * T[6 + i] + (j == 7 + i ? 1.0 : 0.0);
  }
  // dq1q2_dq2(r)[:, j-3] for the quaternion columns of y0 (vicalibrator-utils.h:214-220)
  const int jq = j - 3;
  const double Qc[4] = {jq == 0 ? r.w : jq == 1 ? -r.z : jq == 2 ? r.y : r.x,
                        jq == 0 ? r.z : jq == 1 ? r.w : jq == 2 ? -r.x : r.y,
                        jq == 0 ? -r.y : jq == 1 ? r.x : jq == 2 ? r.w : r.z,
                        jq == 0 ? -r.x : jq == 1 ? -r.y : jq == 2 ? -r.z : r.w};
  const bool isq = j >= 3 && j < 7;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    double s = 0.0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      double q = 0.0;
#pragma unroll
      for (int m = 0; m < 4; ++m) q += a[i * 4 + m] * e[m * 3 + c];
      s += q * h * T[3 + c];
    }
    col[3 + i] = s + (isq ? Qc[i] : 0.0);
  }
  return imu::integrate_pose<double>(y0, k, h);
}

// IntegrateImu, Jacobian + covariance branch (types.h:427-595): C <- A C A^T + G R G^T.
// Team lane j carries column j of [dy/dy0 (10) | dy/db (6)] in registers through the four RK stages.  `on` is
// team-uniform: a team whose interval is finished (or empty) idles through the barriers of its warp mate.
__device__ __forceinline__ Pose<double> integrate_imu_cov(const Pose<double>& pose, const Meas<double>& z0, const Meas<double>& z1,
                                                          Vec<double> bg, Vec<double> ba, const double sf[6], Vec<double> g,
                                                          double sg2, double sa2, Work* W, int j, bool on) {
  const double dt = z1.time - z0.time;
  on = on && dt != 0;  // degenerate step: identity map (the reference leaves its outputs untouched)
  Pose<double> res = pose;
  if (on) {
    double col[10], tot[9], T[9], k1[9], k2[9], k3[9], k4[9];
#pragma unroll
    for (int i = 0; i < 10; ++i) col[i] = (j == i) ? 1.0 : 0.0;  // dy_dy0 = I, dy_db = 0
    StageJac J;
    imu::pose_derivative<double>(pose, g, z0, z1, bg, ba, sf, 0.0, k1);
    stage_jac(pose, z0, z1, bg, ba, 0.0, &J);
    stage_T(col, j, J, T);
#pragma unroll
    for (int i = 0; i < 9; ++i) tot[i] = T[i];
    const Pose<double> y1 = integrate_push(pose, k1, dt * 0.5, T, j, col);
    imu::pose_derivative<double>(y1, g, z0, z1, bg, ba, sf, dt / 2, k2);
    stage_jac(y1, z0, z1, bg, ba, dt / 2, &J);
    stage_T(col, j, J, T);
#pragma unroll
    for (int i = 0; i < 9; ++i) tot[i] += 2.0 * T[i];
    const Pose<double> y2 = integrate_push(pose, k2, dt * 0.5, T, j, col);
    imu::pose_derivative<double>(y2, g, z0, z1, bg, ba, sf, dt / 2, k3);
    stage_jac(y2, z0, z1, bg, ba, dt / 2, &J);
    stage_T(col, j, J, T);
#pragma unroll
    for (int i = 0; i < 9; ++i) tot[i] += 2.0 * T[i];
    const Pose<double> y3 = integrate_push(pose, k3, dt, T, j, col);
    imu::pose_derivative<double>(y3, g, z0, z1, bg, ba, sf, dt, k4);
    stage_jac(y3, z0, z1, bg, ba, dt, &J);
    stage_T(col, j, J, T);
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      tot[i] += T[i];
      k1[i] = k1[i] + 2 * k2[i] + 2 * k3[i] + k4[i];
    }
    res = integrate_push(pose, k1, dt / 6.0, tot, j, col);
    if (j < 10) {
#pragma unroll
      for (int i = 0; i < 10; ++i) W->A[i * 10 + j] = col[i];
    } else {
#pragma unroll
      for (int i = 0; i < 10; ++i) W->Gm[i * 6 + (j - 10)] = col[i];
    }
  }
  __syncwarp();
  if (on) tmm(W->t1, W->A, W->C, 10, 10, 10, j);
  __syncwarp();
  if (on) tmm(W->t2, W->t1, W->A, 10, 10, 10, j, true);
  __syncwarp();
  if (on)
    for (int e = j; e < 100; e += kTeam) {
      const int r = e / 10, c = e - r * 10;
      double s = 0.0;
#pragma unroll
      for (int q = 0; q < 6; ++q) s += W->Gm[r * 6 + q] * (q < 3 ? sg2 : sa2) * W->Gm[c * 6 + q];
      W->C[e] = W->t2[e] + s;
    }
  __syncwarp();
  return res;
}

struct WeightArgs {
  DevProblem dp;
  imu::ImuBuf buf;
  const Ctl* ctl;
  const double* states[2];
  const double* ftime;
  double* wsqrt;
  int ni;
  double sigma_g, sigma_a;
  int deferred;  // 1: the update the persistent solve kernel would have run for the last iteration (ignores `done`)
};
constexpr int kWtWarps = 4;                              // warps per CTA
constexpr int kWtTeams = kWtWarps * (32 / kTeam);        // intervals per CTA

// The weights of one interval: everything after the covariance chain (vicalibrator.h:755-796).  Team-collective;
// `on` team-uniform.  Writes the 9x9 weight_sqrt_ to `out` (left untouched when the information matrix is singular).
// `vec` holds the interval's eigenvectors from its last update (all NaN: none, start from the identity); the
// eigen-decomposition starts from them and leaves its own there.
__device__ __forceinline__ void weight_from_cov(const Pose<double>& y, const double* X2, Work* W, int tl, bool on, double* out,
                                                double* vec) {
  // t12 = T_end * T_2w, T_2w = T_w2^-1
  const Quat<double> q2i = imu::qconj(Quat<double>{X2[0], X2[1], X2[2], X2[3]});
  const Vec<double> t2 = imu::qrot(q2i, Vec<double>{X2[4], X2[5], X2[6]});
  const Vec<double> t2i{-t2.x, -t2.y, -t2.z};
  const Quat<double> q12 = imu::qmul(y.q, q2i);
  const Vec<double> t12 = y.p + imu::qrot(y.q, t2i);
  // Jt (9x10) = [dLog_dSE3(t12) * dt1t2_dt1(T_end, T_2w), 0; 0, I3]   (vicalibrator.h:763-781)
  double* dlog = W->t1;        // 42
  double* dmul = W->t1 + 42;   // 49
  double* Jt = W->t2;          // 90
  if (on) {
    for (int e = tl; e < 49; e += kTeam) dmul[e] = (e % 8 == 0 && e < 3 * 8) ? 1.0 : 0.0;  // identity in the 3x3 corner
    for (int e = tl; e < 90; e += kTeam) Jt[e] = (e == 67 || e == 78 || e == 89) ? 1.0 : 0.0;  // rows 6-8: [0 | I3]
  }
  __syncwarp();
  if (on && tl == 0) dLog_dSE3(q12, t12, dlog);
  if (on && tl == 1) {
    dqx_dq(y.q, t2i, dmul + 3, 7);          // block(0,3) = dqx_dq(t1.q, t2.translation)
    dq1q2_dq1(q2i, dmul + 3 * 7 + 3, 7);    // block(3,3) = dq1q2_dq1(t2.q)
  }
  __syncwarp();
  if (on)
    for (int e = tl; e < 42; e += kTeam) {
      const int i = e / 7, jj = e - i * 7;
      double s = 0.0;
#pragma unroll
      for (int q = 0; q < 7; ++q) s += dlog[i * 7 + q] * dmul[q * 7 + jj];
      Jt[i * 10 + jj] = s;
    }
  __syncwarp();
  // P = Jt C Jt^T (9x9): tmp = Jt C in t1, P in A
  if (on) tmm(W->t1, Jt, W->C, 9, 10, 10, tl);
  __syncwarp();
  double* A = W->A;   // 81: P, then its eigenvalues on the diagonal
  double* V = W->C;   // 81: eigenvectors (the covariance chain is done with C)
  if (on) tmm(A, W->t1, Jt, 9, 10, 9, tl, true);
  __syncwarp();
  // info = P^-1, weight_sqrt = sqrtm(info) (vicalibrator.h:783-796) = V diag(lambda^-1/2) V^T with P = V diag(lambda) V^T:
  // one cyclic Jacobi eigen-decomposition of the symmetrised P (no explicit inverse).  Round r of a sweep holds the
  // four disjoint pairs {i, j}, i + j = r (mod 9), i < j; their rotations are computed from the same matrix by four
  // lanes and applied together (columns of A and V, then rows of A).
  // Warm start: W does not depend on which orthogonal V diagonalises P, so the sweeps start from the interval's
  // eigenvectors of its last update, V_prev, with A = V_prev^T sym(P) V_prev — nearly diagonal when the state moved
  // little.  Without them (NaN: after an upload, a weights upload, a flag change, at the start of a solve) V starts as
  // the identity, and the products below are exact: A = sym(P) bit for bit.
  bool cold = false;
  if (on)
    for (int e = tl; e < 81; e += kTeam) {
      const double v = vec[e];
      cold = cold || v != v;
      V[e] = v;
    }
  cold = ((__ballot_sync(0xffffffffu, cold) >> (threadIdx.x & 16)) & 0xffffu) != 0;  // any lane of this team
  if (on && cold)
    for (int e = tl; e < 81; e += kTeam) V[e] = (e % 10 == 0) ? 1.0 : 0.0;
  __syncwarp();
  if (on)  // t1 = sym(P) V
    for (int e = tl; e < 81; e += kTeam) {
      const int r = e / 9, c = e - r * 9;
      double s = 0.0;
      for (int k = 0; k < 9; ++k) s += 0.5 * (A[r * 9 + k] + A[k * 9 + r]) * V[k * 9 + c];
      W->t1[e] = s;
    }
  __syncwarp();
  if (on)  // A = V^T t1, its upper triangle mirrored
    for (int e = tl; e < 81; e += kTeam) {
      const int r = e / 9, c = e - r * 9;
      if (c >= r) {
        double s = 0.0;
        for (int k = 0; k < 9; ++k) s += V[k * 9 + r] * W->t1[k * 9 + c];
        W->t2[r * 9 + c] = s;
        W->t2[c * 9 + r] = s;
      }
    }
  __syncwarp();
  A = W->t2;
  for (int sweep = 0; sweep < 40; ++sweep) {
    double off = 0.0, dg = 0.0;
    if (on) {
#pragma unroll
      for (int i = 0; i < 9; ++i) {
        dg += A[i * 9 + i] * A[i * 9 + i];
#pragma unroll
        for (int jj = i + 1; jj < 9; ++jj) off += A[i * 9 + jj] * A[i * 9 + jj];
      }
    }
    const bool conv = !on || off <= 1e-30 * dg;
    if (__all_sync(0xffffffffu, conv)) break;
    for (int r = 0; r < 9; ++r) {
      if (on && !conv && tl < 4) {
        // pair number tl of round r: i runs over the residues with i < (r - i) mod 9
        int cnt = 0, pi = 0, qi = 0;
#pragma unroll
        for (int i = 0; i < 9; ++i) {
          const int jj = (r - i + 9) % 9;
          if (i < jj) {
            if (cnt == tl) { pi = i; qi = jj; }
            ++cnt;
          }
        }
        const double apq = A[pi * 9 + qi];
        double c = 1.0, sn = 0.0;
        if (apq != 0.0) {
          const double tau = (A[qi * 9 + qi] - A[pi * 9 + pi]) / (2.0 * apq);
          const double t = (tau >= 0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
          c = rsqrt(1.0 + t * t);
          sn = t * c;
        }
        W->rot[2 * tl] = c; W->rot[2 * tl + 1] = sn;
        W->rpq[2 * tl] = pi; W->rpq[2 * tl + 1] = qi;
      }
      __syncwarp();
      if (on && !conv)
        for (int e = tl; e < 36; e += kTeam) {  // columns p, q of A and V: row k, rotation t
          const int k = e >> 2, t = e & 3, p = W->rpq[2 * t], q = W->rpq[2 * t + 1];
          const double c = W->rot[2 * t], sn = W->rot[2 * t + 1];
          const double akp = A[k * 9 + p], akq = A[k * 9 + q];
          A[k * 9 + p] = c * akp - sn * akq;
          A[k * 9 + q] = sn * akp + c * akq;
          const double vkp = V[k * 9 + p], vkq = V[k * 9 + q];
          V[k * 9 + p] = c * vkp - sn * vkq;
          V[k * 9 + q] = sn * vkp + c * vkq;
        }
      __syncwarp();
      if (on && !conv)
        for (int e = tl; e < 36; e += kTeam) {  // rows p, q of A: column k, rotation t
          const int k = e >> 2, t = e & 3, p = W->rpq[2 * t], q = W->rpq[2 * t + 1];
          const double c = W->rot[2 * t], sn = W->rot[2 * t + 1];
          const double apk = A[p * 9 + k], aqk = A[q * 9 + k];
          A[p * 9 + k] = c * apk - sn * aqk;
          A[q * 9 + k] = sn * apk + c * aqk;
        }
      __syncwarp();
    }
  }
  if (!on) return;
  for (int e = tl; e < 81; e += kTeam) vec[e] = V[e];  // the next update of this interval starts from them
  bool singular = false;
#pragma unroll
  for (int k = 0; k < 9; ++k) singular = singular || !(A[k * 9 + k] > 0.0);
  if (singular) return;
  if (tl < 9) W->t1[tl] = 1.0 / sqrt(A[tl * 9 + tl]);  // lambda^-1/2
  __syncwarp(0xffffu << (threadIdx.x & 16));  // this team only: the other one may have left
  for (int e = tl; e < 81; e += kTeam) {
    const int r = e / 9, c = e - r * 9;
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 9; ++k) s += V[r * 9 + k] * W->t1[k] * V[c * 9 + k];
    out[e] = s;
  }
}

// UpdateImuWeights for interval kk by the team of 16 lanes `tl` belongs to (kk >= ni: the team idles along)
template <class A>
__device__ __forceinline__ void imu_weights_team(const A& a, const double* state, int kk, Work* W, int tl) {
  const int ki = min(kk, a.ni - 1);  // an odd tail team shadows the last interval (never written)
  const double* X1 = state + 7 * static_cast<int64_t>(ki);
  const double* X2 = state + 7 * static_cast<int64_t>(ki + 1);
  const double* V1 = state + a.dp.off_v + 3 * static_cast<int64_t>(ki);
  const double* P = state + a.dp.off_imu;
  const double ts = P[14];
  const double t_start = a.ftime[ki], t_end = a.ftime[ki + 1];
  // measurements.size() == 0 -> continue (vicalibrator.h:731-733)
  bool on = kk < a.ni && (t_start >= a.buf.start_time + ts && t_start <= a.buf.end_time + ts) && a.buf.n > 0;
  const Vec<double> g = imu::gravity_vector<double>(P[0], P[1]);
  const Vec<double> bg{P[2], P[3], P[4]}, ba{P[5], P[6], P[7]};
  double sf[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) sf[i] = P[8 + i];
  Pose<double> y{{X1[4], X1[5], X1[6]}, {X1[0], X1[1], X1[2], X1[3]}, {V1[0], V1[1], V1[2]}};
  __syncwarp();  // the team's previous interval is done with the workspace
  for (int e = tl; e < 100; e += kTeam) W->C[e] = 0.0;
  __syncwarp();
  const double sg2 = a.sigma_g * a.sigma_g, sa2 = a.sigma_a * a.sigma_a;
  int idx = 0;
  Meas<double> prev{}, cur{};
  if (on) prev = imu::get_element<double>(a.buf, t_start, ts, &idx);
  bool more = on;
  while (__any_sync(0xffffffffu, more)) {
    const bool step = more;
    if (step) more = imu::get_next<double>(a.buf, t_end, ts, &idx, &cur);
    y = integrate_imu_cov(y, prev, cur, bg, ba, sf, g, sg2, sa2, W, tl, step);
    if (step) prev = cur;
  }
  weight_from_cov(y, X2, W, tl, on, a.wsqrt + static_cast<int64_t>(ki) * 81, a.wsqrt + static_cast<int64_t>(a.ni + ki) * 81);
}

__global__ void __launch_bounds__(32 * kWtWarps, 2) imu_weights_kernel(WeightArgs a) {
  __shared__ Work work[kWtTeams];
  const int tl = threadIdx.x & (kTeam - 1);
  const int team = threadIdx.x / kTeam;
  if (a.deferred) {
    if (!(a.ctl->iter > 0 && a.ctl->last_accepted)) return;
  } else {
    if (a.ctl->done) return;
    // a rejected step leaves the accepted state — hence the weights — unchanged
    if (a.ctl->iter > 0 && !a.ctl->last_accepted) return;
  }
  if (blockIdx.x * kWtTeams + (threadIdx.x >> 5) * (32 / kTeam) >= a.ni) return;  // whole warp past the end
  imu_weights_team(a, a.states[a.ctl->cur], blockIdx.x * kWtTeams + team, &work[team], tl);
}

}  // namespace wts
}  // namespace vc
