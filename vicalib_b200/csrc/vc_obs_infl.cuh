// Regression diagnostics of every reprojection observation (vcgpu_get_observation_influence(_batch)).  Observation i
// of camera c in frame f touches P = (frame f's 6 pose tangents | camera c's 6 + K globals), p = 12 + K <= 20.  With
// J~ = sqrt(w) J and r~ = sqrt(w) r (w = visual_mult rho'(|r|^2), the solve's SoftLOne weight), the P x P block Sigma_PP
// of the covariance and, on F (the globals whose variance is not 0.0),
//   H   = J~ Sigma_PP J~^T                      (2 x 2 leverage)
//   u   = (I -+ H)^-1 r~                         (- for an active observation, + for a removed one)
//   stud = r~ . u
//   infl = Dg^T Sigma_F^-1 Dg,  Dg = Sigma_gP J~^T u  =  a^T M_P a,  a = J~^T u,
//   M_P  = [[Q_f, Sigma_fc], [Sigma_cf, Sigma_cc]],   Q_f = Sigma_fF Sigma_F^-1 Sigma_Ff
// since Sigma_cF Sigma_F^-1 selects camera c's rows.  Four kernels:
//   infl_sgg_kernel                       Sigma_gg unscaled from the elimination's inverse, one CTA per rig;
//   view_prior_kernel (vc_view_info.cuh)  chol of the Jacobi-scaled Sigma_F = D^-1 Sigma_F D^-1 = L L^T, one CTA per rig;
//   infl_q_kernel                         Q_f = Y^T Y, Y = L^-1 D^-1 Sigma_Ff (G_F x 6), one warp per frame;
//   infl_obs_kernel                       one CTA per tile of at most kInflTile observations of one (frame, camera)
//                                         group, Sigma_PP and M_P staged in shared memory, one thread per observation.
// Every output has one owner and a fixed summation order, so a rig's bits depend on nothing else in the launch.
#pragma once
#include "vc_internal.h"
#include "vc_math.cuh"
#include "vc_view_info.cuh"

namespace vc {

constexpr int kInflTile = 64;     // observations per tile = threads per CTA
constexpr int kInflP = 20;        // P's largest size (12 + 8 intrinsics), the staged matrices' leading dimension
constexpr int kInflQWarps = 4;    // frames per CTA of infl_q_kernel
constexpr int kInflRowsPerLane = 4;  // infl_q_kernel: rows of F per lane, so G_F <= 128
constexpr int kInflMaxGF = 32 * kInflRowsPerLane;

// one rig of a launch
struct InflRig {
  DevProblem dp;              // cameras (model, K, goff), visual_mult
  const double* state;        // the accepted state buffer
  const double* mask;         // [G] the build's 0/1 mask of the globals
  const uint8_t* frame_used;  // [nf] 1 where Sigma_ff is determined (vision: an active observation sees the frame)
  const double* inv;          // the scaled inverse of the reduced system, its globals' block first
  int ldinv;
  const double* scg;          // [G] the globals' Jacobi scale
  const double* gmask;        // [G] 0: a global vcgpu_get_covariance zeroes (constant, or of an unused camera)
  double* Sgg;                // [G][G] unscaled (infl_sgg_kernel)
  const double* Sff;          // [nf][fd][fd]
  const double* Sfg;          // [nf][fd][G]
  const int32_t* fidx;        // [GF] global index of each row of F (view_prior_kernel's)
  const double* L;            // [GF][GF] chol of the Jacobi-scaled Sigma_F (view_prior_kernel)
  const double* D;            // [GF] sqrt(diag Sigma_F)
  const int* prior_ok;        // view_prior_kernel's flag
  double* Q;                  // [nf][36]
  const double* pw;           // [n][3] every observation, sorted by (camera, frame), removed ones included
  const double* pc;           // [n][2]
  const int64_t* idx;         // [n] caller index
  const uint8_t* active;      // [n]
  double *h, *stud, *infl;    // caller order, each may be null
  int64_t warp0;              // infl_q_kernel: this rig's frames are warps [warp0, warp0 + nf)
  int G, GF, fd;
  int cam_used[kMaxCams];     // 1: an active observation sees the camera
};
// one observation's outputs
struct InflOut { double h00, h01, h11, stud, infl; };

// Sigma_gg of each rig as vcgpu_get_covariance returns it: the lower triangle of the scaled inverse, unscaled by
// s_i s_j and mirrored, exact zeros outside F.  One CTA per rig.
__global__ void __launch_bounds__(256) infl_sgg_kernel(const InflRig* __restrict__ rigs) {
  const InflRig& a = rigs[blockIdx.x];
  const int G = a.G;
  for (int e = threadIdx.x; e < G * G; e += blockDim.x) {
    const int i = e / G, j = e % G, hi = max(i, j), lo = min(i, j);
    a.Sgg[e] = a.gmask[i] != 0.0 && a.gmask[j] != 0.0 ? a.scg[hi] * a.scg[lo] * a.inv[static_cast<int64_t>(hi) * a.ldinv + lo] : 0.0;
  }
}

// Q_f = Y^T Y, Y = L^-1 D^-1 Sigma_Ff, by one warp: lane l owns rows l, l + 32, ... of Y; column-oriented forward
// substitution (row j done, then every later row updated in j order), then the 21 entries of Q summed over the lanes.
__global__ void __launch_bounds__(32 * kInflQWarps) infl_q_kernel(const InflRig* __restrict__ rigs, int n_rigs, int64_t n_warps) {
  const int64_t gw = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= n_warps) return;
  int lo = 0, hi = n_rigs - 1;  // the last rig whose warp0 <= gw
  while (lo < hi) {
    const int mid = (lo + hi + 1) / 2;
    if (rigs[mid].warp0 <= gw) lo = mid;
    else hi = mid - 1;
  }
  const InflRig& a = rigs[lo];
  if (!*a.prior_ok) return;
  const int f = static_cast<int>(gw - a.warp0), GF = a.GF, G = a.G;
  const double* sfg = a.Sfg + static_cast<int64_t>(f) * a.fd * G;
  double y[kInflRowsPerLane][6];
#pragma unroll
  for (int m = 0; m < kInflRowsPerLane; ++m) {
    const int i = lane + 32 * m;
#pragma unroll
    for (int k = 0; k < 6; ++k) y[m][k] = i < GF ? sfg[static_cast<int64_t>(k) * G + a.fidx[i]] / a.D[i] : 0.0;
  }
  for (int j = 0; j < GF; ++j) {
    const int owner = j & 31, mj = j >> 5;
    double yj[6];
    const double ljj = a.L[static_cast<int64_t>(j) * GF + j];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      double v = 0.0;
#pragma unroll
      for (int m = 0; m < kInflRowsPerLane; ++m)
        if (m == mj) v = y[m][k];
      v = __shfl_sync(0xffffffffu, v, owner) / ljj;
      yj[k] = v;
    }
#pragma unroll
    for (int m = 0; m < kInflRowsPerLane; ++m) {
      const int i = lane + 32 * m;
      if (i == j) {
#pragma unroll
        for (int k = 0; k < 6; ++k) y[m][k] = yj[k];
      } else if (i > j && i < GF) {
        const double lij = a.L[static_cast<int64_t>(i) * GF + j];
#pragma unroll
        for (int k = 0; k < 6; ++k) y[m][k] -= lij * yj[k];
      }
    }
  }
  double* Q = a.Q + static_cast<int64_t>(f) * 36;
#pragma unroll
  for (int k = 0; k < 6; ++k)
#pragma unroll
    for (int l = 0; l <= k; ++l) {
      double s = 0.0;
#pragma unroll
      for (int m = 0; m < kInflRowsPerLane; ++m) s += y[m][k] * y[m][l];  // rows past G_F are 0
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) { Q[k * 6 + l] = s; Q[l * 6 + k] = s; }
    }
}

// the diagnostics of one observation: J~ and r~ with eval_obs_to_tile's expressions (the pose columns, the extrinsic
// columns as the pose row times A (times_A), the intrinsics), then H, the 2 x 2 solve and the two quadratic forms
template <int MODEL>
__device__ __forceinline__ InflOut infl_obs(const double* T, const double* cam, const double* R, const double* cmask, double vm, V3 pw,
                                            double pcu, double pcv, bool active, const double* S, const double* M) {
  constexpr int K = Cam<MODEL>::K, NP = 12 + K;
  const Q4 q{T[0], T[1], T[2], T[3]};
  const V3 t{T[4], T[5], T[6]};
  const V3 pk = qrot(qconj(q), pw - t);
  const V3 pc = mat_mul(R, pk) + V3{cam[4], cam[5], cam[6]};
  double z[2], dzp[6], dzi[2 * K];
  Cam<MODEL>::project(pc, cam + 7, z, dzp, dzi);
  const double r0 = z[0] - pcu, r1 = z[1] - pcv;
  double rho0, rho1;
  soft_l_one(r0 * r0 + r1 * r1, &rho0, &rho1);
  const double sw = sqrt(vm * rho1);
  double J[2][NP];
#pragma unroll
  for (int row = 0; row < 2; ++row) {
    const double* d = dzp + 3 * row;
    const double m0 = (d[0] * R[0] + d[1] * R[3] + d[2] * R[6]) * sw;
    const double m1 = (d[0] * R[1] + d[1] * R[4] + d[2] * R[7]) * sw;
    const double m2 = (d[0] * R[2] + d[1] * R[5] + d[2] * R[8]) * sw;
    double* o = J[row];
    o[0] = -m0;
    o[1] = -m1;
    o[2] = -m2;
    o[3] = m1 * pk.z - m2 * pk.y;
    o[4] = m2 * pk.x - m0 * pk.z;
    o[5] = m0 * pk.y - m1 * pk.x;
#pragma unroll
    for (int e = 0; e < 6; ++e) o[6 + e] = cmask[e] * times_A(o, e, R);
#pragma unroll
    for (int k = 0; k < K; ++k) o[12 + k] = dzi[row * K + k] * sw * cmask[6 + k];
  }
  const double rt0 = r0 * sw, rt1 = r1 * sw;
  // H = J~ Sigma_PP J~^T, row k of Sigma_PP at a time
  double h00 = 0.0, h01 = 0.0, h11 = 0.0;
#pragma unroll
  for (int k = 0; k < NP; ++k) {
    double s0 = 0.0, s1 = 0.0;
#pragma unroll
    for (int j = 0; j < NP; ++j) {
      const double sk = S[k * kInflP + j];
      s0 += sk * J[0][j];
      s1 += sk * J[1][j];
    }
    h00 += J[0][k] * s0;
    h01 += J[0][k] * s1;
    h11 += J[1][k] * s1;
  }
  InflOut out{h00, h01, h11, NAN, NAN};
  const double sg = active ? -1.0 : 1.0;
  const double a = 1.0 + sg * h00, b = sg * h01, c = 1.0 + sg * h11, det = a * c - b * b;
  if (!(a > 0.0 && det > 0.0)) return out;
  const double u0 = (c * rt0 - b * rt1) / det, u1 = (a * rt1 - b * rt0) / det;
  out.stud = rt0 * u0 + rt1 * u1;
  double v[NP];
#pragma unroll
  for (int k = 0; k < NP; ++k) v[k] = J[0][k] * u0 + J[1][k] * u1;
  double s = 0.0;
#pragma unroll
  for (int k = 0; k < NP; ++k) {
    double mk = 0.0;
#pragma unroll
    for (int j = 0; j < NP; ++j) mk += M[k * kInflP + j] * v[j];
    s += v[k] * mk;
  }
  out.infl = s;
  return out;
}

__global__ void __launch_bounds__(kInflTile) infl_obs_kernel(const InflRig* __restrict__ rigs, const InflTile* __restrict__ tiles) {
  __shared__ double S[kInflP * kInflP], M[kInflP * kInflP], sT[7], sCam[kCamStateStride], sR[9], sMask[6 + 8];
  const InflTile t = tiles[blockIdx.x];
  const InflRig& a = rigs[t.rig];
  const int tid = threadIdx.x, c = t.cam, f = t.frame, G = a.G, fd = a.fd;
  const CamInfo& ci = a.dp.cams[c];
  const int NG = 6 + ci.K, NP = 6 + NG, goff = ci.goff;
  const bool defined = a.cam_used[c] && a.frame_used[f] && *a.prior_ok;
  if (defined) {
    const double* sff = a.Sff + static_cast<int64_t>(f) * fd * fd;
    const double* sfg = a.Sfg + static_cast<int64_t>(f) * fd * G;
    const double* Q = a.Q + static_cast<int64_t>(f) * 36;
    for (int e = tid; e < NP * NP; e += kInflTile) {
      const int i = e / NP, j = e % NP;
      double s, m;
      if (i < 6 && j < 6) { s = sff[i * fd + j]; m = Q[i * 6 + j]; }
      else if (i < 6) s = m = sfg[static_cast<int64_t>(i) * G + goff + j - 6];
      else if (j < 6) s = m = sfg[static_cast<int64_t>(j) * G + goff + i - 6];
      else s = m = a.Sgg[static_cast<int64_t>(goff + i - 6) * G + goff + j - 6];
      S[i * kInflP + j] = s;
      M[i * kInflP + j] = m;
    }
    if (tid < 7) sT[tid] = a.state[7 * static_cast<int64_t>(f) + tid];
    if (tid < kCamStateStride) sCam[tid] = a.state[a.dp.off_cam + kCamStateStride * c + tid];
    if (tid < NG) sMask[tid] = a.mask[goff + tid];
    __syncthreads();
    if (tid == 0) qmat(Q4{sCam[0], sCam[1], sCam[2], sCam[3]}, sR);
    __syncthreads();
  }
  if (tid >= t.count) return;
  const int64_t i = t.start + tid;
  InflOut out{NAN, NAN, NAN, NAN, NAN};
  if (defined) {
    const V3 pw{a.pw[3 * i], a.pw[3 * i + 1], a.pw[3 * i + 2]};
    const double pcu = a.pc[2 * i], pcv = a.pc[2 * i + 1], vm = a.dp.visual_mult;
    const bool act = a.active[i] != 0;
    switch (ci.model) {  // uniform across the tile
      case kLinear: out = infl_obs<kLinear>(sT, sCam, sR, sMask, vm, pw, pcu, pcv, act, S, M); break;
      case kFov: out = infl_obs<kFov>(sT, sCam, sR, sMask, vm, pw, pcu, pcv, act, S, M); break;
      case kPoly2: out = infl_obs<kPoly2>(sT, sCam, sR, sMask, vm, pw, pcu, pcv, act, S, M); break;
      case kPoly3: out = infl_obs<kPoly3>(sT, sCam, sR, sMask, vm, pw, pcu, pcv, act, S, M); break;
      default: out = infl_obs<kKb4>(sT, sCam, sR, sMask, vm, pw, pcu, pcv, act, S, M); break;
    }
  }
  const int64_t o = a.idx[i];
  if (a.h) { a.h[3 * o] = out.h00; a.h[3 * o + 1] = out.h01; a.h[3 * o + 2] = out.h11; }
  if (a.stud) a.stud[o] = out.stud;
  if (a.infl) a.infl[o] = out.infl;
}

}  // namespace vc
