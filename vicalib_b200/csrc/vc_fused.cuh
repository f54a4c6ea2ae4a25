// The reprojection half of the block normal equations: evaluate + Gram build, fused, for every engine.
//
// Each corner (pose chain, camera model, analytic Jacobian, SoftLOne corrector) parks two rows of the
// REDUCED Jacobian  [d/dpose(6) | d/dintrinsics(K) | residual]  in a shared-memory tile, column-major
// over corners; the 16 x 16 Gram matrix of those columns is formed with FP64 tensor-core
// mma.sync.m8n8k4 (DMMA), both operand fragments read straight from the tile.
//
// The six extrinsic (T_ck) columns never enter the tile: for one camera they are a constant linear map
// of the pose columns,  J_ck = J_pose * A  with  A = [[0, -R_ck^T], [-I, 0]]  (right perturbation on both
// sides, vc_math.cuh), so every block that involves them (E's extrinsic columns, the camera's global
// block, its gradient) is A^T / A applied to the summed Gram matrix once per (frame, camera)
// (expand_gram).  That halves the DMMA work (3 instead of 6 8x8 blocks per k-step) and the tile.
//
// Two layouts share the per-corner evaluation, the expansion and the frame-block store:
//   build_frame_warp    one warp per frame, 32 corners per slab: the frame tasks of the persistent kernels
//                       (lm_mega_kernel phase B, eval_mega_kernel phase T)
//   fused_build_kernel  one CTA per frame, 144 corners per pass, a cross-warp reduction: the multi-launch engine
//
// The Jacobian never goes to HBM: a build reads 44 B per corner and writes ~2 KB per (frame, camera).
// Replaces the residual+Jacobian evaluation and J^T J build Ceres does inside ceres::Solve
// (vicalibrator.h:956) for the ImuReprojectionCostFunctor blocks (ceres-cost-functions.h:342-377).
#pragma once
#include "vc_internal.h"
#include "vc_math.cuh"

namespace vc {

constexpr int kFusedThreads = 160;                   // 5 warps
constexpr int kFusedWarps = kFusedThreads / 32;
constexpr int kFusedChunk = 144;                     // corners staged per pass
constexpr int kFusedLd = 2 * kFusedChunk + 4;        // tile leading dimension (== 4 mod 16: conflict-free fragments)
constexpr int kFusedCols = 16;                       // 6 pose + K <= 8 intrinsics + residual, padded
constexpr int kFusedRed = 3 * 64;                    // per-warp partial: blocks (0,0) (1,0) (1,1)
static_assert(kFusedLd % 16 == 4, "fragment loads need ld == 4 (mod 16)");
constexpr int kSlabLd = 64 + 4;                        // 32 corners x 2 residual rows (+4: conflict-free fragments)
constexpr int kSlabDoubles = kFusedCols * kSlabLd;     // one warp's tile
constexpr int kWarpDoubles = kSlabDoubles + 48;        // + frame block (36) + frame gradient (6), padded
static_assert(kSlabLd % 16 == 4, "fragment loads need ld == 4 (mod 16)");

struct FusedArgs {
  DevProblem dp;
  const Ctl* ctl;
  int which;
  const double* state[2];
  const int32_t *grp_start, *grp_count, *group_of;
  const double *pw, *pc;  // AoS [n_obs][3], [n_obs][2]
  int64_t n_obs;
  const double* mask;  // [G]
  Blocks out[2];
  double* Cg;          // [n_groups][kCgStride]
  double* cost_part;   // [n_frames]
};
constexpr size_t kFusedSmemDoubles = static_cast<size_t>(kFusedCols) * kFusedLd + kFusedWarps * kFusedRed + 256 + 36 + 6 +
                                     kFusedWarps + 9;

__device__ __forceinline__ void dmma_m8n8k4(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(d0), "+d"(d1)
               : "d"(a), "d"(b));
}

// residual + reduced tangent Jacobian of one observation, loss-corrected, written to the tile:
// columns [0,6) pose (translation, rotation), [6,6+K) intrinsics (masked), 6+K residual, rest zero
template <int MODEL, int LD = kFusedLd>
__device__ __forceinline__ double eval_obs_to_tile(const double* T, const double* cam, const double* R, const double* mask, V3 pw,
                                                   double pcu, double pcv, double mult, double* tile, int k0, int k1) {
  constexpr int K = Cam<MODEL>::K;
  const Q4 q{T[0], T[1], T[2], T[3]};
  const V3 t{T[4], T[5], T[6]};
  const V3 pk = qrot(qconj(q), pw - t);
  const V3 pc = mat_mul(R, pk) + V3{cam[4], cam[5], cam[6]};
  double z[2], dzp[6], dzi[2 * K];
  Cam<MODEL>::project(pc, cam + 7, z, dzp, dzi);
  const double r0 = z[0] - pcu, r1 = z[1] - pcv;
  double rho0, rho1;
  soft_l_one(r0 * r0 + r1 * r1, &rho0, &rho1);
  const double sc = sqrt(rho1);
#pragma unroll
  for (int row = 0; row < 2; ++row) {
    const double* d = dzp + 3 * row;
    const double m0 = (d[0] * R[0] + d[1] * R[3] + d[2] * R[6]) * sc;
    const double m1 = (d[0] * R[1] + d[1] * R[4] + d[2] * R[7]) * sc;
    const double m2 = (d[0] * R[2] + d[1] * R[5] + d[2] * R[8]) * sc;
    double* o = tile + (row == 0 ? k0 : k1);
    o[0 * LD] = -m0;
    o[1 * LD] = -m1;
    o[2 * LD] = -m2;
    o[3 * LD] = m1 * pk.z - m2 * pk.y;
    o[4 * LD] = m2 * pk.x - m0 * pk.z;
    o[5 * LD] = m0 * pk.y - m1 * pk.x;
#pragma unroll
    for (int k = 0; k < K; ++k) o[(6 + k) * LD] = dzi[row * K + k] * sc * mask[6 + k];
    o[(6 + K) * LD] = (row == 0 ? r0 : r1) * sc;
#pragma unroll
    for (int k = 7 + K; k < kFusedCols; ++k) o[k * LD] = 0.0;
  }
  return 0.5 * rho0 * mult;
}

// eval_obs_to_tile for a camera model known at run time: the one device switch over the models
template <int LD>
__device__ __forceinline__ double eval_obs_any(int model, const double* T, const double* cam, const double* R, const double* mask, V3 pw,
                                               double pcu, double pcv, double mult, double* tile, int k0, int k1) {
  switch (model) {
    case kLinear: return eval_obs_to_tile<kLinear, LD>(T, cam, R, mask, pw, pcu, pcv, mult, tile, k0, k1);
    case kFov: return eval_obs_to_tile<kFov, LD>(T, cam, R, mask, pw, pcu, pcv, mult, tile, k0, k1);
    case kPoly2: return eval_obs_to_tile<kPoly2, LD>(T, cam, R, mask, pw, pcu, pcv, mult, tile, k0, k1);
    case kPoly3: return eval_obs_to_tile<kPoly3, LD>(T, cam, R, mask, pw, pcu, pcv, mult, tile, k0, k1);
    default: return eval_obs_to_tile<kKb4, LD>(T, cam, R, mask, pw, pcu, pcv, mult, tile, k0, k1);
  }
}

// x * A for a 6-vector x = (translation part, rotation part) of the pose columns: the matching
// extrinsic column e (0..2 rotation w_ck, 3..5 translation p_ck)
__device__ __forceinline__ double times_A(const double* x, int e, const double* R) {
  if (e < 3) return -x[3 + e];
  const double* r = R + 3 * (e - 3);
  return -(x[0] * r[0] + x[1] * r[1] + x[2] * r[2]);
}

// packed lower-triangle index of a camera block (at most 14 x 14: 105 entries) -> (row << 4 | col)
__device__ __forceinline__ void fill_tri_lut(unsigned char* lut, int first, int step) {
  for (int e = first; e < 105; e += step) {
    int p = 0;
    while ((p + 1) * (p + 2) / 2 <= e) ++p;
    lut[e] = static_cast<unsigned char>((p << 4) | (e - p * (p + 1) / 2));
  }
}

// Expands the 16 x 16 Gram matrix Gm of one (frame, camera) through A into:  Bp [6][6] += the pose block,
// gp [6] += the pose gradient,  the camera's columns of E_f (Ec = E_f + the camera's goff, rows 0..5 of leading
// dimension G),  and the camera's packed global block Cc (lower triangle over [w_ck p_ck intr], gradient at 105),
// stored, or added to with kAccumulate.  Entries first, first + step, ...: a thread that passes the same (first,
// step) for every frame owns the same entries of Cc.
template <bool kAccumulate>
__device__ __forceinline__ void expand_gram(const double* Gm, const double* R, const double* mask, int K, double* Bp, double* gp,
                                            double* Ec, int G, double* Cc, const unsigned char* tri_lut, int first, int step) {
  const int NG = 6 + K;
  const double* Grf = Gm + (6 + K) * 16;  // residual row: [pose | intrinsics] parts of the gradient
  const int nsym = NG * (NG + 1) / 2;
  const int n_out = 36 + 6 + 6 * NG + nsym + NG;
  for (int e = first; e < n_out; e += step) {
    int o = e;
    if (o < 36) { Bp[o] += Gm[(o / 6) * 16 + (o % 6)]; continue; }
    o -= 36;
    if (o < 6) { gp[o] += Grf[o]; continue; }
    o -= 6;
    if (o < 6 * NG) {  // E_f: row j (pose), column p of this camera's globals
      const int j = o / NG, p = o - j * NG;
      Ec[j * G + p] = p < 6 ? mask[p] * times_A(Gm + j * 16, p, R) : Gm[p * 16 + j];
      continue;
    }
    o -= 6 * NG;
    if (o < nsym) {
      const int p = tri_lut[o] >> 4, q = tri_lut[o] & 15;
      double v;
      if (q >= 6) {
        v = Gm[p * 16 + q];                                      // intrinsics x intrinsics
      } else if (p >= 6) {
        v = mask[q] * times_A(Gm + p * 16, q, R);                // intrinsics x extrinsics
      } else {                                                   // extrinsics x extrinsics: (A^T Gff A)[p][q]
        if (p < 3) {
          v = -times_A(Gm + (3 + p) * 16, q, R);
        } else {
          const double* r = R + 3 * (p - 3);
          v = -(r[0] * times_A(Gm, q, R) + r[1] * times_A(Gm + 16, q, R) + r[2] * times_A(Gm + 32, q, R));
        }
        v *= mask[p] * mask[q];
      }
      if (kAccumulate) Cc[o] += v;
      else Cc[o] = v;
      continue;
    }
    o -= nsym;  // gradient of the camera's globals
    const double v = o < 6 ? mask[o] * times_A(Grf, o, R) : Grf[o];
    if (kAccumulate) Cc[105 + o] += v;
    else Cc[105 + o] = v;
  }
}

// B_f [FD][FD] and g_f [FD] from the pose block Bp [6][6] and gradient gp [6]; velocity rows and columns zero
template <int FD>
__device__ __forceinline__ void store_frame_block(const double* Bp, const double* gp, double* Bf, double* gf, int first, int step) {
  for (int q = first; q < FD * FD; q += step) {
    const int i = q / FD, j = q - i * FD;
    Bf[q] = (i < 6 && j < 6) ? Bp[i * 6 + j] : 0.0;
  }
  for (int q = first; q < FD; q += step) gf[q] = q < 6 ? gp[q] : 0.0;
}

// Reprojection blocks of one frame by one warp.  For every camera that sees the frame: its corners 32 at a time
// through the warp's slab [16][kSlabLd] (the next slab's observation is loaded while this one goes through the DMMAs,
// the accumulators stay in registers across slabs), then the three accumulator blocks mirrored into the 16 x 16 Gram
// matrix (in the slab) and expanded by expand_gram.  cam_obs(c) -> (start, count) of camera c's observations in the
// frame (count 0: the camera does not see it; prepare() never makes an empty group); cam_block(c) -> its packed
// global block, asked for after the corners (no pointer held across the evaluation).  E_f (FD rows) is zeroed unless
// the frame's only camera writes all G of its columns.  Leaves the pose block [36] and gradient [6] in the slab tail
// (slab + kSlabDoubles) and returns cost plus the lane's share of the frame's cost.
template <int FD, bool kAccumulate, class CamObs, class CamBlock>
__device__ __forceinline__ double build_frame_warp(const DevProblem& dp, const double* T, const double* smCam, const double* smRc,
                                                   const double* mask, const double* pw_all, const double* pc_all, double* Ef,
                                                   double* slab, const unsigned char* tri_lut, int lane, double cost,
                                                   CamObs cam_obs, CamBlock cam_block) {
  const int G = dp.G, n_cams = dp.n_cams;
  double* smB = slab + kSlabDoubles;  // [36] | [6]
  double* smg = smB + 36;
  const double* frag = slab + (lane >> 2) * kSlabLd + (lane & 3);
  __syncwarp();
  for (int q = lane; q < 42; q += 32) smB[q] = 0.0;
  if (!(n_cams == 1 && G == 6 + dp.cams[0].K))
    for (int q = lane; q < FD * G; q += 32) Ef[q] = 0.0;
  for (int c = 0; c < n_cams; ++c) {
    const int2 grp = cam_obs(c);
    if (grp.y == 0) continue;
    const CamInfo& ci = dp.cams[c];
    const int K = ci.K, model = ci.model;
    const int start = grp.x, cnt = grp.y;
    const double* cam = smCam + kCamStateStride * c;
    const double* Rc = smRc + 9 * c;
    const double* cmask = mask + ci.goff;
    double acc[3][2];
#pragma unroll
    for (int b = 0; b < 3; ++b) acc[b][0] = acc[b][1] = 0.0;
    double nx[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
    if (lane < cnt) {
      const int64_t i = start + lane;
      nx[0] = pw_all[3 * i]; nx[1] = pw_all[3 * i + 1]; nx[2] = pw_all[3 * i + 2]; nx[3] = pc_all[2 * i]; nx[4] = pc_all[2 * i + 1];
    }
    for (int s0 = 0; s0 < cnt; s0 += 32) {
      const int m = min(32, cnt - s0);
      const int m4 = (m + 3) & ~3;
      const V3 pw{nx[0], nx[1], nx[2]};
      const double pcu = nx[3], pcv = nx[4];
      if (s0 + 32 + lane < cnt) {
        const int64_t i = start + s0 + 32 + lane;
        nx[0] = pw_all[3 * i]; nx[1] = pw_all[3 * i + 1]; nx[2] = pw_all[3 * i + 2]; nx[3] = pc_all[2 * i]; nx[4] = pc_all[2 * i + 1];
      }
      __syncwarp();  // the previous slab's fragment loads are done
      if (lane < m) {
        cost += eval_obs_any<kSlabLd>(model, T, cam, Rc, cmask, pw, pcu, pcv, dp.visual_mult, slab, lane, 32 + lane);
      } else if (lane < m4) {  // zero the padding rows of both halves
#pragma unroll
        for (int q = 0; q < kFusedCols; ++q) {
          slab[q * kSlabLd + lane] = 0.0;
          slab[q * kSlabLd + 32 + lane] = 0.0;
        }
      }
      __syncwarp();
      // SYRK over k: steps [0, m4/4) cover residual row 0, [m4/4, m4/2) residual row 1 (two accumulator sets
      // for six independent DMMA chains measured no faster: the phase is not DMMA-latency bound)
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
    {
      const int rr = lane >> 2, cc = 2 * (lane & 3);
      const double vm = dp.visual_mult;
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        const int i = (b == 0 ? 0 : 8) + rr, j = (b == 2 ? 8 : 0) + cc;
        const double v0 = acc[b][0] * vm, v1 = acc[b][1] * vm;
        // diagonal blocks: both triangles are computed (bitwise equal), keep j <= i and mirror
        if (b == 1 || j <= i) { slab[i * 16 + j] = v0; slab[j * 16 + i] = v0; }
        if (b == 1 || j + 1 <= i) { slab[i * 16 + j + 1] = v1; slab[(j + 1) * 16 + i] = v1; }
      }
    }
    __syncwarp();
    expand_gram<kAccumulate>(slab, Rc, cmask, K, smB, smg, Ef + ci.goff, G, cam_block(c), tri_lut, lane, 32);
  }
  return cost;
}

template <int FD>
__global__ void __launch_bounds__(kFusedThreads, 4) fused_build_kernel(FusedArgs a) {
  extern __shared__ double smem[];
  if (a.ctl->done) return;
  const int buf = a.which ? 1 - a.ctl->cur : a.ctl->cur;
  const double* state = a.state[buf];
  const Blocks& out = a.out[buf];
  double* tile = smem;                                   // [16][kFusedLd]
  double* red = tile + kFusedCols * kFusedLd;            // [warps][3][64]
  double* Gm = red + kFusedWarps * kFusedRed;            // [16][16] Gram matrix of one (frame, camera)
  double* smB = Gm + 256;                                // [36] pose block
  double* smg = smB + 36;                                // [6] pose gradient
  double* wcost = smg + 6;                               // [warps]
  double* smR = wcost + kFusedWarps;                     // [9] R_ck of the current camera
  __shared__ unsigned char tri_lut[128];
  const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int G = a.dp.G, nf = a.dp.n_frames;
  fill_tri_lut(tri_lut, tid, kFusedThreads);
  for (int k = tid; k < 42; k += kFusedThreads) smB[k] = 0.0;
  double* Ef = out.E + static_cast<int64_t>(f) * FD * G;
  for (int k = tid; k < FD * G; k += kFusedThreads) Ef[k] = 0.0;
  const double* T = state + 7 * static_cast<int64_t>(f);
  const double* camBase = state + a.dp.off_cam;
  double cost = 0.0;
  for (int c = 0; c < a.dp.n_cams; ++c) {
    const int g = a.group_of[c * nf + f];
    if (g < 0) continue;
    const CamInfo& ci = a.dp.cams[c];
    const int start = a.grp_start[g], cnt = a.grp_count[g];
    double* Cgg = a.Cg + static_cast<int64_t>(g) * kCgStride;
    double* Ec = Ef + ci.goff;
    const double* cam = camBase + kCamStateStride * c;
    const double* mask = a.mask + ci.goff;
    __syncthreads();  // the previous camera's epilogue is done with smR / Gm
    if (tid < 9) {
      double R[9];
      qmat(Q4{cam[0], cam[1], cam[2], cam[3]}, R);
#pragma unroll
      for (int k = 0; k < 9; ++k)
        if (tid == k) smR[k] = R[k];
    }
    double acc[3][2];
#pragma unroll
    for (int b = 0; b < 3; ++b) acc[b][0] = acc[b][1] = 0.0;
    for (int ch = 0; ch < cnt; ch += kFusedChunk) {
      const int m = min(kFusedChunk, cnt - ch);
      const int m4 = (m + 3) & ~3;  // k range padded to the MMA depth
      __syncthreads();              // previous pass is done with the tile; smR is visible
      if (tid < m) {
        const int64_t i = start + ch + tid;
        const V3 pw{a.pw[3 * i], a.pw[3 * i + 1], a.pw[3 * i + 2]};
        const double pcu = a.pc[2 * i], pcv = a.pc[2 * i + 1];
        cost += eval_obs_any<kFusedLd>(ci.model, T, cam, smR, mask, pw, pcu, pcv, a.dp.visual_mult, tile, tid, kFusedChunk + tid);
      } else if (tid < m4) {  // zero the padding rows of both halves
#pragma unroll
        for (int k = 0; k < kFusedCols; ++k) {
          tile[k * kFusedLd + tid] = 0.0;
          tile[k * kFusedLd + kFusedChunk + tid] = 0.0;
        }
      }
      __syncthreads();
      // SYRK over k: steps [0, m4/4) cover residual row 0, [m4/4, m4/2) residual row 1
      const int ns = m4 >> 2;
      const double* frag = tile + (lane >> 2) * kFusedLd + (lane & 3);
      for (int s = warp; s < 2 * ns; s += kFusedWarps) {
        const int k0 = s < ns ? 4 * s : kFusedChunk + 4 * (s - ns);
        const double a0 = frag[k0], a1 = frag[8 * kFusedLd + k0];
        dmma_m8n8k4(acc[0][0], acc[0][1], a0, a0);  // (0,0)
        dmma_m8n8k4(acc[1][0], acc[1][1], a1, a0);  // (1,0)
        dmma_m8n8k4(acc[2][0], acc[2][1], a1, a1);  // (1,1)
      }
    }
    // cross-warp reduction of the three 8x8 blocks into the symmetric 16 x 16 Gram matrix
    {
      double* rw = red + warp * kFusedRed + (lane >> 2) * 8 + 2 * (lane & 3);
#pragma unroll
      for (int b = 0; b < 3; ++b) { rw[b * 64] = acc[b][0]; rw[b * 64 + 1] = acc[b][1]; }
    }
    __syncthreads();
#pragma unroll 1  // unrolled, this loop's loads cost the kernel spills (ptxas -v)
    for (int e = tid; e < kFusedRed; e += kFusedThreads) {
      const int b = e >> 6, rr = (e >> 3) & 7, cc = e & 7;
      const int i = (b == 0 ? 0 : 8) + rr, j = (b == 2 ? 8 : 0) + cc;
      if (j > i) continue;
      double v = 0.0;
#pragma unroll
      for (int w = 0; w < kFusedWarps; ++w) v += red[w * kFusedRed + e];
      v *= a.dp.visual_mult;
      Gm[i * 16 + j] = v;
      Gm[j * 16 + i] = v;
    }
    __syncthreads();
    expand_gram<false>(Gm, smR, mask, ci.K, smB, smg, Ec, G, Cgg, tri_lut, tid, kFusedThreads);
  }
  // block cost
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cost += __shfl_down_sync(0xffffffffu, cost, o);
  if (lane == 0) wcost[warp] = cost;
  __syncthreads();
  store_frame_block<FD>(smB, smg, out.B + static_cast<int64_t>(f) * FD * FD, out.gf + static_cast<int64_t>(f) * FD, tid, kFusedThreads);
  if (tid == 0) {
    double s = 0.0;
    for (int w = 0; w < kFusedWarps; ++w) s += wcost[w];
    a.cost_part[f] = s;
  }
}

}  // namespace vc
