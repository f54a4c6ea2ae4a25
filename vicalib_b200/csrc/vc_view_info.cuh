// Information a candidate view of the target would add to the globals (vcgpu_get_view_information(_batch)).  A
// candidate is a rig pose T_wp; the corners it sees are observations at their own predicted pixels (residual 0,
// SoftLOne weight 1), which couple only the candidate's pose and the globals.  Marginalising the pose leaves
//   S = C_v - E_v^T B_v^-1 E_v                                    (G x G)
// and the posterior of the globals is (Sigma^-1 + S)^-1.  On F, the rows of Sigma whose diagonal is not 0.0, with
// D = sqrt(diag Sigma_F) and the Jacobi-scaled prior Sigma_F~ = D^-1 Sigma_F D^-1 = L L^T:
//   W = L^T (D S_F D) L,   M = I + W = U diag(d) U^T,   gain = 1/2 sum log d_k = 1/2 log det(I + Sigma_F S_F),
//   Sigma'_F = D L M^-1 L^T D.
// Two kernels: view_prior_kernel factors Sigma_F~ once per rig (one CTA per rig); view_info_kernel takes one candidate
// per CTA:
//   1. visibility: warp c projects the target through camera c (eval_obs_to_tile's expressions, so the residual is 0)
//      and compacts the seen corners (p_w, pixel) into camera c's segment of the CTA's workspace, in corner order;
//   2. frame blocks: warp 0 runs build_frame_warp<6, false> on the workspace: B_v, E_v and each camera's packed block;
//   3. reduction: W = sum_c L_c^T (D C_c D) L_c - V^T V, V = chol(B_v)^-1 E_v D L, into one G_F x G_F matrix that
//      overlays the workspace;
//   4. M = I + W by an in-place LDL^T, M^-1 in place, then Sigma'_F row by row: t = M^-1 l_i, Sigma'_ij = D_i D_j l_j.t
//      for j <= i, mirrored.
// Every entry is owned by one thread and summed in a fixed order, so a candidate's bits depend on nothing else in the
// launch.
#pragma once
#include "vc_internal.h"
#include "vc_math.cuh"
#include "vc_kernels.cuh"
#include "vc_fused.cuh"
#include "vc_proj_cov.cuh"

namespace vc {

constexpr int kViewThreads = 256;  // 8 warps: warp c compacts camera c (kMaxCams == 8)
constexpr int kViewWarps = kViewThreads / 32;
constexpr int kViewMaxPts = 400;   // target corners per call: 8 cameras' segments (40 B per corner) fit the workspace
constexpr int kViewCamRows = 6 + 8;  // globals of one camera
constexpr double kViewQuatTol = 1e-6;  // a candidate's |q| must be within this of 1
static_assert(kViewWarps >= kMaxCams, "one warp per camera");

// one rig of a launch: its candidates are CTAs [cta0, cta0 + n_cand)
struct ViewRig {
  DevProblem dp;          // the handle's cameras, G and visual_mult (build_frame_warp's view of the problem)
  const double* cams;     // [n_cams][kCamStateStride] the accepted state's cameras
  const double* mask;     // [G] the build's 0/1 mask of the globals
  const double* S;        // [G][G] Sigma
  const int32_t* fidx;    // [GF] the global index of each row of F, ascending
  double* L;              // [GF][GF] chol(Sigma_F~), lower, zeros above (view_prior_kernel)
  double* D;              // [GF] sqrt(diag Sigma_F) (view_prior_kernel)
  int* prior_ok;          // 1 where Sigma_F~ was positive definite (view_prior_kernel)
  const double* T;        // [n_cand][7] q | t
  const double* pw;       // [n_pts][3]
  int32_t* n_seen;        // [n_cand][n_cams]
  double* gain;           // [n_cand]
  double* var;            // [n_cand][G], or null
  double* post;           // [n_cand][G][G], or null
  int64_t n_cand, cta0;
  double facing[3];
  double width[kMaxCams], height[kMaxCams];
  int has_facing, n_pts, G, GF;
  int used[kMaxCams];     // 1: an active observation sees the camera
  int f0[kMaxCams + 1];   // camera c's rows of F are [f0[c], f0[c + 1])
};

// leading dimension of a G_F x G_F matrix in shared memory: odd, so a column's doubles fall in different banks
__host__ __device__ inline int view_ld(int n) { return n | 1; }

// the candidate kernel's dynamic shared memory (doubles): workspace / W | E_v | camera blocks | slab | L_c | Z_c |
// P | V | D | tmp | per-warp t | cameras | R_ck
struct ViewSmem {
  int64_t W, Ef, Cc, slab, Lc, Zc, P, V, D, tmp, tw, cam, R, total;
};
__host__ __device__ inline ViewSmem view_smem(int G, int GF, int n_cams, int n_pts) {
  ViewSmem s;
  const int64_t w = static_cast<int64_t>(GF) * view_ld(GF), corners = 5 * static_cast<int64_t>(n_cams) * n_pts;
  int64_t at = 0;
  auto take = [&](int64_t n) { const int64_t o = at; at += (n + 1) & ~int64_t(1); return o; };  // 16-byte aligned
  s.W = take(w > corners ? w : corners);
  s.Ef = take(6 * static_cast<int64_t>(G));
  s.Cc = take(static_cast<int64_t>(kMaxCams) * kCgStride);
  s.slab = take(kWarpDoubles);
  s.Lc = take(static_cast<int64_t>(kViewCamRows) * GF);
  s.Zc = take(static_cast<int64_t>(kViewCamRows) * GF);
  s.P = take(6 * static_cast<int64_t>(GF));
  s.V = take(6 * static_cast<int64_t>(GF));
  s.D = take(GF);
  s.tmp = take(GF);
  s.tw = take(static_cast<int64_t>(kViewWarps) * GF);
  s.cam = take(static_cast<int64_t>(kMaxCams) * kCamStateStride);
  s.R = take(9 * kMaxCams);
  s.total = at;
  return s;
}

// In-place LDL^T of the symmetric n x n matrix whose lower triangle is A (leading dimension ld), by the whole CTA:
// the strict lower triangle becomes the unit factor U, the diagonal keeps the pivots d.  Right-looking, one barrier
// per step: step k updates the trailing triangle with column k unscaled and scales column k - 1.  Every entry is
// updated by one thread in step order.  False (uniformly) where a pivot is not positive; A is then partial.
__device__ bool view_ldl(double* A, int n, int ld) {
  const int tid = threadIdx.x, nt = blockDim.x;
  __syncthreads();
  for (int k = 0; k < n; ++k) {
    const double d = A[k * ld + k];
    if (!(d > 0.0)) return false;  // every thread reads the same pivot
    const double id = 1.0 / d;
    if (k > 0) {
      const double ip = 1.0 / A[(k - 1) * ld + k - 1];
      for (int i = k + tid; i < n; i += nt) A[i * ld + k - 1] *= ip;
    }
    const int m = n - k - 1;
    for (int e = tid; e < m * m; e += nt) {
      const int i = k + 1 + e / m, j = k + 1 + e % m;
      if (j > i) continue;
      A[i * ld + j] -= A[i * ld + k] * (A[j * ld + k] * id);
    }
    __syncthreads();
  }
  return true;
}

// the scaled prior of each rig: Sigma_F~ = D^-1 Sigma_F D^-1 (diagonal exactly 1), L = U sqrt(d).  One CTA per rig.
__global__ void __launch_bounds__(kViewThreads) view_prior_kernel(const ViewRig* __restrict__ rigs) {
  extern __shared__ double sm[];
  const ViewRig& a = rigs[blockIdx.x];
  const int n = a.GF, ld = view_ld(n), G = a.G, tid = threadIdx.x, nt = blockDim.x;
  double* A = sm;
  double* D = A + static_cast<int64_t>(n) * ld;
  for (int i = tid; i < n; i += nt) D[i] = sqrt(a.S[static_cast<int64_t>(a.fidx[i]) * G + a.fidx[i]]);
  __syncthreads();
  for (int e = tid; e < n * n; e += nt) {
    const int i = e / n, j = e % n;
    if (j > i) continue;
    A[i * ld + j] = i == j ? 1.0 : a.S[static_cast<int64_t>(a.fidx[i]) * G + a.fidx[j]] / (D[i] * D[j]);
  }
  bool ok = true;
  for (int i = 0; i < n; ++i) ok = ok && D[i] > 0.0;  // also false for a NaN diagonal
  if (ok) ok = view_ldl(A, n, ld);
  for (int i = tid; i < n; i += nt) a.D[i] = D[i];
  if (ok)
    for (int e = tid; e < n * n; e += nt) {
      const int i = e / n, j = e % n;
      a.L[e] = j > i ? 0.0 : i == j ? sqrt(A[i * ld + i]) : A[i * ld + j] * sqrt(A[j * ld + j]);
    }
  if (tid == 0) *a.prior_ok = ok ? 1 : 0;
}

// corner pw through camera c at pose T: the pixel as eval_obs_to_tile computes it, and whether the corner is seen
template <int MODEL>
__device__ __forceinline__ bool view_sees(const ViewRig& a, const double* T, const double* cam, const double* R, double lim, V3 pw,
                                          double w, double h, double z[2]) {
  const Q4 q{T[0], T[1], T[2], T[3]};
  const V3 t{T[4], T[5], T[6]};
  const V3 pk = qrot(qconj(q), pw - t);
  const V3 pc = mat_mul(R, pk) + V3{cam[4], cam[5], cam[6]};
  Cam<MODEL>::project(pc, cam + 7, z, nullptr, nullptr);
  const double* in = cam + 7;
  bool ok;
  if constexpr (MODEL == kKb4) {
    ok = atan2(sqrt(pc.x * pc.x + pc.y * pc.y), pc.z) < lim;
  } else {
    ok = pc.z > 0.0;
    if constexpr (MODEL == kPoly2 || MODEL == kPoly3) {
      const double u = pc.x / pc.z, v = pc.y / pc.z;
      ok = ok && u * u + v * v < lim;
    } else if constexpr (MODEL == kFov) {
      // the unprojection's rule at the pixel: past its small-rad branch, r_d |w| < pi / 2
      const double xd = (z[0] - in[2]) / in[0], yd = (z[1] - in[3]) / in[1], rd = sqrt(xd * xd + yd * yd);
      const double om = in[4];
      if (om * om > 1e-5) {
        const double fs = 2.0 * tan(0.5 * om) / om, rs = rd / fs;
        ok = ok && (rs * rs < 1e-5 || rd * fabs(om) < 0.5 * M_PI);
      }
    }
  }
  ok = ok && z[0] >= 0.0 && z[0] < w && z[1] >= 0.0 && z[1] < h;
  if (ok && a.has_facing) {
    // (c_w - p_w) . n > 0, in the rig frame: c_k = -R_ck^T p_ck, n_k = R_wp^T n
    const V3 ck = mat_tmul(R, V3{-cam[4], -cam[5], -cam[6]});
    const V3 nk = qrot(qconj(q), V3{a.facing[0], a.facing[1], a.facing[2]});
    ok = dot(ck - pk, nk) > 0.0;
  }
  return ok;
}

__device__ __forceinline__ bool view_sees_any(int model, const ViewRig& a, const double* T, const double* cam, const double* R, double lim,
                                              V3 pw, double w, double h, double z[2]) {
  switch (model) {
    case kLinear: return view_sees<kLinear>(a, T, cam, R, lim, pw, w, h, z);
    case kFov: return view_sees<kFov>(a, T, cam, R, lim, pw, w, h, z);
    case kPoly2: return view_sees<kPoly2>(a, T, cam, R, lim, pw, w, h, z);
    case kPoly3: return view_sees<kPoly3>(a, T, cam, R, lim, pw, w, h, z);
    default: return view_sees<kKb4>(a, T, cam, R, lim, pw, w, h, z);
  }
}

// One CTA per candidate: rigs[r] owns CTAs [cta0, cta0 + n_cand).
__global__ void __launch_bounds__(kViewThreads) view_info_kernel(const ViewRig* __restrict__ rigs, int n_rigs) {
  extern __shared__ double sm[];
  __shared__ unsigned char tri_lut[128];
  __shared__ double sT[7], lim[kMaxCams], Lb[36], iLb[6];
  __shared__ int cnt[kMaxCams], flag;
  int lo = 0, hi = n_rigs - 1;  // the last rig whose cta0 <= blockIdx.x
  while (lo < hi) {
    const int mid = (lo + hi + 1) / 2;
    if (rigs[mid].cta0 <= blockIdx.x) lo = mid;
    else hi = mid - 1;
  }
  const ViewRig& a = rigs[lo];
  if (!*a.prior_ok) return;
  const int64_t ci = blockIdx.x - a.cta0;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nt = blockDim.x;
  const int G = a.G, GF = a.GF, nc = a.dp.n_cams, np = a.n_pts, ld = view_ld(GF);
  const ViewSmem L_ = view_smem(G, GF, nc, np);
  double* W = sm + L_.W;
  double* pw_ws = W;                                  // [nc * np][3]
  double* pc_ws = W + 3 * static_cast<int64_t>(nc) * np;  // [nc * np][2]
  double* Ef = sm + L_.Ef;
  double* Cc = sm + L_.Cc;
  double* slab = sm + L_.slab;
  double* Lc = sm + L_.Lc;
  double* Zc = sm + L_.Zc;
  double* P = sm + L_.P;
  double* V = sm + L_.V;
  double* D = sm + L_.D;
  double* tmp = sm + L_.tmp;
  double* smCam = sm + L_.cam;
  double* smR = sm + L_.R;
  fill_tri_lut(tri_lut, tid, nt);
  if (tid < 7) sT[tid] = a.T[7 * ci + tid];
  for (int e = tid; e < nc * kCamStateStride; e += nt) smCam[e] = a.cams[e];
  for (int i = tid; i < GF; i += nt) D[i] = a.D[i];
  __syncthreads();
  if (tid < nc) {
    const double* cam = smCam + kCamStateStride * tid;
    double R[9];
    qmat(Q4{cam[0], cam[1], cam[2], cam[3]}, R);
    for (int k = 0; k < 9; ++k) smR[9 * tid + k] = R[k];
    const double* in = cam + 7;
    const int m = a.dp.cams[tid].model;
    lim[tid] = m == kPoly2 ? proj_limit<kPoly2>(in) : m == kPoly3 ? proj_limit<kPoly3>(in) : m == kKb4 ? proj_limit<kKb4>(in) : INFINITY;
  }
  __syncthreads();
  // 1. visibility: warp c, corners in order, compacted by ballot
  if (warp < nc) {
    const int c = warp;
    int n = 0;
    for (int j0 = 0; j0 < np; j0 += 32) {
      const int j = j0 + lane;
      double z[2] = {0.0, 0.0};
      V3 pw{0.0, 0.0, 0.0};
      bool seen = false;
      if (j < np) {
        pw = V3{a.pw[3 * j], a.pw[3 * j + 1], a.pw[3 * j + 2]};
        seen = view_sees_any(a.dp.cams[c].model, a, sT, smCam + kCamStateStride * c, smR + 9 * c, lim[c], pw, a.width[c], a.height[c], z);
      }
      const unsigned b = __ballot_sync(0xffffffffu, seen);
      if (seen) {
        const int64_t o = static_cast<int64_t>(c) * np + n + __popc(b & ((1u << lane) - 1u));
        pw_ws[3 * o] = pw.x; pw_ws[3 * o + 1] = pw.y; pw_ws[3 * o + 2] = pw.z;
        pc_ws[2 * o] = z[0]; pc_ws[2 * o + 1] = z[1];
      }
      n += __popc(b);
    }
    if (lane == 0) cnt[c] = n;
  }
  __syncthreads();
  int n_contrib = 0;
  for (int c = 0; c < nc; ++c) n_contrib += a.used[c] ? cnt[c] : 0;
  if (tid < nc) a.n_seen[ci * nc + tid] = cnt[tid];
  const int64_t GG = static_cast<int64_t>(G) * G;
  double* var = a.var ? a.var + ci * G : nullptr;
  double* post = a.post ? a.post + ci * GG : nullptr;
  if (n_contrib == 0) {  // nothing to add: Sigma itself
    if (tid == 0) a.gain[ci] = 0.0;
    if (var)
      for (int i = tid; i < G; i += nt) var[i] = a.S[static_cast<int64_t>(i) * G + i];
    if (post)
      for (int64_t e = tid; e < GG; e += nt) post[e] = a.S[e];
    return;
  }
  // 2. the candidate's frame blocks (warp 0)
  if (n_contrib >= 4 && warp == 0) {
    const int np_ = np;
    build_frame_warp<6, false>(
        a.dp, sT, smCam, smR, a.mask, pw_ws, pc_ws, Ef, slab, tri_lut, lane, 0.0,
        [&](int c) { return make_int2(c * np_, a.used[c] ? cnt[c] : 0); }, [&](int c) { return Cc + c * kCgStride; });
    __syncwarp();
    if (lane == 0) {  // B_v's factor, by the frame elimination's test
      double Lr[6][6], il[6];
      const double* Bp = slab + kSlabDoubles;
      for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) Lr[i][j] = Bp[i * 6 + j];
      flag = frame_chol<6>(Lr, il) ? 1 : 0;
      for (int i = 0; i < 6; ++i) {
        iLb[i] = il[i];
        for (int j = 0; j < 6; ++j) Lb[i * 6 + j] = j <= i ? Lr[i][j] : 0.0;
      }
    }
  }
  __syncthreads();
  if (n_contrib < 4 || !flag) {  // the view does not fix its pose
    if (tid == 0) a.gain[ci] = NAN;
    if (var)
      for (int i = tid; i < G; i += nt) var[i] = NAN;
    if (post)
      for (int64_t e = tid; e < GG; e += nt) post[e] = NAN;
    return;
  }
  // 3. W.  P = chol(B_v)^-1 E_F D (6 x GF), V = P L
  for (int b = tid; b < GF; b += nt) {
    const int g = a.fidx[b];
    double x[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      double s = Ef[k * G + g] * D[b];
      for (int m = 0; m < k; ++m) s -= Lb[k * 6 + m] * x[m];
      x[k] = s * iLb[k];
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) P[k * GF + b] = x[k];
  }
  __syncthreads();
  for (int e = tid; e < 6 * GF; e += nt) {
    const int k = e / GF, b = e % GF;
    double s = 0.0;
    for (int q = b; q < GF; ++q) s += P[k * GF + q] * a.L[static_cast<int64_t>(q) * GF + b];
    V[e] = s;
  }
  // the camera terms into W's lower triangle, cameras in order
  for (int e = tid; e < GF * GF; e += nt) {
    const int i = e / GF, j = e % GF;
    if (j <= i) W[i * ld + j] = 0.0;
  }
  for (int c = 0; c < nc; ++c) {
    const int r0 = a.f0[c], nr = a.f0[c + 1] - r0;
    if (!a.used[c] || cnt[c] == 0 || nr == 0) continue;
    const int goff = a.dp.cams[c].goff;
    const double* Cp = Cc + c * kCgStride;
    __syncthreads();  // the previous camera's Lc / Zc are read
    for (int e = tid; e < nr * GF; e += nt) Lc[e] = a.L[static_cast<int64_t>(r0) * GF + e];
    __syncthreads();
    // Z_c = (D C_c D) L_c
    for (int e = tid; e < nr * GF; e += nt) {
      const int p = e / GF, j = e % GF;
      const int gp = a.fidx[r0 + p] - goff;
      double s = 0.0;
      for (int q = 0; q < nr; ++q) {
        const int gq = a.fidx[r0 + q] - goff;
        const double cpq = gp >= gq ? Cp[gp * (gp + 1) / 2 + gq] : Cp[gq * (gq + 1) / 2 + gp];
        s += (D[r0 + p] * cpq * D[r0 + q]) * Lc[q * GF + j];
      }
      Zc[e] = s;
    }
    __syncthreads();
    for (int e = tid; e < GF * GF; e += nt) {
      const int i = e / GF, j = e % GF;
      if (j > i) continue;
      double s = 0.0;
      for (int p = 0; p < nr; ++p) s += Lc[p * GF + i] * Zc[p * GF + j];
      W[i * ld + j] += s;
    }
  }
  __syncthreads();
  // M = I + W - V^T V
  for (int e = tid; e < GF * GF; e += nt) {
    const int i = e / GF, j = e % GF;
    if (j > i) continue;
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 6; ++k) s += V[k * GF + i] * V[k * GF + j];
    W[i * ld + j] = (W[i * ld + j] - s) + (i == j ? 1.0 : 0.0);
  }
  // 4. M = U diag(d) U^T, the gain, M^-1 in place
  const bool ok = view_ldl(W, GF, ld);
  if (!ok) {
    if (tid == 0) a.gain[ci] = NAN;
    if (var)
      for (int i = tid; i < G; i += nt) var[i] = NAN;
    if (post)
      for (int64_t e = tid; e < GG; e += nt) post[e] = NAN;
    return;
  }
  if (tid == 0) {
    double s = 0.0;
    for (int k = 0; k < GF; ++k) s += log(W[k * ld + k]);
    a.gain[ci] = fmax(0.5 * s, 0.0);
  }
  // the pivots' reciprocals, then X = U^-1 in place, column by column from the right
  for (int k = tid; k < GF; k += nt) tmp[k] = 1.0 / W[k * ld + k];
  double* col = Zc;  // column j of U, kept while it is overwritten
  for (int j = GF - 2; j >= 0; --j) {
    __syncthreads();
    for (int i = j + 1 + tid; i < GF; i += nt) col[i] = W[i * ld + j];
    __syncthreads();
    for (int i = j + 1 + tid; i < GF; i += nt) {
      double s = col[i];
      for (int k = j + 1; k < i; ++k) s += W[i * ld + k] * col[k];
      W[i * ld + j] = -s;
    }
  }
  // M^-1 = X^T diag(1/d) X in place, row by row: row i reads only rows >= i
  for (int i = 0; i < GF; ++i) {
    __syncthreads();
    for (int j = tid; j <= i; j += nt) {
      double s = (j == i ? 1.0 : W[i * ld + j]) * tmp[i];
      for (int k = i + 1; k < GF; ++k) s += W[k * ld + i] * W[k * ld + j] * tmp[k];
      W[i * ld + j] = s;
    }
  }
  __syncthreads();
  // outputs: zeros outside F, then Sigma'_ij = D_i D_j l_j . (M^-1 l_i) for j <= i, mirrored
  if (post)
    for (int64_t e = tid; e < GG; e += nt) post[e] = 0.0;
  if (var)
    for (int i = tid; i < G; i += nt) var[i] = 0.0;
  __syncthreads();
  double* t = sm + L_.tw + static_cast<int64_t>(warp) * GF;
  for (int i = warp; i < GF; i += kViewWarps) {
    const double* li = a.L + static_cast<int64_t>(i) * GF;
    __syncwarp();
    for (int b = lane; b < GF; b += 32) {
      double s = 0.0;
      for (int q = 0; q <= i; ++q) s += (b >= q ? W[b * ld + q] : W[q * ld + b]) * li[q];
      t[b] = s;
    }
    __syncwarp();
    const int gi = a.fidx[i];
    for (int j = post ? lane : (lane == 0 ? i : GF); j <= i; j += post ? 32 : GF + 1) {
      const double* lj = a.L + static_cast<int64_t>(j) * GF;
      double s = 0.0;
      for (int q = 0; q <= j; ++q) s += lj[q] * t[q];
      const double v = D[i] * D[j] * s;
      const int gj = a.fidx[j];
      if (post) { post[static_cast<int64_t>(gi) * G + gj] = v; post[static_cast<int64_t>(gj) * G + gi] = v; }
      if (var && j == i) var[gi] = v;
    }
  }
}

}  // namespace vc
