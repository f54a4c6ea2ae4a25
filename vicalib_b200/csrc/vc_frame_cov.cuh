// Marginal covariance of every frame's tangent (vcgpu_get_frame_covariance): the [f, f] blocks of (J^T J)^-1, by a
// selected inversion of the frame elimination the solve already runs.  Everything here works in the Jacobi-scaled
// system S H S that the eliminations factor; the last step unscales.
//
// Vision (fd = 6, block-diagonal frames): Σ_ff = B_f^-1 + W_f Σ_gg W_f^T with W_f = B_f^-1 E_f, the X that
// frame_solve_kernel stores, and Σ_gg the inverse of the reduced system.
//
// Inertial (fd = 9, block-tridiagonal frames): the chain elimination (vc_chain.cuh) keeps, for every eliminated node p
// of a level, its solution against the chunk's boundary y = (left separator, right separator, globals):
// x_p = -Z_g - M_p x_y with M_p = Z_p[:, 0:2FD+G].  With the interior's block-tridiagonal matrix T (its inverse K)
// and Σ_yy from the level above, the inverse restricted to the chunk is
//   Σ_py = -M_p Σ_yy,   Σ_pq = K_pq + M_p Σ_yy M_q^T.
// The walk starts at the inverse of the dense [globals | top nodes] system and goes down the levels; at every level it
// keeps what the level below needs as its boundary: Σ_kk, Σ_k,k+1 and Σ_kg of every node (SigmaLevel).
//
// The blocks off the diagonal (vcgpu_get_frame_cross_covariance) come from the same two routes: vision Σ_fg = -X_f Σ_gg
// and Σ_f,f+1 = X_f Σ_gg X_f+1^T (frame_cross_cov_block), inertial level 0's Σ_kg and Σ_k,k+1 (frame_cross_cov_out_entry).
#pragma once
#include "vc_chain.cuh"

namespace vc {

// ---------------------------------------------------------------- vision: one warp per frame
struct FrameCovArgs {
  DevProblem dp;
  Blocks b[2];
  const Ctl* ctl;
  const double* scale;
  const double* D2x;           // the frames' damping (0, or 1 on a frame no active observation sees)
  const double* X;             // [nf][FD][G+1] of frame_solve_kernel: B_f^-1 [E_f | g_f]
  const double* Sgg;           // [G*G] inverse of the reduced system
  const uint8_t* frame_used;   // [nf]
  double* out;                 // [nf][FD*FD]
};
constexpr int kFrameCovWarps = 4;

// Frame f's block B_f^-1 + X_f Σ_gg X_f^T, unscaled, by one warp (frame_cov_vision_kernel, cov_frame_mega_batch_kernel).
// b, D2x: the blocks of the normal equations and the frames' damping; sf: frame f's Jacobi scale; Xf: X_f = B_f^-1 E_f,
// [FD][ldx].  (B_f's address is formed after the product: held across it, it costs frame_cov_vision_kernel two registers.)
template <int FD>
__device__ __forceinline__ void frame_cov_block(const Blocks& b, const double* D2x, int f, const double* sf, const double* Xf, int ldx,
                                                const double* Sgg, int G, int lane, double* out) {
  constexpr int NP = FD * (FD + 1) / 2;  // lower triangle, row by row
  const int M = ldx;
  // W Σ_gg W^T: the lanes split the columns q of P = W Σ_gg and sum P[r][q] W[c][q] over their own columns
  double acc[NP];
#pragma unroll
  for (int t = 0; t < NP; ++t) acc[t] = 0.0;
  for (int q = lane; q < G; q += 32) {
    double p[FD];
#pragma unroll
    for (int r = 0; r < FD; ++r) p[r] = 0.0;
    for (int k = 0; k < G; ++k) {
      const double s = Sgg[static_cast<int64_t>(k) * G + q];
#pragma unroll
      for (int r = 0; r < FD; ++r) p[r] += Xf[r * M + k] * s;
    }
    int t = 0;
#pragma unroll
    for (int r = 0; r < FD; ++r)
#pragma unroll
      for (int c = 0; c <= r; ++c) acc[t++] += p[r] * Xf[c * M + q];
  }
#pragma unroll
  for (int t = 0; t < NP; ++t)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[t] += __shfl_xor_sync(0xffffffffu, acc[t], o);
  // B_f^-1: every lane factors the damped, scaled block (as frame_solve_kernel); lane c solves column c
  const double* Bf = b.B + static_cast<int64_t>(f) * FD * FD;
  double L[FD][FD], iL[FD];
#pragma unroll
  for (int i = 0; i < FD; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j) L[i][j] = Bf[i * FD + j] * sf[i] * sf[j] + (i == j ? D2x[static_cast<int64_t>(f) * FD + i] : 0.0);
  frame_chol<FD>(L, iL);  // a failed pivot is flagged by the elimination, which factored the same block
  if (lane < FD) {
    double x[FD];
#pragma unroll
    for (int i = 0; i < FD; ++i) {
      double t = i == lane ? 1.0 : 0.0;
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
    int t = 0;
#pragma unroll
    for (int r = 0; r < FD; ++r)
#pragma unroll
      for (int c = 0; c <= r; ++c, ++t)
        if (c == lane) {
          const double v = (x[r] + acc[t]) * (sf[r] * sf[c]);
          out[r * FD + c] = v;
          out[c * FD + r] = v;
        }
  }
}

template <int FD>
__global__ void __launch_bounds__(32 * kFrameCovWarps) frame_cov_vision_kernel(FrameCovArgs a) {
  const int lane = threadIdx.x & 31, f = blockIdx.x * kFrameCovWarps + (threadIdx.x >> 5);
  if (f >= a.dp.n_frames) return;
  double* out = a.out + static_cast<int64_t>(f) * FD * FD;
  if (!a.frame_used[f]) {
    for (int e = lane; e < FD * FD; e += 32) out[e] = 0.0;
    return;
  }
  const Blocks& b = a.b[a.ctl->cur];
  const int G = a.dp.G, M = G + 1;
  frame_cov_block<FD>(b, a.D2x, f, a.scale + static_cast<int64_t>(f) * FD, a.X + static_cast<int64_t>(f) * FD * M, M, a.Sgg, G, lane, out);
}

// Frame f's blocks off the diagonal (vcgpu_get_frame_cross_covariance), unscaled, by one warp: P_f = X_f Σ_gg is formed
// once, and gives Σ_fg = -P_f and Σ_f,f+1 = P_f X_f+1^T (frame_cross_cov_vision_kernel, cov_frame_cross_mega_batch_kernel).
// Xf, Xn: X_f and X_f+1, [FD][ldx]; Xn null where frame f is the last or frame f+1 unused (its columns of fn are 0, as
// are the columns of fg where mask[q] is 0).  sf, sn, scg: the Jacobi scales of frames f, f+1 and of the globals.  fn
// null: frame f is the last.
template <int FD>
__device__ __forceinline__ void frame_cross_cov_block(const double* Xf, const double* Xn, int ldx, const double* Sgg, int G,
                                                      const double* sf, const double* sn, const double* scg, const double* mask,
                                                      int lane, double* fg, double* fn) {
  constexpr int kOwn = (FD * FD + 31) / 32;  // entry t of Σ_f,f+1 (row-major) is summed by lane t mod 32
  const int M = ldx;
  double own[kOwn];
#pragma unroll
  for (int i = 0; i < kOwn; ++i) own[i] = 0.0;
  for (int q0 = 0; q0 < G; q0 += 32) {  // the lanes split the columns q of P, 32 at a time
    const int q = q0 + lane;
    double p[FD];
#pragma unroll
    for (int r = 0; r < FD; ++r) p[r] = 0.0;
    if (q < G) {
      for (int k = 0; k < G; ++k) {
        const double s = Sgg[static_cast<int64_t>(k) * G + q];
#pragma unroll
        for (int r = 0; r < FD; ++r) p[r] += Xf[r * M + k] * s;
      }
      const bool free_q = mask[q] != 0.0;
      const double sq = scg[q];
#pragma unroll
      for (int r = 0; r < FD; ++r) fg[static_cast<int64_t>(r) * G + q] = free_q ? -(p[r] * (sf[r] * sq)) : 0.0;
    }
    if (Xn) {  // this tile's share of P X_f+1^T, summed over the warp one entry at a time (few registers held)
#pragma unroll
      for (int t = 0; t < FD * FD; ++t) {
        double v = q < G ? p[t / FD] * Xn[(t % FD) * M + q] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((t & 31) == lane) own[t >> 5] += v;
      }
    }
  }
  if (!fn) return;
#pragma unroll
  for (int t = 0; t < FD * FD; ++t)
    if ((t & 31) == lane) fn[t] = Xn ? own[t >> 5] * (sf[t / FD] * sn[t % FD]) : 0.0;
}

// the arguments of frame_cross_cov_vision_kernel: f.out is Σ_fg [nf][FD][G]
struct FrameCrossCovArgs {
  FrameCovArgs f;
  const double* mask;  // [G] 0: constant or unused global
  double* fn;          // [nf - 1][FD][FD] Σ_f,f+1
};
template <int FD>
__global__ void __launch_bounds__(32 * kFrameCovWarps) frame_cross_cov_vision_kernel(FrameCrossCovArgs a) {
  const int lane = threadIdx.x & 31, f = blockIdx.x * kFrameCovWarps + (threadIdx.x >> 5);
  const int nf = a.f.dp.n_frames, G = a.f.dp.G, M = G + 1;
  if (f >= nf) return;
  double* fg = a.f.out + static_cast<int64_t>(f) * FD * G;
  double* fn = f + 1 < nf ? a.fn + static_cast<int64_t>(f) * FD * FD : nullptr;
  if (!a.f.frame_used[f]) {
    for (int e = lane; e < FD * G; e += 32) fg[e] = 0.0;
    if (fn)
      for (int e = lane; e < FD * FD; e += 32) fn[e] = 0.0;
    return;
  }
  const double* Xn = fn && a.f.frame_used[f + 1] ? a.f.X + static_cast<int64_t>(f + 1) * FD * M : nullptr;
  const double* sf = a.f.scale + static_cast<int64_t>(f) * FD;
  frame_cross_cov_block<FD>(a.f.X + static_cast<int64_t>(f) * FD * M, Xn, M, a.f.Sgg, G, sf, sf + FD,
                            a.f.scale + static_cast<int64_t>(nf) * FD, a.mask, lane, fg, fn);
}

// ---------------------------------------------------------------- inertial: one CTA per chunk of a level
struct SelinvArgs {
  int G, c;
  ChainLevel cur;          // level l, as the elimination left it (A + addA, U, Z)
  SigmaLevel sig, up;      // level l's blocks (written) and level l+1's (read)
  const double* Sgg;       // Σ_gg, leading dimension ldg
  int ldg;
  double* scalars;
  // chain_selinv_kernel's NodeSrc of level l = lev[l] (level 0: the normal equations, with the damping in D2x)
  const ChainLevel* lev;
  int l, nf;
  Blocks b[2];
  const Ctl* ctl;
  const double* scale;
  const double* D2x;
};

// shared memory of one chunk of c nodes (chain_selinv_chunk): T [(c-1) FD]^2 | K [(c-1) FD]^2 | P [(c-1) FD][2 FD + G]
template <int FD>
__host__ __device__ inline size_t chain_selinv_smem_bytes(int G, int c) {
  const size_t nT = static_cast<size_t>(c - 1) * FD;
  return (2 * nT * nT + nT * (2 * FD + static_cast<size_t>(G))) * sizeof(double);
}

// entry (k, q) of the boundary covariance Σ_yy of chunk j, y = (node j, node j+1 of level l+1, globals).  Level l+1's
// blocks and Σ_gg are read through L2: in a cluster's walk other CTAs wrote them in the same launch.
template <int FD>
__device__ __forceinline__ double selinv_boundary(const SelinvArgs& a, int j, bool hasR, int k, int q) {
  const int G = a.G;
  const int bk = k < FD ? 0 : k < 2 * FD ? 1 : 2, bq = q < FD ? 0 : q < 2 * FD ? 1 : 2;
  if (!hasR && (bk == 1 || bq == 1)) return 0.0;
  if (bk == 2 && bq == 2) return __ldcg(a.Sgg + static_cast<int64_t>(k - 2 * FD) * a.ldg + (q - 2 * FD));
  if (bq == 2) return __ldcg(a.up.kg + static_cast<int64_t>(j + bk) * FD * G + (k - bk * FD) * G + (q - 2 * FD));
  if (bk == 2) return __ldcg(a.up.kg + static_cast<int64_t>(j + bq) * FD * G + (q - bq * FD) * G + (k - 2 * FD));
  if (bk == bq) return __ldcg(a.up.kk + static_cast<int64_t>(j + bk) * FD * FD + (k - bk * FD) * FD + (q - bq * FD));
  if (bk == 0) return __ldcg(a.up.kn + static_cast<int64_t>(j) * FD * FD + k * FD + (q - FD));
  return __ldcg(a.up.kn + static_cast<int64_t>(j) * FD * FD + q * FD + (k - FD));
}

// Chunk j of level l (separator s = j c, interior nodes s+1 .. s+m) by NT threads: this thread is `tid` of them, sync()
// is their barrier, sm their workspace (chain_selinv_smem_bytes), *bad their pivot flag.  node_A(p, e) and node_U(p, e)
// give entry e of H[p, p] and of H[p-1, p] at level l as the elimination saw them (A + addA and U, or at level 0,
// which the elimination reads on the fly, the scaled and damped normal equations: src_A, src_U).  The caller separates two chunks that
// share a workspace with sync().
template <int FD, int NT, class Sync, class NodeA, class NodeU>
__device__ __forceinline__ void chain_selinv_chunk(const SelinvArgs& a, int j, double* sm, int tid, int* bad, Sync sync, NodeA node_A,
                                                   NodeU node_U) {
  const int G = a.G, c = a.c, ny = 2 * FD + G, w = ny + 1;
  const ChainLevel& L = a.cur;
  const int s = j * c, n = L.n;
  const int m = min(c - 1, n - 1 - s);  // interior nodes s+1 .. s+m
  const bool hasR = s + c < n;          // right separator: node s+m+1 here, node j+1 at level l+1
  const int nT = m * FD;
  double* T = sm;           // [nT][nT] the interior's block-tridiagonal matrix, then its Cholesky factor
  double* K = T + nT * nT;  // [nT][nT] its inverse
  double* P = K + nT * nT;  // [m][FD][ny] M_p Σ_yy
  if (tid == 0) *bad = 0;
  for (int e = tid; e < nT * nT; e += NT) {
    const int r = e / nT, q = e - r * nT, br = r / FD, bq = q / FD, rr = r - br * FD, qq = q - bq * FD;
    const int64_t p = s + 1 + min(br, bq);
    double v = 0.0;
    if (br == bq) v = node_A(p, rr * FD + qq);
    else if (bq == br + 1) v = node_U(p + 1, rr * FD + qq);  // H[p, p+1]
    else if (br == bq + 1) v = node_U(p + 1, qq * FD + rr);  // H[p+1, p] = H[p, p+1]^T
    T[e] = v;
  }
  for (int e = tid; e < nT * ny; e += NT) {
    const int rp = e / ny, q = e - rp * ny;  // rp = i FD + r
    const double* z = L.Z + (static_cast<int64_t>(s + 1) * FD + rp) * w;
    double sum = 0.0;
    for (int k = 0; k < ny; ++k) sum += z[k] * selinv_boundary<FD>(a, j, hasR, k, q);
    P[e] = sum;
  }
  sync();
  for (int jj = 0; jj < nT; ++jj) {  // T = L L^T, in place (lower triangle)
    if (tid == 0) {
      double d = T[jj * nT + jj];
      if (!(d > 0.0)) { *bad = 1; d = 1.0; }
      T[jj * nT + jj] = sqrt(d);
    }
    sync();
    const double dj = T[jj * nT + jj];
    for (int i = jj + 1 + tid; i < nT; i += NT) T[i * nT + jj] /= dj;
    sync();
    const int rem = nT - jj - 1;
    for (int e = tid; e < rem * rem; e += NT) {
      const int i = jj + 1 + e / rem, k = jj + 1 + e % rem;
      if (k <= i) T[i * nT + k] -= T[i * nT + jj] * T[k * nT + jj];
    }
    sync();
  }
  for (int col = tid; col < nT; col += NT) {  // K = T^-1, one column per thread
    for (int i = col; i < nT; ++i) {
      double t = i == col ? 1.0 : 0.0;
      for (int k = col; k < i; ++k) t -= T[i * nT + k] * K[k * nT + col];
      K[i * nT + col] = t / T[i * nT + i];
    }
    for (int i = nT - 1; i >= 0; --i) {
      double t = i >= col ? K[i * nT + col] : 0.0;
      for (int k = i + 1; k < nT; ++k) t -= T[k * nT + i] * K[k * nT + col];
      K[i * nT + col] = t / T[i * nT + i];
    }
  }
  sync();
  if (*bad && tid == 0) a.scalars[kScNotPD] = 1.0;
  // the interior nodes: Σ_pp, Σ_p,p+1 (p+1 interior, or the right separator: -M_p Σ_y,right), Σ_pg = -(M_p Σ_yy)[:, g]
  for (int e = tid; e < m * FD * FD; e += NT) {
    const int i = e / (FD * FD), r = (e / FD) % FD, q = e % FD;
    const int64_t p = s + 1 + i;
    const double* Pr = P + (i * FD + r) * ny;
    const double* zq = L.Z + (p * FD + q) * w;
    double kk = K[(i * FD + r) * nT + i * FD + q];
    for (int k = 0; k < ny; ++k) kk += Pr[k] * zq[k];
    double kn = 0.0;
    if (i + 1 < m) {
      const double* zn = L.Z + ((p + 1) * FD + q) * w;
      kn = K[(i * FD + r) * nT + (i + 1) * FD + q];
      for (int k = 0; k < ny; ++k) kn += Pr[k] * zn[k];
    } else if (hasR) {
      kn = -Pr[FD + q];
    }
    a.sig.kk[p * FD * FD + r * FD + q] = kk;
    a.sig.kn[p * FD * FD + r * FD + q] = kn;
  }
  for (int e = tid; e < m * FD * G; e += NT) {
    const int i = e / (FD * G), r = (e / G) % FD, q = e % G;
    a.sig.kg[(static_cast<int64_t>(s + 1 + i) * FD + r) * G + q] = -P[(i * FD + r) * ny + 2 * FD + q];
  }
  // the chunk's left separator: node j of level l+1; its next node is the first interior one (or the right separator)
  for (int e = tid; e < FD * FD; e += NT) {
    const int r = e / FD, q = e % FD;
    a.sig.kk[static_cast<int64_t>(s) * FD * FD + e] = __ldcg(a.up.kk + static_cast<int64_t>(j) * FD * FD + e);
    a.sig.kn[static_cast<int64_t>(s) * FD * FD + e] =
        m > 0 ? -P[q * ny + r] : (hasR ? __ldcg(a.up.kn + static_cast<int64_t>(j) * FD * FD + e) : 0.0);
  }
  for (int e = tid; e < FD * G; e += NT)
    a.sig.kg[static_cast<int64_t>(s) * FD * G + e] = __ldcg(a.up.kg + static_cast<int64_t>(j) * FD * G + e);
}

// One CTA per chunk of level l (vcgpu_get_frame_covariance), its nodes read as chain_frame_cov_batch_kernel's walk reads
// them: the call refuses frame shards, so level 0 has neither a ghost nor a separator's summed diagonal
template <int FD>
__global__ void __launch_bounds__(kChainThreads) chain_selinv_kernel(SelinvArgs a) {
  extern __shared__ double sm[];
  __shared__ int bad;
  NodeSrc src;
  src.L = a.l > 0 ? a.lev + a.l : nullptr;
  src.b = a.b[a.ctl->cur]; src.scale = a.scale; src.D2x = a.D2x; src.rinv = 0.0; src.G = a.G; src.nf = a.nf;
  src.sepdiag = nullptr; src.rank = 0; src.ghost = 0;
  chain_selinv_chunk<FD, kChainThreads>(
      a, blockIdx.x, sm, threadIdx.x, &bad, [] { __syncthreads(); }, [&](int64_t p, int e) { return src_A<FD>(src, p, e); },
      [&](int64_t p, int e) { return src_U<FD>(src, p, e); });
}

// Level 0's Σ_ff unscaled, s_f Σ_ff s_f, and exactly symmetric: both halves are written from the lower triangle.  Rows
// and columns from `live` on (the velocities of a rotation-only run, which no residual reads) are 0.
template <int FD>
__device__ __forceinline__ double frame_cov_out_entry(int64_t e, int live, const double* kk, const double* scale) {
  const int64_t f = e / (FD * FD);
  const int r = static_cast<int>((e / FD) % FD), q = static_cast<int>(e % FD), hi = max(r, q), lo = min(r, q);
  return hi < live ? kk[f * FD * FD + hi * FD + lo] * (scale[f * FD + hi] * scale[f * FD + lo]) : 0.0;
}
template <int FD>
__global__ void __launch_bounds__(256) frame_cov_out_kernel(int n_frames, int live, const double* kk, const double* scale,
                                                            double* out) {
  const int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= static_cast<int64_t>(n_frames) * FD * FD) return;
  out[e] = frame_cov_out_entry<FD>(e, live, kk, scale);
}

// Level 0's blocks off the diagonal (vcgpu_get_frame_cross_covariance), unscaled: entry e of Σ_fg [nf][FD][G] (e below
// nf FD G) or of Σ_f,f+1 [nf - 1][FD][FD] (the entries after).  Rows and columns of a frame from `live` on, and the
// columns of constant or unused globals (mask 0), are 0.
template <int FD>
__device__ __forceinline__ void frame_cross_cov_out_entry(int64_t e, int nf, int G, int live, const SigmaLevel& sig, const double* scale,
                                                          const double* mask, double* fg, double* fn) {
  const int64_t ng = static_cast<int64_t>(nf) * FD * G;
  if (e < ng) {
    const int64_t f = e / (FD * G);
    const int r = static_cast<int>((e / G) % FD), q = static_cast<int>(e % G);
    fg[e] = r < live && mask[q] != 0.0 ? sig.kg[e] * (scale[f * FD + r] * scale[static_cast<int64_t>(nf) * FD + q]) : 0.0;
  } else {
    const int64_t k = e - ng, f = k / (FD * FD);
    const int r = static_cast<int>((k / FD) % FD), c = static_cast<int>(k % FD);
    fn[k] = r < live && c < live ? sig.kn[k] * (scale[f * FD + r] * scale[(f + 1) * FD + c]) : 0.0;
  }
}
template <int FD>
__host__ __device__ inline int64_t frame_cross_cov_entries(int nf, int G) {
  return static_cast<int64_t>(nf) * FD * G + static_cast<int64_t>(nf - 1) * FD * FD;
}
template <int FD>
__global__ void __launch_bounds__(256) frame_cross_cov_out_kernel(int nf, int G, int live, SigmaLevel sig, const double* scale,
                                                                  const double* mask, double* fg, double* fn) {
  const int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= frame_cross_cov_entries<FD>(nf, G)) return;
  frame_cross_cov_out_entry<FD>(e, nf, G, live, sig, scale, mask, fg, fn);
}

}  // namespace vc
