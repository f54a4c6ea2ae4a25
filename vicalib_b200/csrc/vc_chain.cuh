// Block-tridiagonal + arrow solve for the inertial problem.
//
// With IMU factors the frame block of J^T J is block tridiagonal (each factor couples frames j-1, j;
// vicalibrator.h:628-632) and every frame also couples to the dense global block.  The reference
// hands this to a sparse Cholesky inside ceres::Solve.  Here the chain is eliminated by recursive
// partitioning: every c-th node of a level is a separator, the c-1 nodes between two separators are
// eliminated by one CTA (block Thomas sweep with the couplings to both separators, the global columns
// and the gradient as right-hand sides), which leaves a chain of separators c times shorter.  After
// ~log_c(n) levels the few remaining nodes join the globals in one dense Cholesky; back-substitution
// walks the levels in reverse.  The same structure shards across GPUs (a rank's first frame is a
// separator at every level), which is why it is preferred to a sequential sweep.
//
// Here: the level descriptors, where a level's node blocks come from (NodeSrc: level 0 straight from the normal
// equations), the Schur partials' sum and the dense solve of the multi-launch engine.  The chunk elimination and the
// back-substitution of a node have one definition, chain_eliminate_chunk and chain_backsub_node (vc_imu_mega.cuh), which
// the persistent kernels and the multi-launch engine's chain_eliminate_kernel / chain_backsub_kernel all run.
#pragma once
#include "vc_internal.h"
#include "vc_kernels.cuh"

namespace vc {

struct ChainLevel {
  int n;                        // nodes at this level (including the ghost, if any)
  int ghost;                    // 1: the last node is the next rank's first frame: a forced separator, never eliminated
  double *A, *U, *E, *g;        // node blocks: A[n][FD*FD], U[i] = H[i-1,i], E[n][FD*G], g[n][FD]
  double *addA, *addE, *addg;   // Schur contributions from the chunk on the node's left (null on level 0)
  double* Z;                    // [n][FD][2FD+G+1]: eliminated nodes' solutions against [L | R | E | g]
  int32_t* orig;                // original frame index of each node
};

constexpr int kChainThreads = 128;

// where a level's node blocks come from: level 0 reads the block normal equations and applies the Jacobi scaling and
// the LM damping on the fly (no separate pass, no copy); deeper levels read what the level above left
struct NodeSrc {
  const ChainLevel* L;   // level >= 1 (null at level 0)
  Blocks b;              // level 0
  const double* scale;
  const double* D2x;
  double rinv;
  int G, nf;
  const double* sepdiag;  // sharded: summed diagonal of the ranks' first frames (damping of frame 0; the ghost is damped by its owner)
  int rank, ghost;
};
template <int FD>
__device__ __forceinline__ double src_A(const NodeSrc& s, int64_t p, int e) {
  if (s.L) return s.L->A[p * FD * FD + e] + (s.L->addA ? s.L->addA[p * FD * FD + e] : 0.0);
  const int r = e / FD, c = e - r * FD;
  const double* sf = s.scale + p * FD;
  const double bij = s.b.B[p * FD * FD + e];
  double v = bij * sf[r] * sf[c];
  // frame_damp's rule, written out: through frame_damp the compiler fuses this add differently and the solve's bits change
  if (r == c) {
    const bool is_ghost = s.ghost && p == s.nf - 1;
    if (is_ghost) ;  // damped once, by the rank that owns the frame
    else if (s.D2x) v += s.D2x[p * FD + r];
    else if (s.sepdiag && p == 0) v += lm_damp(s.sepdiag[s.rank * FD + r], sf[r], s.rinv);
    else v += lm_damp(bij, sf[r], s.rinv);
  }
  return v;
}
template <int FD>
__device__ __forceinline__ double src_U(const NodeSrc& s, int64_t p, int e) {  // H[p-1, p]
  if (s.L) return s.L->U[p * FD * FD + e];
  if (p == 0) return 0.0;
  const int r = e / FD, c = e - r * FD;
  return s.b.U[p * FD * FD + e] * s.scale[(p - 1) * FD + r] * s.scale[p * FD + c];
}
template <int FD>
__device__ __forceinline__ double src_E(const NodeSrc& s, int64_t p, int r, int c) {
  const int e = r * s.G + c;
  if (s.L) return s.L->E[p * FD * s.G + e] + (s.L->addE ? s.L->addE[p * FD * s.G + e] : 0.0);
  return s.b.E[p * FD * s.G + e] * s.scale[p * FD + r] * s.scale[static_cast<int64_t>(s.nf) * FD + c];
}
template <int FD>
__device__ __forceinline__ double src_g(const NodeSrc& s, int64_t p, int e) {
  if (s.L) return s.L->g[p * FD + e] + (s.L->addg ? s.L->addg[p * FD + e] : 0.0);
  return s.b.gf[p * FD + e] * s.scale[p * FD + e];
}
// the NodeSrc of level L (null: level 0) at the point the iteration is at (bs[ctl->cur], damped at ctl's radius)
__device__ __forceinline__ NodeSrc chain_src(const ChainLevel* L, const DevProblem& dp, const Blocks* bs, const Ctl* ctl,
                                             const double* scale, const double* D2x, const double* sepdiag) {
  NodeSrc s;
  s.L = L; s.b = bs[ctl->cur]; s.scale = scale; s.D2x = D2x; s.rinv = 1.0 / ctl->radius; s.G = dp.G; s.nf = dp.n_frames;
  s.sepdiag = sepdiag; s.rank = dp.rank; s.ghost = dp.ghost;
  return s;
}

// dynamic shared memory of dense_solve_kernel when it factors (src 0 and 2): S [N^2] | rhs [N]
__host__ inline size_t chain_dense_smem_bytes(int N) { return (static_cast<size_t>(N) * N + N) * sizeof(double); }

// sum of per-CTA partials (coalesced across entries), into out0 or, with `which` >= 0, into whichever of out0 / out1
// belongs to the buffer `which` picks on the device ([C | gc] of the point being evaluated, contiguous in Blocks)
// launch with 256 threads: 32 entries per CTA, 8 partial-slices per entry, fixed summation order
__global__ void __launch_bounds__(256) sum_partials_kernel(const double* part, int n_part, int NS, double* out0, double* out1,
                                                           const Ctl* ctl, int which) {
  __shared__ double sh[8][33];
  if (ctl->done) return;
  double* out = which >= 0 && pick(ctl, which) ? out1 : out0;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int e = blockIdx.x * 32 + tx;
  double s = 0.0;
  if (e < NS) {
    double s1 = 0.0, s2 = 0.0, s3 = 0.0;
    int b = ty;
    for (; b + 24 < n_part; b += 32) {
      s += part[static_cast<int64_t>(b) * NS + e];
      s1 += part[static_cast<int64_t>(b + 8) * NS + e];
      s2 += part[static_cast<int64_t>(b + 16) * NS + e];
      s3 += part[static_cast<int64_t>(b + 24) * NS + e];
    }
    for (; b < n_part; b += 8) s += part[static_cast<int64_t>(b) * NS + e];
    s = (s + s1) + (s2 + s3);
  }
  sh[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && e < NS) {
    double t = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += sh[k][tx];
    out[e] = t;
  }
}

// Blocks of the inverse of a level's system (vcgpu_get_frame_covariance, vc_frame_cov.cuh), in the scaled system: per
// node Σ_kk [n][FD*FD], Σ_k,k+1 [n][FD*FD] (zero for the last node) and Σ_kg [n][FD*G]
struct SigmaLevel {
  double *kk, *kn, *kg;
};

// dense solve of [globals | top-level chain nodes]
struct DenseArgs {
  DevProblem dp;
  Blocks bs[2];
  const Ctl* ctl;
  const double* scale;
  const double* D2x;
  const double* sepdiag;  // sharded: the ranks' first frames' summed diagonal (NodeSrc)
  const double* Ssum;  // [G*G+G] summed Schur partials
  ChainLevel top;      // n may be 0
  const ChainLevel* lev;  // the level table (device memory), top = lev[n_levels - 1]; n_levels 1: the top nodes are
  int n_levels;           // level 0, read from the normal equations (NodeSrc)
  double* delta;
  double* scalars;
  int n_slots;         // frame blocks in the dense system (single GPU: top.n; sharded: one per rank)
  int slot_of[4];      // dense slot of each local top node
  int add_globals;     // 1: this rank contributes C + D and -g_c (exactly one rank does)
  int src;             // the system: 0 assembled here; 1 this rank's partial assembled into buf, and nothing else done;
                       // 2 loaded from buf (the ranks' partials summed)
  double* buf;         // [N*N + N], N = G + n_slots*FD
  double* inv;         // null: solve into delta; else invert: the whole inverse into inv [N*N] ...
  SigmaLevel sig;      // ... and, where sig.kk is set, the top nodes' blocks of it into sig
};
template <int FD>
__global__ void __launch_bounds__(256) dense_solve_kernel(DenseArgs a) {
  extern __shared__ double sm[];
  const int G = a.dp.G, nt = a.top.n, N = G + a.n_slots * FD, tid = threadIdx.x;
  double* S = a.src == 1 ? a.buf : sm;               // [N*N]
  double* rhs = S + N * N;
  __shared__ int bad;
  if (a.ctl->done) return;
  const Blocks& b = a.bs[a.ctl->cur];
  const double rinv = 1.0 / a.ctl->radius;
  if (tid == 0) bad = 0;
  const int64_t nfp = static_cast<int64_t>(a.dp.n_frames) * a.dp.fd;
  const double* sc = a.scale + nfp;
  if (a.src == 2) {
    for (int e = tid; e < N * N + N; e += 256) S[e] = a.buf[e];
  } else {
    for (int e = tid; e < N * N + N; e += 256) S[e] = 0.0;
    __syncthreads();
    for (int e = tid; e < G * G + G; e += 256) {
      if (e < G * G) {
        const int r = e / G, c = e - r * G;
        double v = -a.Ssum[e];
        if (a.add_globals) {
          v += b.C[e] * sc[r] * sc[c];
          if (r == c) v += global_damp(r, b.C[e], sc[r], rinv, a.D2x, nfp);
        }
        S[r * N + c] = v;
      } else {
        const int r = e - G * G;
        rhs[r] = (a.add_globals ? -b.gc[r] * sc[r] : 0.0) + a.Ssum[e];
      }
    }
    const NodeSrc src = chain_src(a.n_levels > 1 ? a.lev + a.n_levels - 1 : nullptr, a.dp, a.bs, a.ctl, a.scale, a.D2x, a.sepdiag);
    for (int t = 0; t < nt; ++t) {
      const int o = G + a.slot_of[t] * FD;
      for (int e = tid; e < FD * FD; e += 256) {
        const int r = e / FD, c = e - r * FD;
        S[(o + r) * N + o + c] = src_A<FD>(src, t, e);
        if (t > 0) {
          const int op = G + a.slot_of[t - 1] * FD;
          const double u = src_U<FD>(src, t, e);  // H[t-1, t]
          S[(op + r) * N + o + c] = u;
          S[(o + c) * N + op + r] = u;
        }
      }
      for (int e = tid; e < FD * G; e += 256) {
        const int r = e / G, c = e - r * G;
        const double v = src_E<FD>(src, t, r, c);
        S[(o + r) * N + c] = v;
        S[c * N + o + r] = v;
      }
      for (int e = tid; e < FD; e += 256) rhs[o + e] = -src_g<FD>(src, t, e);
    }
  }
  if (a.src == 1) return;
  __syncthreads();
  for (int j = 0; j < N; ++j) {
    if (tid == 0) {
      double d = S[j * N + j];
      if (!(d > 0.0)) { bad = 1; d = 1.0; }
      S[j * N + j] = sqrt(d);
    }
    __syncthreads();
    const double dj = S[j * N + j];
    for (int i = j + 1 + tid; i < N; i += 256) S[i * N + j] /= dj;
    __syncthreads();
    const int rem = N - j - 1;
    for (int e = tid; e < rem * rem; e += 256) {
      const int i = j + 1 + e / rem, k = j + 1 + e % rem;
      if (k <= i) S[i * N + k] -= S[i * N + j] * S[k * N + j];
    }
    __syncthreads();
  }
  if (a.inv) {
    // N unit right-hand sides through the factor, one column per thread: L y = e_j (y is zero above row j), L^T x = y
    double* X = a.inv;
    for (int j = tid; j < N; j += 256) {
      for (int i = j; i < N; ++i) {
        double t = i == j ? 1.0 : 0.0;
        for (int k = j; k < i; ++k) t -= S[i * N + k] * X[static_cast<int64_t>(k) * N + j];
        X[static_cast<int64_t>(i) * N + j] = t / S[i * N + i];
      }
      for (int i = N - 1; i >= 0; --i) {
        double t = i >= j ? X[static_cast<int64_t>(i) * N + j] : 0.0;
        for (int k = i + 1; k < N; ++k) t -= S[k * N + i] * X[static_cast<int64_t>(k) * N + j];
        X[static_cast<int64_t>(i) * N + j] = t / S[i * N + i];
      }
    }
    __syncthreads();
    if (bad && tid == 0) a.scalars[kScNotPD] = 1.0;
    if (!a.sig.kk) return;
    for (int e = tid; e < nt * FD * FD; e += 256) {
      const int t = e / (FD * FD), r = (e / FD) % FD, q = e % FD, o = G + a.slot_of[t] * FD;
      a.sig.kk[e] = X[static_cast<int64_t>(o + r) * N + o + q];
      a.sig.kn[e] = t + 1 < nt ? X[static_cast<int64_t>(o + r) * N + G + a.slot_of[t + 1] * FD + q] : 0.0;
    }
    for (int e = tid; e < nt * FD * G; e += 256) {
      const int t = e / (FD * G), r = (e / G) % FD, q = e % G, o = G + a.slot_of[t] * FD;
      a.sig.kg[e] = X[static_cast<int64_t>(o + r) * N + q];
    }
    return;
  }
  if (tid < 32) {  // warp-cooperative triangular solves (column oriented), L L^T x = rhs
    const int lane = tid;
    for (int i = 0; i < N; ++i) {
      const double xi = rhs[i] / S[i * N + i];
      __syncwarp();
      if (lane == 0) rhs[i] = xi;
      for (int k = i + 1 + lane; k < N; k += 32) rhs[k] -= S[k * N + i] * xi;
      __syncwarp();
    }
    for (int i = N - 1; i >= 0; --i) {
      const double xi = rhs[i] / S[i * N + i];
      __syncwarp();
      if (lane == 0) rhs[i] = xi;
      for (int k = lane; k < i; k += 32) rhs[k] -= S[i * N + k] * xi;
      __syncwarp();
    }
    if (bad && lane == 0) a.scalars[kScNotPD] = 1.0;
  }
  __syncthreads();
  for (int i = tid; i < G; i += 256) a.delta[nfp + i] = bad ? 0.0 : rhs[i];
  for (int e = tid; e < nt * FD; e += 256) {
    const int t = e / FD, r = e - t * FD;
    a.delta[static_cast<int64_t>(a.n_levels > 1 ? a.top.orig[t] : t) * FD + r] = bad ? 0.0 : rhs[G + a.slot_of[t] * FD + r];
  }
}

}  // namespace vc
