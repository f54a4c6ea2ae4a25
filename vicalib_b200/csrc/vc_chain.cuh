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
#pragma once
#include "vc_internal.h"

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

// level 0 from the block normal equations: scaled + damped
template <int FD>
__global__ void chain_init_kernel(DevProblem dp, Blocks b0, Blocks b1, const Ctl* ctl, const double* scale,
                                  const double* D2x, ChainLevel L, const double* sepdiag) {
  if (ctl->done) return;
  const Blocks& b = ctl->cur ? b1 : b0;
  const double rinv = 1.0 / ctl->radius;
  const int G = dp.G, f = blockIdx.x, tid = threadIdx.x;
  // sharded chain: a rank's first frame (and its ghost copy on the previous rank) is damped once, by its
  // owner, from the diagonal summed over both ranks; sepdiag[slot*FD + r]
  const bool sep = sepdiag != nullptr && (f == 0 || (dp.ghost && f == dp.n_frames - 1));
  const bool is_ghost = dp.ghost && f == dp.n_frames - 1;
  const double* sd = sep ? sepdiag + (dp.rank + (is_ghost ? 1 : 0)) * FD : nullptr;
  const double* sf = scale + static_cast<int64_t>(f) * FD;
  const double* sc = scale + static_cast<int64_t>(dp.n_frames) * FD;
  for (int e = tid; e < FD * FD; e += blockDim.x) {
    const int r = e / FD, c = e - r * FD;
    const double bij = b.B[static_cast<int64_t>(f) * FD * FD + e];
    double v = bij * sf[r] * sf[c];
    if (r == c) {
      if (D2x) v += D2x[static_cast<int64_t>(f) * FD + r];
      else if (!sep) v += lm_damp(bij, sf[r], rinv);
      else if (!is_ghost) v += lm_damp(sd[r], sf[r], rinv);
    }
    L.A[static_cast<int64_t>(f) * FD * FD + e] = v;
    double u = 0.0;
    if (f > 0) u = b.U[static_cast<int64_t>(f) * FD * FD + e] * scale[static_cast<int64_t>(f - 1) * FD + r] * sf[c];
    L.U[static_cast<int64_t>(f) * FD * FD + e] = u;
  }
  for (int e = tid; e < FD * G; e += blockDim.x) {
    const int r = e / G, c = e - r * G;
    L.E[static_cast<int64_t>(f) * FD * G + e] = b.E[static_cast<int64_t>(f) * FD * G + e] * sf[r] * sc[c];
  }
  for (int e = tid; e < FD; e += blockDim.x) L.g[static_cast<int64_t>(f) * FD + e] = b.gf[static_cast<int64_t>(f) * FD + e] * sf[e];
  if (tid == 0) L.orig[f] = f;
}

// dynamic shared memory of chain_eliminate_kernel<FD> with chunks of c nodes:
// Sacc [G^2 + G] | Al [FD^2] | El [FD G] | gl [FD] | Ap [FD^2] | Uc [FD^2] | V [(c - 1) FD][FD + 2 FD + G + 1]
template <int FD>
__host__ inline size_t chain_eliminate_smem_bytes(int G, int c) {
  const size_t g = static_cast<size_t>(G), w = 2 * FD + g + 1;
  return (g * g + g + 3 * FD * FD + FD * g + FD + static_cast<size_t>(c - 1) * FD * (FD + w)) * sizeof(double);
}
// dynamic shared memory of dense_solve_kernel when it factors (modes 0 and 2): S [N^2] | rhs [N]
__host__ inline size_t chain_dense_smem_bytes(int N) { return (static_cast<size_t>(N) * N + N) * sizeof(double); }

struct ElimArgs {
  int G, c;
  const Ctl* ctl;
  ChainLevel cur, next;
  double* Spart;  // [gridDim][G*G+G]
  double* scalars;
};

template <int FD>
__global__ void __launch_bounds__(kChainThreads, 4) chain_eliminate_kernel(ElimArgs a) {
  extern __shared__ double sm[];
  const int G = a.G, c = a.c, tid = threadIdx.x, NS = G * G + G;
  const int w = 2 * FD + G + 1, VW = FD + w;
  const int oL = FD, oR = 2 * FD, oE = 3 * FD, og = 3 * FD + G;  // column offsets inside a V row
  double* Sacc = sm;                       // [NS]
  double* Al = Sacc + NS;                  // [FD*FD]
  double* El = Al + FD * FD;               // [FD*G]
  double* gl = El + FD * G;                // [FD]
  double* Ap = gl + FD;                    // [FD*FD] pivot / its Cholesky factor
  double* Uc = Ap + FD * FD;               // [FD*FD] U[p]
  double* V = Uc + FD * FD;                // [(c-1)][FD][VW]
  __shared__ int bad;
  if (a.ctl->done) return;
  const ChainLevel& L = a.cur;
  const int j = blockIdx.x, s = j * c, n_eff = L.n - L.ghost;
  const int nsep = (n_eff + c - 1) / c;
  const bool toGhost = L.ghost && !(s + c < n_eff);  // this chunk's right separator is the ghost node
  const bool hasR = s + c < n_eff || toGhost;
  const int m = min(c - 1, n_eff - 1 - s);            // interior nodes s+1 .. s+m
  const int rIdx = s + m + 1;                         // right separator at this level (when hasR)
  const int jr = toGhost ? nsep : j + 1;              // ... and its index at the next level
  const bool add = L.addA != nullptr;
  if (tid == 0) bad = 0;
  for (int e = tid; e < NS; e += kChainThreads) Sacc[e] = 0.0;
  for (int e = tid; e < FD * FD; e += kChainThreads)
    Al[e] = L.A[static_cast<int64_t>(s) * FD * FD + e] + (add ? L.addA[static_cast<int64_t>(s) * FD * FD + e] : 0.0);
  for (int e = tid; e < FD * G; e += kChainThreads)
    El[e] = L.E[static_cast<int64_t>(s) * FD * G + e] + (add ? L.addE[static_cast<int64_t>(s) * FD * G + e] : 0.0);
  for (int e = tid; e < FD; e += kChainThreads)
    gl[e] = L.g[static_cast<int64_t>(s) * FD + e] + (add ? L.addg[static_cast<int64_t>(s) * FD + e] : 0.0);
  __syncthreads();
  // ---- forward sweep
  for (int i = 0; i < m; ++i) {
    const int64_t p = s + 1 + i;
    double* Vi = V + static_cast<int64_t>(i) * FD * VW;
    for (int e = tid; e < FD * FD; e += kChainThreads) {
      const int r = e / FD, q = e - r * FD;
      Ap[e] = L.A[p * FD * FD + e] + (add ? L.addA[p * FD * FD + e] : 0.0);
      Uc[e] = L.U[p * FD * FD + e];
      const bool lastI = i == m - 1;
      const double unext = (!lastI || hasR) ? L.U[(p + 1) * FD * FD + e] : 0.0;  // H[p, p+1]
      Vi[r * VW + q] = lastI ? 0.0 : unext;
      Vi[r * VW + oR + q] = (lastI && hasR) ? unext : 0.0;
      Vi[r * VW + oL + q] = i == 0 ? L.U[p * FD * FD + q * FD + r] : 0.0;  // H[p0, s] = U[p0]^T
    }
    for (int e = tid; e < FD * G; e += kChainThreads) {
      const int r = e / G, q = e - r * G;
      Vi[r * VW + oE + q] = L.E[p * FD * G + e] + (add ? L.addE[p * FD * G + e] : 0.0);
    }
    for (int e = tid; e < FD; e += kChainThreads) Vi[e * VW + og] = L.g[p * FD + e] + (add ? L.addg[p * FD + e] : 0.0);
    __syncthreads();
    if (i > 0) {
      const double* Vp = V + static_cast<int64_t>(i - 1) * FD * VW;
      // A'_i = A_i - U^T V_U(i-1);  R'_i = R_i - U^T V_R(i-1)
      for (int e = tid; e < FD * VW; e += kChainThreads) {
        const int r = e / VW, q = e - r * VW;
        double sum = 0.0;
#pragma unroll
        for (int k = 0; k < FD; ++k) sum += Uc[k * FD + r] * Vp[k * VW + q];
        if (q < FD) Ap[r * FD + q] -= sum;
        else Vi[r * VW + q] -= sum;
      }
      __syncthreads();
    }
    if (tid < VW) {
      // every column-solving thread factors the FD x FD pivot in registers (no serial section, no barrier)
      double Lr[FD][FD], iL[FD];
#pragma unroll
      for (int ii = 0; ii < FD; ++ii)
#pragma unroll
        for (int k = 0; k <= ii; ++k) Lr[ii][k] = Ap[ii * FD + k];
      bool ok = true;
#pragma unroll
      for (int jj = 0; jj < FD; ++jj) {
        double d = Lr[jj][jj];
#pragma unroll
        for (int k = 0; k < jj; ++k) d -= Lr[jj][k] * Lr[jj][k];
        if (!(d > 0.0)) { ok = false; d = 1.0; }
        d = sqrt(d);
        Lr[jj][jj] = d;
        const double inv = 1.0 / d;
        iL[jj] = inv;
#pragma unroll
        for (int ii = jj + 1; ii < FD; ++ii) {
          double t = Lr[ii][jj];
#pragma unroll
          for (int k = 0; k < jj; ++k) t -= Lr[ii][k] * Lr[jj][k];
          Lr[ii][jj] = t * inv;
        }
      }
      if (!ok && tid == 0) bad = 1;
      for (int q = tid; q < VW; q += kChainThreads) {
        double x[FD];
#pragma unroll
        for (int ii = 0; ii < FD; ++ii) {
          double t = Vi[ii * VW + q];
#pragma unroll
          for (int k = 0; k < ii; ++k) t -= Lr[ii][k] * x[k];
          x[ii] = t * iL[ii];
        }
#pragma unroll
        for (int ii = FD - 1; ii >= 0; --ii) {
          double t = x[ii];
#pragma unroll
          for (int k = ii + 1; k < FD; ++k) t -= Lr[k][ii] * x[k];
          x[ii] = t * iL[ii];
        }
#pragma unroll
        for (int ii = 0; ii < FD; ++ii) Vi[ii * VW + q] = x[ii];
      }
    }
    __syncthreads();
  }
  // ---- backward sweep: X_i = V_R(i) - V_U(i) X_{i+1}
  for (int i = m - 2; i >= 0; --i) {
    double* Vi = V + static_cast<int64_t>(i) * FD * VW;
    const double* Vn = V + static_cast<int64_t>(i + 1) * FD * VW;
    for (int e = tid; e < FD * w; e += kChainThreads) {
      const int r = e / w, q = FD + (e - r * w);
      double sum = 0.0;
#pragma unroll
      for (int k = 0; k < FD; ++k) sum += Vi[r * VW + k] * Vn[k * VW + q];
      Vi[r * VW + q] -= sum;
    }
    __syncthreads();
  }
  // ---- store Z, accumulate the Schur terms
  for (int i = 0; i < m; ++i) {
    const int64_t p = s + 1 + i;
    const double* Vi = V + static_cast<int64_t>(i) * FD * VW;
    for (int e = tid; e < FD * w; e += kChainThreads) {
      const int r = e / w, q = e - r * w;
      L.Z[(p * FD + r) * w + q] = Vi[r * VW + FD + q];
    }
    // S += E_i^T X_i[E], rhs += E_i^T X_i[g]  (E_i = the node's own global coupling)
    for (int e = tid; e < NS; e += kChainThreads) {
      const int ra = e < G * G ? e / G : e - G * G;
      const int cb = e < G * G ? oE + (e - ra * G) : og;
      double sum = 0.0;
#pragma unroll
      for (int k = 0; k < FD; ++k) {
        const double ek = L.E[p * FD * G + k * G + ra] + (add ? L.addE[p * FD * G + k * G + ra] : 0.0);
        sum += ek * Vi[k * VW + cb];
      }
      Sacc[e] += sum;
    }
  }
  if (m > 0) {
    const double* X0 = V;                                          // node s+1
    const double* Xl = V + static_cast<int64_t>(m - 1) * FD * VW;  // last interior node
    const double* U0 = L.U + static_cast<int64_t>(s + 1) * FD * FD;  // H[s, s+1]
    const double* Ur = hasR ? L.U + static_cast<int64_t>(rIdx) * FD * FD : nullptr;  // H[rIdx-1, rIdx]
    __syncthreads();
    for (int e = tid; e < FD * w; e += kChainThreads) {
      const int r = e / w, q = e - r * w;  // q indexes [L | R | E | g]
      double sl = 0.0, sr = 0.0;
#pragma unroll
      for (int k = 0; k < FD; ++k) {
        sl += U0[r * FD + k] * X0[k * VW + FD + q];
        if (hasR) sr += Ur[k * FD + r] * Xl[k * VW + FD + q];
      }
      if (q < FD) {
        Al[r * FD + q] -= sl;                                        // A_s -= H[s,p0] Z_L
      } else if (q < 2 * FD) {
        if (hasR) {
          a.next.U[static_cast<int64_t>(jr) * FD * FD + r * FD + (q - FD)] = -sl;     // fill H[s, rIdx]
          a.next.addA[static_cast<int64_t>(jr) * FD * FD + r * FD + (q - FD)] = -sr;  // A_r -= H[r,pl] Z_R
        }
      } else if (q < 2 * FD + G) {
        El[r * G + (q - 2 * FD)] -= sl;
        if (hasR) a.next.addE[static_cast<int64_t>(jr) * FD * G + r * G + (q - 2 * FD)] = -sr;
      } else {
        gl[r] -= sl;
        if (hasR) a.next.addg[static_cast<int64_t>(jr) * FD + r] = -sr;
      }
    }
  } else if (hasR) {
    // no interior node between this separator and the ghost: the coupling passes through unchanged
    for (int e = tid; e < FD * FD; e += kChainThreads) {
      a.next.U[static_cast<int64_t>(jr) * FD * FD + e] = L.U[static_cast<int64_t>(rIdx) * FD * FD + e];
      a.next.addA[static_cast<int64_t>(jr) * FD * FD + e] = 0.0;
    }
    for (int e = tid; e < FD * G; e += kChainThreads) a.next.addE[static_cast<int64_t>(jr) * FD * G + e] = 0.0;
    for (int e = tid; e < FD; e += kChainThreads) a.next.addg[static_cast<int64_t>(jr) * FD + e] = 0.0;
  }
  if (toGhost) {  // carry the ghost node itself to the next level (its Schur updates went to next.add*)
    for (int e = tid; e < FD * FD; e += kChainThreads)
      a.next.A[static_cast<int64_t>(jr) * FD * FD + e] = L.A[static_cast<int64_t>(rIdx) * FD * FD + e] + (add ? L.addA[static_cast<int64_t>(rIdx) * FD * FD + e] : 0.0);
    for (int e = tid; e < FD * G; e += kChainThreads)
      a.next.E[static_cast<int64_t>(jr) * FD * G + e] = L.E[static_cast<int64_t>(rIdx) * FD * G + e] + (add ? L.addE[static_cast<int64_t>(rIdx) * FD * G + e] : 0.0);
    for (int e = tid; e < FD; e += kChainThreads)
      a.next.g[static_cast<int64_t>(jr) * FD + e] = L.g[static_cast<int64_t>(rIdx) * FD + e] + (add ? L.addg[static_cast<int64_t>(rIdx) * FD + e] : 0.0);
    if (tid == 0) a.next.orig[jr] = L.orig[rIdx];
  }
  __syncthreads();
  for (int e = tid; e < FD * FD; e += kChainThreads) {
    a.next.A[static_cast<int64_t>(j) * FD * FD + e] = Al[e];
    if (j == 0) { a.next.U[e] = 0.0; a.next.addA[e] = 0.0; }
  }
  for (int e = tid; e < FD * G; e += kChainThreads) {
    a.next.E[static_cast<int64_t>(j) * FD * G + e] = El[e];
    if (j == 0) a.next.addE[e] = 0.0;
  }
  for (int e = tid; e < FD; e += kChainThreads) {
    a.next.g[static_cast<int64_t>(j) * FD + e] = gl[e];
    if (j == 0) a.next.addg[e] = 0.0;
  }
  if (tid == 0) {
    a.next.orig[j] = L.orig[s];
    if (bad) a.scalars[7] = 1.0;  // kScNotPD
  }
  double* out = a.Spart + static_cast<int64_t>(j) * NS;
  for (int e = tid; e < NS; e += kChainThreads) out[e] = Sacc[e];
}

// sum of the per-CTA Schur partials (coalesced across entries)
// launch with 256 threads: 32 entries per CTA, 8 partial-slices per entry, fixed summation order
__global__ void __launch_bounds__(256) sum_partials_kernel(const double* part, int n_part, int NS, double* out,
                                                           const Ctl* ctl) {
  __shared__ double sh[8][33];
  if (ctl->done) return;
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

// same sum, output selected on the device: [C | gc] of the buffer being evaluated (contiguous in Blocks)
__global__ void __launch_bounds__(256) sum_partials_sel_kernel(const double* part, int n_part, int NS, double* out0,
                                                               double* out1, const Ctl* ctl, int which) {
  __shared__ double sh[8][33];
  if (ctl->done) return;
  double* out = (which ? 1 - ctl->cur : ctl->cur) ? out1 : out0;
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

// dense solve of [globals | top-level chain nodes]
struct DenseArgs {
  DevProblem dp;
  Blocks bs[2];
  const Ctl* ctl;
  const double* scale;
  const double* D2x;
  const double* Ssum;  // [G*G+G] summed Schur partials
  ChainLevel top;      // n may be 0
  double* delta;
  double* scalars;
  int n_slots;         // frame blocks in the dense system (single GPU: top.n; sharded: one per rank)
  int slot_of[4];      // dense slot of each local top node
  int add_globals;     // 1: this rank contributes C + D and -g_c (exactly one rank does)
  int mode;            // 0: assemble + solve; 1: assemble the local partial into buf only; 2: solve the (summed) buf
  double* buf;         // [N*N + N], N = G + n_slots*FD
};
template <int FD>
__global__ void __launch_bounds__(256) dense_solve_kernel(DenseArgs a) {
  extern __shared__ double sm[];
  const int G = a.dp.G, nt = a.top.n, N = G + a.n_slots * FD, tid = threadIdx.x;
  double* S = a.mode == 1 ? a.buf : sm;              // [N*N]
  double* rhs = S + N * N;
  __shared__ int bad;
  if (a.ctl->done) return;
  const Blocks& b = a.bs[a.ctl->cur];
  const double rinv = 1.0 / a.ctl->radius;
  if (tid == 0) bad = 0;
  const int64_t nfp = static_cast<int64_t>(a.dp.n_frames) * a.dp.fd;
  const double* sc = a.scale + nfp;
  if (a.mode == 2) {
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
          if (r == c) v += a.D2x ? a.D2x[nfp + r] : lm_damp(b.C[e], sc[r], rinv);
        }
        S[r * N + c] = v;
      } else {
        const int r = e - G * G;
        rhs[r] = (a.add_globals ? -b.gc[r] * sc[r] : 0.0) + a.Ssum[e];
      }
    }
    const bool add = a.top.addA != nullptr;
    for (int t = 0; t < nt; ++t) {
      const int o = G + a.slot_of[t] * FD;
      for (int e = tid; e < FD * FD; e += 256) {
        const int r = e / FD, c = e - r * FD;
        S[(o + r) * N + o + c] = a.top.A[static_cast<int64_t>(t) * FD * FD + e] + (add ? a.top.addA[static_cast<int64_t>(t) * FD * FD + e] : 0.0);
        if (t > 0) {
          const int op = G + a.slot_of[t - 1] * FD;
          const double u = a.top.U[static_cast<int64_t>(t) * FD * FD + e];  // H[t-1, t]
          S[(op + r) * N + o + c] = u;
          S[(o + c) * N + op + r] = u;
        }
      }
      for (int e = tid; e < FD * G; e += 256) {
        const int r = e / G, c = e - r * G;
        const double v = a.top.E[static_cast<int64_t>(t) * FD * G + e] + (add ? a.top.addE[static_cast<int64_t>(t) * FD * G + e] : 0.0);
        S[(o + r) * N + c] = v;
        S[c * N + o + r] = v;
      }
      for (int e = tid; e < FD; e += 256)
        rhs[o + e] = -(a.top.g[static_cast<int64_t>(t) * FD + e] + (add ? a.top.addg[static_cast<int64_t>(t) * FD + e] : 0.0));
    }
  }
  if (a.mode == 1) return;
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
    if (bad && lane == 0) a.scalars[7] = 1.0;
  }
  __syncthreads();
  for (int i = tid; i < G; i += 256) a.delta[nfp + i] = bad ? 0.0 : rhs[i];
  for (int e = tid; e < nt * FD; e += 256) {
    const int t = e / FD, r = e - t * FD;
    a.delta[static_cast<int64_t>(a.top.orig[t]) * FD + r] = bad ? 0.0 : rhs[G + a.slot_of[t] * FD + r];
  }
}

// back-substitution of one level: x_p = -Z_g - Z_L x_left - Z_R x_right - Z_E dc
struct BacksubArgs {
  const Ctl* ctl;
  int G, c, nfp_off;  // nfp_off unused
  ChainLevel cur;
  double* delta;
  int64_t nfp;
};
template <int FD>
__global__ void __launch_bounds__(128) chain_backsub_kernel(BacksubArgs a) {
  const int G = a.G, c = a.c, w = 2 * FD + G + 1;
  const int lane = threadIdx.x & 31;
  const int p = blockIdx.x * 4 + (threadIdx.x >> 5);  // node index at this level
  const int n_eff = a.cur.n - a.cur.ghost;
  if (a.ctl->done || p >= n_eff || p % c == 0) return;              // separators (and the ghost) are solved at the next level
  const int s = (p / c) * c;
  const int r = s + c < n_eff ? s + c : (a.cur.ghost ? a.cur.n - 1 : a.cur.n);
  const double* xl = a.delta + static_cast<int64_t>(a.cur.orig[s]) * FD;
  const double* xr = r < a.cur.n ? a.delta + static_cast<int64_t>(a.cur.orig[r]) * FD : nullptr;
  const double* dc = a.delta + a.nfp;
  const double* Z = a.cur.Z + static_cast<int64_t>(p) * FD * w;
  double* out = a.delta + static_cast<int64_t>(a.cur.orig[p]) * FD;
#pragma unroll
  for (int rr = 0; rr < FD; ++rr) {
    const double* z = Z + rr * w;
    double sum = 0.0;
    for (int q = lane; q < w - 1; q += 32) {
      const double x = q < FD ? xl[q] : q < 2 * FD ? (xr ? xr[q - FD] : 0.0) : dc[q - 2 * FD];
      sum += z[q] * x;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) out[rr] = -z[w - 1] - sum;
  }
}

}  // namespace vc
