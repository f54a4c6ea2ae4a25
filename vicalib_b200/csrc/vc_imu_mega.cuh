// Persistent (cooperative) kernels of the inertial trust-region iteration — one GPU.
//
// An inertial LM iteration used to be ~21 launches (chain_init, one chain_eliminate per level, sum_partials,
// dense_solve, one chain_backsub per level, backsub_update, fused_build, imu_eval, imu_accumulate, reduce_finalize,
// imu_weights).  Here it is TWO cooperative launches of one CTA per SM, with grid barriers where a launch boundary
// used to be:
//
//   chain_solve_kernel   damped, Jacobi-scaled block-tridiagonal + arrow system (frame chain + dense globals):
//                        level-0 blocks -> partitioned elimination level by level (every kCsChunk-th node a
//                        separator; a chunk of kCsChunk - 1 interior nodes is swept by a GROUP of 128 threads, two groups per CTA, each
//                        keeping its share of the Schur complement of the globals in shared memory across all
//                        levels) -> distributed fixed-order sum of the groups' Schur partials -> dense Cholesky of
//                        [globals | top nodes] by every CTA -> back-substitution level by level -> x (+) step into
//                        the trial state + step statistics
//   eval_kernel          (vc_imu_eval_mega.cuh) residuals + Jacobians + block normal equations at the trial point,
//                        reduction, accept/reject, UpdateImuWeights
//
// Replaces what ceres::Solve does per iteration for the inertial stages (vicalibrator.h:956; SPARSE_NORMAL_CHOLESKY
// on the block-tridiagonal + arrow J^T J, SURVEY §8 a12).  Same arithmetic as vc_chain.cuh's kernels (which remain
// the engine of frame-sharded runs, where an NCCL all-reduce sits between assembling and factoring the dense system).
#pragma once
#include <cooperative_groups.h>

#include "vc_chain.cuh"
#include "vc_kernels.cuh"
#include "vc_mega.cuh"
#include "vc_xchg.cuh"
#include "vc_imu_weights.cuh"

namespace vc {

constexpr int kMaxChainLevels = 10;
constexpr int kCsThreads = 256;              // threads per CTA
constexpr int kCsGroup = 128;                // threads per elimination group
constexpr int kCsGroups = kCsThreads / kCsGroup;
// Shape of the partitioned elimination, for the device and for the host's level table (vc_imu_host.inl) alike:
// every kCsChunk-th node of a level is a separator; a level of at most kCsTop nodes joins the dense solve
constexpr int kCsChunk = 8;
constexpr int kCsTop = 4;
constexpr int kCsBsItem = 16;  // level-0 back-substitution nodes a CTA takes at a time in the closing phase (two per warp)
constexpr int kCsSyncWords = 8;  // counters of one launch (ChainSolveArgs::sync)
constexpr int kCsRedLoads = 16;  // loads a thread of the Schur reduction keeps in flight
// phase clock slots: elimination levels [0, 10), reduce 10, dense 11, back-substitution levels [12, 22), update 22
enum { kCsProfElim = 0, kCsProfReduce = kMaxChainLevels, kCsProfDense, kCsProfBacksub, kCsProfUpdate = kCsProfBacksub + kMaxChainLevels,
       kCsProfWeights, kCsProfCount };

struct ChainSolveArgs {
  DevProblem dp;
  Blocks b[2];
  Ctl* ctl;
  const double* scale;
  const double* D2x;            // explicit damping (inspection hook / dogleg) or null: LM rule
  const ChainLevel* lev;        // [n_levels] level descriptors (device memory)
  int n_levels;
  double* Spart;                // [grid][G*G+G] one Schur partial per CTA, packed (chain_sacc_doubles(G) entries used)
  double* Ssum;                 // [G*G+G]
  double* delta;                // scaled step [nf*9 + G]
  double* scalars;
  double* state[2];
  double* step_part;            // [grid + 1][4]
  int do_update;                // 1: trial state + step statistics
  int narrow_ok;                // 1: levels with fewer chunks than CTAs run one chunk per CTA (0: A/B switch)
  // frame-sharded run (x.nranks > 1): every rank reduces its chain to its first frame (+ the ghost = the next rank's
  // first frame); the partial [globals | one slot per rank] systems meet through the in-kernel exchange
  Xchg x;
  const double* sepdiag;        // [ranks][9] diag(B) of the ranks' first frames summed over both owners, or null
  double* dsys;                 // [NS + ranks * kTopBlock] summed dense system in block form
  unsigned long long* prof;     // [kCsProfCount] ns per phase (CTA 0) or null
  // deferred UpdateImuWeights (the reference's iteration callback, vicalibrator.h:690-721): the weights at the point the
  // previous iteration accepted are needed by the next EVALUATION, not by this solve — CTAs that have run out of
  // elimination work (levels with fewer chunks than CTAs, the dense solve) compute them here, off a queue
  int wts_on;                   // 1: run the update if the previous iteration accepted its step
  int n_solver;                 // CTAs that stay with the solve after the elimination levels
  imu::ImuBuf buf;
  const double* ftime;
  double* wsqrt;
  double sigma_g, sigma_a;
  unsigned long long* sync;     // [kCsSyncWords] {barrier counter, weights queue, CTAs ready for level 0, level-0 items
                                //  handed out, level-0 items done} of this launch
  unsigned long long* sync_next;  // ... of the next launch (the host alternates two sets): zeroed here
};

// the Schur accumulator of a group: lower triangle of S packed row by row (row r at r (r + 1) / 2), then the right-hand
// side — half the square, which is what lets two groups of chunk length 8 fit an SM at G = 67
__host__ __device__ inline int chain_sacc_doubles(int G) { return G * (G + 1) / 2 + G; }
// a group's workspace (chain_eliminate_chunk): Sacc | Al El gl | Ap | Uc | Ur | V | Eo
__host__ __device__ inline size_t chain_group_doubles(int G) {
  constexpr int FD = 9, c = kCsChunk;
  const size_t VW = FD + 2 * FD + G + 1;
  return chain_sacc_doubles(G) + FD * FD + FD * G + FD + (2 * (c - 1) + 1) * FD * FD + (c - 1) * FD * VW + (c - 1) * FD * G;
}
// tiles of the register version that fits N (0: none does — shared-memory version), and the layout of S that goes with it
__host__ __device__ inline int dense_tiles(int N) {
  const int t = (N + 1 + 15) / 16;
  return t <= 6 ? 6 : t <= 7 ? 7 : t <= 9 ? 9 : 0;
}
__host__ __device__ inline int dense_rows(int N) { return dense_tiles(N) ? 16 * dense_tiles(N) : N + 1; }
__host__ __device__ inline int dense_ld(int N) { return dense_tiles(N) ? 16 * dense_tiles(N) + 1 : (N | 1); }
// a top node's blocks in the exchanged dense system: A 81 | U 81 (coupling to the previous slot) | E 9G | -g 9
__host__ __device__ inline int chain_top_block(int G) { return 2 * 81 + 9 * G + 9; }
__host__ __device__ inline size_t chain_solve_smem_doubles(int G, int nranks = 1) {
  const size_t grp = kCsGroups * chain_group_doubles(G);
  const size_t N = static_cast<size_t>(G) + (nranks > kCsTop ? nranks : kCsTop) * 9;
  const size_t dense = static_cast<size_t>(dense_rows(static_cast<int>(N))) * dense_ld(static_cast<int>(N)) + N + 2;
  const size_t wts = (kCsThreads / wts::kTeam) * (sizeof(wts::Work) / sizeof(double) + 1);
  const size_t m = grp > dense ? grp : dense;
  return (m > wts ? m : wts) + 16;
}

// wait (one thread) until a grid-wide counter reaches target; what the arrivals wrote before their increment is visible
__device__ __forceinline__ void spin_until(unsigned long long* c, unsigned long long target) {
  unsigned long long v;
  do {
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(c) : "memory");
  } while (v < target);
  __threadfence();
}

__device__ __forceinline__ void group_sync(int grp) {
  asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "r"(kCsGroup) : "memory");
}

// (r, q) of linear index e = r * W + q, advanced by `step` without a division
__device__ __forceinline__ void adv2(int& r, int& q, int W, int step) {
  q += step;
  while (q >= W) { q -= W; ++r; }
}

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

// 8-byte copy global -> shared that does not pass through a register, and the wait for all of this thread's copies
__device__ __forceinline__ void cp_async8(double* dst, const double* src) {
  const unsigned d = static_cast<unsigned>(__cvta_generic_to_shared(dst));
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(__cvta_generic_to_global(src)) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// *dst(e) += add[e] for e in [0, n), eight loads in flight per thread (element e by thread e mod NT)
template <int NT, class Dst>
__device__ __forceinline__ void add_in_place(const double* add, int n, int tid, Dst dst) {
  constexpr int B = 8;
  for (int e0 = tid; e0 < n; e0 += B * NT) {
    double v[B];
#pragma unroll
    for (int u = 0; u < B; ++u) v[u] = e0 + u * NT < n ? __ldcg(add + e0 + u * NT) : 0.0;
#pragma unroll
    for (int u = 0; u < B; ++u)
      if (e0 + u * NT < n) {
        double* d = dst(e0 + u * NT);
        *d = *d + v[u];
      }
  }
}

// Forward + backward sweep of one chunk (separator s = j*c, interior nodes s+1..s+m) by one group of 128 threads.
// Same algorithm as chain_eliminate_kernel (vc_chain.cuh); here the chunk's blocks arrive by asynchronous copies
// straight into their places in shared memory, all in flight before the first one is used (no register staging: nothing
// grows with the chunk length), the 9 x 9 pivots are factored right-looking with rsqrt, and the group's Schur
// accumulator Sacc lives on across chunks and levels.
// NT: threads working on the chunk — a group of 128 (two chunks per CTA in flight: the wide levels) or the whole CTA of
// 256 (levels with fewer chunks than CTAs, where the other group would idle)
template <int NT>
__device__ __forceinline__ void gsync(int grp) {
  if (NT == kCsThreads) __syncthreads();
  else group_sync(grp);
}
template <int FD, int NT>
__device__ __forceinline__ void chain_eliminate_chunk(const NodeSrc& src, const ChainLevel L, const ChainLevel nxt, int G, int j, double* sm,
                                             int tid, int grp, int* bad, unsigned long long* dbg = nullptr) {
  // dbg: cycle counts of the chunk's phases (measurement hook: phase clocks [40..51], one group)
  long long dbg_t = dbg ? clock64() : 0;
  auto tick = [&](int slot) {
    if (dbg && tid == 0) {
      const long long t = clock64();
      dbg[slot] += static_cast<unsigned long long>(t - dbg_t);
      dbg_t = t;
    }
  };
  constexpr int c = kCsChunk;
  const int NS = chain_sacc_doubles(G), GT = G * (G + 1) / 2;
  const int w = 2 * FD + G + 1, VW = FD + w;
  const int oL = FD, oR = 2 * FD, oE = 3 * FD, og = 3 * FD + G;  // column offsets inside a V row
  double* Sacc = sm;                       // [NS] packed (chain_sacc_doubles)
  double* Al = Sacc + NS;                  // [FD*FD]
  double* El = Al + FD * FD;               // [FD*G]
  double* gl = El + FD * G;                // [FD]
  double* Ap = gl + FD;                    // [(c-1)][FD*FD] pivots
  double* Uc = Ap + (c - 1) * FD * FD;     // [(c-1)][FD*FD] U[p] = H[p-1, p]
  double* Ur = Uc + (c - 1) * FD * FD;     // [FD*FD] U of the right separator
  double* V = Ur + FD * FD;                // [(c-1)][FD][VW]: row r of interior node i is row R = i * FD + r
  double* Eo = V + (c - 1) * FD * VW;      // [(c-1)][FD*G] the interior nodes' own global coupling
  const int s = j * c, n_eff = L.n - L.ghost;
  const int nsep = (n_eff + c - 1) / c;
  const bool toGhost = L.ghost && !(s + c < n_eff);
  const bool hasR = s + c < n_eff || toGhost;
  const int m = min(c - 1, n_eff - 1 - s);
  const int rIdx = s + m + 1;
  const int jr = toGhost ? nsep : j + 1;
  gsync<NT>(grp);  // the previous chunk of this group is done with the workspace
  tick(0);
  const int nn = m + 1;                              // nodes s .. s+m
  const int nu = m + (hasR ? 1 : 0);                 // U blocks of nodes s+1 .. s+m (+ the right separator)
  const int rG0 = tid / G, qG0 = tid - rG0 * G;      // (row, column) of element tid of an FD x G block
  const int rw0 = tid / w, qw0 = tid - rw0 * w;      // ... of an FD x w block
  const int rV0 = tid / VW, qV0 = tid - rV0 * VW;    // ... of an FD x VW block
  const bool lvl0 = src.L == nullptr;
  // level 0: the Jacobi scales of nodes s-1 .. rIdx ([(c+2)][FD], entries [0, kSG)) and of the globals (entries kSG + q)
  // are parked in the coupling columns [0, 3 FD) of V's rows, which nothing else touches before the couplings step
  constexpr int kSG = (c + 2) * FD;
  auto scl = [&](int e) -> double* { return V + (e / (3 * FD)) * VW + e % (3 * FD); };
  // ---- the chunk's blocks as stored (level 0: the unscaled normal equations and the scales), one round of copies
  {
    const double* gA = (lvl0 ? src.b.B : L.A) + static_cast<int64_t>(s) * FD * FD;
    const double* gU = (lvl0 ? src.b.U : L.U) + static_cast<int64_t>(s + 1) * FD * FD;
    const double* gE = (lvl0 ? src.b.E : L.E) + static_cast<int64_t>(s) * FD * G;
    const double* gg = (lvl0 ? src.b.gf : L.g) + static_cast<int64_t>(s) * FD;
    for (int e = tid; e < nn * FD * FD; e += NT) cp_async8(e < FD * FD ? Al + e : Ap + (e - FD * FD), gA + e);
    for (int e = tid; e < nu * FD * FD; e += NT) cp_async8(e < m * FD * FD ? Uc + e : Ur + (e - m * FD * FD), gU + e);
    for (int e = tid, R = rG0, q = qG0; e < nn * FD * G; e += NT, adv2(R, q, G, NT))
      cp_async8(R < FD ? El + e : V + (R - FD) * VW + oE + q, gE + e);
    for (int e = tid; e < nn * FD; e += NT) cp_async8(e < FD ? gl + e : V + (e - FD) * VW + og, gg + e);
    if (lvl0) {
      for (int e = tid; e < (m + 3) * FD; e += NT) {
        const int64_t node = static_cast<int64_t>(s) - 1 + e / FD;
        if (node >= 0 && node < src.nf) cp_async8(scl(e), src.scale + node * FD + e % FD);
        else *scl(e) = 0.0;
      }
      for (int e = tid; e < G; e += NT) cp_async8(scl(kSG + e), src.scale + static_cast<int64_t>(src.nf) * FD + e);
    }
    cp_async_wait_all();
  }
  gsync<NT>(grp);
  tick(1);
  // ---- in place: level 0 scales and damps, deeper levels add the Schur terms of the chunk on the left (add*)
  if (lvl0) {
    for (int e = tid; e < nn * FD * FD; e += NT) {
      const int nd = e / (FD * FD), el = e - nd * FD * FD, r = el / FD, q = el - r * FD;
      double* d = nd == 0 ? Al + el : Ap + (e - FD * FD);
      const double a = *d, sr = *scl((nd + 1) * FD + r), sq = *scl((nd + 1) * FD + q);
      double v = a * sr * sq;
      if (r == q) {
        if (src.D2x) v += src.D2x[static_cast<int64_t>(s + nd) * FD + r];
        else if (src.sepdiag && s + nd == 0) v += lm_damp(src.sepdiag[src.rank * FD + r], sr, src.rinv);
        else v += lm_damp(a, sr, src.rinv);
      }
      *d = v;
    }
    for (int e = tid; e < nu * FD * FD; e += NT) {
      const int nd = e / (FD * FD), el = e - nd * FD * FD, r = el / FD, q = el - r * FD;  // node s + 1 + nd
      // H[p-1, p] scaled by (scale of p-1, row) x (scale of p, column)
      double* d = nd < m ? Uc + e : Ur + el;
      *d = *d * *scl((nd + 1) * FD + r) * *scl((nd + 2) * FD + q);
    }
    for (int e = tid; e < nn * FD; e += NT) {
      double* d = e < FD ? gl + e : V + (e - FD) * VW + og;
      *d = *d * *scl(FD + e);
    }
    for (int e = tid, R = rG0, q = qG0; e < nn * FD * G; e += NT, adv2(R, q, G, NT)) {
      double* d = R < FD ? El + e : V + (R - FD) * VW + oE + q;
      *d = *d * *scl(FD + R) * *scl(kSG + q);
    }
  } else {
    const int64_t o = static_cast<int64_t>(s);
    if (L.addA) add_in_place<NT>(L.addA + o * FD * FD, nn * FD * FD, tid, [&](int e) { return e < FD * FD ? Al + e : Ap + (e - FD * FD); });
    if (L.addg) add_in_place<NT>(L.addg + o * FD, nn * FD, tid, [&](int e) { return e < FD ? gl + e : V + (e - FD) * VW + og; });
    if (L.addE)
      add_in_place<NT>(L.addE + o * FD * G, nn * FD * G, tid, [&](int e) {
        const int R = e / G;
        return R < FD ? El + e : V + (R - FD) * VW + oE + (e - R * G);
      });
  }
  // the interior nodes' E as the sweeps will see it, kept for the Schur product (every thread copies the elements it
  // finished itself: no barrier needed)
  for (int e = tid, R = rG0, q = qG0; e < nn * FD * G; e += NT, adv2(R, q, G, NT))
    if (R >= FD) Eo[e - FD * G] = V[(R - FD) * VW + oE + q];
  gsync<NT>(grp);
  tick(2);
  // couplings of the interior nodes' right-hand sides, from the staged U blocks
  for (int i = 0; i < m; ++i) {
    double* Vi = V + static_cast<int64_t>(i) * FD * VW;
    const bool lastI = i == m - 1;
    const double* Unext = lastI ? Ur : Uc + (i + 1) * FD * FD;  // H[p, p+1]
    for (int e = tid; e < FD * FD; e += NT) {
      const int r = e / FD, q = e - r * FD;
      Vi[r * VW + oL + q] = i == 0 ? Uc[q * FD + r] : 0.0;  // H[p0, s] = U[p0]^T
      const double unext = (!lastI || hasR) ? Unext[e] : 0.0;
      Vi[r * VW + q] = lastI ? 0.0 : unext;
      Vi[r * VW + oR + q] = (lastI && hasR) ? unext : 0.0;
    }
  }
  gsync<NT>(grp);
  tick(4);
  // ---- forward sweep
  for (int i = 0; i < m; ++i) {
    double* Vi = V + static_cast<int64_t>(i) * FD * VW;
    double* Api = Ap + i * FD * FD;
    if (i > 0) {
      const double* Vp = V + static_cast<int64_t>(i - 1) * FD * VW;
      const double* Uci = Uc + i * FD * FD;
      // A'_i = A_i - U^T V_U(i-1);  R'_i = R_i - U^T V_R(i-1)
      for (int e = tid, r = rV0, q = qV0; e < FD * VW; e += NT, adv2(r, q, VW, NT)) {
        double sum = 0.0;
#pragma unroll
        for (int k = 0; k < FD; ++k) sum += Uci[k * FD + r] * Vp[k * VW + q];
        if (q < FD) Api[r * FD + q] -= sum;
        else Vi[r * VW + q] -= sum;
      }
      gsync<NT>(grp);
    }
    if (tid < VW) {
      // every column-solving thread factors the FD x FD pivot in registers (no serial section, no barrier):
      // right-looking Cholesky, reciprocal pivots by rsqrt
      double Lr[FD][FD], iL[FD];
#pragma unroll
      for (int ii = 0; ii < FD; ++ii)
#pragma unroll
        for (int k = 0; k <= ii; ++k) Lr[ii][k] = Api[ii * FD + k];
      bool ok = true;
#pragma unroll
      for (int jj = 0; jj < FD; ++jj) {
        const double d = Lr[jj][jj];
        ok = ok && d > 0.0;
        const double inv = rsqrt(d > 0.0 ? d : 1.0);
        iL[jj] = inv;
#pragma unroll
        for (int ii = jj + 1; ii < FD; ++ii) Lr[ii][jj] *= inv;
#pragma unroll
        for (int ii = jj + 1; ii < FD; ++ii)
#pragma unroll
          for (int k = jj + 1; k <= ii; ++k) Lr[ii][k] -= Lr[ii][jj] * Lr[k][jj];
      }
      if (!ok && tid == 0) *bad = 1;
      const int q = tid;
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
        for (int k = FD - 1; k > ii; --k) t -= Lr[k][ii] * x[k];
        x[ii] = t * iL[ii];
      }
#pragma unroll
      for (int ii = 0; ii < FD; ++ii) Vi[ii * VW + q] = x[ii];
    }
    gsync<NT>(grp);
  }
  tick(5);
  // ---- backward sweep: X_i = V_R(i) - V_U(i) X_{i+1}
  for (int i = m - 2; i >= 0; --i) {
    double* Vi = V + static_cast<int64_t>(i) * FD * VW;
    const double* Vn = V + static_cast<int64_t>(i + 1) * FD * VW;
    for (int e = tid, r = rw0, qq = qw0; e < FD * w; e += NT, adv2(r, qq, w, NT)) {
      const int q = FD + qq;
      double sum = 0.0;
#pragma unroll
      for (int k = 0; k < FD; ++k) sum += Vi[r * VW + k] * Vn[k * VW + q];
      Vi[r * VW + q] -= sum;
    }
    gsync<NT>(grp);
  }
  tick(6);
  // ---- store Z, accumulate the Schur terms: S += E_i^T X_i[E], rhs += E_i^T X_i[g]
  for (int i = 0; i < m; ++i) {
    const int64_t p = s + 1 + i;
    const double* Vi = V + static_cast<int64_t>(i) * FD * VW;
    for (int e = tid, r = rw0, q = qw0; e < FD * w; e += NT, adv2(r, q, w, NT)) L.Z[p * FD * w + e] = Vi[r * VW + FD + q];
  }
  tick(7);
  {  // lower triangle of S (row ra has ra + 1 entries), then the right-hand side; four entries in flight per thread
    int ra = 0, cb = tid;
    while (cb > ra) { cb -= ra + 1; ++ra; }
    while (ra < G) {
      int r4[4], c4[4];
      double sum[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        r4[u] = ra; c4[u] = cb;
        cb += NT;
        while (cb > ra && ra < G) { cb -= ra + 1; ++ra; }
      }
      for (int i = 0; i < m; ++i) {
        const double* Vi = V + static_cast<int64_t>(i) * FD * VW + oE;
        const double* Ei = Eo + i * FD * G;
#pragma unroll
        for (int k = 0; k < FD; ++k) {
#pragma unroll
          for (int u = 0; u < 4; ++u)
            if (r4[u] < G) sum[u] += Ei[k * G + r4[u]] * Vi[k * VW + c4[u]];
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (r4[u] < G) Sacc[r4[u] * (r4[u] + 1) / 2 + c4[u]] += sum[u];
    }
    for (int r = tid; r < G; r += NT) {
      double sum = 0.0;
      for (int i = 0; i < m; ++i) {
        const double* Vi = V + static_cast<int64_t>(i) * FD * VW;
        const double* Ei = Eo + i * FD * G;
#pragma unroll
        for (int k = 0; k < FD; ++k) sum += Ei[k * G + r] * Vi[k * VW + og];
      }
      Sacc[GT + r] += sum;
    }
  }
  tick(8);
  if (m > 0) {
    const double* X0 = V;                                          // node s+1
    const double* Xl = V + static_cast<int64_t>(m - 1) * FD * VW;  // last interior node
    const double* U0 = Uc;                                         // H[s, s+1]
    for (int e = tid, r = rw0, q = qw0; e < FD * w; e += NT, adv2(r, q, w, NT)) {  // q indexes [L | R | E | g]
      double sl = 0.0, sr = 0.0;
#pragma unroll
      for (int k = 0; k < FD; ++k) {
        sl += U0[r * FD + k] * X0[k * VW + FD + q];
        if (hasR) sr += Ur[k * FD + r] * Xl[k * VW + FD + q];  // H[rIdx-1, rIdx]^T
      }
      if (q < FD) {
        Al[r * FD + q] -= sl;                                        // A_s -= H[s,p0] Z_L
      } else if (q < 2 * FD) {
        if (hasR) {
          nxt.U[static_cast<int64_t>(jr) * FD * FD + r * FD + (q - FD)] = -sl;     // fill H[s, rIdx]
          nxt.addA[static_cast<int64_t>(jr) * FD * FD + r * FD + (q - FD)] = -sr;  // A_r -= H[r,pl] Z_R
        }
      } else if (q < 2 * FD + G) {
        El[r * G + (q - 2 * FD)] -= sl;
        if (hasR) nxt.addE[static_cast<int64_t>(jr) * FD * G + r * G + (q - 2 * FD)] = -sr;
      } else {
        gl[r] -= sl;
        if (hasR) nxt.addg[static_cast<int64_t>(jr) * FD + r] = -sr;
      }
    }
  } else if (hasR) {
    // no interior node between this separator and the ghost: the coupling passes through unchanged
    for (int e = tid; e < FD * FD; e += NT) {
      nxt.U[static_cast<int64_t>(jr) * FD * FD + e] = Ur[e];
      nxt.addA[static_cast<int64_t>(jr) * FD * FD + e] = 0.0;
    }
    for (int e = tid; e < FD * G; e += NT) nxt.addE[static_cast<int64_t>(jr) * FD * G + e] = 0.0;
    for (int e = tid; e < FD; e += NT) nxt.addg[static_cast<int64_t>(jr) * FD + e] = 0.0;
  }
  if (toGhost) {  // carry the ghost node itself to the next level (its Schur updates went to nxt.add*)
    for (int e = tid; e < FD * FD; e += NT) nxt.A[static_cast<int64_t>(jr) * FD * FD + e] = src_A<FD>(src, rIdx, e);
    for (int e = tid, r = rG0, q = qG0; e < FD * G; e += NT, adv2(r, q, G, NT)) nxt.E[static_cast<int64_t>(jr) * FD * G + e] = src_E<FD>(src, rIdx, r, q);
    for (int e = tid; e < FD; e += NT) nxt.g[static_cast<int64_t>(jr) * FD + e] = src_g<FD>(src, rIdx, e);
    if (tid == 0) nxt.orig[jr] = src.L ? L.orig[rIdx] : rIdx;
  }
  gsync<NT>(grp);
  for (int e = tid; e < FD * FD; e += NT) {
    nxt.A[static_cast<int64_t>(j) * FD * FD + e] = Al[e];
    if (j == 0) { nxt.U[e] = 0.0; nxt.addA[e] = 0.0; }
  }
  for (int e = tid; e < FD * G; e += NT) {
    nxt.E[static_cast<int64_t>(j) * FD * G + e] = El[e];
    if (j == 0) nxt.addE[e] = 0.0;
  }
  for (int e = tid; e < FD; e += NT) {
    nxt.g[static_cast<int64_t>(j) * FD + e] = gl[e];
    if (j == 0) nxt.addg[e] = 0.0;
  }
  if (tid == 0) nxt.orig[j] = src.L ? L.orig[s] : s;
  tick(9);
}

// Back-substitution of one level: x_p = -Z_g - Z_L x_left - Z_R x_right - Z_E dc for every interior node p, one warp each.
// Node slot t (interior node t mod (c - 1) of chunk t / (c - 1)) of a level's n_chunks * (c - 1) slots.
template <int FD>
__device__ __forceinline__ void chain_backsub_node(const ChainLevel& cur, int l, double* delta, int64_t nfp, int G, int t, int lane) {
  const int w = 2 * FD + G + 1, c = kCsChunk;
  const double* dc = delta + nfp;
  const int n_eff = cur.n - cur.ghost;
  int cl = 1;  // c^l
  for (int k = 0; k < l; ++k) cl *= c;
  // interior node q (0..c-2) of chunk j: p = j*c + 1 + q
  const int jc = t / (c - 1), p = jc * c + 1 + (t - jc * (c - 1));
  if (p >= n_eff) return;
  const int s = jc * c;
  const int r = s + c < n_eff ? s + c : (cur.ghost ? cur.n - 1 : cur.n);
  // original frame of node p of level l: p * c^l (no ghost node on one GPU); a table lookup otherwise
  const int os = cur.ghost ? (l > 0 ? cur.orig[s] : s) : s * cl, op = cur.ghost ? (l > 0 ? cur.orig[p] : p) : p * cl;
  const double* xl = delta + static_cast<int64_t>(os) * FD;
  const double* xr = r < cur.n ? delta + static_cast<int64_t>(cur.ghost ? (l > 0 ? cur.orig[r] : r) : r * cl) * FD : nullptr;
  const double* Z = cur.Z + static_cast<int64_t>(p) * FD * w;
  double* out = delta + static_cast<int64_t>(op) * FD;
  double d[FD];
#pragma unroll
  for (int rr = 0; rr < FD; ++rr) d[rr] = 0.0;
  for (int q = lane; q < w - 1; q += 32) {
    const double x = q < FD ? __ldcg(xl + q) : q < 2 * FD ? (xr ? __ldcg(xr + q - FD) : 0.0) : __ldcg(dc + q - 2 * FD);
#pragma unroll
    for (int rr = 0; rr < FD; ++rr) d[rr] += __ldcg(Z + rr * w + q) * x;
  }
#pragma unroll
  for (int rr = 0; rr < FD; ++rr) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d[rr] += __shfl_xor_sync(0xffffffffu, d[rr], o);
    d[rr] = -__ldcg(Z + rr * w + w - 1) - d[rr];
  }
  if (lane < FD) {
    double v = d[0];
#pragma unroll
    for (int rr = 1; rr < FD; ++rr) v = lane == rr ? d[rr] : v;
    out[lane] = v;
  }
}
__host__ __device__ inline int chain_backsub_slots(const ChainLevel& cur) {
  return (cur.n - cur.ghost + kCsChunk - 1) / kCsChunk * (kCsChunk - 1);
}
// all of a level, warp gw of nw
template <int FD>
__device__ __forceinline__ void chain_backsub_level(const ChainLevel cur, int l, double* delta, int64_t nfp, int G, int gw, int nw, int lane) {
  const int n_slots = chain_backsub_slots(cur);
  for (int t = gw; t < n_slots; t += nw) chain_backsub_node<FD>(cur, l, delta, nfp, G, t, lane);
}

// x (+) step of one frame into the trial state, and the frame's share of the step statistics
// (acc: step.g, step.D2.step, |x_new - x|^2, |x_new|^2)
__device__ __forceinline__ void chain_update_frame(const ChainSolveArgs& a, const Blocks& b, double rinv, int f, const double* d,
                                                   double acc[4]) {
  constexpr int FD = 9;
  const int cur = a.ctl->cur;
  const double* x_cur = a.state[cur];
  double* x_new = a.state[1 - cur];
  double du[FD];
  // sharded: a rank's first frame is damped from the diagonal summed over both owners; its ghost copy on the previous
  // rank moves with the same step but is counted (damping term, norms) by the owner only
  const bool is_ghost = a.dp.ghost && f == a.dp.n_frames - 1;
#pragma unroll
  for (int r = 0; r < FD; ++r) {
    const int64_t k = static_cast<int64_t>(f) * FD + r;
    const double sc = a.scale[k];
    double d2;
    if (is_ghost) d2 = 0.0;
    else if (a.D2x) d2 = a.D2x[k];
    else if (a.sepdiag && f == 0) d2 = lm_damp(a.sepdiag[a.dp.rank * FD + r], sc, rinv);
    else d2 = lm_damp(b.B[k * FD + r], sc, rinv);
    acc[0] += d[r] * b.gf[k] * sc;
    acc[1] += d[r] * d[r] * d2;
    du[r] = d[r] * sc;
  }
  const double* x = x_cur + 7 * static_cast<int64_t>(f);
  double xo[7];
  se3_plus(x, du, xo);
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    x_new[7 * static_cast<int64_t>(f) + k] = xo[k];
    if (!is_ghost) {
      acc[2] += (xo[k] - x[k]) * (xo[k] - x[k]);
      acc[3] += xo[k] * xo[k];
    }
  }
  const double* v = x_cur + a.dp.off_v + 3 * static_cast<int64_t>(f);
  double* vo = x_new + a.dp.off_v + 3 * static_cast<int64_t>(f);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double nv = v[k] + du[6 + k];
    vo[k] = nv;
    if (!is_ghost) {
      acc[2] += (nv - v[k]) * (nv - v[k]);
      acc[3] += nv * nv;
    }
  }
}

// The deferred UpdateImuWeights as a function of its own (its own register allocation: inlined into the solve kernel
// it is slower, with the solve's live values squeezed into the same 255 registers).  Everything by value — a
// reference to the kernel's parameter block would force the whole block into local memory.
struct WeightQueueArgs {
  struct { int64_t off_v, off_imu; } dp;
  imu::ImuBuf buf;
  const double* ftime;
  double* wsqrt;
  int ni;
  double sigma_g, sigma_a;
};
__device__ __noinline__ void chain_weights_queue(const WeightQueueArgs w, const double* xs, unsigned long long* wq, double* smem,
                                                 unsigned long long* wtask) {
  constexpr int kTeams = kCsThreads / wts::kTeam;
  const int tid = threadIdx.x, warp = tid >> 5;
  wts::Work* work = reinterpret_cast<wts::Work*>(smem);
  const int team = tid / wts::kTeam, tl = tid & (wts::kTeam - 1);
  for (;;) {
    __syncthreads();  // the workspace (and *wtask) are free
    if (tid == 0) *wtask = atomicAdd(wq, 1ull);
    __syncthreads();
    const long long base = static_cast<long long>(*wtask) * kTeams;
    if (base >= w.ni) break;
    if (base + (warp * (32 / wts::kTeam)) < w.ni) wts::imu_weights_team(w, xs, static_cast<int>(base) + team, &work[team], tl);
  }
}

// ---- dense L D L^T of the [globals | top nodes] system (one CTA of 256 threads; S: [N + 1][LD], row N = right-hand side)
// shared-memory version: any N
__device__ __noinline__ void dense_ldlt_smem(double* S, int N, int LD, double* wd, int* bad) {
  const int tid = threadIdx.x, ti = tid >> 4, tk = tid & 15;
  if (tid == 0) {
    const double d = S[0];
    const bool okp = d > 0.0;
    wd[0] = 1.0 / (okp ? d : 1.0);
    if (!okp) *bad = 1;
  }
  for (int j = 0; j < N; ++j) {
    __syncthreads();
    const double wj = wd[j];
    for (int i = j + 1 + ti; i <= N; i += 16) {
      double* row = S + i * LD;
      const double lw = row[j] * wj;
      const int kmax = i < N ? i : N - 1;
      for (int k = j + 1 + tk; k <= kmax; k += 16) {
        const double v = row[k] - lw * S[k * LD + j];
        row[k] = v;
        if (k == j + 1 && i == j + 1) {  // the next pivot is final: its reciprocal now
          const bool okp = v > 0.0;
          wd[j + 1] = 1.0 / (okp ? v : 1.0);
          if (!okp) *bad = 1;
        }
      }
    }
  }
  __syncthreads();
}
// register version: T x T tiles of 16 x 16 cover the N + 1 rows.  S is padded to 16 T rows of LD >= 16 T columns (zeros
// outside the system), so nothing in the column loop needs a bounds check: an update that should not happen (row or
// column already finished, padding) only ever lands in an element above the diagonal or in a column that has already
// gone back to shared memory — registers nobody reads again.  ~45 instructions per column instead of ~150; the loop is
// issue-bound (two warps per scheduler, dependent instructions), so that is what counts.
template <int T, int KK>
__device__ __forceinline__ void dense_col_back(const double (&R)[T][T], double* Sc, int LD, int jn, int ti, double* wd, int* bad) {
  // Sc = &S[ti][jn]; rows 16 ii + ti for ii >= KK (rows above the diagonal get dead values)
#pragma unroll
  for (int ii = KK; ii < T; ++ii) Sc[16 * ii * LD] = R[ii][KK];
  if (16 * KK + ti == jn) {  // the pivot: its reciprocal for the next column step
    const double v = R[KK][KK];
    const bool okp = v > 0.0;
    wd[jn] = __drcp_rn(okp ? v : 1.0);
    if (!okp) *bad = 1;
  }
}
template <int T, int JT>
__device__ __forceinline__ void dense_tile_columns(double (&R)[T][T], double* S, int N, int LD, double* wd, int* bad, int ti, int tk) {
  const double* pi = S + ti * LD + 16 * JT;  // S[ti][j]
  const double* pk = S + tk * LD + 16 * JT;  // S[tk][j]
  for (int jr = 0; jr < 16; ++jr, ++pi, ++pk) {
    const int j = 16 * JT + jr;
    if (j >= N) break;
    __syncthreads();  // column j and 1 / d_j are in shared memory
    const double wj = wd[j];
    double ci[T], ck[T];
#pragma unroll
    for (int ii = JT; ii < T; ++ii) ci[ii] = pi[16 * ii * LD] * wj;
#pragma unroll
    for (int kk = JT; kk < T; ++kk) ck[kk] = pk[16 * kk * LD];
    // column tile by column tile, the one that holds column j + 1 first: that column is then final, its owners put it
    // back (and take the pivot's reciprocal) while everybody goes on with the rest of the update
    const int jn = j + 1;
    const bool owner = jn < N && tk == (jn & 15);
#pragma unroll
    for (int kk = JT; kk < T; ++kk) {
#pragma unroll
      for (int ii = kk; ii < T; ++ii) R[ii][kk] -= ci[ii] * ck[kk];
      if (kk == JT && jr < 15 && owner) dense_col_back<T, JT>(R, S + ti * LD + jn, LD, jn, ti, wd, bad);
      if (kk == JT + 1 && jr == 15 && owner) dense_col_back<T, (JT + 1 < T ? JT + 1 : JT)>(R, S + ti * LD + jn, LD, jn, ti, wd, bad);
    }
  }
}
template <int T, int JT>
struct DenseTiles {
  static __device__ __forceinline__ void run(double (&R)[T][T], double* S, int N, int LD, double* wd, int* bad, int ti, int tk) {
    dense_tile_columns<T, JT>(R, S, N, LD, wd, bad, ti, tk);
    if (16 * (JT + 1) < N) DenseTiles<T, JT + 1>::run(R, S, N, LD, wd, bad, ti, tk);
  }
};
template <int T>
struct DenseTiles<T, T> {
  static __device__ __forceinline__ void run(double (&)[T][T], double*, int, int, double*, int*, int, int) {}
};
template <int T>
__device__ __noinline__ void dense_ldlt_tiles(double* S, int N, int LD, double* wd, int* bad) {
  const int tid = threadIdx.x, ti = tid >> 4, tk = tid & 15;
  double R[T][T];  // (only kk <= ii is used)
#pragma unroll
  for (int ii = 0; ii < T; ++ii)
#pragma unroll
    for (int kk = 0; kk <= ii; ++kk) R[ii][kk] = S[(16 * ii + ti) * LD + 16 * kk + tk];
  if (tid == 0) {
    const double d = S[0];
    const bool okp = d > 0.0;
    wd[0] = __drcp_rn(okp ? d : 1.0);
    if (!okp) *bad = 1;
  }
  DenseTiles<T, 0>::run(R, S, N, LD, wd, bad, ti, tk);
  __syncthreads();
}
// One damped solve of the frame-chain + globals system and (optionally) the state update, all in one launch.
__global__ void __launch_bounds__(kCsThreads, 1) chain_solve_kernel(ChainSolveArgs a) {
  extern __shared__ double smem[];
  namespace cg = cooperative_groups;
  constexpr int FD = 9;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int grp = tid / kCsGroup, gtid = tid - grp * kCsGroup;
  const int nb = gridDim.x, bid = blockIdx.x;
  const int n_groups = nb * kCsGroups, gid = bid * kCsGroups + grp;
  const int G = a.dp.G, NS = G * G + G, nf = a.dp.n_frames;
  const int64_t nfp = static_cast<int64_t>(nf) * FD;
  __shared__ int bad_s[kCsGroups];
  __shared__ int bad_dense;
  __shared__ double part[kCsThreads / 32][4];
  __shared__ unsigned long long wtask;
  __shared__ unsigned long long* xbufs[kMaxRanks];
  xchg_stage(a.x, xbufs);  // (visible after the first barrier below)
  if (bid == 0 && tid == 0)
    for (int k = 0; k < kCsSyncWords; ++k) a.sync_next[k] = 0ull;
  if (a.ctl->done) return;  // uniform over the grid: written before this launch
  const Blocks& b = a.b[a.ctl->cur];
  const double rinv = 1.0 / a.ctl->radius;
  unsigned long long t_prev = 0;
  const bool prof = a.prof != nullptr && bid == 0 && tid == 0;
  if (prof) t_prev = global_ns();
  auto mark = [&](int slot) {
    if (prof) {
      const unsigned long long t = global_ns();
      a.prof[slot] += t - t_prev;
      t_prev = t;
    }
  };
  // ---- who does what.  Without a pending weight update every CTA stays with the solve (ns = grid).  With one, the
  // CTAs [ns, grid) leave after their last elimination level and work the weights queue; the solve goes on among the
  // first ns CTAs, which join the queue when they are done.  Barriers therefore count arrivals: everybody who took
  // part in a phase arrives, only those who go on wait.
  const bool wts_go = a.wts_on && !a.dp.rotation_only && a.ctl->iter > 0 && a.ctl->last_accepted;
  const int ns = wts_go ? min(max(a.n_solver, 1), nb) : nb;
  unsigned long long* bar = a.sync;      // this launch's counters (the host alternates the pair)
  unsigned long long* wq = a.sync + 1;
  unsigned long long bar_target = 0;
  int n_act = nb;
  // The CTAs that left come back for the widest phases at the end (back-substitution of level 0, the state update).
  // Those barriers count on a second counter: a CTA that is back early must not be mistaken for an arrival at one of
  // the barriers the solve is still passing through.
  auto barrier = [&](int n_next) -> bool {
    __syncthreads();
    bar_target += static_cast<unsigned long long>(n_act);
    const bool stay = bid < n_next;
    if (tid == 0) {
      __threadfence();
      atomicAdd(bar, 1ull);
      if (stay) {
        unsigned long long v;
        do {
          asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(bar) : "memory");
        } while (v < bar_target);
        __threadfence();
      }
    }
    n_act = n_next;
    __syncthreads();
    return stay;
  };
  double* gsm = smem + static_cast<size_t>(grp) * chain_group_doubles(G);
  if (gtid == 0) bad_s[grp] = 0;
  for (int e = gtid; e < chain_sacc_doubles(G); e += kCsGroup) gsm[e] = 0.0;  // the group's Schur accumulator
  double acc[4] = {0.0, 0.0, 0.0, 0.0};                   // this thread's share of the step statistics

  bool left = false;  // this CTA has left the solve (its elimination work is done): straight to the weights queue
  do {
  // ------------------------------------------------------------ elimination, level by level
  for (int l = 0; l + 1 < a.n_levels; ++l) {
    NodeSrc src;
    src.L = l > 0 ? &a.lev[l] : nullptr;
    src.b = b; src.scale = a.scale; src.D2x = a.D2x; src.rinv = rinv; src.G = G; src.nf = nf;
    src.sepdiag = a.sepdiag; src.rank = a.dp.rank; src.ghost = a.dp.ghost;
    const int nsep = a.lev[l + 1].n - a.dp.ghost;
    const ChainLevel Lc = a.lev[l], Ln = a.lev[l + 1];
    if (nsep > nb || !a.narrow_ok) {  // wide level: two chunks per CTA in flight
      for (int j = gid; j < nsep; j += n_groups)
        chain_eliminate_chunk<FD, kCsGroup>(src, Lc, Ln, G, j, gsm, gtid, grp, &bad_s[grp], nullptr);
    } else {          // narrow level: the whole CTA on one chunk (group 0's workspace and Schur accumulator)
      unsigned long long* dbg = (a.prof && bid == 0 && l == 1) ? a.prof + 40 : nullptr;
      for (int j = bid; j < nsep; j += nb) chain_eliminate_chunk<FD, kCsThreads>(src, Lc, Ln, G, j, smem, tid, 0, &bad_s[0], dbg);
      __syncthreads();
    }
    // who goes on: everybody the next level needs (all of them if it is a wide one), never fewer than ns
    int n_next = ns;
    if (l + 2 < a.n_levels) {
      const int nsep2 = a.lev[l + 2].n - a.dp.ghost;
      n_next = (nsep2 > nb || !a.narrow_ok) ? nb : max(ns, nsep2);
    }
    n_next = min(n_next, n_act);
    if (l + 2 == a.n_levels || bid >= n_next) {  // last level of this CTA: publish its Schur partial (the two groups'
      __syncthreads();                             // accumulators added: half as many partials for the reduction)
      double* out = a.Spart + static_cast<int64_t>(bid) * NS;
      const double* g1 = smem + chain_group_doubles(G);
#pragma unroll 1
      for (int e = tid; e < chain_sacc_doubles(G); e += kCsThreads) out[e] = smem[e] + g1[e];  // packed, as accumulated

      if (gtid == 0 && bad_s[grp]) a.scalars[kScNotPD] = 1.0;
    }
    mark(kCsProfElim + l);
    if (!barrier(n_next)) {
      left = true;
      break;
    }
  }
  if (left) break;
  if (a.n_levels == 1) {  // nothing to eliminate: the top level is the problem itself; zero partials
    const ChainLevel& L = a.lev[0];
    NodeSrc src;
    src.L = nullptr; src.b = b; src.scale = a.scale; src.D2x = a.D2x; src.rinv = rinv; src.G = G; src.nf = nf;
    src.sepdiag = a.sepdiag; src.rank = a.dp.rank; src.ghost = a.dp.ghost;
    if (bid == 0) {
      for (int f = 0; f < nf; ++f) {
        for (int e = tid; e < FD * FD; e += kCsThreads) {
          L.A[static_cast<int64_t>(f) * FD * FD + e] = src_A<FD>(src, f, e);
          L.U[static_cast<int64_t>(f) * FD * FD + e] = src_U<FD>(src, f, e);
        }
        for (int e = tid; e < FD * G; e += kCsThreads) L.E[static_cast<int64_t>(f) * FD * G + e] = src_E<FD>(src, f, e / G, e % G);
        for (int e = tid; e < FD; e += kCsThreads) L.g[static_cast<int64_t>(f) * FD + e] = src_g<FD>(src, f, e);
        if (tid == 0) L.orig[f] = f;
      }
    }
    double* out = a.Spart + static_cast<int64_t>(bid) * NS;
    for (int e = tid; e < NS; e += kCsThreads) out[e] = 0.0;
    if (!barrier(ns)) {
      left = true;
      break;
    }
  }
  // ------------------------------------------------------------ Schur partials -> total (fixed order), distributed
  // Entry e of the square total by one thread of the first ns CTAs: it adds the packed entry up over the nb partials in
  // CTA order, kCsRedLoads loads in flight (neighbouring threads read neighbouring entries), and writes it unpacked:
  // lower triangle, upper triangle 0, then the right-hand side.  32-bit offsets (grid x (G^2 + G) < 2^31 for G <= 127):
  // 64-bit ones cost the kernel more spills.
  for (int e = bid * kCsThreads + tid; e < NS; e += ns * kCsThreads) {
    const int r = e / G, q = e - r * G;
    const int k = r < G ? (q <= r ? r * (r + 1) / 2 + q : -1) : G * (G + 1) / 2 + q;
    double s = 0.0;
    if (k >= 0) {
      const double* p = a.Spart + k;
      int c = 0;
      for (; c + kCsRedLoads <= nb; c += kCsRedLoads) {
        double v[kCsRedLoads];
#pragma unroll
        for (int u = 0; u < kCsRedLoads; ++u) v[u] = __ldcg(p + (c + u) * NS);
#pragma unroll
        for (int u = 0; u < kCsRedLoads; ++u) s += v[u];
      }
      for (; c < nb; ++c) s += __ldcg(p + c * NS);
    }
    a.Ssum[e] = s;
  }
  mark(kCsProfReduce);
  barrier(ns);
  // ------------------------------------------------------------ sharded: the ranks' partial systems meet here
  const bool sharded = a.x.nranks > 1;
  const int TB = chain_top_block(G);
  if (sharded) {
    const ChainLevel& top = a.lev[a.n_levels - 1];
    const bool add = top.addA != nullptr;
    const double* sc = a.scale + nfp;
    const int P = NS + top.n * TB;  // this rank's entries: globals, own first frame (+ the ghost)
    for (int e = bid * kCsThreads + tid; e < P; e += ns * kCsThreads) {
      double v;
      if (e < NS) {
        const double p = __ldcg(a.Ssum + e);
        if (e < G * G) {
          v = -p;
          if (a.x.rank == 0) {  // the globals' own block joins once
            const int r = e / G, c = e - r * G;
            v += b.C[e] * sc[r] * sc[c];
            if (r == c) v += a.D2x ? a.D2x[nfp + r] : lm_damp(b.C[e], sc[r], rinv);
          }
        } else {
          v = p - (a.x.rank == 0 ? b.gc[e - G * G] * sc[e - G * G] : 0.0);
        }
      } else {
        const int t = (e - NS) / TB, o = (e - NS) - t * TB;
        if (o < 81) {
          v = __ldcg(top.A + static_cast<int64_t>(t) * 81 + o) + (add ? __ldcg(top.addA + static_cast<int64_t>(t) * 81 + o) : 0.0);
        } else if (o < 162) {
          v = t > 0 ? __ldcg(top.U + static_cast<int64_t>(t) * 81 + (o - 81)) : 0.0;  // H[own first frame, ghost]
        } else if (o < 162 + FD * G) {
          const int64_t q = static_cast<int64_t>(t) * FD * G + (o - 162);
          v = __ldcg(top.E + q) + (add ? __ldcg(top.addE + q) : 0.0);
        } else {
          const int64_t q = static_cast<int64_t>(t) * FD + (o - 162 - FD * G);
          v = -(__ldcg(top.g + q) + (add ? __ldcg(top.addg + q) : 0.0));
        }
      }
      xchg_put(a.x, xbufs, e, v);
    }
    // one reader per entry of the summed system (slot k = rank k's first frame: its own blocks + the ghost blocks of
    // rank k-1, whose U block is the coupling between slots k-1 and k), ranks in order
    const int Q = NS + a.x.nranks * TB;
    for (int e = bid * kCsThreads + tid; e < Q; e += ns * kCsThreads) {
      double v = 0.0;
      if (e < NS) {
        for (int r = 0; r < a.x.nranks; ++r) v += xchg_get(a.x, xbufs, r, e);
      } else {
        const int k = (e - NS) / TB, o = (e - NS) - k * TB;
        if (o >= 81 && o < 162) {
          v = k > 0 ? xchg_get(a.x, xbufs, k - 1, NS + TB + o) : 0.0;
        } else {
          if (k > 0) v = xchg_get(a.x, xbufs, k - 1, NS + TB + o);
          v += xchg_get(a.x, xbufs, k, NS + o);
        }
      }
      a.dsys[e] = v;
    }
    barrier(ns);
  }
  // ------------------------------------------------------------ dense solve of [globals | top nodes]: CTA 0 (the step
  // of the globals and of the top nodes goes through a.delta; everybody waits at the barrier below)
  long long dt0 = 0;
  if (bid == 0) {
    const ChainLevel& top = a.lev[a.n_levels - 1];
    const int nt = top.n, n_slots = sharded ? a.x.nranks : nt, N = G + n_slots * FD;
    const int slot0 = sharded ? a.x.rank : 0;  // slot of top node 0
    const int LD = dense_ld(N), RT = dense_rows(N);  // odd leading dimension: a column walks all shared-memory banks
    double* S = smem;          // [RT][LD] lower triangle; unscaled columns u_ij (L D L^T: L_ij = u_ij / d_j)
    double* rhs = S + N * LD;  // row N of the same elimination: u_Nj
    double* wd = S + RT * LD;  // 1 / d_j
    const double* sc = a.scale + nfp;
    if (tid == 0) bad_dense = 0;
    for (int e = tid; e < RT * LD; e += kCsThreads) S[e] = 0.0;
    __syncthreads();
    if (sharded) {
      for (int e = tid; e < NS; e += kCsThreads) {
        const double v = __ldcg(a.dsys + e);
        if (e < G * G) S[(e / G) * LD + e % G] = v;
        else rhs[e - G * G] = v;
      }
      for (int k = 0; k < n_slots; ++k) {
        const double* blk = a.dsys + NS + static_cast<int64_t>(k) * TB;
        const int o = G + k * FD, op = o - FD;
        for (int e = tid; e < TB; e += kCsThreads) {
          const double v = __ldcg(blk + e);
          if (e < 81) {
            S[(o + e / FD) * LD + o + e % FD] = v;
          } else if (e < 162) {
            if (k > 0) {
              const int r = (e - 81) / FD, c = (e - 81) % FD;
              S[(op + r) * LD + o + c] = v;
              S[(o + c) * LD + op + r] = v;
            }
          } else if (e < 162 + FD * G) {
            const int r = (e - 162) / G, c = (e - 162) % G;
            S[(o + r) * LD + c] = v;
            S[c * LD + o + r] = v;
          } else {
            rhs[o + e - 162 - FD * G] = v;
          }
        }
      }
    } else {
    for (int e0 = tid; e0 < NS; e0 += 4 * kCsThreads) {  // four entries per round: their loads are all in flight together
      double p[4], cv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int e = e0 + u * kCsThreads;
        p[u] = e < NS ? __ldcg(a.Ssum + e) : 0.0;
        cv[u] = e < NS ? b.C[e] : 0.0;  // C | gc are contiguous
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int e = e0 + u * kCsThreads;
        if (e >= NS) continue;
        if (e < G * G) {
          const int r = e / G, c = e - r * G;
          double v = cv[u] * sc[r] * sc[c] - p[u];
          if (r == c) v += a.D2x ? a.D2x[nfp + r] : lm_damp(cv[u], sc[r], rinv);
          S[r * LD + c] = v;
        } else {
          const int r = e - G * G;
          rhs[r] = -cv[u] * sc[r] + p[u];
        }
      }
    }
    const bool add = top.addA != nullptr;
    for (int t = 0; t < nt; ++t) {
      const int o = G + t * FD;
      for (int e = tid; e < FD * FD; e += kCsThreads) {
        const int r = e / FD, c = e - r * FD;
        S[(o + r) * LD + o + c] = __ldcg(top.A + static_cast<int64_t>(t) * FD * FD + e) + (add ? __ldcg(top.addA + static_cast<int64_t>(t) * FD * FD + e) : 0.0);
        if (t > 0) {
          const int op = o - FD;
          const double u = __ldcg(top.U + static_cast<int64_t>(t) * FD * FD + e);  // H[t-1, t]
          S[(op + r) * LD + o + c] = u;
          S[(o + c) * LD + op + r] = u;
        }
      }
      for (int e = tid; e < FD * G; e += kCsThreads) {
        const int r = e / G, c = e - r * G;
        const double v = __ldcg(top.E + static_cast<int64_t>(t) * FD * G + e) + (add ? __ldcg(top.addE + static_cast<int64_t>(t) * FD * G + e) : 0.0);
        S[(o + r) * LD + c] = v;
        S[c * LD + o + r] = v;
      }
      for (int e = tid; e < FD; e += kCsThreads)
        rhs[o + e] = -(__ldcg(top.g + static_cast<int64_t>(t) * FD + e) + (add ? __ldcg(top.addg + static_cast<int64_t>(t) * FD + e) : 0.0));
    }
    }
    // right-looking L D L^T on the lower triangle, the right-hand side riding along as row N.  The matrix lives in
    // registers for the whole factorisation (16 x 16 thread tiling: thread (ti, tk) owns the elements (i, k) = (ti, tk)
    // mod 16); a finished column goes back to shared memory, is read by everybody after ONE barrier, and nothing else
    // touches shared memory.  (The shared-memory version of this loop — read, update, write every element every column —
    // is slower: every element makes a shared-memory round trip per column, and a sharded run has up to 135 columns.)
    dt0 = clock64();
    __syncthreads();  // the system is assembled
    const int tiles = dense_tiles(N);
    if (tiles == 6) dense_ldlt_tiles<6>(S, N, LD, wd, &bad_dense);
    else if (tiles == 7) dense_ldlt_tiles<7>(S, N, LD, wd, &bad_dense);
    else if (tiles == 9) dense_ldlt_tiles<9>(S, N, LD, wd, &bad_dense);
    else dense_ldlt_smem(S, N, LD, wd, &bad_dense);
    __syncthreads();
    if (prof) { const long long t = clock64(); a.prof[53] += static_cast<unsigned long long>(t - dt0); dt0 = t; }
    if (warp == 0) {  // x_i = (u_Ni - sum_{k>i} u_ki x_k) / d_i
      constexpr int kQ = 5;
      if (N <= 32 * kQ) {
        // the right-hand side lives in registers (entry k in lane k mod 32, slot k / 32): per step one shuffle, one
        // multiply and the lanes' updates — no shared-memory round trip on the dependency chain
        double r[kQ];
#pragma unroll
        for (int q = 0; q < kQ; ++q) r[q] = 32 * q + lane < N ? rhs[32 * q + lane] : 0.0;
#pragma unroll
        for (int q = kQ - 1; q >= 0; --q) {
          for (int l = 31; l >= 0; --l) {
            const int i = 32 * q + l;
            if (i >= N) continue;
            const double xi = __shfl_sync(0xffffffffu, r[q], l) * wd[i];
            if (lane == l) r[q] = xi;
            const double* row = S + i * LD + lane;
#pragma unroll
            for (int qq = 0; qq <= q; ++qq)
              if (32 * qq + lane < i) r[qq] -= row[32 * qq] * xi;
          }
        }
#pragma unroll
        for (int q = 0; q < kQ; ++q)
          if (32 * q + lane < N) rhs[32 * q + lane] = r[q];
      } else {
        for (int i = N - 1; i >= 0; --i) {
          const double xi = rhs[i] * wd[i];
          __syncwarp();
          if (lane == 0) rhs[i] = xi;
          for (int k = lane; k < i; k += 32) rhs[k] -= S[i * LD + k] * xi;
          __syncwarp();
        }
      }
    }
    __syncthreads();
    if (prof) { const long long t = clock64(); a.prof[54] += static_cast<unsigned long long>(t - dt0); dt0 = t; }
    {
      const int bd = bad_dense;
      for (int i = tid; i < G; i += kCsThreads) a.delta[nfp + i] = bd ? 0.0 : rhs[i];
      for (int e = tid; e < nt * FD; e += kCsThreads) {
        const int t = e / FD, r = e - t * FD;
        a.delta[static_cast<int64_t>(a.n_levels > 1 ? top.orig[t] : t) * FD + r] = bd ? 0.0 : rhs[G + (slot0 + t) * FD + r];
      }
      if (tid == 0 && bd) a.scalars[kScNotPD] = 1.0;
      if (a.do_update && tid < nt) {  // the top nodes' frames
        double d[FD];
        for (int r = 0; r < FD; ++r) d[r] = bd ? 0.0 : rhs[G + (slot0 + tid) * FD + r];
        chain_update_frame(a, b, rinv, a.n_levels > 1 ? top.orig[tid] : tid, d, acc);
      }
      // globals: cameras + IMU parameters (one thread; the step.g / step.D2.step sums over the globals by its warp)
      double gs0 = 0.0, gs1 = 0.0;
      if (a.do_update && warp == kCsThreads / 32 - 1) {
        for (int k = lane; k < G; k += 32) {
          const double d2 = a.D2x ? a.D2x[nfp + k] : lm_damp(b.C[k * G + k], sc[k], rinv);
          const double dk = bd ? 0.0 : rhs[k];
          gs0 += dk * b.gc[k] * sc[k];
          gs1 += dk * dk * d2;
        }
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {  // the total lands in lane 31
          const double t0 = __shfl_up_sync(0xffffffffu, gs0, o), t1 = __shfl_up_sync(0xffffffffu, gs1, o);
          if (lane >= o) { gs0 += t0; gs1 += t1; }
        }
      }
      if (a.do_update && tid == kCsThreads - 1) {
        const double* x_cur = a.state[a.ctl->cur];
        double* x_new = a.state[1 - a.ctl->cur];
        double g4[4] = {gs0, gs1, 0.0, 0.0};
        for (int c = 0; c < a.dp.n_cams; ++c) {
          const CamInfo& ci = a.dp.cams[c];
          const double* x = x_cur + a.dp.off_cam + kCamStateStride * c;
          double* xo = x_new + a.dp.off_cam + kCamStateStride * c;
          double du[3];
          for (int k = 0; k < 3; ++k) du[k] = (bd ? 0.0 : rhs[ci.goff + k]) * sc[ci.goff + k];
          double qo[4];
          so3_plus(x, du, qo);
          for (int k = 0; k < 4; ++k) xo[k] = qo[k];
          for (int k = 0; k < 3; ++k) xo[4 + k] = x[4 + k] + (bd ? 0.0 : rhs[ci.goff + 3 + k]) * sc[ci.goff + 3 + k];
          for (int k = 0; k < 10; ++k)
            xo[7 + k] = x[7 + k] + (k < ci.K ? (bd ? 0.0 : rhs[ci.goff + 6 + k]) * sc[ci.goff + 6 + k] : 0.0);
          for (int k = 0; k < 7 + ci.K; ++k) {
            g4[2] += (xo[k] - x[k]) * (xo[k] - x[k]);
            g4[3] += xo[k] * xo[k];
          }
        }
        {
          const double* x = x_cur + a.dp.off_imu;
          double* xo = x_new + a.dp.off_imu;
          for (int k = 0; k < kImuStateSize; ++k) {
            const double dd = (bd ? 0.0 : rhs[a.dp.imu_goff + k]) * sc[a.dp.imu_goff + k];
            xo[k] = x[k] + dd;
            g4[2] += dd * dd;
            g4[3] += xo[k] * xo[k];
          }
        }
        for (int q = 0; q < 4; ++q) a.step_part[4 * static_cast<int64_t>(nb) + q] = g4[q];
      }
    }
  }
  if (prof) { const long long t = clock64(); a.prof[55] += static_cast<unsigned long long>(t - dt0); }
  mark(kCsProfDense);
  if (a.n_levels <= 2) break;  // the next barrier is the one the whole grid meets at
  barrier(ns);
  // ------------------------------------------------------------ back-substitution, top-down, levels >= 1
  for (int l = a.n_levels - 2; l >= 1; --l) {
    chain_backsub_level<FD>(a.lev[l], l, a.delta, nfp, G, bid * (kCsThreads / 32) + warp, ns * (kCsThreads / 32), lane);
    mark(kCsProfBacksub + (a.n_levels - 2 - l));
    if (l > 1) barrier(ns);
  }
  } while (false);
  // step 0: the CTAs that left the solve work the weights queue.  step 1: everybody — back-substitution of level 0,
  // x (+) step, step statistics.  step 2: the CTAs that stayed with the solve take what is left in the queue.
  for (int step = 0; step < 3; ++step) {
    if (step != 1) {
      if (!wts_go || (step == 0) != left) continue;
      // ---------------------------------------------------------- deferred UpdateImuWeights
      WeightQueueArgs wa;
      wa.dp.off_v = a.dp.off_v; wa.dp.off_imu = a.dp.off_imu; wa.buf = a.buf; wa.ftime = a.ftime; wa.wsqrt = a.wsqrt;
      wa.ni = nf - 1; wa.sigma_g = a.sigma_g; wa.sigma_a = a.sigma_a;
      chain_weights_queue(wa, a.state[a.ctl->cur], wq, smem, &wtask);
      if (step == 2) mark(kCsProfWeights);
      continue;
    }
    // ---------------------------------------------------------- closing phases.  The CTAs that stayed with the solve
    // get here when the levels above level 0 are back-substituted, the CTAs that left when the weights queue is empty.
    // Nobody waits for everybody: level 0 is handed out in items of kCsBsItem nodes, off a counter, to whoever is here
    // once the levels above are done — a CTA still busy with its last weights task holds up neither the
    // back-substitution nor the update of the others (the queue used to keep them all at a grid barrier).  Which warp
    // does a node changes nothing in its result, and the update keeps its fixed frames per CTA.
    unsigned long long* ready = a.sync + 2;  // CTAs that stayed with the solve and are done with the levels above
    unsigned long long* items = a.sync + 3;  // level-0 items handed out
    unsigned long long* done = a.sync + 4;   // level-0 items finished
    if (!left) {
      __syncthreads();
      if (tid == 0) {
        __threadfence();
        atomicAdd(ready, 1ull);
      }
    }
    if (a.n_levels >= 2) {
      const ChainLevel L0 = a.lev[0];
      const int n_items = (chain_backsub_slots(L0) + kCsBsItem - 1) / kCsBsItem;
      if (tid == 0) spin_until(ready, static_cast<unsigned long long>(ns));
      __syncthreads();
      for (;;) {
        if (tid == 0) wtask = atomicAdd(items, 1ull);
        __syncthreads();
        const long long it = static_cast<long long>(wtask);
        if (it >= n_items) break;
#pragma unroll
        for (int u = 0; u < kCsBsItem / (kCsThreads / 32); ++u)
          chain_backsub_node<FD>(L0, 0, a.delta, nfp, G, static_cast<int>(it) * kCsBsItem + u * (kCsThreads / 32) + warp, lane);
        __syncthreads();
        if (tid == 0) {
          __threadfence();
          atomicAdd(done, 1ull);
        }
      }
      mark(kCsProfBacksub + (a.n_levels - 2));
      if (a.do_update) {  // the update reads every frame's step
        if (tid == 0) spin_until(done, static_cast<unsigned long long>(n_items));
        __syncthreads();
      }
    }
    if (!a.do_update) continue;
    // ---------------------------------------------------------- x (+) step of every frame, one thread each (the top
    // nodes' frames were done with the dense solve); a serial tail per node inside the level loop above cost more than
    // this one barrier
    {
      const ChainLevel top = a.lev[a.n_levels - 1];
      int ct = 1;  // c^(n_levels - 1): frame of top node t on one GPU
      for (int k = 1; k < a.n_levels; ++k) ct *= kCsChunk;
      for (int f = bid * kCsThreads + tid; f < nf; f += nb * kCsThreads) {
        bool is_top = false;
        if (a.n_levels > 1) {
          for (int t = 0; t < top.n; ++t) is_top = is_top || (top.ghost ? top.orig[t] : t * ct) == f;
        } else {
          is_top = true;
        }
        if (is_top) continue;
        double d[FD];
#pragma unroll
        for (int r = 0; r < FD; ++r) d[r] = __ldcg(a.delta + static_cast<int64_t>(f) * FD + r);
        chain_update_frame(a, b, rinv, f, d, acc);
      }
    }
    // ---------------------------------------------------------- step statistics of this CTA
#pragma unroll
    for (int q = 0; q < 4; ++q) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], o);
    }
    if (lane == 0)
      for (int q = 0; q < 4; ++q) part[warp][q] = acc[q];
    __syncthreads();
    if (tid == 0) {
      for (int q = 0; q < 4; ++q) {
        double sum = 0.0;
        for (int ww = 0; ww < kCsThreads / 32; ++ww) sum += part[ww][q];
        a.step_part[4 * static_cast<int64_t>(bid) + q] = sum;
      }
    }
    mark(kCsProfUpdate);
  }
}

}  // namespace vc
