// Persistent (cooperative) kernels of the inertial trust-region iteration — one GPU.
//
// An inertial LM iteration on the multi-launch engine is ~20 launches (one chain_eliminate per level, sum_partials,
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
// on the block-tridiagonal + arrow J^T J, SURVEY §8 a12).  The multi-launch engine (vc_imu_host.inl; the solves that do
// not fit here, frame shards without mapped exchange buffers, the per-handle covariance calls) runs the same chunk and
// node routines, one level per launch (chain_eliminate_kernel, chain_backsub_kernel below).
#pragma once
#include <cooperative_groups.h>

#include <type_traits>

#include "vc_chain.cuh"
#include "vc_frame_cov.cuh"
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
  double* Ssum;                 // [G*G+G] summed Schur complement; chain_solve_kernel on one GPU: the dense system [RT][LD]
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
// Above level 0 a chunk's Schur terms from the left (add*: A and g of its c nodes, E of its separator) are staged in the
// coupling columns [0, 3 FD) of V's rows until the couplings step; what does not fit there (G > 109) goes past Eo
__host__ __device__ inline int chain_stage_overflow(int G) {
  constexpr int FD = 9, c = kCsChunk;
  const int over = c * (FD * FD + FD) + FD * G - (c - 1) * FD * 3 * FD;
  return over > 0 ? over : 0;
}
// a group's workspace (chain_eliminate_chunk): Sacc | Al El gl | Ap | Uc | Ur | V | Eo | staging overflow
__host__ __device__ inline size_t chain_group_doubles(int G) {
  constexpr int FD = 9, c = kCsChunk;
  const size_t VW = FD + 2 * FD + G + 1;
  return chain_sacc_doubles(G) + FD * FD + FD * G + FD + (2 * (c - 1) + 1) * FD * FD + (c - 1) * FD * VW + (c - 1) * FD * G +
         chain_stage_overflow(G);
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

// 8-byte copy global -> shared that does not pass through a register, and the wait for all of this thread's copies
__device__ __forceinline__ void cp_async8(double* dst, const double* src) {
  const unsigned d = static_cast<unsigned>(__cvta_generic_to_shared(dst));
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(__cvta_generic_to_global(src)) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

template <int NT>
__device__ __forceinline__ void gsync(int grp) {
  if (NT == kCsThreads) __syncthreads();
  else group_sync(grp);
}
// A chunk's Schur terms: S += sum_i E_i^T X_i[E] (packed lower triangle, Sacc[0, GT)) and rhs += sum_i E_i^T X_i[g]
// (Sacc[GT, GT + G)) over its m interior nodes; E_i row k at Eo + (i FD + k) G, X_i row k at X + (i FD + k) VW (column
// G: g).  Each entry is one FMA chain from 0.0, i then k ascending, added to its accumulator once.  A thread takes a
// 2 x 2 tile of the lower triangle (rows 2 br, 2 br + 1; columns 2 bc, 2 bc + 1; bc <= br) or two rows of the right-hand
// side, so every value it loads from shared memory serves two entries.  Not inlined: in chain_solve_kernel the tiles
// would otherwise cost the kernel more spills.
template <int FD, int NT>
__device__ __noinline__ void chain_schur_acc(double* Sacc, const double* Eo, const double* X, int m, int G, int VW, int tid) {
  const int RB = (G + 1) / 2, nT = RB * (RB + 1) / 2, GT = G * (G + 1) / 2;
  for (int t = tid; t < nT + RB; t += NT) {
    int br = t - nT, c0 = G;  // t >= nT: rows 2 br, 2 br + 1 of the right-hand side
    if (t < nT) {
      int bc = t;
      br = 0;
      while (bc > br) { bc -= br + 1; ++br; }
      c0 = 2 * bc;
    }
    const int r0 = 2 * br, r1 = min(r0 + 1, G - 1), c1 = min(c0 + 1, G);  // (clamped loads of a tile's missing row/column)
    double s00 = 0.0, s01 = 0.0, s10 = 0.0, s11 = 0.0;
    for (int i = 0; i < m; ++i) {
      const double* Ei = Eo + i * FD * G;
      const double* Xi = X + i * FD * VW;
#pragma unroll
      for (int k = 0; k < FD; ++k) {
        const double e0 = Ei[k * G + r0], e1 = Ei[k * G + r1], x0 = Xi[k * VW + c0], x1 = Xi[k * VW + c1];
        s00 += e0 * x0;
        s01 += e0 * x1;
        s10 += e1 * x0;
        s11 += e1 * x1;
      }
    }
    const bool two = r0 + 1 < G;
    if (c0 == G) {
      Sacc[GT + r0] += s00;
      if (two) Sacc[GT + r0 + 1] += s10;
    } else {
      const int k0 = r0 * (r0 + 1) / 2 + c0, k1 = k0 + r0 + 1;  // (r0, c0), (r0 + 1, c0)
      Sacc[k0] += s00;
      if (c0 + 1 <= r0) Sacc[k0 + 1] += s01;
      if (two) {
        Sacc[k1] += s10;
        Sacc[k1 + 1] += s11;
      }
    }
  }
}

// Forward + backward sweep of one chunk (separator s = j*c, interior nodes s+1..s+m) by one group of 128 threads, in
// chain_solve and, one chunk per CTA, in the multi-launch engine's chain_eliminate_kernel.  The chunk's blocks (and
// above level 0 the Schur terms from the chunk on its left) arrive by asynchronous copies straight into shared memory,
// all in flight before the first one is used (no register staging: nothing grows with the chunk length), the 9 x 9
// pivots are factored right-looking with rsqrt, each element of an interior node's solution goes to Z as the sweep
// finishes it, and the group's Schur accumulator Sacc lives on across chunks and levels.
// NT: threads working on the chunk — a group of 128 (two chunks per CTA in flight: the wide levels) or the whole CTA of
// 256 (levels with fewer chunks than CTAs, where the other group would idle); either covers a V row, one column each
template <int FD, int NT>
__device__ __forceinline__ void chain_eliminate_chunk(const NodeSrc& src, const ChainLevel L, const ChainLevel nxt, int G, int j, double* sm,
                                             int tid, int grp, int* bad, unsigned long long* dbg = nullptr) {
  // dbg: cycle counts of the chunk's phases (measurement hook: eight phase clock slots from dbg, one group)
  long long dbg_t = dbg ? clock64() : 0;
  auto tick = [&](int slot) {
    if (dbg && tid == 0) {
      const long long t = clock64();
      dbg[slot] += static_cast<unsigned long long>(t - dbg_t);
      dbg_t = t;
    }
  };
  constexpr int c = kCsChunk;
  const int NS = chain_sacc_doubles(G);
  const int w = 2 * FD + G + 1, VW = FD + w;
  const int oE = 3 * FD, og = 3 * FD + G;  // column offsets inside a V row [U | L | R | E | g]
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
  // The coupling columns [0, 3 FD) of V's rows, which nothing else touches before the couplings step, hold what the
  // in-place step reads (entry t at row t / (3 FD)):
  // level 0: the Jacobi scales of nodes s-1 .. rIdx ([(c+2)][FD], entries [0, kSG)) and of the globals (entries kSG + q);
  // above: the Schur terms of the chunk on the left, addA [nn][FD*FD] | addg [nn][FD] | the separator's addE [FD*G]
  // (entries past kPark in the staging overflow after Eo); the interior nodes' addE goes to Eo
  constexpr int kSG = (c + 2) * FD, kPark = (c - 1) * FD * 3 * FD;
  auto scl = [&](int e) -> double* { return V + (e / (3 * FD)) * VW + e % (3 * FD); };  // e < kPark
  auto stg = [&](int e) -> double* { return e < kPark ? scl(e) : Eo + (c - 1) * FD * G + (e - kPark); };
  const bool add = !lvl0 && L.addA != nullptr;  // (the host sets the three add* together)
  const int oSg = nn * FD * FD, oSE = nn * (FD * FD + FD);
  // couplings of the interior nodes' right-hand sides from the staged U blocks: entry t < m * 3 FD * FD of the coupling
  // columns (interior node t / (3 FD * FD): H[p, p+1] | H[p0, s] = U[p0]^T | H[pl, rIdx])
  auto coupling = [&](int t) -> double {
    const int i = t / (3 * FD * FD), rc = t - i * 3 * FD * FD, r = rc / (3 * FD), col = rc - r * 3 * FD;
    const int blk = col / FD, q = col - blk * FD;
    const bool lastI = i == m - 1;
    const double* Unext = lastI ? Ur : Uc + (i + 1) * FD * FD;  // H[p, p+1]
    const double unext = (!lastI || hasR) ? Unext[r * FD + q] : 0.0;
    if (blk == 0) return lastI ? 0.0 : unext;
    if (blk == 1) return i == 0 ? Uc[q * FD + r] : 0.0;
    return (lastI && hasR) ? unext : 0.0;
  };
  // ---- the chunk's blocks as stored (level 0: the unscaled normal equations and the scales; above: the Schur terms of
  // the chunk on the left as well), one round of copies
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
    if (add) {  // (8-byte copies, so .ca: cp.async.cg copies 16 bytes only; the level barrier's acquire orders them, as the blocks)
      const int64_t o = static_cast<int64_t>(s);
      for (int e = tid; e < nn * FD * FD; e += NT) cp_async8(stg(e), L.addA + o * FD * FD + e);
      for (int e = tid; e < nn * FD; e += NT) cp_async8(stg(oSg + e), L.addg + o * FD + e);
      for (int e = tid; e < nn * FD * G; e += NT) cp_async8(e < FD * G ? stg(oSE + e) : Eo + (e - FD * G), L.addE + o * FD * G + e);
    }
    cp_async_wait_all();
  }
  gsync<NT>(grp);
  tick(1);
  // ---- in place: level 0 scales and damps, deeper levels add the Schur terms of the chunk on the left (block + add)
  const int nC = m * 3 * FD * FD;
  if (lvl0) {
    for (int e = tid; e < nn * FD * FD; e += NT) {
      const int nd = e / (FD * FD), el = e - nd * FD * FD, r = el / FD, q = el - r * FD;
      double* d = nd == 0 ? Al + el : Ap + (e - FD * FD);
      const double a = *d, sr = *scl((nd + 1) * FD + r), sq = *scl((nd + 1) * FD + q);
      double v = a * sr * sq;
      // frame_damp's rule, written out as in src_A (a chunk's nodes s .. s + m stop short of the ghost)
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
    // the interior nodes' E also goes to Eo as the sweeps will see it, kept for the Schur product
    for (int e = tid, R = rG0, q = qG0; e < nn * FD * G; e += NT, adv2(R, q, G, NT)) {
      double* d = R < FD ? El + e : V + (R - FD) * VW + oE + q;
      const double v = *d * *scl(FD + R) * *scl(kSG + q);
      *d = v;
      if (R >= FD) Eo[e - FD * G] = v;
    }
    gsync<NT>(grp);
    tick(2);
    for (int t = tid; t < nC; t += NT) *scl(t) = coupling(t);
    gsync<NT>(grp);
    tick(3);
  } else {
    // entry t of the coupling columns is read (staged add) and then written (coupling) by the same thread
    const int nS = add ? oSE + FD * G : 0;
    for (int t = tid; t < max(nS, nC); t += NT) {
      double* st = stg(t);
      if (t < nS) {
        double* d = t < oSg ? (t < FD * FD ? Al + t : Ap + (t - FD * FD))
                  : t < oSE ? (t - oSg < FD ? gl + (t - oSg) : V + (t - oSg - FD) * VW + og)
                            : El + (t - oSE);
        *d = *d + *st;
      }
      if (t < nC) *st = coupling(t);
    }
    // the interior nodes' E: staged add in Eo, where the sum stays for the Schur product
    for (int e = FD * G + tid, R = FD + rG0, q = qG0; e < nn * FD * G; e += NT, adv2(R, q, G, NT)) {
      double* d = V + (R - FD) * VW + oE + q;
      const double v = add ? *d + Eo[e - FD * G] : *d;
      *d = v;
      Eo[e - FD * G] = v;
    }
    gsync<NT>(grp);
    tick(2);
  }
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
      if (i == m - 1 && q >= FD) {  // the last interior node's solution is final here: its Z row, columns [L | R | E | g]
        double* Z = L.Z + (static_cast<int64_t>(s) + 1 + i) * FD * w + (q - FD);
#pragma unroll
        for (int ii = 0; ii < FD; ++ii) Z[ii * w] = x[ii];
      }
    }
    gsync<NT>(grp);
  }
  tick(4);
  // ---- backward sweep: X_i = V_R(i) - V_U(i) X_{i+1}, each element stored to Z as it is finished
  for (int i = m - 2; i >= 0; --i) {
    double* Vi = V + static_cast<int64_t>(i) * FD * VW;
    const double* Vn = V + static_cast<int64_t>(i + 1) * FD * VW;
    double* Z = L.Z + (static_cast<int64_t>(s) + 1 + i) * FD * w;
    for (int e = tid, r = rw0, qq = qw0; e < FD * w; e += NT, adv2(r, qq, w, NT)) {
      const int q = FD + qq;
      double sum = 0.0;
#pragma unroll
      for (int k = 0; k < FD; ++k) sum += Vi[r * VW + k] * Vn[k * VW + q];
      const double x = Vi[r * VW + q] - sum;
      Vi[r * VW + q] = x;
      Z[e] = x;
    }
    gsync<NT>(grp);
  }
  tick(5);
  // ---- the Schur terms: S += E_i^T X_i[E], rhs += E_i^T X_i[g]
  chain_schur_acc<FD, NT>(Sacc, Eo, V + oE, m, G, VW, tid);
  tick(6);
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
  tick(7);
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

// ------------------------------------------------------------------ the multi-launch engine (vc_imu_host.inl)
// One level of the elimination per launch, one CTA per separator-led chunk, chain_solve's chunk routine on the CTA's
// own Schur accumulator.  The CTA's partial is written unpacked, [G*G + G]: both triangles from the packed lower one,
// then the right-hand side, the layout sum_partials_kernel, dense_solve_kernel and the sharded all-reduce take.
// NT: kCsGroup threads where they cover a V row (3 FD + G + 1 columns, one pivot solve each), else kCsThreads.
struct ElimArgs {
  DevProblem dp;
  Blocks b[2];
  const Ctl* ctl;
  const double* scale;
  const double* D2x;
  const double* sepdiag;
  const ChainLevel* lev;  // the level table (device memory)
  int l;                  // the level eliminated: lev[l] -> lev[l + 1]
  double* Spart;          // [gridDim][G*G+G]
  double* scalars;
};
template <int NT>
__global__ void __launch_bounds__(NT) chain_eliminate_kernel(ElimArgs a) {
  extern __shared__ double sm[];  // chain_group_doubles(G)
  __shared__ int bad;
  if (a.ctl->done) return;
  constexpr int FD = 9;
  const int G = a.dp.G, GT = G * (G + 1) / 2, tid = threadIdx.x;
  const NodeSrc src = chain_src(a.l > 0 ? a.lev + a.l : nullptr, a.dp, a.b, a.ctl, a.scale, a.D2x, a.sepdiag);
  if (tid == 0) bad = 0;
  for (int e = tid; e < chain_sacc_doubles(G); e += NT) sm[e] = 0.0;
  chain_eliminate_chunk<FD, NT>(src, a.lev[a.l], a.lev[a.l + 1], G, blockIdx.x, sm, tid, 0, &bad);
  __syncthreads();
  if (tid == 0 && bad) a.scalars[kScNotPD] = 1.0;
  double* out = a.Spart + static_cast<int64_t>(blockIdx.x) * (G * G + G);
  for (int e = tid; e < G * G; e += NT) {
    const int r = e / G, c = e - r * G, hi = max(r, c), lo = min(r, c);
    out[e] = sm[hi * (hi + 1) / 2 + lo];
  }
  for (int r = tid; r < G; r += NT) out[G * G + r] = sm[GT + r];
}

// One level of the back-substitution per launch, one warp per node slot (chain_backsub_slots)
struct BacksubArgs {
  const Ctl* ctl;
  int G, l;
  ChainLevel cur;
  double* delta;
  int64_t nfp;
};
constexpr int kBacksubWarps = 4;
__global__ void __launch_bounds__(32 * kBacksubWarps) chain_backsub_kernel(BacksubArgs a) {
  const int slot = blockIdx.x * kBacksubWarps + (threadIdx.x >> 5);
  if (a.ctl->done || slot >= chain_backsub_slots(a.cur)) return;
  chain_backsub_node<9>(a.cur, a.l, a.delta, a.nfp, a.G, slot, threadIdx.x & 31);
}

// The back-substitution of every level on the cooperative grid, by whichever CTA calls it: items of kCsBsItem nodes at
// level 0 and of one node per warp above it (the levels above have 28 and 224 nodes on the target: items of 16 would
// leave most warps idle and double the rounds of those that work), levels top-down (the items of level l after all those of the levels above), off the counter sync[3].  An item of the
// top level waits for sync[2] (1 once the dense solve has written the globals' and the top nodes' steps), an item of a
// lower level for the count of finished items sync[4] to cover every level above — items are handed out in order, so
// that count cannot include one of its own level before.  wait_all: return when every item is done (the update reads
// every frame's step).  A function of its own with by-value arguments, as chain_weights_queue: inlined into the solve
// kernel it raised the kernel's spills.  prof: CTA 0's phase clocks (thread 0 only, else null), t_prev the time of
// its last mark; returns the time of the last mark here.
template <int FD>
__device__ __noinline__ unsigned long long chain_backsub_items(const ChainLevel* lev, int n_levels, double* delta, int64_t nfp, int G,
                                                               unsigned long long* sync, bool wait_all, unsigned long long* wtask,
                                                               unsigned long long* prof, unsigned long long t_prev) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  unsigned long long* ready = sync + 2;
  unsigned long long* items = sync + 3;
  unsigned long long* done = sync + 4;
  auto item_nodes = [](int l) { return l == 0 ? kCsBsItem : kCsThreads / 32; };
  auto level_items = [&](int l) { return (chain_backsub_slots(lev[l]) + item_nodes(l) - 1) / item_nodes(l); };
  auto mark = [&](int l) {  // the time since the last mark to back-substitution level l's clock
    if (prof) {
      const unsigned long long t = global_ns();
      prof[kCsProfBacksub + (n_levels - 2 - l)] += t - t_prev;
      t_prev = t;
    }
  };
  const int l_top = n_levels - 2;
  int n_items = 0;
  for (int l = l_top; l >= 0; --l) n_items += level_items(l);
  int cl = l_top, n_cl = level_items(l_top);  // level of this CTA's current item, and its items
  int before = 0;                             // items of the levels above cl
  for (;;) {
    if (tid == 0) *wtask = atomicAdd(items, 1ull);
    __syncthreads();
    const int it = static_cast<int>(*wtask);
    if (it >= n_items) break;
    while (it >= before + n_cl) {
      mark(cl);
      before += n_cl;
      n_cl = level_items(--cl);
    }
    if (tid == 0) {
      if (cl == l_top) spin_until(ready, 1ull);
      else spin_until(done, static_cast<unsigned long long>(before));
    }
    __syncthreads();
    const ChainLevel L = lev[cl];
    const int nodes = item_nodes(cl);
    for (int u = 0; u < nodes / (kCsThreads / 32); ++u)
      chain_backsub_node<FD>(L, cl, delta, nfp, G, (it - before) * nodes + u * (kCsThreads / 32) + warp, lane);
    __syncthreads();
    if (tid == 0) {
      __threadfence();
      atomicAdd(done, 1ull);
    }
  }
  mark(cl);
  if (wait_all) {
    if (tid == 0) spin_until(done, static_cast<unsigned long long>(n_items));
    __syncthreads();
  }
  return t_prev;
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
// entry k of the summed Schur complement: the nb CTAs' packed partials p[c * NS] added in CTA order, kCsRedLoads loads
// in flight
__device__ __forceinline__ double schur_entry(const double* p, int nb, int NS) {
  double s = 0.0;
  int c = 0;
  for (; c + kCsRedLoads <= nb; c += kCsRedLoads) {
    double v[kCsRedLoads];
#pragma unroll
    for (int u = 0; u < kCsRedLoads; ++u) v[u] = __ldcg(p + (c + u) * NS);
#pragma unroll
    for (int u = 0; u < kCsRedLoads; ++u) s += v[u];
  }
  for (; c < nb; ++c) s += __ldcg(p + c * NS);
  return s;
}
// The [globals | top nodes] system of a run on one GPU as chain_solve's dense phase factors it — S [RT][LD] with the
// right-hand side as row N and zeros everywhere else — written to a.Ssum, entries e0, e0 + stride, ...  First the
// globals' block and right-hand side (an entry per thread of the solver CTAs, as the Schur reduction alone had: each
// sums the nb partials), then the top nodes' blocks and the zeros.  Every entry is formed by the operations, in the
// order, of the dense phase's own assembly (which sharded runs and clusters keep), so the system is bit for bit the same.
__device__ __forceinline__ void dense_assemble(const ChainSolveArgs& a, const Blocks& b, double rinv, int nb, int e0, int stride) {
  constexpr int FD = 9;
  const int G = a.dp.G, NS = G * G + G;
  const int64_t nfp = static_cast<int64_t>(a.dp.n_frames) * FD;
  const ChainLevel& top = a.lev[a.n_levels - 1];
  const int N = G + top.n * FD, LD = dense_ld(N), RT = dense_rows(N);
  const double* sc = a.scale + nfp;
  double* S = a.Ssum;
  for (int e = e0; e < NS; e += stride) {
    const int r = e / G, q = e - r * G;
    const int k = r < G ? (q <= r ? r * (r + 1) / 2 + q : -1) : G * (G + 1) / 2 + q;
    const double p = k >= 0 ? schur_entry(a.Spart + k, nb, NS) : 0.0;
    const double cv = b.C[e];  // C | gc are contiguous
    if (r < G) {
      double v = cv * sc[r] * sc[q] - p;
      if (r == q) v += global_damp(r, cv, sc[r], rinv, a.D2x, nfp);
      S[r * LD + q] = v;
    } else {
      S[N * LD + q] = -cv * sc[q] + p;
    }
  }
  const bool add = top.addA != nullptr;
  auto entry = [&](int e) -> double {  // a top node's entry, or a zero
    const int r = e / LD, c = e - r * LD;
    double v = 0.0;
    if (r <= N && c < N) {
      const int tc = (c - G) / FD, cc = (c - G) - tc * FD;  // top node and row of column c (c >= G unless G <= r < N)
      if (r == N) {
        const int64_t o = static_cast<int64_t>(tc) * FD + cc;
        v = -(__ldcg(top.g + o) + (add ? __ldcg(top.addg + o) : 0.0));
      } else if (r < G) {  // E of top node tc, transposed
        const int64_t o = static_cast<int64_t>(tc) * FD * G + cc * G + r;
        v = __ldcg(top.E + o) + (add ? __ldcg(top.addE + o) : 0.0);
      } else {
        const int tr = (r - G) / FD, rr = (r - G) - tr * FD;
        if (c < G) {
          const int64_t o = static_cast<int64_t>(tr) * FD * G + rr * G + c;
          v = __ldcg(top.E + o) + (add ? __ldcg(top.addE + o) : 0.0);
        } else if (tc == tr) {
          const int64_t o = static_cast<int64_t>(tr) * FD * FD + rr * FD + cc;
          v = __ldcg(top.A + o) + (add ? __ldcg(top.addA + o) : 0.0);
        } else if (tc == tr + 1) {
          v = __ldcg(top.U + static_cast<int64_t>(tc) * FD * FD + rr * FD + cc);  // H[tr, tc]
        } else if (tr == tc + 1) {
          v = __ldcg(top.U + static_cast<int64_t>(tr) * FD * FD + cc * FD + rr);  // H[tc, tr] transposed
        }
      }
    }
    return v;
  };
  for (int e = e0; e < RT * LD; e += stride) {
    const int r = e / LD, c = e - r * LD;
    if (c < G && (r < G || r == N)) continue;  // written above
    S[e] = entry(e);
  }
}
// DOGLEG's step (vc_dogleg.cuh) of the rig `a` and its update, by the CTAs of one cluster, once every frame's Gauss-Newton
// step x = (H + mu D^2)^-1 (-g) is in a.delta (H = S J^T J S, D = sqrt(clamp(diag H)), g~ = g / D, u = g~ / D, gn = D x).
// The six step scalars of the persistent vision kernel (kDlG2 .. kDlXHx): per CTA, one warp per frame of frames bid * 8
// + warp, + 8 nb, ... — |g~_f|^2, |gn_f|^2, g~_f.gn_f and the frame rows of u.Hu, u.Hx, x.Hx over the block-tridiagonal +
// arrow system: B_f, the couplings U to both neighbours, E_f both ways — the warps added in order, CTA 0 adding the
// globals' rows (C and their own entries); one slot per CTA (a.Spart: the Schur partials are spent by now); a cluster
// barrier; every CTA adds the slots up in CTA order, takes dogleg_point() and the same (cg, cn).  Then x (+) S step of
// every frame and of the globals with step = (cg g~ + cn gn) / D (0 when the solve failed), into acc and the globals'
// step_part slot as the LM update writes them.  The model change -step.g - step.H.step / 2 is expanded over the explicit
// products, as the vision kernel forms it: -(cg |g~|^2 + cn g~.gn) - (cg^2 u.Hu + 2 cg cn u.Hx + cn^2 x.Hx) / 2.
// sm: 3 G doubles of free shared memory.
__device__ __noinline__ void chain_dogleg_update(const ChainSolveArgs& a, ClusterScope scope, double mu, double* sm, double* acc) {
  constexpr int FD = 9;
  constexpr int kWarps = kCsThreads / 32;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nb = scope.nb(), bid = scope.bid();
  const int G = a.dp.G, NS = G * G + G, nf = a.dp.n_frames;
  const int64_t nfp = static_cast<int64_t>(nf) * FD;
  const Blocks& b = a.b[a.ctl->cur];
  const double* s = a.scale;
  __shared__ double wpart[kWarps][kDlParts];
  __shared__ double step_s[3];  // cg, cn, ok
  double* pug = sm;       // [G] s u of the globals
  double* pxg = pug + G;  // [G] s x
  double* dg = pxg + G;   // [G] the globals' step
  for (int k = tid; k < G; k += kCsThreads) {
    double D, gt;
    dl_scaled(b.C[k * G + k], b.gc[k], s[nfp + k], &D, &gt);
    pug[k] = s[nfp + k] * (gt / D);
    pxg[k] = s[nfp + k] * __ldcg(a.delta + nfp + k);
  }
  __syncthreads();
  double q[kDlParts] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int f = bid * kWarps + warp; f < nf; f += nb * kWarps) {
    const int64_t o = static_cast<int64_t>(f) * FD;
    // lane l < 27: entry l % 9 of frame f - 1 + l / 9 (s u, s x); lane r < 9 works row r of frame f
    double pu = 0.0, px = 0.0, gt = 0.0, D = 1.0, x = 0.0;
    {
      const int node = f - 1 + lane / FD, r = lane % FD;
      if (lane < 3 * FD && node >= 0 && node < nf) {
        const int64_t i = static_cast<int64_t>(node) * FD + r;
        dl_scaled(b.B[i * FD + r], b.gf[i], s[i], &D, &gt);
        x = __ldcg(a.delta + i);
        pu = s[i] * (gt / D);
        px = s[i] * x;
      }
    }
    double hu = 0.0, hx = 0.0;
    const int r = lane < FD ? lane : 0;
#pragma unroll
    for (int c = 0; c < FD; ++c) {  // B_f
      const double bv = b.B[(o + r) * FD + c];
      hu += bv * __shfl_sync(0xffffffffu, pu, FD + c);
      hx += bv * __shfl_sync(0xffffffffu, px, FD + c);
    }
#pragma unroll
    for (int c = 0; c < FD; ++c) {  // U[f] = H[f-1, f]: U[f]^T (f - 1);  U[f+1] (f + 1)
      const double ul = f > 0 ? b.U[o * FD + c * FD + r] : 0.0;
      const double ur = f + 1 < nf ? b.U[(o + FD) * FD + r * FD + c] : 0.0;
      hu += ul * __shfl_sync(0xffffffffu, pu, c) + ur * __shfl_sync(0xffffffffu, pu, 2 * FD + c);
      hx += ul * __shfl_sync(0xffffffffu, px, c) + ur * __shfl_sync(0xffffffffu, px, 2 * FD + c);
    }
    double eu = 0.0, ex = 0.0;
#pragma unroll
    for (int rr = 0; rr < FD; ++rr) {  // E_f s u_g, E_f s x_g: lanes split the columns
      double su = 0.0, sx = 0.0;
      for (int c = lane; c < G; c += 32) {
        const double e = b.E[(o + rr) * G + c];
        su += e * pug[c];
        sx += e * pxg[c];
      }
#pragma unroll
      for (int k = 16; k > 0; k >>= 1) {
        su += __shfl_xor_sync(0xffffffffu, su, k);
        sx += __shfl_xor_sync(0xffffffffu, sx, k);
      }
      eu = rr == r ? su : eu;
      ex = rr == r ? sx : ex;
    }
    // the own entry of row r sits in lane 9 + r
    const double pur = __shfl_sync(0xffffffffu, pu, FD + r), pxr = __shfl_sync(0xffffffffu, px, FD + r);
    const double gtr = __shfl_sync(0xffffffffu, gt, FD + r), Dr = __shfl_sync(0xffffffffu, D, FD + r);
    const double xr = __shfl_sync(0xffffffffu, x, FD + r);
    if (lane < FD) {
      const double gn = xr * Dr;
      q[kDlG2] += gtr * gtr;
      q[kDlGn2] += gn * gn;
      q[kDlB] += gtr * gn;
      q[kDlUHu] += pur * (hu + 2.0 * eu);
      q[kDlUHx] += pur * (hx + ex) + pxr * eu;
      q[kDlXHx] += pxr * (hx + 2.0 * ex);
    }
  }
  if (bid == 0) {  // the globals' rows: C and their own entries
    for (int k = tid; k < G; k += kCsThreads) {
      double cu = 0.0, cx = 0.0;
      for (int c = 0; c < G; ++c) {
        const double cv = b.C[k * G + c];
        cu += cv * pug[c];
        cx += cv * pxg[c];
      }
      double D, gt;
      dl_scaled(b.C[k * G + k], b.gc[k], s[nfp + k], &D, &gt);
      const double gn = __ldcg(a.delta + nfp + k) * D;
      q[kDlG2] += gt * gt;
      q[kDlGn2] += gn * gn;
      q[kDlB] += gt * gn;
      q[kDlUHu] += pug[k] * cu;
      q[kDlUHx] += pug[k] * cx;
      q[kDlXHx] += pxg[k] * cx;
    }
  }
#pragma unroll
  for (int j = 0; j < kDlParts; ++j)
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) q[j] += __shfl_xor_sync(0xffffffffu, q[j], k);
  if (lane == 0)
    for (int j = 0; j < kDlParts; ++j) wpart[warp][j] = q[j];
  __syncthreads();
  if (tid == 0) {
    for (int j = 0; j < kDlParts; ++j) {
      double t = 0.0;
      for (int w = 0; w < kWarps; ++w) t += wpart[w][j];
      a.Spart[static_cast<int64_t>(bid) * NS + j] = t;
    }
  }
  scope.sync();
  if (tid == 0) {  // every CTA alike: the totals in CTA order, the dogleg point
    double t[kDlParts] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int c = 0; c < nb; ++c)
      for (int j = 0; j < kDlParts; ++j) t[j] += __ldcg(a.Spart + static_cast<int64_t>(c) * NS + j);
    const int ok = __ldcg(a.scalars + kScNotPD) > 0.0 ? 0 : 1;
    const double alpha = t[kDlG2] / t[kDlUHu];
    double cg, cn;
    const double step_norm = dogleg_point(a.ctl->radius, alpha, t[kDlG2], t[kDlGn2], t[kDlB], &cg, &cn);
    if (!ok) cg = cn = 0.0;
    step_s[0] = cg; step_s[1] = cn; step_s[2] = ok;
    if (bid == 0) {
      Ctl* c = a.ctl;
      c->dl_g2 = t[kDlG2];
      c->dl_alpha = alpha;
      c->dl_gn2 = t[kDlGn2];
      c->dl_b = t[kDlB];
      c->dl_ok = ok;
      c->dl_step_norm = step_norm;
      c->dl_model_change = -(cg * t[kDlG2] + cn * t[kDlB]) - 0.5 * (cg * cg * t[kDlUHu] + 2.0 * cg * cn * t[kDlUHx] + cn * cn * t[kDlXHx]);
    }
  }
  __syncthreads();
  const double cg = step_s[0], cn = step_s[1];
  const bool ok = step_s[2] != 0.0;
  const double* x_cur = a.state[a.ctl->cur];
  double* x_new = a.state[1 - a.ctl->cur];
  for (int f = bid * kCsThreads + tid; f < nf; f += nb * kCsThreads) {  // every frame, the top nodes' too
    double d[FD];
#pragma unroll
    for (int r = 0; r < FD; ++r) {
      const int64_t i = static_cast<int64_t>(f) * FD + r;
      double D, gt;
      dl_scaled(b.B[i * FD + r], b.gf[i], s[i], &D, &gt);
      d[r] = ok ? (cg * gt + cn * (__ldcg(a.delta + i) * D)) / D : 0.0;
    }
    frame_plus<FD>(a.dp, b, s, mu, a.D2x, a.sepdiag, f, d, true, x_cur, x_new, acc);
  }
  if (bid == 0) {
    for (int k = tid; k < G; k += kCsThreads) {
      double D, gt;
      dl_scaled(b.C[k * G + k], b.gc[k], s[nfp + k], &D, &gt);
      dg[k] = ok ? (cg * gt + cn * (__ldcg(a.delta + nfp + k) * D)) / D : 0.0;
    }
    __syncthreads();
    if (tid == kCsThreads - 1) {
      double g4[4] = {0.0, 0.0, 0.0, 0.0};
      for (int k = 0; k < G; ++k) {
        g4[0] += dg[k] * b.gc[k] * s[nfp + k];
        g4[1] += dg[k] * dg[k] * global_damp(k, b.C[k * G + k], s[nfp + k], mu, a.D2x, nfp);
      }
      globals_plus(a.dp, x_cur, x_new, dg, s + nfp, g4 + 2);
      for (int k = 0; k < 4; ++k) a.step_part[4 * static_cast<int64_t>(nb) + k] = g4[k];
    }
  }
}

// One damped solve of the frame-chain + globals system and (optionally) the state update of the rig `a`, by the CTAs
// of `scope` (vc_mega.cuh): the cooperative grid (chain_solve_kernel) or one thread-block cluster (chain_solve_batch_kernel).
// The barriers count arrivals on the rig's own counters (a.sync) either way; the CTAs of a cluster are co-scheduled, as
// those of a cooperative grid are, so a CTA that spins on them never waits for one that has not started.  A cluster is
// never sharded: the exchange is compiled out for it.
// kCov (chain_cov_batch_kernel, with a.D2x set): the elimination, the Schur reduction and the dense factorisation only;
// in place of the dense phase's right-hand side, the G unit right-hand sides of the globals give the globals' block of
// the [globals | top nodes] inverse, unscaled into cov (G x G; mask: 0 on constant globals).  No step, no state update.
// kFrame (with kCov; chain_frame_cov_batch_kernel): no right-hand side at all; the factorisation stays in CTA 0's shared
// memory for the caller (the L D L^T factor S [RT][LD], then 1 / d at S + RT LD).
// Str = kDogleg (clusters only, with a.do_update): the Gauss-Newton step with the damping mu D^2 (mu = Ctl::dl_mu in
// place of LM's 1 / radius in the same damping rule), then chain_dogleg_update in place of the LM update.
template <class Scope, bool kCov = false, bool kFrame = false, Strategy Str = Strategy::kLM>
__device__ __forceinline__ void chain_solve(const ChainSolveArgs& a, Scope scope, const double* mask = nullptr, double* cov = nullptr) {
  constexpr bool kDl = Str == Strategy::kDogleg;
  static_assert(!kDl || (std::is_same<Scope, ClusterScope>::value && !kCov), "DOGLEG runs in the cluster solve");
  extern __shared__ double smem[];
  constexpr int FD = 9;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int grp = tid / kCsGroup, gtid = tid - grp * kCsGroup;
  const int nb = scope.nb(), bid = scope.bid();
  const int n_groups = nb * kCsGroups, gid = bid * kCsGroups + grp;
  const int G = a.dp.G, NS = G * G + G, nf = a.dp.n_frames;
  const int64_t nfp = static_cast<int64_t>(nf) * FD;
  __shared__ int bad_s[kCsGroups];
  __shared__ int bad_dense;
  __shared__ double part[kCsThreads / 32][4];
  __shared__ unsigned long long wtask;
  __shared__ unsigned long long* xbufs[kMaxRanks];
  if constexpr (Scope::kSharded) xchg_stage(a.x, xbufs);  // (visible after the first barrier below)
  if (bid == 0 && tid == 0)
    for (int k = 0; k < kCsSyncWords; ++k) a.sync_next[k] = 0ull;
  if (a.ctl->done) return;  // uniform over the grid: written before this launch
  const Blocks& b = a.b[a.ctl->cur];
  const double rinv = kDl ? a.ctl->dl_mu : 1.0 / a.ctl->radius;  // the damping's multiplier of clamp(diag H)
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
  // The queue is the grid's: a cluster of at most 8 CTAs has none to spare (a batch computes the weights in its
  // evaluation launch), and compiled into the cluster kernel too it would change how ptxas allocates the grid kernel's call.
  constexpr bool kQueue = std::is_same<Scope, GridScope>::value;
  const bool wts_go = kQueue && a.wts_on && !a.dp.rotation_only && a.ctl->iter > 0 && a.ctl->last_accepted;
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
    // chunk phase clocks (measurement hook): level 0 on CTA 0's group 0 in slots [56, 64), level 1 on CTA 0 in [40, 48)
    unsigned long long* dbg = a.prof && bid == 0 && l < 2 ? a.prof + (l == 0 ? 56 : 40) : nullptr;
    if (nsep > nb || !a.narrow_ok) {  // wide level: two chunks per CTA in flight
      for (int j = gid; j < nsep; j += n_groups)
        chain_eliminate_chunk<FD, kCsGroup>(src, Lc, Ln, G, j, gsm, gtid, grp, &bad_s[grp], grp == 0 ? dbg : nullptr);
    } else {          // narrow level: the whole CTA on one chunk (group 0's workspace and Schur accumulator)
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
  // On the grid on one GPU the same threads assemble the dense system as CTA 0 factors it, in its padded [RT][LD]
  // layout, in a.Ssum (sized for it): the operations of the assembly CTA 0 does otherwise, in the same order, so the
  // system is bit for bit the same, and CTA 0 copies it in one round of asynchronous copies.
  const bool sharded = Scope::kSharded && a.x.nranks > 1;
  const bool assemble = kQueue && !sharded;
  if (assemble) {
    dense_assemble(a, b, rinv, nb, bid * kCsThreads + tid, ns * kCsThreads);
  } else {
    for (int e = bid * kCsThreads + tid; e < NS; e += ns * kCsThreads) {
      const int r = e / G, q = e - r * G;
      const int k = r < G ? (q <= r ? r * (r + 1) / 2 + q : -1) : G * (G + 1) / 2 + q;
      a.Ssum[e] = k >= 0 ? schur_entry(a.Spart + k, nb, NS) : 0.0;
    }
  }
  mark(kCsProfReduce);
  barrier(ns);
  // ------------------------------------------------------------ sharded: the ranks' partial systems meet here
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
            if (r == c) v += global_damp(r, b.C[e], sc[r], rinv, a.D2x, nfp);
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
    if (assemble) {  // assembled by the Schur reduction (dense_assemble)
      for (int e = tid; e < RT * LD; e += kCsThreads) cp_async8(S + e, a.Ssum + e);
      cp_async_wait_all();
    } else {
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
          if (r == c) v += global_damp(r, cv[u], sc[r], rinv, a.D2x, nfp);
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
    if constexpr (kCov) {  // one warp per right-hand side at a time, in registers: no shared memory beyond the factors
      if (bad_dense) {
        if (tid == 0) a.scalars[kScNotPD] = 1.0;
        return;
      }
      if constexpr (kFrame) return;
      for (int j = warp; j < G; j += kCsThreads / 32) {
        double x[kCovQ] = {0.0, 0.0, 0.0, 0.0};
        if (mask[j] != 0.0) warp_inverse_column<kCovQ, true>(S, LD, wd, N, j, lane, x);
        cov_store_column<kCovQ>(x, sc, mask, G, j, lane, cov);
      }
      return;
    }
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
      if (!kDl && a.do_update && tid < nt) {  // the top nodes' frames
        double d[FD];
        for (int r = 0; r < FD; ++r) d[r] = bd ? 0.0 : rhs[G + (slot0 + tid) * FD + r];
        frame_plus<FD>(a.dp, b, a.scale, rinv, a.D2x, a.sepdiag, a.n_levels > 1 ? top.orig[tid] : tid, d, true, a.state[a.ctl->cur],
                       a.state[1 - a.ctl->cur], acc);
      }
      // globals: cameras + IMU parameters (one thread; the step.g / step.D2.step sums over the globals by its warp)
      double gs0 = 0.0, gs1 = 0.0;
      if (!kDl && a.do_update && warp == kCsThreads / 32 - 1) {
        for (int k = lane; k < G; k += 32) {
          const double d2 = global_damp(k, b.C[k * G + k], sc[k], rinv, a.D2x, nfp);
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
      if (!kDl && a.do_update && tid == kCsThreads - 1) {
        const double* x_cur = a.state[a.ctl->cur];
        double* x_new = a.state[1 - a.ctl->cur];
        double g4[4] = {gs0, gs1, 0.0, 0.0};
        globals_plus(a.dp, x_cur, x_new, bd ? nullptr : rhs, sc, g4 + 2);
        for (int q = 0; q < 4; ++q) a.step_part[4 * static_cast<int64_t>(nb) + q] = g4[q];
      }
    }
    if constexpr (kQueue) {  // the back-substitution may start: the globals' and the top nodes' steps are in a.delta
      __syncthreads();
      if (tid == 0) {
        __threadfence();
        atomicAdd(a.sync + 2, 1ull);
      }
    }
  }
  if constexpr (kCov) return;  // the other CTAs: nothing after the elimination
  if (prof) { const long long t = clock64(); a.prof[55] += static_cast<unsigned long long>(t - dt0); }
  mark(kCsProfDense);
  if constexpr (kQueue) break;  // every level of the back-substitution is handed out in the closing phases
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
    // get here when they are done with the solve, the CTAs that left when the weights queue is empty.  Nobody waits for
    // everybody: the back-substitution is handed out in items of kCsBsItem nodes, off a counter, to whoever is here —
    // a CTA still busy with its last weights task holds up neither the back-substitution nor the update of the others.
    // On the grid every level is handed out so (chain_backsub_items).  A cluster hands out level 0 only, once its CTAs
    // are done with the levels above.  Which warp does a node changes nothing in its result, and the update keeps its
    // fixed frames per CTA.
    if constexpr (kQueue) {
      if (a.n_levels >= 2) t_prev = chain_backsub_items<FD>(a.lev, a.n_levels, a.delta, nfp, G, a.sync, a.do_update != 0, &wtask,
                                                            prof ? a.prof : nullptr, t_prev);
    } else {
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
    }
    if (!a.do_update) continue;
    if constexpr (kDl) {
      if (a.n_levels < 2) scope.sync();  // (no back-substitution: CTA 0's dense phase wrote every step)
      chain_dogleg_update(a, scope, rinv, smem, acc);
    } else {
    // ---------------------------------------------------------- x (+) step of every frame, one thread each (the top
    // nodes' frames were done with the dense solve); a serial tail per node inside the level loop above cost more than
    // this one barrier
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
        frame_plus<FD>(a.dp, b, a.scale, rinv, a.D2x, a.sepdiag, f, d, true, a.state[a.ctl->cur], a.state[1 - a.ctl->cur], acc);
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

// One rig on the whole cooperative grid.
__global__ void __launch_bounds__(kCsThreads, 1) chain_solve_kernel(ChainSolveArgs a) { chain_solve(a, GridScope()); }

// A batch of rigs, one thread-block cluster each (launched with a cluster dimension; no cooperative launch): cluster k
// solves args[k], an LM or a DOGLEG iteration's solve and update by Str.  The arguments are read where they are, through
// the read-only data path: staged in shared memory they would leave too little of it for the two groups' workspaces of
// the largest rig that fits (G = 67).
template <Strategy Str>
__global__ void __launch_bounds__(kCsThreads, 1) chain_solve_batch_kernel(const ChainSolveArgs* __restrict__ args) {
  ClusterScope scope;
  chain_solve<ClusterScope, false, false, Str>(args[blockIdx.x / scope.nb()], scope);
}

// a rig as chain_cov_batch_kernel takes it: the solve's arguments (D2x set, scalars[kScNotPD] zeroed: set where a pivot
// fails), the constant-global mask [G] and the covariance it writes [G*G]
struct ChainCovArgs {
  ChainSolveArgs s;
  const double* mask;
  double* cov;
  // frame mode (chain_frame_cov_batch_kernel; D2x: the frame damping of vcgpu_get_frame_covariance): every level's Σ
  // blocks, the inverse of [globals | top nodes] [N*N] and the blocks written [nf][81], rows and columns from `live` on 0
  SigmaLevel sig[kMaxChainLevels];
  double* inv;
  double* out;
  int live;
  // cross mode (chain_frame_cross_cov_batch_kernel): frame mode's, with out Σ_fg [nf][9][G] and out_next Σ_f,f+1
  // [nf - 1][81]
  double* out_next;
  // diagonal and cross mode (chain_frame_diag_cross_cov_batch_kernel): cross mode's, and out_ff Σ_ff [nf][81]
  double* out_ff;
};
// A batch of inertial rigs, one thread-block cluster each: cluster k writes the covariance of args[k] (vcgpu_get_covariance_batch).
__global__ void __launch_bounds__(kCsThreads, 1) chain_cov_batch_kernel(const ChainCovArgs* __restrict__ args) {
  ClusterScope scope;
  const ChainCovArgs& a = args[blockIdx.x / scope.nb()];
  chain_solve<ClusterScope, true>(a.s, scope, a.mask, a.cov);
}

// ------------------------------------------------------------------ frame covariance (vcgpu_get_frame_covariance_batch)
// The walk takes two chunks per CTA at a time, one per group of kCsGroup threads, where their workspaces fit in what the
// solve asks for; else one per CTA, and the request grows to one chunk's workspace.
__host__ __device__ inline int chain_walk_chunks(int G) {
  return 2 * chain_selinv_smem_bytes<9>(G, kCsChunk) <= chain_solve_smem_doubles(G) * sizeof(double) ? 2 : 1;
}
__host__ __device__ inline size_t chain_frame_cov_smem_bytes(int G) {
  const size_t solve = chain_solve_smem_doubles(G) * sizeof(double), walk = chain_walk_chunks(G) * chain_selinv_smem_bytes<9>(G, kCsChunk);
  return solve > walk ? solve : walk;
}
// The walk of one inertial rig by its thread-block cluster: the elimination and the dense factorisation of chain_solve;
// CTA 0's warps solve the N unit right-hand sides (the whole inverse of [globals | top nodes], as dense_solve_kernel's
// inversion gives it) and leave the top nodes' blocks; then the levels top-down, a cluster barrier between two, their
// chunks spread over the CTAs (chain_selinv_chunk).  Then out(tid, bid, nb, nf) writes what the call returns from level
// 0's blocks in a.sig[0].
template <class Out>
__device__ __forceinline__ void chain_frame_cov_walk(const ChainCovArgs& a, ClusterScope scope, Out out) {
  extern __shared__ double smem[];
  constexpr int FD = 9;
  chain_solve<ClusterScope, true, true>(a.s, scope);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, grp = tid / kCsGroup, gtid = tid - grp * kCsGroup;
  const int bid = scope.bid(), nb = scope.nb();
  const int G = a.s.dp.G, nl = a.s.n_levels, nf = a.s.dp.n_frames;
  const ChainLevel top = a.s.lev[nl - 1];
  const int nt = top.n, N = G + nt * FD;
  if (bid == 0) {
    const int LD = dense_ld(N), RT = dense_rows(N);
    for (int j = warp; j < N; j += kCsThreads / 32) {
      double x[kCovQ] = {0.0, 0.0, 0.0, 0.0};
      warp_inverse_column<kCovQ, true>(smem, LD, smem + RT * LD, N, j, lane, x);
#pragma unroll
      for (int q = 0; q < kCovQ; ++q)
        if (32 * q + lane < N) a.inv[static_cast<int64_t>(32 * q + lane) * N + j] = x[q];
    }
    __syncthreads();
    const SigmaLevel& t = a.sig[nl - 1];
    for (int e = tid; e < nt * FD * FD; e += kCsThreads) {
      const int k = e / (FD * FD), r = (e / FD) % FD, q = e % FD, o = G + k * FD;
      t.kk[e] = a.inv[static_cast<int64_t>(o + r) * N + o + q];
      t.kn[e] = k + 1 < nt ? a.inv[static_cast<int64_t>(o + r) * N + o + FD + q] : 0.0;
    }
    for (int e = tid; e < nt * FD * G; e += kCsThreads) {
      const int k = e / (FD * G), r = (e / G) % FD, q = e % G;
      t.kg[e] = a.inv[static_cast<int64_t>(G + k * FD + r) * N + q];
    }
  }
  scope.sync();
  __shared__ int bad[kCsGroups];
  const bool two = chain_walk_chunks(G) == 2;
  const size_t ws = chain_selinv_smem_bytes<FD>(G, kCsChunk) / sizeof(double);
  for (int l = nl - 2; l >= 0; --l) {
    SelinvArgs sa;
    sa.G = G; sa.c = kCsChunk; sa.cur = a.s.lev[l]; sa.sig = a.sig[l]; sa.up = a.sig[l + 1];
    sa.Sgg = a.inv; sa.ldg = N; sa.scalars = a.s.scalars;
    NodeSrc src;
    src.L = l > 0 ? &a.s.lev[l] : nullptr;
    src.b = a.s.b[a.s.ctl->cur]; src.scale = a.s.scale; src.D2x = a.s.D2x; src.rinv = 0.0; src.G = G; src.nf = nf;
    src.sepdiag = nullptr; src.rank = 0; src.ghost = 0;
    auto node_A = [&](int64_t p, int e) { return src_A<FD>(src, p, e); };
    auto node_U = [&](int64_t p, int e) { return src_U<FD>(src, p, e); };
    const int n_chunks = a.s.lev[l + 1].n;
    if (two) {
      auto sync = [grp] { group_sync(grp); };
      for (int j = bid * kCsGroups + grp; j < n_chunks; j += nb * kCsGroups) {
        chain_selinv_chunk<FD, kCsGroup>(sa, j, smem + grp * ws, gtid, &bad[grp], sync, node_A, node_U);
        sync();
      }
    } else {
      auto sync = [] { __syncthreads(); };
      for (int j = bid; j < n_chunks; j += nb) {
        chain_selinv_chunk<FD, kCsThreads>(sa, j, smem, tid, &bad[0], sync, node_A, node_U);
        sync();
      }
    }
    scope.sync();
  }
  out(tid, bid, nb, nf);
}
// A batch of inertial rigs, one thread-block cluster each: cluster k writes the frame covariance of args[k], the walk's
// level 0 Σ_kk unscaled.
__global__ void __launch_bounds__(kCsThreads, 1) chain_frame_cov_batch_kernel(const ChainCovArgs* __restrict__ args) {
  constexpr int FD = 9;
  ClusterScope scope;
  const ChainCovArgs& a = args[blockIdx.x / scope.nb()];
  chain_frame_cov_walk(a, scope, [&](int tid, int bid, int nb, int nf) {
    const double* kk = a.sig[0].kk;
    for (int64_t e = static_cast<int64_t>(bid) * kCsThreads + tid; e < static_cast<int64_t>(nf) * FD * FD; e += static_cast<int64_t>(nb) * kCsThreads)
      a.out[e] = frame_cov_out_entry<FD>(e, a.live, kk, a.s.scale);
  });
}
// ... the frame blocks off the diagonal of args[k] (vcgpu_get_frame_cross_covariance_batch): level 0's Σ_kg and
// Σ_k,k+1 unscaled
__global__ void __launch_bounds__(kCsThreads, 1) chain_frame_cross_cov_batch_kernel(const ChainCovArgs* __restrict__ args) {
  constexpr int FD = 9;
  ClusterScope scope;
  const ChainCovArgs& a = args[blockIdx.x / scope.nb()];
  chain_frame_cov_walk(a, scope, [&](int tid, int bid, int nb, int nf) {
    const int G = a.s.dp.G;
    for (int64_t e = static_cast<int64_t>(bid) * kCsThreads + tid; e < frame_cross_cov_entries<FD>(nf, G); e += static_cast<int64_t>(nb) * kCsThreads)
      frame_cross_cov_out_entry<FD>(e, nf, G, a.live, a.sig[0], a.s.scale, a.mask, a.out, a.out_next);
  });
}
// ... both: level 0's Σ_kk, Σ_kg and Σ_k,k+1 unscaled, from one walk (vcgpu_get_observation_influence_batch)
__global__ void __launch_bounds__(kCsThreads, 1) chain_frame_diag_cross_cov_batch_kernel(const ChainCovArgs* __restrict__ args) {
  constexpr int FD = 9;
  ClusterScope scope;
  const ChainCovArgs& a = args[blockIdx.x / scope.nb()];
  chain_frame_cov_walk(a, scope, [&](int tid, int bid, int nb, int nf) {
    const int G = a.s.dp.G;
    const int64_t nd = static_cast<int64_t>(nf) * FD * FD, nc = frame_cross_cov_entries<FD>(nf, G);
    for (int64_t e = static_cast<int64_t>(bid) * kCsThreads + tid; e < nd + nc; e += static_cast<int64_t>(nb) * kCsThreads) {
      if (e < nd) a.out_ff[e] = frame_cov_out_entry<FD>(e, a.live, a.sig[0].kk, a.s.scale);
      else frame_cross_cov_out_entry<FD>(e - nd, nf, G, a.live, a.sig[0], a.s.scale, a.mask, a.out, a.out_next);
    }
  });
}

}  // namespace vc
