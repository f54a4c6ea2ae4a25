// Persistent trust-region kernel for the vision-only problem (one GPU, or frame shards on several).
//
// One cooperative launch runs up to n_iters trust-region iterations, Levenberg-Marquardt or (one GPU) DOGLEG: the kernel
// is instantiated per strategy (Strategy::kLM, kDogleg).  The loop itself (mega_solve) is written against a scope — the
// CTAs that share the rig and their barrier: the cooperative grid here (lm_mega_kernel), or one thread-block cluster per
// rig in lm_mega_batch_kernel, which solves many rigs in one launch ("grid" below: the scope).  One CTA per SM, every
// frame owned by the same WARP of the same CTA for the whole solve (frame f -> CTA f mod grid, warp
// (f / grid) mod warps).  An iteration is a chain of per-frame warp phases and small every-CTA phases,
// separated by grid barriers instead of launches:
//
//   S  per frame (warp):  L = chol(B_f + D_f),  X_f = (B_f + D_f)^-1 [E_f | g_f],  CTA partial of E^T X
//      (schur_accumulate)
//   -- grid barrier; every CTA leaves here, together, if CTA 0 published "stop" (or a peer timed out)
//   R1 entry e of the Schur sum is added up over the CTAs by one warp of CTA (e mod grid) and published:
//      one GPU: plain totals + grid barrier; shards: tagged words into every rank's buffer, readers poll
//   G  every CTA, redundantly: reduced system C + D - sum E^T X (reduced_system_entry), Cholesky, globals' step
//   U  per frame (warp):  back-substitution (frame_backsub), x (+) step, step statistics; trial camera states
//      DOGLEG: U1 per frame (warp): back-substitution x_f, CTA partials of the step scalars; one more grid barrier;
//      every CTA sums them, takes the dogleg point (dogleg_point, vc_dogleg.cuh) and the model change; U2 as U with
//      the dogleg step in place of x
//   B  per frame (warp): fused evaluate + Gram build at the trial point (build_frame_warp, vc_fused.cuh), 32
//      corners at a time through the warp's own shared-memory slab and FP64 DMMA (no block barrier anywhere in
//      the phase); the camera blocks are accumulated per warp, packed per camera
//   -- grid barrier
//   R2 packed camera blocks / scalars added up and published, as R1
//   D  every CTA, redundantly: expands the packed blocks, takes the accept-reject decision of Ceres'
//      TrustRegionMinimizer (decide_step) on its own copy of Ctl
//
// Every CTA (of every rank) reads bit-identical totals, so all take the same decision and the loop needs
// no broadcast; all sums run in a fixed order (deterministic).  The Schur accumulation, the reduced system's entries and the
// back-substitution are vc_kernels.cuh's routines, shared with the multi-launch kernels.  Replaces the body of ceres::Solve
// (vicalibrator.h:956) for the staged vision solves; the inertial path has its own persistent kernels
// (vc_imu_mega.cuh, vc_imu_eval_mega.cuh), and frame-sharded DOGLEG runs the multi-launch engine (vc_engine.inl).
//
// DOGLEG (vc_dogleg.cuh's header) on the same Jacobi-scaled system H = S J^T J S, g = S J^T r: S and G solve
// (H + mu D^2) x = -g (the damping mu clamp(diag H) in place of LM's clamp(diag H) / radius).  Every product with H the
// step needs is local to a frame once the CTA holds the globals' parts (replicated), so U1 needs no mat-vec pass: per
// frame the partials |g~_f|^2, u_f.(Hu)_f-share, |gn_f|^2, g~_f.gn_f, u.Hx and x.Hx frame shares (u = g~ / D, gn = D x),
// the globals' shares added by every CTA alike.  Then step~ = cg g~ + cn gn, step = step~ / D and the model change
// -step.g - step.H.step / 2 = -(cg |g~|^2 + cn g~.gn) - (cg^2 u.Hu + 2 cg cn u.Hx + cn^2 x.Hx) / 2.
#pragma once
#include <cooperative_groups.h>

#include "vc_frame_cov.cuh"
#include "vc_dogleg.cuh"
#include "vc_fused.cuh"
#include "vc_kernels.cuh"

namespace vc {
namespace cg = cooperative_groups;

constexpr int kMegaMaxWarps = 16;
constexpr int kMegaMaxThreads = 32 * kMegaMaxWarps;
constexpr int kGtabMax = 256;
constexpr int kMegaPartExtra = 8;  // scalars appended to each CTA's partial slot (kScCost .. kScNotPD)
// Totals buffer: every rank owns one (32 MiB, the vision kernel uses the first 4); in a frame-sharded run (one process per GPU) all ranks of the
// node map all of them (CUDA IPC).  A total is published as two 64-bit words {low half | tag}, {high half | tag}
// (tag = exchange number): an 8-byte store is single-copy atomic, so a reader that sees both tags has the value —
// no fence, no flag, no barrier between publishing and reading.  Layout in 64-bit words: Schur totals
// [2 parities][ranks][NS+8][2] at 0, packed camera blocks [2][ranks][NP+8][2] at kXchgCOff, control words at
// kXchgCtlOff: exchange counters (S, C), exit word (bit 0: CTA 0 decided to stop, bit 1: a reader timed out).
constexpr int kMaxRanks = 8;
constexpr size_t kXchgBytes = 32u << 20;  // the inertial kernels' regions follow the vision kernel's (vc_xchg.cuh)
constexpr int kXchgCOff = 409600;
constexpr int kXchgCtlOff = 442368;
// sharded runs: the totals summed over the ranks, as plain doubles, for this rank's CTAs (one reader per entry polls
// the tagged words and writes here; a grid barrier later everybody reads the plain copy)
constexpr int kXchgPlainS = kXchgCtlOff + 64;
constexpr int kXchgPlainC = kXchgPlainS + 32768;
constexpr int kMegaCommFailed = 1000;  // Ctl::done value when a peer never showed up
enum { kProfS = 0, kProfG, kProfU, kProfB, kProfD, kProfSync, kProfCount };

struct MegaArgs {
  DevProblem dp;
  Ctl* ctl;
  double* state[2];
  Blocks blk[2];
  const int32_t *grp_start, *grp_count, *group_of;
  const double *pw, *pc;
  const double* mask;
  const uint8_t* frame_used;  // [nf] 0: no active observation sees the frame (left as it is)
  const double* scale;   // Jacobi scale [nf*6 + G]
  double* X;             // [nf][6][G+1]
  double* partS;         // [grid][NS + 8]   Schur partial (lower triangle) | flags
  double* partC;         // [grid][n_cams*kCgStride + 8]   packed camera blocks | scalars
  double* delta;         // scaled step [nf*6 + G]
  double* scalars;       // kSc* of the last evaluated point (for the host)
  int n_iters;
  int n_warps;
  int rank, nranks;                      // frame shards (nranks = 1: a single GPU)
  unsigned long long* xbuf[kMaxRanks];   // totals buffer of every rank (peer pointers; [rank] is local)
  unsigned long long* prof;  // [kProfCount] ns per phase (CTA 0), or null
};

// DOGLEG's step scalars: U1's per-CTA partials (in the Schur partial slot's unused entries partS[NS + 0 .. 5], summed by
// every CTA after U1's barrier) and the globals' shares of them
enum { kDlG2 = 0, kDlUHu, kDlGn2, kDlB, kDlUHx, kDlXHx, kDlParts };
// dynamic shared memory of lm_mega_kernel (strategy: 0 LM, 1 DOGLEG); DOGLEG adds u_g, D_g, g~_g and its scalars
__host__ __device__ inline size_t mega_smem_doubles(int G, int n_cams, int n_warps, int strategy) {
  const size_t NS = static_cast<size_t>(G) * G + G;
  return static_cast<size_t>(n_warps) * (kWarpDoubles + n_cams * kCgStride) + 3 * NS + G + kMaxCams * (kCamStateStride + 9) +
         kScCount + 8 * kMegaMaxWarps + n_cams * kCgStride + kMegaPartExtra + sizeof(Ctl) / sizeof(double) + 8 +
         (strategy == 1 ? 3 * static_cast<size_t>(G) + 8 : 0);
}

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// Entry e's sum (is_max: maximum) over the nparts CTA partials part[b * stride + e], by the calling warp in a fixed
// order; every lane gets it.
__device__ __forceinline__ double partials_total(const double* part, int stride, int nparts, int e, bool is_max, int lane) {
  const double* p = part + e;
  double s0 = 0.0, s1 = 0.0;
  int b = lane;
  if (is_max) {
    for (; b < nparts; b += 32) s0 = fmax(s0, __ldcg(p + static_cast<int64_t>(b) * stride));
  } else {
    for (; b + 32 < nparts; b += 64) {
      s0 += __ldcg(p + static_cast<int64_t>(b) * stride);
      s1 += __ldcg(p + static_cast<int64_t>(b + 32) * stride);
    }
    if (b < nparts) s0 += __ldcg(p + static_cast<int64_t>(b) * stride);
    s0 += s1;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double t = __shfl_xor_sync(0xffffffffu, s0, o);
    s0 = is_max ? fmax(s0, t) : s0 + t;
  }
  return s0;
}

// Single GPU: entry e is added up over the CTAs by one warp of CTA (e mod grid) into tot[e]; a grid barrier
// later every CTA reads tot[] (cheaper than polling tagged words when nobody is remote: no tag checks, no polling).
// (bid of nb: the CTAs sharing the work — the whole grid unless the caller says otherwise)
__device__ inline void mega_reduce_stage1(const double* part, int stride, int nparts, int n, double* tot, int max_a, int max_b,
                                          int bid = blockIdx.x, int nb = gridDim.x) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int e = bid + warp * nb; e < n; e += nwarps * nb) {
    const double s = partials_total(part, stride, nparts, e, e == max_a || e == max_b, lane);
    if (lane == 0) tot[e] = s;
  }
}

// ---- the two reductions of an iteration: CTA partials -> totals (over the CTAs and, sharded, over the GPUs) ----
// Publish: entry e is added up over this GPU's CTAs by one warp of CTA (e mod grid) — fixed order — and stored,
// tagged, into slot [parity][my rank][e] of EVERY rank's totals buffer (lane r -> rank r; NVLink peer stores).
__device__ inline void mega_publish(const double* part, int stride, int nparts, int n, const MegaArgs& a, int off, int parity,
                                    unsigned tag, int max_a, int max_b) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int e = blockIdx.x + warp * gridDim.x; e < n; e += nwarps * gridDim.x) {
    const double s0 = partials_total(part, stride, nparts, e, e == max_a || e == max_b, lane);
    if (lane < a.nranks) {
      const unsigned long long bits = static_cast<unsigned long long>(__double_as_longlong(s0));
      const unsigned long long hi_tag = static_cast<unsigned long long>(tag) << 32;
      unsigned long long* w = a.xbuf[lane] + off + 2 * (static_cast<size_t>(parity * a.nranks + a.rank) * stride + e);
      asm volatile("st.volatile.global.v2.u64 [%0], {%1, %2};" ::"l"(w), "l"((bits & 0xffffffffull) | hi_tag),
                   "l"((bits >> 32) | hi_tag)
                   : "memory");
    }
  }
}
// Read: the total of entry e over the ranks, in rank order; spins until every rank's words carry `tag`.
// A reader that waits longer than 2 s sets the abort bit of the exit word and gives up (the value is then junk;
// every CTA leaves the loop together at the next grid barrier).
__device__ inline double mega_total(const MegaArgs& a, int off, int stride, int parity, unsigned tag, int e, bool is_max) {
  unsigned long long* ctlw = a.xbuf[a.rank] + kXchgCtlOff;
  const unsigned long long* w = a.xbuf[a.rank] + off + 2 * (static_cast<size_t>(parity) * a.nranks * stride + e);
  double s = 0.0;
  for (int r = 0; r < a.nranks; ++r, w += 2 * static_cast<size_t>(stride)) {
    unsigned long long w0, w1;
    unsigned polls = 0;
    unsigned long long t0 = 0;
    for (;;) {
      asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(w) : "memory");
      if (static_cast<unsigned>(w0 >> 32) == tag && static_cast<unsigned>(w1 >> 32) == tag) break;
      __nanosleep(polls < 8 ? 100 : 400);  // thousands of threads poll: keep the L2 free for the publishers
      if ((++polls & 1023u) == 0) {
        const unsigned long long now = global_ns();
        if (t0 == 0) t0 = now;
        if (now - t0 > 2000000000ull || (*reinterpret_cast<volatile unsigned long long*>(ctlw + 2) & 2ull)) {
          atomicOr(ctlw + 2, 2ull);
          return 0.0;
        }
      }
    }
    const double v = __longlong_as_double(static_cast<long long>((w0 & 0xffffffffull) | (w1 << 32)));
    s = is_max ? fmax(s, v) : s + v;
  }
  return s;
}

// Reduced-system solve, one warp.  S: lower triangle [G][G] row-major followed by the right-hand side [G];
// the solution overwrites the right-hand side.  The right-hand side is carried through the factorisation as an
// extra row (so L y = rhs comes for free) and the pivots are kept as reciprocals.  Rows are spread over the
// lanes, column updates batched by four.  (Register-resident variants — lane r owning row r, columns broadcast
// with shuffles — were slower in this phase: the row array ends up in local memory.)
__device__ inline void mega_chol_solve_smem(double* S, int G, int lane, double* invd, int* bad) {
  double* rhs = S + G * G;
  for (int j = 0; j < G; ++j) {
    double d = S[j * G + j];
    if (!(d > 0.0)) { if (lane == 0) *bad = 1; d = 1.0; }
    const double inv = rsqrt(d);
    __syncwarp();
    if (lane == 0) { S[j * G + j] = d * inv; invd[j] = inv; }
    for (int r = j + 1 + lane; r <= G; r += 32) {
      double* row = r < G ? S + r * G : rhs;
      row[j] *= inv;
    }
    __syncwarp();
    for (int r = j + 1 + lane; r <= G; r += 32) {
      double* row = r < G ? S + r * G : rhs;
      const double lrj = row[j];
      const int qmax = min(r, G - 1);
      int q = j + 1;
      for (; q + 3 <= qmax; q += 4) {
        const double l0 = S[q * G + j], l1 = S[(q + 1) * G + j], l2 = S[(q + 2) * G + j], l3 = S[(q + 3) * G + j];
        const double r0 = row[q], r1 = row[q + 1], r2 = row[q + 2], r3 = row[q + 3];
        row[q] = r0 - lrj * l0; row[q + 1] = r1 - lrj * l1; row[q + 2] = r2 - lrj * l2; row[q + 3] = r3 - lrj * l3;
      }
      for (; q <= qmax; ++q) row[q] -= lrj * S[q * G + j];
    }
    __syncwarp();
  }
  for (int i = G - 1; i >= 0; --i) {  // L^T x = y
    const double xi = rhs[i] * invd[i];
    __syncwarp();
    if (lane == 0) rhs[i] = xi;
    for (int q = lane; q < i; q += 32) rhs[q] -= S[i * G + q] * xi;
    __syncwarp();
  }
}

// The CTAs that share one rig's solve.  A scope supplies what the solve loop needs from "the grid": this CTA's index
// among them, their count, and a barrier over them that orders their global-memory writes.
//   GridScope: the whole cooperative grid (lm_mega_kernel: one rig per launch; frame shards allowed).
//   ClusterScope: one thread-block cluster (lm_mega_batch_kernel: one rig per cluster, many clusters per launch, none
//   of which ever waits for another).  Never sharded, so mega_publish / mega_total are not instantiated for it.
struct GridScope {
  static constexpr bool kSharded = true;
  cg::grid_group g = cg::this_grid();
  __device__ __forceinline__ int bid() const { return blockIdx.x; }
  __device__ __forceinline__ int nb() const { return gridDim.x; }
  __device__ __forceinline__ void sync() { g.sync(); }
};
struct ClusterScope {
  static constexpr bool kSharded = false;
  cg::cluster_group c = cg::this_cluster();
  __device__ __forceinline__ int bid() const { return static_cast<int>(c.block_rank()); }
  __device__ __forceinline__ int nb() const { return static_cast<int>(c.num_blocks()); }
  __device__ __forceinline__ void sync() { c.sync(); }  // barrier.cluster.arrive.release + wait.acquire
};

// The solve loop: up to a.n_iters trust-region iterations of strategy Str on the rig `a`, by the CTAs of `scope`.
template <Strategy Str, class Scope>
__device__ __forceinline__ void mega_solve(const MegaArgs& a, Scope scope) {
  constexpr bool kDl = Str == Strategy::kDogleg;
  extern __shared__ double smem[];
  constexpr int FD = 6;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nthreads = blockDim.x, nwarps = nthreads >> 5;
  const int bid = scope.bid(), nb = scope.nb();
  const int n_cams = a.dp.n_cams;
  const int G = a.dp.G, M = G + 1, NS = G * G + G, PS = NS + kMegaPartExtra, nf = a.dp.n_frames;
  const int NP = n_cams * kCgStride, PC = NP + kMegaPartExtra;  // packed camera blocks
  const int64_t nfp = static_cast<int64_t>(nf) * FD;
  const int nk = bid < nf ? (nf - bid + nb - 1) / nb : 0;  // frames of this CTA: f = bid + k * nb, warp k mod nwarps

  double* wmem = smem;                                               // [nwarps][kWarpDoubles]; also phase scratch
  double* Cw = wmem + static_cast<size_t>(nwarps) * kWarpDoubles;    // [nwarps][NP] packed camera blocks per warp
  double* Cacc = Cw + static_cast<size_t>(nwarps) * NP;              // [2][NS]  C | gc of the two points
  double* Swork = Cacc + 2 * NS;                                     // [NS] Schur accumulator / reduced system
  double* dg = Swork + NS;                                           // [G] globals' step (scaled)
  double* smCam = dg + G;                                            // [kMaxCams][17] trial camera states
  double* smRc = smCam + kMaxCams * kCamStateStride;                 // [kMaxCams][9]
  double* sc = smRc + kMaxCams * 9;                                  // [kScCount]
  double* wred = sc + kScCount;                                      // [kMegaMaxWarps][8] per-warp scalars
  double* totc = wred + 8 * kMegaMaxWarps;                           // [NP + 8] packed camera blocks / scalars, grid (and rank) totals
  Ctl* ctl = reinterpret_cast<Ctl*>(totc + NP + kMegaPartExtra);
  double* dl_u = reinterpret_cast<double*>(ctl + 1);                 // DOGLEG: [G] u_g = g~_g / D_g
  double* dl_D = dl_u + G;                                           // [G] D_g
  double* dl_gt = dl_D + G;                                          // [G] g~_g
  double* dl_s = dl_gt + G;                                          // [8] globals' shares (kDl*), then cg, cn
  __shared__ int bad;
  __shared__ int2 gtab[kGtabMax];          // (start, count) of the observations of this CTA's (frame slot, camera) pairs
  __shared__ unsigned char tri_lut[128];   // packed lower-triangle index -> (row << 4 | col)
  const double* scg = a.scale + nfp;
  unsigned long long* ctlw = a.xbuf[a.rank] + kXchgCtlOff;  // [0] S exchanges, [1] C exchanges, [2] exit word
  __shared__ unsigned long long exit_s;

  if (tid == 0) *ctl = *a.ctl;
  const bool use_gtab = nk * n_cams <= kGtabMax;
  if (use_gtab)  // frame ownership is static: look the groups up once per launch
    for (int e = tid; e < nk * n_cams; e += nthreads) {
      const int k = e / n_cams, c = e - k * n_cams;
      const int g = a.group_of[c * nf + bid + k * nb];
      gtab[e] = g < 0 ? make_int2(0, 0) : make_int2(a.grp_start[g], a.grp_count[g]);
    }
  fill_tri_lut(tri_lut, tid, nthreads);
  __syncthreads();
  if (ctl->done) return;
  if (bid == 0 && tid == 0 && !(ctlw[2] & 2ull)) {  // the stop bit of the previous launch; the abort bit is sticky
    ctlw[2] = 0;
    __threadfence();
  }
  {
    const Blocks& b0 = a.blk[ctl->cur];
    double* C0 = Cacc + ctl->cur * NS;
    for (int e = tid; e < NS; e += nthreads) C0[e] = e < G * G ? b0.C[e] : b0.gc[e - G * G];
  }
  // (start, count) of the observations of (frame slot k, camera c); count 0: the camera does not see the frame
  auto lookup = [&](int k, int c) -> int2 {
    if (use_gtab) return gtab[k * n_cams + c];
    const int g = a.group_of[c * nf + bid + k * nb];
    return g < 0 ? make_int2(0, 0) : make_int2(a.grp_start[g], a.grp_count[g]);
  };
  const bool sharded = Scope::kSharded && a.nranks > 1;
  unsigned epS = static_cast<unsigned>(ctlw[0]), epC = static_cast<unsigned>(ctlw[1]);  // same on every CTA of every rank
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

  for (int it = 0; it < a.n_iters; ++it) {
    __syncthreads();
    // A CTA never leaves the loop on its own: it idles through phase S and leaves with everybody else right
    // after the next grid barrier, on the word CTA 0 published (so a junk total can never split the grid).
    const bool skip = ctl->done != 0;
    const int cur = ctl->cur;
    const Blocks& bc = a.blk[cur];
    const Blocks& bt = a.blk[1 - cur];
    const double* x_cur = a.state[cur];
    double* x_new = a.state[1 - cur];
    // the damping's multiplier: LM clamp(diag) / radius; DOGLEG mu clamp(diag), the Gauss-Newton solve's regularisation
    const double dmul = kDl ? ctl->dl_mu : 1.0 / ctl->radius;
    const double* Ccur = Cacc + cur * NS;
    double notpd = 0.0;

    // ------------------------------------------------------------ S: per-frame solves + Schur partial
    if (!skip) {
      double* Sacc = Swork;
      for (int k = tid; k < NS; k += nthreads) Sacc[k] = 0.0;
      for (int base = 0; base < nk; base += nwarps) {
        const int k = base + warp;
        __syncthreads();
        if (k < nk) {
          const int f = bid + k * nb;
          double* Esw = wmem + static_cast<size_t>(warp) * kWarpDoubles;  // [FD][M] scaled [E | g], then X [FD][M]
          double* Xw = Esw + FD * M;
          const double* sf = a.scale + static_cast<int64_t>(f) * FD;
          const double* Bf = bc.B + static_cast<int64_t>(f) * FD * FD;
          const double* Ef = bc.E + static_cast<int64_t>(f) * FD * G;
          double s[FD], L[FD][FD], iL[FD];
#pragma unroll
          for (int i = 0; i < FD; ++i) s[i] = sf[i];
#pragma unroll
          for (int i = 0; i < FD; ++i)
#pragma unroll
            for (int j = 0; j <= i; ++j) {
              const double bij = Bf[i * FD + j];
              double v = bij * s[i] * s[j];
              if (i == j) v = frame_damp<FD>(v, f, i, bij, s[i], dmul, nullptr, nullptr, 0, false);
              L[i][j] = v;
            }
          bool ok = true;
#pragma unroll
          for (int j = 0; j < FD; ++j) {
            double d = L[j][j];
#pragma unroll
            for (int q = 0; q < j; ++q) d -= L[j][q] * L[j][q];
            if (!(d > 0.0)) { ok = false; d = 1.0; }
            const double inv = rsqrt(d);
            L[j][j] = d * inv;
            iL[j] = inv;
#pragma unroll
            for (int i = j + 1; i < FD; ++i) {
              double t = L[i][j];
#pragma unroll
              for (int q = 0; q < j; ++q) t -= L[i][q] * L[j][q];
              L[i][j] = t * inv;
            }
          }
          if (!ok) notpd = 1.0;
          double* Xf = a.X + static_cast<int64_t>(f) * FD * M;
          for (int c = lane; c < M; c += 32) {
            double x[FD];
            const double scc = c < G ? scg[c] : 1.0;
#pragma unroll
            for (int i = 0; i < FD; ++i) {
              const double r = (c < G ? Ef[i * G + c] : bc.gf[static_cast<int64_t>(f) * FD + i]) * s[i] * scc;
              Esw[i * M + c] = r;
              x[i] = r;
            }
#pragma unroll
            for (int i = 0; i < FD; ++i) {
              double t = x[i];
#pragma unroll
              for (int q = 0; q < i; ++q) t -= L[i][q] * x[q];
              x[i] = t * iL[i];
            }
#pragma unroll
            for (int i = FD - 1; i >= 0; --i) {
              double t = x[i];
#pragma unroll
              for (int q = i + 1; q < FD; ++q) t -= L[q][i] * x[q];
              x[i] = t * iL[i];
            }
#pragma unroll
            for (int i = 0; i < FD; ++i) {
              Xw[i * M + c] = x[i];
              Xf[i * M + c] = x[i];
            }
          }
        }
        __syncthreads();
        schur_accumulate<FD>(Sacc, wmem, kWarpDoubles, min(nwarps, nk - base), G, tid, nthreads);
      }
      __syncthreads();
      double* out = a.partS + static_cast<int64_t>(bid) * PS;
      for (int k = tid; k < NS; k += nthreads) out[k] = Sacc[k];
      const unsigned any = __ballot_sync(0xffffffffu, notpd > 0.0);
      if (lane == 0) wred[8 * warp] = any ? 1.0 : 0.0;
      __syncthreads();
      if (tid == 0) {
        double v = 0.0;
        for (int w = 0; w < nwarps; ++w) v = fmax(v, wred[8 * w]);
        out[NS + kScNotPD] = v;
      }
    }
    mark(kProfS);
    scope.sync();
    if (tid == 0) exit_s = *reinterpret_cast<volatile unsigned long long*>(ctlw + 2);
    __syncthreads();
    if (exit_s) break;
    mark(kProfSync);

    // ------------------------------------------------------------ G: reduced system, every CTA the same
    {
      double* S = Swork;  // [G*G] lower triangle, then rhs [G]
      ++epS;
      const int parS = static_cast<int>(epS & 1);
      // plain totals: in the exchange buffer itself on one GPU, next to the tagged words in a sharded run
      double* totS = reinterpret_cast<double*>(a.xbuf[a.rank] + (sharded ? kXchgPlainS : 0));
      if (sharded) {
        // every rank's CTA sums go to every rank (tagged words over NVLink); ONE thread of this grid per entry waits for
        // them and adds them up in rank order (every rank computes the same bits)
        if constexpr (Scope::kSharded) {
          mega_publish(a.partS, PS, nb, PS, a, 0, parS, epS, NS + kScNotPD, -1);
          for (int e = bid * nthreads + tid; e < PS; e += nb * nthreads) totS[e] = mega_total(a, 0, PS, parS, epS, e, e == NS + kScNotPD);
        }
      } else {
        mega_reduce_stage1(a.partS, PS, nb, PS, totS, NS + kScNotPD, -1, bid, nb);
      }
      mark(kProfG);
      scope.sync();
      mark(kProfSync);
      for (int e = tid; e < NS; e += nthreads) {
        if (e < G * G && e % G > e / G) continue;  // lower triangle only
        S[e] = reduced_system_entry(e, G, Ccur[e], __ldcg(totS + e), scg, dmul, nullptr, 0);
      }
      if (tid == 0) {
        sc[kScNotPD] = __ldcg(totS + NS + kScNotPD);
        bad = 0;
      }
      __syncthreads();
      if (warp == 0) {
        mega_chol_solve_smem(S, G, lane, dg, &bad);
      }
      __syncthreads();
      for (int i = tid; i < G; i += nthreads) {
        const double v = bad ? 0.0 : S[G * G + i];
        dg[i] = v;
        if (bid == 0) a.delta[nfp + i] = v;
      }
      if (tid == 0 && bad) sc[kScNotPD] = 1.0;
      __syncthreads();
    }
    mark(kProfG);

    // ------------------------------------------------------------ U1 (DOGLEG): Gauss-Newton step, step scalars
    if constexpr (kDl) {
      for (int i = tid; i < G; i += nthreads) {
        double D, gt;
        dl_scaled(Ccur[i * G + i], Ccur[G * G + i], scg[i], &D, &gt);
        dl_D[i] = D;
        dl_gt[i] = gt;
        dl_u[i] = gt / D;
      }
      __syncthreads();
      double part[kDlParts] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};  // lane 0 of each warp: its frames' shares
      if (warp == nwarps - 1) {  // the globals' shares, the same bits in every CTA (x_g = dg)
        double q[kDlParts] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        for (int r = lane; r < G; r += 32) {
          double cu = 0.0, cx = 0.0;  // rows of (S C S) u_g, (S C S) x_g
          for (int c = 0; c < G; ++c) {
            const double h = Ccur[r * G + c] * scg[r] * scg[c];
            cu += h * dl_u[c];
            cx += h * dg[c];
          }
          const double gn = dg[r] * dl_D[r];
          q[kDlG2] += dl_gt[r] * dl_gt[r];
          q[kDlUHu] += dl_u[r] * cu;
          q[kDlGn2] += gn * gn;
          q[kDlB] += dl_gt[r] * gn;
          q[kDlUHx] += dl_u[r] * cx;
          q[kDlXHx] += dg[r] * cx;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
          for (int j = 0; j < kDlParts; ++j) q[j] += __shfl_xor_sync(0xffffffffu, q[j], o);
        if (lane == 0)
          for (int j = 0; j < kDlParts; ++j) dl_s[j] = q[j];
      }
      for (int k = warp; k < nk; k += nwarps) {
        const int f = bid + k * nb;
        const double* Xf = a.X + static_cast<int64_t>(f) * FD * M;
        const double* Ef = bc.E + static_cast<int64_t>(f) * FD * G;
        double x[FD], ex[FD], eu[FD];  // x_f, then rows of E S x_g and E S u_g (the frame's row scale not yet applied)
#pragma unroll
        for (int r = 0; r < FD; ++r) {
          double s = 0.0, t = 0.0, v = 0.0;
          for (int c = lane; c < G; c += 32) {
            s += Xf[r * M + c] * dg[c];
            const double e = Ef[r * G + c] * scg[c];
            t += e * dg[c];
            v += e * dl_u[c];
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            s += __shfl_xor_sync(0xffffffffu, s, o);
            t += __shfl_xor_sync(0xffffffffu, t, o);
            v += __shfl_xor_sync(0xffffffffu, v, o);
          }
          x[r] = -Xf[r * M + G] - s;
          ex[r] = t;
          eu[r] = v;
        }
        if (lane == 0) {
          const double* sf = a.scale + static_cast<int64_t>(f) * FD;
          const double* Bf = bc.B + static_cast<int64_t>(f) * FD * FD;
          const double* gf = bc.gf + static_cast<int64_t>(f) * FD;
          double u[FD], wu[FD], wx[FD];
#pragma unroll
          for (int r = 0; r < FD; ++r) {
            double D, gt;
            dl_scaled(Bf[r * FD + r], gf[r], sf[r], &D, &gt);
            const double gn = x[r] * D;
            u[r] = gt / D;
            wu[r] = sf[r] * u[r];
            wx[r] = sf[r] * x[r];
            part[kDlG2] += gt * gt;
            part[kDlGn2] += gn * gn;
            part[kDlB] += gt * gn;
            a.delta[static_cast<int64_t>(f) * FD + r] = x[r];
          }
#pragma unroll
          for (int r = 0; r < FD; ++r) {
            double bu = 0.0, bx = 0.0;
#pragma unroll
            for (int j = 0; j < FD; ++j) {
              bu += Bf[r * FD + j] * wu[j];
              bx += Bf[r * FD + j] * wx[j];
            }
            const double hu = sf[r] * (bu + eu[r]), hx = sf[r] * (bx + ex[r]);  // rows of H u, H x of the frame
            const double gu = sf[r] * eu[r], gx = sf[r] * ex[r];                // rows of (S E S) u_g, (S E S) x_g
            part[kDlUHu] += u[r] * hu + u[r] * gu;  // u_f.(S B S) u_f + 2 u_f.(S E S) u_g
            part[kDlUHx] += u[r] * hx + x[r] * gu;  // u_f.(S B S) x_f + u_f.(S E S) x_g + x_f.(S E S) u_g
            part[kDlXHx] += x[r] * hx + x[r] * gx;  // x_f.(S B S) x_f + 2 x_f.(S E S) x_g
          }
        }
      }
      if (lane == 0)
        for (int j = 0; j < kDlParts; ++j) wred[8 * warp + j] = part[j];
      __syncthreads();
      if (tid == 0) {
        double* out = a.partS + static_cast<int64_t>(bid) * PS + NS;
        for (int j = 0; j < kDlParts; ++j) {
          double v = 0.0;
          for (int w = 0; w < nwarps; ++w) v += wred[8 * w + j];
          out[j] = v;
        }
      }
      mark(kProfU);
      scope.sync();
      mark(kProfSync);
      if (warp == 0) {  // every CTA adds up the CTA partials alike, then the dogleg point and the model change
        double t[kDlParts] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        for (int b = lane; b < nb; b += 32)
          for (int j = 0; j < kDlParts; ++j) t[j] += __ldcg(a.partS + static_cast<int64_t>(b) * PS + NS + j);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
          for (int j = 0; j < kDlParts; ++j) t[j] += __shfl_xor_sync(0xffffffffu, t[j], o);
        if (lane == 0) {
          for (int j = 0; j < kDlParts; ++j) t[j] += dl_s[j];
          ctl->dl_g2 = t[kDlG2];
          ctl->dl_alpha = t[kDlG2] / t[kDlUHu];
          ctl->dl_gn2 = t[kDlGn2];
          ctl->dl_b = t[kDlB];
          ctl->dl_ok = sc[kScNotPD] > 0.0 ? 0 : 1;
          double cg, cn;
          ctl->dl_step_norm = dogleg_point(ctl->radius, ctl->dl_alpha, ctl->dl_g2, ctl->dl_gn2, ctl->dl_b, &cg, &cn);
          if (!ctl->dl_ok) cg = cn = 0.0;
          // step.g = cg |g~|^2 + cn g~.gn;  step.H.step = cg^2 u.Hu + 2 cg cn u.Hx + cn^2 x.Hx
          ctl->dl_model_change = -(cg * t[kDlG2] + cn * t[kDlB]) -
                                 0.5 * (cg * cg * t[kDlUHu] + 2.0 * cg * cn * t[kDlUHx] + cn * cn * t[kDlXHx]);
          dl_s[6] = cg;
          dl_s[7] = cn;
        }
      }
      __syncthreads();
      for (int i = tid; i < G; i += nthreads) {  // the globals' step (cg g~ + cn gn) / D replaces x_g
        const double v = ctl->dl_ok ? (dl_s[6] * dl_gt[i] + dl_s[7] * (dg[i] * dl_D[i])) / dl_D[i] : 0.0;
        dg[i] = v;
        if (bid == 0) a.delta[nfp + i] = v;
      }
      __syncthreads();
    }

    // ------------------------------------------------------------ U: back-substitution, trial states
    // (DOGLEG: the dogleg step in place of the back-substitution)
    double ustat[4] = {0.0, 0.0, 0.0, 0.0};  // lane 0 of each warp: kScDotG .. kScXnorm2
    {
      if (warp == nwarps - 1) {  // trial camera states (every CTA needs them; the last warp is the one most likely
                                 // to own no frame); CTA 0 also stores the globals
        if (lane < n_cams) {
          const int c = lane;
          const double* x = x_cur + a.dp.off_cam + kCamStateStride * c;
          double* xo = smCam + kCamStateStride * c;
          double R[9];
          cam_plus(a.dp, c, x, dg, scg, xo);
          qmat(Q4{xo[0], xo[1], xo[2], xo[3]}, R);
#pragma unroll
          for (int q = 0; q < 9; ++q) smRc[9 * c + q] = R[q];
          if (bid == 0) {
            double* xg = x_new + a.dp.off_cam + kCamStateStride * c;
            for (int q = 0; q < kCamStateStride; ++q) xg[q] = xo[q];
          }
        }
        __syncwarp();
        if (bid == 0 && a.rank == 0 && lane == 0) {  // the globals' share of the step statistics, counted once
          for (int c = 0; c < n_cams; ++c) {
            const double* x = x_cur + a.dp.off_cam + kCamStateStride * c;
            cam_stats(a.dp, c, x, smCam + kCamStateStride * c, ustat + 2);
          }
          for (int q = 0; q < kImuStateSize; ++q) x_new[a.dp.off_imu + q] = x_cur[a.dp.off_imu + q];
          for (int q = 0; q < G; ++q) {
            const double d2 = global_damp(q, Ccur[q * G + q], scg[q], dmul, nullptr, 0);
            ustat[0] += dg[q] * Ccur[G * G + q] * scg[q];
            ustat[1] += dg[q] * dg[q] * d2;
          }
        }
      }
      for (int k = warp; k < nk; k += nwarps) {
        const int f = bid + k * nb;
        double d[FD];
        if constexpr (kDl) {  // (cg g~ + cn gn) / D from U1's x_f (in delta)
          const double* sf = a.scale + static_cast<int64_t>(f) * FD;
          const double* Bf = bc.B + static_cast<int64_t>(f) * FD * FD;
          const double* gf = bc.gf + static_cast<int64_t>(f) * FD;
#pragma unroll
          for (int r = 0; r < FD; ++r) {
            double D, gt;
            dl_scaled(Bf[r * FD + r], gf[r], sf[r], &D, &gt);
            d[r] = ctl->dl_ok ? (dl_s[6] * gt + dl_s[7] * (a.delta[static_cast<int64_t>(f) * FD + r] * D)) / D : 0.0;
          }
        } else {
          frame_backsub<FD>(a.X + static_cast<int64_t>(f) * FD * M, dg, G, lane, d);
        }
        if constexpr (kDl) __syncwarp();  // every lane has read x_f before lane 0 overwrites it
        if (lane == 0) {
#pragma unroll
          for (int r = 0; r < FD; ++r) a.delta[static_cast<int64_t>(f) * FD + r] = d[r];
          frame_plus<FD>(a.dp, bc, a.scale, dmul, nullptr, nullptr, f, d, a.frame_used[f] != 0, x_cur, x_new, ustat);
        }
      }
      for (int e = tid; e < nwarps * NP; e += nthreads) Cw[e] = 0.0;
      __syncthreads();  // trial camera states and the trial poses are visible to every warp
    }
    mark(kProfU);

    // ------------------------------------------------------------ B: fused evaluate + build at the trial point
    // No block barrier in this phase: each warp runs its frames on its own slab, at its own pace.
    double cost = 0.0, gf2 = 0.0, gfmax = 0.0;
    {
      double* slab = wmem + static_cast<size_t>(warp) * kWarpDoubles;  // [16][kSlabLd]; reused as the 16 x 16 Gram matrix
      const double* smg = slab + kSlabDoubles + 36;
      double* Cmine = Cw + static_cast<size_t>(warp) * NP;
      for (int k = warp; k < nk; k += nwarps) {
        const int f = bid + k * nb;
        // the camera blocks are added up per warp: the same lane owns an entry for every frame of this warp
        cost = build_frame_warp<FD, true>(a.dp, x_new + 7 * static_cast<int64_t>(f), smCam, smRc, a.mask, a.pw, a.pc,
                                          bt.E + static_cast<int64_t>(f) * FD * G, slab, tri_lut, lane, cost,
                                          [&](int c) { return lookup(k, c); }, [&](int c) { return Cmine + c * kCgStride; });
        __syncwarp();
        store_frame_block<FD>(slab + kSlabDoubles, smg, bt.B + static_cast<int64_t>(f) * FD * FD, bt.gf + static_cast<int64_t>(f) * FD,
                              lane, 32);
        if (lane < 6) {
          const double gv = smg[lane];
          gf2 += gv * gv;
          gfmax = fmax(gfmax, fabs(gv));
        }
      }
    }
    // CTA partials: scalars, then the warps' packed camera blocks in fixed order
    {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        cost += __shfl_xor_sync(0xffffffffu, cost, o);
        gf2 += __shfl_xor_sync(0xffffffffu, gf2, o);
        gfmax = fmax(gfmax, __shfl_xor_sync(0xffffffffu, gfmax, o));
      }
      if (lane == 0) {
        double* w = wred + 8 * warp;
        w[kScCost] = cost; w[kScGnorm2] = gf2; w[kScGmax] = gfmax;
#pragma unroll
        for (int q = 0; q < 4; ++q) w[kScDotG + q] = ustat[q];
      }
      __syncthreads();
      double* out = a.partC + static_cast<int64_t>(bid) * PC;
      for (int e = tid; e < NP; e += nthreads) {
        double v = 0.0;
        for (int w = 0; w < nwarps; ++w) v += Cw[static_cast<size_t>(w) * NP + e];
        out[e] = v;
      }
      if (tid == 0) {
        double t[kScNotPD] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        for (int w = 0; w < nwarps; ++w) {
          const double* p = wred + 8 * w;
#pragma unroll
          for (int q = 0; q < kScGmax; ++q) t[q] += p[q];
          t[kScGmax] = fmax(t[kScGmax], p[kScGmax]);
        }
        for (int q = 0; q < kScNotPD; ++q) out[NP + q] = t[q];
        out[NP + kScNotPD] = 0.0;
      }
    }
    mark(kProfB);
    scope.sync();
    mark(kProfSync);

    // ------------------------------------------------------------ D: global block of the trial point, decision
    {
      double* Ctrial = Cacc + (1 - cur) * NS;
      ++epC;
      const int parC = static_cast<int>(epC & 1);
      double* totC = reinterpret_cast<double*>(a.xbuf[a.rank] + (sharded ? kXchgPlainC : kXchgCOff));
      if (sharded) {
        if constexpr (Scope::kSharded) {
          mega_publish(a.partC, PC, nb, PC, a, kXchgCOff, parC, epC, NP + kScGmax, NP + kScNotPD);
          for (int e = bid * nthreads + tid; e < PC; e += nb * nthreads)
            totC[e] = mega_total(a, kXchgCOff, PC, parC, epC, e, e == NP + kScGmax || e == NP + kScNotPD);
        }
      } else {
        mega_reduce_stage1(a.partC, PC, nb, PC, totC, NP + kScGmax, NP + kScNotPD, bid, nb);
      }
      mark(kProfD);
      scope.sync();
      mark(kProfSync);
      for (int e = tid; e < PC; e += nthreads) totc[e] = __ldcg(totC + e);
      __syncthreads();
      for (int e = tid; e < NS; e += nthreads) {  // packed per-camera blocks -> dense C | gc
        const int r = e < G * G ? e / G : e - G * G;
        const int cc = e < G * G ? e - r * G : -1;
        double v = 0.0;
        for (int c = 0; c < n_cams; ++c) {
          const CamInfo& ci = a.dp.cams[c];
          const int p = r - ci.goff;
          if (p < 0 || p >= 6 + ci.K) continue;
          if (cc < 0) {
            v = totc[c * kCgStride + 105 + p];
          } else {
            const int q = cc - ci.goff;
            if (q >= 0 && q < 6 + ci.K) {
              const int hi = max(p, q), lo = min(p, q);
              v = totc[c * kCgStride + hi * (hi + 1) / 2 + lo];
            }
          }
        }
        Ctrial[e] = v;
      }
      __syncthreads();
      if (warp == 0) {
        double g2 = 0.0, gm = 0.0;
        for (int q = lane; q < G; q += 32) {
          const double gv = Ctrial[G * G + q];
          g2 += gv * gv;
          gm = fmax(gm, fabs(gv));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          g2 += __shfl_xor_sync(0xffffffffu, g2, o);
          gm = fmax(gm, __shfl_xor_sync(0xffffffffu, gm, o));
        }
        if (lane == 0) {
          double t[kScNotPD];
#pragma unroll
          for (int q = 0; q < kScNotPD; ++q) t[q] = totc[NP + q];
          t[kScGnorm2] += g2;
          t[kScGmax] = fmax(t[kScGmax], gm);
          finish_scalars<Str>(ctl, sc, bid == 0 ? bt.cost : nullptr, t, true, 1);
          if (bid == 0) {
            if (ctl->done) atomicOr(ctlw + 2, 1ull);
            *a.ctl = *ctl;
            for (int q = 0; q <= kScNotPD; ++q) a.scalars[q] = sc[q];
          }
        }
      }
      __syncthreads();
    }
    mark(kProfD);
  }
  // hand the accepted point's global block back to the multi-launch engine / inspection hooks
  __syncthreads();
  if (bid == 0 && tid == 0) {
    ctlw[0] = epS;
    ctlw[1] = epC;
    if (*reinterpret_cast<volatile unsigned long long*>(ctlw + 2) & 2ull) a.ctl->done = kMegaCommFailed;
  }
  if (bid == 0) {
    const Blocks& bf = a.blk[ctl->cur];
    const double* Cf = Cacc + ctl->cur * NS;
    for (int e = tid; e < NS; e += nthreads) {
      if (e < G * G) bf.C[e] = Cf[e];
      else bf.gc[e - G * G] = Cf[e];
    }
  }
}

// One rig on the whole cooperative grid.
template <Strategy Str>
__global__ void __launch_bounds__(kMegaMaxThreads, 1) lm_mega_kernel(MegaArgs a) {
  mega_solve<Str>(a, GridScope());
}

// A batch of rigs, one thread-block cluster each (launched with a cluster dimension; no cooperative launch): cluster k
// solves args[k].  The clusters share nothing and leave on their own rig's exit word.  The rig's arguments are staged in
// shared memory once per CTA (the loop reads them all the time).
template <Strategy Str>
__global__ void __launch_bounds__(kMegaMaxThreads, 1) lm_mega_batch_kernel(const MegaArgs* args) {
  static_assert(sizeof(MegaArgs) % sizeof(unsigned long long) == 0, "MegaArgs is copied in 8-byte words");
  __shared__ __align__(16) unsigned long long words[sizeof(MegaArgs) / sizeof(unsigned long long)];
  ClusterScope scope;
  const unsigned long long* src = reinterpret_cast<const unsigned long long*>(args + blockIdx.x / scope.nb());
  for (int k = threadIdx.x; k < static_cast<int>(sizeof(MegaArgs) / sizeof(unsigned long long)); k += blockDim.x) words[k] = src[k];
  __syncthreads();
  mega_solve<Str>(*reinterpret_cast<const MegaArgs*>(words), scope);
}

// ------------------------------------------------------------------ covariance of the globals (vcgpu_get_covariance_batch)
// The [globals, globals] block of the inverse of the Jacobi-scaled, undamped arrow system S J^T J S (+ 1 on the diagonal
// of constant globals) is the inverse of the reduced system the frame elimination produces.  One factorisation, then G
// unit right-hand sides, one warp each.
constexpr int kCovQ = 4;  // register slots per lane of a right-hand side: systems of up to 128 unknowns

// Column j of the inverse of a factored n x n system, by one warp (n <= 32 kQ).  A: the factor's lower triangle,
// row-major with leading dimension ld; p: the reciprocals of its pivots.  kLdlt = false: Cholesky M = L L^T (A = L,
// p_i = 1 / L_ii).  kLdlt = true: M = L D L^T as chain_solve's dense phase keeps it (A_ik = L_ik d_k, p_i = 1 / d_i).
// Entry k of the column lands in lane k mod 32, slot k / 32 of x.
template <int kQ, bool kLdlt>
__device__ __forceinline__ void warp_inverse_column(const double* A, int ld, const double* p, int n, int j, int lane, double (&x)[kQ]) {
#pragma unroll
  for (int q = 0; q < kQ; ++q) x[q] = 32 * q + lane == j ? 1.0 : 0.0;
  // forward, from row j on (the rows above are zero): t_k = r_k p_k, r_i -= A_ik t_k below it.  Cholesky keeps t = L^-1 e_j,
  // L D L^T keeps r = L^-1 e_j (unit L)
#pragma unroll
  for (int q = 0; q < kQ; ++q) {
    for (int l = 0; l < 32; ++l) {
      const int k = 32 * q + l;
      if (k < j || k >= n) continue;
      const double t = __shfl_sync(0xffffffffu, x[q], l) * p[k];
      if (!kLdlt && lane == l) x[q] = t;
#pragma unroll
      for (int qq = q; qq < kQ; ++qq) {
        const int i = 32 * qq + lane;
        if (i > k && i < n) x[qq] -= A[i * ld + k] * t;
      }
    }
  }
  // backward, both forms: x_i = r_i p_i, r_k -= A_ik x_i above it
#pragma unroll
  for (int q = kQ - 1; q >= 0; --q) {
    for (int l = 31; l >= 0; --l) {
      const int i = 32 * q + l;
      if (i >= n) continue;
      const double xi = __shfl_sync(0xffffffffu, x[q], l) * p[i];
      if (lane == l) x[q] = xi;
      const double* row = A + i * ld + lane;
#pragma unroll
      for (int qq = 0; qq <= q; ++qq)
        if (32 * qq + lane < i) x[qq] -= row[32 * qq] * xi;
    }
  }
}

// Column j of the covariance from column j of the scaled inverse (x: warp_inverse_column's layout, the globals first):
// entries i >= j into cov[i][j] and cov[j][i] (one triangle, mirrored: the matrix is exactly symmetric), unscaled by
// s_i s_j.  Rows and columns of constant globals (mask 0) are exactly 0.
template <int kQ>
__device__ __forceinline__ void cov_store_column(const double (&x)[kQ], const double* sc, const double* mask, int G, int j, int lane,
                                                 double* cov) {
  const bool free_j = mask[j] != 0.0;
#pragma unroll
  for (int q = 0; q < kQ; ++q) {
    const int i = 32 * q + lane;
    if (i < j || i >= G) continue;
    const double v = free_j && mask[i] != 0.0 ? sc[i] * sc[j] * x[q] : 0.0;
    cov[static_cast<int64_t>(i) * G + j] = v;
    cov[static_cast<int64_t>(j) * G + i] = v;
  }
}

// a vision rig as cov_mega_batch_kernel takes it
struct CovArgs {
  int n_frames, G;
  Blocks b;             // the blocks of the evaluated point
  const double* scale;  // Jacobi scale [nf*6 + G]
  const double* D2x;    // explicit damping [nf*6 + G]: 0 on frames and free globals, 1 on constant globals
  const double* mask;   // [G] 0: constant global
  double* part;         // [cluster CTAs][G*G + G] CTA partials of the Schur sum
  double* tot;          // [G*G + G] their total
  double* cov;          // [G*G] the covariance, row-major (frame mode: Σ_gg, the whole scaled inverse)
  double* notpd;        // set to 1 where a pivot fails (zeroed before the launch)
  // frame mode (cov_frame_mega_batch_kernel): D2x also 1 on the frames no active observation sees (frame_used 0), whose
  // blocks of fcov [nf][36] are 0
  const uint8_t* frame_used;
  double* fcov;
  // cross mode (cov_frame_cross_mega_batch_kernel): frame mode's D2x and frame_used; fcov Σ_fg [nf][6][G], fcov_next
  // Σ_f,f+1 [nf - 1][36]
  double* fcov_next;
  // diagonal and cross mode (cov_frame_diag_cross_mega_batch_kernel): cross mode's, and fcov_diag Σ_ff [nf][36]
  double* fcov_diag;
};
// dynamic shared memory of cov_mega_batch_kernel: per warp its frame's scaled [E | g] and X, the reduced system, pivots
__host__ __device__ inline size_t cov_mega_smem_doubles(int G, int n_warps) {
  return static_cast<size_t>(n_warps) * 12 * (G + 1) + static_cast<size_t>(G) * G + 2 * static_cast<size_t>(G);
}

// One vision rig by one thread-block cluster.  Frames are owned as in mega_solve (frame f -> CTA f mod cluster size, warp
// (f / size) mod warps); every CTA forms and factors the reduced system (the same bits everywhere), then the cluster's
// warps share the right-hand sides.  kCovGlobals: the covariance of the globals.  kCovFrames: all G unit right-hand
// sides give Σ_gg; after a cluster barrier one warp per frame refactors B_f, forms X_f = B_f^-1 E_f again and writes
// B_f^-1 + X_f Σ_gg X_f^T (frame_cov_block).  kCovCross: as kCovFrames, but the warp forms X_f and X_f+1 and writes
// -X_f Σ_gg and X_f Σ_gg X_f+1^T (frame_cross_cov_block).  kCovDiagCross: kCovFrames' pass into fcov_diag, then
// kCovCross' pass: one elimination leaves Σ_gg, Σ_ff and Σ_fg on the device (vcgpu_get_observation_influence_batch).
enum CovMode { kCovGlobals, kCovFrames, kCovCross, kCovDiagCross };
template <CovMode kMode>
__device__ __forceinline__ void cov_mega(const CovArgs& a, ClusterScope scope) {
  extern __shared__ double smem[];
  constexpr int FD = 6;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nthreads = blockDim.x, nwarps = nthreads >> 5;
  const int bid = scope.bid(), nb = scope.nb();
  const int G = a.G, M = G + 1, NS = G * G + G, nf = a.n_frames;
  const int64_t nfp = static_cast<int64_t>(nf) * FD;
  const int nk = bid < nf ? (nf - bid + nb - 1) / nb : 0;
  double* wmem = smem;                                           // [nwarps][2][FD][M]
  double* S = wmem + static_cast<size_t>(nwarps) * 2 * FD * M;   // [NS] Schur accumulator, then the reduced system
  double* invd = S + NS;                                         // [G]
  __shared__ int bad;
  const double* scg = a.scale + nfp;
  for (int e = tid; e < NS; e += nthreads) S[e] = 0.0;
  if (tid == 0) bad = 0;
  bool frame_bad = false;
  // this warp's frame f: its damped, scaled block factored in registers, then its scaled [E | 0] and X into Esw and Xw
  // (the warp's slots of wmem; kCovCross passes one slot as both, which leaves X there)
  auto frame_x = [&](int f, double* Esw, double* Xw) {
    const double* sf = a.scale + static_cast<int64_t>(f) * FD;
    const double* Bf = a.b.B + static_cast<int64_t>(f) * FD * FD;
    const double* Ef = a.b.E + static_cast<int64_t>(f) * FD * G;
    double s[FD], L[FD][FD], iL[FD];
#pragma unroll
    for (int i = 0; i < FD; ++i) s[i] = sf[i];
#pragma unroll
    for (int i = 0; i < FD; ++i)
#pragma unroll
      for (int j = 0; j <= i; ++j) {
        const double bij = Bf[i * FD + j];
        double v = bij * s[i] * s[j];
        if (i == j) v = frame_damp<FD>(v, f, i, bij, s[i], 0.0, a.D2x, nullptr, 0, false);
        L[i][j] = v;
      }
#pragma unroll
    for (int j = 0; j < FD; ++j) {
      double d = L[j][j];
#pragma unroll
      for (int q = 0; q < j; ++q) d -= L[j][q] * L[j][q];
      if (!(d > 0.0)) { frame_bad = true; d = 1.0; }
      const double inv = rsqrt(d);
      L[j][j] = d * inv;
      iL[j] = inv;
#pragma unroll
      for (int i = j + 1; i < FD; ++i) {
        double t = L[i][j];
#pragma unroll
        for (int q = 0; q < j; ++q) t -= L[i][q] * L[j][q];
        L[i][j] = t * inv;
      }
    }
    for (int c = lane; c < M; c += 32) {
      double x[FD];
      const double scc = c < G ? scg[c] : 1.0;
#pragma unroll
      for (int i = 0; i < FD; ++i) {
        const double r = (c < G ? Ef[i * G + c] : 0.0) * s[i] * scc;  // the right-hand side plays no part
        Esw[i * M + c] = r;
        x[i] = r;
      }
#pragma unroll
      for (int i = 0; i < FD; ++i) {
        double t = x[i];
#pragma unroll
        for (int q = 0; q < i; ++q) t -= L[i][q] * x[q];
        x[i] = t * iL[i];
      }
#pragma unroll
      for (int i = FD - 1; i >= 0; --i) {
        double t = x[i];
#pragma unroll
        for (int q = i + 1; q < FD; ++q) t -= L[q][i] * x[q];
        x[i] = t * iL[i];
      }
#pragma unroll
      for (int i = 0; i < FD; ++i) Xw[i * M + c] = x[i];
    }
  };
  for (int base = 0; base < nk; base += nwarps) {
    const int k = base + warp;
    __syncthreads();
    double* Esw = wmem + static_cast<size_t>(warp) * 2 * FD * M;
    if (k < nk) frame_x(bid + k * nb, Esw, Esw + FD * M);
    __syncthreads();
    schur_accumulate<FD>(S, wmem, 2 * FD * M, min(nwarps, nk - base), G, tid, nthreads);
  }
  if (frame_bad) *a.notpd = 1.0;
  __syncthreads();
  double* out = a.part + static_cast<int64_t>(bid) * NS;
  for (int e = tid; e < NS; e += nthreads) out[e] = S[e];
  scope.sync();
  mega_reduce_stage1(a.part, NS, nb, NS, a.tot, -1, -1, bid, nb);  // entry e by CTA e mod size, CTAs in order
  scope.sync();
  for (int e = tid; e < NS; e += nthreads) {
    if (e < G * G && e % G > e / G) continue;  // lower triangle only
    S[e] = e < G * G ? reduced_system_entry(e, G, a.b.C[e], __ldcg(a.tot + e), scg, 0.0, a.D2x, nfp) : 0.0;
  }
  __syncthreads();
  if (warp == 0) mega_chol_solve_smem(S, G, lane, invd, &bad);
  __syncthreads();
  if (bad) {
    if (bid == 0 && tid == 0) *a.notpd = 1.0;
    return;
  }
  if constexpr (kMode == kCovGlobals) {
    for (int j = bid * nwarps + warp; j < G; j += nb * nwarps) {
      double x[kCovQ] = {0.0, 0.0, 0.0, 0.0};
      if (a.mask[j] != 0.0) warp_inverse_column<kCovQ, false>(S, G, invd, G, j, lane, x);
      cov_store_column<kCovQ>(x, scg, a.mask, G, j, lane, a.cov);
    }
  } else {
    for (int j = bid * nwarps + warp; j < G; j += nb * nwarps) {
      double x[kCovQ] = {0.0, 0.0, 0.0, 0.0};
      warp_inverse_column<kCovQ, false>(S, G, invd, G, j, lane, x);
#pragma unroll
      for (int q = 0; q < kCovQ; ++q)
        if (32 * q + lane < G) a.cov[static_cast<int64_t>(32 * q + lane) * G + j] = x[q];
    }
    scope.sync();
    if constexpr (kMode == kCovFrames || kMode == kCovDiagCross) {
      // kCovDiagCross: the diagonal blocks first, in their own pass (X_f formed again: held across both products, the
      // two blocks' registers spill)
      for (int k = warp; k < nk; k += nwarps) {
        const int f = bid + k * nb;
        double* out = (kMode == kCovFrames ? a.fcov : a.fcov_diag) + static_cast<int64_t>(f) * FD * FD;
        if (!a.frame_used[f]) {
          for (int e = lane; e < FD * FD; e += 32) out[e] = 0.0;
          continue;
        }
        double* Esw = wmem + static_cast<size_t>(warp) * 2 * FD * M;
        frame_x(f, Esw, Esw + FD * M);
        __syncwarp();
        const double* Xw = wmem + static_cast<size_t>(warp) * 2 * FD * M + FD * M;
        frame_cov_block<FD>(a.b, a.D2x, f, a.scale + static_cast<int64_t>(f) * FD, Xw, M, a.cov, G, lane, out);
        __syncwarp();
      }
    }
    if constexpr (kMode == kCovCross || kMode == kCovDiagCross) {
      // X_f into the warp's second slot, X_f+1 (its owner's bits: the same routine on the same inputs) into its first
      for (int k = warp; k < nk; k += nwarps) {
        const int f = bid + k * nb;
        double* fg = a.fcov + static_cast<int64_t>(f) * FD * G;
        double* fn = f + 1 < nf ? a.fcov_next + static_cast<int64_t>(f) * FD * FD : nullptr;
        if (!a.frame_used[f]) {
          for (int e = lane; e < FD * G; e += 32) fg[e] = 0.0;
          if (fn)
            for (int e = lane; e < FD * FD; e += 32) fn[e] = 0.0;
          continue;
        }
        double* Xn = wmem + static_cast<size_t>(warp) * 2 * FD * M;
        double* Xf = Xn + FD * M;
        frame_x(f, Xf, Xf);
        const bool next = fn && a.frame_used[f + 1];
        if (next) frame_x(f + 1, Xn, Xn);
        __syncwarp();
        const double* sf = a.scale + static_cast<int64_t>(f) * FD;
        frame_cross_cov_block<FD>(Xf, next ? Xn : nullptr, M, a.cov, G, sf, sf + FD, scg, a.mask, lane, fg, fn);
        __syncwarp();
      }
    }
  }
}

// A batch of vision rigs, one thread-block cluster each: cluster k writes the covariance of args[k].
__global__ void __launch_bounds__(kMegaMaxThreads, 1) cov_mega_batch_kernel(const CovArgs* __restrict__ args) {
  ClusterScope scope;
  cov_mega<kCovGlobals>(args[blockIdx.x / scope.nb()], scope);
}
// ... the frame covariance of args[k] (vcgpu_get_frame_covariance_batch)
__global__ void __launch_bounds__(kMegaMaxThreads, 1) cov_frame_mega_batch_kernel(const CovArgs* __restrict__ args) {
  ClusterScope scope;
  cov_mega<kCovFrames>(args[blockIdx.x / scope.nb()], scope);
}
// ... the frame blocks off the diagonal of args[k] (vcgpu_get_frame_cross_covariance_batch)
__global__ void __launch_bounds__(kMegaMaxThreads, 1) cov_frame_cross_mega_batch_kernel(const CovArgs* __restrict__ args) {
  ClusterScope scope;
  cov_mega<kCovCross>(args[blockIdx.x / scope.nb()], scope);
}
// ... the frame blocks on and off the diagonal of args[k] from one elimination (vcgpu_get_observation_influence_batch)
__global__ void __launch_bounds__(kMegaMaxThreads, 1) cov_frame_diag_cross_mega_batch_kernel(const CovArgs* __restrict__ args) {
  ClusterScope scope;
  cov_mega<kCovDiagCross>(args[blockIdx.x / scope.nb()], scope);
}

}  // namespace vc
