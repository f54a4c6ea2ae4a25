// Hand-eye alignment of the gyro stream with the vision poses (vcgpu_align_imu, include/vcgpu.h): the rotation Q from
// the IMU's axes to the rig's, the time offset ts and the gyro bias b_g.  Over usable interval j (frames f, f+1):
//   a_j = log(R_f^T R_f+1)                the rig's turn from the frame poses of the accepted state
//   b_j(s, b_g) = log(dR_j)               the attitude integrate_imu reaches from the identity over GetRange(t_f, t_f+1, s)
// and a_j = Q b_j at the truth.  Kernels, each over a table of rigs (AlignRig):
//   align_prep_kernel    one thread per usable interval: a_j
//   align_grid_kernel    one CTA per (rig, candidate s, tile of kAlignThreads intervals): each thread integrates its
//                        interval's attitude; the CTA reduces the kAlignSums sums (M = sum a b^T, sum |b|^2, sum |a|^2)
//                        into the tile's partial
//   align_cost_kernel    one thread per (rig, candidate): the tiles in order, Horn's 4 x 4 matrix, its largest
//                        eigenpair (cyclic Jacobi), cost(s) and the candidate's Q
//   align_refine_kernel  one CTA per rig: the argmin, then Gauss-Newton on (dtheta, s, b_g) with step halving, rms and
//                        the excitation eigenvalues
// Every sum runs in an order fixed by the rig's own sizes (its interval count, its tiles), so a rig's outputs are the
// same bits whatever else is in the table.
#pragma once
#include "vc_imu_math.cuh"
#include "vc_imu_poses.cuh"

namespace vc {
namespace imu {

constexpr int kAlignThreads = 128;       // intervals per grid tile
constexpr int kAlignRefineThreads = 256;
constexpr int kAlignSums = 11;           // M (9, row-major M[i][k] = sum a_i b_k) | sum |b|^2 | sum |a|^2
constexpr int kAlignHalvings = 10;       // step halvings a Gauss-Newton iteration may try
constexpr int kAlignOut = 16;            // Q (x y z w) | ts | b_g (3) | excitation (3) | n | iterations | failed | rms | 0
constexpr int kAlignN = 7;               // Gauss-Newton unknowns: dtheta (3) | s | b_g (3)

// one usable interval: its frame times and its first frame
struct AlignIv {
  double t0, t1;
  int f, pad_;
};

// one rig's entry in the argument table
struct AlignRig {
  ImuBuf buf;
  const double* state;   // the accepted state: T_wp at 0, the IMU block at off_imu (b_g at 2, sf_g at 8, ts at 14)
  int64_t off_imu;
  const AlignIv* iv;     // [n]
  double* a;             // [n][3]
  double* part;          // [n_cand][n_tiles][kAlignSums]
  double* curve;         // [n_cand] cost(s)
  double* horn;          // [n_cand][4] each candidate's Q (x y z w)
  double* out;           // [kAlignOut]
  double ts_lo, ts_hi, step;  // candidate c: ts_lo + c * step, the last one ts_hi
  int n, n_cand, n_tiles;
  int fit_ts, max_iters;
  int64_t blk0;          // the rig's first grid CTA
  int iv0, cand0;        // its first interval and candidate over the table
};

// candidate c's s; no contraction, so the host's restatement (ts_lo + c * step) gives the same double
__device__ __forceinline__ double align_cand_ts(const AlignRig& g, int c) {
  if (!g.fit_ts) return g.state[g.off_imu + 14];
  return c == g.n_cand - 1 && g.n_cand > 1 ? g.ts_hi : __dadd_rn(g.ts_lo, __dmul_rn(static_cast<double>(c), g.step));
}

// the rig of table entry t: the last rig whose first entry (member `first`) is <= t
template <class K>
__device__ __forceinline__ int align_rig(const AlignRig* rigs, int n_rigs, int64_t t, K first) {
  int lo = 0, hi = n_rigs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (first(rigs[mid]) <= t) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// log of the attitude integrate_imu reaches from the identity over GetRange(t0, t1, ts), with gyro scale sfg and bias bg
// (the accelerometer terms do not reach the attitude and are left at zero)
template <class T>
__device__ inline Vec<T> align_attitude(const ImuBuf& buf, double t0, double t1, T ts, Vec<T> bg, const double sfg[3]) {
  const T sf[6] = {T(sfg[0]), T(sfg[1]), T(sfg[2]), T(1.0), T(1.0), T(1.0)};
  const Vec<T> zero{T(0.0), T(0.0), T(0.0)};
  Pose<T> y{zero, {T(0.0), T(0.0), T(0.0), T(1.0)}, zero};
  NoTangent nt;
  int idx;
  Meas<T> prev = get_element<T>(buf, t0, ts, &idx), cur;
  bool more = true;
  while (more) {
    more = get_next<T>(buf, t1, ts, &idx, &cur);
    y = integrate_imu(y, prev, cur, bg, zero, sf, zero, nt);
    prev = cur;
  }
  T th;
  return so3_log(y.q, &th);
}

__device__ __forceinline__ void align_sfg_bg(const AlignRig& g, double sfg[3], Vec<double>* bg) {
  const double* P = g.state + g.off_imu;
  sfg[0] = P[8]; sfg[1] = P[9]; sfg[2] = P[10];
  *bg = Vec<double>{P[2], P[3], P[4]};
}

// a_j of every usable interval of every rig, one thread each
__global__ void __launch_bounds__(kAlignThreads) align_prep_kernel(const AlignRig* rigs, int n_rigs, int total) {
  const int t = blockIdx.x * kAlignThreads + threadIdx.x;
  if (t >= total) return;
  const AlignRig& g = rigs[align_rig(rigs, n_rigs, t, [](const AlignRig& r) { return static_cast<int64_t>(r.iv0); })];
  const int j = t - g.iv0;
  const double* X = g.state + 7 * static_cast<int64_t>(g.iv[j].f);
  const Quat<double> q = qmul(qconj(Quat<double>{X[0], X[1], X[2], X[3]}), Quat<double>{X[7], X[8], X[9], X[10]});
  double th;
  const Vec<double> a = so3_log(q, &th);
  g.a[3 * j] = a.x; g.a[3 * j + 1] = a.y; g.a[3 * j + 2] = a.z;
}

// sum of v[0 .. N) over the CTA, in a fixed order: a butterfly within each warp, then the warps in order by thread 0.
// Every thread's v is overwritten; thread 0 returns with the totals.  red: [blockDim.x / 32][N] shared doubles.
template <int N>
__device__ __forceinline__ void align_block_sum(double v[N], double* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int k = 0; k < N; ++k)
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], d);
  __syncthreads();  // red may still be read by an earlier call
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < N; ++k) red[wid * N + k] = v[k];
  __syncthreads();
  if (threadIdx.x == 0)
    for (int k = 0; k < N; ++k) {
      double s = red[k];
      for (int w = 1; w < nw; ++w) s += red[w * N + k];
      v[k] = s;
    }
}

__global__ void __launch_bounds__(kAlignThreads) align_grid_kernel(const AlignRig* rigs, int n_rigs) {
  __shared__ double red[kAlignThreads / 32 * kAlignSums];
  const AlignRig& g = rigs[align_rig(rigs, n_rigs, blockIdx.x, [](const AlignRig& r) { return r.blk0; })];
  const int local = static_cast<int>(blockIdx.x - g.blk0);
  const int c = local / g.n_tiles, tile = local - c * g.n_tiles;
  const int j = tile * kAlignThreads + threadIdx.x;
  double v[kAlignSums];
#pragma unroll
  for (int k = 0; k < kAlignSums; ++k) v[k] = 0.0;
  if (j < g.n) {
    double sfg[3];
    Vec<double> bg;
    align_sfg_bg(g, sfg, &bg);
    const AlignIv iv = g.iv[j];
    const Vec<double> b = align_attitude<double>(g.buf, iv.t0, iv.t1, align_cand_ts(g, c), bg, sfg);
    const double a[3] = {g.a[3 * j], g.a[3 * j + 1], g.a[3 * j + 2]};
    const double bb[3] = {b.x, b.y, b.z};
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int k = 0; k < 3; ++k) v[3 * i + k] = a[i] * bb[k];
    v[9] = dot(b, b);
    v[10] = a[0] * a[0] + a[1] * a[1] + a[2] * a[2];
  }
  align_block_sum<kAlignSums>(v, red);
  if (threadIdx.x == 0) {
    double* o = g.part + (static_cast<int64_t>(c) * g.n_tiles + tile) * kAlignSums;
#pragma unroll
    for (int k = 0; k < kAlignSums; ++k) o[k] = v[k];
  }
}

// eigen-decomposition of a symmetric N x N matrix by cyclic Jacobi rotations, one thread: A becomes diagonal (its
// eigenvalues), V's columns the eigenvectors.  Sweeps stop when every off-diagonal entry is exactly 0, or after 32.
template <int N>
__device__ inline void align_jacobi(double A[N][N], double V[N][N]) {
  for (int i = 0; i < N; ++i)
    for (int k = 0; k < N; ++k) V[i][k] = i == k ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 32; ++sweep) {
    bool any = false;
    for (int p = 0; p < N - 1; ++p)
      for (int q = p + 1; q < N; ++q) {
        const double apq = A[p][q];
        // an entry below the rounding of both diagonal entries is set to 0 (Numerical Recipes' jacobi test)
        if (fabs(apq) * 1e18 <= fabs(A[p][p]) && fabs(apq) * 1e18 <= fabs(A[q][q])) {
          A[p][q] = A[q][p] = 0.0;
          continue;
        }
        if (apq == 0.0) continue;
        any = true;
        const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double cs = 1.0 / sqrt(t * t + 1.0), sn = t * cs;
        for (int k = 0; k < N; ++k) {
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = cs * akp - sn * akq;
          A[k][q] = sn * akp + cs * akq;
        }
        for (int k = 0; k < N; ++k) {
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = cs * apk - sn * aqk;
          A[q][k] = sn * apk + cs * aqk;
        }
        A[p][q] = A[q][p] = 0.0;
        for (int k = 0; k < N; ++k) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = cs * vkp - sn * vkq;
          V[k][q] = sn * vkp + cs * vkq;
        }
      }
    if (!any) break;
  }
}

// Horn's closed form from the kAlignSums sums s: the Q (x y z w) that maximises sum a . Q b, and
// cost = (sum |a|^2 + sum |b|^2 - 2 lambda_max) / n
__device__ inline double align_horn(const double s[kAlignSums], int n, double Qo[4]) {
  // S = sum b a^T = M^T: S[x][y] = M[y][x]
  auto S = [&](int x, int y) { return s[3 * y + x]; };
  double N[4][4] = {
      {S(0, 0) + S(1, 1) + S(2, 2), S(1, 2) - S(2, 1), S(2, 0) - S(0, 2), S(0, 1) - S(1, 0)},
      {S(1, 2) - S(2, 1), S(0, 0) - S(1, 1) - S(2, 2), S(0, 1) + S(1, 0), S(2, 0) + S(0, 2)},
      {S(2, 0) - S(0, 2), S(0, 1) + S(1, 0), -S(0, 0) + S(1, 1) - S(2, 2), S(1, 2) + S(2, 1)},
      {S(0, 1) - S(1, 0), S(2, 0) + S(0, 2), S(1, 2) + S(2, 1), -S(0, 0) - S(1, 1) + S(2, 2)}};
  double V[4][4];
  align_jacobi<4>(N, V);
  int m = 0;
  for (int k = 1; k < 4; ++k)
    if (N[k][k] > N[m][m]) m = k;
  // (w x y z) -> (x y z w)
  Qo[0] = V[1][m]; Qo[1] = V[2][m]; Qo[2] = V[3][m]; Qo[3] = V[0][m];
  return (s[10] + s[9] - 2.0 * N[m][m]) / static_cast<double>(n);
}

// cost(s) of every candidate of every rig, one thread each
__global__ void __launch_bounds__(kAlignThreads) align_cost_kernel(const AlignRig* rigs, int n_rigs, int total) {
  const int t = blockIdx.x * kAlignThreads + threadIdx.x;
  if (t >= total) return;
  const AlignRig& g = rigs[align_rig(rigs, n_rigs, t, [](const AlignRig& r) { return static_cast<int64_t>(r.cand0); })];
  const int c = t - g.cand0;
  double s[kAlignSums];
  const double* p = g.part + static_cast<int64_t>(c) * g.n_tiles * kAlignSums;
  for (int k = 0; k < kAlignSums; ++k) s[k] = p[k];
  for (int tile = 1; tile < g.n_tiles; ++tile)
    for (int k = 0; k < kAlignSums; ++k) s[k] += p[tile * kAlignSums + k];
  double Q[4];
  g.curve[c] = align_horn(s, g.n, Q);
  for (int k = 0; k < 4; ++k) g.horn[4 * c + k] = Q[k];
}

// ---------------------------------------------------------------- refinement
struct AlignPoint {
  Quat<double> Q;
  double s;
  Vec<double> bg;
};

// mean |a_j - Q b_j|^2 at x over the rig's intervals; every thread returns it
__device__ inline double align_cost_at(const AlignRig& g, const AlignPoint& x, const double sfg[3], double* red,
                                       double* bcast) {
  double v[1] = {0.0};
  for (int j = threadIdx.x; j < g.n; j += blockDim.x) {
    const Vec<double> b = align_attitude<double>(g.buf, g.iv[j].t0, g.iv[j].t1, x.s, x.bg, sfg);
    const Vec<double> qb = qrot(x.Q, b);
    const double r0 = g.a[3 * j] - qb.x, r1 = g.a[3 * j + 1] - qb.y, r2 = g.a[3 * j + 2] - qb.z;
    v[0] += r0 * r0 + r1 * r1 + r2 * r2;
  }
  align_block_sum<1>(v, red);
  if (threadIdx.x == 0) *bcast = v[0] / static_cast<double>(g.n);
  __syncthreads();
  return *bcast;
}

// the Gauss-Newton normal equations at x: H (upper triangle, 28) | -J^T r (7), summed over the rig's intervals.  J's
// s and b_g columns come from D1 duals seeded along one direction each; s only when fit_ts.
constexpr int kAlignNe = kAlignN * (kAlignN + 1) / 2 + kAlignN;
__device__ inline void align_normal(const AlignRig& g, const AlignPoint& x, const double sfg[3], double v[kAlignNe]) {
  for (int k = 0; k < kAlignNe; ++k) v[k] = 0.0;
  for (int j = threadIdx.x; j < g.n; j += blockDim.x) {
    const AlignIv iv = g.iv[j];
    const Vec<double> b = align_attitude<double>(g.buf, iv.t0, iv.t1, x.s, x.bg, sfg);
    const Vec<double> qb = qrot(x.Q, b);
    const double r[3] = {g.a[3 * j] - qb.x, g.a[3 * j + 1] - qb.y, g.a[3 * j + 2] - qb.z};
    // J = [ [Q b]_x | -Q db/ds | -Q db/db_g ]
    double J[3][kAlignN];
    J[0][0] = 0.0;   J[0][1] = -qb.z; J[0][2] = qb.y;
    J[1][0] = qb.z;  J[1][1] = 0.0;   J[1][2] = -qb.x;
    J[2][0] = -qb.y; J[2][1] = qb.x;  J[2][2] = 0.0;
    for (int d = 0; d < 4; ++d) {
      Vec<double> db{0.0, 0.0, 0.0};
      if (d > 0 || g.fit_ts) {
        const D1 ts(x.s, d == 0 ? 1.0 : 0.0);
        const Vec<D1> bg{D1(x.bg.x, d == 1 ? 1.0 : 0.0), D1(x.bg.y, d == 2 ? 1.0 : 0.0), D1(x.bg.z, d == 3 ? 1.0 : 0.0)};
        const Vec<D1> bd = align_attitude<D1>(g.buf, iv.t0, iv.t1, ts, bg, sfg);
        db = qrot(x.Q, Vec<double>{bd.x.v, bd.y.v, bd.z.v});
      }
      J[0][3 + d] = -db.x; J[1][3 + d] = -db.y; J[2][3 + d] = -db.z;
    }
    int o = 0;
    for (int p = 0; p < kAlignN; ++p)
      for (int q = p; q < kAlignN; ++q) v[o++] += J[0][p] * J[0][q] + J[1][p] * J[1][q] + J[2][p] * J[2][q];
    for (int p = 0; p < kAlignN; ++p) v[o++] -= J[0][p] * r[0] + J[1][p] * r[1] + J[2][p] * r[2];
  }
}

// solve H d = rhs (H from its upper triangle) by Cholesky; false where a pivot is not positive
__device__ inline bool align_chol_solve(const double* ne, double d[kAlignN]) {
  double L[kAlignN][kAlignN];
  int o = 0;
  for (int p = 0; p < kAlignN; ++p)
    for (int q = p; q < kAlignN; ++q) L[q][p] = ne[o++];
  for (int k = 0; k < kAlignN; ++k) {
    double s = L[k][k];
    for (int m = 0; m < k; ++m) s -= L[k][m] * L[k][m];
    if (!(s > 0.0)) return false;
    L[k][k] = sqrt(s);
    for (int i = k + 1; i < kAlignN; ++i) {
      double t = L[i][k];
      for (int m = 0; m < k; ++m) t -= L[i][m] * L[k][m];
      L[i][k] = t / L[k][k];
    }
  }
  for (int i = 0; i < kAlignN; ++i) {
    double t = ne[kAlignN * (kAlignN + 1) / 2 + i];
    for (int m = 0; m < i; ++m) t -= L[i][m] * d[m];
    d[i] = t / L[i][i];
  }
  for (int i = kAlignN - 1; i >= 0; --i) {
    double t = d[i];
    for (int m = i + 1; m < kAlignN; ++m) t -= L[m][i] * d[m];
    d[i] = t / L[i][i];
  }
  return true;
}

// one CTA per rig
__global__ void __launch_bounds__(kAlignRefineThreads) align_refine_kernel(const AlignRig* rigs) {
  __shared__ double red[kAlignRefineThreads / 32 * kAlignNe];
  __shared__ double bcast;
  __shared__ int arg_i[kAlignRefineThreads];
  __shared__ double arg_v[kAlignRefineThreads];
  __shared__ AlignPoint xs, xc;  // the current point, the trial point
  __shared__ int state;          // 0 running, 1 done, 2 numeric failure
  const AlignRig& g = rigs[blockIdx.x];
  double sfg[3];
  Vec<double> bg0;
  align_sfg_bg(g, sfg, &bg0);
  // the least cost, the lowest index among equals (NaN never wins)
  int bi = -1;
  double bv = 0.0;
  for (int c = threadIdx.x; c < g.n_cand; c += blockDim.x) {
    const double v = g.curve[c];
    if (v == v && (bi < 0 || v < bv)) { bi = c; bv = v; }
  }
  arg_i[threadIdx.x] = bi;
  arg_v[threadIdx.x] = bv;
  __syncthreads();
  double* out = g.out;
  int iters = 0;
  if (threadIdx.x == 0) {
    int m = -1;
    double mv = 0.0;
    for (int t = 0; t < blockDim.x; ++t)
      if (arg_i[t] >= 0 && (m < 0 || arg_v[t] < mv || (arg_v[t] == mv && arg_i[t] < m))) { m = arg_i[t]; mv = arg_v[t]; }
    if (m < 0) m = 0;  // every cost NaN: fewer than one usable interval
    xs.Q = Quat<double>{g.horn[4 * m], g.horn[4 * m + 1], g.horn[4 * m + 2], g.horn[4 * m + 3]};
    xs.s = align_cand_ts(g, m);
    xs.bg = bg0;
    state = g.n < 3 ? 2 : 0;
  }
  __syncthreads();
  if (state == 0) {
    double cost = align_cost_at(g, xs, sfg, red, &bcast);
    for (int it = 0; it < g.max_iters; ++it) {
      double v[kAlignNe];
      align_normal(g, xs, sfg, v);
      align_block_sum<kAlignNe>(v, red);
      double d[kAlignN];
      if (threadIdx.x == 0) {
        if (!g.fit_ts) {  // s is no unknown: a unit row and column and a zero right-hand side keep it exactly
          int o = 0;
          for (int p = 0; p < kAlignN; ++p)
            for (int q = p; q < kAlignN; ++q, ++o)
              if (p == 3 || q == 3) v[o] = p == q ? 1.0 : 0.0;
          v[kAlignN * (kAlignN + 1) / 2 + 3] = 0.0;
        }
        if (!align_chol_solve(v, d)) state = 2;
      }
      __syncthreads();
      if (state != 0) break;
      bool accepted = false;
      double alpha = 1.0;
      for (int hv = 0; hv <= kAlignHalvings && !accepted; ++hv, alpha *= 0.5) {
        if (threadIdx.x == 0) {
          const Quat<double> dq = so3_exp(Vec<double>{alpha * d[0], alpha * d[1], alpha * d[2]});
          Quat<double> q = qmul(dq, xs.Q);
          const double nq = sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
          xc.Q = Quat<double>{q.x / nq, q.y / nq, q.z / nq, q.w / nq};
          xc.s = g.fit_ts ? fmin(fmax(xs.s + alpha * d[3], g.ts_lo), g.ts_hi) : xs.s;
          xc.bg = Vec<double>{xs.bg.x + alpha * d[4], xs.bg.y + alpha * d[5], xs.bg.z + alpha * d[6]};
        }
        __syncthreads();
        const double c2 = align_cost_at(g, xc, sfg, red, &bcast);
        if (c2 < cost) {
          accepted = true;
          cost = c2;
          __syncthreads();
          if (threadIdx.x == 0) xs = xc;
          __syncthreads();
        }
      }
      if (!accepted) break;
      ++iters;
    }
  }
  // excitation: the eigenvalues of (1/n) sum b b^T at the result (at the start point if the fit failed)
  {
    double v[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int j = threadIdx.x; j < g.n; j += blockDim.x) {
      const Vec<double> b = align_attitude<double>(g.buf, g.iv[j].t0, g.iv[j].t1, xs.s, xs.bg, sfg);
      v[0] += b.x * b.x; v[1] += b.x * b.y; v[2] += b.x * b.z; v[3] += b.y * b.y; v[4] += b.y * b.z; v[5] += b.z * b.z;
    }
    align_block_sum<6>(v, red);
    if (threadIdx.x == 0) {
      const double inv = 1.0 / static_cast<double>(g.n);
      double A[3][3] = {{v[0] * inv, v[1] * inv, v[2] * inv}, {v[1] * inv, v[3] * inv, v[4] * inv},
                        {v[2] * inv, v[4] * inv, v[5] * inv}};
      double V[3][3];
      align_jacobi<3>(A, V);
      double e[3] = {A[0][0], A[1][1], A[2][2]};
      for (int i = 0; i < 2; ++i)
        for (int k = 0; k < 2 - i; ++k)
          if (e[k + 1] < e[k]) { const double t = e[k]; e[k] = e[k + 1]; e[k + 1] = t; }
      out[8] = e[0]; out[9] = e[1]; out[10] = e[2];
    }
  }
  if (threadIdx.x == 0) {
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    out[11] = g.n;
    out[12] = iters;
    out[13] = state == 2 ? 1.0 : 0.0;
    out[14] = out[15] = 0.0;
    if (state == 2) {
      for (int k = 0; k < 8; ++k) out[k] = nan;
    } else {
      const double sg = xs.Q.w < 0.0 ? -1.0 : 1.0;
      out[0] = sg * xs.Q.x; out[1] = sg * xs.Q.y; out[2] = sg * xs.Q.z; out[3] = sg * xs.Q.w;
      out[4] = xs.s;
      out[5] = xs.bg.x; out[6] = xs.bg.y; out[7] = xs.bg.z;
    }
  }
  // rms at the result (its cost pass runs with every thread)
  if (state != 2) {
    const double c = align_cost_at(g, xs, sfg, red, &bcast);
    if (threadIdx.x == 0) out[14] = sqrt(c);
  } else if (threadIdx.x == 0) {
    out[14] = __longlong_as_double(0x7ff8000000000000LL);
  }
}

}  // namespace imu
}  // namespace vc
