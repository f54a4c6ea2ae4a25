// Batched pose initialisation: the pose of the planar calibration target in every (frame, camera) view, one WARP per
// view — the step right before the calibration solve (SURVEY §8 f3).
//
// Replaces the per-frame, per-camera call `PosePnPRansac(camera, ellipses, target.Circles3D(), ellipse_target_map, 0, 0,
// &t_cw)` at src/vicalib-task.cc:322-325 (Calibu's PosePnPRansac over OpenCV's iterative solvePnP; both un-vendored):
//   1. unproject the detected centres through the camera model to normalised coordinates (lane per point)
//   2. homography target plane -> normalised image: Hartley-normalised DLT, A^T A (45 sums per lane, warp-reduced),
//      its null vector by a cyclic Jacobi eigen-decomposition in the warp's shared memory
//   3. pose from the homography columns, target in front of the camera
//   4. 12 Levenberg-Marquardt iterations on the 6-DoF pose (left perturbation): one pass over the points per iteration
//      (cost, J^T J, J^T r at the candidate: 28 sums per lane, warp-reduced), 6 x 6 Cholesky in registers
//   robust_its > 0: RANSAC over 4-point homographies (deterministic sample sequence), steps 2-4 on the inliers.
// CPU restatement: oracle/pnp.py.  The frame pose handed to the solve is T_wp = T_cw^-1 * T_ck (vicalib-task.cc:341-349).
#pragma once
#include "vc_internal.h"
#include "vc_math.cuh"

namespace vc {
namespace pnp {

constexpr int kLmIters = 12;
constexpr int kNewtonIters = 8;
constexpr int kWarps = 4;

__device__ inline void unproject(int model, const double* p, double u, double v, double* x, double* y) {
  const double xd = (u - p[2]) / p[0], yd = (v - p[3]) / p[1];
  const double rd = sqrt(xd * xd + yd * yd);
  double ru = rd, limit = 1.0;
  if (model == kFov) {
    const double w = p[4], m = 2.0 * tan(w / 2.0);
    ru = tan(fmin(rd * w, 1.5)) / m;
    limit = w / m;
  } else if (model == kPoly2 || model == kPoly3) {
    const double k0 = p[4], k1 = p[5], k2 = model == kPoly3 ? p[6] : 0.0;
    for (int it = 0; it < kNewtonIters; ++it) {
      const double r2 = ru * ru;
      const double f = 1 + r2 * (k0 + r2 * (k1 + r2 * k2));
      const double df = f + ru * ru * (2 * k0 + r2 * (4 * k1 + r2 * 6 * k2));
      ru = ru - (ru * f - rd) / df;
    }
  } else if (model == kKb4) {
    double th = rd;
    for (int it = 0; it < kNewtonIters; ++it) {
      const double t2 = th * th;
      const double d = th * (1 + t2 * (p[4] + t2 * (p[5] + t2 * (p[6] + t2 * p[7]))));
      const double dd = 1 + t2 * (3 * p[4] + t2 * (5 * p[5] + t2 * (7 * p[6] + t2 * 9 * p[7])));
      th = th - (d - rd) / dd;
    }
    ru = tan(fmin(th, 1.5));
  }
  const double s = rd <= 1e-12 ? limit : ru / rd;
  *x = xd * s;
  *y = yd * s;
}

__device__ __forceinline__ double wsum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Hartley normalisation of the selected points: scale s and centre (cx, cy) with T = [s 0 -s cx; 0 s -s cy; 0 0 1]
__device__ inline void hartley(const double* pts, int stride, int ox, int oy, const unsigned char* use, int cnt, int lane, double* s,
                               double* cx, double* cy) {
  double sx = 0, sy = 0, n = 0;
  for (int i = lane; i < cnt; i += 32)
    if (use[i]) { sx += pts[i * stride + ox]; sy += pts[i * stride + oy]; n += 1.0; }
  sx = wsum(sx); sy = wsum(sy); n = wsum(n);
  *cx = sx / n; *cy = sy / n;
  double d = 0;
  for (int i = lane; i < cnt; i += 32)
    if (use[i]) {
      const double dx = pts[i * stride + ox] - *cx, dy = pts[i * stride + oy] - *cy;
      d += sqrt(dx * dx + dy * dy);
    }
  d = wsum(d) / n;
  *s = d > 0 ? sqrt(2.0) / d : 1.0;
}

// cyclic Jacobi on the symmetric 9 x 9 matrix A (shared memory), eigenvectors in V; round-robin pairing: round r
// holds the four disjoint pairs {i, j}, i + j = r (mod 9)
__device__ inline void jacobi9(double* A, double* V, double* rot, int* rpq, int lane) {
  for (int e = lane; e < 81; e += 32) V[e] = (e / 9 == e % 9) ? 1.0 : 0.0;
  __syncwarp();
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off = 0.0, dg = 0.0;
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      dg += A[i * 9 + i] * A[i * 9 + i];
#pragma unroll
      for (int j = i + 1; j < 9; ++j) off += A[i * 9 + j] * A[i * 9 + j];
    }
    if (off <= 1e-30 * dg) break;
    for (int r = 0; r < 9; ++r) {
      if (lane < 4) {
        int cnt = 0, pi = 0, qi = 0;
#pragma unroll
        for (int i = 0; i < 9; ++i) {
          const int j = (r - i + 9) % 9;
          if (i < j) {
            if (cnt == lane) { pi = i; qi = j; }
            ++cnt;
          }
        }
        const double apq = A[pi * 9 + qi];
        double c = 1.0, sn = 0.0;
        if (apq != 0.0) {
          const double tau = (A[qi * 9 + qi] - A[pi * 9 + pi]) / (2.0 * apq);
          const double t = (tau >= 0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
          c = 1.0 / sqrt(1.0 + t * t);
          sn = t * c;
        }
        rot[2 * lane] = c; rot[2 * lane + 1] = sn;
        rpq[2 * lane] = pi; rpq[2 * lane + 1] = qi;
      }
      __syncwarp();
      for (int e = lane; e < 36; e += 32) {
        const int k = e >> 2, t = e & 3, p = rpq[2 * t], q = rpq[2 * t + 1];
        const double c = rot[2 * t], sn = rot[2 * t + 1];
        const double akp = A[k * 9 + p], akq = A[k * 9 + q];
        A[k * 9 + p] = c * akp - sn * akq;
        A[k * 9 + q] = sn * akp + c * akq;
        const double vkp = V[k * 9 + p], vkq = V[k * 9 + q];
        V[k * 9 + p] = c * vkp - sn * vkq;
        V[k * 9 + q] = sn * vkp + c * vkq;
      }
      __syncwarp();
      for (int e = lane; e < 36; e += 32) {
        const int k = e >> 2, t = e & 3, p = rpq[2 * t], q = rpq[2 * t + 1];
        const double c = rot[2 * t], sn = rot[2 * t + 1];
        const double apk = A[p * 9 + k], aqk = A[q * 9 + k];
        A[p * 9 + k] = c * apk - sn * aqk;
        A[q * 9 + k] = sn * apk + c * aqk;
      }
      __syncwarp();
    }
  }
}

struct WarpMem {
  double A[81], V[81], rot[8];
  int rpq[8];
};

// homography xy ~ H (X, Y, 1) of the points with use[i] != 0 (at least 4); H row-major in registers of every lane
__device__ inline void homography(const double* pw, const double* xy, const unsigned char* use, int cnt, WarpMem* sm, int lane, double H[9]) {
  double sa, cax, cay, sb, cbx, cby;
  hartley(pw, 3, 0, 1, use, cnt, lane, &sa, &cax, &cay);
  hartley(xy, 2, 0, 1, use, cnt, lane, &sb, &cbx, &cby);
  double M[45];
#pragma unroll
  for (int k = 0; k < 45; ++k) M[k] = 0.0;
  for (int i = lane; i < cnt; i += 32) {
    if (!use[i]) continue;
    const double X = sa * (pw[3 * i] - cax), Y = sa * (pw[3 * i + 1] - cay);
    const double x = sb * (xy[2 * i] - cbx), y = sb * (xy[2 * i + 1] - cby);
    const double r1[9] = {X, Y, 1, 0, 0, 0, -x * X, -x * Y, -x};
    const double r2[9] = {0, 0, 0, X, Y, 1, -y * X, -y * Y, -y};
    int k = 0;
#pragma unroll
    for (int a = 0; a < 9; ++a)
#pragma unroll
      for (int b = 0; b <= a; ++b, ++k) M[k] += r1[a] * r1[b] + r2[a] * r2[b];
  }
  __syncwarp();
  {
    int k = 0;
#pragma unroll
    for (int a = 0; a < 9; ++a)
#pragma unroll
      for (int b = 0; b <= a; ++b, ++k) {
        const double v = wsum(M[k]);
        if (lane == 0) { sm->A[a * 9 + b] = v; sm->A[b * 9 + a] = v; }
      }
  }
  __syncwarp();
  jacobi9(sm->A, sm->V, sm->rot, sm->rpq, lane);
  int best = 0;
#pragma unroll
  for (int k = 1; k < 9; ++k) best = sm->A[k * 9 + k] < sm->A[best * 9 + best] ? k : best;
  double h[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) h[k] = sm->V[k * 9 + best];
  // H = Tb^-1 h Ta,  Ta = [sa 0 -sa cax; 0 sa -sa cay; 0 0 1],  Tb^-1 = [1/sb 0 cbx; 0 1/sb cby; 0 0 1]
  double G[9];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    G[r * 3] = h[r * 3] * sa;
    G[r * 3 + 1] = h[r * 3 + 1] * sa;
    G[r * 3 + 2] = h[r * 3 + 2] - sa * (h[r * 3] * cax + h[r * 3 + 1] * cay);
  }
  const double isb = 1.0 / sb;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    H[c] = G[c] * isb + cbx * G[6 + c];
    H[3 + c] = G[3 + c] * isb + cby * G[6 + c];
    H[6 + c] = G[6 + c];
  }
  __syncwarp();
}

// cost, J^T J (21, lower triangle row-major) and J^T r (6) of the selected points at (R, t): sums over the warp
__device__ inline void lm_system(const double R[9], const double t[3], const double* pw, const double* xy, const unsigned char* use,
                                 int cnt, int lane, double* cost, double JtJ[21], double Jtr[6]) {
  double c = 0.0, a[21], g[6];
#pragma unroll
  for (int k = 0; k < 21; ++k) a[k] = 0.0;
#pragma unroll
  for (int k = 0; k < 6; ++k) g[k] = 0.0;
  for (int i = lane; i < cnt; i += 32) {
    if (!use[i]) continue;
    const double X = pw[3 * i], Y = pw[3 * i + 1], Z = pw[3 * i + 2];
    const double px = R[0] * X + R[1] * Y + R[2] * Z + t[0], py = R[3] * X + R[4] * Y + R[5] * Z + t[1],
                 pz = R[6] * X + R[7] * Y + R[8] * Z + t[2];
    const double iz = 1.0 / pz;
    const double r0 = px * iz - xy[2 * i], r1 = py * iz - xy[2 * i + 1];
    c += r0 * r0 + r1 * r1;
    // J = dpi * [I | -[p]x],  dpi = [iz 0 -px iz^2; 0 iz -py iz^2]
    const double d02 = -px * iz * iz, d12 = -py * iz * iz;
    // rows of dpi * [I | -[p]x] with -[p]x = [0 pz -py; -pz 0 px; py -px 0]
    const double J0[6] = {iz, 0.0, d02, d02 * py, iz * pz - d02 * px, -iz * py};
    const double J1[6] = {0.0, iz, d12, -iz * pz + d12 * py, -d12 * px, iz * px};
    int k = 0;
#pragma unroll
    for (int p = 0; p < 6; ++p) {
#pragma unroll
      for (int q = 0; q <= p; ++q, ++k) a[k] += J0[p] * J0[q] + J1[p] * J1[q];
      g[p] += J0[p] * r0 + J1[p] * r1;
    }
  }
  *cost = wsum(c);
#pragma unroll
  for (int k = 0; k < 21; ++k) JtJ[k] = wsum(a[k]);
#pragma unroll
  for (int k = 0; k < 6; ++k) Jtr[k] = wsum(g[k]);
}

__device__ inline void rodrigues(const double w[3], double R[9]) {
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], th = sqrt(th2);
  const double K[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
  double a, b;
  if (th < 1e-10) { a = 1.0; b = 0.0; }
  else { a = sin(th) / th; b = (1.0 - cos(th)) / th2; }
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      double kk = 0.0;
#pragma unroll
      for (int q = 0; q < 3; ++q) kk += K[i * 3 + q] * K[q * 3 + j];
      R[i * 3 + j] = (i == j ? 1.0 : 0.0) + a * K[i * 3 + j] + b * kk;
    }
}

// rotation matrix -> unit quaternion (x, y, z, w), w >= 0 (same branches as the host-side helper)
__device__ inline void mat_to_quat(const double m[9], double q[4]) {
  const double tr = m[0] + m[4] + m[8];
  if (tr > 0) {
    const double s = sqrt(tr + 1.0) * 2;
    q[0] = (m[7] - m[5]) / s; q[1] = (m[2] - m[6]) / s; q[2] = (m[3] - m[1]) / s; q[3] = 0.25 * s;
  } else if (m[0] > m[4] && m[0] > m[8]) {
    const double s = sqrt(1.0 + m[0] - m[4] - m[8]) * 2;
    q[0] = 0.25 * s; q[1] = (m[1] + m[3]) / s; q[2] = (m[2] + m[6]) / s; q[3] = (m[7] - m[5]) / s;
  } else if (m[4] > m[8]) {
    const double s = sqrt(1.0 + m[4] - m[0] - m[8]) * 2;
    q[0] = (m[1] + m[3]) / s; q[1] = 0.25 * s; q[2] = (m[5] + m[7]) / s; q[3] = (m[2] - m[6]) / s;
  } else {
    const double s = sqrt(1.0 + m[8] - m[0] - m[4]) * 2;
    q[0] = (m[2] + m[6]) / s; q[1] = (m[5] + m[7]) / s; q[2] = 0.25 * s; q[3] = (m[3] - m[1]) / s;
  }
  const double sg = q[3] < 0 ? -1.0 : 1.0;
  const double n = sg / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
#pragma unroll
  for (int k = 0; k < 4; ++k) q[k] *= n;
}

// One view on one warp: cnt correspondences pix [cnt][2] / pw [cnt][3] of a camera of `model` / `intr`, scratch xy
// [cnt][2] / use [cnt]; the RANSAC draws are seeded by (seed, draw).  Writes T_cw [7], *rmse and *n_used.
__device__ __forceinline__ void pose_pnp_view(int seed, int cnt, const double* pix, const double* pw, int model, const double* intr,
                                              int robust_its, double robust_tol, double* xy, unsigned char* use, WarpMem* sm,
                                              int lane, double* T_cw, double* rmse, int32_t* n_used) {
  if (lane == 0) { *n_used = 0; *rmse = 0.0; }
  if (lane < 7) T_cw[lane] = lane == 3 ? 1.0 : 0.0;
  if (cnt < 4) return;
  for (int i = lane; i < cnt; i += 32) {
    unproject(model, intr, pix[2 * i], pix[2 * i + 1], &xy[2 * i], &xy[2 * i + 1]);
    use[i] = 1;
  }
  __syncwarp();
  double H[9];
  int n_use = cnt;
  if (robust_its > 0) {
    double Hbest[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    int best = -1;
    for (int it = 0; it < robust_its; ++it) {
      // 4 distinct indices from a linear congruential sequence seeded by (view, draw): the same on every lane
      int idx[4];
      unsigned s = static_cast<unsigned>(seed) * 2654435761u + static_cast<unsigned>(it) * 40503u + 12345u;
      int got = 0;
      while (got < 4) {
        s = s * 1664525u + 1013904223u;
        const int k = static_cast<int>((s >> 8) % static_cast<unsigned>(cnt));
        bool dup = false;
        for (int q = 0; q < got; ++q) dup = dup || idx[q] == k;
        if (!dup) idx[got++] = k;
      }
      for (int i = lane; i < cnt; i += 32) use[i] = (i == idx[0] || i == idx[1] || i == idx[2] || i == idx[3]) ? 1 : 0;
      __syncwarp();
      homography(pw, xy, use, cnt, sm, lane, H);
      int inl = 0;
      for (int i = lane; i < cnt; i += 32) {
        const double X = pw[3 * i], Y = pw[3 * i + 1];
        const double qz = H[6] * X + H[7] * Y + H[8];
        const double ex = (H[0] * X + H[1] * Y + H[2]) / qz - xy[2 * i], ey = (H[3] * X + H[4] * Y + H[5]) / qz - xy[2 * i + 1];
        inl += sqrt(ex * ex + ey * ey) < robust_tol ? 1 : 0;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) inl += __shfl_xor_sync(0xffffffffu, inl, o);
      if (inl > best) {
        best = inl;
#pragma unroll
        for (int k = 0; k < 9; ++k) Hbest[k] = H[k];
      }
      __syncwarp();
    }
    n_use = 0;
    for (int i = lane; i < cnt; i += 32) {
      const double X = pw[3 * i], Y = pw[3 * i + 1];
      const double qz = Hbest[6] * X + Hbest[7] * Y + Hbest[8];
      const double ex = (Hbest[0] * X + Hbest[1] * Y + Hbest[2]) / qz - xy[2 * i], ey = (Hbest[3] * X + Hbest[4] * Y + Hbest[5]) / qz - xy[2 * i + 1];
      const int ok = sqrt(ex * ex + ey * ey) < robust_tol ? 1 : 0;
      use[i] = static_cast<unsigned char>(ok);
      n_use += ok;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n_use += __shfl_xor_sync(0xffffffffu, n_use, o);
    __syncwarp();
    if (n_use < 4) return;
  }
  homography(pw, xy, use, cnt, sm, lane, H);
  // pose from the homography columns
  double R[9], t[3];
  {
    const double n1 = sqrt(H[0] * H[0] + H[3] * H[3] + H[6] * H[6]), n2 = sqrt(H[1] * H[1] + H[4] * H[4] + H[7] * H[7]);
    const double sc = 2.0 / (n1 + n2);
    double sg = H[8] * sc < 0 ? -1.0 : 1.0;
    double r1[3] = {sg * H[0] / n1, sg * H[3] / n1, sg * H[6] / n1}, r2[3] = {sg * H[1] / n2, sg * H[4] / n2, sg * H[7] / n2};
    t[0] = sg * H[2] * sc; t[1] = sg * H[5] * sc; t[2] = sg * H[8] * sc;
    double r3[3] = {r1[1] * r2[2] - r1[2] * r2[1], r1[2] * r2[0] - r1[0] * r2[2], r1[0] * r2[1] - r1[1] * r2[0]};
    const double n3 = sqrt(r3[0] * r3[0] + r3[1] * r3[1] + r3[2] * r3[2]);
    for (int k = 0; k < 3; ++k) r3[k] /= n3;
    r2[0] = r3[1] * r1[2] - r3[2] * r1[1]; r2[1] = r3[2] * r1[0] - r3[0] * r1[2]; r2[2] = r3[0] * r1[1] - r3[1] * r1[0];
    for (int k = 0; k < 3; ++k) { R[k * 3] = r1[k]; R[k * 3 + 1] = r2[k]; R[k * 3 + 2] = r3[k]; }
  }
  // Levenberg-Marquardt, left perturbation T <- exp(d) T
  double lam = 1e-3, cost, JtJ[21], Jtr[6];
  lm_system(R, t, pw, xy, use, cnt, lane, &cost, JtJ, Jtr);
  for (int it = 0; it < kLmIters; ++it) {
    // (J^T J + lam diag) d = -J^T r : Cholesky in registers (every lane the same)
    double L[21], d[6];
    {
      int k = 0;
#pragma unroll
      for (int p = 0; p < 6; ++p)
#pragma unroll
        for (int q = 0; q <= p; ++q, ++k) L[k] = JtJ[k] * (p == q ? 1.0 + lam : 1.0);
    }
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      double dj = L[j * (j + 1) / 2 + j];
#pragma unroll
      for (int q = 0; q < j; ++q) dj -= L[j * (j + 1) / 2 + q] * L[j * (j + 1) / 2 + q];
      ok = ok && dj > 0.0;
      dj = sqrt(dj > 0.0 ? dj : 1.0);
      L[j * (j + 1) / 2 + j] = dj;
#pragma unroll
      for (int i = j + 1; i < 6; ++i) {
        double s = L[i * (i + 1) / 2 + j];
#pragma unroll
        for (int q = 0; q < j; ++q) s -= L[i * (i + 1) / 2 + q] * L[j * (j + 1) / 2 + q];
        L[i * (i + 1) / 2 + j] = s / dj;
      }
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      double s = -Jtr[i];
#pragma unroll
      for (int q = 0; q < i; ++q) s -= L[i * (i + 1) / 2 + q] * d[q];
      d[i] = s / L[i * (i + 1) / 2 + i];
    }
#pragma unroll
    for (int i = 5; i >= 0; --i) {
      double s = d[i];
#pragma unroll
      for (int q = i + 1; q < 6; ++q) s -= L[q * (q + 1) / 2 + i] * d[q];
      d[i] = s / L[i * (i + 1) / 2 + i];
    }
    double dR[9], R2[9], t2[3], c2, A2[21], g2[6];
    rodrigues(d + 3, dR);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
      for (int j = 0; j < 3; ++j) R2[i * 3 + j] = dR[i * 3] * R[j] + dR[i * 3 + 1] * R[3 + j] + dR[i * 3 + 2] * R[6 + j];
      t2[i] = dR[i * 3] * t[0] + dR[i * 3 + 1] * t[1] + dR[i * 3 + 2] * t[2] + d[i];
    }
    lm_system(R2, t2, pw, xy, use, cnt, lane, &c2, A2, g2);
    if (ok && c2 < cost) {
#pragma unroll
      for (int k = 0; k < 9; ++k) R[k] = R2[k];
#pragma unroll
      for (int k = 0; k < 3; ++k) t[k] = t2[k];
#pragma unroll
      for (int k = 0; k < 21; ++k) JtJ[k] = A2[k];
#pragma unroll
      for (int k = 0; k < 6; ++k) Jtr[k] = g2[k];
      cost = c2;
      lam = fmax(lam * 0.1, 1e-9);
    } else {
      lam = fmin(lam * 10.0, 1e6);
    }
  }
  double q[4];
  mat_to_quat(R, q);
  if (lane < 4) T_cw[lane] = q[lane];
  else if (lane < 7) T_cw[lane] = t[lane - 4];
  if (lane == 0) {
    *n_used = n_use;
    *rmse = sqrt(cost / n_use);
  }
}

// vcgpu_pose_pnp_ransac and its batch: one warp per view of every rig, the views of a rig one after the other and each
// view's correspondences packed behind the previous view's.  A view reads its camera from its rig's table and seeds its
// RANSAC draws with its index within its rig, so a rig's poses do not depend on the rest of the batch.
struct BatchRig {
  int32_t model[kMaxCams];
  double intr[kMaxCams][10];
};
struct BatchView {
  int64_t at;     // first correspondence of the view in pix / pw / xy / use
  int32_t rig;    // index into rigs
  int32_t index;  // the view's index within its rig: the RANSAC seed
  int32_t cam, count;
};
struct BatchArgs {
  int64_t n_views;
  const BatchRig* rigs;
  const BatchView* views;
  const double* pix;   // [N][2]
  const double* pw;    // [N][3]
  int robust_its;
  double robust_tol;
  double* xy;          // [N][2] scratch
  unsigned char* use;  // [N] scratch
  double* T_cw;        // [n_views][7]
  double* rmse;        // [n_views]
  int32_t* n_used;     // [n_views]
};
__global__ void __launch_bounds__(32 * kWarps) pose_pnp_batch_kernel(BatchArgs a) {
  __shared__ WarpMem wm[kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t v = static_cast<int64_t>(blockIdx.x) * kWarps + warp;
  if (v >= a.n_views) return;
  const BatchView w = a.views[v];
  const BatchRig& r = a.rigs[w.rig];
  pose_pnp_view(w.index, w.count, a.pix + 2 * w.at, a.pw + 3 * w.at, r.model[w.cam], r.intr[w.cam], a.robust_its, a.robust_tol,
                a.xy + 2 * w.at, a.use + w.at, &wm[warp], lane, a.T_cw + 7 * v, a.rmse + v, a.n_used + v);
}

}  // namespace pnp
}  // namespace vc
