// Pixel covariance of projected points (vcgpu_get_projection_covariance(_batch)): for a pixel z of camera c and a
// depth d, the ray through z, the point d * ray (or the point at infinity along it), the 2 x (6+K) Jacobian of its
// projection with respect to the camera's globals (w_ck | p_ck | intrinsics) and Sigma_z = J Sigma_c J^T, Sigma_c the
// camera's diagonal block of vcgpu_get_covariance's matrix.  One thread per point; a CTA takes 256 consecutive points
// of one rig and stages that rig's camera blocks and camera states in shared memory.
//
// Unprojection (Cam<MODEL>::project inverted at the current intrinsics; x_d = ((u - u0) / fu, (v - v0) / fv), r_d = |x_d|):
//   linear   ray ~ (x_d, 1).
//   FOV      w^2 <= 1e-5: ray ~ (x_d, 1).  Otherwise, m = 2 tan(w / 2): where the undistorted radius r_d w / m of the
//            small-rad branch has r^2 < 1e-5, that branch (f = m / w); else r = tan(r_d w) / m, which needs
//            r_d |w| < pi / 2.  ray ~ (x_d / f, 1), f = r_d / r.
//   poly     r f(r) = r_d, f = 1 + k1 r^2 + k2 r^4 (+ k3 r^6), on [0, r_fold), r_fold the first zero of
//            (r f(r))' = 1 + 3 k1 r^2 + 5 k2 r^4 (+ 7 k3 r^6).  ray ~ (x_d / f(r), 1).
//   KB4      theta (1 + k0 theta^2 + ... + k3 theta^8) = r_d on [0, theta_max), theta_max = min(pi, the first zero of
//            the left side's derivative).  ray = (sin theta x_d / r_d, cos theta): beyond 90 degrees it points behind the
//            image plane.
// The folds are the first zeros of polynomials in s = r^2 (theta^2), found per camera by proj_first_zero.  A pixel whose
// radius is not below the image of its model's limit is outside the domain.  Newton starts at r = r_d (theta = r_d) and
// takes at most kProjNewtonIters steps; it has converged where the image radius matches r_d to kProjImageTol (near a fold
// rounding keeps the steps above the step test), or after a step |dr| <= kProjNewtonTol * r.  Every derivative it
// divides by must be positive and every iterate must stay in [0, limit).  A pixel outside the domain, or one where Newton
// fails, gets NaN in every output.
#pragma once
#include "vc_internal.h"
#include "vc_math.cuh"

namespace vc {

constexpr int kProjThreads = 256;
constexpr int kProjNewtonIters = 50;
constexpr double kProjNewtonTol = 1e-14;  // a step |dr| <= kProjNewtonTol * r ends the iteration
constexpr double kProjImageTol = 1e-15;   // so does |r f(r) - r_d| <= kProjImageTol * r_d, before the step
constexpr int kProjMaxN = 6 + 8;  // globals of one camera

// one rig of a launch: its points are tiles [tile0, tile0 + ceil(n / kProjThreads))
struct ProjRig {
  const double* S;      // [G][G] row-major: vcgpu_get_covariance's matrix
  const double* cams;   // [n_cams][kCamStateStride] the accepted state's cameras: q_ck 4 | p_ck 3 | intrinsics
  const int32_t* cam;   // [n]
  const double* pix;    // [n][2]
  const double* depth;  // [n], or null: every point at infinity
  double* cov;          // [n][3] S_uu, S_uv, S_vv
  double* ray;          // [n][3]
  int64_t n, tile0;
  int G, n_cams, rig_frame;
  int model[kMaxCams], goff[kMaxCams];
};

__device__ __forceinline__ double proj_peval(const double* c, int n, double s) {
  double v = c[n];
  for (int i = n - 1; i >= 0; --i) v = v * s + c[i];
  return v;
}
// the zeros of the degree-N polynomial c in (0, S), ascending, into z; their count.  Between consecutive zeros of the
// derivative the polynomial is monotone, so each such piece holds at most one zero, which bisection narrows to adjacent
// doubles (z gets the end nearer 0).
template <int N>
__device__ int proj_zeros(const double* c, double S, double* z) {
  if constexpr (N == 1) {
    if (c[1] == 0.0) return 0;
    const double s = -c[0] / c[1];
    z[0] = s;
    return s > 0.0 && s < S ? 1 : 0;
  } else {
    double d[N], k[N + 1];
    for (int i = 0; i < N; ++i) d[i] = (i + 1) * c[i + 1];
    const int m = proj_zeros<N - 1>(d, S, k + 1);
    k[0] = 0.0;
    k[m + 1] = S;
    int nz = 0;
    for (int p = 0; p <= m; ++p) {
      double lo = k[p], hi = k[p + 1];
      const double flo = proj_peval(c, N, lo), fhi = proj_peval(c, N, hi);
      if (fhi == 0.0 && p < m) { z[nz++] = hi; continue; }
      if (!((flo < 0.0 && fhi > 0.0) || (flo > 0.0 && fhi < 0.0))) continue;
      for (int it = 0; it < 2100; ++it) {
        const double mid = 0.5 * (lo + hi);
        if (!(mid > lo && mid < hi)) break;
        if ((proj_peval(c, N, mid) > 0.0) == (flo > 0.0)) lo = mid;
        else hi = mid;
      }
      z[nz++] = lo;
    }
    return nz;
  }
}
// the first zero in (0, S) of a polynomial with c[0] = 1, or S where it has none
template <int N>
__device__ double proj_first_zero(const double* c, double S) {
  double z[N];
  return proj_zeros<N>(c, S, z) > 0 ? z[0] : S;
}

// the per-camera limit of the radial models: poly r_fold^2, KB4 theta_max (infinite: no limit)
template <int MODEL>
__device__ double proj_limit(const double* in) {
  if constexpr (MODEL == kPoly2 || MODEL == kPoly3) {
    constexpr int N = MODEL == kPoly2 ? 2 : 3;
    const double c[4] = {1.0, 3.0 * in[4], 5.0 * in[5], N == 3 ? 7.0 * in[6] : 0.0};
    // every zero lies below the Cauchy bound of the polynomial's effective degree
    int deg = N;
    while (deg > 0 && c[deg] == 0.0) --deg;
    if (deg == 0) return INFINITY;
    double b = 0.0;
    for (int i = 0; i < deg; ++i) b = fmax(b, fabs(c[i] / c[deg]));
    const double S = 2.0 * (1.0 + b);
    const double s = proj_first_zero<N>(c, S);
    return s < S ? s : INFINITY;
  } else if constexpr (MODEL == kKb4) {
    const double c[5] = {1.0, 3.0 * in[4], 5.0 * in[5], 7.0 * in[6], 9.0 * in[7]};
    const double S = M_PI * M_PI;
    const double s = proj_first_zero<4>(c, S);
    return s < S ? sqrt(s) : M_PI;
  } else {
    return INFINITY;
  }
}

// r (poly) or theta (KB4) with image r_d: Newton as the header describes; false outside the domain
template <int MODEL>
__device__ bool proj_radius(const double* in, double lim, double rd, double* out) {
  constexpr bool kb = MODEL == kKb4;
  const double k1 = in[4], k2 = in[5], k3 = MODEL == kPoly2 ? 0.0 : in[6], k4 = kb ? in[7] : 0.0;
  // image radius and its derivative
  auto img = [&](double r, double* d) {
    const double s = r * r;
    if (kb) {
      *d = 1.0 + s * (3.0 * k1 + s * (5.0 * k2 + s * (7.0 * k3 + s * 9.0 * k4)));
      return r * (1.0 + s * (k1 + s * (k2 + s * (k3 + s * k4))));
    }
    *d = 1.0 + s * (3.0 * k1 + s * (5.0 * k2 + s * 7.0 * k3));
    return r * (1.0 + s * (k1 + s * (k2 + s * k3)));
  };
  // in r: poly's limit is r_fold^2
  const double rmax = kb ? lim : sqrt(lim);
  double dd;
  if (rmax < INFINITY && !(rd < img(rmax, &dd))) return false;
  double r = rd;
  for (int it = 0; it < kProjNewtonIters; ++it) {
    const double g = img(r, &dd) - rd;
    if (!(dd > 0.0)) return false;
    if (fabs(g) <= kProjImageTol * rd) {
      *out = r;
      return true;
    }
    const double step = g / dd;
    r -= step;
    if (!(r >= 0.0 && r < rmax)) return false;
    if (fabs(step) <= kProjNewtonTol * r) {
      *out = r;
      return true;
    }
  }
  return false;
}

// the unit ray whose projection is the pixel (px, py); false outside the model's domain
template <int MODEL>
__device__ bool proj_unproject(const double* in, double lim, double px, double py, V3* ray) {
  const double xd = (px - in[2]) / in[0], yd = (py - in[3]) / in[1];
  const double rd = sqrt(xd * xd + yd * yd);
  V3 p{xd, yd, 1.0};
  if constexpr (MODEL == kFov) {
    const double w = in[4];
    if (w * w > 1e-5) {
      const double m = 2.0 * tan(0.5 * w), fs = m / w, rs = rd / fs;
      double f = fs;
      if (!(rs * rs < 1e-5)) {
        if (!(rd * fabs(w) < 0.5 * M_PI)) return false;
        f = rd / (tan(rd * w) / m);
      }
      p = V3{xd / f, yd / f, 1.0};
    }
  } else if constexpr (MODEL == kPoly2 || MODEL == kPoly3) {
    double r;
    if (!proj_radius<MODEL>(in, lim, rd, &r)) return false;
    const double s = r * r, k3 = MODEL == kPoly3 ? in[6] : 0.0;
    const double f = 1.0 + s * (in[4] + s * (in[5] + s * k3));
    p = V3{xd / f, yd / f, 1.0};
  } else if constexpr (MODEL == kKb4) {
    double th;
    if (!proj_radius<MODEL>(in, lim, rd, &th)) return false;
    double sn, cs;
    sincos(th, &sn, &cs);
    *ray = rd > 0.0 ? V3{sn * xd / rd, sn * yd / rd, cs} : V3{0.0, 0.0, 1.0};
    return true;
  }
  if (!(fabs(p.x) < INFINITY && fabs(p.y) < INFINITY)) return false;
  *ray = p * (1.0 / sqrt(dot(p, p)));
  return true;
}

// one point: its ray, then J and Sigma_z = J Sigma_c J^T with the products in a fixed order
template <int MODEL>
__device__ void proj_point(const double* cs, const double* Sc, double lim, bool rig_frame, double px, double py, double d,
                           double out_cov[3], double out_ray[3]) {
  constexpr int K = Cam<MODEL>::K, N = 6 + K;
  const double* in = cs + 7;
  V3 ray;
  if (!proj_unproject<MODEL>(in, lim, px, py, &ray)) {
    for (int k = 0; k < 3; ++k) out_cov[k] = out_ray[k] = NAN;
    return;
  }
  out_ray[0] = ray.x; out_ray[1] = ray.y; out_ray[2] = ray.z;
  const bool inf = !(d > 0.0);
  const V3 pc = inf ? ray : ray * d;
  double z[2], dzp[6], dzi[2 * K], J[2][N];
  Cam<MODEL>::project(pc, in, z, dzp, dzi);
  double R[9];
  qmat(Q4{cs[0], cs[1], cs[2], cs[3]}, R);
  // the point in the rig frame; at infinity its direction, whose scale cancels against dz/dp_c's
  const V3 pk = mat_tmul(R, inf ? ray : pc - V3{cs[4], cs[5], cs[6]});
#pragma unroll
  for (int row = 0; row < 2; ++row) {
    const double* dp = dzp + 3 * row;
    // eval_reproj_kernel's w_ck and p_ck columns
    const double m0 = dp[0] * R[0] + dp[1] * R[3] + dp[2] * R[6];
    const double m1 = dp[0] * R[1] + dp[1] * R[4] + dp[2] * R[7];
    const double m2 = dp[0] * R[2] + dp[1] * R[5] + dp[2] * R[8];
    const double w0 = m1 * pk.z - m2 * pk.y;
    const double w1 = m2 * pk.x - m0 * pk.z;
    const double w2 = m0 * pk.y - m1 * pk.x;
    const bool pose = rig_frame, trans = rig_frame && !inf;
    J[row][0] = pose ? -w0 : 0.0;
    J[row][1] = pose ? -w1 : 0.0;
    J[row][2] = pose ? -w2 : 0.0;
    J[row][3] = trans ? dp[0] : 0.0;
    J[row][4] = trans ? dp[1] : 0.0;
    J[row][5] = trans ? dp[2] : 0.0;
#pragma unroll
    for (int k = 0; k < K; ++k) J[row][6 + k] = dzi[row * K + k];
  }
  // t = Sigma_c J^T row by row (j ascending), then S_ab = sum_i J_a[i] t_b[i] (i ascending)
  double suu = 0.0, suv = 0.0, svv = 0.0;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    double tu = 0.0, tv = 0.0;
#pragma unroll
    for (int j = 0; j < N; ++j) {
      tu = fma(Sc[i * N + j], J[0][j], tu);
      tv = fma(Sc[i * N + j], J[1][j], tv);
    }
    suu = fma(J[0][i], tu, suu);
    suv = fma(J[0][i], tv, suv);
    svv = fma(J[1][i], tv, svv);
  }
  out_cov[0] = suu; out_cov[1] = suv; out_cov[2] = svv;
}

// One CTA per tile of kProjThreads consecutive points of one rig: rigs[r] owns tiles [tile0, next rig's tile0).
__global__ void __launch_bounds__(kProjThreads) proj_cov_kernel(const ProjRig* __restrict__ rigs, int n_rigs) {
  __shared__ double Sc[kMaxCams][kProjMaxN * kProjMaxN];
  __shared__ double cs[kMaxCams][kCamStateStride];
  __shared__ double lim[kMaxCams];
  int lo = 0, hi = n_rigs - 1;  // the last rig whose tile0 <= blockIdx.x
  while (lo < hi) {
    const int mid = (lo + hi + 1) / 2;
    if (rigs[mid].tile0 <= blockIdx.x) lo = mid;
    else hi = mid - 1;
  }
  const ProjRig& a = rigs[lo];
  const int nc = a.n_cams;
  for (int e = threadIdx.x; e < nc * kProjMaxN * kProjMaxN; e += blockDim.x) {
    const int c = e / (kProjMaxN * kProjMaxN), ij = e % (kProjMaxN * kProjMaxN), N = 6 + num_intr(a.model[c]);
    if (ij < N * N) Sc[c][ij] = a.S[static_cast<int64_t>(a.goff[c] + ij / N) * a.G + a.goff[c] + ij % N];
  }
  for (int e = threadIdx.x; e < nc * kCamStateStride; e += blockDim.x) cs[e / kCamStateStride][e % kCamStateStride] = a.cams[e];
  __syncthreads();
  if (threadIdx.x < nc) {
    const double* in = cs[threadIdx.x] + 7;
    const int m = a.model[threadIdx.x];
    lim[threadIdx.x] = m == kPoly2 ? proj_limit<kPoly2>(in) : m == kPoly3 ? proj_limit<kPoly3>(in) : m == kKb4 ? proj_limit<kKb4>(in) : INFINITY;
  }
  __syncthreads();
  const int64_t i = (blockIdx.x - a.tile0) * static_cast<int64_t>(kProjThreads) + threadIdx.x;
  if (i >= a.n) return;
  const int c = a.cam[i];
  const double px = a.pix[2 * i], py = a.pix[2 * i + 1], d = a.depth ? a.depth[i] : 0.0;
  double cov[3], ray[3];
  switch (a.model[c]) {
    case kLinear: proj_point<kLinear>(cs[c], Sc[c], lim[c], a.rig_frame, px, py, d, cov, ray); break;
    case kFov: proj_point<kFov>(cs[c], Sc[c], lim[c], a.rig_frame, px, py, d, cov, ray); break;
    case kPoly2: proj_point<kPoly2>(cs[c], Sc[c], lim[c], a.rig_frame, px, py, d, cov, ray); break;
    case kPoly3: proj_point<kPoly3>(cs[c], Sc[c], lim[c], a.rig_frame, px, py, d, cov, ray); break;
    default: proj_point<kKb4>(cs[c], Sc[c], lim[c], a.rig_frame, px, py, d, cov, ray); break;
  }
  for (int k = 0; k < 3; ++k) a.cov[3 * i + k] = cov[k];
  if (a.ray)
    for (int k = 0; k < 3; ++k) a.ray[3 * i + k] = ray[k];
}

}  // namespace vc
