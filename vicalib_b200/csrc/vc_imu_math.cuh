// Device-side IMU residual math: RK4 integration of (p, q, v) through interpolated gyro / accel
// samples, the SE3 log residual, a one-direction dual number for the tangent directions that reach the
// attitude, and the (p, v)-only tangents that ride along the same chain in plain doubles (AccelTangent).
//
// Reference being reproduced:
//   SwitchedFullImuCostFunction::operator()   ceres-cost-functions.h:402-484
//   IntegratePoseJet / GetPoseDerivativeJet / IntegrateImuJet / IntegrateResidualJet
//                                             ceres-cost-functions.h:38-56, 79-105, 138-177, 199-227
//   InterpolationBufferT::{GetRange,GetElement,GetNext,HasElement,InterpolateElements}
//                                             interpolation-buffer.h:100-117,122-125,136-155,160-203,208-226
//   GetGravityVector                          types.h:93-104
// The reference differentiates with ceres::Jet<double,35> in ambient coordinates and multiplies by
// LocalParamSe3::ComputeJacobian (local-param-se3.h:28-91); seeding a 1-wide dual with the matching
// column of that matrix gives the same tangent-space derivative directly.
#pragma once
#include "vc_math.cuh"

namespace vc {
namespace imu {

struct D1 {  // value + derivative along this lane's direction
  double a, v;
  __host__ __device__ D1() : a(0.0), v(0.0) {}
  __host__ __device__ D1(double s) : a(s), v(0.0) {}  // NOLINT
  __host__ __device__ D1(double s, double d) : a(s), v(d) {}
};
__device__ __forceinline__ D1 operator+(D1 x, D1 y) { return {x.a + y.a, x.v + y.v}; }
__device__ __forceinline__ D1 operator-(D1 x, D1 y) { return {x.a - y.a, x.v - y.v}; }
__device__ __forceinline__ D1 operator-(D1 x) { return {-x.a, -x.v}; }
__device__ __forceinline__ D1 operator*(D1 x, D1 y) { return {x.a * y.a, x.a * y.v + x.v * y.a}; }
__device__ __forceinline__ D1 operator/(D1 x, D1 y) {
  const double inv = 1.0 / y.a, q = x.a * inv;
  return {q, (x.v - q * y.v) * inv};
}
__device__ __forceinline__ D1 dsqrt(D1 x) { const double s = sqrt(x.a); return {s, 0.5 * x.v / s}; }
__device__ __forceinline__ double dsqrt(double x) { return sqrt(x); }
__device__ __forceinline__ void dsincos(D1 x, D1* s, D1* c) {
  double sn, cs;
  sincos(x.a, &sn, &cs);
  *s = {sn, cs * x.v};
  *c = {cs, -sn * x.v};
}
__device__ __forceinline__ void dsincos(double x, double* s, double* c) { sincos(x, s, c); }
__device__ __forceinline__ D1 dtan(D1 x) { const double t = tan(x.a); return {t, (1.0 + t * t) * x.v}; }
__device__ __forceinline__ double dtan(double x) { return tan(x); }
__device__ __forceinline__ D1 datan(D1 x) { return {atan(x.a), x.v / (1.0 + x.a * x.a)}; }
__device__ __forceinline__ double datan(double x) { return atan(x); }
__device__ __forceinline__ double val(D1 x) { return x.a; }
__device__ __forceinline__ double val(double x) { return x; }

template <class T> struct Vec { T x, y, z; };
template <class T> struct Quat { T x, y, z, w; };

template <class T> __device__ __forceinline__ Vec<T> operator+(Vec<T> a, Vec<T> b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
template <class T> __device__ __forceinline__ Vec<T> operator-(Vec<T> a, Vec<T> b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
template <class T> __device__ __forceinline__ Vec<T> scale(Vec<T> a, T s) { return {a.x * s, a.y * s, a.z * s}; }
template <class T> __device__ __forceinline__ Vec<T> cross(Vec<T> a, Vec<T> b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
template <class T> __device__ __forceinline__ T dot(Vec<T> a, Vec<T> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

template <class T> __device__ __forceinline__ Quat<T> qmul(Quat<T> a, Quat<T> b) {
  return {a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
          a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
template <class T> __device__ __forceinline__ Quat<T> qconj(Quat<T> q) { return {-q.x, -q.y, -q.z, q.w}; }
// rotate by a (unit) quaternion: v + w*uv + q.vec x uv, uv = 2 q.vec x v  (== R(q) v; the reference
// uses both so3().Adj()*v and so3()*v, ceres-cost-functions.h:98,101 — identical on unit quaternions)
template <class T> __device__ __forceinline__ Vec<T> qrot(Quat<T> q, Vec<T> v) {
  const Vec<T> qv{q.x, q.y, q.z};
  Vec<T> uv = cross(qv, v);
  uv = uv + uv;
  return v + scale(uv, q.w) + cross(qv, uv);
}

// Sophus SO3::exp: imag = sin(theta/2)/theta, real = cos(theta/2).  Below theta^2 = 1e-3 both are evaluated by their
// Taylor series to theta^8 / theta^10 (truncation < 1e-25 relative, i.e. the same double as the closed form): an IMU
// sub-step rotates by milliradians, and the series needs no square root, sine / cosine or division — which matters
// most when T is a dual number.  Sophus' own theta < 1e-10 branch is the first two terms of the same series.
template <class T> __device__ inline Quat<T> so3_exp(Vec<T> om) {
  const T th2 = dot(om, om);
  T imag, real;
  if (val(th2) < 1e-3) {
    imag = T(0.5) + th2 * (T(-1.0 / 48.0) + th2 * (T(1.0 / 3840.0) + th2 * (T(-1.0 / 645120.0) + th2 * T(1.0 / 185794560.0))));
    real = T(1.0) + th2 * (T(-1.0 / 8.0) + th2 * (T(1.0 / 384.0) + th2 * (T(-1.0 / 46080.0) + th2 * (T(1.0 / 10321920.0) +
                                                                                                   th2 * T(-1.0 / 3715891200.0)))));
  } else {
    const T th = dsqrt(th2);
    T s, c;
    dsincos(th * T(0.5), &s, &c);
    imag = s / th;
    real = c;
  }
  return {imag * om.x, imag * om.y, imag * om.z, real};
}
// Sophus SO3::logAndTheta
template <class T> __device__ inline Vec<T> so3_log(Quat<T> q, T* theta) {
  const T n2 = q.x * q.x + q.y * q.y + q.z * q.z;
  T f, n = T(0.0);
  if (val(n2) < kSophusEps * kSophusEps) {
    f = T(2.0) / q.w - T(2.0) * n2 / (q.w * q.w * q.w);
    if (val(n2) > 0.0) n = dsqrt(n2);
  } else {
    n = dsqrt(n2);
    if (fabs(val(q.w)) < kSophusEps) f = T(val(q.w) > 0.0 ? M_PI : -M_PI) / n;
    else f = T(2.0) * datan(n / q.w) / n;
  }
  *theta = f * n;
  return {f * q.x, f * q.y, f * q.z};
}
// Sophus SE3::log of (q, t): out = (upsilon, omega), upsilon = V^-1 t
template <class T> __device__ inline void se3_log(Quat<T> q, Vec<T> t, T out[6]) {
  T th;
  const Vec<T> om = so3_log(q, &th);
  T c;
  if (fabs(val(th)) < kSophusEps) c = T(1.0 / 12.0);
  else c = (T(1.0) - th / (T(2.0) * dtan(th * T(0.5)))) / (th * th);
  const Vec<T> ot = cross(om, t);
  const Vec<T> oot = cross(om, ot);
  const Vec<T> u = t - scale(ot, T(0.5)) + scale(oot, c);
  out[0] = u.x; out[1] = u.y; out[2] = u.z;
  out[3] = om.x; out[4] = om.y; out[5] = om.z;
}

// IMU sample buffer on the device: SoA [7][n] = t, w3, a3  (+ the reference's running statistics)
struct ImuBuf {
  const double* d;  // base; channel c at d + c*n
  int n;
  double start_time, end_time, average_dt;
};
template <class T> struct Meas { Vec<T> w, a; T time; };

template <class T> __device__ __forceinline__ Meas<T> load_meas(const ImuBuf& b, int i) {
  const int64_t n = b.n;
  return {{T(b.d[n + i]), T(b.d[2 * n + i]), T(b.d[3 * n + i])},
          {T(b.d[4 * n + i]), T(b.d[5 * n + i]), T(b.d[6 * n + i])}, T(b.d[i])};
}
// interpolation-buffer.h:136-155
template <class T> __device__ inline Meas<T> interpolate(const ImuBuf& b, int ai, int bi, T ts, double time) {
  const Meas<T> ma = load_meas<T>(b, ai), mb = load_meas<T>(b, bi);
  const T t_a = ma.time + ts, t_b = mb.time + ts, t_out = T(time);
  const T fr = (t_out - t_a) / (t_b - t_a), omf = T(1.0) - fr;
  return {scale(ma.w, omf) + scale(mb.w, fr), scale(ma.a, omf) + scale(mb.a, fr), t_out};
}
// interpolation-buffer.h:160-203 (index logic on the scalar part of ts only)
template <class T> __device__ inline Meas<T> get_element(const ImuBuf& b, double time, T ts, int* idx) {
  const double off = val(ts);
  const int n = b.n;
  double gd = (time - b.start_time + off) / b.average_dt;
  if (!(gd > 0.0)) gd = 0.0;
  int guess = gd >= static_cast<double>(n) ? n - 1 : static_cast<int>(gd);
  guess = min(guess, n - 1);
  Meas<T> r;
  if (b.d[guess] + off > time) {
    if (guess == 0) {
      r = load_meas<T>(b, 0);
      r.time = r.time + ts;
      *idx = 0;
    } else {
      while ((guess - 1) > 0 && b.d[guess - 1] + off > time) --guess;
      r = interpolate<T>(b, guess - 1, guess, ts, time);
      *idx = guess - 1;
    }
  } else {
    if (guess == n - 1) {
      *idx = guess;
      r = load_meas<T>(b, n - 1);
      r.time = r.time + ts;
    } else {
      while ((guess + 1) < n && (b.d[guess + 1] + off) < time) ++guess;
      r = interpolate<T>(b, guess, guess + 1, ts, time);
      *idx = guess;
    }
  }
  return r;
}
// interpolation-buffer.h:100-117
template <class T> __device__ inline bool get_next(const ImuBuf& b, double max_time, T ts, int* idx, Meas<T>* out) {
  if (*idx + 1 >= b.n || b.d[*idx + 1] + val(ts) > max_time) {
    *out = get_element<T>(b, max_time, ts, idx);
    return false;
  }
  *out = load_meas<T>(b, ++*idx);
  out->time = out->time + ts;
  return true;
}

template <class T> struct Pose { Vec<T> p; Quat<T> q; Vec<T> v; };

// ceres-cost-functions.h:38-56
template <class T> __device__ inline Pose<T> integrate_pose(const Pose<T>& y0, const T k[9], T dt) {
  const Quat<T> dq = so3_exp(Vec<T>{k[3] * dt, k[4] * dt, k[5] * dt});
  Pose<T> y;
  y.p = y0.p + Vec<T>{k[0] * dt, k[1] * dt, k[2] * dt};
  y.q = qmul(dq, y0.q);  // left-multiplied, no renormalisation (:47-51)
  y.v = y0.v + Vec<T>{k[6] * dt, k[7] * dt, k[8] * dt};
  return y;
}
// ceres-cost-functions.h:79-105
template <class T> __device__ inline void pose_derivative(const Pose<T>& y, Vec<T> g, const Meas<T>& z0, const Meas<T>& z1,
                                                          Vec<T> bg, Vec<T> ba, const T sf[6], T dt, T k[9],
                                                          Vec<T>* za_out = nullptr) {
  const T alpha = (z1.time - (z0.time + dt)) / (z1.time - z0.time), oma = T(1.0) - alpha;
  const Vec<T> zg = scale(z0.w, alpha) + scale(z1.w, oma);
  const Vec<T> za = scale(z0.a, alpha) + scale(z1.a, oma);
  if (za_out) *za_out = za;
  k[0] = y.v.x; k[1] = y.v.y; k[2] = y.v.z;
  const Vec<T> w = qrot(y.q, Vec<T>{zg.x * sf[0] + bg.x, zg.y * sf[1] + bg.y, zg.z * sf[2] + bg.z});
  k[3] = w.x; k[4] = w.y; k[5] = w.z;
  const Vec<T> a = qrot(y.q, Vec<T>{za.x * sf[3] + ba.x, za.y * sf[4] + ba.y, za.z * sf[5] + ba.z}) - g;
  k[6] = a.x; k[7] = a.y; k[8] = a.z;
}
// A (p, v)-only tangent carried beside the RK4 chain in plain doubles.  k[3..8] depend on q and the measurements but
// never on p or v, so a direction that moves neither q, the gyro terms nor the sample times (pose1 translation, v1,
// gravity, accelerometer bias and scale) never reaches q: along it k_v moves by R(q_s) du_s - dg at stage s, with
// du_s = (fb + fz za_s[ax]) e_ax the derivative of the accelerometer term, and k_p by the velocity tangent.  This
// accumulates the accelerometer part along the attitude path the chain integrates (RK4 per step:
// dv += dt/6 (b1 + 2 b2 + 2 b3 + b4), dp += dt dv + dt^2/6 (b1 + b2 + b3)) and the integrated time `dur`; the seeds'
// own part is linear in it (dp0 + dur dv0 - dur^2/2 dg, dv0 - dur dg) and is added by the caller.
struct AccelTangent {
  int ax;          // du = (fb + fz za[ax]) e_ax
  double fb, fz;
  double dur = 0.0;
  Vec<double> dp{0.0, 0.0, 0.0}, dv{0.0, 0.0, 0.0};
  Vec<double> b3, b6;  // b1 + b2 + b3 and b1 + 2 b2 + 2 b3 + b4 of the current step
  template <class T_>
  __device__ __forceinline__ void stage(int s, const Quat<T_>& q, const Vec<T_>& za) {
    const double u = fb + fz * (ax == 0 ? val(za.x) : ax == 1 ? val(za.y) : val(za.z));
    const Vec<double> b = qrot(Quat<double>{val(q.x), val(q.y), val(q.z), val(q.w)},
                               Vec<double>{ax == 0 ? u : 0.0, ax == 1 ? u : 0.0, ax == 2 ? u : 0.0});
    if (s == 0) {
      b3 = b;
      b6 = b;
    } else if (s < 3) {
      b3 = b3 + b;
      b6 = b6 + scale(b, 2.0);
    } else {
      b6 = b6 + b;
    }
  }
  __device__ __forceinline__ void step(double dt) {
    dp = dp + scale(dv, dt) + scale(b3, dt * dt / 6.0);
    dv = dv + scale(b6, dt / 6.0);
    dur += dt;
  }
};

// ceres-cost-functions.h:138-177 (RK4); `at` follows an AccelTangent along the step.  w_out (null: not asked for)
// receives k.segment<3>(3) of the unnormalised sum k1 + 2 k2 + 2 k3 + k4, the w_w_ of types.h:592; a zero-length step
// leaves it untouched, as the reference leaves the whole pose.
template <class T, class AT>
__device__ inline Pose<T> integrate_imu(const Pose<T>& y0, const Meas<T>& z0, const Meas<T>& z1, Vec<T> bg, Vec<T> ba,
                                        const T sf[6], Vec<T> g, AT& at, Vec<T>* w_out = nullptr) {
  if (val(z1.time) == val(z0.time)) return y0;
  const T dt = z1.time - z0.time;
  T k1[9], k2[9], k3[9], k4[9];
  Vec<T> za;
  pose_derivative(y0, g, z0, z1, bg, ba, sf, T(0.0), k1, &za);
  at.stage(0, y0.q, za);
  const Pose<T> y1 = integrate_pose(y0, k1, dt * T(0.5));
  pose_derivative(y1, g, z0, z1, bg, ba, sf, dt / T(2.0), k2, &za);
  at.stage(1, y1.q, za);
  const Pose<T> y2 = integrate_pose(y0, k2, dt * T(0.5));
  pose_derivative(y2, g, z0, z1, bg, ba, sf, dt / T(2.0), k3, &za);
  at.stage(2, y2.q, za);
  const Pose<T> y3 = integrate_pose(y0, k3, dt);
  pose_derivative(y3, g, z0, z1, bg, ba, sf, dt, k4, &za);
  at.stage(3, y3.q, za);
  at.step(val(dt));
#pragma unroll
  for (int i = 0; i < 9; ++i) k1[i] = k1[i] + T(2.0) * k2[i] + T(2.0) * k3[i] + k4[i];
  if (w_out) *w_out = Vec<T>{k1[3], k1[4], k1[5]};
  return integrate_pose(y0, k1, dt / T(6.0));
}

// types.h:93-104
template <class T> __device__ inline Vec<T> gravity_vector(T p, T q) {
  T sp, cp, sq, cq;
  dsincos(p, &sp, &cp);
  dsincos(q, &sq, &cq);
  const T mg = T(-9.8007);
  return {cp * sq * mg, -sp * mg, cp * cq * mg};
}

// The pose and velocity at t_end integrated from (x1, v1) at t_start (ceres-cost-functions.h:440-470); returns false
// when the interval has no measurements (:452-455).  `at` follows an AccelTangent along the way.
template <class T, class AT>
__device__ inline bool imu_integrate(const ImuBuf& buf, double t_start, double t_end, const T x1[7], const T v1[3],
                                     const T g2[2], const T b[6], const T sf[6], T ts, Pose<T>* end, AT& at) {
  // HasElement (interpolation-buffer.h:122-125)
  if (!(t_start >= buf.start_time + val(ts) && t_start <= buf.end_time + val(ts)) || buf.n == 0) return false;
  const Vec<T> g = gravity_vector<T>(g2[0], g2[1]);
  const Vec<T> bg{b[0], b[1], b[2]}, ba{b[3], b[4], b[5]};
  Pose<T> y{{x1[4], x1[5], x1[6]}, {x1[0], x1[1], x1[2], x1[3]}, {v1[0], v1[1], v1[2]}};
  int idx;
  Meas<T> prev = get_element<T>(buf, t_start, ts, &idx), cur;
  bool more = true;
  while (more) {
    more = get_next<T>(buf, t_end, ts, &idx, &cur);
    y = integrate_imu(y, prev, cur, bg, ba, sf, g, at);
    prev = cur;
  }
  *end = y;
  return true;
}

// Unweighted residual of the integrated end state y: (log(T_end * T_2^-1), v_end - v2)
template <class T>
__device__ inline void imu_end_residual(const Pose<T>& y, const T x2[7], const T v2[3], T r[9]) {
  // T_end * T_2^-1
  const Quat<T> q2i = qconj(Quat<T>{x2[0], x2[1], x2[2], x2[3]});
  const Vec<T> t2i = qrot(q2i, Vec<T>{x2[4], x2[5], x2[6]});
  const Quat<T> qe = qmul(y.q, q2i);
  const Vec<T> te = y.p - qrot(y.q, t2i);
  se3_log(qe, te, r);
  r[6] = y.v.x - v2[0];
  r[7] = y.v.y - v2[1];
  r[8] = y.v.z - v2[2];
}

}  // namespace imu
}  // namespace vc
