// TEST INFRASTRUCTURE ONLY: flat C entry points over the oracle's restatement of UpdateImuWeights
// (oracle/imu_weights.h), for tests/imu_mahalanobis_ref.py, which compiles this file into a temporary directory.
//   vo_imu_mahalanobis  UpdateOneImuWeight's `mahalanobis` output for every interval (vicalibrator.h:786-794)
//   vo_imu_interval     one interval's P = Jt C Jt^T (9 x 9) and residual r (9) as the loop body forms them
//                       (vicalibrator.h:755-788), for the numpy model of the device formula
#include <cmath>
#include <limits>

#include "imu_weights.h"

using namespace vo;  // NOLINT

namespace {

InterpolationBuffer make_buffer(int n, const double* t, const double* w, const double* a) {
  InterpolationBuffer buf;
  for (int i = 0; i < n; ++i)
    buf.AddElement({{w[3 * i], w[3 * i + 1], w[3 * i + 2]}, {a[3 * i], a[3 * i + 1], a[3 * i + 2]}, t[i]});
  return buf;
}

}  // namespace

extern "C" {

// dist[k], k < nf - 1: NaN where the interval has no measurements (the reference logs nothing there) or P is singular
void vo_imu_mahalanobis(int n, const double* t, const double* w, const double* a, int nf, const double* ftime,
                        const double* T_wp, const double* v_w, const double* g, const double* b, const double* sf,
                        double ts, double sigma_g, double sigma_a, double* dist) {
  const InterpolationBuffer buf = make_buffer(n, t, w, a);
  for (int k = 0; k + 1 < nf; ++k) {
    double W[81];
    dist[k] = std::numeric_limits<double>::quiet_NaN();
    UpdateOneImuWeight(buf, ftime[k], ftime[k + 1], ts, T_wp + 7 * k, v_w + 3 * k, T_wp + 7 * (k + 1),
                       v_w + 3 * (k + 1), b, sf, g, sigma_g, sigma_a, W, dist + k);
  }
}

// Returns the number of measurements GetRange yields (0: nothing written)
int vo_imu_interval(int n, const double* t, const double* w, const double* a, double t_start, double t_end,
                    const double* T_w1, const double* v1, const double* T_w2, const double* v2, const double* g,
                    const double* b, const double* sf, double ts, double sigma_g, double sigma_a, double* P_out,
                    double* r_out) {
  const InterpolationBuffer buf = make_buffer(n, t, w, a);
  std::vector<ImuMeas<double>> meas;
  buf.GetRange(t_start, t_end, ts, &meas);
  if (meas.empty()) return 0;
  const SE3<double> t_2w = se3_inv(se3_from(T_w2));
  DPose pose{se3_from(T_w1), {v1[0], v1[1], v1[2]}};
  Mat<10, 10> c;
  Mat<6, 6> R;
  for (int i = 0; i < 3; ++i) { R(i, i) = powi(sigma_g, 2); R(3 + i, 3 + i) = powi(sigma_a, 2); }
  const Vec3<double> bg{b[0], b[1], b[2]}, ba{b[3], b[4], b[5]};
  const Vec3<double> gv = GetGravityVector<double>(g, gravity());
  const ImuMeas<double>* prev = nullptr;
  for (const ImuMeas<double>& m : meas) {
    if (prev) {
      Mat<10, 6> dy_db;
      Mat<10, 10> dy_dy;
      pose = IntegrateImuD(pose, *prev, m, bg, ba, sf, gv, &dy_db, &dy_dy, &c, R);
    }
    prev = &m;
  }
  const SE3<double> t12 = se3_mul(pose.t_wp, t_2w);
  Mat<9, 10> Jt;
  SetBlock(&Jt, 0, 0, dLog_dSE3(t12) * dt1t2_dt1(pose.t_wp, t_2w));
  SetBlock(&Jt, 6, 7, Mat<3, 3>::Identity());
  const Mat<9, 9> P = Jt * c * Tr(Jt);
  for (int i = 0; i < 81; ++i) P_out[i] = P.m[i];
  se3_log(t12, r_out);
  r_out[6] = pose.v_w.x - v2[0]; r_out[7] = pose.v_w.y - v2[1]; r_out[8] = pose.v_w.z - v2[2];
  return static_cast<int>(meas.size());
}

}  // extern "C"
