// TEST INFRASTRUCTURE ONLY: flat C entry points over two CPU restatements of ViCalibrator::GetIntegrationPoses
// (vicalibrator.h:508-533), for tests/integration_poses_ref.py, which compiles this file into a temporary directory.
//   vo_integration_poses      the oracle's GetRange and IntegrateImuD (oracle/cost_functors.h, oracle/imu_weights.h);
//                             w_w from the oracle's stage functions, GetPoseDerivativeD summed as types.h:588
//   mirror_integration_poses  the host mirror's own GetIntegrationPoses (vicalib_b200/host/vicalibrator.h) on a
//                             ViCalibrator whose members are set directly.  No device is touched: the three C-ABI calls
//                             its constructor and destructor make are stubbed below.
// Both return one interval's poses, 14 doubles each (q x y z w | t | v_w | w_w | time), and their number.
//   mirror_all_integration_poses  the mirror's GetIntegrationPoses(k) for every k on one object, timed (the probe's arm)
#include <chrono>
#include <cmath>
#include <cstdint>

#include "imu_weights.h"
#include "../../vicalib_b200/host/vicalibrator.h"

extern "C" {
int vcgpu_create(const vcgpu_config*, vcgpu_handle** out) { *out = nullptr; return VCGPU_OK; }
int vcgpu_destroy(vcgpu_handle*) { return VCGPU_OK; }
void vcgpu_default_options(vcgpu_options* o) { *o = vcgpu_options(); }
}

namespace {

vo::InterpolationBuffer make_buffer(int n, const double* t, const double* w, const double* a) {
  vo::InterpolationBuffer buf;
  for (int i = 0; i < n; ++i)
    buf.AddElement({{w[3 * i], w[3 * i + 1], w[3 * i + 2]}, {a[3 * i], a[3 * i + 1], a[3 * i + 2]}, t[i]});
  return buf;
}

void put(double* o, const double* q, const double* t, const double* v, const double* w, double time) {
  for (int k = 0; k < 4; ++k) o[k] = q[k];
  for (int k = 0; k < 3; ++k) { o[4 + k] = t[k]; o[7 + k] = v[k]; o[10 + k] = w[k]; }
  o[13] = time;
}

// the mirror with nf frames and its IMU inputs set as the solve would leave them: inertial, not rotation-only
class Mirror : public visual_inertial_calibration::ViCalibrator {
 public:
  Mirror(int n, const double* t, const double* w, const double* a, int nf, const double* ftime, const double* T_wp,
         const double* v_w, const double* g, const double* b, const double* sf, double ts) {
    using namespace visual_inertial_calibration;  // NOLINT
    for (int i = 0; i < n; ++i)
      imu_.push_back(ImuMeasurement{{{w[3 * i], w[3 * i + 1], w[3 * i + 2]}}, {{a[3 * i], a[3 * i + 1], a[3 * i + 2]}}, t[i]});
    for (int f = 0; f < nf; ++f) {
      SE3d T;
      std::memcpy(T.d, T_wp + 7 * f, 7 * sizeof(double));
      AddFrameUnlocked(T, ftime[f]);
      t_wk_[f]->v_w_ = Vector3d{{v_w[3 * f], v_w[3 * f + 1], v_w[3 * f + 2]}};
    }
    g_[0] = g[0]; g_[1] = g[1];
    for (int i = 0; i < 6; ++i) { biases_[i] = b[i]; scale_factors_[i] = sf[i]; }
    time_offset_ = ts;
    is_inertial_active_ = true;
    optimize_rotation_only_ = false;
  }
};

}  // namespace

extern "C" {

int vo_integration_poses(int n, const double* t, const double* w, const double* a, double t_start, double t_end,
                         const double* x1, const double* v1, const double* g, const double* b, const double* sf,
                         double ts, double* out, int max_n) {
  using namespace vo;  // NOLINT
  const InterpolationBuffer buf = make_buffer(n, t, w, a);
  std::vector<ImuMeas<double>> meas;
  buf.GetRange(t_start, t_end, ts, &meas);
  const int m = static_cast<int>(meas.size());
  if (m == 0) return 0;
  const Vec3<double> bg{b[0], b[1], b[2]}, ba{b[3], b[4], b[5]};
  const Vec3<double> gv = GetGravityVector<double>(g, gravity());
  DPose y{se3_from(x1), {v1[0], v1[1], v1[2]}};
  double wv[3] = {0.0, 0.0, 0.0}, time = t_start;
  Mat<6, 6> R;
  for (int i = 0; i < m && i < max_n; ++i) {
    if (i > 0 && meas[i].time - meas[i - 1].time != 0) {
      const ImuMeas<double>& z0 = meas[i - 1];
      const ImuMeas<double>& z1 = meas[i];
      const double dt = z1.time - z0.time;
      double k1[9], k2[9], k3[9], k4[9];
      GetPoseDerivativeD(y, gv, z0, z1, bg, ba, sf, 0, k1, nullptr, nullptr);
      GetPoseDerivativeD(IntegratePoseD(y, k1, dt * 0.5, nullptr, nullptr), gv, z0, z1, bg, ba, sf, dt / 2, k2, nullptr, nullptr);
      GetPoseDerivativeD(IntegratePoseD(y, k2, dt * 0.5, nullptr, nullptr), gv, z0, z1, bg, ba, sf, dt / 2, k3, nullptr, nullptr);
      GetPoseDerivativeD(IntegratePoseD(y, k3, dt, nullptr, nullptr), gv, z0, z1, bg, ba, sf, dt, k4, nullptr, nullptr);
      for (int k = 0; k < 3; ++k) wv[k] = k1[3 + k] + 2 * k2[3 + k] + 2 * k3[3 + k] + k4[3 + k];
      Mat<10, 6> dy_db;
      Mat<10, 10> dy_dy;
      y = IntegrateImuD(y, z0, z1, bg, ba, sf, gv, &dy_db, &dy_dy, nullptr, R);
      time = z1.time;
    }
    const double q[4] = {y.t_wp.q.x, y.t_wp.q.y, y.t_wp.q.z, y.t_wp.q.w}, tt[3] = {y.t_wp.t.x, y.t_wp.t.y, y.t_wp.t.z};
    const double v[3] = {y.v_w.x, y.v_w.y, y.v_w.z};
    put(out + 14 * i, q, tt, v, wv, time);
  }
  return m;
}

int mirror_integration_poses(int n, const double* t, const double* w, const double* a, double t_start, double t_end,
                             const double* x1, const double* v1, const double* g, const double* b, const double* sf,
                             double ts, double* out, int max_n) {
  const double ft[2] = {t_start, t_end};
  double T2[14] = {0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0}, v2[6] = {0, 0, 0, 0, 0, 0};  // frame 1's are not read
  std::memcpy(T2, x1, 7 * sizeof(double));
  std::memcpy(v2, v1, 3 * sizeof(double));
  Mirror cal(n, t, w, a, 2, ft, T2, v2, g, b, sf, ts);
  const std::vector<visual_inertial_calibration::ImuPose> poses = cal.GetIntegrationPoses(0);
  const int m = static_cast<int>(poses.size());
  for (int i = 0; i < m && i < max_n; ++i)
    put(out + 14 * i, poses[i].t_wp_.d, poses[i].t_wp_.d + 4, poses[i].v_w_.data(), poses[i].w_w_.data(), poses[i].time_);
  return m;
}

// the mirror's GetIntegrationPoses(k) for k = 0 .. nf - 2 on one object, as a GUI redraw calls it: the total number of
// poses, and the wall time of the loop alone in *seconds
int64_t mirror_all_integration_poses(int n, const double* t, const double* w, const double* a, int nf, const double* ftime,
                                     const double* T_wp, const double* v_w, const double* g, const double* b,
                                     const double* sf, double ts, double* seconds) {
  Mirror cal(n, t, w, a, nf, ftime, T_wp, v_w, g, b, sf, ts);
  int64_t total = 0;
  const auto t0 = std::chrono::steady_clock::now();
  for (int k = 0; k + 1 < nf; ++k) total += static_cast<int64_t>(cal.GetIntegrationPoses(k).size());
  *seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return total;
}

}  // extern "C"
