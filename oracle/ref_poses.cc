// ORACLE — TEST INFRASTRUCTURE ONLY.
// oracle/_ref/libvicalib_ref_poses.so: ViCalibrator::GetIntegrationPoses (vicalibrator.h:508-533) through the
// reference's OWN headers, compiled UNMODIFIED from the reference's include/ against the stand-ins of oracle/ref_shim,
// as oracle/_ref/libvicalib_ref.so is (oracle/ref_main.cc, oracle/README.md):
//   include/vicalib/types.h                  GetGravityVector, ImuPoseT, ImuMeasurementT, ImuResidualT::IntegrateResidual
//                                            (the double RK4 of IntegrateImu, no Jacobians)
//   include/vicalib/interpolation-buffer.h   InterpolationBufferT (AddElement, GetRange)
// This file only marshals flat arrays and restates the method's glue: GetRange over the interval, then IntegrateResidual
// from the frame's ImuPoseT.  Built by `make -C oracle -f ref_poses.mk` (only where the reference tree exists); used by
// tests/integration_poses_ref.py.
#include <vector>

#include <ceres/ceres.h>
#include <glog/logging.h>

// include order of include/vicalib/vicalibrator.h:51-53
#include <vicalib/types.h>
#include <vicalib/vicalibrator-utils.h>
#include <vicalib/interpolation-buffer.h>

namespace visual_inertial_calibration {
int debug_level_threshold = 0;
int debug_level = 0;
}  // namespace visual_inertial_calibration

using namespace visual_inertial_calibration;  // NOLINT
typedef InterpolationBufferT<ImuMeasurementT, double> ImuBuffer;

extern "C" {

// GetIntegrationPoses(id) for the interval [t_start, t_end]: GetRange(t_start, t_end, ts), then IntegrateResidual
// without Jacobians (types.h:611-687) from the frame's ImuPoseT (pose x1 = [qx qy qz qw | t], velocity v1, w_w_ = 0,
// time t_start).  Returns the number of poses (0: no measurements); out rows: q (x y z w), t (3), v_w (3), w_w (3), time.
int ref_integration_poses(int n, const double* t, const double* w, const double* a, double t_start, double t_end,
                          const double* x1, const double* v1, const double* g, const double* b, const double* sf, double ts,
                          double* out, int max_n) {
  ImuBuffer buf(n);
  for (int i = 0; i < n; ++i)
    buf.AddElement(ImuMeasurementT<double>(Eigen::Vector3d(w[3 * i], w[3 * i + 1], w[3 * i + 2]),
                                           Eigen::Vector3d(a[3 * i], a[3 * i + 1], a[3 * i + 2]), t[i]));
  aligned_vector<ImuMeasurementT<double> > measurements;
  buf.GetRange(t_start, t_end, ts, &measurements);
  if (measurements.empty()) return 0;
  const Sophus::SE3d t_w1 = Sophus::SE3d(Eigen::Map<const Sophus::SE3d>(x1));
  const ImuPoseT<double> start_pose(t_w1, Eigen::Vector3d(v1[0], v1[1], v1[2]), Eigen::Vector3d::Zero(), t_start);
  aligned_vector<ImuPoseT<double> > poses;
  Vector6d biases, scale_factors;
  for (int i = 0; i < 6; ++i) { biases[i] = b[i]; scale_factors[i] = sf[i]; }
  const Eigen::Matrix<double, 2, 1> gdir(g[0], g[1]);
  ImuResidualT<double>::IntegrateResidual(start_pose, measurements, biases.head<3>(), biases.tail<3>(), scale_factors,
                                          GetGravityVector(gdir, gravity()), poses);
  const int m = static_cast<int>(poses.size());
  for (int i = 0; i < m && i < max_n; ++i) {
    double* o = out + 14 * i;
    const Sophus::SE3d& T = poses[i].t_wp_;
    for (int k = 0; k < 4; ++k) o[k] = T.so3().unit_quaternion().coeffs()[k];
    for (int k = 0; k < 3; ++k) {
      o[4 + k] = T.translation()[k];
      o[7 + k] = poses[i].v_w_[k];
      o[10 + k] = poses[i].w_w_[k];
    }
    o[13] = poses[i].time_;
  }
  return m;
}

}  // extern "C"
