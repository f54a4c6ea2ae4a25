// Drives the C++ ViCalibrator mirror (vicalib_b200/host/vicalibrator.h) through its staged flow on a problem written by
// tests/test_gpu_integration_poses.py (the layout of host_mirror_main.cc's input), then compares the device's
// GetAllIntegrationPoses() with the host GetIntegrationPoses(k) of every interval k:
//   final <intervals> <poses> <counts equal> <times equal> <worst q> <worst t> <worst v_w> <worst w_w>
// (worst: largest difference relative to the group's scale over the interval, 1 for q), then the gate of
// vicalibrator.h:510 in a rotation-only and a vision stage set afterwards:
//   rotation_only <device poses> <host poses>
//   vision <device poses> <host poses>
#include <unistd.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../vicalib_b200/host/vicalibrator.h"

using namespace visual_inertial_calibration;  // NOLINT

template <class T>
static std::vector<T> rd(FILE* f, size_t n) {
  std::vector<T> v(n);
  if (n && fread(v.data(), sizeof(T), n, f) != n) { std::fprintf(stderr, "short read\n"); std::exit(2); }
  return v;
}

static void put(const ImuPose& y, double* o) {
  for (int k = 0; k < 7; ++k) o[k] = y.t_wp_.d[k];
  for (int k = 0; k < 3; ++k) { o[7 + k] = y.v_w_[k]; o[10 + k] = y.w_w_[k]; }
}

static size_t total(const std::vector<std::vector<ImuPose>>& v) {
  size_t n = 0;
  for (const auto& x : v) n += x.size();
  return n;
}

static std::vector<std::vector<ImuPose>> host_all(ViCalibrator& cal) {
  std::vector<std::vector<ImuPose>> out;
  for (size_t k = 0; k + 1 < cal.NumFrames(); ++k) out.push_back(cal.GetIntegrationPoses(static_cast<unsigned>(k)));
  return out;
}

int main(int argc, char** argv) {
  if (argc < 3) { std::fprintf(stderr, "usage: %s problem.bin result.txt\n", argv[0]); return 2; }
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<int64_t> hd = rd<int64_t>(f, 8);  // n_cams n_frames n_obs n_imu inertial has_initial_guess max_iters mode
  const int nc = static_cast<int>(hd[0]), nf = static_cast<int>(hd[1]);
  const int64_t nobs = hd[2], nimu = hd[3];
  std::vector<int32_t> model = rd<int32_t>(f, nc);
  std::vector<double> intr = rd<double>(f, 10 * nc), q = rd<double>(f, 4 * nc), p = rd<double>(f, 3 * nc);
  std::vector<double> T = rd<double>(f, 7 * nf), tm = rd<double>(f, nf);
  std::vector<int32_t> of = rd<int32_t>(f, nobs), oc = rd<int32_t>(f, nobs);
  std::vector<double> pw = rd<double>(f, 3 * nobs), pc = rd<double>(f, 2 * nobs);
  std::vector<double> it = rd<double>(f, nimu), iw = rd<double>(f, 3 * nimu), ia = rd<double>(f, 3 * nimu);
  fclose(f);

  static const char* kTypes[5] = {"calibu_fu_fv_u0_v0", "calibu_fu_fv_u0_v0_w", "calibu_fu_fv_u0_v0_k1_k2",
                                  "calibu_fu_fv_u0_v0_k1_k2_k3", "calibu_fu_fv_u0_v0_kb4"};
  static const int kK[5] = {4, 5, 6, 7, 8};
  CalibratorFlags flags;
  flags.max_iters = static_cast<int>(hd[6]);
  flags.trust_region_strategy = 0;
  ViCalibrator cal(flags);
  for (int c = 0; c < nc; ++c) {
    std::vector<double> params(intr.begin() + 10 * c, intr.begin() + 10 * c + kK[model[c]]);
    cal.AddCamera(std::shared_ptr<CameraInterface>(new CameraInterface(kTypes[model[c]], 640, 480, params)), SE3d(&q[4 * c], &p[3 * c]));
  }
  for (int fr = 0; fr < nf; ++fr) cal.AddFrame(SE3d(&T[7 * fr], &T[7 * fr + 4]), tm[fr]);
  for (int64_t i = 0; i < nobs; ++i)
    cal.AddObservation(of[i], oc[i], Vector3d{{pw[3 * i], pw[3 * i + 1], pw[3 * i + 2]}}, Vector2d{{pc[2 * i], pc[2 * i + 1]}}, tm[of[i]]);
  for (int64_t i = 0; i < nimu; ++i)
    cal.AddImuMeasurements(Vector3d{{iw[3 * i], iw[3 * i + 1], iw[3 * i + 2]}}, Vector3d{{ia[3 * i], ia[3 * i + 1], ia[3 * i + 2]}}, it[i]);
  cal.SetFunctionTolerance(1e-10);
  cal.SetOptimizationFlags(true, true, false, true);  // vicalib-task.cc:227-235 (an initial guess)
  cal.Start();
  while (cal.IsRunning()) usleep(2000);
  cal.Stop();

  FILE* o = fopen(argv[2], "w");
  {
    const std::vector<std::vector<ImuPose>> dev = cal.GetAllIntegrationPoses(), host = host_all(cal);
    bool counts = dev.size() == host.size(), times = true;
    double worst[4] = {0, 0, 0, 0};
    for (size_t k = 0; counts && k < dev.size(); ++k) {
      if (dev[k].size() != host[k].size()) { counts = false; break; }
      double scale[4] = {1.0, 1e-3, 1e-3, 1e-3}, diff[4] = {0, 0, 0, 0};
      for (size_t i = 0; i < dev[k].size(); ++i) {
        double a[13], b[13];
        put(dev[k][i], a);
        put(host[k][i], b);
        times = times && dev[k][i].time_ == host[k][i].time_;
        for (int j = 0; j < 13; ++j) {
          const int g = j < 4 ? 0 : j < 7 ? 1 : j < 10 ? 2 : 3;
          if (g > 0) scale[g] = std::max(scale[g], std::fabs(b[j]));
          diff[g] = std::max(diff[g], std::fabs(a[j] - b[j]));
        }
      }
      for (int g = 0; g < 4; ++g) worst[g] = std::max(worst[g], diff[g] / scale[g]);
    }
    std::fprintf(o, "final %zu %zu %d %d %.6g %.6g %.6g %.6g\n", dev.size(), total(dev), counts ? 1 : 0, times ? 1 : 0, worst[0],
                 worst[1], worst[2], worst[3]);
  }
  cal.SetOptimizationFlags(true, true, true, true);
  std::fprintf(o, "rotation_only %zu %zu\n", total(cal.GetAllIntegrationPoses()), total(host_all(cal)));
  cal.SetOptimizationFlags(false, false, false, false);
  std::fprintf(o, "vision %zu %zu\n", total(cal.GetAllIntegrationPoses()), total(host_all(cal)));
  fclose(o);
  return 0;
}
