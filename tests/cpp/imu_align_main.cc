// Drives the C++ ViCalibrator mirror (vicalib_b200/host/vicalibrator.h) through its vision-only flow on a problem
// written by tests/test_gpu_host_mirror.py's _write_problem, then aligns the IMU twice: vcgpu_align_imu without apply on
// the mirror's handle, then ViCalibrator::AlignImu, which applies it.
// result.bin: per path (C-ABI, then method) Q[4] ts b_g[3] rms excitation[3]; then the mirror's state after AlignImu:
// T_ck q of every camera [n_cams][4], every frame's t_wp_ [n_frames][7], time_offset(), GetBiases()[6].
#include <unistd.h>

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

static void put(FILE* out, const vcgpu_imu_alignment& r) {
  fwrite(r.Q, sizeof(double), 4, out);
  fwrite(&r.ts, sizeof(double), 1, out);
  fwrite(r.b_g, sizeof(double), 3, out);
  fwrite(&r.rms, sizeof(double), 1, out);
  fwrite(r.excitation, sizeof(double), 3, out);
}

int main(int argc, char** argv) {
  if (argc < 3) { std::fprintf(stderr, "usage: %s problem.bin result.bin\n", argv[0]); return 2; }
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
  flags.calibrate_imu = false;
  flags.max_iters = static_cast<int>(hd[6]);
  flags.trust_region_strategy = 0;
  ViCalibrator cal(flags);
  for (int c = 0; c < nc; ++c) {
    std::vector<double> params(intr.begin() + 10 * c, intr.begin() + 10 * c + kK[model[c]]);
    cal.AddCamera(std::shared_ptr<CameraInterface>(new CameraInterface(kTypes[model[c]], 640, 480, params)),
                  SE3d(&q[4 * c], &p[3 * c]));
  }
  for (int fr = 0; fr < nf; ++fr) cal.AddFrame(SE3d(&T[7 * fr], &T[7 * fr + 4]), tm[fr]);
  for (int64_t i = 0; i < nobs; ++i)
    cal.AddObservation(of[i], oc[i], Vector3d{{pw[3 * i], pw[3 * i + 1], pw[3 * i + 2]}}, Vector2d{{pc[2 * i], pc[2 * i + 1]}}, tm[of[i]]);
  for (int64_t i = 0; i < nimu; ++i)
    cal.AddImuMeasurements(Vector3d{{iw[3 * i], iw[3 * i + 1], iw[3 * i + 2]}}, Vector3d{{ia[3 * i], ia[3 * i + 1], ia[3 * i + 2]}}, it[i]);
  cal.Start();
  while (cal.IsRunning()) usleep(2000);
  cal.Stop();

  const vcgpu_imu_align_opts o{-0.05, 0.05, 21, 1, 20, 0};
  vcgpu_imu_alignment a{};
  if (vcgpu_align_imu(cal.handle(), &o, &a) != VCGPU_OK) {
    std::fprintf(stderr, "%s\n", vcgpu_last_error(cal.handle()));
    return 1;
  }
  const vcgpu_imu_alignment b = cal.AlignImu(-0.05, 0.05, 21, true);
  FILE* out = fopen(argv[2], "wb");
  put(out, a);
  put(out, b);
  for (int c = 0; c < nc; ++c) fwrite(cal.GetCamera(c).T_ck.d, sizeof(double), 4, out);
  for (int fr = 0; fr < nf; ++fr) fwrite(cal.GetFrame(fr)->t_wp_.d, sizeof(double), 7, out);
  const double ts = cal.time_offset();
  fwrite(&ts, sizeof(double), 1, out);
  const Vector6d bias = cal.GetBiases();
  fwrite(bias.data(), sizeof(double), 6, out);
  fclose(out);
  return 0;
}
