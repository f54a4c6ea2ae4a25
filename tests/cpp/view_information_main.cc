// Drives the C++ ViCalibrator mirror (vicalib_b200/host/vicalibrator.h) through its staged flow on a problem written by
// tests/test_gpu_host_mirror.py's _write_problem, with each camera's image size from the views file, then scores the
// candidate views with ViCalibrator::GetViewInformation and with vcgpu_get_view_information on the same handle.
// views.bin: int64 n_cand, n_pts, has_facing | int32 width[n_cams], height[n_cams] | T_wp[n_cand][7] | p_w[n_pts][3] |
// facing[3].  result.bin: int64 G | per path (method, then C-ABI): gain[n_cand], var[n_cand][G], n_seen[n_cand][n_cams]
// (as doubles).
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

static void put(FILE* o, const std::vector<double>& gain, const std::vector<double>& var, const std::vector<int32_t>& seen) {
  fwrite(gain.data(), sizeof(double), gain.size(), o);
  fwrite(var.data(), sizeof(double), var.size(), o);
  for (int32_t s : seen) {
    const double d = s;
    fwrite(&d, sizeof(double), 1, o);
  }
}

int main(int argc, char** argv) {
  if (argc < 4) { std::fprintf(stderr, "usage: %s problem.bin views.bin result.bin\n", argv[0]); return 2; }
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<int64_t> hd = rd<int64_t>(f, 8);  // n_cams n_frames n_obs n_imu inertial has_initial_guess max_iters mode
  const int nc = static_cast<int>(hd[0]), nf = static_cast<int>(hd[1]);
  const int64_t nobs = hd[2];
  std::vector<int32_t> model = rd<int32_t>(f, nc);
  std::vector<double> intr = rd<double>(f, 10 * nc), q = rd<double>(f, 4 * nc), p = rd<double>(f, 3 * nc);
  std::vector<double> T = rd<double>(f, 7 * nf), tm = rd<double>(f, nf);
  std::vector<int32_t> of = rd<int32_t>(f, nobs), oc = rd<int32_t>(f, nobs);
  std::vector<double> pw = rd<double>(f, 3 * nobs), pc = rd<double>(f, 2 * nobs);
  fclose(f);
  f = fopen(argv[2], "rb");
  if (!f) return 2;
  std::vector<int64_t> vh = rd<int64_t>(f, 3);
  const int64_t n_cand = vh[0], n_pts = vh[1];
  std::vector<int32_t> width = rd<int32_t>(f, nc), height = rd<int32_t>(f, nc);
  std::vector<double> cand = rd<double>(f, 7 * n_cand), target = rd<double>(f, 3 * n_pts), facing = rd<double>(f, 3);
  fclose(f);
  if (!vh[2]) facing.clear();

  static const char* kTypes[5] = {"calibu_fu_fv_u0_v0", "calibu_fu_fv_u0_v0_w", "calibu_fu_fv_u0_v0_k1_k2",
                                  "calibu_fu_fv_u0_v0_k1_k2_k3", "calibu_fu_fv_u0_v0_kb4"};
  static const int kK[5] = {4, 5, 6, 7, 8};
  CalibratorFlags flags;
  flags.calibrate_imu = false;  // a vision solve
  flags.max_iters = static_cast<int>(hd[6]);
  flags.trust_region_strategy = 0;
  ViCalibrator cal(flags);
  cal.SetEmulateBlockDuplication(false);
  for (int c = 0; c < nc; ++c) {
    std::vector<double> params(intr.begin() + 10 * c, intr.begin() + 10 * c + kK[model[c]]);
    cal.AddCamera(std::shared_ptr<CameraInterface>(new CameraInterface(kTypes[model[c]], width[c], height[c], params)),
                  SE3d(&q[4 * c], &p[3 * c]));
  }
  for (int fr = 0; fr < nf; ++fr) cal.AddFrame(SE3d(&T[7 * fr], &T[7 * fr + 4]), tm[fr]);
  for (int64_t i = 0; i < nobs; ++i)
    cal.AddObservation(of[i], oc[i], Vector3d{{pw[3 * i], pw[3 * i + 1], pw[3 * i + 2]}}, Vector2d{{pc[2 * i], pc[2 * i + 1]}}, tm[of[i]]);
  cal.SetFunctionTolerance(1e-10);
  cal.Start();
  while (cal.IsRunning()) usleep(2000);
  cal.Stop();

  std::vector<double> var;
  std::vector<int32_t> seen;
  const std::vector<double> gain = cal.GetViewInformation(cand, target, facing, &var, &seen);
  int G = 0;
  vcgpu_num_globals(cal.handle(), &G);
  std::vector<double> gain2(n_cand), var2(static_cast<size_t>(n_cand) * G);
  std::vector<int32_t> seen2(static_cast<size_t>(n_cand) * nc);
  const vcgpu_view_candidates v{n_cand, cand.data(), static_cast<int>(n_pts), target.data(), facing.empty() ? nullptr : facing.data(),
                                width.data(), height.data(), seen2.data(), gain2.data(), var2.data(), nullptr};
  if (vcgpu_get_view_information(cal.handle(), nullptr, &v) != VCGPU_OK) {
    std::fprintf(stderr, "%s\n", vcgpu_last_error(cal.handle()));
    return 1;
  }
  FILE* o = fopen(argv[3], "wb");
  const int64_t g64 = G;
  fwrite(&g64, sizeof(int64_t), 1, o);
  put(o, gain, var, seen);
  put(o, gain2, var2, seen2);
  fclose(o);
  return 0;
}
