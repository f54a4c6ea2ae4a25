// Host-side mirror of the reference's ViCalibrator (include/vicalib/vicalibrator.h:119-1086) on top of
// the C-ABI in include/vcgpu.h.  Same public method names, argument meaning and error behaviour, so
// VicalibTask / VicalibEngine call sites (vicalib-task.cc:128-147,227-245,339-363,607-610,689;
// vicalib-engine.cc:301-303,356,365,388-399,415-418) keep compiling against it; everything that used to
// happen inside ceres::Problem / ceres::Solve now happens on the GPU.
//
// Calibu / Sophus / Eigen are not vendored by the reference and are not in this image, so the few
// value types those call sites touch are provided as minimal stand-ins with the same member names:
//   Sophus::SE3d        -> SE3d   (7 doubles: unit quaternion x,y,z,w + translation; Sophus' own storage)
//   calibu::CameraInterface<double> -> CameraInterface (Type(), GetParams(), NumParams(), Width/Height, RDF, Pose)
// A build that has the real libraries can replace these two typedefs and nothing else.
#ifndef VICALIB_B200_HOST_VICALIBRATOR_H_
#define VICALIB_B200_HOST_VICALIBRATOR_H_

#include <pthread.h>

#include <array>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iomanip>
#include <memory>
#include <sstream>
#include <stdexcept>
#include <cctype>
#include <string>
#include <vector>

#include "../../include/vcgpu.h"

namespace visual_inertial_calibration {

// reference: glog CHECK aborts (vicalibrator.h:254,302,356,377,396,456)
#define VICALIB_CHECK(cond, msg)                                              \
  do {                                                                        \
    if (!(cond)) {                                                            \
      std::fprintf(stderr, "Check failed: %s  %s\n", #cond, msg);             \
      std::abort();                                                           \
    }                                                                         \
  } while (0)

typedef std::array<double, 3> Vector3d;
typedef std::array<double, 2> Vector2d;
typedef std::array<double, 6> Vector6d;

// ---- Sophus::SE3d stand-in (storage order of Sophus: quaternion coefficients x,y,z,w then translation)
struct SE3d {
  double d[7] = {0, 0, 0, 1, 0, 0, 0};
  SE3d() {}
  SE3d(const double q[4], const double t[3]) {
    for (int i = 0; i < 4; ++i) d[i] = q[i];
    for (int i = 0; i < 3; ++i) d[4 + i] = t[i];
  }
  double* data() { return d; }
  const double* data() const { return d; }
  void rotation(double R[9]) const {
    const double x = d[0], y = d[1], z = d[2], w = d[3];
    R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - w * z); R[2] = 2 * (x * z + w * y);
    R[3] = 2 * (x * y + w * z); R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - w * x);
    R[6] = 2 * (x * z - w * y); R[7] = 2 * (y * z + w * x); R[8] = 1 - 2 * (x * x + y * y);
  }
  SE3d inverse() const {
    double R[9];
    rotation(R);
    SE3d o;
    o.d[0] = -d[0]; o.d[1] = -d[1]; o.d[2] = -d[2]; o.d[3] = d[3];
    for (int i = 0; i < 3; ++i) o.d[4 + i] = -(R[0 * 3 + i] * d[4] + R[1 * 3 + i] * d[5] + R[2 * 3 + i] * d[6]);
    return o;
  }
  SE3d operator*(const SE3d& b) const {
    const double *p = d, *q = b.d;
    SE3d o;
    o.d[0] = p[3] * q[0] + p[0] * q[3] + p[1] * q[2] - p[2] * q[1];
    o.d[1] = p[3] * q[1] + p[1] * q[3] + p[2] * q[0] - p[0] * q[2];
    o.d[2] = p[3] * q[2] + p[2] * q[3] + p[0] * q[1] - p[1] * q[0];
    o.d[3] = p[3] * q[3] - p[0] * q[0] - p[1] * q[1] - p[2] * q[2];
    double R[9];
    rotation(R);
    for (int i = 0; i < 3; ++i) o.d[4 + i] = d[4 + i] + R[i * 3] * q[4] + R[i * 3 + 1] * q[5] + R[i * 3 + 2] * q[6];
    return o;
  }
  void matrix3x4(double M[12]) const {
    double R[9];
    rotation(R);
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) M[i * 4 + j] = R[i * 3 + j];
      M[i * 4 + 3] = d[4 + i];
    }
  }
  static SE3d FromRotation(const double R[9]) {  // rotation matrix -> SE3 with zero translation
    SE3d o;
    const double t = R[0] + R[4] + R[8];
    double q[4];
    if (t > 0) { const double s = std::sqrt(t + 1.0) * 2; q[3] = 0.25 * s; q[0] = (R[7] - R[5]) / s; q[1] = (R[2] - R[6]) / s; q[2] = (R[3] - R[1]) / s; }
    else if (R[0] > R[4] && R[0] > R[8]) { const double s = std::sqrt(1.0 + R[0] - R[4] - R[8]) * 2; q[3] = (R[7] - R[5]) / s; q[0] = 0.25 * s; q[1] = (R[1] + R[3]) / s; q[2] = (R[2] + R[6]) / s; }
    else if (R[4] > R[8]) { const double s = std::sqrt(1.0 + R[4] - R[0] - R[8]) * 2; q[3] = (R[2] - R[6]) / s; q[0] = (R[1] + R[3]) / s; q[1] = 0.25 * s; q[2] = (R[5] + R[7]) / s; }
    else { const double s = std::sqrt(1.0 + R[8] - R[0] - R[4]) * 2; q[3] = (R[3] - R[1]) / s; q[0] = (R[2] + R[6]) / s; q[1] = (R[5] + R[7]) / s; q[2] = 0.25 * s; }
    for (int i = 0; i < 4; ++i) o.d[i] = q[i];
    return o;
  }
};

// calibu::RdfRobotics / RdfVision (SURVEY App. A.2)
static const double kRdfRobotics[9] = {0, 1, 0, 0, 0, 1, 1, 0, 0};
static const double kRdfVision[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};

// ---- calibu::CameraInterface<double> stand-in
class CameraInterface {
 public:
  // type strings as written by the reference (vicalib-engine.cc:210,220,230,250,260)
  CameraInterface(const std::string& type, int width, int height, const std::vector<double>& params)
      : type_(type), width_(width), height_(height), params_(params) {
    std::memcpy(rdf_, kRdfVision, sizeof rdf_);
    VICALIB_CHECK(ModelId() >= 0, "Don't know how to optimize CameraModel");  // vicalibrator.h:455-458
    VICALIB_CHECK(static_cast<int>(params_.size()) == NumParams(), "parameter count does not match the model");
  }
  const std::string& Type() const { return type_; }
  int ModelId() const {
    if (type_ == "calibu_fu_fv_u0_v0") return VCGPU_CAM_LINEAR;
    if (type_ == "calibu_fu_fv_u0_v0_w") return VCGPU_CAM_FOV;
    if (type_ == "calibu_fu_fv_u0_v0_k1_k2") return VCGPU_CAM_POLY2;
    if (type_ == "calibu_fu_fv_u0_v0_k1_k2_k3") return VCGPU_CAM_POLY3;
    if (type_ == "calibu_fu_fv_u0_v0_kb4") return VCGPU_CAM_KB4;
    return -1;
  }
  int NumParams() const {
    static const int k[5] = {4, 5, 6, 7, 8};
    return k[ModelId()];
  }
  std::vector<double>& GetParams() { return params_; }
  const std::vector<double>& GetParams() const { return params_; }
  int Width() const { return width_; }
  int Height() const { return height_; }
  void SetIndex(int i) { index_ = i; }
  int Index() const { return index_; }
  void SetRDF(const double R[9]) { std::memcpy(rdf_, R, sizeof rdf_); }
  const double* RDF() const { return rdf_; }
  void SetPose(const SE3d& T) { pose_ = T; }
  const SE3d& Pose() const { return pose_; }

 private:
  std::string type_;
  int width_, height_, index_ = 0;
  std::vector<double> params_;
  double rdf_[9];
  SE3d pose_;
};

// ---- calibu::ReadXmlRig stand-in: reads the rig files WriteCameraModels writes (and Calibu's own: same tags).
// The reference uses it for `-model_files` warm starts and keeps only cameras_[0] of every file with an identity
// pose (vicalib-engine.cc:188-196); pose and RDF are parsed as well.  Throws std::runtime_error on a malformed file.
namespace xml_detail {
inline std::string Between(const std::string& s, const std::string& open, const std::string& close, size_t from, size_t* end) {
  const size_t a = s.find(open, from);
  if (a == std::string::npos) { *end = std::string::npos; return std::string(); }
  const size_t b = s.find(close, a + open.size());
  if (b == std::string::npos) throw std::runtime_error("rig xml: missing " + close);
  *end = b + close.size();
  return s.substr(a + open.size(), b - a - open.size());
}
inline std::vector<double> Numbers(const std::string& text) {  // "[ a; b, c ]" -> {a, b, c}
  std::vector<double> v;
  std::string tok;
  for (size_t i = 0; i <= text.size(); ++i) {
    const char ch = i < text.size() ? text[i] : ' ';
    if (std::isdigit(static_cast<unsigned char>(ch)) || ch == '-' || ch == '+' || ch == '.' || ch == 'e' || ch == 'E' ||
        ch == 'n' || ch == 'a' || ch == 'i' || ch == 'f') {
      tok.push_back(ch);
    } else if (!tok.empty()) {
      v.push_back(std::strtod(tok.c_str(), nullptr));
      tok.clear();
    }
  }
  return v;
}
inline std::string Attribute(const std::string& tag, const std::string& name) {
  const size_t a = tag.find(name + "=\"");
  if (a == std::string::npos) return std::string();
  const size_t b = tag.find('"', a + name.size() + 2);
  return tag.substr(a + name.size() + 2, b - a - name.size() - 2);
}
}  // namespace xml_detail

inline std::vector<std::shared_ptr<CameraInterface>> ReadXmlRig(const std::string& filename) {
  std::ifstream in(filename.c_str());
  if (!in) throw std::runtime_error("rig xml: cannot open " + filename);
  std::stringstream ss;
  ss << in.rdbuf();
  const std::string s = ss.str();
  std::vector<std::shared_ptr<CameraInterface>> rig;
  size_t pos = 0;
  for (;;) {
    size_t end = 0;
    const std::string cam = xml_detail::Between(s, "<camera>", "</camera>", pos, &end);
    if (end == std::string::npos) break;
    pos = end;
    const size_t m0 = cam.find("<camera_model");
    if (m0 == std::string::npos) throw std::runtime_error("rig xml: <camera> without <camera_model>");
    const std::string head = cam.substr(m0, cam.find('>', m0) - m0);
    const std::string type = xml_detail::Attribute(head, "type");
    size_t e = 0;
    const std::vector<double> w = xml_detail::Numbers(xml_detail::Between(cam, "<width>", "</width>", 0, &e));
    const std::vector<double> h = xml_detail::Numbers(xml_detail::Between(cam, "<height>", "</height>", 0, &e));
    const std::vector<double> params = xml_detail::Numbers(xml_detail::Between(cam, "<params>", "</params>", 0, &e));
    if (w.size() != 1 || h.size() != 1) throw std::runtime_error("rig xml: bad <width>/<height>");
    std::shared_ptr<CameraInterface> c(new CameraInterface(type, static_cast<int>(w[0]), static_cast<int>(h[0]), params));
    const std::string idx = xml_detail::Attribute(head, "index");
    if (!idx.empty()) c->SetIndex(std::atoi(idx.c_str()));
    const std::vector<double> r = xml_detail::Numbers(xml_detail::Between(cam, "<right>", "</right>", 0, &e));
    const std::vector<double> d = xml_detail::Numbers(xml_detail::Between(cam, "<down>", "</down>", 0, &e));
    const std::vector<double> f = xml_detail::Numbers(xml_detail::Between(cam, "<forward>", "</forward>", 0, &e));
    if (r.size() == 3 && d.size() == 3 && f.size() == 3) {  // right / down / forward are the columns of the RDF matrix
      const double R[9] = {r[0], d[0], f[0], r[1], d[1], f[1], r[2], d[2], f[2]};
      c->SetRDF(R);
    }
    const std::vector<double> T = xml_detail::Numbers(xml_detail::Between(cam, "<T_wc>", "</T_wc>", 0, &e));
    if (T.size() == 12) {
      const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
      SE3d pose = SE3d::FromRotation(R);
      pose.d[4] = T[3]; pose.d[5] = T[7]; pose.d[6] = T[11];
      c->SetPose(pose);
    } else if (!T.empty()) {
      throw std::runtime_error("rig xml: <T_wc> is not 3x4");
    }
    rig.push_back(c);
  }
  if (rig.empty()) throw std::runtime_error("rig xml: no <camera> in " + filename);
  return rig;
}

struct CameraAndPose {  // vicalibrator.h:65-73
  CameraAndPose(const std::shared_ptr<CameraInterface>& c, const SE3d& T) : camera(c), T_ck(T) {}
  std::shared_ptr<CameraInterface> camera;
  SE3d T_ck;
};

struct VicalibFrame {  // vicalibrator.h:76-97 (ImuPoseT fields the call sites read)
  SE3d t_wp_;
  Vector3d v_w_{{0, 0, 0}}, w_w_{{0, 0, 0}};
  double time_ = 0;
  std::vector<bool> has_measurements_from_cam;
  void SetHasMeasurementsFromCam(size_t cam_id, bool val) {
    while (has_measurements_from_cam.size() <= cam_id) has_measurements_from_cam.push_back(false);
    has_measurements_from_cam[cam_id] = val;
  }
};

struct ImuMeasurement { Vector3d w_, a_; double time; };

struct ImuPose {  // ImuPoseT<double> (types.h:170-205): what GetIntegrationPoses hands to the GUI
  SE3d t_wp_;
  Vector3d v_w_{{0, 0, 0}}, w_w_{{0, 0, 0}};
  double time_ = 0;
};

// Flags the reference reads from gflags (vicalibrator.h:56-60; defaults vicalib-engine.cc:94, :30-104)
struct CalibratorFlags {
  bool calibrate_imu = true;
  int max_iters = 200;
  bool remove_outliers = false;    // DEFINE_bool(remove_outliers, false, ...) vicalib-engine.cc:100
  double outlier_threshold = 2.0;  // vicalib-engine.cc:102
  // 1 = DOGLEG, the reference's solver_options_ (vicalibrator.h:151); 0 = LEVENBERG_MARQUARDT (what north_star
  // benchmarks; the only strategy of frame-sharded multi-GPU solves)
  int trust_region_strategy = 1;
};

class ViCalibrator {
 public:
  explicit ViCalibrator(const CalibratorFlags& flags = CalibratorFlags(), int device = -1) : FLAGS_(flags) {
    vcgpu_config cfg;
    cfg.device = device;
    const int rc = vcgpu_create(&cfg, &h_);
    if (rc != VCGPU_OK) throw std::runtime_error("vcgpu_create failed: a CUDA device is required (no CPU fallback)");
    vcgpu_default_options(&opts_);
    opts_.max_iters = FLAGS_.max_iters;  // vicalibrator.h:142
    opts_.function_tol = 1e-6;           // vicalibrator.h:149
    opts_.strategy = FLAGS_.trust_region_strategy;
    Clear();
  }
  virtual ~ViCalibrator() {
    Stop();
    vcgpu_destroy(h_);
  }

  std::vector<double> GetCameraProjRMSE() const { return camera_proj_rmse_; }  // :160

  // Write XML file containing configuration of camera rig (vicalibrator.h:208-229; Calibu WriteXmlRig)
  void WriteCameraModels(const std::string& filename) {
    std::ofstream of(filename.c_str());
    of << std::setprecision(17);
    of << "<rig>\n";
    for (size_t c = 0; c < cameras_.size(); ++c) {
      CameraInterface& cam = *cameras_[c]->camera;
      if (FLAGS_.calibrate_imu) {  // :214-219
        cam.SetRDF(kRdfRobotics);
        double Rt[9];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Rt[i * 3 + j] = kRdfRobotics[j * 3 + i];
        cam.SetPose(cameras_[c]->T_ck.inverse() * SE3d::FromRotation(Rt));
      } else {  // :221-224
        cam.SetRDF(kRdfVision);
        cam.SetPose(cameras_[c]->T_ck.inverse());
      }
      const double* R = cam.RDF();
      double M[12];
      cam.Pose().matrix3x4(M);
      of << "    <camera>\n        <camera_model name=\"\" index=\"" << c << "\" serialno=\"0\" type=\"" << cam.Type()
         << "\" version=\"8\">\n";
      of << "            <width> " << cam.Width() << " </width>\n            <height> " << cam.Height() << " </height>\n";
      // right / down / forward = columns of the RDF matrix
      of << "            <right> [ " << R[0] << "; " << R[3] << "; " << R[6] << " ] </right>\n";
      of << "            <down> [ " << R[1] << "; " << R[4] << "; " << R[7] << " ] </down>\n";
      of << "            <forward> [ " << R[2] << "; " << R[5] << "; " << R[8] << " ] </forward>\n";
      of << "            <params> [ ";
      for (size_t k = 0; k < cam.GetParams().size(); ++k) of << cam.GetParams()[k] << (k + 1 < cam.GetParams().size() ? "; " : " ");
      of << "] </params>\n        </camera_model>\n        <pose>\n            <T_wc> [ ";
      for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 4; ++j) of << M[i * 4 + j] << (j < 3 ? ", " : "");
        of << (i < 2 ? "; " : " ");
      }
      of << "] </T_wc>\n        </pose>\n    </camera>\n";
    }
    of << "</rig>\n";
  }

  void Clear() {  // :232-249
    Stop();
    t_wk_.clear();
    cameras_.clear();
    obs_frame_.clear(); obs_cam_.clear(); obs_pw_.clear(); obs_pc_.clear();
    imu_.clear();
    mse_ = 0;
    num_iterations_ = 0;
    is_bias_active_ = false;
    is_scale_factor_active_ = false;
    is_inertial_active_ = false;
    is_visual_active_ = true;
    optimize_rotation_only_ = true;
    is_finished_ = false;
    is_gravity_initialized_ = false;
    outliers_removed_ = false;
    num_solves_ = 0;
    // the device still holds the previous problem: the next SetupProblem must upload observations / IMU samples again
    // and restart the residual-block multiplicities (the reference resets num_imu_residuals_ and proj_costs_, :236-241)
    problem_uploaded_ = false;
    visual_adds_ = imu_adds_ = 0;
    n_removed_ = 0;
    stopped_by_user_ = false;
    g_[0] = g_[1] = 0;
    time_offset_ = 0;
    for (int i = 0; i < 6; ++i) { biases_[i] = 0; scale_factors_[i] = 1; }
  }

  void SetOptimizationFlags(bool bias_active, bool inertial_active, bool rotation_only, bool optimize_imu_time_offset) {  // :252-260
    VICALIB_CHECK(!is_running_, "SetOptimizationFlags while running");
    is_scale_factor_active_ = bias_active;
    is_bias_active_ = bias_active;
    is_inertial_active_ = inertial_active;
    optimize_rotation_only_ = rotation_only;
    optimize_time_offset_ = optimize_imu_time_offset;
  }

  void Start() {  // :263-274
    if (!is_running_) {
      should_run_ = true;
      stopped_by_user_ = false;
      is_running_ = true;
      pthread_create(&thread_, NULL, &ViCalibrator::SolveThreadStatic, this);
      thread_valid_ = true;
    } else {
      std::fprintf(stderr, "Already Running.\n");
    }
  }
  void SetFunctionTolerance(double tolerance) { VICALIB_CHECK(!is_running_, ""); opts_.function_tol = tolerance; }  // :277
  unsigned int GetNumIterations() { return num_iterations_; }                                                       // :283
  Vector6d GetBiases() const { return biases_; }                                                                     // :286
  void SetSigmas(double gyro_sigma, double accel_sigma) { VICALIB_CHECK(!is_running_, ""); gyro_sigma_ = gyro_sigma; accel_sigma_ = accel_sigma; }  // :290
  void SetTimeOffset(double offset) { time_offset_ = offset; }                                                       // :296
  void SetBiases(const Vector6d& b) { VICALIB_CHECK(!is_running_, ""); biases_ = b; }                                // :301
  Vector6d GetScaleFactor() { return scale_factors_; }                                                               // :306
  void SetScaleFactor(const Vector6d& s) { VICALIB_CHECK(!is_running_, ""); scale_factors_ = s; }                    // :308
  bool IsRunning() { return is_running_ && !is_finished_; }                                                          // :314
  void Stop() {                                                                                                      // :317-328
    if (thread_valid_) {
      should_run_ = false;
      pthread_join(thread_, NULL);
      thread_valid_ = false;
    }
  }

  int AddCamera(const std::shared_ptr<CameraInterface>& cam, const SE3d& t_ck = SE3d()) {  // :332-342
    VICALIB_CHECK(!is_running_, "AddCamera while running");
    const int id = static_cast<int>(cameras_.size());
    cameras_.push_back(std::unique_ptr<CameraAndPose>(new CameraAndPose(cam, t_ck)));
    cameras_.back()->camera->SetIndex(id);
    camera_proj_rmse_.resize(cameras_.size());
    return id;
  }
  void FixCameraIntrinsics(bool should_fix = true) { VICALIB_CHECK(!is_running_, ""); fix_intrinsics_ = should_fix; }  // :346

  int AddFrame(const SE3d& t_wk, double time) {  // :355-367
    VICALIB_CHECK(!is_running_, "AddFrame while running");
    pthread_mutex_lock(&update_mutex_);
    const int id = AddFrameUnlocked(t_wk, time);
    pthread_mutex_unlock(&update_mutex_);
    return id;
  }
  bool AddImuMeasurements(const Vector3d& gyro, const Vector3d& accel, double time) {  // :370-380
    VICALIB_CHECK(!is_running_, "AddImuMeasurements while running");
    VICALIB_CHECK(imu_.empty() || time > imu_.back().time, "Timestamps are not unique!");
    imu_.push_back(ImuMeasurement{gyro, accel, time});
    return true;
  }
  void AddObservation(size_t frame, size_t camera_id, const Vector3d& p_w, const Vector2d& p_c, double time) {  // :385-468
    VICALIB_CHECK(!is_running_, "AddObservation while running");
    pthread_mutex_lock(&update_mutex_);
    while (NumFrames() < frame) AddFrameUnlocked(SE3d(), time);  // :392-394 (the reference would self-deadlock here)
    VICALIB_CHECK(camera_id < NumCameras(), "camera_id out of range");  // :396
    VICALIB_CHECK(frame < NumFrames(), "frame out of range");
    t_wk_[frame]->SetHasMeasurementsFromCam(camera_id, true);
    obs_frame_.push_back(static_cast<int32_t>(frame));
    obs_cam_.push_back(static_cast<int32_t>(camera_id));
    obs_pw_.insert(obs_pw_.end(), p_w.begin(), p_w.end());
    obs_pc_.insert(obs_pc_.end(), p_c.begin(), p_c.end());
    pthread_mutex_unlock(&update_mutex_);
  }

  size_t NumFrames() const { return t_wk_.size(); }                       // :471
  double time_offset() const { return time_offset_; }                     // :474
  std::shared_ptr<VicalibFrame> GetFrame(size_t i) { VICALIB_CHECK(i < t_wk_.size(), "GetFrame()"); return t_wk_[i]; }  // :477
  size_t NumCameras() const { return cameras_.size(); }                   // :484
  const std::vector<ImuMeasurement>& imu_buffer() { return imu_; }        // :487
  CameraAndPose& GetCamera(size_t i) { VICALIB_CHECK(i < cameras_.size(), "GetCamera()"); return *cameras_[i]; }  // :492
  double MeanSquaredError() const { return mse_; }                        // :506
  const double* gravity_angles() const { return g_; }
  int num_solves() const { return num_solves_; }
  int64_t num_outliers_removed() const { return n_removed_; }

  // The poses the IMU integration passes through between frame `id` and frame `id + 1` with the current
  // biases / scale factors / gravity / time offset (vicalibrator.h:508-533; ImuResidualT::IntegrateResidual,
  // types.h:611-687, double branch of IntegrateImu :575-590).  Host-side: the GUI polls it while drawing.
  std::vector<ImuPose> GetIntegrationPoses(unsigned int id) {
    std::vector<ImuPose> poses;
    if (!(is_inertial_active_ && !optimize_rotation_only_)) return poses;
    if (static_cast<size_t>(id) + 1 >= t_wk_.size()) return poses;  // the reference reads t_wk_[id + 1] unchecked (:517)
    const VicalibFrame& f0 = *t_wk_[id];
    const VicalibFrame& f1 = *t_wk_[id + 1];
    std::vector<ImuMeasurement> meas;
    GetRange(f0.time_, f1.time_, time_offset_, &meas);
    if (meas.empty()) return poses;
    const double sp = std::sin(g_[0]), cp = std::cos(g_[0]), sq = std::sin(g_[1]), cq = std::cos(g_[1]);
    const double gv[3] = {-9.8007 * cp * sq, 9.8007 * sp, -9.8007 * cp * cq};  // GetGravityVector, types.h:93-104
    ImuPose y;
    y.t_wp_ = f0.t_wp_;
    y.v_w_ = f0.v_w_;
    y.time_ = f0.time_;
    poses.push_back(y);
    for (size_t i = 1; i < meas.size(); ++i) {
      y = IntegrateImu(y, meas[i - 1], meas[i], gv);
      poses.push_back(y);
    }
    return poses;
  }

  // GetSolutionCovariance (vicalibrator.h:802-857, behind COMPUTE_VICALIB_COVARIANCE upstream): covariance of the
  // calibration parameters at the current solution, tangent space, G x G row-major — per camera (w_ck 3 | p_ck 3 |
  // intrinsics K), then (g 2 | b 6 | sf 6 | ts 1) when the inertial terms are on; constant blocks have zero rows /
  // columns (ceres::Covariance convention).  Call after the solve has finished (not while IsRunning()).
  std::vector<double> GetSolutionCovariance(int* n_globals = nullptr) {
    int G = 0;
    Check(vcgpu_num_globals(h_, &G), "num_globals");
    std::vector<double> cov(static_cast<size_t>(G) * G, 0.0);
    Check(vcgpu_get_covariance(h_, cov.data()), "get_covariance");
    if (n_globals) *n_globals = G;
    return cov;
  }

  // GetCovarianceBlock(t_wp, t_wp) for every frame, and (v_w, v_w) when the inertial terms are on: the marginal
  // covariance of each frame's tangent at the current solution, NumFrames() blocks of fd x fd row-major (fd: 6 | 9, the
  // frame's rows of the normal equations).  A frame no active observation sees has a zero block.  Call after the solve
  // has finished (not while IsRunning()).
  std::vector<double> GetFrameCovariance(int* frame_dim = nullptr) {
    int fd = 0;
    Check(vcgpu_frame_dim(h_, &fd), "frame_dim");
    std::vector<double> cov(NumFrames() * fd * fd, 0.0);
    Check(vcgpu_get_frame_covariance(h_, cov.data()), "get_frame_covariance");
    if (frame_dim) *frame_dim = fd;
    return cov;
  }

  // GetCovarianceBlock(t_wp[f], calibration) and (t_wp[f], t_wp[f+1]) for every frame, with v_w likewise when the
  // inertial terms are on: *frame_globals gets NumFrames() blocks of fd x G row-major (rows as GetFrameCovariance's,
  // columns as GetSolutionCovariance's), *frame_next NumFrames() - 1 blocks of fd x fd (rows frame f, columns frame
  // f+1); either may be null, not both.  With GetFrameCovariance, the covariance of the motion from frame f to f+1 is
  // S_ff + S_f+1,f+1 - S_f,f+1 - S_f,f+1^T.  Call after the solve has finished (not while IsRunning()).
  void GetFrameCrossCovariance(std::vector<double>* frame_globals, std::vector<double>* frame_next, int* frame_dim = nullptr,
                               int* n_globals = nullptr) {
    int fd = 0, G = 0;
    Check(vcgpu_frame_dim(h_, &fd), "frame_dim");
    Check(vcgpu_num_globals(h_, &G), "num_globals");
    const size_t nf = NumFrames();
    if (frame_globals) frame_globals->assign(nf * fd * G, 0.0);
    if (frame_next) frame_next->assign((nf > 0 ? nf - 1 : 0) * fd * fd, 0.0);
    Check(vcgpu_get_frame_cross_covariance(h_, frame_globals ? frame_globals->data() : nullptr, frame_next ? frame_next->data() : nullptr),
          "get_frame_cross_covariance");
    if (frame_dim) *frame_dim = fd;
    if (n_globals) *n_globals = G;
  }

  // The Mahalanobis distance UpdateImuWeights logs for each IMU interval against chi2inv(0.95, 9) = 16.919
  // (vicalibrator.h:786-794), at the current solution: NumFrames() - 1 entries, NaN for an interval with no measurements
  // (the reference logs nothing there) or whose covariance is not positive definite.  The inertial terms must be on.
  // Call after the solve has finished (not while IsRunning()).
  std::vector<double> GetImuMahalanobis() {
    const size_t nf = NumFrames();
    std::vector<double> dist(nf > 1 ? nf - 1 : 0, 0.0);
    Check(vcgpu_get_imu_mahalanobis(h_, dist.data(), nullptr), "get_imu_mahalanobis");
    return dist;
  }

  // The pixel covariance the calibration leaves at points of camera `cam`: pixels (u, v) interleaved, depth one distance
  // along each pixel's ray (empty: every point at infinity), the point fixed in the rig frame (rig_frame) or the camera
  // frame.  Three values per point, S_uu S_uv S_vv, for unit observation variance (scale by the residual variance); NaN
  // where a pixel lies outside the lens model's domain.  Call after the solve has finished (not while IsRunning()).
  std::vector<double> GetProjectionCovariance(int cam, const std::vector<double>& pixels, const std::vector<double>& depth,
                                              bool rig_frame) {
    const int64_t n = static_cast<int64_t>(pixels.size() / 2);
    std::vector<int32_t> cam_id(n, cam);
    std::vector<double> cov(3 * n, 0.0);
    const vcgpu_proj_points pts{n, cam_id.data(), pixels.data(), depth.empty() ? nullptr : depth.data(),
                                rig_frame ? VCGPU_PROJ_RIG : VCGPU_PROJ_CAMERA, cov.data(), nullptr};
    Check(vcgpu_get_projection_covariance(h_, nullptr, &pts), "get_projection_covariance");
    return cov;
  }

  // The information each candidate view of the target would add to the calibration (vcgpu_get_view_information):
  // T_wp holds 7 doubles (q | t) per candidate rig pose, p_w 3 per target point in the world frame, facing the target's
  // front normal (empty: every side is the front).  Each camera's image is its CameraInterface's Width() x Height().
  // Returns one gain per candidate, the entropy in nats the view removes from the globals (NaN where the view does not
  // fix its own pose); var (if not null) gets NumGlobals() posterior variances per candidate and n_seen (if not null)
  // the corners each camera sees.  Call after the solve has finished (not while IsRunning()).
  std::vector<double> GetViewInformation(const std::vector<double>& T_wp, const std::vector<double>& p_w,
                                         const std::vector<double>& facing = {}, std::vector<double>* var = nullptr,
                                         std::vector<int32_t>* n_seen = nullptr) {
    VICALIB_CHECK(!IsRunning(), "GetViewInformation while running");
    VICALIB_CHECK(facing.empty() || facing.size() == 3, "GetViewInformation: facing needs 3 values");
    const int64_t n = static_cast<int64_t>(T_wp.size() / 7);
    int G = 0;
    Check(vcgpu_num_globals(h_, &G), "num_globals");
    std::vector<int32_t> width, height, seen(static_cast<size_t>(n) * cameras_.size());
    for (const auto& c : cameras_) {
      width.push_back(c->camera->Width());
      height.push_back(c->camera->Height());
    }
    std::vector<double> gain(n);
    if (var) var->assign(static_cast<size_t>(n) * G, 0.0);
    const vcgpu_view_candidates v{n, T_wp.data(), static_cast<int>(p_w.size() / 3), p_w.data(),
                                  facing.empty() ? nullptr : facing.data(), width.data(), height.data(), seen.data(),
                                  gain.data(), var ? var->data() : nullptr, nullptr};
    Check(vcgpu_get_view_information(h_, nullptr, &v), "get_view_information");
    if (n_seen) *n_seen = seen;
    return gain;
  }

  // The regression diagnostics of every observation, active or removed, in upload order
  // (vcgpu_get_observation_influence): h 3 doubles per observation (H_uu, H_uv, H_vv of the leverage), stud the
  // studentized residual (a removed observation's predictive residual), infl the shift of the calibration its deletion
  // causes, measured in the calibration's covariance.  stud and infl assume unit observation variance.  Any output may
  // be null, not all three.  The outputs cover the observations the solve was given (the last upload), which after a
  // Clear() may differ from those added since.
  void GetObservationInfluence(std::vector<double>* h, std::vector<double>* stud, std::vector<double>* infl) {
    VICALIB_CHECK(!IsRunning(), "GetObservationInfluence while running");
    VICALIB_CHECK(h || stud || infl, "GetObservationInfluence: every output is null");
    const size_t n = n_uploaded_obs_;
    if (h) h->assign(3 * n, 0.0);
    if (stud) stud->assign(n, 0.0);
    if (infl) infl->assign(n, 0.0);
    vcgpu_obs_influence out{h ? h->data() : nullptr, stud ? stud->data() : nullptr, infl ? infl->data() : nullptr};
    Check(vcgpu_get_observation_influence(h_, &out), "get_observation_influence");
  }

  // The regression diagnostics of every IMU interval k < NumFrames() - 1 (vcgpu_get_imu_influence): h 81 doubles per
  // interval (its 9 x 9 leverage, row-major), stud the studentized residual, infl the shift of the calibration its
  // deletion causes, measured in the calibration's covariance.  stud and infl assume unit observation variance; NaN in
  // all three for an interval with no measurements.  Any output may be null, not all three.  The inertial terms must be
  // active in the handle's last solve.  Call after the solve has finished (not while IsRunning()).
  void GetImuInfluence(std::vector<double>* h, std::vector<double>* stud, std::vector<double>* infl) {
    VICALIB_CHECK(!IsRunning(), "GetImuInfluence while running");
    VICALIB_CHECK(h || stud || infl, "GetImuInfluence: every output is null");
    VICALIB_CHECK(FLAGS_.calibrate_imu && is_inertial_active_, "GetImuInfluence: the inertial terms are not active");
    const size_t nf = NumFrames(), ni = nf > 1 ? nf - 1 : 0;
    if (h) h->assign(81 * ni, 0.0);
    if (stud) stud->assign(ni, 0.0);
    if (infl) infl->assign(ni, 0.0);
    vcgpu_imu_influence out{h ? h->data() : nullptr, stud ? stud->data() : nullptr, infl ? infl->data() : nullptr};
    Check(vcgpu_get_imu_influence(h_, &out, nullptr), "get_imu_influence");
  }

  // The hand-eye alignment of the gyro stream with the frame poses (vcgpu_align_imu, applied): the rotation Q from the
  // IMU's axes to the rig's, the time offset and the gyro bias, from n_ts candidate offsets in [ts_lo, ts_hi] (without
  // find_time_offset the current offset is kept) and a Gauss-Newton refinement of at most max_iters steps.  On success
  // every camera's T_ck and every frame's rotation are right-multiplied by Q, and time_offset() and the gyro part of
  // GetBiases() take the result; camera poses T_wk T_ck^-1 do not change.  Returns the call's outputs; a fit that fails
  // (fewer than 3 usable intervals, a singular system) aborts as every other device error does.  Call between the
  // vision-only solve and the inertial stages, after the solve has finished (not while IsRunning()).
  vcgpu_imu_alignment AlignImu(double ts_lo, double ts_hi, int n_ts, bool find_time_offset, int max_iters = 20) {
    VICALIB_CHECK(!IsRunning(), "AlignImu while running");
    VICALIB_CHECK(problem_uploaded_, "AlignImu before the problem is on the device (run the vision solve first)");
    const vcgpu_imu_align_opts o{ts_lo, ts_hi, n_ts, find_time_offset ? 1 : 0, max_iters, 1};
    vcgpu_imu_alignment r{};
    Check(vcgpu_align_imu(h_, &o, &r), "align_imu");
    ReadBackState();
    return r;
  }

  // GetIntegrationPoses(k) for every k < NumFrames() - 1, computed on the device from the current solution: one vector
  // per interval, empty where the interval has no IMU measurements, and all empty unless the inertial terms are active
  // and the stage is not rotation-only (the reference's gate, vicalibrator.h:510).  Call after the solve has finished
  // (not while IsRunning()); GetIntegrationPoses stays the host-side call a GUI can poll during the solve.
  std::vector<std::vector<ImuPose>> GetAllIntegrationPoses() {
    VICALIB_CHECK(!IsRunning(), "GetAllIntegrationPoses while running");
    const size_t nf = NumFrames();
    std::vector<std::vector<ImuPose>> out(nf > 1 ? nf - 1 : 0);
    if (!(is_inertial_active_ && !optimize_rotation_only_) || nf < 2) return out;
    std::vector<int64_t> start(nf);
    Check(vcgpu_get_integration_poses(h_, start.data(), nullptr), "get_integration_poses");
    std::vector<double> p(static_cast<size_t>(start[nf - 1]) * 14);
    Check(vcgpu_get_integration_poses(h_, start.data(), p.data()), "get_integration_poses");
    for (size_t k = 0; k + 1 < nf; ++k)
      for (int64_t i = start[k]; i < start[k + 1]; ++i) {
        const double* o = p.data() + 14 * i;
        ImuPose y;
        std::memcpy(y.t_wp_.d, o, 7 * sizeof(double));
        for (int j = 0; j < 3; ++j) { y.v_w_[j] = o[7 + j]; y.w_w_[j] = o[10 + j]; }
        y.time_ = o[13];
        out[k].push_back(y);
      }
    return out;
  }

  // Pose seeds for AddFrame: what VicalibTask::AddSuperFrame computes per frame and camera with
  // calibu::PosePnPRansac(camera, ellipses, target.Circles3D(), ellipse_target_map, 0, 0, &t_cw) and
  // t_wp = t_cw.inverse() * t_ck (src/vicalib-task.cc:322-325, 341-349) — here for ALL views in one device call.
  // views[v] = (camera id, detected centres in pixels, their target points); the cameras must have been added.
  // Returns one T_wp per view (identity with ok[v] = false when fewer than 4 usable correspondences).
  struct PnpView {
    int camera_id;
    std::vector<Vector2d> pixels;
    std::vector<Vector3d> target_points;
  };
  std::vector<SE3d> InitialPosesFromTarget(const std::vector<PnpView>& views, std::vector<bool>* ok = nullptr, int robust_its = 0,
                                           double robust_tol = 0.0) {
    UploadCameras();
    std::vector<int32_t> cam(views.size()), count(views.size());
    std::vector<int64_t> start(views.size());
    std::vector<double> pix, pw;
    for (size_t v = 0; v < views.size(); ++v) {
      VICALIB_CHECK(views[v].pixels.size() == views[v].target_points.size(), "one target point per detected centre");
      cam[v] = views[v].camera_id;
      start[v] = static_cast<int64_t>(pix.size() / 2);
      count[v] = static_cast<int32_t>(views[v].pixels.size());
      for (size_t k = 0; k < views[v].pixels.size(); ++k) {
        pix.push_back(views[v].pixels[k][0]); pix.push_back(views[v].pixels[k][1]);
        for (int q = 0; q < 3; ++q) pw.push_back(views[v].target_points[k][q]);
      }
    }
    std::vector<double> T_cw(views.size() * 7, 0.0);
    std::vector<int32_t> used(views.size(), 0);
    Check(vcgpu_pose_pnp_ransac(h_, static_cast<int>(views.size()), cam.data(), start.data(), count.data(), pix.data(), pw.data(),
                                robust_its, robust_tol, T_cw.data(), nullptr, used.data()), "pose_pnp_ransac");
    std::vector<SE3d> out(views.size());
    if (ok) ok->assign(views.size(), false);
    for (size_t v = 0; v < views.size(); ++v) {
      if (used[v] < 4) continue;
      const SE3d t_cw(&T_cw[7 * v], &T_cw[7 * v + 4]);
      out[v] = t_cw.inverse() * cameras_[views[v].camera_id]->T_ck;
      if (ok) (*ok)[v] = true;
    }
    return out;
  }

  void PrintResults() {  // :536-544
    std::printf("------------------------------------------\n");
    for (size_t c = 0; c < cameras_.size(); ++c) {
      std::printf("Camera: %zu\n", c);
      for (double v : cameras_[c]->camera->GetParams()) std::printf("%.10g ", v);
      double M[12];
      cameras_[c]->T_ck.matrix3x4(M);
      std::printf("\n");
      for (int i = 0; i < 3; ++i) std::printf("%.10g %.10g %.10g %.10g\n", M[i * 4], M[i * 4 + 1], M[i * 4 + 2], M[i * 4 + 3]);
    }
  }

 protected:
  int AddFrameUnlocked(const SE3d& t_wk, double time) {
    const int id = static_cast<int>(t_wk_.size());
    std::shared_ptr<VicalibFrame> f(new VicalibFrame());
    f->t_wp_ = t_wk;
    f->time_ = time;
    t_wk_.push_back(f);
    return id;
  }
  void Check(int rc, const char* what) {
    if (rc != VCGPU_OK) throw std::runtime_error(std::string(what) + ": " + vcgpu_last_error(h_));
  }

  // the cameras alone (models, intrinsics, T_ck): what the pose initialisation needs before any frame exists
  void UploadCameras() {
    const int nc = static_cast<int>(cameras_.size());
    VICALIB_CHECK(nc > 0, "no camera added");
    std::vector<int32_t> model(nc);
    std::vector<double> intr(10 * static_cast<size_t>(nc), 0.0), q(4 * static_cast<size_t>(nc)), p(3 * static_cast<size_t>(nc));
    for (int c = 0; c < nc; ++c) {
      model[c] = cameras_[c]->camera->ModelId();
      const std::vector<double>& pr = cameras_[c]->camera->GetParams();
      std::copy(pr.begin(), pr.end(), intr.begin() + 10 * c);
      std::memcpy(&q[4 * c], cameras_[c]->T_ck.d, 4 * sizeof(double));
      std::memcpy(&p[3 * c], cameras_[c]->T_ck.d + 4, 3 * sizeof(double));
    }
    Check(vcgpu_set_cameras(h_, nc, model.data(), intr.data(), q.data(), p.data()), "set_cameras");
  }

  // SetupProblem (vicalibrator.h:548-679): hand the parameter blocks, residual data and masks to the device
  void SetupProblem() {
    pthread_mutex_lock(&update_mutex_);
    const int nc = static_cast<int>(cameras_.size()), nf = static_cast<int>(t_wk_.size());
    std::vector<int32_t> model(nc);
    std::vector<double> intr(10 * nc, 0.0), q(4 * nc), p(3 * nc), T(7 * nf), v(3 * nf), tm(nf);
    for (int c = 0; c < nc; ++c) {
      model[c] = cameras_[c]->camera->ModelId();
      const std::vector<double>& pr = cameras_[c]->camera->GetParams();
      std::copy(pr.begin(), pr.end(), intr.begin() + 10 * c);
      std::memcpy(&q[4 * c], cameras_[c]->T_ck.d, 4 * sizeof(double));
      std::memcpy(&p[3 * c], cameras_[c]->T_ck.d + 4, 3 * sizeof(double));
    }
    for (int f = 0; f < nf; ++f) {
      std::memcpy(&T[7 * f], t_wk_[f]->t_wp_.d, 7 * sizeof(double));
      std::memcpy(&v[3 * f], t_wk_[f]->v_w_.data(), 3 * sizeof(double));
      tm[f] = t_wk_[f]->time_;
    }
    Check(vcgpu_set_cameras(h_, nc, model.data(), intr.data(), q.data(), p.data()), "set_cameras");
    Check(vcgpu_set_frames(h_, nf, T.data(), v.data(), tm.data()), "set_frames");
    if (!problem_uploaded_) {  // residual blocks are added once; later stages only change masks / multiplicities
      Check(vcgpu_set_observations(h_, static_cast<int64_t>(obs_frame_.size()), obs_frame_.data(), obs_cam_.data(),
                                   obs_pw_.data(), obs_pc_.data()), "set_observations");
      n_uploaded_obs_ = obs_frame_.size();
      std::vector<double> t(imu_.size()), w(3 * imu_.size()), a(3 * imu_.size());
      for (size_t i = 0; i < imu_.size(); ++i) {
        t[i] = imu_[i].time;
        for (int k = 0; k < 3; ++k) { w[3 * i + k] = imu_[i].w_[k]; a[3 * i + k] = imu_[i].a_[k]; }
      }
      Check(vcgpu_set_imu(h_, static_cast<int>(imu_.size()), t.data(), w.data(), a.data(), gyro_sigma_, accel_sigma_), "set_imu");
      problem_uploaded_ = true;
    }
    Check(vcgpu_set_imu_params(h_, g_, biases_.data(), scale_factors_.data(), time_offset_), "set_imu_params");
    vcgpu_flags fl;
    vcgpu_default_flags(&fl);
    fl.inertial = (FLAGS_.calibrate_imu && is_inertial_active_) ? 1 : 0;  // :651
    fl.rotation_only = optimize_rotation_only_ ? 1 : 0;
    fl.bias_active = is_bias_active_ ? 1 : 0;
    fl.scale_active = is_scale_factor_active_ ? 1 : 0;
    fl.optimize_ts = optimize_time_offset_ ? 1 : 0;
    fl.fix_intrinsics = fix_intrinsics_ ? 1 : 0;
    fl.visual = is_visual_active_ ? 1 : 0;
    // SetupProblem re-adds every residual block at each stage without removing the old ones
    // (vicalibrator.h:641-656, SURVEY §0.5): visual blocks appear 1x,2x,3x,... and IMU blocks 0x,1x,2x,...
    if (emulate_block_duplication_) {
      ++visual_adds_;
      if (fl.inertial) ++imu_adds_;
      fl.visual_mult = visual_adds_;
      fl.imu_mult = imu_adds_ > 0 ? imu_adds_ : 1;
    }
    Check(vcgpu_set_flags(h_, &fl), "set_flags");
    Check(vcgpu_set_options(h_, &opts_), "set_options");
    pthread_mutex_unlock(&update_mutex_);
  }

  void ReadBackState() {
    const int nc = static_cast<int>(cameras_.size()), nf = static_cast<int>(t_wk_.size());
    std::vector<double> intr(10 * nc), q(4 * nc), p(3 * nc), T(7 * nf), v(3 * nf);
    Check(vcgpu_get_state(h_, intr.data(), q.data(), p.data(), T.data(), v.data(), g_, biases_.data(), scale_factors_.data(),
                          &time_offset_), "get_state");
    for (int c = 0; c < nc; ++c) {
      std::vector<double>& pr = cameras_[c]->camera->GetParams();
      std::copy(intr.begin() + 10 * c, intr.begin() + 10 * c + pr.size(), pr.begin());
      std::memcpy(cameras_[c]->T_ck.d, &q[4 * c], 4 * sizeof(double));
      std::memcpy(cameras_[c]->T_ck.d + 4, &p[3 * c], 3 * sizeof(double));
    }
    for (int f = 0; f < nf; ++f) {
      std::memcpy(t_wk_[f]->t_wp_.d, &T[7 * f], 7 * sizeof(double));
      std::memcpy(t_wk_[f]->v_w_.data(), &v[3 * f], 3 * sizeof(double));
    }
  }

  static int IterationCallback(const vcgpu_iteration* it, void* user) {  // vicalibrator.h:690-721
    ViCalibrator* self = static_cast<ViCalibrator*>(user);
    ++self->num_iterations_;
    if (self->num_residuals_ > 0) self->mse_ = it->cost / self->num_residuals_;
    if (!self->should_run_) self->stopped_by_user_ = true;  // Stop(): abort the solve (the reference lets Ceres finish)
    return self->should_run_ ? 0 : 1;  // UpdateImuWeights and the gradient-norm rule run on the device
  }

  static void* SolveThreadStatic(void* p) {
    static_cast<ViCalibrator*>(p)->SolveThread();
    return NULL;
  }

  // vicalibrator.h:919-1040
  void SolveThread() {
    is_running_ = true;
    try {
      while (should_run_ && !is_finished_) {
        SetupProblem();
        // gravity initialisation from the mid-frame accelerometer sample (:927-949)
        if (is_inertial_active_ && !optimize_rotation_only_ && !is_gravity_initialized_ && !imu_.empty()) {
          const VicalibFrame& fr = *t_wk_[t_wk_.size() / 2];
          const Vector3d a = InterpolateAccel(fr.time_);
          const double n = std::sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
          double R[9];
          fr.t_wp_.rotation(R);
          const double gb[3] = {a[0] / n, a[1] / n, a[2] / n};
          const double gw[3] = {R[0] * gb[0] + R[1] * gb[1] + R[2] * gb[2], R[3] * gb[0] + R[4] * gb[1] + R[5] * gb[2],
                                R[6] * gb[0] + R[7] * gb[1] + R[8] * gb[2]};
          const double pp = std::asin(gw[1]);
          g_[0] = pp;
          g_[1] = std::asin(-gw[0] / std::cos(pp));
          is_gravity_initialized_ = true;
          Check(vcgpu_set_imu_params(h_, g_, biases_.data(), scale_factors_.data(), time_offset_), "set_imu_params");
        }
        Check(vcgpu_num_residuals(h_, &num_residuals_), "num_residuals");
        while (num_residuals_ > 0 && should_run_ && !is_finished_) {
          vcgpu_summary summary;
          Check(vcgpu_solve(h_, &ViCalibrator::IterationCallback, this, &summary), "solve");  // :956
          ++num_solves_;
          ReadBackState();
          for (size_t c = 0; c < cameras_.size(); ++c) {  // :958-971
            double cost = 0;
            int64_t n = 0;
            Check(vcgpu_evaluate(h_, static_cast<int>(c), &cost, NULL, &n), "evaluate");
            camera_proj_rmse_[c] = n > 0 ? std::sqrt(cost / n) : 0.0;
          }
          mse_ = summary.num_residuals > 0 ? summary.final_cost / summary.num_residuals : 0.0;  // :975
          // a solve cut short by Stop() must not advance the stage machine (it did not converge; the reference's
          // Stop() never interrupts ceres::Solve)
          if (stopped_by_user_) break;
          const bool converged = summary.termination != VCGPU_TERM_NO_CONVERGENCE;
          if (converged && FLAGS_.calibrate_imu) {  // :976-1022
            if (!is_inertial_active_) {
              is_inertial_active_ = true;
            } else if (optimize_rotation_only_) {
              optimize_rotation_only_ = false;
              is_bias_active_ = true;
            } else if (!is_scale_factor_active_) {
              is_scale_factor_active_ = true;
            } else if (FLAGS_.remove_outliers && !outliers_removed_) {
              RemoveOutliers();
              outliers_removed_ = true;
            } else {
              PrintResults();
              is_finished_ = true;
            }
            break;
          } else if (converged) {  // :1023-1031
            if (FLAGS_.remove_outliers && !outliers_removed_) {
              RemoveOutliers();
              outliers_removed_ = true;
            } else {
              is_finished_ = true;
            }
          }
        }
      }
    } catch (const std::exception& e) {  // :1033-1035 (the reference logs and retries; a device error is fatal here)
      std::fprintf(stderr, "ViCalibrator: %s\n", e.what());
      is_finished_ = true;
    }
    is_running_ = false;
  }

  // InterpolationBufferT::GetRange (interpolation-buffer.h:208-226): [element(start), samples inside, element(end)],
  // sample i valid at time_i + offset
  void GetRange(double t0, double t1, double off, std::vector<ImuMeasurement>* out) const {
    if (imu_.empty() || !(t0 >= imu_.front().time + off && t0 <= imu_.back().time + off)) return;
    auto element = [&](double t, size_t* idx) {
      ImuMeasurement m;
      if (imu_.front().time + off > t) { m = imu_.front(); m.time += off; *idx = 0; return m; }
      size_t i = 0;
      while (i + 1 < imu_.size() && imu_[i + 1].time + off < t) ++i;
      if (i + 1 >= imu_.size()) { m = imu_.back(); m.time += off; *idx = imu_.size() - 1; return m; }
      const double ta = imu_[i].time + off, tb = imu_[i + 1].time + off, f = (t - ta) / (tb - ta);
      for (int k = 0; k < 3; ++k) {
        m.w_[k] = imu_[i].w_[k] * (1 - f) + imu_[i + 1].w_[k] * f;
        m.a_[k] = imu_[i].a_[k] * (1 - f) + imu_[i + 1].a_[k] * f;
      }
      m.time = t;
      *idx = i;
      return m;
    };
    size_t idx = 0;
    out->push_back(element(t0, &idx));
    while (idx + 1 < imu_.size() && !(imu_[idx + 1].time + off > t1)) {
      ImuMeasurement m = imu_[++idx];
      m.time += off;
      out->push_back(m);
    }
    out->push_back(element(t1, &idx));
  }
  // GetPoseDerivative (types.h:380-425, value only)
  void PoseDerivative(const ImuPose& y, const ImuMeasurement& z0, const ImuMeasurement& z1, double dt, const double gv[3],
                      double k[9]) const {
    const double alpha = (z1.time - (z0.time + dt)) / (z1.time - z0.time);
    double R[9], w[3], a[3];
    y.t_wp_.rotation(R);
    for (int i = 0; i < 3; ++i) {
      w[i] = (z0.w_[i] * alpha + z1.w_[i] * (1.0 - alpha)) * scale_factors_[i] + biases_[i];
      a[i] = (z0.a_[i] * alpha + z1.a_[i] * (1.0 - alpha)) * scale_factors_[3 + i] + biases_[3 + i];
    }
    for (int i = 0; i < 3; ++i) {
      k[i] = y.v_w_[i];
      k[3 + i] = R[i * 3] * w[0] + R[i * 3 + 1] * w[1] + R[i * 3 + 2] * w[2];
      k[6 + i] = R[i * 3] * a[0] + R[i * 3 + 1] * a[1] + R[i * 3 + 2] * a[2] - gv[i];
    }
  }
  // IntegratePose (types.h:330-378, value only): p += k_v dt, q <- exp(k_w dt) * q (no renormalisation), v += k_a dt
  static ImuPose IntegratePose(const ImuPose& y0, const double k[9], double dt) {
    ImuPose y = y0;
    const double wx = k[3] * dt, wy = k[4] * dt, wz = k[5] * dt, th2 = wx * wx + wy * wy + wz * wz, th = std::sqrt(th2);
    double imag, real;
    if (th < 1e-10) { imag = 0.5 - th2 / 48.0; real = 1.0 - th2 / 8.0; }
    else { imag = std::sin(0.5 * th) / th; real = std::cos(0.5 * th); }
    const double e[4] = {imag * wx, imag * wy, imag * wz, real};
    const double* q = y0.t_wp_.d;
    y.t_wp_.d[0] = e[3] * q[0] + e[0] * q[3] + e[1] * q[2] - e[2] * q[1];
    y.t_wp_.d[1] = e[3] * q[1] + e[1] * q[3] + e[2] * q[0] - e[0] * q[2];
    y.t_wp_.d[2] = e[3] * q[2] + e[2] * q[3] + e[0] * q[1] - e[1] * q[0];
    y.t_wp_.d[3] = e[3] * q[3] - e[0] * q[0] - e[1] * q[1] - e[2] * q[2];
    for (int i = 0; i < 3; ++i) {
      y.t_wp_.d[4 + i] += k[i] * dt;
      y.v_w_[i] += k[6 + i] * dt;
    }
    return y;
  }
  // IntegrateImu, RK4 (types.h:575-594)
  ImuPose IntegrateImu(const ImuPose& y0, const ImuMeasurement& z0, const ImuMeasurement& z1, const double gv[3]) const {
    const double dt = z1.time - z0.time;
    if (dt == 0) return y0;
    double k1[9], k2[9], k3[9], k4[9], k[9];
    PoseDerivative(y0, z0, z1, 0.0, gv, k1);
    PoseDerivative(IntegratePose(y0, k1, dt * 0.5), z0, z1, dt / 2, gv, k2);
    PoseDerivative(IntegratePose(y0, k2, dt * 0.5), z0, z1, dt / 2, gv, k3);
    PoseDerivative(IntegratePose(y0, k3, dt), z0, z1, dt, gv, k4);
    for (int i = 0; i < 9; ++i) k[i] = k1[i] + 2 * k2[i] + 2 * k3[i] + k4[i];
    ImuPose res = IntegratePose(y0, k, dt / 6.0);
    for (int i = 0; i < 3; ++i) res.w_w_[i] = k[3 + i];
    res.time_ = z1.time;
    return res;
  }

  void RemoveOutliers() {  // :859-916
    int64_t n = 0;
    Check(vcgpu_remove_outliers(h_, camera_proj_rmse_.data(), FLAGS_.outlier_threshold, &n), "remove_outliers");
    n_removed_ += n;
  }

  // InterpolationBufferT::GetElement(time) with zero offset (interpolation-buffer.h:160-203): the first / last
  // element outside the buffer's time span, linear interpolation between the two neighbours inside it
  Vector3d InterpolateAccel(double time) const {
    if (imu_.empty()) return Vector3d{{0, 0, 0}};
    if (!(imu_.front().time < time)) return imu_.front().a_;
    if (!(time < imu_.back().time)) return imu_.back().a_;
    size_t i = 0;
    while (i + 2 < imu_.size() && imu_[i + 1].time < time) ++i;
    const double f = (time - imu_[i].time) / (imu_[i + 1].time - imu_[i].time);
    Vector3d a;
    for (int k = 0; k < 3; ++k) a[k] = imu_[i].a_[k] * (1 - f) + imu_[i + 1].a_[k] * f;
    return a;
  }

 public:
  // The staged flow of the reference re-adds residual blocks (SURVEY §0.5); on by default for
  // bug-compatibility, off gives every block weight 1 in every stage.
  void SetEmulateBlockDuplication(bool on) { emulate_block_duplication_ = on; }
  vcgpu_handle* handle() { return h_; }

 protected:
  CalibratorFlags FLAGS_;
  vcgpu_handle* h_ = nullptr;
  vcgpu_options opts_;
  pthread_mutex_t update_mutex_ = PTHREAD_MUTEX_INITIALIZER;
  pthread_t thread_;
  bool thread_valid_ = false;
  volatile bool should_run_ = false, is_running_ = false, stopped_by_user_ = false;
  bool fix_intrinsics_ = false, problem_uploaded_ = false, emulate_block_duplication_ = true;
  size_t n_uploaded_obs_ = 0;  // observations the handle holds (GetObservationInfluence's output size); Clear() keeps it
  int visual_adds_ = 0, imu_adds_ = 0;
  std::vector<std::shared_ptr<VicalibFrame> > t_wk_;
  std::vector<std::unique_ptr<CameraAndPose> > cameras_;
  std::vector<int32_t> obs_frame_, obs_cam_;
  std::vector<double> obs_pw_, obs_pc_;
  std::vector<ImuMeasurement> imu_;
  std::vector<double> camera_proj_rmse_;
  double g_[2] = {0, 0}, time_offset_ = 0;
  Vector6d biases_{{0, 0, 0, 0, 0, 0}}, scale_factors_{{1, 1, 1, 1, 1, 1}};
  double gyro_sigma_ = 5.3088444e-5, accel_sigma_ = 0.001883649;  // types.h:34-35
  unsigned int num_iterations_ = 0;
  int num_residuals_ = 0, num_solves_ = 0;
  int64_t n_removed_ = 0;
  bool is_bias_active_ = false, is_scale_factor_active_ = false, is_inertial_active_ = false, is_visual_active_ = true;
  bool optimize_rotation_only_ = true, is_gravity_initialized_ = false, outliers_removed_ = false, optimize_time_offset_ = true;
  volatile bool is_finished_ = false;
  double mse_ = 0;
};

}  // namespace visual_inertial_calibration
#endif  // VICALIB_B200_HOST_VICALIBRATOR_H_
