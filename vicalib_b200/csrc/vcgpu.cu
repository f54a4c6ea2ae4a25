// libvcgpu.so — host side of the C-ABI declared in include/vcgpu.h.
//
// Replaces, for ViCalibrator, what ceres::Problem + ceres::Solve + Problem::Evaluate do
// (vicalibrator.h:152, 548-679, 859-916, 956-971).  The trust-region loop below is the Ceres
// loop (TrustRegionMinimizer + LevenbergMarquardtStrategy, SURVEY App. A.3) driven from the host
// with every arithmetic step — the accept/reject decision included — on the device; the candidate
// point is evaluated *with* its Jacobian blocks (speculatively) so an accepted step needs no second
// pass.  Engines: vc_mega.cuh (persistent kernel, vision solves) and vc_engine.inl (multi-launch).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <tuple>

#include <nccl.h>

#include "vc_internal.h"
#include "vc_kernels.cuh"
#include "vc_imu.cuh"
#include "vc_chain.cuh"
#include "vc_fused.cuh"
#include "vc_peak.cuh"
#include "vc_mega.cuh"
#include "vc_dogleg.cuh"
#include "vc_imu_weights.cuh"
#include "vc_imu_mega.cuh"
#include "vc_imu_eval_mega.cuh"
#include "vc_pnp.cuh"

using namespace vc;

#define CUDA_TRY(h, expr)                                                                   \
  do {                                                                                      \
    cudaError_t e__ = (expr);                                                               \
    if (e__ != cudaSuccess) {                                                               \
      (h)->err = std::string(#expr) + ": " + cudaGetErrorString(e__);                       \
      return VCGPU_ERR_CUDA;                                                                \
    }                                                                                       \
  } while (0)
#define VC_TRY(expr)                 \
  do {                               \
    int rc__ = (expr);               \
    if (rc__ != VCGPU_OK) return rc__; \
  } while (0)

static int fail(vcgpu_handle* h, int code, const std::string& msg) {
  h->err = msg;
  return code;
}

// device buffers are reused across prepare() calls when they are already large enough (a re-upload of
// a same-sized problem then costs no cudaMalloc / cudaFree)
template <class T>
static int dev_alloc(vcgpu_handle* h, T** p, size_t n) {
  if (n == 0) n = 1;
  const size_t bytes = n * sizeof(T);
  void* key = static_cast<void*>(p);
  auto it = h->capacity.find(key);
  if (*p && it != h->capacity.end() && it->second >= bytes) return VCGPU_OK;
  if (*p) cudaFree(*p);
  *p = nullptr;
  CUDA_TRY(h, cudaMalloc(reinterpret_cast<void**>(p), bytes));
  h->capacity[key] = bytes;
  return VCGPU_OK;
}
template <class T>
static void dev_free(T** p) {
  if (*p) cudaFree(*p);
  *p = nullptr;
}

// ------------------------------------------------------------------ stage timers
struct StageScope {
  vcgpu_handle* h;
  int s;
  StageScope(vcgpu_handle* h_, int s_) : h(h_), s(s_) {
    if (h->profiling) { cudaEventRecord(h->st_ev[s][0], h->stream); h->st_l0 = h->launches; }
  }
  ~StageScope() {
    if (h->profiling) {
      cudaEventRecord(h->st_ev[s][1], h->stream);
      h->st_used[s] = true;
      h->st_n[s] += h->launches - h->st_l0;
    }
  }
};
static void stage_collect(vcgpu_handle* h) {  // call after a stream synchronise
  if (!h->profiling) return;
  for (int s = 0; s < VCGPU_STAGE_COUNT; ++s)
    if (h->st_used[s]) {
      float ms = 0;
      if (cudaEventElapsedTime(&ms, h->st_ev[s][0], h->st_ev[s][1]) == cudaSuccess) h->st_ms[s] += ms;
      h->st_used[s] = false;
    }
}
static void xchg_release(vcgpu_handle* h);
static int imu_mega_prepare(vcgpu_handle* h);
#include "vc_imu_host.inl"

extern "C" int vcgpu_set_profiling(vcgpu_handle* h, int profile, int flush_l2) {
  if (!h) return VCGPU_ERR_INVALID;
  CUDA_TRY(h, cudaSetDevice(h->device));
  if ((profile || flush_l2) && !h->it_ev[0]) {
    for (int s = 0; s < VCGPU_STAGE_COUNT; ++s)
      for (int k = 0; k < 2; ++k) CUDA_TRY(h, cudaEventCreate(&h->st_ev[s][k]));
    CUDA_TRY(h, cudaEventCreate(&h->it_ev[0]));
    CUDA_TRY(h, cudaEventCreate(&h->it_ev[1]));
  }
  if (flush_l2 && !h->d_flush) CUDA_TRY(h, cudaMalloc(&h->d_flush, 256u << 20));
  h->profiling = (profile & 1) != 0;
  h->materialize = (profile & 2) != 0;  // bit 1: use the two-pass path that materialises J in HBM
  h->multi_launch = (profile & 4) != 0; // bit 2: multi-launch engine even where the persistent kernel applies
  h->phase_clocks = (profile & 8) != 0; // bit 3: persistent kernel records per-phase device clocks
  h->flush_l2 = flush_l2 != 0;
  for (int s = 0; s < VCGPU_STAGE_COUNT; ++s) { h->st_ms[s] = 0; h->st_n[s] = 0; h->st_used[s] = false; }
  for (int k = 0; k < vc::kImuProfSlots; ++k) h->phase_ns[k] = 0;
  return VCGPU_OK;
}
extern "C" int vcgpu_get_phase_clocks(vcgpu_handle* h, uint64_t ns[64]) {
  if (!h || !ns) return VCGPU_ERR_INVALID;
  for (int k = 0; k < 64; ++k) ns[k] = h->phase_ns[k];
  return VCGPU_OK;
}
extern "C" int vcgpu_get_stage_times(vcgpu_handle* h, double ms_total[VCGPU_STAGE_COUNT], int64_t launches[VCGPU_STAGE_COUNT]) {
  if (!h || !ms_total || !launches) return VCGPU_ERR_INVALID;
  for (int s = 0; s < VCGPU_STAGE_COUNT; ++s) { ms_total[s] = h->st_ms[s]; launches[s] = h->st_n[s]; }
  return VCGPU_OK;
}

// FP64 throughput of this device (vector DFMA and tensor DMMA), for the roofline of the FP64-bound kernels
extern "C" int vcgpu_fp64_peak(int device, double* dfma_tflops, double* dmma_tflops) {
  if (!dfma_tflops || !dmma_tflops) return VCGPU_ERR_INVALID;
  cudaDeviceProp prop;
  if (cudaSetDevice(device) != cudaSuccess || cudaGetDeviceProperties(&prop, device) != cudaSuccess) return VCGPU_ERR_CUDA;
  double* out = nullptr;
  cudaEvent_t e0, e1;
  if (cudaMalloc(&out, sizeof(double)) != cudaSuccess) return VCGPU_ERR_CUDA;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int ctas = prop.multiProcessorCount * 8, threads = 256, iters = 4096;
  double best[2] = {0.0, 0.0};
  for (int which = 0; which < 2; ++which)
    for (int rep = 0; rep < 5; ++rep) {
      cudaEventRecord(e0);
      if (which == 0) vc::dfma_peak_kernel<<<ctas, threads>>>(out, iters, 1.0);
      else vc::dmma_peak_kernel<<<ctas, threads>>>(out, iters, 1.0);
      cudaEventRecord(e1);
      if (cudaEventSynchronize(e1) != cudaSuccess) { cudaFree(out); return VCGPU_ERR_CUDA; }
      float ms = 0.f;
      cudaEventElapsedTime(&ms, e0, e1);
      // DFMA: 8 chains x 2 flop per thread-iteration; DMMA: 8 x (8*8*4*2 flop) per warp-iteration
      const double flop = which == 0 ? 16.0 * iters * static_cast<double>(ctas) * threads
                                     : 8.0 * 512.0 * iters * static_cast<double>(ctas) * (threads / 32);
      if (rep > 0) best[which] = std::max(best[which], flop / (ms * 1e-3) / 1e12);
    }
  cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(out);
  *dfma_tflops = best[0];
  *dmma_tflops = best[1];
  return VCGPU_OK;
}

// ------------------------------------------------------------------ lifecycle
extern "C" void vcgpu_default_flags(vcgpu_flags* f) {
  std::memset(f, 0, sizeof *f);
  f->visual = 1;
  f->visual_mult = 1.0;
  f->imu_mult = 1.0;
}
extern "C" void vcgpu_default_options(vcgpu_options* o) {
  o->max_iters = 200;
  o->function_tol = 1e-6;
  o->gradient_tol = 1e-10;
  o->param_tol = 1e-8;
  o->init_radius = 1e4;
  o->strategy = 0;
  o->jacobi_scaling = 1;
  o->update_imu_weights = 1;
  o->update_state_every_iteration = 0;
}

extern "C" int vcgpu_create(const vcgpu_config* cfg, vcgpu_handle** out) {
  if (!out) return VCGPU_ERR_INVALID;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return VCGPU_ERR_CUDA;  // no CPU fallback
  vcgpu_handle* h = new vcgpu_handle();
  vcgpu_default_flags(&h->flags);
  vcgpu_default_options(&h->opts);
  int dev = cfg ? cfg->device : -1;
  if (dev < 0) cudaGetDevice(&dev);
  h->device = dev;
  if (cudaSetDevice(dev) != cudaSuccess || cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&h->stream2, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&h->ev_dec, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&h->ev_wts, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreate(&h->ev0) != cudaSuccess || cudaEventCreate(&h->ev1) != cudaSuccess ||
      cudaMallocHost(reinterpret_cast<void**>(&h->h_scalars), kScCount * sizeof(double)) != cudaSuccess ||
      cudaMallocHost(reinterpret_cast<void**>(&h->h_ctl), sizeof(Ctl)) != cudaSuccess ||
      cudaMalloc(reinterpret_cast<void**>(&h->d_ctl), sizeof(Ctl)) != cudaSuccess) {
    delete h;
    return VCGPU_ERR_CUDA;
  }
  *out = h;
  return VCGPU_OK;
}

extern "C" int vcgpu_destroy(vcgpu_handle* h) {
  if (!h) return VCGPU_OK;
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->stream);
  dev_free(&h->d_state[0]); dev_free(&h->d_state[1]);
  dev_free(&h->d_pw); dev_free(&h->d_pc); dev_free(&h->d_obs_frame);
  dev_free(&h->d_grp_start); dev_free(&h->d_grp_count); dev_free(&h->d_group_of);
  dev_free(&h->d_mask); dev_free(&h->d_frame_used); dev_free(&h->d_r); dev_free(&h->d_J); dev_free(&h->d_cost_part);
  dev_free(&h->d_Cg); dev_free(&h->d_Cpart);
  dev_free(&h->d_blk_mem[0]); dev_free(&h->d_blk_mem[1]);
  dev_free(&h->d_scale); dev_free(&h->d_X); dev_free(&h->d_Spart); dev_free(&h->d_delta);
  dev_free(&h->d_red); dev_free(&h->d_scalars); dev_free(&h->d_Ssum); dev_free(&h->d_red_part); dev_free(&h->d_counter);
  dev_free(&h->d_dl); dev_free(&h->d_dl_part); dev_free(&h->d_partS); dev_free(&h->d_partC); dev_free(&h->d_batch_args); dev_free(&h->d_batch_cs); dev_free(&h->d_batch_ev); dev_free(&h->d_batch_cov); dev_free(&h->d_batch_ccov); dev_free(&h->d_cov); dev_free(&h->d_prof); dev_free(&h->d_prof2); dev_free(&h->d_csync);
  dev_free(&h->d_imu); dev_free(&h->d_wsqrt); h->d_wvec = nullptr; dev_free(&h->d_imu_r); dev_free(&h->d_imu_J);
  imu_free(h);
  dev_free(&h->d_mg); dev_free(&h->d_sep); dev_free(&h->d_dense); dev_free(&h->d_dsys);
  xchg_release(h);
  if (h->comm) ncclCommDestroy(static_cast<ncclComm_t>(h->comm));
  if (h->h_scalars) cudaFreeHost(h->h_scalars);
  if (h->h_ctl) cudaFreeHost(h->h_ctl);
  if (h->d_ctl) cudaFree(h->d_ctl);
  if (h->d_flush) cudaFree(h->d_flush);
  if (h->it_ev[0]) {
    for (int s = 0; s < VCGPU_STAGE_COUNT; ++s)
      for (int k = 0; k < 2; ++k) cudaEventDestroy(h->st_ev[s][k]);
    cudaEventDestroy(h->it_ev[0]);
    cudaEventDestroy(h->it_ev[1]);
  }
  cudaEventDestroy(h->ev0);
  cudaEventDestroy(h->ev1);
  if (h->ev_dec) cudaEventDestroy(h->ev_dec);
  if (h->ev_wts) cudaEventDestroy(h->ev_wts);
  if (h->stream2) cudaStreamDestroy(h->stream2);
  cudaStreamDestroy(h->stream);
  delete h;
  return VCGPU_OK;
}

extern "C" const char* vcgpu_last_error(const vcgpu_handle* h) { return h ? h->err.c_str() : "null handle"; }

// ------------------------------------------------------------------ uploads
extern "C" int vcgpu_set_cameras(vcgpu_handle* h, int n, const int32_t* model, const double* intr,
                                 const double* q_ck, const double* p_ck) {
  if (!h || n <= 0 || n > kMaxCams || !model || !intr || !q_ck || !p_ck)
    return h ? fail(h, VCGPU_ERR_INVALID, "set_cameras: bad arguments (1..8 cameras)") : VCGPU_ERR_INVALID;
  for (int i = 0; i < n; ++i)
    if (model[i] < 0 || model[i] > 4) return fail(h, VCGPU_ERR_INVALID, "set_cameras: unknown camera model");
  if (n != h->n_cams || !std::equal(model, model + n, h->h_model.begin())) h->dirty = true;
  h->n_cams = n;
  h->h_model.assign(model, model + n);
  h->h_intr.assign(intr, intr + 10 * n);
  h->h_qck.assign(q_ck, q_ck + 4 * n);
  h->h_pck.assign(p_ck, p_ck + 3 * n);
  h->state_dirty = true;
  h->wvec_cold = true;
  return VCGPU_OK;
}
extern "C" int vcgpu_set_frames(vcgpu_handle* h, int n, const double* T_wp, const double* v_w, const double* time) {
  if (!h || n <= 0 || !T_wp || !v_w || !time) return h ? fail(h, VCGPU_ERR_INVALID, "set_frames: bad arguments") : VCGPU_ERR_INVALID;
  if (n != h->n_frames) h->dirty = true;
  h->n_frames = n;
  h->h_T.assign(T_wp, T_wp + 7 * n);
  h->h_v.assign(v_w, v_w + 3 * n);
  if (h->h_time.size() != static_cast<size_t>(n) || !std::equal(time, time + n, h->h_time.begin())) h->dirty = true;
  h->h_time.assign(time, time + n);
  h->state_dirty = true;
  h->wvec_cold = true;
  return VCGPU_OK;
}
extern "C" int vcgpu_set_observations(vcgpu_handle* h, int64_t n, const int32_t* frame_id, const int32_t* cam_id,
                                      const double* p_w, const double* p_c) {
  if (!h || n < 0 || (n > 0 && (!frame_id || !cam_id || !p_w || !p_c)))
    return h ? fail(h, VCGPU_ERR_INVALID, "set_observations: bad arguments") : VCGPU_ERR_INVALID;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));  // an earlier upload may still be reading the page-locked copies
  h->n_obs_all = n;
  // one thread on purpose: copies split over several cores are slower end to end (the DMA that follows reads lines
  // still owned by the other cores' caches)
  h->h_obs_frame.assign(frame_id, frame_id + n);
  h->h_obs_cam.assign(cam_id, cam_id + n);
  h->h_pw.assign(p_w, p_w + 3 * n);
  h->h_pc.assign(p_c, p_c + 2 * n);
  h->h_active.assign(n, 1);
  h->dirty = true;
  return VCGPU_OK;
}
extern "C" int vcgpu_set_imu(vcgpu_handle* h, int n, const double* t, const double* w, const double* a,
                             double sigma_g, double sigma_a) {
  if (!h || n < 0 || (n > 0 && (!t || !w || !a))) return h ? fail(h, VCGPU_ERR_INVALID, "set_imu: bad arguments") : VCGPU_ERR_INVALID;
  for (int i = 1; i < n; ++i)
    if (!(t[i] > t[i - 1])) return fail(h, VCGPU_ERR_INVALID, "set_imu: timestamps are not unique/increasing");  // vicalibrator.h:377
  h->h_imu_t.assign(t, t + n);
  h->h_imu_w.assign(w, w + 3 * n);
  h->h_imu_a.assign(a, a + 3 * n);
  h->sigma_g = sigma_g;
  h->sigma_a = sigma_a;
  h->dirty = true;
  h->wvec_cold = true;
  return VCGPU_OK;
}
extern "C" int vcgpu_set_imu_params(vcgpu_handle* h, const double g[2], const double b[6], const double sf[6], double ts) {
  if (!h || !g || !b || !sf) return h ? fail(h, VCGPU_ERR_INVALID, "set_imu_params: bad arguments") : VCGPU_ERR_INVALID;
  std::memcpy(h->h_g, g, sizeof h->h_g);
  std::memcpy(h->h_b, b, sizeof h->h_b);
  std::memcpy(h->h_sf, sf, sizeof h->h_sf);
  h->h_ts = ts;
  h->state_dirty = true;
  h->wvec_cold = true;
  return VCGPU_OK;
}
extern "C" int vcgpu_set_flags(vcgpu_handle* h, const vcgpu_flags* f) {
  if (!h || !f) return VCGPU_ERR_INVALID;
  if ((f->inertial != 0) != (h->flags.inertial != 0)) h->dirty = true;
  h->flags = *f;
  h->blocks_valid = false;
  h->wvec_cold = true;
  return VCGPU_OK;
}
extern "C" int vcgpu_set_options(vcgpu_handle* h, const vcgpu_options* o) {
  if (!h || !o) return VCGPU_ERR_INVALID;
  if (o->strategy != 0 && o->strategy != 1) return fail(h, VCGPU_ERR_INVALID, "set_options: unknown strategy");
  h->opts = *o;
  return VCGPU_OK;
}
extern "C" int vcgpu_register_mirrors(vcgpu_handle* h, double* intr, double* q_ck, double* p_ck, double* T_wp,
                                      double* v_w, double* g, double* b, double* sf, double* ts) {
  if (!h) return VCGPU_ERR_INVALID;
  double* m[9] = {intr, q_ck, p_ck, T_wp, v_w, g, b, sf, ts};
  std::memcpy(h->mirror, m, sizeof m);
  return VCGPU_OK;
}

// ------------------------------------------------------------------ prepare: sort, allocate, upload
static void fill_mask(const vcgpu_handle* h, std::vector<double>* mask) {
  const DevProblem& dp = h->dp;
  mask->assign(dp.G, 1.0);
  const vcgpu_flags& f = h->flags;
  for (int c = 0; c < dp.n_cams; ++c) {
    const CamInfo& ci = dp.cams[c];
    if (c == 0) {  // vicalibrator.h:572-587
      const double rot = f.inertial ? 1.0 : 0.0;
      const double trans = (f.inertial && !f.rotation_only) ? 1.0 : 0.0;
      for (int i = 0; i < 3; ++i) (*mask)[ci.goff + i] = rot;
      for (int i = 0; i < 3; ++i) (*mask)[ci.goff + 3 + i] = trans;
    }
    if (f.fix_intrinsics)
      for (int i = 0; i < ci.K; ++i) (*mask)[ci.goff + 6 + i] = 0.0;
    // A camera no active observation sees is in no residual (the IMU residual takes no camera block): Ceres removes
    // its blocks (Program::RemoveFixedBlocks), so they are never moved and stay out of x_norm, like an unused frame's.
    // A frame shard sees its own frames' observations only, so a sharded handle keeps every camera.
    if (ci.n_obs == 0 && h->nranks == 1)
      for (int i = 0; i < 6 + ci.K; ++i) (*mask)[ci.goff + i] = 0.0;
  }
  if (f.inertial) {  // vicalibrator.h:657-676
    const int o = dp.imu_goff;
    (*mask)[o] = (*mask)[o + 1] = f.rotation_only ? 0.0 : 1.0;
    for (int i = 0; i < 6; ++i) (*mask)[o + 2 + i] = f.bias_active ? 1.0 : 0.0;
    for (int i = 0; i < 6; ++i) (*mask)[o + 8 + i] = f.scale_active ? 1.0 : 0.0;
    (*mask)[o + 14] = f.optimize_ts ? 1.0 : 0.0;
  }
}

static void pack_state(const vcgpu_handle* h, std::vector<double>* s) {
  const DevProblem& dp = h->dp;
  s->assign(dp.state_size, 0.0);
  std::copy(h->h_T.begin(), h->h_T.end(), s->begin());
  std::copy(h->h_v.begin(), h->h_v.end(), s->begin() + dp.off_v);
  for (int c = 0; c < dp.n_cams; ++c) {
    double* p = s->data() + dp.off_cam + kCamStateStride * c;
    std::copy(&h->h_qck[4 * c], &h->h_qck[4 * c] + 4, p);
    std::copy(&h->h_pck[3 * c], &h->h_pck[3 * c] + 3, p + 4);
    std::copy(&h->h_intr[10 * c], &h->h_intr[10 * c] + 10, p + 7);
  }
  double* p = s->data() + dp.off_imu;
  p[0] = h->h_g[0]; p[1] = h->h_g[1];
  for (int i = 0; i < 6; ++i) { p[2 + i] = h->h_b[i]; p[8 + i] = h->h_sf[i]; }
  p[14] = h->h_ts;
}
static void unpack_state(vcgpu_handle* h, const std::vector<double>& s) {
  const DevProblem& dp = h->dp;
  std::copy(s.begin(), s.begin() + 7 * dp.n_frames, h->h_T.begin());
  std::copy(s.begin() + dp.off_v, s.begin() + dp.off_v + 3 * dp.n_frames, h->h_v.begin());
  for (int c = 0; c < dp.n_cams; ++c) {
    const double* p = s.data() + dp.off_cam + kCamStateStride * c;
    std::copy(p, p + 4, &h->h_qck[4 * c]);
    std::copy(p + 4, p + 7, &h->h_pck[3 * c]);
    std::copy(p + 7, p + 17, &h->h_intr[10 * c]);
  }
  const double* p = s.data() + dp.off_imu;
  h->h_g[0] = p[0]; h->h_g[1] = p[1];
  for (int i = 0; i < 6; ++i) { h->h_b[i] = p[2 + i]; h->h_sf[i] = p[8 + i]; }
  h->h_ts = p[14];
}

static int upload_state(vcgpu_handle* h) {
  std::vector<double> s;
  pack_state(h, &s);
  CUDA_TRY(h, cudaMemcpyAsync(h->d_state[h->cur], s.data(), s.size() * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->state_dirty = false;
  h->blocks_valid = false;
  return VCGPU_OK;
}
static int download_state(vcgpu_handle* h) {
  std::vector<double> s(h->dp.state_size);
  CUDA_TRY(h, cudaMemcpyAsync(s.data(), h->d_state[h->cur], s.size() * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  unpack_state(h, s);
  return VCGPU_OK;
}
static void write_mirrors(vcgpu_handle* h) {
  const size_t nc = h->n_cams, nf = h->n_frames;
  if (h->mirror[0]) std::memcpy(h->mirror[0], h->h_intr.data(), 10 * nc * sizeof(double));
  if (h->mirror[1]) std::memcpy(h->mirror[1], h->h_qck.data(), 4 * nc * sizeof(double));
  if (h->mirror[2]) std::memcpy(h->mirror[2], h->h_pck.data(), 3 * nc * sizeof(double));
  if (h->mirror[3]) std::memcpy(h->mirror[3], h->h_T.data(), 7 * nf * sizeof(double));
  if (h->mirror[4]) std::memcpy(h->mirror[4], h->h_v.data(), 3 * nf * sizeof(double));
  if (h->mirror[5]) std::memcpy(h->mirror[5], h->h_g, sizeof h->h_g);
  if (h->mirror[6]) std::memcpy(h->mirror[6], h->h_b, sizeof h->h_b);
  if (h->mirror[7]) std::memcpy(h->mirror[7], h->h_sf, sizeof h->h_sf);
  if (h->mirror[8]) *h->mirror[8] = h->h_ts;
}

static inline int64_t perm_at(const vcgpu_handle* h, int64_t k) { return h->perm_identity ? k : h->perm[k]; }

// residual / Jacobian buffers of the two-pass (materialising) path and the inspection hooks
static int ensure_rJ(vcgpu_handle* h) {
  VC_TRY(dev_alloc(h, &h->d_r, 2 * static_cast<size_t>(std::max<int64_t>(h->n_obs, 1))));
  VC_TRY(dev_alloc(h, &h->d_J, static_cast<size_t>(std::max<int64_t>(h->j_doubles, 1))));
  return VCGPU_OK;
}

// device attributes: once per handle (SM count; shared-memory opt-in, 0 without cooperative launch)
static int device_attrs(vcgpu_handle* h) {
  if (h->dev_sms != 0) return VCGPU_OK;
  int coop = 0, smem_optin = 0, sms = 0;
  CUDA_TRY(h, cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, h->device));
  CUDA_TRY(h, cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device));
  CUDA_TRY(h, cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device));
  h->dev_sms = sms;
  h->dev_smem_optin = coop ? smem_optin : 0;
  return VCGPU_OK;
}

// The most warps per CTA (0: none) whose dynamic request fits `avail` bytes: what the per-block opt-in leaves beside the
// static shared memory of the kernel that runs the loop (the group table; the batch kernel also stages its arguments)
static int mega_warps_in(const DevProblem& dp, int st, size_t avail) {
  int warps = vc::kMegaMaxWarps;
  while (warps > 0 && vc::mega_smem_doubles(dp.G, dp.n_cams, warps, st) * sizeof(double) > avail) --warps;
  return 12 * (dp.G + 1) > vc::kWarpDoubles ? 0 : warps;
}
// persistent vision kernel: pick the team count that fits shared memory, allocate the partial slots.  Each instantiation
// (LM, and DOGLEG with its three extra G-vectors) gets its own team count, shared-memory attribute and occupancy check,
// since the strategy may change between solves without a new prepare().
template <vc::Strategy S>
static int mega_fit(vcgpu_handle* h, int* warps_out) {
  const DevProblem& dp = h->dp;
  const int st = S == vc::Strategy::kDogleg ? 1 : 0;
  *warps_out = 0;
  cudaFuncAttributes fa{};
  CUDA_TRY(h, cudaFuncGetAttributes(&fa, vc::lm_mega_kernel<S>));
  const int warps = mega_warps_in(dp, st, static_cast<size_t>(h->dev_smem_optin) - fa.sharedSizeBytes);
  if (warps == 0) return VCGPU_OK;
  const size_t smem = vc::mega_smem_doubles(dp.G, dp.n_cams, warps, st) * sizeof(double);
  // the opt-in belongs to the function, not to a handle: it is only ever raised, so that handles of different rigs
  // (several may be live at once, and a batch prepares them all before any runs) keep each other's launches valid
  if (smem > static_cast<size_t>(fa.maxDynamicSharedSizeBytes))
    CUDA_TRY(h, cudaFuncSetAttribute(vc::lm_mega_kernel<S>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  int per_sm = 0;
  CUDA_TRY(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, vc::lm_mega_kernel<S>, 32 * warps, smem));
  if (per_sm < 1) return VCGPU_OK;
  *warps_out = warps;
  return VCGPU_OK;
}
static int mega_prepare(vcgpu_handle* h) {
  const DevProblem& dp = h->dp;
  h->mega_warps[0] = h->mega_warps[1] = 0;
  if (dp.inertial || (h->nranks > 1 && !h->xchg_ready)) return VCGPU_OK;
  VC_TRY(device_attrs(h));
  if (h->dev_smem_optin == 0) return VCGPU_OK;
  int warps[2];
  VC_TRY(mega_fit<vc::Strategy::kLM>(h, &warps[0]));
  VC_TRY(mega_fit<vc::Strategy::kDogleg>(h, &warps[1]));
  if (warps[0] == 0 && warps[1] == 0) return VCGPU_OK;
  const size_t PS = static_cast<size_t>(dp.G) * dp.G + dp.G + vc::kMegaPartExtra;
  const size_t PC = static_cast<size_t>(dp.n_cams) * vc::kCgStride + vc::kMegaPartExtra;
  if (PS > 32768 || 4 * h->nranks * PS > static_cast<size_t>(vc::kXchgCOff) ||
      4 * h->nranks * PC > static_cast<size_t>(vc::kXchgCtlOff - vc::kXchgCOff))
    return VCGPU_OK;  // the totals do not fit the totals buffer: multi-launch engine
  if (!h->xchg_local) {  // single GPU: the totals buffer is local only
    void* p = nullptr;
    CUDA_TRY(h, cudaMalloc(&p, vc::kXchgBytes));
    CUDA_TRY(h, cudaMemset(p, 0, vc::kXchgBytes));
    h->xchg_local = static_cast<double*>(p);
    h->xchg_peer[0] = h->xchg_local;
  }
  h->mega_grid = h->dev_sms;
  h->mega_warps[0] = warps[0];
  h->mega_warps[1] = warps[1];
  VC_TRY(dev_alloc(h, &h->d_partS, h->mega_grid * PS));
  VC_TRY(dev_alloc(h, &h->d_partC, h->mega_grid * PC));
  CUDA_TRY(h, cudaMemsetAsync(h->d_partS, 0, h->mega_grid * PS * sizeof(double), h->stream));
  CUDA_TRY(h, cudaMemsetAsync(h->d_partC, 0, h->mega_grid * PC * sizeof(double), h->stream));
  VC_TRY(dev_alloc(h, &h->d_prof, vc::kProfCount));
  CUDA_TRY(h, cudaMemsetAsync(h->d_prof, 0, vc::kProfCount * sizeof(unsigned long long), h->stream));
  return VCGPU_OK;
}

static int prepare(vcgpu_handle* h) {
  CUDA_TRY(h, cudaSetDevice(h->device));
  if (h->n_cams <= 0 || h->n_frames <= 0) return fail(h, VCGPU_ERR_INVALID, "cameras and frames must be set first");
  if (h->dirty) {
    DevProblem& dp = h->dp;
    std::memset(&dp, 0, sizeof dp);
    dp.n_cams = h->n_cams;
    dp.n_frames = h->n_frames;
    const int nf = h->n_frames, nc = h->n_cams;
    // Optimistic upload: when no observation is switched off, start the DMAs from the page-locked caller-order
    // copies right away; they run while the pass below validates and checks the order on the CPU.  If the order
    // turns out not to be sorted by (camera, frame), the sorted staging copy simply overwrites them (stream order).
    bool uploaded = false;
    if (h->n_obs_all > 0 && std::memchr(h->h_active.data(), 0, static_cast<size_t>(h->n_obs_all)) == nullptr) {
      const size_t n = static_cast<size_t>(h->n_obs_all);
      VC_TRY(dev_alloc(h, &h->d_pw, 3 * n));
      VC_TRY(dev_alloc(h, &h->d_pc, 2 * n));
      VC_TRY(dev_alloc(h, &h->d_obs_frame, n));
      CUDA_TRY(h, cudaMemcpyAsync(h->d_pw, h->h_pw.data(), 3 * n * sizeof(double), cudaMemcpyHostToDevice, h->stream));
      CUDA_TRY(h, cudaMemcpyAsync(h->d_pc, h->h_pc.data(), 2 * n * sizeof(double), cudaMemcpyHostToDevice, h->stream));
      CUDA_TRY(h, cudaMemcpyAsync(h->d_obs_frame, h->h_obs_frame.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
      uploaded = true;
    }
    // Validate ids, count per (camera, frame), detect an already-sorted caller order.  Fast pass first: with every
    // observation active (`uploaded`), one branch-light sweep checks bounds and order and records the run boundaries;
    // the per-group counts of a sorted input are just the run lengths.
    std::vector<int64_t> count(static_cast<size_t>(nc) * nf + 1, 0);
    bool sorted = false;
    int64_t n_act = 0;
    if (uploaded) {
      const int32_t* cam = h->h_obs_cam.data();
      const int32_t* frm = h->h_obs_frame.data();
      const int64_t n = h->n_obs_all;
      bool in_range = true, ordered = true;
      int64_t prev_key = -1, run_start = 0;
      for (int64_t i = 0; i < n; ++i) {
        const int32_t c = cam[i], f = frm[i];
        in_range &= static_cast<uint32_t>(c) < static_cast<uint32_t>(nc) && static_cast<uint32_t>(f) < static_cast<uint32_t>(nf);
        const int64_t key = static_cast<int64_t>(c) * nf + f;
        if (key != prev_key) {
          if (in_range && prev_key >= 0) count[prev_key + 1] = i - run_start;
          ordered &= key > prev_key;
          if (!ordered || !in_range) break;  // the general pass below reports / sorts
          prev_key = key;
          run_start = i;
        }
      }
      if (in_range && ordered) {
        if (prev_key >= 0) count[prev_key + 1] = n - run_start;
        sorted = true;
        n_act = n;
      } else {
        std::fill(count.begin(), count.end(), 0);
      }
    }
    if (!sorted) {
      bool ordered = true;
      int64_t prev_key = -1;
      for (int64_t i = 0; i < h->n_obs_all; ++i) {
        const int32_t c = h->h_obs_cam[i], f = h->h_obs_frame[i];
        if (c < 0 || c >= nc) return fail(h, VCGPU_ERR_INVALID, "observation with unknown camera id");  // vicalibrator.h:396
        if (f < 0 || f >= nf) return fail(h, VCGPU_ERR_INVALID, "observation with unknown frame id");
        if (!h->h_active[i]) continue;
        const int64_t key = static_cast<int64_t>(c) * nf + f;
        ordered &= key >= prev_key;
        prev_key = key;
        ++count[key + 1];
        ++n_act;
      }
      sorted = ordered;
    }
    for (size_t k = 1; k < count.size(); ++k) count[k] += count[k - 1];
    h->n_obs = n_act;
    h->perm_identity = sorted && n_act == h->n_obs_all;
    h->perm.clear();
    if (!h->perm_identity) {  // stable counting sort by (camera, frame)
      h->perm.assign(h->n_obs, 0);
      std::vector<int64_t> pos(count.begin(), count.end() - 1);
      for (int64_t i = 0; i < h->n_obs_all; ++i)
        if (h->h_active[i]) h->perm[pos[static_cast<size_t>(h->h_obs_cam[i]) * nf + h->h_obs_frame[i]]++] = i;
    }
    std::vector<int32_t> grp_start, grp_count, group_of(static_cast<size_t>(nc) * nf, -1);
    int goff = 0;
    int64_t joff = 0;
    for (int c = 0; c < nc; ++c) {
      CamInfo& ci = dp.cams[c];
      ci.model = h->h_model[c];
      ci.K = num_intr(ci.model);
      ci.goff = goff;
      goff += 6 + ci.K;
      ci.obs_start = static_cast<int>(count[static_cast<size_t>(c) * nf]);
      ci.n_obs = static_cast<int>(count[static_cast<size_t>(c + 1) * nf] - count[static_cast<size_t>(c) * nf]);
      ci.group_start = static_cast<int>(grp_start.size());
      for (int f = 0; f < nf; ++f) {
        const int64_t s = count[static_cast<size_t>(c) * nf + f], e = count[static_cast<size_t>(c) * nf + f + 1];
        if (e > s) {
          group_of[static_cast<size_t>(c) * nf + f] = static_cast<int32_t>(grp_start.size());
          grp_start.push_back(static_cast<int32_t>(s));
          grp_count.push_back(static_cast<int32_t>(e - s));
        }
      }
      ci.n_groups = static_cast<int>(grp_start.size()) - ci.group_start;
      ci.joff = joff;
      joff += static_cast<int64_t>(2 * (12 + ci.K)) * ci.n_obs;
    }
    h->n_groups = static_cast<int>(grp_start.size());
    dp.inertial = h->flags.inertial ? 1 : 0;
    dp.fd = dp.inertial ? 9 : 6;
    dp.rank = h->rank;
    dp.nranks = h->nranks;
    // sharded inertial run: the caller appended the next rank's first frame (the cross-shard IMU factor needs it)
    dp.ghost = (dp.inertial && h->nranks > 1 && h->rank < h->nranks - 1) ? 1 : 0;
    dp.n_own = nf - dp.ghost;
    if (dp.ghost && nf < 2) return fail(h, VCGPU_ERR_INVALID, "a sharded inertial rank needs its own frames plus the ghost frame");
    dp.imu_goff = goff;
    dp.G = goff + (dp.inertial ? 15 : 0);
    dp.off_v = 7LL * nf;
    dp.off_cam = 10LL * nf;
    dp.off_imu = dp.off_cam + kCamStateStride * nc;
    dp.state_size = dp.off_imu + kImuStateSize;
    const int fd = dp.fd, G = dp.G;
    const int64_t n = h->n_obs;
    // observations to the device: straight DMA from the page-locked caller-order copies when they are
    // already sorted, else through a sorted page-locked staging copy
    VC_TRY(dev_alloc(h, &h->d_pw, 3 * static_cast<size_t>(n)));
    VC_TRY(dev_alloc(h, &h->d_pc, 2 * static_cast<size_t>(n)));
    VC_TRY(dev_alloc(h, &h->d_obs_frame, static_cast<size_t>(n)));
    if (n > 0 && !(uploaded && h->perm_identity)) {
      const double *src_pw = h->h_pw.data(), *src_pc = h->h_pc.data();
      const int32_t* src_fr = h->h_obs_frame.data();
      if (!h->perm_identity) {
        h->h_stage_pw.resize(3 * n); h->h_stage_pc.resize(2 * n); h->h_stage_frame.resize(n);
        for (int64_t k = 0; k < n; ++k) {
          const int64_t i = h->perm[k];
          h->h_stage_pw[3 * k] = h->h_pw[3 * i]; h->h_stage_pw[3 * k + 1] = h->h_pw[3 * i + 1]; h->h_stage_pw[3 * k + 2] = h->h_pw[3 * i + 2];
          h->h_stage_pc[2 * k] = h->h_pc[2 * i]; h->h_stage_pc[2 * k + 1] = h->h_pc[2 * i + 1];
          h->h_stage_frame[k] = h->h_obs_frame[i];
        }
        src_pw = h->h_stage_pw.data(); src_pc = h->h_stage_pc.data(); src_fr = h->h_stage_frame.data();
      }
      CUDA_TRY(h, cudaMemcpyAsync(h->d_pw, src_pw, 3 * n * sizeof(double), cudaMemcpyHostToDevice, h->stream));
      CUDA_TRY(h, cudaMemcpyAsync(h->d_pc, src_pc, 2 * n * sizeof(double), cudaMemcpyHostToDevice, h->stream));
      CUDA_TRY(h, cudaMemcpyAsync(h->d_obs_frame, src_fr, n * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
    }
    VC_TRY(dev_alloc(h, &h->d_grp_start, grp_start.size()));
    VC_TRY(dev_alloc(h, &h->d_grp_count, grp_count.size()));
    VC_TRY(dev_alloc(h, &h->d_group_of, group_of.size()));
    if (!grp_start.empty()) {
      CUDA_TRY(h, cudaMemcpyAsync(h->d_grp_start, grp_start.data(), grp_start.size() * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
      CUDA_TRY(h, cudaMemcpyAsync(h->d_grp_count, grp_count.data(), grp_count.size() * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
    }
    CUDA_TRY(h, cudaMemcpyAsync(h->d_group_of, group_of.data(), group_of.size() * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
    h->h_frame_used.assign(nf, h->flags.inertial ? 1 : 0);
    for (int c = 0; c < nc; ++c)
      for (int f = 0; f < nf; ++f)
        if (group_of[static_cast<size_t>(c) * nf + f] >= 0) h->h_frame_used[f] = 1;
    VC_TRY(dev_alloc(h, &h->d_frame_used, nf));
    CUDA_TRY(h, cudaMemcpyAsync(h->d_frame_used, h->h_frame_used.data(), nf, cudaMemcpyHostToDevice, h->stream));
    // work buffers
    VC_TRY(dev_alloc(h, &h->d_state[0], dp.state_size));
    VC_TRY(dev_alloc(h, &h->d_state[1], dp.state_size));
    VC_TRY(dev_alloc(h, &h->d_mask, G));
    h->j_doubles = joff;  // residual / Jacobian buffers of the two-pass path are allocated on first use (ensure_rJ)
    h->n_cost_part = 0;
    for (int c = 0; c < nc; ++c) h->n_cost_part += (dp.cams[c].n_obs + 255) / 256;
    VC_TRY(dev_alloc(h, &h->d_cost_part, std::max(h->n_cost_part, nf)));
    VC_TRY(dev_alloc(h, &h->d_Cg, static_cast<size_t>(h->n_groups) * kCgStride));
    CUDA_TRY(h, cudaMemsetAsync(h->d_Cg, 0, std::max<size_t>(1, static_cast<size_t>(h->n_groups) * kCgStride) * sizeof(double), h->stream));
    const size_t NS = static_cast<size_t>(G) * G + G;
    VC_TRY(dev_alloc(h, &h->d_Cpart, kReduceBlocks * NS));
    const size_t blk_sz = 2 * static_cast<size_t>(nf) * fd * fd + static_cast<size_t>(nf) * fd * G +
                          static_cast<size_t>(nf) * fd + NS + 1;
    for (int b = 0; b < 2; ++b) {
      VC_TRY(dev_alloc(h, &h->d_blk_mem[b], blk_sz));
      CUDA_TRY(h, cudaMemsetAsync(h->d_blk_mem[b], 0, blk_sz * sizeof(double), h->stream));
      double* p = h->d_blk_mem[b];
      h->blk[b].B = p; p += static_cast<size_t>(nf) * fd * fd;
      h->blk[b].U = p; p += static_cast<size_t>(nf) * fd * fd;
      h->blk[b].E = p; p += static_cast<size_t>(nf) * fd * G;
      h->blk[b].gf = p; p += static_cast<size_t>(nf) * fd;
      h->blk[b].C = p; p += static_cast<size_t>(G) * G;
      h->blk[b].gc = p; p += G;
      h->blk[b].cost = p;
    }
    const size_t np = static_cast<size_t>(nf) * fd + G;
    VC_TRY(dev_alloc(h, &h->d_scale, 2 * np));  // [scale | D2]
    VC_TRY(dev_alloc(h, &h->d_X, static_cast<size_t>(nf) * fd * (G + 1)));
    VC_TRY(device_attrs(h));
    h->n_solve_blocks = std::min((nf + kSolveWarps - 1) / kSolveWarps, h->dev_sms);
    VC_TRY(dev_alloc(h, &h->d_Spart, static_cast<size_t>(h->n_solve_blocks) * NS));
    VC_TRY(dev_alloc(h, &h->d_Ssum, NS));
    VC_TRY(dev_alloc(h, &h->d_delta, np));
    VC_TRY(dev_alloc(h, &h->d_red, 4 * (static_cast<size_t>(nf) + 2)));
    VC_TRY(dev_alloc(h, &h->d_red_part, 8 * kReduceBlocks));
    VC_TRY(dev_alloc(h, &h->d_mg, NS + kScGmax + h->nranks + 18 * h->nranks));
    VC_TRY(dev_alloc(h, &h->d_sep, 18 * h->nranks));
    {
      const size_t N = static_cast<size_t>(G) + 9 * h->nranks;
      VC_TRY(dev_alloc(h, &h->d_dense, N * N + N));
    }
    VC_TRY(dev_alloc(h, &h->d_counter, 8));
    CUDA_TRY(h, cudaMemsetAsync(h->d_counter, 0, 8 * sizeof(unsigned), h->stream));
    VC_TRY(dev_alloc(h, &h->d_scalars, kScCount));
    CUDA_TRY(h, cudaMemsetAsync(h->d_scalars, 0, kScCount * sizeof(double), h->stream));
    VC_TRY(mega_prepare(h));
    VC_TRY(imu_prepare(h));
    VC_TRY(imu_mega_prepare(h));
    h->cur = 0;
    h->dirty = false;
    h->state_dirty = true;
  }
  {
    DevProblem& dp = h->dp;
    dp.rotation_only = h->flags.rotation_only ? 1 : 0;
    dp.visual_mult = h->flags.visual ? h->flags.visual_mult : 0.0;
    dp.imu_mult = h->flags.imu_mult;
    std::vector<double> mask;
    fill_mask(h, &mask);
    CUDA_TRY(h, cudaMemcpyAsync(h->d_mask, mask.data(), mask.size() * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    dp.free_blocks = 0;
    for (int c = 0; c < dp.n_cams; ++c)
      for (int k = 0; k < 3; ++k)
        if (mask[dp.cams[c].goff + 3 * k]) dp.free_blocks |= 1u << (kFreeCam * c + k);
    if (dp.inertial) {
      const int first[4] = {0, 2, 8, 14};  // g b sf ts
      for (int k = 0; k < 4; ++k)
        if (mask[dp.imu_goff + first[k]]) dp.free_blocks |= 1u << (kFreeImu + k);
    }
  }
  if (h->state_dirty) VC_TRY(upload_state(h));
  // the next weights update starts its eigen-decompositions from the identity (NaN: no vectors)
  if (h->wvec_cold && h->dp.inertial && h->d_wvec) {
    CUDA_TRY(h, cudaMemsetAsync(h->d_wvec, 0xff, static_cast<size_t>(h->n_frames - 1) * 81 * sizeof(double), h->stream));
    h->wvec_cold = false;
  }
  return VCGPU_OK;
}

#include "vc_engine.inl"

extern "C" int vcgpu_solve(vcgpu_handle* h, vcgpu_iter_cb cb, void* user, vcgpu_summary* out) {
  if (!h) return VCGPU_ERR_INVALID;
  return run_solve(h, cb, user, out, 0);
}
extern "C" int vcgpu_solve_batch(vcgpu_handle* const* handles, int n, vcgpu_summary* out) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  return run_solve_batch(handles, n, out);
}
extern "C" int vcgpu_batch_plan(vcgpu_handle* h, int* cluster_size, int* warps, int* resident_clusters) {
  if (!h) return VCGPU_ERR_INVALID;
  return batch_plan_of(h, cluster_size, warps, resident_clusters);
}
extern "C" int vcgpu_solve_batch_inertial(vcgpu_handle* const* handles, int n, vcgpu_summary* out) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  return run_solve_batch_inertial(handles, n, out);
}
extern "C" int vcgpu_batch_plan_inertial(vcgpu_handle* h, int* cluster_size, int* resident_clusters) {
  if (!h) return VCGPU_ERR_INVALID;
  return imu_batch_plan_of(h, cluster_size, resident_clusters);
}
extern "C" int vcgpu_get_covariance_batch(vcgpu_handle* const* handles, int n, double* const* cov, int* status) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  if (!cov) return batch_refuse(handles, n, 0, "null cov array", "vcgpu_get_covariance_batch");
  return run_covariance_batch(handles, n, cov, status);
}
extern "C" int vcgpu_iterate(vcgpu_handle* h, int n, vcgpu_summary* out) {
  if (!h || n <= 0) return VCGPU_ERR_INVALID;
  return run_solve(h, nullptr, nullptr, out, n);
}

// ------------------------------------------------------------------ evaluation entry points
extern "C" int vcgpu_cost(vcgpu_handle* h, double* cost) {
  if (!h || !cost) return VCGPU_ERR_INVALID;
  VC_TRY(prepare(h));
  VC_TRY(ctl_reset(h, 0, 0));
  VC_TRY(evaluate_into(h, 0, false, -1));
  VC_TRY(read_scalars(h));
  *cost = h->h_scalars[kScCost];
  return VCGPU_OK;
}

extern "C" int vcgpu_evaluate(vcgpu_handle* h, int cam, double* cost, double* residuals, int64_t* n_blocks) {
  if (!h) return VCGPU_ERR_INVALID;
  VC_TRY(prepare(h));
  const DevProblem& dp = h->dp;
  if (cam >= dp.n_cams) return fail(h, VCGPU_ERR_INVALID, "evaluate: camera index out of range");
  VC_TRY(ctl_reset(h, 0, 0));
  VC_TRY(eval_reproj(h, 0, false, false, h->d_mask));
  const int64_t n = h->n_obs;
  std::vector<double> r(2 * std::max<int64_t>(n, 1));
  CUDA_TRY(h, cudaMemcpyAsync(r.data(), h->d_r, 2 * n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->blocks_valid = false;
  // caller order: gather the sorted residuals back through perm
  const int c0 = cam < 0 ? 0 : cam, c1 = cam < 0 ? dp.n_cams : cam + 1;
  std::vector<std::pair<int64_t, int64_t>> idx;  // (caller index, sorted index)
  for (int c = c0; c < c1; ++c)
    for (int64_t k = dp.cams[c].obs_start; k < dp.cams[c].obs_start + dp.cams[c].n_obs; ++k) idx.emplace_back(perm_at(h, k), k);
  std::sort(idx.begin(), idx.end());
  double s = 0;
  int64_t o = 0;
  for (const auto& pr : idx) {
    const double a = r[pr.second], b = r[n + pr.second];
    s += a * a + b * b;
    if (residuals) { residuals[2 * o] = a; residuals[2 * o + 1] = b; }
    ++o;
  }
  if (cost) *cost = 0.5 * s;
  if (n_blocks) *n_blocks = o;
  return VCGPU_OK;
}

extern "C" int vcgpu_remove_outliers(vcgpu_handle* h, const double* rmse, double threshold, int64_t* n_removed) {
  if (!h || !rmse) return VCGPU_ERR_INVALID;
  VC_TRY(prepare(h));
  const DevProblem& dp = h->dp;
  VC_TRY(ctl_reset(h, 0, 0));
  VC_TRY(eval_reproj(h, 0, false, false, h->d_mask));
  const int64_t n = h->n_obs;
  std::vector<double> r(2 * std::max<int64_t>(n, 1));
  CUDA_TRY(h, cudaMemcpyAsync(r.data(), h->d_r, 2 * n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  int64_t removed = 0;
  for (int c = 0; c < dp.n_cams; ++c)
    for (int64_t k = dp.cams[c].obs_start; k < dp.cams[c].obs_start + dp.cams[c].n_obs; ++k) {
      const double err = std::sqrt(r[k] * r[k] + r[n + k] * r[n + k]);
      if (err > threshold * rmse[c]) { h->h_active[perm_at(h, k)] = 0; ++removed; }  // vicalibrator.h:890-893
    }
  if (removed) h->dirty = true;
  if (n_removed) *n_removed = removed;
  return VCGPU_OK;
}
extern "C" int vcgpu_get_obs_active(vcgpu_handle* h, uint8_t* active) {
  if (!h || !active) return VCGPU_ERR_INVALID;
  std::memcpy(active, h->h_active.data(), h->h_active.size());
  return VCGPU_OK;
}

extern "C" int vcgpu_get_state(vcgpu_handle* h, double* intr, double* q_ck, double* p_ck, double* T_wp, double* v_w,
                               double* g, double* b, double* sf, double* ts) {
  if (!h) return VCGPU_ERR_INVALID;
  if (!h->dirty && !h->state_dirty) VC_TRY(download_state(h));
  const size_t nc = h->n_cams, nf = h->n_frames;
  if (intr) std::memcpy(intr, h->h_intr.data(), 10 * nc * sizeof(double));
  if (q_ck) std::memcpy(q_ck, h->h_qck.data(), 4 * nc * sizeof(double));
  if (p_ck) std::memcpy(p_ck, h->h_pck.data(), 3 * nc * sizeof(double));
  if (T_wp) std::memcpy(T_wp, h->h_T.data(), 7 * nf * sizeof(double));
  if (v_w) std::memcpy(v_w, h->h_v.data(), 3 * nf * sizeof(double));
  if (g) std::memcpy(g, h->h_g, sizeof h->h_g);
  if (b) std::memcpy(b, h->h_b, sizeof h->h_b);
  if (sf) std::memcpy(sf, h->h_sf, sizeof h->h_sf);
  if (ts) *ts = h->h_ts;
  return VCGPU_OK;
}
extern "C" int vcgpu_num_residuals(vcgpu_handle* h, int* out) {
  if (!h || !out) return VCGPU_ERR_INVALID;
  *out = num_residuals(h);
  return VCGPU_OK;
}
extern "C" int vcgpu_frame_dim(vcgpu_handle* h, int* out) {
  if (!h || !out) return VCGPU_ERR_INVALID;
  *out = h->flags.inertial ? 9 : 6;
  return VCGPU_OK;
}
extern "C" int vcgpu_num_globals(vcgpu_handle* h, int* out) {
  if (!h || !out) return VCGPU_ERR_INVALID;
  int g = 0;
  for (int c = 0; c < h->n_cams; ++c) g += 6 + num_intr(h->h_model[c]);
  *out = g + (h->flags.inertial ? 15 : 0);
  return VCGPU_OK;
}

// ------------------------------------------------------------------ inspection hooks
extern "C" int vcgpu_eval_reproj(vcgpu_handle* h, double* r_out, double* J_out) {
  if (!h || !r_out) return VCGPU_ERR_INVALID;
  VC_TRY(prepare(h));
  const DevProblem& dp = h->dp;
  const int64_t n = h->n_obs;
  double* ones = nullptr;
  VC_TRY(dev_alloc(h, &ones, dp.G));
  std::vector<double> hones(dp.G, 1.0);
  CUDA_TRY(h, cudaMemcpy(ones, hones.data(), dp.G * sizeof(double), cudaMemcpyHostToDevice));
  VC_TRY(ctl_reset(h, 0, 0));
  VC_TRY(eval_reproj(h, 0, J_out != nullptr, false, ones));
  std::vector<double> r(2 * std::max<int64_t>(n, 1));
  CUDA_TRY(h, cudaMemcpyAsync(r.data(), h->d_r, 2 * n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  cudaFree(ones);
  h->blocks_valid = false;
  for (int64_t k = 0; k < n; ++k) {
    r_out[2 * perm_at(h, k)] = r[k];
    r_out[2 * perm_at(h, k) + 1] = r[n + k];
  }
  if (J_out) {
    for (int c = 0; c < dp.n_cams; ++c) {
      const CamInfo& ci = dp.cams[c];
      const int NT = 12 + ci.K;
      std::vector<double> J(static_cast<size_t>(2 * NT) * std::max(ci.n_obs, 1));
      CUDA_TRY(h, cudaMemcpy(J.data(), h->d_J + ci.joff, static_cast<size_t>(2 * NT) * ci.n_obs * sizeof(double), cudaMemcpyDeviceToHost));
      for (int li = 0; li < ci.n_obs; ++li) {
        double* o = J_out + 44 * perm_at(h, ci.obs_start + li);
        std::memset(o, 0, 44 * sizeof(double));
        for (int row = 0; row < 2; ++row)
          for (int k = 0; k < NT; ++k) o[row * 22 + k] = J[static_cast<size_t>(row * NT + k) * ci.n_obs + li];
      }
    }
  }
  return VCGPU_OK;
}

extern "C" int vcgpu_normal_equations(vcgpu_handle* h, double* B, double* U, double* E, double* gf, double* C,
                                      double* gc, double* cost) {
  if (!h) return VCGPU_ERR_INVALID;
  VC_TRY(prepare(h));
  VC_TRY(ctl_reset(h, 0, 0));
  VC_TRY(evaluate_into(h, 0, false, -1));
  VC_TRY(read_scalars(h));
  const DevProblem& dp = h->dp;
  const size_t nf = dp.n_frames, fd = dp.fd, G = dp.G;
  const Blocks& b = h->blk[h->cur];
  if (B) CUDA_TRY(h, cudaMemcpy(B, b.B, nf * fd * fd * sizeof(double), cudaMemcpyDeviceToHost));
  if (U) CUDA_TRY(h, cudaMemcpy(U, b.U, nf * fd * fd * sizeof(double), cudaMemcpyDeviceToHost));
  if (E) CUDA_TRY(h, cudaMemcpy(E, b.E, nf * fd * G * sizeof(double), cudaMemcpyDeviceToHost));
  if (gf) CUDA_TRY(h, cudaMemcpy(gf, b.gf, nf * fd * sizeof(double), cudaMemcpyDeviceToHost));
  if (C) CUDA_TRY(h, cudaMemcpy(C, b.C, G * G * sizeof(double), cudaMemcpyDeviceToHost));
  if (gc) CUDA_TRY(h, cudaMemcpy(gc, b.gc, G * sizeof(double), cudaMemcpyDeviceToHost));
  if (cost) *cost = h->h_scalars[kScCost];
  return VCGPU_OK;
}

extern "C" int vcgpu_solve_arrow(vcgpu_handle* h, const double* scale, const double* D2, double* x) {
  if (!h || !scale || !D2 || !x) return VCGPU_ERR_INVALID;
  VC_TRY(prepare(h));
  VC_TRY(ctl_reset(h, 0, 0));
  VC_TRY(evaluate_into(h, 0, false, -1));
  const DevProblem& dp = h->dp;
  const int64_t np = static_cast<int64_t>(dp.n_frames) * dp.fd + dp.G;
  CUDA_TRY(h, cudaMemcpyAsync(h->d_scale, scale, np * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(h->d_scale + np, D2, np * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(h->d_scalars + kScNotPD, 0, sizeof(double), h->stream));
  VC_TRY(solve_and_update(h, h->d_scale + np, false));
  VC_TRY(read_scalars(h));
  if (h->h_scalars[kScNotPD] > 0) return fail(h, VCGPU_ERR_NUMERIC, "arrow system is not positive definite");
  CUDA_TRY(h, cudaMemcpy(x, h->d_delta, np * sizeof(double), cudaMemcpyDeviceToHost));
  return VCGPU_OK;
}

// Solution covariance of the global parameters (GetSolutionCovariance, vicalibrator.h:802-857, compiled out upstream
// behind COMPUTE_VICALIB_COVARIANCE because ceres::Covariance on the full problem "can run out of memory"): the
// [globals, globals] block of (J^T J)^-1 at the current state, i.e. the inverse of the Schur complement of the frames —
// one solve of the (undamped, unscaled) arrow system per global column on the device, through the same frame
// elimination the trust-region step uses.  Tangent space: per camera (w_ck 3 | p_ck 3 | intrinsics K), then with
// inertial terms (g 2 | b 6 | sf 6 | ts 1); rows / columns of constant or unused parameters (fill_mask) are zero like
// ceres::Covariance's.
extern "C" int vcgpu_get_covariance(vcgpu_handle* h, double* cov) {
  if (!h || !cov) return VCGPU_ERR_INVALID;
  VC_TRY(prepare(h));
  VC_TRY(ctl_reset(h, 0, 0));
  VC_TRY(evaluate_into(h, 0, false, -1));
  const DevProblem& dp = h->dp;
  const int G = dp.G;
  const int64_t nfp = static_cast<int64_t>(dp.n_frames) * dp.fd, np = nfp + G;
  std::vector<double> mask;
  fill_mask(h, &mask);
  const Blocks& b = h->blk[h->cur];
  std::vector<double> gf0(nfp), gc0(G), D2(np, 0.0), col(G, 0.0), x(np);
  CUDA_TRY(h, cudaMemcpyAsync(gf0.data(), b.gf, nfp * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(gc0.data(), b.gc, G * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  for (int k = 0; k < G; ++k) D2[nfp + k] = mask[k] != 0.0 ? 0.0 : 1.0;  // constant columns are empty: keep the system definite
  // Jacobi-scaled like the trust-region steps (focal lengths next to distortion coefficients and a time offset: the raw
  // J^T J does not survive an unpivoted Cholesky): cov = S (S H S)^-1 S
  jacobi_scale_kernel<<<static_cast<int>((np + 255) / 256), 256, 0, h->stream>>>(dp, h->blk[0], h->blk[1], h->d_ctl, h->d_scale, nullptr);
  ++h->launches;
  std::vector<double> sc(G);
  CUDA_TRY(h, cudaMemcpyAsync(sc.data(), h->d_scale + nfp, G * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(h->d_scale + np, D2.data(), np * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(b.gf, 0, nfp * sizeof(double), h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  std::fill(cov, cov + static_cast<size_t>(G) * G, 0.0);
  int rc = VCGPU_OK;
  for (int j = 0; j < G && rc == VCGPU_OK; ++j) {
    if (mask[j] == 0.0) continue;
    std::fill(col.begin(), col.end(), 0.0);
    col[j] = -1.0;  // the solver forms the right-hand side -g_c * scale and returns the scaled solution
    CUDA_TRY(h, cudaMemcpyAsync(b.gc, col.data(), G * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaMemsetAsync(h->d_scalars + kScNotPD, 0, sizeof(double), h->stream));
    rc = solve_and_update(h, h->d_scale + np, false);
    if (rc != VCGPU_OK) break;
    CUDA_TRY(h, cudaMemcpyAsync(x.data(), h->d_delta, np * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    rc = read_scalars(h);
    if (rc == VCGPU_OK && h->h_scalars[kScNotPD] > 0) rc = fail(h, VCGPU_ERR_NUMERIC, "covariance: J^T J is singular at the current state");
    for (int i = 0; i < G; ++i) cov[static_cast<size_t>(i) * G + j] = mask[i] != 0.0 ? sc[i] * x[nfp + i] : 0.0;
  }
  // put the gradient back; the Jacobi scale is recomputed by the next solve
  CUDA_TRY(h, cudaMemcpyAsync(b.gf, gf0.data(), nfp * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(b.gc, gc0.data(), G * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->blocks_valid = false;
  return rc;
}

// Batched PosePnPRansac (vicalib-task.cc:322-325): pose of the planar target in every (frame, camera) view, one warp
// per view (vc_pnp.cuh).  Cameras (model, intrinsics) are the ones given to vcgpu_set_cameras.
extern "C" int vcgpu_pose_pnp_ransac(vcgpu_handle* h, int n_views, const int32_t* cam_id, const int64_t* start, const int32_t* count,
                                     const double* pix, const double* pw, int robust_its, double robust_tol, double* T_cw,
                                     double* rmse, int32_t* n_used) {
  if (!h || n_views < 0 || (n_views > 0 && (!cam_id || !start || !count || !pix || !pw || !T_cw)))
    return h ? fail(h, VCGPU_ERR_INVALID, "pose_pnp_ransac: bad arguments") : VCGPU_ERR_INVALID;
  if (h->n_cams <= 0) return fail(h, VCGPU_ERR_INVALID, "pose_pnp_ransac: cameras must be set first");
  if (n_views == 0) return VCGPU_OK;
  CUDA_TRY(h, cudaSetDevice(h->device));
  int64_t N = 0;
  for (int v = 0; v < n_views; ++v) {
    if (cam_id[v] < 0 || cam_id[v] >= h->n_cams || start[v] < 0 || count[v] < 0)
      return fail(h, VCGPU_ERR_INVALID, "pose_pnp_ransac: bad view description");
    N = std::max<int64_t>(N, start[v] + count[v]);
  }
  int32_t *d_cam = nullptr, *d_count = nullptr, *d_model = nullptr, *d_used = nullptr;
  int64_t* d_start = nullptr;
  double *d_pix = nullptr, *d_pw = nullptr, *d_intr = nullptr, *d_xy = nullptr, *d_T = nullptr, *d_rmse = nullptr;
  unsigned char* d_use = nullptr;
  auto release = [&] {
    cudaFree(d_cam); cudaFree(d_count); cudaFree(d_model); cudaFree(d_used); cudaFree(d_start); cudaFree(d_pix); cudaFree(d_pw);
    cudaFree(d_intr); cudaFree(d_xy); cudaFree(d_T); cudaFree(d_rmse); cudaFree(d_use);
  };
  const size_t nv = static_cast<size_t>(n_views), np_ = static_cast<size_t>(std::max<int64_t>(N, 1));
  cudaError_t e = cudaSuccess;
  auto up = [&](void** d, const void* src, size_t bytes) {
    if (e != cudaSuccess) return;
    e = cudaMalloc(d, std::max<size_t>(bytes, 8));
    if (e == cudaSuccess && src) e = cudaMemcpyAsync(*d, src, bytes, cudaMemcpyHostToDevice, h->stream);
  };
  up(reinterpret_cast<void**>(&d_cam), cam_id, nv * sizeof(int32_t));
  up(reinterpret_cast<void**>(&d_start), start, nv * sizeof(int64_t));
  up(reinterpret_cast<void**>(&d_count), count, nv * sizeof(int32_t));
  up(reinterpret_cast<void**>(&d_pix), pix, 2 * np_ * sizeof(double));
  up(reinterpret_cast<void**>(&d_pw), pw, 3 * np_ * sizeof(double));
  up(reinterpret_cast<void**>(&d_model), h->h_model.data(), h->n_cams * sizeof(int32_t));
  up(reinterpret_cast<void**>(&d_intr), h->h_intr.data(), 10 * h->n_cams * sizeof(double));
  up(reinterpret_cast<void**>(&d_xy), nullptr, 2 * np_ * sizeof(double));
  up(reinterpret_cast<void**>(&d_use), nullptr, np_);
  up(reinterpret_cast<void**>(&d_T), nullptr, 7 * nv * sizeof(double));
  up(reinterpret_cast<void**>(&d_rmse), nullptr, nv * sizeof(double));
  up(reinterpret_cast<void**>(&d_used), nullptr, nv * sizeof(int32_t));
  if (e != cudaSuccess) { release(); h->err = std::string("pose_pnp_ransac: ") + cudaGetErrorString(e); return VCGPU_ERR_CUDA; }
  vc::pnp::Args a;
  a.n_views = n_views; a.cam = d_cam; a.start = d_start; a.count = d_count; a.pix = d_pix; a.pw = d_pw; a.model = d_model; a.intr = d_intr;
  a.robust_its = robust_its; a.robust_tol = robust_tol; a.xy = d_xy; a.use = d_use; a.T_cw = d_T; a.rmse = d_rmse; a.n_used = d_used;
  vc::pnp::pose_pnp_kernel<<<(n_views + vc::pnp::kWarps - 1) / vc::pnp::kWarps, 32 * vc::pnp::kWarps, 0, h->stream>>>(a);
  ++h->launches;
  std::vector<double> hr(nv);
  std::vector<int32_t> hu(nv);
  e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpyAsync(T_cw, d_T, 7 * nv * sizeof(double), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(hr.data(), d_rmse, nv * sizeof(double), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(hu.data(), d_used, nv * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  release();
  if (e != cudaSuccess) { h->err = std::string("pose_pnp_ransac: ") + cudaGetErrorString(e); return VCGPU_ERR_CUDA; }
  if (rmse) std::copy(hr.begin(), hr.end(), rmse);
  if (n_used) std::copy(hu.begin(), hu.end(), n_used);
  return VCGPU_OK;
}

extern "C" int vcgpu_eval_imu(vcgpu_handle* h, double* r, double* J) {
  if (!h || !r) return VCGPU_ERR_INVALID;
  VC_TRY(prepare(h));
  return imu_eval_hook(h, r, J);
}
extern "C" int vcgpu_update_imu_weights(vcgpu_handle* h) {
  if (!h) return VCGPU_ERR_INVALID;
  VC_TRY(prepare(h));
  if (!h->dp.inertial) return VCGPU_OK;
  VC_TRY(ctl_reset(h, 0, 0));
  VC_TRY(imu_update_weights(h));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return VCGPU_OK;
}
extern "C" int vcgpu_get_imu_weights(vcgpu_handle* h, double* w) {
  if (!h || !w) return VCGPU_ERR_INVALID;
  VC_TRY(prepare(h));
  if (h->n_frames < 2 || !h->d_wsqrt) return VCGPU_OK;
  CUDA_TRY(h, cudaMemcpy(w, h->d_wsqrt, static_cast<size_t>(h->n_frames - 1) * 81 * sizeof(double), cudaMemcpyDeviceToHost));
  return VCGPU_OK;
}
extern "C" int vcgpu_set_imu_weights(vcgpu_handle* h, const double* w) {
  if (!h || !w) return VCGPU_ERR_INVALID;
  h->wvec_cold = true;
  VC_TRY(prepare(h));
  if (h->n_frames < 2 || !h->d_wsqrt) return VCGPU_OK;
  CUDA_TRY(h, cudaMemcpy(h->d_wsqrt, w, static_cast<size_t>(h->n_frames - 1) * 81 * sizeof(double), cudaMemcpyHostToDevice));
  return VCGPU_OK;
}

extern "C" int vcgpu_comm_unique_id(uint8_t id[VCGPU_UNIQUE_ID_BYTES]) {
  static_assert(sizeof(ncclUniqueId) <= VCGPU_UNIQUE_ID_BYTES, "unique id does not fit");
  if (!id) return VCGPU_ERR_INVALID;
  ncclUniqueId u;
  if (ncclGetUniqueId(&u) != ncclSuccess) return VCGPU_ERR_COMM;
  std::memset(id, 0, VCGPU_UNIQUE_ID_BYTES);
  std::memcpy(id, &u, sizeof u);
  return VCGPU_OK;
}
// Map one exchange buffer per rank into every rank (CUDA IPC; all ranks are processes of one node) so the
// persistent kernel can do its two per-iteration reductions with NVLink peer stores instead of NCCL launches.
static void xchg_release(vcgpu_handle* h) {
  if (h->xchg_local) {
    if (h->comm && h->xchg_ready) {  // nobody may unmap / free while a peer can still store into it
      int* d = nullptr;
      if (cudaMalloc(&d, sizeof(int)) == cudaSuccess) {
        cudaMemset(d, 0, sizeof(int));
        ncclAllReduce(d, d, 1, ncclInt, ncclSum, static_cast<ncclComm_t>(h->comm), h->stream);
        cudaStreamSynchronize(h->stream);
        cudaFree(d);
      }
    }
    for (int r = 0; r < 8; ++r) {
      if (h->xchg_peer[r] && h->xchg_peer[r] != h->xchg_local) cudaIpcCloseMemHandle(h->xchg_peer[r]);
      h->xchg_peer[r] = nullptr;
    }
    cudaFree(h->xchg_local);
    h->xchg_local = nullptr;
  }
  h->xchg_ready = false;
}
static void xchg_setup(vcgpu_handle* h) {
  xchg_release(h);
  if (h->nranks < 2 || h->nranks > vc::kMaxRanks) return;
  const ncclComm_t comm = static_cast<ncclComm_t>(h->comm);
  cudaIpcMemHandle_t mine;
  cudaIpcMemHandle_t* d_all = nullptr;
  std::vector<cudaIpcMemHandle_t> all(h->nranks);
  int ok = 1;
  if (cudaMalloc(&h->xchg_local, vc::kXchgBytes) != cudaSuccess) { h->xchg_local = nullptr; ok = 0; }
  if (ok && cudaMemset(h->xchg_local, 0, vc::kXchgBytes) != cudaSuccess) ok = 0;
  if (ok && cudaIpcGetMemHandle(&mine, h->xchg_local) != cudaSuccess) ok = 0;
  if (!ok) std::memset(&mine, 0, sizeof mine);
  // every rank takes part in the collectives below whatever happened above, so nobody is left waiting
  if (cudaMalloc(&d_all, sizeof(cudaIpcMemHandle_t) * (h->nranks + 1)) != cudaSuccess) { cudaGetLastError(); return; }
  cudaMemcpy(d_all + h->nranks, &mine, sizeof mine, cudaMemcpyHostToDevice);
  ncclAllGather(d_all + h->nranks, d_all, sizeof mine, ncclChar, comm, h->stream);
  cudaStreamSynchronize(h->stream);
  cudaMemcpy(all.data(), d_all, sizeof(cudaIpcMemHandle_t) * h->nranks, cudaMemcpyDeviceToHost);
  for (int r = 0; ok && r < h->nranks; ++r) {
    if (r == h->rank) { h->xchg_peer[r] = h->xchg_local; continue; }
    void* p = nullptr;
    if (cudaIpcOpenMemHandle(&p, all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = 0; break; }
    h->xchg_peer[r] = static_cast<double*>(p);
  }
  // all ranks must agree: one failure anywhere disables the peer path everywhere
  int* d_ok = reinterpret_cast<int*>(d_all);
  cudaMemcpy(d_ok, &ok, sizeof(int), cudaMemcpyHostToDevice);
  ncclAllReduce(d_ok, d_ok, 1, ncclInt, ncclMin, comm, h->stream);
  cudaStreamSynchronize(h->stream);
  cudaMemcpy(&ok, d_ok, sizeof(int), cudaMemcpyDeviceToHost);
  cudaFree(d_all);
  h->xchg_ready = ok != 0;
  if (!h->xchg_ready) {
    for (int r = 0; r < 8; ++r) {
      if (h->xchg_peer[r] && h->xchg_peer[r] != h->xchg_local) cudaIpcCloseMemHandle(h->xchg_peer[r]);
      h->xchg_peer[r] = nullptr;
    }
    cudaGetLastError();
  }
}

extern "C" int vcgpu_comm_init(vcgpu_handle* h, const uint8_t id[VCGPU_UNIQUE_ID_BYTES], int rank, int nranks) {
  if (!h || !id || nranks < 1 || rank < 0 || rank >= nranks) return h ? fail(h, VCGPU_ERR_INVALID, "comm_init: bad arguments") : VCGPU_ERR_INVALID;
  CUDA_TRY(h, cudaSetDevice(h->device));
  xchg_release(h);
  h->dirty = true;  // the totals buffer is gone: prepare() must set the persistent kernel up again
  if (h->comm) { ncclCommDestroy(static_cast<ncclComm_t>(h->comm)); h->comm = nullptr; }
  h->rank = rank;
  h->nranks = nranks;
  if (nranks == 1) return VCGPU_OK;
  ncclUniqueId u;
  std::memcpy(&u, id, sizeof u);
  ncclComm_t c;
  const ncclResult_t rc = ncclCommInitRank(&c, nranks, u, rank);
  if (rc != ncclSuccess) return fail(h, VCGPU_ERR_COMM, std::string("ncclCommInitRank: ") + ncclGetErrorString(rc));
  h->comm = c;
  h->dirty = true;
  xchg_setup(h);  // optional: without peer access the sharded solve stays on the NCCL multi-launch engine
  return VCGPU_OK;
}
