// libvcgpu.so — host side of the C-ABI declared in include/vcgpu.h.
//
// Replaces, for ViCalibrator, what ceres::Problem + ceres::Solve + Problem::Evaluate do
// (vicalibrator.h:152, 548-679, 859-916, 956-971).  The trust-region loop below is the Ceres
// loop (TrustRegionMinimizer + LevenbergMarquardtStrategy, SURVEY App. A.3) driven from the host
// with every arithmetic step — the accept/reject decision included — on the device; the candidate
// point is evaluated *with* its Jacobian blocks (speculatively) so an accepted step needs no second
// pass.  Engines: vc_mega.cuh (persistent kernel, vision solves) and vc_engine.inl (multi-launch); the batch
// calls, one thread-block cluster per rig: vc_batch.inl.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>

#include <nccl.h>

#include "vc_internal.h"
#include "vc_kernels.cuh"
#include "vc_imu.cuh"
#include "vc_chain.cuh"
#include "vc_frame_cov.cuh"
#include "vc_fused.cuh"
#include "vc_peak.cuh"
#include "vc_mega.cuh"
#include "vc_dogleg.cuh"
#include "vc_imu_weights.cuh"
#include "vc_imu_poses.cuh"
#include "vc_imu_mega.cuh"
#include "vc_imu_eval_mega.cuh"
#include "vc_pnp.cuh"
#include "vc_eval_batch.cuh"
#include "vc_proj_cov.cuh"
#include "vc_view_info.cuh"
#include "vc_obs_infl.cuh"
#include "vc_imu_infl.cuh"
#include "vc_imu_align.cuh"

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
  if (profile & ~(1 | 4 | 8)) return fail(h, VCGPU_ERR_INVALID, "set_profiling: unknown bit in " + std::to_string(profile) + " (bits: 1, 4, 8)");
  CUDA_TRY(h, cudaSetDevice(h->device));
  if ((profile || flush_l2) && !h->it_ev[0]) {
    for (int s = 0; s < VCGPU_STAGE_COUNT; ++s)
      for (int k = 0; k < 2; ++k) CUDA_TRY(h, cudaEventCreate(&h->st_ev[s][k]));
    CUDA_TRY(h, cudaEventCreate(&h->it_ev[0]));
    CUDA_TRY(h, cudaEventCreate(&h->it_ev[1]));
  }
  if (flush_l2 && !h->d_flush) CUDA_TRY(h, cudaMalloc(&h->d_flush, 256u << 20));
  h->profiling = (profile & 1) != 0;
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
  dev_free(&h->d_dl); dev_free(&h->d_dl_part); dev_free(&h->d_partS); dev_free(&h->d_partC); dev_free(&h->d_batch_args); dev_free(&h->d_eval); dev_free(&h->d_pnp); dev_free(&h->d_mahal); dev_free(&h->d_pstart); dev_free(&h->d_poses); dev_free(&h->d_proj); dev_free(&h->d_view); dev_free(&h->d_infl); dev_free(&h->d_infl_obs); h->infl_obs_valid = false; dev_free(&h->d_align); dev_free(&h->d_rank); dev_free(&h->d_cov); dev_free(&h->d_fcov); dev_free(&h->d_prof); dev_free(&h->d_prof2); dev_free(&h->d_csync);
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

// residual / Jacobian buffers of vcgpu_eval_reproj
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
    h->infl_obs_valid = false;  // vcgpu_get_observation_influence's sorted copy of the observations
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
    h->j_doubles = joff;  // the residual / Jacobian buffers of vcgpu_eval_reproj are allocated on first use (ensure_rJ)
    VC_TRY(dev_alloc(h, &h->d_cost_part, nf));
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
#include "vc_batch.inl"

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
extern "C" int vcgpu_calibrate_batch(vcgpu_handle* const* handles, int n, const vcgpu_flow* flow, vcgpu_flow_summary* out,
                                     double* const* cam_rmse) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  if (!flow) return batch_refuse(handles, n, 0, "null flow", "vcgpu_calibrate_batch");
  return run_calibrate_batch(handles, n, *flow, out, cam_rmse);
}
extern "C" int vcgpu_batch_plan_inertial(vcgpu_handle* h, int* cluster_size, int* resident_clusters) {
  if (!h) return VCGPU_ERR_INVALID;
  return imu_batch_plan_of(h, cluster_size, resident_clusters);
}
extern "C" int vcgpu_get_covariance_batch(vcgpu_handle* const* handles, int n, double* const* cov, int* status) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  if (!cov) return batch_refuse(handles, n, 0, "null cov array", "vcgpu_get_covariance_batch");
  return run_cov_batch(handles, n, cov, status, kCovGlobals);
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

// Problem::Evaluate of one camera's or every camera's residual blocks, without the loss (vicalibrator.h:873-887, 958-966):
// run_evaluate_batch of this handle alone, then the asked camera's share of its per-camera results.  Frame shards
// evaluate their own observations.
extern "C" int vcgpu_evaluate(vcgpu_handle* h, int cam, double* cost, double* residuals, int64_t* n_blocks) {
  if (!h) return VCGPU_ERR_INVALID;
  if (cam >= h->n_cams) return fail(h, VCGPU_ERR_INVALID, "evaluate: camera index out of range");
  double cam_cost[kMaxCams];
  int64_t cam_blocks[kMaxCams];
  std::vector<double> all;  // one camera's residuals are picked from every camera's
  double* res = residuals;
  if (residuals && cam >= 0) {
    all.resize(2 * static_cast<size_t>(h->n_obs_all));
    res = all.data();
  }
  double* cp = cam_cost;
  int64_t* bp = cam_blocks;
  VC_TRY(run_evaluate_batch(&h, 1, EvalBatchOut{&cp, &bp, &res, nullptr, 0.0, nullptr}, "vcgpu_evaluate",
                            [](const vcgpu_handle*, int) -> const char* { return nullptr; }));
  const int c0 = cam < 0 ? 0 : cam, c1 = cam < 0 ? h->dp.n_cams : cam + 1;
  double s = 0;
  int64_t o = 0;
  for (int c = c0; c < c1; ++c) { s += cam_cost[c]; o += cam_blocks[c]; }
  if (residuals && cam >= 0)  // the camera's active observations in caller order
    for (int64_t k = 0, a = 0, m = 0; k < h->n_obs_all; ++k) {
      if (!h->h_active[k]) continue;
      if (h->h_obs_cam[k] == cam) { residuals[2 * m] = all[2 * a]; residuals[2 * m + 1] = all[2 * a + 1]; ++m; }
      ++a;
    }
  if (cost) *cost = s;
  if (n_blocks) *n_blocks = o;
  return VCGPU_OK;
}

// RemoveOutliers (vicalibrator.h:859-916): run_evaluate_batch of this handle alone
extern "C" int vcgpu_remove_outliers(vcgpu_handle* h, const double* rmse, double threshold, int64_t* n_removed) {
  if (!h || !rmse) return VCGPU_ERR_INVALID;
  return run_evaluate_batch(&h, 1, EvalBatchOut{nullptr, nullptr, nullptr, &rmse, threshold, n_removed}, "vcgpu_remove_outliers",
                            [](const vcgpu_handle*, int) -> const char* { return nullptr; });
}
// the batch calls refuse frame shards
static const char* eval_batch_refusal(const vcgpu_handle* h) { return h->nranks > 1 ? "frame shards (use the per-handle call)" : nullptr; }
extern "C" int vcgpu_evaluate_batch(vcgpu_handle* const* handles, int n, double* const* cam_cost, int64_t* const* cam_blocks,
                                    double* const* residuals_or_null) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  if (!cam_cost) return batch_refuse(handles, n, 0, "null cam_cost array", "vcgpu_evaluate_batch");
  return run_evaluate_batch(handles, n, EvalBatchOut{cam_cost, cam_blocks, residuals_or_null, nullptr, 0.0, nullptr}, "vcgpu_evaluate_batch",
                            [&](const vcgpu_handle* h, int i) { return cam_cost[i] ? eval_batch_refusal(h) : "null cam_cost pointer"; });
}
extern "C" int vcgpu_remove_outliers_batch(vcgpu_handle* const* handles, int n, const double* const* rmse, double threshold,
                                           int64_t* n_removed) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  if (!rmse) return batch_refuse(handles, n, 0, "null rmse array", "vcgpu_remove_outliers_batch");
  return run_evaluate_batch(handles, n, EvalBatchOut{nullptr, nullptr, nullptr, rmse, threshold, n_removed}, "vcgpu_remove_outliers_batch",
                            [&](const vcgpu_handle* h, int i) { return rmse[i] ? eval_batch_refusal(h) : "null rmse pointer"; });
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
  VC_TRY(eval_reproj(h, J_out != nullptr, ones));
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
  VC_TRY(solve_and_update(h, h->d_scale + np));
  VC_TRY(read_scalars(h));
  if (h->h_scalars[kScNotPD] > 0) return fail(h, VCGPU_ERR_NUMERIC, "arrow system is not positive definite");
  CUDA_TRY(h, cudaMemcpy(x, h->d_delta, np * sizeof(double), cudaMemcpyDeviceToHost));
  return VCGPU_OK;
}

// The frames' elimination and the inverse of the system it leaves into w.inv [N*N]: vision: the solve's frame
// elimination and Schur sum (summed over frame shards), then the inverse of the reduced system [globals].  kCovFrames:
// then the blocks (vc_frame_cov.cuh) into w.out [nf][fd*fd]; kCovCross: Σ_fg into w.out and Σ_f,f+1 into w.out_next;
// one warp per frame.
static int cov_vision(vcgpu_handle* h, const double* D2x, CovMode mode, const CovSpace& w) {
  const DevProblem& dp = h->dp;
  const int G = dp.G;
  VC_TRY(vision_frame_solve(h, D2x));
  VC_TRY(all_reduce(h, h->d_Ssum, static_cast<size_t>(G) * G + G));
  DenseArgs da{};
  da.dp = dp; da.bs[0] = h->blk[0]; da.bs[1] = h->blk[1]; da.ctl = h->d_ctl; da.scale = h->d_scale; da.D2x = D2x;
  da.Ssum = h->d_Ssum; da.delta = h->d_delta; da.scalars = h->d_scalars; da.add_globals = 1; da.src = 0; da.inv = w.inv;
  VC_TRY(kernel_smem_optin(h));
  dense_solve_kernel<6><<<1, 256, vc::chain_dense_smem_bytes(G), h->stream>>>(da);
  ++h->launches;
  if (mode != kCovGlobals) {
    vc::FrameCovArgs fa;
    fa.dp = dp; fa.b[0] = h->blk[0]; fa.b[1] = h->blk[1]; fa.ctl = h->d_ctl; fa.scale = h->d_scale; fa.D2x = D2x; fa.X = h->d_X;
    fa.Sgg = w.inv; fa.frame_used = h->d_frame_used; fa.out = w.out;
    const int grid = (dp.n_frames + vc::kFrameCovWarps - 1) / vc::kFrameCovWarps;
    if (mode == kCovFrames) vc::frame_cov_vision_kernel<6><<<grid, 32 * vc::kFrameCovWarps, 0, h->stream>>>(fa);
    else vc::frame_cross_cov_vision_kernel<6><<<grid, 32 * vc::kFrameCovWarps, 0, h->stream>>>({fa, h->d_mask, w.out_next});
    ++h->launches;
    if (mode == kCovDiagCross) {  // the diagonal blocks too, from the same X_f and Σ_gg
      fa.out = w.out_ff;
      vc::frame_cov_vision_kernel<6><<<grid, 32 * vc::kFrameCovWarps, 0, h->stream>>>(fa);
      ++h->launches;
    }
  }
  CUDA_TRY(h, cudaGetLastError());
  return VCGPU_OK;
}
// Inertial: the chain elimination, the inverse of [globals | top nodes] (on frame shards: of the ranks' summed
// partials).  Frame modes: with the top nodes' blocks, then the levels top-down (chain_selinv_kernel), then level 0's
// Σ_kk (kCovFrames) or Σ_kg and Σ_k,k+1 (kCovCross) unscaled; rows and columns from `live` on are 0.
static int cov_inertial(vcgpu_handle* h, const double* D2x, CovMode mode, int live, const CovSpace& w) {
  constexpr int FD = 9;
  vc::ImuDev* d = imu_dev(h);
  const DevProblem& dp = h->dp;
  const int G = dp.G, nl = static_cast<int>(d->levels.size());
  VC_TRY(imu_chain_eliminate(h, D2x));
  VC_TRY(imu_chain_dense(h, D2x, w.inv, mode != kCovGlobals ? &w.sig.back() : nullptr));
  if (mode == kCovGlobals) return VCGPU_OK;
  const size_t sm = vc::chain_selinv_smem_bytes<FD>(G, kChainC);
  if (nl > 1 && sm > h->selinv_smem_max)
    return fail(h, VCGPU_ERR_INVALID, "frame covariance: G = " + std::to_string(G) + " needs " + std::to_string(sm) +
                                          " B of shared memory per block, the device allows " + std::to_string(h->selinv_smem_max));
  for (int l = nl - 2; l >= 0; --l) {
    vc::SelinvArgs sa;
    sa.G = G; sa.c = kChainC; sa.cur = d->levels[l]; sa.sig = w.sig[l]; sa.up = w.sig[l + 1];
    sa.Sgg = w.inv; sa.ldg = w.N; sa.scalars = h->d_scalars;
    sa.lev = d->d_levels; sa.l = l; sa.nf = dp.n_frames; sa.b[0] = h->blk[0]; sa.b[1] = h->blk[1]; sa.ctl = h->d_ctl; sa.scale = h->d_scale; sa.D2x = D2x;
    vc::chain_selinv_kernel<FD><<<d->levels[l + 1].n, vc::kChainThreads, sm, h->stream>>>(sa);
    ++h->launches;
  }
  if (mode == kCovFrames || mode == kCovDiagCross) {
    const int64_t ne = static_cast<int64_t>(dp.n_frames) * FD * FD;
    vc::frame_cov_out_kernel<FD><<<static_cast<int>((ne + 255) / 256), 256, 0, h->stream>>>(dp.n_frames, live, w.sig[0].kk, h->d_scale, w.out_ff);
  }
  if (mode == kCovDiagCross) ++h->launches;
  if (mode != kCovFrames) {
    const int64_t ne = vc::frame_cross_cov_entries<FD>(dp.n_frames, G);
    vc::frame_cross_cov_out_kernel<FD><<<static_cast<int>((ne + 255) / 256), 256, 0, h->stream>>>(dp.n_frames, G, live, w.sig[0], h->d_scale,
                                                                                                  h->d_mask, w.out, w.out_next);
  }
  ++h->launches;
  CUDA_TRY(h, cudaGetLastError());
  return VCGPU_OK;
}

// vcgpu_get_covariance (kCovGlobals), vcgpu_get_frame_covariance (kCovFrames) and vcgpu_get_frame_cross_covariance
// (kCovCross) of one handle, the per-handle counterpart of run_cov_batch: cov_prelude, the frames' elimination and one
// inversion of the system it leaves; the globals' block of that inverse, or the frames' blocks from it.  kCovCross:
// Σ_fg into cov and Σ_f,f+1 into cov_next, either of them null.  Writes no state buffer.
// kCovDiagCross: cov is not read; the workspace, with Σ_gg (scaled, in inv), Σ_fg (out) and Σ_ff (out_ff) on the device,
// goes to *keep.
static int run_cov(vcgpu_handle* h, double* cov, CovMode mode, double* cov_next = nullptr, CovSpace* keep = nullptr) {
  VC_TRY(prepare(h));
  const bool frames = mode != kCovGlobals;
  std::vector<double> D2;
  int live = 0;
  VC_TRY(cov_prelude(h, frames, &D2, &live));
  const DevProblem& dp = h->dp;
  const size_t G = dp.G, nfp = static_cast<size_t>(dp.n_frames) * dp.fd;
  const double* D2x = h->d_scale + nfp + G;
  CUDA_TRY(h, cudaMemsetAsync(h->d_scalars + kScNotPD, 0, sizeof(double), h->stream));
  CovSpace w;
  int rc = cov_space(h, mode, &w);
  if (rc == VCGPU_OK) rc = dp.inertial ? cov_inertial(h, D2x, mode, live, w) : cov_vision(h, D2x, mode, w);
  h->blocks_valid = false;  // the Jacobi scale is the next solve's to set
  if (rc != VCGPU_OK) return rc;
  std::vector<double> inv(frames ? 0 : G * G), sc(frames ? 0 : G);
  if (!frames) {  // Σ_gg: the globals' block of the inverse, row stride N, and the globals' Jacobi scale
    CUDA_TRY(h, cudaMemcpy2DAsync(inv.data(), G * sizeof(double), w.inv, w.N * sizeof(double), G * sizeof(double), G,
                                  cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(sc.data(), h->d_scale + nfp, G * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  }
  VC_TRY(read_scalars(h));
  if (h->h_scalars[kScNotPD] > 0)
    return fail(h, VCGPU_ERR_NUMERIC, std::string(mode == kCovCross ? "frame cross covariance" : mode == kCovDiagCross ? "observation influence"
                                                  : frames ? "frame covariance" : "covariance") +
                                          ": J^T J is singular at the current state");
  if (mode == kCovDiagCross) {
    *keep = w;
    return VCGPU_OK;
  }
  if (mode == kCovFrames) {
    CUDA_TRY(h, cudaMemcpy(cov, w.out, nfp * dp.fd * sizeof(double), cudaMemcpyDeviceToHost));
    return VCGPU_OK;
  }
  if (mode == kCovCross) {
    if (cov) CUDA_TRY(h, cudaMemcpy(cov, w.out, nfp * G * sizeof(double), cudaMemcpyDeviceToHost));
    if (cov_next && dp.n_frames > 1)
      CUDA_TRY(h, cudaMemcpy(cov_next, w.out_next, (nfp - dp.fd) * dp.fd * sizeof(double), cudaMemcpyDeviceToHost));
    return VCGPU_OK;
  }
  // as cov_store_column: the lower triangle unscaled by s_i s_j and mirrored; constant or unused globals exactly 0
  std::vector<double> mask;
  fill_mask(h, &mask);
  for (size_t j = 0; j < G; ++j)
    for (size_t i = j; i < G; ++i)
      cov[i * G + j] = cov[j * G + i] = mask[j] != 0.0 && mask[i] != 0.0 ? sc[i] * sc[j] * inv[i * G + j] : 0.0;
  return VCGPU_OK;
}

// Solution covariance of the global parameters (GetSolutionCovariance, vicalibrator.h:802-857, compiled out upstream
// behind COMPUTE_VICALIB_COVARIANCE because ceres::Covariance on the full problem "can run out of memory"): the
// [globals, globals] block of (J^T J)^-1 at the current state, i.e. the inverse of the Schur complement of the frames.
// run_cov eliminates the frames once, as the trust-region step does, and inverts the system left, [globals] (vision)
// or [globals | top nodes] (inertial), whose globals' block this is.  Tangent space: per camera (w_ck 3 | p_ck 3 |
// intrinsics K), then with inertial terms (g 2 | b 6 | sf 6 | ts 1); rows / columns of constant or unused parameters
// (fill_mask) are zero like ceres::Covariance's.
extern "C" int vcgpu_get_covariance(vcgpu_handle* h, double* cov) {
  if (!h || !cov) return VCGPU_ERR_INVALID;
  return run_cov(h, cov, kCovGlobals);
}

// Marginal covariance of every frame's tangent (GetCovarianceBlock(t_wp, t_wp) and (v_w, v_w) of ceres::Covariance):
// the [f, f] blocks of (J^T J)^-1 on the system vcgpu_get_covariance inverts, by a selected inversion of the frame
// elimination (vc_frame_cov.cuh); no step forms more than a chunk-sized or [globals | top nodes]-sized matrix.
extern "C" int vcgpu_get_frame_covariance(vcgpu_handle* h, double* cov) {
  if (!h || !cov) return VCGPU_ERR_INVALID;
  if (h->nranks > 1) return fail(h, VCGPU_ERR_INVALID, "vcgpu_get_frame_covariance is one-GPU only: frame shards are not supported");
  return run_cov(h, cov, kCovFrames);
}
extern "C" int vcgpu_get_frame_covariance_batch(vcgpu_handle* const* handles, int n, double* const* cov, int* status) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  if (!cov) return batch_refuse(handles, n, 0, "null cov array", "vcgpu_get_frame_covariance_batch");
  return run_cov_batch(handles, n, cov, status, kCovFrames);
}

// The frame blocks off the block diagonal of (J^T J)^-1 (GetCovarianceBlock(t_wp[f], globals) and (t_wp[f], t_wp[f+1])
// of ceres::Covariance, with v_w[f] on the inertial path), on the system vcgpu_get_frame_covariance inverts, from the
// same selected inversion: vision Σ_fg = -X_f Σ_gg and Σ_f,f+1 = X_f Σ_gg X_f+1^T, inertial level 0's Σ_kg and Σ_k,k+1
// of the level walk (vc_frame_cov.cuh).
extern "C" int vcgpu_get_frame_cross_covariance(vcgpu_handle* h, double* cov_fg, double* cov_fn) {
  if (!h) return VCGPU_ERR_INVALID;
  if (!cov_fg && !cov_fn) return fail(h, VCGPU_ERR_INVALID, "vcgpu_get_frame_cross_covariance: cov_fg and cov_fn are both null");
  if (h->nranks > 1) return fail(h, VCGPU_ERR_INVALID, "vcgpu_get_frame_cross_covariance is one-GPU only: frame shards are not supported");
  return run_cov(h, cov_fg, kCovCross, cov_fn);
}
extern "C" int vcgpu_get_frame_cross_covariance_batch(vcgpu_handle* const* handles, int n, double* const* cov_fg,
                                                      double* const* cov_fn, int* status) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  if (!cov_fg && !cov_fn) return batch_refuse(handles, n, 0, "null cov_fg and cov_fn arrays", "vcgpu_get_frame_cross_covariance_batch");
  // one null array stands for n null pointers
  std::vector<double*> fg(n, nullptr), fn(n, nullptr);
  for (int i = 0; i < n; ++i) {
    if (cov_fg) fg[i] = cov_fg[i];
    if (cov_fn) fn[i] = cov_fn[i];
  }
  return run_cov_batch(handles, n, fg.data(), status, kCovCross, fn.data());
}

// The pixel covariance a calibration leaves at projected points (vc_proj_cov.cuh): the matrix of vcgpu_get_covariance
// (run_cov) or the caller's, then run_proj_cov of this handle alone.  Both paths hand the kernel a host matrix, so a
// given matrix gives the same bits on either.
extern "C" int vcgpu_get_projection_covariance(vcgpu_handle* h, const double* globals_cov, const vcgpu_proj_points* pts) {
  if (!h) return VCGPU_ERR_INVALID;
  const std::string why = proj_refusal(h, pts);
  if (!why.empty()) return fail(h, VCGPU_ERR_INVALID, "vcgpu_get_projection_covariance: " + why);
  std::vector<double> own;
  if (!globals_cov) {
    int G = 0;
    vcgpu_num_globals(h, &G);
    own.resize(static_cast<size_t>(G) * G);
    VC_TRY(run_cov(h, own.data(), kCovGlobals));
    globals_cov = own.data();
  } else {
    VC_TRY(prepare(h));
  }
  return run_proj_cov(&h, 1, &globals_cov, pts);
}
extern "C" int vcgpu_get_projection_covariance_batch(vcgpu_handle* const* handles, int n, const vcgpu_proj_points* pts, int* status) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  if (!pts) return batch_refuse(handles, n, 0, "null pts array", "vcgpu_get_projection_covariance_batch");
  return run_proj_cov_batch(handles, n, pts, status);
}

// The information candidate views would add (vc_view_info.cuh): the matrix of vcgpu_get_covariance (run_cov) or the
// caller's, then run_view_info of this handle alone.  Both paths hand the kernels a host matrix, so a given matrix
// gives the same bits on either.
extern "C" int vcgpu_get_view_information(vcgpu_handle* h, const double* globals_cov, const vcgpu_view_candidates* v) {
  if (!h) return VCGPU_ERR_INVALID;
  const std::string why = view_refusal(h, v);
  if (!why.empty()) return fail(h, VCGPU_ERR_INVALID, "vcgpu_get_view_information: " + why);
  if (v->n_cand == 0) return VCGPU_OK;
  std::vector<double> own;
  if (!globals_cov) {
    int G = 0;
    vcgpu_num_globals(h, &G);
    own.resize(static_cast<size_t>(G) * G);
    VC_TRY(run_cov(h, own.data(), kCovGlobals));
    globals_cov = own.data();
  } else {
    VC_TRY(prepare(h));
  }
  int st = VCGPU_OK;
  VC_TRY(run_view_info(&h, 1, &globals_cov, v, &st));
  if (st != VCGPU_OK) return fail(h, st, "vcgpu_get_view_information: Sigma_F is not positive definite");
  return VCGPU_OK;
}
extern "C" int vcgpu_get_view_information_batch(vcgpu_handle* const* handles, int n, const vcgpu_view_candidates* v, int* status) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  if (!v) return batch_refuse(handles, n, 0, "null candidates array", "vcgpu_get_view_information_batch");
  return run_view_info_batch(handles, n, v, status);
}

// The regression diagnostics of every reprojection observation (vc_obs_infl.cuh): Σ_gg, Σ_ff and Σ_fg from one
// elimination and selected inversion of this handle (run_cov, kCovDiagCross; Σ_ff and Σ_fg stay on the device), then
// run_obs_infl of this handle alone.
extern "C" int vcgpu_get_observation_influence(vcgpu_handle* h, vcgpu_obs_influence* out) {
  if (!h) return VCGPU_ERR_INVALID;
  const std::string why = infl_refusal(h, out);
  if (!why.empty()) return fail(h, VCGPU_ERR_INVALID, "vcgpu_get_observation_influence: " + why);
  CovSpace w;
  VC_TRY(run_cov(h, nullptr, kCovDiagCross, nullptr, &w));
  const InflSrc src{w.inv, w.N, w.out_ff, w.out, w.out_next};
  int st = VCGPU_OK;
  VC_TRY(run_obs_infl(&h, 1, &src, out, &st));
  if (st != VCGPU_OK) return fail(h, st, "vcgpu_get_observation_influence: Sigma_F is not positive definite");
  return VCGPU_OK;
}
extern "C" int vcgpu_get_observation_influence_batch(vcgpu_handle* const* handles, int n, const vcgpu_obs_influence* out, int* status) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  if (!out) return batch_refuse(handles, n, 0, "null out array", "vcgpu_get_observation_influence_batch");
  return run_obs_infl_batch(handles, n, out, status);
}

// The regression diagnostics of every IMU interval (vc_imu_infl.cuh), and of every observation where obs is given, from
// one elimination and selected inversion of this handle (run_cov, kCovDiagCross), then run_imu_infl of this handle alone.
extern "C" int vcgpu_get_imu_influence(vcgpu_handle* h, vcgpu_imu_influence* imu, vcgpu_obs_influence* obs) {
  if (!h) return VCGPU_ERR_INVALID;
  const std::string why = imu_infl_refusal(h, imu, obs);
  if (!why.empty()) return fail(h, VCGPU_ERR_INVALID, "vcgpu_get_imu_influence: " + why);
  CovSpace w;
  const int rc = run_cov(h, nullptr, kCovDiagCross, nullptr, &w);
  if (rc == VCGPU_ERR_NUMERIC) return fail(h, rc, "vcgpu_get_imu_influence: J^T J is singular at the current state");
  VC_TRY(rc);
  const InflSrc src{w.inv, w.N, w.out_ff, w.out, w.out_next};
  int st = VCGPU_OK;
  VC_TRY(run_imu_infl(&h, 1, &src, imu, obs, &st));
  if (st != VCGPU_OK) return fail(h, st, "vcgpu_get_imu_influence: Sigma_F is not positive definite");
  return VCGPU_OK;
}
extern "C" int vcgpu_get_imu_influence_batch(vcgpu_handle* const* handles, int n, const vcgpu_imu_influence* imu,
                                             const vcgpu_obs_influence* obs, int* status) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  if (!imu) return batch_refuse(handles, n, 0, "null imu array", "vcgpu_get_imu_influence_batch");
  return run_imu_infl_batch(handles, n, imu, obs, status);
}


// Batched PosePnPRansac (vicalib-task.cc:322-325): pose of the planar target in every (frame, camera) view, one warp
// per view (vc_pnp.cuh): run_pnp_batch of this handle alone.  Cameras (model, intrinsics) are the ones given to
// vcgpu_set_cameras.
extern "C" int vcgpu_pose_pnp_ransac(vcgpu_handle* h, int n_views, const int32_t* cam_id, const int64_t* start, const int32_t* count,
                                     const double* pix, const double* pw, int robust_its, double robust_tol, double* T_cw,
                                     double* rmse, int32_t* n_used) {
  if (!h) return VCGPU_ERR_INVALID;
  const vcgpu_pnp_views views{n_views, cam_id, start, count, pix, pw, T_cw, rmse, n_used};
  return run_pnp_batch(&h, 1, &views, robust_its, robust_tol, "vcgpu_pose_pnp_ransac");
}

extern "C" int vcgpu_pose_pnp_ransac_batch(vcgpu_handle* const* handles, int n, const vcgpu_pnp_views* views, int robust_its,
                                           double robust_tol) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  if (!views) return batch_refuse(handles, n, 0, "null views array", "vcgpu_pose_pnp_ransac_batch");
  return run_pnp_batch(handles, n, views, robust_its, robust_tol, "vcgpu_pose_pnp_ransac_batch");
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

// Each IMU interval's Mahalanobis distance as UpdateImuWeights logs it (vicalibrator.h:786-794): run_imu_mahalanobis_batch
// of this handle alone
extern "C" int vcgpu_get_imu_mahalanobis(vcgpu_handle* h, double* dist, double* r_or_null) {
  if (!h) return VCGPU_ERR_INVALID;
  return run_imu_mahalanobis_batch(&h, 1, &dist, &r_or_null, "vcgpu_get_imu_mahalanobis");
}
extern "C" int vcgpu_get_imu_mahalanobis_batch(vcgpu_handle* const* handles, int n, double* const* dist, double* const* r) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  if (!dist) return batch_refuse(handles, n, 0, "null dist array", "vcgpu_get_imu_mahalanobis_batch");
  return run_imu_mahalanobis_batch(handles, n, dist, r, "vcgpu_get_imu_mahalanobis_batch");
}

// GetIntegrationPoses of every interval (vicalibrator.h:508-533): run_integration_poses_batch of this handle alone
extern "C" int vcgpu_get_integration_poses(vcgpu_handle* h, int64_t* start, double* poses_or_null) {
  if (!h) return VCGPU_ERR_INVALID;
  return run_integration_poses_batch(&h, 1, &start, &poses_or_null, "vcgpu_get_integration_poses");
}
extern "C" int vcgpu_get_integration_poses_batch(vcgpu_handle* const* handles, int n, int64_t* const* start,
                                                 double* const* poses) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  if (!start) return batch_refuse(handles, n, 0, "null start array", "vcgpu_get_integration_poses_batch");
  return run_integration_poses_batch(handles, n, start, poses, "vcgpu_get_integration_poses_batch");
}

// hand-eye alignment of the gyro stream with the vision poses: run_align_imu_batch of this handle alone
extern "C" int vcgpu_align_imu(vcgpu_handle* h, const vcgpu_imu_align_opts* opts, vcgpu_imu_alignment* out) {
  if (!h) return VCGPU_ERR_INVALID;
  if (!opts || !out) return fail(h, VCGPU_ERR_INVALID, "vcgpu_align_imu: null opts or out");
  return run_align_imu_batch(&h, 1, opts, out, nullptr, "vcgpu_align_imu");
}
extern "C" int vcgpu_align_imu_batch(vcgpu_handle* const* handles, int n, const vcgpu_imu_align_opts* opts,
                                     vcgpu_imu_alignment* out, int* status) {
  if (!handles || n <= 0) return VCGPU_ERR_INVALID;
  if (!opts) return batch_refuse(handles, n, 0, "null opts array", "vcgpu_align_imu_batch");
  if (!out) return batch_refuse(handles, n, 0, "null out array", "vcgpu_align_imu_batch");
  return run_align_imu_batch(handles, n, opts, out, status, "vcgpu_align_imu_batch");
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
