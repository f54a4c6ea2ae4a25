// vcgpu_evaluate, vcgpu_remove_outliers and their batches: the loss-free reprojection residuals (reproj_residual) of
// every camera of one or many rigs in one launch, reduced per (rig, camera) on the device.
//
// The work is cut into tiles of kEvalTile consecutive observations of one (rig, camera) in the rig's sorted (camera,
// frame) order, one CTA per tile.  The tiling is a function of the rig alone, so a large rig spreads over the whole GPU
// and a rig's sums run in the same order whatever else is in the launch.  Each tile writes its partial of sum |r|^2 to
// a slot of its own; the tile that takes the last ticket of its (rig, camera) adds the partials in tile order.
#pragma once
#include "vc_internal.h"
#include "vc_math.cuh"
#include "vc_kernels.cuh"

namespace vc {

constexpr int kEvalTile = 256;  // observations per tile = threads per CTA

// one rig of the launch; observation arrays are the rig's sorted device copies
struct EvalBatchRig {
  const double* state[2];
  const Ctl* ctl;            // the evaluated buffer is pick(ctl, 0)
  int64_t off_cam;           // state offset of camera 0's 17 doubles
  const int32_t* frame;
  const double *pw, *pc;     // AoS [n][3], [n][2]
  const int32_t* rank;       // sorted index -> index among the active observations in caller order; null: the same
  double* res;               // null, or [2 * n_obs]: the active observations' residuals in caller order
  uint8_t* mark;             // null, or [n_obs] sorted: 1 where |r| > limit[camera]
  int model[kMaxCams], obs_start[kMaxCams], n_obs[kMaxCams];
  double limit[kMaxCams];    // threshold * rmse[c], formed on the host
};
// tile `tile` of the n_tiles of camera `cam` of rig `rig`; its partial goes to part[part0 + tile], the camera's cost and
// ticket counter are entry `sum`
struct EvalTile { int rig, cam, tile, n_tiles, part0, sum; };
struct EvalBatchArgs {
  const EvalBatchRig* rigs;
  const EvalTile* tiles;
  double* part;
  double* cost;        // 1/2 sum |r|^2 per (rig, camera) entry
  unsigned* counter;   // tickets per (rig, camera) entry, zero at launch
};

// the residual of sorted observation i of camera c of rig g
template <int MODEL>
__device__ __forceinline__ void eval_batch_residual(const EvalBatchRig& g, const double* state, int c, int64_t i, double* r0, double* r1) {
  V3 pk;
  double R[9];
  reproj_residual<MODEL>(state + 7 * static_cast<int64_t>(g.frame[i]), state + g.off_cam + kCamStateStride * c, g.pw + 3 * i, g.pc + 2 * i,
                         r0, r1, &pk, R, nullptr, nullptr);
}

// sum of v over the CTA in a fixed order (lanes by shuffle, then warps in order); the result is valid in thread 0
__device__ __forceinline__ double eval_batch_block_sum(double v, double* wsum) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kEvalTile / 32; ++w) s += wsum[w];
  __syncthreads();
  return s;
}

__global__ void __launch_bounds__(kEvalTile) eval_batch_kernel(EvalBatchArgs a) {
  __shared__ double wsum[kEvalTile / 32];
  __shared__ int is_last;
  const EvalTile t = a.tiles[blockIdx.x];
  const EvalBatchRig& g = a.rigs[t.rig];
  const int c = t.cam, local = t.tile * kEvalTile + static_cast<int>(threadIdx.x);
  double s = 0.0;
  if (local < g.n_obs[c]) {
    const int64_t i = static_cast<int64_t>(g.obs_start[c]) + local;
    const double* state = g.state[pick(g.ctl, 0)];
    double r0, r1;
    switch (g.model[c]) {  // uniform across the tile
      case kLinear: eval_batch_residual<kLinear>(g, state, c, i, &r0, &r1); break;
      case kFov: eval_batch_residual<kFov>(g, state, c, i, &r0, &r1); break;
      case kPoly2: eval_batch_residual<kPoly2>(g, state, c, i, &r0, &r1); break;
      case kPoly3: eval_batch_residual<kPoly3>(g, state, c, i, &r0, &r1); break;
      default: eval_batch_residual<kKb4>(g, state, c, i, &r0, &r1); break;
    }
    // not contracted into an FMA: |r| is sqrt(r0 * r0 + r1 * r1) with every operation rounded, as RemoveOutliers forms it
    // (vicalibrator.h:890-893)
    s = __dadd_rn(__dmul_rn(r0, r0), __dmul_rn(r1, r1));
    if (g.res) {
      const int64_t o = g.rank ? static_cast<int64_t>(g.rank[i]) : i;
      g.res[2 * o] = r0;
      g.res[2 * o + 1] = r1;
    }
    if (g.mark) g.mark[i] = sqrt(s) > g.limit[c] ? 1 : 0;
  }
  const double tile_sum = eval_batch_block_sum(s, wsum);
  if (threadIdx.x == 0) {
    a.part[t.part0 + t.tile] = tile_sum;
    __threadfence();
    is_last = atomicAdd(a.counter + t.sum, 1u) == static_cast<unsigned>(t.n_tiles - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  double p = 0.0;
  for (int k = threadIdx.x; k < t.n_tiles; k += kEvalTile) p += __ldcg(a.part + t.part0 + k);
  const double total = eval_batch_block_sum(p, wsum);
  if (threadIdx.x == 0) a.cost[t.sum] = 0.5 * total;
}

}  // namespace vc
