// ViCalibrator::GetIntegrationPoses for every interval of a batch of rigs (vicalibrator.h:508-533): the poses the
// double-precision RK4 of ImuResidualT::IntegrateResidual (types.h:611-687, the no-Jacobian branch of IntegrateImu
// :575-594) passes through from frame k over the measurements GetRange(t_k, t_k+1, ts) returns
// (interpolation-buffer.h:208-226).  One thread per interval; the interpolation and the RK4 step are vc_imu_math.cuh's.
//   count pass   each interval's number of measurements (= its number of poses) into start[k]
//   scan         one CTA per rig turns start[0 .. ni-1] into offsets, start[ni] the rig's total
//   fill pass    the start pose, then one pose per later measurement, kPoseOut doubles each
// Nothing is written but the outputs: state, IMU weights and the weight update's eigenvectors stay as they are.
#pragma once
#include "vc_imu_math.cuh"

namespace vc {
namespace imu {

constexpr int kPoseOut = 14;  // q (x y z w), t (3), v_w (3), w_w (3), time
constexpr int kPoseThreads = 128;
constexpr int kPoseScanThreads = 1024;

// one rig's entry in the argument table
struct PosesRig {
  ImuBuf buf;
  const double* ftime;  // [ni + 1] frame times
  const double* state;  // the accepted state
  int64_t off_v, off_imu;
  int64_t* start;       // [ni + 1]: counts after the count pass, offsets after the scan
  double* poses;        // [start[ni]][kPoseOut], null: the fill pass skips the rig
  int ni, i0;           // intervals; the first one's index over the whole table
};

struct NoTangent {  // integrate_imu's tangent hook, unused here
  template <class Q, class Z>
  __device__ __forceinline__ void stage(int, const Q&, const Z&) {}
  __device__ __forceinline__ void step(double) {}
};

__device__ __forceinline__ void put_pose(double* o, const Pose<double>& y, const Vec<double>& w, double time) {
  o[0] = y.q.x; o[1] = y.q.y; o[2] = y.q.z; o[3] = y.q.w;
  o[4] = y.p.x; o[5] = y.p.y; o[6] = y.p.z;
  o[7] = y.v.x; o[8] = y.v.y; o[9] = y.v.z;
  o[10] = w.x; o[11] = w.y; o[12] = w.z;
  o[13] = time;
}

// interval k of rig a.  kFill false: its count into a.start[k]; true: its poses at a.poses + kPoseOut * a.start[k]
template <bool kFill>
__device__ void integration_poses_interval(const PosesRig& a, int k) {
  const double* X1 = a.state + 7 * static_cast<int64_t>(k);
  const double* V1 = a.state + a.off_v + 3 * static_cast<int64_t>(k);
  const double* P = a.state + a.off_imu;
  const double ts = P[14];
  const double t_start = a.ftime[k], t_end = a.ftime[k + 1];
  // GetRange adds nothing unless HasElement(t_start) (interpolation-buffer.h:122-125, 217)
  if (!(t_start >= a.buf.start_time + ts && t_start <= a.buf.end_time + ts) || a.buf.n == 0) {
    if (!kFill) a.start[k] = 0;
    return;
  }
  int idx;
  Meas<double> prev = get_element<double>(a.buf, t_start, ts, &idx), cur;
  if constexpr (!kFill) {
    int64_t m = 1;  // GetElement(t_start), then one per GetNext: the last one (false) interpolates t_end
    while (get_next<double>(a.buf, t_end, ts, &idx, &cur)) ++m;
    a.start[k] = m + 1;
  } else {
    double* o = a.poses + kPoseOut * a.start[k];
    const Vec<double> g = gravity_vector<double>(P[0], P[1]);
    const Vec<double> bg{P[2], P[3], P[4]}, ba{P[5], P[6], P[7]};
    double sf[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) sf[i] = P[8 + i];
    // the frame's ImuPoseT: its pose, velocity, w_w_ = 0 and time (types.h:178-180)
    Pose<double> y{{X1[4], X1[5], X1[6]}, {X1[0], X1[1], X1[2], X1[3]}, {V1[0], V1[1], V1[2]}};
    Vec<double> w{0.0, 0.0, 0.0};
    double time = t_start;
    put_pose(o, y, w, time);
    NoTangent nt;
    bool more = true;
    while (more) {
      more = get_next<double>(a.buf, t_end, ts, &idx, &cur);
      y = integrate_imu(y, prev, cur, bg, ba, sf, g, nt, &w);
      if (cur.time != prev.time) time = cur.time;  // dt == 0: the previous pose, time and w_w_ included (types.h:440-442)
      prev = cur;
      o += kPoseOut;
      put_pose(o, y, w, time);
    }
  }
}

// the rig of table entry t (an interval index over the whole table): the last with i0 <= t
__device__ __forceinline__ int poses_rig(const PosesRig* rigs, int n_rigs, int t) {
  int lo = 0, hi = n_rigs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (rigs[mid].i0 <= t) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// count (kFill false) or fill pass over the `intervals` intervals of n_rigs rigs, one thread each
template <bool kFill>
__global__ void __launch_bounds__(kPoseThreads) integration_poses_kernel(const PosesRig* rigs, int n_rigs, int intervals) {
  const int t = blockIdx.x * kPoseThreads + threadIdx.x;
  if (t >= intervals) return;
  const PosesRig& a = rigs[poses_rig(rigs, n_rigs, t)];
  if (kFill && !a.poses) return;
  integration_poses_interval<kFill>(a, t - a.i0);
}

// exclusive prefix sum of rig blockIdx.x's counts, in place: start[k] = sum of counts before k, start[ni] = the total
__global__ void __launch_bounds__(kPoseScanThreads) integration_poses_scan_kernel(const PosesRig* rigs) {
  __shared__ int64_t warp_sum[kPoseScanThreads / 32];
  const PosesRig& a = rigs[blockIdx.x];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int64_t carry = 0;
  for (int base = 0; base < a.ni; base += kPoseScanThreads) {
    const int k = base + threadIdx.x;
    const int64_t v = k < a.ni ? a.start[k] : 0;
    int64_t s = v;  // inclusive scan within the warp
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int64_t u = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += u;
    }
    if (lane == 31) warp_sum[wid] = s;
    __syncthreads();
    if (wid == 0) {
      int64_t x = warp_sum[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int64_t u = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += u;
      }
      warp_sum[lane] = x;  // inclusive over warps
    }
    __syncthreads();
    const int64_t before = carry + (wid > 0 ? warp_sum[wid - 1] : 0);
    if (k < a.ni) a.start[k] = before + s - v;
    carry += warp_sum[kPoseScanThreads / 32 - 1];
    __syncthreads();  // warp_sum is rewritten by the next chunk
  }
  if (threadIdx.x == 0) a.start[a.ni] = carry;
}

}  // namespace imu
}  // namespace vc
