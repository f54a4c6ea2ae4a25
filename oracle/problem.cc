// ORACLE — TEST INFRASTRUCTURE ONLY.  Parity unpinned (see oracle/README.md).
// See problem.h for the reference lines each piece restates.
#include "problem.h"

#include <cmath>
#include <cstring>
#include <thread>

#include "imu_weights.h"

namespace vo {

// ------------------------------------------------------------------ layout
void NormalEq::Resize(int nf_, int fd_, int G_) {
  nf = nf_; fd = fd_; G = G_;
  B.assign(static_cast<size_t>(nf) * fd * fd, 0.0);
  U.assign(static_cast<size_t>(nf) * fd * fd, 0.0);
  E.assign(static_cast<size_t>(nf) * fd * G, 0.0);
  gf.assign(static_cast<size_t>(nf) * fd, 0.0);
  C.assign(static_cast<size_t>(G) * G, 0.0);
  gc.assign(G, 0.0);
  cost = 0;
}
void NormalEq::Zero() {
  std::fill(B.begin(), B.end(), 0.0);
  std::fill(U.begin(), U.end(), 0.0);
  std::fill(E.begin(), E.end(), 0.0);
  std::fill(gf.begin(), gf.end(), 0.0);
  std::fill(C.begin(), C.end(), 0.0);
  std::fill(gc.begin(), gc.end(), 0.0);
  cost = 0;
}

int Problem::CamOffset(int c) const {
  int off = 0;
  for (int i = 0; i < c; ++i) off += 6 + NumIntrinsics(model[i]);
  return off;
}
int Problem::ImuOffset() const { return CamOffset(n_cams); }
int Problem::NumGlobals() const { return ImuOffset() + (flags.inertial ? 15 : 0); }

// vicalibrator.h:572-592, 657-676.  A camera no active observation sees is in no residual (the IMU residual takes no
// camera block, vicalibrator.h:628-632): Ceres removes its blocks like those of an unused frame.
void Problem::GlobalMask(std::vector<double>* mask) const {
  mask->assign(NumGlobals(), 1.0);
  std::vector<uint8_t> seen(n_cams, 0);
  for (int64_t i = 0; i < n_obs; ++i)
    if (obs_active[i]) seen[obs_cam[i]] = 1;
  for (int c = 0; c < n_cams; ++c) {
    const int off = CamOffset(c), K = NumIntrinsics(model[c]);
    if (c == 0) {
      const double rot = flags.inertial ? 1.0 : 0.0;
      const double trans = (flags.inertial && !flags.rotation_only) ? 1.0 : 0.0;
      for (int i = 0; i < 3; ++i) (*mask)[off + i] = rot;
      for (int i = 0; i < 3; ++i) (*mask)[off + 3 + i] = trans;
    }
    if (flags.fix_intrinsics)
      for (int i = 0; i < K; ++i) (*mask)[off + 6 + i] = 0.0;
    if (!seen[c])
      for (int i = 0; i < 6 + K; ++i) (*mask)[off + i] = 0.0;
  }
  if (flags.inertial) {
    const int o = ImuOffset();
    const double gact = flags.rotation_only ? 0.0 : 1.0;
    (*mask)[o] = (*mask)[o + 1] = gact;
    for (int i = 0; i < 6; ++i) (*mask)[o + 2 + i] = flags.bias_active ? 1.0 : 0.0;
    for (int i = 0; i < 6; ++i) (*mask)[o + 8 + i] = flags.scale_active ? 1.0 : 0.0;
    (*mask)[o + 14] = flags.optimize_ts ? 1.0 : 0.0;
  }
}

int Problem::NumResiduals() const {
  int64_t n = 0;
  if (flags.visual) {
    int64_t act = 0;
    for (int64_t i = 0; i < n_obs; ++i) act += obs_active[i];
    n += static_cast<int64_t>(2 * act * flags.visual_mult);
  }
  if (flags.inertial && n_frames > 1) n += static_cast<int64_t>(9 * (n_frames - 1) * flags.imu_mult);
  return static_cast<int>(n);
}

void Problem::ResetImuWeights() {
  const int ni = n_frames > 1 ? n_frames - 1 : 0;
  w_sqrt.assign(static_cast<size_t>(ni) * 81, 0.0);
  for (int k = 0; k < ni; ++k)
    for (int i = 0; i < 9; ++i) w_sqrt[static_cast<size_t>(k) * 81 + i * 9 + i] = 500.0;
}

void Problem::UpdateImuWeights() {
  // vicalibrator.h:725
  if (!(flags.inertial && !flags.rotation_only)) return;
  const int ni = n_frames - 1;
  auto work = [&](int k0, int k1) {
    for (int k = k0; k < k1; ++k)
      UpdateOneImuWeight(imu, ftime[k], ftime[k + 1], ts, &T_wp[7 * k], &v_w[3 * k],
                         &T_wp[7 * (k + 1)], &v_w[3 * (k + 1)], b, sf, g, sigma_g, sigma_a,
                         &w_sqrt[static_cast<size_t>(k) * 81]);
  };
  const int nt = std::max(1, opts.num_threads);
  if (nt == 1 || ni < 64) { work(0, ni); return; }
  std::vector<std::thread> th;
  for (int t = 0; t < nt; ++t) th.emplace_back(work, ni * t / nt, ni * (t + 1) / nt);
  for (auto& t : th) t.join();
}

// ------------------------------------------------------------------ residual blocks
template <class Cam>
static void EvalReprojT(const Problem& P, int64_t i, double r[2], double* J) {
  constexpr int K = Cam::K, N = 14 + K, NT = 12 + K;
  const int f = P.obs_frame[i], c = P.obs_cam[i];
  const double* twk = &P.T_wp[7 * f];
  const double* qck = &P.q_ck[4 * c];
  const double* pck = &P.p_ck[3 * c];
  const double* ip = &P.intr[10 * c];
  if (J == nullptr) {
    ReprojectionResidual<Cam, double>(twk, qck, pck, ip, &P.p_w[3 * i], &P.p_c[2 * i], r);
    return;
  }
  using D = Dual<N>;
  D a[7], q[4], t[3], cp[K], res[2];
  for (int k = 0; k < 7; ++k) a[k] = D(twk[k], k);
  for (int k = 0; k < 4; ++k) q[k] = D(qck[k], 7 + k);
  for (int k = 0; k < 3; ++k) t[k] = D(pck[k], 11 + k);
  for (int k = 0; k < K; ++k) cp[k] = D(ip[k], 14 + k);
  ReprojectionResidual<Cam, D>(a, q, t, cp, &P.p_w[3 * i], &P.p_c[2 * i], res);
  double L7[42], L4[12];
  LocalParamSe3Jacobian(twk, L7);
  LocalParamSo3Jacobian(qck, L4);
  for (int row = 0; row < 2; ++row) {
    r[row] = res[row].a;
    double* Jr = J + row * NT;
    for (int col = 0; col < 6; ++col) {
      double s = 0;
      for (int k = 0; k < 7; ++k) s += res[row].v[k] * L7[k * 6 + col];
      Jr[col] = s;
    }
    for (int col = 0; col < 3; ++col) {
      double s = 0;
      for (int k = 0; k < 4; ++k) s += res[row].v[7 + k] * L4[k * 3 + col];
      Jr[6 + col] = s;
    }
    for (int k = 0; k < 3 + K; ++k) Jr[9 + k] = res[row].v[11 + k];
  }
}

void Problem::EvalReprojection(int64_t i, double r[2], double* J) const {
  switch (model[obs_cam[i]]) {
    case kLinear: EvalReprojT<LinearCam>(*this, i, r, J); break;
    case kFov: EvalReprojT<FovCam>(*this, i, r, J); break;
    case kPoly2: EvalReprojT<Poly2Cam>(*this, i, r, J); break;
    case kPoly3: EvalReprojT<Poly3Cam>(*this, i, r, J); break;
    case kKb4: EvalReprojT<Kb4Cam>(*this, i, r, J); break;
  }
}

void Problem::EvalImu(int k, double r[9], double* J) const {
  const double* x2 = &T_wp[7 * (k + 1)];
  const double* x1 = &T_wp[7 * k];
  const double* v2 = &v_w[3 * (k + 1)];
  const double* v1 = &v_w[3 * k];
  const double* W = &w_sqrt[static_cast<size_t>(k) * 81];
  const bool sw = flags.rotation_only != 0;
  if (J == nullptr) {
    ImuResidual<double>(imu, ftime[k], ftime[k + 1], W, sw, x2, x1, v2, v1, g, b, sf, &ts, r);
    return;
  }
  using D = Dual<35>;
  D a2[7], a1[7], d2[3], d1[3], dg[2], db[6], dsf[6], dts, res[9];
  int o = 0;
  for (int i = 0; i < 7; ++i) a2[i] = D(x2[i], o++);
  for (int i = 0; i < 7; ++i) a1[i] = D(x1[i], o++);
  for (int i = 0; i < 3; ++i) d2[i] = D(v2[i], o++);
  for (int i = 0; i < 3; ++i) d1[i] = D(v1[i], o++);
  for (int i = 0; i < 2; ++i) dg[i] = D(g[i], o++);
  for (int i = 0; i < 6; ++i) db[i] = D(b[i], o++);
  for (int i = 0; i < 6; ++i) dsf[i] = D(sf[i], o++);
  dts = D(ts, o++);
  ImuResidual<D>(imu, ftime[k], ftime[k + 1], W, sw, a2, a1, d2, d1, dg, db, dsf, &dts, res);
  double L2[42], L1[42];
  LocalParamSe3Jacobian(x2, L2);
  LocalParamSe3Jacobian(x1, L1);
  for (int row = 0; row < 9; ++row) {
    r[row] = res[row].a;
    double* Jr = J + row * 33;
    for (int col = 0; col < 6; ++col) {
      double s2 = 0, s1 = 0;
      for (int i = 0; i < 7; ++i) {
        s2 += res[row].v[i] * L2[i * 6 + col];
        s1 += res[row].v[7 + i] * L1[i * 6 + col];
      }
      Jr[col] = s2;
      Jr[6 + col] = s1;
    }
    for (int i = 0; i < 21; ++i) Jr[12 + i] = res[row].v[14 + i];
  }
}

// ------------------------------------------------------------------ evaluation
namespace {
struct Accum {
  NormalEq* ne;
  double cost = 0;
};

void AccumulateRange(const Problem& P, const std::vector<double>& mask, int64_t o0, int64_t o1, int k0,
                     int k1, NormalEq* ne, double* cost_out) {
  const int fd = P.FrameDim(), G = P.NumGlobals();
  double cost = 0;
  double r[9], J[9 * 33];
  if (P.flags.visual) {
    const double m = P.flags.visual_mult;
    for (int64_t i = o0; i < o1; ++i) {
      if (!P.obs_active[i]) continue;
      const int f = P.obs_frame[i], c = P.obs_cam[i];
      const int K = NumIntrinsics(P.model[c]), NT = 12 + K, NG = 6 + K, off = P.CamOffset(c);
      P.EvalReprojection(i, r, ne ? J : nullptr);
      const double s = r[0] * r[0] + r[1] * r[1];
      double rho[3];
      SoftLOne(0.5, s, rho);  // vicalibrator.h:127
      cost += 0.5 * rho[0] * m;
      if (!ne) continue;
      const double sc = std::sqrt(rho[1]);  // corrector with rho'' < 0: scale r and J by sqrt(rho')
      r[0] *= sc; r[1] *= sc;
      for (int row = 0; row < 2; ++row) {
        double* Jr = J + row * NT;
        for (int k = 0; k < 6; ++k) Jr[k] *= sc;
        for (int k = 0; k < NG; ++k) Jr[6 + k] *= sc * mask[off + k];
      }
      double* B = &ne->B[static_cast<size_t>(f) * fd * fd];
      double* E = &ne->E[static_cast<size_t>(f) * fd * G];
      double* gf = &ne->gf[static_cast<size_t>(f) * fd];
      for (int row = 0; row < 2; ++row) {
        const double* Jr = J + row * NT;
        for (int a = 0; a < 6; ++a) {
          const double ja = Jr[a] * m;
          for (int bb = 0; bb < 6; ++bb) B[a * fd + bb] += ja * Jr[bb];
          for (int bb = 0; bb < NG; ++bb) E[a * G + off + bb] += ja * Jr[6 + bb];
          gf[a] += ja * r[row];
        }
        for (int a = 0; a < NG; ++a) {
          const double ja = Jr[6 + a] * m;
          double* Crow = &ne->C[static_cast<size_t>(off + a) * G + off];
          for (int bb = 0; bb < NG; ++bb) Crow[bb] += ja * Jr[6 + bb];
          ne->gc[off + a] += ja * r[row];
        }
      }
    }
  }
  if (P.flags.inertial) {
    const double m = P.flags.imu_mult;
    const int io = P.ImuOffset();
    for (int k = k0; k < k1; ++k) {
      P.EvalImu(k, r, ne ? J : nullptr);
      double s = 0;
      for (int i = 0; i < 9; ++i) s += r[i] * r[i];
      double rho[3];
      Cauchy(100.0, s, rho);  // vicalibrator.h:133
      cost += 0.5 * rho[0] * m;
      if (!ne) continue;
      const double sc = std::sqrt(rho[1]);
      // local J: [frame k (pose1 6, v1 3) | frame k+1 (pose2 6, v2 3) | imu globals 15]
      double Jl[9 * 33];
      for (int row = 0; row < 9; ++row) {
        const double* Jr = J + row * 33;
        double* o = Jl + row * 33;
        for (int i = 0; i < 6; ++i) o[i] = Jr[6 + i] * sc;
        for (int i = 0; i < 3; ++i) o[6 + i] = Jr[15 + i] * sc;
        for (int i = 0; i < 6; ++i) o[9 + i] = Jr[i] * sc;
        for (int i = 0; i < 3; ++i) o[15 + i] = Jr[12 + i] * sc;
        for (int i = 0; i < 15; ++i) o[18 + i] = Jr[18 + i] * sc * mask[io + i];
        r[row] *= sc;
      }
      double* B1 = &ne->B[static_cast<size_t>(k) * 81];
      double* B2 = &ne->B[static_cast<size_t>(k + 1) * 81];
      double* U2 = &ne->U[static_cast<size_t>(k + 1) * 81];
      double* E1 = &ne->E[static_cast<size_t>(k) * 9 * G];
      double* E2 = &ne->E[static_cast<size_t>(k + 1) * 9 * G];
      double* g1 = &ne->gf[static_cast<size_t>(k) * 9];
      double* g2 = &ne->gf[static_cast<size_t>(k + 1) * 9];
      for (int row = 0; row < 9; ++row) {
        const double* o = Jl + row * 33;
        for (int a = 0; a < 9; ++a) {
          const double j1 = o[a] * m, j2 = o[9 + a] * m;
          for (int bb = 0; bb < 9; ++bb) {
            B1[a * 9 + bb] += j1 * o[bb];
            B2[a * 9 + bb] += j2 * o[9 + bb];
            U2[a * 9 + bb] += j1 * o[9 + bb];
          }
          for (int bb = 0; bb < 15; ++bb) {
            E1[a * G + io + bb] += j1 * o[18 + bb];
            E2[a * G + io + bb] += j2 * o[18 + bb];
          }
          g1[a] += j1 * r[row];
          g2[a] += j2 * r[row];
        }
        for (int a = 0; a < 15; ++a) {
          const double ja = o[18 + a] * m;
          double* Crow = &ne->C[static_cast<size_t>(io + a) * G + io];
          for (int bb = 0; bb < 15; ++bb) Crow[bb] += ja * o[18 + bb];
          ne->gc[io + a] += ja * r[row];
        }
      }
    }
  }
  *cost_out = cost;
}
}  // namespace

double Problem::Evaluate(NormalEq* ne) const {
  const int fd = FrameDim(), G = NumGlobals();
  std::vector<double> mask;
  GlobalMask(&mask);
  if (ne) {
    if (ne->nf != n_frames || ne->fd != fd || ne->G != G) ne->Resize(n_frames, fd, G);
    ne->Zero();
  }
  const int ni = (flags.inertial && n_frames > 1) ? n_frames - 1 : 0;
  const int nt = std::max(1, opts.num_threads);
  double cost = 0;
  if (nt == 1) {
    AccumulateRange(*this, mask, 0, n_obs, 0, ni, ne, &cost);
  } else {
    std::vector<NormalEq> parts(ne ? nt - 1 : 0);
    std::vector<double> costs(nt, 0.0);
    std::vector<std::thread> th;
    for (int t = 0; t < nt; ++t) {
      NormalEq* target = nullptr;
      if (ne) {
        if (t == 0) target = ne;
        else { parts[t - 1].Resize(n_frames, fd, G); target = &parts[t - 1]; }
      }
      th.emplace_back(AccumulateRange, std::cref(*this), std::cref(mask), n_obs * t / nt,
                      n_obs * (t + 1) / nt, ni * t / nt, ni * (t + 1) / nt, target, &costs[t]);
    }
    for (auto& t : th) t.join();
    for (int t = 0; t < nt; ++t) cost += costs[t];
    if (ne) {
      for (auto& p : parts) {
        for (size_t i = 0; i < ne->B.size(); ++i) ne->B[i] += p.B[i];
        for (size_t i = 0; i < ne->U.size(); ++i) ne->U[i] += p.U[i];
        for (size_t i = 0; i < ne->E.size(); ++i) ne->E[i] += p.E[i];
        for (size_t i = 0; i < ne->gf.size(); ++i) ne->gf[i] += p.gf[i];
        for (size_t i = 0; i < ne->C.size(); ++i) ne->C[i] += p.C[i];
        for (size_t i = 0; i < ne->gc.size(); ++i) ne->gc[i] += p.gc[i];
      }
    }
  }
  if (ne) ne->cost = cost;
  return cost;
}

double Problem::EvaluateCamera(int cam, std::vector<double>* residuals) const {
  double cost = 0;
  if (residuals) residuals->clear();
  for (int64_t i = 0; i < n_obs; ++i) {
    if (obs_cam[i] != cam || !obs_active[i]) continue;
    double r[2];
    EvalReprojection(i, r, nullptr);
    cost += 0.5 * (r[0] * r[0] + r[1] * r[1]);
    if (residuals) { residuals->push_back(r[0]); residuals->push_back(r[1]); }
  }
  return cost;
}

int Problem::RemoveOutliers(const std::vector<double>& rmse, double threshold_mult) {
  int removed = 0;
  for (int64_t i = 0; i < n_obs; ++i) {
    if (!obs_active[i]) continue;
    double r[2];
    EvalReprojection(i, r, nullptr);
    const double err = std::sqrt(r[0] * r[0] + r[1] * r[1]);
    if (err > threshold_mult * rmse[obs_cam[i]]) { obs_active[i] = 0; ++removed; }
  }
  return removed;
}

// ------------------------------------------------------------------ state
Problem::State Problem::Save() const {
  State s;
  s.intr = intr; s.q_ck = q_ck; s.p_ck = p_ck; s.T_wp = T_wp; s.v_w = v_w;
  std::memcpy(s.g, g, sizeof g); std::memcpy(s.b, b, sizeof b); std::memcpy(s.sf, sf, sizeof sf);
  s.ts = ts;
  return s;
}
void Problem::Restore(const State& s) {
  intr = s.intr; q_ck = s.q_ck; p_ck = s.p_ck; T_wp = s.T_wp; v_w = s.v_w;
  std::memcpy(g, s.g, sizeof g); std::memcpy(b, s.b, sizeof b); std::memcpy(sf, s.sf, sizeof sf);
  ts = s.ts;
}
// Ceres minimises over the blocks that are neither constant nor unused (Program::RemoveFixedBlocks): those are never
// moved and are not part of x_norm.  Constant blocks are the zero entries of GlobalMask.  Every frame of an inertial
// run is in an IMU residual; a frame of a vision-only run is used iff an active observation sees it.
void Problem::FramesUsed(std::vector<uint8_t>* used) const {
  used->assign(n_frames, flags.inertial ? 1 : 0);
  if (flags.inertial) return;
  for (int64_t i = 0; i < n_obs; ++i)
    if (obs_active[i]) (*used)[obs_frame[i]] = 1;
}
double Problem::StateNorm() const {
  std::vector<double> mask;
  std::vector<uint8_t> used;
  GlobalMask(&mask);
  FramesUsed(&used);
  double s = 0;
  for (int f = 0; f < n_frames; ++f) {
    if (!used[f]) continue;
    for (int i = 0; i < 7; ++i) s += T_wp[7 * f + i] * T_wp[7 * f + i];
    if (flags.inertial) for (int i = 0; i < 3; ++i) s += v_w[3 * f + i] * v_w[3 * f + i];
  }
  for (int c = 0; c < n_cams; ++c) {
    const int off = CamOffset(c), K = NumIntrinsics(model[c]);
    if (mask[off]) for (int i = 0; i < 4; ++i) s += q_ck[4 * c + i] * q_ck[4 * c + i];
    if (mask[off + 3]) for (int i = 0; i < 3; ++i) s += p_ck[3 * c + i] * p_ck[3 * c + i];
    if (K > 0 && mask[off + 6]) for (int i = 0; i < K; ++i) s += intr[10 * c + i] * intr[10 * c + i];
  }
  if (flags.inertial) {
    const int o = ImuOffset();
    if (mask[o]) s += g[0] * g[0] + g[1] * g[1];
    for (int i = 0; i < 6; ++i) {
      if (mask[o + 2 + i]) s += b[i] * b[i];
      if (mask[o + 8 + i]) s += sf[i] * sf[i];
    }
    if (mask[o + 14]) s += ts * ts;
  }
  return std::sqrt(s);
}

// A constant or unused block is left as it is: the rotations' Plus renormalises, which can change the last bits of a
// quaternion even with a zero step.
void Problem::Plus(const std::vector<double>& delta) {
  std::vector<double> mask;
  std::vector<uint8_t> used;
  GlobalMask(&mask);
  FramesUsed(&used);
  const int fd = FrameDim();
  double out[7];
  for (int f = 0; f < n_frames; ++f) {
    if (!used[f]) continue;
    const double* d = &delta[static_cast<size_t>(f) * fd];
    LocalParamSe3Plus(&T_wp[7 * f], d, out);
    std::memcpy(&T_wp[7 * f], out, sizeof out);
    if (fd == 9) for (int i = 0; i < 3; ++i) v_w[3 * f + i] += d[6 + i];
  }
  const double* dg = &delta[static_cast<size_t>(n_frames) * fd];
  for (int c = 0; c < n_cams; ++c) {
    const int off = CamOffset(c), K = NumIntrinsics(model[c]);
    if (mask[off]) {
      LocalParamSo3Plus(&q_ck[4 * c], dg + off, out);
      std::memcpy(&q_ck[4 * c], out, 4 * sizeof(double));
    }
    if (mask[off + 3]) for (int i = 0; i < 3; ++i) p_ck[3 * c + i] += dg[off + 3 + i];
    if (K > 0 && mask[off + 6]) for (int i = 0; i < K; ++i) intr[10 * c + i] += dg[off + 6 + i];
  }
  if (flags.inertial) {
    const int o = ImuOffset();
    const double* di = dg + o;
    if (mask[o]) { g[0] += di[0]; g[1] += di[1]; }
    for (int i = 0; i < 6; ++i) {
      if (mask[o + 2 + i]) b[i] += di[2 + i];
      if (mask[o + 8 + i]) sf[i] += di[8 + i];
    }
    if (mask[o + 14]) ts += di[14];
  }
}

// ------------------------------------------------------------------ linear algebra
namespace {
// in-place lower Cholesky of n x n row-major; returns false if not PD
bool Chol(double* A, int n) {
  for (int j = 0; j < n; ++j) {
    double d = A[j * n + j];
    for (int k = 0; k < j; ++k) d -= A[j * n + k] * A[j * n + k];
    if (!(d > 0.0)) return false;
    d = std::sqrt(d);
    A[j * n + j] = d;
    for (int i = j + 1; i < n; ++i) {
      double s = A[i * n + j];
      for (int k = 0; k < j; ++k) s -= A[i * n + k] * A[j * n + k];
      A[i * n + j] = s / d;
    }
  }
  return true;
}
// solve L L^T X = R for m right-hand sides; R is n x m row-major, overwritten
void CholSolve(const double* L, int n, double* R, int m) {
  for (int i = 0; i < n; ++i) {
    for (int k = 0; k < i; ++k) {
      const double l = L[i * n + k];
      for (int c = 0; c < m; ++c) R[i * m + c] -= l * R[k * m + c];
    }
    const double inv = 1.0 / L[i * n + i];
    for (int c = 0; c < m; ++c) R[i * m + c] *= inv;
  }
  for (int i = n - 1; i >= 0; --i) {
    for (int k = i + 1; k < n; ++k) {
      const double l = L[k * n + i];
      for (int c = 0; c < m; ++c) R[i * m + c] -= l * R[k * m + c];
    }
    const double inv = 1.0 / L[i * n + i];
    for (int c = 0; c < m; ++c) R[i * m + c] *= inv;
  }
}
}  // namespace

bool SolveArrow(const NormalEq& ne, const std::vector<double>& scale, const std::vector<double>& D2,
                std::vector<double>* delta) {
  const int nf = ne.nf, fd = ne.fd, G = ne.G, M = G + 1;
  const double* sc = &scale[static_cast<size_t>(nf) * fd];
  std::vector<double> A(static_cast<size_t>(nf) * fd * fd);   // Cholesky factors of pivots
  std::vector<double> Us(static_cast<size_t>(nf) * fd * fd);  // scaled couplings
  std::vector<double> Y(static_cast<size_t>(nf) * fd * M);    // forward-eliminated rhs [E | g]
  std::vector<double> Es(static_cast<size_t>(nf) * fd * G);
  std::vector<double> W(static_cast<size_t>(fd) * (fd + M));
  bool any_u = false;
  for (int f = 0; f < nf; ++f) {
    const double* sf_ = &scale[static_cast<size_t>(f) * fd];
    double* Af = &A[static_cast<size_t>(f) * fd * fd];
    double* Yf = &Y[static_cast<size_t>(f) * fd * M];
    double* Ef = &Es[static_cast<size_t>(f) * fd * G];
    for (int a = 0; a < fd; ++a) {
      for (int bb = 0; bb < fd; ++bb)
        Af[a * fd + bb] = ne.B[(static_cast<size_t>(f) * fd + a) * fd + bb] * sf_[a] * sf_[bb];
      Af[a * fd + a] += D2[static_cast<size_t>(f) * fd + a];
      for (int c = 0; c < G; ++c) {
        const double e = ne.E[(static_cast<size_t>(f) * fd + a) * G + c] * sf_[a] * sc[c];
        Ef[a * G + c] = e;
        Yf[a * M + c] = e;
      }
      Yf[a * M + G] = ne.gf[static_cast<size_t>(f) * fd + a] * sf_[a];
    }
    if (f > 0) {
      const double* sp = &scale[static_cast<size_t>(f - 1) * fd];
      double* Uf = &Us[static_cast<size_t>(f) * fd * fd];
      bool nz = false;
      for (int a = 0; a < fd; ++a)
        for (int bb = 0; bb < fd; ++bb) {
          const double u = ne.U[(static_cast<size_t>(f) * fd + a) * fd + bb] * sp[a] * sf_[bb];
          Uf[a * fd + bb] = u;
          nz |= (u != 0.0);
        }
      if (nz) {
        any_u = true;
        // W = A_{f-1}^{-1} [U_f | Y_{f-1}]
        const double* Lp = &A[static_cast<size_t>(f - 1) * fd * fd];
        const double* Yp = &Y[static_cast<size_t>(f - 1) * fd * M];
        const int WM = fd + M;
        for (int a = 0; a < fd; ++a) {
          for (int bb = 0; bb < fd; ++bb) W[a * WM + bb] = Uf[a * fd + bb];
          for (int c = 0; c < M; ++c) W[a * WM + fd + c] = Yp[a * M + c];
        }
        CholSolve(Lp, fd, W.data(), WM);
        // A_f -= U^T W[:, :fd];  Y_f -= U^T W[:, fd:]
        for (int a = 0; a < fd; ++a)
          for (int k = 0; k < fd; ++k) {
            const double u = Uf[k * fd + a];
            if (u == 0.0) continue;
            for (int bb = 0; bb < fd; ++bb) Af[a * fd + bb] -= u * W[k * WM + bb];
            for (int c = 0; c < M; ++c) Yf[a * M + c] -= u * W[k * WM + fd + c];
          }
      }
    }
    if (!Chol(Af, fd)) return false;
  }
  // back substitution: X_f = A_f^{-1} (Y_f - U_{f+1} X_{f+1}); stored in Y
  for (int f = nf - 1; f >= 0; --f) {
    double* Yf = &Y[static_cast<size_t>(f) * fd * M];
    if (any_u && f + 1 < nf) {
      const double* Un = &Us[static_cast<size_t>(f + 1) * fd * fd];
      const double* Xn = &Y[static_cast<size_t>(f + 1) * fd * M];
      for (int a = 0; a < fd; ++a)
        for (int k = 0; k < fd; ++k) {
          const double u = Un[a * fd + k];
          if (u == 0.0) continue;
          for (int c = 0; c < M; ++c) Yf[a * M + c] -= u * Xn[k * M + c];
        }
    }
    CholSolve(&A[static_cast<size_t>(f) * fd * fd], fd, Yf, M);
  }
  // Schur complement onto the globals
  std::vector<double> S(static_cast<size_t>(G) * G), rhs(G);
  for (int a = 0; a < G; ++a) {
    for (int bb = 0; bb < G; ++bb) S[a * G + bb] = ne.C[a * G + bb] * sc[a] * sc[bb];
    S[a * G + a] += D2[static_cast<size_t>(nf) * fd + a];
    rhs[a] = -ne.gc[a] * sc[a];
  }
  for (int f = 0; f < nf; ++f) {
    const double* Ef = &Es[static_cast<size_t>(f) * fd * G];
    const double* Xf = &Y[static_cast<size_t>(f) * fd * M];
    for (int k = 0; k < fd; ++k)
      for (int a = 0; a < G; ++a) {
        const double e = Ef[k * G + a];
        if (e == 0.0) continue;
        for (int bb = 0; bb < G; ++bb) S[a * G + bb] -= e * Xf[k * M + bb];
        rhs[a] += e * Xf[k * M + G];
      }
  }
  delta->assign(static_cast<size_t>(nf) * fd + G, 0.0);
  double* dc = &(*delta)[static_cast<size_t>(nf) * fd];
  if (G > 0) {
    if (!Chol(S.data(), G)) return false;
    CholSolve(S.data(), G, rhs.data(), 1);
    for (int a = 0; a < G; ++a) dc[a] = rhs[a];
  }
  for (int f = 0; f < nf; ++f) {
    const double* Xf = &Y[static_cast<size_t>(f) * fd * M];
    for (int a = 0; a < fd; ++a) {
      double s = -Xf[a * M + G];
      for (int c = 0; c < G; ++c) s -= Xf[a * M + c] * dc[c];
      (*delta)[static_cast<size_t>(f) * fd + a] = s;
    }
  }
  return true;
}

void ArrowMatVec(const NormalEq& ne, const std::vector<double>& scale, const std::vector<double>& x,
                 std::vector<double>* y) {
  const int nf = ne.nf, fd = ne.fd, G = ne.G;
  const size_t n = static_cast<size_t>(nf) * fd + G;
  std::vector<double> xs(n);
  for (size_t i = 0; i < n; ++i) xs[i] = x[i] * scale[i];
  y->assign(n, 0.0);
  const double* xc = &xs[static_cast<size_t>(nf) * fd];
  double* yc = &(*y)[static_cast<size_t>(nf) * fd];
  for (int f = 0; f < nf; ++f) {
    const double* xf = &xs[static_cast<size_t>(f) * fd];
    double* yf = &(*y)[static_cast<size_t>(f) * fd];
    for (int a = 0; a < fd; ++a) {
      double s = 0;
      for (int bb = 0; bb < fd; ++bb) s += ne.B[(static_cast<size_t>(f) * fd + a) * fd + bb] * xf[bb];
      for (int c = 0; c < G; ++c) {
        const double e = ne.E[(static_cast<size_t>(f) * fd + a) * G + c];
        s += e * xc[c];
        yc[c] += e * xf[a];
      }
      yf[a] += s;
    }
    if (f > 0) {
      const double* xp = &xs[static_cast<size_t>(f - 1) * fd];
      double* yp = &(*y)[static_cast<size_t>(f - 1) * fd];
      for (int a = 0; a < fd; ++a)
        for (int bb = 0; bb < fd; ++bb) {
          const double u = ne.U[(static_cast<size_t>(f) * fd + a) * fd + bb];
          yp[a] += u * xf[bb];
          yf[bb] += u * xp[a];
        }
    }
  }
  for (int a = 0; a < G; ++a) {
    double s = 0;
    for (int bb = 0; bb < G; ++bb) s += ne.C[a * G + bb] * xc[bb];
    yc[a] += s;
  }
  for (size_t i = 0; i < n; ++i) (*y)[i] *= scale[i];
}

void ArrowDiagonal(const NormalEq& ne, std::vector<double>* diag) {
  const int nf = ne.nf, fd = ne.fd, G = ne.G;
  diag->assign(static_cast<size_t>(nf) * fd + G, 0.0);
  for (int f = 0; f < nf; ++f)
    for (int a = 0; a < fd; ++a)
      (*diag)[static_cast<size_t>(f) * fd + a] = ne.B[(static_cast<size_t>(f) * fd + a) * fd + a];
  for (int a = 0; a < G; ++a) (*diag)[static_cast<size_t>(nf) * fd + a] = ne.C[a * G + a];
}
void ArrowGradient(const NormalEq& ne, std::vector<double>* grad) {
  grad->assign(ne.gf.begin(), ne.gf.end());
  grad->insert(grad->end(), ne.gc.begin(), ne.gc.end());
}
void ArrowToDense(const NormalEq& ne, std::vector<double>* H, std::vector<double>* grad) {
  const int nf = ne.nf, fd = ne.fd, G = ne.G;
  const size_t n = static_cast<size_t>(nf) * fd + G;
  H->assign(n * n, 0.0);
  for (int f = 0; f < nf; ++f) {
    const size_t o = static_cast<size_t>(f) * fd;
    for (int a = 0; a < fd; ++a) {
      for (int bb = 0; bb < fd; ++bb) {
        (*H)[(o + a) * n + o + bb] = ne.B[(o + a) * fd + bb];
        if (f > 0) {
          const double u = ne.U[(o + a) * fd + bb];
          (*H)[(o - fd + a) * n + o + bb] = u;
          (*H)[(o + bb) * n + o - fd + a] = u;
        }
      }
      for (int c = 0; c < G; ++c) {
        const double e = ne.E[(o + a) * G + c];
        (*H)[(o + a) * n + nf * fd + c] = e;
        (*H)[(static_cast<size_t>(nf) * fd + c) * n + o + a] = e;
      }
    }
  }
  for (int a = 0; a < G; ++a)
    for (int bb = 0; bb < G; ++bb)
      (*H)[(static_cast<size_t>(nf) * fd + a) * n + nf * fd + bb] = ne.C[a * G + bb];
  ArrowGradient(ne, grad);
}

// ------------------------------------------------------------------ trust-region loop
Summary Problem::Solve() {
  Summary sum;
  sum.num_residuals = NumResiduals();
  const int fd = FrameDim(), G = NumGlobals();
  const size_t n = static_cast<size_t>(n_frames) * fd + G;
  if (opts.update_imu_weights) UpdateImuWeights();  // vicalibrator.h:955

  NormalEq ne;
  double cost = Evaluate(&ne);
  sum.initial_cost = cost;
  std::vector<double> grad, diag, scale(n, 1.0), D2(n), step, Hs, delta(n);
  ArrowGradient(ne, &grad);
  if (opts.jacobi_scaling) {
    ArrowDiagonal(ne, &diag);
    for (size_t i = 0; i < n; ++i) scale[i] = 1.0 / (1.0 + std::sqrt(diag[i]));
  }
  auto norms = [&](double* gmax, double* gnorm) {
    double m = 0, s = 0;
    for (double v : grad) { m = std::max(m, std::fabs(v)); s += v * v; }
    *gmax = m; *gnorm = std::sqrt(s);
  };
  double gmax, gnorm;
  norms(&gmax, &gnorm);
  double x_norm = StateNorm();
  double radius = opts.init_radius, decrease_factor = 2.0;
  bool reuse_diagonal = false;
  // dogleg state
  double mu = 1e-8, dogleg_step_norm = 0, alpha = 0;
  bool dl_reuse = false;
  std::vector<double> dl_diag(n), dl_grad(n), dl_gn(n);

  sum.rows.push_back({0, cost, 0, gmax, gnorm, 0, 0, radius, 1});
  if (gmax <= opts.gradient_tol) { sum.termination = 2; sum.final_cost = cost; return sum; }
  auto callback = [&](double gn) {  // vicalibrator.h:690-721
    if (opts.update_imu_weights) UpdateImuWeights();
    return gn > 0 && gn < opts.callback_gnorm_stop;
  };
  if (callback(gnorm)) { sum.termination = 4; sum.final_cost = cost; return sum; }

  std::vector<double> scaled_diag(n), gs(n);
  for (int it = 1;; ++it) {
    if (it > opts.max_iters) { sum.termination = 0; break; }
    if (radius < opts.min_radius) { sum.termination = 5; break; }
    sum.iterations = it;
    bool ok = true;
    double model_change = 0;
    for (size_t i = 0; i < n; ++i) gs[i] = grad[i] * scale[i];
    if (opts.strategy == 0) {
      // LevenbergMarquardtStrategy::ComputeStep
      if (!reuse_diagonal) {
        ArrowDiagonal(ne, &diag);
        for (size_t i = 0; i < n; ++i)
          scaled_diag[i] = std::min(std::max(diag[i] * scale[i] * scale[i], 1e-6), 1e32);
      }
      for (size_t i = 0; i < n; ++i) D2[i] = scaled_diag[i] / radius;
      ok = SolveArrow(ne, scale, D2, &step);
      reuse_diagonal = true;
    } else {
      // DoglegStrategy (TRADITIONAL_DOGLEG)
      if (!dl_reuse) {
        dl_reuse = true;
        ArrowDiagonal(ne, &diag);
        for (size_t i = 0; i < n; ++i)
          dl_diag[i] = std::sqrt(std::min(std::max(diag[i] * scale[i] * scale[i], 1e-6), 1e32));
        for (size_t i = 0; i < n; ++i) dl_grad[i] = gs[i] / dl_diag[i];
        // Cauchy point: alpha = |g|^2 / |J D^-2 g... |^2 with implicit scaling
        std::vector<double> sg(n), Hv;
        double g2 = 0;
        for (size_t i = 0; i < n; ++i) { sg[i] = dl_grad[i] / dl_diag[i]; g2 += dl_grad[i] * dl_grad[i]; }
        ArrowMatVec(ne, scale, sg, &Hv);
        double jg2 = 0;
        for (size_t i = 0; i < n; ++i) jg2 += sg[i] * Hv[i];
        alpha = g2 / jg2;
        // Gauss-Newton step, regularised by mu
        for (;;) {
          for (size_t i = 0; i < n; ++i) D2[i] = dl_diag[i] * dl_diag[i] * mu;
          ok = SolveArrow(ne, scale, D2, &step);
          if (ok) break;
          mu *= 10.0;
          if (mu > 1.0) break;
        }
        if (ok) for (size_t i = 0; i < n; ++i) dl_gn[i] = step[i] * dl_diag[i];
      }
      if (ok) {
        step.assign(n, 0.0);
        double gn_norm = 0, grad_norm = 0;
        for (size_t i = 0; i < n; ++i) { gn_norm += dl_gn[i] * dl_gn[i]; grad_norm += dl_grad[i] * dl_grad[i]; }
        gn_norm = std::sqrt(gn_norm); grad_norm = std::sqrt(grad_norm);
        if (gn_norm <= radius) {
          step = dl_gn; dogleg_step_norm = gn_norm;
        } else if (grad_norm * alpha >= radius) {
          for (size_t i = 0; i < n; ++i) step[i] = -(radius / grad_norm) * dl_grad[i];
          dogleg_step_norm = radius;
        } else {
          double b_dot_a = 0;
          for (size_t i = 0; i < n; ++i) b_dot_a += dl_grad[i] * dl_gn[i];
          b_dot_a *= -alpha;
          const double a_sq = std::pow(alpha * grad_norm, 2.0);
          const double bma_sq = a_sq - 2 * b_dot_a + gn_norm * gn_norm;
          const double c = b_dot_a - a_sq;
          const double d = std::sqrt(c * c + bma_sq * (radius * radius - a_sq));
          const double beta = (c <= 0) ? (d - c) / bma_sq : (radius * radius - a_sq) / (d + c);
          double s2 = 0;
          for (size_t i = 0; i < n; ++i) {
            step[i] = (-alpha * (1.0 - beta)) * dl_grad[i] + beta * dl_gn[i];
            s2 += step[i] * step[i];
          }
          dogleg_step_norm = std::sqrt(s2);
        }
        for (size_t i = 0; i < n; ++i) step[i] /= dl_diag[i];
      }
    }
    if (ok) {
      // model_cost_change = -(J step).(r + J step / 2) = -step.g - step.H.step / 2
      ArrowMatVec(ne, scale, step, &Hs);
      double sg = 0, sHs = 0;
      for (size_t i = 0; i < n; ++i) { sg += step[i] * gs[i]; sHs += step[i] * Hs[i]; }
      model_change = -sg - 0.5 * sHs;
    }
    if (!ok || !(model_change > 0.0)) {
      // invalid step
      if (opts.strategy == 0) { radius /= decrease_factor; decrease_factor *= 2.0; reuse_diagonal = true; }
      else { mu *= 10.0; dl_reuse = false; }
      sum.rows.push_back({it, cost, 0, gmax, 0, 0, 0, radius, 0});
      if (callback(0.0)) { sum.termination = 4; break; }
      continue;
    }
    for (size_t i = 0; i < n; ++i) delta[i] = step[i] * scale[i];
    const State saved = Save();
    Plus(delta);
    const double cand = Evaluate(nullptr);
    // step norm in ambient coordinates
    double sn = 0;
    {
      const State& o = saved;
      for (size_t i = 0; i < T_wp.size(); ++i) sn += (T_wp[i] - o.T_wp[i]) * (T_wp[i] - o.T_wp[i]);
      for (size_t i = 0; i < v_w.size(); ++i) sn += (v_w[i] - o.v_w[i]) * (v_w[i] - o.v_w[i]);
      for (size_t i = 0; i < q_ck.size(); ++i) sn += (q_ck[i] - o.q_ck[i]) * (q_ck[i] - o.q_ck[i]);
      for (size_t i = 0; i < p_ck.size(); ++i) sn += (p_ck[i] - o.p_ck[i]) * (p_ck[i] - o.p_ck[i]);
      for (size_t i = 0; i < intr.size(); ++i) sn += (intr[i] - o.intr[i]) * (intr[i] - o.intr[i]);
      sn += (g[0] - o.g[0]) * (g[0] - o.g[0]) + (g[1] - o.g[1]) * (g[1] - o.g[1]) + (ts - o.ts) * (ts - o.ts);
      for (int i = 0; i < 6; ++i) sn += (b[i] - o.b[i]) * (b[i] - o.b[i]) + (sf[i] - o.sf[i]) * (sf[i] - o.sf[i]);
      sn = std::sqrt(sn);
    }
    const double cost_change = cost - cand;
    if (sn <= opts.param_tol * (x_norm + opts.param_tol)) {
      Restore(saved);
      sum.rows.push_back({it, cost, cost_change, gmax, 0, sn, 0, radius, 0});
      sum.termination = 3;
      break;
    }
    if (std::fabs(cost_change) <= opts.function_tol * cost) {
      Restore(saved);
      sum.rows.push_back({it, cost, cost_change, gmax, 0, sn, 0, radius, 0});
      sum.termination = 1;
      break;
    }
    const double rho = cost_change / model_change;
    double cb_gnorm = 0;
    if (rho > opts.min_rel_decrease) {
      cost = Evaluate(&ne);  // Jacobian at the accepted point (weights as currently set)
      x_norm = StateNorm();
      ArrowGradient(ne, &grad);
      norms(&gmax, &gnorm);
      cb_gnorm = gnorm;
      ++sum.successful_steps;
      if (opts.strategy == 0) {
        radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * rho - 1.0, 3));
        radius = std::min(opts.max_radius, radius);
        decrease_factor = 2.0;
        reuse_diagonal = false;
      } else {
        if (rho < 0.25) radius *= 0.5;
        if (rho > 0.75) radius = std::max(radius, 3.0 * dogleg_step_norm);
        mu = std::max(1e-8, 2.0 * mu / 10.0);
        dl_reuse = false;
      }
      sum.rows.push_back({it, cost, cost_change, gmax, gnorm, sn, rho, radius, 1});
      if (gmax <= opts.gradient_tol) { sum.termination = 2; callback(cb_gnorm); break; }
    } else {
      Restore(saved);
      if (opts.strategy == 0) { radius /= decrease_factor; decrease_factor *= 2.0; reuse_diagonal = true; }
      else { radius *= 0.5; dl_reuse = true; }
      sum.rows.push_back({it, cost, cost_change, gmax, 0, sn, rho, radius, 0});
    }
    if (callback(cb_gnorm)) { sum.termination = 4; break; }
  }
  sum.final_cost = cost;
  return sum;
}

}  // namespace vo
