// TEST INFRASTRUCTURE ONLY — never loaded by the abr_control_b200 package.
// hostsim.cpp plus the Joint / Sliding rollouts: runs ctrl_rollout_step (abrb_osc.cuh), the per-step body of
// ctrl_rollout_kernel, with the path rows read by the kernel's own ctrl_path_rows, so that `pytest -m "not gpu"` checks
// them against the oracle.
#include "hostsim.cpp"

namespace {

struct CtrlIo {
  int kind;
  double k1, k2;  // Joint: kp, kv;  Sliding: kd, lamb
  int flag;       // Joint: account_for_gravity;  Sliding: cartesian
  double *q, *dq;  // (B, n) in/out
  const double *path, *pv, *pa;
  int ps, pvs, pas, steps;
  double dt, effort;
  double *q_traj, *dq_traj, *u_traj, *x_traj, *cost;  // each may be nullptr
  int64_t B;
};

template <typename T, int N, bool ORTHO, int KIND>
void ctrl_loop_kind(const ChainHost &h, int frame, const double *xoff, const CtrlIo &io) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  CtrlK<T> G;
  G.kp = G.kd = T(io.k1);
  G.kv = G.lamb = T(io.k2);
  G.gravity = G.cartesian = io.flag;
  constexpr int L = CtrlRow<N>::kMax;
  const T xo[3] = {T(xoff ? xoff[0] : 0), T(xoff ? xoff[1] : 0), T(xoff ? xoff[2] : 0)};
  for (int64_t b = 0; b < io.B; ++b) {
    T q[N], dq[N], tg[L], tv[L], ta[L], u[N], x[3];
    double tgd[L], tvd[L], tad[L];
    T cost = T(0);
    for (int k = 0; k < N; ++k) {
      q[k] = T(io.q[b * N + k]);
      dq[k] = T(io.dq[b * N + k]);
    }
    for (int t = 0; t < io.steps; ++t) {
      ctrl_path_rows<double, N, KIND>(io.path, io.ps, io.pv, io.pvs, io.pa, io.pas, io.flag != 0, t, io.B, b, tgd, tvd,
                                      tad);
      for (int k = 0; k < L; ++k) {
        tg[k] = T(tgd[k]);
        tv[k] = T(tvd[k]);
        ta[k] = T(tad[k]);
      }
      Kin<T, N, ORTHO> K;
      ctrl_rollout_step<T, N, KIND>(P, G, frame, xo, q, dq, tg, io.pv ? tv : nullptr, io.pa ? ta : nullptr, T(io.dt),
                                    T(io.effort), u, x, cost, K);
      const int64_t row = (int64_t)t * io.B + b;
      for (int k = 0; k < N; ++k) {
        if (io.q_traj) io.q_traj[row * N + k] = double(q[k]);
        if (io.dq_traj) io.dq_traj[row * N + k] = double(dq[k]);
        if (io.u_traj) io.u_traj[row * N + k] = double(u[k]);
      }
      for (int c = 0; c < 3; ++c)
        if (io.x_traj) io.x_traj[row * 3 + c] = double(x[c]);
    }
    for (int k = 0; k < N; ++k) {
      io.q[b * N + k] = double(q[k]);
      io.dq[b * N + k] = double(dq[k]);
    }
    if (io.cost) io.cost[b] = double(cost);
  }
}

template <typename T, int N, bool ORTHO>
void ctrl_rollout_loop(const ChainHost &h, int frame, const double *xoff, const CtrlIo &io) {
  if (io.kind == kCtrlJoint)
    ctrl_loop_kind<T, N, ORTHO, kCtrlJoint>(h, frame, xoff, io);
  else
    ctrl_loop_kind<T, N, ORTHO, kCtrlSliding>(h, frame, xoff, io);
}

}  // namespace

extern "C" {

// kind 0 (Joint: k1 = kp, k2 = kv, flag = account_for_gravity) or 1 (Sliding: kd, lamb, cartesian); strides 0 or the
// row width (3 for cartesian Sliding, n otherwise); pv and pa may be nullptr; records as the kernel's
int cs_rollout(const abrb_chain_desc *d, int f32, int kind, double k1, double k2, int flag, int frame,
               const double *xoff, double *q, double *dq, const double *path, int ps, const double *pv, int pvs,
               const double *pa, int pas, int steps, double dt, double effort, double *q_traj, double *dq_traj,
               double *u_traj, double *x_traj, double *cost, int64_t B) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const CtrlIo io{kind, k1, k2, flag, q, dq, path, pv, pa, ps, pvs, pas, steps, dt, effort, q_traj, dq_traj, u_traj,
                  x_traj, cost, B};
  const bool ortho = h.ortho;
  DISPATCH_N(ctrl_rollout_loop, h, frame, xoff, io);
  return 0;
}
}
