// abrb_grad.cuh — derivatives of the plant (DESIGN.md S3.6): one forward-mode dual evaluation per input direction.
//
// A lane (dyn_jac_kernel, plant_vjp_kernel, joint_vjp_kernel) or a loop iteration (tests/hostsim/gradsim.cpp,
// jointgradsim.cpp) seeds direction j of the
// inputs with a unit tangent and runs the per-state code of abrb_rbd.cuh on Dual<T>; the tangents of the outputs are
// column j of the Jacobian.  The chain constants are a ChainK<Dual<T>, N> with zero tangents.
//
// The dual evaluation runs in out-of-line phases — the walk; M, g and C dq; the factorisation and what follows — at the
// K.sync() boundaries of the real code.  Fully inlined, the general-frame dual evaluation is one body that ptxas does
// not keep in registers (tens of KB of stack per thread); in phases, each body is small enough and the arrays handed
// from one phase to the next live in the thread's stack frame.
#pragma once
#include "abrb_dual.cuh"
#include "abrb_osc.cuh"
#include "abrb_rbd.cuh"

namespace abrb {

template <typename T, int N, class K_>
ABRB_HD_NOINLINE void phase_walk(const ChainK<T, N> &P, const T *q, int frame, K_ &K) {
  K.sync();
  walk<T, N>(P, q, frame, K);
  K.sync();
}
template <typename T, int N, class K_>
ABRB_HD_NOINLINE void phase_terms(const ChainK<T, N> &P, const T *dq, T (*M)[N], T *g, T *cdq, K_ &K) {
  plant_terms<T, N>(P, dq, M, g, cdq, K);
  K.sync();
}
template <typename T, int N>
ABRB_HD_NOINLINE void phase_forward_solve(T (*M)[N], const T *g, const T *cdq, const T *u, T *ddq) {
  forward_solve<T, N>(M, g, cdq, u, ddq);
}
template <typename T, int N>
ABRB_HD_NOINLINE void phase_inverse_apply(const T (*M)[N], const T *g, const T *cdq, const T *ddq, T *u) {
  inverse_apply<T, N>(M, g, cdq, ddq, u);
}
template <typename T, int N>
ABRB_HD_NOINLINE void phase_advance(T (*M)[N], const T *g, const T *cdq, T *q, T *dq, const T *u, bool comp_g,
                                    const T *x, const T *p, T dt, T effort, T *tau, T &cost) {
  plant_advance<T, N>(M, g, cdq, q, dq, u, comp_g, x, p, dt, effort, tau, cost);
}

// plant_step in phases (the same calls in the same order)
template <typename T, int N, class K_>
ABRB_HD void plant_step_phased(const ChainK<T, N> &P, int frame, const T *xoff, T *q, T *dq, const T *u, bool comp_g,
                               const T *p, T dt, T effort, T *tau, T *x, T &cost, K_ &K) {
  phase_walk<T, N>(P, q, frame, K);
  frame_point(K.F, xoff, x);
  T M[N][N], g[N], cdq[N];
  phase_terms<T, N>(P, dq, M, g, cdq, K);
  phase_advance<T, N>(M, g, cdq, q, dq, u, comp_g, x, p, dt, effort, tau, cost);
}

template <typename T>
ABRB_HD T unit_if(bool on) {
  return on ? T(1) : T(0);
}

// Column j (< 3N) of the derivatives of one state's forward dynamics (kind 0: ddq of (q, dq, u)) or inverse dynamics
// (kind 1: u of (q, dq, ddq)): col[i] = d out_i / d in_j, with in = (q, dq, u or ddq).
template <typename T, int N, class K_>
ABRB_HD void dyn_jac_column(const ChainK<Dual<T>, N> &P, int kind, int j, const T *q, const T *dq, const T *in,
                            T *col, K_ &K) {
  typedef Dual<T> D;
  D qd[N], dqd[N], ind[N], out[N];
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    qd[k] = D(q[k], unit_if<T>(j == k));
    dqd[k] = D(dq[k], unit_if<T>(j == N + k));
    ind[k] = D(in[k], unit_if<T>(j == 2 * N + k));
  }
  phase_walk<D, N>(P, qd, 0, K);
  D M[N][N], g[N], cdq[N];
  phase_terms<D, N>(P, dqd, M, g, cdq, K);
  if (kind == 0)
    phase_forward_solve<D, N>(M, g, cdq, ind, out);
  else
    phase_inverse_apply<D, N>(M, g, cdq, ind, out);
  ABRB_UNROLL
  for (int i = 0; i < N; ++i) col[i] = out[i].d;
}

// One lane's share of the backward step t of the rollout's vector-Jacobian product (DESIGN.md S3.6).  Direction j of
// (q_t, dq_t, u_t) is pushed through one dual plant_step from the recorded state x_t = (q, dq); the result is
//     gcost dc_t/dj + gx . dx_t/dj + gtau . dtau_t/dj + mu . dx_{t+1}/dj
// that is lambda_t[j] for j < 2N and the torque cotangent gu_t[j - 2N] for j >= 2N.  mu = (mu_q, mu_dq) is the
// cotangent of x_{t+1}; gx (3) and gtau (N) may be nullptr (zero).
template <typename T, int N, class K_>
ABRB_HD T plant_vjp_lane(const ChainK<Dual<T>, N> &P, int frame, const Dual<T> *xoff, int j, const T *q, const T *dq,
                         const T *u, bool comp_g, const T *p, T dt, T effort, const T *mu, T gcost, const T *gx,
                         const T *gtau, K_ &K) {
  typedef Dual<T> D;
  D qd[N], dqd[N], ud[N], tau[N], x[3], pd[3];
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    qd[k] = D(q[k], unit_if<T>(j == k));
    dqd[k] = D(dq[k], unit_if<T>(j == N + k));
    ud[k] = D(u[k], unit_if<T>(j == 2 * N + k));
  }
  if (p != nullptr) {
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) pd[c] = D(p[c]);
  }
  D cost = D(0);
  plant_step_phased<D, N>(P, frame, xoff, qd, dqd, ud, comp_g, p != nullptr ? pd : nullptr, D(dt), D(effort), tau, x,
                          cost, K);
  T s = gcost * cost.d;
  if (gx != nullptr) {
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) s += gx[c] * x[c].d;
  }
  if (gtau != nullptr) {
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) s += gtau[k] * tau[k].d;
  }
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) s += mu[k] * qd[k].d + mu[N + k] * dqd[k].d;
  return s;
}

// ------------------------------------------------------------------------------------------------ the Joint closed loop
template <typename T, int N, class K_>
ABRB_HD_NOINLINE void phase_joint_torque(const ChainK<T, N> &P, T kp, T kv, bool gravity, const T *q, const T *dq,
                                         const T *target, const T *tv, T *u, K_ &K) {
  joint_torque<T, N>(P, kp, kv, gravity, q, dq, target, tv, u, K);
}
// The plant's tail for the Joint step: phase_advance's body in an out-of-line function of its own.  Calling
// phase_advance from a second kernel changes the register allocation ptxas gives plant_vjp_kernel around it.
template <typename T, int N>
ABRB_HD_NOINLINE void phase_joint_advance(T (*M)[N], const T *g, const T *cdq, T *q, T *dq, const T *u, const T *x,
                                          T dt, T effort, T &cost) {
  T tau[N];
  plant_advance<T, N>(M, g, cdq, q, dq, u, false, x, (const T *)nullptr, dt, effort, tau, cost);
}

// ctrl_rollout_step<KIND = kCtrlJoint> in phases (the same calls in the same order, each with its own walk: the
// controller's at the base frame, the plant's at `frame`)
template <typename T, int N, class K_>
ABRB_HD void joint_step_phased(const ChainK<T, N> &P, T kp, T kv, bool gravity, int frame, const T *xoff, T *q, T *dq,
                               const T *target, const T *tv, T dt, T effort, T *u, T *x, T &cost, K_ &K) {
  phase_walk<T, N>(P, q, 0, K);
  phase_joint_torque<T, N>(P, kp, kv, gravity, q, dq, target, tv, u, K);
  T e = T(0);
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    const T d = wrap_pm_pi(target[k] - q[k]);
    e += d * d;
  }
  phase_walk<T, N>(P, q, frame, K);
  frame_point(K.F, xoff, x);
  T M[N][N], g[N], cdq[N];
  phase_terms<T, N>(P, dq, M, g, cdq, K);
  phase_joint_advance<T, N>(M, g, cdq, q, dq, u, x, dt, effort, cost);
  cost += e;
}

// One lane's share of the backward step t of the Joint closed loop's vector-Jacobian product (DESIGN.md S3.6).  Lane j
// seeds one direction of (q_t, dq_t, p_t, v_t, kp, kv):
//     j < N: q_t;  N <= j < 2N: dq_t;  2N <= j < 3N: p_t;  3N <= j < 4N: v_t;  j = 4N: kp;  j = 4N + 1: kv
// and pushes it through one dual Joint step from the recorded state x_t = (q, dq); the result is
//     gcost dc_t/dj + gx . dx_t/dj + gu . du_t/dj + mu . dx_{t+1}/dj
// that is lambda_t[j] for j < 2N, the path (velocity) cotangent of step t for 2N <= j < 4N and step t's share of the
// gain cotangent for j >= 4N.  `v` (the path velocity row) may be nullptr (zero, and lanes 3N..4N-1 then idle); gx (3)
// and gu (N) may be nullptr (zero).
template <typename T, int N, class K_>
ABRB_HD T joint_vjp_lane(const ChainK<Dual<T>, N> &P, T kp, T kv, bool gravity, int frame, const Dual<T> *xoff, int j,
                         const T *q, const T *dq, const T *p, const T *v, T dt, T effort, const T *mu, T gcost,
                         const T *gx, const T *gu, K_ &K) {
  typedef Dual<T> D;
  D qd[N], dqd[N], pd[N], vd[N], u[N], x[3];
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    qd[k] = D(q[k], unit_if<T>(j == k));
    dqd[k] = D(dq[k], unit_if<T>(j == N + k));
    pd[k] = D(p[k], unit_if<T>(j == 2 * N + k));
    vd[k] = D(v != nullptr ? v[k] : T(0), unit_if<T>(j == 3 * N + k));
  }
  D cost = D(0);
  joint_step_phased<D, N>(P, D(kp, unit_if<T>(j == 4 * N)), D(kv, unit_if<T>(j == 4 * N + 1)), gravity, frame, xoff, qd,
                          dqd, pd, v != nullptr ? vd : nullptr, D(dt), D(effort), u, x, cost, K);
  T s = gcost * cost.d;
  if (gx != nullptr) {
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) s += gx[c] * x[c].d;
  }
  if (gu != nullptr) {
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) s += gu[k] * u[k].d;
  }
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) s += mu[k] * qd[k].d + mu[N + k] * dqd[k].d;
  return s;
}

}  // namespace abrb
