// TEST INFRASTRUCTURE ONLY — never loaded by the abr_control_b200 package.
// ctrlsim.cpp plus the derivatives of the Joint closed loop: joint_vjp_kernel's recursion with the per-lane function
// joint_vjp_lane (abrb_grad.cuh) run on the host one direction after another, and forward-mode dual rollouts of one
// seeded direction, either through ctrl_rollout_step itself or through the phased step the kernel uses.
#include "ctrlsim.cpp"

#include "../../abr_control_b200/csrc/abrb_grad.cuh"

namespace {

struct JointIo {
  double kp, kv;
  int gravity;
  const double *q0, *dq0, *path, *pv;
  int ps, pvs, steps;
  double dt, effort;
  int64_t B;
};

struct JointCot {
  const double *q_traj, *dq_traj;
  const double *g_cost, *g_q, *g_dq, *g_q_traj, *g_dq_traj, *g_u_traj, *g_x_traj;
  double *g_path, *g_pv, *g_gains, *gq0, *gdq0;
};

template <int N>
const double *jrow(const double *a, int stride, int t, int64_t B, int64_t b) {
  return torque_row<double, N>(a, stride, t, B, b);
}

// joint_vjp_kernel's recursion with the warp's lanes as a loop over j (lanes whose output is not wanted are skipped)
template <typename T, int N, bool ORTHO>
void joint_vjp_loop(const ChainHost &h, int frame, const double *xoff, const JointIo &io, const JointCot &c) {
  ChainK<Dual<T>, N> P;
  fill_chain<Dual<T>, N>(h, P);
  const Dual<T> xo[3] = {Dual<T>(xoff ? xoff[0] : 0.0), Dual<T>(xoff ? xoff[1] : 0.0), Dual<T>(xoff ? xoff[2] : 0.0)};
  for (int64_t b = 0; b < io.B; ++b) {
    T mu[2 * N], val[4 * N + 2], gain[2] = {T(0), T(0)};
    for (int k = 0; k < N; ++k) {
      mu[k] = c.g_q ? T(c.g_q[b * N + k]) : T(0);
      mu[N + k] = c.g_dq ? T(c.g_dq[b * N + k]) : T(0);
    }
    const T gc = c.g_cost ? T(c.g_cost[b]) : T(0);
    for (int t = io.steps - 1; t >= 0; --t) {
      const int64_t row = (int64_t)t * io.B + b;
      for (int k = 0; k < N; ++k) {
        if (c.g_q_traj) mu[k] += T(c.g_q_traj[row * N + k]);
        if (c.g_dq_traj) mu[N + k] += T(c.g_dq_traj[row * N + k]);
      }
      const double *qs = t > 0 ? c.q_traj + (row - io.B) * N : io.q0 + b * N;
      const double *dqs = t > 0 ? c.dq_traj + (row - io.B) * N : io.dq0 + b * N;
      const double *pt = jrow<N>(io.path, io.ps, t, io.B, b);
      const double *vt = io.pv ? jrow<N>(io.pv, io.pvs, t, io.B, b) : nullptr;
      T q[N], dq[N], pr[N], vr[N], gx[3], gu[N];
      for (int k = 0; k < N; ++k) {
        q[k] = T(qs[k]);
        dq[k] = T(dqs[k]);
        pr[k] = T(pt[k]);
        vr[k] = vt ? T(vt[k]) : T(0);
        if (c.g_u_traj) gu[k] = T(c.g_u_traj[row * N + k]);
      }
      for (int i = 0; i < 3; ++i)
        if (c.g_x_traj) gx[i] = T(c.g_x_traj[row * 3 + i]);
      for (int j = 0; j < 4 * N + 2; ++j) {
        const bool work = j < 2 * N || (j < 3 * N && c.g_path) || (j >= 3 * N && j < 4 * N && c.g_pv) ||
                          (j >= 4 * N && c.g_gains);
        if (!work) continue;
        Kin<Dual<T>, N, ORTHO> K;
        val[j] = joint_vjp_lane<T, N>(P, T(io.kp), T(io.kv), io.gravity != 0, frame, xo, j, q, dq, pr,
                                      vt ? vr : nullptr, T(io.dt), T(io.effort), mu, gc, c.g_x_traj ? gx : nullptr,
                                      c.g_u_traj ? gu : nullptr, K);
      }
      for (int k = 0; k < N; ++k) {
        if (c.g_path) c.g_path[row * N + k] = double(val[2 * N + k]);
        if (c.g_pv) c.g_pv[row * N + k] = double(val[3 * N + k]);
      }
      if (c.g_gains) {
        gain[0] += val[4 * N];
        gain[1] += val[4 * N + 1];
      }
      for (int k = 0; k < 2 * N; ++k) mu[k] = val[k];
    }
    for (int k = 0; k < N; ++k) {
      c.gq0[b * N + k] = double(mu[k]);
      c.gdq0[b * N + k] = double(mu[N + k]);
    }
    if (c.g_gains) {
      c.g_gains[b * 2] = double(gain[0]);
      c.g_gains[b * 2 + 1] = double(gain[1]);
    }
  }
}

struct JointJvp {
  const double *a, *bt, *tp, *tv;  // tangents of q0, dq0 (B, n) and of the path, path velocity (laid out as they are)
  double tkp, tkv;                 // tangents of the gains
  double *q, *dq, *u, *x, *cost;   // values of the records (as the forward rollout's) and of the cost
  double *t_q, *t_dq, *t_u, *t_x, *t_cost, *t_qf, *t_dqf;
};

// forward-mode dual rollout along one direction of (q0, dq0, path, path velocity, kp, kv): through ctrl_rollout_step
// itself (phased = 0) or through joint_step_phased, the step joint_vjp_lane runs (phased = 1)
template <typename T, int N, bool ORTHO>
void joint_jvp_loop(const ChainHost &h, int frame, const double *xoff, int phased, const JointIo &io,
                    const JointJvp &o) {
  typedef Dual<T> D;
  ChainK<D, N> P;
  fill_chain<D, N>(h, P);
  const D xo[3] = {D(xoff ? xoff[0] : 0.0), D(xoff ? xoff[1] : 0.0), D(xoff ? xoff[2] : 0.0)};
  CtrlK<D> G;
  G.kp = D(T(io.kp), T(o.tkp));
  G.kv = D(T(io.kv), T(o.tkv));
  G.kd = G.lamb = D(0);
  G.gravity = io.gravity;
  G.cartesian = 0;
  for (int64_t b = 0; b < io.B; ++b) {
    D q[N], dq[N], pr[N], vr[N], u[N], x[3];
    D cost = D(0);
    for (int k = 0; k < N; ++k) {
      q[k] = D(T(io.q0[b * N + k]), T(o.a[b * N + k]));
      dq[k] = D(T(io.dq0[b * N + k]), T(o.bt[b * N + k]));
    }
    for (int t = 0; t < io.steps; ++t) {
      const double *pt = jrow<N>(io.path, io.ps, t, io.B, b), *tpt = jrow<N>(o.tp, io.ps, t, io.B, b);
      for (int k = 0; k < N; ++k) pr[k] = D(T(pt[k]), T(tpt[k]));
      if (io.pv) {
        const double *vt = jrow<N>(io.pv, io.pvs, t, io.B, b), *tvt = jrow<N>(o.tv, io.pvs, t, io.B, b);
        for (int k = 0; k < N; ++k) vr[k] = D(T(vt[k]), T(tvt[k]));
      }
      Kin<D, N, ORTHO> K;
      if (phased)
        joint_step_phased<D, N>(P, G.kp, G.kv, io.gravity != 0, frame, xo, q, dq, pr, io.pv ? vr : nullptr,
                                D(T(io.dt)), D(T(io.effort)), u, x, cost, K);
      else
        ctrl_rollout_step<D, N, kCtrlJoint>(P, G, frame, xo, q, dq, pr, io.pv ? vr : nullptr, (const D *)nullptr,
                                            D(T(io.dt)), D(T(io.effort)), u, x, cost, K);
      const int64_t row = (int64_t)t * io.B + b;
      for (int k = 0; k < N; ++k) {
        o.q[row * N + k] = double(q[k].v);
        o.dq[row * N + k] = double(dq[k].v);
        o.u[row * N + k] = double(u[k].v);
        o.t_q[row * N + k] = double(q[k].d);
        o.t_dq[row * N + k] = double(dq[k].d);
        o.t_u[row * N + k] = double(u[k].d);
      }
      for (int i = 0; i < 3; ++i) {
        o.x[row * 3 + i] = double(x[i].v);
        o.t_x[row * 3 + i] = double(x[i].d);
      }
    }
    for (int k = 0; k < N; ++k) {
      o.t_qf[b * N + k] = double(q[k].d);
      o.t_dqf[b * N + k] = double(dq[k].d);
    }
    o.cost[b] = double(cost.v);
    o.t_cost[b] = double(cost.d);
  }
}

}  // namespace

extern "C" {

// the arguments of abrb_joint_rollout_path_vjp_* (host arrays; strides 0 or n; g_path, g_path_velocity, g_gains and
// every cotangent NULL or given)
int jg_rollout_vjp(const abrb_chain_desc *d, int f32, double kp, double kv, int gravity, int frame, const double *xoff,
                   const double *q0, const double *dq0, const double *path, int ps, const double *pv, int pvs,
                   int steps, double dt, double effort, const double *q_traj, const double *dq_traj,
                   const double *g_cost, const double *g_q, const double *g_dq, const double *g_q_traj,
                   const double *g_dq_traj, const double *g_u_traj, const double *g_x_traj, double *g_path,
                   double *g_pv, double *g_gains, double *gq0, double *gdq0, int64_t B) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const JointIo io{kp, kv, gravity, q0, dq0, path, pv, ps, pvs, steps, dt, effort, B};
  const JointCot c{q_traj, dq_traj, g_cost, g_q, g_dq, g_q_traj, g_dq_traj, g_u_traj, g_x_traj,
                   g_path, g_pv, g_gains, gq0, gdq0};
  const bool ortho = h.ortho;
  DISPATCH_N(joint_vjp_loop, h, frame, xoff, io, c);
  return 0;
}

// a dual rollout along (a, bt, tp, tv, tkp, tkv); values and tangents of the records (steps, B, .), the cost (B) and
// the tangents of the final state (B, n)
int jg_rollout_jvp(const abrb_chain_desc *d, int f32, int phased, double kp, double kv, int gravity, int frame,
                   const double *xoff, const double *q0, const double *dq0, const double *path, int ps,
                   const double *pv, int pvs, int steps, double dt, double effort, const double *a, const double *bt,
                   const double *tp, const double *tv, double tkp, double tkv, double *q, double *dq, double *u,
                   double *x, double *cost, double *t_q, double *t_dq, double *t_u, double *t_x, double *t_cost,
                   double *t_qf, double *t_dqf, int64_t B) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const JointIo io{kp, kv, gravity, q0, dq0, path, pv, ps, pvs, steps, dt, effort, B};
  const JointJvp o{a, bt, tp, tv, tkp, tkv, q, dq, u, x, cost, t_q, t_dq, t_u, t_x, t_cost, t_qf, t_dqf};
  const bool ortho = h.ortho;
  DISPATCH_N(joint_jvp_loop, h, frame, xoff, phased, io, o);
  return 0;
}
}
