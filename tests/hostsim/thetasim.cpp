// TEST INFRASTRUCTURE ONLY — never loaded by the abr_control_b200 package.
// gradsim.cpp plus the link-inertia gradient of the plant rollout: theta_vjp_state (abrb_theta.cuh), the per-state body
// of theta_vjp_kernel, summed over each trajectory's steps in order, and a forward-mode dual rollout of the phased plant
// step whose chain carries the tangent of a direction v of theta in its inertial constants (and none in its kinematic
// ones), that the tests pair the gradient against.
#include "gradsim.cpp"

#include "../../abr_control_b200/csrc/abrb_theta.cuh"

namespace {

struct ThetaIo {
  const double *q0, *dq0, *u;
  int u_stride, comp_g, steps;
  double effort;
  const double *q_traj, *dq_traj, *gu, *g_cost, *g_u_traj;
  double *g_theta;
  int64_t B;
};

template <typename T, int N, bool ORTHO>
void theta_loop(const ChainHost &h, const double *gravity, const ThetaIo &io) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  T grav[6];
  for (int c = 0; c < 6; ++c) grav[c] = T(gravity[c]);
  for (int64_t b = 0; b < io.B; ++b) {
    T acc[6 * N];
    for (int p = 0; p < 6 * N; ++p) acc[p] = T(0);
    const T ec = io.g_cost ? T(2) * T(io.effort) * T(io.g_cost[b]) : T(0);
    for (int t = 0; t < io.steps; ++t) {
      const int64_t row = (int64_t)t * io.B + b;
      const double *qs = t > 0 ? io.q_traj + (row - io.B) * N : io.q0 + b * N;
      const double *dqs = t > 0 ? io.dq_traj + (row - io.B) * N : io.dq0 + b * N;
      const double *ut = torque_row<double, N>(io.u, io.u_stride, t, io.B, b);
      T q[N], dq[N], ur[N], gu[N], gt[N];
      for (int k = 0; k < N; ++k) {
        q[k] = T(qs[k]);
        dq[k] = T(dqs[k]);
        ur[k] = T(ut[k]);
        gu[k] = T(io.gu[row * N + k]);
        gt[k] = io.g_u_traj ? T(io.g_u_traj[row * N + k]) : T(0);
      }
      Kin<T, N, ORTHO> K;
      theta_vjp_state<T, N>(P, grav, q, dq, ur, io.comp_g != 0, gu, ec, io.g_u_traj ? gt : nullptr, acc, K);
    }
    for (int p = 0; p < 6 * N; ++p) io.g_theta[b * 6 * N + p] = double(acc[p]);
  }
}

// the chain with the tangent v (6N, theta's order) on its inertial constants, as chain_from_desc forms them
template <typename T, int N>
void fill_chain_theta_tangent(const ChainHost &h, const double *gravity, const double *v, ChainK<Dual<T>, N> &P) {
  typedef Dual<T> D;
  fill_chain<D, N>(h, P);
  for (int l = 1; l <= N; ++l)
    for (int c = 0; c < 3; ++c) {
      P.Wp[l][c] = D(T(h.Wp[l][c]), T(v[6 * (l - 1) + c]));
      P.gp[l][c] = D(T(h.gp[l][c]), T(v[6 * (l - 1) + c] * gravity[c]));
    }
  for (int k = 0; k < N; ++k)
    for (int c = 0; c < 3; ++c) {
      double s = 0, sg = 0;
      for (int l = k + 1; l <= N; ++l) {
        s += v[6 * (l - 1) + 3 + c];
        sg += v[6 * (l - 1) + 3 + c] * gravity[3 + c];
      }
      P.Wos[k][c] = D(T(h.Wos[k][c]), T(s));
      P.gos[k][c] = D(T(h.gos[k][c]), T(sg));
    }
}

struct ThetaJvpIo {
  const double *q0, *dq0, *u, *path;
  int u_stride, comp_g, path_stride, steps;
  double dt, effort;
  const double *v;                                        // (6N,) direction of theta
  double *t_q, *t_dq, *t_u, *t_x, *t_cost, *t_qf, *t_dqf;  // tangents of the records, the cost and the final state
  int64_t B;
};

template <typename T, int N, bool ORTHO>
void theta_jvp_loop(const ChainHost &h, const double *gravity, int frame, const double *xoff, const ThetaJvpIo &io) {
  typedef Dual<T> D;
  ChainK<D, N> P;
  fill_chain_theta_tangent<T, N>(h, gravity, io.v, P);
  const D xo[3] = {D(xoff ? xoff[0] : 0.0), D(xoff ? xoff[1] : 0.0), D(xoff ? xoff[2] : 0.0)};
  for (int64_t b = 0; b < io.B; ++b) {
    D q[N], dq[N], ur[N], tau[N], x[3], pr[3];
    D cost = D(0);
    for (int k = 0; k < N; ++k) {
      q[k] = D(T(io.q0[b * N + k]));
      dq[k] = D(T(io.dq0[b * N + k]));
    }
    for (int t = 0; t < io.steps; ++t) {
      const double *ut = torque_row<double, N>(io.u, io.u_stride, t, io.B, b);
      for (int k = 0; k < N; ++k) ur[k] = D(T(ut[k]));
      if (io.path) {
        const double *pt = path_row(io.path, io.path_stride, t, io.B, b);
        for (int c = 0; c < 3; ++c) pr[c] = D(T(pt[c]));
      }
      Kin<D, N, ORTHO> K;
      plant_step_phased<D, N>(P, frame, xo, q, dq, ur, io.comp_g != 0, io.path ? pr : nullptr, D(T(io.dt)),
                              D(T(io.effort)), tau, x, cost, K);
      const int64_t row = (int64_t)t * io.B + b;
      for (int k = 0; k < N; ++k) {
        io.t_q[row * N + k] = double(q[k].d);
        io.t_dq[row * N + k] = double(dq[k].d);
        io.t_u[row * N + k] = double(tau[k].d);
      }
      for (int c = 0; c < 3; ++c) io.t_x[row * 3 + c] = double(x[c].d);
    }
    for (int k = 0; k < N; ++k) {
      io.t_qf[b * N + k] = double(q[k].d);
      io.t_dqf[b * N + k] = double(dq[k].d);
    }
    io.t_cost[b] = double(cost.d);
  }
}

}  // namespace

extern "C" {

// the arguments of abrb_plant_rollout_theta_vjp_* (host arrays; g_cost and g_u_traj NULL or given)
int th_rollout_theta_vjp(const abrb_chain_desc *d, int f32, const double *q0, const double *dq0, const double *u,
                         int u_stride, int comp_g, int steps, double effort, const double *q_traj,
                         const double *dq_traj, const double *gu, const double *g_cost, const double *g_u_traj,
                         double *g_theta, int64_t B) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const ThetaIo io{q0, dq0, u, u_stride, comp_g, steps, effort, q_traj, dq_traj, gu, g_cost, g_u_traj, g_theta, B};
  const bool ortho = h.ortho;
  DISPATCH_N(theta_loop, h, d->gravity, io);
  return 0;
}

// forward-mode dual rollout along the direction v of theta (fp64: f32 must be 0)
int th_rollout_theta_jvp(const abrb_chain_desc *d, int f32, int frame, const double *xoff, const double *q0,
                         const double *dq0, const double *u, int u_stride, int comp_g, const double *path,
                         int path_stride, int steps, double dt, double effort, const double *v, double *t_q,
                         double *t_dq, double *t_u, double *t_x, double *t_cost, double *t_qf, double *t_dqf,
                         int64_t B) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const ThetaJvpIo io{q0, dq0, u, path, u_stride, comp_g, path_stride, steps, dt, effort, v,
                      t_q, t_dq, t_u, t_x, t_cost, t_qf, t_dqf, B};
  const bool ortho = h.ortho;
  DISPATCH_N(theta_jvp_loop, h, d->gravity, frame, xoff, io);
  return 0;
}
}
