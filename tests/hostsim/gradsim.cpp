// TEST INFRASTRUCTURE ONLY — never loaded by the abr_control_b200 package.
// plantsim.cpp plus the derivatives of the plant: the per-lane functions of dyn_jac_kernel and plant_vjp_kernel
// (abrb_grad.cuh) run on the host, one direction after another, and a forward-mode dual rollout of plant_step itself
// (not the phased step the kernels use) that the tests compare the adjoint against.
#include "plantsim.cpp"

#include "../../abr_control_b200/csrc/abrb_grad.cuh"

namespace {

template <typename T, int N, bool ORTHO>
void jac_loop(const ChainHost &h, int kind, const double *q, const double *dq, const double *in, int64_t B,
              double *d_q, double *d_dq, double *d_in) {
  ChainK<Dual<T>, N> P;
  fill_chain<Dual<T>, N>(h, P);
  const int ncol = d_in != nullptr ? 3 * N : 2 * N;
  for (int64_t b = 0; b < B; ++b) {
    T qq[N], dd[N], ii[N], col[N];
    for (int k = 0; k < N; ++k) {
      qq[k] = T(q[b * N + k]);
      dd[k] = T(dq[b * N + k]);
      ii[k] = T(in[b * N + k]);
    }
    for (int j = 0; j < ncol; ++j) {
      Kin<Dual<T>, N, ORTHO> K;
      dyn_jac_column<T, N>(P, kind, j, qq, dd, ii, col, K);
      double *dst = j < N ? d_q : (j < 2 * N ? d_dq : d_in);
      for (int i = 0; i < N; ++i) dst[(b * N + i) * N + j % N] = double(col[i]);
    }
  }
}

struct VjpIo {
  const double *q0, *dq0, *u, *path;
  int u_stride, comp_g, path_stride, steps;
  double dt, effort;
  const double *q_traj, *dq_traj;
  const double *g_cost, *g_q, *g_dq, *g_q_traj, *g_dq_traj, *g_u_traj, *g_x_traj;
  double *gu, *gq0, *gdq0;
  int64_t B;
};

// plant_vjp_kernel's recursion with the warp's lanes as a loop over j
template <typename T, int N, bool ORTHO>
void vjp_loop(const ChainHost &h, int frame, const double *xoff, const VjpIo &io) {
  ChainK<Dual<T>, N> P;
  fill_chain<Dual<T>, N>(h, P);
  const Dual<T> xo[3] = {Dual<T>(xoff ? xoff[0] : 0.0), Dual<T>(xoff ? xoff[1] : 0.0), Dual<T>(xoff ? xoff[2] : 0.0)};
  for (int64_t b = 0; b < io.B; ++b) {
    T mu[2 * N], val[3 * N];
    for (int k = 0; k < N; ++k) {
      mu[k] = io.g_q ? T(io.g_q[b * N + k]) : T(0);
      mu[N + k] = io.g_dq ? T(io.g_dq[b * N + k]) : T(0);
    }
    const T gc = io.g_cost ? T(io.g_cost[b]) : T(0);
    for (int t = io.steps - 1; t >= 0; --t) {
      const int64_t row = (int64_t)t * io.B + b;
      for (int k = 0; k < N; ++k) {
        if (io.g_q_traj) mu[k] += T(io.g_q_traj[row * N + k]);
        if (io.g_dq_traj) mu[N + k] += T(io.g_dq_traj[row * N + k]);
      }
      const double *qs = t > 0 ? io.q_traj + (row - io.B) * N : io.q0 + b * N;
      const double *dqs = t > 0 ? io.dq_traj + (row - io.B) * N : io.dq0 + b * N;
      const double *ut = torque_row<double, N>(io.u, io.u_stride, t, io.B, b);
      T q[N], dq[N], ur[N], pr[3], gx[3], gt[N];
      for (int k = 0; k < N; ++k) {
        q[k] = T(qs[k]);
        dq[k] = T(dqs[k]);
        ur[k] = T(ut[k]);
        if (io.g_u_traj) gt[k] = T(io.g_u_traj[row * N + k]);
      }
      if (io.path) {
        const double *pt = path_row(io.path, io.path_stride, t, io.B, b);
        for (int c = 0; c < 3; ++c) pr[c] = T(pt[c]);
      }
      for (int c = 0; c < 3; ++c)
        if (io.g_x_traj) gx[c] = T(io.g_x_traj[row * 3 + c]);
      for (int j = 0; j < 3 * N; ++j) {
        Kin<Dual<T>, N, ORTHO> K;
        val[j] = plant_vjp_lane<T, N>(P, frame, xo, j, q, dq, ur, io.comp_g != 0, io.path ? pr : nullptr, T(io.dt),
                                      T(io.effort), mu, gc, io.g_x_traj ? gx : nullptr, io.g_u_traj ? gt : nullptr, K);
      }
      for (int k = 0; k < N; ++k) io.gu[row * N + k] = double(val[2 * N + k]);
      for (int k = 0; k < 2 * N; ++k) mu[k] = val[k];
    }
    for (int k = 0; k < N; ++k) {
      io.gq0[b * N + k] = double(mu[k]);
      io.gdq0[b * N + k] = double(mu[N + k]);
    }
  }
}

struct JvpIo {
  const double *q0, *dq0, *u, *path;
  int u_stride, comp_g, path_stride, steps;
  double dt, effort;
  const double *v, *a, *bt;  // tangents of u (laid out as u), q0 and dq0 (B, n)
  double *t_q, *t_dq, *t_u, *t_x, *t_cost, *t_qf, *t_dqf;  // tangents of the records, the cost and the final state
  int64_t B;
};

// forward-mode dual rollout of plant_step along (v, a, bt)
template <typename T, int N, bool ORTHO>
void jvp_loop(const ChainHost &h, int frame, const double *xoff, const JvpIo &io) {
  typedef Dual<T> D;
  ChainK<D, N> P;
  fill_chain<D, N>(h, P);
  const D xo[3] = {D(xoff ? xoff[0] : 0.0), D(xoff ? xoff[1] : 0.0), D(xoff ? xoff[2] : 0.0)};
  for (int64_t b = 0; b < io.B; ++b) {
    D q[N], dq[N], ur[N], tau[N], x[3], pr[3];
    D cost = D(0);
    for (int k = 0; k < N; ++k) {
      q[k] = D(T(io.q0[b * N + k]), T(io.a[b * N + k]));
      dq[k] = D(T(io.dq0[b * N + k]), T(io.bt[b * N + k]));
    }
    for (int t = 0; t < io.steps; ++t) {
      const double *ut = torque_row<double, N>(io.u, io.u_stride, t, io.B, b);
      const double *vt = torque_row<double, N>(io.v, io.u_stride, t, io.B, b);
      for (int k = 0; k < N; ++k) ur[k] = D(T(ut[k]), T(vt[k]));
      if (io.path) {
        const double *pt = path_row(io.path, io.path_stride, t, io.B, b);
        for (int c = 0; c < 3; ++c) pr[c] = D(T(pt[c]));
      }
      Kin<D, N, ORTHO> K;
      plant_step<D, N>(P, frame, xo, q, dq, ur, io.comp_g != 0, io.path ? pr : nullptr, D(T(io.dt)), D(T(io.effort)),
                       tau, x, cost, K);
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

// kind 0: derivatives of the forward dynamics (in = u), kind 1: of the inverse dynamics (in = ddq); d_in may be NULL
int gr_dyn_jac(const abrb_chain_desc *d, int f32, int kind, const double *q, const double *dq, const double *in,
               int64_t B, double *d_q, double *d_dq, double *d_in) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const bool ortho = h.ortho;
  DISPATCH_N(jac_loop, h, kind, q, dq, in, B, d_q, d_dq, d_in);
  return 0;
}

// the arguments of abrb_plant_rollout_vjp_* (host arrays, every cotangent NULL or given)
int gr_rollout_vjp(const abrb_chain_desc *d, int f32, int frame, const double *xoff, const double *q0,
                   const double *dq0, const double *u, int u_stride, int comp_g, const double *path, int path_stride,
                   int steps, double dt, double effort, const double *q_traj, const double *dq_traj,
                   const double *g_cost, const double *g_q, const double *g_dq, const double *g_q_traj,
                   const double *g_dq_traj, const double *g_u_traj, const double *g_x_traj, double *gu, double *gq0,
                   double *gdq0, int64_t B) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const VjpIo io{q0, dq0, u, path, u_stride, comp_g, path_stride, steps, dt, effort, q_traj, dq_traj, g_cost, g_q,
                 g_dq, g_q_traj, g_dq_traj, g_u_traj, g_x_traj, gu, gq0, gdq0, B};
  const bool ortho = h.ortho;
  DISPATCH_N(vjp_loop, h, frame, xoff, io);
  return 0;
}

int gr_rollout_jvp(const abrb_chain_desc *d, int f32, int frame, const double *xoff, const double *q0,
                   const double *dq0, const double *u, int u_stride, int comp_g, const double *path, int path_stride,
                   int steps, double dt, double effort, const double *v, const double *a, const double *bt,
                   double *t_q, double *t_dq, double *t_u, double *t_x, double *t_cost, double *t_qf, double *t_dqf,
                   int64_t B) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const JvpIo io{q0, dq0, u, path, u_stride, comp_g, path_stride, steps, dt, effort, v, a, bt,
                 t_q, t_dq, t_u, t_x, t_cost, t_qf, t_dqf, B};
  const bool ortho = h.ortho;
  DISPATCH_N(jvp_loop, h, frame, xoff, io);
  return 0;
}
}
