// TEST INFRASTRUCTURE ONLY — never loaded by the abr_control_b200 package.
// hostsim.cpp plus the plant: runs plant_step (abrb_rbd.cuh), the per-step body of plant_kernel, with the torque rows
// addressed as the kernel addresses them and the path rows by the kernel's own path_row, and the single-state forward
// and inverse dynamics of dyn_kernel, so that `pytest -m "not gpu"` checks them against the oracle.
#include "hostsim.cpp"

namespace {

struct PlantIo {
  double *q, *dq;  // (B, n) in/out
  const double *u, *path;
  int u_stride, comp_g, path_stride, steps;
  double dt, effort;
  double *q_traj, *dq_traj, *u_traj, *x_traj, *cost;  // each may be nullptr
  int64_t B;
};

template <typename T, int N, bool ORTHO>
void plant_loop(const ChainHost &h, int frame, const double *xoff, const PlantIo &io) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  const T xo[3] = {T(xoff ? xoff[0] : 0), T(xoff ? xoff[1] : 0), T(xoff ? xoff[2] : 0)};
  for (int64_t b = 0; b < io.B; ++b) {
    T q[N], dq[N], ur[N], tau[N], x[3], pr[6];
    T cost = T(0);
    for (int k = 0; k < N; ++k) {
      q[k] = T(io.q[b * N + k]);
      dq[k] = T(io.dq[b * N + k]);
    }
    for (int t = 0; t < io.steps; ++t) {
      const double *ut = torque_row<double, N>(io.u, io.u_stride, t, io.B, b);
      for (int k = 0; k < N; ++k) ur[k] = T(ut[k]);
      if (io.path) {
        const double *pt = path_row(io.path, io.path_stride, t, io.B, b);
        for (int c = 0; c < 6; ++c) pr[c] = T(pt[c]);
      }
      Kin<T, N, ORTHO> K;
      plant_step<T, N>(P, frame, xo, q, dq, ur, io.comp_g != 0, io.path ? pr : nullptr, T(io.dt), T(io.effort), tau,
                       x, cost, K);
      const int64_t row = (int64_t)t * io.B + b;
      for (int k = 0; k < N; ++k) {
        if (io.q_traj) io.q_traj[row * N + k] = double(q[k]);
        if (io.dq_traj) io.dq_traj[row * N + k] = double(dq[k]);
        if (io.u_traj) io.u_traj[row * N + k] = double(tau[k]);
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
void dyn_loop(const ChainHost &h, int kind, const double *q, const double *dq, const double *in, int64_t B,
              double *out) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  for (int64_t b = 0; b < B; ++b) {
    T qq[N], dd[N], ii[N], oo[N];
    for (int k = 0; k < N; ++k) {
      qq[k] = T(q[b * N + k]);
      dd[k] = T(dq[b * N + k]);
      ii[k] = T(in[b * N + k]);
    }
    Kin<T, N, ORTHO> K;
    if (kind == 0)
      forward_dynamics_state<T, N>(P, qq, dd, ii, oo, K);
    else
      inverse_dynamics_state<T, N>(P, qq, dd, ii, oo, K);
    for (int k = 0; k < N; ++k) out[b * N + k] = double(oo[k]);
  }
}

}  // namespace

extern "C" {

// u_stride is n (per trajectory) or 0 (shared), path_stride 6 or 0, path may be nullptr; records as the kernel's
int pl_rollout(const abrb_chain_desc *d, int f32, int frame, const double *xoff, double *q, double *dq,
               const double *u, int u_stride, int comp_g, const double *path, int path_stride, int steps, double dt,
               double effort, double *q_traj, double *dq_traj, double *u_traj, double *x_traj, double *cost,
               int64_t B) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const PlantIo io{q, dq, u, path, u_stride, comp_g, path_stride, steps, dt, effort, q_traj, dq_traj, u_traj, x_traj,
                   cost, B};
  const bool ortho = h.ortho;
  DISPATCH_N(plant_loop, h, frame, xoff, io);
  return 0;
}

// kind 0: out = forward dynamics ddq of in = u;  kind 1: out = inverse dynamics u of in = ddq
int pl_dynamics(const abrb_chain_desc *d, int f32, int kind, const double *q, const double *dq, const double *in,
                int64_t B, double *out) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const bool ortho = h.ortho;
  DISPATCH_N(dyn_loop, h, kind, q, dq, in, B, out);
  return 0;
}
}
