// TEST INFRASTRUCTURE ONLY — never loaded by the abr_control_b200 package.
// hostsim.cpp plus the path-following rollout: runs rollout_step (abrb_osc.cuh), the per-step body of rollout_kernel,
// with the path rows addressed by the kernel's own path_row, and with the instantiation the
// kernel picks for a call (rollout_path_go, kernels.cu: plain iff osc_plain with the path velocity as the target
// velocity) or the general one on request, so that `pytest -m "not gpu"` checks the step against the oracle.
#include "hostsim.cpp"

namespace {

struct PathIo {
  double *q, *dq;  // (B, n) in/out
  const double *path, *pv;
  int path_stride, pv_stride, steps;
  double dt, effort;
  double *q_traj, *dq_traj, *u_traj, *x_traj, *cost, *ierr;  // each may be nullptr (ierr iff ki != 0)
  int64_t B;
};

template <typename T, int N, bool ORTHO, int KD, bool PLAIN>
void path_traj(const ChainK<T, N> &P, const OscK<T, N> &O, const PathIo &io, int64_t b) {
  T q[N], dq[N], tg[6], tv[6], ie[6], u[N], x[3];
  T cost = T(0);
  for (int k = 0; k < N; ++k) {
    q[k] = T(io.q[b * N + k]);
    dq[k] = T(io.dq[b * N + k]);
  }
  for (int c = 0; c < 6; ++c) ie[c] = io.ierr ? T(io.ierr[b * 6 + c]) : T(0);
  for (int t = 0; t < io.steps; ++t) {
    const double *pt = path_row(io.path, io.path_stride, t, io.B, b);
    for (int c = 0; c < 6; ++c) tg[c] = T(pt[c]);
    if (io.pv) {
      const double *vt = path_row(io.pv, io.pv_stride, t, io.B, b);
      for (int c = 0; c < 6; ++c) tv[c] = T(vt[c]);
    }
    Kin<T, N, ORTHO> K;
    SeqCoop seq;
    rollout_step<T, N, KD, PLAIN, true>(P, O, q, dq, tg, io.pv ? tv : nullptr, io.ierr ? ie : nullptr, T(io.dt),
                                        T(io.effort), u, x, cost, K, seq);
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
  for (int c = 0; c < 6; ++c)
    if (io.ierr) io.ierr[b * 6 + c] = double(ie[c]);
  if (io.cost) io.cost[b] = double(cost);
}

int g_picked_plain = -1;

template <typename T, int N, bool ORTHO>
void path_loop(const ChainHost &h, const abrb_osc_params &p, int frame, const double *xoff, const PathIo &io,
               bool allow_plain) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  OscK<T, N> O;
  fill_osc<T, N>(p, frame, xoff, O);
  const bool kd6 = (O.dof_mask & 56u) != 0;
  const bool plain = allow_plain && osc_plain(p, N, frame, kd6 ? 6 : 3, io.pv != nullptr, io.ierr != nullptr);
  g_picked_plain = plain ? 1 : 0;
  for (int64_t b = 0; b < io.B; ++b) {
    if (kd6) {
      if (plain)
        path_traj<T, N, ORTHO, 6, true>(P, O, io, b);
      else
        path_traj<T, N, ORTHO, 6, false>(P, O, io, b);
    } else {
      if (plain)
        path_traj<T, N, ORTHO, 3, true>(P, O, io, b);
      else
        path_traj<T, N, ORTHO, 3, false>(P, O, io, b);
    }
  }
}

}  // namespace

extern "C" {

// Returns 1 if the plain instantiation ran, 0 if the general one, < 0 on a bad argument.  general != 0 runs the general
// instantiation even for calls that qualify for the plain one.
int ps_rollout_path(const abrb_chain_desc *d, const abrb_osc_params *p, int f32, int general, int frame,
                    const double *xoff, double *q, double *dq, const double *path, int path_stride, const double *pv,
                    int pv_stride, int steps, double dt, double effort, double *q_traj, double *dq_traj,
                    double *u_traj, double *x_traj, double *cost, double *ierr, int64_t B) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  if (!check_osc(h.n, *p).empty()) return ABRB_EUNSUP;
  if ((p->ki != 0.0) != (ierr != nullptr)) return ABRB_EINVAL;
  const PathIo io{q, dq, path, pv, path_stride, pv_stride, steps, dt, effort, q_traj, dq_traj, u_traj, x_traj, cost,
                  ierr, B};
  const bool ortho = h.ortho;
  DISPATCH_N(path_loop, h, *p, frame, xoff, io, general == 0);
  return g_picked_plain;
}
}
