// TEST INFRASTRUCTURE ONLY — never loaded by the abr_control_b200 package.
// Instantiates the __host__ __device__ per-state functions of abr_control_b200/csrc with g++ so that
// the kernel arithmetic can be unit-tested against the oracle on a machine without a GPU
// (`pytest -m "not gpu"`).  The shipped library (libabrb.so) reaches the same functions only through
// CUDA kernels.
#include <type_traits>
#include <vector>

#include "../../abr_control_b200/csrc/abrb_host.hpp"
#include "../../abr_control_b200/csrc/abrb_rbd.cuh"

using namespace abrb;

namespace {

template <typename T>
struct Sink {  // receives each finished per-state record from rbd_state
  double *dst[kOutCount];
  int64_t b;
  template <int LEN>
  void put(int which, const T *rec) {
    if (dst[which])
      for (int i = 0; i < LEN; ++i) dst[which][b * LEN + i] = double(rec[i]);
  }
};

template <typename T, int N, bool ORTHO>
void rbd_loop(const ChainHost &h, int frame, const double *xoff, const double *q, const double *dq, int64_t B,
              unsigned want, double *Tx, double *Tm, double *R, double *Tinv, double *quat, double *J, double *dJ,
              double *M, double *g, double *C) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  T xo[3] = {T(xoff ? xoff[0] : 0), T(xoff ? xoff[1] : 0), T(xoff ? xoff[2] : 0)};
  for (int64_t b = 0; b < B; ++b) {
    T qq[N], dd[N];
    for (int k = 0; k < N; ++k) {
      qq[k] = T(q[b * N + k]);
      dd[k] = dq ? T(dq[b * N + k]) : T(0);
    }
    Sink<T> sink{{Tx, Tm, R, Tinv, quat, J, dJ, M, g, C}, b};
    Kin<T, N, ORTHO> K;
    rbd_state<T, N, true, true, true>(P, qq, dd, frame, xo, want, K, sink);
  }
}

template <typename T, int N, bool ORTHO>
void osc_loop(const ChainHost &h, const abrb_osc_params &p, int frame, const double *xoff, const double *q,
              const double *dq, const double *target, int tstride, const double *tv, int tvstride, int64_t B,
              double *u, double *train, double *ddq, double *ierr) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  OscK<T, N> O;
  fill_osc<T, N>(p, frame, xoff, O);
  const bool kd6 = (O.dof_mask & 56u) != 0;
  for (int64_t b = 0; b < B; ++b) {
    T qq[N], dd[N], tg[6], tvv[6], uu[N], tr[N], acc[N], ie[6];
    for (int k = 0; k < N; ++k) {
      qq[k] = T(q[b * N + k]);
      dd[k] = T(dq[b * N + k]);
    }
    for (int c = 0; c < 6; ++c) {
      tg[c] = T(target[b * tstride + c]);
      tvv[c] = tv ? T(tv[b * tvstride + c]) : T(0);
      ie[c] = ierr ? T(ierr[b * 6 + c]) : T(0);
    }
    Kin<T, N, ORTHO> K;
    if (kd6)
      osc_state<T, N, 6, true>(P, O, qq, dd, tg, tv ? tvv : nullptr, ierr ? ie : nullptr, uu, tr, acc, K);
    else
      osc_state<T, N, 3, true>(P, O, qq, dd, tg, tv ? tvv : nullptr, ierr ? ie : nullptr, uu, tr, acc, K);
    for (int c = 0; c < 6; ++c)
      if (ierr) ierr[b * 6 + c] = double(ie[c]);
    for (int k = 0; k < N; ++k) {
      u[b * N + k] = double(uu[k]);
      if (train) train[b * N + k] = double(tr[k]);
      if (ddq) ddq[b * N + k] = double(acc[k]);
    }
  }
}

template <typename T, int N, bool ORTHO>
void null_loop(const ChainHost &h, const abrb_null_params &z, const double *q, const double *dq, int64_t B, double *u) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  NullK<T, N> Z;
  fill_null<T, N>(z, Z);
  for (int64_t b = 0; b < B; ++b) {
    T qq[N], dd[N], uu[N];
    for (int k = 0; k < N; ++k) {
      qq[k] = T(q[b * N + k]);
      dd[k] = T(dq[b * N + k]);
    }
    Kin<T, N, ORTHO> K;
    null_state<T, N>(P, Z, qq, dd, uu, K);
    for (int k = 0; k < N; ++k) u[b * N + k] = double(uu[k]);
  }
}

template <typename T, int N, bool ORTHO>
void sliding_loop(const ChainHost &h, double kd, double lamb, int cartesian, int frame, const double *xoff,
                  const double *q, const double *dq, const double *target, const double *tv, const double *ta,
                  int64_t B, double *u, double *s) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  const int w = cartesian ? 3 : N;
  constexpr int L = CtrlRow<N>::kMax;  // a cartesian row is 3 wide whatever N is
  T xo[3] = {T(xoff ? xoff[0] : 0), T(xoff ? xoff[1] : 0), T(xoff ? xoff[2] : 0)};
  for (int64_t b = 0; b < B; ++b) {
    T qq[N], dd[N], tg[L], tvv[L], taa[L], uu[N], ss[N];
    for (int k = 0; k < N; ++k) {
      qq[k] = T(q[b * N + k]);
      dd[k] = T(dq[b * N + k]);
    }
    for (int k = 0; k < L; ++k) {
      tg[k] = k < w ? T(target[b * w + k]) : T(0);
      tvv[k] = (k < w && tv) ? T(tv[b * w + k]) : T(0);
      taa[k] = (k < w && ta) ? T(ta[b * w + k]) : T(0);
    }
    Kin<T, N, ORTHO> K;
    sliding_state<T, N>(P, T(kd), T(lamb), cartesian != 0, frame, xo, qq, dd, tg, tvv, taa, uu, ss, K);
    for (int k = 0; k < N; ++k) {
      u[b * N + k] = double(uu[k]);
      if (s) s[b * N + k] = double(ss[k]);
    }
  }
}

template <typename T, int N, bool ORTHO>
void ik_loop(const ChainHost &h, double max_dx, double max_dr, double max_dq, int method, double dt, int steps,
             const double *position, const double *target, int64_t B, double *pos_path, double *vel_path) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  for (int64_t b = 0; b < B; ++b) {
    T q[N], dq[N], tg[3], Qd[4];
    for (int k = 0; k < N; ++k) q[k] = T(position[b * N + k]);
    for (int c = 0; c < 3; ++c) tg[c] = T(target[b * 6 + c]);
    quat_from_euler_sxyz(T(target[b * 6 + 3]), T(target[b * 6 + 4]), T(target[b * 6 + 5]), Qd);
    const T nq = T(1) / sqrt_t(Qd[0] * Qd[0] + Qd[1] * Qd[1] + Qd[2] * Qd[2] + Qd[3] * Qd[3]);
    for (int i = 0; i < 4; ++i) Qd[i] *= nq;
    for (int t = 0; t < steps; ++t) {
      Kin<T, N, ORTHO> K;
      ik_step<T, N>(P, T(max_dx * dt), T(max_dr * dt), T(max_dq * dt), method, q, tg, Qd, dq, K);
      for (int k = 0; k < N; ++k) {
        pos_path[((int64_t)t * B + b) * N + k] = double(q[k]);  // (steps, B, n) like the kernel
        vel_path[((int64_t)t * B + b) * N + k] = double(dq[k]);
        q[k] += dq[k];
      }
    }
  }
}

template <typename T, int N, bool ORTHO>
void ctrl_loop(const ChainHost &h, int kind, double kp, double kv, int fa, int fb, const double *q, const double *dq,
               const double *target, const double *tv, int64_t B, double *u) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  for (int64_t b = 0; b < B; ++b) {
    T qq[N], dd[N], tg[N], tvv[N], uu[N];
    for (int k = 0; k < N; ++k) {
      qq[k] = T(q[b * N + k]);
      dd[k] = dq ? T(dq[b * N + k]) : T(0);
      tg[k] = target ? T(target[b * N + k]) : T(0);
      tvv[k] = tv ? T(tv[b * N + k]) : T(0);
    }
    Kin<T, N, ORTHO> K;
    if (kind == 0)
      joint_state<T, N>(P, T(kp), T(kv), fa != 0, qq, dd, tg, tv ? tvv : nullptr, uu, K);
    else
      floating_state<T, N>(P, fa != 0, fb != 0, qq, dd, uu, K);
    for (int k = 0; k < N; ++k) u[b * N + k] = double(uu[k]);
  }
}

}  // namespace

#define DISPATCH_N(FN, ...)                                       \
  switch (h.n) {                                                  \
    case 1: DISPATCH_T(FN, 1, __VA_ARGS__); break;                \
    case 2: DISPATCH_T(FN, 2, __VA_ARGS__); break;                \
    case 3: DISPATCH_T(FN, 3, __VA_ARGS__); break;                \
    case 4: DISPATCH_T(FN, 4, __VA_ARGS__); break;                \
    case 5: DISPATCH_T(FN, 5, __VA_ARGS__); break;                \
    case 6: DISPATCH_T(FN, 6, __VA_ARGS__); break;                \
    case 7: DISPATCH_T(FN, 7, __VA_ARGS__); break;                \
    default: return ABRB_ESHAPE;                                  \
  }
#define DISPATCH_T(FN, N, ...)                                    \
  if (f32) {                                                      \
    if (ortho) FN<float, N, true>(__VA_ARGS__); else FN<float, N, false>(__VA_ARGS__);   \
  } else {                                                        \
    if (ortho) FN<double, N, true>(__VA_ARGS__); else FN<double, N, false>(__VA_ARGS__); \
  }

extern "C" {

// force_general != 0 runs the non-orthonormal code path even for orthonormal chains
int hs_rbd(const abrb_chain_desc *d, int f32, int force_general, int frame, const double *xoff, const double *q,
           const double *dq, int64_t B, double *Tx, double *Tm, double *R, double *Tinv, double *quat, double *J,
           double *dJ, double *M, double *g, double *C) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const bool ortho = h.ortho && !force_general;
  unsigned want = 0;
  if (Tx) want |= kWantTx;
  if (Tm) want |= kWantT;
  if (R) want |= kWantR;
  if (Tinv) want |= kWantTinv;
  if (quat) want |= kWantQuat;
  if (J) want |= kWantJ;
  if (dJ) want |= kWantdJ | kWantJ;
  if (M) want |= kWantM;
  if (g) want |= kWantg;
  if (C) want |= kWantC;
  DISPATCH_N(rbd_loop, h, frame, xoff, q, dq, B, want, Tx, Tm, R, Tinv, quat, J, dJ, M, g, C);
  return 0;
}

int hs_osc(const abrb_chain_desc *d, const abrb_osc_params *p, int f32, int force_general, int frame,
           const double *xoff, const double *q, const double *dq, const double *target, int tstride, const double *tv,
           int tvstride, int64_t B, double *u, double *train, double *ddq, double *ierr) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  if (!check_osc(h.n, *p).empty()) return ABRB_EUNSUP;
  if ((p->ki != 0.0) != (ierr != nullptr)) return ABRB_EINVAL;
  const bool ortho = h.ortho && !force_general;
  DISPATCH_N(osc_loop, h, *p, frame, xoff, q, dq, target, tstride, tv, tvstride, B, u, train, ddq, ierr);
  return 0;
}

int hs_null(const abrb_chain_desc *d, const abrb_null_params *z, int f32, int force_general, const double *q,
            const double *dq, int64_t B, double *u) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const bool ortho = h.ortho && !force_general;
  DISPATCH_N(null_loop, h, *z, q, dq, B, u);
  return 0;
}

int hs_ctrl(const abrb_chain_desc *d, int f32, int force_general, int kind, double kp, double kv, int fa, int fb,
            const double *q, const double *dq, const double *target, const double *tv, int64_t B, double *u) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const bool ortho = h.ortho && !force_general;
  DISPATCH_N(ctrl_loop, h, kind, kp, kv, fa, fb, q, dq, target, tv, B, u);
  return 0;
}

int hs_sliding(const abrb_chain_desc *d, int f32, int force_general, double kd, double lamb, int cartesian, int frame,
               const double *xoff, const double *q, const double *dq, const double *target, const double *tv,
               const double *ta, int64_t B, double *u, double *s) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const bool ortho = h.ortho && !force_general;
  DISPATCH_N(sliding_loop, h, kd, lamb, cartesian, frame, xoff, q, dq, target, tv, ta, B, u, s);
  return 0;
}

int hs_ik(const abrb_chain_desc *d, int f32, int force_general, double max_dx, double max_dr, double max_dq, int method,
          double dt, int steps, const double *position, const double *target, int64_t B, double *pos_path,
          double *vel_path) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const bool ortho = h.ortho && !force_general;
  DISPATCH_N(ik_loop, h, max_dx, max_dr, max_dq, method, dt, steps, position, target, B, pos_path, vel_path);
  return 0;
}

int hs_frame_id(int n, const char *name) { return parse_frame(n, name); }

// which = 0: w = A^T pinv(A A^T, rcond) y (6 values) for a K x 6 matrix A (K = 6 or 3) through the one-sided Jacobi route
// of the OSC kernels (pinv_rows_jacobi_seq: the sequential walk over the schedule the warp-cooperative device code runs
// in parallel); which = 1: x = pinv(S, rcond) y (K values) for a symmetric K x K matrix S through the cyclic Jacobi routine.
int hs_pinv(int K, const double *A_or_S, unsigned active, double rcond, const double *y, double *x, int which) {
  if (K != 6 && K != 3) return -1;
  if (which == 0) {
    double zero[6] = {0, 0, 0, 0, 0, 0}, wz[6];
    if (K == 6) pinv_rows_jacobi_seq<6, 6>(A_or_S, rcond, y, zero, false, x, wz);
    else pinv_rows_jacobi_seq<6, 3>(A_or_S, rcond, y, zero, false, x, wz);
    return 1;
  }
  double Sf[36], yi[6];
  for (int a = 0; a < K * K; ++a) Sf[a] = A_or_S[a];
  for (int a = 0; a < K; ++a) yi[a] = y[a];
  if (K == 6) pinv_apply_sym<double, 6>(Sf, active, rcond, yi, x);
  else pinv_apply_sym<double, 3>(Sf, active, rcond, yi, x);
  return 1;
}
}
