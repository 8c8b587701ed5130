// abrb_rbd.cuh — one state of the batched rigid-body quantities {Tx, T, R, T_inv, quaternion, J, dJ, M, g, C}
// (reference: /root/reference/abr_control/arms/base_config.py:210-415).
#pragma once
#include "abrb_math.cuh"

namespace abrb {

enum : unsigned {
  kWantTx = 1u << 0,
  kWantT = 1u << 1,
  kWantR = 1u << 2,
  kWantTinv = 1u << 3,
  kWantQuat = 1u << 4,
  kWantJ = 1u << 5,
  kWantdJ = 1u << 6,
  kWantM = 1u << 7,
  kWantg = 1u << 8,
  kWantC = 1u << 9,
};

enum { kOutTx = 0, kOutT, kOutR, kOutTinv, kOutQuat, kOutJ, kOutdJ, kOutM, kOutg, kOutC, kOutCount };

// One state.  Every requested quantity is handed to `out.template put<LEN>(which, record)` as soon as it is complete,
// so that no more than one or two output records are ever live in registers (the kernel's `put` stages the record
// through shared memory and writes it out coalesced; the host test shim copies it into an array).
// DYN: M and/or g requested; CMAT: C requested; XTRA: any of Tx/T/R/T_inv/quaternion/dJ requested (compiled out of
// the common {J, M, g, C} instantiations: less code to fetch, fewer live registers).  `want` is uniform over the launch.
// `K` is the caller-provided kinematic scratch (register- or shared-memory-backed, see Kin in abrb_math.cuh).
template <typename T, int N, bool DYN, bool CMAT, bool XTRA, class K_, class Out>
ABRB_HD void rbd_state(const ChainK<T, N> &P, const T *q, const T *dq, int frame, const T *xoff, unsigned want,
                       K_ &K, Out &out) {
  if (!XTRA) want &= (kWantJ | kWantM | kWantg | kWantC);
  K.sync();
  walk<T, N>(P, q, frame, K);
  K.sync();
  const int dep = frame_dep<N>(frame);
  T pF[3];
  frame_point(K.F, xoff, pF);
  if (XTRA && (want & kWantTx)) out.template put<3>(kOutTx, pF);
  if (XTRA && (want & kWantT)) {  // base_config.py:338-369
    T Tm[16];
    ABRB_UNROLL
    for (int i = 0; i < 12; ++i) Tm[i] = K.F[i];
    Tm[12] = Tm[13] = Tm[14] = T(0);
    Tm[15] = T(1);
    out.template put<16>(kOutT, Tm);
  }
  if (XTRA && (want & (kWantR | kWantQuat))) {  // base_config.py:647-676, :304-318
    T R[9];
    ABRB_UNROLL
    for (int r = 0; r < 3; ++r)
      ABRB_UNROLL
    for (int c = 0; c < 3; ++c) R[r * 3 + c] = K.F[r * 4 + c];
    if (want & kWantR) out.template put<9>(kOutR, R);
    if (want & kWantQuat) {
      T qt[4];
      quat_from_R(R, qt);
      out.template put<4>(kOutQuat, qt);
    }
  }
  if (XTRA && (want & kWantTinv)) {  // [[R^T, -R^T t],[0,1]] with the TRANSPOSE (base_config.py:820-824)
    T Ti[16];
    ABRB_UNROLL
    for (int r = 0; r < 3; ++r) {
      T s = T(0);
      ABRB_UNROLL
      for (int c = 0; c < 3; ++c) {
        Ti[r * 4 + c] = K.F[c * 4 + r];
        s -= K.F[c * 4 + r] * K.F[c * 4 + 3];
      }
      Ti[r * 4 + 3] = s;
    }
    Ti[12] = Ti[13] = Ti[14] = T(0);
    Ti[15] = T(1);
    out.template put<16>(kOutTinv, Ti);
  }
  K.sync();
  if (want & (kWantJ | kWantdJ)) {
    T J[6][N];
    jacobian<T, N>(K, pF, dep, J);
    if (want & kWantJ) out.template put<6 * N>(kOutJ, &J[0][0]);
    if (XTRA && (want & kWantdJ)) {
      T dJ[6][N];
      jacobian_dot<T, N>(K, J, dq, dep, dJ);
      out.template put<6 * N>(kOutdJ, &dJ[0][0]);
    }
  }
  if (DYN) {
    T M[N][N], g[N];
    dynamics_Mg<T, N, false>(P, K, dq, M, g, nullptr);
    ABRB_UNROLL
    for (int a = 0; a < N; ++a)
      ABRB_UNROLL
    for (int b = 0; b < N; ++b)
      if (b < a) M[a][b] = M[b][a];
    if (want & kWantM) out.template put<N * N>(kOutM, &M[0][0]);
    if (want & kWantg) out.template put<N>(kOutg, g);
  }
  K.sync();
  if (CMAT) {
    T C[N][N];
    dynamics_C<T, N>(P, K, dq, C);
    out.template put<N * N>(kOutC, &C[0][0]);
  }
}

// ------------------------------------------------------------------------------------------------ the plant
// The rollouts' plant (reference semi-implicit Euler, arms/twojoint/arm_sim.py:131-132) on its own:
//     ddq = M(q)^-1 (tau + g(q) - C(q, dq) dq),   u = M(q) ddq + C(q, dq) dq - g(q)
// g is the generalized gravity force the controllers subtract (base_config.py:417-468) and C dq the product
// dynamics_Mg<T, N, true> returns.  The operations and their order are those of osc_eval's PLANT branch, so a torque
// sequence recorded by a closed-loop rollout replays to the same track.

// M (full, symmetric), g and C dq of the state whose walk K holds
template <typename T, int N, class K_>
ABRB_HD void plant_terms(const ChainK<T, N> &P, const T *dq, T (*M)[N], T *g, T *cdq, K_ &K) {
  K.sync();
  dynamics_Mg<T, N, true>(P, K, dq, M, g, cdq);
  ABRB_UNROLL
  for (int a = 0; a < N; ++a)
    ABRB_UNROLL
  for (int b = 0; b < N; ++b)
    if (b < a) M[a][b] = M[b][a];
}

// Forward dynamics of one state: ddq = M^-1 (u + g - C dq)
template <typename T, int N, class K_>
ABRB_HD void forward_dynamics_state(const ChainK<T, N> &P, const T *q, const T *dq, const T *u, T *ddq, K_ &K) {
  K.sync();
  walk<T, N>(P, q, 0, K);
  T M[N][N], Mi[N], g[N], cdq[N];
  plant_terms<T, N>(P, dq, M, g, cdq, K);
  K.sync();
  chol<T, N>(M, Mi);
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) ddq[k] = u[k] + g[k] - cdq[k];
  fwd_solve<T, N>(M, Mi, ddq);
  bwd_solve<T, N>(M, Mi, ddq);
}

// Inverse dynamics of one state: u = M ddq + C dq - g
template <typename T, int N, class K_>
ABRB_HD void inverse_dynamics_state(const ChainK<T, N> &P, const T *q, const T *dq, const T *ddq, T *u, K_ &K) {
  K.sync();
  walk<T, N>(P, q, 0, K);
  T M[N][N], g[N], cdq[N];
  plant_terms<T, N>(P, dq, M, g, cdq, K);
  ABRB_UNROLL
  for (int a = 0; a < N; ++a) {
    T s = T(0);
    ABRB_UNROLL
    for (int b = 0; b < N; ++b) s += M[a][b] * ddq[b];
    u[a] = s + cdq[a] - g[a];
  }
}

// Row t of trajectory b of a torque sequence of abrb_plant_rollout_*: (steps, B, N) when stride != 0 (== N), one
// (steps, N) sequence for every trajectory when stride == 0.
template <typename T, int N>
ABRB_HD const T *torque_row(const T *u, int stride, int t, int64_t B, int64_t b) {
  return u + (stride != 0 ? ((int64_t)t * B + b) * N : (int64_t)t * N);
}

// One step of the open-loop plant rollout (plant_kernel), for the torque row `u` and the path row `p` (3 values used,
// or nullptr):
//     tau = u, or u - g with comp_g (the residual-torque form);  x = control point (frame + xoff) at q
//     ddq = M^-1 (tau + g - C dq);  dq += ddq dt;  q += dq dt
//     cost += |x - p[:3]|^2 (with a path) + effort |tau|^2
// `tau` and `x` belong to the state BEFORE the update, as in rollout_step.
template <typename T, int N, class K_>
ABRB_HD void plant_step(const ChainK<T, N> &P, int frame, const T *xoff, T *q, T *dq, const T *u, bool comp_g,
                        const T *p, T dt, T effort, T *tau, T *x, T &cost, K_ &K) {
  K.sync();
  walk<T, N>(P, q, frame, K);
  K.sync();
  frame_point(K.F, xoff, x);
  T M[N][N], Mi[N], g[N], cdq[N], rhs[N];
  plant_terms<T, N>(P, dq, M, g, cdq, K);
  K.sync();
  chol<T, N>(M, Mi);
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    tau[k] = comp_g ? u[k] - g[k] : u[k];
    rhs[k] = tau[k] + g[k] - cdq[k];
  }
  fwd_solve<T, N>(M, Mi, rhs);
  bwd_solve<T, N>(M, Mi, rhs);
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    dq[k] += rhs[k] * dt;
    q[k] += dq[k] * dt;
  }
  T ex = T(0), eu = T(0);
  if (p != nullptr) {
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) {
      const T d = x[c] - p[c];
      ex += d * d;
    }
  }
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) eu += tau[k] * tau[k];
  cost += ex + effort * eu;
}

}  // namespace abrb
