// abrb_theta.cuh — the gradient of the plant rollout with respect to the link inertias theta (DESIGN.md S3.8).
//
// theta = link_inertia[1:] flattened, as in abrb_regress.cuh.  At a fixed applied torque tau, Y(q, dq, ddq) theta = tau
// gives d ddq / d theta = -M^-1 Y(q, dq, ddq), and with compensate_gravity tau = u - g = u + Y(q, 0, 0) theta.  Step t
// of the rollout (state (q_t, dq_t) before the step, applied torque tau_t) then contributes
//     -Y(q_t, dq_t, ddq_t)^T w_t + c_g Y(q_t, 0, 0)^T gu_t,     w_t = gu_t - 2 e gcost tau_t - gtau_t
// where gu_t is the torque cotangent of abrb_plant_rollout_vjp_* (per trajectory), e the effort weight, gcost the cost
// cotangent and gtau_t that of the recorded tau_t; w_t = M^-1 (dt^2 mu_q + dt mu_dq) is the part of gu_t that flows
// through ddq_t.  ddq_t is recomputed from (q_t, dq_t, tau_t) by the plant's own terms and Cholesky solve.
#pragma once
#include "abrb_rbd.cuh"
#include "abrb_regress.cuh"

namespace abrb {

// Output functor for inverse_dynamics_regressor: contracts each finished half of the record with the weights w,
// acc[6 (l - 1) + 3 h + c] += sum_a half[c N + a] w[a] (h = 0 translational, 1 rotational), instead of storing Y^T
template <typename T, int N>
struct ThetaContract {
  const T *w;  // N
  T *acc;      // 6N, theta's order
  template <int LEN>
  ABRB_HD void put(int off, const T *half) {
    typedef RegressorLayout<N> L;
    const int p0 = 6 * (off / L::kParams) + 3 * ((off % L::kParams) / L::kHalf);
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) {
      T s = T(0);
      ABRB_UNROLL
      for (int a = 0; a < N; ++a) s += half[c * N + a] * w[a];
      acc[p0 + c] += s;
    }
  }
};

// walk, M, g and C dq of (q, dq), then the applied torque and ddq exactly as plant_advance forms them
template <typename T, int N, class K_>
ABRB_HD_NOINLINE void theta_phase_plant(const ChainK<T, N> &P, const T *q, const T *dq, const T *u, bool comp_g,
                                        T *tau, T *ddq, K_ &K) {
  K.sync();
  walk<T, N>(P, q, 0, K);
  T M[N][N], g[N], cdq[N], Mi[N];
  plant_terms<T, N>(P, dq, M, g, cdq, K);
  K.sync();
  chol<T, N>(M, Mi);
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    tau[k] = comp_g ? u[k] - g[k] : u[k];
    ddq[k] = tau[k] + g[k] - cdq[k];
  }
  fwd_solve<T, N>(M, Mi, ddq);
  bwd_solve<T, N>(M, Mi, ddq);
}

// acc += Y(q, dq, ddq)^T w
template <typename T, int N, class K_>
ABRB_HD_NOINLINE void theta_phase_regress(const ChainK<T, N> &P, const T *gravity, const T *q, const T *dq,
                                          const T *ddq, const T *w, T *acc, K_ &K) {
  ThetaContract<T, N> sink{w, acc};
  inverse_dynamics_regressor<T, N>(P, gravity, q, dq, ddq, sink, K);
}

// One step's contribution to theta's cotangent, added to acc (6N): the state (q, dq) before the step, its torque row
// u, the torque cotangent gu, ec = 2 e gcost and gtau (N, or nullptr: zero)
template <typename T, int N, class K_>
ABRB_HD void theta_vjp_state(const ChainK<T, N> &P, const T *gravity, const T *q, const T *dq, const T *u,
                             bool comp_g, const T *gu, T ec, const T *gtau, T *acc, K_ &K) {
  T tau[N], ddq[N], nw[N];
  theta_phase_plant<T, N>(P, q, dq, u, comp_g, tau, ddq, K);
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) nw[k] = ec * tau[k] + (gtau != nullptr ? gtau[k] : T(0)) - gu[k];  // -w
  theta_phase_regress<T, N>(P, gravity, q, dq, ddq, nw, acc, K);
  if (comp_g) {
    T zero[N];
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) zero[k] = T(0);
    theta_phase_regress<T, N>(P, gravity, q, zero, zero, gu, acc, K);
  }
}

}  // namespace abrb
