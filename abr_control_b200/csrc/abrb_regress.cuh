// abrb_regress.cuh — the inverse-dynamics regressor of one state: u = M ddq + C dq - g = Y(q, dq, ddq) theta.
//
// theta is the diagonal link inertias of links 1..N, flattened: parameter p = 6 (l - 1) + c is link_inertia[l][c]
// (c = 0..5: m_x, m_y, m_z, I_xx, I_yy, I_zz).  Link 0 never moves, so it never enters.  Y is the coefficient of every
// inertia constant in dynamics_Mg<T, N, true> and inverse_apply (DESIGN.md S3.7):
//   translational, link l, axis c:  v_la[c] (sum_b v_lb[c] ddq_b + acc_l[c] - gravity[c])
//     with v_la = d p_l / d q_a and acc_l the C dq accumulator of link l before its product with Wp[l];
//   rotational: the inertias enter only through Wos[k][c] = sum_{l>k} I_l[c] (and gos = Wos o gravity[3:]), so the
//     coefficient of each Wos[k] is formed first (M ddq, C dq and -g restricted to the terms with max(a, b) = k) and
//     link l's rotational columns are its prefix sum over k < l.
#pragma once
#include "abrb_math.cuh"

namespace abrb {

// Record of one state: Y^T, (6N, N) row-major, element (p, a) = d u_a / d theta_p.  Link l's block of 6N values
// (rows 6 (l - 1) .. 6 l - 1) is contiguous; its translational half (rows c = 0..2) and its rotational half (c = 3..5)
// are each handed to `out.template put<3 N>(offset, half)` as soon as they are complete, with `offset` the half's first
// element in the record, so only one half is live at a time.
template <int N>
struct RegressorLayout {
  static constexpr int kParams = 6 * N;
  static constexpr int kRecord = 6 * N * N;
  static constexpr int kHalf = 3 * N;
  static ABRB_HD constexpr int trans(int l) { return 6 * N * (l - 1); }  // link l = 1..N
  static ABRB_HD constexpr int rot(int l) { return 6 * N * (l - 1) + 3 * N; }
};

template <typename T, int N, class K_, class Out>
ABRB_HD void inverse_dynamics_regressor(const ChainK<T, N> &P, const T *gravity, const T *q, const T *dq, const T *ddq,
                                        Out &out, K_ &K) {
  constexpr bool ORTHO = K_::kOrtho;
  typedef RegressorLayout<N> L;
  K.sync();
  walk<T, N>(P, q, 0, K);
  K.sync();
  // ---- translational halves: per link, the columns v_la and the link's C dq accumulator (dynamics_Mg's loop body)
  Spin<T, ORTHO> Wl;
  Wl.clear();
  ABRB_UNROLL
  for (int l = 1; l <= N; ++l) {
    T v[N][3];
    link_columns<T, N>(K, l, v);
    Wl.add(K, l - 1, dq[l - 1]);
    Spin<T, ORTHO> tail;
    tail.clear();
    T suf[3] = {T(0), T(0), T(0)}, f[3] = {T(0), T(0), T(0)};
    ABRB_UNROLL
    for (int j = N - 1; j >= 0; --j) {
      if (j < l) {
        tail.add(K, j, dq[j]);
        ABRB_UNROLL
        for (int c = 0; c < 3; ++c) suf[c] += dq[j] * v[j][c];
        T a1[3], a2[3];
        spin_diff_apply(Wl, tail, v[j], a1);  // W_j v_j
        omega_apply(K, j, suf, a2);           // Omega_j suf_j
        ABRB_UNROLL
        for (int c = 0; c < 3; ++c) f[c] += dq[j] * (a1[c] + a2[c]) + ddq[j] * v[j][c];
      }
    }
    T half[3 * N];
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) {
      const T fc = f[c] - gravity[c];  // COM acceleration minus gravity, axis c
      ABRB_UNROLL
      for (int a = 0; a < N; ++a) half[c * N + a] = a < l ? v[a][c] * fc : T(0);
    }
    out.template put<L::kHalf>(L::trans(l), half);
  }
  // ---- rotational halves.  Coefficient of Wos[m][c] in u_a (zero for a > m), with
  //   Pz = sum_{j<=m} dq_j z_j,  Pd = sum_{j<=m} dq_j zd_j,  Pa = sum_{j<=m} ddq_j z_j,  zd_j = W_j z_j,
  //   X_a = zd_a - sum_{a<k<m} dq_k Omega_a z_k:
  //   a < m:   z_a z_m ddq_m + dq_m (z_m X_a + z_a zd_m - (Omega_a z_m) Pz)      (componentwise in c)
  //   a == m:  z_m Pa + zd_m Pz + z_m Pd - z_m gravity[3 + c]
  // (M ddq, then dM/dt dq and -1/2 d/dq (dq^T M dq) of dynamics_Mg_rotational, then -g.)
  K.sync();
  Spin<T, ORTHO> W;
  W.clear();
  T Pz[3] = {T(0), T(0), T(0)}, Pd[3] = {T(0), T(0), T(0)}, Pa[3] = {T(0), T(0), T(0)};
  T X[N][3], rot[3 * N];
  ABRB_UNROLL
  for (int i = 0; i < 3 * N; ++i) rot[i] = T(0);
  ABRB_UNROLL
  for (int m = 0; m < N; ++m) {
    T zm[3], zdm[3];
    K.z(m, zm);
    W.apply(zm, zdm);
    W.add(K, m, dq[m]);
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) {
      Pz[c] += dq[m] * zm[c];
      Pd[c] += dq[m] * zdm[c];
      Pa[c] += ddq[m] * zm[c];
    }
    ABRB_UNROLL
    for (int a = 0; a < N; ++a) {
      if (a < m) {
        T za[3], oz[3];
        K.z(a, za);
        omega_apply(K, a, zm, oz);
        ABRB_UNROLL
        for (int c = 0; c < 3; ++c) {
          rot[c * N + a] += za[c] * zm[c] * ddq[m] + dq[m] * (zm[c] * X[a][c] + za[c] * zdm[c] - oz[c] * Pz[c]);
          X[a][c] -= dq[m] * oz[c];
        }
      }
    }
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) {
      rot[c * N + m] += zm[c] * (Pa[c] + Pd[c] - gravity[3 + c]) + zdm[c] * Pz[c];
      X[m][c] = zdm[c];
    }
    out.template put<L::kHalf>(L::rot(m + 1), rot);
  }
}

}  // namespace abrb
