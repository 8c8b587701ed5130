// abrb_osc.cuh — one state of OSC.generate (and the secondary controllers), fully fused:
// chain walk -> J, M, g, (C dq) -> Cholesky(M) -> task-space inertia -> task PD -> joint torques ->
// null-space filtered secondary torques.  Reference: /root/reference/abr_control/controllers/osc.py:217-320,
// damping.py:21-32, resting_config.py:25-42 + joint.py:104-131, avoid_obstacles.py:38-120.
#pragma once
#include "abrb_math.cuh"
#include "abrb_rbd.cuh"

namespace abrb {

enum { kNullDamping = 1, kNullResting = 2, kNullAvoid = 3, kNullLimits = 4 };

template <typename T, int N>
struct NullK {
  int kind;
  int n_obs;
  unsigned rest_mask;
  int pad_;
  T kp, kv;
  T rest[N];
  T threshold, gain, maximum;
  T obs[kMaxObstacles][4];
  // AvoidJointLimits shares the storage: rest[] = lower limits, obs[0..1] = upper limits, obs[2..3] = max torque,
  // rest_mask bits 0-7 cross_zero, 8-15 gradient, 16-23 no lower limit, 24-31 no upper limit (abrb_host.hpp)
  ABRB_HD T lim_hi(int k) const { return obs[k >> 2][k & 3]; }
  ABRB_HD T lim_torque(int k) const { return obs[2 + (k >> 2)][k & 3]; }
};

// AvoidJointLimits.generate (controllers/avoid_joint_limits.py:83-142): a function of q alone
template <typename T, int N>
ABRB_HD void joint_limits_generate(const NullK<T, N> &Z, const T *q, T *u) {
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    const T x = q[k] - T(3.14159265358979323846);  // :91
    const T lo = Z.rest[k], hi = Z.lim_hi(k), tq = Z.lim_torque(k);
    const bool cross = (Z.rest_mask >> k) & 1u, grad = (Z.rest_mask >> (8 + k)) & 1u;
    const bool no_lo = (Z.rest_mask >> (16 + k)) & 1u, no_hi = (Z.rest_mask >> (24 + k)) & 1u;
    const T dlo = x - lo, dhi = x - hi;
    const bool nearer_hi = abs_t(dlo) >= abs_t(dhi);  // the reference's `closer_to_min_index` (:94-96)
    const bool nearer_lo = abs_t(dlo) <= abs_t(dhi);  // the reference's `closer_to_max_index` (:97-99)
    T a_lo = T(0), a_hi = T(0);
    if (grad) {  // :108-115
      const T e_lo = exp_t(T(1) / dlo), e_hi = exp_t(T(-1) / dhi);
      a_lo = e_lo < tq ? e_lo : tq;
      a_hi = -(e_hi < tq ? e_hi : tq);
    }
    bool below = dlo < T(0), above = dhi > T(0);  // :118-119
    if (cross) {                                 // :124-134
      below = below && (dhi > T(0)) && nearer_lo;
      above = above && (dlo < T(0)) && nearer_hi;
    }
    if (below) a_lo = tq;
    if (no_lo) a_lo = T(0);
    if (above) a_hi = -tq;
    if (no_hi) a_hi = T(0);
    u[k] = a_lo + a_hi;
  }
}

template <typename T, int N>
struct OscK {
  T kp, ko, kv, ki;
  T lim_xyz, lim_abg;  // vmax[0]/kp*kv, vmax[1]/ko*kv   (osc.py:109-115)
  T thr;               // |det| threshold of _Mx (osc.py:120,138)
  T xoff[3];
  unsigned dof_mask;   // bit r = ctrlr_dof[r]
  int use_vmax, use_g, use_C, alg, n_null, frame;
  NullK<T, N> nul[kMaxNull];
};

// pinv of a 3 x N matrix (the position or the orientation rows of a Jacobian) as numpy.linalg.pinv computes it
// (rcond = 1e-15), applied to right-hand sides: a one-sided (Hestenes) Jacobi SVD of the rows — rotations of row pairs
// until they are mutually orthogonal give J = V^T diag(sigma) U^T with sigma_i u_i = rotated row i, so
// pinv(J) y = sum_i row_i (v_i . y) / sigma_i^2 over the sigma_i > 1e-15 sigma_max.  (Going through J J^T would square
// the condition number.)  The sweep loop is rolled around three rotations with static indices.
template <typename T, int N>
struct RowPinv3 {
  T b0[N], b1[N], b2[N], v0[3], v1[3], v2[3], i0, i1, i2;

  ABRB_HD static void rotate(T *bi, T *bj, T *vi, T *vj) {
    T al = T(0), be = T(0), ga = T(0);
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) {
      al += bi[k] * bi[k];
      be += bj[k] * bj[k];
      ga += bi[k] * bj[k];
    }
    if (ga * ga > (sizeof(T) == 8 ? T(1e-32) : T(1e-14)) * al * be && ga != T(0)) {
      const T zeta = (be - al) / (T(2) * ga);
      const T t = (zeta >= T(0) ? T(1) : T(-1)) / (abs_t(zeta) + sqrt_t(T(1) + zeta * zeta));
      const T c = T(1) / sqrt_t(T(1) + t * t), sn = c * t;
      ABRB_UNROLL
      for (int k = 0; k < N; ++k) {
        const T x = bi[k], y = bj[k];
        bi[k] = c * x - sn * y;
        bj[k] = sn * x + c * y;
      }
      ABRB_UNROLL
      for (int k = 0; k < 3; ++k) {
        const T x = vi[k], y = vj[k];
        vi[k] = c * x - sn * y;
        vj[k] = sn * x + c * y;
      }
    }
  }

  // cut_rel: squared singular values <= cut_rel * largest are dropped (numpy.linalg.pinv of the 3 x N matrix with
  // rcond = 1e-15: pinv_cut2, 1e-30 in fp64 and 1e-12 in fp32; pinv(J J^T, rcond) of the symmetric product: rcond
  // itself)
  ABRB_HD void build(const T *r0, const T *r1, const T *r2, T cut_rel = pinv_cut2<T>()) {
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) {
      b0[k] = r0[k];
      b1[k] = r1[k];
      b2[k] = r2[k];
    }
    ABRB_UNROLL
    for (int k = 0; k < 3; ++k) {
      v0[k] = k == 0 ? T(1) : T(0);
      v1[k] = k == 1 ? T(1) : T(0);
      v2[k] = k == 2 ? T(1) : T(0);
    }
    ABRB_NOUNROLL
    for (int sweep = 0; sweep < 8; ++sweep) {
      rotate(b0, b1, v0, v1);
      rotate(b0, b2, v0, v2);
      rotate(b1, b2, v1, v2);
    }
    T s0 = T(0), s1 = T(0), s2 = T(0);
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) {
      s0 += b0[k] * b0[k];
      s1 += b1[k] * b1[k];
      s2 += b2[k] * b2[k];
    }
    const T smax = s0 > s1 ? (s0 > s2 ? s0 : s2) : (s1 > s2 ? s1 : s2);
    const T cut = cut_rel * smax;
    i0 = s0 > cut ? T(1) / s0 : T(0);
    i1 = s1 > cut ? T(1) / s1 : T(0);
    i2 = s2 > cut ? T(1) / s2 : T(0);
  }

  // out = pinv(J J^T, cut_rel) y: the eigenvalues of J J^T are the squared singular values, its eigenvectors the rows of V
  ABRB_HD void apply_sym(const T *y, T *out) const {
    const T c0 = (v0[0] * y[0] + v0[1] * y[1] + v0[2] * y[2]) * i0;
    const T c1 = (v1[0] * y[0] + v1[1] * y[1] + v1[2] * y[2]) * i1;
    const T c2 = (v2[0] * y[0] + v2[1] * y[1] + v2[2] * y[2]) * i2;
    ABRB_UNROLL
    for (int k = 0; k < 3; ++k) out[k] = v0[k] * c0 + v1[k] * c1 + v2[k] * c2;
  }

  ABRB_HD void apply(const T *y, T *out) const {  // out = pinv(J) y
    const T c0 = (v0[0] * y[0] + v0[1] * y[1] + v0[2] * y[2]) * i0;
    const T c1 = (v1[0] * y[0] + v1[1] * y[1] + v1[2] * y[2]) * i1;
    const T c2 = (v2[0] * y[0] + v2[1] * y[1] + v2[2] * y[2]) * i2;
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) out[k] = b0[k] * c0 + b1[k] * c1 + b2[k] * c2;
  }
};

// AvoidObstacles.generate — the rare, data-dependent secondary controller; not inlined and self-contained
// (re-walks the chain) so that the main path's register allocation is unaffected.
// Lm: Cholesky factor of M (row-major N x N, lower).
template <typename T, int N, bool ORTHO>
ABRB_HD_NOINLINE void avoid_generate(const ChainK<T, N> &P, const NullK<T, N> &A, const T *q, const T *Lm,
                                     T *u_out) {
  Kin<T, N, ORTHO> K;  // private register/local copy: this path is rare
  T LFs[N][12];
  walk<T, N>(P, q, 2 * N + 1, K, LFs);  // K.F = EE frame, LFs[i] = link(i+1) frame
  T up[N];
  for (int k = 0; k < N; ++k) up[k] = T(0);
  const T thr = A.threshold;
  for (int seg = 0; seg < N; ++seg) {
    const T *LF = LFs[seg];
    T p1[3], p2[3];
    K.t(seg, p1);
    K.t(seg + 1 < N ? seg + 1 : N - 1, p2);
    if (seg == N - 1)
      for (int r = 0; r < 3; ++r) p2[r] = K.F[r * 4 + 3];
    for (int ob = 0; ob < A.n_obs; ++ob) {
      const T *O = A.obs[ob];
      T line[3], obl[3];
      for (int r = 0; r < 3; ++r) {
        line[r] = p2[r] - p1[r];
        obl[r] = O[r] - p1[r];
      }
      const T proj = dot3(obl, line) / dot3(line, line);
      T cl[3];
      for (int r = 0; r < 3; ++r) cl[r] = proj < T(0) ? p1[r] : (proj > T(1) ? p2[r] : p1[r] + proj * line[r]);
      T d[3] = {O[0] - cl[0], O[1] - cl[1], O[2] - cl[2]};
      const T dist = sqrt_t(dot3(d, d));
      T rho = dist - O[3];
      const T floor_ = thr / T(50);
      rho = rho > floor_ ? rho : floor_;
      if (!(rho < thr)) continue;
      const T mag = T(0.02) * (T(1) / rho - T(1) / thr) * T(1) / (rho * sqrt_t(rho));
      T F[3];
      for (int r = 0; r < 3; ++r) F[r] = mag * (d[r] / rho);
      // m = T_inv(link) [closest;1] with the reference's TRANSPOSE inverse (base_config.py:820-824)
      T dl[3] = {cl[0] - LF[3], cl[1] - LF[7], cl[2] - LF[11]};
      T m[3], pw[3];
      for (int cc = 0; cc < 3; ++cc) m[cc] = LF[0 * 4 + cc] * dl[0] + LF[1 * 4 + cc] * dl[1] + LF[2 * 4 + cc] * dl[2];
      frame_point(LF, m, pw);
      // Jp (3 x N) of that point, W = L^-1 Jp^T (N x 3)
      T Jp[3][N], Wc[3][N];
      for (int k = 0; k < N; ++k) {
        T tk[3], v[3];
        K.t(k, tk);
        T dd[3] = {pw[0] - tk[0], pw[1] - tk[1], pw[2] - tk[2]};
        omega_apply(K, k, dd, v);
        for (int r = 0; r < 3; ++r) Jp[r][k] = k < seg + 1 ? v[r] : T(0);
      }
      for (int r = 0; r < 3; ++r) {
        for (int i = 0; i < N; ++i) {
          T sacc = Jp[r][i];
          for (int k = 0; k < i; ++k) sacc -= Lm[i * N + k] * Wc[r][k];
          Wc[r][i] = sacc / Lm[i * N + i];
        }
      }
      // Mx_pt F = pinv(Jp M^-1 Jp^T, rcond = 0.01) F  (avoid_obstacles.py:113-116): Jp M^-1 Jp^T = Wc Wc^T, so its
      // eigen-decomposition is the one-sided Jacobi SVD of the three rows of Wc (registers, no 3 x 3 matrix formed)
      T x3[3];
      RowPinv3<T, N> rp;
      rp.build(Wc[0], Wc[1], Wc[2], T(0.01));
      rp.apply_sym(F, x3);
      for (int k = 0; k < N; ++k) up[k] -= Jp[0][k] * x3[0] + Jp[1][k] * x3[1] + Jp[2][k] * x3[2];
    }
  }
  for (int k = 0; k < N; ++k) {
    T v = up[k] * A.gain;
    v = v > A.maximum ? A.maximum : v;
    v = v < -A.maximum ? -A.maximum : v;
    u_out[k] = v;
  }
}

// python-style (x mod 2pi) in [0, 2pi)
template <typename T>
ABRB_HD T wrap_pm_pi(T d) {
  const T two_pi = T(6.283185307179586476925286766559);
  const T pi = T(3.14159265358979323846264338327950288);
  T r = fmod_t(d + pi, two_pi);
  r = r < T(0) ? r + two_pi : r;
  return r - pi;
}

// Sequential stand-in for the warp-cooperative truncating pseudo-inverse (abrb_coop.cuh): used by the host
// instantiation (tests/hostsim), where a "warp" is one state.
struct SeqCoop {
  template <typename T, int N, int KD, class K_, class LGet>
  ABRB_HD void pinv(bool slow, K_ &K, LGet, const T *y, const T *z, T *wy, T *wz, bool two, double rcond) const {
    if (!slow) return;
    double A[KD * N], yd[KD], zd[KD], oy[N], oz[N];
    for (int r = 0; r < KD; ++r) {
      yd[r] = double(y[r]);
      zd[r] = double(z[r]);
      for (int k = 0; k < N; ++k) A[r * N + k] = double(K.s.ld(K_::aslot(r, k)));
    }
    pinv_rows_jacobi_seq<N, KD>(A, rcond, yd, zd, two, oy, oz);
    for (int k = 0; k < N; ++k) {
      wy[k] = T(oy[k]);
      wz[k] = T(oz[k]);
    }
  }
};

// One OSC evaluation.  KD = 3: only (a subset of) x,y,z controlled; KD = 6: any mask.
// PLANT: also return ddq = M^-1 (u + g - C dq) for the rollout kernel.
// `K`: caller-provided kinematic scratch (registers or shared memory).  Once the dynamics are done its t_k / z_k
// slots are overwritten IN PLACE by the task Jacobian (column k of J only needs t_k, z_k), which later becomes
// A = (L^-1 J^T)^T; so J, A never occupy registers of their own.
// `ierr`: the state's integrated task-space error (osc.py:81-82, :262-264), 6 values updated in place, or nullptr
// when ki == 0.
// `coop`: how the states whose task-space inertia needs the TRUNCATING pseudo-inverse (osc.py:138-145, a few percent
// of random UR5 states) are finished.  On the GPU every lane of the warp reaches coop.pinv() together and the lanes
// work on those states jointly (abrb_coop.cuh) instead of one lane walking a long serial path while 31 wait.
// PLAIN: the caller has established (osc_plain, abrb_host.hpp) that there is no secondary controller, no target
// velocity and no integrator, that all KD task rows of the EE frame are controlled, and that use_g and use_C are set.
// Those branches, their arrays and the per-row mask and per-joint frame selects then vanish at compile time; for the
// fp64 OSC kernels this is the difference between ~2.5 KB of local-memory spills per thread and none (DESIGN.md S4.1).
// `x`: receives the control point (ref_frame + xyz_offset) at q, 3 values, or nullptr.
template <typename T, int N, int KD, bool PLANT, bool PLAIN, class K_, class Coop>
ABRB_HD void osc_eval(const ChainK<T, N> &P, const OscK<T, N> &O, const T *q, const T *dq, const T *target,
                      const T *tv, T *ierr, T *u, T *train, T *ddq, K_ &K, Coop &coop, T *x = nullptr) {
  constexpr bool ORTHO = K_::kOrtho;
  auto Aslot = [](int r, int k) { return K_::aslot(r, k); };
  T M[N][N], Mi[N], g[N], cdq[N], un[N], y[KD], z[KD];
  // (read at each use, as the parameter itself is: a copy would hold a register through the whole evaluation)
  auto dof_mask = [&]() { return PLAIN ? (1u << KD) - 1u : O.dof_mask; };
  auto n_null = [&]() { return PLAIN ? 0 : O.n_null; };
  if (PLAIN) {
    tv = nullptr;
    ierr = nullptr;
  }
  const bool any_null = n_null() > 0;
  const T rcond = O.thr * T(0.1);
  K.sync();
  walk<T, N>(P, q, PLAIN ? 2 * N + 1 : O.frame, K);
  K.sync();
  const int dep = frame_dep<N>(PLAIN ? 2 * N + 1 : O.frame);
  T pF[3];
  frame_point(K.F, O.xoff, pF);
  if (x != nullptr) {
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) x[c] = pF[c];
  }

  // ---- task-space error (osc.py:250-272), needs only the frame
  T err[6] = {T(0), T(0), T(0), T(0), T(0), T(0)};
  if (dof_mask() & 7u) {
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) err[c] = pF[c] - target[c];
  }
  if (KD == 6 && (dof_mask() & 56u)) {
    T R[9];
    ABRB_UNROLL
    for (int r = 0; r < 3; ++r)
      ABRB_UNROLL
    for (int c = 0; c < 3; ++c) R[r * 3 + c] = K.F[r * 4 + c];
    if (O.alg == 0) {
      T qd[4], qe[4], qr[4];
      quat_from_euler_rxyz(target[3], target[4], target[5], qd);
      const T nd = inv_sqrt_t(qd[0] * qd[0] + qd[1] * qd[1] + qd[2] * qd[2] + qd[3] * qd[3]);
      ABRB_UNROLL
      for (int i = 0; i < 4; ++i) qd[i] *= nd;
      quat_from_R(R, qe);
      qe[1] = -qe[1];
      qe[2] = -qe[2];
      qe[3] = -qe[3];
      quat_mul(qd, qe, qr);
      const T sg = qr[0] > T(0) ? T(1) : (qr[0] < T(0) ? T(-1) : T(0));  // numpy.sign
      ABRB_UNROLL
      for (int c = 0; c < 3; ++c) err[3 + c] = -qr[1 + c] * sg;
    } else {
      T Rd[9], Red[9], qed[4];
      R_from_euler_rxyz(target[3], target[4], target[5], Rd);
      ABRB_UNROLL
      for (int r = 0; r < 3; ++r)
        ABRB_UNROLL
      for (int c = 0; c < 3; ++c) Red[r * 3 + c] = R[0 * 3 + r] * Rd[0 * 3 + c] + R[1 * 3 + r] * Rd[1 * 3 + c] + R[2 * 3 + r] * Rd[2 * 3 + c];
      quat_from_R(Red, qed);
      ABRB_UNROLL
      for (int r = 0; r < 3; ++r) err[3 + r] = -(R[r * 3 + 0] * qed[1] + R[r * 3 + 1] * qed[2] + R[r * 3 + 2] * qed[3]);
    }
  }
  if (ierr != nullptr) {  // osc.py:262-264: integrated_error += u_task; u_task += ki * integrated_error
    ABRB_UNROLL
    for (int c = 0; c < 6; ++c) {
      ierr[c] += err[c];
      err[c] += O.ki * ierr[c];
    }
  }
  if (O.use_vmax) {  // osc.py:198-215
    const T nx = sqrt_t(err[0] * err[0] + err[1] * err[1] + err[2] * err[2]);
    const T na = sqrt_t(err[3] * err[3] + err[4] * err[4] + err[5] * err[5]);
    const T sx = nx > O.lim_xyz ? O.lim_xyz / nx : T(1);
    const T sa = na > O.lim_abg ? O.lim_abg / na : T(1);
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) {
      err[c] = O.kv * sx * (O.kp / O.kv) * err[c];
      err[3 + c] = O.kv * sa * (O.ko / O.kv) * err[3 + c];
    }
  } else {
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) {
      err[c] *= O.kp;
      err[3 + c] *= O.ko;
    }
  }

  // ---- joint-space dynamics
  K.sync();
  if (PLANT || PLAIN || O.use_C)
    dynamics_Mg<T, N, true>(P, K, dq, M, g, cdq);
  else
    dynamics_Mg<T, N, false>(P, K, dq, M, g, nullptr);
  ABRB_UNROLL
  for (int a = 0; a < N; ++a)
    ABRB_UNROLL
  for (int b = 0; b < N; ++b)
    if (b < a) M[a][b] = M[b][a];

  // secondary controllers that are M.(something): accumulate the something
  T wn[N], ud[N];  // ud: secondary controllers that are plain joint torques (AvoidJointLimits)
  bool any_avoid = false;
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    wn[k] = T(0);
    ud[k] = T(0);
  }
  for (int i = 0; i < n_null(); ++i) {
    const NullK<T, N> &Z = O.nul[i];
    if (Z.kind == kNullDamping) {
      ABRB_UNROLL
      for (int k = 0; k < N; ++k) wn[k] -= Z.kv * dq[k];
    } else if (Z.kind == kNullResting) {
      ABRB_UNROLL
      for (int k = 0; k < N; ++k) {
        const T qt = ((Z.rest_mask >> k) & 1u) ? wrap_pm_pi(Z.rest[k] - q[k]) : T(0);
        wn[k] += Z.kp * qt - Z.kv * dq[k];
      }
    } else if (Z.kind == kNullLimits) {
      T ul[N];
      joint_limits_generate<T, N>(Z, q, ul);
      ABRB_UNROLL
      for (int k = 0; k < N; ++k) ud[k] += ul[k];
    } else {
      any_avoid = true;
    }
  }
  // velocity compensation (osc.py:275-282): joint space if the target velocity is all zero
  bool tv_zero = true;
  if (tv != nullptr) {
    ABRB_UNROLL
    for (int c = 0; c < 6; ++c) tv_zero = tv_zero && (tv[c] == T(0));
  }
  ABRB_UNROLL
  for (int a = 0; a < N; ++a) {
    T s1 = T(0), s2 = T(0);
    ABRB_UNROLL
    for (int b = 0; b < N; ++b) {
      s1 += M[a][b] * dq[b];
      s2 += M[a][b] * wn[b];
    }
    u[a] = tv_zero ? -O.kv * s1 : T(0);
    un[a] = s2 + ud[a];
  }

  K.sync();
  // ---- task Jacobian rows of the controlled DOF written in place over t_k / z_k (osc.py:242-244):
  //      Uncontrolled rows are zero.
  T xdot[KD];
  ABRB_UNROLL
  for (int r = 0; r < KD; ++r) xdot[r] = T(0);
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    T tk[3], zk[3], d[3], v[3];
    K.t(k, tk);
    K.z(k, zk);
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) d[c] = pF[c] - tk[c];
    omega_apply(K, k, d, v);
    const bool on = k < dep;
    ABRB_UNROLL
    for (int r = 0; r < KD; ++r) {
      const T val = (on && ((dof_mask() >> r) & 1u)) ? (r < 3 ? v[r < 3 ? r : 0] : zk[r < 3 ? 0 : r - 3]) : T(0);
      K.s.st(Aslot(r, k), val);
      xdot[r] += val * dq[k];
    }
  }
  if (!tv_zero) {
    ABRB_UNROLL
    for (int r = 0; r < KD; ++r) err[r] += O.kv * (xdot[r] - tv[r]);
  }
  ABRB_UNROLL
  for (int r = 0; r < KD; ++r) y[r] = ((dof_mask() >> r) & 1u) ? err[r] : T(0);

  K.sync();
  // ---- M = L L^T   (osc.py:136)
  chol<T, N>(M, Mi);
  // ---- secondary controllers that go through the null-space filter  I - J^T Mx J M^-1  (osc.py:310-318): their
  //      task-space image z = J M^-1 u_null = A (L^-1 u_null) is formed so that Mx is applied to y and z in ONE place
  //      (the truncating route decomposes once for both right-hand sides).  w = L^-1 u_null is taken here, while L is
  //      at hand; z itself falls out of the S loop below.
  T w[N];
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) w[k] = T(0);
  if (any_null) {
    if (any_avoid) {
      T Lf[N * N];
      ABRB_UNROLL
      for (int a = 0; a < N; ++a)
        ABRB_UNROLL
      for (int b = 0; b < N; ++b) Lf[a * N + b] = M[a][b];
      for (int i = 0; i < n_null(); ++i) {
        if (O.nul[i].kind == kNullAvoid) {
          T ua[N], qa[N];  // private copies: only these (not the caller's register arrays) have their address taken
          ABRB_UNROLL
          for (int k = 0; k < N; ++k) qa[k] = q[k];
          avoid_generate<T, N, ORTHO>(P, O.nul[i], qa, Lf, ua);
          ABRB_UNROLL
          for (int k = 0; k < N; ++k) un[k] += ua[k];
        }
      }
    }
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) w[k] = un[k];
    fwd_solve<T, N>(M, Mi, w);  // L^-1 u_null
  }
  // ---- A <- rows of (L^-1 J^T)^T   (in place over J)
  ABRB_UNROLL
  for (int r = 0; r < KD; ++r) {
    T row[N];
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) row[k] = K.s.ld(Aslot(r, k));
    fwd_solve<T, N>(M, Mi, row);
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) K.s.st(Aslot(r, k), row[k]);
  }
  // ---- nothing below needs 1/diag(L), g, C dq until the task-space solve is done: with the scratch in
  //      shared memory they are parked there (slots that are free by now) instead of being carried in registers across
  //      the 6x6 factorisation, where the register allocator would otherwise spill them to local memory
  typedef typename K_::S SL;
  constexpr bool PARK = K_::kSharedScratch;
  if (PARK) {
    ABRB_UNROLL
    for (int a = 0; a < N; ++a) {
      K.s.st(SL::kPl + a, Mi[a]);
      K.s.st(SL::kPl + N + a, g[a]);
      K.s.st(SL::kPl + 2 * N + a, (PLANT || PLAIN || O.use_C) ? cdq[a] : T(0));
    }
  }
  // ---- S = J M^-1 J^T = A A^T (osc.py:137), built straight into the array that is then factorised in place; z = A w
  T Sc[KD][KD], Si[KD];
  ABRB_UNROLL
  for (int a = 0; a < KD; ++a) {
    T ra[N];
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) ra[k] = K.s.ld(Aslot(a, k));
    T za = T(0);
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) za += ra[k] * w[k];
    z[a] = (!PLAIN && ((dof_mask() >> a) & 1u)) ? za : T(0);  // (PLAIN: w = 0, and z is read only with any_null)
    ABRB_UNROLL
    for (int b = 0; b < KD; ++b) {
      if (b <= a) {
        T s = T(0);
        ABRB_UNROLL
        for (int k = 0; k < N; ++k) s += ra[k] * K.s.ld(Aslot(b, k));
        const bool on = ((dof_mask() >> a) & 1u) && ((dof_mask() >> b) & 1u);
        Sc[a][b] = on ? s : (a == b ? T(1) : T(0));
        Sc[b][a] = Sc[a][b];
      }
    }
  }
  // ---- Mx: inverse if |det| >= threshold else pinv(rcond = threshold*0.1)   (osc.py:138-145)
  const bool pd = chol<T, KD>(Sc, Si);
  T det = T(1);
  ABRB_UNROLL
  for (int a = 0; a < KD; ++a) det *= Sc[a][a] * Sc[a][a];
  bool fast = pd && (det >= O.thr);
  if (pd && !fast) {
    // pinv == inv whenever no eigenvalue is truncated; certify that cheaply before sending the state down the
    // truncating route:  lambda_max <= trace(S_active) and 1/lambda_min <= ||S^-1||_F, so nothing is truncated if
    // rcond * trace * ||S^-1||_F < 1.  (S^-1)_aa >= 1/L_aa^2 bounds ||S^-1||_F from below with values already at hand:
    // when that bound alone breaks the inequality (every UR5 6-DOF state that gets here) the solves are skipped.
    T tr = T(0), big = T(0);
    ABRB_UNROLL
    for (int a = 0; a < KD; ++a) {
      if ((dof_mask() >> a) & 1u) {
        T saa = T(0);  // S_aa = sum_k L_ak^2
        ABRB_UNROLL
        for (int b = 0; b < KD; ++b)
          if (b <= a) saa += Sc[a][b] * Sc[a][b];
        tr += saa;
        big = Si[a] * Si[a] > big ? Si[a] * Si[a] : big;
      }
    }
    if (rcond * tr * big < T(1)) {
      T fro = T(0);
      ABRB_UNROLL
      for (int a = 0; a < KD; ++a) {
        if ((dof_mask() >> a) & 1u) {
          T e[KD];
          ABRB_UNROLL
          for (int b = 0; b < KD; ++b) e[b] = b == a ? T(1) : T(0);
          fwd_solve<T, KD>(Sc, Si, e);
          bwd_solve<T, KD>(Sc, Si, e);
          ABRB_UNROLL
          for (int b = 0; b < KD; ++b) fro += e[b] * e[b];
        }
      }
      fast = rcond * tr * sqrt_t(fro) < T(1);
    }
  }
  // y <- Mx y,  z <- Mx z: two triangular solves in the regular case ...
  if (fast) {
    fwd_solve<T, KD>(Sc, Si, y);
    bwd_solve<T, KD>(Sc, Si, y);
    if (any_null) {
      fwd_solve<T, KD>(Sc, Si, z);
      bwd_solve<T, KD>(Sc, Si, z);
    }
  }
  // ... and the truncating pseudo-inverse otherwise (always in double: the matrices that end up here have eigenvalue
  // ratios down to 1e-16).  When nothing is below the cut-off it returns S^-1 y itself, as numpy's pinv does.
  // wy = A^T Mx y, wz = A^T Mx z  (J^T x = L (A^T x), osc.py:285-288): from the solved y, z in the regular case; for the
  // states on the truncating route the cooperative step provides them directly (zero if the state was deferred: the
  // CTA's flush then adds the task-space term to the stored row)
  T wy[N], wz[N];
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    T sy = T(0), sz = T(0);
    ABRB_UNROLL
    for (int r = 0; r < KD; ++r) {
      const T ark = K.s.ld(Aslot(r, k));
      sy += ark * y[r];
      sz += ark * z[r];
    }
    wy[k] = sy;
    wz[k] = sz;
  }
  coop.template pinv<T, N, KD>(!fast, K, [&](int a, int b) { return M[a][b]; }, y, z, wy, wz, any_null, double(rcond));
  if (PARK) {
    ABRB_UNROLL
    for (int a = 0; a < N; ++a) {
      Mi[a] = K.s.ld(SL::kPl + a);
      g[a] = K.s.ld(SL::kPl + N + a);
      cdq[a] = K.s.ld(SL::kPl + 2 * N + a);
    }
  }

  auto L_apply = [&](const T *w, T *out) {
    ABRB_UNROLL
    for (int i = 0; i < N; ++i) {
      T s = T(0);
      ABRB_UNROLL
      for (int k = 0; k < N; ++k)
        if (k <= i) s += M[i][k] * w[k];
      out[i] = s;
    }
  };
  {
    T jt[N];
    L_apply(wy, jt);
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) u[k] -= jt[k];
  }
  if (PLAIN || O.use_C) {
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) u[k] -= cdq[k];
  }
  if (train != nullptr) {
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) train[k] = u[k];  // osc.py:297
  }
  if (PLAIN || O.use_g) {
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) u[k] -= g[k];
  }
  // ---- secondary controllers, filtered:  u += u_null - J^T Mx J M^-1 u_null   (osc.py:310-318)
  if (any_null) {
    T jt[N];
    L_apply(wz, jt);
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) u[k] += un[k] - jt[k];
  }
  if (PLANT) {
    T rhs[N];
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) rhs[k] = u[k] + g[k] - cdq[k];
    fwd_solve<T, N>(M, Mi, rhs);
    bwd_solve<T, N>(M, Mi, rhs);
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) ddq[k] = rhs[k];
  }
}

template <typename T, int N, int KD, bool PLANT, bool PLAIN = false, class K_>
ABRB_HD void osc_state(const ChainK<T, N> &P, const OscK<T, N> &O, const T *q, const T *dq, const T *target,
                       const T *tv, T *ierr, T *u, T *train, T *ddq, K_ &K) {
  SeqCoop seq;
  osc_eval<T, N, KD, PLANT, PLAIN>(P, O, q, dq, target, tv, ierr, u, train, ddq, K, seq);
}

// Row t of trajectory b of a path (or path velocity) of abrb_osc_rollout_path_*: (steps, B, 6) when stride == 6, one
// (steps, 6) path for every trajectory when stride == 0.
template <typename T>
ABRB_HD const T *path_row(const T *path, int stride, int t, int64_t B, int64_t b) {
  return path + (stride != 0 ? ((int64_t)t * B + b) * 6 : (int64_t)t * 6);
}

// One step of the closed-loop rollouts (rollout_kernel, fixed target and path):
//     u = OSC(q, dq, target, tv);  ddq = M^-1 (u + g - C dq);  dq += ddq dt;  q += dq dt
// (semi-implicit Euler).  PATH: also `x` = the control point at the state BEFORE the update, and
//     cost += |x - target[:3]|^2 + effort |u|^2.
template <typename T, int N, int KD, bool PLAIN, bool PATH, class K_, class Coop>
ABRB_HD void rollout_step(const ChainK<T, N> &P, const OscK<T, N> &O, T *q, T *dq, const T *target, const T *tv,
                          T *ierr, T dt, T effort, T *u, T *x, T &cost, K_ &K, Coop &coop) {
  T acc[N];
  osc_eval<T, N, KD, true, PLAIN>(P, O, q, dq, target, tv, ierr, u, (T *)nullptr, acc, K, coop, PATH ? x : (T *)nullptr);
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    dq[k] += acc[k] * dt;
    q[k] += dq[k] * dt;
  }
  if (PATH) {
    T ex = T(0), eu = T(0);
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) {
      const T d = x[c] - target[c];
      ex += d * d;
    }
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) eu += u[k] * u[k];
    cost += ex + effort * eu;
  }
}

// Standalone secondary controller (`Damping/RestingConfig/AvoidObstacles.generate`)
template <typename T, int N, class K_>
ABRB_HD void null_state(const ChainK<T, N> &P, const NullK<T, N> &Z, const T *q, const T *dq, T *u, K_ &K) {
  constexpr bool ORTHO = K_::kOrtho;
  if (Z.kind == kNullLimits) {
    joint_limits_generate<T, N>(Z, q, u);
    return;
  }
  walk<T, N>(P, q, 0, K);
  T M[N][N], g[N];
  dynamics_Mg<T, N, false>(P, K, dq, M, g, nullptr);
  ABRB_UNROLL
  for (int a = 0; a < N; ++a)
    ABRB_UNROLL
  for (int b = 0; b < N; ++b)
    if (b < a) M[a][b] = M[b][a];
  if (Z.kind == kNullAvoid) {
    T Mi[N];
    chol<T, N>(M, Mi);
    T Lf[N * N];
    ABRB_UNROLL
    for (int a = 0; a < N; ++a)
      ABRB_UNROLL
    for (int b = 0; b < N; ++b) Lf[a * N + b] = M[a][b];
    T ua[N], qa[N];
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) qa[k] = q[k];
    avoid_generate<T, N, ORTHO>(P, Z, qa, Lf, ua);
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) u[k] = ua[k];
    return;
  }
  T w[N];
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    if (Z.kind == kNullDamping) {
      w[k] = -Z.kv * dq[k];
    } else {
      const T qt = ((Z.rest_mask >> k) & 1u) ? wrap_pm_pi(Z.rest[k] - q[k]) : T(0);
      w[k] = Z.kp * qt - Z.kv * dq[k];
    }
  }
  ABRB_UNROLL
  for (int a = 0; a < N; ++a) {
    T s = T(0);
    ABRB_UNROLL
    for (int b = 0; b < N; ++b) s += M[a][b] * w[b];
    u[a] = s;
  }
}

// The tail of joint_state once the walk of q is in K: M, g and the torque
template <typename T, int N, class K_>
ABRB_HD void joint_torque(const ChainK<T, N> &P, T kp, T kv, bool gravity, const T *q, const T *dq, const T *target,
                          const T *tv, T *u, K_ &K) {
  T M[N][N], g[N];
  dynamics_Mg<T, N, false>(P, K, dq, M, g, nullptr);
  T w[N];
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) w[k] = kp * wrap_pm_pi(target[k] - q[k]) + kv * ((tv != nullptr ? tv[k] : T(0)) - dq[k]);
  ABRB_UNROLL
  for (int a = 0; a < N; ++a) {
    T s = T(0);
    ABRB_UNROLL
    for (int b = 0; b < N; ++b) s += (b >= a ? M[a][b] : M[b][a]) * w[b];
    u[a] = gravity ? s - g[a] : s;
  }
}

// Joint.generate (controllers/joint.py:104-131)
template <typename T, int N, class K_>
ABRB_HD void joint_state(const ChainK<T, N> &P, T kp, T kv, bool gravity, const T *q, const T *dq, const T *target,
                         const T *tv, T *u, K_ &K) {
  walk<T, N>(P, q, 0, K);
  joint_torque<T, N>(P, kp, kv, gravity, q, dq, target, tv, u, K);
}

// Floating.generate (controllers/floating.py:27-71)
template <typename T, int N, class K_>
ABRB_HD void floating_state(const ChainK<T, N> &P, bool task_space, bool dynamic, const T *q, const T *dq, T *u,
                            K_ &K) {
  constexpr bool ORTHO = K_::kOrtho;
  walk<T, N>(P, q, 2 * N + 1, K);
  T M[N][N], g[N];
  dynamics_Mg<T, N, false>(P, K, dq, M, g, nullptr);
  ABRB_UNROLL
  for (int a = 0; a < N; ++a)
    ABRB_UNROLL
  for (int b = 0; b < N; ++b)
    if (b < a) M[a][b] = M[b][a];
  T Mdq[N];
  ABRB_UNROLL
  for (int a = 0; a < N; ++a) {
    T s = T(0);
    ABRB_UNROLL
    for (int b = 0; b < N; ++b) s += M[a][b] * dq[b];
    Mdq[a] = s;
  }
  if (!task_space) {
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) u[k] = -g[k] - (dynamic ? Mdq[k] : T(0));
    return;
  }
  // J = J("EE")[:3];  A = (L^-1 J^T)^T;  S = J M^-1 J^T;  u = J^T (-Mx^T J M^-1 g) = -L A^T Mx A (L^-1 g)
  T pF[3] = {K.F[3], K.F[7], K.F[11]};
  T J[6][N];
  jacobian<T, N>(K, pF, N, J);
  T Mi[N];
  chol<T, N>(M, Mi);
  T A[3][N];
  ABRB_UNROLL
  for (int r = 0; r < 3; ++r) {
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) A[r][k] = J[r][k];
    fwd_solve<T, N>(M, Mi, A[r]);
  }
  T S[3][3], Sc[3][3], Si[3];
  ABRB_UNROLL
  for (int a = 0; a < 3; ++a)
    ABRB_UNROLL
  for (int b = 0; b < 3; ++b) {
    T s = T(0);
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) s += A[a][k] * A[b][k];
    S[a][b] = s;
    Sc[a][b] = s;
  }
  const bool pd = chol<T, 3>(Sc, Si);
  T det = T(1);
  ABRB_UNROLL
  for (int a = 0; a < 3; ++a) det *= Sc[a][a] * Sc[a][a];
  T w[N], z[3];
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) w[k] = g[k];
  fwd_solve<T, N>(M, Mi, w);
  ABRB_UNROLL
  for (int r = 0; r < 3; ++r) {
    T s = T(0);
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) s += A[r][k] * w[k];
    z[r] = s;
  }
  if (pd && det > T(1e-3)) {  // note the strict '>' of floating.py:52 (osc.py uses '>=')
    fwd_solve<T, 3>(Sc, Si, z);
    bwd_solve<T, 3>(Sc, Si, z);
  } else {
    T Sf[9], zi[3], zo[3];
    ABRB_UNROLL
    for (int a = 0; a < 3; ++a) {
      zi[a] = z[a];
      ABRB_UNROLL
      for (int b = 0; b < 3; ++b) Sf[a * 3 + b] = S[a][b];
    }
    pinv_apply_sym<T, 3>(Sf, 7u, T(1e-4), zi, zo);
    ABRB_UNROLL
    for (int a = 0; a < 3; ++a) z[a] = zo[a];
  }
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    T s = T(0);
    ABRB_UNROLL
    for (int r = 0; r < 3; ++r) s += A[r][k] * z[r];
    w[k] = s;
  }
  ABRB_UNROLL
  for (int i = 0; i < N; ++i) {
    T s = T(0);
    ABRB_UNROLL
    for (int k = 0; k < N; ++k)
      if (k <= i) s += M[i][k] * w[k];
    u[i] = -s - (dynamic ? Mdq[i] : T(0));
  }
  (void)ORTHO;
}

// Sliding.generate (controllers/sliding.py:34-99); pinv(J[:3]) through RowPinv3.
template <typename T, int N, class K_>
ABRB_HD void sliding_state(const ChainK<T, N> &P, T kd, T lamb, bool cartesian, int frame, const T *xoff, const T *q,
                           const T *dq, const T *target, const T *tv, const T *ta, T *u, T *s_out, K_ &K) {
  walk<T, N>(P, q, cartesian ? frame : 0, K);
  T dq_ref[N], ddq_ref[N];
  if (cartesian) {
    const int dep = frame_dep<N>(frame);
    T pF[3];
    frame_point(K.F, xoff, pF);
    T J[6][N], dJ[6][N];
    jacobian<T, N>(K, pF, dep, J);
    RowPinv3<T, N> Jp;
    Jp.build(J[0], J[1], J[2]);
    auto pinv_J = [&](const T *y, T *out) { Jp.apply(y, out); };
    T r1[3], r2[3];
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) r1[c] = (tv != nullptr ? tv[c] : T(0)) + lamb * (target[c] - pF[c]);
    pinv_J(r1, dq_ref);
    jacobian_dot<T, N>(K, J, dq, dep, dJ);
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) {
      T dx = T(0), dj = T(0);
      ABRB_UNROLL
      for (int k = 0; k < N; ++k) {
        dx += J[c][k] * dq[k];
        dj += dJ[c][k] * dq_ref[k];
      }
      r2[c] = (ta != nullptr ? ta[c] : T(0)) + lamb * ((tv != nullptr ? tv[c] : T(0)) - dx) - dj;
    }
    pinv_J(r2, ddq_ref);
  } else {
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) {
      const T tvk = tv != nullptr ? tv[k] : T(0);
      dq_ref[k] = tvk - lamb * (q[k] - target[k]);
      ddq_ref[k] = (ta != nullptr ? ta[k] : T(0)) - lamb * (dq[k] - tvk);
    }
  }
  T M[N][N], g[N], Cm[N][N];
  dynamics_Mg<T, N, false>(P, K, dq, M, g, nullptr);
  dynamics_C<T, N>(P, K, dq, Cm);
  ABRB_UNROLL
  for (int a = 0; a < N; ++a) {
    T acc = T(0);
    ABRB_UNROLL
    for (int b = 0; b < N; ++b) acc += (b >= a ? M[a][b] : M[b][a]) * ddq_ref[b] + Cm[a][b] * dq_ref[b];
    const T sa = dq[a] - dq_ref[a];
    if (s_out != nullptr) s_out[a] = sa;
    u[a] = acc + g[a] - kd * sa;
  }
}

// ------------------------------------------------------------------------------------------------ Joint / Sliding rollouts
// The closed-loop rollouts of the trajectory-tracking controllers other than OSC (ctrl_rollout_kernel): the controller
// (joint_state / sliding_state) and the plant (plant_step) as they are, one after the other, each with its own walk.
// KIND is compile-time because the two live sets differ widely (Sliding carries J, dJ, C and RowPinv3).
enum { kCtrlJoint = 0, kCtrlSliding = 1 };

template <typename T>
struct CtrlK {
  T kp, kv;       // Joint
  T kd, lamb;     // Sliding
  int gravity;    // Joint: account_for_gravity
  int cartesian;  // Sliding: task-space target (rows of 3) or joint-space target (rows of N)
};

// Width of the path rows of a ctrl rollout, and the length of the arrays they are loaded into (>= 3, so that a
// cartesian row fits whatever N is)
template <int N>
struct CtrlRow {
  static constexpr int kMax = N > 3 ? N : 3;
};

// Row t of trajectory b of one of a ctrl rollout's path arrays, addressed by torque_row<T, W> ((steps, B, W) for stride
// W, one (steps, W) row sequence for stride 0), copied into `out` and padded with zeros; nullptr gives a zero row.
template <typename T, int W, int LEN>
ABRB_HD void ctrl_row(const T *a, int stride, int t, int64_t B, int64_t b, T *out) {
  const T *r = a != nullptr ? torque_row<T, W>(a, stride, t, B, b) : nullptr;
  ABRB_UNROLL
  for (int k = 0; k < LEN; ++k) out[k] = (r != nullptr && k < W) ? r[k] : T(0);
}

// Path, path velocity and path acceleration rows of step t: width 3 for cartesian Sliding, N otherwise
template <typename T, int N, int KIND>
ABRB_HD void ctrl_path_rows(const T *path, int ps, const T *pv, int pvs, const T *pa, int pas, bool cartesian, int t,
                            int64_t B, int64_t b, T *tg, T *tv, T *ta) {
  constexpr int L = CtrlRow<N>::kMax;
  if (KIND == kCtrlSliding && cartesian) {
    ctrl_row<T, 3, L>(path, ps, t, B, b, tg);
    ctrl_row<T, 3, L>(pv, pvs, t, B, b, tv);
    ctrl_row<T, 3, L>(pa, pas, t, B, b, ta);
  } else {
    ctrl_row<T, N, L>(path, ps, t, B, b, tg);
    ctrl_row<T, N, L>(pv, pvs, t, B, b, tv);
    if (KIND == kCtrlSliding) ctrl_row<T, N, L>(pa, pas, t, B, b, ta);
  }
}

// One step of the Joint / Sliding rollouts, for the path rows `target`, `tv` and `ta` (tv, ta nullptr: zero):
//     u = Joint.generate(q, dq, target, tv)   or   Sliding.generate(q, dq, target, tv, ta, frame, xoff)
//     x = control point (frame + xoff) at q;  ddq = M^-1 (u + g - C dq);  dq += ddq dt;  q += dq dt
//     cost += e + effort |u|^2,  e = |wrap(target - q)|^2 (Joint), |x - target|^2 (cartesian Sliding),
//                                    |q - target|^2 (joint-mode Sliding: not wrapped, as in the reference)
// `u`, `x` and e belong to the state BEFORE the update, as in rollout_step and plant_step.
template <typename T, int N, int KIND, class K_>
ABRB_HD void ctrl_rollout_step(const ChainK<T, N> &P, const CtrlK<T> &G, int frame, const T *xoff, T *q, T *dq,
                               const T *target, const T *tv, const T *ta, T dt, T effort, T *u, T *x, T &cost,
                               K_ &K) {
  K.sync();
  if (KIND == kCtrlJoint)
    joint_state<T, N>(P, G.kp, G.kv, G.gravity != 0, q, dq, target, tv, u, K);
  else
    sliding_state<T, N>(P, G.kd, G.lamb, G.cartesian != 0, frame, xoff, q, dq, target, tv, ta, u, (T *)nullptr, K);
  const bool task = KIND == kCtrlSliding && G.cartesian != 0;
  T e = T(0);
  if (!task) {
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) {
      const T d = KIND == kCtrlJoint ? wrap_pm_pi(target[k] - q[k]) : q[k] - target[k];
      e += d * d;
    }
  }
  T tau[N];
  plant_step<T, N>(P, frame, xoff, q, dq, u, false, (const T *)nullptr, dt, effort, tau, x, cost, K);
  if (task) {
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) {
      const T d = x[c] - target[c];
      e += d * d;
    }
  }
  cost += e;
}

// One iteration of InverseKinematics.generate_path (controllers/path_planners/inverse_kinematics.py:83-137): the joint
// step dq towards the task-space target from the current q.  `Qd`: unit target quaternion (the reference builds it
// with axes="sxyz" whatever `axes` it was given, :72-81).  max_dx / max_dr / max_dq are already multiplied by dt.
//   method 1: dq = pinv(J) [dx, dr];   2: dq = J^T (J J^T + 0.001 I)^-1 [dx, 0.3 dr];
//   method 3: dq = pinv(Jx) dx + (I - pinv(Jx) Jx) pinv(Jr) dr      (Jx = J[:3], Jr = J[3:])
template <typename T, int N, class K_>
ABRB_HD void ik_step(const ChainK<T, N> &P, T max_dx, T max_dr, T max_dq, int method, const T *q, const T *target,
                     const T *Qd, T *dq, K_ &K) {
  walk<T, N>(P, q, 2 * N + 1, K);
  T pF[3] = {K.F[3], K.F[7], K.F[11]};
  T J[6][N];
  jacobian<T, N>(K, pF, N, J);
  T R[9], Qe[4];
  ABRB_UNROLL
  for (int r = 0; r < 3; ++r)
    ABRB_UNROLL
  for (int c = 0; c < 3; ++c) R[r * 3 + c] = K.F[r * 4 + c];
  quat_from_R(R, Qe);
  T dx[3], dr[3];
  ABRB_UNROLL
  for (int c = 0; c < 3; ++c) dx[c] = target[c] - pF[c];
  // dr = Qe[0] Qd[1:] - Qd[0] Qe[1:] - Qd[1:] x Qe[1:]   (:93)
  T cr[3];
  cross3(Qd + 1, Qe + 1, cr);
  ABRB_UNROLL
  for (int c = 0; c < 3; ++c) dr[c] = Qe[0] * Qd[1 + c] - Qd[0] * Qe[1 + c] - cr[c];
  const T ndx = sqrt_t(dx[0] * dx[0] + dx[1] * dx[1] + dx[2] * dx[2]);
  const T ndr = sqrt_t(dr[0] * dr[0] + dr[1] * dr[1] + dr[2] * dr[2]);
  if (ndx > max_dx) {
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) dx[c] = dx[c] / ndx * max_dx;
  }
  if (ndr > max_dr) {
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) dr[c] = dr[c] / ndr * max_dr;
  }
  if (method == 1) {
    T Af[6 * N], yf[6], of[N];  // private copies: the out-of-line routine takes addresses
    ABRB_UNROLL
    for (int r = 0; r < 6; ++r) {
      yf[r] = r < 3 ? dx[r < 3 ? r : 0] : dr[r < 3 ? 0 : r - 3];
      ABRB_UNROLL
      for (int k = 0; k < N; ++k) Af[r * N + k] = J[r][k];
    }
    pinv_rows_apply<T, 6, N>(Af, yf, of);
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) dq[k] = of[k];
  } else if (method == 2) {
    T S[6][6], Si[6], y[6];
    ABRB_UNROLL
    for (int a = 0; a < 6; ++a) {
      y[a] = a < 3 ? dx[a < 3 ? a : 0] : T(0.3) * dr[a < 3 ? 0 : a - 3];
      ABRB_UNROLL
      for (int b = 0; b < 6; ++b) {
        T acc = a == b ? T(0.001) : T(0);
        ABRB_UNROLL
        for (int k = 0; k < N; ++k) acc += J[a][k] * J[b][k];
        S[a][b] = acc;
      }
    }
    chol<T, 6>(S, Si);  // J J^T + 0.001 I is positive definite
    fwd_solve<T, 6>(S, Si, y);
    bwd_solve<T, 6>(S, Si, y);
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) {
      T acc = T(0);
      ABRB_UNROLL
      for (int a = 0; a < 6; ++a) acc += J[a][k] * y[a];
      dq[k] = acc;
    }
  } else {
    RowPinv3<T, N> Px, Pr;
    Px.build(J[0], J[1], J[2]);
    Pr.build(J[3], J[4], J[5]);
    T a[N], w[N], jw[3], pw[N];
    Px.apply(dx, a);
    Pr.apply(dr, w);
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) {
      T acc = T(0);
      ABRB_UNROLL
      for (int k = 0; k < N; ++k) acc += J[c][k] * w[k];
      jw[c] = acc;
    }
    Px.apply(jw, pw);
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) dq[k] = a[k] + w[k] - pw[k];
  }
  T big = T(0);
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) big = abs_t(dq[k]) > big ? abs_t(dq[k]) : big;
  if (big > max_dq) {
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) dq[k] = dq[k] / big * max_dq;
  }
}

}  // namespace abrb
