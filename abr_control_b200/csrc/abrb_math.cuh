// abrb_math.cuh — per-state arithmetic of the batched arm engine (one joint state per thread).
//
// Everything here is a template over the scalar type T (float / double), the joint count N and
// ORTHO (all constant frames orthonormal -> joint-axis operators reduce to cross products).
// The functions are __host__ __device__ so the very same code can be instantiated by g++ for the
// CPU-side unit tests in tests/hostsim (test infrastructure only: the shipped library launches them
// exclusively from CUDA kernels, see kernels.cu).
//
// Formulation (DESIGN.md S3).  The reference differentiates symbolic products of 4x4 factors
// (/root/reference/abr_control/arms/base_config.py:559-563, :504-507, :706-714).  Here the same exact
// derivatives are obtained from per-joint operators.  For joint k let R_k, t_k be the rotation block and
// origin of frame "joint k" (before its own rotation) and
//        Omega_k = R_k E R_k^-1,   E = [[0,-1,0],[1,0,0],[0,0,0]]
// (for an orthonormal R_k, Omega_k v = z_k x v).  For any point p rigidly attached downstream of joint k:
//        dp/dq_k          = Omega_k (p - t_k)
//        d2p/dq_i dq_k    = Omega_min(i,k) dp/dq_max(i,k)
//        dz_a/dq_i        = Omega_i z_a   (i < a),  0 otherwise
// which holds for non-orthonormal constant frames too (Jaco2, SURVEY.md S0.4) because Omega_k commutes
// with the joint's own rotation.  M, g, C then follow the reference's definitions
// (base_config.py:625-632, :448-455, :706-714) with the diagonal link inertias left un-rotated.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define ABRB_HD __host__ __device__ __forceinline__
#define ABRB_HD_NOINLINE __host__ __device__ __noinline__
#define ABRB_UNROLL _Pragma("unroll")
#define ABRB_NOUNROLL _Pragma("unroll 1")
#else
#define ABRB_HD inline
#define ABRB_HD_NOINLINE __attribute__((noinline))
#define ABRB_UNROLL
#define ABRB_NOUNROLL
#endif

namespace abrb {

constexpr int kMaxJoints = 7;
constexpr int kMaxNull = 4;
constexpr int kMaxObstacles = 16;
constexpr int kMaxPeers = 8;  // GPUs of one box (fused all-gather of the control outputs)

// sin and cos of a joint angle in double.  The CUDA library routine is ~115 executed instructions per call with a
// Payne-Hanek slow path inlined at each of the nine call sites of an OSC evaluation (1.9 k static instructions, 12 % of
// the executed ones, in kernels that stall on instruction fetch).  Joint angles are small numbers, so on the device:
// three-term Cody-Waite reduction by pi/2 (exact products through FMA; |x| < 1024, beyond that — and for NaN — one
// shared out-of-line call of the library routine) and the classic degree-13 / degree-14 kernel polynomials on
// [-pi/4, pi/4]; measured against long-double references over [0, 2 pi) and [-50, 50]: <= 1.5 ulp.
#ifdef __CUDA_ARCH__
__device__ __noinline__ void sincos_cold(double x, double *s, double *c) { ::sincos(x, s, c); }
__device__ __forceinline__ void sincos_t(double x, double *s, double *c) {
  if (!(::fabs(x) < 1024.0)) {
    sincos_cold(x, s, c);
    return;
  }
  const double k = ::rint(x * 0.63661977236758138);  // 2 / pi
  double r = ::fma(-k, 1.5707963267948966, x);        // pi/2 = hi + mid + lo
  r = ::fma(-k, 6.123233995736766e-17, r);
  r = ::fma(-k, -1.4973849048591698e-33, r);
  const double z = r * r;
  double ps = 1.58969099521155010221e-10;
  ps = ::fma(ps, z, -2.50507602534068634195e-08);
  ps = ::fma(ps, z, 2.75573137070700676789e-06);
  ps = ::fma(ps, z, -1.98412698298579493134e-04);
  ps = ::fma(ps, z, 8.33333333332248946124e-03);
  ps = ::fma(ps, z, -1.66666666666666324348e-01);
  const double sn = ::fma(r * z, ps, r);
  double pc = -1.13596475577881948265e-11;
  pc = ::fma(pc, z, 2.08757232129817482790e-09);
  pc = ::fma(pc, z, -2.75573143513906633035e-07);
  pc = ::fma(pc, z, 2.48015872894767294178e-05);
  pc = ::fma(pc, z, -1.38888888888741095749e-03);
  pc = ::fma(pc, z, 4.16666666666666019037e-02);
  const double cs = ::fma(z * z, pc, ::fma(-0.5, z, 1.0));
  const int n = (int)k;
  const double a = (n & 1) ? cs : sn, b = (n & 1) ? sn : cs;
  *s = (n & 2) ? -a : a;
  *c = ((n + 1) & 2) ? -b : b;
}
#else
ABRB_HD void sincos_t(double x, double *s, double *c) { ::sincos(x, s, c); }
#endif
ABRB_HD void sincos_t(float x, float *s, float *c) { ::sincosf(x, s, c); }
ABRB_HD double sqrt_t(double x) { return ::sqrt(x); }
ABRB_HD float sqrt_t(float x) { return ::sqrtf(x); }
// Reciprocal and reciprocal square root of the pivots and norms of the small factorisations: the hardware seed
// (rcp / rsqrt.approx.ftz.f64, ~23 bits) refined by two Newton steps to ~1 ulp — the IEEE double division / square root
// are ~30-instruction dependent sequences each, and these kernels are bound by exactly such chains.  Operands are far
// from the subnormal range.
ABRB_HD float inv_t(float x) { return 1.0f / x; }
ABRB_HD float inv_sqrt_t(float x) { return 1.0f / ::sqrtf(x); }
ABRB_HD double inv_t(double x) {
  double r;
#ifdef __CUDA_ARCH__
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
#else
  const double ax = ::fabs(x);
  if (!(ax > 1e-30 && ax < 1e30)) return 1.0 / x;
  r = (double)(1.0f / (float)x);  // host stand-in for the hardware seed (tests/hostsim)
#endif
  r = ::fma(r, ::fma(-x, r, 1.0), r);
  return ::fma(r, ::fma(-x, r, 1.0), r);
}
ABRB_HD double inv_sqrt_t(double x) {
  double y;
#ifdef __CUDA_ARCH__
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
#else
  if (!(x > 1e-30 && x < 1e30)) return 1.0 / ::sqrt(x);
  y = (double)(1.0f / ::sqrtf((float)x));
#endif
  const double hx = 0.5 * x;
  y = ::fma(y, ::fma(-hx * y, y, 0.5), y);
  return ::fma(y, ::fma(-hx * y, y, 0.5), y);
}
// 1 / sqrt(x) to ~2^-45: the hardware seed and ONE Newton step.  Only for the Jacobi rotations of the truncating
// pseudo-inverse, whose rounds are a pure dependent chain: a rotation whose (c, s) are off by 1e-13 is still applied
// identically to the row and to its row of V, and the iteration converges to the same decomposition (measured:
// 5e-13 instead of 4e-14 on the pseudo-inverse, against a 1e-9 parity tolerance; two steps buy nothing there).
ABRB_HD double inv_sqrt1_t(double x) {
  double y;
#ifdef __CUDA_ARCH__
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
#else
  if (!(x > 1e-30 && x < 1e30)) return 1.0 / ::sqrt(x);
  y = (double)(1.0f / ::sqrtf((float)x));
#endif
  return ::fma(y, ::fma(-0.5 * x * y, y, 0.5), y);
}
ABRB_HD double abs_t(double x) { return ::fabs(x); }
ABRB_HD float abs_t(float x) { return ::fabsf(x); }
ABRB_HD double fmod_t(double x, double y) { return ::fmod(x, y); }
ABRB_HD float fmod_t(float x, float y) { return ::fmodf(x, y); }
ABRB_HD double exp_t(double x) { return ::exp(x); }
ABRB_HD float exp_t(float x) { return ::expf(x); }
ABRB_HD double pow_t(double x, double y) { return ::pow(x, y); }
ABRB_HD float pow_t(float x, float y) { return ::powf(x, y); }

// ------------------------------------------------------------------------------------------------
// Chain constants in compute precision; passed to the kernels BY VALUE (kernel-parameter constant bank:
// every lane reads the same constant at the same time, so the constant cache broadcast is the right
// staging level — no shared-memory copy is needed for a one-state-per-thread mapping).
// Affine blocks are 3x4 row-major [R|t].
template <typename T, int N>
struct ChainK {
  T G0[12];          // world -> joint0 frame            (L0 . A_0)
  T L0[12];          // world -> link0 frame
  T Bf[N][12];       // rotated joint-i frame -> link(i+1) COM frame          (B_i)
  T BA[N][12];       // rotated joint-i frame -> joint(i+1) frame (B_i . A_{i+1}); BA[N-1] = B_{N-1} . E -> EE
  T Wp[N + 1][3];    // translational part of diag link inertia l
  T Wos[N][3];       // Wos[k] = sum_{l>k} rotational diag inertia of link l
  T gp[N + 1][3];    // Wp[l][c] * gravity[c]
  T gos[N][3];       // sum_{l>k} Wo[l][c] * gravity[3+c]
};

// frame ids: link l -> l (0..N), joint j -> N+1+j, EE -> 2N+1
template <int N>
ABRB_HD int frame_dep(int frame) {  // number of joints the frame moves with == reference `end_point`
  return frame <= N ? frame : (frame <= 2 * N ? frame - (N + 1) : N);
}

// Per-state kinematic scratch: joint origins t_k, joint axes z_k, link COMs and (non-orthonormal chains only)
// columns 0,1 of R_k and rows 0,1 of R_k^-1.  The values live in a "slot store": registers (RegStore) or a strided
// shared-memory column per thread (StridedStore, slot-major so consecutive lanes hit consecutive words), which is
// what the fp64 kernels use to keep register pressure, and so local-memory spills, down.
// Phase barrier of the CTA (`sync()`), called by the per-state code at points every thread of the CTA reaches.  The
// evaluations are ~10^4 straight-line instructions per state, far beyond the instruction caches, and instruction fetch
// is their top stall reason; a barrier at the phase boundaries keeps the warps of a CTA inside the same code window so
// that they share the fetched lines.  It pays for the long OSC and rollout kernels and costs the shorter rbd kernels,
// so the kernel decides (`psync`).
template <typename T, int COUNT>
struct RegStore {
  static constexpr bool kShared = false;
  T v[COUNT];
  bool psync = false;
  ABRB_HD T ld(int i) const { return v[i]; }
  ABRB_HD void st(int i, T x) { v[i] = x; }
  ABRB_HD void sync() const {
#ifdef __CUDA_ARCH__
    if (psync) __syncthreads();
#endif
  }
};
template <typename T, int COUNT>
struct StridedStore {
  static constexpr bool kShared = true;
  T *base;
  int stride;
  bool psync = false;
  ABRB_HD T ld(int i) const { return base[i * stride]; }
  ABRB_HD void st(int i, T x) { base[i * stride] = x; }
  ABRB_HD void sync() const {
#ifdef __CUDA_ARCH__
    if (psync) __syncthreads();
#endif
  }
};

template <int N, bool ORTHO>
struct KinSlots {
  static constexpr int kT = 0, kZ = 3 * N, kPl = 6 * N, kR0 = 9 * N, kR1 = 12 * N, kS0 = 15 * N, kS1 = 18 * N;
  // osc_eval parks 1/diag(L), g and C dq in the 3 N link-COM slots at kPl (free by then) while the task-space system is
  // solved.
  static constexpr int kCount = ORTHO ? 9 * N : 21 * N;
};

template <typename T, int N, bool ORTHO_, template <typename, int> class Store = RegStore>
struct Kin {
  typedef T Scalar;
  static constexpr int kN = N;
  static constexpr bool kOrtho = ORTHO_;
  typedef KinSlots<N, ORTHO_> S;
  static constexpr bool kSharedScratch = Store<T, S::kCount>::kShared;
  Store<T, S::kCount> s;
  T F[12];  // the requested frame
  ABRB_HD void ld3(int slot, T *o) const {
    o[0] = s.ld(slot);
    o[1] = s.ld(slot + 1);
    o[2] = s.ld(slot + 2);
  }
  ABRB_HD void st3(int slot, const T *v) {
    s.st(slot, v[0]);
    s.st(slot + 1, v[1]);
    s.st(slot + 2, v[2]);
  }
  ABRB_HD void sync() const { s.sync(); }
  // slot of element (r, k) of the task-space matrices that osc_eval writes over t_k / z_k (J, then A = (L^-1 J^T)^T)
  static ABRB_HD int aslot(int r, int k) { return r < 3 ? S::kT + 3 * k + r : S::kZ + 3 * k + (r - 3); }
  ABRB_HD void t(int k, T *o) const { ld3(S::kT + 3 * k, o); }
  ABRB_HD void z(int k, T *o) const { ld3(S::kZ + 3 * k, o); }
  ABRB_HD void pl(int l, T *o) const { ld3(S::kPl + 3 * l, o); }
};

template <typename T>
ABRB_HD void cross3(const T *a, const T *b, T *o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
template <typename T>
ABRB_HD T dot3(const T *a, const T *b) {
  return a[0] * b[0] + a[1] * b[1] + a[2] * b[2];
}

// out = X . C for two affine 3x4 blocks
template <typename T>
ABRB_HD void aff_mul(const T *X, const T *C, T *o) {
  ABRB_UNROLL
  for (int r = 0; r < 3; ++r) {
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c)
      o[r * 4 + c] = X[r * 4 + 0] * C[c] + X[r * 4 + 1] * C[4 + c] + X[r * 4 + 2] * C[8 + c];
    o[r * 4 + 3] = X[r * 4 + 0] * C[3] + X[r * 4 + 1] * C[7] + X[r * 4 + 2] * C[11] + X[r * 4 + 3];
  }
}

// Omega_k v
template <class K>
ABRB_HD void omega_apply(const K &kin, int k, const typename K::Scalar *v, typename K::Scalar *o) {
  typedef typename K::Scalar T;
  if (K::kOrtho) {
    T zk[3];
    kin.z(k, zk);
    cross3(zk, v, o);
  } else {
    T r0[3], r1[3], s0[3], s1[3];
    kin.ld3(K::S::kR0 + 3 * k, r0);
    kin.ld3(K::S::kR1 + 3 * k, r1);
    kin.ld3(K::S::kS0 + 3 * k, s0);
    kin.ld3(K::S::kS1 + 3 * k, s1);
    const T a = dot3(s0, v), b = dot3(s1, v);
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) o[c] = r1[c] * a - r0[c] * b;
  }
}

// Running sum  W_j = sum_{i<j} dq_i Omega_i  (angular-velocity operator seen by joint j)
template <typename T, bool ORTHO>
struct Spin {
  T w[ORTHO ? 3 : 9];
  ABRB_HD void clear() {
    ABRB_UNROLL
    for (int i = 0; i < (ORTHO ? 3 : 9); ++i) w[i] = T(0);
  }
  template <class K>
  ABRB_HD void add(const K &kin, int k, T dqk) {
    if (ORTHO) {
      T zk[3];
      kin.z(k, zk);
      ABRB_UNROLL
      for (int c = 0; c < 3; ++c) w[c] += dqk * zk[c];
    } else {
      T r0[3], r1[3], s0[3], s1[3];
      kin.ld3(K::S::kR0 + 3 * k, r0);
      kin.ld3(K::S::kR1 + 3 * k, r1);
      kin.ld3(K::S::kS0 + 3 * k, s0);
      kin.ld3(K::S::kS1 + 3 * k, s1);
      ABRB_UNROLL
      for (int r = 0; r < 3; ++r)
        ABRB_UNROLL
      for (int c = 0; c < 3; ++c) w[r * 3 + c] += dqk * (r1[r] * s0[c] - r0[r] * s1[c]);
    }
  }
  ABRB_HD void apply(const T *v, T *o) const {
    if (ORTHO) {
      cross3(w, v, o);
    } else {
      ABRB_UNROLL
      for (int r = 0; r < 3; ++r) o[r] = w[r * 3] * v[0] + w[r * 3 + 1] * v[1] + w[r * 3 + 2] * v[2];
    }
  }
};

// ------------------------------------------------------------------------------------------------
// Forward walk along the chain (SURVEY.md Appendix A.1): fills joint origins/axes, link COMs and the
// full transform of `frame`.
template <typename T, int N, class K>
ABRB_HD void walk(const ChainK<T, N> &P, const T *q, int frame, K &kin,
                  T (*link_frames)[12] = nullptr) {  // optional: all link(i+1) frames (rare paths only)
  T X[12];
  ABRB_UNROLL
  for (int i = 0; i < 12; ++i) X[i] = P.G0[i];
  if (frame == 0) {
    ABRB_UNROLL
    for (int i = 0; i < 12; ++i) kin.F[i] = P.L0[i];
  }
  ABRB_UNROLL
  for (int i = 0; i < N; ++i) {
    {
      const T tk[3] = {X[3], X[7], X[11]}, zk[3] = {X[2], X[6], X[10]};
      kin.st3(K::S::kT + 3 * i, tk);
      kin.st3(K::S::kZ + 3 * i, zk);
    }
    if (!K::kOrtho) {
      T c0[3], c1[3], c2[3], c12[3], c20[3];
      ABRB_UNROLL
      for (int r = 0; r < 3; ++r) {
        c0[r] = X[r * 4 + 0];
        c1[r] = X[r * 4 + 1];
        c2[r] = X[r * 4 + 2];
      }
      cross3(c1, c2, c12);
      cross3(c2, c0, c20);
      const T inv = T(1) / dot3(c0, c12);
      ABRB_UNROLL
      for (int r = 0; r < 3; ++r) {
        c12[r] *= inv;
        c20[r] *= inv;
      }
      kin.st3(K::S::kR0 + 3 * i, c0);
      kin.st3(K::S::kR1 + 3 * i, c1);
      kin.st3(K::S::kS0 + 3 * i, c12);
      kin.st3(K::S::kS1 + 3 * i, c20);
    }
    if (frame == N + 1 + i) {
      ABRB_UNROLL
      for (int j = 0; j < 12; ++j) kin.F[j] = X[j];
    }
    T s, c;
    sincos_t(q[i], &s, &c);
    ABRB_UNROLL
    for (int r = 0; r < 3; ++r) {
      const T a = X[r * 4 + 0], b = X[r * 4 + 1];
      X[r * 4 + 0] = c * a + s * b;
      X[r * 4 + 1] = c * b - s * a;
    }
    {
      T p[3];
      ABRB_UNROLL
      for (int r = 0; r < 3; ++r)
        p[r] = X[r * 4 + 0] * P.Bf[i][3] + X[r * 4 + 1] * P.Bf[i][7] + X[r * 4 + 2] * P.Bf[i][11] + X[r * 4 + 3];
      kin.st3(K::S::kPl + 3 * i, p);
    }
    if (frame == i + 1) aff_mul(X, P.Bf[i], kin.F);
    if (link_frames != nullptr) aff_mul(X, P.Bf[i], link_frames[i]);
    T Y[12];
    aff_mul(X, P.BA[i], Y);
    ABRB_UNROLL
    for (int j = 0; j < 12; ++j) X[j] = Y[j];
  }
  if (frame == 2 * N + 1) {
    ABRB_UNROLL
    for (int j = 0; j < 12; ++j) kin.F[j] = X[j];
  }
}

// point `x` of the requested frame in world coordinates  (reference Tx, base_config.py:371-392)
template <typename T>
ABRB_HD void frame_point(const T *F, const T *x, T *p) {
  ABRB_UNROLL
  for (int r = 0; r < 3; ++r) p[r] = F[r * 4 + 0] * x[0] + F[r * 4 + 1] * x[1] + F[r * 4 + 2] * x[2] + F[r * 4 + 3];
}

// J[6][N] of world point p attached to a frame that moves with the first `dep` joints
// (reference J, base_config.py:522-592: rows 0-2 dTx/dq_k, rows 3-5 J_orientation[k] for k < end_point)
template <typename T, int N, class K>
ABRB_HD void jacobian(const K &kin, const T *p, int dep, T (*J)[N]) {
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    T d[3], v[3], tk[3], zk[3];
    kin.t(k, tk);
    kin.z(k, zk);
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) d[c] = p[c] - tk[c];
    omega_apply(kin, k, d, v);
    const bool on = k < dep;
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) {
      J[c][k] = on ? v[c] : T(0);
      J[3 + c][k] = on ? zk[c] : T(0);
    }
  }
}

// dJ/dt = sum_i dJ/dq_i dq_i (reference dJ, base_config.py:470-520) given J's position rows
template <typename T, int N, class K_>
ABRB_HD void jacobian_dot(const K_ &K, const T (*J)[N], const T *dq, int dep, T (*dJ)[N]) {
  constexpr bool ORTHO = K_::kOrtho;
  // suffix sums s_k = sum_{k<=i<dep} dq_i v_i
  T suf[N][3];
  T run[3] = {T(0), T(0), T(0)};
  ABRB_UNROLL
  for (int k = N - 1; k >= 0; --k) {
    if (k < dep) {
      ABRB_UNROLL
      for (int c = 0; c < 3; ++c) run[c] += dq[k] * J[c][k];
    }
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) suf[k][c] = run[c];
  }
  Spin<T, ORTHO> W;
  W.clear();
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    T v[3] = {J[0][k], J[1][k], J[2][k]};
    T a[3], b[3], zd[3], zk[3];
    K.z(k, zk);
    W.apply(v, a);
    omega_apply(K, k, suf[k], b);
    W.apply(zk, zd);
    const bool on = k < dep;
    ABRB_UNROLL
    for (int c = 0; c < 3; ++c) {
      dJ[c][k] = on ? a[c] + b[c] : T(0);
      dJ[3 + c][k] = on ? zd[c] : T(0);
    }
    W.add(K, k, dq[k]);
  }
}

// ------------------------------------------------------------------------------------------------
// Joint-space dynamics, written for a small live set (one link at a time, only the link's Jacobian columns
// v_k = d p_l / d q_k are kept; everything else is accumulated on the fly).
//   M = sum_l J_l^T W_l J_l            base_config.py:625-632      (upper triangle a<=b is filled)
//   g = sum_l J_l^T W_l gravity        base_config.py:448-455
//   C[k][j] = sum_i 1/2 (d_i M_kj + d_j M_ki - d_k M_ij) dq_i     base_config.py:706-714
// Translational part of C:  sum_l v_lk . W_l (d/dt v_lj)  — the second derivatives of a point are symmetric, so
// the symmetric pieces of the Christoffel sum cancel exactly (DESIGN.md S3.3).  With
//   W_j = sum_{i<j} dq_i Omega_i,   suf_j = sum_{j<=i<l} dq_i v_li
// d/dt v_lj = W_j v_lj + Omega_j suf_j; walking j downwards needs only the running tail of both sums.
// Rotational part: explicit Christoffel sum over the derivative index (C matrix) or the product form (C dq).

// difference of two running operator sums applied to v:  (A - B) v
template <typename T, bool ORTHO>
ABRB_HD void spin_diff_apply(const Spin<T, ORTHO> &A, const Spin<T, ORTHO> &B, const T *v, T *o) {
  Spin<T, ORTHO> D;
  ABRB_UNROLL
  for (int i = 0; i < (ORTHO ? 3 : 9); ++i) D.w[i] = A.w[i] - B.w[i];
  D.apply(v, o);
}

// Jacobian columns of link l's COM: v[k] = Omega_k (p_l - t_k), k < l
template <typename T, int N, class K_>
ABRB_HD void link_columns(const K_ &K, int l, T (*v)[3]) {
  T pl[3];
  K.pl(l - 1, pl);
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) {
    if (k < l) {
      T d[3], tk[3];
      K.t(k, tk);
      ABRB_UNROLL
      for (int c = 0; c < 3; ++c) d[c] = pl[c] - tk[c];
      omega_apply(K, k, d, v[k]);
    }
  }
}

// rotational contributions to M, g (and C.dq)
template <typename T, int N, bool CDQ, class K_>
ABRB_HD void dynamics_Mg_rotational(const ChainK<T, N> &P, const K_ &K, const T *dq, T (*M)[N], T *g, T *cdq) {
  constexpr bool ORTHO = K_::kOrtho;
  // ---- rotational part: M_ab += sum_c z_a[c] Wos[max(a,b)][c] z_b[c]
  K.sync();
  T Z[N][3];
  ABRB_UNROLL
  for (int a = 0; a < N; ++a) K.z(a, Z[a]);
  ABRB_UNROLL
  for (int a = 0; a < N; ++a) {
    g[a] += dot3(Z[a], P.gos[a]);
    ABRB_UNROLL
    for (int b = a; b < N; ++b)
      M[a][b] += Z[a][0] * P.Wos[b][0] * Z[b][0] + Z[a][1] * P.Wos[b][1] * Z[b][1] + Z[a][2] * P.Wos[b][2] * Z[b][2];
  }
  if (CDQ) {
    // (C dq)_k = (dM/dt dq)_k - 1/2 d/dq_k (dq^T M dq), rotational part, with
    //   zd_a = W_a z_a,  hz_k = sum_j dq_j Wos[max(k,j)] o z_j,  hd_k = sum_j dq_j Wos[max(k,j)] o zd_j
    //   (dM/dt dq)_k = zd_k . hz_k + z_k . hd_k ;   1/2 d_k(..) = sum_{i>k} dq_i (Omega_k z_i) . hz_i
    T zd[N][3];
    Spin<T, ORTHO> W;
    W.clear();
    ABRB_UNROLL
    for (int a = 0; a < N; ++a) {
      W.apply(Z[a], zd[a]);
      W.add(K, a, dq[a]);
    }
    // hz_k = Wos[k] o (sum_{j<=k} dq_j z_j) + sum_{j>k} dq_j Wos[j] o z_j: a running prefix and a stored suffix instead of
    // the O(N^2) double loop (likewise hd with zd)
    T Qz[N][3], Qd[N][3];
    {
      T rz[3] = {T(0), T(0), T(0)}, rd[3] = {T(0), T(0), T(0)};
      ABRB_UNROLL
      for (int k = N - 1; k >= 0; --k) {
        ABRB_UNROLL
        for (int c = 0; c < 3; ++c) {
          Qz[k][c] = rz[c];
          Qd[k][c] = rd[c];
          rz[c] += dq[k] * P.Wos[k][c] * Z[k][c];
          rd[c] += dq[k] * P.Wos[k][c] * zd[k][c];
        }
      }
    }
    T Pz[3] = {T(0), T(0), T(0)}, Pd[3] = {T(0), T(0), T(0)};
    T hzs[N][3];
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) {
      T hd[3];
      ABRB_UNROLL
      for (int c = 0; c < 3; ++c) {
        Pz[c] += dq[k] * Z[k][c];
        Pd[c] += dq[k] * zd[k][c];
        hzs[k][c] = P.Wos[k][c] * Pz[c] + Qz[k][c];
        hd[c] = P.Wos[k][c] * Pd[c] + Qd[k][c];
      }
      cdq[k] += dot3(zd[k], hzs[k]) + dot3(Z[k], hd);
    }
    // -(1/2) d/dq_i terms: state i receives from every k > i:  - dq_k (Omega_i z_k) . hz_k
    if (ORTHO) {
      // (z_i x z_k) . hz_k = z_i . (z_k x hz_k): one cross product per k and a running suffix sum
      T acc[3] = {T(0), T(0), T(0)};
      ABRB_UNROLL
      for (int i = N - 2; i >= 0; --i) {
        T v[3];
        cross3(Z[i + 1], hzs[i + 1], v);
        ABRB_UNROLL
        for (int c = 0; c < 3; ++c) acc[c] += dq[i + 1] * v[c];
        cdq[i] -= dot3(Z[i], acc);
      }
    } else {
      ABRB_UNROLL
      for (int k = 0; k < N; ++k) {
        ABRB_UNROLL
        for (int i = 0; i < N; ++i) {
          if (i < k) {
            T oz[3];
            omega_apply(K, i, Z[k], oz);
            cdq[i] -= dq[k] * dot3(oz, hzs[k]);
          }
        }
      }
    }
  }
}

template <typename T, int N, class K_>
ABRB_HD void dynamics_C_rotational(const ChainK<T, N> &P, const K_ &K, const T *dq, T (*C)[N]) {
  // ---- rotational part, one derivative index d at a time.  With dz_a = Omega_d z_a (a > d, else 0) and
  //   D(a,b) = sum_c Wos[max(a,b)][c] (dz_a[c] z_b[c] + z_a[c] dz_b[c])   (= d M_ab / d q_d, symmetric)
  //   E_a    = sum_i dq_i D(a,i)
  // the Christoffel sum contributes  C[k][j] += 1/2 dq_d D(k,j),  C[k][d] += 1/2 E_k,  C[d][j] -= 1/2 E_j.
  T Z[N][3];
  ABRB_UNROLL
  for (int a = 0; a < N; ++a) K.z(a, Z[a]);
  ABRB_UNROLL
  for (int d = 0; d < N; ++d) {
    T dz[N][3], E[N];
    K.sync();
    ABRB_UNROLL
    for (int a = 0; a < N; ++a) {
      E[a] = T(0);
      if (a > d) {
        omega_apply(K, d, Z[a], dz[a]);
      } else {
        dz[a][0] = dz[a][1] = dz[a][2] = T(0);
      }
    }
    ABRB_UNROLL
    for (int a = 0; a < N; ++a) {
      ABRB_UNROLL
      for (int b = a; b < N; ++b) {
        if (b > d) {  // D(a,b) vanishes unless max(a,b) > d
          T Dab = T(0);
          ABRB_UNROLL
          for (int c = 0; c < 3; ++c) Dab += P.Wos[b][c] * (dz[a][c] * Z[b][c] + Z[a][c] * dz[b][c]);
          const T h = T(0.5) * dq[d] * Dab;
          C[a][b] += h;
          E[a] += dq[b] * Dab;
          if (b != a) {
            C[b][a] += h;
            E[b] += dq[a] * Dab;
          }
        }
      }
    }
    ABRB_UNROLL
    for (int k = 0; k < N; ++k) {
      C[k][d] += T(0.5) * E[k];
      C[d][k] -= T(0.5) * E[k];
    }
  }
}

// M (upper triangle), g and, if CDQ, the product C.dq
template <typename T, int N, bool CDQ, class K_>
ABRB_HD void dynamics_Mg(const ChainK<T, N> &P, const K_ &K, const T *dq, T (*M)[N], T *g, T *cdq) {
  constexpr bool ORTHO = K_::kOrtho;
  ABRB_UNROLL
  for (int a = 0; a < N; ++a) {
    g[a] = T(0);
    if (CDQ) cdq[a] = T(0);
    ABRB_UNROLL
    for (int b = 0; b < N; ++b) M[a][b] = T(0);
  }
  Spin<T, ORTHO> Wl;  // sum_{i<l} dq_i Omega_i, carried from link to link
  Wl.clear();
  ABRB_UNROLL
  for (int l = 1; l <= N; ++l) {
    T v[N][3];
    K.sync();
    link_columns<T, N>(K, l, v);
    ABRB_UNROLL
    for (int b = 0; b < N; ++b) {
      if (b < l) {
        const T wb[3] = {P.Wp[l][0] * v[b][0], P.Wp[l][1] * v[b][1], P.Wp[l][2] * v[b][2]};
        g[b] += dot3(v[b], P.gp[l]);
        ABRB_UNROLL
        for (int a = 0; a < N; ++a)
          if (a <= b) M[a][b] += dot3(v[a], wb);
      }
    }
    if (CDQ) {
      Wl.add(K, l - 1, dq[l - 1]);
      Spin<T, ORTHO> tail;
      tail.clear();
      T suf[3] = {T(0), T(0), T(0)}, acc[3] = {T(0), T(0), T(0)};
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
          for (int c = 0; c < 3; ++c) acc[c] += dq[j] * (a1[c] + a2[c]);
        }
      }
      ABRB_UNROLL
      for (int c = 0; c < 3; ++c) acc[c] *= P.Wp[l][c];
      ABRB_UNROLL
      for (int k = 0; k < N; ++k)
        if (k < l) cdq[k] += dot3(v[k], acc);
    }
  }
  dynamics_Mg_rotational<T, N, CDQ>(P, K, dq, M, g, cdq);
}

// The full Coriolis matrix C (only the rbd kernel materialises it)
template <typename T, int N, class K_>
ABRB_HD void dynamics_C(const ChainK<T, N> &P, const K_ &K, const T *dq, T (*C)[N]) {
  constexpr bool ORTHO = K_::kOrtho;
  ABRB_UNROLL
  for (int a = 0; a < N; ++a)
    ABRB_UNROLL
  for (int b = 0; b < N; ++b) C[a][b] = T(0);
  Spin<T, ORTHO> Wl;
  Wl.clear();
  ABRB_UNROLL
  for (int l = 1; l <= N; ++l) {
    T v[N][3];
    K.sync();
    link_columns<T, N>(K, l, v);
    Wl.add(K, l - 1, dq[l - 1]);
    Spin<T, ORTHO> tail;
    tail.clear();
    T suf[3] = {T(0), T(0), T(0)};
    ABRB_UNROLL
    for (int j = N - 1; j >= 0; --j) {
      if (j < l) {
        tail.add(K, j, dq[j]);
        ABRB_UNROLL
        for (int c = 0; c < 3; ++c) suf[c] += dq[j] * v[j][c];
        T a1[3], a2[3], wa[3];
        spin_diff_apply(Wl, tail, v[j], a1);
        omega_apply(K, j, suf, a2);
        ABRB_UNROLL
        for (int c = 0; c < 3; ++c) wa[c] = P.Wp[l][c] * (a1[c] + a2[c]);
        ABRB_UNROLL
        for (int k = 0; k < N; ++k)
          if (k < l) C[k][j] += dot3(v[k], wa);
      }
    }
  }
  dynamics_C_rotational<T, N>(P, K, dq, C);
}

// ------------------------------------------------------------------------------------------------
// Unit quaternion (w,x,y,z), w >= 0, of a (nearly) rotation matrix R[9] row-major.
// Reference: utils/transformations.py:1192-1271 (isprecise=False): eigenvector of the largest eigenvalue
// of the symmetric 4x4 matrix K/3.  For a rotation, K/3 + I/3 = (4/3) q q^T, so the dominant eigenvector is
// reached by power iteration on K/3 + I/3 from its column with the largest diagonal; the other
// eigenvalues are O(|R^T R - I|), i.e. each iteration gains >= 3 digits for the arms' measured frames.
template <typename T>
ABRB_HD void quat_from_R(const T *m, T *qo) {
  const T third = T(1) / T(3);
  T Kp[4][4];
  Kp[0][0] = (m[0] - m[4] - m[8]) * third + third;
  Kp[1][1] = (m[4] - m[0] - m[8]) * third + third;
  Kp[2][2] = (m[8] - m[0] - m[4]) * third + third;
  Kp[3][3] = (m[0] + m[4] + m[8]) * third + third;
  Kp[0][1] = Kp[1][0] = (m[1] + m[3]) * third;
  Kp[0][2] = Kp[2][0] = (m[2] + m[6]) * third;
  Kp[1][2] = Kp[2][1] = (m[5] + m[7]) * third;
  Kp[0][3] = Kp[3][0] = (m[7] - m[5]) * third;
  Kp[1][3] = Kp[3][1] = (m[2] - m[6]) * third;
  Kp[2][3] = Kp[3][2] = (m[3] - m[1]) * third;
  // start from the column with the largest diagonal entry (branch-free select)
  T v[4] = {Kp[0][0], Kp[1][0], Kp[2][0], Kp[3][0]};
  T best = Kp[0][0];
  ABRB_UNROLL
  for (int j = 1; j < 4; ++j) {
    const bool take = Kp[j][j] > best;
    best = take ? Kp[j][j] : best;
    ABRB_UNROLL
    for (int r = 0; r < 4; ++r) v[r] = take ? Kp[r][j] : v[r];
  }
  ABRB_UNROLL
  for (int it = 0; it < 5; ++it) {
    T w[4];
    ABRB_UNROLL
    for (int r = 0; r < 4; ++r) w[r] = Kp[r][0] * v[0] + Kp[r][1] * v[1] + Kp[r][2] * v[2] + Kp[r][3] * v[3];
    const T inv = inv_sqrt_t(w[0] * w[0] + w[1] * w[1] + w[2] * w[2] + w[3] * w[3]);
    ABRB_UNROLL
    for (int r = 0; r < 4; ++r) v[r] = w[r] * inv;
  }
  const T sgn = v[3] < T(0) ? T(-1) : T(1);  // reference: flip so that q[0] (w) >= 0
  qo[0] = sgn * v[3];
  qo[1] = sgn * v[0];
  qo[2] = sgn * v[1];
  qo[3] = sgn * v[2];
}

// quaternion_from_euler(a, b, g, axes="rxyz")  (utils/transformations.py:1096-1147, _AXES2TUPLE['rxyz']=(2,1,0,1))
template <typename T>
ABRB_HD void quat_from_euler_rxyz(T al, T be, T ga, T *qo) {
  T si, ci, sj, cj, sk, ck;
  sincos_t(ga * T(0.5), &si, &ci);   // frame=1 swaps first/last angle
  sincos_t(-be * T(0.5), &sj, &cj);  // parity=1 negates the middle angle
  sincos_t(al * T(0.5), &sk, &ck);
  const T cc = ci * ck, cs = ci * sk, sc = si * ck, ss = si * sk;
  qo[0] = cj * cc + sj * ss;
  qo[3] = cj * sc - sj * cs;     // i = 3
  qo[2] = -(cj * ss + sj * cc);  // j = 2, parity flips its sign
  qo[1] = cj * cs - sj * sc;     // k = 1
}

// quaternion_from_euler(ai, aj, ak, axes="sxyz")  (utils/transformations.py:1096-1147 with the axes tuple (0,0,0,0):
// i, j, k = 1, 2, 3, no parity flip, no frame swap)
template <typename T>
ABRB_HD void quat_from_euler_sxyz(T ai, T aj, T ak, T *qo) {
  T si, ci, sj, cj, sk, ck;
  sincos_t(ai * T(0.5), &si, &ci);
  sincos_t(aj * T(0.5), &sj, &cj);
  sincos_t(ak * T(0.5), &sk, &ck);
  const T cc = ci * ck, cs = ci * sk, sc = si * ck, ss = si * sk;
  qo[0] = cj * cc + sj * ss;
  qo[1] = cj * sc - sj * cs;
  qo[2] = cj * ss + sj * cc;
  qo[3] = cj * cs - sj * sc;
}

// Relative cut on the squared singular values of the row-Jacobi pseudo-inverses (pinv_rows_apply, RowPinv3): those at
// or below pinv_cut2<T>() * the largest are dropped.  fp64: 1e-30, numpy.linalg.pinv's rcond = 1e-15.  fp32: 1e-12,
// i.e. sigma <= 1e-6 sigma_max (~8 eps32): a null row of J in fp32 keeps a Jacobi residual of a few eps32 sigma_max
// (squared ~1e-14), which 1e-30 would keep and then amplify by 1 / residual^2 (DESIGN.md, "fp32 pseudo-inverse cut").
template <typename T>
ABRB_HD constexpr T pinv_cut2() {
  return sizeof(T) == 8 ? T(1e-30) : T(1e-12);
}

// out = pinv(A) y for an R x N matrix A (row-major, R <= N expected), numpy.linalg.pinv's rcond = 1e-15 in fp64
// (pinv_cut2): one-sided Jacobi on the rows as in RowPinv3 (abrb_osc.cuh) but for any R, with every loop rolled over
// local-memory arrays — the 15 row pairs of R = 6 unrolled would be ~3 k instructions, and this is a latency-bound
// sequential caller anyway.
template <typename T, int R, int N>
ABRB_HD_NOINLINE void pinv_rows_apply(const T *A, const T *y, T *out) {
  T Bm[R][N], V[R][R];
  ABRB_NOUNROLL
  for (int i = 0; i < R; ++i) {
    ABRB_NOUNROLL
    for (int k = 0; k < N; ++k) Bm[i][k] = A[i * N + k];
    ABRB_NOUNROLL
    for (int k = 0; k < R; ++k) V[i][k] = i == k ? T(1) : T(0);
  }
  const T tol = sizeof(T) == 8 ? T(1e-32) : T(1e-14);
  ABRB_NOUNROLL
  for (int sweep = 0; sweep < 12; ++sweep) {
    bool rotated = false;
    ABRB_NOUNROLL
    for (int i = 0; i < R - 1; ++i) {
      ABRB_NOUNROLL
      for (int j = i + 1; j < R; ++j) {
        T al = T(0), be = T(0), ga = T(0);
        ABRB_NOUNROLL
        for (int k = 0; k < N; ++k) {
          al += Bm[i][k] * Bm[i][k];
          be += Bm[j][k] * Bm[j][k];
          ga += Bm[i][k] * Bm[j][k];
        }
        if (!(ga * ga > tol * al * be) || ga == T(0)) continue;
        rotated = true;
        const T zeta = (be - al) / (T(2) * ga);
        const T t = (zeta >= T(0) ? T(1) : T(-1)) / (abs_t(zeta) + sqrt_t(T(1) + zeta * zeta));
        const T c = T(1) / sqrt_t(T(1) + t * t), sn = c * t;
        ABRB_NOUNROLL
        for (int k = 0; k < N; ++k) {
          const T x = Bm[i][k], w = Bm[j][k];
          Bm[i][k] = c * x - sn * w;
          Bm[j][k] = sn * x + c * w;
        }
        ABRB_NOUNROLL
        for (int k = 0; k < R; ++k) {
          const T x = V[i][k], w = V[j][k];
          V[i][k] = c * x - sn * w;
          V[j][k] = sn * x + c * w;
        }
      }
    }
    if (!rotated) break;
  }
  T s2[R], smax = T(0);
  ABRB_NOUNROLL
  for (int i = 0; i < R; ++i) {
    T acc = T(0);
    ABRB_NOUNROLL
    for (int k = 0; k < N; ++k) acc += Bm[i][k] * Bm[i][k];
    s2[i] = acc;
    smax = acc > smax ? acc : smax;
  }
  ABRB_NOUNROLL
  for (int k = 0; k < N; ++k) out[k] = T(0);
  ABRB_NOUNROLL
  for (int i = 0; i < R; ++i) {
    if (!(s2[i] > pinv_cut2<T>() * smax)) continue;
    T c = T(0);
    ABRB_NOUNROLL
    for (int k = 0; k < R; ++k) c += V[i][k] * y[k];
    c /= s2[i];
    ABRB_NOUNROLL
    for (int k = 0; k < N; ++k) out[k] += Bm[i][k] * c;
  }
}

// euler_matrix(a, b, g, axes="rxyz")[:3,:3]  (utils/transformations.py:973-1035), row-major R[9]
template <typename T>
ABRB_HD void R_from_euler_rxyz(T al, T be, T ga, T *R) {
  T si, ci, sj, cj, sk, ck;
  sincos_t(-ga, &si, &ci);
  sincos_t(-be, &sj, &cj);
  sincos_t(-al, &sk, &ck);
  const T cc = ci * ck, cs = ci * sk, sc = si * ck, ss = si * sk;
  // (i, j, k) = (2, 1, 0)
  R[2 * 3 + 2] = cj * ck;
  R[2 * 3 + 1] = sj * sc - cs;
  R[2 * 3 + 0] = sj * cc + ss;
  R[1 * 3 + 2] = cj * sk;
  R[1 * 3 + 1] = sj * ss + cc;
  R[1 * 3 + 0] = sj * cs - sc;
  R[0 * 3 + 2] = -sj;
  R[0 * 3 + 1] = cj * si;
  R[0 * 3 + 0] = cj * ci;
}

template <typename T>
ABRB_HD void quat_mul(const T *q1, const T *q0, T *o) {  // utils/transformations.py:1274-1290
  o[0] = -q1[1] * q0[1] - q1[2] * q0[2] - q1[3] * q0[3] + q1[0] * q0[0];
  o[1] = q1[1] * q0[0] + q1[2] * q0[3] - q1[3] * q0[2] + q1[0] * q0[1];
  o[2] = -q1[1] * q0[3] + q1[2] * q0[0] + q1[3] * q0[1] + q1[0] * q0[2];
  o[3] = q1[1] * q0[2] - q1[2] * q0[1] + q1[3] * q0[0] + q1[0] * q0[3];
}

// ------------------------------------------------------------------------------------------------
// Small dense linear algebra on register-resident matrices (static indices only).
// In-place lower Cholesky of the symmetric S (reads the upper OR lower triangle consistently: we use
// S[i][j], j<=i).  Returns false if a pivot is not positive.
template <typename T, int S_>
ABRB_HD bool chol(T (*A)[S_], T *invd) {  // invd[j] = 1 / L[j][j] (the solves multiply instead of dividing)
  bool ok = true;
  ABRB_UNROLL
  for (int j = 0; j < S_; ++j) {
    T d = A[j][j];
    ABRB_UNROLL
    for (int k = 0; k < S_; ++k)
      if (k < j) d -= A[j][k] * A[j][k];
    ok = ok && (d > T(0));
    const T dpos = d > T(0) ? d : T(1);
    const T inv = inv_sqrt_t(dpos);
    const T ljj = dpos * inv;
    A[j][j] = ljj;
    invd[j] = inv;
    ABRB_UNROLL
    for (int i = 0; i < S_; ++i) {
      if (i > j) {
        T s = A[i][j];
        ABRB_UNROLL
        for (int k = 0; k < S_; ++k)
          if (k < j) s -= A[i][k] * A[j][k];
        A[i][j] = s * inv;
      }
    }
  }
  return ok;
}
template <typename T, int S_>
ABRB_HD void fwd_solve(const T (*L)[S_], const T *invd, T *b) {  // L y = b
  ABRB_UNROLL
  for (int i = 0; i < S_; ++i) {
    T s = b[i];
    ABRB_UNROLL
    for (int k = 0; k < S_; ++k)
      if (k < i) s -= L[i][k] * b[k];
    b[i] = s * invd[i];
  }
}
template <typename T, int S_>
ABRB_HD void bwd_solve(const T (*L)[S_], const T *invd, T *b) {  // L^T x = b
  ABRB_UNROLL
  for (int i = S_ - 1; i >= 0; --i) {
    T s = b[i];
    ABRB_UNROLL
    for (int k = 0; k < S_; ++k)
      if (k > i) s -= L[k][i] * b[k];
    b[i] = s * invd[i];
  }
}

// x = pinv(S, rcond) y for a symmetric positive semi-definite S (numpy.linalg.pinv semantics: singular
// values <= rcond * largest are dropped; for symmetric PSD they are the eigenvalues).  Cyclic Jacobi.
// `active` marks the rows that belong to the problem (others are identity rows and are ignored when
// looking for the largest eigenvalue).  Deliberately NOT inlined: this is the rare, divergent path and
// works on a private copy so the hot path keeps its registers.
template <typename T, int S_>
ABRB_HD_NOINLINE void pinv_apply_sym(const T *Sin, unsigned active, T rcond, const T *y, T *x) {
  // NOTE: every loop here is kept rolled (ABRB_NOUNROLL): the fully unrolled, register-resident form of these
  // rotations has been seen not to converge on the device with nvcc 12.9 -O3 (tools/dbg/pinv_test.cu checks it: sum of
  // squares not preserved) while the rolled form matches the host bit for bit.  This is the rare
  // path, so local-memory arrays are fine.
  T A[S_][S_], V[S_][S_];
  ABRB_NOUNROLL
  for (int i = 0; i < S_; ++i) {
    ABRB_NOUNROLL
    for (int j = 0; j < S_; ++j) {
      A[i][j] = Sin[i * S_ + j];
      V[i][j] = i == j ? T(1) : T(0);
    }
  }
  const T eps = sizeof(T) == 8 ? T(1e-30) : T(1e-14);
  ABRB_NOUNROLL
  for (int sweep = 0; sweep < 30; ++sweep) {
    T off = T(0), diag = T(0);
    ABRB_NOUNROLL
    for (int i = 0; i < S_; ++i) {
      if ((active >> i) & 1u) diag += A[i][i] * A[i][i];  // identity rows must not set the scale
      ABRB_NOUNROLL
      for (int j = i + 1; j < S_; ++j) off += A[i][j] * A[i][j];
    }
    if (off <= eps * diag) break;
    ABRB_NOUNROLL
    for (int p = 0; p < S_ - 1; ++p) {
      ABRB_NOUNROLL
      for (int q = p + 1; q < S_; ++q) {
        const T apq = A[p][q];
        if (apq == T(0)) continue;
        const T theta = (A[q][q] - A[p][p]) / (T(2) * apq);
        const T t = (theta >= T(0) ? T(1) : T(-1)) / (abs_t(theta) + sqrt_t(theta * theta + T(1)));
        const T c = T(1) / sqrt_t(t * t + T(1)), s = t * c;
        ABRB_NOUNROLL
        for (int k = 0; k < S_; ++k) {
          const T akp = A[k][p], akq = A[k][q];
          A[k][p] = c * akp - s * akq;
          A[k][q] = s * akp + c * akq;
        }
        ABRB_NOUNROLL
        for (int k = 0; k < S_; ++k) {
          const T apk = A[p][k], aqk = A[q][k];
          A[p][k] = c * apk - s * aqk;
          A[q][k] = s * apk + c * aqk;
        }
        ABRB_NOUNROLL
        for (int k = 0; k < S_; ++k) {
          const T vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq;
          V[k][q] = s * vkp + c * vkq;
        }
      }
    }
  }
  T lmax = T(0);
  ABRB_NOUNROLL
  for (int i = 0; i < S_; ++i)
    if ((active >> i) & 1u) lmax = abs_t(A[i][i]) > lmax ? abs_t(A[i][i]) : lmax;
  ABRB_NOUNROLL
  for (int i = 0; i < S_; ++i) x[i] = T(0);
  ABRB_NOUNROLL
  for (int e = 0; e < S_; ++e) {
    // identity rows (inactive) have eigenvalue exactly 1 and never couple to y (y is zero on them)
    const T lam = A[e][e];
    if (!(abs_t(lam) > rcond * lmax)) continue;
    T proj = T(0);
    ABRB_NOUNROLL
    for (int k = 0; k < S_; ++k) proj += V[k][e] * y[k];
    proj /= lam;
    ABRB_NOUNROLL
    for (int k = 0; k < S_; ++k) x[k] += V[k][e] * proj;
  }
}

// ------------------------------------------------------------------------------------------------
// x = pinv(A A^T, rcond) y for a KD x N matrix A (the rows of L^-1 J^T, so that A A^T = J M^-1 J^T), the route taken
// by OSC._Mx when |det| is below its threshold (/root/reference/abr_control/controllers/osc.py:138-145).
// numpy.linalg.pinv drops the singular values <= rcond * largest; for the symmetric positive semi-definite A A^T
// they are its eigenvalues, i.e. the SQUARED singular values of A.  A one-sided (Hestenes) Jacobi SVD of the rows
// of A finds them without ever forming A A^T (whose eigenvalue ratios reach 1e-16 here): pairs of rows are rotated
// until all rows are mutually orthogonal, B = G A, B B^T = diag(s2), and then
//   pinv(A A^T) y = sum_{i: s2_i > rcond * max s2} G_i^T (G y)_i / s2_i .
// The pairs of one round (round-robin tournament schedule) are disjoint, so a round is ONE parallel step: on the GPU
// each row lives in its own lane of a six- (eight-) lane group of the warp and the partners exchange rows with shuffles
// (abrb_coop.cuh); the host instantiation (tests/hostsim) walks the same schedule sequentially.  Both use the
// per-row step below, so the arithmetic is the same.
template <int N, int KD>
struct JacobiRow {
  double b[N];  // the (rotated) row of A
  double t[2];  // its entries of the rotated right-hand sides G y and G z (G: the accumulated rotations)
};
// (The accumulated rotations themselves are never needed: with B = G A, B B^T = diag(s2), the product the controller
// wants is  A^T pinv(A A^T) y = B^T diag(keep / s2) G y = sum_i b_i (G y)_i / s2_i  — J^T Mx y is L times that.)

// Partner of player i in round r of a round-robin tournament of n (even) players, r = 0 .. n-2: player n-1 stays,
// the others move around a circle (i + j = 2 r mod n-1).
ABRB_HD int rr_partner(int n, int i, int r) {
  if (i == n - 1) return r;
  int j = 2 * r - i;
  j = j < 0 ? j + (n - 1) : j;
  j = j >= n - 1 ? j - (n - 1) : j;
  return j == i ? n - 1 : j;
}

// One row's share of the rotation of a pair of rows.  `lo`: this row has the smaller index of the two.  Returns
// 0 (already orthogonal to rounding: untouched), 1 (rotated, the cosine of the angle was below 1e-6: the quadratically
// convergent iteration is finished by this very rotation) or 2 (rotated, not yet converged).
template <int N, int KD>
ABRB_HD int jacobi_pair(bool lo, JacobiRow<N, KD> &me, const JacobiRow<N, KD> &other) {
  // (pairwise sums: the three inner products are the head of the round's dependent chain — depth 4 instead of 6 for
  // six columns — and these rounds are pure latency)
  double pm[(N + 1) / 2], pt[(N + 1) / 2], pg[(N + 1) / 2];
  ABRB_UNROLL
  for (int k = 0; k + 1 < N; k += 2) {
    pm[k / 2] = ::fma(me.b[k + 1], me.b[k + 1], me.b[k] * me.b[k]);
    pt[k / 2] = ::fma(other.b[k + 1], other.b[k + 1], other.b[k] * other.b[k]);
    pg[k / 2] = ::fma(me.b[k + 1], other.b[k + 1], me.b[k] * other.b[k]);
  }
  if (N & 1) {
    pm[N / 2] = me.b[N - 1] * me.b[N - 1];
    pt[N / 2] = other.b[N - 1] * other.b[N - 1];
    pg[N / 2] = me.b[N - 1] * other.b[N - 1];
  }
  ABRB_UNROLL
  for (int w = 1; w < (N + 1) / 2; w *= 2) {
    ABRB_UNROLL
    for (int k = 0; k + w < (N + 1) / 2; k += 2 * w) {
      pm[k] += pm[k + w];
      pt[k] += pt[k + w];
      pg[k] += pg[k + w];
    }
  }
  const double mine = pm[0], theirs = pt[0], ga = pg[0];
  const double prod = mine * theirs, g2 = ga * ga;
  if (!(g2 > 1e-30 * prod)) return 0;
  // rows (lo, hi) with squared norms (al, be):  lo' = c lo - s hi,  hi' = s lo + c hi  with the rotation angle
  //   tan 2 theta = 2 ga / d,  d = be - al  (|theta| <= pi/4).  With h = sqrt(d^2 + 4 ga^2):
  //   cos 2 theta = |d| / h,   c^2 = (1 + |d| / h) / 2  (in [1/2, 1]),   s = sgn(d) ga / (h c)
  // — two reciprocal square roots, no division, and no cancellation anywhere.
  const double d = lo ? theirs - mine : mine - theirs;
  const double r1 = inv_sqrt1_t(d * d + 4.0 * g2);  // 1 / h
  const double c2 = 0.5 + 0.5 * abs_t(d) * r1;
  const double r2 = inv_sqrt1_t(c2);                // 1 / c
  const double c = c2 * r2;
  const double sn = (d >= 0.0 ? ga : -ga) * r1 * r2;
  const double sp = lo ? -sn : sn;
  ABRB_UNROLL
  for (int k = 0; k < N; ++k) me.b[k] = c * me.b[k] + sp * other.b[k];
  me.t[0] = c * me.t[0] + sp * other.t[0];
  me.t[1] = c * me.t[1] + sp * other.t[1];
  return g2 > 1e-12 * prod ? 2 : 1;
}

constexpr int kJacobiMaxSweeps = 24;

// Sequential walk over the same schedule (host instantiation).  A: KD x N row-major.  Returns
// wy = A^T pinv(A A^T, rcond) y and wz likewise (N values each).
template <int N, int KD>
ABRB_HD void pinv_rows_jacobi_seq(const double *A, double rcond, const double *y, const double *z, bool two, double *wy,
                                  double *wz) {
  constexpr int NRR = KD + (KD & 1);
  JacobiRow<N, KD> row[NRR], old[NRR];
  for (int i = 0; i < NRR; ++i) {
    for (int k = 0; k < N; ++k) row[i].b[k] = i < KD ? A[i * N + k] : 0.0;
    row[i].t[0] = i < KD ? y[i] : 0.0;
    row[i].t[1] = (i < KD && two) ? z[i] : 0.0;
  }
  for (int sweep = 0; sweep < kJacobiMaxSweeps; ++sweep) {
    bool big = false;
    for (int r = 0; r < NRR - 1; ++r) {
      for (int i = 0; i < NRR; ++i) old[i] = row[i];
      for (int i = 0; i < NRR; ++i) {
        const int p = rr_partner(NRR, i, r);
        big = (jacobi_pair<N, KD>(i < p, row[i], old[p]) == 2) || big;
      }
    }
    if (!big) break;
  }
  double s2[KD], smax = 0.0;
  for (int i = 0; i < KD; ++i) {
    double acc = 0.0;
    for (int k = 0; k < N; ++k) acc += row[i].b[k] * row[i].b[k];
    s2[i] = acc;
    smax = acc > smax ? acc : smax;
  }
  for (int k = 0; k < N; ++k) wy[k] = wz[k] = 0.0;
  for (int i = 0; i < KD; ++i) {
    if (!(s2[i] > rcond * smax)) continue;
    const double cy = row[i].t[0] / s2[i], cz = row[i].t[1] / s2[i];
    for (int k = 0; k < N; ++k) {
      wy[k] += row[i].b[k] * cy;
      wz[k] += row[i].b[k] * cz;
    }
  }
}

}  // namespace abrb
